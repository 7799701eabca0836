"""GPU tier: the kernels across the float32 range of input scales.

Each op runs on ``2^k x`` for k on one ladder (``LADDER``; 15 is int16 PCM passed without the 1/32768), trimmed per op
to the rungs where the float64 reference's output, and the kernel's intermediates, are normal floats.  Every rung is
held to two checks:

(a) the float64 reference on the scaled input, the error normalised by the reference's own scale at that rung, with
    the bound the op's unit-scale test uses;
(b) homogeneity: an op of degree d must give ``op(2^k x) == 2^(d k) op(x)`` bit for bit, since a power-of-two scale
    is exact and every rounding repeats while the intermediates stay normal.

and the all-zero input is held to the reference.  Magnitudes are where the scale used to matter: a squared norm
underflows below |X| ~ 2^-63 (sqrt.approx.ftz then returns 0 and the gradients 0) and overflows above 2^64, and
__fdividef returns 0 for divisors above 2^126, which made the fused phase of (1.5e38, 1.5e38) 0.  kb_cabs and the
scaled division in kb_atan2 keep those rungs exact; the Magnitude, gradient and fused-phase tests hold them.

MUFU: every magnitude here goes through sqrt.approx (MUFU.SQRT on sm_90a); measured on an NVIDIA H100 80GB HBM3 at a
700 W power limit it is exponent-separable for even exponent shifts (the squared norm's shift is always even):
Magnitude gave 2^k |X| bit for bit at every rung from 2^-120 to 2^120, so the magnitude modes are asserted bit-exact
like the rest.  The decibel modes go through MUFU.LG2, whose result for
2^(2k) v is log2 v + 2k rounded once, so they are held to the oracle and to the dB shift within float32 rounding of
the shifted value."""
import math

import numpy as np
import pytest

torch = pytest.importorskip('torch')

import oracle as O  # noqa: E402

pytestmark = pytest.mark.gpu

LADDER = (-120, -90, -60, -40, -20, 0, 15, 20, 40, 60, 90, 120)
FLT_MAX = float(np.finfo(np.float32).max)
FLT_MIN = float(np.finfo(np.float32).tiny)
DB_PER_OCTAVE = 10.0 * math.log10(2.0)   # kapre's decibels are 10 log10 of the input


@pytest.fixture(scope='module')
def K():
    assert torch.cuda.is_available(), 'GPU tier needs a CUDA device'
    import kapre_b200
    from kapre_b200 import _native
    _native.lib()
    return kapre_b200


def rungs(lo, hi):
    return [k for k in LADDER if lo <= k <= hi]


def usable(ref, headroom=8):
    """True where the reference's scale is a normal float32 with 24 bits below it and ``headroom`` octaves above."""
    s = float(np.abs(ref).max())
    return FLT_MIN * 2.0 ** 24 <= s <= FLT_MAX * 2.0 ** -headroom


def scaled(x, k):
    """2^k x, computed exactly in float32 (subnormal or zero where 2^k x is)."""
    x = np.asarray(x)
    if np.iscomplexobj(x):
        out = np.empty_like(x)
        out.real, out.imag = np.ldexp(x.real, k), np.ldexp(x.imag, k)
        return out
    return np.ldexp(x, k).astype(x.dtype)


def nerr(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return float(np.abs(a - b).max() / max(float(np.abs(b).max()), 1e-300))


def bits(t):
    t = t.contiguous()
    if t.is_complex():
        t = torch.view_as_real(t)
    return t.view(torch.int32)


def exact(a, b):
    """a and b have the same bits (NaN payloads and signed zeros included)."""
    return a.shape == b.shape and bool(torch.equal(bits(a), bits(b)))


def p2(t, k):
    """2^k t for a float or complex tensor t, exact (signed zeros included) while the result is normal."""
    if t.is_complex():
        return torch.view_as_complex(torch.view_as_real(t) * (2.0 ** k))
    return t * (2.0 ** k)


def ulps(a, b):
    a, b = bits(a).long(), bits(b).long()
    a = torch.where(a < 0, -(a & 0x7fffffff), a)
    b = torch.where(b < 0, -(b & 0x7fffffff), b)
    return int((a - b).abs().max())


def _wave(rng, shape):
    """uniform(-1, 1) samples, none below 2^-12 in magnitude, so every product of a sample with a window or twiddle
    factor stays normal down to the lowest rung a transform is held to."""
    x = rng.uniform(-1, 1, size=shape)
    return (np.sign(x) * np.maximum(np.abs(x), 2.0 ** -12)).astype(np.float32)


def _cplx(rng, shape):
    """complex64 values whose parts lie in [2^-4, 1] in magnitude: every rung in LADDER keeps them normal."""
    re = np.sign(rng.uniform(-1, 1, shape)) * rng.uniform(2.0 ** -4, 1, shape)
    im = np.sign(rng.uniform(-1, 1, shape)) * rng.uniform(2.0 ** -4, 1, shape)
    return (re + 1j * im).astype(np.complex64)


# --------------------------------------------------------------------------------------- fused STFT (all variants)
MODE_COMPLEX, MODE_MAG, MODE_MAG_DB, MODE_MAG_PHASE = 0, 1, 2, 5
DB = (1.0, 2e-38, 1e9)      # (ref, amin, dynamic range): a clamp that binds at no rung held to the dB shift
# (n_fft, channels, launch switch, launch tag): K1 single-channel, K1b all-channel, mixed radix, direct DFT
# (K1b takes interleaved channels_last input; its tests transpose to channels_first for the checks)
VARIANTS = [(512, 1, {}, r'^Q8 '), (512, 2, {}, r'^MC Q'), (512, 2, {'NOMC': 1}, r'^Q8 '), (400, 1, {}, r'^MR '),
            (98, 1, {}, r'^DFT')]


def _stft(n_fft, mode):
    """The fused forward on a channels_first waveform; a multi-channel one goes in as an interleaved channels_last view
    (the all-channel kernel's input) and comes out channels_first."""
    from kapre_b200 import ops
    hop = n_fft // 4
    plan = ops.StftPlan(n_fft, n_fft, hop, O.get_window('hann_window', n_fft).astype(np.float32))

    def fwd(x):
        db = DB if mode == MODE_MAG_DB else None
        if x.shape[1] == 1:
            return ops.stft_forward(x, plan, 'channels_first', 'channels_first', True, True, mode, None, db)
        y = ops.stft_forward(x.transpose(1, 2).contiguous(), plan, 'channels_last', 'channels_last', True, True, mode,
                             None, db)
        return y.permute(0, 3, 1, 2).contiguous()
    return fwd, hop


def _launch(monkeypatch, switches):
    for k in ('NOMC',):
        monkeypatch.delenv('KAPRE_B200_' + k, raising=False)
    for k, v in switches.items():
        monkeypatch.setenv('KAPRE_B200_' + k, str(v))


@pytest.mark.parametrize('n_fft,C,switches,tag', VARIANTS, ids=['k1', 'k1b', 'k1_nomc', 'mr', 'dft'])
def test_stft_complex_is_homogeneous_and_matches_the_oracle(K, monkeypatch, n_fft, C, switches, tag):
    import re
    from kapre_b200 import _native
    _launch(monkeypatch, switches)
    rng = np.random.default_rng(n_fft + C)
    fwd, hop = _stft(n_fft, MODE_COMPLEX)
    x = _wave(rng, (2, C, 9 * hop + 3))
    xt = torch.from_numpy(x).cuda()
    y0 = fwd(xt)
    assert re.search(tag, _native.last_launch_info()), _native.last_launch_info()
    for k in LADDER:
        xs = scaled(x, k)
        ref = O.stft_layer(xs, n_fft, n_fft, hop, 'hann_window', True, True, 'channels_first', 'channels_first')
        if not usable(ref):
            continue
        y = fwd(torch.from_numpy(xs).cuda())
        assert nerr(y.cpu().numpy(), ref) < 2e-6, k
        if -60 <= k <= 90:
            assert exact(y, p2(y0, k)), k
    assert not fwd(torch.zeros_like(xt)).abs().max()


@pytest.mark.parametrize('n_fft,C,switches,tag', VARIANTS, ids=['k1', 'k1b', 'k1_nomc', 'mr', 'dft'])
def test_stft_magnitude_modes_are_homogeneous_and_match_the_oracle(K, monkeypatch, n_fft, C, switches, tag):
    _launch(monkeypatch, switches)
    rng = np.random.default_rng(n_fft + C + 1)
    modes = {98: (MODE_MAG,), 400: (MODE_MAG, MODE_MAG_DB)}.get(n_fft, (MODE_MAG, MODE_MAG_DB, MODE_MAG_PHASE))
    hop = n_fft // 4
    x = _wave(rng, (2, C, 9 * hop + 3))
    for mode in modes:
        fwd, _ = _stft(n_fft, mode)
        y0 = fwd(torch.from_numpy(x).cuda())
        for k in LADDER:
            xs = scaled(x, k)
            spec = O.stft_layer(xs, n_fft, n_fft, hop, 'hann_window', True, True, 'channels_first', 'channels_first')
            mag = np.abs(spec)
            if not usable(mag):
                continue
            y = fwd(torch.from_numpy(xs).cuda())
            yn = y.double().cpu().numpy()
            if mode == MODE_MAG_DB:
                lin = 10.0 ** (yn / 10.0)
                # 2e-6 plus two float32 roundings at the dB value's magnitude (log2 |X| and the dB value), which
                # reach 7.4e-6 relative at 190 dB (k = 60) on the H100
                tol = 2e-6 + 2 * np.spacing(np.float32(np.abs(yn).max())) * math.log(10.0) / 10.0
                assert nerr(lin, np.maximum(mag, DB[1])) < tol, k
                # the dB shift: 10 k log10(2), within the float32 rounding of the shifted value
                d = yn - y0.double().cpu().numpy() - DB_PER_OCTAVE * k
                assert np.abs(d).max() <= 4 * np.spacing(np.float32(np.abs(yn).max())) + 1e-5, k
                continue
            m = yn[:, :C]
            assert nerr(m, mag) < 2e-6, k
            if -60 <= k <= 90:
                assert exact(y[:, :C], p2(y0[:, :C], k)), (mode, k, ulps(y[:, :C], p2(y0[:, :C], k)))
            if mode == MODE_MAG_PHASE:
                ph = yn[:, C:]
                ok = mag > 1e-3 * mag.max()
                assert np.abs(np.angle(np.exp(1j * (ph - np.angle(spec)))))[ok].max() < 1e-3, k
                if -60 <= k <= 90:
                    assert exact(y[:, C:], y0[:, C:]), k     # degree 0


# ----------------------------------------------------------------------------- Magnitude, Phase and their gradients
def test_magnitude_over_the_whole_float_range(K):
    """|X| for parts in [2^-4, 1] at every rung: tiny (k <= -90) gave 0 and huge (k >= 90) gave inf before kb_cabs."""
    rng = np.random.default_rng(3)
    X = _cplx(rng, (4, 3, 257))
    Xt = torch.from_numpy(X).cuda()
    y0 = K.Magnitude()(Xt)
    for k in LADDER:
        Xs = scaled(X, k)
        y = K.Magnitude()(torch.from_numpy(Xs).cuda())
        ref = np.abs(Xs.astype(np.complex128))
        assert nerr(y.cpu().numpy(), ref) < 2e-6, k       # test_gpu_grad's Magnitude bound at unit scale
        assert exact(y, p2(y0, k)), (k, ulps(y, p2(y0, k)))
    assert not K.Magnitude()(torch.zeros_like(Xt)).abs().max()
    # subnormal parts: still |X|, within the rounding of the subnormal inputs
    sub = torch.tensor([complex(3e-42, 4e-42), complex(0.0, 1e-44), complex(1e-40, 0.0)], dtype=torch.complex64)
    got = K.Magnitude()(sub.cuda()).cpu().double()
    want = sub.to(torch.complex128).abs()
    assert float((got - want).abs().max()) <= 2.0 ** -149


def test_phase_is_degree_zero(K):
    rng = np.random.default_rng(4)
    X = _cplx(rng, (4, 3, 257))
    y0 = K.Phase()(torch.from_numpy(X).cuda())
    for k in LADDER:
        Xs = scaled(X, k)
        y = K.Phase()(torch.from_numpy(Xs).cuda())
        assert np.abs(y.cpu().numpy() - np.angle(Xs.astype(np.complex128))).max() < 1e-6, k
        assert exact(y, y0), k


def test_fused_phase_at_the_top_and_bottom_of_the_range(K):
    """One frame holding an impulse a at n0 = 224 under a rectangular window: X[f] = a exp(2 pi i f / 8), so bin 1 is
    (a, a) / sqrt(2).  The fused mode-5 phase divides min / max with __fdividef, which returned 0 for a divisor above
    2^126 (huge, a = 1.5e38: phase 0 instead of pi / 4) before the scaled division."""
    from kapre_b200 import ops
    n_fft, hop = 256, 256
    plan = ops.StftPlan(n_fft, n_fft, hop, np.ones(n_fft, np.float32))
    n0 = 224
    for a in (1.5e38, 1e38, 1.0, 2.0 ** -120):
        x = torch.zeros((1, 1, n_fft), device='cuda')
        x[0, 0, n0] = a
        y = ops.stft_forward(x, plan, 'channels_first', 'channels_first', False, False, MODE_MAG_PHASE)
        ref = np.angle(np.exp(-2j * np.pi * np.arange(n_fft // 2 + 1) * n0 / n_fft))
        ph = y[0, 1, 0].double().cpu().numpy()
        assert np.abs(np.angle(np.exp(1j * (ph - ref)))).max() < 1e-6, a
        assert abs(ph[1] - math.pi / 4) < 1e-6, (a, ph[1])
        assert np.abs(y[0, 0, 0].double().cpu().numpy() - float(np.float32(a))).max() <= 2e-6 * float(np.float32(a))


def _grad_ref(X, g_mag=None, g_ph=None):
    X = X.astype(np.complex128)
    u = X / np.abs(X)
    out = np.zeros_like(X)
    if g_mag is not None:
        out += g_mag * u
    if g_ph is not None:
        out += 1j * u * g_ph / np.abs(X)
    return out


def test_magnitude_and_phase_gradients_over_the_whole_float_range(K):
    """d|X|/dX = g X / |X| is degree 0 in X and d angle(X)/dX degree -1; tiny X gave 0 and huge X gave 0 or NaN before
    kb_cabs (and the phase gradient's (g / |X|) / |X| overflowed for |X| below 2^-64)."""
    from kapre_b200 import ops
    rng = np.random.default_rng(5)
    X = _cplx(rng, (2, 3, 5, 33))
    gm = rng.standard_normal(X.shape).astype(np.float32)
    gp = rng.standard_normal(X.shape).astype(np.float32)
    Xt, gmt, gpt = (torch.from_numpy(v).cuda() for v in (X, gm, gp))
    m0 = ops.magnitude_backward(Xt, gmt)
    p0 = ops.phase_backward(Xt, gpt)
    for k in LADDER:
        Xs = scaled(X, k)
        Xst = torch.from_numpy(Xs).cuda()
        m = ops.magnitude_backward(Xst, gmt)
        p = ops.phase_backward(Xst, gpt)
        mp = ops.mag_phase_backward(Xst, gmt, gpt, 'channels_first')
        assert nerr(m.cpu().numpy(), _grad_ref(Xs, gm)) < 1e-5, k          # test_gpu_grad's bound
        assert exact(m, m0), k
        want_p = _grad_ref(Xs, None, gp)
        if usable(want_p, 0):
            assert nerr(p.cpu().numpy(), want_p) < 1e-5, k
            assert nerr(mp.cpu().numpy(), _grad_ref(Xs, gm, gp)) < 1e-5, k
            assert exact(p, p2(p0, -k)), k
    # a part that is exactly 0 (STFT DC and Nyquist bins) with a gradient 1 / |X| that overflows: the other part of
    # the phase gradient is 0, as in float64, not inf * 0
    Xz = torch.tensor([complex(2.0 ** -130, 0.0), complex(0.0, -(2.0 ** -128))], dtype=torch.complex64).cuda()
    gz = torch.full((2,), 2.0 ** 16, device='cuda')
    for got in (ops.phase_backward(Xz, gz), ops.mag_phase_backward(Xz.view(1, 1, 1, 2), None, gz.view(1, 1, 1, 2),
                                                                   'channels_first').view(2)):
        assert float(got[0].real) == 0 and float(got[1].imag) == 0, got
        assert torch.isinf(got[0].imag) and torch.isinf(got[1].real), got
    z = torch.zeros_like(Xt)
    for got in (ops.magnitude_backward(z, gmt), ops.phase_backward(z, gpt), ops.mag_phase_backward(z, gmt, gpt,
                                                                                                   'channels_first')):
        assert not got.abs().max()


# ------------------------------------------------------------------------------------- degree-1 linear transforms
def _stft_f64(x, n_fft, hop):
    """kapre's STFT (pad_begin, pad_end, periodic Hann) of a float64 (B, C, L) tensor, differentiable."""
    w = torch.from_numpy(O.get_window('hann_window', n_fft))
    L = x.shape[-1]
    T = -(-(L + n_fft - hop) // hop)
    xp = torch.nn.functional.pad(x, (n_fft - hop, T * hop + n_fft - hop - (L + n_fft - hop)))
    frames = xp.unfold(-1, n_fft, hop)[..., :T, :]
    return torch.fft.rfft(frames * w, dim=-1)



def test_inverse_stft_and_the_stft_adjoints_are_homogeneous(K):
    from kapre_b200 import ops
    rng = np.random.default_rng(6)
    n_fft, hop = 512, 128
    Xc = _cplx(rng, (2, 1, 12, n_fft // 2 + 1))
    Xt = torch.from_numpy(Xc).cuda()
    istft = K.InverseSTFT(n_fft=n_fft, hop_length=hop, forward_window_name='hann_window',
                          input_data_format='channels_first', output_data_format='channels_first')
    plan = ops.StftPlan(n_fft, n_fft, hop, O.get_window('hann_window', n_fft).astype(np.float32))
    y0 = istft(Xt)
    L = 11 * hop - 308                 # pad_begin + pad_end: ceil((L + n_fft - hop) / hop) = 12 frames
    s0 = ops.stft_backward(Xt, plan, 'channels_first', 'channels_first', True, True, L)
    for k in rungs(-60, 90):
        Xs = torch.from_numpy(scaled(Xc, k)).cuda()
        assert exact(istft(Xs), p2(y0, k)), k
        # stft_backward against the float64 adjoint of the oracle's STFT at this scale
        xd = torch.zeros((2, 1, L), dtype=torch.float64, requires_grad=True)
        spec = _stft_f64(xd, n_fft, hop)
        want, = torch.autograd.grad(spec, xd, Xs.cpu().to(torch.complex128))
        got = ops.stft_backward(Xs, plan, 'channels_first', 'channels_first', True, True, L)
        assert nerr(got.double().cpu().numpy(), want.numpy()) < 2e-6, k
        assert exact(ops.stft_backward(Xs, plan, 'channels_first', 'channels_first', True, True, L),
                     p2(s0, k)), k
    for k in LADDER:
        Xs = scaled(Xc, k)
        want = O.istft_layer(Xs, n_fft, n_fft, hop, 'hann_window', 'channels_first', 'channels_first')
        if usable(want):
            assert nerr(istft(torch.from_numpy(Xs).cuda()).cpu().numpy(), want) < 2e-6, k
    assert not istft(torch.zeros_like(Xt)).abs().max()


def test_frame_delta_and_filterbank_are_homogeneous(K):
    rng = np.random.default_rng(7)
    x = _wave(rng, (2, 1000, 2))
    spec = (rng.random((2, 2, 9, 257)) * 0.75 + 0.25).astype(np.float32)
    fbl = K.ApplyFilterbank('mel', dict(sample_rate=16000, n_freq=257, n_mels=40), data_format='channels_first')
    ops_ = [(K.Frame(64, 16, pad_end=True, data_format='channels_last'), x,
             lambda v: O.frame_layer(v, 64, 16, True, 0, 'channels_last'), 0.0),
            (K.Delta(win_length=5, mode='symmetric', data_format='channels_first'), spec,
             lambda v: O.delta(v, 5, 'symmetric', 'channels_first'), 2e-6),
            (fbl, spec, lambda v: np.einsum('bctf,fm->bctm', v, np.asarray(fbl.filterbank, np.float64)), 2e-6)]
    for layer, v, ref, tol in ops_:
        y0 = layer(torch.from_numpy(v).cuda())
        for k in LADDER:
            vs = scaled(v, k)
            y = layer(torch.from_numpy(vs).cuda())
            want = ref(vs.astype(np.float64))
            if usable(want, 0):
                assert nerr(y.double().cpu().numpy(), want) <= tol, (layer, k)
            if -60 <= k <= 90:
                assert exact(y, p2(y0, k)), (layer, k)
        assert not layer(torch.zeros_like(torch.from_numpy(v)).cuda()).abs().max()


def test_magnitude_to_decibel_shifts_by_10_k_log10_2(K):
    rng = np.random.default_rng(8)
    x = (rng.random((3, 1, 9, 40)) * 0.75 + 0.25).astype(np.float32)
    layer = K.MagnitudeToDecibel(ref_value=1.0, amin=2e-38, dynamic_range=1e9)     # the clamp is inactive
    y0 = layer(torch.from_numpy(x).cuda()).double().cpu().numpy()
    for k in rungs(-90, 120):
        xs = scaled(x, k)
        y = layer(torch.from_numpy(xs).cuda()).double().cpu().numpy()
        ref = O.magnitude_to_decibel(xs.astype(np.float64), 1.0, 2e-38, 1e9)
        assert np.abs(y - ref).max() < 2e-4 + 1e-6 * np.abs(ref).max(), k
        d = y - y0 - DB_PER_OCTAVE * k
        assert np.abs(d).max() <= 4 * np.spacing(np.float32(np.abs(y).max())) + 1e-5, k


# ------------------------------------------------- the correctly rounded magnitude form: CQT, chroma, time stretch
def _tone(seed, L=22050):
    """0.1 noise plus a 0.4 sinusoid (test_gpu_cqt's signal), (1, 1, L) float32."""
    rng = np.random.default_rng(seed)
    t = np.arange(L) / 22050
    x = 0.1 * rng.standard_normal((1, 1, L)) + 0.4 * np.sin(2 * np.pi * rng.uniform(40, 7000) * t + rng.uniform(0, 6))
    return x.astype(np.float32)


def test_cqt_magnitude_and_its_gradient_at_the_ends_of_the_range(K):
    """|C| and its gradient at 2^-90 (|C|^2 underflowed to 0) and 2^90 (it overflowed to inf) as at unit scale: within
    test_gpu_cqt's derived bounds, and the magnitude 2^k |C| bit for bit."""
    import cqt_ref as R
    from kapre_b200 import ops
    from kapre_b200.time_frequency import CQT
    q = CQT(input_data_format='channels_first', output_data_format='channels_first')
    x = _tone(21)
    rng = np.random.default_rng(22)
    y0 = ops.cqt(torch.from_numpy(x).cuda(), q.plan, 'channels_first', 'channels_first', True)
    g = torch.from_numpy(rng.standard_normal(tuple(y0.shape)).astype(np.float32)).cuda()
    for k in (-90, -60, 0, 60, 90):
        xs = scaled(x, k)
        xg = torch.from_numpy(xs).cuda().requires_grad_(True)
        y = ops.cqt(xg, q.plan, 'channels_first', 'channels_first', True)
        xd = torch.from_numpy(xs).double()
        err = np.abs(y.detach().double().cpu().numpy() - R.cqt(xd, q.plan, True).numpy())
        assert (err <= R.forward_bound(xd, q.plan, True).numpy()).all(), k
        assert exact(y.detach(), p2(y0, k)), k
        y.backward(g)
        gd = g.cpu().double()
        err = np.abs(xg.grad.double().cpu().numpy() - R.vjp(xd, q.plan, gd, True).numpy())
        assert (err <= R.backward_bound(xd, q.plan, gd, True).numpy()).all(), k


def test_chroma_is_degree_zero_through_the_cqt_and_complex_inputs(K):
    """chroma_cqt from the waveform (|C| in the CQT kernel) and from a complex C (|C| in the chroma kernel), and the
    gradient with respect to C (degree -1), at scales where |C|^2 left the float range."""
    from kapre_b200 import ops, signal
    x = _tone(23, 3 * 22050)
    cqt, _ = signal._cqt_chroma_plans(22050, 512, None, 0.0, 12, 7, 36, True, 41)
    Cc = ops.cqt(torch.from_numpy(x).cuda(), cqt, 'channels_first', 'channels_first', False)
    w0 = signal.chroma_cqt(torch.from_numpy(x).cuda(), data_format='channels_first')
    c0 = signal.chroma_cqt(C=Cc, data_format='channels_first')
    assert torch.equal(c0, w0)
    Cg = Cc.clone().requires_grad_(True)
    gy = torch.randn(tuple(c0.shape), device='cuda', generator=torch.Generator(device='cuda').manual_seed(24))
    d0, = torch.autograd.grad(signal.chroma_cqt(C=Cg, data_format='channels_first'), Cg, gy)
    for k in (-90, -60, -20, 20, 60, 90):
        assert exact(signal.chroma_cqt(torch.from_numpy(scaled(x, k)).cuda(), data_format='channels_first'), w0), k
        Cs = torch.view_as_complex(torch.view_as_real(Cc) * 2.0 ** k).requires_grad_(True)
        assert exact(signal.chroma_cqt(C=Cs, data_format='channels_first'), c0), k
        d, = torch.autograd.grad(signal.chroma_cqt(C=Cs, data_format='channels_first'), Cs, gy)
        # degree -1 within float32 rounding: at 2^-90 some products in the normalisation's backward go subnormal
        assert nerr(torch.view_as_real(d).cpu().numpy(), torch.view_as_real(p2(d0, -k)).cpu().numpy()) < 1e-5, k


def test_time_stretch_is_homogeneous(K):
    """The phase vocoder blends |X| (the correctly rounded kb_cabs) with a degree-0 phase: degree 1, bit for bit,
    including 2^-90 and 2^90 where |X|^2 left the float range.  (At 2^-120 small output parts are subnormal.)"""
    from kapre_b200.augmentation import TimeStretch
    layer = TimeStretch(0.8, data_format='channels_first')
    X = _cplx(np.random.default_rng(25), (2, 1, 40, 257))
    y0 = layer(torch.from_numpy(X).cuda())
    for k in rungs(-90, 120):
        Xs = scaled(X, k)
        y = layer(torch.from_numpy(Xs).cuda())
        assert exact(y, p2(y0, k)), k
