"""Gradients of Phase, get_stft_mag_phase, Delta, Frame, Energy, ConcatenateFrequencyMap and SpecAugment on the H100:
vector-Jacobian products against the float64 restatement (grad_ref_adjacent.py), adjoint identities at the BASELINE
cfg2 shape, a training chain through the log-mel front end, and the promise that every public layer records a
gradient while the no-grad path stays as it was.

Tolerances follow test_gpu_grad.py and are relative to the largest reference value (``_rel``) or the reference's
norm (``_rel_l2``):
* linear layers (Delta, Frame, ConcatenateFrequencyMap, SpecAugment) and Energy: 1e-4.  Each output is a float32
  sum of at most 2n taps (Delta) or ceil(frame_length / hop) frames, or a copy;
* anything through a decibel or a phase (Phase, get_stft_mag_phase, the training chain): 2e-3 in L2.  The phase's
  gradient g / |X| amplifies the float32 error of weak bins, d dB / dx = 10 / (ln 10 x) that of small magnitudes,
  and an element within rounding of the dynamic-range threshold may be clamped on one side only.  The test signals
  are white noise, whose bins stay well away from zero apart from the deliberate exact zeros.
"""
import numpy as np
import pytest
import torch

import grad_ref as R
import grad_ref_adjacent as RA

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    import kapre_b200 as K
    from kapre_b200 import _native as N

CL, CF = 'channels_last', 'channels_first'
FMTS = (CF, CL)


def _rel(got, want, tol):
    got = got.detach().cpu().to(want.dtype)
    want = want.detach().cpu()
    err = float((got - want).abs().max())
    scale = float(want.abs().max())
    assert err <= tol * scale, (err, scale)


def _rel_l2(got, want, tol):
    got = got.detach().cpu().to(want.dtype)
    want = want.detach().cpu()
    err = float(torch.linalg.vector_norm(got - want))
    assert err <= tol * float(torch.linalg.vector_norm(want)), (err, float(torch.linalg.vector_norm(want)))


def _grad(layer, x, g, **kw):
    """(output, d<layer(x), g>/dx) through kapre_b200 on the GPU; also checks that recording for autograd leaves the
    forward output bit-identical."""
    xd = x.cuda().requires_grad_(True)
    y = layer(xd, **kw)
    assert y.grad_fn is not None
    with torch.no_grad():
        y0 = layer(x.cuda(), **kw)
    assert torch.equal(y.detach(), y0)
    (gx,) = torch.autograd.grad(y, xd, grad_outputs=g.cuda().to(y.dtype))
    return y, gx


def _randn(rng, shape, dtype=np.float32):
    return torch.from_numpy(rng.standard_normal(shape).astype(dtype))


def _cplx(rng, shape):
    return torch.from_numpy((rng.standard_normal(shape) + 1j * rng.standard_normal(shape)).astype(np.complex64))


# ------------------------------------------------------------------------------ per-layer vector-Jacobian products
@pytest.mark.parametrize('fmt', FMTS)
def test_phase_vjp(fmt):
    rng = np.random.default_rng(1)
    X = _cplx(rng, (2, 9, 257, 2) if fmt == CL else (2, 2, 9, 257))
    X.view(-1)[[0, 11, 500]] = 0
    g = _randn(rng, tuple(X.shape))
    _, gX = _grad(K.Phase(), X, g)
    _rel_l2(gX, R.vjp(RA.phase, X.to(torch.complex128), g.double())[1], 2e-3)
    flat = gX.reshape(-1).cpu()
    assert flat[0] == 0 and flat[11] == 0 and flat[500] == 0


@pytest.mark.parametrize('mode', ['symmetric', 'reflect', 'constant'])
@pytest.mark.parametrize('win', [3, 5, 9])
@pytest.mark.parametrize('fmt', FMTS)
def test_delta_vjp(mode, win, fmt):
    rng = np.random.default_rng(win + len(mode))
    layer = K.Delta(win_length=win, mode=mode, data_format=fmt)
    for T in (1, 2, win // 2, win, 2 * win + 1, 50):
        shape = (2, T, 40, 2) if fmt == CL else (2, 2, T, 40)
        x, g = _randn(rng, shape), _randn(rng, shape)
        _, gx = _grad(layer, x, g)
        _rel(gx, R.vjp(lambda t: RA.delta(t, win, mode, fmt), x.double(), g.double())[1], 1e-4)


FRAME_CASES = [(512, 128, False), (512, 128, True), (300, 300, False), (300, 300, True), (100, 160, False),
               (100, 160, True)]


@pytest.mark.parametrize('case', FRAME_CASES, ids=lambda c: 'fl%d_h%d_pe%d' % c)
@pytest.mark.parametrize('fmt', FMTS)
def test_frame_and_energy_vjp(case, fmt):
    fl, hop, pe = case
    rng = np.random.default_rng(fl + hop)
    x = _randn(rng, (2, 4001, 2) if fmt == CL else (2, 2, 4001))
    if hop <= fl:
        layer = K.Frame(frame_length=fl, hop_length=hop, pad_end=pe, pad_value=0.5, data_format=fmt)
        y0 = layer(x.cuda())
        g = _randn(rng, tuple(y0.shape))
        _, gx = _grad(layer, x, g)
        _rel(gx, R.vjp(lambda t: RA.frame(t, fl, hop, pe, 0.5, fmt), x.double(), g.double())[1], 1e-4)
    layer = K.Energy(sample_rate=16000, ref_duration=0.1, frame_length=fl, hop_length=hop, pad_end=pe, pad_value=0.5,
                     data_format=fmt)
    y0 = layer(x.cuda())
    g = _randn(rng, tuple(y0.shape))
    _, gx = _grad(layer, x, g)
    scale = 0.1 / (fl / 16000)
    _rel(gx, R.vjp(lambda t: RA.energy(t, fl, hop, pe, 0.5, scale, fmt), x.double(), g.double())[1], 1e-4)


@pytest.mark.parametrize('fmt', FMTS)
def test_concat_frequency_map_vjp(fmt):
    rng = np.random.default_rng(4)
    x = _randn(rng, (3, 20, 64, 2) if fmt == CL else (3, 2, 20, 64))
    g = _randn(rng, (3, 20, 64, 3) if fmt == CL else (3, 3, 20, 64))
    _, gx = _grad(K.ConcatenateFrequencyMap(data_format=fmt), x, g)
    _rel(gx, R.vjp(lambda t: RA.concat_frequency_map(t, fmt), x.double(), g.double())[1], 0.0)


@pytest.mark.parametrize('fmt', FMTS)
def test_spec_augment_vjp_reuses_the_forward_masks(fmt):
    rng = np.random.default_rng(6)
    shape = (4, 60, 40, 1) if fmt == CL else (4, 1, 60, 40)
    x, g = _randn(rng, shape), _randn(rng, shape)
    layer = K.SpecAugment(freq_mask_param=10, time_mask_param=12, n_freq_masks=2, n_time_masks=2, mask_value=-3.0,
                          data_format=fmt, seed=11)
    xd = x.cuda().requires_grad_(True)
    y = layer(xd, training=True)
    tm, fm = layer.last_masks
    layer(x.cuda(), training=True)                     # draws other masks; the backward must not see them
    assert not (np.array_equal(tm, layer.last_masks[0]) and np.array_equal(fm, layer.last_masks[1]))
    (gx,) = torch.autograd.grad(y, xd, grad_outputs=g.cuda())
    _rel(y.detach(), RA.spec_augment(x.double(), tm, fm, -3.0, fmt), 0.0)
    _rel(gx, R.vjp(lambda t: RA.spec_augment(t, tm, fm, -3.0, fmt), x.double(), g.double())[1], 0.0)
    assert layer(xd, training=False) is xd             # inference: identity, the graph passes through


# ------------------------------------------------------------------------------ get_stft_mag_phase
@pytest.mark.parametrize('db,dyn', [(False, 80.0), (True, 80.0), (True, 15.0)], ids=['lin', 'db80', 'db15'])
@pytest.mark.parametrize('fmt', FMTS)
@pytest.mark.parametrize('n_fft,hop', [(512, 128), (1024, 256), (2048, 512), (400, 160), (1000, 250)])
def test_stft_mag_phase_vjp(n_fft, hop, fmt, db, dyn):
    rng = np.random.default_rng(n_fft + int(dyn) + db)
    model = K.get_stft_mag_phase(None, n_fft=n_fft, hop_length=hop, return_decibel=db, db_dynamic_range=dyn,
                                 input_data_format=fmt, output_data_format=fmt)
    fused = model.stft.plan.supports_mode(N.OUT_MAG_PHASE)
    assert fused == (n_fft in (512, 1024, 2048))      # 400 and 1000 take the unfused torch.cat route
    x = _randn(rng, (2, 9000, 1) if fmt == CL else (2, 1, 9000))
    y0 = model(x.cuda())
    g = _randn(rng, tuple(y0.shape))
    _, gx = _grad(model, x, g)
    dbt = (1.0, 1e-5, dyn) if db else None
    _, want = R.vjp(lambda t: RA.mag_phase(t, n_fft, n_fft, hop, None, False, False, fmt, fmt, dbt), x.double(),
                    g.double())
    _rel_l2(gx, want, 2e-3)


def test_stft_mag_phase_clamp_binds():
    """At 15 dB the dynamic-range clamp holds about 1% of the bins of white noise (some hundreds per item here), so the
    db15 cases above exercise the threshold's gradient."""
    rng = np.random.default_rng(0)
    x = _randn(rng, (2, 1, 9000))
    model = K.get_stft_mag_phase(None, n_fft=1024, hop_length=256, return_decibel=True, db_dynamic_range=15.0,
                                 input_data_format=CF, output_data_format=CF)
    y = model(x.cuda())
    mag = y[:, :1]
    thr = mag.amax(dim=(1, 2, 3), keepdim=True) - 15.0
    assert float((mag <= thr + 1e-4).float().mean()) > 0.002


# ------------------------------------------------------------------------------ adjoint identities at cfg2
def _dot(a, b):
    return float((a.double() * b.double()).sum())


def _norm(a):
    return float(a.detach().double().square().sum()) ** 0.5


def _linear_adjoint(layer, x, affine=False):
    """|<A x, y> - <x, A^T y>| relative to |A x| |y|, in float64; affine: A x = layer(x) - layer(0)."""
    xg = x.clone().requires_grad_(True)
    y = layer(xg)
    yr = torch.randn_like(y)
    (gx,) = torch.autograd.grad(y, xg, grad_outputs=yr)
    Ax = y.detach()
    if affine:
        Ax = Ax - layer(torch.zeros_like(x))
    lhs, rhs = _dot(Ax, yr), _dot(x, gx)
    return abs(lhs - rhs) / (_norm(Ax) * _norm(yr))


def test_adjoint_identities_cfg2():
    """Delta and ConcatenateFrequencyMap on the (256, 1, 427, 128) log-mel of BASELINE cfg2 (batch 256, 5 s at
    22.05 kHz, n_fft 1024, hop 256, 128 mel), Frame on its 256 x 110250 waveform."""
    torch.manual_seed(0)
    mel = torch.randn(256, 1, 427, 128, device='cuda')
    for mode in ('symmetric', 'reflect', 'constant'):
        assert _linear_adjoint(K.Delta(win_length=9, mode=mode, data_format=CF), mel) <= 1e-5
    assert _linear_adjoint(K.ConcatenateFrequencyMap(data_format=CF), mel, affine=True) <= 1e-6
    del mel
    wav = torch.randn(256, 1, 110250, device='cuda')
    assert _linear_adjoint(K.Frame(frame_length=1024, hop_length=256, pad_end=True, data_format=CF), wav) <= 1e-5
    torch.cuda.empty_cache()


def test_energy_gradient_cfg2():
    """d<E(x), y>/dx for Energy's defaults (2205-sample frames every 1102) on the cfg2 waveform, against the
    restatement run in float64 on the same device."""
    torch.manual_seed(1)
    x = torch.randn(256, 110250, 1, device='cuda')
    layer = K.Energy(sample_rate=22050, data_format=CL)
    y = layer(x)
    yr = torch.randn_like(y)
    xg = x.clone().requires_grad_(True)
    (gx,) = torch.autograd.grad(layer(xg), xg, grad_outputs=yr)
    xd = x.double().requires_grad_(True)
    (want,) = torch.autograd.grad(RA.energy(xd, 2205, 1102, False, 0.0, 0.1 / (2205 / 22050), CL), xd,
                                  grad_outputs=yr.double())
    err = float((gx.double() - want).abs().max())
    assert err <= 1e-4 * float(want.abs().max()), err
    del x, y, yr, xg, gx, xd, want
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------ a training chain
def test_training_chain_gain_and_waveform():
    """clean + learnable gain * noise -> log-mel (dB) -> Delta -> SpecAugment(training) -> ConcatenateFrequencyMap -> loss.
    (A gain on the whole waveform would only shift the decibels by a constant, which Delta removes: its gradient is 0.
    SpecAugment takes depth-1 spectrograms, so it comes before the frequency map adds its channel.)"""
    rng = np.random.default_rng(8)
    n_fft, hop, sr, n_mels = 512, 128, 16000, 64
    mel = K.get_melspectrogram_layer(n_fft=n_fft, hop_length=hop, sample_rate=sr, n_mels=n_mels, return_decibel=True,
                                     input_data_format=CL, output_data_format=CL)
    delta = K.Delta(win_length=5, data_format=CL)
    aug = K.SpecAugment(freq_mask_param=8, time_mask_param=10, data_format=CL, seed=3)
    cfm = K.ConcatenateFrequencyMap(data_format=CL)
    x = _randn(rng, (2, 16000, 1))
    noise = _randn(rng, (2, 16000, 1))
    gain = torch.tensor(0.7, device='cuda', requires_grad=True)
    xw = x.cuda().requires_grad_(True)
    y = cfm(aug(delta(mel(xw + gain * noise.cuda())), training=True))
    w = _randn(rng, tuple(y.shape)).cuda()
    (y * w).sum().backward()
    tm, fm = aug.last_masks

    fb = mel.layers[2].filterbank
    gr = torch.tensor(0.7, dtype=torch.float64, requires_grad=True)
    xr = x.double().requires_grad_(True)
    s = R.magnitude_to_decibel(R.apply_filterbank(R.magnitude(R.stft(xr + gr * noise.double(), n_fft, n_fft, hop, None,
                                                                     False, False, CL, CL)), fb, CL))
    yr = RA.concat_frequency_map(RA.spec_augment(RA.delta(s, 5, 'symmetric', CL), tm, fm, 0.0, CL), CL)
    (yr * w.cpu().double()).sum().backward()
    _rel_l2(xw.grad, xr.grad, 2e-3)
    assert abs(float(gain.grad) - float(gr.grad)) <= 2e-3 * abs(float(gr.grad)), (float(gain.grad), float(gr.grad))


# ------------------------------------------------------------------------------ coverage and the no-grad path
def _public_cases():
    """name -> (callable that builds a model, input shape, call kwargs) for every layer and factory in __all__."""
    mel_kw = dict(n_fft=512, hop_length=128, input_data_format=CL, output_data_format=CL)
    return {
        'STFT': (lambda: K.STFT(**mel_kw), (2, 4000, 1), {}),
        'InverseSTFT': (lambda: K.InverseSTFT(n_fft=512, hop_length=128, input_data_format=CL, output_data_format=CL),
                        (2, 10, 257, 1), {}),
        'Magnitude': (K.Magnitude, (2, 10, 257, 1), {}),
        'Phase': (K.Phase, (2, 10, 257, 1), {}),
        'MagnitudeToDecibel': (K.MagnitudeToDecibel, (2, 10, 257, 1), {}),
        'ApplyFilterbank': (lambda: K.ApplyFilterbank('mel', dict(sample_rate=16000, n_freq=257, n_mels=40),
                                                      data_format=CL), (2, 10, 257, 1), {}),
        'Delta': (lambda: K.Delta(data_format=CL), (2, 10, 40, 1), {}),
        'ConcatenateFrequencyMap': (lambda: K.ConcatenateFrequencyMap(data_format=CL), (2, 10, 40, 1), {}),
        'Frame': (lambda: K.Frame(frame_length=256, hop_length=64, data_format=CL), (2, 4000, 1), {}),
        'Energy': (lambda: K.Energy(data_format=CL), (2, 8000, 1), {}),
        'LogmelToMFCC': (lambda: K.LogmelToMFCC(data_format=CL), (2, 10, 40, 1), {}),
        'SpecAugment': (lambda: K.SpecAugment(freq_mask_param=5, time_mask_param=3, data_format=CL, seed=0),
                        (2, 10, 40, 1), {'training': True}),
        'Sequential': (lambda: K.Sequential([K.STFT(**mel_kw), K.Magnitude(), K.Delta(data_format=CL)]),
                       (2, 4000, 1), {}),
        'get_stft_magnitude_layer': (lambda: K.get_stft_magnitude_layer(return_decibel=True, **mel_kw), (2, 4000, 1), {}),
        'get_melspectrogram_layer': (lambda: K.get_melspectrogram_layer(return_decibel=True, **mel_kw), (2, 4000, 1), {}),
        'get_log_frequency_spectrogram_layer': (
            lambda: K.get_log_frequency_spectrogram_layer(sample_rate=16000, return_decibel=True, **mel_kw),
            (2, 4000, 1), {}),
        'get_perfectly_reconstructing_stft_istft': (
            lambda: K.Sequential(list(K.get_perfectly_reconstructing_stft_istft(512, 128, CL, CL))), (2, 4000, 1), {}),
        'get_stft_mag_phase': (lambda: K.get_stft_mag_phase(None, return_decibel=True, **mel_kw), (2, 4000, 1), {}),
    }


_NOT_LAYERS = {'__version__', 'VERSION', 'backend', 'composed', 'augmentation', 'Layer'}


def _input(shape, complex_in):
    x = torch.randn(shape, device='cuda')
    return torch.complex(x, torch.randn_like(x)) if complex_in else x


def test_every_public_layer_records_a_gradient():
    cases = _public_cases()
    assert set(K.__all__) - _NOT_LAYERS == set(cases)
    for name, (make, shape, kw) in cases.items():
        complex_in = name in ('InverseSTFT', 'Magnitude', 'Phase')
        x = _input(shape, complex_in).requires_grad_(True)
        y = make()(x, **kw)
        assert y.grad_fn is not None, name
        (gx,) = torch.autograd.grad(y.abs().sum() if y.is_complex() else y.sum(), x)
        assert gx.shape == x.shape and bool(torch.isfinite(torch.view_as_real(gx) if gx.is_complex() else gx).all()), name


def test_no_grad_path_is_unchanged():
    """Same launches, in the same number, and the same bits with and without requires_grad (and under no_grad)."""
    for name, (make, shape, kw) in _public_cases().items():
        complex_in = name in ('InverseSTFT', 'Magnitude', 'Phase')
        torch.manual_seed(5)
        x = _input(shape, complex_in)
        outs, counts = [], []
        for variant in ('plain', 'requires_grad', 'no_grad'):
            layer = make()
            layer(x, **kw)                                  # plans, filterbanks, workspaces made on first use
            layer = make() if name == 'SpecAugment' else layer     # the same masks in every variant
            xi = x.clone().requires_grad_(variant != 'plain')
            torch.cuda.synchronize()
            n0 = N.launch_count()
            if variant == 'no_grad':
                with torch.no_grad():
                    y = layer(xi, **kw)
            else:
                y = layer(xi, **kw)
            torch.cuda.synchronize()
            counts.append(N.launch_count() - n0)
            outs.append(y.detach())
            assert (y.grad_fn is None) == (variant != 'requires_grad'), (name, variant)
        assert counts[0] == counts[1] == counts[2], (name, counts)
        assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2]), name


@pytest.mark.parametrize('name', ['Phase', 'Delta', 'Frame', 'Energy', 'ConcatenateFrequencyMap', 'SpecAugment',
                                  'get_stft_mag_phase'])
def test_double_backward_raises(name):
    make, shape, kw = _public_cases()[name]
    x = _input(shape, name == 'Phase').requires_grad_(True)
    y = make()(x, **kw)
    (gx,) = torch.autograd.grad(y.square().sum(), x, create_graph=True)
    with pytest.raises(RuntimeError, match='twice'):
        (gx.abs() if gx.is_complex() else gx).sum().backward()
