"""CPU tier: the homogeneity checks of test_gpu_scale_range.py on the CPU emulation of the kernel bodies.

The emulation builds the same sources with host math (std::sqrt for kb_sqrt, a true division for __fdividef), so
what it catches is scale dependence in the algorithm itself: absolute constants, the rescaled branches of kb_cabs and
kb_atan2, a clamp that binds.  An op of degree d must give ``op(2^k x) == 2^(d k) op(x)`` bit for bit on every rung
where the intermediates stay normal; the GPU tier adds the hardware intrinsics."""
import math

import numpy as np
import pytest

import emu_harness as E
import oracle as O

LADDER = (-120, -90, -60, -40, -20, 0, 15, 20, 40, 60, 90, 120)
CF = 'channels_first'


def rungs(lo, hi):
    return [k for k in LADDER if lo <= k <= hi]


def scaled(x, k):
    x = np.asarray(x)
    if np.iscomplexobj(x):
        out = np.empty_like(x)
        out.real, out.imag = np.ldexp(x.real, k), np.ldexp(x.imag, k)
        return out
    return np.ldexp(x, k).astype(x.dtype)


def same(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and a.tobytes() == b.tobytes()


def homogeneous(y, y0, k):
    """y == 2^k y0 bit for bit wherever 2^k y0 is a normal float or zero.  An output that is rounding noise of a
    cancellation (1e-19 where its neighbours are 1) leaves the normal range first, and is only held to stay tiny."""
    want = scaled(y0, k)
    parts = (lambda v: (v.real, v.imag)) if np.iscomplexobj(want) else (lambda v: (v,))
    for a, b in zip(parts(np.asarray(y)), parts(want)):
        ok = (np.abs(b) >= np.finfo(np.float32).tiny) | (b == 0)
        if not same(a[ok], b[ok]) or np.abs(a[~ok]).max(initial=0) > 2 * np.finfo(np.float32).tiny:
            return False
    return True


def _wave(rng, shape):
    x = rng.uniform(-1, 1, size=shape)
    return (np.sign(x) * np.maximum(np.abs(x), 2.0 ** -12)).astype(np.float32)


def _cplx(rng, shape):
    re = np.sign(rng.uniform(-1, 1, shape)) * rng.uniform(2.0 ** -4, 1, shape)
    im = np.sign(rng.uniform(-1, 1, shape)) * rng.uniform(2.0 ** -4, 1, shape)
    return (re + 1j * im).astype(np.complex64)


def _forward(kind, n_fft, mode):
    hop = n_fft // 4
    w = O.get_window('hann_window', n_fft).astype(np.float32)
    if kind == 'k1':
        return lambda x: E.emu_stft(x, n_fft, n_fft, hop, w, True, True, mode, CF, CF, TF=8, n_warps=2)[0]
    if kind == 'mc':
        return lambda x: E.emu_stft_mc(x, n_fft, n_fft, hop, w, True, True, mode, CF, CF)[0]
    if kind == 'mr':
        return lambda x: E.emu_mr(x, n_fft, n_fft, hop, w, True, True, mode, CF, CF)
    return lambda x: E.emu_dft(x, n_fft, n_fft, hop, w, True, True, mode, CF, CF)


# (kind, n_fft, channels, modes): K1 single-channel, K1b all-channel, mixed radix, direct DFT
FAMILIES = [('k1', 512, 1, (E.MODE_COMPLEX, E.MODE_MAG, E.MODE_MAG_PHASE)),
            ('mc', 512, 2, (E.MODE_COMPLEX, E.MODE_MAG, E.MODE_MAG_PHASE)),
            ('mr', 400, 1, (E.MODE_COMPLEX, E.MODE_MAG)),
            ('dft', 98, 1, (E.MODE_COMPLEX, E.MODE_MAG))]


@pytest.mark.parametrize('kind,n_fft,C,modes', FAMILIES, ids=[f[0] for f in FAMILIES])
def test_forward_transforms_are_homogeneous(kind, n_fft, C, modes):
    """Complex and magnitude outputs of degree 1, the fused phase of degree 0, from 2^-60 to 2^90: 2^120 overflows the
    spectrum, and at 2^-90 some FFT partial sums that cancel go subnormal and round differently."""
    rng = np.random.default_rng(n_fft + C)
    x = _wave(rng, (2, C, 9 * (n_fft // 4) + 3))
    for mode in modes:
        fwd = _forward(kind, n_fft, mode)
        y0 = fwd(x)
        for k in rungs(-60, 90):
            y = fwd(scaled(x, k))
            if mode == E.MODE_MAG_PHASE:
                assert homogeneous(y[:, :C], y0[:, :C], k), (mode, k)
                assert same(y[:, C:], y0[:, C:]), (mode, k)
            else:
                assert homogeneous(y, y0, k), (mode, k)
        assert not np.abs(fwd(np.zeros_like(x))).max()


@pytest.mark.parametrize('kind', ['istft', 'idft'])
def test_inverse_transforms_are_homogeneous(kind):
    rng = np.random.default_rng(11)
    n_fft = 512 if kind == 'istft' else 400
    hop = n_fft // 4
    X = _cplx(rng, (2, 1, 12, n_fft // 2 + 1))
    dual = O.inverse_stft_window(n_fft, hop, O.get_window('hann_window', n_fft)).astype(np.float32)
    inv = E.emu_istft if kind == 'istft' else E.emu_idft
    y0 = inv(X, n_fft, n_fft, hop, dual, CF, CF)
    for k in rungs(-60, 90):
        assert homogeneous(inv(scaled(X, k), n_fft, n_fft, hop, dual, CF, CF), y0, k), k
    assert not np.abs(inv(np.zeros_like(X), n_fft, n_fft, hop, dual, CF, CF)).max()


def test_filterbank_is_homogeneous():
    rng = np.random.default_rng(12)
    S = (rng.random((2, 2, 9, 257)) * 0.75 + 0.25).astype(np.float32)
    fb = O.filterbank_mel(16000, 257, 40, 0.0, None, False, 'slaney').astype(np.float32)
    y0 = E.emu_fb(S, fb, CF)
    for k in rungs(-60, 90):
        assert homogeneous(E.emu_fb(scaled(S, k), fb, CF), y0, k), k


def test_atan2_is_degree_zero_over_the_whole_float_range():
    """Every rung keeps the parts of _cplx normal; kb_atan2's scaled division holds above 2^126 and below 2^-100."""
    rng = np.random.default_rng(13)
    X = _cplx(rng, 4096)
    y0 = E.emu_atan2(X.imag.copy(), X.real.copy())
    assert np.abs(y0 - np.angle(X.astype(np.complex128))).max() < 1e-6
    for k in LADDER:
        Xs = scaled(X, k)
        assert same(E.emu_atan2(Xs.imag.copy(), Xs.real.copy()), y0), k
    top = np.float32(3e38)
    assert abs(float(E.emu_atan2(np.array([top], np.float32), np.array([top], np.float32))[0]) - math.pi / 4) < 1e-6


def test_decibel_tail_shifts_by_10_k_log10_2():
    rng = np.random.default_rng(14)
    x = (rng.random(4096) * 0.75 + 0.25).astype(np.float32)
    y0 = E.emu_db_tail(x, amin=2e-38).astype(np.float64)
    for k in rungs(-90, 120):
        y = E.emu_db_tail(scaled(x, k), amin=2e-38).astype(np.float64)
        d = y - y0 - 10.0 * math.log10(2.0) * k
        assert np.abs(d).max() <= 4 * np.spacing(np.float32(np.abs(y).max())) + 1e-5, k


@pytest.mark.parametrize('rn', [0, 1], ids=['approx_form', 'rounded_form'])
def test_cabs_matches_float64_over_the_whole_float_range(rn):
    """kb_cabs in both forms (rn = 1: sqrtf(fmaf) of the CQT, chroma, time-stretch and Kaldi magnitudes; rn = 0:
    kb_sqrt(cnorm) of the STFT family) against |X| in float64, for parts from subnormal to FLT_MAX: within 2 ulps of
    a normal result, within the subnormal spacing of a subnormal one, inf exactly where |X| exceeds FLT_MAX, NaN
    where a part is NaN, and 2^k |X| bit for bit across the ladder."""
    rng = np.random.default_rng(15 + rn)
    X = _cplx(rng, 4096)
    y0 = E.emu_cabs(X.real, X.imag, rn)
    for k in LADDER:
        Xs = scaled(X, k)
        assert same(E.emu_cabs(Xs.real, Xs.imag, rn), scaled(y0, k)), k
    # every exponent of both parts, zero and the extremes included
    e = rng.integers(-149, 128, size=(2, 20000))
    parts = np.ldexp(rng.uniform(1, 2, size=e.shape), e) * np.sign(rng.uniform(-1, 1, size=e.shape))
    parts = np.where(np.abs(parts) > np.finfo(np.float32).max, np.finfo(np.float32).max, parts).astype(np.float32)
    parts[:, :8] = np.float32([[0, 0, 0, 1e-45, 3.4028235e38, 3.4028235e38, 1e-45, 2e38],
                               [0, 1e-45, -1e-45, 0, 3.4028235e38, 0, 1e-45, 2e38]])
    got = E.emu_cabs(parts[0], parts[1], rn).astype(np.float64)
    want = np.hypot(parts[0].astype(np.float64), parts[1].astype(np.float64))
    over = want > np.finfo(np.float32).max
    assert np.isinf(got[over]).all() and np.isfinite(got[~over]).all()
    tiny = np.finfo(np.float32).tiny
    sub = ~over & (want < tiny)
    assert (np.abs(got[sub] - want[sub]) <= 2.0 ** -149).all()
    nrm = ~over & ~sub
    assert (np.abs(got[nrm] - want[nrm]) <= 2 * np.spacing(np.minimum(want[nrm], np.finfo(np.float32).max).astype(np.float32)).astype(np.float64)).all()
    nan = np.float32(np.nan)
    assert np.isnan(E.emu_cabs(np.float32([nan, 1.0, nan]), np.float32([1.0, nan, np.inf]), rn)).all()
