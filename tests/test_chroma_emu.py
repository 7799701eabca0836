"""Chroma on the CPU: the kernel bodies of chroma_core.cuh (run by a CPU emulation) against the float64 restatement
(chroma_ref.py): the projection and its gradient within the derived bound in every input mode, norm and layout, the
tuning estimate's peaks bit for bit against a float32 restatement with its median and histogram index exact, the CENS
quantisation and smoothing, tile orders and CTA counts, the host tables against independent anchors, gradcheck of
the restatement and validation."""
import ctypes
import hashlib
import os
import subprocess
import tempfile

import numpy as np
import pytest
import torch

import chroma_ref as R
from emu_harness import Checked
from kapre_b200 import backend, signal

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, 'emu', 'kb_emu_chroma.cpp')
_CSRC = os.path.join(_HERE, '..', 'kapre_b200', 'csrc')
_lib_handle = None
CL, CF = 'channels_last', 'channels_first'
NORMS = {None: 0, np.inf: 1, 1: 2, 2: 3}
ORDERS = [(0, 0), (1, 0), (2, 0), (0, 3), (1, 5)]


def _lib():
    """tests/emu/kb_emu_chroma.cpp built with g++ into the temporary directory (keyed by the sources' contents)."""
    global _lib_handle
    if _lib_handle is None:
        hs = hashlib.sha256()
        for f in [_SRC] + sorted(os.path.join(_CSRC, n) for n in os.listdir(_CSRC) if n.endswith(('.h', '.cuh'))):
            with open(f, 'rb') as fh:
                hs.update(fh.read())
        out = os.path.join(tempfile.gettempdir(), 'kapre_b200_emu_chroma_%s.so' % hs.hexdigest()[:16])
        if not os.path.exists(out):
            tmp = '%s.%d.tmp' % (out, os.getpid())
            subprocess.check_call(['g++', '-O2', '-std=c++17', '-shared', '-fPIC', '-DKB_HOST_EMU', '-Wno-unknown-pragmas',
                                   '-o', tmp, _SRC])
            os.replace(tmp, out)
        lib = ctypes.CDLL(out)
        lib.kb_emu_chroma.argtypes = [ctypes.c_void_p, ctypes.c_float] + [ctypes.c_void_p] * 10 + [ctypes.c_int] * 2
        lib.kb_emu_tuning.argtypes = [ctypes.c_void_p, ctypes.c_float, ctypes.c_float, ctypes.c_double] + \
            [ctypes.c_void_p] * 10 + [ctypes.c_int] * 2
        lib.kb_emu_cens.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_void_p] + [ctypes.c_int] * 3 + \
            [ctypes.c_void_p] * 3 + [ctypes.c_int] * 2
        _lib_handle = Checked(lib)
    return _lib_handle


def _p(a):
    return None if a is None else ctypes.c_void_p(a.__array_interface__['data'][0])


def _strides(a, fmt):
    """Element strides (b, c, t, k) of a 4-D array in ``fmt``."""
    st = [s // a.itemsize for s in a.strides]
    return np.array([st[0], st[3], st[1], st[2]] if fmt == CL else st, np.int64)


def _to_fmt(a, fmt):
    """(B, C, M, K) -> the layout of ``fmt`` (a copy)."""
    return np.ascontiguousarray(a.transpose(0, 2, 3, 1) if fmt == CL else a)


def _from_fmt(a, fmt):
    return a.transpose(0, 3, 1, 2) if fmt == CL else a


def emu_chroma(x, W, mode, norm, fmt, thr=None, tab=None, order=0, n_cta=0, cens=False, g=None):
    """x: (B, C, M, K) float32 (complex64 for mode 2); W: (T, NC, K).  Returns (B, C, M, NC) or the input gradient."""
    B, C, M, K = x.shape
    W32 = np.ascontiguousarray(W, np.float32)
    NC = W.shape[1]
    xin = _to_fmt(x, fmt)
    ic = np.array([NC, K, mode, NORMS[norm], int(cens), int(thr is not None), B, C, M], np.int32)
    tb = None if tab is None else np.ascontiguousarray(tab, np.int32)
    out = _to_fmt(np.full((B, C, M, NC), -7.0, np.float32), fmt)
    xs, os_ = _strides(xin, fmt), _strides(out, fmt)
    if g is None:
        rc = _lib().kb_emu_chroma(_p(ic), 0.0 if thr is None else thr, _p(W32), _p(tb), _p(xin), _p(xs), _p(out),
                                  _p(os_), None, None, None, None, order, n_cta)
        assert rc == 0
        return _from_fmt(out, fmt)
    gin = _to_fmt(np.asarray(g, np.float32), fmt)
    gx = _to_fmt(np.full(x.shape, -7.0, x.dtype), fmt)
    gs, gxs = _strides(gin, fmt), _strides(gx, fmt)
    rc = _lib().kb_emu_chroma(_p(ic), 0.0 if thr is None else thr, _p(W32), _p(tb), _p(xin), _p(xs), None, None,
                              _p(gin), _p(gs), _p(gx), _p(gxs), order, n_cta)
    assert rc == 0
    return _from_fmt(gx, fmt)


def emu_tuning(S, sr, n_fft, lo, hi, resolution=0.01, bpo=12, mode=0, fmt=CF, order=0, n_cta=0):
    """S: (B, C, M, K) float32.  Returns (tuning, index, mag, pitch, hist)."""
    B, C, M, K = S.shape
    edges = backend.tuning_edges(resolution)
    nres = edges.size - 1
    cap = (hi - lo + 1) // 2
    xin = _to_fmt(S, fmt)
    ic = np.array([K, lo, hi, mode, nres, B, C, M], np.int32)
    mag = np.full((B * C, M, cap), 7.0, np.float32)
    pitch = np.full((B * C, M, cap), 7.0, np.float32)
    hist = np.zeros((B, 4, 256), np.uint32)
    above = np.full(B, 0xffffffff, np.uint32)
    res = np.zeros((B, nres), np.uint32)
    tuning = np.full(B, 9.0)
    tab = np.full(B, -1, np.int32)
    xs = _strides(xin, fmt)
    rc = _lib().kb_emu_tuning(_p(ic), sr, float(n_fft), float(bpo), _p(edges), _p(xin), _p(xs),
                              _p(mag), _p(pitch), _p(hist), _p(above), _p(res), _p(tuning), _p(tab), order, n_cta)
    assert rc == 0
    return tuning, tab, mag, pitch, hist


def emu_cens(q, taps, fmt=CF, order=0, n_cta=0):
    B, C, M, NC = q.shape
    w = np.ascontiguousarray(taps, np.float32)
    qc = np.ascontiguousarray(q, np.float32)
    out = _to_fmt(np.full(q.shape, -7.0, np.float32), fmt)
    os_ = _strides(out, fmt)
    rc = _lib().kb_emu_cens(NC, len(w), _p(w), B, C, M, _p(qc), _p(out), _p(os_), order, n_cta)
    assert rc == 0
    return _from_fmt(out, fmt)


def _mag(rng, B, C, M, K):
    """A magnitude-like spectrogram: log-uniform values with a few strong partials."""
    x = (10.0 ** rng.uniform(-3, 0, size=(B, C, M, K))).astype(np.float32)
    for _ in range(4):
        x[..., rng.integers(20, K - 20)] *= 30
    return x


# ---- host tables against independent anchors -------------------------------------------------------------------------
@pytest.mark.parametrize('n_chroma', [12, 24, 7])
def test_filterbank_columns_unit_norm_and_pitch_classes(n_chroma):
    W = backend.chroma_filterbank(22050, 4096, n_chroma=n_chroma, octwidth=None)
    np.testing.assert_allclose(np.sqrt((W ** 2).sum(axis=0)), 1.0, rtol=1e-12)
    if n_chroma % 12:
        return
    # a bin centred on pitch class p (C = 0) peaks in chroma p * n_chroma / 12
    for midi in range(48, 84):
        f = 440.0 * 2.0 ** ((midi - 69) / 12.0)
        k = f * 4096 / 22050
        if abs(k - round(k)) > 0.05:
            continue
        assert W[:, int(round(k))].argmax() == (midi % 12) * n_chroma // 12, midi


def test_filterbank_peaks_on_exact_bin_frequencies():
    # sr = 440 * n_fft / 40: bin 40 is A4 exactly, bin 20 A3; A is chroma 9 with C first, 0 without base_c
    n_fft = 4096
    sr = 440.0 * n_fft / 40
    W = backend.chroma_filterbank(sr, n_fft)
    assert W[:, 40].argmax() == 9 and W[:, 20].argmax() == 9
    assert backend.chroma_filterbank(sr, n_fft, base_c=False)[:, 40].argmax() == 0
    # tuning +0.5 chroma bin moves A4's bump half-way to A#
    Wt = backend.chroma_filterbank(sr, n_fft, tuning=0.5, octwidth=None)
    W0 = backend.chroma_filterbank(sr, n_fft, octwidth=None)
    assert Wt[9, 40] < W0[9, 40] and Wt[8, 40] > W0[8, 40]


@pytest.mark.parametrize('bpo,n_chroma,f_min', [(36, 12, None), (12, 12, None), (24, 12, 55.0), (48, 24, 100.0)])
def test_cq_to_chroma_maps_each_bin_to_its_pitch_class(bpo, n_chroma, f_min):
    n_bins = 7 * bpo
    M = backend.cq_to_chroma(n_bins, bpo, n_chroma, f_min)
    assert M.shape == (n_chroma, n_bins)
    np.testing.assert_array_equal(M.sum(axis=0), 1.0)
    freqs = backend.cqt_frequencies(n_bins, f_min, bpo)
    midi = backend.hz_to_midi(freqs)
    for k in range(n_bins):
        pc = midi[k] * n_chroma / 12.0
        if abs(pc - round(pc)) < 1e-6:        # a bin centred on a pitch class
            assert M[:, k].argmax() == int(round(pc)) % n_chroma, k
    with pytest.raises(ValueError):
        backend.cq_to_chroma(84, 12, 24)


def test_tuning_grid_tables_equal_fixed_tuning_tables():
    edges = backend.tuning_edges(0.01)
    assert edges.size == 101 and edges[0] == -0.5 and edges[-1] == 0.5
    plan = signal._stft_chroma_plans(22050, 1024, 256, None, 12, None, 5.0, 2.0, True)[1]
    for k in (0, 17, 50, 99):
        fixed = signal._stft_chroma_plans(22050, 1024, 256, None, 12, float(edges[k]), 5.0, 2.0, True)[1]
        np.testing.assert_array_equal(plan.tables[k], fixed.tables[0])
    np.testing.assert_array_equal(plan.tables[100], backend.chroma_filterbank(22050, 1024))


def test_cens_window_matches_scipy_and_smoothing_matches_ndimage():
    import scipy.ndimage
    import scipy.signal
    for n in (1, 2, 41, 8):
        w = scipy.signal.get_window('hann', n + 2, fftbins=False)
        np.testing.assert_allclose(backend.cens_window(n), w / w.sum(), atol=1e-15)
        q = np.random.default_rng(n).uniform(size=(30, 5))
        want = scipy.ndimage.convolve(q, (w / w.sum())[:, None], mode='constant')
        np.testing.assert_allclose(R.smooth(q, backend.cens_window(n)), want, atol=1e-14)


def test_validation():
    for kw in [dict(norm=3), dict(norm='l2'), dict(n_chroma=0), dict(n_chroma=65), dict(n_fft=16384),
               dict(win_length=1024)]:
        a = dict(sample_rate=22050, tuning=0.0)
        a.update(kw)
        with pytest.raises(ValueError):
            from kapre_b200.time_frequency import ChromaSTFT
            ChromaSTFT(**a)
    for r in (0.0, -0.1, 1.5, 0.0009):
        with pytest.raises(ValueError):
            backend.tuning_edges(r)
    from kapre_b200.time_frequency import ChromaCENS, ChromaCQT
    with pytest.raises(ValueError):
        ChromaCQT(bins_per_octave=30)
    with pytest.raises(ValueError):
        ChromaCQT(tuning=None)
    with pytest.raises(ValueError):
        ChromaCENS(win_len_smooth=600)
    with pytest.raises(ValueError):
        ChromaCQT(n_octaves=13)


def test_layers_round_trip_and_aliases():
    from kapre.signal import chroma_cens, chroma_cqt, chroma_stft, estimate_tuning  # noqa: F401
    from kapre.time_frequency import ChromaCENS, ChromaCQT, ChromaSTFT
    for layer in (ChromaSTFT(n_fft=1024, norm=2, tuning=0.1), ChromaSTFT(), ChromaCQT(threshold=None, norm=1),
                  ChromaCENS(win_len_smooth=None, data_format='channels_first')):
        cfg = layer.get_config()
        again = type(layer).from_config(cfg)
        assert again.get_config() == cfg


# ---- projection ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('mode', [0, 1, 2])
@pytest.mark.parametrize('norm', [np.inf, 1, 2, None])
@pytest.mark.parametrize('fmt', [CL, CF])
def test_projection_within_bound(mode, norm, fmt):
    rng = np.random.default_rng(mode * 7 + NORMS[norm])
    B, C, M, K = 2, 2, 37, 129
    x = _mag(rng, B, C, M, K)
    x[0, 1, 3] = 0.0                                    # a silent frame stays 0
    if mode == 2:
        x = (x * np.exp(1j * rng.uniform(0, 6.3, size=x.shape))).astype(np.complex64)
    W = backend.chroma_filterbank(256 * 22050 / 1024.0 / 2, 256)[None]
    thr = 0.05 if norm == 2 else None
    got = emu_chroma(x, W, mode, norm, fmt, thr=thr).astype(np.float64)
    s = np.abs(x).astype(np.float64) ** (2 if mode == 1 else 1)
    if mode == 1:
        s = (np.abs(x).astype(np.float32) ** 2).astype(np.float64)     # the kernel's own float32 square...
    want, bound = R.project(s, W[0], norm, thr)
    bound = bound + (R.gamma(2) * np.abs(want) if mode else 0)         # ...or modulus, rounded once
    assert (np.abs(got - want) <= bound).all(), float((np.abs(got - want) - bound).max())
    np.testing.assert_array_equal(got[0, 1, 3], 0.0)


@pytest.mark.parametrize('n_chroma', [12, 24, 40, 64])
def test_projection_tile_orders_cta_counts_and_tables(n_chroma):
    rng = np.random.default_rng(n_chroma)
    B, C, M, K = 3, 1, 300, 65
    x = _mag(rng, B, C, M, K)
    W = np.stack([backend.chroma_filterbank(8000, 128, n_chroma, t) for t in (0.0, 0.3, -0.2)])
    tab = np.array([2, 0, 1], np.int32)
    ref = emu_chroma(x, W, 1, np.inf, CF, tab=tab)
    for order, n_cta in ORDERS:
        np.testing.assert_array_equal(emu_chroma(x, W, 1, np.inf, CL, tab=tab, order=order, n_cta=n_cta), ref)
    # item by item, the per-item table equals a single-table call
    for b in range(B):
        np.testing.assert_array_equal(emu_chroma(x[b:b + 1], W[tab[b]:tab[b] + 1], 1, np.inf, CF), ref[b:b + 1])
    s = (x.astype(np.float32) ** 2).astype(np.float64)
    for b in range(B):
        want, bound = R.project(s[b], W[tab[b]], np.inf)
        assert (np.abs(ref[b] - want) <= bound + R.gamma(2) * want).all()


@pytest.mark.parametrize('mode', [0, 1, 2])
@pytest.mark.parametrize('norm', [np.inf, 1, 2, None])
def test_projection_gradient_within_bound(mode, norm):
    rng = np.random.default_rng(11 + mode)
    B, C, M, K = 2, 1, 19, 65
    x = _mag(rng, B, C, M, K)
    x[1, 0, 4] = 0.0
    if mode == 2:
        x = (x * np.exp(1j * rng.uniform(0, 6.3, size=x.shape))).astype(np.complex64)
    W = backend.chroma_filterbank(8000, 128)[None]
    g = rng.standard_normal((B, C, M, 12)).astype(np.float32)
    thr = 0.02 if norm == 1 else None
    got = None
    for fmt, (order, n_cta) in zip([CF, CL, CF], [(0, 0), (1, 3), (2, 0)]):
        r = emu_chroma(x, W, mode, norm, fmt, thr=thr, g=g, order=order, n_cta=n_cta)
        if got is None:
            got = r
        np.testing.assert_array_equal(r, got)
    xa = np.abs(x).astype(np.float64)
    s = (np.abs(x).astype(np.float32) ** 2).astype(np.float64) if mode == 1 else xa
    xx = x.astype(np.complex128) if mode == 2 else xa
    want, bound = R.project_grad(s, W[0], norm, g.astype(np.float64), thr,
                                 {0: 'linear', 1: 'square', 2: 'complex'}[mode], xx)
    # the recomputed y carries the forward's relative error into the normalisation's derivative
    err = np.abs(got.astype(np.complex128 if mode == 2 else np.float64) - want)
    assert (err <= 4 * bound).all(), float((err - 4 * bound).max())


def test_gradcheck_of_the_restatement():
    rng = np.random.default_rng(3)
    W = torch.from_numpy(backend.chroma_filterbank(8000, 64))
    for norm in (np.inf, 1, 2, None):
        x = torch.from_numpy(rng.uniform(0.1, 1.0, size=(5, 33))).requires_grad_(True)

        def f(x):
            y = (x ** 2) @ W.T
            if norm is None:
                return y
            if norm == np.inf:
                n = y.abs().max(dim=-1, keepdim=True).values
            else:
                n = y.abs().pow(norm).sum(dim=-1, keepdim=True).pow(1.0 / norm)
            return y / n
        assert torch.autograd.gradcheck(f, (x,))
        g = rng.standard_normal((5, 12))
        want = torch.autograd.grad(f(x), x, torch.from_numpy(g))[0].numpy()
        s = x.detach().numpy() ** 2
        got, _ = R.project_grad(s, W.numpy(), norm, g, None, 'square', x.detach().numpy())
        np.testing.assert_allclose(got, want, rtol=1e-10, atol=1e-12)


def test_non_finite_frame_stays_local():
    rng = np.random.default_rng(5)
    x = _mag(rng, 2, 1, 40, 65)
    y = x.copy()
    y[1, 0, 7, 30] = np.nan
    W = backend.chroma_filterbank(8000, 128)[None]
    a, b = emu_chroma(x, W, 1, np.inf, CF), emu_chroma(y, W, 1, np.inf, CF)
    assert np.isnan(b[1, 0, 7]).all()
    keep = np.ones(40, bool)
    keep[7] = False
    np.testing.assert_array_equal(a[1, 0, keep], b[1, 0, keep])
    np.testing.assert_array_equal(a[0], b[0])


# ---- tuning estimate ----------------------------------------------------------------------------------------------------
def _power(rng, B, C, M, n_fft, sr, detune):
    """Power spectrogram of tones plus noise (numpy STFT), each item detuned by detune[b] semitones."""
    L = (M - 1) * (n_fft // 4) + n_fft
    t = np.arange(L) / sr
    S = np.zeros((B, C, M, n_fft // 2 + 1), np.float32)
    w = 0.5 - 0.5 * np.cos(2 * np.pi * np.arange(n_fft) / n_fft)
    for b in range(B):
        for c in range(C):
            sig = 0.01 * rng.standard_normal(L)
            for midi in rng.choice(np.arange(50, 80), 3, replace=False):
                f = 440.0 * 2.0 ** ((midi - 69 + detune[b]) / 12.0)
                sig += rng.uniform(0.3, 1.0) * np.sin(2 * np.pi * f * t + rng.uniform(0, 6))
            fr = np.lib.stride_tricks.sliding_window_view(sig, n_fft)[::n_fft // 4][:M] * w
            S[b, c] = (np.abs(np.fft.rfft(fr, axis=-1)) ** 2).astype(np.float32)
    return S


@pytest.mark.parametrize('fmt', [CF, CL])
def test_tuning_peaks_median_and_index_exact(fmt):
    sr, n_fft = 22050, 1024
    rng = np.random.default_rng(1)
    B, C, M = 4, 2, 30
    S = _power(rng, B, C, M, n_fft, sr, [0.0, 0.235, -0.315, 0.4])
    S[3] = 0.0                                           # an item without peaks
    S[2, 1, 5, 100] = np.inf                             # its frame contributes no peaks
    lo, hi = backend.piptrack_bins(sr, n_fft)
    ref = None
    for order, n_cta in ORDERS:
        got = emu_tuning(S, sr, n_fft, lo, hi, fmt=fmt, order=order, n_cta=n_cta)
        if ref is None:
            ref = got
        for u, v in zip(got, ref):
            np.testing.assert_array_equal(u, v)
    tuning, tab, mag, pitch, hist = ref
    cap = (hi - lo + 1) // 2
    for b in range(B):
        want_t, want_i, _, n = R.estimate_tuning(S[b], sr, n_fft, lo, hi)
        assert tuning[b] == want_t and tab[b] == want_i, (b, tuning[b], want_t)
        assert int(hist[b, 0].sum()) == n
        for c in range(C):
            peaks = R.piptrack32(S[b, c], sr, n_fft, lo, hi)
            for m in range(M):
                row = b * C + c
                slots = np.nonzero(mag[row, m] >= 0)[0]
                assert len(slots) == len(peaks[m])
                for s_, (k, mg, pt) in zip(slots, peaks[m]):
                    assert s_ == (k - lo) // 2
                    assert mag[row, m, s_].tobytes() == np.float32(mg).tobytes()
                    assert pitch[row, m, s_].tobytes() == np.float32(pt).tobytes()
    assert tuning[3] == 0.0 and tab[3] == 100


@pytest.mark.parametrize('n', [1, 2, 3, 4, 257, 1000, 1001])
def test_median_selection_exact_with_ties(n):
    """The radix selection on hand-made peak sets: many equal mags, an even and odd count, values across binary
    exponents (all above a tenth of their frame's maximum, so each one is a peak)."""
    sr, n_fft = 8000, 256
    lo, hi = backend.piptrack_bins(sr, n_fft)
    rng = np.random.default_rng(n)
    K = n_fft // 2 + 1
    per = max(1, min((hi - lo) // 4, 20))
    M = -(-n // per)
    S = np.zeros((1, 1, M, K), np.float32)
    vals = rng.choice(np.float32([1.0, 1.0, 2.5, 0.5, 0.375, 3.0, 1.0000001]), n)
    i = 0
    for m in range(M):
        for j in range(per):
            if i == n:
                break
            S[0, 0, m, lo + 1 + 4 * j] = vals[i]
            i += 1
    got = emu_tuning(S, sr, n_fft, lo, hi)
    want = R.estimate_tuning(S[0], sr, n_fft, lo, hi)
    assert got[0][0] == want[0] and got[1][0] == want[1]
    assert int(got[4][0, 0].sum()) == want[3] == n


# ---- CENS ---------------------------------------------------------------------------------------------------------------
def test_cens_quantisation_and_smoothing():
    rng = np.random.default_rng(9)
    B, C, M, K = 2, 1, 150, 84
    x = _mag(rng, B, C, M, K)
    Mq = backend.cq_to_chroma(K, 12, 12)[None]
    l1 = emu_chroma(x, Mq, 0, 1, CF, thr=0.0)
    q = emu_chroma(x, Mq, 0, None, CF, thr=0.0, cens=True)
    np.testing.assert_array_equal(q, R.quantize(l1))
    for win in (41, 8, None):
        taps = backend.cens_window(win)
        ref = None
        for fmt, (order, n_cta) in zip([CF, CL, CF], [(0, 0), (1, 2), (2, 0)]):
            got = emu_cens(q, taps, fmt, order, n_cta)
            if ref is None:
                ref = got
            np.testing.assert_array_equal(got, ref)
        want, bound = R.cens_from_q(q, taps)
        assert (np.abs(ref - want) <= bound).all()
    # NaN reaches only the frames whose window holds it
    qn = q.copy()
    qn[0, 0, 70, 3] = np.nan
    taps = backend.cens_window(41)
    got = emu_cens(qn, taps)
    bad = np.isnan(got[0, 0]).any(axis=-1)
    assert bad[70 - 21:70 + 22].all() and not bad[:70 - 21].any() and not bad[70 + 22:].any()
