"""Onsets, tempo and beats on the CPU: the kernel bodies of rhythm_core.cuh (run by a CPU emulation) against the
float64 restatements of rhythm_ref.py: onset strength within 1 ulp (the median exact), the tie rules, the gradient
against torch.autograd, the tempogram within a derived bound, the tempo, peak-pick and beat decisions, the block-
parallel DP against a serial loop, bit equality across tile orders, CTA counts, layouts and strides, isolation of
non-finite and all-zero rows, and validation."""
import ctypes
import hashlib
import os
import subprocess
import tempfile

import numpy as np
import pytest
import torch

import rhythm_ref as R
from emu_harness import Checked

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, 'emu', 'kb_emu_rhythm.cpp')
_CSRC = os.path.join(_HERE, '..', 'kapre_b200', 'csrc')
_lib_handle = None
CL, CF = 'channels_last', 'channels_first'
EPS32 = 2.0 ** -24


def _lib():
    """tests/emu/kb_emu_rhythm.cpp built with g++ into the temporary directory (keyed by the sources' contents)."""
    global _lib_handle
    if _lib_handle is None:
        hs = hashlib.sha256()
        for f in [_SRC] + sorted(os.path.join(_CSRC, n) for n in os.listdir(_CSRC) if n.endswith(('.h', '.cuh'))):
            with open(f, 'rb') as fh:
                hs.update(fh.read())
        out = os.path.join(tempfile.gettempdir(), 'kapre_b200_emu_rhythm_%s.so' % hs.hexdigest()[:16])
        if not os.path.exists(out):
            tmp = '%s.%d.tmp' % (out, os.getpid())
            subprocess.check_call(['g++', '-O2', '-std=c++17', '-shared', '-fPIC', '-DKB_HOST_EMU', '-Wno-unknown-pragmas',
                                   '-o', tmp, _SRC])
            os.replace(tmp, out)
        lib = ctypes.CDLL(out)
        vp, ci = ctypes.c_void_p, ctypes.c_int
        lib.kb_emu_onset.argtypes = [vp] * 5 + [ci] * 2
        lib.kb_emu_onset_bwd.argtypes = [vp] * 8 + [ci] * 2
        lib.kb_emu_tempogram.argtypes = [vp] * 5 + [ci] * 2
        lib.kb_emu_tempo.argtypes = [vp] * 4 + [ctypes.c_double] + [vp] * 2 + [ci] * 2
        lib.kb_emu_peak.argtypes = [vp, ctypes.c_double] + [vp] * 4 + [ci] * 2
        lib.kb_emu_beat.argtypes = [vp, vp, vp, ctypes.c_float] + [vp] * 6 + [ci] * 2
        _lib_handle = Checked(lib)
    return _lib_handle


def _p(a):
    return None if a is None else ctypes.c_void_p(a.__array_interface__['data'][0])


def _strides(x, perm):
    """Element strides of array x, reordered by perm (axis of x for b, c, t[, k])."""
    st = [s // x.itemsize for s in x.strides]
    return np.array([st[a] for a in perm], np.int64)


def _spec(S, fmt):
    """Canonical (B, C, T, K) -> (array in fmt, strides (b, c, t, k))."""
    if fmt == CL:
        x = np.ascontiguousarray(S.transpose(0, 2, 3, 1))
        return x, _strides(x, (0, 3, 1, 2))
    x = np.ascontiguousarray(S)
    return x, _strides(x, (0, 1, 2, 3))


def _rows(B, C, T, fmt, dtype=np.float32, fill=np.nan):
    """A (B, T, C) / (B, C, T) array and its strides (b, c, t)."""
    if fmt == CL:
        x = np.full((B, T, C), fill, dtype)
        return x, _strides(x, (0, 2, 1))
    x = np.full((B, C, T), fill, dtype)
    return x, _strides(x, (0, 1, 2))


def _canon_rows(x, fmt):
    return x.transpose(0, 2, 1) if fmt == CL else x


def _env_in(e, fmt):
    """Canonical (B, C, T) -> (array in fmt, strides)."""
    if fmt == CL:
        x = np.ascontiguousarray(e.transpose(0, 2, 1))
        return x, _strides(x, (0, 2, 1))
    x = np.ascontiguousarray(e)
    return x, _strides(x, (0, 1, 2))


def emu_onset(S, lag=1, max_size=1, aggregate='mean', pad=0, fmt=CF, order=0, n_cta=0, xin=None):
    B, C, T, K = S.shape
    ic = np.array([B, C, T, K, lag, max_size, 0 if aggregate == 'mean' else 1, pad], np.int32)
    x, xs = xin if xin is not None else _spec(S, fmt)
    out, os_ = _rows(B, C, T, fmt)
    assert _lib().kb_emu_onset(_p(ic), _p(x), _p(xs), _p(out), _p(os_), order, n_cta) == 0
    return _canon_rows(out, fmt)


def emu_onset_bwd(S, g, lag=1, max_size=1, aggregate='mean', pad=0, fmt=CF, order=0, n_cta=0):
    B, C, T, K = S.shape
    ic = np.array([B, C, T, K, lag, max_size, 0 if aggregate == 'mean' else 1, pad], np.int32)
    x, xs = _spec(S, fmt)
    gi, gs = _env_in(g.astype(np.float32), fmt)
    gx, gxs = _spec(np.full(S.shape, np.nan, np.float32), fmt)
    ws = np.zeros(2 * S.size, np.int32)
    assert _lib().kb_emu_onset_bwd(_p(ic), _p(x), _p(xs), _p(gi), _p(gs), _p(gx), _p(gxs), _p(ws), order, n_cta) == 0
    return gx.transpose(0, 3, 1, 2) if fmt == CL else gx


def emu_tempogram(e, W, center=True, norm=True, fmt=CF, order=0, n_cta=0):
    B, C, T = e.shape
    n_out = T if center else T - W + 1
    ei, es = _env_in(e, fmt)
    out, os_ = _spec(np.full((B, C, n_out, W), np.nan, np.float32), fmt)
    ic = np.array([B, C, T, W, int(center), int(norm)], np.int32)
    assert _lib().kb_emu_tempogram(_p(ic), _p(ei), _p(es), _p(out), _p(os_), order, n_cta) == n_out
    return out.transpose(0, 3, 1, 2) if fmt == CL else out


def emu_tempo(tg, logprior, bpm_scale, per_frame=False, fmt=CF, order=0, n_cta=0):
    B, C, T, W = tg.shape
    gi, gs = _spec(tg, fmt)
    ic = np.array([B, C, T, W, int(per_frame)], np.int32)
    lp = np.ascontiguousarray(logprior, np.float64)
    if per_frame:
        out, os_ = _rows(B, C, T, fmt)
    else:
        out, os_ = np.full((B, C), np.nan, np.float32), None
    assert _lib().kb_emu_tempo(_p(ic), _p(gi), _p(gs), _p(lp), bpm_scale, _p(out), _p(os_), order, n_cta) == 0
    return _canon_rows(out, fmt) if per_frame else out


def emu_peak(e, pre_max, post_max, pre_avg, post_avg, wait, delta=0.07, normalize=True, fmt=CF, order=0, n_cta=0):
    B, C, T = e.shape
    ei, es = _env_in(e, fmt)
    mask, ms = _rows(B, C, T, fmt, np.uint8, 7)
    ic = np.array([B, C, T, pre_max, post_max, pre_avg, post_avg, wait, int(normalize)], np.int32)
    assert _lib().kb_emu_peak(_p(ic), delta, _p(ei), _p(es), _p(mask), _p(ms), order, n_cta) == 0
    return _canon_rows(mask, fmt)


def emu_beat(e, bpm, sr=22050, hop=512, tightness=100.0, trim=True, fmt=CF, order=0, n_cta=0):
    """(tempo (B, C), mask (B, C, T), workspace (ls, cs, back) per row)."""
    B, C, T = e.shape
    ei, es = _env_in(e, fmt)
    mask, ms = _rows(B, C, T, fmt, np.uint8, 7)
    tempo = np.full((B, C), -1.0, np.float32)
    ic = np.array([B, C, T, int(trim)], np.int32)
    dc = np.array([sr / hop, tightness], np.float64)
    ws = np.zeros(B * C * 3 * T, np.float64)
    bp = None if np.isscalar(bpm) else np.ascontiguousarray(bpm, np.float32)
    bc = float(bpm) if np.isscalar(bpm) else 0.0
    assert _lib().kb_emu_beat(_p(ic), _p(dc), _p(bp), bc, _p(ei), _p(es), _p(tempo), _p(mask), _p(ms), _p(ws), order,
                              n_cta) == 0
    w = ws.reshape(B * C, 3 * T)
    ls, cs = w[:, :T], w[:, T:2 * T]
    back = w[:, 2 * T:].view(np.int32)[:, :T]
    return tempo, _canon_rows(mask, fmt).astype(bool), (ls, cs, back)


def _ulp_diff(a, b):
    a = np.asarray(a, np.float32)
    b = np.asarray(b, np.float32)
    ia = a.view(np.int32).astype(np.int64)
    ib = b.view(np.int32).astype(np.int64)
    return np.abs(ia - ib)


# ----------------------------------------------------------------------------------------------------- onset strength
@pytest.mark.parametrize('aggregate', ['mean', 'median'])
@pytest.mark.parametrize('K', [7, 8, 128, 1025])
@pytest.mark.parametrize('max_size,lag,pad', [(1, 1, 2), (3, 3, 0), ('K', 1, 0), (3, 1, 2)])
def test_onset_against_reference(aggregate, K, max_size, lag, pad):
    if K == 1025 and max_size == 'K' and aggregate == 'median':
        pytest.skip('covered at smaller K')
    m = K if max_size == 'K' else max_size
    rng = np.random.default_rng(K + m + lag)
    S = rng.standard_normal((2, 2, 23, K)).astype(np.float32) * 10
    S[0, 1, 5] = S[0, 1, 4]                         # ties and zeros of D
    got = emu_onset(S, lag, m, aggregate, pad)
    for b in range(2):
        for c in range(2):
            ref = R.onset_strength_row(S[b, c], lag, m, aggregate, pad)
            if aggregate == 'median':
                np.testing.assert_array_equal(got[b, c], ref)
            else:
                assert _ulp_diff(got[b, c], ref).max() <= 1


@pytest.mark.parametrize('aggregate', ['mean', 'median'])
def test_onset_invariance(aggregate):
    rng = np.random.default_rng(3)
    S = rng.standard_normal((3, 2, 70, 33)).astype(np.float32)
    ref = emu_onset(S, 2, 5, aggregate, 3)
    for fmt in (CF, CL):
        for order, n_cta in ((0, 0), (1, 0), (2, 0), (0, 3), (1, 5)):
            np.testing.assert_array_equal(emu_onset(S, 2, 5, aggregate, 3, fmt, order, n_cta), ref)
    np.testing.assert_array_equal(emu_onset(S[1:2], 2, 5, aggregate, 3), ref[1:2])
    big = np.zeros((3, 3, 80, 40), np.float32)
    big[:, ::2][:, :, 4:74, 3:36] = S
    view = big[:, ::2, 4:74, 3:36]
    xs = _strides(view, (0, 1, 2, 3))
    np.testing.assert_array_equal(emu_onset(S, 2, 5, aggregate, 3, xin=(big[:, ::2, 4:, 3:], xs)), ref)


def test_onset_tie_rules():
    # two equal maxima in a window: the gradient goes to the lower bin; the median of even K splits 0.5 / 0.5
    S = np.zeros((1, 1, 3, 4), np.float32)
    S[0, 0, 0] = [1, 3, 3, 0]
    S[0, 0, 1] = [5, 5, 5, 5]
    g = np.array([[[0, 1, 0]]], np.float32)
    gx = emu_onset_bwd(S, g, 1, 3, 'mean')
    # D[1] = 5 - R[0], R[0] = [3, 3, 3, 3] from bins 1, 1, 1, 2 (lowest tied bin)
    np.testing.assert_allclose(gx[0, 0, 0], [0, -0.75, -0.25, 0])
    np.testing.assert_allclose(gx[0, 0, 1], [0.25] * 4)
    S2 = np.zeros((1, 1, 2, 4), np.float32)
    S2[0, 0, 1] = [4, 1, 2, 3]
    gx = emu_onset_bwd(S2, np.array([[[0, 1]]], np.float32), 1, 1, 'median')
    np.testing.assert_allclose(gx[0, 0, 1], [0, 0, 0.5, 0.5])
    assert emu_onset(S2, 1, 1, 'median')[0, 0, 1] == np.float32(2.5)


@pytest.mark.parametrize('aggregate', ['mean', 'median'])
@pytest.mark.parametrize('K,m,lag,pad', [(9, 1, 1, 2), (8, 3, 2, 0), (6, 6, 1, 1)])
@pytest.mark.parametrize('fmt', [CF, CL])
def test_onset_gradient(aggregate, K, m, lag, pad, fmt):
    rng = np.random.default_rng(K * 7 + m)
    B, C, T = 2, 1, 12
    S = (rng.permutation(B * C * T * K).reshape(B, C, T, K) * 0.01 - 3).astype(np.float32)   # tie-free
    g = rng.standard_normal((B, C, T)).astype(np.float32)
    got = emu_onset_bwd(S, g, lag, m, aggregate, pad, fmt)
    for b in range(B):
        St = torch.tensor(S[b, 0], dtype=torch.float64, requires_grad=True)
        R.onset_strength_torch(St, lag, m, aggregate, pad).backward(torch.tensor(g[b, 0], dtype=torch.float64))
        np.testing.assert_allclose(got[b, 0], St.grad.numpy(), rtol=1e-6, atol=1e-6)
    np.testing.assert_array_equal(emu_onset_bwd(S, g, lag, m, aggregate, pad, fmt, order=2, n_cta=3), got)


def test_onset_nonfinite_isolation():
    rng = np.random.default_rng(5)
    S = rng.standard_normal((2, 2, 20, 16)).astype(np.float32)
    ref = emu_onset(S, 1, 3, 'median')
    S2 = S.copy()
    S2[1, 0, 7, 3] = np.nan
    S2[0, 1, 9, 2] = np.inf
    got = emu_onset(S2, 1, 3, 'median')
    np.testing.assert_array_equal(got[0, 0], ref[0, 0])
    np.testing.assert_array_equal(got[1, 1], ref[1, 1])
    assert np.isnan(got[1, 0, 7]) and np.isnan(got[1, 0, 8])


# ---------------------------------------------------------------------------------------------------------- tempogram
@pytest.mark.parametrize('W,center', [(2, True), (7, True), (64, True), (384, True), (33, False), (4096, True)])
@pytest.mark.parametrize('norm', [True, False])
def test_tempogram_against_reference(W, center, norm):
    rng = np.random.default_rng(W)
    T = 50 if W <= 384 else 9
    e = np.abs(rng.standard_normal((2, 1, T))).astype(np.float32)
    got = emu_tempogram(e, W, center, norm)
    for b in range(2):
        ref = R.tempogram_row(e[b, 0], W, center, norm)
        # |y_j y_{j+l}| summed is at most ||y||^2 <= max_l |ac[l]| (Cauchy-Schwarz, ac[0] = ||y||^2); the float32
        # window and products add 3 rounding errors per term, the chain W - 1, and the division one: relative to the
        # frame's maximum the error is below (W + 4) 2^-24 (plus the reference's FFT error)
        scale = 1.0 if norm else np.abs(ref).max(axis=1, keepdims=True)
        bound = (W + 4) * EPS32 * scale + 1e-12
        assert np.all(np.abs(got[b, 0] - ref) <= bound)


def test_tempogram_invariance():
    rng = np.random.default_rng(11)
    e = np.abs(rng.standard_normal((3, 2, 40))).astype(np.float32)
    ref = emu_tempogram(e, 24)
    for fmt in (CF, CL):
        for order, n_cta in ((1, 0), (2, 0), (0, 2)):
            np.testing.assert_array_equal(emu_tempogram(e, 24, fmt=fmt, order=order, n_cta=n_cta), ref)
    np.testing.assert_array_equal(emu_tempogram(e[2:], 24), ref[2:])


def test_tempogram_ramps_match_numpy():
    e = np.array([[[3.0, 1.0, 2.0, 5.0]]], np.float32)
    W = 8
    got = emu_tempogram(e, W, True, False)
    ref = R.tempogram_row(e[0, 0], W, True, False)
    np.testing.assert_allclose(got[0, 0], ref, rtol=1e-6, atol=1e-6)


# -------------------------------------------------------------------------------------------------------------- tempo
MARGIN = 1e-6


def _decided(scores):
    """True when the first maximum leads the runner-up by more than the relative margin."""
    s = np.sort(scores[np.isfinite(scores)])
    return s.size < 2 or s[-1] - s[-2] > MARGIN * max(1.0, abs(s[-1]))


@pytest.mark.parametrize('per_frame', [False, True])
def test_tempo_decisions(per_frame):
    sr, hop, W = 22050, 512, 344
    bpm, lp = R.tempo_prior(W, sr, hop)
    rng = np.random.default_rng(2)
    e = np.abs(rng.standard_normal((3, 2, 60))).astype(np.float32)
    e[:, :, ::21] += 3
    tg = emu_tempogram(e, W)
    got = emu_tempo(tg, lp, 60.0 * sr / hop, per_frame)
    checked = 0
    for b in range(3):
        for c in range(2):
            rows = tg[b, c].astype(np.float64)
            ref = R.tempo_row(rows, lp, bpm, per_frame)
            if per_frame:
                for t in range(rows.shape[0]):
                    if _decided(R.tempo_scores(rows[t], lp)):
                        assert got[b, c, t] == np.float32(ref[t])
                        checked += 1
            elif _decided(R.tempo_scores(rows.mean(axis=0), lp)):
                assert got[b, c] == np.float32(ref)
                checked += 1
    assert checked > 0
    for fmt in (CF, CL):
        np.testing.assert_array_equal(emu_tempo(tg, lp, 60.0 * sr / hop, per_frame, fmt, 2, 3), got)


def test_tempo_from_default_tempogram():
    # the default 384-lag tempogram, decided with its own lag count
    sr, hop, W = 22050, 512, 384
    bpm, lp = R.tempo_prior(W, sr, hop)
    rng = np.random.default_rng(12)
    e = np.abs(rng.standard_normal((2, 1, 80))).astype(np.float32)
    e[:, :, ::22] += 3
    tg = emu_tempogram(e, W)
    got = emu_tempo(tg, lp, 60.0 * sr / hop)
    checked = 0
    for b in range(2):
        if _decided(R.tempo_scores(tg[b, 0].astype(np.float64).mean(axis=0), lp)):
            assert got[b, 0] == np.float32(R.tempo_row(tg[b, 0], lp, bpm))
            checked += 1
    assert checked > 0


def test_tempo_skips_nan_scores():
    # g < -1e-6 makes log1p NaN: those lags are skipped (np.nanargmax), lag 0 included; all NaN gives NaN
    W = 40
    bpm, lp = R.tempo_prior(W, 22050, 512)
    rng = np.random.default_rng(13)
    tg = rng.random((1, 3, 6, W)).astype(np.float32)
    tg[0, 0, :, :10] = -0.5
    tg[0, 0, :, 0] = -0.5
    tg[0, 1, :, 25] = -0.25
    tg[0, 2] = -1.0
    for per_frame in (False, True):
        got = emu_tempo(tg, lp, 60.0 * 22050 / 512, per_frame)
        for c in range(3):
            ref = R.tempo_row(tg[0, c], lp, bpm, per_frame)
            np.testing.assert_array_equal(got[0, c], np.float32(ref))
    assert np.isnan(emu_tempo(tg, lp, 60.0 * 22050 / 512)[0, 2])


def test_tempo_nonfinite_rows():
    bpm, lp = R.tempo_prior(16, 22050, 512)
    tg = np.random.default_rng(1).random((1, 2, 5, 16)).astype(np.float32)
    ref = emu_tempo(tg, lp, 60.0 * 22050 / 512)
    tg[0, 1, 2, 3] = np.inf
    got = emu_tempo(tg, lp, 60.0 * 22050 / 512)
    assert got[0, 0] == ref[0, 0] and np.isnan(got[0, 1])
    pf = emu_tempo(tg, lp, 60.0 * 22050 / 512, per_frame=True)
    assert np.isnan(pf[0, 1, 2]) and np.isfinite(pf[0, 1, [0, 1, 3, 4]]).all()


# ------------------------------------------------------------------------------------------------------- peak picking
@pytest.mark.parametrize('normalize', [True, False])
@pytest.mark.parametrize('params', [R.detect_defaults(22050, 512), dict(pre_max=3, post_max=2, pre_avg=0, post_avg=1,
                                                                          wait=0)])
def test_peak_pick(normalize, params):
    rng = np.random.default_rng(4)
    e = np.abs(rng.standard_normal((2, 2, 300))).astype(np.float32)
    e[:, :, ::17] += 4
    got = emu_peak(e, delta=0.07, normalize=normalize, **params)
    for b in range(2):
        for c in range(2):
            ref, margin = R.peak_pick_row(e[b, c], delta=0.07, normalize=normalize, return_scores=True, **params)
            assert np.abs(margin).min() > MARGIN     # no candidate decided by rounding
            np.testing.assert_array_equal(got[b, c].astype(bool), ref)
    for fmt in (CF, CL):
        np.testing.assert_array_equal(emu_peak(e, delta=0.07, normalize=normalize, fmt=fmt, order=1, n_cta=3,
                                               **params), got)


def test_peak_pick_empty_rows():
    e = np.zeros((1, 3, 50), np.float32)
    e[0, 1, 10] = 1
    e[0, 2, 10] = 1
    e[0, 2, 20] = np.nan
    got = emu_peak(e, 1, 1, 2, 3, 1)
    assert not got[0, 0].any() and got[0, 1, 10] and not got[0, 2].any()


# ------------------------------------------------------------------------------------------------------ beat tracking
def _clicks(T, per, rng, noise=0.05):
    e = noise * np.abs(rng.standard_normal(T))
    e[3::per] += 1.0
    return e.astype(np.float32)


@pytest.mark.parametrize('p', [1, 2, 7, 22, 31, 4096])
def test_beat_dp_block_parallel_equals_serial(p):
    rng = np.random.default_rng(p)
    T = 9000 if p == 4096 else 400
    e = _clicks(T, max(p, 2), rng)[None, None]
    bpm = 60.0 * (22050 / 512) / p
    tempo, mask, (ls, cs, back) = emu_beat(e, bpm)
    cs_ref, back_ref = R.beat_dp(ls[0], p)
    np.testing.assert_array_equal(cs[0], cs_ref)
    np.testing.assert_array_equal(back[0], back_ref)
    np.testing.assert_allclose(ls[0], R.local_score(e[0, 0], p), rtol=1e-12, atol=1e-12)
    np.testing.assert_array_equal(np.nonzero(mask[0, 0])[0], R.beats_from(ls[0], cs[0], back_ref))
    assert tempo[0, 0] == np.float32(bpm)


@pytest.mark.parametrize('trim', [True, False])
def test_beat_against_reference(trim):
    rng = np.random.default_rng(8)
    e = np.stack([_clicks(500, 21, rng), _clicks(500, 29, rng, 0.3)])[None]
    bpms = np.array([[60 * 22050 / 512 / 21, 60 * 22050 / 512 / 29]], np.float32)
    tempo, mask, _ = emu_beat(e, bpms, trim=trim)
    for c in range(2):
        t, beats = R.beat_track_row(e[0, c], float(bpms[0, c]), 22050, 512, trim=trim)
        np.testing.assert_array_equal(np.nonzero(mask[0, c])[0], beats)
        assert tempo[0, c] == np.float32(t)
        assert beats.size > 5
    for fmt in (CF, CL):
        t2, m2, _ = emu_beat(e, bpms, trim=trim, fmt=fmt, order=1, n_cta=1)
        np.testing.assert_array_equal(m2, mask)
        np.testing.assert_array_equal(t2, tempo)


def test_beat_negative_envelope():
    # every local score negative: no frame reaches 0.01 max, so i0 = T and every backlink is -1
    rng = np.random.default_rng(14)
    e = -(1.0 + _clicks(400, 21, rng))[None, None]
    bpm = 60.0 * (22050 / 512) / 21
    tempo, mask, (ls, cs, back) = emu_beat(e, bpm)
    assert (ls[0] < 0).all() and (back[0] == -1).all()
    cs_ref, back_ref = R.beat_dp(ls[0], 21)
    np.testing.assert_array_equal(cs[0], cs_ref)
    np.testing.assert_array_equal(back[0], back_ref)
    _, beats = R.beat_track_row(e[0, 0], bpm, 22050, 512)
    np.testing.assert_array_equal(np.nonzero(mask[0, 0])[0], beats)
    # a detrended-looking envelope with both signs
    e2 = (_clicks(400, 21, rng) - 0.3)[None, None]
    tempo, mask, (ls, cs, back) = emu_beat(e2, bpm)
    np.testing.assert_array_equal(back[0], R.beat_dp(ls[0], 21)[1])
    np.testing.assert_array_equal(np.nonzero(mask[0, 0])[0], R.beat_track_row(e2[0, 0], bpm, 22050, 512)[1])


def test_beat_special_rows():
    rng = np.random.default_rng(9)
    e = np.stack([_clicks(300, 20, rng), np.zeros(300, np.float32), _clicks(300, 20, rng)])[None]
    e[0, 2, 50] = np.nan
    tempo, mask, _ = emu_beat(e, 120.0)
    assert tempo[0, 0] == np.float32(120.0) and mask[0, 0].any()
    assert tempo[0, 1] == 0 and not mask[0, 1].any()
    assert np.isnan(tempo[0, 2]) and not mask[0, 2].any()
    t1, m1, _ = emu_beat(e[:, :1], 120.0)
    np.testing.assert_array_equal(m1[0, 0], mask[0, 0])


# --------------------------------------------------------------------------------------------------------- validation
def test_validation():
    from kapre_b200 import ops, signal
    with pytest.raises(ValueError):
        ops.onset_config(lag=0)
    with pytest.raises(ValueError):
        ops.onset_config(max_size=0)
    with pytest.raises(ValueError):
        ops.onset_config(aggregate='max')
    with pytest.raises(ValueError):
        ops.tempogram_check(1)
    with pytest.raises(ValueError):
        ops.tempogram_check(4097)
    with pytest.raises(ValueError):
        ops.tempogram_check(10, frames=5, center=False)
    with pytest.raises(ValueError):
        ops.onset_detect_config(1, 0, 1, 1, 1, 0.07, True)
    with pytest.raises(ValueError):
        ops.onset_detect_config(-1, 1, 1, 1, 1, 0.07, True)
    with pytest.raises(ValueError):
        ops.beat_config(22050, 512, 0.0, True)
    with pytest.raises(ValueError):
        signal._tempo_plan(22050, 512, 8.0, -1.0, 1.0, 320.0)
    with pytest.raises(ValueError):
        signal._tempo_plan(22050, 512, 8.0, 120.0, 0.0, 320.0)
    with pytest.raises(ValueError):
        signal._tempo_plan(22050, 512, 200.0, 120.0, 1.0, 320.0)      # W > 4096
    with pytest.raises(ValueError):
        signal.tempo(onset_envelope=object(), aggregate='median')
    with pytest.raises(ValueError):
        signal.beat_track(onset_envelope=object(), bpm=0.5)              # p > 4096
    with pytest.raises(ValueError):
        signal.beat_track(onset_envelope=object(), tightness=-1.0)
    with pytest.raises(ValueError):
        signal.onset_strength(waveform=None, S=None)
    with pytest.raises(ValueError):
        signal.tempogram(onset_envelope=object(), norm=2)
    with pytest.raises(ValueError):
        ops.onset_detect_config(1, 1, 1, 1, (1 << 30) + 1, 0.07, True)
    with pytest.raises(ValueError):
        ops.onset_detect_config(1, 1 << 31, 1, 1, 1, 0.07, True)
    wave = torch.zeros((1, 22050, 1))
    with pytest.raises(ValueError):
        signal.onset_strength(wave, hop_length=0)                       # ValueError, not ZeroDivisionError
    with pytest.raises(ValueError):
        signal.onset_strength(S=torch.zeros((1, 4, 8, 1)), n_fft=1)      # n_fft checked with S too
    with pytest.raises(ValueError):
        signal.onset_strength(wave, max_size=129)                        # > n_mels, before any launch
    with pytest.raises(ValueError):
        signal.onset_strength(torch.zeros((1, 512, 1)), lag=2)          # 2 frames: lag must be below them
    with pytest.raises(ValueError):
        signal.tempo(tg=torch.zeros((1, 5, 1, 1)))                       # a given tg of 1 lag
    plan = signal._tempo_plan(22050, 512, 8.0, 120.0, 1.0, 320.0, win_length=384)
    assert plan.W == 384


def test_layers_config_roundtrip():
    from kapre_b200 import time_frequency as tf
    layer = tf.OnsetStrength(sample_rate=16000, lag=2, max_size=3, aggregate='median', n_mels=64, data_format=CF)
    cfg = layer.get_config()
    assert cfg['lag'] == 2 and cfg['aggregate'] == 'median' and cfg['data_format'] == CF
    tg = tf.Tempogram(win_length=200, hop_length=256)
    assert tg.get_config()['win_length'] == 200
    with pytest.raises(ValueError):
        tf.OnsetStrength(aggregate='max')
    with pytest.raises(ValueError):
        tf.Tempogram(win_length=1)
    with pytest.raises(ValueError):
        tf.OnsetStrength(max_size=65, n_mels=64)
