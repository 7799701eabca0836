"""YIN / pYIN on the CPU: the kernel bodies of pitch_core.cuh (run by a CPU emulation) against the float64
restatement (pitch_ref.py): the CMNDF within its derived bound, the decisions against the float64 rule applied to the
kernel's own CMNDF, the pYIN observations, the Viterbi path's score, bit-independence of the batch position, the
grid and the layout, tonal / vibrato / silence / noise anchors, the host tables, validation and non-finite input."""
import ctypes
import hashlib
import os
import subprocess
import tempfile

import numpy as np
import pytest

import pitch_ref as R
from emu_harness import Checked
from kapre_b200 import backend, ops

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, 'emu', 'kb_emu_pitch.cpp')
_CSRC = os.path.join(_HERE, '..', 'kapre_b200', 'csrc')
_lib_handle = None
CL, CF = 'channels_last', 'channels_first'


def _lib():
    """tests/emu/kb_emu_pitch.cpp built with g++ into the temporary directory (keyed by the sources' contents)."""
    global _lib_handle
    if _lib_handle is None:
        hs = hashlib.sha256()
        for f in [_SRC] + sorted(os.path.join(_CSRC, n) for n in os.listdir(_CSRC) if n.endswith(('.h', '.cuh'))):
            with open(f, 'rb') as fh:
                hs.update(fh.read())
        out = os.path.join(tempfile.gettempdir(), 'kapre_b200_emu_pitch_%s.so' % hs.hexdigest()[:16])
        if not os.path.exists(out):
            tmp = '%s.%d.tmp' % (out, os.getpid())
            subprocess.check_call(['g++', '-O2', '-std=c++17', '-shared', '-fPIC', '-DKB_HOST_EMU', '-Wno-unknown-pragmas',
                                   '-o', tmp, _SRC])
            os.replace(tmp, out)
        lib = ctypes.CDLL(out)
        lib.kb_emu_pitch.argtypes = [ctypes.c_void_p, ctypes.c_float, ctypes.c_double] + [ctypes.c_void_p] * 11 + \
            [ctypes.c_int, ctypes.c_int]
        _lib_handle = Checked(lib)
    return _lib_handle


def _p(a):
    return None if a is None else ctypes.c_void_p(a.__array_interface__['data'][0])


def _ic(plan):
    g = plan.geometry
    q = plan.pyin or {}
    return np.array([g['frame_length'], g['win_length'], g['hop_length'], int(g['center']), g['min_period'],
                     g['max_period'], int(plan.pyin is not None), q.get('n_thresholds', 0), q.get('n_pitch', 0)],
                    np.int32)


def plan_of(sr=8000, fmin=100.0, fmax=1000.0, F=256, W=None, h=None, center=True, thresh=0.1, pyin=None, **kw):
    q = None if pyin is None else dict(pyin, **kw)
    return ops.PitchPlan(sr, fmin, fmax, F, W, h, center, thresh, q)


def tiling(plan):
    out = np.zeros(8, np.int32)
    assert _lib().kb_emu_pitch_tiling(_p(_ic(plan)), _p(out)) == 0
    return dict(zip(['share', 'G', 'KB', 'TF', 'NSEG', 'SPAN', 'smem'], out.tolist()))


def emu_pitch(x, plan, fmt, order=0, n_cta=0, cmndf=True, view=None):
    """The difference-function body on x ((B, L, C) channels_last or (B, C, L)): (out (B, C, M), CMNDF (B, C, M, n),
    candidates (counts, bins, probabilities per (row, frame)))."""
    xv = x if view is None else view
    B, L, C = xv.shape if fmt == CL else (xv.shape[0], xv.shape[2], xv.shape[1])
    M = plan.num_frames(L)
    st = [s // 4 for s in xv.strides]
    xs = np.array([st[0], st[2], st[1]] if fmt == CL else st, np.int64)
    out = np.full((B, C, M), -7.0, np.float32)
    os_ = np.array([s // 4 for s in out.strides], np.int64)
    cm = np.full((B, C, M, plan.n_lags), -7.0, np.float32) if cmndf else None
    cs = np.array([s // 4 for s in cm.strides], np.int64) if cmndf else None
    g = plan.geometry
    cmax = (g['n_lags'] + 1) // 2
    tabs, keep = None, []
    cn = cb = cp = None
    if plan.pyin is not None:
        t = plan._tables
        keep = [np.ascontiguousarray(t[k]) for k in ('beta_probs', 'boltzmann_pow', 'boltzmann_norm',
                                                     'no_trough_bonus', 'period_edges')]
        tabs = (ctypes.c_void_p * 5)(*[a.ctypes.data for a in keep])
        cn = np.full(B * C * M, -1, np.int32)
        cb = np.zeros(B * C * M * cmax, np.uint16)
        cp = np.zeros(B * C * M * cmax, np.float32)
    dims = np.array([B, C, L, M], np.int32)
    base = xv.__array_interface__['data'][0]
    rc = _lib().kb_emu_pitch(_p(_ic(plan)), g['sample_rate'], float(plan.cfg.trough_threshold), _p(dims),
                             ctypes.c_void_p(base), _p(xs), _p(out), _p(os_), _p(cm), _p(cs), tabs, _p(cn), _p(cb),
                             _p(cp), order, n_cta)
    assert rc == 0
    return out, cm, (cn, cb.reshape(-1, cmax) if cb is not None else None, cp.reshape(-1, cmax) if cp is not None
                     else None)


def emu_viterbi(plan, cands, vp, order=0, n_cta=0, nt=None):
    """The Viterbi body on the candidates and voiced probabilities (B, C, M) of emu_pitch: (f0, flag, vp)."""
    q, t = plan.pyin, plan._tables
    B, C, M = vp.shape
    vp = np.ascontiguousarray(vp, np.float32).copy()
    f0 = np.full_like(vp, -7.0)
    flag = np.full(vp.shape, 7, np.uint8)
    os_ = np.array([s // 4 for s in vp.strides], np.int64)
    cn, cb, cp = cands
    cmax = cb.shape[1]
    vi = np.array([q['n_pitch'], q['band_width'], M, C, B * C, cmax], np.int32)
    cfg = plan.cfg
    vf = np.array([cfg.log_stay, cfg.log_switch, cfg.log_init_voiced, cfg.log_init_unvoiced, cfg.fill_na], np.float32)
    keep = [np.ascontiguousarray(t[k]) for k in ('log_triangle', 'log_row_norm', 'freqs')]
    tabs = (ctypes.c_void_p * 3)(*[a.ctypes.data for a in keep])
    bp = np.zeros(B * C * M * 2 * q['n_pitch'], np.uint16)
    nt = nt or min(1024, (q['n_pitch'] + 31) // 32 * 32)
    assert _lib().kb_emu_viterbi(_p(vi), _p(vf), tabs, _p(np.ascontiguousarray(cn)), _p(np.ascontiguousarray(cb)),
                                 _p(np.ascontiguousarray(cp)), _p(vp), _p(f0), _p(flag), _p(os_), _p(bp), nt, order,
                                 n_cta) == 0
    return f0, flag.astype(bool), vp


def emu_pyin(x, plan, fmt=CF, **kw):
    vp, cm, cands = emu_pitch(x, plan, fmt, **kw)
    f0, flag, vp2 = emu_viterbi(plan, cands, vp)
    return f0, flag, vp2, cm, cands, vp


def _tone(f0, sr, L, harmonics=4, rng=None, noise=0.0, amp=0.5):
    t = np.arange(L) / sr
    f0 = np.broadcast_to(np.asarray(f0, np.float64), (L,)) if np.ndim(f0) else np.full(L, float(f0))
    ph = 2 * np.pi * np.cumsum(f0) / sr
    x = sum(amp / k * np.sin(k * ph + 0.3 * k) for k in range(1, harmonics + 1))
    if noise:
        x = x + noise * rng.standard_normal(L)
    return x.astype(np.float32)


def _batch(rng, B, C, L, sr):
    x = np.empty((B, C, L), np.float32)
    for b in range(B):
        for c in range(C):
            x[b, c] = _tone(rng.uniform(120, 700), sr, L, rng=rng, noise=0.05 * rng.uniform(), amp=rng.uniform(0.05, 1))
    return x


# ---------------------------------------------------------------------------------------------------- the CMNDF
@pytest.mark.parametrize('F,W,h,center', [
    (256, 128, 64, True),      # hop divides W: segments of gcd = 64 shared by two frames
    (256, 128, 64, False),
    (256, 128, 48, True),      # gcd 16: one segment per frame
    (256, 100, 60, False),     # gcd 20, hop not dividing W
    (300, 96, 200, True),      # hop above the window
])
@pytest.mark.parametrize('fmt', [CL, CF])
def test_cmndf_within_bound(F, W, h, center, fmt):
    rng = np.random.default_rng(F + W + h)
    plan = plan_of(F=F, W=W, h=h, center=center)
    x = _batch(rng, 2, 3, 1500, 8000)
    if fmt == CL:
        big = np.zeros((2, 1500, 7), np.float32)      # odd channel stride
        big[:, :, 1:7:2] = x.transpose(0, 2, 1)
        view = big[:, :, 1:7:2]
    else:
        big = np.zeros((2, 3, 1500 * 3), np.float32)  # odd sample stride
        big[:, :, ::3] = x
        view = big[:, :, ::3]
    _, cm, _ = emu_pitch(big, plan, fmt, view=view)
    g = plan.geometry
    for b in range(2):
        for c in range(3):
            ref, bound = R.cmndf_bound(x[b, c], g)
            err = np.abs(cm[b, c].astype(np.float64) - ref)
            assert cm.shape[2] == ref.shape[0]
            assert (err <= bound).all(), (b, c, float((err - bound).max()))


def test_sharing_is_used_where_it_pays():
    assert tiling(plan_of(F=256, W=128, h=64))['share'] == 1
    assert tiling(plan_of(F=256, W=128, h=48))['share'] == 0
    t = tiling(ops.PitchPlan(22050, 65.40639, 2093.0047))
    assert t['share'] == 1 and t['G'] == 512 and t['TF'] >= 2


def test_smallest_lag_range():
    # min_period = floor(sr / fmax), max_period = F - W - 1 = min_period + 2: three lags
    plan = ops.PitchPlan(8000, 2000.0, 4000.0, 9, 4, 2, True)
    assert plan.n_lags == 3
    rng = np.random.default_rng(1)
    x = rng.standard_normal((1, 1, 100)).astype(np.float32)
    out, cm, _ = emu_pitch(x, plan, CF)
    ref, bound = R.cmndf_bound(x[0, 0], plan.geometry)
    assert (np.abs(cm[0, 0] - ref) <= bound).all()
    for m in range(out.shape[2]):
        k, f0 = R.yin_decide(cm[0, 0, m], plan.geometry, 0.1, 8000)
        np.testing.assert_allclose(out[0, 0, m], f0, rtol=1e-6)


# ------------------------------------------------------------------------------------------------ decisions
@pytest.mark.parametrize('h', [64, 48])
def test_yin_decisions_match_float64_rule_on_kernel_cmndf(h):
    rng = np.random.default_rng(h)
    plan = plan_of(F=256, h=h, thresh=0.15)
    x = _batch(rng, 3, 2, 2000, 8000)
    x[1, 0] = rng.standard_normal(2000).astype(np.float32)       # noise: many frames fall back to the argmin
    out, cm, _ = emu_pitch(x, plan, CF)
    g = plan.geometry
    n_fallback = 0
    for b, c, m in np.ndindex(out.shape):
        row = cm[b, c, m].astype(np.float64)
        k, f0 = R.yin_decide(row, g, 0.15, 8000)
        n_fallback += not (R.is_trough(row) & (row < 0.15)).any()
        np.testing.assert_allclose(out[b, c, m], f0, rtol=1e-6)
        assert abs(8000 / out[b, c, m] - g['min_period'] - k) < 1.0
    assert n_fallback > 0


def test_pyin_observations_match_float64_on_kernel_cmndf():
    rng = np.random.default_rng(3)
    plan = plan_of(F=256, pyin={})
    x = _batch(rng, 2, 2, 2000, 8000)
    x[0, 1] = 0.3 * rng.standard_normal(2000).astype(np.float32)
    vp, cm, (cn, cb, cp) = emu_pitch(x, plan, CF)
    g, q, t = plan.geometry, plan.pyin, plan._tables
    M = vp.shape[2]
    edges = t['period_edges']
    for b, c, m in np.ndindex(vp.shape):
        obs, vref, per = R.pyin_observe(cm[b, c, m].astype(np.float64), g, q, t)
        fi = (b * 2 + c) * M + m
        got = {int(cb[fi, e]): float(cp[fi, e]) for e in range(cn[fi])}
        assert cn[fi] == len(got)
        # bins agree except for a refined period within 1e-5 of a bin edge (float32 shift against float64)
        near = any(np.min(np.abs(R.refined_period(cm[b, c, m].astype(np.float64), k, g['min_period']) / edges - 1))
                   < 1e-5 for k, _ in per)
        if not near:
            assert sorted(got) == sorted(obs), (b, c, m)
            for k in obs:
                np.testing.assert_allclose(got[k], obs[k], rtol=1e-4, atol=1e-7)
        np.testing.assert_allclose(vp[b, c, m], vref, rtol=1e-4, atol=1e-6)
        assert len(got) <= (g['n_lags'] + 1) // 2


def _decode_reference(plan, obs_list, vps):
    q, t = plan.pyin, plan._tables
    A, band = R.transition(q, t)
    lobs = R.log_obs(obs_list, vps, q)
    path, best = R.viterbi(lobs, A, band)
    return lobs, R.log_transition(A, band), path, best


def _state_path(plan, f0, flag):
    """Decoded states from (f0, voiced_flag): voiced bins from f0, unvoiced ones unknown (-1)."""
    B = 12 * plan.pyin['bins_per_semitone']
    fmin = plan.geometry['fmin']
    return np.where(flag, np.round(B * np.log2(np.where(flag, f0, fmin) / fmin)).astype(np.int64), -1)


def test_viterbi_path_score_within_bound_of_optimum():
    rng = np.random.default_rng(4)
    plan = plan_of(F=256, pyin={})
    x = np.concatenate([_tone(np.linspace(150, 600, 4000), 8000, 4000, rng=rng, noise=0.2),
                        0.2 * rng.standard_normal(2000).astype(np.float32)])[None, None]
    f0, flag, vp, cm, (cn, cb, cp), _ = emu_pyin(x, plan)
    M = vp.shape[2]
    obs = [{int(cb[m, e]): float(cp[m, e]) for e in range(cn[m])} for m in range(M)]
    lobs, la, path, best = _decode_reference(plan, obs, vp[0, 0].astype(np.float64))
    # the kernel's path: its voiced states are known from f0; recover the unvoiced ones from the reference's optimum
    # restricted to the kernel's voicing, so the score compared is a lower bound of the kernel path's own score
    n = plan.pyin['n_pitch']
    sp = _state_path(plan, f0[0, 0], flag[0, 0])
    q, t = plan.pyin, plan._tables
    A, band = R.transition(q, t)
    mask = np.full(lobs.shape, -np.inf)
    for m in range(M):
        if sp[m] >= 0:
            mask[m, sp[m]] = 0.0
        else:
            mask[m, n:] = 0.0
    kpath, kscore = R.viterbi(lobs + mask, A, band)
    kscore = R.path_score(kpath, lobs, la, np.log(np.concatenate([np.zeros(n), np.full(n, 1.0 / n)]) + R.TINY))
    assert kscore >= best - R.path_bound(M, lobs, la), (kscore, best)
    assert flag[0, 0, :M // 2].mean() > 0.8 and flag[0, 0, -4:].mean() < 0.5


# -------------------------------------------------------------------------------------------------- anchors
@pytest.mark.parametrize('f0', [110.0, 220.0, 440.0, 830.0])
def test_harmonic_tone_anchors(f0):
    sr = 8000
    plan = plan_of(F=256, thresh=0.1)
    x = _tone(f0, sr, 4000)[None, None]
    out, _, _ = emu_pitch(x, plan, CF)
    inner = out[0, 0, 2:-2]
    assert np.all(np.abs(inner / f0 - 1) < 0.005), inner
    pplan = plan_of(F=256, pyin={})
    pf0, flag, vp, cm, cands, _ = emu_pyin(x, pplan)
    B = 12 * pplan.pyin['bins_per_semitone']
    assert flag[0, 0, 2:-2].all()
    assert np.all(np.abs(B * np.log2(pf0[0, 0, 2:-2] / f0)) <= 1.0 + 1e-6)
    # on a clean tone the decoded path is the float64 reference's path
    M = vp.shape[2]
    cn, cb, cp = cands
    obs = [{int(cb[m, e]): float(cp[m, e]) for e in range(cn[m])} for m in range(M)]
    _, _, path, _ = _decode_reference(pplan, obs, vp[0, 0].astype(np.float64))
    n = pplan.pyin['n_pitch']
    np.testing.assert_array_equal(flag[0, 0], path < n)
    np.testing.assert_array_equal(_state_path(pplan, pf0[0, 0], flag[0, 0])[path < n], path[path < n])


def test_vibrato_is_tracked():
    sr = 8000
    t = np.arange(8000) / sr
    f = 300 * 2 ** (0.5 / 12 * np.sin(2 * np.pi * 5 * t))
    x = _tone(f, sr, 8000)[None, None]
    plan = plan_of(F=256, pyin={})
    f0, flag, vp, _, _, _ = emu_pyin(x, plan)
    h = plan.geometry['hop_length']
    m = np.arange(f0.shape[2])
    truth = 300 * 2 ** (0.5 / 12 * np.sin(2 * np.pi * 5 * m * h / sr))
    inner = slice(3, -3)
    assert flag[0, 0, inner].all()
    assert np.abs(12 * np.log2(f0[0, 0, inner] / truth[inner])).max() < 0.25
    yplan = plan_of(F=256)
    y, _, _ = emu_pitch(x, yplan, CF)
    assert np.abs(y[0, 0, inner] / truth[inner] - 1).max() < 0.02


def test_silence_is_unvoiced_and_noise_mostly_unvoiced():
    rng = np.random.default_rng(5)
    plan = plan_of(F=256, pyin={})
    x = np.stack([np.zeros(4000, np.float32), rng.standard_normal(4000).astype(np.float32)])[:, None]
    f0, flag, vp, _, _, _ = emu_pyin(x, plan)
    assert not flag[0].any() and np.isnan(f0[0]).all()
    assert flag[1].mean() < 0.3


def test_non_finite_input_stays_local():
    rng = np.random.default_rng(6)
    x = _batch(rng, 2, 2, 3000, 8000)
    y = x.copy()
    y[0, 1, 1500] = np.nan
    y[1, 0, 10] = np.inf
    plan = plan_of(F=256)
    a, _, _ = emu_pitch(x, plan, CF)
    b_, _, _ = emu_pitch(y, plan, CF)
    g = plan.geometry
    for (bi, ci, s) in [(0, 1, 1500), (1, 0, 10)]:
        start = np.arange(a.shape[2]) * g['hop_length'] - g['pad']
        hit = (start <= s) & (s < start + g['frame_length'])
        assert np.isnan(b_[bi, ci, hit]).all() and not np.isnan(b_[bi, ci, ~hit]).any()
        np.testing.assert_array_equal(b_[bi, ci, ~hit], a[bi, ci, ~hit])
    np.testing.assert_array_equal(b_[0, 0], a[0, 0])
    np.testing.assert_array_equal(b_[1, 1], a[1, 1])
    pplan = plan_of(F=256, pyin={})
    fa, la, va, _, _, _ = emu_pyin(x, pplan)
    fb, lb, vb, _, _, _ = emu_pyin(y, pplan)
    for bi, ci in [(0, 1), (1, 0)]:
        assert np.isnan(fb[bi, ci]).all() and not lb[bi, ci].any() and np.isnan(vb[bi, ci]).all()
    for bi, ci in [(0, 0), (1, 1)]:
        np.testing.assert_array_equal(fb[bi, ci], fa[bi, ci])
        np.testing.assert_array_equal(vb[bi, ci], va[bi, ci])


# ------------------------------------------------------------------------------------------ bit-independence
@pytest.mark.parametrize('h', [64, 48])
def test_bits_independent_of_batch_position_grid_and_layout(h):
    rng = np.random.default_rng(7 + h)
    x = _batch(rng, 3, 2, 2500, 8000)
    plan = plan_of(F=256, h=h, pyin={})
    ref = emu_pyin(x, plan, CF)
    assert tiling(plan)['TF'] < ref[2].shape[2]          # several tiles per row
    variants = [emu_pyin(x[::-1].copy(), plan, CF), emu_pyin(x, plan, CF, order=1), emu_pyin(x, plan, CF, order=2),
                emu_pyin(x, plan, CF, n_cta=3), emu_pyin(np.ascontiguousarray(x.transpose(0, 2, 1)), plan, CL)]
    for i, v in enumerate(variants):
        for a, b in zip(ref[:4], v[:4]):
            bb = b[::-1] if i == 0 else b
            np.testing.assert_array_equal(a, bb)
    # the Viterbi: few CTAs walking the rows, descending order, fewer threads than bins
    vp, _, cands = emu_pitch(x, plan, CF)
    base = emu_viterbi(plan, cands, vp)
    for kw in (dict(n_cta=2), dict(order=1), dict(nt=128)):
        for a, b in zip(base, emu_viterbi(plan, cands, vp, **kw)):
            np.testing.assert_array_equal(a, b)


# ---------------------------------------------------------------------------------------------- host tables
def test_beta_cdf_against_scipy():
    from scipy.stats import beta
    x = np.linspace(0, 1, 201)
    for a, b in [(2, 18), (1, 1), (0.5, 3.0), (7.5, 2.25)]:
        np.testing.assert_allclose(backend.beta_cdf(x, a, b), beta.cdf(x, a, b), rtol=1e-12, atol=1e-14)


def test_transition_band_against_dense_build():
    plan = plan_of(sr=22050, fmin=65.0, fmax=1000.0, F=2048, pyin={})
    q, t = plan.pyin, plan._tables
    A, band = R.transition(q, t)
    n, w = q['n_pitch'], q['band_width']
    assert w == 101
    for i in (0, 3, n // 2, n - 1):
        for j in range(n):
            qq = j - i + w // 2
            if 0 <= qq < w:
                want = np.log(A[i, j] / (1 - q['switch_prob']))
                np.testing.assert_allclose(t['log_triangle'][qq] + t['log_row_norm'][i], want, rtol=1e-12)
            else:
                assert not band[i, j]
    from scipy.signal.windows import triang
    for w in (1, 2, 7, 10, 101):
        np.testing.assert_allclose(backend.triangle_window(w), triang(w), rtol=0, atol=1e-15)


# ----------------------------------------------------------------------------------------------- validation
@pytest.mark.parametrize('kw', [
    dict(fmin=0.0), dict(fmin=-5.0), dict(fmin=500.0, fmax=500.0), dict(fmin=600.0, fmax=500.0), dict(fmax=4500.0),
    dict(W=256), dict(W=300), dict(fmax=4000.0, sr=3000), dict(F=16384, W=8192), dict(F=16, W=8, fmin=3000.0, fmax=4000.0),
])
def test_value_errors(kw):
    kw = dict(kw)
    sr = kw.pop('sr', 8000)
    with pytest.raises(ValueError):
        plan_of(sr=sr, **kw)


def test_pyin_value_errors():
    with pytest.raises(ValueError):      # 2 n_pitch states over uint16 (and the bin limit)
        plan_of(sr=48000, fmin=30.0, fmax=20000.0, F=4096, pyin=dict(resolution=0.01))
    with pytest.raises(ValueError):
        plan_of(F=256, pyin=dict(n_thresholds=5000))
    with pytest.raises(ValueError):
        plan_of(F=256, pyin=dict(switch_prob=1.5))
    with pytest.raises(ValueError):
        plan_of(F=256, pyin=dict(resolution=0.0))


def test_largest_frame_fits():
    plan = ops.PitchPlan(48000, 30.0, 2000.0, 8192)
    t = tiling(plan)
    assert t['smem'] <= 220 * 1024 and t['TF'] >= 1
    plan = ops.PitchPlan(48000, 5.9, 2000.0, 8192, 64, 4096)
    assert tiling(plan)['smem'] <= 220 * 1024


def test_layer_config_round_trip():
    from kapre_b200.signal import PYIN, YIN
    y = YIN(22050, 65.0, 2000.0, hop_length=256, data_format=CF)
    cfg = y.get_config()
    y2 = YIN.from_config(cfg)
    assert y2.get_config() == cfg and y2.plan is y.plan
    p = PYIN(16000, 50.0, 600.0, frame_length=1024, switch_prob=0.02, data_format=CL)
    cfg = p.get_config()
    assert PYIN.from_config(cfg).get_config() == cfg
    import kapre
    assert kapre.signal.YIN is YIN and kapre.signal.pyin is not None


def test_exported_from_signal_not_from_the_package_root():
    # the package root mirrors kapre's hot-path import surface, every name of which records a gradient; the pitch
    # trackers have none, so they live in kapre_b200.signal (kapre.signal) like loudness and add_noise
    import kapre_b200
    from kapre_b200 import signal
    for name in ('yin', 'pyin', 'YIN', 'PYIN'):
        assert name in signal.__all__ and name not in kapre_b200.__all__
