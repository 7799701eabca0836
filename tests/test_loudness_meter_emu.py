"""The loudness meter on the CPU: the float64 restatement (loudness_meter_ref.py) against direct definitions and EBU's
test signals, the kernel bodies of meter_core.cuh (run by a CPU emulation) against the restatement within the derived
bounds at every rate, 1, 2 and 5 channels, both formats, with and without lengths, short, silent and NaN items; the
range's index rule, the true-peak gradient against torch.autograd, validation, configs and the register budget."""
import ctypes
import hashlib
import math
import os
import re
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

import loudness_meter_ref as MR
import loudness_ref as LR
from emu_harness import Checked

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, 'emu', 'kb_emu_meter.cpp')
_CSRC = os.path.join(_HERE, '..', 'kapre_b200', 'csrc')
_LIB = os.path.join(_HERE, '..', 'kapre_b200', '_lib', 'libkapre_b200.so')
_lib_handle = None
RATES = (8000, 11025, 16000, 44100, 48000)


def _lib():
    """tests/emu/kb_emu_meter.cpp built with g++ into the temporary directory (keyed by the sources' contents)."""
    global _lib_handle
    if _lib_handle is None:
        hs = hashlib.sha256()
        for f in [_SRC] + sorted(os.path.join(_CSRC, n) for n in os.listdir(_CSRC) if n.endswith(('.h', '.cuh'))):
            with open(f, 'rb') as fh:
                hs.update(fh.read())
        out = os.path.join(tempfile.gettempdir(), 'kapre_b200_emu_meter_%s.so' % hs.hexdigest()[:16])
        if not os.path.exists(out):
            tmp = '%s.%d.tmp' % (out, os.getpid())
            subprocess.check_call(['g++', '-O2', '-std=c++17', '-shared', '-fPIC', '-DKB_HOST_EMU', '-Wno-unknown-pragmas',
                                   '-o', tmp, _SRC])
            os.replace(tmp, out)
        lib = ctypes.CDLL(out)
        P, I = ctypes.c_void_p, ctypes.c_int
        lib.kb_emu_meter_geometry.argtypes = [I, I, I, I, P]
        lib.kb_emu_loudness_stats.argtypes = [P, P, P, I, I, I, I, I, I, P, P, P, P, I]
        lib.kb_emu_lra.argtypes = [P, P, I, I, P]
        lib.kb_emu_true_peak.argtypes = [P, P, P, I, I, I, P, P, P, P, I]
        lib.kb_emu_true_peak_backward.argtypes = [P, P, I, I, I, P, P, P, P, P]
        _lib_handle = Checked(lib)
    return _lib_handle


def _p(a):
    return ctypes.c_void_p(a.__array_interface__['data'][0]) if a is not None else None


def _strides(a, fmt):
    """Element strides (b, c, l) and (B, C, L) of a (B, C, L) ('bcl') or (B, L, C) ('blc') float32 array or view."""
    s = [v // 4 for v in a.strides]
    if fmt == 'blc':
        return np.array([s[0], s[2], s[1]], np.int64), (a.shape[0], a.shape[2], a.shape[1])
    return np.array(s, np.int64), a.shape


def _len(lengths, B):
    return None if lengths is None else np.ascontiguousarray(np.broadcast_to(np.asarray(lengths, np.int32), (B,)))


def emu_stats(y, sr, lengths=None, fmt='bcl', order=0):
    """(integrated, momentary, short_term, lra) of the K-weighted float32 y."""
    st, (B, C, L) = _strides(y, fmt)
    G, S, G3 = MR.geometry(sr)
    J = np.zeros(2, np.int32)
    _lib().kb_emu_meter_geometry(L, G, S, G3, _p(J))
    out = [np.full(B, 7.0, np.float32), np.full((B, J[0]), 7.0, np.float32), np.full((B, J[1]), 7.0, np.float32),
           np.full(B, 7.0, np.float32)]
    assert _lib().kb_emu_loudness_stats(_p(y), _p(st), _p(_len(lengths, B)), B, C, L, G, S, G3,
                                        *[_p(o) for o in out], order) == 0
    return out


def emu_true_peak(x, lengths=None, fmt='bcl', order=0):
    """(dBTP (B, C), z[t*], t*)."""
    st, (B, C, L) = _strides(x, fmt)
    out = np.full((B, C), 7.0, np.float32)
    zs = np.full((B, C), 7.0, np.float32)
    ts = np.zeros((B, C), np.uint32)
    taps = MR.tp_taps()
    assert _lib().kb_emu_true_peak(_p(x), _p(st), _p(_len(lengths, B)), B, C, L, _p(taps), _p(out), _p(zs), _p(ts),
                                   order) == 0
    return out, zs, ts


def emu_true_peak_backward(g, zs, ts, shape, lengths=None):
    B, C, L = shape
    gx = np.full((B, C, L), np.nan, np.float32)
    gst = np.array([C * L, L, 1], np.int64)
    g = np.ascontiguousarray(g, np.float32)
    assert _lib().kb_emu_true_peak_backward(_p(g), _p(_len(lengths, B)), B, C, L, _p(MR.tp_taps()), _p(zs), _p(ts),
                                            _p(gx), _p(gst)) == 0
    return gx


def _noise(shape, seed, scale=0.1):
    return np.random.default_rng(seed).standard_normal(shape) * scale


def _sections(C, sr, levels, seed, seconds=1.0):
    """(1, C, L) noise in consecutive sections of `seconds` at the given amplitudes."""
    n = int(seconds * sr)
    return np.concatenate([_noise((1, C, n), seed + i, a) for i, a in enumerate(levels)], axis=2)


def _weighted32(x, sr):
    y = LR.weight(x, LR.normalised(LR.k_weighting(sr)))
    return y, y.astype(np.float32)


def _check_stats(x, sr, lengths, fmt, got=None):
    """The emulated meter on x (B, C, L) against the restatement within the bounds; returns the emulated outputs."""
    G, S, G3 = MR.geometry(sr)
    y, y32 = _weighted32(x, sr)
    yin = y32 if fmt == 'bcl' else np.ascontiguousarray(y32.transpose(0, 2, 1))
    integ, mom, sht, lra = got if got is not None else emu_stats(yin, sr, lengths, fmt)
    delta = float(np.nan_to_num(np.abs(y - y32), nan=0.0).max())
    # integrated: kapre_loudness's own passes
    ref = LR.gated(y, G, S, lengths)[0]
    fin = np.isfinite(ref)
    assert np.array_equal(np.isnan(integ), np.isnan(ref)) and np.array_equal(np.isneginf(integ), np.isneginf(ref))
    assert np.all(np.abs(integ[fin] - ref[fin]) <= LR.lkfs_bound(y, G, S, delta, lengths)[fin])
    for W, got_s in ((G, mom), (G3, sht)):
        ref = MR.series(y, W, S, lengths)
        assert got_s.shape == ref.shape
        assert np.array_equal(np.isnan(got_s), np.isnan(ref)) and np.array_equal(np.isneginf(got_s), np.isneginf(ref))
        fin = np.isfinite(ref)
        assert np.all(np.abs(got_s[fin] - ref[fin]) <= MR.series_bound(y, W, S, delta, lengths)[fin]), W
    ref = MR.loudness_range(y, G3, S, lengths)
    bound = MR.lra_bound(y, G3, S, delta, lengths)
    margin = MR.lra_margin(y, G3, S, lengths)
    ok = np.isfinite(ref)
    assert np.array_equal(np.isnan(lra), np.isnan(ref))
    assert np.all(margin[ok] > 10 * bound[ok]), (margin, bound)         # the gate decisions cannot differ
    assert np.all(np.abs(lra[ok] - ref[ok]) <= bound[ok]), (lra, ref, bound)
    return integ, mom, sht, lra


# ------------------------------------------------------------------------------------------ the restatement
def test_restatement_series_and_integrated_are_loudness_ref_s():
    sr = 8000
    x = _sections(2, sr, (0.3, 0.01, 0.2, 0.05), 3)
    G, S, G3 = MR.geometry(sr)
    y = LR.weight(x, LR.k_weighting(sr))
    m = MR.series(y, G, S)
    # ungated momentary blocks are the gate pass's blocks
    E = (LR.WEIGHTS[:2, None] * LR.blocks(y[0], G, S, x.shape[2])).sum(0)
    np.testing.assert_allclose(m[0], -0.691 + 10 * np.log10(E), rtol=0, atol=1e-12)
    # a direct short-term window
    j = 5
    e = (y[0, :, j * S:j * S + G3] ** 2).mean(axis=1)
    assert abs(MR.series(y, G3, S)[0, j] - (-0.691 + 10 * math.log10(e.sum()))) < 1e-12
    assert MR.series(y, G, S, lengths=[G + S - 1]).tolist()[0][1:] == [-np.inf] * (m.shape[1] - 1)


@pytest.mark.parametrize('n', [1, 2, 10, 21])
def test_lra_index_rule_against_a_sort(n):
    rng = np.random.default_rng(n)
    E = 10 ** rng.uniform(-4, -1, size=n)
    j2, _ = MR.lra_gate(E)
    v = np.sort((-0.691 + 10 * np.log10(E))[j2])
    k = len(v)
    assert k >= 1
    assert MR.lra_of_energies(E) == v[((k - 1) * 95 + 50) // 100] - v[((k - 1) * 10 + 50) // 100]
    # the emulated range pass on the same energies, alone and with other items and lengths around it
    lra = np.full(3, 7.0, np.float32)
    e = np.zeros((3, n + 4))
    e[1, :n] = E
    e[0] = 10 ** rng.uniform(-4, -1, size=n + 4)
    e[2, :] = 1e-3
    counts = np.array([n + 4, n, 0], np.int32)
    _lib().kb_emu_lra(_p(np.ascontiguousarray(e)), _p(counts), 3, n + 4, _p(lra))
    assert lra[1] == np.float32(MR.lra_of_energies(E))
    assert lra[0] == np.float32(MR.lra_of_energies(e[0])) and lra[2] == 0.0


def test_lra_ties_and_equal_energies():
    E = np.array([1e-3, 1e-3, 2e-3, 2e-3, 2e-3, 1e-3])
    lra = np.full(1, 7.0, np.float32)
    _lib().kb_emu_lra(_p(np.ascontiguousarray(E[None])), None, 1, len(E), _p(lra))
    assert lra[0] == np.float32(MR.lra_of_energies(E)) and lra[0] > 0
    _lib().kb_emu_lra(_p(np.full((1, 9), 0.01)), None, 1, 9, _p(lra))
    assert lra[0] == 0.0


# ------------------------------------------------------------------------------------------ EBU anchors
def _sine(sr, seconds, dbfs, C=2, f=1000.0):
    t = np.arange(int(seconds * sr)) / sr
    return np.broadcast_to(10 ** (dbfs / 20) * np.sin(2 * np.pi * f * t), (1, C, len(t))).copy()


def test_tech3341_sine_at_minus_23():
    sr = 48000
    x = _sine(sr, 20, -23.0)
    integ, mom, sht, lra = emu_stats(_weighted32(x, sr)[1], sr)
    ref = MR.stats(x, sr)
    for v in (integ, mom, sht, ref[0], ref[1], ref[2]):
        assert np.all(np.abs(np.asarray(v) + 23.0) < 0.1), v
    assert abs(lra[0]) < 0.1


@pytest.mark.parametrize('levels, want', [((-20, -30), 10), ((-20, -15), 5), ((-40, -20), 20),
                                          ((-50, -35, -20, -35, -50), 15)])
def test_tech3342_loudness_range(levels, want):
    sr = 16000
    x = np.concatenate([_sine(sr, 20, v) for v in levels], axis=2)
    G, S, G3 = MR.geometry(sr)
    y, y32 = _weighted32(x, sr)
    ref = MR.loudness_range(y, G3, S)[0]
    assert abs(ref - want) <= 1, ref
    got = emu_stats(y32, sr)[3][0]
    assert abs(got - want) <= 1 and abs(got - ref) <= MR.lra_bound(y, G3, S, float(np.abs(y - y32).max()))[0]


def test_true_peak_of_a_quarter_rate_sine():
    sr = 48000
    A = 0.5
    n = np.arange(sr)
    fade = np.ones(sr)                                                # 50 ms raised-cosine ends: no edge overshoot
    fade[:2400] = np.sin(np.pi / 2 * np.arange(2400) / 2400) ** 2
    fade[-2400:] = fade[:2400][::-1]
    x = (A * fade * np.sin(np.pi * n / 2 + np.pi / 4)).astype(np.float32)[None, None]
    sample_peak = 20 * np.log10(np.abs(x).max())
    assert abs(sample_peak - (20 * np.log10(A) - 3.0103)) < 1e-4
    ref = MR.true_peak(x)[0, 0]
    got = emu_true_peak(x)[0][0, 0]
    # measured with scipy: the filter's passband ripple at sr / 4 puts the true peak 0.015 dB above the amplitude
    assert abs(ref - 20 * np.log10(A)) < 0.02, ref - 20 * np.log10(A)
    assert abs(got - ref) <= MR.true_peak_bound(x)[0, 0]


# ------------------------------------------------------------------------------------------ the kernels
@pytest.mark.parametrize('sr', RATES)
@pytest.mark.parametrize('C', [1, 2, 5])
@pytest.mark.parametrize('fmt', ['bcl', 'blc'])
def test_stats_within_bound(sr, C, fmt):
    x = np.concatenate([_sections(C, sr, (0.3, 0.005, 0.2, 0.05, 0.1), 7 + C),
                        _sections(C, sr, (0.1, 0.4, 0.02, 0.2, 0.01), 70 + C)])
    lengths = None if fmt == 'bcl' else [int(4.3 * sr), 5 * sr]
    _check_stats(x, sr, lengths, fmt)
    if fmt == 'bcl':
        _check_stats(x, sr, [int(3.7 * sr), int(2.2 * sr)], fmt)


def test_short_silent_and_nan_items():
    sr = 11025
    C = 2
    G, S, G3 = MR.geometry(sr)
    base = _sections(C, sr, (0.2, 0.02, 0.3, 0.1), 1)
    x = np.concatenate([base, base, base, np.zeros_like(base), base, base]).astype(np.float64)
    x[5, 1, int(2.5 * sr)] = np.nan
    lengths = [4 * sr, G - 1, G3 - 1, 4 * sr, 0, 4 * sr]          # full, < G, < G3, silent, empty, NaN
    integ, mom, sht, lra = _check_stats(x, sr, lengths, 'bcl')
    assert np.isneginf(mom[1]).all() and np.isfinite(mom[2, :count(G3 - 1, G, S)]).all()
    assert np.isneginf(sht[1:5]).all() and (lra[1:5] == 0).all()
    assert np.isneginf(integ[[1, 3, 4]]).all() and np.isneginf(mom[3]).all()
    assert np.isnan(integ[5]) and np.isnan(lra[5]) and np.isnan(mom[5]).any() and np.isnan(sht[5]).any()
    assert np.isfinite(integ[[0, 2]]).all() and np.isfinite(lra[0])
    tp = emu_true_peak(x.astype(np.float32), lengths)[0]
    ref = MR.true_peak(x.astype(np.float32), lengths)
    assert np.array_equal(np.isneginf(tp), np.isneginf(ref)) and np.isnan(tp[5, 1]) and np.isfinite(tp[5, 0])


def count(L, W, S):
    return MR.count(L, W, S)


def test_bits_do_not_depend_on_order_position_strides_format_or_lengths():
    sr = 16000
    C, L = 2, int(4.6 * sr)
    x = np.concatenate([_sections(C, sr, (0.2, 0.01, 0.3, 0.1, 0.05), 20 + i)[:, :, :L] for i in range(3)])
    _, y32 = _weighted32(x, sr)
    x32 = x.astype(np.float32)
    base = emu_stats(y32, sr)
    tbase = emu_true_peak(x32)
    for order in (1, 2):
        assert all(np.array_equal(a, b) for a, b in zip(emu_stats(y32, sr, order=order), base))
        assert all(np.array_equal(a, b) for a, b in zip(emu_true_peak(x32, order=order), tbase))
    one = emu_stats(np.ascontiguousarray(y32[2:3]), sr)
    assert all(np.array_equal(a, b[2:3]) for a, b in zip(one, base))
    assert np.array_equal(emu_true_peak(np.ascontiguousarray(x32[2:3]))[0], tbase[0][2:3])
    blc = np.ascontiguousarray(y32.transpose(0, 2, 1))
    assert all(np.array_equal(a, b) for a, b in zip(emu_stats(blc, sr, fmt='blc'), base))
    assert np.array_equal(emu_true_peak(np.ascontiguousarray(x32.transpose(0, 2, 1)), fmt='blc')[0], tbase[0])
    big = np.zeros((3, C + 2, L + 11), np.float32)
    big[:, 1:C + 1, 5:5 + L] = x32
    assert np.array_equal(emu_true_peak(big[:, 1:C + 1, 5:5 + L])[0], tbase[0])
    cut = [L, int(3.2 * sr), 3 * sr + 7]
    got = emu_stats(y32, sr, lengths=cut)
    tgot = emu_true_peak(x32, lengths=cut)[0]
    for b, n in enumerate(cut):
        alone = emu_stats(np.ascontiguousarray(y32[b:b + 1, :, :n]), sr)
        assert alone[0] == got[0][b] and alone[3] == got[3][b]
        for a, g in ((alone[1], got[1]), (alone[2], got[2])):
            assert np.array_equal(a[0], g[b, :a.shape[1]]) and np.isneginf(g[b, a.shape[1]:]).all()
        assert np.array_equal(emu_true_peak(np.ascontiguousarray(x32[b:b + 1, :, :n]))[0][0], tgot[b])


@pytest.mark.parametrize('C, fmt', [(1, 'bcl'), (2, 'blc'), (7, 'bcl')])
def test_true_peak_within_bound(C, fmt):
    x = np.concatenate([_noise((1, C, 5000), 3 + C, 0.3), _noise((1, C, 5000), 4 + C, 1e-3)]).astype(np.float32)
    x[1, 0, 2345] = 0.9                                               # an isolated spike
    lengths = [5000, 4100] if fmt == 'blc' else None
    xin = x if fmt == 'bcl' else np.ascontiguousarray(x.transpose(0, 2, 1))
    got, zs, ts = emu_true_peak(xin, lengths, fmt)
    ref = MR.true_peak(x, lengths)
    assert np.all(np.abs(got - ref) <= MR.true_peak_bound(x, lengths)), (got - ref)
    # t* is the argmax of the float64 z within the bound, and z[t*] its value
    for b in range(2):
        n = 5000 if lengths is None else lengths[b]
        for c in range(C):
            z = scipy_z(x[b, c, :n])
            assert abs(abs(z[ts[b, c]]) - 10 ** (ref[b, c] / 20)) <= 1e-5 * 10 ** (ref[b, c] / 20)
            assert abs(zs[b, c] - z[ts[b, c]]) <= 1e-5 * abs(z[ts[b, c]])


def scipy_z(x):
    import scipy.signal
    return scipy.signal.resample_poly(np.asarray(x, np.float64), 4, 1)


def test_true_peak_ties_go_to_the_lowest_index_and_silence_is_minus_inf():
    x = np.zeros((2, 1, 3000), np.float32)
    x[0, 0, 500] = 0.5
    x[0, 0, 2500] = 0.5                                               # the same |z| again, later
    x[0, 0, 1500] = -0.5
    got, zs, ts = emu_true_peak(x)
    assert ts[0, 0] == 4 * 500 and zs[0, 0] > 0
    assert np.isneginf(got[1, 0]) and zs[1, 0] == 0
    gx = emu_true_peak_backward(np.ones((2, 1), np.float32), zs, ts, (2, 1, 3000))
    assert np.all(gx[1] == 0) and np.count_nonzero(gx[0]) <= 21 and np.all(gx[0, 0, :480] == 0)


@pytest.mark.parametrize('lengths', [None, [3000, 1700]])
def test_true_peak_backward_is_torch_autograd(lengths):
    C = 2
    x = np.concatenate([_noise((1, C, 3000), 5, 0.3), _noise((1, C, 3000), 6, 0.01)]).astype(np.float32)
    x[1, 1] = 0.0                                                     # a silent channel: exactly 0
    _, zs, ts = emu_true_peak(x, lengths)
    g = np.array([[0.7, -1.3], [2.0, 0.5]], np.float32)
    got = emu_true_peak_backward(g, zs, ts, x.shape, lengths)
    want = MR.true_peak_vjp(x, g, lengths)
    assert np.all(got[1, 1] == 0)
    assert np.all(np.abs(got - want) <= 1e-4 * np.abs(want).max() + 1e-30)
    assert np.count_nonzero(got[0, 0]) > 10


# ------------------------------------------------------------------------------------------ validation and the ABI
def _kb():
    if not os.path.exists(_LIB):
        pytest.skip('needs the built library')


def test_exports_validation_and_config():
    _kb()
    import torch

    import kapre
    from kapre_b200 import signal as KS
    from kapre_b200._native import KapreNativeError
    from kapre_b200.augmentation import LoudnessNormalization
    for name in ('loudness_stats', 'true_peak', 'LoudnessStats'):
        assert name in KS.__all__ and getattr(kapre.signal, name) is getattr(KS, name)
    assert KS.LoudnessStats._fields == ('integrated', 'momentary', 'short_term', 'loudness_range', 'true_peak')
    with pytest.raises(KapreNativeError):
        KS.true_peak(torch.zeros(1, 100, 1))
    with pytest.raises(KapreNativeError):
        KS.loudness_stats(torch.zeros(1, 16000, 1), 16000)
    for bad in (np.nan, np.inf, 'loud', True):
        with pytest.raises(ValueError):
            LoudnessNormalization(16000, true_peak_limit=bad)
    norm = LoudnessNormalization(16000, lufs_range=(-20.0, -14.0), seed=1, true_peak_limit=-1)
    cfg = norm.get_config()
    assert cfg['true_peak_limit'] == -1.0 and LoudnessNormalization.from_config(cfg).get_config() == cfg
    assert LoudnessNormalization(16000).get_config()['true_peak_limit'] is None
    assert np.array_equal(MR.tp_taps(), KS.resample_filter(4, 1))


def test_workspace_sizes_and_bad_arguments():
    _kb()
    from kapre_b200 import _native as N
    lib = N.lib()
    st = ctypes.c_int64(-7)
    # 3 x 2 channels of 5000 samples: three 2048-sample tiles a column, 8 B a key, in 256 B units; (z, t) of 4 B a
    # column, each region in 256 B units
    assert lib.kapre_true_peak_workspace_bytes(3, 2, 5000, ctypes.byref(st)) == 256 and st.value == 512
    assert lib.kapre_true_peak_workspace_bytes(64, 2, 480000, None) == 64 * 2 * 235 * 8
    assert lib.kapre_true_peak_workspace_bytes(0, 1, 100, None) == 0
    for bad in ((-1, 1, 100), (1, 0, 100), (1, 1, -1), (1, 1, 2 ** 30 + 1)):
        assert lib.kapre_true_peak_workspace_bytes(*bad, None) < 0, bad
    assert lib.kapre_true_peak_workspace_bytes(1, 1, 2 ** 30, None) > 0
    G, S, G3 = MR.geometry(16000)
    assert lib.kapre_loudness_stats_workspace_bytes(256, 1, 80000, G, S, G3) > 0
    for bad in ((1, 6, 100, 40, 10, 300), (1, 1, 100, 40, 10, 39), (1, 1, 100, 40, 0, 300), (-1, 1, 100, 40, 10, 300)):
        assert lib.kapre_loudness_stats_workspace_bytes(*bad) < 0, bad


@pytest.mark.skipif(shutil.which('cuobjdump') is None or not os.path.exists(_LIB),
                    reason='needs cuobjdump and the built library')
def test_meter_kernels_have_no_stack_or_spills():
    out = subprocess.run(['cuobjdump', '-res-usage', _LIB], capture_output=True, text=True, check=True).stdout
    budget = {'kb_tp_peak_kernel': 64, 'kb_tp_fold_kernel': 64, 'kb_tp_bwd_kernel': 40, 'kb_meter_series_kernel': 64,
              'kb_meter_lra_kernel': 64}
    for name, regs in budget.items():
        m = re.search(r'Function \S*%s\S*:\s*\n\s*REG:(\d+) STACK:(\d+)' % name, out)
        assert m, name + ' not in the library'
        assert int(m.group(1)) <= regs, (name, m.group(1))
        assert int(m.group(2)) == 0, (name, m.group(2))
