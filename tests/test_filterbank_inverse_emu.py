"""Filterbank inversion on the CPU: the kernel body of fbinv_core.cuh (run by a CPU emulation) against the float64
restatement (fbinv_ref.py), the plan's step and back-projection weights, convergence against scipy's NNLS and
torchaudio's method, tile-shape, layout and stride invariance, decibel input, NaN containment, the unsupported-size
rule, and the ``InverseFilterbank`` layer's validation and config.

Tolerances.  Each FISTA step rounds a band dot (four float32 partial sums), a column dot, one FMA for the gradient step
and one for the momentum update.  The iteration map is non-expansive for the projected gradient part, but the momentum
term (coefficient up to ~1) carries each step's rounding into the next, so the error of a float32 run grows with the
iterations and with the conditioning of the bank.  A float32 twin of the same loop (``fbinv_ref.fista`` in float32,
NumPy's summation order) measures that growth for each case: on the banks here it drifts from the float64 run by
1e-7 of the frame's largest bin at 0 and 1 iterations, up to 5e-7 at 10 and up to 2e-5 at 100 (the 128-band 22.05 kHz
banks drift most).  The kernel sums in a different order than NumPy, so it does not reproduce the twin's bits, but its
error measured the same way is within 2x of the twin's.  It is held to 10x the twin's drift, with a floor of 1e-6 of
the frame's largest bin.
"""
import ctypes
import hashlib
import os
import subprocess
import tempfile

import numpy as np
import pytest

import fbinv_ref as FR
import oracle
from emu_harness import Checked

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, 'emu', 'kb_emu_fbinv.cpp')
_CSRC = os.path.join(_HERE, '..', 'kapre_b200', 'csrc')
_lib_handle = None
CL, CF = 'channels_last', 'channels_first'
H100_SMEM = 232448   # cudaDevAttrMaxSharedMemoryPerBlockOptin of an H100


def _lib():
    """tests/emu/kb_emu_fbinv.cpp built with g++ into the temporary directory (keyed by the sources' contents, so the
    checkout itself may be read-only)."""
    global _lib_handle
    if _lib_handle is None:
        h = hashlib.sha256()
        for f in [_SRC] + sorted(os.path.join(_CSRC, n) for n in os.listdir(_CSRC) if n.endswith(('.h', '.cuh'))):
            with open(f, 'rb') as fh:
                h.update(fh.read())
        out = os.path.join(tempfile.gettempdir(), 'kapre_b200_emu_fbinv_%s.so' % h.hexdigest()[:16])
        if not os.path.exists(out):
            tmp = '%s.%d.tmp' % (out, os.getpid())
            subprocess.check_call(['g++', '-O2', '-std=c++17', '-shared', '-fPIC', '-DKB_HOST_EMU', '-Wno-unknown-pragmas',
                                   '-o', tmp, _SRC])
            os.replace(tmp, out)
        lib = ctypes.CDLL(out)
        P, I, F = ctypes.c_void_p, ctypes.c_int, ctypes.c_float
        lib.kb_emu_fbi_tables.argtypes = [P, I, I, P, P, P]
        lib.kb_emu_fbi_pick_r.argtypes = [I, I, I]
        lib.kb_emu_fbi.argtypes = [P, I, I, P, P, I, I, I, I, I, F, F, P, P, I, I]
        _lib_handle = Checked(lib)
    return _lib_handle


def tables(fb):
    """(step float32, ||A||_2^2 float64, 1 / d float32) of the plan."""
    fb = np.ascontiguousarray(fb, np.float32)
    step, norm2 = ctypes.c_float(), ctypes.c_double()
    inv_d = np.zeros(fb.shape[1], np.float32)
    _lib().kb_emu_fbi_tables(fb.ctypes.data, fb.shape[0], fb.shape[1], ctypes.byref(step), ctypes.byref(norm2),
                             inv_d.ctypes.data)
    return np.float32(step.value), norm2.value, inv_d


def _strides(a, fmt):
    """(B, C, T, K) and the (b, c, t, k) element strides of a (B, T, K, C) channels_last / (B, C, T, K) array view."""
    s = [v // 4 for v in a.strides]
    if fmt == CL:
        B, T, K, C = a.shape
        return (B, C, T, K), np.array([s[0], s[3], s[1], s[2]], np.int64)
    B, C, T, K = a.shape
    return (B, C, T, K), np.array(s, np.int64)


def emu_invert(fb, x, fmt, n_iter, from_db=False, ref=1.0, amin=1e-5, R=32, n_cta=3):
    """x: a float32 (B, T, M, C) / (B, C, T, M) array (any strides) -> contiguous (B, T, F, C) / (B, C, T, F)."""
    fb = np.ascontiguousarray(fb, np.float32)
    assert x.dtype == np.float32
    (B, C, T, M), xs = _strides(x, fmt)
    F = fb.shape[0]
    out = np.full((B, T, F, C) if fmt == CL else (B, C, T, F), np.nan, np.float32)
    _, os_ = _strides(out, fmt)
    # the emulation reads x through its base pointer and element strides (a view into a larger buffer is fine)
    rc = _lib().kb_emu_fbi(fb.ctypes.data, F, M, x.ctypes.data, xs.ctypes.data, B, C, T, n_iter, int(from_db), ref, amin,
                           out.ctypes.data, os_.ctypes.data, R, n_cta)
    assert rc == 0
    return out


def _canon(a, fmt):
    """(B, T, K, C) / (B, C, T, K) -> (B, C, T, K) float64."""
    return np.ascontiguousarray(np.transpose(a, (0, 3, 1, 2)) if fmt == CL else a).astype(np.float64)


def _to_fmt(a, fmt):
    """(B, C, T, K) -> float32 array in `fmt`."""
    return np.ascontiguousarray(np.transpose(a, (0, 2, 3, 1)) if fmt == CL else a).astype(np.float32)


# ------------------------------------------------------------------------------ banks and inputs
# (kind, sample rate, n_fft, bands)
BANKS = [('mel', 22050, 256, 32), ('mel', 16000, 400, 80), ('mel', 22050, 1024, 128), ('mel', 22050, 2048, 128),
         ('mel', 22050, 4096, 64), ('log', 22050, 1024, 84), ('log', 44100, 2048, 48)]
BANK_IDS = ['%s%d_%d' % (k, n, m) for k, _, n, m in BANKS]


def _frame_err(got, want):
    """Per frame max|got - want| / max|want| over the bins: (..., T, F) -> (..., T)."""
    return np.abs(got - want).max(-1) / np.maximum(np.abs(want).max(-1), 1e-300)


def _reference(fb, m, n_iter):
    """(float64 restatement with the plan's step and weights, the float32 twin's worst per-frame drift)."""
    step, _, inv_d = tables(fb)
    A = FR.matrix(fb)
    mf = m.reshape(-1, m.shape[-1]).astype(np.float64)
    want = FR.fista(A, mf, n_iter, step=float(step), inv_d=inv_d.astype(np.float64))
    twin = FR.fista(A, mf, n_iter, step=step, inv_d=inv_d, dtype=np.float32)
    drift = float(_frame_err(twin.astype(np.float64), want).max())
    return want.reshape(m.shape[:-1] + (A.shape[1],)), drift


def _bound(drift):
    return max(1e-6, 10 * drift)


# ------------------------------------------------------------------------------ plan tables
@pytest.mark.parametrize('bank', BANKS, ids=BANK_IDS)
def test_step_and_back_projection_weights(bank):
    fb = FR.bank(*bank)
    A = FR.matrix(fb)
    step, norm2, inv_d = tables(fb)
    ref = np.linalg.norm(A, 2) ** 2
    assert abs(norm2 - ref) <= 1e-9 * ref, (norm2, ref)
    assert abs(float(step) * ref - 1.0) <= 1.2e-7, (step, 1 / ref)
    want = FR.inv_d_of(A)
    np.testing.assert_allclose(inv_d, want, rtol=1.2e-7, atol=0)
    assert np.all((inv_d == 0) == (want == 0))


# ------------------------------------------------------------------------------ parity with the restatement
@pytest.mark.parametrize('bank', BANKS, ids=BANK_IDS)
@pytest.mark.parametrize('n_iter', [0, 1, 10, 100])
def test_emulated_kernel_matches_restatement(bank, n_iter):
    kind, sr, n_fft, _ = bank
    fb = FR.bank(*bank)
    T = 5 if n_fft >= 4096 else 37
    m = FR.consistent_input(fb, sr, n_fft, 1, 2, T)
    want, drift = _reference(fb, m, n_iter)
    got = _canon(emu_invert(fb, _to_fmt(m, CF), CF, n_iter, R=16 if n_fft >= 4096 else 32), CF)
    err = float(_frame_err(got, want).max())
    assert err <= _bound(drift), (err, drift)


@pytest.mark.parametrize('bank', [BANKS[1], BANKS[2], BANKS[5]], ids=[BANK_IDS[1], BANK_IDS[2], BANK_IDS[5]])
def test_formats_views_and_tiles_give_identical_bits(bank):
    """channels_first / channels_last, a strided view (every other frame, a band-padded buffer, a channel slice), tile
    sizes R = 32 ... 1 and CTA counts: the same bits for every frame, and within the bound of the restatement."""
    kind, sr, n_fft, M = bank
    fb = FR.bank(*bank)
    m = FR.consistent_input(fb, sr, n_fft, 2, 2, 11)
    base = _canon(emu_invert(fb, _to_fmt(m, CF), CF, 10), CF)
    want, drift = _reference(fb, m, 10)
    assert float(_frame_err(base, want).max()) <= _bound(drift)
    np.testing.assert_array_equal(_canon(emu_invert(fb, _to_fmt(m, CL), CL, 10), CL), base)
    for R, n_cta in ((16, 1), (8, 5), (4, 2), (1, 7)):
        np.testing.assert_array_equal(_canon(emu_invert(fb, _to_fmt(m, CF), CF, 10, R=R, n_cta=n_cta), CF), base)
    for fmt in (CF, CL):
        big = np.full((2, 3, 22, M + 5), np.nan, np.float32)   # (B, C, T, M + 5)
        big[:, 1:, ::2, 2:M + 2] = m
        bigf = _to_fmt(big, fmt) if fmt == CL else big
        view = bigf[:, ::2, 2:M + 2, 1:] if fmt == CL else bigf[:, 1:, ::2, 2:M + 2]
        np.testing.assert_array_equal(_canon(emu_invert(fb, view, fmt, 10, R=8), fmt), base)
    # a frame alone, and at another place in a longer batch
    alone = _canon(emu_invert(fb, _to_fmt(m[1:2, :, 7:8], CF), CF, 10), CF)
    np.testing.assert_array_equal(alone[0, :, 0], base[1, :, 7])


def test_empty_and_single_frame():
    fb = FR.bank('mel', 22050, 256, 32)
    assert emu_invert(fb, np.zeros((0, 1, 4, 32), np.float32), CF, 5).shape == (0, 1, 4, 129)
    assert emu_invert(fb, np.zeros((2, 0, 32, 1), np.float32), CL, 5).shape == (2, 0, 129, 1)
    m = FR.consistent_input(fb, 22050, 256, 1, 1, 1)
    want, drift = _reference(fb, m, 10)
    assert float(_frame_err(_canon(emu_invert(fb, _to_fmt(m, CF), CF, 10), CF), want).max()) <= _bound(drift)


# ------------------------------------------------------------------------------ what the iteration achieves
_CONV = [('mel', 22050, 1024, 128), ('mel', 22050, 2048, 128), ('mel', 16000, 400, 80), ('log', 22050, 1024, 84)]


@pytest.mark.parametrize('bank', _CONV, ids=['%s%d' % (b[0], b[2]) for b in _CONV])
def test_converges_on_consistent_input_and_beats_lstsq_relu(bank):
    """At the default 100 iterations the residual ||A s - m|| is below 1e-3 of ||m|| in every frame; scipy's NNLS
    reaches 0 there (the input is reachable); and the residual over the input is below that of relu(lstsq(A, m)), which
    is what torchaudio.transforms.InverseMelScale computes, taken with this matrix.  For the 22.05 kHz mel banks that
    holds in every frame.  For the 16 kHz / 80-band bank the least-squares solution of many frames of this signal is
    already non-negative, so relu(lstsq) is exact there to float64 rounding and beats a float32 iteration frame by
    frame, while it leaves large residuals in the other frames: that bank is compared over the whole input only.  The
    log bank (84 overlapping bumps) has that property in every frame, so relu(lstsq) is not compared there: the
    iteration only reaches its float32 floor (about 1e-7)."""
    from scipy.optimize import nnls
    kind, sr, n_fft, _ = bank
    fb = FR.bank(*bank)
    m = FR.consistent_input(fb, sr, n_fft, 1, 1, 24, seed=3)
    got = _canon(emu_invert(fb, _to_fmt(m, CF), CF, 100), CF)[0, 0]
    A = FR.matrix(fb)
    mf = m[0, 0].astype(np.float64)
    res = FR.residual(A, got, mf)
    assert res.max() < 1e-3, res.max()
    for t in range(0, 24, 6):
        _, rn = nnls(A, mf[t], maxiter=50 * A.shape[1])
        assert rn <= 1e-6 * np.linalg.norm(mf[t]), (t, rn)
    if kind != 'mel':
        return
    s_ls = FR.lstsq_relu(A, mf)
    total = np.linalg.norm(got @ A.T - mf) / np.linalg.norm(mf)
    total_ls = np.linalg.norm(s_ls @ A.T - mf) / np.linalg.norm(mf)
    assert total < total_ls, (total, total_ls)
    if sr == 22050 and kind == 'mel':
        res_ls = FR.residual(A, s_ls, mf)
        assert np.all(res < res_ls), (res.max(), res_ls.min())


@pytest.mark.parametrize('bank', [BANKS[2], BANKS[5]], ids=[BANK_IDS[2], BANK_IDS[5]])
def test_non_negative_and_untouched_bins_zero(bank):
    kind, sr, n_fft, _ = bank
    fb = FR.bank(*bank)
    rng = np.random.default_rng(4)
    m = np.concatenate([FR.consistent_input(fb, sr, n_fft, 1, 1, 6),
                        rng.uniform(0, 2, size=(1, 1, 6, fb.shape[1])).astype(np.float32)], axis=2)   # consistent, random
    untouched = ~np.any(fb != 0, axis=1)
    assert untouched.any()
    for n_iter in (0, 3, 100):
        got = emu_invert(fb, m, CF, n_iter)
        assert np.all(got >= 0)
        assert np.all(got[..., untouched] == 0)


# ------------------------------------------------------------------------------ decibel input
def _db(m, ref, amin, dyn=80.0):
    """oracle's magnitude_to_decibel per item over (B, C, T, M)."""
    return np.stack([oracle.magnitude_to_decibel(m[b:b + 1].astype(np.float64), ref, amin, dyn)[0]
                     for b in range(m.shape[0])]).astype(np.float32)


@pytest.mark.parametrize('ref,amin', [(1.0, 1e-5), (0.5, 1e-4), (1e-6, 1e-3)])
def test_decibel_input_round_trips(ref, amin):
    """dB in, converted on load: the same result as the magnitudes in, to float32 tolerance where the clamp did not
    bind; an element the clamp raised comes back as the clamp floor."""
    fb = FR.bank('mel', 22050, 1024, 128)
    m = FR.consistent_input(fb, 22050, 1024, 2, 1, 9)
    m[1] *= 1e6
    m[1, 0, 4, :] = 1e-9            # a quiet frame in a loud item: the clamp binds there
    d = _db(m, ref, amin)
    scale = max(amin, ref)
    floor_db = d.reshape(2, -1).min(axis=1)
    m_eff = np.where(d <= floor_db[:, None, None, None] + 1e-4, 10.0 ** (floor_db[:, None, None, None] / 10) * scale,
                     np.maximum(m, amin))
    for n_iter in (0, 10):
        got = _canon(emu_invert(fb, d, CF, n_iter, from_db=True, ref=ref, amin=amin), CF)
        want = _canon(emu_invert(fb, m_eff.astype(np.float32), CF, n_iter), CF)
        assert float(_frame_err(got, want).max()) <= 2e-5
    clamped = d[1, 0, 4] <= floor_db[1] + 1e-4
    assert clamped.all()


# ------------------------------------------------------------------------------ NaN
def test_nan_stays_inside_its_frame():
    fb = FR.bank('mel', 22050, 1024, 128)
    m = FR.consistent_input(fb, 22050, 1024, 2, 1, 40)
    clean = emu_invert(fb, m, CF, 20)
    bad = m.copy()
    bad[1, 0, 33, 17] = np.nan
    got = emu_invert(fb, bad, CF, 20)
    assert np.isnan(got[1, 0, 33]).any()
    keep = np.ones(got.shape[:3], bool)
    keep[1, 0, 33] = False
    np.testing.assert_array_equal(got[keep], clean[keep])


# ------------------------------------------------------------------------------ sizes
def test_tile_size_rule_and_unsupported_size():
    """R shrinks with the spectrum length; every n_fft up to 16384 fits an H100; a filterbank whose single-frame state
    does not fit shared memory gets R = 0, which the library reports as KAPRE_E_UNSUPPORTED."""
    lib = _lib()
    assert lib.kb_emu_fbi_pick_r(513, 128, H100_SMEM) == 32
    assert lib.kb_emu_fbi_pick_r(1025, 128, H100_SMEM) == 16
    for n_fft in (4096, 8192, 16384):
        assert lib.kb_emu_fbi_pick_r(n_fft // 2 + 1, 512, H100_SMEM) >= 1
    assert lib.kb_emu_fbi_pick_r(16385, 128, H100_SMEM) == 0
    assert lib.kb_emu_fbi_pick_r(8193, 8000, H100_SMEM) == 0


def test_largest_fft_runs():
    fb = FR.bank('mel', 44100, 16384, 64)
    m = FR.consistent_input(fb, 44100, 16384, 1, 1, 2)
    want, drift = _reference(fb, m, 4)
    got = _canon(emu_invert(fb, _to_fmt(m, CF), CF, 4, R=_lib().kb_emu_fbi_pick_r(8193, 64, H100_SMEM)), CF)
    assert float(_frame_err(got, want).max()) <= _bound(drift)


def test_kernel_register_and_spill_budget():
    """The inversion kernel fits 64 registers (one 1024-thread CTA fills the register file) and does not spill."""
    import re
    import shutil
    lib = os.path.join(_HERE, '..', 'kapre_b200', '_lib', 'libkapre_b200.so')
    if shutil.which('cuobjdump') is None or not os.path.exists(lib):
        pytest.skip('needs cuobjdump and the built library')
    out = subprocess.run(['cuobjdump', '-res-usage', lib], capture_output=True, text=True, check=True).stdout
    lines = out.splitlines()
    found = [(lines[i], lines[i + 1]) for i in range(len(lines) - 1) if 'kb_fbi_' in lines[i]]
    assert len(found) == 1, found
    for name, res in found:
        m = re.search(r'REG:(\d+) STACK:(\d+).*LOCAL:(\d+)', res)
        assert m and int(m.group(1)) <= 64 and int(m.group(2)) == 0 and int(m.group(3)) == 0, (name, res)


# ------------------------------------------------------------------------------ the layer and the factory
_MEL_KW = dict(sample_rate=16000, n_freq=257, n_mels=40)


def test_layer_validation():
    from kapre_b200.time_frequency import InverseFilterbank
    for kw in ({'n_iter': -1}, {'n_iter': 2.0}, {'n_iter': True}, {'from_decibel': 1}, {'db_ref_value': 0.0},
               {'db_ref_value': -1.0}, {'db_ref_value': float('inf')}, {'db_amin': 0}, {'db_amin': float('nan')},
               {'db_amin': '1e-5'}, {'data_format': 'channels_middle'}):
        with pytest.raises(ValueError):
            InverseFilterbank('mel', _MEL_KW, **kw)
    with pytest.raises(ValueError):
        InverseFilterbank('linear', _MEL_KW)
    InverseFilterbank('mel', _MEL_KW, n_iter=0)
    InverseFilterbank('log', dict(sample_rate=22050, n_freq=513), n_iter=np.int64(3), from_decibel=True, db_amin=1e-10)


def test_layer_config_round_trip_and_alias():
    from kapre_b200.time_frequency import ApplyFilterbank, InverseFilterbank
    import kapre
    import kapre_b200
    from kapre_b200 import time_frequency
    assert kapre.time_frequency.InverseFilterbank is InverseFilterbank
    assert 'InverseFilterbank' in time_frequency.__all__ and 'InverseFilterbank' not in kapre_b200.__all__
    assert time_frequency.get_registered_object('Kapre>InverseFilterbank') is InverseFilterbank
    layer = InverseFilterbank('mel', _MEL_KW, n_iter=30, from_decibel=True, db_ref_value=0.5, db_amin=1e-4,
                              data_format='channels_first', name='inv_x')
    cfg = layer.get_config()
    assert cfg['type'] == 'mel' and cfg['filterbank_kwargs'] == _MEL_KW and cfg['n_iter'] == 30
    assert cfg['from_decibel'] is True and cfg['db_ref_value'] == 0.5 and cfg['db_amin'] == 1e-4
    assert cfg['data_format'] == 'channels_first' and cfg['name'] == 'inv_x'
    assert InverseFilterbank.from_config(cfg).get_config() == cfg
    d = InverseFilterbank('log', dict(sample_rate=22050, n_freq=513)).get_config()
    assert d['n_iter'] == 100 and d['from_decibel'] is False and d['db_ref_value'] == 1.0 and d['db_amin'] == 1e-5
    assert d['data_format'] == 'default'
    np.testing.assert_array_equal(layer.filterbank, ApplyFilterbank('mel', _MEL_KW).filterbank)


def test_factory_shares_the_melspectrogram_arguments():
    from kapre_b200 import composed
    from kapre_b200.time_frequency import GriffinLim, InverseFilterbank
    kw = dict(n_fft=512, win_length=400, hop_length=160, window_name='hamming_window', sample_rate=16000, n_mels=64,
              mel_f_min=50.0, mel_f_max=7000.0, mel_htk=True, mel_norm=None, return_decibel=True, db_amin=1e-4,
              db_ref_value=2.0)
    fwd = composed.get_melspectrogram_layer(input_data_format=CL, output_data_format=CF, **kw)
    inv = composed.get_inverse_melspectrogram_layer(nnls_iter=50, griffin_lim_iter=8, momentum=0.5, init='ones', seed=4,
                                                    input_data_format=CF, output_data_format=CL, **kw)
    assert 'get_inverse_melspectrogram_layer' in composed.__all__
    assert [type(l) for l in inv.layers] == [InverseFilterbank, GriffinLim]
    ifb, gl = inv.layers
    np.testing.assert_array_equal(ifb.filterbank, fwd.layers[2].filterbank)
    assert ifb.n_iter == 50 and ifb.from_decibel and ifb.db_amin == 1e-4 and ifb.db_ref_value == 2.0
    assert ifb.data_format == CF and gl.input_data_format == CF and gl.output_data_format == CL
    g = gl.get_config()
    assert (g['n_fft'], g['win_length'], g['hop_length'], g['window_name']) == (512, 400, 160, 'hamming_window')
    assert (g['n_iter'], g['momentum'], g['init'], g['seed']) == (8, 0.5, 'ones', 4)
    d = composed.get_inverse_melspectrogram_layer()
    assert d.layers[0].n_iter == 100 and not d.layers[0].from_decibel and d.layers[1].n_iter == 32
    assert d.layers[0].filterbank.shape == (1025, 128)
    assert type(composed.Sequential.from_config(inv.get_config()).layers[0]) is InverseFilterbank
