"""PCEN on the CPU: the float64 restatement (pcen_ref.py) against scipy's ``lfilter`` and the naive formula, its
autograd gradients against finite differences, and the kernel bodies of pcen_core.cuh (run by a CPU emulation)
against the restatement, forward and backward, unchunked and chunked; plus the ``PCEN`` layer's validation,
config and weights.

Tolerances, float32 against float64.  Every step of the smoother rounds once (an FMA and a product), and the
recurrence is a contraction by 1 - s, so the error of M stays below about eps32 / s relative to M (1e-5 at
s = 0.0286; chunking adds the fold, K terms of the same size).  u, log1p and expm1 each add a few ulps, so y is
held to 1e-4 relative to |y| + 1e-4 max|y| (the absolute part covers y near 0, where u << d).  The gradients
propagate the same relative errors through at most five more rounded operations per frame; lam sums terms that
decay by 1 - s, so gE is held to 1e-4 of max|gE|, and each parameter gradient, a float32 sum over frames, to
1e-4 of the sum of its absolute per-element contributions (pcen_ref.grads), which bounds any cancellation.
s = 0 and s = 1 are exact in the smoother (M = E[0] or M = E).
"""
import ctypes
import hashlib
import math
import os
import subprocess
import tempfile

import numpy as np
import pytest
import torch

import pcen_ref as PR
from emu_harness import Checked

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, 'emu', 'kb_emu_pcen.cpp')
_CSRC = os.path.join(_HERE, '..', 'kapre_b200', 'csrc')
_lib_handle = None
CL, CF = 'channels_last', 'channels_first'
EPS = 1e-6


def _lib():
    """tests/emu/kb_emu_pcen.cpp built with g++ into the temporary directory (keyed by the sources' contents, so the
    checkout itself may be read-only)."""
    global _lib_handle
    if _lib_handle is None:
        h = hashlib.sha256()
        for f in [_SRC] + sorted(os.path.join(_CSRC, n) for n in os.listdir(_CSRC) if n.endswith(('.h', '.cuh'))):
            with open(f, 'rb') as fh:
                h.update(fh.read())
        out = os.path.join(tempfile.gettempdir(), 'kapre_b200_emu_pcen_%s.so' % h.hexdigest()[:16])
        if not os.path.exists(out):
            tmp = '%s.%d.tmp' % (out, os.getpid())
            subprocess.check_call(['g++', '-O2', '-std=c++17', '-shared', '-fPIC', '-DKB_HOST_EMU', '-Wno-unknown-pragmas',
                                   '-o', tmp, _SRC])
            os.replace(tmp, out)
        lib = ctypes.CDLL(out)
        P = ctypes.c_void_p
        lib.kb_emu_pcen.argtypes = [P, P, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, P, P, ctypes.c_float,
                                    ctypes.c_int, P, P, P, P]
        lib.kb_emu_pcen_backward.argtypes = [P, P, P, P, P, P, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                             P, P, ctypes.c_float, ctypes.c_int, P, P, P]
        lib.kb_emu_pcen_chunks.argtypes = [ctypes.c_longlong, ctypes.c_int, ctypes.c_longlong]
        _lib_handle = Checked(lib)
    return _lib_handle


def _fp(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _dims_strides(x, fmt):
    """(B, C, T, F) and the (b, c, t, f) element strides of a (B, T, F, C) channels_last / (B, C, T, F) array."""
    s = [v // 4 for v in x.strides]
    if fmt == CL:
        B, T, F, C = x.shape
        return (B, C, T, F), np.array([s[0], s[3], s[1], s[2]], np.int64)
    B, C, T, F = x.shape
    return (B, C, T, F), np.array(s, np.int64)


def _alloc(fmt, B, C, T, F):
    a = np.full((B, T, F, C) if fmt == CL else (B, C, T, F), np.nan, np.float32)
    return a, _dims_strides(a, fmt)[1]


class _Params:
    """The four parameters as host float32 arrays for the emulation (stride 0: shared, 1: per band)."""

    def __init__(self, gain, bias, power, smooth):
        self.values = [np.atleast_1d(np.asarray(v, np.float32)) for v in (gain, bias, power, smooth)]
        self.ptrs = (ctypes.c_void_p * 4)(*[v.ctypes.data for v in self.values])
        self.strides = np.array([1 if v.size > 1 else 0 for v in self.values], np.int32)
        self.ref = [v if v.size > 1 else float(v[0]) for v in (x.astype(np.float64) for x in self.values)]


def emu_pcen(x, fmt, prm, Tc=0, with_M=True):
    (B, C, T, F), es = _dims_strides(x, fmt)
    y, ys = _alloc(fmt, B, C, T, F)
    M, ms = _alloc(fmt, B, C, T, F) if with_M else (None, None)
    K = _lib().kb_emu_pcen(x.ctypes.data, _fp(es), B, C, T, F, prm.ptrs, _fp(prm.strides), EPS, Tc, _fp(y), _fp(ys),
                           _fp(M) if with_M else None, _fp(ms) if with_M else None)
    return y, M, K


def emu_pcen_backward(x, M, gy, fmt, prm, Tc=0):
    """(gE, [g_gain, g_bias, g_power, g_smooth]) with each parameter gradient reduced to its own shape."""
    (B, C, T, F), es = _dims_strides(x, fmt)
    ms, gs = _dims_strides(M, fmt)[1], _dims_strides(gy, fmt)[1]
    gE, os_ = _alloc(fmt, B, C, T, F)
    K = -(-T // Tc) if (Tc > 0 and T > 0) else 1
    part = np.full((4, K, B, C, F), np.nan, np.float32)
    rc = _lib().kb_emu_pcen_backward(x.ctypes.data, _fp(es), M.ctypes.data, _fp(ms), gy.ctypes.data, _fp(gs), B, C, T, F,
                                     prm.ptrs, _fp(prm.strides), EPS, Tc, _fp(gE), _fp(os_), _fp(part))
    assert rc == (K if B * C * F * T else 0)
    g = []
    for j, v in enumerate(prm.values):
        band = part[j].astype(np.float64).sum(axis=(0, 1, 2)) if T else np.zeros(F)
        g.append(band if v.size > 1 else band.sum())
    return gE, g


def _canon(x, fmt):
    """(B, C, T, F) float64 torch tensor of an array in `fmt`."""
    t = torch.from_numpy(np.ascontiguousarray(x, np.float64))
    return t.permute(0, 3, 1, 2) if fmt == CL else t


def _spectrogram(rng, fmt, B, C, T, F):
    """Non-negative, spread over four decades like mel magnitudes."""
    x = (10.0 ** rng.uniform(-2, 2, size=(B, T, F, C) if fmt == CL else (B, C, T, F))).astype(np.float32)
    return x


def _close(got, want, rel, scale):
    want = np.asarray(want, np.float64)
    got = np.asarray(got, np.float64)
    assert got.shape == want.shape, (got.shape, want.shape)
    if got.size:
        err = np.abs(got - want)
        bound = rel * (np.abs(want) + scale)
        assert np.all(err <= bound), (float((err / np.maximum(bound, 1e-300)).max()), float(err.max()))


def _check_forward(x, fmt, prm, Tc=0):
    y, M, K = emu_pcen(x, fmt, prm, Tc)
    yr, Mr = PR.pcen(_canon(x, fmt), *prm.ref, eps=EPS, return_M=True)
    yr, Mr = yr.numpy(), Mr.numpy()
    to = (lambda a: np.ascontiguousarray(_canon(a, fmt).numpy()))
    ysc = 1e-4 * float(np.abs(yr).max()) if yr.size else 0.0
    _close(to(y), yr, 1e-4, ysc)
    _close(to(M), Mr, 1e-4, 1e-4 * float(np.abs(Mr).max()) if Mr.size else 0.0)
    y2, _, _ = emu_pcen(x, fmt, prm, Tc, with_M=False)
    np.testing.assert_array_equal(y2, y)               # writing M does not change a bit of y
    return y, M, K


def _check_backward(x, M, fmt, prm, rng, Tc=0):
    gy = rng.uniform(-1, 1, size=x.shape).astype(np.float32)
    gE, g = emu_pcen_backward(x, M, gy, fmt, prm, Tc)
    gEr, gr, scale = PR.grads(_canon(x, fmt), prm.ref, _canon(gy, fmt), eps=EPS)
    gE_c = np.ascontiguousarray(_canon(gE, fmt).numpy())
    _close(gE_c, gEr.numpy(), 0.0, 0.0) if not gE.size else \
        _close(gE_c, gEr.numpy(), 1e-4, float(np.abs(gEr.numpy()).max()))
    for got, want, sc in zip(g, gr, scale):
        want = want.numpy()
        assert np.all(np.abs(got - want) <= 1e-4 * sc.numpy() + 1e-30), (got, want, sc)
    return gE, g


# ------------------------------------------------------------------------------ the restatement
@pytest.mark.parametrize('s', [0.0, 0.0286, 0.3, 1.0])
def test_smoother_matches_lfilter(s):
    sig = pytest.importorskip('scipy.signal')
    E = np.random.default_rng(1).uniform(0, 5, size=(2, 3, 50, 4))
    want = sig.lfilter([s], [1, s - 1], E, axis=2, zi=(1 - s) * E[:, :, :1])[0]
    got = PR.smoother(torch.from_numpy(E), s).numpy()
    np.testing.assert_allclose(got, want, rtol=1e-12, atol=1e-12)


def test_cancellation_free_form_matches_naive():
    """Where (u + d)^r - d^r is accurate (u not small against d), the expm1 / log1p form agrees with it."""
    E = torch.from_numpy(np.random.default_rng(2).uniform(0.5, 50, size=(1, 1, 40, 6)))
    for gain, bias, power in ((0.98, 2.0, 0.5), (0.5, 0.1, 0.25), (0.0, 1.0, 2.0)):
        got = PR.pcen(E, gain, bias, power, 0.1)
        want = PR.pcen_naive(E, gain, bias, power, 0.1)
        torch.testing.assert_close(got, want, rtol=1e-12, atol=1e-12)
    # and where it is not: u = 1e-12 d, the naive form loses everything
    tiny = torch.full((1, 1, 3, 1), 1e-12, dtype=torch.float64)
    got = PR.pcen(tiny, 0.0, 1.0, 0.5, 0.5)
    assert torch.allclose(got, torch.full_like(tiny, 0.5e-12), rtol=1e-9)


def test_smooth_coef_from_time_constant():
    assert abs(PR.smooth_coef(0.4, 22050, 256) - 0.0286) < 5e-5
    assert abs(PR.smooth_coef(0.4, 22050, 512) - 0.0564) < 5e-5


@pytest.mark.parametrize('per_band', [False, True])
def test_restatement_gradcheck(per_band):
    rng = np.random.default_rng(3)
    E = torch.from_numpy(rng.uniform(0.1, 3, size=(2, 1, 6, 3))).requires_grad_()
    shape = (3,) if per_band else ()
    ps = [torch.from_numpy(np.asarray(rng.uniform(lo, hi, size=shape))).requires_grad_()
          for lo, hi in ((0.5, 1.0), (1.0, 3.0), (0.3, 0.8), (0.1, 0.6))]
    assert torch.autograd.gradcheck(lambda e, a, d, r, s: PR.pcen(e, a, d, r, s, eps=1e-6), (E, *ps))


# ------------------------------------------------------------------------------ the emulated bodies
_SCALAR = (0.98, 2.0, 0.5, 0.0564)


def _per_band(F, seed=4):
    rng = np.random.default_rng(seed)
    return (rng.uniform(0.5, 1.0, F), rng.uniform(0.5, 3.0, F), rng.uniform(0.2, 0.8, F), rng.uniform(0.01, 0.5, F))


@pytest.mark.parametrize('T', [0, 1, 2, 17, 40])
@pytest.mark.parametrize('C', [1, 2, 3])
@pytest.mark.parametrize('fmt', [CF, CL])
@pytest.mark.parametrize('per_band', [False, True])
def test_emulated_forward_and_backward(T, C, fmt, per_band):
    """Bands not a multiple of 32 (37), T not a multiple of the register tiles (16 and 8), several batch items."""
    rng = np.random.default_rng(T * 10 + C)
    F = 37
    prm = _Params(*(_per_band(F) if per_band else _SCALAR))
    x = _spectrogram(rng, fmt, 2, C, T, F)
    _, M, K = _check_forward(x, fmt, prm)
    assert K in (0, 1)
    _check_backward(x, M, fmt, prm, rng)


@pytest.mark.parametrize('s', [0.0, 1.0])
@pytest.mark.parametrize('fmt', [CF, CL])
def test_emulated_smooth_coef_limits(s, fmt):
    rng = np.random.default_rng(5)
    x = _spectrogram(rng, fmt, 1, 2, 23, 5)
    prm = _Params(0.9, 1.5, 0.4, s)
    y, M, _ = _check_forward(x, fmt, prm)
    E = _canon(x, fmt).numpy()
    want_M = np.broadcast_to(E[:, :, :1], E.shape) if s == 0.0 else E
    np.testing.assert_array_equal(_canon(M, fmt).numpy(), want_M.astype(np.float32))
    _check_backward(x, M, fmt, prm, rng)


@pytest.mark.parametrize('view', ['time_stride', 'band_slice', 'channel_slice', 'batch_stride', 'transposed'])
@pytest.mark.parametrize('fmt', [CF, CL])
def test_emulated_body_on_views(view, fmt):
    rng = np.random.default_rng(6)
    full = _spectrogram(rng, fmt, 3, 3, 30, 40)
    t_ax, f_ax, c_ax = (1, 2, 3) if fmt == CL else (2, 3, 1)
    sl = [slice(None)] * 4
    if view == 'time_stride':
        sl[t_ax] = slice(None, None, 2)
    elif view == 'band_slice':
        sl[f_ax] = slice(3, 36)
    elif view == 'channel_slice':
        sl[c_ax] = slice(1, 3)
    elif view == 'batch_stride':
        sl[0] = slice(None, None, 2)
    x = full[tuple(sl)]
    if view == 'transposed':            # the other format's memory order under this format's shape
        x = np.ascontiguousarray(np.moveaxis(full, c_ax, 1 if fmt == CL else 3))
        x = np.moveaxis(x, 1 if fmt == CL else 3, c_ax)
    prm = _Params(*_per_band(x.shape[f_ax], seed=7))
    _, M, _ = _check_forward(x, fmt, prm)
    _check_backward(x, M, fmt, prm, rng)


@pytest.mark.parametrize('fmt', [CF, CL])
@pytest.mark.parametrize('per_band', [False, True])
def test_emulated_chunks_at_every_offset(fmt, per_band):
    """The chunked passes with chunk lengths 1..T-1 of a 13-frame signal: a chunk boundary at every offset."""
    rng = np.random.default_rng(8)
    T, F = 13, 33
    prm = _Params(*(_per_band(F, seed=9) if per_band else (0.98, 2.0, 0.5, 0.2)))
    x = _spectrogram(rng, fmt, 2, 2, T, F)
    y1, M1, _ = emu_pcen(x, fmt, prm)
    for Tc in range(1, T):
        y, M, K = _check_forward(x, fmt, prm, Tc)
        assert K == -(-T // Tc)
        _check_backward(x, M, fmt, prm, np.random.default_rng(Tc), Tc)
        _close(y, y1, 1e-5, 1e-5 * float(np.abs(y1).max()))


@pytest.mark.parametrize('fmt', [CF, CL])
def test_emulated_chunks_long(fmt):
    """32 chunks of 40 frames (the most the library uses) on a long column set, small smoothing coefficient."""
    rng = np.random.default_rng(10)
    prm = _Params(0.98, 2.0, 0.5, 0.0286)
    x = _spectrogram(rng, fmt, 1, 1, 1280, 5)
    _, M, K = _check_forward(x, fmt, prm, Tc=40)
    assert K == 32
    _check_backward(x, M, fmt, prm, rng, Tc=40)


def test_emulated_backward_is_deterministic():
    rng = np.random.default_rng(11)
    prm = _Params(*_per_band(9))
    x = _spectrogram(rng, CL, 2, 2, 50, 9)
    _, M, _ = emu_pcen(x, CL, prm, Tc=7)
    gy = rng.uniform(-1, 1, size=x.shape).astype(np.float32)
    a = emu_pcen_backward(x, M, gy, CL, prm, Tc=7)
    b = emu_pcen_backward(x, M, gy, CL, prm, Tc=7)
    np.testing.assert_array_equal(a[0], b[0])
    for u, v in zip(a[1], b[1]):
        np.testing.assert_array_equal(u, v)


def test_chunk_choice():
    """One chunk while the columns fill a sixteenth of the resident threads; else up to 32, none under 64 frames."""
    lib = _lib()
    resident = 132 * 2048
    assert lib.kb_emu_pcen_chunks(256 * 128, 427, resident) == 1          # cfg2 mel shape
    assert lib.kb_emu_pcen_chunks(128, 51680, resident) == 32             # 10 min at 22.05 kHz, hop 256
    assert lib.kb_emu_pcen_chunks(128, 200, resident) == 3                # short: chunks of at least 64 frames
    assert lib.kb_emu_pcen_chunks(128, 100, resident) == 1
    assert lib.kb_emu_pcen_chunks(8 * 128, 5000, resident) == 32
    assert lib.kb_emu_pcen_chunks(10000, 5000, resident) == 7


def test_kernel_register_and_spill_budget():
    """The four PCEN kernels do not spill (the register tiles must stay in registers)."""
    import re
    import shutil
    lib = os.path.join(_HERE, '..', 'kapre_b200', '_lib', 'libkapre_b200.so')
    if shutil.which('cuobjdump') is None or not os.path.exists(lib):
        pytest.skip('needs cuobjdump and the built library')
    out = subprocess.run(['cuobjdump', '-res-usage', lib], capture_output=True, text=True, check=True).stdout
    lines = out.splitlines()
    found = [(lines[i], lines[i + 1]) for i in range(len(lines) - 1) if 'kb_pcen' in lines[i]]
    assert len(found) == 4, found
    for name, res in found:
        m = re.search(r'REG:(\d+) STACK:(\d+)', res)
        assert m and int(m.group(1)) <= 128 and int(m.group(2)) == 0, (name, res)


# ------------------------------------------------------------------------------ the layer
def test_layer_validation():
    from kapre_b200.time_frequency import PCEN
    for kw in ({'gain': -0.1}, {'bias': 0.0}, {'power': 0.0}, {'eps': 0.0}, {'time_constant': 0.0},
               {'smooth_coef': -0.01}, {'smooth_coef': 1.01}, {'gain': float('nan')}, {'bias': float('inf')},
               {'power': [0.5, float('nan')]}, {'sample_rate': 0}, {'hop_length': -1}, {'gain': [[1.0]]},
               {'bias': []}, {'data_format': 'channels_middle'}):
        with pytest.raises(ValueError):
            PCEN(**kw)
    PCEN(smooth_coef=0.0)
    PCEN(smooth_coef=1.0, gain=0.0)


def test_layer_config_round_trip():
    from kapre_b200.time_frequency import PCEN
    import kapre
    assert kapre.time_frequency.PCEN is PCEN
    import kapre_b200
    assert 'PCEN' not in kapre_b200.__all__
    from kapre_b200 import time_frequency
    assert 'PCEN' in time_frequency.__all__
    layer = PCEN(sample_rate=16000, hop_length=160, time_constant=0.3, gain=[0.9, 0.8, 0.7], bias=1.5, power=0.25,
                 eps=1e-5, data_format='channels_first', name='pcen_x', trainable=False)
    cfg = layer.get_config()
    assert cfg['sample_rate'] == 16000 and cfg['hop_length'] == 160 and cfg['time_constant'] == 0.3
    assert cfg['smooth_coef'] is None and cfg['gain'] == [0.9, 0.8, 0.7] and cfg['bias'] == 1.5
    assert cfg['power'] == 0.25 and cfg['eps'] == 1e-5 and cfg['data_format'] == 'channels_first'
    assert cfg['name'] == 'pcen_x' and cfg['trainable'] is False
    again = PCEN.from_config(cfg)
    assert again.get_config() == cfg
    assert abs(layer.smooth_coef_value - PR.smooth_coef(0.3, 16000, 160)) < 1e-12
    assert PCEN(smooth_coef=0.1).get_config()['smooth_coef'] == 0.1


def test_layer_weights_before_build():
    from kapre_b200.time_frequency import PCEN
    layer = PCEN(gain=[0.9] * 4)
    assert layer.weights == [] and not layer.built
    with pytest.raises(ValueError):
        layer.count_params()


def test_layer_builds_weights_on_the_cpu_description():
    """Weight shapes and the band check come from the band count alone (``build``), without a GPU."""
    from kapre_b200.time_frequency import PCEN
    layer = PCEN(gain=[0.9, 0.8, 0.7, 0.6], power=0.4, smooth_coef=[0.1] * 4)
    layer.build(4, torch.device('cpu'))
    w = layer.weights
    assert [tuple(t.shape) for t in w] == [(4,), (), (), (4,)]
    assert all(t.dtype == torch.float32 and t.requires_grad for t in w)
    assert layer.count_params() == 4 + 1 + 1 + 4
    np.testing.assert_allclose(w[0].detach().numpy(), [0.9, 0.8, 0.7, 0.6], rtol=1e-7)
    assert math.isclose(float(w[1].detach()), 2.0) and math.isclose(float(w[2].detach()), 0.4, rel_tol=1e-7)
    with pytest.raises(ValueError):
        PCEN(gain=[0.9, 0.8]).build(3, torch.device('cpu'))
    frozen = PCEN(trainable=False)
    frozen.build(7, torch.device('cpu'))
    assert not any(t.requires_grad for t in frozen.weights) and frozen.count_params() == 4
