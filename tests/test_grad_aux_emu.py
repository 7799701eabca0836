"""Gradients of the layers next to the hot path, on the CPU: the float64 restatement (grad_ref_adjacent.py) against
the oracle, and the backward bodies of grad_aux_core.cuh (run by a CPU emulation) against the restatement's
vector-Jacobian products.

The emulated bodies compute in float32 like the kernels; the linear ones sum at most a handful of terms per output
(Delta: 2n taps per mirror image, Frame / Energy: ceil(frame_length / hop) frames), so they are held to 1e-5 of the
largest reference value.  Phase and magnitude + phase divide by |X| (and |X|^2): 1e-5 with test signals that keep
|X| away from zero except at the deliberate exact zeros.
"""
import ctypes
import hashlib
import os
import subprocess
import tempfile

import numpy as np
import pytest
import torch

import grad_ref as R
import grad_ref_adjacent as RA
from oracle import reference as ref

LL = ctypes.c_longlong
FMTS = ('channels_first', 'channels_last')
CL, CF = 'channels_last', 'channels_first'

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, 'emu', 'kb_emu_grad_aux.cpp')
_CSRC = os.path.join(_HERE, '..', 'kapre_b200', 'csrc')
_lib_handle = None


def _lib():
    """tests/emu/kb_emu_grad_aux.cpp built with g++ into the temporary directory (keyed by the sources' contents, so
    the checkout itself may be read-only)."""
    global _lib_handle
    if _lib_handle is None:
        h = hashlib.sha256()
        for f in [_SRC] + sorted(os.path.join(_CSRC, n) for n in os.listdir(_CSRC) if n.endswith(('.h', '.cuh'))):
            with open(f, 'rb') as fh:
                h.update(fh.read())
        out = os.path.join(tempfile.gettempdir(), 'kapre_b200_emu_grad_aux_%s.so' % h.hexdigest()[:16])
        if not os.path.exists(out):
            tmp = '%s.%d.tmp' % (out, os.getpid())
            subprocess.check_call(['g++', '-O2', '-std=c++17', '-shared', '-fPIC', '-DKB_HOST_EMU', '-Wno-unknown-pragmas',
                                   '-o', tmp, _SRC])
            os.replace(tmp, out)
        lib = ctypes.CDLL(out)
        lib.kb_emu_pad_index.restype = ctypes.c_longlong
        lib.kb_emu_pad_index.argtypes = [ctypes.c_longlong, ctypes.c_longlong, ctypes.c_int]
        _lib_handle = lib
    return _lib_handle


def _fp(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _strides(a, order):
    """Element strides of the numpy array `a` along its axes listed in `order`."""
    return np.array([a.strides[i] // a.itemsize for i in order], dtype=np.int64)


def _close(got, want, tol=1e-5):
    want = np.asarray(want)
    scale = max(float(np.abs(want).max()), 1e-30)
    err = float(np.abs(np.asarray(got) - want).max())
    assert err <= tol * scale, (err, scale)


def _vjp(fn, x, g):
    return R.vjp(fn, torch.from_numpy(np.asarray(x)).to(torch.complex128 if np.iscomplexobj(x) else torch.float64),
                 torch.from_numpy(np.asarray(g)))


# ------------------------------------------------------------------------------ the restatement
@pytest.mark.parametrize('fmt', FMTS)
def test_restatement_forward_equals_oracle(fmt):
    rng = np.random.default_rng(3)
    X = rng.standard_normal((2, 3, 5, 7)) + 1j * rng.standard_normal((2, 3, 5, 7))
    np.testing.assert_allclose(RA.phase(torch.from_numpy(X)).numpy(), ref.phase(X), rtol=0, atol=1e-15)

    for n_fft, win, hop, pb, pe, db in [(512, 512, 128, False, False, None), (400, 400, 160, True, True, None),
                                        (256, 200, 64, False, True, (1.0, 1e-5, 15.0))]:
        x = rng.standard_normal((2, 2000, 1) if fmt == CL else (2, 1, 2000))
        want = ref.stft_mag_phase_layer(x, n_fft, win, hop, None, pb, pe, db is not None,
                                        *(db[1], db[0], db[2]) if db else (1e-5, 1.0, 80.0), fmt, fmt)
        got = RA.mag_phase(torch.from_numpy(x), n_fft, win, hop, None, pb, pe, fmt, fmt, db)
        np.testing.assert_allclose(got.numpy(), want, rtol=0, atol=1e-9 * np.abs(want).max())

    spec = rng.standard_normal((2, 11, 6, 2) if fmt == CL else (2, 2, 11, 6))
    for mode in ('symmetric', 'reflect', 'constant'):
        for win in (3, 5, 9):           # T = 11 > n: the kernels' extension is tf.pad's
            np.testing.assert_allclose(RA.delta(torch.from_numpy(spec), win, mode, fmt).numpy(),
                                       ref.delta(spec, win, mode, fmt), rtol=0, atol=1e-12)
    np.testing.assert_allclose(RA.concat_frequency_map(torch.from_numpy(spec), fmt).numpy(),
                               ref.concat_frequency_map(spec, fmt), rtol=0, atol=0)

    wav = rng.standard_normal((2, 1000, 2) if fmt == CL else (2, 2, 1000))
    for fl, hop, pe in [(256, 64, False), (256, 64, True), (100, 100, True), (100, 130, False), (100, 130, True)]:
        if hop <= fl:
            np.testing.assert_allclose(RA.frame(torch.from_numpy(wav), fl, hop, pe, 0.5, fmt).numpy(),
                                       ref.frame_layer(wav, fl, hop, pe, 0.5, fmt), rtol=0, atol=0)
        sr, dur = 16000, 0.1
        np.testing.assert_allclose(RA.energy(torch.from_numpy(wav), fl, hop, pe, 0.5, dur / (fl / sr), fmt).numpy(),
                                   ref.energy_layer(wav, sr, dur, fl, hop, pe, 0.5, fmt), rtol=1e-12)

    mono = rng.standard_normal((3, 20, 16, 1) if fmt == CL else (3, 1, 20, 16))
    tm = np.array([[[2, 3]], [[0, 0]], [[15, 4]]], np.int32)
    fm = np.array([[[5, 1], [9, 0]], [[0, 2], [14, 1]], [[3, 3], [3, 0]]], np.int32)
    np.testing.assert_allclose(RA.spec_augment(torch.from_numpy(mono), tm, fm, -1.5, fmt).numpy(),
                               ref.spec_augment(mono, tm, fm, -1.5, fmt), rtol=0, atol=0)


def test_pad_index_matches_kernel():
    lib = _lib()
    for T in range(1, 12):
        for mode in range(3):
            for t in range(-6, T + 6):
                assert RA.pad_index(t, T, mode) == lib.kb_emu_pad_index(t, T, mode), (t, T, mode)


# ------------------------------------------------------------------------------ emulated backward bodies
@pytest.mark.parametrize('mode', ['symmetric', 'reflect', 'constant'])
@pytest.mark.parametrize('win', [3, 5, 9])
@pytest.mark.parametrize('fmt', FMTS)
def test_emu_delta_backward(mode, win, fmt):
    rng = np.random.default_rng(win)
    n = (win - 1) // 2
    md = {'symmetric': 0, 'reflect': 1, 'constant': 2}[mode]
    inv = np.float32(1.0 / (2 * sum(m * m for m in range(1, n + 1))))
    for T in list(range(1, 2 * n + 4)) + [4 * n + 7]:
        shape = (2, T, 5, 2) if fmt == CL else (2, 2, T, 5)
        x = rng.standard_normal(shape)
        g = rng.standard_normal(shape).astype(np.float32)
        _, want = _vjp(lambda t: RA.delta(t, win, mode, fmt), x, g.astype(np.float64))
        outer, inner = (2, 10) if fmt == CL else (4, 5)
        gx = np.full(shape, np.nan, np.float32)
        assert _lib().kb_emu_delta_bwd(_fp(g), _fp(gx), LL(outer), LL(T), LL(inner), n, ctypes.c_float(inv), md) == 0
        _close(gx, want.numpy())


def _wave_strides(a, fmt):
    return _strides(a, (0, 2, 1) if fmt == CL else (0, 1, 2))


def _frames_strides(a, fmt):
    return _strides(a, (0, 3, 1, 2) if fmt == CL else (0, 1, 2, 3))


FRAME_CASES = [(64, 16, False), (64, 16, True), (50, 50, False), (50, 50, True), (30, 45, False), (30, 45, True),
               (7, 3, True)]


@pytest.mark.parametrize('case', FRAME_CASES, ids=lambda c: 'fl%d_h%d_pe%d' % c)
@pytest.mark.parametrize('fmt', FMTS)
def test_emu_frame_and_energy_backward(case, fmt):
    fl, hop, pe = case
    rng = np.random.default_rng(fl + hop + pe)
    B, C, L = 2, 3, 311
    x = rng.standard_normal((B, L, C) if fmt == CL else (B, C, L)).astype(np.float32)
    T = ref.num_frames(L, fl, hop, pe)
    if hop <= fl:                     # Frame requires frame_length >= hop_length
        g = rng.standard_normal((B, T, fl, C) if fmt == CL else (B, C, T, fl)).astype(np.float32)
        _, want = _vjp(lambda t: RA.frame(t, fl, hop, pe, 0.25, fmt), x, g.astype(np.float64))
        gx = np.full_like(x, np.nan)
        assert _lib().kb_emu_frame_bwd(_fp(g), _fp(_frames_strides(g, fmt)), _fp(gx), _fp(_wave_strides(gx, fmt)),
                                       B, C, L, T, fl, hop) == 0
        _close(gx, want.numpy())
    scale = 0.37
    g = rng.standard_normal((B, T, C) if fmt == CL else (B, C, T)).astype(np.float32)
    _, want = _vjp(lambda t: RA.energy(t, fl, hop, pe, 0.25, scale, fmt), x, g.astype(np.float64))
    gx = np.full_like(x, np.nan)
    assert _lib().kb_emu_energy_bwd(_fp(x), _fp(_wave_strides(x, fmt)), _fp(g), _fp(_wave_strides(g, fmt)), _fp(gx),
                                    _fp(_wave_strides(gx, fmt)), B, C, L, T, fl, hop, ctypes.c_float(scale)) == 0
    _close(gx, want.numpy())
    if hop > fl:                      # samples in the gaps between frames get exactly 0
        s = np.arange(L)
        gap = (s % hop >= fl) & (s < T * hop)
        assert np.all((gx[:, gap, :] if fmt == CL else gx[:, :, gap]) == 0)


def test_emu_frame_backward_channels_last_strides():
    """A channels_last gradient read through the strides of a transposed view, into a channels_first gx."""
    rng = np.random.default_rng(9)
    B, C, L, fl, hop = 1, 2, 97, 16, 5
    T = ref.num_frames(L, fl, hop, True)
    g_cl = rng.standard_normal((B, T, fl, C)).astype(np.float32)
    g_cf = g_cl.transpose(0, 3, 1, 2)           # same memory, (b, c, t, n) view
    _, want = _vjp(lambda t: RA.frame(t, fl, hop, True, 0.0, CF), rng.standard_normal((B, C, L)),
                   np.ascontiguousarray(g_cf).astype(np.float64))
    gx = np.full((B, C, L), np.nan, np.float32)
    assert _lib().kb_emu_frame_bwd(_fp(g_cl), _fp(_strides(g_cf, (0, 1, 2, 3))), _fp(gx), _fp(_strides(gx, (0, 1, 2))),
                                   B, C, L, T, fl, hop) == 0
    _close(gx, want.numpy())


def test_emu_phase_backward():
    rng = np.random.default_rng(1)
    X = (rng.standard_normal(301) + 1j * rng.standard_normal(301)).astype(np.complex64)
    X[[0, 7, 300]] = 0
    g = rng.standard_normal(301).astype(np.float32)
    gX = np.full_like(X, np.nan)
    assert _lib().kb_emu_phase_bwd(_fp(X), _fp(g), _fp(gX), LL(X.size)) == 0
    _, want = _vjp(RA.phase, X.astype(np.complex128), g.astype(np.float64))
    _close(gX, want.numpy())
    assert gX[0] == 0 and gX[7] == 0 and gX[300] == 0


@pytest.mark.parametrize('fmt', FMTS)
@pytest.mark.parametrize('halves', ['both', 'mag', 'phase'])
def test_emu_mag_phase_backward(fmt, halves):
    rng = np.random.default_rng(len(halves) + len(fmt))
    B, C, T, F = 2, 2, 5, 9
    shape = (B, T, F, C) if fmt == CL else (B, C, T, F)
    X = (rng.standard_normal(shape) + 1j * rng.standard_normal(shape)).astype(np.complex64)
    X.reshape(-1)[[3, 17]] = 0
    gshape = (B, T, F, 2 * C) if fmt == CL else (B, 2 * C, T, F)
    g = rng.standard_normal(gshape).astype(np.float32)
    if halves == 'mag':
        (g[..., C:] if fmt == CL else g[:, C:])[...] = 0
    elif halves == 'phase':
        (g[..., :C] if fmt == CL else g[:, :C])[...] = 0
    gm, gp = (g[..., :C], g[..., C:]) if fmt == CL else (g[:, :C], g[:, C:])
    order = (0, 3, 1, 2) if fmt == CL else (0, 1, 2, 3)
    Xf = X.view(np.float32)           # complex strides counted in complex elements
    gX = np.full_like(X, np.nan)
    lib = _lib()
    null = ctypes.c_void_p(None)
    assert lib.kb_emu_mag_phase_bwd(
        _fp(Xf), _fp(_strides(X, order)),
        _fp(gm) if halves != 'phase' else null, _fp(_strides(gm, order)),
        _fp(gp) if halves != 'mag' else null, _fp(_strides(gp, order)),
        _fp(gX), _fp(_strides(gX, order)), LL(B), LL(C), LL(T), LL(F), int(fmt == CL)) == 0

    def f(t):
        return torch.cat([t.abs(), torch.angle(t)], dim=3 if fmt == CL else 1)
    _, want = _vjp(f, X.astype(np.complex128), g.astype(np.float64))
    _close(gX, want.numpy())
    assert gX.reshape(-1)[3] == 0 and gX.reshape(-1)[17] == 0


@pytest.mark.parametrize('fmt', FMTS)
def test_emu_concat_frequency_map_backward(fmt):
    rng = np.random.default_rng(2)
    B, C, T, F = 2, 3, 4, 5
    x = rng.standard_normal((B, T, F, C) if fmt == CL else (B, C, T, F))
    g = rng.standard_normal((B, T, F, C + 1) if fmt == CL else (B, C + 1, T, F)).astype(np.float32)
    gx = np.full(x.shape, np.nan, np.float32)
    assert _lib().kb_emu_concat_fm_bwd(_fp(g), _fp(gx), LL(B), LL(C), LL(T), LL(F), int(fmt == CL)) == 0
    _, want = _vjp(lambda t: RA.concat_frequency_map(t, fmt), x, g.astype(np.float64))
    np.testing.assert_array_equal(gx, want.numpy().astype(np.float32))
