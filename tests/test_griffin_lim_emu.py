"""Griffin-Lim on the CPU: the float64 restatement (gl_ref.py) pinned to ``torchaudio.functional.griffinlim``, the
element passes of gl_core.cuh (run by a CPU emulation) against the restatement, the random-phase hash bit for bit,
and the ``GriffinLim`` layer's validation and config.

Tolerances.  The init pass rounds S cos and S sin once each, after a phasor within an ulp or two: X is held to 4e-7
of |S| per element.  The projection rounds A = Y - beta Yprev once (an FMA), then |A| (an FMA, a product, a square
root), the quotient S / (|A| + 1e-16) and the two products: a few ulps of |S|, held to 1e-6 of |S|.
"""
import ctypes
import hashlib
import os
import subprocess
import tempfile

import numpy as np
import pytest
import torch

import gl_ref as GR
from emu_harness import Checked

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, 'emu', 'kb_emu_gl.cpp')
_CSRC = os.path.join(_HERE, '..', 'kapre_b200', 'csrc')
_lib_handle = None
CL, CF = 'channels_last', 'channels_first'


def _lib():
    """tests/emu/kb_emu_gl.cpp built with g++ into the temporary directory (keyed by the sources' contents, so the
    checkout itself may be read-only)."""
    global _lib_handle
    if _lib_handle is None:
        h = hashlib.sha256()
        for f in [_SRC] + sorted(os.path.join(_CSRC, n) for n in os.listdir(_CSRC) if n.endswith(('.h', '.cuh'))):
            with open(f, 'rb') as fh:
                h.update(fh.read())
        out = os.path.join(tempfile.gettempdir(), 'kapre_b200_emu_gl_%s.so' % h.hexdigest()[:16])
        if not os.path.exists(out):
            tmp = '%s.%d.tmp' % (out, os.getpid())
            subprocess.check_call(['g++', '-O2', '-std=c++17', '-shared', '-fPIC', '-DKB_HOST_EMU', '-Wno-unknown-pragmas',
                                   '-o', tmp, _SRC])
            os.replace(tmp, out)
        lib = ctypes.CDLL(out)
        P, I = ctypes.c_void_p, ctypes.c_int
        lib.kb_emu_gl_init.argtypes = [P, P, I, I, I, I, I, ctypes.c_ulonglong, P]
        lib.kb_emu_gl_project.argtypes = [P, P, I, I, I, I, P, P, ctypes.c_float, P]
        lib.kb_emu_gl_u.argtypes = [ctypes.c_ulonglong, ctypes.c_longlong]
        lib.kb_emu_gl_u.restype = ctypes.c_float
        lib.kb_emu_gl_phasor.argtypes = [ctypes.c_float, P, P]
        _lib_handle = Checked(lib)
    return _lib_handle


def _dims_strides(S, fmt):
    """(B, C, T, F) and the (b, c, t, f) element strides of a (B, T, F, C) channels_last / (B, C, T, F) array."""
    s = [v // 4 for v in S.strides]
    if fmt == CL:
        B, T, F, C = S.shape
        return (B, C, T, F), np.array([s[0], s[3], s[1], s[2]], np.int64)
    B, C, T, F = S.shape
    return (B, C, T, F), np.array(s, np.int64)


def _canon(S, fmt):
    return np.ascontiguousarray(np.transpose(S, (0, 3, 1, 2)) if fmt == CL else S).astype(np.float64)


def emu_init(S, fmt, init, seed):
    (B, C, T, F), ss = _dims_strides(S, fmt)
    X = np.full((B, C, T, F), np.nan, np.complex64)
    _lib().kb_emu_gl_init(S.ctypes.data, ss.ctypes.data, B, C, T, F, init, seed, X.ctypes.data)
    return X


def emu_project(S, fmt, Y, Yprev, beta, out=None):
    (B, C, T, F), ss = _dims_strides(S, fmt)
    X = np.full((B, C, T, F), np.nan, np.complex64) if out is None else out
    _lib().kb_emu_gl_project(S.ctypes.data, ss.ctypes.data, B, C, T, F, Y.ctypes.data,
                             None if Yprev is None else Yprev.ctypes.data, beta, X.ctypes.data)
    return X


def _magnitudes(rng, fmt, B, C, T, F):
    """Positive, over three decades."""
    return (10.0 ** rng.uniform(-1.5, 1.5, size=(B, T, F, C) if fmt == CL else (B, C, T, F))).astype(np.float32)


def _complex(rng, shape):
    return (rng.standard_normal(shape) + 1j * rng.standard_normal(shape)).astype(np.complex64)


def _within(got, want, S, rel):
    err = np.abs(got.astype(np.complex128) - want)
    assert np.all(err <= rel * S), float((err / np.maximum(S, 1e-300)).max())


# ------------------------------------------------------------------------------ the restatement
def _chirp(C, L, seed=0):
    t = np.arange(L) / 22050.0
    x = [np.sin(2 * np.pi * (200 + 1500 * c + 900 * t) * t) for c in range(C)]
    return np.stack(x) + 0.05 * np.random.default_rng(seed).standard_normal((C, L))


@pytest.mark.parametrize('momentum', [0.0, 0.99])
def test_restatement_matches_torchaudio(momentum):
    """With torch's centred transforms and A_0 = 1 the restatement is torchaudio's loop (spectrograms there are
    (..., freq, time))."""
    ta = pytest.importorskip('torchaudio')
    n_fft, hop = 1024, 256
    win = torch.hann_window(n_fft, dtype=torch.float64)
    x = torch.from_numpy(_chirp(2, 22050))
    S = torch.stft(x, n_fft, hop, window=win, return_complex=True).abs()

    def stft_fn(y):
        return torch.stft(y, n_fft, hop, window=win, return_complex=True).transpose(-1, -2)

    def istft_fn(X):
        return torch.istft(X.transpose(-1, -2), n_fft, hop, window=win)

    got = GR.griffin_lim(S.transpose(-1, -2), stft_fn, istft_fn, 8, momentum, 1.0)
    want = ta.functional.griffinlim(S, win, n_fft, hop, n_fft, 1.0, 8, momentum, None, False)
    assert got.shape == want.shape
    assert float((got - want).abs().max()) <= 1e-12 * float(want.abs().max())


def test_kapre_instance_reconstructs():
    """Over the oracle's pair: the true phase with no iteration gives the signal back where the frames cover it
    fully, and from zero phase the spectral convergence falls with the iterations (momentum 0 cannot increase it)."""
    n_fft, hop = 512, 128
    stft_fn, istft_fn = GR.kapre_pair(n_fft, n_fft, hop)
    x = torch.from_numpy(_chirp(1, 8192, seed=1))
    X = stft_fn(x)
    y = GR.griffin_lim(X.abs(), stft_fn, istft_fn, 0, 0.0, X / X.abs())
    L = y.shape[-1]
    assert L == (X.shape[-2] - 1) * hop + n_fft
    torch.testing.assert_close(y[..., n_fft - hop:L - (n_fft - hop)], x[..., n_fft - hop:L - (n_fft - hop)],
                               rtol=0, atol=1e-10)
    sc = [GR.spectral_convergence(GR.griffin_lim(X.abs(), stft_fn, istft_fn, n, 0.0, 1.0), X.abs(), stft_fn)
          for n in (0, 1, 4, 8)]
    assert all(a >= b for a, b in zip(sc, sc[1:])) and sc[-1] < 0.8 * sc[0], sc


# ------------------------------------------------------------------------------ the random-phase hash
@pytest.mark.parametrize('seed', [0, 1, 12345, 2 ** 63, 2 ** 64 - 1])
def test_hash_bit_for_bit(seed):
    lib = _lib()
    idx = list(range(0, 600)) + [2 ** 31 - 1, 2 ** 32, 3 * 2 ** 40 + 7, 2 ** 62 + 5]
    for i in idx:
        assert lib.kb_emu_gl_u(seed, i) == GR.phase_u(seed, i), (seed, i)
    u = np.array([GR.phase_u(seed, i) for i in range(4096)])
    np.testing.assert_array_equal(GR.phase_u_table(seed, 4096), u)
    assert 0.0 <= u.min() and u.max() < 1.0 and abs(u.mean() - 0.5) < 0.03     # a sanity check of the spread


def test_seeds_give_different_phases():
    a = [GR.phase_u(0, i) for i in range(64)]
    b = [GR.phase_u(1, i) for i in range(64)]
    assert sum(x == y for x, y in zip(a, b)) <= 1


def test_phasor_within_ulps():
    lib = _lib()
    s, c = ctypes.c_float(), ctypes.c_float()
    for u in np.concatenate([np.arange(0, 1 << 24, 4099) / float(1 << 24), [0.0, 0.25, 0.5, 0.75, 1 - 2 ** -24]]):
        u32 = np.float32(u)
        lib.kb_emu_gl_phasor(u32, ctypes.byref(s), ctypes.byref(c))
        a = 2 * np.pi * float(u32)
        for got, want in ((s.value, np.sin(a)), (c.value, np.cos(a))):
            assert abs(got - want) <= 2 * float(np.spacing(np.float32(max(abs(want), 2 ** -24)))), (u, got, want)


# ------------------------------------------------------------------------------ the emulated bodies
def _views(rng, fmt):
    """A contiguous S and a strided view of a larger one (every other frame, a channel slice), both 3 x 2 channels."""
    full = _magnitudes(rng, fmt, 3, 3, 14, 33)
    t_ax, c_ax = (1, 3) if fmt == CL else (2, 1)
    sl = [slice(None)] * 4
    sl[t_ax] = slice(None, None, 2)
    sl[c_ax] = slice(1, 3)
    return [_magnitudes(rng, fmt, 3, 2, 7, 33), full[tuple(sl)]]


@pytest.mark.parametrize('fmt', [CF, CL])
@pytest.mark.parametrize('init', [0, 1])
def test_emulated_init(fmt, init):
    rng = np.random.default_rng(10 + init)
    for S in _views(rng, fmt):
        Sc = _canon(S, fmt)
        X = emu_init(S, fmt, init, seed=77)
        B, C, T, F = Sc.shape
        want = Sc * (GR.random_phase(77, B, C, T, F).numpy() if init == 1 else 1.0)
        _within(X, want, Sc, 4e-7)
        if init == 0:
            assert np.all(X.imag == 0) and np.array_equal(X.real, Sc.astype(np.float32))


def test_emulated_init_does_not_depend_on_layout():
    rng = np.random.default_rng(12)
    S = _magnitudes(rng, CF, 2, 3, 5, 17)
    Scl = np.ascontiguousarray(np.transpose(S, (0, 2, 3, 1)))
    np.testing.assert_array_equal(emu_init(S, CF, 1, 5), emu_init(Scl, CL, 1, 5))


def _project_ref(Sc, Y, Yprev, beta):
    A = Y.astype(np.complex128)
    if Yprev is not None:
        A = A - np.float64(np.float32(beta)) * Yprev.astype(np.complex128)
    return Sc * A / (np.abs(A) + 1e-16)


@pytest.mark.parametrize('fmt', [CF, CL])
@pytest.mark.parametrize('case', ['momentum', 'first', 'momentum0'])
def test_emulated_project(fmt, case):
    rng = np.random.default_rng(20)
    beta = {'momentum': 0.99 / 1.99, 'first': 0.99 / 1.99, 'momentum0': 0.0}[case]
    for S in _views(rng, fmt):
        Sc = _canon(S, fmt)
        Y = _complex(rng, Sc.shape)
        Yprev = None if case == 'first' else _complex(rng, Sc.shape)
        X = emu_project(S, fmt, Y, Yprev, beta)
        _within(X, _project_ref(Sc, Y, Yprev, beta), Sc, 1e-6)
        if case == 'momentum0':                   # beta = 0 reads Yprev but gives the first-iteration result
            np.testing.assert_array_equal(X, emu_project(S, fmt, Y, None, beta))


def test_emulated_project_zero_and_in_place():
    """A = 0 gives X = 0 (not NaN); writing X over Yprev, as the library does, gives the same bits."""
    rng = np.random.default_rng(21)
    S = _magnitudes(rng, CF, 2, 2, 6, 9)
    Y = _complex(rng, S.shape)
    Yprev = _complex(rng, S.shape)
    Y[0, 1, 2, :] = 0
    Yprev[0, 1, 2, :] = 0
    Y[1, 0, :, 4] = 0
    beta = 0.5 / 1.5
    X = emu_project(S, CF, Y, Yprev, beta)
    assert np.all(X[0, 1, 2, :] == 0) and np.all(np.isfinite(X))
    _within(X, _project_ref(S.astype(np.float64), Y, Yprev, beta), S.astype(np.float64), 1e-6)
    buf = Yprev.copy()
    np.testing.assert_array_equal(emu_project(S, CF, Y, buf, beta, out=buf), X)


def test_emulated_empty():
    S = np.zeros((0, 1, 4, 9), np.float32)
    assert emu_init(S, CF, 1, 0).size == 0
    assert emu_project(S, CF, np.zeros(S.shape, np.complex64), None, 0.0).size == 0


def test_kernel_register_and_spill_budget():
    """The two Griffin-Lim element kernels do not spill."""
    import re
    import shutil
    lib = os.path.join(_HERE, '..', 'kapre_b200', '_lib', 'libkapre_b200.so')
    if shutil.which('cuobjdump') is None or not os.path.exists(lib):
        pytest.skip('needs cuobjdump and the built library')
    out = subprocess.run(['cuobjdump', '-res-usage', lib], capture_output=True, text=True, check=True).stdout
    lines = out.splitlines()
    found = [(lines[i], lines[i + 1]) for i in range(len(lines) - 1) if 'kb_gl_' in lines[i]]
    assert len(found) == 2, found
    for name, res in found:
        m = re.search(r'REG:(\d+) STACK:(\d+).*LOCAL:(\d+)', res)
        assert m and int(m.group(1)) <= 64 and int(m.group(2)) == 0 and int(m.group(3)) == 0, (name, res)


# ------------------------------------------------------------------------------ the layer
def test_layer_validation():
    from kapre_b200.time_frequency import GriffinLim
    for kw in ({'n_iter': -1}, {'n_iter': 2.0}, {'n_iter': True}, {'momentum': 1.0}, {'momentum': -0.1},
               {'momentum': float('nan')}, {'momentum': '0.5'}, {'init': 'zeros'}, {'seed': -1}, {'seed': 2 ** 64},
               {'seed': 1.5}, {'seed': True}, {'input_data_format': 'channels_middle'},
               {'output_data_format': 'channels_middle'}):
        with pytest.raises(ValueError):
            GriffinLim(**kw)
    GriffinLim(n_iter=0, momentum=0.0, init='ones', seed=None)
    GriffinLim(seed=2 ** 64 - 1, n_iter=np.int64(3))


def test_layer_config_round_trip_and_alias():
    from kapre_b200.time_frequency import GriffinLim
    import kapre
    import kapre_b200
    from kapre_b200 import time_frequency
    assert kapre.time_frequency.GriffinLim is GriffinLim
    assert 'GriffinLim' in time_frequency.__all__ and 'GriffinLim' not in kapre_b200.__all__
    assert time_frequency.get_registered_object('Kapre>GriffinLim') is GriffinLim
    layer = GriffinLim(n_fft=512, hop_length=128, window_name='hamming_window', n_iter=10, momentum=0.5, init='ones',
                       seed=9, input_data_format='channels_first', output_data_format='channels_last', name='gl_x')
    cfg = layer.get_config()
    assert cfg['n_fft'] == 512 and cfg['win_length'] == 512 and cfg['hop_length'] == 128
    assert cfg['window_name'] == 'hamming_window' and cfg['n_iter'] == 10 and cfg['momentum'] == 0.5
    assert cfg['init'] == 'ones' and cfg['seed'] == 9 and cfg['name'] == 'gl_x'
    assert cfg['input_data_format'] == 'channels_first' and cfg['output_data_format'] == 'channels_last'
    assert GriffinLim.from_config(cfg).get_config() == cfg
    d = GriffinLim(n_fft=400).get_config()
    assert d['win_length'] == 400 and d['hop_length'] == 100 and d['seed'] == 0 and d['init'] == 'random'
    assert d['n_iter'] == 32 and d['momentum'] == 0.99
    assert GriffinLim(seed=None).get_config()['seed'] is None
