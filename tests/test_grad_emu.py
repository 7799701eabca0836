"""Gradients on the CPU: the float64 restatement (grad_ref.py) against the oracle and TensorFlow's tie rules, and
the backward passes' kernel bodies (grad_core.cuh, run by the CPU emulation together with the existing transform
bodies and their adjoint windows) against the restatement's vector-Jacobian products."""
import ctypes
import hashlib
import os
import subprocess
import tempfile

import numpy as np
import pytest
import torch

import emu_harness as E
import grad_ref as R
from oracle import reference as ref
from emu_harness import Checked

LL = ctypes.c_longlong
FMTS = ('channels_first', 'channels_last')


def _fp(a):
    return a.ctypes.data_as(ctypes.c_void_p)


_HERE = os.path.dirname(os.path.abspath(__file__))
_GRAD_SRC = os.path.join(_HERE, 'emu', 'kb_emu_grad.cpp')
_CSRC = os.path.join(_HERE, '..', 'kapre_b200', 'csrc')
_grad_lib_handle = None


def _grad_lib():
    """The CPU emulation of grad_core.cuh (tests/emu/kb_emu_grad.cpp), built with g++ into the temporary directory
    (keyed by the sources' contents, so the checkout itself may be read-only)."""
    global _grad_lib_handle
    if _grad_lib_handle is None:
        h = hashlib.sha256()
        for f in [_GRAD_SRC] + sorted(os.path.join(_CSRC, n) for n in os.listdir(_CSRC) if n.endswith(('.h', '.cuh'))):
            with open(f, 'rb') as fh:
                h.update(fh.read())
        out = os.path.join(tempfile.gettempdir(), 'kapre_b200_emu_grad_%s.so' % h.hexdigest()[:16])
        if not os.path.exists(out):
            tmp = '%s.%d.tmp' % (out, os.getpid())
            subprocess.check_call(['g++', '-O2', '-std=c++17', '-shared', '-fPIC', '-DKB_HOST_EMU', '-Wno-unknown-pragmas',
                                   '-o', tmp, _GRAD_SRC])
            os.replace(tmp, out)
        _grad_lib_handle = Checked(ctypes.CDLL(out))
    return _grad_lib_handle


def _spec_strides(shape, fmt):
    """(b, c, t, k) element strides of a contiguous spectrum array in `fmt`."""
    if fmt == 'channels_last':
        B, T, F, C = shape
        return T * F * C, 1, F * C, C
    B, C, T, F = shape
    return C * T * F, T * F, F, 1


def _wave(rng, B, C, L, fmt):
    x = rng.standard_normal((B, L, C) if fmt == 'channels_last' else (B, C, L))
    return x.astype(np.float32)


def _spec(rng, B, C, T, F, fmt):
    shape = (B, T, F, C) if fmt == 'channels_last' else (B, C, T, F)
    return (rng.standard_normal(shape) + 1j * rng.standard_normal(shape)).astype(np.complex64)


def _close(got, want, rtol=3e-5):
    want = np.asarray(want)
    scale = max(float(np.abs(want).max()), 1e-30)
    err = float(np.abs(np.asarray(got) - want).max())
    assert err <= rtol * scale, (err, scale)


# ------------------------------------------------------------------------------ the restatement
@pytest.mark.parametrize('seed', range(4))
def test_restatement_forward_equals_oracle(seed):
    rng = np.random.default_rng(seed)
    n_fft = int(rng.choice([96, 256, 400, 512]))
    win = int(rng.choice([n_fft // 2, n_fft, n_fft + 16]))
    hop = int(rng.choice([win // 4, win // 2, win + 8]))
    pb, pe = bool(rng.integers(2)), bool(rng.integers(2))
    if pb and hop > n_fft:
        pb = False
    fi, fo = FMTS[rng.integers(2)], FMTS[rng.integers(2)]
    wname = [None, 'hamming_window'][rng.integers(2)]
    x = _wave(rng, 2, 2, 3 * n_fft + 37, fi).astype(np.float64)
    s_ref = ref.stft_layer(x, n_fft, win, hop, wname, pb, pe, fi, fo)
    s = R.stft(torch.from_numpy(x), n_fft, win, hop, wname, pb, pe, fi, fo)
    np.testing.assert_allclose(s.numpy(), s_ref, rtol=0, atol=1e-9 * np.abs(s_ref).max())
    m = R.magnitude(s)
    fb = R.filterbank_mel(n_fft, 16000, 40)
    fbo = R.apply_filterbank(m, fb, fo)
    np.testing.assert_allclose(fbo.numpy(), ref.apply_filterbank(np.abs(s_ref), fb.astype(np.float64), fo), rtol=1e-10,
                               atol=1e-12)
    db = R.magnitude_to_decibel(fbo, 1.0, 1e-5, 30.0)
    np.testing.assert_allclose(db.numpy(), ref.magnitude_to_decibel(fbo.numpy(), 1.0, 1e-5, 30.0), rtol=0, atol=1e-9)
    y = R.istft(s, n_fft, win, hop, wname, fo, fi)
    y_ref = ref.istft_layer(s_ref, n_fft, win, hop, wname, fo, fi)
    np.testing.assert_allclose(y.numpy(), y_ref, rtol=0, atol=1e-9 * max(np.abs(y_ref).max(), 1.0))


def _db_grad(x, g, **kw):
    return R.vjp(lambda t: R.magnitude_to_decibel(t, **kw), torch.tensor(x, dtype=torch.float64),
                 torch.tensor(g, dtype=torch.float64))[1].numpy()


def test_restatement_tie_rules():
    k = 10.0 / np.log(10.0)
    # x == amin: the gradient goes to x (tf.maximum passes ties to its first argument); x < amin: nothing
    amin = 0.25
    x = np.array([[1.0, amin, 0.125]])
    gx = _db_grad(x, np.ones_like(x), amin=amin, dynamic_range=100.0)
    np.testing.assert_allclose(gx, [[k / 1.0, k / amin, 0.0]])
    # an element exactly at the threshold keeps its gradient; one below sends it to the maximum
    x = np.array([[1.0, 0.1, 0.05]])           # 0 dB, -10 dB, -13 dB; threshold -10 dB
    g = np.array([[1.0, 2.0, 3.0]])
    gx = _db_grad(x, g, amin=1e-5, dynamic_range=10.0)
    np.testing.assert_allclose(gx, [[k * (1.0 + 3.0), k * 2.0 / 0.1, 0.0]], rtol=1e-12)
    # two tied maxima split the threshold's gradient equally
    x = np.array([[2.0, 2.0, 1e-3]])
    g = np.array([[1.0, 1.0, 4.0]])
    gx = _db_grad(x, g, amin=1e-5, dynamic_range=20.0)
    np.testing.assert_allclose(gx, [[k * 3.0 / 2.0, k * 3.0 / 2.0, 0.0]], rtol=1e-12)


# ------------------------------------------------------------------------------ emulated backward bodies
def _emu_stft_adj(G, ola, B, C, L, T, n_fft, hop, win_eff, pad_left, w, spec_fmt, wave_fmt):
    lib = _grad_lib()
    gx = np.full((B, L, C) if wave_fmt == 'channels_last' else (B, C, L), np.nan, np.float32)
    xs = (L * C, 1, C) if wave_fmt == 'channels_last' else (C * L, L, 1)
    gs = _spec_strides(G.shape, spec_fmt)
    G = np.ascontiguousarray(G, np.complex64)
    ola = np.ascontiguousarray(ola, np.float32)
    w = np.ascontiguousarray(w, np.float32)
    assert lib.kb_emu_stft_adj(_fp(G), *[LL(s) for s in gs], _fp(ola), LL(ola.shape[-1]), _fp(gx), *[LL(s) for s in xs],
                               B, C, L, T, n_fft, hop, win_eff, pad_left, _fp(w)) == 0
    return gx


def _emu_istft_adj(gX, fmt, n_fft):
    lib = _grad_lib()
    gX = np.ascontiguousarray(gX, np.complex64)
    sb, sc, st, sk = _spec_strides(gX.shape, fmt)
    B, C, T = (gX.shape[0], gX.shape[3], gX.shape[1]) if fmt == 'channels_last' else gX.shape[:3]
    assert lib.kb_emu_istft_adj(_fp(gX), LL(sb), LL(sc), LL(st), LL(sk), B, C, T, n_fft) == 0
    return gX


# n_fft, win_length, hop: fused sizes, mixed-radix sizes (400, 1000, 96, odd 75) and a prime factor above 5 (98)
CASES = [(256, 256, 64), (512, 384, 128), (1024, 1024, 256), (2048, 2048, 512), (400, 400, 160), (1000, 1000, 250),
         (96, 128, 32), (75, 75, 25), (98, 98, 49), (256, 200, 240), (512, 512, 600)]
PADS = [(False, False), (True, False), (False, True), (True, True)]


def _body(n_fft, kind):
    """Which emulated transform bodies serve n_fft."""
    if n_fft in (256, 512, 1024, 2048):
        return kind[0]
    P = n_fft if n_fft % 2 else n_fft // 2
    for r in (2, 3, 5):
        while P % r == 0:
            P //= r
    return kind[1] if P == 1 else kind[2]


@pytest.mark.parametrize('case', CASES, ids=lambda c: 'n%d_w%d_h%d' % c)
@pytest.mark.parametrize('pads', PADS, ids=lambda p: 'pb%d_pe%d' % p)
def test_emu_stft_adjoint(case, pads):
    n_fft, win, hop = case
    pb, pe = pads
    if pb and hop > n_fft:
        pytest.skip('pad_begin needs hop <= n_fft')
    rng = np.random.default_rng(n_fft + 7 * hop + 3 * pb + pe)
    win_eff = min(win, n_fft)
    for i, (fi, fo) in enumerate([('channels_first', 'channels_last'), ('channels_last', 'channels_first')]):
        B, C = 1, 1 + i
        L = 2 * max(n_fft, win) + 3 * hop + 11
        x = _wave(rng, B, C, L, fi)
        pad_left = n_fft - hop if pb else 0
        T = ref.num_frames(L + pad_left, win, hop, pe)
        G = _spec(rng, B, C, T, n_fft // 2 + 1, fo)
        _, want = R.vjp(lambda t: R.stft(t, n_fft, win, hop, None, pb, pe, fi, fo), torch.from_numpy(x.astype(np.float64)),
                        torch.from_numpy(G.astype(np.complex128)))
        w = ref.get_window(None, win).astype(np.float32)
        dual_adj = np.zeros(win, np.float32)
        dual_adj[:win_eff] = w[:win_eff].astype(np.float64) * n_fft / 2
        body = _body(n_fft, ('istft', 'idft', 'idft'))
        olas = []
        if body == 'istft':
            olas.append(E.emu_istft(G, n_fft, win, hop, dual_adj, fo, 'channels_first', seg=5))
            R_ = -(-win_eff // hop)
            olas.append(E.emu_istft(G, n_fft, win, hop, dual_adj, fo, 'channels_first', TFc=max(16, R_ + 2)))
        else:
            olas.append(E.emu_idft(G, n_fft, win, hop, dual_adj, fo, 'channels_first'))
        for ola in olas:
            got = _emu_stft_adj(G, ola, B, C, L, T, n_fft, hop, win_eff, pad_left, w[:win_eff], fo, fi)
            _close(got, want.numpy())


@pytest.mark.parametrize('case', CASES, ids=lambda c: 'n%d_w%d_h%d' % c)
def test_emu_istft_adjoint(case):
    n_fft, win, hop = case
    rng = np.random.default_rng(n_fft + hop)
    for i, (fs, fw) in enumerate([('channels_first', 'channels_last'), ('channels_last', 'channels_first')]):
        B, C, T = 1, 1 + i, 5
        X = _spec(rng, B, C, T, n_fft // 2 + 1, fs)
        out_len = (T - 1) * hop + win
        gy = _wave(rng, B, C, out_len, fw)
        # hamming: no zero samples, so the dual window stays finite when hop > win_length
        _, want = R.vjp(lambda t: R.istft(t, n_fft, win, hop, 'hamming_window', fs, fw),
                        torch.from_numpy(X.astype(np.complex128)), torch.from_numpy(gy.astype(np.float64)))
        dual = ref.inverse_stft_window(win, hop, ref.get_window('hamming_window', win))
        w_adj = (dual * 2.0 / n_fft).astype(np.float32)
        body = _body(n_fft, ('stft', 'mr', 'dft'))
        if body == 'stft':
            fwd, _ = E.emu_stft(gy, n_fft, win, hop, w_adj, False, False, E.MODE_COMPLEX, fw, fs)
        elif body == 'mr':
            fwd = E.emu_mr(gy, n_fft, win, hop, w_adj, False, False, E.MODE_COMPLEX, fw, fs)
        else:
            fwd = E.emu_dft(gy, n_fft, win, hop, w_adj, False, False, E.MODE_COMPLEX, fw, fs)
        got = _emu_istft_adj(fwd, fs, n_fft)
        _close(got, want.numpy())


def test_emu_magnitude_backward():
    rng = np.random.default_rng(1)
    X = (rng.standard_normal(257) + 1j * rng.standard_normal(257)).astype(np.complex64)
    X[[0, 5]] = 0
    g = rng.standard_normal(257).astype(np.float32)
    gX = np.full_like(X, np.nan)
    assert _grad_lib().kb_emu_mag_bwd(_fp(X), _fp(g), _fp(gX), LL(X.size)) == 0
    _, want = R.vjp(R.magnitude, torch.from_numpy(X.astype(np.complex128)), torch.from_numpy(g.astype(np.float64)))
    _close(gX, want.numpy(), 1e-6)
    assert gX[0] == 0 and gX[5] == 0


def _emu_db_bwd(x, g, ref_value=1.0, amin=1e-5, dynamic_range=80.0, chunks=2, nt=64):
    x = np.ascontiguousarray(x, np.float32)
    g = np.ascontiguousarray(g, np.float32)
    n_items = x.shape[0] if x.ndim > 1 else 1
    gx = np.full_like(x, np.nan)
    ws = np.zeros(3 * n_items, np.uint32)
    f = ctypes.c_float
    assert _grad_lib().kb_emu_db_bwd(_fp(x), _fp(g), _fp(gx), LL(n_items), LL(x.size // n_items), f(amin),
                                  f(10 * np.log10(2.0)), f(10 * np.log10(max(amin, ref_value))), f(dynamic_range),
                                  f(10 / np.log(10.0)), _fp(ws), chunks, nt) == 0
    return gx, ws


@pytest.mark.parametrize('dyn', [80.0, 25.0])
def test_emu_decibel_backward(dyn):
    rng = np.random.default_rng(int(dyn))
    x = (rng.random((3, 7, 33)) ** 6).astype(np.float32)
    x[0, 0, :4] = 0.0                                           # below amin
    x[1, 2, 3] = x[1, 4, 5] = x[1].max() * 1.5                  # two tied maxima
    g = rng.standard_normal(x.shape).astype(np.float32)
    gx, ws = _emu_db_bwd(x, g, dynamic_range=dyn)
    _, want = R.vjp(lambda t: R.magnitude_to_decibel(t, 1.0, 1e-5, dyn), torch.from_numpy(x.astype(np.float64)),
                    torch.from_numpy(g.astype(np.float64)))
    np.testing.assert_allclose(gx, want.numpy(), rtol=2e-5, atol=1e-6 * np.abs(want.numpy()).max())
    # the emulated passes leave the sums and counts behind; the CUDA entry point clears them (self-cleaning)
    assert ws[:3].view(np.float32).max() > 0


def test_emu_decibel_backward_tie_rules():
    k = 10.0 / np.log(10.0)
    gx, _ = _emu_db_bwd(np.array([[1.0, 0.25, 0.125]]), np.ones((1, 3)), amin=0.25, dynamic_range=100.0)
    np.testing.assert_allclose(gx, [[k, k / 0.25, 0.0]], rtol=1e-6)
    gx, _ = _emu_db_bwd(np.array([[2.0, 2.0, 1e-3]]), np.array([[1.0, 1.0, 4.0]]), dynamic_range=20.0)
    np.testing.assert_allclose(gx, [[k * 1.5, k * 1.5, 0.0]], rtol=1e-6)
