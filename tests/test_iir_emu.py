"""The IIR filter on the CPU: the float64 restatement (iir_ref.py) against scipy and torchaudio, the biquad designs
against torchaudio's helpers, the kernel bodies of iir_core.cuh (run by a CPU emulation) against the restatement
within the derived error bound, their bit-independence of grid, loader, batch position, strides, broadcasting,
format and length, the adjoint identities, the layers' validation and configuration, and the register budget."""
import ctypes
import hashlib
import os
import re
import shutil
import subprocess
import tempfile

import numpy as np
import pytest
import scipy.signal
import torch

import iir_ref as IR

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, 'emu', 'kb_emu_iir.cpp')
_CSRC = os.path.join(_HERE, '..', 'kapre_b200', 'csrc')
_LIB = os.path.join(_HERE, '..', 'kapre_b200', '_lib', 'libkapre_b200.so')
_lib_handle = None


def _lib():
    """tests/emu/kb_emu_iir.cpp built with g++ into the temporary directory (keyed by the sources' contents)."""
    global _lib_handle
    if _lib_handle is None:
        hs = hashlib.sha256()
        for f in [_SRC] + sorted(os.path.join(_CSRC, n) for n in os.listdir(_CSRC) if n.endswith(('.h', '.cuh'))):
            with open(f, 'rb') as fh:
                hs.update(fh.read())
        out = os.path.join(tempfile.gettempdir(), 'kapre_b200_emu_iir_%s.so' % hs.hexdigest()[:16])
        if not os.path.exists(out):
            tmp = '%s.%d.tmp' % (out, os.getpid())
            subprocess.check_call(['g++', '-O2', '-std=c++17', '-shared', '-fPIC', '-DKB_HOST_EMU', '-Wno-unknown-pragmas',
                                   '-o', tmp, _SRC])
            os.replace(tmp, out)
        lib = ctypes.CDLL(out)
        I, P, LL = ctypes.c_int, ctypes.c_void_p, ctypes.c_longlong
        lib.kb_emu_lfilter.argtypes = [P, P, P, P, P, P, P, I, I, I, I, I, I, P, P, P, P, I, I, LL]
        lib.kb_emu_iir_powers.argtypes = [P, I, P]
        _lib_handle = lib
    return _lib_handle


def _p(a):
    return ctypes.c_void_p(a.__array_interface__['data'][0]) if a is not None else None


def _es(a):
    return np.array([s // 4 for s in a.strides], np.int64)


def emu(x, b, a, flags=0, bwd=False, xr=None, yr=None, tile_order=0, bulk=1, fmt='bcl', coef_strides=None):
    """Run the bodies on float32 x (B, C, L) ('bcl') or (B, L, C) ('blc'; views allowed) with float32 coefficients
    b, a of shape (Bc, Cc, n) (1 broadcasts through stride 0).  Returns (y (B, C, L), part or None)."""
    if fmt == 'blc':
        B, L, C = x.shape
        xs = _es(x)[[0, 2, 1]]
    else:
        B, C, L = x.shape
        xs = _es(x)
    n = b.shape[-1]
    y = np.full((B, C, L), np.nan, np.float32)
    if coef_strides is None:
        cs = np.array([0 if b.shape[0] == 1 else b.shape[1] * n, 0 if b.shape[1] == 1 else n,
                       0 if a.shape[0] == 1 else a.shape[1] * n, 0 if a.shape[1] == 1 else n], np.int64)
    else:
        cs = np.asarray(coef_strides, np.int64)
    part = rs = None
    if xr is not None:
        K = -(-L // IR.TC)
        part = np.full((2 * n - 1, B * C, K), np.nan, np.float32)
        xr = np.ascontiguousarray(xr, np.float32)
        yr = np.ascontiguousarray(yr, np.float32)
        rs = np.concatenate([_es(xr), _es(yr)])
    base = x if x.base is None else x.base
    numel = int(base.size) - (x.__array_interface__['data'][0] - base.__array_interface__['data'][0]) // 4
    rc = _lib().kb_emu_lfilter(_p(x), _p(xs), _p(y), _p(_es(y)), _p(b), _p(a), _p(cs), n - 1, B, C, L, flags, int(bwd),
                               _p(xr), _p(yr), _p(rs), _p(part), tile_order, bulk, numel)
    assert rc == 0
    return y, part


def _f32(b, a):
    b32, a32 = IR.normalised32(b, a)
    return b32, a32


def _filters():
    """(name, b, a) float64 designs the tests run (normalised to float32 by the callers)."""
    out = [('preemph', np.array([1.0, -0.97]), np.array([1.0, 0.0])),
           ('fir', np.array([0.2, -0.5, 0.3, 0.1, 0.05]), np.array([1.0, 0.0, 0.0, 0.0, 0.0]))]
    for kind in ('lowpass', 'highpass', 'bandpass', 'bandreject', 'allpass', 'equalizer'):
        for f in (100.0, 1000.0, 6000.0):
            Q = 30.0 if (kind == 'bandpass' and f == 100.0) else 0.707
            b, a = IR.biquad(kind, 16000, f, Q, 6.0)
            out.append(('%s-%g' % (kind, f), b, a))
    for order, wn in ((4, 0.1), (8, 0.2), (8, 0.4)):
        b, a = scipy.signal.butter(order, wn)
        out.append(('butter%d-%g' % (order, wn), b, a))
    return out


FILTERS = _filters()


def _check_against_ref(x, b32, a32, y, what=''):
    ref = IR.lfilter_fast(x, b32, a32)
    bound = IR.error_bound(b32, a32, np.abs(x).max(), np.abs(ref).max(), IR.local_max(x, b32, a32))
    err = np.abs(y - ref).max()
    assert err <= bound, (what, err, bound)
    return err, bound


# ------------------------------------------------------------------------------------------ the restatement
def test_restatement_matches_scipy_and_torchaudio():
    F = pytest.importorskip('torchaudio.functional')
    rng = np.random.default_rng(0)
    x = rng.uniform(-1, 1, (2, 3, 300))
    for b, a in ((np.array([0.3, 0.2, 0.1]), np.array([2.0, -0.5, 0.3])),               # a0 != 1
                 (np.array([1.0, -0.97]), np.array([1.0, 0.0])),
                 scipy.signal.butter(4, 0.2)):
        ref = IR.lfilter(x, b / a[0], a / a[0])
        assert np.abs(ref - scipy.signal.lfilter(b, a, x, axis=-1)).max() <= 1e-12
        ta = F.lfilter(torch.from_numpy(x), torch.from_numpy(a), torch.from_numpy(b), clamp=False).numpy()
        assert np.abs(ref - ta).max() <= 1e-12
        ta_c = F.lfilter(torch.from_numpy(x * 4), torch.from_numpy(a), torch.from_numpy(b), clamp=True).numpy()
        assert np.abs(IR.lfilter(x * 4, b / a[0], a / a[0], clamp=True) - ta_c).max() <= 1e-12
        ff = F.filtfilt(torch.from_numpy(x), torch.from_numpy(a), torch.from_numpy(b)).numpy()
        assert np.abs(IR.filtfilt(x, b / a[0], a / a[0]) - ff).max() <= 1e-12
    # 2-D coefficients: one filter per channel (torchaudio's batching form)
    bs = np.array([[0.3, 0.2, 0.1], [1.0, 0.5, 0.0], [0.1, 0.0, -0.1]])
    as_ = np.array([[1.0, -0.5, 0.3], [1.5, 0.2, 0.0], [1.0, -1.8, 0.9]])
    ta = F.lfilter(torch.from_numpy(x), torch.from_numpy(as_), torch.from_numpy(bs), clamp=False, batching=True).numpy()
    for c in range(3):
        assert np.abs(IR.lfilter(x[:, c], bs[c] / as_[c, 0], as_[c] / as_[c, 0]) - ta[:, c]).max() <= 1e-12


def test_biquad_coefficients_are_torchaudio_s():
    F = pytest.importorskip('torchaudio.functional')
    import torchaudio.functional.filtering as TF
    from kapre_b200.backend import BIQUAD_KINDS, biquad_coefficients
    seen = []
    orig = TF.biquad

    def spy(waveform, b0, b1, b2, a0, a1, a2):
        seen.append(np.array([float(v) for v in (b0, b1, b2, a0, a1, a2)]))
        return orig(waveform, b0, b1, b2, a0, a1, a2)

    x = torch.zeros(1, 16, dtype=torch.float64)
    TF.biquad = spy
    try:
        for kind in BIQUAD_KINDS:
            for f, Q, g in ((100.0, 30.0, 3.0), (1000.0, 0.707, -6.0), (6000.0, 2.0, 12.0)):
                seen.clear()
                if kind == 'equalizer':
                    F.equalizer_biquad(x, 16000, f, g, Q)
                else:
                    getattr(F, kind + '_biquad')(x, 16000, f, Q)
                b, a = biquad_coefficients(kind, 16000, f, Q, g)
                assert len(seen) == 1, kind
                np.testing.assert_allclose(np.r_[b, a], seen[0], rtol=0, atol=1e-12)
                rb, ra = IR.biquad(kind, 16000, f, Q, g)
                np.testing.assert_allclose(np.r_[rb, ra], seen[0], rtol=0, atol=1e-12)
    finally:
        TF.biquad = orig
    # arrays give one filter per element
    b, a = biquad_coefficients('lowpass', 16000, [100.0, 200.0], 0.707)
    assert b.shape == (2, 3) and np.allclose(b[1], biquad_coefficients('lowpass', 16000, 200.0)[0])
    for bad in (dict(kind='notch'), dict(freq=9000.0), dict(freq=0.0), dict(Q=0.0)):
        kw = dict(kind='lowpass', sample_rate=16000, freq=1000.0, Q=0.707)
        kw.update(bad)
        with pytest.raises(ValueError):
            biquad_coefficients(**kw)


def test_the_stated_test_filters():
    b, a = IR.biquad('bandpass', 16000, 100.0, 30.0)
    assert abs(np.abs(np.roots(a / a[0])).max() - 0.99935) < 5e-5
    assert 2.0e4 < IR.impulse_l1(a / a[0]) < 3.0e4
    b, a = IR.biquad('lowpass', 16000, 1000.0, 0.707)
    assert 5 < IR.impulse_l1(a / a[0]) < 15
    # butter(8, 0.05) in direct form: stable in float64, unstable once its denominator is rounded to float32
    b, a = scipy.signal.butter(8, 0.05)
    assert np.abs(np.roots(a)).max() < 1 < np.abs(np.roots(a.astype(np.float32).astype(np.float64))).max()
    for wn in (0.2, 0.4):
        b, a = scipy.signal.butter(8, wn)
        assert np.abs(np.roots(a.astype(np.float32).astype(np.float64))).max() < 1


def test_adjoint_is_the_transpose_and_coefficient_gradients_match_autograd():
    F = pytest.importorskip('torchaudio.functional')
    rng = np.random.default_rng(1)
    for b, a, L in ((np.array([0.3, 0.2, 0.1]), np.array([1.0, -0.5, 0.3]), 1),
                    (np.array([0.3, 0.2, 0.1]), np.array([1.0, -0.5, 0.3]), 7),
                    (*scipy.signal.butter(4, 0.3), 40),
                    (*IR.biquad('bandpass', 16000, 100.0, 30.0), 50)):
        b, a = b / a[0], a / a[0]
        M = IR.matrix(b, a, L)
        x, dx, gy = rng.standard_normal(L), rng.standard_normal(L), rng.standard_normal(L)
        assert np.abs(M @ x - IR.lfilter(x, b, a)).max() <= 1e-12 * max(1, np.abs(M @ x).max())
        gx, gb, ga = IR.vjp(x, gy, b, a)
        assert np.abs(gx - M.T @ gy).max() <= 1e-12 * max(1, np.abs(gx).max())
        assert abs(np.dot(M @ dx, gy) - np.dot(dx, gx)) <= 1e-12 * max(1, abs(np.dot(dx, gx)))
        # the coefficient gradients against float64 torchaudio autograd
        tb = torch.tensor(b, requires_grad=True)
        ta = torch.tensor(a, requires_grad=True)
        y = F.lfilter(torch.from_numpy(x)[None], ta, tb, clamp=False)[0]
        (y * torch.from_numpy(gy)).sum().backward()
        scale = max(1.0, np.abs(tb.grad.numpy()).max(), np.abs(ta.grad.numpy()).max())
        assert np.abs(tb.grad.numpy() - gb).max() <= 1e-10 * scale
        # torchaudio's a0 = 1 here: its gradient to a[0] is that of the division, which ours leaves to torch
        assert np.abs(ta.grad.numpy()[1:] - ga[1:]).max() <= 1e-10 * scale


# ------------------------------------------------------------------------------------------ the kernel bodies
def test_powers_are_the_companion_matrix_powers():
    for name, b, a in FILTERS[:6] + FILTERS[-3:]:
        b32, a32 = _f32(b, a)
        n = len(a32) - 1
        out = np.zeros((6, 8, 8))
        _lib().kb_emu_iir_powers(_p(a32), n, _p(out))
        Phi = np.zeros((8, 8))
        Phi[0, :n] = -a32[1:].astype(np.float64)
        Phi[np.arange(1, 8), np.arange(7)] = 1.0
        P = np.linalg.matrix_power(Phi, IR.TC)
        for j in range(6):
            assert np.abs(out[j] - P).max() <= 1e-7 * max(1.0, np.abs(P).max()), (name, j)   # float64, far below float32
            P = P @ P


LENGTHS = [1, 8, IR.TC - 1, IR.TC, IR.TC + 1, IR.TC * IR.W - 1, IR.TC * IR.W, IR.TC * IR.W + 1, 3 * IR.TC * IR.W + 77]


@pytest.mark.parametrize('name,b,a', FILTERS, ids=[f[0] for f in FILTERS])
def test_forward_within_bound(name, b, a):
    rng = np.random.default_rng(abs(hash(name)) % 1000)
    b32, a32 = _f32(b, a)
    for L in LENGTHS:
        x = rng.uniform(-1, 1, (2, 1, L)).astype(np.float32)
        y, _ = emu(x, b32[None, None], a32[None, None])
        _check_against_ref(x, b32, a32, y, (name, L))


@pytest.mark.parametrize('name', ['preemph', 'bandpass-100', 'lowpass-1000', 'butter8-0.2'])
def test_forward_long_signal_within_bound(name):
    _, b, a = next(f for f in FILTERS if f[0] == name)
    b32, a32 = _f32(b, a)
    x = np.random.default_rng(3).uniform(-1, 1, (1, 1, 1_000_003)).astype(np.float32)
    y, _ = emu(x, b32[None, None], a32[None, None])
    err, bound = _check_against_ref(x, b32, a32, y, name)
    print('%s: max|err| %.3g, bound %.3g' % (name, err, bound))


def test_clamp_and_reverse():
    b32, a32 = _f32(*IR.biquad('lowpass', 16000, 1000.0))
    x = np.random.default_rng(4).uniform(-3, 3, (2, 2, 3000)).astype(np.float32)
    y, _ = emu(x, b32[None, None], a32[None, None])
    yc, _ = emu(x, b32[None, None], a32[None, None], flags=1)
    assert np.array_equal(yc, np.clip(y, -1, 1)) and np.abs(y).max() > 1
    yr, _ = emu(np.ascontiguousarray(x[..., ::-1]), b32[None, None], a32[None, None])
    yrev, _ = emu(x, b32[None, None], a32[None, None], flags=2)
    assert np.array_equal(yrev, yr[..., ::-1])


def test_bits_do_not_depend_on_grid_loader_position_strides_broadcast_format_or_length():
    rng = np.random.default_rng(5)
    b32, a32 = _f32(*scipy.signal.butter(8, 0.2))
    B, C, L = 3, 2, 2 * IR.TC * IR.W + 300
    x = rng.uniform(-1, 1, (B, C, L)).astype(np.float32)
    bb, ab = b32[None, None], a32[None, None]
    ref, _ = emu(x, bb, ab)
    assert np.array_equal(emu(x, bb, ab, tile_order=1)[0], ref)
    assert np.array_equal(emu(x, bb, ab, bulk=0)[0], ref)
    for flags in (0, 2):
        r0, _ = emu(x, bb, ab, flags=flags)
        assert np.array_equal(emu(x, bb, ab, flags=flags, bulk=0)[0], r0)
    # materialised coefficients per item and channel
    bm = np.ascontiguousarray(np.broadcast_to(bb, (B, C, 9)))
    am = np.ascontiguousarray(np.broadcast_to(ab, (B, C, 9)))
    assert np.array_equal(emu(x, bm, am)[0], ref)
    # each item alone and a batch that starts elsewhere
    for i in range(B):
        assert np.array_equal(emu(x[i:i + 1], bb, ab)[0], ref[i:i + 1])
    assert np.array_equal(emu(x[1:], bb, ab)[0], ref[1:])
    # a strided view (offset items, narrowed time, every other channel)
    big = rng.uniform(-1, 1, (B + 1, 2 * C, L + 11)).astype(np.float32)
    big[1:, ::2, 5:L + 5] = x
    assert np.array_equal(emu(big[1:, ::2, 5:L + 5], bb, ab)[0], ref)
    # channels-last (interleaved) input gives the channels-first bits
    xl = np.ascontiguousarray(x.transpose(0, 2, 1))
    assert np.array_equal(emu(xl, bb, ab, fmt='blc')[0], ref)
    # mono: either format
    assert np.array_equal(emu(np.ascontiguousarray(x[:, :1].transpose(0, 2, 1)), bb, ab, fmt='blc')[0], ref[:, :1])
    # a prefix of a longer signal
    for n in (1, IR.TC, IR.TC * IR.W + 3, L - 1):
        assert np.array_equal(emu(np.ascontiguousarray(x[..., :n]), bb, ab)[0], ref[..., :n]), n


def test_per_item_and_per_channel_coefficients():
    rng = np.random.default_rng(6)
    B, C, L = 3, 2, 4000
    x = rng.uniform(-1, 1, (B, C, L)).astype(np.float32)
    freqs = [[300.0, 3000.0], [500.0, 100.0], [1000.0, 7000.0]]
    bb = np.zeros((B, C, 3), np.float32)
    ab = np.zeros((B, C, 3), np.float32)
    for i in range(B):
        for c in range(C):
            bb[i, c], ab[i, c] = _f32(*IR.biquad('lowpass', 16000, freqs[i][c]))
    y, _ = emu(x, bb, ab)
    for i in range(B):
        for c in range(C):
            _check_against_ref(x[i, c], bb[i, c], ab[i, c], y[i, c])
            # the same bits as that filter alone
            yi, _ = emu(x[i:i + 1, c:c + 1].copy(), bb[i:i + 1, c:c + 1].copy(), ab[i:i + 1, c:c + 1].copy())
            assert np.array_equal(yi[0, 0], y[i, c])
    # one filter per channel, shared over the batch
    y2, _ = emu(x, bb[:1].copy(), ab[:1].copy())
    for c in range(C):
        _check_against_ref(x[:, c], bb[0, c], ab[0, c], y2[:, c])


@pytest.mark.parametrize('name', ['preemph', 'fir', 'lowpass-1000', 'bandpass-100', 'butter4-0.1', 'butter8-0.2'])
@pytest.mark.parametrize('L', [1, 9, IR.TC + 1, IR.TC * IR.W + 1, 5000])
def test_backward_within_bound(name, L):
    _, b, a = next(f for f in FILTERS if f[0] == name)
    b32, a32 = _f32(b, a)
    rng = np.random.default_rng(L)
    x = rng.uniform(-1, 1, (2, 1, L)).astype(np.float32)
    gy = rng.uniform(-1, 1, (2, 1, L)).astype(np.float32)
    y, _ = emu(x, b32[None, None], a32[None, None])
    gx, part = emu(gy, b32[None, None], a32[None, None], bwd=True, xr=x, yr=y)
    gx_ref, gb_ref, ga_ref = IR.vjp(x, gy, b32, a32)
    # gx: the same recursion run backwards on gy; its bound is the forward's with gy as input
    v = IR.allpole_adjoint(gy, a32)
    bound = IR.error_bound(b32, a32, 1.0, max(np.abs(gx_ref).max(), np.abs(v).max()), IR.local_max(gy[..., ::-1], [1.0], a32))
    bound *= 1 + np.abs(b32).sum()
    assert np.abs(gx - gx_ref).max() <= bound, (np.abs(gx - gx_ref).max(), bound)
    # the coefficient sums: per-chunk float32 sums of terms of at most |v| max(|x|, |y|)
    n = len(b32)
    s = part.astype(np.float64).sum(axis=(1, 2))
    terms = L * 2 * max(np.abs(v).max(), 1e-30) * max(1.0, np.abs(y).max())
    tol = bound * 2 * L * max(1.0, np.abs(y).max()) + (IR.TC + 2) * IR.EPS32 * terms
    assert np.abs(s[:n] - gb_ref).max() <= tol
    assert np.abs(s[n:] - ga_ref[1:]).max() <= tol
    # without the sums gx has the same bits
    gx2, _ = emu(gy, b32[None, None], a32[None, None], bwd=True)
    assert np.array_equal(gx2, gx)


def test_backward_of_reverse_is_the_forward_adjoint():
    rng = np.random.default_rng(8)
    b32, a32 = _f32(*IR.biquad('highpass', 16000, 500.0))
    x = rng.uniform(-1, 1, (1, 1, 3000)).astype(np.float32)
    gy = rng.uniform(-1, 1, (1, 1, 3000)).astype(np.float32)
    gx, _ = emu(gy, b32[None, None], a32[None, None], flags=2, bwd=True)
    gx_ref, _, _ = IR.vjp(x[..., ::-1], gy[..., ::-1], b32, a32)
    assert np.abs(gx - gx_ref[..., ::-1]).max() <= 1e-5


# ------------------------------------------------------------------------------------------ layers
def _kb():
    if not os.path.exists(_LIB):
        pytest.skip('needs the built library')


def test_functional_validation_before_any_launch():
    _kb()
    from kapre_b200 import ops
    x = torch.zeros(4, 100, 2)
    ops.iir_check(x, torch.zeros(3), torch.zeros(3), 'channels_last')
    ops.iir_check(x, torch.zeros(2, 9), torch.zeros(2, 9), 'channels_last')
    ops.iir_check(x, torch.zeros(4, 1, 3), torch.zeros(4, 1, 3), 'channels_last')
    for b, a in ((torch.zeros(10), torch.zeros(10)),              # order 9
                 (torch.zeros(3), torch.zeros(4)),                # mismatched
                 (torch.zeros(3, 3), torch.zeros(3, 3)),          # 3 filters for 2 channels
                 (torch.zeros(2, 2, 3), torch.zeros(2, 2, 3)),    # batch 2 for 4 items
                 (torch.zeros(0), torch.zeros(0)),
                 (torch.zeros(1, 1, 1, 3), torch.zeros(1, 1, 1, 3))):
        with pytest.raises(ValueError):
            ops.iir_check(x, b, a, 'channels_last')


def test_layer_validation_and_config():
    _kb()
    from kapre_b200.augmentation import RandomBiquad
    from kapre_b200.signal import Biquad, IIRFilter
    import kapre
    assert kapre.signal.IIRFilter is IIRFilter and kapre.signal.Biquad is Biquad
    assert kapre.augmentation.RandomBiquad is RandomBiquad
    assert kapre.signal.lfilter is not None and kapre.signal.filtfilt is not None
    for b, a in (([1.0] * 10, [1.0] * 10), ([1.0, 0.5], [1.0]), ([1.0, 0.5], [0.0, 0.5]), ([1.0, np.nan], [1.0, 0.0])):
        with pytest.raises(ValueError):
            IIRFilter(b, a)
    f = IIRFilter([1.0, -0.97], [1.0, 0.0], clamp=False, trainable=True, data_format='channels_first')
    cfg = f.get_config()
    g = IIRFilter.from_config(cfg)
    assert g.get_config() == cfg and g.trainable and not g.clamp and np.array_equal(g.b, [1.0, -0.97])
    q = Biquad('bandpass', 16000, 100.0, Q=30.0)
    cfg = q.get_config()
    assert Biquad.from_config(cfg).get_config() == cfg
    np.testing.assert_allclose(q.a, IR.biquad('bandpass', 16000, 100.0, 30.0)[1] / IR.biquad('bandpass', 16000, 100.0, 30.0)[1][0])
    for bad in (dict(kind='notch'), dict(freq=8000.0), dict(Q=-1.0)):
        kw = dict(kind='lowpass', sample_rate=16000, freq=1000.0)
        kw.update(bad)
        with pytest.raises(ValueError):
            Biquad(**kw)
    r = RandomBiquad('equalizer', 16000, (100.0, 4000.0), (0.5, 2.0), (-6.0, 6.0), seed=3)
    cfg = r.get_config()
    r2 = RandomBiquad.from_config(cfg)
    d1, d2 = r.draw(5), r2.draw(5)
    assert all(np.array_equal(u, v) for u, v in zip(d1, d2))
    rng = np.random.default_rng(3)
    freq = np.exp(rng.uniform(np.log(100.0), np.log(4000.0), 5))
    assert np.array_equal(d1[0], freq)
    assert np.all((d1[1] >= 0.5) & (d1[1] <= 2.0)) and np.all((d1[2] >= -6) & (d1[2] <= 6))
    for bad in (dict(freq_range=(100.0, 9000.0)), dict(freq_range=(400.0, 100.0)), dict(Q_range=(0.0, 1.0)),
                dict(kind='notch')):
        kw = dict(kind='lowpass', sample_rate=16000, freq_range=(100.0, 1000.0))
        kw.update(bad)
        with pytest.raises(ValueError):
            RandomBiquad(**kw)


# ------------------------------------------------------------------------------------------ register budget
@pytest.mark.skipif(shutil.which('cuobjdump') is None or not os.path.exists(_LIB),
                    reason='needs cuobjdump and the built library')
def test_iir_kernels_register_and_spill_budget():
    out = subprocess.run(['cuobjdump', '-res-usage', _LIB], capture_output=True, text=True, check=True).stdout
    for name, cap in (('kb_iir_powers_kernel', 64), ('kb_iir_state_kernel', 128), ('kb_iir_carry_kernel', 128),
                      ('kb_iir_out_kernel', 128)):
        m = re.search(r'Function \S*%s\S*:\s*\n\s*REG:(\d+) STACK:(\d+)' % name, out)
        assert m, name + ' not in the library'
        assert int(m.group(1)) <= cap, (name, m.group(1))
        assert int(m.group(2)) == 0, (name, m.group(2))      # no spills, no stack
