"""The partitioned FFT convolution on the CPU: the multiply-accumulate body of conv_core.cuh (run by a CPU emulation)
against the float64 restatement (conv_ref.py), its bit-independence of tiling, grid, strides, layout, batch position
and broadcasting, the adjoint identities, the whole chain (STFT body -> MAC body -> inverse body) against
``scipy.signal.fftconvolve``, the block-size rule and the crops, the ``Convolve`` / ``Reverb`` layers' validation and
configuration, the RIR preparation and seeded draws, and the kernel's register budget.
"""
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

import conv_ref as CR
import emu_harness as EH

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, 'emu', 'kb_emu_conv.cpp')
_CSRC = os.path.join(_HERE, '..', 'kapre_b200', 'csrc')
_LIB = os.path.join(_HERE, '..', 'kapre_b200', '_lib', 'libkapre_b200.so')
_lib_handle = None


def _lib():
    """tests/emu/kb_emu_conv.cpp built with g++ into the temporary directory (keyed by the sources' contents)."""
    global _lib_handle
    if _lib_handle is None:
        hs = hashlib.sha256()
        for f in [_SRC] + sorted(os.path.join(_CSRC, n) for n in os.listdir(_CSRC) if n.endswith(('.h', '.cuh'))):
            with open(f, 'rb') as fh:
                hs.update(fh.read())
        out = os.path.join(tempfile.gettempdir(), 'kapre_b200_emu_conv_%s.so' % hs.hexdigest()[:16])
        if not os.path.exists(out):
            tmp = '%s.%d.tmp' % (out, os.getpid())
            subprocess.check_call(['g++', '-O2', '-std=c++17', '-shared', '-fPIC', '-DKB_HOST_EMU', '-Wno-unknown-pragmas',
                                   '-o', tmp, _SRC])
            os.replace(tmp, out)
        lib = ctypes.CDLL(out)
        I, P = ctypes.c_int, ctypes.c_void_p
        lib.kb_emu_spec_conv.argtypes = [P, P, I, P, P, I, P, P, I, I, I, I, I, I, I]
        lib.kb_emu_conv_block_size.restype = ctypes.c_longlong
        lib.kb_emu_conv_block_size.argtypes = [ctypes.c_longlong]
        _lib_handle = lib
    return _lib_handle


def _fp(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _estrides(a):
    """Element strides (b, c, t, f) of a 4-D complex64 array; size-1 dims may be broadcast by passing 0."""
    return np.array([s // 8 for s in a.strides], np.int64)


def emu_mac(a, b, To, correlate, n_cta=3, a_strides=None, b_strides=None, out_layout='bctf'):
    """Run the body on complex64 arrays a (Ba, Ca, S, F), b (Bn, C, Tb, F) (views allowed); a's batch / channel of
    size 1 are broadcast with stride 0.  out_layout 'btfc' writes through a channels-last view."""
    Bn, C, Tb, F = b.shape
    S = a.shape[2]
    as_ = _estrides(a) if a_strides is None else np.asarray(a_strides, np.int64)
    if a_strides is None:
        if a.shape[0] == 1:
            as_[0] = 0
        if a.shape[1] == 1:
            as_[1] = 0
    bs = _estrides(b) if b_strides is None else np.asarray(b_strides, np.int64)
    if out_layout == 'btfc':
        buf = np.full((Bn, To, F, C), np.nan + 0j, np.complex64)
        out = buf.transpose(0, 3, 1, 2)
    else:
        buf = out = np.full((Bn, C, To, F), np.nan + 0j, np.complex64)
    os_ = _estrides(out)
    abase = a if a.base is None else a.base
    bbase = b if b.base is None else b.base
    rc = _lib().kb_emu_spec_conv(ctypes.c_void_p(a.__array_interface__['data'][0]), _fp(as_), S,
                                 ctypes.c_void_p(b.__array_interface__['data'][0]), _fp(bs), Tb,
                                 ctypes.c_void_p(out.__array_interface__['data'][0]), _fp(os_), Bn, C, F, To,
                                 int(correlate), 256, n_cta)
    assert rc == 0
    del abase, bbase, buf
    return np.ascontiguousarray(out)


def _cplx(rng, shape):
    return (rng.standard_normal(shape) + 1j * rng.standard_normal(shape)).astype(np.complex64)


# ------------------------------------------------------------------------------------------ the MAC body
@pytest.mark.parametrize('correlate', [0, 1])
@pytest.mark.parametrize('S,Tb,To', [(1, 5, 5), (3, 10, 12), (8, 70, 77), (40, 45, 6), (70, 3, 72), (33, 100, 68)])
def test_mac_against_float64(correlate, S, Tb, To):
    rng = np.random.default_rng(S * 100 + Tb + correlate)
    F = 37
    a, b = _cplx(rng, (2, 2, S, F)), _cplx(rng, (2, 2, Tb, F))
    got = emu_mac(a, b, To, correlate)
    want = CR.mac(a.astype(np.complex128), b.astype(np.complex128), To, correlate)
    # |sum of S products| error: S + 1 roundings of terms of size |a||b| ~ 2
    tol = 4 * (S + 2) * CR.EPS32 * 2 * np.sqrt(S)
    assert np.abs(got - want).max() <= tol * 2


@pytest.mark.parametrize('correlate', [0, 1])
def test_mac_bits_do_not_depend_on_grid_layout_position_or_broadcast(correlate):
    rng = np.random.default_rng(7)
    Bn, C, S, Tb, F = 5, 3, 37, 80, 65
    To = Tb + S - 1 if not correlate else Tb
    a1 = _cplx(rng, (1, 1, S, F))
    b = _cplx(rng, (Bn, C, Tb, F))
    ref = emu_mac(a1, b, To, correlate)
    for n_cta in (1, 2, 7, 1000):
        assert np.array_equal(emu_mac(a1, b, To, correlate, n_cta=n_cta), ref)
    # the broadcast filter gives the bits of its copy per item and channel
    a_full = np.ascontiguousarray(np.broadcast_to(a1, (Bn, C, S, F)))
    assert np.array_equal(emu_mac(a_full, b, To, correlate), ref)
    # a channels-last b (bins C apart) and output, and a strided view of b
    b_cl = np.ascontiguousarray(b.transpose(0, 2, 3, 1)).transpose(0, 3, 1, 2)
    assert np.array_equal(emu_mac(a1, b_cl, To, correlate, out_layout='btfc'), ref)
    big = _cplx(rng, (Bn + 2, C + 1, Tb + 3, F + 5))
    big[1:Bn + 1, 1:, 2:Tb + 2, 3:F + 3] = b
    assert np.array_equal(emu_mac(a1, big[1:Bn + 1, 1:, 2:Tb + 2, 3:F + 3], To, correlate), ref)
    # each item alone, and a batch that starts elsewhere
    for i in (0, 3):
        assert np.array_equal(emu_mac(a1, b[i:i + 1], To, correlate), ref[i:i + 1])
    assert np.array_equal(emu_mac(a1, b[2:], To, correlate), ref[2:])


def test_adjoint_identities_on_explicit_matrices():
    rng = np.random.default_rng(3)
    for S, J in ((1, 1), (4, 9), (9, 4), (16, 79)):
        T = J + S - 1
        a = rng.standard_normal(S) + 1j * rng.standard_normal(S)
        x = rng.standard_normal(J) + 1j * rng.standard_normal(J)
        g = rng.standard_normal(T) + 1j * rng.standard_normal(T)
        Mf = CR.mac_matrix(a, J, T, False)            # Y = Mf X
        Mc = CR.mac_matrix(a, T, J, True)             # gX = Mc G
        assert np.abs(Mc - Mf.conj().T).max() <= 1e-12
        y = Mf @ x
        lhs, rhs = np.vdot(g, y), np.vdot(Mc @ g, x)
        assert abs(lhs - rhs) <= 1e-12 * max(1.0, abs(lhs))
        # gH_p = sum_j conj(X_j) G_{j + p}: the adjoint of a -> Y at fixed X
        Mx = CR.mac_matrix(x, S, T, False)            # Y = Mx a (convolution is symmetric in its operands)
        assert np.abs(Mx @ a - y).max() <= 1e-12
        gH = CR.mac(x[None, :, None], g[None, :, None], S, True)[0, :, 0]
        assert np.abs(gH - Mx.conj().T @ g).max() <= 1e-12


def test_restated_scheme_is_the_convolution_and_its_tail_is_zero():
    rng = np.random.default_rng(0)
    for B in CR.BLOCKS:
        for L, K in ((1, 1), (1000, 1), (500, 300), (333, 2777)):
            x, h = rng.standard_normal(L), rng.standard_normal(K)
            y = CR.convolve_full(x, h, B)
            ref = np.convolve(x, h)
            assert np.abs(y[:L + K - 1] - ref).max() < 1e-9 * max(1.0, np.abs(ref).max())
            assert np.abs(y[L + K - 1:]).max() < 1e-9


# ------------------------------------------------------------------------------------------ the whole chain
def emu_chain(x, h, B, fmt='channels_first'):
    """STFT body -> MAC body -> inverse body, as kapre_convolve runs them (x (Bn, C, L) / (Bn, L, C); h (K,))."""
    Xs, _ = EH.emu_stft(x, 2 * B, B, B, np.ones(B, np.float32), False, True, EH.MODE_COMPLEX, fmt, 'channels_first')
    Hs, _ = EH.emu_stft(h.reshape(1, 1, -1).astype(np.float32), 2 * B, B, B, np.ones(B, np.float32), False, True,
                        EH.MODE_COMPLEX, 'channels_first', 'channels_first')
    J, P = Xs.shape[2], Hs.shape[2]
    Y = emu_mac(Hs, Xs, J + P - 1, 0)
    return EH.emu_istft(Y, 2 * B, 2 * B, B, np.ones(2 * B, np.float32), 'channels_first', fmt)


@pytest.mark.parametrize('B', CR.BLOCKS)
def test_emulated_chain_against_fftconvolve(B):
    rng = np.random.default_rng(B)
    for L, K in ((3000, 5 * B + 17), (B // 2, 3 * B), (700, 1), (2 * B, 8 * B)):
        x = rng.uniform(-1, 1, (2, 2, L)).astype(np.float32)
        h = rng.standard_normal(K).astype(np.float32)
        y = emu_chain(x, h, B)
        ref = scipy.signal.fftconvolve(x.astype(np.float64), h.astype(np.float64)[None, None, :], axes=-1)
        scale = np.sqrt(np.mean(x.astype(np.float64) ** 2)) * np.linalg.norm(h.astype(np.float64))
        P = -(-K // B)
        assert y.shape[-1] == (-(-L // B) + P) * B
        err = np.abs(y[..., :L + K - 1] - ref).max() / scale
        assert err <= CR.error_bound(B, P), (B, L, K, err)
        assert np.abs(y[..., L + K - 1:]).max() / scale <= CR.error_bound(B, P)


def test_emulated_chain_channels_last_gives_the_channels_first_bits():
    rng = np.random.default_rng(5)
    x = rng.uniform(-1, 1, (2, 2, 1500)).astype(np.float32)
    h = rng.standard_normal(700).astype(np.float32)
    yf = emu_chain(x, h, 128)
    yl = emu_chain(np.ascontiguousarray(x.transpose(0, 2, 1)), h, 128, 'channels_last')
    assert np.array_equal(yl.transpose(0, 2, 1), yf)


# ------------------------------------------------------------------------------------------ rule, crops, layers
def test_block_size_rule():
    for K in (1, 100, 1024, 1025, 2000, 2048, 2049, 4096, 4097, 8192, 8193, 16000, 48000):
        assert _lib().kb_emu_conv_block_size(K) == CR.block_size(K)
    assert [CR.block_size(K) for K in (100, 2000, 16000)] == [128, 256, 1024]
    if os.path.exists(_LIB):
        from kapre_b200 import ops
        for K in (1, 100, 2000, 16000, 48000):
            assert ops.convolve_block_size(K) == CR.block_size(K)
        from kapre_b200 import _native as N
        with pytest.raises(N.KapreNativeError):
            ops.convolve_block_size(0)


def _torchaudio_crop(full, L, K, mode):
    """torchaudio.functional.functional._apply_convolve_mode, restated."""
    if mode == 'full':
        return full
    if mode == 'valid':
        target = max(L, K) - min(L, K) + 1
        start = (full.shape[-1] - target) // 2
        return full[..., start:start + target]
    start = (full.shape[-1] - L) // 2
    return full[..., start:start + L]


@pytest.mark.parametrize('mode', ['full', 'same', 'valid'])
def test_mode_spans_follow_torchaudio(mode):
    from kapre_b200 import ops
    for L, K in ((10, 3), (3, 10), (7, 7), (1, 1), (1000, 257), (256, 1000)):
        full = np.arange(L + K - 1)
        start, n = ops.convolve_span(L, K, mode)
        assert np.array_equal(full[start:start + n], _torchaudio_crop(full, L, K, mode))
        assert (start, n) == CR.span(L, K, mode)


def test_convolve_layer_validation_and_config():
    from kapre_b200.signal import Convolve
    with pytest.raises(ValueError):
        Convolve(mode='circular')
    with pytest.raises(ValueError):
        Convolve(data_format='channels_middle')
    layer = Convolve(mode='same', data_format='channels_first')
    cfg = layer.get_config()
    assert cfg['mode'] == 'same' and cfg['data_format'] == 'channels_first'
    again = Convolve.from_config(cfg)
    assert again.mode == 'same' and again.data_format == 'channels_first'
    import kapre
    assert kapre.signal.Convolve is Convolve


def test_convolve_shape_validation():
    import torch

    from kapre_b200 import ops
    x = torch.zeros(4, 100, 2)
    ops._conv_check(x, torch.zeros(7), 'channels_last')
    for h in (torch.zeros(1, 7, 2), torch.zeros(4, 7, 1), torch.zeros(4, 7, 2)):
        ops._conv_check(x, h, 'channels_last')
    for h in (torch.zeros(2, 7, 2), torch.zeros(1, 7, 3), torch.zeros(7, 2), torch.zeros(0)):
        with pytest.raises(ValueError):
            ops._conv_check(x, h, 'channels_last')
    with pytest.raises(ValueError):
        ops._conv_check(torch.zeros(4, 0, 2), torch.zeros(3), 'channels_last')


def test_rir_preparation():
    from kapre_b200.augmentation import prepare_rirs
    a = np.array([0.0, 0.1, -2.0, 0.5, 0.25])
    b = np.array([3.0, 1.0])
    bank = prepare_rirs([a, b])
    assert bank.dtype == np.float32 and bank.shape == (2, 3)
    ta = a[2:] / np.linalg.norm(a[2:])
    np.testing.assert_allclose(bank[0], ta, rtol=0, atol=1e-7)
    np.testing.assert_allclose(bank[1], np.r_[b / np.linalg.norm(b), 0.0], rtol=0, atol=1e-7)
    assert np.array_equal(prepare_rirs(np.stack([a, a])), np.stack([bank[0], bank[0]]))
    for bad in ([], [np.zeros(4)], [np.array([1.0, np.nan])], [np.array([1.0, np.inf])], [np.zeros((2, 2))],
                np.zeros(3), [np.array([])]):
        with pytest.raises(ValueError):
            prepare_rirs(bad)


def test_reverb_draws_config_and_validation():
    if not os.path.exists(_LIB):
        pytest.skip('needs the built library (the block-size rule)')
    from kapre_b200.augmentation import Reverb
    rng = np.random.default_rng(1)
    rirs = [rng.standard_normal(n) for n in (50, 300, 1200)]
    r1, r2 = Reverb(rirs, seed=11), Reverb(rirs, seed=11)
    d1 = [r1._choice(8, None) for _ in range(3)]
    d2 = [r2._choice(8, None) for _ in range(3)]
    assert all(np.array_equal(u, v) for u, v in zip(d1, d2))
    want = np.random.default_rng(11).integers(0, 3, size=8)
    assert np.array_equal(d1[0], want)
    assert np.array_equal(r1._choice(4, 2), [2, 2, 2, 2])
    assert np.array_equal(r1._choice(3, [0, 2, 1]), [0, 2, 1])
    for bad in (3, -1, [0, 1], 1.5, [[0, 1, 2]]):
        with pytest.raises(ValueError):
            r1._choice(3, bad)
    assert r1.plan.block == CR.block_size(r1.bank.shape[1])
    cfg = r1.get_config()
    assert cfg['seed'] == 11 and cfg['data_format'] == 'default'
    again = Reverb.from_config(cfg)
    np.testing.assert_allclose(again.bank, r1.bank, rtol=0, atol=1e-7)
    import kapre
    assert kapre.augmentation.Reverb is Reverb
    with pytest.raises(ValueError):
        Reverb([])


# ------------------------------------------------------------------------------------------ register budget
@pytest.mark.skipif(shutil.which('cuobjdump') is None or not os.path.exists(_LIB),
                    reason='needs cuobjdump and the built library')
def test_mac_kernel_register_and_spill_budget():
    out = subprocess.run(['cuobjdump', '-res-usage', _LIB], capture_output=True, text=True, check=True).stdout
    m = re.search(r'Function \S*kb_spec_conv_kernel\S*:\s*\n\s*REG:(\d+) STACK:(\d+)', out)
    assert m, 'kb_spec_conv_kernel not in the library'
    regs, stack = int(m.group(1)), int(m.group(2))
    assert regs <= 64, regs          # 256 threads x 4 CTAs per SM fit in the register file
    assert stack == 0, stack         # no spills
