"""Builds and drives the CPU emulation of the CUDA kernel bodies (tests/emu/kb_emu.cpp).

Test infrastructure: lets the CPU-only test tier check the fused kernels' arithmetic
(the exact source the GPU compiles) against the oracle.
"""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, 'emu', 'kb_emu.cpp')
_OUT = os.path.join(_HERE, 'emu', '_build', 'libkb_emu.so')
_CSRC = os.path.join(_HERE, '..', 'kapre_b200', 'csrc')

MODE_COMPLEX, MODE_MAG, MODE_MAG_DB, MODE_FB, MODE_FB_DB, MODE_MAG_PHASE = range(6)


def _needs_build():
    if not os.path.exists(_OUT):
        return True
    t = os.path.getmtime(_OUT)
    deps = [_SRC] + [os.path.join(_CSRC, f) for f in os.listdir(_CSRC) if f.endswith(('.h', '.cuh'))]
    return any(os.path.getmtime(d) > t for d in deps)


class Checked:
    """An emulation library whose every call is checked against the host model of the async staging primitives
    (stft_core.cuh): the model is reset before the call and must count no violation after it.  `raw` is the
    unchecked library."""

    def __init__(self, lib):
        lib.kb_emu_async_violations.restype = ctypes.c_longlong
        self.raw = lib

    def __getattr__(self, name):
        fn = getattr(self.raw, name)

        def call(*args):
            self.raw.kb_emu_async_reset()
            out = fn(*args)
            n = self.raw.kb_emu_async_violations()
            assert n == 0, '%s: %d violations of the async staging protocol' % (name, n)
            return out
        return call


_lib_handle = None


def load():
    global _lib_handle
    if _lib_handle is None:
        if _needs_build():
            os.makedirs(os.path.dirname(_OUT), exist_ok=True)
            subprocess.check_call(['g++', '-O2', '-std=c++17', '-shared', '-fPIC', '-DKB_HOST_EMU',
                                   '-Wno-unknown-pragmas', '-o', _OUT, _SRC])
        _lib_handle = Checked(ctypes.CDLL(_OUT))
    return _lib_handle


def _fp(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def emu_stft(x, n_fft, win_length, hop, window, pad_begin, pad_end, mode, in_fmt, out_fmt,
             fb=None, amin=1e-5, ref=1.0, TF=16, n_warps=4, n_cta=3, dbuf=1, bulk=1, db_on=0, fb_mma=0):
    """x: (B, L, C) channels_last or (B, C, L) channels_first float32.  Returns (out, item_max)."""
    lib = load()
    x = np.ascontiguousarray(x, dtype=np.float32)
    if in_fmt == 'channels_last':
        B, L, C = x.shape
        sb, sl, sc = L * C, C, 1
    else:
        B, C, L = x.shape
        sb, sc, sl = C * L, L, 1
    pad_left = (n_fft - hop) if pad_begin else 0
    Lp = L + pad_left
    T = -(-Lp // hop) if pad_end else max(0, 1 + (Lp - win_length) // hop)
    F = n_fft // 2 + 1
    K = fb.shape[1] if mode in (MODE_FB, MODE_FB_DB) else F
    dt = np.complex64 if mode == MODE_COMPLEX else np.float32
    Co = 2 * C if mode == MODE_MAG_PHASE else C   # mag+phase: phases live in channels [C, 2C)
    if out_fmt == 'channels_last':
        out = np.full((B, T, K, Co), np.nan, dtype=dt)
        osb, ost, osk, osc = T * K * Co, K * Co, Co, 1
    else:
        out = np.full((B, Co, T, K), np.nan, dtype=dt)
        osb, osc, ost, osk = Co * T * K, T * K, K, 1
    item_max = np.zeros(B, dtype=np.uint32)
    window = np.ascontiguousarray(window, dtype=np.float32)
    fbp, nfreq, nb = None, 0, 0
    if fb is not None:
        fb = np.ascontiguousarray(fb, dtype=np.float32)
        fbp, nfreq, nb = _fp(fb), fb.shape[0], fb.shape[1]
    db_mul = 10.0 * np.log10(2.0)
    db_sub = 10.0 * np.log10(max(amin, ref))
    LL = ctypes.c_longlong
    rc = lib.kb_emu_stft(_fp(x), LL(sb), LL(sc), LL(sl), B, C, L, n_fft, win_length, hop, pad_left, T,
                         _fp(window), mode, _fp(out), LL(osb), LL(osc), LL(ost), LL(osk),
                         fbp, nfreq, nb, ctypes.c_float(amin), ctypes.c_float(db_mul),
                         ctypes.c_float(db_sub), _fp(item_max), TF, n_warps, n_cta, dbuf, bulk, LL(x.size),
                         db_on, LL(C * osc), int(fb_mma))
    assert rc == 0
    return out, item_max.view(np.float32)


def emu_stft_mc(x, n_fft, win_length, hop, window, pad_begin, pad_end, mode, in_fmt, out_fmt,
                fb=None, amin=1e-5, ref=1.0, TF=2, n_warps=4, n_cta=3, db_on=0):
    """Multi-channel tile kernel (stft_mc_core.cuh); same conventions as emu_stft, TF = time frames per tile."""
    lib = load()
    x = np.ascontiguousarray(x, dtype=np.float32)
    if in_fmt == 'channels_last':
        B, L, C = x.shape
        sb, sl, sc = L * C, C, 1
    else:
        B, C, L = x.shape
        sb, sc, sl = C * L, L, 1
    pad_left = (n_fft - hop) if pad_begin else 0
    Lp = L + pad_left
    T = -(-Lp // hop) if pad_end else max(0, 1 + (Lp - win_length) // hop)
    F = n_fft // 2 + 1
    K = fb.shape[1] if mode in (MODE_FB, MODE_FB_DB) else F
    dt = np.complex64 if mode == MODE_COMPLEX else np.float32
    Co = 2 * C if mode == MODE_MAG_PHASE else C
    if out_fmt == 'channels_last':
        out = np.full((B, T, K, Co), np.nan, dtype=dt)
        osb, ost, osk, osc = T * K * Co, K * Co, Co, 1
    else:
        out = np.full((B, Co, T, K), np.nan, dtype=dt)
        osb, osc, ost, osk = Co * T * K, T * K, K, 1
    item_max = np.zeros(B, dtype=np.uint32)
    window = np.ascontiguousarray(window, dtype=np.float32)
    fbp, nfreq, nb = None, 0, 0
    if fb is not None:
        fb = np.ascontiguousarray(fb, dtype=np.float32)
        fbp, nfreq, nb = _fp(fb), fb.shape[0], fb.shape[1]
    db_mul = 10.0 * np.log10(2.0)
    db_sub = 10.0 * np.log10(max(amin, ref))
    LL = ctypes.c_longlong
    rc = lib.kb_emu_stft_mc(_fp(x), LL(sb), LL(sc), LL(sl), B, C, L, n_fft, win_length, hop, pad_left, T,
                            _fp(window), mode, _fp(out), LL(osb), LL(osc), LL(ost), LL(osk),
                            ctypes.c_float(amin), ctypes.c_float(db_mul), ctypes.c_float(db_sub), _fp(item_max),
                            TF, n_warps, n_cta, db_on, LL(C * osc), fbp, nfreq, nb)
    assert rc == 0, rc
    return out, item_max.view(np.float32)


def emu_istft(X, n_fft, win_length, hop, dual_window, in_fmt, out_fmt, TFc=16, n_warps=4, n_cta=3, seg=None):
    """X: (B, T, F, C) channels_last or (B, C, T, F) channels_first complex64.  seg=None: the class-ordered overlap-add
    body (kb_istft_cta, tiles of TFc frames); seg=k: the streaming body (kb_istft2_cta, tiles of k output hops)."""
    lib = load()
    X = np.ascontiguousarray(X, dtype=np.complex64)
    if in_fmt == 'channels_last':
        B, T, F, C = X.shape
        sb, st, sk, sc = T * F * C, F * C, C, 1
    else:
        B, C, T, F = X.shape
        sb, sc, st, sk = C * T * F, T * F, F, 1
    out_len = (T - 1) * hop + win_length
    if out_fmt == 'channels_last':
        y = np.full((B, out_len, C), np.nan, dtype=np.float32)
        ysb, ysl, ysc = out_len * C, C, 1
    else:
        y = np.full((B, C, out_len), np.nan, dtype=np.float32)
        ysb, ysc, ysl = C * out_len, out_len, 1
    dual = np.ascontiguousarray(dual_window, dtype=np.float32)
    LL = ctypes.c_longlong
    if seg is not None:
        rc = lib.kb_emu_istft2(_fp(X), LL(sb), LL(sc), LL(st), LL(sk), B, C, T, n_fft, win_length, hop,
                               _fp(dual), _fp(y), LL(ysb), LL(ysc), LL(ysl), int(seg), n_warps, n_cta)
    else:
        rc = lib.kb_emu_istft(_fp(X), LL(sb), LL(sc), LL(st), LL(sk), B, C, T, n_fft, win_length, hop,
                              _fp(dual), _fp(y), LL(ysb), LL(ysc), LL(ysl), TFc, n_warps, n_cta)
    assert rc == 0
    return y


def _strides4(shape, fmt):
    """(shape of the array, element strides (b, c, t, k)) of a (B, C, T, K) tensor in `fmt`."""
    B, C, T, K = shape
    if fmt == 'channels_last':
        return (B, T, K, C), (T * K * C, 1, K * C, C)
    return (B, C, T, K), (C * T * K, T * K, K, 1)


def emu_dft(x, n_fft, win_length, hop, window, pad_begin, pad_end, mode, in_fmt, out_fmt, n_cta=3):
    """Generic-n_fft forward kernel body (aux_core.cuh kb_dft_cta): complex or magnitude output."""
    lib = load()
    x = np.ascontiguousarray(x, dtype=np.float32)
    if in_fmt == 'channels_last':
        B, L, C = x.shape
        sb, sl, sc = L * C, C, 1
    else:
        B, C, L = x.shape
        sb, sc, sl = C * L, L, 1
    pad_left = (n_fft - hop) if pad_begin else 0
    Lp = L + pad_left
    T = -(-Lp // hop) if pad_end else max(0, 1 + (Lp - win_length) // hop)
    shape, (osb, osc, ost, osk) = _strides4((B, C, T, n_fft // 2 + 1), out_fmt)
    out = np.full(shape, np.nan, dtype=np.complex64 if mode == MODE_COMPLEX else np.float32)
    window = np.ascontiguousarray(window, dtype=np.float32)
    LL = ctypes.c_longlong
    rc = lib.kb_emu_dft(_fp(x), LL(sb), LL(sc), LL(sl), B, C, L, n_fft, win_length, hop, pad_left, T, _fp(window),
                        mode, _fp(out), LL(osb), LL(osc), LL(ost), LL(osk), n_cta)
    assert rc == 0
    return out


def emu_mr(x, n_fft, win_length, hop, window, pad_begin, pad_end, mode, in_fmt, out_fmt, n_warps=4, fpw=2, n_cta=3, group=1,
           fb=None, amin=1e-5, ref=1.0, frt=8, with_item_max=False):
    """Mixed-radix Stockham forward kernel body (mr_core.cuh kb_mr_cta): complex or magnitude output, or the fused
    tail (MODE_MAG_DB, MODE_FB, MODE_FB_DB; filterbank tiles of `frt` frames).  Returns None when n_fft has a prime
    factor above 5 (the library then uses the direct DFT); (out, item_max) with with_item_max."""
    lib = load()
    x = np.ascontiguousarray(x, dtype=np.float32)
    if in_fmt == 'channels_last':
        B, L, C = x.shape
        sb, sl, sc = L * C, C, 1
    else:
        B, C, L = x.shape
        sb, sc, sl = C * L, L, 1
    pad_left = (n_fft - hop) if pad_begin else 0
    Lp = L + pad_left
    T = -(-Lp // hop) if pad_end else max(0, 1 + (Lp - win_length) // hop)
    K = fb.shape[1] if mode in (MODE_FB, MODE_FB_DB) else n_fft // 2 + 1
    shape, (osb, osc, ost, osk) = _strides4((B, C, T, K), out_fmt)
    out = np.full(shape, np.nan, dtype=np.complex64 if mode == MODE_COMPLEX else np.float32)
    window = np.ascontiguousarray(window, dtype=np.float32)
    item_max = np.zeros(B, dtype=np.uint32)
    fbp, nfreq, nb = None, 0, 0
    if fb is not None:
        fb = np.ascontiguousarray(fb, dtype=np.float32)
        fbp, nfreq, nb = _fp(fb), fb.shape[0], fb.shape[1]
    db_mul = 10.0 * np.log10(2.0)
    db_sub = 10.0 * np.log10(max(amin, ref))
    LL = ctypes.c_longlong
    rc = lib.kb_emu_mr(_fp(x), LL(sb), LL(sc), LL(sl), B, C, L, n_fft, win_length, hop, pad_left, T, _fp(window),
                       mode, _fp(out), LL(osb), LL(osc), LL(ost), LL(osk), n_warps, fpw, n_cta, group,
                       fbp, nfreq, nb, ctypes.c_float(amin), ctypes.c_float(db_mul), ctypes.c_float(db_sub),
                       _fp(item_max), int(frt))
    if rc == -3:
        return None
    assert rc == 0, rc
    return (out, item_max.view(np.float32)) if with_item_max else out


def emu_idft(X, n_fft, win_length, hop, dual_window, in_fmt, out_fmt, n_cta=3):
    """Generic-n_fft inverse kernel body (kb_idft_cta)."""
    lib = load()
    X = np.ascontiguousarray(X, dtype=np.complex64)
    if in_fmt == 'channels_last':
        B, T, F, C = X.shape
    else:
        B, C, T, F = X.shape
    _, (sb, sc, st, sk) = _strides4((B, C, T, F), in_fmt)
    out_len = (T - 1) * hop + win_length
    if out_fmt == 'channels_last':
        y = np.full((B, out_len, C), np.nan, dtype=np.float32)
        ysb, ysl, ysc = out_len * C, C, 1
    else:
        y = np.full((B, C, out_len), np.nan, dtype=np.float32)
        ysb, ysc, ysl = C * out_len, out_len, 1
    dual = np.ascontiguousarray(dual_window, dtype=np.float32)
    LL = ctypes.c_longlong
    rc = lib.kb_emu_idft(_fp(X), LL(sb), LL(sc), LL(st), LL(sk), B, C, T, n_fft, win_length, hop, _fp(dual), _fp(y),
                         LL(ysb), LL(ysc), LL(ysl), n_cta)
    assert rc == 0
    return y


def emu_fb(x, fb, fmt, n_cta=3, R=32):
    """Stand-alone ApplyFilterbank kernel body (kb_fb_cta) on a (B, T, F, C) / (B, C, T, F) float tensor."""
    lib = load()
    x = np.ascontiguousarray(x, dtype=np.float32)
    if fmt == 'channels_last':
        B, T, F, C = x.shape
    else:
        B, C, T, F = x.shape
    _, (sb, sc, st, sk) = _strides4((B, C, T, F), fmt)
    fb = np.ascontiguousarray(fb, dtype=np.float32)
    M = fb.shape[1]
    shape, (osb, osc, ost, osk) = _strides4((B, C, T, M), fmt)
    out = np.full(shape, np.nan, dtype=np.float32)
    LL = ctypes.c_longlong
    rc = lib.kb_emu_fb(_fp(x), LL(sb), LL(sc), LL(st), LL(sk), B, C, T, _fp(fb), fb.shape[0], M, _fp(out), LL(osb),
                       LL(osc), LL(ost), LL(osk), n_cta, R)
    assert rc == 0
    return out


def emu_db_tail(x, amin=1e-5, ref=1.0):
    """The fused kernels' decibel tail (db_mul * log2(max(x, amin)) - db_sub, host build of the same source) on a
    float32 array, with the constants emu_stft passes."""
    lib = load()
    x = np.ascontiguousarray(x, np.float32)
    out = np.empty_like(x)
    lib.kb_emu_db_tail(_fp(x), _fp(out), ctypes.c_longlong(x.size), ctypes.c_float(amin),
                       ctypes.c_float(10.0 * np.log10(2.0)), ctypes.c_float(10.0 * np.log10(max(amin, ref))))
    return out


def emu_atan2(y, x):
    """kb_atan2 of kapre_b200/csrc/stft_core.cuh (host build of the same source) on float32 arrays."""
    lib = load()
    y = np.ascontiguousarray(y, np.float32)
    x = np.ascontiguousarray(x, np.float32)
    out = np.empty_like(y)
    lib.kb_emu_atan2(_fp(y), _fp(x), _fp(out), ctypes.c_longlong(y.size))
    return out


def emu_cabs(re, im, rn):
    """kb_cabs<rn> of kapre_b200/csrc/stft_core.cuh (host build of the same source) on float32 arrays."""
    lib = load()
    re = np.ascontiguousarray(re, np.float32)
    im = np.ascontiguousarray(im, np.float32)
    out = np.empty_like(re)
    lib.kb_emu_cabs(_fp(re), _fp(im), _fp(out), ctypes.c_longlong(re.size), ctypes.c_int(int(rn)))
    return out
