"""CPU tier: the backward passes at every launch shape their transform launchers can pick, and the pre-decibel
values the fused stack's backward recomputes.

* STFT^T is the inverse-STFT launch with the dual window w N/2 (either body: the streaming one with its segment length,
  the class-ordered one with its tile length and warp count) followed by the edge/crop pass.  The inverse bodies sum
  overlapping frames in an order that follows the tile length, so every shape is held to the float64 vector-Jacobian
  product (grad_ref.py), within the 3e-5 of the maximum that test_grad_emu.py allows the same bodies, and samples that
  no frame covers must be exactly 0.
* ISTFT^T is the forward launch with the window dual 2/N followed by the DC/Nyquist pass.  The forward bodies give
  the same bits at every tile shape, CTA count and staging path (test_emu_launch_invariance.py), and so must they
  with the adjoint's window, including at odd sample offsets where a cosine-sum adjoint window is read from the table
  rather than formed in registers.  One launch per case is held to the float64 product.
* The fused stack's backward recomputes the pre-decibel magnitudes (MODE_MAG) or filterbank energies (MODE_FB) with a
  second launch and re-derives the dynamic-range clamp and the item maximum from them.  That is only consistent with
  the forward if MODE_MAG_DB / MODE_FB_DB are, bit for bit, the decibel tail applied to MODE_MAG / MODE_FB, and if the
  forward's item maximum is the maximum of max(MODE_MAG, amin).  Both are checked at every tile shape, pair-step form
  and filterbank phase, for the single-channel, all-channel and mixed-radix bodies.
"""
import numpy as np
import pytest
import torch

import emu_harness as E
import grad_ref as R
from oracle import reference as ref
from test_emu_launch_invariance import mel, same_bits, sc_shapes
from test_grad_emu import _close, _emu_istft_adj, _emu_stft_adj, _spec, _wave

CF, CL = 'channels_first', 'channels_last'
ISTFT_NW = 4            # KB_ISTFT_MAX_WARPS: the streaming body always runs 4-warp CTAs


def _istft_shapes(n_fft, win, hop):
    """The inverse launches kapre_istft_inverse may make: the streaming body with seg = m * FR - (R - 1) output hops
    for m = 1..8 (KAPRE_B200_ISTFT2_M), and the class-ordered body with TFc = R * NW * FPW for NW = 4, 2, 1
    (KAPRE_B200_ISTFT2=0 with KAPRE_B200_INW)."""
    fpw = 32 // (n_fft // 64)
    R_ = -(-min(win, n_fft) // hop)
    out = [dict(seg=m * ISTFT_NW * fpw - (R_ - 1), n_warps=ISTFT_NW) for m in range(1, 9)
           if m * ISTFT_NW * fpw - (R_ - 1) >= 1]
    out += [dict(TFc=max(R_ * nw * fpw, R_), n_warps=nw) for nw in (4, 2, 1)]
    return out


# n_fft, win_length, hop: the fused sizes, a window shorter than n_fft, and gaps between frames (hop > win_length)
STFT_ADJ_CASES = [(256, 256, 64), (512, 384, 128), (1024, 1024, 256), (2048, 2048, 512), (256, 200, 240),
                  (512, 300, 400)]
PADS = [(False, False), (True, False), (False, True), (True, True)]


@pytest.mark.parametrize('pads', PADS, ids=lambda p: 'pb%d_pe%d' % p)
@pytest.mark.parametrize('case', STFT_ADJ_CASES, ids=lambda c: 'n%d_w%d_h%d' % c)
def test_stft_adjoint_at_every_inverse_shape(case, pads):
    n_fft, win, hop = case
    pb, pe = pads
    rng = np.random.default_rng(n_fft + win + hop + 2 * pb + pe)
    win_eff = min(win, n_fft)
    B, C = 3, 2
    L = 9 * max(n_fft, win) + 3 * hop + 7
    pad_left = n_fft - hop if pb else 0
    T = ref.num_frames(L + pad_left, win, hop, pe)
    fi, fo = CF, CL
    x = _wave(rng, B, C, L, fi)
    G = _spec(rng, B, C, T, n_fft // 2 + 1, fo)
    _, want = R.vjp(lambda t: R.stft(t, n_fft, win, hop, None, pb, pe, fi, fo), torch.from_numpy(x.astype(np.float64)),
                    torch.from_numpy(G.astype(np.complex128)))
    want = want.numpy()
    w = ref.get_window(None, win).astype(np.float32)
    dual_adj = np.zeros(win, np.float32)
    dual_adj[:win_eff] = w[:win_eff].astype(np.float64) * n_fft / 2
    # samples of the signal that no frame's first win_eff samples reach: they do not enter the STFT
    u = np.arange(L) + pad_left
    covered = np.zeros(L, bool)
    for t in range(T):
        covered |= (u >= t * hop) & (u < t * hop + win_eff)
    shapes = _istft_shapes(n_fft, win, hop)
    assert sum('seg' in s for s in shapes) >= 4 and sum('TFc' in s for s in shapes) == 3
    for i, kw in enumerate(shapes):
        ola = E.emu_istft(G, n_fft, win, hop, dual_adj, fo, CF, n_cta=(1, 2, 5)[i % 3], **kw)
        got = _emu_stft_adj(G, ola, B, C, L, T, n_fft, hop, win_eff, pad_left, w[:win_eff], fo, fi)
        _close(got, want)
        assert not got[:, :, ~covered].any(), kw


HANN_HAMMING = ['hann_window', 'hamming_window']


def _istft_adj_window(n_fft, win, hop, wname):
    dual = ref.inverse_stft_window(win, hop, ref.get_window(wname, win))
    return (dual * 2.0 / n_fft).astype(np.float32)


def _is_cosine(w, n_fft):
    lib = E.load()
    wh, cwq, a0 = np.zeros(n_fft, np.float32), np.zeros(4 * (n_fft // 64), np.float32), np.zeros(1, np.float32)
    return lib.kb_emu_window_tables(E._fp(np.ascontiguousarray(w)), len(w), n_fft, E._fp(wh), E._fp(cwq),
                                    E._fp(a0)) == 1


@pytest.mark.parametrize('wname', HANN_HAMMING)
@pytest.mark.parametrize('n_fft,hop', [(256, 64), (512, 128), (1024, 256), (2048, 512)])
def test_istft_adjoint_same_bits_at_every_forward_shape(n_fft, hop, wname):
    """Every single-channel tile shape, CTA count, double buffer and bulk copy; gradients of odd length (items at odd
    sample offsets, which read the adjoint window's table) and of even length; each item alone."""
    win = n_fft
    w_adj = _istft_adj_window(n_fft, win, hop, wname)
    assert _is_cosine(w_adj, n_fft)               # the register-window path is in play
    rng = np.random.default_rng(n_fft + len(wname))
    B, T = 4, 37
    out_len = (T - 1) * hop + win
    shapes = sc_shapes(n_fft, hop, E.MODE_COMPLEX, None)
    assert len(shapes) >= 6, shapes
    X = _spec(rng, B, 1, T, n_fft // 2 + 1, CF)
    base = rng.standard_normal((B, 1, out_len + 1)).astype(np.float32)
    _, want = R.vjp(lambda t: R.istft(t, n_fft, win, hop, wname, CF, CF), torch.from_numpy(X.astype(np.complex128)),
                    torch.from_numpy(base[:, :, :out_len].astype(np.float64)))
    for odd in (False, True):
        # one extra sample past the last frame: the same frames, but items 1 and 3 start at odd offsets
        gy = base if odd else np.ascontiguousarray(base[:, :, :out_len])

        def run(g, tf, nw, **kw):
            out, _ = E.emu_stft(g, n_fft, win, hop, w_adj, False, False, E.MODE_COMPLEX, CF, CF, TF=tf, n_warps=nw,
                                **kw)
            assert out.shape[2] == T
            return out

        tf0, nw0 = shapes[0]
        ref0 = run(gy, tf0, nw0, n_cta=3, dbuf=0, bulk=1)
        if odd:
            assert same_bits(ref0, even_ref)
        even_ref = ref0
        for i, (tf, nw) in enumerate(shapes):
            kw = dict(n_cta=(1, 2, 5)[i % 3], dbuf=i % 2, bulk=(i // 2) % 2)
            assert same_bits(run(gy, tf, nw, **kw), ref0), (tf, nw, kw, odd)
        for b in range(B):
            assert same_bits(run(np.ascontiguousarray(gy[b:b + 1]), tf0, nw0, n_cta=2), ref0[b:b + 1]), (b, odd)
    _close(_emu_istft_adj(even_ref.copy(), CF, n_fft), want.numpy())


@pytest.mark.parametrize('C', [2, 3, 7, 16, 31, 32])
def test_istft_adjoint_same_bits_at_every_all_channel_shape(C):
    n_fft, hop = (512, 128) if C % 2 else (1024, 256)
    win = n_fft
    w_adj = _istft_adj_window(n_fft, win, hop, 'hann_window')
    rng = np.random.default_rng(C)
    B, T = 2, 9
    out_len = (T - 1) * hop + win
    X = _spec(rng, B, C, T, n_fft // 2 + 1, CL)
    gy = rng.standard_normal((B, out_len, C)).astype(np.float32)
    _, want = R.vjp(lambda t: R.istft(t, n_fft, win, hop, 'hann_window', CL, CL),
                    torch.from_numpy(X.astype(np.complex128)), torch.from_numpy(gy.astype(np.float64)))
    fpw = 32 // (n_fft // 64)
    ref0, ran = None, 0
    for nw in (1, 2, 4, 8):
        for tf in (1, 2, 3, 5, 8):
            if tf * C > 8 * nw * fpw or nw * 32 < C:      # more than kb_pick_mc_cfg's 8 rounds, or too few loaders
                continue
            out, _ = E.emu_stft_mc(gy, n_fft, win, hop, w_adj, False, False, E.MODE_COMPLEX, CL, CL, TF=tf, n_warps=nw,
                                   n_cta=(1, 2, 5)[ran % 3])
            if ref0 is None:
                ref0 = out
                _close(_emu_istft_adj(out.copy(), CL, n_fft), want.numpy())
            assert same_bits(out, ref0), (nw, tf)
            ran += 1
    assert ran >= 3


@pytest.mark.parametrize('n_fft', [400, 1000, 480])
def test_istft_adjoint_same_bits_at_every_mixed_radix_shape(n_fft):
    hop = n_fft // 4
    w_adj = _istft_adj_window(n_fft, n_fft, hop, 'hamming_window')
    rng = np.random.default_rng(n_fft)
    B, T = 3, 11
    out_len = (T - 1) * hop + n_fft
    X = _spec(rng, B, 1, T, n_fft // 2 + 1, CF)
    gy = rng.standard_normal((B, 1, out_len + 1)).astype(np.float32)   # odd item stride
    _, want = R.vjp(lambda t: R.istft(t, n_fft, n_fft, hop, 'hamming_window', CF, CF),
                    torch.from_numpy(X.astype(np.complex128)), torch.from_numpy(gy[:, :, :out_len].astype(np.float64)))
    ref0, ran = None, 0
    for nw, fpw, group in ((4, 2, 1), (8, 1, 1), (8, 2, 2), (16, 1, 4), (2, 4, 1)):
        out = E.emu_mr(gy, n_fft, n_fft, hop, w_adj, False, False, E.MODE_COMPLEX, CF, CF, n_warps=nw, fpw=fpw,
                       group=group, n_cta=(1, 2, 5)[ran % 3])
        assert out.shape[2] == T
        if ref0 is None:
            ref0 = out
            _close(_emu_istft_adj(out.copy(), CF, n_fft), want.numpy())
        assert same_bits(out, ref0), (nw, fpw, group)
        ran += 1
    for b in range(B):
        out = E.emu_mr(np.ascontiguousarray(gy[b:b + 1, :, :out_len]), n_fft, n_fft, hop, w_adj, False, False,
                       E.MODE_COMPLEX, CF, CF)
        assert same_bits(out, ref0[b:b + 1]), b


# --------------------------------------------------------------------------- the fused stack's pre-decibel values
def _pair_check(db_out, lin_out, db_max, B):
    """db_out must be the decibel tail of lin_out bit for bit, and the forward's item maximum the maximum of
    max(lin_out, amin) per item."""
    assert same_bits(db_out, E.emu_db_tail(lin_out))
    floored = np.maximum(lin_out.reshape(B, -1), np.float32(1e-5))
    assert same_bits(db_max, floored.max(axis=1))


@pytest.mark.parametrize('n_fft,hop', [(256, 64), (512, 128), (1024, 256), (2048, 512)])
def test_decibel_modes_are_the_tail_of_the_linear_modes_single_channel(n_fft, hop):
    rng = np.random.default_rng(n_fft)
    B = 3
    x = rng.uniform(-1, 1, size=(B, 1, 21 * hop + hop // 2 + 1)).astype(np.float32)
    x[1] *= 1e-4                                          # values near and below amin
    w = ref.get_window('hann_window', n_fft).astype(np.float32)
    fb = mel(n_fft)
    ran = 0
    for lin_mode, db_mode in ((E.MODE_MAG, E.MODE_MAG_DB), (E.MODE_FB, E.MODE_FB_DB)):
        fbm = fb if lin_mode == E.MODE_FB else None
        # fb_mma bits: 1 tensor-core filterbank, 2 band descriptors, 4 the other pair-step form
        variants = (0, 1, 2, 4) if fbm is not None else (0, 4)
        for var in variants:
            for i, (tf, nw) in enumerate(sc_shapes(n_fft, hop, lin_mode, fbm)):
                kw = dict(fb=fbm, TF=tf, n_warps=nw, n_cta=(1, 2, 5)[i % 3], fb_mma=var)
                lin, _ = E.emu_stft(x, n_fft, n_fft, hop, w, True, True, lin_mode, CF, CF, **kw)
                db, db_max = E.emu_stft(x, n_fft, n_fft, hop, w, True, True, db_mode, CF, CF, db_on=0, **kw)
                _pair_check(db, lin, db_max, B)
                ran += 1
    assert ran >= 20


@pytest.mark.parametrize('C', [2, 3, 7, 16])
def test_decibel_modes_are_the_tail_of_the_linear_modes_all_channel(C):
    n_fft, hop = (512, 128) if C % 2 else (1024, 256)
    rng = np.random.default_rng(C)
    B = 2
    x = rng.uniform(-1, 1, size=(B, 11 * hop + 1, C)).astype(np.float32)
    w = ref.get_window('hann_window', n_fft).astype(np.float32)
    fb = mel(n_fft)
    fpw = 32 // (n_fft // 64)
    ran = 0
    for nw in (1, 2, 4, 8):
        for tf in (1, 2, 3, 5):
            if tf * C > 8 * nw * fpw or nw * 32 < C:
                continue
            lin, _ = E.emu_stft_mc(x, n_fft, n_fft, hop, w, True, True, E.MODE_MAG, CL, CL, TF=tf, n_warps=nw)
            db, db_max = E.emu_stft_mc(x, n_fft, n_fft, hop, w, True, True, E.MODE_MAG_DB, CL, CL, TF=tf, n_warps=nw)
            _pair_check(db, lin, db_max, B)
            ran += 1
    assert ran >= 3
    for nw in (2, 4, 8):                                  # filterbank tiles: TF = NW * FPW / C frames (kb_pick_mcfb_cfg)
        if nw * fpw < C or nw * 32 < C or nw * fpw > 32:
            continue
        tf = nw * fpw // C
        lin, _ = E.emu_stft_mc(x, n_fft, n_fft, hop, w, True, True, E.MODE_FB, CL, CL, fb=fb, TF=tf, n_warps=nw)
        db, db_max = E.emu_stft_mc(x, n_fft, n_fft, hop, w, True, True, E.MODE_FB_DB, CL, CL, fb=fb, TF=tf,
                                   n_warps=nw)
        _pair_check(db, lin, db_max, B)


@pytest.mark.parametrize('n_fft', [400, 1000])
def test_decibel_modes_are_the_tail_of_the_linear_modes_mixed_radix(n_fft):
    hop = n_fft // 4
    rng = np.random.default_rng(n_fft)
    B = 3
    x = rng.uniform(-1, 1, size=(B, 1, 30 * hop + 1)).astype(np.float32)
    w = ref.get_window('hann_window', n_fft).astype(np.float32)
    fb = mel(n_fft)
    for nw, fpw, group in ((4, 2, 1), (8, 2, 2), (16, 1, 4)):
        lin = E.emu_mr(x, n_fft, n_fft, hop, w, True, True, E.MODE_MAG, CF, CF, n_warps=nw, fpw=fpw, group=group)
        db, db_max = E.emu_mr(x, n_fft, n_fft, hop, w, True, True, E.MODE_MAG_DB, CF, CF, n_warps=nw, fpw=fpw,
                              group=group, with_item_max=True)
        _pair_check(db, lin, db_max, B)
        for frt in (32, 16, 8):
            if frt % (nw // group) or nw // group > frt:
                continue
            lin = E.emu_mr(x, n_fft, n_fft, hop, w, True, True, E.MODE_FB, CF, CF, n_warps=nw, fpw=fpw, group=group,
                           fb=fb, frt=frt)
            db, db_max = E.emu_mr(x, n_fft, n_fft, hop, w, True, True, E.MODE_FB_DB, CF, CF, n_warps=nw, fpw=fpw,
                                  group=group, fb=fb, frt=frt, with_item_max=True)
            _pair_check(db, lin, db_max, B)
