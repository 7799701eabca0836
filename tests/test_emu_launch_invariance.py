"""CPU tier: the forward kernel bodies give the same bits whatever the launch shape, the staging path or the place of
an item in the batch.

The single-channel kernel (kb_stft_cta) windows a frame in registers when its first sample sits at an even offset in
shared memory and reads the window table otherwise.  The table holds exactly the register form's values, so the
choice -- which follows the item's offset in the batch, the bulk copy's shift and the tile boundaries -- does not show
in the output.  These tests sweep every tile shape the launcher can pick (kb_pick_fwd_cfg) with the number of CTAs,
the double buffer and the bulk copy, and compare each item with the same item run alone.  The all-channel and
mixed-radix bodies are pinned to the same invariances."""
from fractions import Fraction

import numpy as np
import pytest

import emu_harness as E
import oracle as O

SMEM_OPTIN = 227 * 1024   # per-block shared memory limit of an H100
ALL_MODES = [E.MODE_COMPLEX, E.MODE_MAG, E.MODE_MAG_DB, E.MODE_FB, E.MODE_FB_DB, E.MODE_MAG_PHASE]
MODE_NAMES = {E.MODE_COMPLEX: 'complex', E.MODE_MAG: 'mag', E.MODE_MAG_DB: 'mag_db', E.MODE_FB: 'fb',
              E.MODE_FB_DB: 'fb_db', E.MODE_MAG_PHASE: 'mag_phase'}
FB_MODES = (E.MODE_FB, E.MODE_FB_DB)


def nerr(a, b):
    return float(np.abs(a - b).max() / max(float(np.abs(b).max()), 1e-30))


def same_bits(a, b):
    """Bit-identical arrays (NaN patterns included)."""
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and a.tobytes() == b.tobytes()


def mel(n_fft, n_mels=40):
    return O.filterbank_mel(22050, n_fft // 2 + 1, n_mels, 0.0, None, False, 'slaney').astype(np.float32)


def sc_shapes(n_fft, hop, mode, fb):
    """Every (TF, NW) kb_pick_fwd_cfg may choose for the single-channel kernel: NW in {1, 2, 4, 8} (16 only at
    n_fft 2048 in the filterbank modes), FR = NW * 32 / Q frames per round <= 32, TF a power of two that is a
    multiple of FR (equal to it in the filterbank modes), and a shared-memory footprint within the opt-in limit."""
    lib = E.load()
    Q = n_fft // 64
    fpw = 32 // Q
    fbm = mode in FB_MODES
    n_bands = fb.shape[1] if fbm else 0
    n_chunks = lib.kb_emu_fb_chunks(E._fp(fb), fb.shape[0], fb.shape[1]) if fbm else 0
    out = []
    for nw in (1, 2, 4, 8, 16):
        if nw == 16 and not (Q == 32 and fbm):
            continue
        fr = nw * fpw
        if fr > 32:
            continue
        for tf in (32, 16, 8, 4, 2, 1):
            if (tf != fr) if fbm else (tf % fr):
                continue
            if lib.kb_emu_stft_smem(n_fft, hop, tf, nw, mode, n_bands, n_chunks) > SMEM_OPTIN:
                continue
            out.append((tf, nw))
    return out


def oracle_check(out, x, n_fft, win, hop, wname, pads, mode, fb):
    """The same oracle tolerances as the rest of the suite."""
    fmt = 'channels_first'
    spec = O.stft_layer(x, n_fft, win, hop, wname, pads[0], pads[1], fmt, fmt)
    mag = np.abs(spec)
    if mode == E.MODE_COMPLEX:
        assert nerr(out, spec) < 2e-6
    elif mode == E.MODE_MAG:
        assert nerr(out, mag) < 2e-6
    elif mode == E.MODE_MAG_PHASE:
        C = x.shape[1]
        m, ph = out[:, :C], out[:, C:]
        assert nerr(m, mag) < 2e-6
        ok = mag > 1e-3 * mag.max()
        assert np.abs(np.angle(np.exp(1j * (ph - np.angle(spec)))))[ok].max() < 1e-3
    else:
        # decibel outputs (before the dynamic-range clamp): back to linear, then the linear tolerance
        lin = mag if mode == E.MODE_MAG_DB else np.einsum('bctf,fm->bctm', mag, fb.astype(np.float64))
        got = 10.0 ** (out.astype(np.float64) / 10.0) if mode in (E.MODE_MAG_DB, E.MODE_FB_DB) else out
        if mode != E.MODE_FB:
            lin = np.maximum(lin, 1e-5)
        assert nerr(got, lin) < 2e-6


SC_CASES = [(256, 64), (512, 128), (1024, 256), (2048, 512)]
# (window name, win_length as a fraction of n_fft, odd L): hann and hamming are evaluated in registers at even sample
# offsets; a window shorter than n_fft always comes from the table
SC_WINDOWS = [('hann_window', 1, True), ('hamming_window', 1, True), ('hann_window', 0.75, True),
              ('hann_window', 1, False)]


@pytest.mark.parametrize('mode', ALL_MODES, ids=lambda m: MODE_NAMES[m])
@pytest.mark.parametrize('wname,wfrac,odd', SC_WINDOWS, ids=['hann-oddL', 'hamming-oddL', 'short-oddL', 'hann-evenL'])
@pytest.mark.parametrize('n_fft,hop', SC_CASES)
def test_single_channel_bits_do_not_depend_on_launch(n_fft, hop, wname, wfrac, odd, mode):
    win = int(n_fft * wfrac)
    pads = (True, True) if wname == 'hann_window' else (False, True)
    B = 3
    L = 37 * hop + (hop // 2) + (1 if odd else 0)   # > 32 frames: every item spans two tiles at TF = 32
    rng = np.random.default_rng(n_fft + 7 * mode + win)
    x = rng.uniform(-1, 1, size=(B, 1, L)).astype(np.float32)
    w = O.get_window(wname, win).astype(np.float32)
    fb = mel(n_fft) if mode in FB_MODES else None
    shapes = sc_shapes(n_fft, hop, mode, fb)
    assert len(shapes) >= (3 if mode in FB_MODES else 6), shapes

    def run(xx, tf, nw, **kw):
        out, _ = E.emu_stft(xx, n_fft, win, hop, w, pads[0], pads[1], mode, 'channels_first', 'channels_first',
                            fb=fb, TF=tf, n_warps=nw, **kw)
        return out

    tf0, nw0 = shapes[0]
    ref = run(x, tf0, nw0, n_cta=3, dbuf=0, bulk=1)
    oracle_check(ref, x, n_fft, win, hop, wname, pads, mode, fb)
    # every shape, the number of CTAs (1: one CTA walks every tile), the double buffer and the bulk copy
    for i, (tf, nw) in enumerate(shapes):
        kw = dict(n_cta=(1, 2, 5)[i % 3], dbuf=i % 2, bulk=(i // 2) % 2)
        assert same_bits(run(x, tf, nw, **kw), ref), (tf, nw, kw)
    assert same_bits(run(x, tf0, nw0, n_cta=4, dbuf=1, bulk=0), ref)
    # each item alone (at offset 0, its last tile the last of the tensor) against its place in the batch
    for b in range(B):
        assert same_bits(run(x[b:b + 1], tf0, nw0, n_cta=2, dbuf=0, bulk=1), ref[b:b + 1]), b


def test_sixteen_warp_shape_is_swept():
    """kb_stft_kernel_w16 (n_fft 2048, filterbank modes) is among the shapes the sweep above compares."""
    for mode in FB_MODES:
        assert (16, 16) in sc_shapes(2048, 512, mode, mel(2048))


# ------------------------------------------------------------------------------------------- the window table
def _round32(v):
    """Nearest float32 to the exact rational v, ties to even."""
    best = np.float32(float(v))
    for g in (np.nextafter(best, np.float32(-np.inf)), np.nextafter(best, np.float32(np.inf))):
        d, db = abs(Fraction(float(g)) - v), abs(Fraction(float(best)) - v)
        if d < db or (d == db and (int(g.view(np.uint32)) & 1) == 0):
            best = g
    return best


def _fma32(a, b, c):
    return _round32(Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c)))


def _cos32_q(t):
    return np.float32(0.0) if t == 8 else np.float32(np.cos(2.0 * np.pi * t / 32.0))


def _cos32(t):
    return _cos32_q(t) if t <= 8 else -_cos32_q(16 - t)


def _sin32(t):
    return _cos32_q(8 - t) if t <= 8 else _cos32_q(t - 8)


@pytest.mark.parametrize('n_fft', [256, 512, 1024, 2048])
@pytest.mark.parametrize('wname', ['hann_window', 'hamming_window'])
def test_window_table_equals_register_form(n_fft, wname):
    """wh[2(q + Q j) + e] == fma(ss_e, sin(2 pi j/32), fma(cc_e, -cos(2 pi j/32), a0)), each fma rounded once."""
    lib = E.load()
    Q = n_fft // 64
    w = O.get_window(wname, n_fft).astype(np.float32)
    wh = np.zeros(n_fft, np.float32)
    cwq = np.zeros((Q, 4), np.float32)
    a0 = np.zeros(1, np.float32)
    assert lib.kb_emu_window_tables(E._fp(w), n_fft, n_fft, E._fp(wh), E._fp(cwq), E._fp(a0)) == 1
    want = np.zeros(n_fft, np.float32)
    for q in range(Q):
        for j in range(32):
            cj = _cos32(j) if j <= 16 else _cos32(32 - j)
            sj = _sin32(j) if j <= 16 else -_sin32(32 - j)
            for e in range(2):
                v = a0[0]
                if cj != 0:
                    v = _fma32(cwq[q, e], -cj, v)
                if sj != 0:
                    v = _fma32(cwq[q, 2 + e], sj, v)
                want[2 * (q + Q * j) + e] = v
    assert same_bits(wh, want)
    assert np.abs(wh.astype(np.float64) - 0.5 * w).max() < 3e-7    # still the window, within its float32 rounding
    # a window that is no cosine-sum window over n_fft samples keeps 0.5 * window, zero-padded
    ws = O.get_window(wname, n_fft - 64).astype(np.float32)
    assert lib.kb_emu_window_tables(E._fp(ws), n_fft - 64, n_fft, E._fp(wh), E._fp(cwq), E._fp(a0)) == 0
    assert same_bits(wh, np.concatenate([np.float32(0.5) * ws, np.zeros(64, np.float32)]))


# ------------------------------------------------------------------------------------- all-channel tile bodies
def mc_shapes(n_fft, C, mode):
    """(TF, NW) of the all-channel bodies: kb_pick_mc_cfg's range (TF <= 32, at most 8 rounds of FR columns), and
    for the filterbank modes kb_pick_mcfb_cfg's (NW in {2, 4, 8}, TF = FR / C)."""
    Q = n_fft // 64
    fpw = 32 // Q
    out = []
    if mode in FB_MODES:
        for nw in (2, 4, 8):
            fr = nw * fpw
            if fr <= 32 and fr >= C:
                out.append((fr // C, nw))
        return out
    for nw in (1, 2, 4, 8):
        fr = nw * fpw
        if fr > 32 or nw * 32 < C:
            continue
        for tf in (1, 2, 3, 5, 8):
            if (tf * C + fr - 1) // fr <= 8:
                out.append((tf, nw))
    return out


@pytest.mark.parametrize('mode', ALL_MODES, ids=lambda m: MODE_NAMES[m])
@pytest.mark.parametrize('n_fft,hop,C', [(512, 128, 2), (1024, 256, 3), (256, 64, 5), (2048, 512, 2), (512, 125, 3)])
def test_all_channel_bits_do_not_depend_on_launch(n_fft, hop, C, mode):
    B = 3
    L = 21 * hop + 1
    rng = np.random.default_rng(C * n_fft + mode)
    x = rng.uniform(-1, 1, size=(B, L, C)).astype(np.float32)
    w = O.get_window(None, n_fft).astype(np.float32)
    fb = mel(n_fft) if mode in FB_MODES else None
    shapes = mc_shapes(n_fft, C, mode)
    assert len(shapes) >= (1 if mode in FB_MODES else 3), shapes

    def run(xx, tf, nw, n_cta):
        out, _ = E.emu_stft_mc(xx, n_fft, n_fft, hop, w, True, True, mode, 'channels_last', 'channels_first',
                               fb=fb, TF=tf, n_warps=nw, n_cta=n_cta)
        return out

    ref = run(x, *shapes[0], 3)
    oracle_check(ref, np.ascontiguousarray(x.transpose(0, 2, 1)), n_fft, n_fft, hop, None, (True, True), mode, fb)
    for i, (tf, nw) in enumerate(shapes):
        assert same_bits(run(x, tf, nw, (1, 2, 7)[i % 3]), ref), (tf, nw)
    for b in range(B):
        assert same_bits(run(x[b:b + 1], *shapes[-1], 2), ref[b:b + 1]), b


# ------------------------------------------------------------------------------------------ mixed-radix body
@pytest.mark.parametrize('mode', [E.MODE_COMPLEX, E.MODE_MAG, E.MODE_MAG_DB, E.MODE_FB, E.MODE_FB_DB],
                         ids=lambda m: MODE_NAMES[m])
@pytest.mark.parametrize('n_fft,hop', [(400, 160), (480, 120), (1000, 250)])
def test_mixed_radix_bits_do_not_depend_on_launch(n_fft, hop, mode):
    B, C = 3, 1
    L = 20 * hop + 3
    rng = np.random.default_rng(n_fft + mode)
    x = rng.uniform(-1, 1, size=(B, C, L)).astype(np.float32)
    w = O.get_window(None, n_fft).astype(np.float32)
    fb = mel(n_fft) if mode in FB_MODES else None
    # (n_warps, frames per group, group, filterbank tile) in kb_mr_pick's range: 8 or 16 warps, groups of G warps with
    # 32 G lanes at most max(32, 2 P / largest radix), a filterbank tile of 8, 16 or 32 whole frames per group
    launches = [(8, 16, 1, 8), (16, 4, 2, 8), (8, 8, 2, 16), (16, 16, 1, 16), (16, 8, 2, 32)]
    if n_fft == 1000:
        launches.append((16, 4, 4, 32))

    def run(xx, nw, fpw, group, frt, n_cta):
        return E.emu_mr(xx, n_fft, n_fft, hop, w, True, True, mode, 'channels_first', 'channels_first', n_warps=nw,
                        fpw=fpw, n_cta=n_cta, group=group, fb=fb, frt=frt)

    ref = run(x, *launches[0], 3)
    oracle_check(ref, x, n_fft, n_fft, hop, None, (True, True), mode, fb)
    for i, lc in enumerate(launches[1:]):
        assert same_bits(run(x, *lc, (1, 2, 5)[i % 3]), ref), lc
    for b in range(B):
        assert same_bits(run(x[b:b + 1], *launches[1], 2), ref[b:b + 1]), b
