"""CPU tier: the bodies that stage input through the TMA bulk copy and an mbarrier use the protocol correctly.

The emulation (stft_core.cuh, KB_HOST_EMU) models the barrier: a bulk copy fills its destination with NaN and lands
only when the wait that completes its phase runs, and every misuse the hardware would turn into a hang, a fault or a
silent race -- a wrong parity, a second arrival in a phase, a misaligned or oversized copy, a wait with nothing in
flight, a CTA that leaves a copy in flight -- counts as a violation.  Every emulation library checks the count after
each call (emu_harness.Checked), so every emulation test checks the protocol; the tests here run each staging body
where it is most exposed: every emulated CTA walks three or more tiles, so it reuses its buffer and its barrier
reaches later phases; its walk mixes bulk tiles with cooperative ones (a tile whose rounded span leaves the input, or
that reaches past an item's ends, is staged by the cooperative loader); and the input starts 0-3 floats after a 16 B
boundary, which moves every tile's head and tail rounding.  Each run has the bits of the cooperative loader's run at
offset 0 and stays within the bound its kernel's emulation test holds it to against the float64 restatement."""
import numpy as np
import pytest
import scipy.signal

import emu_harness as E
import iir_ref as IR
import resample_ref as RR
import sinc_ref as SR
from test_emu_launch_invariance import SC_CASES, mel, oracle_check, same_bits, sc_shapes
from test_iir_emu import _f32, emu as emu_iir
from test_resample_emu import _close as _close_resample, _ref as _ref_resample, emu_resample
from test_sinc_emu import CF, CL, _close as _close_sinc, _ref as _ref_sinc, emu_sinc

OFFSETS = (0, 1, 2, 3)


def at_offset(a, k):
    """A C-contiguous copy of `a` whose first element lies k floats after a 16 B boundary (the rest of its buffer
    around it)."""
    buf = np.zeros(a.size + 8, np.float32)
    i0 = (-(buf.ctypes.data // 4)) % 4
    out = buf[i0 + k:i0 + k + a.size].reshape(a.shape)
    out[...] = a
    assert (out.ctypes.data // 4) % 4 == k
    return out


def test_checker_flags_every_misuse():
    """The model catches each misuse, played on a private buffer (the host only: nothing here runs on a GPU), and
    passes the correct protocol: bit 0 wrong parity, 1 read before the wait, 2 two arrivals in one phase, 3 a
    misaligned destination, source or size, 4 size 0 or 1 MiB, 5 a wait that would hang, 6 re-initialisation with a
    copy in flight, 7 exit with a copy in flight, 8 the correct protocol over three phases."""
    assert E.load().kb_emu_async_selftest() == 0x1ff


# ------------------------------------------------------------------------------------------ STFT (kb_stft_cta)
@pytest.mark.parametrize('mode', [E.MODE_MAG, E.MODE_FB_DB], ids=['mag', 'fb_db'])
@pytest.mark.parametrize('n_fft,hop', SC_CASES)
def test_stft_walks(n_fft, hop, mode):
    """Every Q and every (TF, n_warps) the launcher may pick.  The body stages each tile in its one sample buffer
    (KbStftParams.dbuf is not read), so the next tile's copy must not be issued before the last round has read the
    current one.  Tiles whose rounded span leaves the input (the first at a nonzero offset, the last of the tensor)
    take the cooperative loader."""
    B = 2
    L = 67 * hop + hop // 2 + 1
    w = np.hanning(n_fft + 1)[:-1].astype(np.float32)
    fb = mel(n_fft) if mode in (E.MODE_FB, E.MODE_FB_DB) else None
    x = np.random.default_rng(n_fft + mode).uniform(-1, 1, size=(B, 1, L)).astype(np.float32)

    def run(xx, tf, nw, **kw):
        out, _ = E.emu_stft(xx, n_fft, n_fft, hop, w, True, True, mode, 'channels_first', 'channels_first', fb=fb,
                            TF=tf, n_warps=nw, **kw)
        return out

    shapes = sc_shapes(n_fft, hop, mode, fb)
    T = -(-(L + n_fft - hop) // hop)
    ref = None
    for tf, nw in shapes:
        tiles = B * -(-T // tf)
        n_cta = max(1, tiles // 3 - 1)             # every CTA walks >= 3 tiles
        want = run(x, tf, nw, n_cta=n_cta, dbuf=0, bulk=0)
        if ref is None:
            ref = want
            oracle_check(ref, x, n_fft, n_fft, hop, 'hann_window', (True, True), mode, fb)
        assert same_bits(want, ref), (tf, nw)
        for k in OFFSETS:
            got = run(at_offset(x, k), tf, nw, n_cta=n_cta, dbuf=0, bulk=1)
            assert same_bits(got, ref), (tf, nw, n_cta, k)


# ------------------------------------------------------------------------------------------ IIR (state and output passes)
@pytest.mark.parametrize('k', OFFSETS)
def test_iir_walks(k):
    """Forward (and the reversed scan filtfilt runs second) and backward with the coefficient partials: a block
    whose staged span reaches past either end of the signal takes the cooperative loader, so every column runs
    cooperative, bulk x 4, cooperative, and the emulator walks all of them on one shared-memory buffer."""
    rng = np.random.default_rng(20 + k)
    b32, a32 = _f32(*scipy.signal.butter(8, 0.2))
    bb, ab = b32[None, None], a32[None, None]
    B, C, L = 2, 2, 5 * IR.TC * IR.W + 300
    x = rng.uniform(-1, 1, (B, C, L)).astype(np.float32)
    gy = rng.uniform(-1, 1, (B, C, L)).astype(np.float32)
    for flags in (0, 2):
        want, _ = emu_iir(x, bb, ab, flags=flags, bulk=0)
        got, _ = emu_iir(at_offset(x, k), bb, ab, flags=flags)
        assert same_bits(got, want), flags
    y, _ = emu_iir(x, bb, ab)
    for i, c in ((0, 0), (B - 1, C - 1)):
        ref = IR.lfilter_fast(x[i, c], b32, a32)
        bound = IR.error_bound(b32, a32, np.abs(x[i, c]).max(), np.abs(ref).max(), IR.local_max(x[i, c], b32, a32))
        assert np.abs(y[i, c] - ref).max() <= bound
    gx_want, part_want = emu_iir(gy, bb, ab, bwd=True, xr=x, yr=y, bulk=0)
    gx, part = emu_iir(at_offset(gy, k), bb, ab, bwd=True, xr=x, yr=y)
    assert same_bits(gx, gx_want) and same_bits(part, part_want)
    gx_ref, _, _ = IR.vjp(x[:1, :1], gy[:1, :1], b32, a32)
    v = IR.allpole_adjoint(gy[:1, :1], a32)
    bound = IR.error_bound(b32, a32, 1.0, max(np.abs(gx_ref).max(), np.abs(v).max()),
                           IR.local_max(gy[:1, :1, ::-1], [1.0], a32)) * (1 + np.abs(b32).sum())
    assert np.abs(gx[:1, :1] - gx_ref).max() <= bound


# ------------------------------------------------------------------------------------------ sinc (forward and adjoint)
@pytest.mark.parametrize('k', OFFSETS)
@pytest.mark.parametrize('C,fmt', [(1, CF), (3, CL)], ids=['G1', 'GC'])
@pytest.mark.parametrize('adjoint', [False, True], ids=['fwd', 'adj'])
def test_sinc_walks(adjoint, C, fmt, k):
    """About 10 tiles per (item, channel group) and 7 CTAs: each CTA walks 4-5 tiles, and as 7 does not divide the
    tiles per item its walk alternates between edge tiles (cooperative) and interior ones (bulk)."""
    ratio, offset, B = 2.0 ** (-4 / 12), 1.5, 3
    rng = np.random.default_rng(30 + 4 * C + k + 8 * adjoint)
    Lx = 1500
    L_in = SR.output_length(Lx, ratio) if adjoint else Lx
    x = rng.uniform(-1, 1, size=(B, L_in, C) if fmt == CL else (B, C, L_in)).astype(np.float32)
    kw = dict(length=Lx if adjoint else None, offset=offset, adjoint=adjoint, NT=128)
    want = emu_sinc(x, fmt, ratio, n_cta=2, bulk=0, **kw)
    got = emu_sinc(at_offset(x, k), fmt, ratio, n_cta=7, **kw)
    assert same_bits(got, want)
    if adjoint:
        A = SR.matrix(Lx, ratio, L_in, offset)
        x64 = x.astype(np.float64)
        ref = np.einsum('ml,bmc->blc', A, x64) if fmt == CL else np.einsum('ml,bcm->bcl', A, x64)
        _close_sinc(got, ref, ratio, float(np.abs(x).max()), adjoint=True)
    else:
        _close_sinc(got, _ref_sinc(x, fmt, ratio, offset=offset), ratio, float(np.abs(x).max()))


# ------------------------------------------------------------------------------------------ polyphase resampler
@pytest.mark.parametrize('k', OFFSETS)
@pytest.mark.parametrize('C,fmt', [(1, CF), (2, CL)], ids=['G1', 'GC'])
@pytest.mark.parametrize('orig,target', [(48000, 16000), (16000, 22050)])
def test_resample_walks(orig, target, C, fmt, k):
    """Tiles of 64 outputs, 5 CTAs: every CTA walks 4 or more tiles, mixing edge (cooperative) and interior (bulk)
    ones."""
    from kapre_b200.signal import resample_filter
    up, down = RR.up_down(orig, target)
    rng = np.random.default_rng(40 + C + k)
    L = 1500
    x = rng.uniform(-1, 1, size=(3, L, C) if fmt == CL else (3, C, L)).astype(np.float32)
    h = resample_filter(up, down)
    want = emu_resample(x, fmt, up, down, h, NT=64, n_cta=2, bulk=0)
    got = emu_resample(at_offset(x, k), fmt, up, down, h, NT=64, n_cta=5)
    assert same_bits(got, want)
    _close_resample(got, _ref_resample(x, fmt, up, down), float(np.abs(x).max()))
