"""The band-limited interpolator on the CPU: the kernel body of sinc_core.cuh (run by a CPU emulation) against the
float64 restatement (sinc_ref.py) within the bound derived there, its independence of tiling and staging, the adjoint
through the exchanged numbers, ``scipy.signal.resample_poly`` as a sanity check, the ``Speed`` and ``PitchShift``
layers' validation and config, and the restated ``PitchShift`` chain on a sinusoid, a tone burst and an impulse.
"""
import ctypes
import hashlib
import math
import os
import re
import shutil
import subprocess
import tempfile

import numpy as np
import pytest
import torch

import sinc_ref as SR

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, 'emu', 'kb_emu_sinc.cpp')
_CSRC = os.path.join(_HERE, '..', 'kapre_b200', 'csrc')
_lib_handle = None
CL, CF = 'channels_last', 'channels_first'
RATIOS = [0.25, 0.5, 2.0 ** (-4 / 12), 0.9, 1.1, 2.0 ** (5 / 12), 2.0, 4.0]
THREADS = 512
SMEM_HALF = 232448 // 2 - 2048          # the library's first shared-memory budget on an H100: two CTAs per SM


def _lib():
    """tests/emu/kb_emu_sinc.cpp built with g++ into the temporary directory (keyed by the sources' contents, so the
    checkout itself may be read-only)."""
    global _lib_handle
    if _lib_handle is None:
        hs = hashlib.sha256()
        for f in [_SRC] + sorted(os.path.join(_CSRC, n) for n in os.listdir(_CSRC) if n.endswith(('.h', '.cuh'))):
            with open(f, 'rb') as fh:
                hs.update(fh.read())
        out = os.path.join(tempfile.gettempdir(), 'kapre_b200_emu_sinc_%s.so' % hs.hexdigest()[:16])
        if not os.path.exists(out):
            tmp = '%s.%d.tmp' % (out, os.getpid())
            subprocess.check_call(['g++', '-O2', '-std=c++17', '-shared', '-fPIC', '-DKB_HOST_EMU', '-Wno-unknown-pragmas',
                                   '-o', tmp, _SRC])
            os.replace(tmp, out)
        lib = ctypes.CDLL(out)
        I, D, P = ctypes.c_int, ctypes.c_double, ctypes.c_void_p
        lib.kb_emu_sinc.argtypes = [P, P, ctypes.c_longlong, I, I, I, P, P, I, D, D, I, I, I, I, I, I]
        lib.kb_emu_sinc_integral.restype = D
        lib.kb_emu_sinc_h.restype = D
        lib.kb_emu_sinc_h.argtypes = [D]
        lib.kb_emu_sinc_table.argtypes = [P]
        lib.kb_emu_sinc_smem.argtypes = [I, D, I, I]
        _lib_handle = lib
    return _lib_handle


def _fp(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def pick_nt(ratio, adjoint, G):
    """The library's tile: the largest power of two <= 2048 whose staged span fits beside the table."""
    for nt in (2048, 1024, 512, 256, 128, 64, 32, 16, 8, 4, 2, 1):
        if _lib().kb_emu_sinc_smem(nt, ratio, int(adjoint), G) <= SMEM_HALF:
            return nt
    raise AssertionError('no tile fits')


def emu_sinc(x, fmt, ratio, length=None, offset=0.0, adjoint=False, NT=None, n_threads=THREADS, n_cta=3, bulk=None):
    """Run the kernel body on the NumPy array `x` ((B, L, C) channels_last or (B, C, L), any strides, possibly a view
    into a larger buffer) with the library's choice of channel grouping, tile and loader unless overridden."""
    if fmt == CL:
        B, L, C = x.shape
        sb, sl, sc = (s // 4 for s in x.strides)
    else:
        B, C, L = x.shape
        sb, sc, sl = (s // 4 for s in x.strides)
    base = x.base if x.base is not None else x
    numel = ((B - 1) * sb + (C - 1) * sc + (L - 1) * sl + 1) if x.size else 0
    assert numel <= base.size
    Lo = SR.output_length(L, ratio) if length is None else length
    y = np.full((B, Lo, C) if fmt == CL else (B, C, Lo), np.nan, dtype=np.float32)
    ys = np.array([y.strides[0], y.strides[2], y.strides[1]] if fmt == CL else [s for s in y.strides], np.int64) // 4
    xs = np.array([sb, sc, sl], np.int64)
    G = C if (1 < C <= n_threads and abs(sc) < abs(sl)) else 1            # kb_sinc_launch's choice
    can_bulk = int((G == 1 and sl == 1) or (G == C and sc == 1 and sl == C))
    if NT is None:
        NT = pick_nt(ratio, adjoint, G)
    rc = _lib().kb_emu_sinc(x.ctypes.data, _fp(xs), numel, B, C, L, _fp(y), _fp(ys), Lo, float(ratio), float(offset),
                            int(adjoint), G, NT, n_threads, n_cta, can_bulk if bulk is None else int(bulk and can_bulk))
    assert rc == 0
    return y


def _ref(x, fmt, ratio, length=None, offset=0.0):
    """Restatement on a (B, L, C) / (B, C, L) array, same layout out."""
    t = torch.from_numpy(np.ascontiguousarray(x, np.float64))
    if fmt == CL:
        return SR.resample(t.transpose(1, 2), ratio, length, offset).transpose(1, 2).numpy()
    return SR.resample(t, ratio, length, offset).numpy()


def _close(got, want, ratio, xmax, adjoint=False):
    assert got.shape == want.shape, (got.shape, want.shape)
    if got.size:
        err = float(np.abs(got - want).max())
        assert err <= SR.error_bound(ratio, adjoint) * xmax, (err, SR.error_bound(ratio, adjoint) * xmax)


def _signal(rng, fmt, B, C, L):
    return rng.uniform(-1, 1, size=(B, L, C) if fmt == CL else (B, C, L)).astype(np.float32)


# ------------------------------------------------------------------------------------------ the filter and its table
def test_filter_integral_and_table():
    lib = _lib()
    u = np.linspace(-10.5, 10.5, 2001)
    got = np.array([lib.kb_emu_sinc_h(float(v)) for v in u])
    np.testing.assert_allclose(got, SR.h(u), rtol=0, atol=1e-14)
    assert abs(lib.kb_emu_sinc_integral() - SR.INTEGRAL) <= 1e-11
    tab = np.empty((SR.Z * SR.Q + 1, 2), np.float32)
    lib.kb_emu_sinc_table(_fp(tab))
    hk = SR.h(np.arange(SR.Z * SR.Q + 2) / SR.Q)
    np.testing.assert_array_equal(tab[:, 0], hk[:-1].astype(np.float32))
    np.testing.assert_array_equal(tab[:-1, 1], np.diff(hk[:-1]).astype(np.float32))
    assert tab[-1, 0] == 0 and tab[-1, 1] == 0                       # positions past the support read weight 0
    # the derived bound is of the size the float64 experiment measured (1.4e-6 of outputs up to 3.9 at Q = 1024)
    assert 5e-6 < SR.error_bound(1.0) < 2e-5 and 5e-6 < SR.error_bound(0.25) < 2.5e-5


# ------------------------------------------------------------------------------------------ the emulated kernel body
@pytest.mark.parametrize('ratio', RATIOS)
@pytest.mark.parametrize('offset', [0.0, 3.37, -7.25])
@pytest.mark.parametrize('C,fmt', [(1, CF), (2, CL)])
def test_emulated_body_matches_restatement(ratio, offset, C, fmt):
    x = _signal(np.random.default_rng(int(ratio * 1000) + C), fmt, 2, C, 3001)
    got = emu_sinc(x, fmt, ratio, offset=offset)
    _close(got, _ref(x, fmt, ratio, offset=offset), ratio, float(np.abs(x).max()))


@pytest.mark.parametrize('ratio', [0.25, 2.0 ** (-4 / 12), 1.1, 4.0])
@pytest.mark.parametrize('L', [0, 1, 5, 37])
@pytest.mark.parametrize('fmt', [CF, CL])
def test_signals_shorter_than_the_filter(ratio, L, fmt):
    x = _signal(np.random.default_rng(L), fmt, 2, 2, L)
    got = emu_sinc(x, fmt, ratio, offset=0.5)
    _close(got, _ref(x, fmt, ratio, offset=0.5), ratio, 1.0)


@pytest.mark.parametrize('ratio', [0.5, 2.0 ** (5 / 12)])
def test_any_output_length_with_exact_trailing_zeros(ratio):
    L = 700
    x = _signal(np.random.default_rng(3), CF, 1, 1, L)
    natural = SR.output_length(L, ratio)
    short = emu_sinc(x, CF, ratio, length=natural - 100)
    long = emu_sinc(x, CF, ratio, length=natural + 500)
    full = emu_sinc(x, CF, ratio)
    assert np.array_equal(short, full[..., :natural - 100]) and np.array_equal(long[..., :natural], full)
    _close(long, _ref(x, CF, ratio, length=natural + 500), ratio, 1.0)
    support = math.ceil((L - 1 + SR.Z / min(1.0, ratio)) * ratio) + 1         # outputs past it see no sample
    tail = long[..., support:]
    assert tail.size > 0 and not tail.any() and not np.signbit(tail).any()


@pytest.mark.parametrize('view', ['time_stride', 'channel_slice', 'batch_stride', 'misaligned'])
@pytest.mark.parametrize('fmt', [CF, CL])
def test_emulated_body_on_views(view, fmt):
    """Non-contiguous inputs: the cooperative loader (strided time axis, a slice of the channels) and the
    bulk copy of a span that does not start on a 16 B boundary."""
    ratio = 2.0 ** (-4 / 12)
    full = _signal(np.random.default_rng(5), fmt, 3, 4, 3100)
    t_ax, c_ax = (1, 2) if fmt == CL else (2, 1)
    sl = [slice(None)] * 3
    if view == 'time_stride':
        sl[t_ax] = slice(None, None, 2)
    elif view == 'channel_slice':
        sl[c_ax] = slice(1, 3)
    elif view == 'batch_stride':
        sl[0] = slice(None, None, 2)
    elif view == 'misaligned':
        sl[t_ax] = slice(3, 3001)
        sl[c_ax] = slice(0, 1)
    x = full[tuple(sl)]
    got = emu_sinc(x, fmt, ratio, offset=1.5, NT=128, n_cta=2)
    _close(got, _ref(x, fmt, ratio, offset=1.5), ratio, float(np.abs(x).max()))


@pytest.mark.parametrize('ratio', [0.25, 2.0 ** (-4 / 12), 2.0 ** (5 / 12), 4.0])
@pytest.mark.parametrize('C,fmt', [(1, CF), (2, CL), (3, CF)])
def test_output_does_not_depend_on_tiling_or_staging(ratio, C, fmt):
    """The same bits for every tile size, thread count, grid, loader and batch position."""
    x = _signal(np.random.default_rng(9), fmt, 2, C, 2500)
    want = emu_sinc(x, fmt, ratio, offset=0.3)
    for NT, n_threads, n_cta, bulk in [(64, 512, 3, 1), (37, 96, 1, 1), (512, 256, 5, 0), (2048, 32, 2, 1), (1, 64, 7, 0)]:
        if NT == 2048 and ratio < 0.5:
            NT = 1024
        got = emu_sinc(x, fmt, ratio, offset=0.3, NT=NT, n_threads=n_threads, n_cta=n_cta, bulk=bulk)
        assert np.array_equal(got, want), (NT, n_threads, n_cta, bulk)
    swapped = emu_sinc(np.ascontiguousarray(x[::-1]), fmt, ratio, offset=0.3)
    assert np.array_equal(swapped[::-1], want)
    other = np.ascontiguousarray(np.swapaxes(x, 1, 2))                 # the other data format: same numbers
    got = emu_sinc(other, CL if fmt == CF else CF, ratio, offset=0.3)
    assert np.array_equal(np.swapaxes(got, 1, 2), want)


@pytest.mark.parametrize('ratio', RATIOS)
@pytest.mark.parametrize('fmt', [CF, CL])
def test_emulated_adjoint_identity(ratio, fmt):
    """<A x, g> = <x, A^T g> with A^T g = the body run with step, offset and s exchanged (kb_sinc_args), to float32
    rounding, and A^T g against the transpose of the explicit float64 matrix."""
    rng = np.random.default_rng(11)
    L, offset = 900, 2.25
    x = _signal(rng, fmt, 2, 2, L)
    y = emu_sinc(x, fmt, ratio, offset=offset)
    g = rng.uniform(-1, 1, size=y.shape).astype(np.float32)
    gx = emu_sinc(g, fmt, ratio, length=L, offset=offset, adjoint=True)
    lhs = float(np.dot(y.astype(np.float64).ravel(), g.astype(np.float64).ravel()))
    rhs = float(np.dot(x.astype(np.float64).ravel(), gx.astype(np.float64).ravel()))
    assert abs(lhs - rhs) <= 1e-5 * np.sqrt(float((y.astype(np.float64) ** 2).sum() * (g.astype(np.float64) ** 2).sum()))
    A = SR.matrix(L, ratio, y.shape[1 if fmt == CL else 2], offset)
    g64 = g.astype(np.float64)
    want = np.einsum('ml,bmc->blc', A, g64) if fmt == CL else np.einsum('ml,bcm->bcl', A, g64)
    _close(gx, want, ratio, 1.0, adjoint=True)
    # the exchanged numbers are the transpose in exact arithmetic too
    t = torch.from_numpy(np.ascontiguousarray(g64[0, :, 0] if fmt == CL else g64[0, 0]))
    by_formula = SR.resample(t, ratio, L, _numbers=SR.adjoint_numbers(ratio, offset)).numpy()
    np.testing.assert_allclose(by_formula, want[0, :, 0] if fmt == CL else want[0, 0], rtol=0, atol=1e-12)


@pytest.mark.parametrize('up,down,tol', [(160, 441, 1e-6), (1, 3, 6e-4), (3, 2, 6e-4), (2, 1, 6e-4)])
def test_close_to_resample_poly(up, down, tol):
    """At rational ratios this is scipy's polyphase resampler up to its normalisation (scipy divides by the tap sum,
    this divides by the integral): a sanity check, the definition is the restatement."""
    sig = pytest.importorskip('scipy.signal')
    x = np.random.default_rng(2).standard_normal((1, 1, 4000)).astype(np.float32)
    want = sig.resample_poly(x.astype(np.float64), up, down, axis=-1)
    got = emu_sinc(x, CF, up / down, length=want.shape[-1])
    assert float(np.abs(got - want).max()) <= tol


def test_kernel_register_and_spill_budget():
    """kb_sinc_resample_kernel runs 512 threads per CTA, two CTAs per SM: at most 64 registers, no spills."""
    lib = os.path.join(_HERE, '..', 'kapre_b200', '_lib', 'libkapre_b200.so')
    if shutil.which('cuobjdump') is None or not os.path.exists(lib):
        pytest.skip('needs cuobjdump and the built library')
    out = subprocess.run(['cuobjdump', '-res-usage', lib], capture_output=True, text=True, check=True).stdout
    lines = out.splitlines()
    found = [(lines[i], lines[i + 1]) for i in range(len(lines) - 1) if 'kb_sinc_resample_kernel' in lines[i]]
    assert len(found) == 1, found
    m = re.search(r'REG:(\d+) STACK:(\d+)', found[0][1])
    assert m and int(m.group(1)) <= 64 and int(m.group(2)) == 0, found[0]


# ------------------------------------------------------------------------------------------ the layers
def test_speed_validation_and_config():
    from kapre_b200.signal import Speed
    import kapre
    assert kapre.signal.Speed is Speed
    for bad in (0, -1.0, 4.5, 0.2, float('nan'), float('inf'), True, '1.1', None):
        with pytest.raises(ValueError):
            Speed(bad)
    with pytest.raises(ValueError):
        Speed(1.1, data_format='channels_middle')
    layer = Speed(1.1, data_format='channels_first', name='sp')
    cfg = layer.get_config()
    assert cfg['factor'] == 1.1 and cfg['data_format'] == 'channels_first' and cfg['name'] == 'sp'
    assert Speed.from_config(cfg).get_config() == cfg
    assert Speed(4).factor == 4.0 and Speed(np.float32(0.25)).factor == 0.25
    assert layer.output_length(1000) == math.ceil(1000 / 1.1)


def test_pitch_shift_validation_and_config():
    from kapre_b200.augmentation import PitchShift
    import kapre
    assert kapre.augmentation.PitchShift is PitchShift
    for bad in (24.5, -25, float('nan'), float('inf'), True, '4', None):
        with pytest.raises(ValueError):
            PitchShift(bad)
    for bad in (0, -12, 12.0, True):
        with pytest.raises(ValueError):
            PitchShift(1, bins_per_octave=bad)
    with pytest.raises(ValueError):
        PitchShift(4, data_format='channels_middle')
    layer = PitchShift(-3.5, bins_per_octave=24, n_fft=512, hop_length=64, window_name='hann_window',
                       data_format='channels_last', name='ps')
    assert layer.rate(-3.5) == 2.0 ** (3.5 / 24)
    cfg = layer.get_config()
    assert cfg['n_steps'] == -3.5 and cfg['bins_per_octave'] == 24 and cfg['n_fft'] == 512 and cfg['win_length'] == 512
    assert cfg['hop_length'] == 64 and cfg['window_name'] == 'hann_window' and cfg['data_format'] == 'channels_last'
    assert PitchShift.from_config(cfg).get_config() == cfg
    assert PitchShift(24).rate(24) == 0.25 and PitchShift(-24).rate(-24) == 4.0
    # the four steps share the framing, and the offset is the derivation's
    assert layer.stft.pad_begin and layer.stft.pad_end and layer.istft.hop_length == 64
    rate = layer.rate(-3.5)
    assert layer.offset(rate) == SR.pitch_shift_offset(rate, 512, 512, 64)


# ------------------------------------------------------------------------------------------ the PitchShift chain, float64
@pytest.mark.parametrize('n_steps', [-5, 4, 0.5])
def test_restated_pitch_shift_moves_a_sinusoid(n_steps):
    sr, f0, n_fft, hop = 16000, 440.0, 1024, 256
    L = sr
    t = torch.arange(L, dtype=torch.float64) / sr
    x = torch.sin(2 * math.pi * f0 * t).view(1, -1, 1)
    y = SR.pitch_shift(x, n_steps, n_fft=n_fft, hop=hop, window_name='hann_window')
    assert y.shape == x.shape
    mid = y[0, n_fft:L - n_fft, 0]
    spec = torch.fft.rfft(mid * torch.hann_window(mid.numel(), dtype=torch.float64)).abs()
    f_peak = float(spec.argmax()) * sr / mid.numel()
    assert abs(f_peak - f0 * 2.0 ** (n_steps / 12)) <= sr / n_fft, f_peak
    assert 0.5 < float(mid.abs().max()) < 1.5


@pytest.mark.parametrize('n_steps', [-5, 4, 0.5])
@pytest.mark.parametrize('i', [4000, 6555])
def test_restated_pitch_shift_is_time_aligned(n_steps, i):
    """The output is time-aligned with the input.  The offset aligns the frames exactly: the energy of the stretched
    frames, read at the frame centres, has its centroid where the derivation puts it.  Inside a frame a phase vocoder
    moves events (it scales each frame's group delay relative to the first frame's by 1 / rate), so in the waveform a
    tone burst is held to hop_length and a click to half a window."""
    import grad_ref as R
    import time_stretch_ref as TR
    n_fft, hop, L = 1024, 256, 12000
    t = torch.arange(L, dtype=torch.float64)
    burst = (torch.exp(-0.5 * ((t - i) / 600) ** 2) * torch.sin(0.1 * math.pi * t)).view(1, -1, 1)
    rate = 2.0 ** (-n_steps / 12)
    S = TR.time_stretch(R.stft(burst, n_fft, n_fft, hop, 'hann_window', True, True, CL, CF), rate)
    e = (S.abs() ** 2).sum(-1)[0, 0]
    centre = float((e * torch.arange(e.numel())).sum() / e.sum()) * hop + n_fft / 2       # in the inverse's output
    m = (centre - SR.pitch_shift_offset(rate, n_fft, n_fft, hop)) * rate                   # the output sample reading it
    assert abs(m - i) <= 2.0, m
    y = SR.pitch_shift(burst, n_steps, n_fft=n_fft, hop=hop, window_name='hann_window')[0, :, 0]
    assert abs(float((y * y * t).sum() / (y * y).sum()) - i) <= hop
    click = torch.zeros((1, L, 1), dtype=torch.float64)
    click[0, i, 0] = 1.0
    y = SR.pitch_shift(click, n_steps, n_fft=n_fft, hop=hop, window_name='hann_window')[0, :, 0]
    env = torch.nn.functional.avg_pool1d((y * y).view(1, 1, -1), hop + 1, 1, hop // 2).view(-1)
    assert abs(int(env.argmax()) - i) <= n_fft // 2, int(env.argmax())
