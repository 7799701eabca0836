"""The polyphase resampler on the CPU: the NumPy filter design against scipy's, the float64 restatement
(resample_ref.py) against ``scipy.signal.resample_poly``, and the kernel body of resample_core.cuh (run by a CPU
emulation) against the restatement, plus the ``Resample`` layer's validation and config.

The emulated body computes in float32 like the kernel: each output is a dot product of at most 2 hl / up + 2 taps
(62 at 48 kHz -> 16 kHz) whose weights sum to about 1, so it is held to 1e-5 of max|x|.
"""
import ctypes
import hashlib
import itertools
import os
import subprocess
import tempfile

import numpy as np
import pytest
import torch

import resample_ref as RR
from emu_harness import Checked

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, 'emu', 'kb_emu_resample.cpp')
_CSRC = os.path.join(_HERE, '..', 'kapre_b200', 'csrc')
_lib_handle = None
CL, CF = 'channels_last', 'channels_first'


def _lib():
    """tests/emu/kb_emu_resample.cpp built with g++ into the temporary directory (keyed by the sources' contents, so
    the checkout itself may be read-only)."""
    global _lib_handle
    if _lib_handle is None:
        h = hashlib.sha256()
        for f in [_SRC] + sorted(os.path.join(_CSRC, n) for n in os.listdir(_CSRC) if n.endswith(('.h', '.cuh'))):
            with open(f, 'rb') as fh:
                h.update(fh.read())
        out = os.path.join(tempfile.gettempdir(), 'kapre_b200_emu_resample_%s.so' % h.hexdigest()[:16])
        if not os.path.exists(out):
            tmp = '%s.%d.tmp' % (out, os.getpid())
            subprocess.check_call(['g++', '-O2', '-std=c++17', '-shared', '-fPIC', '-DKB_HOST_EMU', '-Wno-unknown-pragmas',
                                   '-o', tmp, _SRC])
            os.replace(tmp, out)
        lib = ctypes.CDLL(out)
        lib.kb_emu_resample.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_longlong, ctypes.c_int, ctypes.c_int,
                                        ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int,
                                        ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_double, ctypes.c_int,
                                        ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int]
        _lib_handle = Checked(lib)
    return _lib_handle


def _fp(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def emu_resample(x, fmt, up, down, h32, gain=None, length=None, NT=64, n_cta=3, bulk=None):
    """Run the kernel body on the NumPy array `x` ((B, L, C) channels_last or (B, C, L), any strides, possibly a view
    into a larger buffer) with the library's choice of channel grouping and loader unless overridden."""
    if fmt == CL:
        B, L, C = x.shape
        sb, sl, sc = (s // 4 for s in x.strides)
    else:
        B, C, L = x.shape
        sb, sc, sl = (s // 4 for s in x.strides)
    base = x.base if x.base is not None else x
    numel = ((B - 1) * sb + (C - 1) * sc + (L - 1) * sl + 1) if x.size else 0
    assert numel <= base.size
    Lo = RR.output_length(L, up, down) if length is None else length
    y = np.full((B, Lo, C) if fmt == CL else (B, C, Lo), np.nan, dtype=np.float32)
    ys = np.array([y.strides[0], y.strides[2], y.strides[1]] if fmt == CL else [s for s in y.strides], np.int64) // 4
    xs = np.array([sb, sc, sl], np.int64)
    G = C if (1 < C <= 256 and abs(sc) < abs(sl)) else 1           # kb_resample_launch's choice
    can_bulk = int((G == 1 and sl == 1) or (G == C and sc == 1 and sl == C))
    h32 = np.ascontiguousarray(h32, np.float32)
    rc = _lib().kb_emu_resample(x.ctypes.data, _fp(xs), numel, B, C, L, _fp(y), _fp(ys), Lo, up, down, _fp(h32), h32.size,
                                float(up if gain is None else gain), G, NT, 256, n_cta,
                                can_bulk if bulk is None else int(bulk and can_bulk))
    assert rc == 0
    return y


def _ref(x, fmt, up, down, length=None):
    """Restatement on a (B, L, C) / (B, C, L) array, same layout out."""
    t = torch.from_numpy(np.ascontiguousarray(x, np.float64))
    if fmt == CL:
        return RR.resample(t.transpose(1, 2), up, down, length=length).transpose(1, 2).numpy()
    return RR.resample(t, up, down, length=length).numpy()


def _close(got, want, scale, tol=1e-5):
    assert got.shape == want.shape, (got.shape, want.shape)
    if got.size:
        err = float(np.abs(got - want).max())
        assert err <= tol * scale, (err, scale)


# ------------------------------------------------------------------------------ filter and restatement vs scipy
@pytest.mark.parametrize('orig,target', [p for p in itertools.permutations(RR.RATES, 2)])
def test_filter_matches_firwin(orig, target):
    sig = pytest.importorskip('scipy.signal')
    from kapre_b200.signal import resample_filter
    up, down = RR.up_down(orig, target)
    M = max(up, down)
    want = sig.firwin(20 * M + 1, 1.0 / M, window=('kaiser', 5.0))
    got = resample_filter(up, down)
    assert got.dtype == np.float32 and got.shape == want.shape
    np.testing.assert_allclose(got, want, rtol=1e-6, atol=1e-9 / M)
    np.testing.assert_array_equal(got, got[::-1])
    np.testing.assert_allclose(RR.taps(up, down), want, rtol=1e-12, atol=1e-15)


@pytest.mark.parametrize('orig,target', RR.COMMON_PAIRS + ((96000, 8000), (22050, 44100)))
@pytest.mark.parametrize('L', [1, 7, 301, 4000])
def test_restatement_matches_scipy(orig, target, L):
    sig = pytest.importorskip('scipy.signal')
    up, down = RR.up_down(orig, target)
    x = np.random.default_rng(L).standard_normal((2, L))
    want = sig.resample_poly(x, up, down, axis=-1)
    got = RR.resample(torch.from_numpy(x), up, down).numpy()
    assert got.shape == want.shape
    assert float(np.abs(got - want).max()) <= 1e-12 * float(np.abs(x).max())


# ------------------------------------------------------------------------------ the emulated kernel body
def _case_signal(rng, fmt, B, C, L):
    return rng.uniform(-1, 1, size=(B, L, C) if fmt == CL else (B, C, L)).astype(np.float32)


@pytest.mark.parametrize('orig,target', [(48000, 16000), (44100, 16000), (16000, 22050), (8000, 11025)])
@pytest.mark.parametrize('L', [0, 1, 37, 2900])
@pytest.mark.parametrize('C', [1, 2, 3])
@pytest.mark.parametrize('fmt', [CF, CL])
def test_emulated_body_matches_restatement(orig, target, L, C, fmt):
    up, down = RR.up_down(orig, target)
    x = _case_signal(np.random.default_rng(L * 7 + C), fmt, 2, C, L)
    from kapre_b200.signal import resample_filter
    got = emu_resample(x, fmt, up, down, resample_filter(up, down))
    _close(got, _ref(x, fmt, up, down), max(float(np.abs(x).max()) if x.size else 1.0, 1e-30))


@pytest.mark.parametrize('view', ['time_stride', 'channel_slice', 'batch_stride', 'misaligned'])
@pytest.mark.parametrize('fmt', [CF, CL])
def test_emulated_body_on_views(view, fmt):
    """Non-contiguous inputs: the cooperative loader (strided time axis, a slice of the channels) and the bulk copy
    of a span that does not start on a 16 B boundary."""
    up, down = RR.up_down(44100, 16000)
    rng = np.random.default_rng(5)
    full = _case_signal(rng, fmt, 3, 4, 3100)
    t_ax, c_ax = (1, 2) if fmt == CL else (2, 1)
    sl = [slice(None)] * 3
    if view == 'time_stride':
        sl[t_ax] = slice(None, None, 2)
    elif view == 'channel_slice':
        sl[c_ax] = slice(1, 3)
    elif view == 'batch_stride':
        sl[0] = slice(None, None, 2)
    else:
        sl[t_ax] = slice(3, 3001)
        sl[c_ax] = slice(0, 1)
    x = full[tuple(sl)]
    from kapre_b200.signal import resample_filter
    got = emu_resample(x, fmt, up, down, resample_filter(up, down), NT=128, n_cta=2)
    _close(got, _ref(x, fmt, up, down), float(np.abs(x).max()))


@pytest.mark.parametrize('orig,target', [(48000, 16000), (44100, 16000), (16000, 22050), (11025, 32000)])
@pytest.mark.parametrize('fmt', [CF, CL])
def test_emulated_adjoint_identity(orig, target, fmt):
    """<A x, g> = <x, A^T g> with A^T g = the body run with up and down exchanged (gain up), cropped to L samples."""
    up, down = RR.up_down(orig, target)
    rng = np.random.default_rng(11)
    L = 1500
    x = _case_signal(rng, fmt, 2, 2, L)
    from kapre_b200.signal import resample_filter
    h = resample_filter(up, down)
    y = emu_resample(x, fmt, up, down, h)
    g = rng.uniform(-1, 1, size=y.shape).astype(np.float32)
    gx = emu_resample(g, fmt, down, up, h, gain=up, length=L)
    lhs = float(np.dot(y.astype(np.float64).ravel(), g.astype(np.float64).ravel()))
    rhs = float(np.dot(x.astype(np.float64).ravel(), gx.astype(np.float64).ravel()))
    assert abs(lhs - rhs) <= 1e-5 * np.sqrt(float((y.astype(np.float64) ** 2).sum() * (g.astype(np.float64) ** 2).sum()))
    # and against the restatement's exact VJP
    xt = torch.from_numpy(np.ascontiguousarray(x, np.float64)).requires_grad_()
    yt = RR.resample(xt.transpose(1, 2) if fmt == CL else xt, up, down)
    gt = torch.from_numpy(np.ascontiguousarray(g, np.float64))
    (want,) = torch.autograd.grad(yt, xt, gt.transpose(1, 2) if fmt == CL else gt)
    _close(gx, want.numpy(), float(np.abs(want.numpy()).max()))


def test_table_row_stride_spreads_banks():
    """Rows are Kp floats apart with Kp a multiple of 4 and Kp / 4 odd (when there is more than one row), so that 8
    consecutive rows read as 16 B vectors land in 8 distinct bank groups."""
    lib = _lib()
    for orig, target in itertools.permutations(RR.RATES, 2):
        up, down = RR.up_down(orig, target)
        n_taps = 20 * max(up, down) + 1
        kp = lib.kb_emu_resample_kp(up, n_taps)
        assert kp % 4 == 0 and kp >= 2 * ((n_taps - 1) // 2 // up) + 2
        if up > 1:
            assert (kp // 4) % 2 == 1
            assert len({(r * kp // 4) % 8 for r in range(8)}) == 8


def test_kernel_register_and_spill_budget():
    """kb_resample_kernel runs 256 threads per CTA and relies on several CTAs per SM: at most 64 registers, no spills."""
    import shutil
    lib = os.path.join(_HERE, '..', 'kapre_b200', '_lib', 'libkapre_b200.so')
    if shutil.which('cuobjdump') is None or not os.path.exists(lib):
        pytest.skip('needs cuobjdump and the built library')
    out = subprocess.run(['cuobjdump', '-res-usage', lib], capture_output=True, text=True, check=True).stdout
    lines = out.splitlines()
    found = [(lines[i], lines[i + 1]) for i in range(len(lines) - 1) if 'kb_resample_kernel' in lines[i]]
    assert len(found) == 1, found
    import re
    m = re.search(r'REG:(\d+) STACK:(\d+)', found[0][1])
    assert m and int(m.group(1)) <= 64 and int(m.group(2)) == 0, found[0]


# ------------------------------------------------------------------------------ the layer
def test_layer_validation_and_config():
    from kapre_b200.signal import Resample
    import kapre
    assert kapre.signal.Resample is Resample
    for bad in (0, -16000, 16000.0, 1.5, True, '16000', None):
        with pytest.raises(ValueError):
            Resample(bad, 16000)
        with pytest.raises(ValueError):
            Resample(48000, bad)
    with pytest.raises(ValueError):
        Resample(48000, 16000, data_format='channels_middle')
    layer = Resample(44100, 16000, data_format='channels_first', name='rs')
    assert (layer.up, layer.down) == (160, 441)
    cfg = layer.get_config()
    assert cfg['orig_sample_rate'] == 44100 and cfg['target_sample_rate'] == 16000
    assert cfg['data_format'] == 'channels_first' and cfg['name'] == 'rs'
    again = Resample.from_config(cfg)
    assert again.get_config() == cfg and (again.up, again.down) == (160, 441)
    assert Resample(np.int64(16000), 16000).plan is None            # equal rates: no kernel at all
    import kapre_b200
    assert 'Resample' not in kapre_b200.__all__
