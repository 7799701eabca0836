"""Functional layer over the C ABI: torch tensors in, torch tensors out.

PyTorch is only the device-memory carrier and the stream provider here; every computation
is a launch of the kernels in ``csrc/`` through ``libkapre_b200.so``.  There is no fallback:
a missing library, a CPU-only process or a non-CUDA tensor raises.
"""
from __future__ import annotations

import collections
import ctypes
import math
import threading

import numpy as np
import torch

from . import _native as N
from .backend import _CH_FIRST_STR, _CH_LAST_STR

_lock = threading.Lock()


def _require_cuda():
    if not torch.cuda.is_available():
        raise N.KapreNativeError('kapre_b200 needs a CUDA device (H100, sm_90a); there is no CPU path')


def _stream_ptr():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr())


def to_device(x, dtype=None):
    """NumPy array / CPU tensor / CUDA tensor -> CUDA tensor on the current device.
    Returns (tensor, was_host)."""
    _require_cuda()
    was_host = True
    if isinstance(x, np.ndarray):
        t = torch.from_numpy(np.ascontiguousarray(x))
    elif isinstance(x, torch.Tensor):
        t = x
        was_host = not x.is_cuda
    else:
        t = torch.as_tensor(np.asarray(x))
    if dtype is not None and t.dtype != dtype:
        t = t.to(dtype)
    if not t.is_cuda:
        t = t.to(torch.device('cuda', torch.cuda.current_device()), non_blocking=True)
    return t, was_host


def to_host(t: torch.Tensor) -> np.ndarray:
    """CUDA tensor -> NumPy through pinned memory (torch's caching host allocator)."""
    host = torch.empty(t.shape, dtype=t.dtype, pin_memory=True)
    host.copy_(t, non_blocking=True)
    torch.cuda.current_stream().synchronize()
    return host.numpy()


_ws_cache = {}
_ws_retired = []   # outgrown workspaces stay alive: a captured CUDA graph may have their address baked in


def new_workspace(n_items: int, device) -> torch.Tensor:
    """Zeroed scratch of the decibel modes: 2 words per item (maximum + clamp-pass arrival counter)."""
    return torch.zeros(2 * max(int(n_items), 1), dtype=torch.int32, device=device)


def _workspace(n_items: int, device) -> torch.Tensor:
    """Per-(device, stream) zero-initialised scratch for the per-item dB maxima.  The kernels leave
    it zeroed (self-cleaning contract of the C ABI), so it is allocated and cleared only once.
    Objects that record launches into a CUDA graph own a private workspace instead (``workspace=``
    of ``stft_forward``), so nothing this cache does can invalidate a captured address."""
    n = max(int(n_items), 1)
    key = (device.index if device.index is not None else torch.cuda.current_device(),
           torch.cuda.current_stream(device).cuda_stream)
    ws = _ws_cache.get(key)
    if ws is None or ws.numel() < 2 * n:
        if ws is not None:
            _ws_retired.append(ws)
        ws = new_workspace(max(n, 1024), device)
        _ws_cache[key] = ws
    return ws


def _scratch(n: int, device) -> torch.Tensor:
    """Device scratch of the ``n`` bytes a ``kapre_*_workspace_bytes`` function returned; raises on its error code."""
    n = int(n)
    if n < 0:
        N.check(n)
    return torch.empty(max(n, 1), dtype=torch.uint8, device=device)


def _wants_grad(t) -> bool:
    """True when a CUDA tensor input should be recorded for autograd (see ``autograd.py``)."""
    return isinstance(t, torch.Tensor) and t.is_cuda and t.requires_grad and torch.is_grad_enabled()


def _device_of_first_arg(fn):
    """Run an op with the device of its first (tensor) argument current; host inputs keep the current device."""
    import functools

    @functools.wraps(fn)
    def wrapped(x, *a, **k):
        if isinstance(x, torch.Tensor) and x.is_cuda:
            with torch.cuda.device(x.device):
                return fn(x, *a, **k)
        return fn(x, *a, **k)
    return wrapped


def _on_device_of(t: torch.Tensor):
    """Context that makes the tensor's device current: plans, filterbanks, workspaces and the launch
    stream are all taken from the CURRENT device, which must be the one that owns the data."""
    if not t.is_cuda:
        raise N.KapreNativeError('kapre_b200 needs CUDA tensors (there is no CPU path)')
    return torch.cuda.device(t.device)


class _Handle:
    """Owns one C-ABI object and frees it with the matching destroy function."""

    def __init__(self, ptr, destroy):
        self.ptr = ptr
        self._destroy = destroy

    def __del__(self):
        try:
            if self.ptr:
                self._destroy(self.ptr)
                self.ptr = None
        except Exception:
            pass


class _PerDevice:
    """One C-ABI object per CUDA device, made on first use on that device.  Subclasses set ``_per_device = {}`` in
    their constructor, name the destroy function in ``_destroy`` and make the object in ``_create(lib, out)``, which
    returns the library's status and writes the new pointer through ``out``."""

    _destroy = None

    def handle(self):
        _require_cuda()
        dev = torch.cuda.current_device()
        with _lock:
            h = self._per_device.get(dev)
            if h is None:
                lib = N.lib()
                out = ctypes.c_void_p()
                N.check(self._create(lib, ctypes.byref(out)))
                h = _Handle(out, getattr(lib, self._destroy))
                self._per_device[dev] = h
        return h.ptr


class StftPlan(_PerDevice):
    """kapre_stft_plan per CUDA device for one (n_fft, win_length, hop, window)."""

    def __init__(self, n_fft, win_length, hop_length, window: np.ndarray):
        self.n_fft, self.win_length, self.hop_length = int(n_fft), int(win_length), int(hop_length)
        self.window = np.ascontiguousarray(window, dtype=np.float32)
        if self.window.shape != (self.win_length,):
            raise ValueError('window must have win_length=%d samples, got %s' % (self.win_length, self.window.shape))
        self._per_device = {}

    _destroy = 'kapre_stft_plan_destroy'

    def _create(self, lib, out):
        return lib.kapre_stft_plan_create(self.n_fft, self.win_length, self.hop_length,
                                          self.window.ctypes.data_as(ctypes.c_void_p), out)

    def num_frames(self, length, pad_begin, pad_end):
        lp = int(length) + ((self.n_fft - self.hop_length) if pad_begin else 0)
        if pad_end:
            return -(-lp // self.hop_length)
        return max(0, 1 + (lp - self.win_length) // self.hop_length)

    def supports_mode(self, mode):
        return bool(N.lib().kapre_stft_supports_mode(self.handle(), int(mode)))


class IstftPlan(_PerDevice):
    def __init__(self, n_fft, win_length, hop_length, dual_window: np.ndarray):
        self.n_fft, self.win_length, self.hop_length = int(n_fft), int(win_length), int(hop_length)
        self.dual = np.ascontiguousarray(dual_window, dtype=np.float32)
        self._per_device = {}

    _destroy = 'kapre_istft_plan_destroy'

    def _create(self, lib, out):
        return lib.kapre_istft_plan_create(self.n_fft, self.win_length, self.hop_length,
                                           self.dual.ctypes.data_as(ctypes.c_void_p), out)


class Filterbank(_PerDevice):
    """kapre_filterbank per CUDA device for one (n_freq, n_bands) matrix."""

    def __init__(self, matrix: np.ndarray):
        self.matrix = np.ascontiguousarray(matrix, dtype=np.float32)
        if self.matrix.ndim != 2:
            raise ValueError('filterbank must be (n_freq, n_bands)')
        self.n_freq, self.n_bands = self.matrix.shape
        self._per_device = {}
        self._transposed = None

    def transposed(self) -> 'Filterbank':
        """The (n_bands, n_freq) filterbank: applying it to the gradient of ``apply_filterbank``'s output
        gives the gradient of its input."""
        if self._transposed is None:
            self._transposed = Filterbank(self.matrix.T)
        return self._transposed

    _destroy = 'kapre_filterbank_destroy'

    def _create(self, lib, out):
        return lib.kapre_filterbank_create(self.matrix.ctypes.data_as(ctypes.c_void_p), self.n_freq, self.n_bands, out)


class FilterbankInversePlan(_PerDevice):
    """kapre_fb_inverse_plan per CUDA device for one (n_freq, n_bands) filterbank matrix: the row and column band
    lists of its transpose and the gradient step 1 / ||A||_2^2 of the NNLS iteration."""

    def __init__(self, matrix: np.ndarray):
        self.matrix = np.ascontiguousarray(matrix, dtype=np.float32)
        if self.matrix.ndim != 2:
            raise ValueError('filterbank must be (n_freq, n_bands)')
        self.n_freq, self.n_bands = self.matrix.shape
        self._per_device = {}

    _destroy = 'kapre_fb_inverse_plan_destroy'

    def _create(self, lib, out):
        return lib.kapre_fb_inverse_plan_create(self.matrix.ctypes.data_as(ctypes.c_void_p), self.n_freq, self.n_bands,
                                                out)


class ResamplePlan(_PerDevice):
    """kapre_resample_plan per CUDA device for one (up, down, filter)."""

    def __init__(self, up, down, taps: np.ndarray):
        self.up, self.down = int(up), int(down)
        self.taps = np.ascontiguousarray(taps, dtype=np.float32)
        if self.taps.ndim != 1:
            raise ValueError('resampling filter must be 1-D, got shape %s' % (self.taps.shape,))
        self._per_device = {}

    _destroy = 'kapre_resample_plan_destroy'

    def _create(self, lib, out):
        return lib.kapre_resample_plan_create(self.up, self.down, self.taps.ctypes.data_as(ctypes.c_void_p),
                                              self.taps.size, out)

    def output_length(self, length):
        """ceil(length * up / down), the output length of ``scipy.signal.resample_poly``."""
        return -(-int(length) * self.up // self.down)


def _wave_desc(t: torch.Tensor, data_format: str):
    """(B, L, C) channels_last or (B, C, L) channels_first -> kapre_wave_desc."""
    if t.dim() != 3:
        raise ValueError('waveform batch must be 3-D, got shape %s' % (tuple(t.shape),))
    if data_format == _CH_LAST_STR:
        B, L, C = t.shape
        sb, sl, sc = t.stride()
    else:
        B, C, L = t.shape
        sb, sc, sl = t.stride()
    return N.WaveDesc(B, C, L, sb, sc, sl), (B, C, L)


def _wave_alloc(B, C, L, data_format, device):
    """Contiguous (B, L, C) / (B, C, L) float32 waveform and its descriptor."""
    if data_format == _CH_LAST_STR:
        y = torch.empty((B, L, C), dtype=torch.float32, device=device)
        sb, sl, sc = y.stride()
    else:
        y = torch.empty((B, C, L), dtype=torch.float32, device=device)
        sb, sc, sl = y.stride()
    return y, N.WaveDesc(B, C, L, sb, sc, sl)


def _spec_alloc(B, C, T, K, data_format, dtype, device):
    if data_format == _CH_LAST_STR:
        out = torch.empty((B, T, K, C), dtype=dtype, device=device)
        sb, st, sk, sc = out.stride()
    else:
        out = torch.empty((B, C, T, K), dtype=dtype, device=device)
        sb, sc, st, sk = out.stride()
    return out, N.SpecDesc(sb, sc, st, sk)


def _spec_desc(t: torch.Tensor, data_format: str):
    if t.dim() != 4:
        raise ValueError('spectrogram batch must be 4-D, got shape %s' % (tuple(t.shape),))
    if data_format == _CH_LAST_STR:
        B, T, K, C = t.shape
        sb, st, sk, sc = t.stride()
    else:
        B, C, T, K = t.shape
        sb, sc, st, sk = t.stride()
    return N.SpecDesc(sb, sc, st, sk), (B, C, T, K)


def stft_forward(x: torch.Tensor, plan: StftPlan, input_data_format, output_data_format, pad_begin, pad_end,
                 mode=N.OUT_COMPLEX, fb: Filterbank = None, db=None, workspace: torch.Tensor = None):
    """One fused launch: waveform -> (complex STFT | magnitude | filterbank) [-> dB].
    ``db`` = (ref_value, amin, dynamic_range); ``workspace``: caller-owned decibel scratch (``new_workspace``)."""
    if not x.is_cuda:
        raise N.KapreNativeError('stft_forward needs a CUDA tensor')
    if _wants_grad(x):
        from . import autograd
        return autograd.stft_forward(x, plan, input_data_format, output_data_format, pad_begin, pad_end, mode, fb, db,
                                     workspace)
    with _on_device_of(x):
        return _stft_forward(x, plan, input_data_format, output_data_format, pad_begin, pad_end, mode, fb, db, workspace)


def _stft_forward(x, plan, input_data_format, output_data_format, pad_begin, pad_end, mode, fb, db, workspace):
    if x.dtype != torch.float32:
        x = x.float()
    if pad_begin and plan.hop_length > plan.n_fft:
        # kapre/time_frequency.py:169-172 pads by n_fft - hop_length; tf.pad rejects a negative amount
        raise ValueError('pad_begin needs hop_length <= n_fft: the padding is n_fft - hop_length = %d'
                         % (plan.n_fft - plan.hop_length))
    xd, (B, C, L) = _wave_desc(x, input_data_format)
    T = plan.num_frames(L, pad_begin, pad_end)
    fbmode = mode in (N.OUT_FB, N.OUT_FB_DB)
    K = fb.n_bands if fbmode else plan.n_fft // 2 + 1
    dtype = torch.complex64 if mode == N.OUT_COMPLEX else torch.float32
    c_out = 2 * C if mode == N.OUT_MAG_PHASE else C   # mag+phase: phases in channels [C, 2C)
    out, od = _spec_alloc(B, c_out, T, K, output_data_format, dtype, x.device)
    dbc, ws = None, None
    if mode in (N.OUT_MAG_DB, N.OUT_FB_DB) or (mode == N.OUT_MAG_PHASE and db is not None):
        dbc = N.DbCfg(float(db[0]), float(db[1]), float(db[2]))
        ws = workspace if workspace is not None else _workspace(B, x.device)
        if ws.device != x.device or ws.numel() < 2 * B:
            raise ValueError('decibel workspace must live on %s and hold 2 x %d words' % (x.device, B))
    if out.numel() == 0:
        return out
    try:
        N.check(N.lib().kapre_stft_forward(
            plan.handle(), _ptr(x), ctypes.byref(xd), int(bool(pad_begin)), int(bool(pad_end)), int(mode), _ptr(out),
            ctypes.byref(od), fb.handle() if fbmode else None, ctypes.byref(dbc) if dbc is not None else None,
            _ptr(ws) if ws is not None else None, _stream_ptr()))
    except N.KapreNativeError:
        if ws is not None and not torch.cuda.is_current_stream_capturing():
            ws.zero_()          # a failed call may have left maxima behind: restore the all-zero contract
        raise
    return out


@_device_of_first_arg
def istft(X: torch.Tensor, plan: IstftPlan, input_data_format, output_data_format):
    if not X.is_cuda:
        raise N.KapreNativeError('istft needs a CUDA tensor')
    if _wants_grad(X):
        from . import autograd
        return autograd.istft(X, plan, input_data_format, output_data_format)
    if X.dtype != torch.complex64:
        X = X.to(torch.complex64)
    sd, (B, C, T, F) = _spec_desc(X, input_data_format)
    if F != plan.n_fft // 2 + 1:
        raise ValueError('expected %d frequency bins for n_fft=%d, got %d' % (plan.n_fft // 2 + 1, plan.n_fft, F))
    out_len = (T - 1) * plan.hop_length + plan.win_length if T > 0 else 0
    y, yd = _wave_alloc(B, C, out_len, output_data_format, X.device)
    if y.numel() == 0:
        return y
    N.check(N.lib().kapre_istft_inverse(plan.handle(), _ptr(X), B, C, T, ctypes.byref(sd), _ptr(y),
                                        ctypes.byref(yd), _stream_ptr()))
    return y


@_device_of_first_arg
def apply_filterbank(x: torch.Tensor, fb: Filterbank, data_format):
    if not x.is_cuda:
        raise N.KapreNativeError('apply_filterbank needs a CUDA tensor')
    if _wants_grad(x):
        from . import autograd
        return autograd.apply_filterbank(x, fb, data_format)
    if x.dtype != torch.float32:
        x = x.float()
    xd, (B, C, T, F) = _spec_desc(x, data_format)
    if F != fb.n_freq:
        raise ValueError('filterbank expects %d frequency bins, input has %d' % (fb.n_freq, F))
    out, od = _spec_alloc(B, C, T, fb.n_bands, data_format, torch.float32, x.device)
    if out.numel() == 0:
        return out
    N.check(N.lib().kapre_apply_filterbank(fb.handle(), _ptr(x), B, C, T, ctypes.byref(xd), _ptr(out),
                                           ctypes.byref(od), _stream_ptr()))
    return out


@_device_of_first_arg
def magnitude(x: torch.Tensor):
    if not x.is_cuda:
        raise N.KapreNativeError('magnitude needs a CUDA tensor')
    if not x.is_complex():
        return x.abs()  # tf.abs of a real tensor: plain |x| (not on the hot path)
    if _wants_grad(x):
        from . import autograd
        return autograd.magnitude(x)
    x = x.to(torch.complex64).contiguous()
    out = torch.empty(x.shape, dtype=torch.float32, device=x.device)
    if out.numel():
        N.check(N.lib().kapre_magnitude(_ptr(x), _ptr(out), x.numel(), _stream_ptr()))
    return out


@_device_of_first_arg
def phase(x: torch.Tensor):
    if not x.is_cuda:
        raise N.KapreNativeError('phase needs a CUDA tensor')
    if _wants_grad(x):
        from . import autograd
        return autograd.phase(x)
    x = x.to(torch.complex64).contiguous()
    out = torch.empty(x.shape, dtype=torch.float32, device=x.device)
    if out.numel():
        N.check(N.lib().kapre_phase(_ptr(x), _ptr(out), x.numel(), _stream_ptr()))
    return out


@_device_of_first_arg
def magnitude_to_decibel(x, ref_value=1.0, amin=1e-5, dynamic_range=80.0):
    if _wants_grad(x):
        from . import autograd
        return autograd.magnitude_to_decibel(x, ref_value, amin, dynamic_range)
    t, was_host = to_device(x, torch.float32)
    t = t.contiguous()
    out = torch.empty_like(t)
    if t.numel():
        if t.dim() > 1:
            n_items, item = t.shape[0], t.numel() // t.shape[0]
        else:
            n_items, item = 1, t.numel()
        ws = _workspace(n_items, t.device)
        dbc = N.DbCfg(float(ref_value), float(amin), float(dynamic_range))
        N.check(N.lib().kapre_magnitude_to_decibel(_ptr(t), _ptr(out), n_items, item, ctypes.byref(dbc), _ptr(ws),
                                                   _stream_ptr()))
    return to_host(out) if was_host and isinstance(x, np.ndarray) else out


# ------------------------------------------------------------------------------- backward passes
def _raw(t: torch.Tensor) -> torch.Tensor:
    """Materialise lazy conjugate / negative views: the kernels read the tensor's memory as it is."""
    return t.resolve_conj().resolve_neg()


@_device_of_first_arg
def stft_backward(g: torch.Tensor, plan: StftPlan, input_data_format, output_data_format, pad_begin, pad_end, length):
    """Gradient of ``stft_forward(..., OUT_COMPLEX)`` with respect to its waveform of ``length`` samples, given the
    gradient ``g`` of the complex spectrum (any strides)."""
    g = _raw(g.to(torch.complex64))
    gd, (B, C, T, F) = _spec_desc(g, output_data_format)
    L = int(length)
    gx, xd = _wave_alloc(B, C, L, input_data_format, g.device)
    if gx.numel() == 0:
        return gx
    lib = N.lib()
    nbytes = int(lib.kapre_stft_backward_workspace_bytes(plan.handle(), B, C, L, int(bool(pad_begin)), int(bool(pad_end))))
    ws = _scratch(nbytes, g.device) if nbytes else None
    N.check(lib.kapre_stft_backward(plan.handle(), _ptr(g), ctypes.byref(gd), B, C, T, int(bool(pad_begin)),
                                    int(bool(pad_end)), _ptr(gx), ctypes.byref(xd), _ptr(ws) if ws is not None else None,
                                    _stream_ptr()))
    return gx


@_device_of_first_arg
def istft_backward(gy: torch.Tensor, plan: IstftPlan, input_data_format, output_data_format, frames):
    """Gradient of ``istft`` with respect to its complex spectrum of ``frames`` frames, given the gradient ``gy`` of
    the waveform (any strides)."""
    gy = _raw(gy.to(torch.float32))
    yd, (B, C, _) = _wave_desc(gy, output_data_format)
    gX, sd = _spec_alloc(B, C, int(frames), plan.n_fft // 2 + 1, input_data_format, torch.complex64, gy.device)
    if gX.numel() == 0:
        return gX
    N.check(N.lib().kapre_istft_backward(plan.handle(), _ptr(gy), ctypes.byref(yd), B, C, int(frames), _ptr(gX),
                                         ctypes.byref(sd), _stream_ptr()))
    return gX


@_device_of_first_arg
def magnitude_backward(X: torch.Tensor, g: torch.Tensor):
    """Gradient of ``magnitude`` with respect to the complex64 tensor ``X``: ``g X / |X|``, 0 where ``|X| = 0``."""
    X = _raw(X.to(torch.complex64)).contiguous()
    g = _raw(g.to(torch.float32)).contiguous()
    if g.shape != X.shape:
        raise ValueError('gradient shape %s does not match %s' % (tuple(g.shape), tuple(X.shape)))
    gX = torch.empty_like(X)
    if X.numel():
        N.check(N.lib().kapre_magnitude_backward(_ptr(X), _ptr(g), _ptr(gX), X.numel(), _stream_ptr()))
    return gX


@_device_of_first_arg
def magnitude_to_decibel_backward(x: torch.Tensor, g: torch.Tensor, ref_value=1.0, amin=1e-5, dynamic_range=80.0):
    """Gradient of ``magnitude_to_decibel`` with respect to its input ``x`` (items along axis 0, as the forward),
    with TensorFlow's tie rules."""
    x = x.to(torch.float32).contiguous()
    g = _raw(g.to(torch.float32)).contiguous()
    if g.shape != x.shape:
        raise ValueError('gradient shape %s does not match %s' % (tuple(g.shape), tuple(x.shape)))
    gx = torch.empty_like(x)
    if x.numel():
        n_items, item = (x.shape[0], x.numel() // x.shape[0]) if x.dim() > 1 else (1, x.numel())
        ws = torch.zeros(3 * max(n_items, 1), dtype=torch.int32, device=x.device)
        dbc = N.DbCfg(float(ref_value), float(amin), float(dynamic_range))
        N.check(N.lib().kapre_magnitude_to_decibel_backward(_ptr(x), _ptr(g), _ptr(gx), n_items, item,
                                                            ctypes.byref(dbc), _ptr(ws), _stream_ptr()))
    return gx


@_device_of_first_arg
def phase_backward(X: torch.Tensor, g: torch.Tensor):
    """Gradient of ``phase`` with respect to the complex64 tensor ``X``: ``g i X / |X|^2``, 0 where ``|X| = 0``."""
    X = _raw(X.to(torch.complex64)).contiguous()
    g = _raw(g.to(torch.float32)).contiguous()
    if g.shape != X.shape:
        raise ValueError('gradient shape %s does not match %s' % (tuple(g.shape), tuple(X.shape)))
    gX = torch.empty_like(X)
    if X.numel():
        N.check(N.lib().kapre_phase_backward(_ptr(X), _ptr(g), _ptr(gX), X.numel(), _stream_ptr()))
    return gX


@_device_of_first_arg
def mag_phase_backward(X: torch.Tensor, g_mag, g_phase, data_format):
    """Gradient of the magnitude + phase pair of the complex spectrum ``X`` (``data_format`` layout, any strides)
    with respect to ``X``: ``X / |X| (g_mag + i g_phase / |X|)``.  ``g_mag`` / ``g_phase``: float tensors of X's
    shape (any strides, e.g. the two halves of the 2C-channel gradient), or None for zero."""
    X = _raw(X.to(torch.complex64))
    xd, (B, C, T, F) = _spec_desc(X, data_format)
    gX, od = _spec_alloc(B, C, T, F, data_format, torch.complex64, X.device)
    descs = []
    for g in (g_mag, g_phase):
        if g is None:
            descs.append((None, None))
            continue
        g = _raw(g.to(torch.float32))
        if g.shape != X.shape:
            raise ValueError('gradient shape %s does not match %s' % (tuple(g.shape), tuple(X.shape)))
        descs.append((g, _spec_desc(g, data_format)[0]))
    if gX.numel() == 0:
        return gX
    (gm, gmd), (gp, gpd) = descs
    N.check(N.lib().kapre_mag_phase_backward(
        _ptr(X), ctypes.byref(xd), _ptr(gm) if gm is not None else None, ctypes.byref(gmd) if gmd is not None else None,
        _ptr(gp) if gp is not None else None, ctypes.byref(gpd) if gpd is not None else None, _ptr(gX),
        ctypes.byref(od), B, C, T, F, _stream_ptr()))
    return gX


# ------------------------------------------------------------------------------- adjacent layers
_PAD_MODES = {'symmetric': 0, 'reflect': 1, 'constant': 2}


@_device_of_first_arg
def delta(x: torch.Tensor, win_length: int, mode: str, data_format: str):
    """kapre.Delta along the time axis of (b, t, f, ch) / (b, ch, t, f)."""
    if not x.is_cuda:
        raise N.KapreNativeError('delta needs a CUDA tensor')
    if _wants_grad(x):
        from . import autograd
        return autograd.delta(x, win_length, mode, data_format)
    x = x.float().contiguous()
    outer, frames, inner = _delta_view(x, data_format)
    out = torch.empty_like(x)
    if x.numel():
        N.check(N.lib().kapre_delta(_ptr(x), _ptr(out), outer, frames, inner, int(win_length),
                                    _PAD_MODES[mode.lower()], _stream_ptr()))
    return out


def _delta_view(x, data_format):
    """(outer, frames, inner) of a contiguous 4-D batch whose time axis is 1 (channels_last) or 2."""
    if x.dim() != 4:
        raise ValueError('Delta expects a 4-D batch, got shape %s' % (tuple(x.shape),))
    if data_format == _CH_LAST_STR:
        return x.shape[0], x.shape[1], x.shape[2] * x.shape[3]
    return x.shape[0] * x.shape[1], x.shape[2], x.shape[3]


@_device_of_first_arg
def delta_backward(g: torch.Tensor, win_length: int, mode: str, data_format: str):
    """Gradient of ``delta`` with respect to its input, given the gradient ``g`` of its output."""
    g = _raw(g.to(torch.float32)).contiguous()
    outer, frames, inner = _delta_view(g, data_format)
    gx = torch.empty_like(g)
    if g.numel():
        N.check(N.lib().kapre_delta_backward(_ptr(g), _ptr(gx), outer, frames, inner, int(win_length),
                                             _PAD_MODES[mode.lower()], _stream_ptr()))
    return gx


@_device_of_first_arg
def concat_frequency_map(x: torch.Tensor, data_format: str):
    """kapre.ConcatenateFrequencyMap: (b, t, f, ch) -> (b, t, f, ch + 1) or (b, ch, t, f) -> (b, ch + 1, t, f)."""
    if not x.is_cuda:
        raise N.KapreNativeError('concat_frequency_map needs a CUDA tensor')
    if _wants_grad(x):
        from . import autograd
        return autograd.concat_frequency_map(x, data_format)
    x = x.float().contiguous()
    if x.dim() != 4:
        raise ValueError('ConcatenateFrequencyMap expects a 4-D batch, got shape %s' % (tuple(x.shape),))
    cl = data_format == _CH_LAST_STR
    if cl:
        B, T, F, C = x.shape
        out = torch.empty((B, T, F, C + 1), dtype=torch.float32, device=x.device)
    else:
        B, C, T, F = x.shape
        out = torch.empty((B, C + 1, T, F), dtype=torch.float32, device=x.device)
    if out.numel():
        N.check(N.lib().kapre_concat_frequency_map(_ptr(x), _ptr(out), B, C, T, F, int(cl), _stream_ptr()))
    return out


@_device_of_first_arg
def spec_augment(x: torch.Tensor, time_masks: np.ndarray, freq_masks: np.ndarray, mask_value: float, data_format: str):
    """kapre.SpecAugment with given masks: x (b, t, f, 1) or (b, 1, t, f); masks (b, n, 2) int32 (start, width)."""
    if not x.is_cuda:
        raise N.KapreNativeError('spec_augment needs a CUDA tensor')
    B, _, _ = _spec_augment_dims(x, data_format)
    if x.numel() == 0:
        return torch.empty_like(x, dtype=torch.float32)
    tm = torch.as_tensor(np.ascontiguousarray(time_masks, dtype=np.int32).reshape(B, -1, 2)).to(x.device)
    fm = torch.as_tensor(np.ascontiguousarray(freq_masks, dtype=np.int32).reshape(B, -1, 2)).to(x.device)
    if _wants_grad(x):
        from . import autograd
        return autograd.spec_augment(x, tm, fm, mask_value, data_format)
    return spec_augment_masked(x, tm, fm, mask_value, data_format)


def _spec_augment_dims(x, data_format):
    if data_format == _CH_LAST_STR:
        B, T, F, C = x.shape
    else:
        B, C, T, F = x.shape
    if C != 1:
        raise RuntimeError('SpecAugment does not support spectrograms with depth greater than 1')
    return B, T, F


@_device_of_first_arg
def spec_augment_masked(x: torch.Tensor, tm: torch.Tensor, fm: torch.Tensor, mask_value: float, data_format: str):
    """The masking launch of ``spec_augment`` with device masks ``tm`` / ``fm`` ((b, n, 2) int32).  Run on a gradient
    with ``mask_value`` 0 and the forward's masks, it is the layer's backward pass."""
    x = _raw(x.float()).contiguous()
    B, T, F = _spec_augment_dims(x, data_format)
    out = torch.empty_like(x)
    if x.numel() == 0:
        return out
    N.check(N.lib().kapre_spec_augment(_ptr(x), _ptr(out), B, T, F, _ptr(tm) if tm.numel() else None, tm.shape[1],
                                       _ptr(fm) if fm.numel() else None, fm.shape[1], ctypes.c_float(mask_value), _stream_ptr()))
    return out


def _frames_for(length, frame_length, hop, pad_end):
    return -(-length // hop) if pad_end else max(0, 1 + (length - frame_length) // hop)


@_device_of_first_arg
def frame(x: torch.Tensor, frame_length, hop_length, pad_end, pad_value, data_format):
    """kapre.Frame: (b, t, ch) -> (b, frames, frame_length, ch) or (b, ch, t) -> (b, ch, frames, frame_length)."""
    if not x.is_cuda:
        raise N.KapreNativeError('frame needs a CUDA tensor')
    if _wants_grad(x):
        from . import autograd
        return autograd.frame(x, frame_length, hop_length, pad_end, pad_value, data_format)
    x = x.float()
    xd, (B, C, L) = _wave_desc(x, data_format)
    T = _frames_for(L, frame_length, hop_length, pad_end)
    out, od = _spec_alloc(B, C, T, frame_length, data_format, torch.float32, x.device)
    if out.numel():
        N.check(N.lib().kapre_frame(_ptr(x), ctypes.byref(xd), int(frame_length), int(hop_length), int(bool(pad_end)),
                                    ctypes.c_float(pad_value), _ptr(out), ctypes.byref(od), _stream_ptr()))
    return out


@_device_of_first_arg
def energy(x: torch.Tensor, frame_length, hop_length, pad_end, pad_value, scale, data_format):
    """kapre.Energy: scale * sum of squares per frame; (b, t, ch) -> (b, frames, ch), (b, ch, t) -> (b, ch, frames)."""
    if not x.is_cuda:
        raise N.KapreNativeError('energy needs a CUDA tensor')
    if _wants_grad(x):
        from . import autograd
        return autograd.energy(x, frame_length, hop_length, pad_end, pad_value, scale, data_format)
    x = x.float()
    xd, (B, C, L) = _wave_desc(x, data_format)
    T = _frames_for(L, frame_length, hop_length, pad_end)
    out, od = _wave_alloc(B, C, T, data_format, x.device)     # one value per frame: a waveform of T samples
    if out.numel():
        N.check(N.lib().kapre_energy(_ptr(x), ctypes.byref(xd), int(frame_length), int(hop_length), int(bool(pad_end)),
                                     ctypes.c_float(pad_value), ctypes.c_float(scale), _ptr(out), ctypes.byref(od),
                                     _stream_ptr()))
    return out


@_device_of_first_arg
def frame_backward(g: torch.Tensor, frame_length, hop_length, data_format, length):
    """Gradient of ``frame`` with respect to its waveform of ``length`` samples, given the gradient ``g`` of the
    frames (any strides)."""
    g = _raw(g.to(torch.float32))
    gd, (B, C, T, _) = _spec_desc(g, data_format)
    gx, xd = _wave_alloc(B, C, int(length), data_format, g.device)
    if gx.numel():
        N.check(N.lib().kapre_frame_backward(_ptr(g), ctypes.byref(gd), T, int(frame_length), int(hop_length), _ptr(gx),
                                             ctypes.byref(xd), _stream_ptr()))
    return gx


@_device_of_first_arg
def energy_backward(x: torch.Tensor, g: torch.Tensor, frame_length, hop_length, scale, data_format):
    """Gradient of ``energy`` with respect to its float32 input ``x``, given the gradient ``g`` of the per-frame
    energies (any strides)."""
    xd, (B, C, L) = _wave_desc(x, data_format)
    g = _raw(g.to(torch.float32))
    if g.dim() != 3:
        raise ValueError('energy gradient must be 3-D, got shape %s' % (tuple(g.shape),))
    if data_format == _CH_LAST_STR:
        sb, st, sc = g.stride()
        T = g.shape[1]
    else:
        sb, sc, st = g.stride()
        T = g.shape[2]
    gd = N.WaveDesc(B, C, T, sb, sc, st)
    gx, od = _wave_alloc(B, C, L, data_format, x.device)
    if gx.numel():
        N.check(N.lib().kapre_energy_backward(_ptr(x), ctypes.byref(xd), _ptr(g), ctypes.byref(gd), int(frame_length),
                                              int(hop_length), ctypes.c_float(scale), _ptr(gx), ctypes.byref(od),
                                              _stream_ptr()))
    return gx


@_device_of_first_arg
def resample(x: torch.Tensor, plan: ResamplePlan, data_format):
    """Polyphase resampling along the time axis of (b, t, ch) / (b, ch, t): ``scipy.signal.resample_poly(x, up, down)``."""
    if not x.is_cuda:
        raise N.KapreNativeError('resample needs a CUDA tensor')
    if _wants_grad(x):
        from . import autograd
        return autograd.resample(x, plan, data_format)
    if x.dtype != torch.float32:
        x = x.float()
    xd, (B, C, L) = _wave_desc(x, data_format)
    y, yd = _wave_alloc(B, C, plan.output_length(L), data_format, x.device)
    if y.numel():
        N.check(N.lib().kapre_resample(plan.handle(), _ptr(x), ctypes.byref(xd), _ptr(y), ctypes.byref(yd), _stream_ptr()))
    return y


@_device_of_first_arg
def resample_backward(g: torch.Tensor, plan: ResamplePlan, data_format, length):
    """Gradient of ``resample`` with respect to its input of ``length`` samples, given the gradient ``g`` of its
    output (any strides)."""
    g = _raw(g.to(torch.float32))
    gd, (B, C, _) = _wave_desc(g, data_format)
    gx, xd = _wave_alloc(B, C, int(length), data_format, g.device)
    if gx.numel():
        N.check(N.lib().kapre_resample_backward(plan.handle(), _ptr(g), ctypes.byref(gd), _ptr(gx), ctypes.byref(xd),
                                                _stream_ptr()))
    return gx


class SincPlan(_PerDevice):
    """kapre_sinc_plan per CUDA device: the table of the band-limited interpolation filter.  Nothing in it depends on
    a ratio, so the module holds one instance (``_sinc_plan``) that every ``Speed`` and ``PitchShift`` layer shares."""

    def __init__(self):
        self._per_device = {}

    _destroy = 'kapre_sinc_plan_destroy'

    def _create(self, lib, out):
        return lib.kapre_sinc_plan_create(out)


_sinc_plan = SincPlan()
SINC_RATIO_MIN, SINC_RATIO_MAX = 0.25, 4.0


def _check_ratio(ratio, name='ratio'):
    if isinstance(ratio, (bool, np.bool_)) or not isinstance(ratio, (int, float, np.integer, np.floating)) \
            or not SINC_RATIO_MIN <= float(ratio) <= SINC_RATIO_MAX:
        raise ValueError('%s must be a number in [%g, %g], got: %r' % (name, SINC_RATIO_MIN, SINC_RATIO_MAX, ratio))
    return float(ratio)


def _check_offset(offset):
    if isinstance(offset, (bool, np.bool_)) or not isinstance(offset, (int, float, np.integer, np.floating)) \
            or not math.isfinite(float(offset)):
        raise ValueError('offset must be a finite number, got: %r' % (offset,))
    return float(offset)


@_device_of_first_arg
def sinc_resample(x: torch.Tensor, ratio, length, offset=0.0, data_format=_CH_LAST_STR):
    """Band-limited interpolation along the time axis of (b, t, ch) / (b, ch, t) by any ``ratio`` (output rate /
    input rate) in [0.25, 4]: output sample ``m`` of ``length`` is the input at position ``offset + m / ratio``,
    low-passed to the lower of the two Nyquist rates (see ``include/kapre_b200.h``).  One launch, no per-ratio state."""
    if not x.is_cuda:
        raise N.KapreNativeError('sinc_resample needs a CUDA tensor')
    ratio, offset = _check_ratio(ratio), _check_offset(offset)
    if _wants_grad(x):
        from . import autograd
        return autograd.sinc_resample(x, ratio, length, offset, data_format)
    if x.dtype != torch.float32:
        x = x.float()
    xd, (B, C, L) = _wave_desc(x, data_format)
    y, yd = _wave_alloc(B, C, int(length), data_format, x.device)
    if y.numel():
        N.check(N.lib().kapre_sinc_resample(_sinc_plan.handle(), _ptr(x), ctypes.byref(xd), _ptr(y), ctypes.byref(yd),
                                            ratio, offset, _stream_ptr()))
    return y


@_device_of_first_arg
def sinc_resample_backward(g: torch.Tensor, ratio, offset, data_format, length):
    """Gradient of ``sinc_resample`` with respect to its input of ``length`` samples, given the gradient ``g`` of its
    output (any strides)."""
    g = _raw(g.to(torch.float32))
    gd, (B, C, _) = _wave_desc(g, data_format)
    gx, xd = _wave_alloc(B, C, int(length), data_format, g.device)
    if gx.numel():
        N.check(N.lib().kapre_sinc_resample_backward(_sinc_plan.handle(), _ptr(g), ctypes.byref(gd), _ptr(gx),
                                                     ctypes.byref(xd), _check_ratio(ratio), _check_offset(offset),
                                                     _stream_ptr()))
    return gx


class ConvolvePlan(_PerDevice):
    """kapre_convolve_plan per CUDA device for one block size: the STFT (n_fft 2B, window ones(B), hop B) and the
    inverse (dual window ones(2B)) of the partitioned convolution.  One instance per block size (``convolve_plan``)."""

    def __init__(self, block):
        self.block = int(block)
        self._per_device = {}

    _destroy = 'kapre_convolve_plan_destroy'

    def _create(self, lib, out):
        return lib.kapre_convolve_plan_create(self.block, out)


_conv_plans = {}
CONVOLVE_MODES = ('full', 'same', 'valid')


def convolve_block_size(ir_length):
    """The partition's block size B for a filter of ``ir_length`` taps (``kapre_convolve_block_size``)."""
    b = int(N.lib().kapre_convolve_block_size(int(ir_length)))
    if b < 0:
        N.check(b)
    return b


def convolve_plan(block):
    with _lock:
        plan = _conv_plans.get(block)
        if plan is None:
            plan = _conv_plans[block] = ConvolvePlan(block)
    return plan


def convolve_span(length, ir_length, mode):
    """(start, length) of torchaudio.functional.fftconvolve's ``mode`` inside the full convolution."""
    full = length + ir_length - 1
    if mode == 'full':
        return 0, full
    target = length if mode == 'same' else max(length, ir_length) - min(length, ir_length) + 1
    return (full - target) // 2, target


def _time_axis(data_format):
    return 2 if data_format == _CH_FIRST_STR else 1


def _spec_contiguous_desc(H, broadcast_b=False, broadcast_c=False):
    """Descriptor of a contiguous (B, C, frames, F) complex tensor; a broadcast dimension gets stride 0."""
    sb, sc, st, sf = H.stride()
    return N.SpecDesc(0 if broadcast_b else sb, 0 if broadcast_c else sc, st, sf)


def _conv_check(x, h, data_format):
    """Shapes of ``convolve``'s operands: x (B, L, C) / (B, C, L); h (K,) or 3-D in x's format with batch in {1, B}
    and channels in {1, C}.  Returns (h as a 3-D tensor, (B, C, L), (Bh, Ch, K))."""
    if x.dim() != 3:
        raise ValueError('convolve expects a 3-D signal batch, got shape %s' % (tuple(x.shape),))
    B, C, L = (x.shape[0], x.shape[2], x.shape[1]) if data_format == _CH_LAST_STR else tuple(x.shape)
    if h.dim() == 1:
        h = h.view(1, 1, -1) if data_format == _CH_FIRST_STR else h.view(1, -1, 1)
    elif h.dim() != 3:
        raise ValueError('the filter must be 1-D or 3-D, got shape %s' % (tuple(h.shape),))
    Bh, Ch, K = (h.shape[0], h.shape[2], h.shape[1]) if data_format == _CH_LAST_STR else tuple(h.shape)
    if Bh not in (1, B) or Ch not in (1, C):
        raise ValueError('filter batch %d and channels %d must be 1 or the signal\'s (%d, %d)' % (Bh, Ch, B, C))
    if L < 1 or K < 1:
        raise ValueError('signal and filter need at least one sample, got %d and %d' % (L, K))
    return h, (B, C, L), (Bh, Ch, K)


def convolve_ir_spectrum(h, plan: ConvolvePlan, data_format):
    """The block spectra H (Bh, Ch, P, B + 1) complex64 of a 3-D filter tensor in ``data_format`` (one launch)."""
    if h.dtype != torch.float32:
        h = h.float()
    hd, (Bh, Ch, K) = _wave_desc(h, data_format)
    P = -(-K // plan.block)
    H = torch.empty((Bh, Ch, P, plan.block + 1), dtype=torch.complex64, device=h.device)
    if H.numel():
        N.check(N.lib().kapre_convolve_ir_spectrum(plan.handle(), _ptr(h), ctypes.byref(hd), _ptr(H),
                                                   ctypes.byref(N.SpecDesc(*H.stride())), _stream_ptr()))
    return H


def _conv_workspace_bytes(plan, B, C, L, P, backward=False):
    fn = N.lib().kapre_convolve_backward_workspace_bytes if backward else N.lib().kapre_convolve_workspace_bytes
    n = int(fn(plan.handle(), B, C, L, P))
    if n < 0:
        N.check(n)
    return n


def convolve_full(x, H, plan: ConvolvePlan, data_format):
    """x * h from the filter's block spectra H (``convolve_ir_spectrum``; batch and channels 1 broadcast): the
    untrimmed (T + 1) B samples of ``kapre_convolve`` and the workspace, which begins with the signal spectra X."""
    if x.dtype != torch.float32:
        x = x.float()
    xd, (B, C, L) = _wave_desc(x, data_format)
    P, blk = H.shape[2], plan.block
    nbytes = _conv_workspace_bytes(plan, B, C, L, P)
    T = -(-L // blk) + P - 1
    y, yd = _wave_alloc(B, C, (T + 1) * blk, data_format, x.device)
    ws = _scratch(nbytes, x.device)
    if y.numel():
        Hd = _spec_contiguous_desc(H, H.shape[0] == 1, H.shape[1] == 1)
        N.check(N.lib().kapre_convolve(plan.handle(), _ptr(x), ctypes.byref(xd), _ptr(H), ctypes.byref(Hd), P, _ptr(y),
                                       ctypes.byref(yd), _ptr(ws), _stream_ptr()))
    return y, ws


def convolve_backward(g_full, H, X, plan: ConvolvePlan, data_format, length, want_x, want_h):
    """Gradients of ``convolve_full`` given the gradient of its untrimmed output: (gx or None, per-(item, channel) gH
    (B, C, P, B + 1) or None).  ``X``: the signal spectra ``convolve_full`` left in its workspace (for gH)."""
    g_full = _raw(g_full.to(torch.float32))
    gd, (B, C, _) = _wave_desc(g_full, data_format)
    P, blk = H.shape[2], plan.block
    gx, xd = _wave_alloc(B, C, int(length), data_format, g_full.device)
    gH = torch.empty((B, C, P, blk + 1), dtype=torch.complex64, device=g_full.device) if want_h else None
    ws = _scratch(_conv_workspace_bytes(plan, B, C, int(length), P, backward=True), g_full.device)
    Hd = _spec_contiguous_desc(H, H.shape[0] == 1, H.shape[1] == 1)
    Xd = N.SpecDesc(*X.stride()) if want_h else None
    gHd = N.SpecDesc(*gH.stride()) if want_h else None
    N.check(N.lib().kapre_convolve_backward(
        plan.handle(), _ptr(g_full), ctypes.byref(gd), _ptr(H), ctypes.byref(Hd),
        _ptr(X) if want_h else None, ctypes.byref(Xd) if want_h else None, P,
        _ptr(gx) if want_x else None, ctypes.byref(xd), _ptr(gH) if want_h else None,
        ctypes.byref(gHd) if want_h else None, _ptr(ws), _stream_ptr()))
    return (gx if want_x else None), gH


def convolve_ir_spectrum_backward(gH, plan: ConvolvePlan, ir_length):
    """Gradient of ``convolve_ir_spectrum`` given gH (Bh, Ch, P, B + 1): a (Bh, Ch, K) channels_first filter gradient.
    It is computed for the P B samples the blocks cover (no scratch needed) and cropped to K."""
    gH = _raw(gH).contiguous()
    Bh, Ch, P, _ = gH.shape
    gh, hd = _wave_alloc(Bh, Ch, P * plan.block, _CH_FIRST_STR, gH.device)
    N.check(N.lib().kapre_convolve_ir_spectrum_backward(plan.handle(), _ptr(gH), ctypes.byref(N.SpecDesc(*gH.stride())),
                                                        P, _ptr(gh), ctypes.byref(hd), None, _stream_ptr()))
    return gh[:, :, :int(ir_length)]


def _crop(y, start, length, data_format):
    return y.narrow(_time_axis(data_format), start, length)


@_device_of_first_arg
def convolve(x: torch.Tensor, h: torch.Tensor, mode='full', data_format=_CH_LAST_STR):
    """``torchaudio.functional.fftconvolve`` along the time axis of x (B, L, C) / (B, C, L) with a filter h: (K,)
    shared by every item and channel, or 3-D in x's format with batch in {1, B} and channels in {1, C} (1
    broadcasts).  ``mode``: 'full' (L + K - 1 samples), 'same' (L) or 'valid' (max(L, K) - min(L, K) + 1); the
    result may be a view of the untrimmed output.  Four launches: the filter's spectra, then ``kapre_convolve``'s
    three.  Differentiable with respect to x and h."""
    if not (isinstance(x, torch.Tensor) and x.is_cuda and isinstance(h, torch.Tensor) and h.is_cuda):
        raise N.KapreNativeError('convolve needs CUDA tensors')
    if x.device != h.device:
        raise ValueError('signal on %s, filter on %s' % (x.device, h.device))
    if mode not in CONVOLVE_MODES:
        raise ValueError('mode must be one of %s, got: %r' % (CONVOLVE_MODES, mode))
    h3, (B, C, L), (Bh, Ch, K) = _conv_check(x, h, data_format)
    plan = convolve_plan(convolve_block_size(K))
    _conv_workspace_bytes(plan, B, C, L, -(-K // plan.block))      # size checks before anything is launched
    if _wants_grad(x) or _wants_grad(h):
        from . import autograd
        return autograd.convolve(x, h, h3, plan, mode, data_format)
    start, n = convolve_span(L, K, mode)
    y, _ = convolve_full(x, convolve_ir_spectrum(h3, plan, data_format), plan, data_format)
    return _crop(y, start, n, data_format)


@_device_of_first_arg
def convolve_spectrum(x: torch.Tensor, H: torch.Tensor, plan: ConvolvePlan, start, length, data_format=_CH_LAST_STR):
    """``kapre_convolve`` with given filter spectra H (a constant: the gradient reaches x only), cropped to
    [start, start + length) of the untrimmed output."""
    if not x.is_cuda:
        raise N.KapreNativeError('convolve needs a CUDA tensor')
    if _wants_grad(x):
        from . import autograd
        return autograd.convolve_spectrum(x, H, plan, start, length, data_format)
    y, _ = convolve_full(x, H, plan, data_format)
    return _crop(y, start, length, data_format)


RIR_RECORD = 14                 # float64 per item: room[3], source[3], beta[6], max_order (-1: none), start
RIR_MAX_IMAGES = 1 << 24        # kapre_rir_ism's cap on a response's image bound (KB_RIR_MAX_IMAGES)
_rir_captured = []              # pinned records of captures made without a holder: a graph may replay them at any time


def rir_ism(records, mics, output_length, filter_length, sample_rate, sound_speed, data_format=_CH_LAST_STR,
            unit_norm=False, keep=None):
    """``kapre_rir_ism`` on the current device: ``records`` (B, 14) and ``mics`` (B, M, 3) host float64 arrays, the
    responses as float32 (B, L, M) channels_last or (B, M, L) channels_first.  Values the kernel cannot take raise
    ValueError before anything is launched.  The records go up in one host-to-device copy; under CUDA graph capture
    they are staged in a pinned buffer appended to ``keep`` (a list the caller holds for the graph's life; by default
    one kept for the process), because the graph's copy node reads it on every replay.  ``unit_norm``: each response scaled to unit L2 norm (a second
    launch)."""
    _require_cuda()
    records = np.ascontiguousarray(records, np.float64)
    mics = np.ascontiguousarray(mics, np.float64)
    B, M = mics.shape[0], mics.shape[1]
    L = int(output_length)
    host = torch.from_numpy(np.concatenate([records.ravel(), mics.ravel()]))
    dev = torch.device('cuda', torch.cuda.current_device())
    if data_format == _CH_LAST_STR:
        out = torch.empty((B, L, M), dtype=torch.float32, device=dev)
        sb, st, sm = out.stride()
    else:
        out = torch.empty((B, M, L), dtype=torch.float32, device=dev)
        sb, sm, st = out.stride()
    lib = N.lib()
    args = (int(filter_length), float(sample_rate), float(sound_speed), N.RIR_UNIT_NORM if unit_norm else 0)
    # validation alone (null device pointers), so that a bad value raises before the upload and the launch
    if lib.kapre_rir_ism(_ptr(host), None, B, M, L, *args, None, sb, sm, st, _stream_ptr()) == -1:
        raise ValueError(lib.kapre_last_error().decode())
    if B == 0:
        return out
    if torch.cuda.is_current_stream_capturing():
        host = host.pin_memory()
        (_rir_captured if keep is None else keep).append(host)
    rec_dev = host.to(dev, non_blocking=True)
    N.check(lib.kapre_rir_ism(_ptr(host), _ptr(rec_dev), B, M, L, *args, _ptr(out), sb, sm, st, _stream_ptr()))
    return out


IIR_MAX_ORDER = 8


def iir_check(x, b, a, data_format):
    """Shapes of ``lfilter``'s operands: x (B, L, C) / (B, C, L); b and a of one shape, (N + 1,), (C, N + 1) or
    (B, C, N + 1) with N <= 8.  Returns (B, C, L), (Bc, Cc, N + 1): the coefficients' batch and channels (1 when
    shared)."""
    if x.dim() != 3:
        raise ValueError('lfilter expects a 3-D waveform batch, got shape %s' % (tuple(x.shape),))
    B, C, L = (x.shape[0], x.shape[2], x.shape[1]) if data_format == _CH_LAST_STR else tuple(x.shape)
    if tuple(b.shape) != tuple(a.shape):
        raise ValueError('a_coeffs %s and b_coeffs %s must have the same shape' % (tuple(a.shape), tuple(b.shape)))
    if a.dim() == 1:
        Bc, Cc = 1, 1
    elif a.dim() == 2:
        Bc, Cc = 1, a.shape[0]
    elif a.dim() == 3:
        Bc, Cc = a.shape[0], a.shape[1]
    else:
        raise ValueError('coefficients must be 1-D, 2-D or 3-D, got shape %s' % (tuple(a.shape),))
    n = a.shape[-1]
    if n < 1:
        raise ValueError('coefficients need at least one value per filter')
    if n - 1 > IIR_MAX_ORDER:
        raise ValueError('IIR order %d is above the supported %d (at most %d coefficients)'
                         % (n - 1, IIR_MAX_ORDER, IIR_MAX_ORDER + 1))
    if a.dim() == 2 and Cc != C:
        raise ValueError('2-D coefficients need one filter per channel: %d filters for %d channels' % (Cc, C))
    if a.dim() == 3 and (Bc not in (1, B) or Cc not in (1, C)):
        raise ValueError('3-D coefficients: batch %d and channels %d must be 1 or the waveform\'s (%d, %d)'
                         % (Bc, Cc, B, C))
    return (B, C, L), (Bc, Cc, n)


def _iir_coeffs(b, a):
    """kapre_iir_coeffs over normalised (Bc, Cc, N + 1) float32 tensors; a batch or channel axis of 1 is shared through
    a zero stride."""
    b = b.detach().to(torch.float32).contiguous()
    a = a.detach().to(torch.float32).contiguous()
    st = []
    for t in (b, a):
        st += [0 if t.shape[0] == 1 else t.stride(0), 0 if t.shape[1] == 1 else t.stride(1)]
    return N.IirCoeffs(b.data_ptr(), a.data_ptr(), *st, int(a.shape[-1]) - 1), (b, a)


def lfilter_workspace(B, C, L, order, device):
    return _scratch(N.lib().kapre_lfilter_workspace_bytes(B, C, L, order), device)


def lfilter_forward(x, b, a, flags, data_format):
    """y = ``kapre_lfilter`` of x with normalised (Bc, Cc, N + 1) coefficients on x's device: four launches."""
    x = _raw(x.to(torch.float32))
    xd, (B, C, L) = _wave_desc(x, data_format)
    y, yd = _wave_alloc(B, C, L, data_format, x.device)
    if y.numel():
        cf, keep = _iir_coeffs(b, a)
        ws = lfilter_workspace(B, C, L, cf.order, x.device)
        N.check(N.lib().kapre_lfilter(_ptr(x), ctypes.byref(xd), ctypes.byref(cf), int(flags), _ptr(y), ctypes.byref(yd),
                                      _ptr(ws), _stream_ptr()))
    return y


def lfilter_backward(gy, x, y, b, a, flags, data_format, want_coeffs):
    """Gradients of ``lfilter_forward`` (unclamped) at output gradient gy: (gx, gb, ga), gb and ga shaped like b and
    a (summed over their shared axes; ga[..., 0] = 0) or None without ``want_coeffs``.  Four launches; x and y (the
    unclamped output) are read only for the coefficient gradients.  The kernel writes per-(chunk, item, channel)
    partial sums and torch adds them, so the result is deterministic."""
    gy = _raw(gy.to(torch.float32))
    gd, (B, C, L) = _wave_desc(gy, data_format)
    gx, od = _wave_alloc(B, C, L, data_format, gy.device)
    cf, keep = _iir_coeffs(b, a)
    n = cf.order + 1
    part = None
    if want_coeffs:
        K = -(-L // 65)
        part = torch.empty((2 * n - 1, B, C, K), dtype=torch.float32, device=gy.device)
        x = _raw(x.to(torch.float32))
        xd, _ = _wave_desc(x, data_format)
        yd, _ = _wave_desc(y, data_format)
    if gx.numel():
        ws = lfilter_workspace(B, C, L, cf.order, gy.device)
        N.check(N.lib().kapre_lfilter_backward(
            _ptr(gy), ctypes.byref(gd), _ptr(x) if want_coeffs else None, ctypes.byref(xd) if want_coeffs else None,
            _ptr(y) if want_coeffs else None, ctypes.byref(yd) if want_coeffs else None, ctypes.byref(cf), int(flags),
            _ptr(gx), ctypes.byref(od), _ptr(part) if want_coeffs else None, _ptr(ws), _stream_ptr()))
    if not want_coeffs:
        return gx, None, None
    s = part.sum(dim=3) if part.shape[3] else torch.zeros(part.shape[:3], dtype=torch.float32, device=gy.device)
    gb = s[:n].permute(1, 2, 0)                                                       # (B, C, N + 1)
    ga = torch.cat([torch.zeros_like(s[:1]), s[n:]], 0).permute(1, 2, 0)
    Bc, Cc = b.shape[0], b.shape[1]
    if Bc == 1:
        gb, ga = gb.sum(0, keepdim=True), ga.sum(0, keepdim=True)
    if Cc == 1:
        gb, ga = gb.sum(1, keepdim=True), ga.sum(1, keepdim=True)
    return gx, gb, ga


@_device_of_first_arg
def lfilter(x, b, a, clamp=True, reverse=False, data_format=_CH_LAST_STR):
    """IIR filter along the time axis of x (B, L, C) / (B, C, L) with normalised float32 coefficients b, a on x's
    device, each (Bc, Cc, N + 1) with Bc in {1, B}, Cc in {1, C} (1 shares the filter).  ``reverse`` runs it in
    reverse time.  Everything is validated before any launch.  Differentiable with respect to x, b and a: under
    autograd the kernel writes the unclamped output and ``torch.clamp`` applies the clamp (the same bits)."""
    if not (isinstance(x, torch.Tensor) and x.is_cuda and b.is_cuda and a.is_cuda):
        raise N.KapreNativeError('lfilter needs CUDA tensors')
    if b.device != x.device or a.device != x.device:
        raise ValueError('waveform on %s, coefficients on %s / %s' % (x.device, b.device, a.device))
    if b.dim() != 3:
        raise ValueError('normalised coefficients must be 3-D (batch, channels, order + 1)')
    (B, C, L), (_, _, n) = iir_check(x, b, a, data_format)
    lfilter_workspace(B, C, L, n - 1, x.device)            # size checks before anything is launched
    flags = N.IIR_REVERSE if reverse else 0
    if _wants_grad(x) or _wants_grad(b) or _wants_grad(a):
        from . import autograd
        y = autograd.lfilter(x, b, a, flags, data_format)
        return torch.clamp(y, -1.0, 1.0) if clamp else y
    return lfilter_forward(x, b, a, flags | (N.IIR_CLAMP if clamp else 0), data_format)


SOS_MAX_SECTIONS = 8


def _shared_axes(shape, B, C, what):
    """(Bc, Cc) of a per-filter tensor whose leading axes are () , (ch,) or (batch, ch), each 1 (shared) or the
    waveform's."""
    if len(shape) == 0:
        return 1, 1
    Bc, Cc = (1, shape[0]) if len(shape) == 1 else shape
    if Bc not in (1, B) or Cc not in (1, C):
        raise ValueError('%s: batch %d and channels %d must be 1 or the waveform\'s (%d, %d)' % (what, Bc, Cc, B, C))
    return Bc, Cc


def sos_check(x, sos, data_format):
    """Shapes of ``sosfilt``'s operands: x (B, L, C) / (B, C, L); sos (S, 6), (C, S, 6) or (B, C, S, 6) with axes of 1
    shared and 1 <= S <= 8.  Returns (B, C, L), (Bc, Cc, S)."""
    if x.dim() != 3:
        raise ValueError('sosfilt expects a 3-D waveform batch, got shape %s' % (tuple(x.shape),))
    B, C, L = (x.shape[0], x.shape[2], x.shape[1]) if data_format == _CH_LAST_STR else tuple(x.shape)
    if sos.dim() not in (2, 3, 4) or sos.shape[-1] != 6:
        raise ValueError('sos must be (S, 6), (ch, S, 6) or (batch, ch, S, 6), got shape %s' % (tuple(sos.shape),))
    S = sos.shape[-2]
    if not 1 <= S <= SOS_MAX_SECTIONS:
        raise ValueError('%d sections: 1 to %d are supported' % (S, SOS_MAX_SECTIONS))
    Bc, Cc = _shared_axes(tuple(sos.shape[:-2]), B, C, 'sos')
    return (B, C, L), (Bc, Cc, S)


def sos_state_check(z, B, C, S, name):
    """A state tensor of ``sosfilt``: (S, 2), (C, S, 2) or (B, C, S, 2) with axes of 1 shared.  Returns (Bz, Cz)."""
    if z.dim() not in (2, 3, 4) or tuple(z.shape[-2:]) != (S, 2):
        raise ValueError('%s must be (%d, 2), (ch, %d, 2) or (batch, ch, %d, 2), got shape %s'
                         % (name, S, S, S, tuple(z.shape)))
    return _shared_axes(tuple(z.shape[:-2]), B, C, name)


def sosfilt_workspace(B, C, L, S, device):
    return _scratch(N.lib().kapre_sosfilt_workspace_bytes(B, C, L, S), device)


def _sos_state_desc(z):
    """kapre_sos_state_desc of a (Bz, Cz, S, 2) tensor whose last axis is contiguous; axes of 1 get stride 0."""
    return N.SosStateDesc(0 if z.shape[0] == 1 else z.stride(0), 0 if z.shape[1] == 1 else z.stride(1), z.stride(2))


def sosfilt_forward(x, sos, zi, reverse, data_format, want_zf):
    """(y, zf) = ``kapre_sosfilt`` of x with float32 coefficients sos (Bc, Cc, S, 6) and initial state zi
    (Bz, Cz, S, 2) or None, on x's device: four launches.  zf (B, C, S, 2) is None unless ``want_zf``."""
    x = _raw(x.to(torch.float32))
    xd, (B, C, L) = _wave_desc(x, data_format)
    y, yd = _wave_alloc(B, C, L, data_format, x.device)
    S = sos.shape[2]
    zf = torch.empty((B, C, S, 2), dtype=torch.float32, device=x.device) if want_zf else None
    if zi is not None:
        zi = zi.detach().to(torch.float32).contiguous()
    if y.numel() == 0:
        if zf is not None:
            zf.copy_(zi.expand(B, C, S, 2) if zi is not None else torch.zeros_like(zf))
        return y, zf
    sos = sos.detach().to(torch.float32).contiguous()
    cf = N.SosCoeffs(sos.data_ptr(), 0 if sos.shape[0] == 1 else sos.stride(0), 0 if sos.shape[1] == 1 else sos.stride(1),
                     S)
    zd = _sos_state_desc(zi) if zi is not None else None
    fd = _sos_state_desc(zf) if zf is not None else None
    ws = sosfilt_workspace(B, C, L, S, x.device)
    N.check(N.lib().kapre_sosfilt(_ptr(x), ctypes.byref(xd), ctypes.byref(cf), _ptr(zi) if zi is not None else None,
                                  ctypes.byref(zd) if zd is not None else None, N.IIR_REVERSE if reverse else 0, _ptr(y),
                                  ctypes.byref(yd), _ptr(zf) if zf is not None else None,
                                  ctypes.byref(fd) if fd is not None else None, _ptr(ws), _stream_ptr()))
    return y, zf


@_device_of_first_arg
def sosfilt(x, sos, zi=None, scale=None, dc_gain=None, reverse=False, data_format=_CH_LAST_STR, want_zf=False):
    """Second-order-section cascade along the time axis of x (B, L, C) / (B, C, L) with float32 coefficients sos
    (Bc, Cc, S, 6) on x's device (a0 is not read), from the initial state zi (Bz, Cz, S, 2) or zero.  With ``scale``
    ((B, C)) the initial state is ``zi * scale``, where zi must be the unit-step steady state of the cascade and
    ``dc_gain`` ((Bc, Cc)) its DC gain: that is how ``sosfiltfilt`` starts, and the gradient reaches ``scale``.
    ``reverse`` runs it in reverse time.  Returns (y, zf), zf None unless ``want_zf``; zf carries no gradient.
    Everything is validated before any launch.  Differentiable with respect to x (and ``scale``)."""
    if not (isinstance(x, torch.Tensor) and x.is_cuda and sos.is_cuda):
        raise N.KapreNativeError('sosfilt needs CUDA tensors')
    if sos.device != x.device or (zi is not None and zi.device != x.device):
        raise ValueError('waveform on %s, coefficients or state elsewhere' % (x.device,))
    if sos.dim() != 4:
        raise ValueError('coefficients must be 4-D (batch, channels, sections, 6)')
    (B, C, L), (_, _, S) = sos_check(x, sos, data_format)
    if zi is not None:
        sos_state_check(zi, B, C, S, 'zi')
    if torch.is_grad_enabled() and (sos.requires_grad or (zi is not None and zi.requires_grad)):
        raise ValueError('sosfilt has no gradient with respect to sos or zi; detach them')
    sosfilt_workspace(B, C, L, S, x.device)                 # size checks before anything is launched
    if _wants_grad(x) or _wants_grad(scale):
        from . import autograd
        return autograd.sosfilt(x, scale, sos, zi, dc_gain, reverse, data_format, want_zf)
    if scale is not None:
        zi = zi * scale.to(zi.dtype).reshape(B, C, 1, 1)
    return sosfilt_forward(x, sos, zi, reverse, data_format, want_zf)


def add_noise_workspace_bytes(B, C, L):
    """``kapre_add_noise_workspace_bytes``; raises on a negative size or an overflow."""
    n = int(N.lib().kapre_add_noise_workspace_bytes(B, C, L))
    if n < 0:
        N.check(n)
    return n


def add_noise_workspace(B, C, L, device):
    return _scratch(add_noise_workspace_bytes(B, C, L), device)


def _noise_source(noise, bank, data_format):
    """kapre_noise_source of a float32 noise tensor in ``data_format`` or of a bank (flat clips, start, clip_len,
    offset), and the tensors it points into."""
    if bank is not None:
        flat, start, clip, offset = bank
        return N.NoiseSource(N.NOISE_BANK, None, N.WaveDesc(), flat.data_ptr(), flat.numel(), start.data_ptr(),
                             clip.data_ptr(), offset.data_ptr())
    nd, _ = _wave_desc(noise, data_format)
    return N.NoiseSource(N.NOISE_TENSOR, noise.data_ptr(), nd, None, 0, None, None, None)


def _snr_desc(snr, lengths):
    """kapre_snr_desc over (B, C) float32 snr and int32 lengths (or None) views; a stride of 0 broadcasts."""
    if lengths is None:
        return N.SnrDesc(snr.data_ptr(), snr.stride(0), snr.stride(1), None, 0, 0)
    return N.SnrDesc(snr.data_ptr(), snr.stride(0), snr.stride(1), lengths.data_ptr(), lengths.stride(0),
                     lengths.stride(1))


def add_noise_forward(x, noise, bank, snr, lengths, data_format, want_stats):
    """y = ``kapre_add_noise`` (two launches) and, with ``want_stats``, the (B, C, 2) float64 energies (Ex, En)."""
    x = _raw(x.to(torch.float32))
    xd, (B, C, L) = _wave_desc(x, data_format)
    y, yd = _wave_alloc(B, C, L, data_format, x.device)
    # every column's (Ex, En) is written by the tile of its first segment
    stats = torch.empty((B, C, 2), dtype=torch.float64, device=x.device) if want_stats else None
    if y.numel():
        ws = add_noise_workspace(B, C, L, x.device)
        src = _noise_source(noise, bank, data_format)
        N.check(N.lib().kapre_add_noise(_ptr(x), ctypes.byref(xd), ctypes.byref(src), ctypes.byref(_snr_desc(snr, lengths)),
                                        _ptr(y), ctypes.byref(yd), _ptr(stats) if want_stats else None, _ptr(ws),
                                        _stream_ptr()))
    return y, stats


def add_noise_backward(g, x, noise, bank, snr, lengths, stats, data_format, want_noise, want_snr):
    """Gradients of ``add_noise_forward`` at output gradient g: (gx, gn or None, gsnr (B, C) or None), per element
    and column, two launches; the caller's autograd sums gn and gsnr over broadcast axes."""
    g = _raw(g.to(torch.float32))
    gd, (B, C, L) = _wave_desc(g, data_format)
    xd, _ = _wave_desc(x, data_format)
    gx, od = _wave_alloc(B, C, L, data_format, g.device)
    gn, nd = _wave_alloc(B, C, L, data_format, g.device) if want_noise else (None, None)
    gsnr = torch.zeros((B, C), dtype=torch.float32, device=g.device) if want_snr else None
    if gx.numel():
        ws = add_noise_workspace(B, C, L, g.device)
        src = _noise_source(noise, bank, data_format)
        N.check(N.lib().kapre_add_noise_backward(
            _ptr(g), ctypes.byref(gd), _ptr(x), ctypes.byref(xd), ctypes.byref(src),
            ctypes.byref(_snr_desc(snr, lengths)), _ptr(stats), _ptr(gx), ctypes.byref(od),
            _ptr(gn) if want_noise else None, ctypes.byref(nd) if want_noise else None,
            _ptr(gsnr) if want_snr else None, _ptr(ws), _stream_ptr()))
    return gx, gn, gsnr


def _per_column(v, B, C, dtype, device, name):
    """A number, array or tensor broadcastable to (B, C) by torch's rules, on ``device`` (cast to ``dtype``)."""
    if not isinstance(v, torch.Tensor):
        a = np.asarray(v)
        if a.dtype.kind not in 'iuf':
            raise ValueError('%s must be real numbers, got: %r' % (name, v))
        v = torch.from_numpy(np.ascontiguousarray(a))
    if v.dtype == torch.bool or v.dtype.is_complex:
        raise ValueError('%s must be real numbers, got dtype %s' % (name, v.dtype))
    if v.dim() > 2 or any(n not in (1, m) for n, m in zip(v.shape[::-1], (C, B))):
        raise ValueError('%s of shape %s does not broadcast to (batch, channels) = (%d, %d)'
                         % (name, tuple(v.shape), B, C))
    if v.is_cuda and v.device != device:
        raise ValueError('%s on %s, the waveform on %s' % (name, v.device, device))
    return v.to(device=device, dtype=dtype) if dtype is not None else v.to(device=device)


def noise_check(x, noise, data_format):
    """Shapes of ``add_noise``'s operands: x (B, L, C) / (B, C, L); noise 3-D in the same format with batch in {1, B},
    channels in {1, C} and L samples.  Returns (B, C, L)."""
    if x.dim() != 3:
        raise ValueError('add_noise expects a 3-D waveform batch, got shape %s' % (tuple(x.shape),))
    B, C, L = (x.shape[0], x.shape[2], x.shape[1]) if data_format == _CH_LAST_STR else tuple(x.shape)
    if noise is not None:
        if noise.dim() != 3:
            raise ValueError('the noise must be 3-D like the waveform, got shape %s' % (tuple(noise.shape),))
        Bn, Cn, Ln = (noise.shape[0], noise.shape[2], noise.shape[1]) if data_format == _CH_LAST_STR \
            else tuple(noise.shape)
        if Bn not in (1, B) or Cn not in (1, C) or Ln != L:
            raise ValueError('noise of shape %s does not match the waveform %s (batch and channels may be 1)'
                             % (tuple(noise.shape), tuple(x.shape)))
    return B, C, L


@_device_of_first_arg
def add_noise(x, noise, snr, lengths=None, data_format=_CH_LAST_STR, bank=None):
    """``torchaudio.functional.add_noise`` per (item, channel) column of x (B, L, C) / (B, C, L) on the GPU:
    ``y = x + s n`` with ``s = sqrt(Ex / En) 10^(-snr / 20)`` and the energies over ``t < lengths``; ``s = 0`` where
    either energy is 0 (torchaudio gives NaN for silent noise).  ``noise``: 3-D in x's format with batch and channels
    1 or x's (broadcast without a copy), or None with ``bank = (flat clips, start, clip_len, offset)`` (per-item int64
    CUDA tensors; item b reads ``flat[start + (offset + t) mod clip_len]``).  ``snr`` and ``lengths``: numbers or
    tensors broadcastable to (B, C) by torch's rules; lengths are clamped to [0, L] on the device, without a sync.
    Everything is checked before any launch.  Two launches; differentiable with respect to x, a tensor noise and
    snr."""
    if not (isinstance(x, torch.Tensor) and x.is_cuda):
        raise N.KapreNativeError('add_noise needs a CUDA waveform')
    if noise is not None and not isinstance(noise, torch.Tensor):
        noise = torch.as_tensor(np.asarray(noise, np.float32))
    B, C, L = noise_check(x, noise, data_format)
    if noise is not None:
        if noise.is_cuda and noise.device != x.device:
            raise ValueError('noise on %s, the waveform on %s' % (noise.device, x.device))
        noise = noise.to(device=x.device, dtype=torch.float32)
        noise = noise.expand(B, L, C) if data_format == _CH_LAST_STR else noise.expand(B, C, L)
    elif bank is None:
        raise ValueError('add_noise needs a noise tensor or a bank')
    snr = _per_column(snr, B, C, torch.float32, x.device, 'snr').expand(B, C)
    if lengths is not None:
        lengths = _per_column(lengths, B, C, None, x.device, 'lengths')
        if lengths.dtype.is_floating_point:
            raise ValueError('lengths must be integers, got dtype %s' % (lengths.dtype,))
        lengths = torch.clamp(lengths, 0, L).to(torch.int32).expand(B, C)
    add_noise_workspace_bytes(B, C, L)                     # size checks before anything is launched
    if _wants_grad(x) or _wants_grad(noise) or _wants_grad(snr):
        from . import autograd
        return autograd.add_noise(x, noise, snr, lengths, bank, data_format)
    y, _ = add_noise_forward(x, noise, bank, snr, lengths, data_format, False)
    return y


LOUDNESS_MAX_CHANNELS = 5
_k_weighting = {}


def loudness_geometry(sample_rate):
    """(G, S): the 400 ms gate and its 75 %-overlap step in samples, rounded as torchaudio rounds them."""
    G = int(round(0.4 * sample_rate))
    return G, int(round(G * 0.25))


def k_weighting(sample_rate, device):
    """The K-weighting's two normalised filters as ((b, a), (b, a)) float32 (1, 1, 3) tensors on ``device``, made once
    per (device, rate): nothing is copied to the device on later calls, so a call can be captured in a CUDA graph."""
    from .backend import k_weighting_coefficients
    key = (device.index if device.index is not None else torch.cuda.current_device(), float(sample_rate))
    c = _k_weighting.get(key)
    if c is None:
        c = tuple(tuple(torch.tensor(v, dtype=torch.float32, device=device).reshape(1, 1, 3) for v in (b / a[0], a / a[0]))
                  for b, a in k_weighting_coefficients(sample_rate))
        _k_weighting[key] = c
    return c


def loudness_sizes(B, C, L, G, S):
    """(workspace bytes, stats bytes) of ``kapre_loudness``; raises on a bad size or an overflow."""
    stats = ctypes.c_int64(0)
    n = int(N.lib().kapre_loudness_workspace_bytes(B, C, L, G, S, ctypes.byref(stats)))
    if n < 0:
        N.check(n)
    return n, int(stats.value)


def loudness_forward(y, lengths, G, S, data_format):
    """(LKFS (B,) float32, stats) of the K-weighted y: ``kapre_loudness``, two launches."""
    y = _raw(y.to(torch.float32))
    yd, (B, C, L) = _wave_desc(y, data_format)
    nw, ns = loudness_sizes(B, C, L, G, S)
    out = torch.empty(B, dtype=torch.float32, device=y.device)
    stats = _scratch(ns, y.device)
    if B:
        ws = _scratch(nw, y.device)
        N.check(N.lib().kapre_loudness(_ptr(y), ctypes.byref(yd), _ptr(lengths) if lengths is not None else None, G, S,
                                       _ptr(out), _ptr(stats), _ptr(ws), _stream_ptr()))
    return out, stats


def loudness_backward(gl, y, lengths, G, S, stats, data_format):
    """The gradient of ``loudness_forward`` with respect to y at output gradient gl (B,): one launch."""
    y = _raw(y.to(torch.float32))
    yd, (B, C, L) = _wave_desc(y, data_format)
    gl = gl.to(torch.float32).contiguous()
    gy, gd = _wave_alloc(B, C, L, data_format, y.device)
    if gy.numel():
        N.check(N.lib().kapre_loudness_backward(_ptr(gl), _ptr(y), ctypes.byref(yd),
                                                _ptr(lengths) if lengths is not None else None, G, S, _ptr(stats),
                                                _ptr(gy), ctypes.byref(gd), _stream_ptr()))
    return gy


def _item_lengths(lengths, B, L, device):
    """A number or (B,) integers as (B,) int32 on ``device``, clamped to [0, L] there (no sync)."""
    if not isinstance(lengths, torch.Tensor):
        a = np.asarray(lengths)
        if a.dtype.kind not in 'iu':
            raise ValueError('lengths must be integers, got: %r' % (lengths,))
        lengths = torch.as_tensor(a)
    if lengths.dtype.is_floating_point or lengths.dtype.is_complex or lengths.dtype == torch.bool:
        raise ValueError('lengths must be integers, got dtype %s' % (lengths.dtype,))
    if lengths.dim() > 1 or (lengths.dim() == 1 and lengths.shape[0] != B):
        raise ValueError('lengths must be a number or (batch,) = (%d,) values, got shape %s' % (B, tuple(lengths.shape)))
    if lengths.is_cuda and lengths.device != device:
        raise ValueError('lengths on %s, the waveform on %s' % (lengths.device, device))
    return torch.clamp(lengths.to(device), 0, L).to(torch.int32).expand(B).contiguous()


@_device_of_first_arg
def loudness(x, sample_rate, lengths=None, data_format=_CH_LAST_STR):
    """``torchaudio.functional.loudness`` per item of x (B, L, C) / (B, C, L), C <= 5: the K-weighting as two
    ``kapre_lfilter`` calls with the clamp (four launches each), then ``kapre_loudness`` (two launches).  Everything is
    checked before any launch.  Differentiable with respect to x."""
    if not (isinstance(x, torch.Tensor) and x.is_cuda):
        raise N.KapreNativeError('loudness needs a CUDA waveform')
    if x.dim() != 3:
        raise ValueError('loudness expects a 3-D waveform batch, got shape %s' % (tuple(x.shape),))
    B, C, L = (x.shape[0], x.shape[2], x.shape[1]) if data_format == _CH_LAST_STR else tuple(x.shape)
    if not 1 <= C <= LOUDNESS_MAX_CHANNELS:
        raise ValueError('loudness supports 1 to %d channels, got %d' % (LOUDNESS_MAX_CHANNELS, C))
    (b1, a1), (b2, a2) = k_weighting(sample_rate, x.device)
    G, S = loudness_geometry(sample_rate)
    if lengths is not None:
        lengths = _item_lengths(lengths, B, L, x.device)
    loudness_sizes(B, C, L, G, S)                           # size checks before anything is launched
    lfilter_workspace(B, C, L, 2, x.device)
    y = lfilter(x, b1, a1, clamp=True, data_format=data_format)
    y = lfilter(y, b2, a2, clamp=True, data_format=data_format)
    if _wants_grad(y):
        from . import autograd
        return autograd.loudness(y, lengths, G, S, data_format)
    return loudness_forward(y, lengths, G, S, data_format)[0]


LoudnessStats = collections.namedtuple('LoudnessStats',
                                       ['integrated', 'momentary', 'short_term', 'loudness_range', 'true_peak'])
_true_peak_taps = None


def true_peak_taps():
    """The 81 float32 taps of ``signal.resample_filter(4, 1)``, made once on the host."""
    global _true_peak_taps
    if _true_peak_taps is None:
        from .signal import resample_filter
        _true_peak_taps = np.ascontiguousarray(resample_filter(4, 1), np.float32)
    return _true_peak_taps


def _taps_ptr():
    return true_peak_taps().ctypes.data_as(ctypes.c_void_p)


def true_peak_sizes(B, C, L):
    """(workspace bytes, stats bytes) of ``kapre_true_peak``; raises on a bad size or an overflow."""
    stats = ctypes.c_int64(0)
    n = int(N.lib().kapre_true_peak_workspace_bytes(B, C, L, ctypes.byref(stats)))
    if n < 0:
        N.check(n)
    return n, int(stats.value)


def true_peak_forward(x, lengths, data_format):
    """(dBTP (B, C) float32, stats) of x: ``kapre_true_peak``, two launches."""
    x = _raw(x.to(torch.float32))
    xd, (B, C, L) = _wave_desc(x, data_format)
    nw, ns = true_peak_sizes(B, C, L)
    out = torch.empty((B, C), dtype=torch.float32, device=x.device)
    stats = _scratch(ns, x.device)
    if B:
        ws = _scratch(nw, x.device)
        N.check(N.lib().kapre_true_peak(_ptr(x), ctypes.byref(xd), _ptr(lengths) if lengths is not None else None,
                                        _taps_ptr(), _ptr(out), _ptr(stats), _ptr(ws), _stream_ptr()))
    return out, stats


def true_peak_backward(g, lengths, stats, shape, data_format, device):
    """The gradient of ``true_peak_forward`` with respect to x of (B, C, L) = ``shape`` at output gradient g (B, C):
    one launch."""
    B, C, L = shape
    g = g.to(torch.float32).contiguous()
    gx, gd = _wave_alloc(B, C, L, data_format, device)
    if gx.numel():
        N.check(N.lib().kapre_true_peak_backward(_ptr(g), _ptr(lengths) if lengths is not None else None, _taps_ptr(),
                                                 _ptr(stats), _ptr(gx), ctypes.byref(gd), _stream_ptr()))
    return gx


def _meter_input(x, name, data_format, max_channels):
    if not (isinstance(x, torch.Tensor) and x.is_cuda):
        raise N.KapreNativeError('%s needs a CUDA waveform' % name)
    if x.dim() != 3:
        raise ValueError('%s expects a 3-D waveform batch, got shape %s' % (name, tuple(x.shape)))
    B, C, L = (x.shape[0], x.shape[2], x.shape[1]) if data_format == _CH_LAST_STR else tuple(x.shape)
    if not 1 <= C <= max_channels:
        raise ValueError('%s supports 1 to %d channels, got %d' % (name, max_channels, C))
    return B, C, L


@_device_of_first_arg
def true_peak(x, lengths=None, data_format=_CH_LAST_STR):
    """True peak (dBTP) per (item, channel) of x (B, L, C) / (B, C, L): ``kapre_true_peak`` (two launches).  Checked
    before any launch; differentiable with respect to x (one backward launch)."""
    B, C, L = _meter_input(x, 'true_peak', data_format, 2 ** 31 - 1)
    if lengths is not None:
        lengths = _item_lengths(lengths, B, L, x.device)
    true_peak_sizes(B, C, L)
    if _wants_grad(x):
        from . import autograd
        return autograd.true_peak(x, lengths, data_format)
    return true_peak_forward(x, lengths, data_format)[0]


def loudness_stats_sizes(B, C, L, G, S, G3):
    """Workspace bytes of ``kapre_loudness_stats``; raises on a bad size or an overflow."""
    n = int(N.lib().kapre_loudness_stats_workspace_bytes(B, C, L, G, S, G3))
    if n < 0:
        N.check(n)
    return n


@_device_of_first_arg
def loudness_stats(x, sample_rate, lengths=None, data_format=_CH_LAST_STR):
    """``LoudnessStats`` of x (B, L, C) / (B, C, L), C <= 5: the K-weighting as in ``loudness`` (eight launches), then
    ``kapre_loudness_stats`` (six) and ``kapre_true_peak`` on x (two).  Everything is checked before any launch; no
    gradient (an input that requires grad under grad mode raises)."""
    if _wants_grad(x):
        raise ValueError('loudness_stats has no gradient: use loudness and true_peak, which are differentiable, or call '
                         'it under torch.no_grad() or on a detached waveform')
    B, C, L = _meter_input(x, 'loudness_stats', data_format, LOUDNESS_MAX_CHANNELS)
    (b1, a1), (b2, a2) = k_weighting(sample_rate, x.device)
    G, S = loudness_geometry(sample_rate)
    G3 = int(round(3 * sample_rate))
    if lengths is not None:
        lengths = _item_lengths(lengths, B, L, x.device)
    nw = loudness_stats_sizes(B, C, L, G, S, G3)            # size checks before anything is launched
    true_peak_sizes(B, C, L)
    lfilter_workspace(B, C, L, 2, x.device)
    y = lfilter(x, b1, a1, clamp=True, data_format=data_format)
    y = _raw(lfilter(y, b2, a2, clamp=True, data_format=data_format))
    yd, _ = _wave_desc(y, data_format)
    Jm, Js = ((L - g) // S + 1 if L >= g else 0 for g in (G, G3))
    dev = x.device
    integrated = torch.empty(B, dtype=torch.float32, device=dev)
    momentary = torch.empty((B, Jm), dtype=torch.float32, device=dev)
    short_term = torch.empty((B, Js), dtype=torch.float32, device=dev)
    lra = torch.empty(B, dtype=torch.float32, device=dev)
    if B:
        ws = _scratch(nw, dev)
        N.check(N.lib().kapre_loudness_stats(_ptr(y), ctypes.byref(yd), _ptr(lengths) if lengths is not None else None,
                                             G, S, G3, _ptr(integrated), _ptr(momentary), _ptr(short_term), _ptr(lra),
                                             _ptr(ws), _stream_ptr()))
    return LoudnessStats(integrated, momentary, short_term, lra, true_peak_forward(x, lengths, data_format)[0])


def _pcen_params(params, eps, device):
    """kapre_pcen_params over the four parameter tensors (gain, bias, power, smooth_coef): float32, 0-d (one value
    for every band) or 1-d (one per band), on ``device``."""
    ts = []
    for t in params:
        if t.device != device:
            raise ValueError('PCEN parameters live on %s, the input on %s' % (t.device, device))
        ts.append(t.detach().to(torch.float32).contiguous())
    prm = N.PcenParams(*[t.data_ptr() for t in ts], *[int(t.dim() == 1) for t in ts], float(eps))
    return prm, ts


def _pcen_workspace(B, C, T, F, device):
    """(chunks, scratch tensor or None) the library uses for this shape on the current device."""
    k, nbytes = ctypes.c_int(1), ctypes.c_int64(0)
    N.check(N.lib().kapre_pcen_workspace(B, C, T, F, ctypes.byref(k), ctypes.byref(nbytes)))
    return k.value, _scratch(nbytes.value, device) if nbytes.value else None


@_device_of_first_arg
def pcen(E: torch.Tensor, params, eps, data_format):
    """Per-channel energy normalisation along the time axis of (b, t, band, ch) / (b, ch, t, band).  ``params``:
    gain, bias, power and smooth_coef tensors, each 0-d or with one value per band."""
    if not E.is_cuda:
        raise N.KapreNativeError('pcen needs a CUDA tensor')
    if torch.is_grad_enabled() and (E.requires_grad or any(p.requires_grad for p in params)):
        from . import autograd
        return autograd.pcen(E, params, eps, data_format)
    return pcen_forward(E, params, eps, data_format, save_M=False)[0]


def pcen_forward(E, params, eps, data_format, save_M):
    """(y, M): one launch (two when the time axis is chunked); M is written only with ``save_M``, else None."""
    E = _raw(E.to(torch.float32))
    ed, (B, C, T, F) = _spec_desc(E, data_format)
    prm, keep = _pcen_params(params, eps, E.device)
    y, yd = _spec_alloc(B, C, T, F, data_format, torch.float32, E.device)
    M, md = _spec_alloc(B, C, T, F, data_format, torch.float32, E.device) if save_M else (None, None)
    if y.numel():
        _, ws = _pcen_workspace(B, C, T, F, E.device)
        N.check(N.lib().kapre_pcen(_ptr(E), ctypes.byref(ed), B, C, T, F, ctypes.byref(prm), _ptr(y), ctypes.byref(yd),
                                   _ptr(M) if save_M else None, ctypes.byref(md) if save_M else None,
                                   _ptr(ws) if ws is not None else None, _stream_ptr()))
    return y, M


@_device_of_first_arg
def pcen_backward(E: torch.Tensor, M: torch.Tensor, gy: torch.Tensor, params, eps, data_format):
    """Gradients of ``pcen`` given its input ``E``, the smoother state ``M`` its forward wrote and the output
    gradient ``gy``: (gE, [g_gain, g_bias, g_power, g_smooth]), each parameter gradient shaped like the parameter.
    The kernel writes per-(chunk, item, channel, band) partial sums; summing them here keeps the result
    deterministic."""
    E = _raw(E.to(torch.float32))
    gy = _raw(gy.to(torch.float32))
    ed, (B, C, T, F) = _spec_desc(E, data_format)
    md, _ = _spec_desc(M, data_format)
    gd, _ = _spec_desc(gy, data_format)
    if gy.shape != E.shape or M.shape != E.shape:
        raise ValueError('PCEN gradient shapes %s / %s do not match %s' % (tuple(gy.shape), tuple(M.shape), tuple(E.shape)))
    prm, keep = _pcen_params(params, eps, E.device)
    gE, od = _spec_alloc(B, C, T, F, data_format, torch.float32, E.device)
    K, ws = _pcen_workspace(B, C, T, F, E.device)
    part = torch.empty((4, K, B, C, F), dtype=torch.float32, device=E.device)
    if part.numel():
        N.check(N.lib().kapre_pcen_backward(_ptr(E), ctypes.byref(ed), _ptr(M), ctypes.byref(md), _ptr(gy),
                                            ctypes.byref(gd), B, C, T, F, ctypes.byref(prm), _ptr(gE), ctypes.byref(od),
                                            _ptr(part), _ptr(ws) if ws is not None else None, _stream_ptr()))
    per_band = part.sum(dim=(1, 2, 3))
    grads = [per_band[j] if p.dim() == 1 else per_band[j].sum() for j, p in enumerate(params)]
    return gE, grads


@_device_of_first_arg
def griffin_lim(S: torch.Tensor, stft_plan: StftPlan, istft_plan: IstftPlan, n_iter, momentum, init, seed,
                input_data_format, output_data_format):
    """Griffin-Lim reconstruction of a (b, t, f, ch) / (b, ch, t, f) magnitude spectrogram by one library call that
    enqueues the whole loop.  Returns the untrimmed (b, L, ch) / (b, ch, L) waveform, L = (T - 1) hop + win_length,
    as ``istft`` does.  ``init``: ``N.GL_INIT_ONES`` or ``N.GL_INIT_RANDOM``; ``seed``: an int in [0, 2^64).
    The loop has no gradient: an input that requires grad under grad mode raises rather than being detached."""
    if not S.is_cuda:
        raise N.KapreNativeError('griffin_lim needs a CUDA tensor')
    if _wants_grad(S):
        raise RuntimeError('Griffin-Lim is not differentiable: call it under torch.no_grad() or on a detached input')
    if S.dtype != torch.float32:
        S = S.float()
    sd, (B, C, T, F) = _spec_desc(S, input_data_format)
    if F != stft_plan.n_fft // 2 + 1:
        raise ValueError('expected %d frequency bins for n_fft=%d, got %d' % (stft_plan.n_fft // 2 + 1, stft_plan.n_fft, F))
    L = (T - 1) * stft_plan.hop_length + stft_plan.win_length if T > 0 else 0
    y, yd = _wave_alloc(B, C, L, output_data_format, S.device)
    if y.numel() == 0:
        return y
    lib = N.lib()
    ws = _scratch(lib.kapre_griffin_lim_workspace_bytes(stft_plan.handle(), B, C, T), S.device)
    cfg = N.GlCfg(int(n_iter), float(momentum), int(init), int(seed))
    N.check(lib.kapre_griffin_lim(stft_plan.handle(), istft_plan.handle(), _ptr(S), ctypes.byref(sd), B, C, T,
                                  ctypes.byref(cfg), _ptr(y), ctypes.byref(yd), _ptr(ws), _stream_ptr()))
    return y


def time_stretch_frames(frames, rate):
    """ceil(frames / rate): the output frames of ``time_stretch`` (the length of torch.arange(0, frames, rate))."""
    return math.ceil(int(frames) / float(rate))


def _check_rate(rate):
    if isinstance(rate, (bool, np.bool_)) or not isinstance(rate, (int, float, np.integer, np.floating)) \
            or not math.isfinite(float(rate)) or not float(rate) > 0.0:
        raise ValueError('rate must be a finite number > 0, got: %r' % (rate,))
    return float(rate)


def _time_stretch_workspace(B, C, T, F, rate, device):
    """(chunks, scratch tensor or None) the library uses for this shape on the current device."""
    k, nbytes = ctypes.c_int(1), ctypes.c_int64(0)
    N.check(N.lib().kapre_time_stretch_workspace(B, C, T, F, rate, ctypes.byref(k), ctypes.byref(nbytes)))
    return k.value, _scratch(nbytes.value, device) if nbytes.value else None


@_device_of_first_arg
def time_stretch(X: torch.Tensor, rate, data_format):
    """Phase-vocoder time stretch of a complex (b, t, f, ch) / (b, ch, t, f) spectrogram along time:
    ``torchaudio.functional.phase_vocoder`` with ``ceil(t / rate)`` output frames (see ``include/kapre_b200.h``).
    ``rate == 1`` returns ``X`` itself."""
    if not X.is_cuda:
        raise N.KapreNativeError('time_stretch needs a CUDA tensor')
    if not X.is_complex():
        raise TypeError('time_stretch needs a complex spectrogram, got %s' % (X.dtype,))
    rate = _check_rate(rate)
    if rate == 1.0:
        return X
    if _wants_grad(X):
        from . import autograd
        return autograd.time_stretch(X, rate, data_format)
    return time_stretch_forward(X, rate, data_format)


def time_stretch_forward(X, rate, data_format):
    X = _raw(X.to(torch.complex64))
    xd, (B, C, T, F) = _spec_desc(X, data_format)
    Y, yd = _spec_alloc(B, C, time_stretch_frames(T, rate), F, data_format, torch.complex64, X.device)
    if Y.numel():
        _, ws = _time_stretch_workspace(B, C, T, F, rate, X.device)
        N.check(N.lib().kapre_time_stretch(_ptr(X), ctypes.byref(xd), B, C, T, F, rate, _ptr(Y), ctypes.byref(yd),
                                           _ptr(ws) if ws is not None else None, _stream_ptr()))
    return Y


@_device_of_first_arg
def time_stretch_backward(X: torch.Tensor, Y: torch.Tensor, G: torch.Tensor, rate, data_format):
    """Gradient of ``time_stretch`` with respect to ``X`` given the output ``Y`` it wrote and the output gradient
    ``G`` (any strides)."""
    X = _raw(X.to(torch.complex64))
    Y = _raw(Y.to(torch.complex64))
    G = _raw(G.to(torch.complex64))
    rate = _check_rate(rate)
    xd, (B, C, T, F) = _spec_desc(X, data_format)
    yd, _ = _spec_desc(Y, data_format)
    gd, _ = _spec_desc(G, data_format)
    if G.shape != Y.shape or _spec_desc(Y, data_format)[1] != (B, C, time_stretch_frames(T, rate), F):
        raise ValueError('time-stretch gradient shapes %s / %s do not match input %s at rate %g'
                         % (tuple(G.shape), tuple(Y.shape), tuple(X.shape), rate))
    gX, od = _spec_alloc(B, C, T, F, data_format, torch.complex64, X.device)
    if gX.numel():
        _, ws = _time_stretch_workspace(B, C, T, F, rate, X.device)
        N.check(N.lib().kapre_time_stretch_backward(_ptr(X), ctypes.byref(xd), _ptr(Y), ctypes.byref(yd), _ptr(G),
                                                    ctypes.byref(gd), B, C, T, F, rate, _ptr(gX), ctypes.byref(od),
                                                    _ptr(ws) if ws is not None else None, _stream_ptr()))
    return gX


@_device_of_first_arg
def invert_filterbank(x: torch.Tensor, plan: FilterbankInversePlan, n_iter, from_decibel, ref_value, amin,
                      data_format):
    """Non-negative least-squares inversion of a filterbank output, one launch: (b, t, n_bands, ch) /
    (b, ch, t, n_bands) -> float32 (b, t, n_freq, ch) / (b, ch, t, n_freq) in the same data format (see
    ``kapre_filterbank_invert``).  ``from_decibel``: the input is ``magnitude_to_decibel(., ref_value, amin)``.
    No gradient: an input that requires grad under grad mode raises rather than being detached."""
    if not x.is_cuda:
        raise N.KapreNativeError('invert_filterbank needs a CUDA tensor')
    if _wants_grad(x):
        raise RuntimeError('InverseFilterbank is not differentiable: call it under torch.no_grad() or on a detached '
                           'input')
    if x.dtype != torch.float32:
        x = x.float()
    xd, (B, C, T, M) = _spec_desc(x, data_format)
    if M != plan.n_bands:
        raise ValueError('the filterbank has %d bands, the input has %d' % (plan.n_bands, M))
    out, od = _spec_alloc(B, C, T, plan.n_freq, data_format, torch.float32, x.device)
    if out.numel() == 0:
        return out
    cfg = N.FbInvCfg(int(n_iter), int(bool(from_decibel)), float(ref_value), float(amin))
    N.check(N.lib().kapre_filterbank_invert(plan.handle(), ctypes.byref(cfg), _ptr(x), B, C, T, ctypes.byref(xd),
                                            _ptr(out), ctypes.byref(od), _stream_ptr()))
    return out


@_device_of_first_arg
def concat_frequency_map_backward(g: torch.Tensor, data_format):
    """Gradient of ``concat_frequency_map`` with respect to its input: the first C of the C + 1 channels of ``g``."""
    g = _raw(g.to(torch.float32)).contiguous()
    if g.dim() != 4:
        raise ValueError('ConcatenateFrequencyMap gradient must be 4-D, got shape %s' % (tuple(g.shape),))
    cl = data_format == _CH_LAST_STR
    if cl:
        B, T, F, C1 = g.shape
        gx = torch.empty((B, T, F, C1 - 1), dtype=torch.float32, device=g.device)
    else:
        B, C1, T, F = g.shape
        gx = torch.empty((B, C1 - 1, T, F), dtype=torch.float32, device=g.device)
    if gx.numel():
        N.check(N.lib().kapre_concat_frequency_map_backward(_ptr(g), _ptr(gx), B, C1 - 1, T, F, int(cl), _stream_ptr()))
    return gx


# ------------------------------------------------------------------------------- Kaldi features
KALDI_COMMON = dict(blackman_coeff=0.42, dither=0.0, energy_floor=1.0, frame_length=25.0, frame_shift=10.0,
                    min_duration=0.0, preemphasis_coefficient=0.97, raw_energy=True, remove_dc_offset=True,
                    round_to_power_of_two=True, sample_frequency=16000.0, snip_edges=True, subtract_mean=False,
                    window_type='povey')
_KALDI_MEL = dict(high_freq=0.0, htk_compat=False, low_freq=20.0, num_mel_bins=23, use_energy=False, vtln_high=-500.0,
                  vtln_low=100.0, vtln_warp=1.0)
# torchaudio.compliance.kaldi's keywords and defaults per function (without `channel`: every channel is computed)
KALDI_DEFAULTS = {
    'fbank': dict(KALDI_COMMON, **_KALDI_MEL, use_log_fbank=True, use_power=True),
    'mfcc': dict(KALDI_COMMON, **_KALDI_MEL, cepstral_lifter=22.0, num_ceps=13),
    'spectrogram': dict(KALDI_COMMON),
}
_KALDI_KIND = {'fbank': 0, 'mfcc': 1, 'spectrogram': 2}


def kaldi_options(kind, **kwargs):
    """torchaudio's keywords for ``kind`` ('fbank', 'mfcc', 'spectrogram') with their defaults filled in; raises on an
    unknown keyword or a non-finite number."""
    if kind not in KALDI_DEFAULTS:
        raise ValueError('kind must be one of %s, got %r' % (tuple(KALDI_DEFAULTS), kind))
    unknown = set(kwargs) - set(KALDI_DEFAULTS[kind])
    if unknown:
        raise TypeError('kaldi %s got unknown keyword(s) %s' % (kind, sorted(unknown)))
    o = dict(KALDI_DEFAULTS[kind], **kwargs)
    for k, v in o.items():
        if isinstance(v, float) and not math.isfinite(v):
            raise ValueError('%s must be finite, got %r' % (k, v))
    return o


class KaldiPlan(_PerDevice):
    """kapre_kaldi_plan per CUDA device for one set of options (as ``kaldi_options`` returns them): the window, the
    mel banks (VTLN included) and the DCT with the lifter are built here in float64 and held by the plan."""

    def __init__(self, kind, options):
        from . import backend
        o = dict(options)
        self.kind, self.options = kind, o
        W, H, Np = backend.kaldi_window_properties(o['sample_frequency'], o['frame_shift'], o['frame_length'],
                                                   o['round_to_power_of_two'])
        if W < 2 or H < 1:
            raise ValueError('window size %d and shift %d (samples) must be >= 2 and >= 1' % (W, H))
        if Np not in backend.KALDI_PADDED_SIZES:
            raise N.KapreNativeError('kaldi %s: padded window size %d is not supported; the supported sizes are %s '
                                     '(round_to_power_of_two=True with a window of 129 to 2048 samples)'
                                     % (kind, Np, ', '.join(map(str, backend.KALDI_PADDED_SIZES))))
        if not 0.0 <= o['preemphasis_coefficient'] <= 1.0:
            raise ValueError('preemphasis_coefficient must be in [0, 1]')
        if o['dither'] < 0.0:
            raise ValueError('dither must be >= 0')
        if o['energy_floor'] < 0.0:
            raise ValueError('energy_floor must be >= 0')
        self.W, self.H, self.N = W, H, Np
        self.window = backend.kaldi_window(o['window_type'], W, o['blackman_coeff']).astype(np.float32)
        M, n_ceps, banks, dct = 0, 0, None, None
        if kind != 'spectrogram':
            M = int(o['num_mel_bins'])
            banks = np.ascontiguousarray(backend.kaldi_mel_banks(
                M, Np, o['sample_frequency'], o['low_freq'], o['high_freq'], o['vtln_low'], o['vtln_high'],
                o['vtln_warp']), dtype=np.float32)
        if kind == 'mfcc':
            n_ceps = int(o['num_ceps'])
            if n_ceps > M:
                raise ValueError('num_ceps %d cannot be larger than num_mel_bins %d' % (n_ceps, M))
            d = backend.kaldi_dct(n_ceps, M, o['cepstral_lifter'])
            if o['htk_compat'] and not o['use_energy']:
                d[:, 0] *= math.sqrt(2.0)
            dct = np.ascontiguousarray(d, dtype=np.float32)
        self.banks, self.dct = banks, dct
        self.min_length = int(math.ceil(o['min_duration'] * o['sample_frequency'])) if o['min_duration'] > 0 else 0
        self.cfg = N.KaldiCfg(_KALDI_KIND[kind], W, H, Np, int(bool(o['snip_edges'])), self.min_length, M, n_ceps,
                              int(bool(o.get('use_energy', False))), int(bool(o.get('htk_compat', False))),
                              int(bool(o['raw_energy'])), int(bool(o.get('use_power', True))),
                              int(bool(o.get('use_log_fbank', True))), int(bool(o['remove_dc_offset'])),
                              int(bool(o['subtract_mean'])), float(o['preemphasis_coefficient']),
                              float(o['energy_floor']))
        self.K = M + int(bool(o.get('use_energy', False))) if kind == 'fbank' else (n_ceps if kind == 'mfcc'
                                                                                    else Np // 2 + 1)
        self._per_device = {}

    _destroy = 'kapre_kaldi_plan_destroy'

    def _create(self, lib, out):
        def p(a):
            return a.ctypes.data_as(ctypes.c_void_p) if a is not None else None
        return lib.kapre_kaldi_plan_create(ctypes.byref(self.cfg), p(self.window), p(self.banks), p(self.dct), out)

    def num_frames(self, length):
        from . import backend
        return backend.kaldi_num_frames(length, self.W, self.H, self.cfg.snip_edges, self.min_length)


_kaldi_plans = {}


def kaldi_plan(kind, options):
    key = (kind, tuple(sorted((k, v) for k, v in options.items() if k != 'dither')))
    with _lock:
        p = _kaldi_plans.get(key)
    if p is None:
        p = KaldiPlan(kind, options)
        with _lock:
            p = _kaldi_plans.setdefault(key, p)
    return p


def _kaldi_lengths(lengths, B, L, device):
    """(host int32 array, device int32 tensor) of per-item lengths in [0, L], or (None, None)."""
    if lengths is None:
        return None, None
    if isinstance(lengths, torch.Tensor):
        if lengths.dtype.is_floating_point or lengths.dtype.is_complex or lengths.dtype == torch.bool:
            raise ValueError('lengths must be integers, got dtype %s' % (lengths.dtype,))
        h = lengths.detach().to('cpu').numpy()
    else:
        h = np.asarray(lengths)
        if h.dtype.kind not in 'iu':
            raise ValueError('lengths must be integers, got %r' % (lengths,))
    h = np.ascontiguousarray(h.reshape(-1), dtype=np.int64)
    if h.shape != (B,):
        raise ValueError('lengths must have shape (batch,) = (%d,), got %s' % (B, h.shape))
    if (h < 0).any() or (h > L).any():
        raise ValueError('lengths must be in [0, %d], got %s' % (L, h))
    h = h.astype(np.int32)
    return h, torch.from_numpy(h).to(device)


def kaldi_forward(x, plan: KaldiPlan, lengths_h, lengths_d, data_format, dither, seed):
    """(B, L, C) / (B, C, L) float32 -> (B, T, K, C) / (B, C, T, K) features: one launch (two with subtract_mean)."""
    x = _raw(x.to(torch.float32))
    xd, (B, C, L) = _wave_desc(x, data_format)
    T = int(plan.num_frames(lengths_h).max()) if lengths_h is not None and B else (plan.num_frames(L) if B else 0)
    y, yd = _spec_alloc(B, C, T, plan.K, data_format, torch.float32, x.device)
    if y.numel():
        h = plan.handle()
        N.check(N.lib().kapre_kaldi_workspace_bytes(h, B, C, T, 0))
        lp = lengths_h.ctypes.data_as(ctypes.c_void_p) if lengths_h is not None else None
        N.check(N.lib().kapre_kaldi_features(h, _ptr(x), ctypes.byref(xd), lp,
                                             _ptr(lengths_d) if lengths_d is not None else None, T, float(dither),
                                             int(seed) & 0xFFFFFFFFFFFFFFFF, _ptr(y), ctypes.byref(yd), None,
                                             _stream_ptr()))
    return y


def kaldi_backward(gy, x, plan: KaldiPlan, lengths_h, lengths_d, data_format, dither, seed):
    """Gradient of ``kaldi_forward`` to x: two launches (three with subtract_mean)."""
    gy = _raw(gy.to(torch.float32))
    xd, (B, C, L) = _wave_desc(x, data_format)
    gd, (_, _, T, _) = _spec_desc(gy, data_format)
    gx, od = _wave_alloc(B, C, L, data_format, x.device)
    if gx.numel():
        h = plan.handle()
        ws = _scratch(N.lib().kapre_kaldi_workspace_bytes(h, B, C, T, 1), x.device)
        lp = lengths_h.ctypes.data_as(ctypes.c_void_p) if lengths_h is not None else None
        N.check(N.lib().kapre_kaldi_features_backward(
            h, _ptr(gy), ctypes.byref(gd), _ptr(x), ctypes.byref(xd), lp,
            _ptr(lengths_d) if lengths_d is not None else None, T, float(dither), int(seed) & 0xFFFFFFFFFFFFFFFF,
            _ptr(gx), ctypes.byref(od), _ptr(ws), _stream_ptr()))
    return gx


@_device_of_first_arg
def kaldi_features(x, plan: KaldiPlan, lengths=None, data_format=_CH_LAST_STR, dither=0.0, seed=0):
    """Kaldi features of every (item, channel) of a float32 CUDA waveform (B, L, C) / (B, C, L) under ``plan``:
    (B, T, K, C) / (B, C, T, K), T the largest frame count of the batch, frames past an item's count 0.
    Differentiable with respect to x; requiring grad changes neither the bits nor the launch count."""
    if not (isinstance(x, torch.Tensor) and x.is_cuda):
        raise N.KapreNativeError('kaldi features need a CUDA waveform')
    if x.dim() != 3:
        raise ValueError('kaldi features expect a 3-D waveform batch, got shape %s' % (tuple(x.shape),))
    if x.dtype != torch.float32:
        raise ValueError('kaldi features take a float32 waveform, got %s' % (x.dtype,))
    dither = float(dither)
    if not math.isfinite(dither) or dither < 0.0:
        raise ValueError('dither must be finite and >= 0, got %r' % (dither,))
    B, C, L = (x.shape[0], x.shape[2], x.shape[1]) if data_format == _CH_LAST_STR else tuple(x.shape)
    lh, ld = _kaldi_lengths(lengths, B, L, x.device)
    if _wants_grad(x):
        from . import autograd
        return autograd.kaldi_features(x, plan, lh, ld, data_format, dither, seed)
    return kaldi_forward(x, plan, lh, ld, data_format, dither, seed)


# ------------------------------------------------------------------------------- constant-Q transform
class CqtPlan(_PerDevice):
    """kapre_cqt_plan per CUDA device for one CQT configuration: the per-octave tap tables (``backend.cqt_filters``,
    float64, rounded here once to complex64) and the 2:1 decimation filter ``resample_filter(1, 2)``."""

    def __init__(self, sample_rate, hop_length, f_min=None, n_bins=84, bins_per_octave=12, filter_scale=1.0,
                 gamma=0.0, scale=True):
        from . import backend
        from .signal import resample_filter
        self.geometry = backend.cqt_geometry(sample_rate, hop_length, f_min, n_bins, bins_per_octave, filter_scale,
                                             gamma)
        self.hop_length, self.n_bins, self.bins_per_octave = int(hop_length), int(n_bins), int(bins_per_octave)
        self.n_octaves = self.geometry['n_octaves']
        self.tables = [t.astype(np.complex64) for t in backend.cqt_filters(sample_rate, f_min, n_bins, bins_per_octave,
                                                                           filter_scale, gamma, scale)]
        self.decimator = resample_filter(1, 2)
        taps = [t.shape[1] for t in self.tables] + [0] * (N.CQT_MAX_OCTAVES - len(self.tables))
        self.cfg = N.CqtCfg(self.n_bins, self.bins_per_octave, self.hop_length, (ctypes.c_int * N.CQT_MAX_OCTAVES)(*taps))
        self._flat = np.ascontiguousarray(np.concatenate([t.reshape(-1) for t in self.tables]))
        self._per_device = {}

    _destroy = 'kapre_cqt_plan_destroy'

    def _create(self, lib, out):
        return lib.kapre_cqt_plan_create(ctypes.byref(self.cfg), self._flat.ctypes.data_as(ctypes.c_void_p),
                                         self.decimator.ctypes.data_as(ctypes.c_void_p), self.decimator.size, out)

    def num_frames(self, length):
        return 1 + int(length) // self.hop_length

    def workspace(self, B, C, L, backward, device):
        return _scratch(N.lib().kapre_cqt_workspace_bytes(self.handle(), B, C, L, int(backward)), device)


def cqt_forward(x, plan: CqtPlan, input_data_format, output_data_format, magnitude):
    """(B, L, C) / (B, C, L) float32 -> (B, M, n_bins, C) / (B, C, M, n_bins) complex64 (or float32 |C|), and the
    workspace holding the pyramid: n_octaves - 1 resampling launches and one transform launch."""
    x = _raw(x.to(torch.float32))
    xd, (B, C, L) = _wave_desc(x, input_data_format)
    out, od = _spec_alloc(B, C, plan.num_frames(L), plan.n_bins, output_data_format,
                          torch.float32 if magnitude else torch.complex64, x.device)
    ws = plan.workspace(B, C, L, False, x.device)
    if out.numel():
        N.check(N.lib().kapre_cqt(plan.handle(), _ptr(x), ctypes.byref(xd), int(bool(magnitude)), _ptr(out),
                                  ctypes.byref(od), _ptr(ws), _stream_ptr()))
    return out, ws


def cqt_backward(g, x, fwd_ws, plan: CqtPlan, input_data_format, output_data_format, magnitude):
    """Gradient of ``cqt_forward`` to x: 2 n_octaves - 1 launches.  ``fwd_ws``: the forward's pyramid (magnitude mode)."""
    g = _raw(g.to(torch.float32 if magnitude else torch.complex64))
    x = _raw(x.to(torch.float32))
    xd, (B, C, L) = _wave_desc(x, input_data_format)
    gd, _ = _spec_desc(g, output_data_format)
    gx, gxd = _wave_alloc(B, C, L, input_data_format, x.device)
    if gx.numel():
        ws = plan.workspace(B, C, L, True, x.device)
        N.check(N.lib().kapre_cqt_backward(plan.handle(), _ptr(x), ctypes.byref(xd),
                                           _ptr(fwd_ws) if fwd_ws is not None else None, _ptr(g), ctypes.byref(gd),
                                           int(bool(magnitude)), _ptr(gx), ctypes.byref(gxd), _ptr(ws), _stream_ptr()))
    return gx


@_device_of_first_arg
def cqt(x, plan: CqtPlan, input_data_format=_CH_LAST_STR, output_data_format=_CH_LAST_STR, magnitude=False):
    """Constant-Q transform of a float32 CUDA waveform batch under ``plan`` (see ``time_frequency.CQT``).
    Differentiable with respect to x; requiring grad changes neither the bits nor the launch count."""
    if not (isinstance(x, torch.Tensor) and x.is_cuda):
        raise N.KapreNativeError('cqt needs a CUDA waveform')
    if x.dim() != 3:
        raise ValueError('cqt expects a 3-D waveform batch, got shape %s' % (tuple(x.shape),))
    if _wants_grad(x):
        from . import autograd
        return autograd.cqt(x, plan, input_data_format, output_data_format, magnitude)
    return cqt_forward(x, plan, input_data_format, output_data_format, magnitude)[0]


# ------------------------------------------------------------------------------- pitch tracking (YIN / pYIN)
class PitchPlan(_PerDevice):
    """kapre_pitch_plan per CUDA device for one YIN configuration (``backend.pitch_geometry``), or with ``pyin`` (a
    dict of ``backend.pyin_geometry``'s keyword arguments) one pYIN configuration, whose float64 tables
    (``backend.pyin_tables``) are uploaded once per device."""

    def __init__(self, sample_rate, fmin, fmax, frame_length=2048, win_length=None, hop_length=None, center=True,
                 trough_threshold=0.1, pyin=None, fill_na=float('nan')):
        from . import backend
        self.geometry = g = backend.pitch_geometry(sample_rate, fmin, fmax, frame_length, win_length, hop_length,
                                                   center)
        if isinstance(trough_threshold, bool) or not np.isfinite(float(trough_threshold)):
            raise ValueError('trough_threshold must be finite, got %r' % (trough_threshold,))
        self.pyin = None
        self.n_lags = g['n_lags']
        n_thr = n_pitch = band = 0
        ls = lw = lpv = lpu = 0.0
        self._tables = None
        if pyin is not None:
            self.pyin = q = backend.pyin_geometry(g, **pyin)
            t = {k: np.ascontiguousarray(v, dtype=np.float64) for k, v in backend.pyin_tables(g, q).items()}
            self._tables = t
            self._tab = N.PitchTables(*[t[name].ctypes.data_as(ctypes.c_void_p) for name, _ in N.PitchTables._fields_])
            n_thr, n_pitch, band = q['n_thresholds'], q['n_pitch'], q['band_width']
            tiny = backend.PITCH_TINY
            ls, lw = np.log(1.0 - q['switch_prob'] + tiny), np.log(q['switch_prob'] + tiny)
            lpv, lpu = np.log(tiny), np.log(1.0 / n_pitch + tiny)
        self.fill_na = float(fill_na)
        self.cfg = N.PitchCfg(g['sample_rate'], g['frame_length'], g['win_length'], g['hop_length'], int(g['center']),
                              g['min_period'], g['max_period'], float(trough_threshold), n_thr, n_pitch, band, ls, lw,
                              lpv, lpu, self.fill_na)
        self._per_device = {}

    _destroy = 'kapre_pitch_plan_destroy'

    def _create(self, lib, out):
        return lib.kapre_pitch_plan_create(ctypes.byref(self.cfg), ctypes.byref(self._tab) if self.pyin else None, out)

    def num_frames(self, length):
        g = self.geometry
        lp = int(length) + 2 * g['pad']
        return 0 if lp < g['frame_length'] else 1 + (lp - g['frame_length']) // g['hop_length']

    def workspace(self, B, C, L, device):
        return _scratch(N.lib().kapre_pitch_workspace_bytes(self.handle(), B, C, L), device)


def _frames_alloc(B, C, M, data_format, dtype, device):
    if data_format == _CH_LAST_STR:
        y = torch.empty((B, M, C), dtype=dtype, device=device)
        sb, st, sc = y.stride()
    else:
        y = torch.empty((B, C, M), dtype=dtype, device=device)
        sb, sc, st = y.stride()
    return y, N.FramesDesc(sb, sc, st)


def _pitch_input(x, name):
    if not (isinstance(x, torch.Tensor) and x.is_cuda):
        raise N.KapreNativeError('%s needs a CUDA waveform' % name)
    if x.dim() != 3:
        raise ValueError('%s expects a 3-D waveform batch, got shape %s' % (name, tuple(x.shape)))
    if x.dtype != torch.float32:
        raise ValueError('%s expects float32 samples, got %s' % (name, x.dtype))
    return x.detach()


def _cmndf_desc(cmndf, B, C, M, plan):
    """The (B, C, frames, n_lags) float32 CUDA tensor the caller passed for the CMNDF, or None."""
    if cmndf is None:
        return None, None
    if (not isinstance(cmndf, torch.Tensor) or not cmndf.is_cuda or cmndf.dtype != torch.float32
            or tuple(cmndf.shape) != (B, C, M, plan.n_lags)):
        raise ValueError('cmndf must be a float32 CUDA tensor of shape %s' % ((B, C, M, plan.n_lags),))
    return cmndf, N.SpecDesc(*cmndf.stride())


@_device_of_first_arg
def yin(x, plan: PitchPlan, data_format=_CH_LAST_STR, cmndf=None):
    """YIN f0 of a float32 CUDA waveform batch (``(B, L, C)`` channels_last or ``(B, C, L)``) under ``plan``, as
    ``(B, frames, C)`` / ``(B, C, frames)`` float32 (see ``signal.yin``).  ``cmndf`` (optional): a ``(B, C, frames,
    n_lags)`` float32 tensor that also receives the CMNDF at lags min_period .. max_period.  One launch.  Not
    differentiable: the output carries no ``grad_fn``."""
    x = _pitch_input(x, 'yin')
    xd, (B, C, L) = _wave_desc(x, data_format)
    M = plan.num_frames(L)
    f0, fd = _frames_alloc(B, C, M, data_format, torch.float32, x.device)
    cm, cd = _cmndf_desc(cmndf, B, C, M, plan)
    if f0.numel():
        N.check(N.lib().kapre_yin(plan.handle(), _ptr(x), ctypes.byref(xd), _ptr(f0), ctypes.byref(fd),
                                  _ptr(cm) if cm is not None else None, ctypes.byref(cd) if cd is not None else None,
                                  _stream_ptr()))
    return f0


@_device_of_first_arg
def pyin(x, plan: PitchPlan, data_format=_CH_LAST_STR, cmndf=None):
    """pYIN of a float32 CUDA waveform batch under a pYIN ``plan``: ``(f0, voiced_flag, voiced_prob)``, each ``(B,
    frames, C)`` / ``(B, C, frames)`` (float32, bool, float32; see ``signal.pyin``).  ``cmndf`` as in ``yin``.  Two
    launches.  Not differentiable: the outputs carry no ``grad_fn``."""
    if plan.pyin is None:
        raise ValueError('pyin needs a PitchPlan made with pyin parameters')
    x = _pitch_input(x, 'pyin')
    xd, (B, C, L) = _wave_desc(x, data_format)
    M = plan.num_frames(L)
    f0, fd = _frames_alloc(B, C, M, data_format, torch.float32, x.device)
    flag, _ = _frames_alloc(B, C, M, data_format, torch.bool, x.device)
    vp, _ = _frames_alloc(B, C, M, data_format, torch.float32, x.device)
    cm, cd = _cmndf_desc(cmndf, B, C, M, plan)
    if f0.numel():
        ws = plan.workspace(B, C, L, x.device)
        N.check(N.lib().kapre_pyin(plan.handle(), _ptr(x), ctypes.byref(xd), _ptr(f0), _ptr(flag), _ptr(vp),
                                   ctypes.byref(fd), _ptr(cm) if cm is not None else None,
                                   ctypes.byref(cd) if cd is not None else None, _ptr(ws), _stream_ptr()))
    return f0, flag, vp


# ------------------------------------------------------------------------------- chroma
class ChromaPlan(_PerDevice):
    """kapre_chroma_plan per CUDA device: ``tables``, float64 (n_tables, n_chroma, n_bins) filterbanks (rounded once
    to float32 on upload), optionally the CENS smoothing taps ``smooth`` and the tuning estimate's geometry ``tuning``
    (a dict of ``edges``, ``lo``, ``hi``, ``sample_rate``, ``n_fft`` and ``bins_per_octave``)."""

    def __init__(self, tables, smooth=None, tuning=None, n_chroma=None, n_bins=None):
        if tables is None:
            self.tables = np.zeros((0, int(n_chroma), int(n_bins)))
        else:
            self.tables = np.ascontiguousarray(tables, dtype=np.float64)
        if self.tables.ndim != 3:
            raise ValueError('chroma tables must be (n_tables, n_chroma, n_bins)')
        self.n_tables, self.n_chroma, self.n_bins = self.tables.shape
        self.smooth = None if smooth is None else np.ascontiguousarray(smooth, dtype=np.float64)
        self.tuning = tuning
        self._edges = None
        nres, lo, hi, sr, nfft, bpo = 0, 0, 0, 0.0, 0.0, 0.0
        if tuning is not None:
            self._edges = np.ascontiguousarray(tuning['edges'], dtype=np.float64)
            nres = self._edges.size - 1
            lo, hi = tuning['lo'], tuning['hi']
            sr, nfft, bpo = tuning['sample_rate'], tuning['n_fft'], tuning['bins_per_octave']
        vp = lambda a: None if a is None else a.ctypes.data_as(ctypes.c_void_p)  # noqa: E731
        self.desc = N.ChromaPlanDesc(self.n_chroma, self.n_bins, self.n_tables, vp(self.tables) if self.n_tables
                                     else None, 0 if self.smooth is None else self.smooth.size, vp(self.smooth), nres,
                                     vp(self._edges), lo, hi, sr, nfft, bpo)
        self._per_device = {}

    _destroy = 'kapre_chroma_plan_destroy'

    def _create(self, lib, out):
        return lib.kapre_chroma_plan_create(ctypes.byref(self.desc), out)


def _chroma_input(x, plan: ChromaPlan, data_format, complex_ok):
    """The spectrogram input of a chroma op: (tensor, its SpecDesc, (B, C, M)); its bins must match the plan."""
    if not (isinstance(x, torch.Tensor) and x.is_cuda):
        raise N.KapreNativeError('chroma needs a CUDA spectrogram')
    if x.dim() != 4:
        raise ValueError('chroma expects a 4-D spectrogram batch, got shape %s' % (tuple(x.shape),))
    if x.dtype == torch.complex64 and not complex_ok:
        raise ValueError('this chroma input must be real')
    if x.dtype not in (torch.float32, torch.complex64):
        raise ValueError('chroma expects float32 (or complex64) input, got %s' % (x.dtype,))
    x = _raw(x)
    xd, (B, C, M, K) = _spec_desc(x, data_format)
    if K != plan.n_bins:
        raise ValueError('the chroma filterbank expects %d bins, the input has %d' % (plan.n_bins, K))
    return x, xd, (B, C, M)


def chroma_forward(x, plan: ChromaPlan, cfg, data_format, table=None):
    x, xd, (B, C, M) = _chroma_input(x, plan, data_format, True)
    out, od = _spec_alloc(B, C, M, plan.n_chroma, data_format, torch.float32, x.device)
    if out.numel():
        N.check(N.lib().kapre_chroma(plan.handle(), ctypes.byref(cfg), _ptr(x), ctypes.byref(xd), B, C, M,
                                     _ptr(table) if table is not None else None, _ptr(out), ctypes.byref(od),
                                     _stream_ptr()))
    return out


def chroma_backward(g, x, plan: ChromaPlan, cfg, data_format, table=None):
    x, xd, (B, C, M) = _chroma_input(x, plan, data_format, True)
    g = _raw(g.to(torch.float32))
    gd, _ = _spec_desc(g, data_format)
    gx, gxd = _spec_alloc(B, C, M, plan.n_bins, data_format, x.dtype, x.device)
    if gx.numel():
        N.check(N.lib().kapre_chroma_backward(plan.handle(), ctypes.byref(cfg), _ptr(x), ctypes.byref(xd), B, C, M,
                                              _ptr(table) if table is not None else None, _ptr(g), ctypes.byref(gd),
                                              _ptr(gx), ctypes.byref(gxd), _stream_ptr()))
    return gx


@_device_of_first_arg
def chroma(x, plan: ChromaPlan, in_mode, norm, threshold=None, data_format=_CH_LAST_STR, table=None):
    """Chroma of a CUDA spectrogram batch ``(B, M, K, C)`` / ``(B, C, M, K)`` under ``plan``: float32 ``(B, M,
    n_chroma, C)`` / ``(B, C, M, n_chroma)``.  ``in_mode``: ``N.CHROMA_IN_*`` (the input as it is, squared, or the
    modulus of complex64); ``norm``: ``N.CHROMA_NORM_*``; ``table``: an int32 CUDA tensor of one filterbank index per
    item (else table 0).  One launch.  Differentiable with respect to x; ``table`` is a constant."""
    cfg = N.ChromaCfg(int(in_mode), int(norm), int(threshold is not None),
                      0.0 if threshold is None else float(threshold))
    if _wants_grad(x):
        from . import autograd
        return autograd.chroma(x, plan, cfg, data_format, table)
    return chroma_forward(x, plan, cfg, data_format, table)


@_device_of_first_arg
def chroma_cens(x, plan: ChromaPlan, in_mode, data_format=_CH_LAST_STR):
    """CENS of a CUDA spectrogram batch under a plan with smoothing taps: the L1-normalised chroma (threshold 0)
    quantised, smoothed along time and L2-normalised.  Two launches.  No gradient: the output carries no
    ``grad_fn``."""
    x, xd, (B, C, M) = _chroma_input(x.detach(), plan, data_format, True)
    out, od = _spec_alloc(B, C, M, plan.n_chroma, data_format, torch.float32, x.device)
    if out.numel():
        ws = _scratch(N.lib().kapre_chroma_cens_workspace_bytes(plan.handle(), B, C, M), x.device)
        N.check(N.lib().kapre_chroma_cens(plan.handle(), int(in_mode), _ptr(x), ctypes.byref(xd), B, C, M, _ptr(out),
                                          ctypes.byref(od), _ptr(ws), _stream_ptr()))
    return out


@_device_of_first_arg
def chroma_tuning(x, plan: ChromaPlan, in_mode, data_format=_CH_LAST_STR):
    """librosa's ``estimate_tuning`` per item of a CUDA spectrogram batch (power with ``N.CHROMA_IN_SQUARE`` of a
    magnitude, or as given with ``N.CHROMA_IN_LINEAR``): ``(tuning, table)``, a float64 ``(B,)`` tensor and the int32
    index of each item's filterbank table.  Seven launches; nothing is read back to the host.  No gradient."""
    x, xd, (B, C, M) = _chroma_input(x.detach(), plan, data_format, False)
    tuning = torch.empty(B, dtype=torch.float64, device=x.device)
    table = torch.empty(B, dtype=torch.int32, device=x.device)
    if B:
        ws = _scratch(N.lib().kapre_chroma_tuning_workspace_bytes(plan.handle(), B, C, M), x.device)
        N.check(N.lib().kapre_chroma_tuning(plan.handle(), int(in_mode), _ptr(x), ctypes.byref(xd), B, C, M,
                                            _ptr(tuning), _ptr(table), _ptr(ws), _stream_ptr()))
    return tuning, table


# ------------------------------------------------------------------------------- harmonic/percussive separation
def _hpss_pair(v, name):
    if isinstance(v, (tuple, list)):
        if len(v) != 2:
            raise ValueError('%s must be a number or a pair, got %r' % (name, v))
        return v[0], v[1]
    return v, v


def hpss_config(kernel_size=31, power=2.0, mask=False, margin=1.0):
    """The ``kapre_hpss_config`` of ``hpss``'s arguments; a bad argument raises ``ValueError`` here, before any launch.
    ``kernel_size`` and ``margin``: a number or a pair (harmonic, percussive)."""
    kh, kp = _hpss_pair(kernel_size, 'kernel_size')
    for k in (kh, kp):
        if isinstance(k, (bool, np.bool_)) or not isinstance(k, (int, np.integer)) or not 1 <= k <= N.HPSS_MAX_KERNEL:
            raise ValueError('kernel_size must be integers in [1, %d], got %r' % (N.HPSS_MAX_KERNEL, kernel_size))
    mh, mp = _hpss_pair(margin, 'margin')
    for m in (mh, mp):
        if isinstance(m, (bool, np.bool_)) or not isinstance(m, (int, float, np.integer, np.floating)) \
                or not np.isfinite(float(m)) or not float(m) >= 1.0:
            raise ValueError('margin must be finite and >= 1, got %r' % (margin,))
    if isinstance(power, (bool, np.bool_)) or not isinstance(power, (int, float, np.integer, np.floating)) \
            or not float(power) > 0.0:
        raise ValueError('power must be > 0 (inf allowed), got %r' % (power,))
    return N.HpssCfg(int(kh), int(kp), float(power), float(mh), float(mp), int(bool(mask)))


def _hpss_input(S, data_format):
    if not isinstance(S, torch.Tensor):
        raise ValueError('hpss expects a torch tensor, got %s' % (type(S).__name__,))
    if S.dim() != 4:
        raise ValueError('hpss expects a 4-D spectrogram batch, got shape %s' % (tuple(S.shape),))
    if S.dtype not in (torch.float32, torch.complex64):
        raise ValueError('hpss expects float32 or complex64 input, got %s' % (S.dtype,))
    if not S.is_cuda:
        raise ValueError('hpss needs a CUDA spectrogram')
    S = _raw(S)
    sd, dims = _spec_desc(S, data_format)
    return S, sd, dims


def hpss_forward(S, cfg, data_format, want_h=True, want_p=True):
    """(harmonic, percussive) of ``kapre_hpss`` (None for a component not wanted).  One launch."""
    S, sd, (B, C, T, K) = _hpss_input(S, data_format)
    dt = torch.float32 if cfg.mask else S.dtype
    outs, descs = [None, None], [None, None]
    for i, want in enumerate((want_h, want_p)):
        if want:
            outs[i], descs[i] = _spec_alloc(B, C, T, K, data_format, dt, S.device)
    if S.numel():
        N.check(N.lib().kapre_hpss(ctypes.byref(cfg), _ptr(S), int(S.is_complex()), ctypes.byref(sd), B, C, T, K,
                                   _ptr(outs[0]) if want_h else None, ctypes.byref(descs[0]) if want_h else None,
                                   _ptr(outs[1]) if want_p else None, ctypes.byref(descs[1]) if want_p else None,
                                   _stream_ptr()))
    return outs[0], outs[1]


def hpss_backward(gh, gp, S, cfg, data_format):
    """Gradient of ``hpss_forward`` with respect to S given its outputs' gradients (either may be None).  Two
    launches over a workspace of ``kapre_hpss_workspace_bytes``."""
    S, sd, (B, C, T, K) = _hpss_input(S, data_format)
    gdt = torch.float32 if cfg.mask else S.dtype
    gs = [None, None]
    ds = [None, None]
    for i, g in enumerate((gh, gp)):
        if g is not None:
            gs[i] = _raw(g.to(gdt))
            ds[i], _ = _spec_desc(gs[i], data_format)
    gS, gSd = _spec_alloc(B, C, T, K, data_format, S.dtype, S.device)
    if gS.numel():
        ws = _scratch(N.lib().kapre_hpss_workspace_bytes(B, C, T, K), S.device)
        N.check(N.lib().kapre_hpss_backward(ctypes.byref(cfg), _ptr(S), int(S.is_complex()), ctypes.byref(sd), B, C, T,
                                            K, _ptr(gs[0]) if gs[0] is not None else None,
                                            ctypes.byref(ds[0]) if gs[0] is not None else None,
                                            _ptr(gs[1]) if gs[1] is not None else None,
                                            ctypes.byref(ds[1]) if gs[1] is not None else None,
                                            _ptr(gS), ctypes.byref(gSd), _ptr(ws), _stream_ptr()))
    return gS


@_device_of_first_arg
def hpss(S, cfg, data_format=_CH_LAST_STR, want_h=True, want_p=True):
    """Harmonic/percussive separation of a CUDA spectrogram batch ``(B, T, K, C)`` / ``(B, C, T, K)`` (float32
    magnitudes or complex64) under ``cfg`` (``hpss_config``): ``(harmonic, percussive)``, None for a component not
    wanted.  One launch.  Differentiable with respect to S."""
    if _wants_grad(S):
        from . import autograd
        return autograd.hpss(S, cfg, data_format, want_h, want_p)
    return hpss_forward(S, cfg, data_format, want_h, want_p)


# ------------------------------------------------------------------------------- onsets, tempo and beats
def _check_int(name, v, lo, hi=None):
    if isinstance(v, (bool, np.bool_)) or not isinstance(v, (int, np.integer)) or v < lo or (hi is not None and v > hi):
        raise ValueError('%s must be an integer in [%d, %s], got %r' % (name, lo, 'inf' if hi is None else hi, v))
    return int(v)


def _frames_desc(t: torch.Tensor, data_format: str):
    """(B, T, C) channels_last or (B, C, T) channels_first -> kapre_frames_desc, (B, C, T)."""
    if t.dim() != 3:
        raise ValueError('expected a 3-D (batch, frames, ch) / (batch, ch, frames) tensor, got shape %s'
                         % (tuple(t.shape),))
    if data_format == _CH_LAST_STR:
        B, T, C = t.shape
        sb, st, sc = t.stride()
    else:
        B, C, T = t.shape
        sb, sc, st = t.stride()
    return N.FramesDesc(sb, sc, st), (B, C, T)


def _envelope_input(e, name, data_format):
    if not (isinstance(e, torch.Tensor) and e.is_cuda):
        raise N.KapreNativeError('%s needs a CUDA tensor' % name)
    if e.dtype != torch.float32:
        raise ValueError('%s expects float32, got %s' % (name, e.dtype))
    e = _raw(e.detach())
    ed, dims = _frames_desc(e, data_format)
    return e, ed, dims


def onset_config(lag=1, max_size=1, aggregate='mean', pad_frames=0):
    """The ``kapre_onset_config`` of ``onset_strength``'s arguments; a bad one raises ``ValueError`` here."""
    lag = _check_int('lag', lag, 1)
    max_size = _check_int('max_size', max_size, 1)
    if aggregate not in ('mean', 'median'):
        raise ValueError("aggregate must be 'mean' or 'median', got %r" % (aggregate,))
    pad_frames = _check_int('pad_frames', pad_frames, 0, 1 << 28)
    return N.OnsetCfg(lag, max_size, N.ONSET_MEAN if aggregate == 'mean' else N.ONSET_MEDIAN, pad_frames)


def _onset_input(S, cfg, data_format):
    if not (isinstance(S, torch.Tensor) and S.is_cuda):
        raise N.KapreNativeError('onset_strength needs a CUDA spectrogram')
    if S.dtype != torch.float32:
        raise ValueError('onset_strength expects a float32 spectrogram, got %s' % (S.dtype,))
    S = _raw(S.detach())
    sd, (B, C, T, K) = _spec_desc(S, data_format)
    onset_limits(cfg, K, T)
    return S, sd, (B, C, T, K)


def onset_limits(cfg, K, T):
    """The limits of ``kapre_onset_strength`` for K bins and T frames; raises ``ValueError``."""
    if not 1 <= K <= N.ONSET_MAX_BINS:
        raise ValueError('onset_strength supports 1 to %d bins, got %d' % (N.ONSET_MAX_BINS, K))
    if cfg.max_size > K:
        raise ValueError('max_size (%d) must not exceed the %d bins' % (cfg.max_size, K))
    if T and cfg.lag >= T:
        raise ValueError('lag (%d) must be below the %d frames' % (cfg.lag, T))


def onset_strength_forward(S, cfg, data_format):
    """The envelope ``(B, T, C)`` / ``(B, C, T)`` of ``kapre_onset_strength``: one launch."""
    S, sd, (B, C, T, K) = _onset_input(S, cfg, data_format)
    out, od = _frames_alloc(B, C, T, data_format, torch.float32, S.device)
    if out.numel():
        N.check(N.lib().kapre_onset_strength(ctypes.byref(cfg), _ptr(S), ctypes.byref(sd), B, C, T, K, _ptr(out),
                                             ctypes.byref(od), _stream_ptr()))
    return out


def onset_strength_backward(g, S, cfg, data_format):
    """Gradient of ``onset_strength_forward`` with respect to S: two launches over a workspace of 8 bytes per
    element."""
    S, sd, (B, C, T, K) = _onset_input(S, cfg, data_format)
    g = _raw(g.to(torch.float32))
    gd, _ = _frames_desc(g, data_format)
    gS, gSd = _spec_alloc(B, C, T, K, data_format, torch.float32, S.device)
    if gS.numel():
        ws = _scratch(N.lib().kapre_onset_strength_workspace_bytes(B, C, T, K), S.device)
        N.check(N.lib().kapre_onset_strength_backward(ctypes.byref(cfg), _ptr(S), ctypes.byref(sd), B, C, T, K,
                                                      _ptr(g), ctypes.byref(gd), _ptr(gS), ctypes.byref(gSd),
                                                      _ptr(ws), _stream_ptr()))
    return gS


@_device_of_first_arg
def onset_strength(S, cfg, data_format=_CH_LAST_STR):
    """Onset strength envelope of a float32 CUDA spectrogram ``(B, T, K, C)`` / ``(B, C, T, K)`` under ``cfg``
    (``onset_config``).  One launch; differentiable with respect to S."""
    _onset_input(S, cfg, data_format)
    if _wants_grad(S):
        from . import autograd
        return autograd.onset_strength(S, cfg, data_format)
    return onset_strength_forward(S, cfg, data_format)


def tempogram_check(win_length, frames=None, center=True):
    win_length = _check_int('win_length', win_length, 2, N.TEMPOGRAM_MAX_WIN)
    if not center and frames is not None and frames < win_length:
        raise ValueError('without center the envelope needs at least win_length=%d frames, got %d'
                         % (win_length, frames))
    return win_length


@_device_of_first_arg
def tempogram(e, win_length=384, center=True, norm_inf=True, data_format=_CH_LAST_STR):
    """Autocorrelation tempogram of a float32 CUDA envelope ``(B, T, C)`` / ``(B, C, T)``: ``(B, frames, W, C)`` /
    ``(B, C, frames, W)`` float32.  One launch; no gradient (an input that requires grad under grad mode raises)."""
    if _wants_grad(e):
        raise ValueError('tempogram has no gradient: call it under torch.no_grad() or on a detached envelope')
    e, ed, (B, C, T) = _envelope_input(e, 'tempogram', data_format)
    W = tempogram_check(win_length, T, center)
    n_out = T if center else T - W + 1
    out, od = _spec_alloc(B, C, n_out, W, data_format, torch.float32, e.device)
    if out.numel():
        N.check(N.lib().kapre_tempogram(_ptr(e), ctypes.byref(ed), B, C, T, W, int(bool(center)), int(bool(norm_inf)),
                                        _ptr(out), ctypes.byref(od), _stream_ptr()))
    return out


class TempoPlan:
    """The float64 log-prior over the lags of one tempo configuration, built on the host and kept per device."""

    def __init__(self, win_length, sample_rate, hop_length, start_bpm=120.0, std_bpm=1.0, max_tempo=320.0):
        self.W = tempogram_check(win_length)
        self.bpm_scale = 60.0 * float(sample_rate) / float(hop_length)
        lags = np.arange(self.W, dtype=np.float64)
        with np.errstate(divide='ignore'):
            bpm = self.bpm_scale / lags
            prior = -0.5 * ((np.log2(bpm) - np.log2(float(start_bpm))) / float(std_bpm)) ** 2
        if max_tempo is not None:
            prior[:int(np.argmax(bpm < float(max_tempo)))] = -np.inf
        prior[0] = -np.inf
        self.logprior = prior
        self._per_device = {}

    def table(self, device):
        t = self._per_device.get(device)
        if t is None:
            t = torch.from_numpy(self.logprior).to(device)
            self._per_device[device] = t
        return t


@_device_of_first_arg
def tempo(tg, plan: TempoPlan, per_frame=False, data_format=_CH_LAST_STR):
    """Tempo (bpm) from a float32 CUDA tempogram ``(B, frames, W, C)`` / ``(B, C, frames, W)``: ``(B, C)``, or per
    frame ``(B, frames, C)`` / ``(B, C, frames)``.  Two launches (one per frame); no gradient."""
    if not (isinstance(tg, torch.Tensor) and tg.is_cuda):
        raise N.KapreNativeError('tempo needs a CUDA tempogram')
    if tg.dtype != torch.float32:
        raise ValueError('tempo expects a float32 tempogram, got %s' % (tg.dtype,))
    tg = _raw(tg.detach())
    gd, (B, C, T, W) = _spec_desc(tg, data_format)
    if W != plan.W:
        raise ValueError('the tempogram has %d lags, the plan %d' % (W, plan.W))
    if not per_frame and B * C and T < 1:
        raise ValueError('tempo needs at least one frame')
    if per_frame:
        out, od = _frames_alloc(B, C, T, data_format, torch.float32, tg.device)
    else:
        out, od = torch.empty((B, C), dtype=torch.float32, device=tg.device), None
    if out.numel():
        ws = None
        if not per_frame:
            ws = _scratch(N.lib().kapre_tempo_workspace_bytes(B, C, T, W), tg.device)
        N.check(N.lib().kapre_tempo(_ptr(tg), ctypes.byref(gd), B, C, T, W, _ptr(plan.table(tg.device)),
                                    ctypes.c_double(plan.bpm_scale), int(bool(per_frame)), _ptr(out),
                                    ctypes.byref(od) if od is not None else None,
                                    _ptr(ws) if ws is not None else None, _stream_ptr()))
    return out


def onset_detect_config(pre_max, post_max, pre_avg, post_avg, wait, delta, normalize):
    args = (('pre_max', pre_max, 0), ('post_max', post_max, 1), ('pre_avg', pre_avg, 0), ('post_avg', post_avg, 1),
            ('wait', wait, 0))
    vals = [_check_int(n, v, lo, N.PEAK_MAX_WINDOW) for n, v, lo in args]
    if isinstance(delta, (bool, np.bool_)) or not np.isfinite(float(delta)):
        raise ValueError('delta must be a finite number, got %r' % (delta,))
    return N.OnsetDetectCfg(*vals, int(bool(normalize)), float(delta))


@_device_of_first_arg
def onset_detect(e, cfg, data_format=_CH_LAST_STR):
    """Onset mask (bool, the envelope's shape) of a float32 CUDA envelope under ``cfg`` (``onset_detect_config``).
    One launch."""
    e, ed, (B, C, T) = _envelope_input(e, 'onset_detect', data_format)
    mask, md = _frames_alloc(B, C, T, data_format, torch.bool, e.device)
    if mask.numel():
        N.check(N.lib().kapre_onset_detect(_ptr(e), ctypes.byref(ed), B, C, T, ctypes.byref(cfg), _ptr(mask),
                                           ctypes.byref(md), _stream_ptr()))
    return mask


def beat_config(sample_rate, hop_length, tightness, trim):
    fps = float(sample_rate) / float(hop_length)
    if not (np.isfinite(fps) and fps > 0):
        raise ValueError('sample_rate / hop_length must be positive, got %r / %r' % (sample_rate, hop_length))
    if isinstance(tightness, (bool, np.bool_)) or not (np.isfinite(float(tightness)) and float(tightness) > 0):
        raise ValueError('tightness must be positive, got %r' % (tightness,))
    return N.BeatCfg(fps, float(tightness), int(bool(trim)))


@_device_of_first_arg
def beat_track(e, cfg, bpm, data_format=_CH_LAST_STR):
    """(tempo (B, C) float32, beat mask (bool, the envelope's shape)) of a float32 CUDA envelope under ``cfg``
    (``beat_config``); ``bpm`` is a float for every row or a ``(B, C)`` float32 CUDA tensor.  One launch over a
    workspace of 24 bytes per frame."""
    e, ed, (B, C, T) = _envelope_input(e, 'beat_track', data_format)
    bpm_t, bpm_v = None, 0.0
    if isinstance(bpm, torch.Tensor):
        if bpm.shape != (B, C) or bpm.dtype != torch.float32 or bpm.device != e.device:
            raise ValueError('bpm must be a (%d, %d) float32 tensor on %s' % (B, C, e.device))
        bpm_t = bpm.detach().contiguous()
    else:
        bpm_v = float(bpm)
        p = np.rint(60.0 * cfg.fps / bpm_v) if bpm_v > 0 and np.isfinite(bpm_v) else 0
        if not 1 <= p <= N.BEAT_MAX_PERIOD:
            raise ValueError('bpm=%r gives a beat period of %r frames, outside [1, %d]'
                             % (bpm, p, N.BEAT_MAX_PERIOD))
    tempo_out = torch.empty((B, C), dtype=torch.float32, device=e.device)
    mask, md = _frames_alloc(B, C, T, data_format, torch.bool, e.device)
    if B * C and T < 1:
        raise ValueError('beat_track needs at least one frame')
    if tempo_out.numel():
        ws = _scratch(N.lib().kapre_beat_track_workspace_bytes(B, C, T), e.device)
        N.check(N.lib().kapre_beat_track(_ptr(e), ctypes.byref(ed), B, C, T, ctypes.byref(cfg),
                                         _ptr(bpm_t) if bpm_t is not None else None, ctypes.c_float(bpm_v),
                                         _ptr(tempo_out), _ptr(mask), ctypes.byref(md), _ptr(ws), _stream_ptr()))
    return tempo_out, mask
