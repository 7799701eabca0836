"""Float64 torch restatement of the five hot-path layers, differentiable by torch autograd.

Test infrastructure for the gradient tests: built from ``oracle.reference``'s windows, dual windows, filterbank
conventions and frame counts; ``test_grad_emu.py`` pins its forward to ``oracle.reference``.  The decibel layer
uses ``clamp_min`` and ``where``/``amax`` so that autograd applies TensorFlow's tie rules (``torch.maximum`` would
split the gradient of ties): ``tf.maximum(a, b)`` passes the gradient to ``a`` where ``a >= b``, and
``reduce_max`` splits it equally among tied maxima.
"""
import numpy as np
import torch

from oracle import reference as ref

CL, CF = 'channels_last', 'channels_first'


def _t(a):
    return torch.as_tensor(np.asarray(a, dtype=np.float64))


def stft(x, n_fft, win_length, hop, window_name=None, pad_begin=False, pad_end=False, in_fmt=CF, out_fmt=CF):
    """x: (B, L, C) / (B, C, L) float64 tensor -> complex128 (B, T, F, C) / (B, C, T, F)."""
    if in_fmt == CL:
        x = x.transpose(1, 2)
    if pad_begin:
        x = torch.nn.functional.pad(x, (n_fft - hop, 0))
    L = x.shape[-1]
    T = ref.num_frames(L, win_length, hop, pad_end)
    need = (T - 1) * hop + win_length if T > 0 else 0
    if need > L:
        x = torch.nn.functional.pad(x, (0, need - L))
    idx = torch.arange(T)[:, None] * hop + torch.arange(win_length)[None, :]
    frames = x[..., idx] * _t(ref.get_window(window_name, win_length))
    s = torch.fft.rfft(frames, n=n_fft, dim=-1)
    return s.permute(0, 2, 3, 1) if out_fmt == CL else s


def istft(X, n_fft, win_length, hop, forward_window_name=None, in_fmt=CF, out_fmt=CF):
    """complex (B, T, F, C) / (B, C, T, F) -> float64 (B, L, C) / (B, C, L), L = (T-1) hop + win_length."""
    if in_fmt == CL:
        X = X.permute(0, 3, 1, 2)
    T = X.shape[2]
    fr = torch.fft.irfft(X, n=n_fft, dim=-1)
    fr = fr[..., :win_length] if n_fft >= win_length else torch.nn.functional.pad(fr, (0, win_length - n_fft))
    dual = ref.inverse_stft_window(win_length, hop, ref.get_window(forward_window_name, win_length))
    fr = fr * _t(dual)
    out_len = (T - 1) * hop + win_length if T > 0 else 0
    out = fr.new_zeros(fr.shape[:2] + (out_len,))
    for t in range(T):
        out = out.index_add(2, torch.arange(t * hop, t * hop + win_length), fr[:, :, t])
    return out.transpose(1, 2) if out_fmt == CL else out


def magnitude(X):
    return X.abs()


def apply_filterbank(x, fb, data_format=CF):
    fb = _t(fb)
    if data_format == CF:
        return torch.tensordot(x, fb, dims=([3], [0]))
    return torch.tensordot(x, fb, dims=([2], [0])).permute(0, 1, 3, 2)


def magnitude_to_decibel(x, ref_value=1.0, amin=1e-5, dynamic_range=80.0):
    log_spec = 10.0 * torch.log10(x.clamp_min(amin)) - 10.0 * np.log10(max(amin, ref_value))
    dims = tuple(range(1, x.dim())) if x.dim() > 1 else tuple(range(x.dim()))
    thr = log_spec.amax(dim=dims, keepdim=True) - dynamic_range
    return torch.where(log_spec >= thr, log_spec, thr)


def filterbank_mel(n_fft, sample_rate, n_mels, **kw):
    return ref.filterbank_mel(sample_rate, n_fft // 2 + 1, n_mels, **kw)


def filterbank_log(n_fft, sample_rate, n_bins=84, **kw):
    return ref.filterbank_log(sample_rate, n_fft // 2 + 1, n_bins, **kw)


def vjp(fn, x, g):
    """(fn(x), d<fn(x), g>/dx) in float64 / complex128, PyTorch's complex convention."""
    x = x.detach().clone().requires_grad_(True)
    y = fn(x)
    (gx,) = torch.autograd.grad(y, x, grad_outputs=g.to(y.dtype))
    return y.detach(), gx
