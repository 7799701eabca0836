"""Float64 restatement of per-channel energy normalisation (PCEN) in torch, independent of the CUDA code.

``E`` is a (batch, ch, time, band) tensor.  Each parameter is a scalar, a per-band (band,) tensor, or a tensor of
E's full shape (then every element has its own copy, so autograd returns each element's contribution to the
parameter's gradient).  Gradients come from torch autograd on these formulas.
"""
import math

import torch


def smooth_coef(time_constant, sample_rate, hop_length):
    """librosa's ``b`` from a time constant: the pole of a one-pole filter whose step response takes
    ``time_constant`` seconds (``t_frames`` frames) to settle."""
    t = time_constant * sample_rate / hop_length
    return (math.sqrt(1.0 + 4.0 * t * t) - 1.0) / (2.0 * t * t)


def smoother(E, s):
    """M[-1] = E[0], M[t] = (1 - s) M[t-1] + s E[t] along axis 2; returns M (same shape as E)."""
    s = torch.as_tensor(s, dtype=E.dtype)
    T = E.shape[2]
    if T == 0:
        return E.clone()
    # unbind once: indexing frame by frame would make autograd build a full-size gradient for every frame
    Et = E.unbind(2)
    st = s.unbind(2) if s.dim() == 4 else [s] * T
    out = []
    m = Et[0]
    for t in range(T):
        m = (1 - st[t]) * m + st[t] * Et[t]
        out.append(m)
    return torch.stack(out, dim=2)


def pcen(E, gain=0.98, bias=2.0, power=0.5, smooth=0.0564, eps=1e-6, return_M=False):
    """y = d^r expm1(r log1p(u / d)), u = E exp(-a log(eps + M)) with a = gain, d = bias, r = power."""
    a, d, r = (torch.as_tensor(v, dtype=E.dtype) for v in (gain, bias, power))
    M = smoother(E, smooth)
    u = E * torch.exp(-a * torch.log(eps + M))
    y = d ** r * torch.expm1(r * torch.log1p(u / d))
    return (y, M) if return_M else y


def pcen_naive(E, gain=0.98, bias=2.0, power=0.5, smooth=0.0564, eps=1e-6):
    """The textbook form (E / (eps + M)^a + d)^r - d^r, which cancels when u << d."""
    M = smoother(E, smooth)
    return (E / (eps + M) ** gain + bias) ** power - bias ** power


def grads(E, params, gy, eps=1e-6):
    """(gE, [g_gain, g_bias, g_power, g_smooth], [scale_gain, ...]) in float64 for output gradient ``gy``.

    ``params``: four scalars or (band,) arrays.  Each parameter gradient has the parameter's shape; its scale is
    the sum of the absolute per-element contributions, which bounds the float32 rounding of the sum whatever
    cancellation happens inside it."""
    E = E.detach().double().requires_grad_()
    full = [torch.as_tensor(p, dtype=torch.float64).expand(E.shape).clone().requires_grad_() for p in params]
    y = pcen(E, *full, eps=eps)
    gs = torch.autograd.grad(y, [E] + full, gy.double(), allow_unused=True, materialize_grads=True)
    gE, contrib = gs[0], gs[1:]
    out, scale = [], []
    for p, c in zip(params, contrib):
        per_band = torch.as_tensor(p).dim() == 1
        dims = (0, 1, 2) if per_band else (0, 1, 2, 3)
        out.append(c.sum(dims))
        scale.append(c.abs().sum(dims))
    return gE, out, scale
