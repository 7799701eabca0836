"""Float64 restatement of the phase-vocoder time stretch (``kapre_b200/csrc/ts_core.cuh``), differentiable with torch
autograd, on canonical (B, C, T, F) complex tensors.

Output frame u of T' = ceil(T / rate) reads frames k = floor(u rate) and k + 1 (zeros past T), alpha = u rate - k:
    m[u] = alpha |X[k + 1]| + (1 - alpha) |X[k]|,   phi[u] = angle(X[0]) + sum_{v < u} (angle(X[k_v + 1]) - angle(X[k_v]))
and Y = m exp(i phi).  This is torchaudio.functional.phase_vocoder modulo 2 pi for any phase_advance (the wrapped
advance cancels), with u rate formed as one float64 product.
"""
import math

import torch


def steps(T, rate):
    """(k, alpha) for the ceil(T / rate) output frames: k int64, alpha float64."""
    n = math.ceil(T / rate)
    ts = torch.arange(n, dtype=torch.float64) * rate
    k = torch.floor(ts)
    return k.long(), ts - k


def _frames(X, T, rate):
    k, alpha = steps(T, rate)
    B, C, _, F = X.shape
    Xp = torch.cat([X, torch.zeros((B, C, 2, F), dtype=X.dtype)], dim=2)
    return Xp[:, :, k], Xp[:, :, k + 1], alpha.to(X.real.dtype).view(1, 1, -1, 1)


def phases(X, rate, dtype=torch.complex128):
    """(m, phi): the magnitudes and the unwrapped phases of the stretched frames, (B, C, T', F), computed in
    ``dtype`` (complex64 gives the float32 twin the tests measure rounding drift with)."""
    X = X.to(dtype)
    T = X.shape[2]
    X0, X1, alpha = _frames(X, T, rate)
    m = alpha * X1.abs() + (1 - alpha) * X0.abs()
    d = X1.angle() - X0.angle()
    if d.shape[2] == 0:
        return m, d
    phi = X[:, :, :1].angle() + torch.cat([torch.zeros_like(d[:, :, :1]), torch.cumsum(d, dim=2)[:, :, :-1]], dim=2)
    return m, phi


def time_stretch(X, rate, dtype=torch.complex128):
    """The stretched spectrogram; differentiable in X.  rate == 1 returns X."""
    if rate == 1.0:
        return X
    m, phi = phases(X, rate, dtype)
    return torch.polar(m, phi)


def torchaudio_layout(X):
    """(B, C, T, F) -> torchaudio's (B, C, F, T) and back (the same transpose)."""
    return X.transpose(-1, -2)
