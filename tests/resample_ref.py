"""Float64 restatement of the polyphase resampler (``scipy.signal.resample_poly`` with its defaults), in torch so that
autograd gives its exact vector-Jacobian product.  Needs no scipy: the tests pin it to scipy where scipy exists.

    M = max(up, down), hl = 10 M, h = Kaiser(beta 5)-windowed sinc((k - hl) / M) / M normalised to unit sum
    y[n] = up * sum_i x[i] h[hl + n down - i up],   n < ceil(L up / down), terms outside h or the signal are zero
"""
import math

import numpy as np
import torch

RATES = (8000, 11025, 16000, 22050, 24000, 32000, 44100, 48000, 88200, 96000)
COMMON_PAIRS = ((48000, 16000), (44100, 22050), (44100, 16000), (16000, 22050), (8000, 11025), (11025, 32000),
                (32000, 11025))


def up_down(orig, target):
    g = math.gcd(orig, target)
    return target // g, orig // g


def taps(up, down):
    """h in float64 (the library rounds the same formula to float32)."""
    M = max(up, down)
    hl = 10 * M
    n = 2 * hl + 1
    k = np.arange(n, dtype=np.float64)
    h = np.sinc((k - hl) / M) / M * np.kaiser(n, 5.0)
    return h / h.sum()


def output_length(length, up, down):
    return -(-length * up // down)


def resample(x, up, down, h=None, length=None, chunk=1 << 16):
    """x: float64 tensor (..., L), resampled along the last axis to ``length`` (default ceil(L up / down)) samples."""
    h = torch.as_tensor(taps(up, down) if h is None else h, dtype=torch.float64)
    hl = (h.numel() - 1) // 2
    L = x.shape[-1]
    Lo = output_length(L, up, down) if length is None else int(length)
    K = 2 * (hl // up) + 2
    xp = torch.cat([x, torch.zeros(x.shape[:-1] + (1,), dtype=x.dtype)], dim=-1)     # index L reads zero
    outs = []
    for n0 in range(0, Lo, chunk):
        n = torch.arange(n0, min(Lo, n0 + chunk), dtype=torch.int64)
        t = n * down
        i = (-((hl - t) // up))[:, None] + torch.arange(K)[None, :]       # i >= ceil((t - hl) / up)
        off = hl + t[:, None] - i * up                                      # index into h
        ok = (off >= 0) & (off <= 2 * hl) & (i >= 0) & (i < L)
        w = torch.where(ok, up * h[off.clamp(0, 2 * hl)], torch.zeros((), dtype=torch.float64))
        idx = torch.where(ok, i, torch.full_like(i, L))
        outs.append((xp[..., idx] * w).sum(-1))
    if not outs:
        return x.new_zeros(x.shape[:-1] + (0,))
    return torch.cat(outs, dim=-1)
