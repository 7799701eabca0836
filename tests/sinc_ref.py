"""Float64 restatement of the band-limited interpolator (``kapre_b200/csrc/sinc_core.cuh``) with the exact filter (no
table), in torch so that autograd gives its vector-Jacobian product, plus the explicit matrix for the adjoint and the
``PitchShift`` chain built from it.  Needs no scipy.

    h(u) = sinc(u) I0(5 sqrt(1 - (u / Z)^2)) / I0(5) for |u| < Z = 10, else 0;    I = integral of h over [-Z, Z]
    y[m] = (gain / I) sum_j x[j] h(s (offset + m step - j)),   x[j] = 0 outside [0, L)
    forward of ratio rho: step = 1 / rho, s = gain = min(1, rho)
"""
import math

import numpy as np
import torch

Z, BETA, Q = 10, 5.0, 1024
CL, CF = 'channels_last', 'channels_first'


def h(u):
    u = np.asarray(u, dtype=np.float64)
    a = np.abs(u) / Z
    w = np.i0(BETA * np.sqrt(np.clip(1.0 - a * a, 0.0, None))) / np.i0(BETA)
    return np.where(a < 1.0, np.sinc(u) * w, 0.0)


def _simpson(f, n_per_unit):
    n = Z * n_per_unit
    v = f(np.arange(n + 1, dtype=np.float64) / n_per_unit)
    return 2.0 * (v[0] + v[-1] + 4.0 * v[1:-1:2].sum() + 2.0 * v[2:-1:2].sum()) / (3.0 * n_per_unit)


INTEGRAL = _simpson(h, 1 << 13)                          # I
L1 = _simpson(lambda u: np.abs(h(u)), 1 << 13)           # integral of |h|


def numbers(ratio, offset=0.0):
    """(step, offset, s, gain) of the forward sum."""
    s = min(1.0, float(ratio))
    return 1.0 / float(ratio), float(offset), s, s


def output_length(length, ratio):
    return math.ceil(length * ratio)


def _weights(m, L, step, offset, s, gain):
    """(j, w): input indices (len(m), K) and their float64 weights, zero where j is outside [0, L)."""
    pos = offset + m.astype(np.float64) * step
    half = math.ceil(Z / s) + 1
    j = np.floor(pos).astype(np.int64)[:, None] + np.arange(-half + 1, half + 1)[None, :]
    w = (gain / INTEGRAL) * h(s * (pos[:, None] - j))
    ok = (j >= 0) & (j < L)
    return np.where(ok, j, L), np.where(ok, w, 0.0)


def resample(x, ratio, length=None, offset=0.0, chunk=1 << 13, _numbers=None):
    """x: float64 tensor (..., L) -> (..., length) along the last axis (default ceil(L ratio)); differentiable in x."""
    step, offset, s, gain = numbers(ratio, offset) if _numbers is None else _numbers
    L = x.shape[-1]
    Lo = output_length(L, ratio) if length is None else int(length)
    xp = torch.cat([x, torch.zeros(x.shape[:-1] + (1,), dtype=x.dtype)], dim=-1)     # index L reads zero
    outs = []
    for m0 in range(0, Lo, chunk):
        j, w = _weights(np.arange(m0, min(Lo, m0 + chunk)), L, step, offset, s, gain)
        outs.append((xp[..., torch.from_numpy(j)] * torch.from_numpy(w)).sum(-1))
    if not outs:
        return x.new_zeros(x.shape[:-1] + (0,))
    return torch.cat(outs, dim=-1)


def matrix(L, ratio, length, offset=0.0):
    """The dense (length, L) float64 matrix A of ``resample``: y = A x.  Its transpose is the adjoint."""
    step, offset, s, gain = numbers(ratio, offset)
    A = np.zeros((length, L + 1))
    j, w = _weights(np.arange(length), L, step, offset, s, gain)
    np.add.at(A, (np.arange(length)[:, None].repeat(j.shape[1], 1), j), w)
    return A[:, :L]


def adjoint_numbers(ratio, offset=0.0):
    """(step, offset, s, gain) with which the same sum, run over the output gradient, gives A^T g (h is even)."""
    step, offset, s, gain = numbers(ratio, offset)
    return float(ratio), -offset * float(ratio), s / float(ratio), gain


def error_bound(ratio, adjoint=False):
    """Bound on |kernel output - restatement| per unit of max|x|, from the three error sources of sinc_core.cuh:
    linear interpolation of the table (max|h''| / (8 Q^2) per tap), the float32 table position (2e-7 per tap) and
    float32 accumulation (one rounding of a partial sum <= gain / I * L1 / s per tap of a wing, plus the product, the
    final sum and the scale)."""
    _, _, s, gain = adjoint_numbers(ratio) if adjoint else numbers(ratio)
    taps = 2 * math.ceil(Z / s)
    d2 = np.abs(np.diff(h(np.arange(-4096, 4097) / 4096.0), 2)).max() * 4096.0 ** 2          # max|h''|, at u = 0
    per_tap = d2 / (8.0 * Q * Q) + 2e-7
    partial = gain / INTEGRAL * L1 / s
    return gain / INTEGRAL * taps * per_tap + (taps / 2 + 4) * 2.0 ** -24 * partial


# ---------------------------------------------------------------------------------------------- the PitchShift chain
def pitch_shift_offset(rate, n_fft, win_length, hop):
    """Position of output sample 0 in the untrimmed inverse STFT of the stretched frames.  Input sample t sits at the
    centre of the (fractional) frame k = (t + pad_left - win / 2) / hop, pad_left = n_fft - hop being what pad_begin
    prepends; the stretch maps frame k to frame k / rate, whose centre the inverse puts at k / rate * hop + win / 2."""
    return win_length / 2.0 + ((n_fft - hop) - win_length / 2.0) / rate


def pitch_shift(x, n_steps, bins_per_octave=12, n_fft=2048, win_length=None, hop=None, window_name=None):
    """x: (B, L, C) float64 -> (B, L, C): STFT (pad_begin, pad_end) -> phase vocoder at rate 2^(-n_steps / bins) ->
    inverse STFT with the dual window -> band-limited interpolation by `rate` to L samples at `pitch_shift_offset`."""
    import grad_ref as R
    import time_stretch_ref as TR
    win_length = n_fft if win_length is None else win_length
    hop = win_length // 4 if hop is None else hop
    rate = 2.0 ** (-float(n_steps) / bins_per_octave)
    if rate == 1.0:
        return x
    S = R.stft(x, n_fft, win_length, hop, window_name, True, True, CL, CF)
    y = R.istft(TR.time_stretch(S, rate), n_fft, win_length, hop, window_name, CF, CF)
    return resample(y, rate, x.shape[1], pitch_shift_offset(rate, n_fft, win_length, hop)).transpose(1, 2)
