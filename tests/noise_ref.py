"""Float64 restatement of additive noise at a target SNR (kapre_add_noise, torchaudio.functional.add_noise), its
vector-Jacobian product and the error bounds of the float32 kernel (kapre_b200/csrc/noise_core.cuh).

Per (item, channel) column, with x and n the float32 values the kernel received (upcast), snr the float32 SNR and the
mask t < len:

    Ex = sum_{t < len} x[t]^2,  En = sum_{t < len} n[t]^2,  s = sqrt(Ex / En) 10^(-snr / 20)  (0 where Ex or En is 0)
    y[t] = x[t] + s n[t]   (every t < L)

Error bound of the kernel.  Every product x[t]^2, n[t]^2, g[t] n[t] of float32 values is exact in float64, so only
the float64 additions round.  A sum of m terms in any fixed tree whose longest path has d additions is within
d 2^-53 sum |terms| of the exact sum; here d <= 128 (a lane's samples of a segment) + 5 (the tree) + the segment
count.  Ex and En are sums of non-negative terms, so they carry a relative error of at most d 2^-53, and s (a ratio,
a square root, an exponential and a product in float64) a relative error of at most (d + 8) 2^-53 = e64.  The kernel
then rounds s once to float32 (relative 2^-24) and forms y = fmaf(s32, n, x) with one more rounding:

    |y - y_exact| <= |s32 - s| |n| + 2^-24 |x + s32 n| <= (2^-24 + e64) |s n| + 2^-24 (|y| + (2^-24 + e64) |s n|),

which is below 2^-23 (|s n| + |y|) + e64 |s n| (``forward_bound``).  The gradient is formed in float64 and rounded
once: gx = fl32(g + [t < len] (D s / Ex) x) with D = sum g n a signed sum, whose absolute error is at most
d 2^-53 sum |g n|; the coefficients D s / Ex and D s / En carry that error times s / Ex (s / En) plus a relative
(d + 16) 2^-53 of their own.  ``backward_bounds`` states the resulting per-element bounds of gx, gn and gsnr.
"""
import numpy as np

EPS32 = 2.0 ** -24
EPS64 = 2.0 ** -53
SEG = 4096                  # samples per segment
LN10_20 = np.log(10.0) / 20.0


def _depth(L):
    return 128 + 5 + -(-int(L) // SEG)


def _mask(shape, lengths):
    """(B, C, L) boolean t < len (all True without lengths)."""
    B, C, L = shape
    if lengths is None:
        return np.ones(shape, bool)
    ln = np.broadcast_to(np.asarray(lengths, np.int64), (B, C))
    return np.arange(L)[None, None, :] < ln[:, :, None]


def energies(x, n, lengths=None):
    """(Ex, En) per column, float64."""
    x = np.asarray(x, np.float64)
    n = np.broadcast_to(np.asarray(n, np.float64), x.shape)
    m = _mask(x.shape, lengths)
    return np.where(m, x * x, 0.0).sum(-1), np.where(m, n * n, 0.0).sum(-1)


def scale(ex, en, snr):
    """s per column: 0 where Ex or En is 0 (torchaudio gives NaN for En == 0)."""
    snr = np.asarray(snr, np.float64)
    with np.errstate(divide='ignore', invalid='ignore'):
        s = np.sqrt(ex / en) * 10.0 ** (-snr / 20.0)
    return np.where((ex == 0) | (en == 0), 0.0, s)


def add_noise(x, n, snr, lengths=None):
    """y (B, C, L) float64 and s (B, C) for x (B, C, L), n broadcastable to it, snr and lengths broadcastable to
    (B, C)."""
    x = np.asarray(x, np.float64)
    n = np.broadcast_to(np.asarray(n, np.float64), x.shape)
    ex, en = energies(x, n, lengths)
    s = scale(ex, en, np.broadcast_to(np.asarray(snr, np.float64), ex.shape))
    return x + s[..., None] * n, s


def vjp(x, n, snr, g, lengths=None):
    """(gx, gn, gsnr) of ``add_noise`` at output gradient g, every term through s 0 where Ex or En is 0."""
    x = np.asarray(x, np.float64)
    n = np.broadcast_to(np.asarray(n, np.float64), x.shape)
    g = np.asarray(g, np.float64)
    ex, en = energies(x, n, lengths)
    s = scale(ex, en, np.broadcast_to(np.asarray(snr, np.float64), ex.shape))
    D = (g * n).sum(-1)
    ok = s != 0
    with np.errstate(divide='ignore', invalid='ignore'):
        cx = np.where(ok, D * s / ex, 0.0)
        cn = np.where(ok, D * s / en, 0.0)
    m = _mask(x.shape, lengths)
    gx = g + np.where(m, cx[..., None] * x, 0.0)
    gn = s[..., None] * g - np.where(m, cn[..., None] * n, 0.0)
    return gx, gn, -D * s * LN10_20


def forward_bound(x, n, snr, lengths=None):
    """Per-element bound on |y_kernel - y| (module docstring)."""
    y, s = add_noise(x, n, snr, lengths)
    n = np.broadcast_to(np.asarray(n, np.float64), y.shape)
    sn = np.abs(s[..., None] * n)
    e64 = (_depth(y.shape[-1]) + 8) * EPS64
    return 2 * EPS32 * (sn + np.abs(y)) + e64 * sn


def backward_bounds(x, n, snr, g, lengths=None):
    """Per-element bounds on gx and gn and per-column bound on gsnr (module docstring)."""
    x = np.asarray(x, np.float64)
    n = np.broadcast_to(np.asarray(n, np.float64), x.shape)
    g = np.asarray(g, np.float64)
    gx, gn, gsnr = vjp(x, n, snr, g, lengths)
    ex, en = energies(x, n, lengths)
    s = scale(ex, en, np.broadcast_to(np.asarray(snr, np.float64), ex.shape))
    d = _depth(x.shape[-1])
    dD = d * EPS64 * np.abs(g * n).sum(-1)                  # the float64 error of D
    D = np.abs((g * n).sum(-1))
    rel = (d + 16) * EPS64
    with np.errstate(divide='ignore', invalid='ignore'):
        ecx = np.where(s != 0, s / ex * (dD + rel * D), 0.0)
        ecn = np.where(s != 0, s / en * (dD + rel * D), 0.0)
    bx = 2 * EPS32 * np.abs(gx) + ecx[..., None] * np.abs(x)
    bn = 2 * EPS32 * np.abs(gn) + ecn[..., None] * np.abs(n) + rel * np.abs(s[..., None] * g)
    bs = 2 * EPS32 * np.abs(gsnr) + s * LN10_20 * (dD + rel * D)
    return (gx, gn, gsnr), (bx, bn, bs)


def bank_excerpt(clips, index, offset, L):
    """(B, L) float64: item b's clip ``clips[index[b]]`` read from ``offset[b]`` on, looping."""
    out = np.empty((len(index), L))
    for b, (i, o) in enumerate(zip(index, offset)):
        c = np.asarray(clips[i], np.float64)
        out[b] = c[(int(o) + np.arange(L)) % c.size]
    return out
