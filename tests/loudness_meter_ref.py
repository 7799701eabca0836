"""Float64 restatement of the loudness meter (kapre_loudness_stats and kapre_true_peak, kapre_b200/csrc/meter_core.cuh)
and the error bounds of the float32 kernels against it.

    momentary / short-term:  s_j = -0.691 + 10 log10(sum_c g_c e_cj) over [jS, jS + W), W = G or G3; -inf past the
                             item's own count (len - W) // S + 1
    loudness range (EBU Tech 3342, short-term windows):  J1 = {s_j > -70}, Gamma = -0.691 + 10 log10(mean_J1 E_j) - 20,
                             J2 = {j in J1 : s_j > Gamma}, v = sorted s_j over J2, n = |J2|,
                             LRA = v[((n-1) 95 + 50) // 100] - v[((n-1) 10 + 50) // 100]   (0 when n = 0)
    true peak:               20 log10 max_t |resample_poly(x[:len], 4, 1)[t]|
"""

import numpy as np
import scipy.signal

import loudness_ref as LR

EPS32 = LR.EPS32
DB = LR.DB


def geometry(sample_rate):
    """(G, S, G3)."""
    G, S = LR.geometry(sample_rate)
    return G, S, int(round(3 * sample_rate))


def count(L, W, S):
    return (L - W) // S + 1 if L >= W else 0


def _lengths(lengths, B, L):
    return [L] * B if lengths is None else [int(min(max(v, 0), L)) for v in np.broadcast_to(lengths, (B,))]


def window_energies(y, W, S, length):
    """E_j = sum_c g_c e_cj (J,) of one K-weighted item y (C, L) over windows of W samples stepping by S."""
    e = LR.blocks(y, W, S, length)
    return (LR.WEIGHTS[:len(e), None] * e).sum(axis=0), e


def series(y, W, S, lengths=None):
    """(B, count(L, W, S)) loudness series of the K-weighted y (B, C, L)."""
    B, C, L = y.shape
    out = np.full((B, count(L, W, S)), -np.inf)
    for b, n in enumerate(_lengths(lengths, B, L)):
        E, _ = window_energies(y[b], W, S, n)
        with np.errstate(divide='ignore', invalid='ignore'):
            out[b, :len(E)] = -0.691 + 10 * np.log10(E)
    return out


def lra_index(n):
    """(lo, hi) nearest-rank indices of the 10th and 95th percentiles among n values."""
    return ((n - 1) * 10 + 50) // 100, ((n - 1) * 95 + 50) // 100


def lra_gate(E):
    """(J2 mask, Gamma) of one item's short-term energies E, or (None, None) when one is not finite."""
    if not np.all(np.isfinite(E)):
        return None, None
    with np.errstate(divide='ignore', invalid='ignore'):
        s = -0.691 + 10 * np.log10(E)
        j1 = s > -70.0
        if not j1.any():
            return np.zeros(E.shape, bool), -np.inf
        rel = -0.691 + 10 * np.log10(E[j1].mean()) - 20.0
    return j1 & (s > rel), rel


def lra_of_energies(E):
    """Loudness range (LU) of one item's short-term energies E."""
    j2, _ = lra_gate(E)
    if j2 is None:
        return float('nan')
    n = int(j2.sum())
    if n == 0:
        return 0.0
    v = np.sort(-0.691 + 10 * np.log10(E[j2]))
    lo, hi = lra_index(n)
    return float(v[hi] - v[lo])


def loudness_range(y, G3, S, lengths=None):
    B, C, L = y.shape
    return np.array([lra_of_energies(window_energies(y[b], G3, S, n)[0])
                     for b, n in enumerate(_lengths(lengths, B, L))])


def true_peak(x, lengths=None):
    """(B, C) dBTP of x (B, C, L) with scipy's resample_poly in float64."""
    x = np.asarray(x, np.float64)
    B, C, L = x.shape
    out = np.full((B, C), -np.inf)
    for b, n in enumerate(_lengths(lengths, B, L)):
        for c in range(C):
            if n == 0:
                continue
            z = scipy.signal.resample_poly(x[b, c, :n], 4, 1)
            with np.errstate(divide='ignore'):
                out[b, c] = 20 * np.log10(np.abs(z).max()) if not np.isnan(z).any() else np.nan
    return out


def stats(x, sample_rate, lengths=None, coeffs=None):
    """(integrated, momentary, short_term, loudness_range, true_peak) of x (B, C, L) in float64."""
    G, S, G3 = geometry(sample_rate)
    y = LR.weight(x, coeffs or LR.k_weighting(sample_rate))
    return (LR.gated(y, G, S, lengths)[0], series(y, G, S, lengths), series(y, G3, S, lengths),
            loudness_range(y, G3, S, lengths), true_peak(x, lengths))


# ------------------------------------------------------------------------------------------ error bounds
def series_bound(y, W, S, delta, lengths=None):
    """Bound on |s_kernel - s| per window when every sample of y is off by at most delta, as loudness_ref.lkfs_bound
    derives it: |dE_j| <= sum_c g_c (2 sqrt(e_cj) delta + delta^2) plus a relative 1e-12 for the float64 sums, then
    |ds_j| <= (10 / ln 10) |dE_j| / (E_j - |dE_j|) and one float32 rounding.  0 where s is -inf (exact there)."""
    B, C, L = y.shape
    out = np.zeros((B, count(L, W, S)))
    for b, n in enumerate(_lengths(lengths, B, L)):
        E, e = window_energies(y[b], W, S, n)
        if not E.size:
            continue
        dE = (LR.WEIGHTS[:len(e), None] * (2 * np.sqrt(e) * delta + delta ** 2)).sum(axis=0) + 1e-12 * E
        with np.errstate(divide='ignore', invalid='ignore'):
            s = -0.691 + 10 * np.log10(E)
            out[b, :len(E)] = np.where(E > 0, DB * dE / np.maximum(E - dE, 1e-300) + np.abs(s) * EPS32 + 1e-30, 0.0)
    return out


def lra_bound(y, G3, S, delta, lengths=None):
    """Bound on |LRA_kernel - LRA|: an order statistic moves by at most the largest perturbation of the values it is
    taken from, so twice the largest series bound over J2, plus one float32 rounding (gate decisions agreeing)."""
    B, C, L = y.shape
    sb = series_bound(y, G3, S, delta, lengths)
    ref = loudness_range(y, G3, S, lengths)
    out = np.zeros(B)
    for b, n in enumerate(_lengths(lengths, B, L)):
        E, _ = window_energies(y[b], G3, S, n)
        j2, _ = lra_gate(E)
        if j2 is not None and j2.any():
            out[b] = 2 * sb[b, :len(E)][j2].max() + abs(ref[b]) * EPS32 + 1e-30
    return out


def lra_margin(y, G3, S, lengths=None):
    """Per item the smallest distance (LU) of a short-term loudness from either of the range's gates."""
    B, C, L = y.shape
    m = np.full(B, np.inf)
    for b, n in enumerate(_lengths(lengths, B, L)):
        E, _ = window_energies(y[b], G3, S, n)
        j2, rel = lra_gate(E)
        if j2 is None or not E.size:
            continue
        with np.errstate(divide='ignore'):
            s = -0.691 + 10 * np.log10(E)
        m[b] = min(np.abs(s + 70).min(), np.abs(s - rel).min() if np.isfinite(rel) else np.inf)
    return m


def tp_taps():
    """The float32 taps the kernel receives (signal.resample_filter(4, 1)), restated."""
    n, hl, M = 81, 40, 4
    k = np.arange(n, dtype=np.float64)
    h = np.sinc((k - hl) / M) / M * np.kaiser(n, 5.0)
    h = 0.5 * (h + h[::-1])
    return (h / h.sum()).astype(np.float32)


def true_peak_bound(x, lengths=None):
    """Bound on |TP_kernel - TP| (dB) per column.  Each z[t] is 21 float32 products in four fmaf chains of at most six
    terms and two additions: at most 8 roundings on any term, so |dz| <= 8 u sum|w x|; the float32 taps differ from
    scipy's float64 ones by at most u |w|, one more u sum|w x|.  With W = max_r ||w_r||_1 and X = max |x|,
    |d max|z|| <= D = 9 u W X (u = 2^-24, first-order, rounded up to 10), so |dTP| <= (20 / ln 10) D / (peak - D)
    plus one float32 rounding."""
    w = 4.0 * tp_taps().astype(np.float64)
    W = max(np.abs(w[r::4]).sum() for r in range(4))
    ref = true_peak(x, lengths)
    x = np.asarray(x, np.float64)
    B, C, L = x.shape
    out = np.zeros((B, C))
    for b, n in enumerate(_lengths(lengths, B, L)):
        for c in range(C):
            if not np.isfinite(ref[b, c]):
                continue
            D = 10 * EPS32 * W * np.abs(x[b, c, :n]).max()
            peak = 10 ** (ref[b, c] / 20)
            out[b, c] = 2 * DB * D / max(peak - D, 1e-300) + abs(ref[b, c]) * EPS32 + 1e-30
    return out


def true_peak_vjp(x, g, lengths=None):
    """The gradient of true_peak at output gradient g (B, C), through float64 torch.autograd: resample_poly as a
    torch convolution with the float64 taps, amax, 20 log10."""
    import torch
    x = torch.tensor(np.asarray(x, np.float64), requires_grad=True)
    B, C, L = x.shape
    h = torch.tensor(np.asarray(tp_taps(), np.float64))
    total = torch.zeros((), dtype=torch.float64)
    for b, n in enumerate(_lengths(lengths, B, L)):
        if n == 0:
            continue
        u = torch.zeros((C, 4 * n), dtype=torch.float64)
        u = u.index_put((torch.arange(C)[:, None], torch.arange(0, 4 * n, 4)[None, :]), x[b, :, :n])
        z = torch.nn.functional.conv1d(torch.nn.functional.pad(u, (40, 40))[:, None], (4 * h).flip(0)[None, None])[:, 0]
        m = z.abs().amax(dim=1)
        keep = m > 0
        tp = 20 * torch.log10(torch.where(keep, m, torch.ones_like(m)))
        total = total + (tp * torch.tensor(np.asarray(g[b], np.float64)) * keep).sum()
    total.backward()
    return x.grad.numpy()
