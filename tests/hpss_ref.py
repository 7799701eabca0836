"""Restatements of the harmonic/percussive separation (kapre_b200/csrc/hpss_core.cuh), written from librosa 0.10's
``decompose.hpss`` and ``util.softmask`` and scipy's ``median_filter(mode='reflect')``:

* ``medians``: the two medians in numpy (reflected windows, rank k // 2, NaN where a window holds NaN);
* ``select``: the element each median selects under the tie rule (value, position in the reflected window);
* ``hpss32``: masks and outputs in float32, one rounded operation per step in the kernels' order, so that powers
  1, 2 and inf are equal bit for bit;
* ``hpss64``: a float64 torch restatement that gathers the medians at given indices, differentiable, for the
  gradient checks.
"""
import numpy as np
import torch

TINY = np.float32(np.finfo(np.float32).tiny)


def reflect(i, n):
    m = np.mod(i, 2 * n)
    return np.where(m < n, m, 2 * n - 1 - m)


def windows(n, k):
    """(n, k) indices of each output's reflected window along an axis of n."""
    return reflect(np.arange(n)[:, None] - k // 2 + np.arange(k)[None, :], n)


def medians(S, kh, kp):
    """H (along axis -2, frames) and P (along axis -1, bins) of a (..., T, K) float32 array."""
    T, K = S.shape[-2:]
    wh = S[..., windows(T, kh), :]                          # (..., T, kh, K)
    H = np.sort(wh, axis=-2)[..., kh // 2, :]
    H = np.where(np.isnan(wh).any(axis=-2), np.float32(np.nan), H)
    wp = S[..., windows(K, kp)]                             # (..., T, K, kp)
    P = np.sort(wp, axis=-1)[..., kp // 2]
    P = np.where(np.isnan(wp).any(axis=-1), np.float32(np.nan), P)
    return H.astype(np.float32), P.astype(np.float32)


def select(S, kh, kp):
    """Indices (frame for H, bin for P) of the elements the medians select: rank k // 2 under (value, window
    position), mapped back through the reflection; a window holding NaN selects its first NaN."""
    T, K = S.shape[-2:]
    out = []
    for axis, k, n in ((-2, kh, T), (-1, kp, K)):
        w = windows(n, k)
        if axis == -2:
            vals = np.moveaxis(S[..., w, :], -1, -2)        # (..., T, K, k)
        else:
            vals = S[..., w]                                # (..., T, K, k)
        key = np.where(np.isnan(vals), np.inf, vals)
        order = np.argsort(key, axis=-1, kind='stable')
        pos = order[..., k // 2]
        first_nan = np.argmax(np.isnan(vals), axis=-1)
        pos = np.where(np.isnan(vals).any(axis=-1), first_nan, pos)
        idx = np.arange(n)
        if axis == -2:
            src = reflect(idx[:, None] - k // 2 + pos, n)   # pos (..., T, K): frame t = axis -2
        else:
            src = reflect(idx[None, :] - k // 2 + pos, n)
        out.append(src.astype(np.int64))
    return out[0], out[1]


def softmask32(a, b, power, split):
    a = np.asarray(a, np.float32)
    b = np.asarray(b, np.float32)
    with np.errstate(all='ignore'):
        if np.isinf(power):
            m = (a > b).astype(np.float32)
        else:
            z = np.maximum(a, b)
            zs = np.where(z < TINY, np.float32(1), z)
            a1, b1 = a / zs, b / zs
            if power == 1:
                pa, pb = a1, b1
            elif power == 2:
                pa, pb = a1 * a1, b1 * b1
            else:
                pa, pb = np.power(a1, np.float32(power)), np.power(b1, np.float32(power))
            m = pa / (pa + pb)
            m = np.where(z < TINY, np.float32(0.5 if split else 0.0), m)
    return np.where(np.isnan(a) | np.isnan(b), np.float32(np.nan), m).astype(np.float32)


def hpss32(S, X, kh, kp, power, margin=(1.0, 1.0), mask=False):
    """(harmonic, percussive) of magnitudes S (..., T, K) float32; X: the complex input (or None for float)."""
    H, P = medians(S, kh, kp)
    mh, mp = np.float32(margin[0]), np.float32(margin[1])
    split = margin[0] == 1 and margin[1] == 1
    with np.errstate(all='ignore'):
        Mh = softmask32(H, mh * P, power, split)
        Mp = softmask32(P, mp * H, power, split)
        if mask:
            return Mh, Mp
        if X is None:
            return S * Mh, S * Mp
        return ((Mh * X.real) + 1j * (Mh * X.imag)).astype(np.complex64), \
            ((Mp * X.real) + 1j * (Mp * X.imag)).astype(np.complex64)


def _softmask64(a, b, power, split):
    if np.isinf(power):
        return (a > b).to(a.dtype)
    z = torch.maximum(a, b)
    bad = z < float(TINY)
    zs = torch.where(bad, torch.ones_like(z), z)
    pa, pb = (a / zs) ** power, (b / zs) ** power
    m = pa / (pa + pb)
    return torch.where(bad, torch.full_like(m, 0.5 if split else 0.0), m)


def hpss64(S, srcH, srcP, kh, kp, power, margin=(1.0, 1.0), mask=False, X=None):
    """float64 torch restatement with the medians gathered at srcH / srcP (from ``select``) out of S (..., T, K).
    X: complex128 input whose |X| is S (S then is computed from X here), or None."""
    if X is not None:
        S = X.abs()
    H = torch.gather(S, -2, torch.as_tensor(srcH))
    P = torch.gather(S, -1, torch.as_tensor(srcP))
    split = margin[0] == 1 and margin[1] == 1
    Mh = _softmask64(H, margin[0] * P, power, split)
    Mp = _softmask64(P, margin[1] * H, power, split)
    if mask:
        return Mh, Mp
    base = S if X is None else X
    return base * Mh, base * Mp
