"""Float64 restatement of gated loudness (kapre_loudness, torchaudio.functional.loudness, ITU-R BS.1770-4), its VJP and
the error bound of the float32 K-weighting plus the float64 gated-energy kernels (kapre_b200/csrc/loudness_core.cuh).

    y = clamp(lfilter(clamp(lfilter(x, shelf)), high-pass)),   blocks [jS, jS + G) for j <= (len - G) // S,
    e_cj = mean of y_c^2 over block j,   E_j = sum_c g_c e_cj,   l_j = -0.691 + 10 log10(E_j),
    J1 = {l_j > -70},   Gamma = -0.691 + 10 log10(mean_J1 E_j) - 10,   J2 = {j in J1 : l_j > Gamma},
    LKFS = -0.691 + 10 log10(mean_J2 E_j)   (-inf for an empty J2; NaN when a block energy is not finite).
"""
import math

import numpy as np
import scipy.signal

import iir_ref as IR

WEIGHTS = np.array([1.0, 1.0, 1.0, 1.41, 1.41])
EPS32 = 2.0 ** -24
DB = 10.0 / math.log(10.0)


def geometry(sample_rate):
    """(G, S) as torchaudio computes them."""
    G = int(round(0.4 * sample_rate))
    return G, int(round(G * 0.25))


def k_weighting(sample_rate):
    """torchaudio's two designs, restated: ((b, a) of treble_biquad(gain 4, 1500 Hz, Q 1 / sqrt 2), (b, a) of
    highpass_biquad(38 Hz, Q 0.5)), float64, not normalised."""
    w0 = 2 * math.pi * 1500.0 / sample_rate
    alpha = math.sin(w0) / 2 / (1 / math.sqrt(2))
    A = math.exp(4.0 / 40 * math.log(10))
    t1, t2, t3 = 2 * math.sqrt(A) * alpha, (A - 1) * math.cos(w0), (A + 1) * math.cos(w0)
    shelf = (np.array([A * ((A + 1) + t2 + t1), -2 * A * ((A - 1) + t3), A * ((A + 1) + t2 - t1)]),
             np.array([(A + 1) - t2 + t1, 2 * ((A - 1) - t3), (A + 1) - t2 - t1]))
    return shelf, IR.biquad('highpass', sample_rate, 38.0, 0.5)


def normalised(coeffs):
    """The float32 coefficients the kernels receive: each pair divided by a[0] in float64, then rounded."""
    return [((b / a[0]).astype(np.float32), (a / a[0]).astype(np.float32)) for b, a in coeffs]


def weight(x, coeffs):
    """The clamped K-weighting of x (..., L) in float64 with the given (b, a) pairs."""
    y = np.asarray(x, np.float64)
    for b, a in coeffs:
        y = IR.lfilter_fast(y, np.asarray(b, np.float64), np.asarray(a, np.float64), clamp=True)
    return y


def blocks(y, G, S, length):
    """(C, J) block energies e_cj of one item y (C, L) cut to `length`."""
    J = (length - G) // S + 1 if length >= G else 0
    sq = np.asarray(y, np.float64)[:, :length] ** 2
    return np.stack([sq[:, j * S:j * S + G].mean(axis=1) for j in range(J)], axis=1) if J else np.zeros((len(y), 0))


def gate(e):
    """(LKFS, E2, J2 mask) of one item's block energies e (C, J)."""
    E = (WEIGHTS[:len(e), None] * e).sum(axis=0)
    if not np.all(np.isfinite(E)):
        return float('nan'), float('nan'), np.zeros(E.shape, bool)
    with np.errstate(divide='ignore', invalid='ignore'):
        l = -0.691 + 10 * np.log10(E)
        j1 = l > -70.0
        rel = -0.691 + 10 * np.log10(E[j1].mean()) - 10 if j1.any() else float('nan')
        j2 = j1 & (l > rel)
    if not j2.any():
        return float('-inf'), 0.0, j2
    E2 = float(E[j2].mean())
    return -0.691 + 10 * math.log10(E2), E2, j2


def gated(y, G, S, lengths=None):
    """Per item of the K-weighted y (B, C, L): (LKFS (B,), E2 (B,), [J2 masks], block energies)."""
    B, C, L = y.shape
    lengths = [L] * B if lengths is None else [int(min(max(v, 0), L)) for v in np.broadcast_to(lengths, (B,))]
    out, E2, masks, es = np.zeros(B), np.zeros(B), [], []
    for b in range(B):
        e = blocks(y[b], G, S, lengths[b])
        out[b], E2[b], m = gate(e)
        masks.append(m)
        es.append(e)
    return out, E2, masks, es


def loudness(x, sample_rate, lengths=None, coeffs=None):
    """LKFS per item of x (B, C, L); coeffs: the (b, a) pairs (default torchaudio's float64 designs)."""
    G, S = geometry(sample_rate)
    return gated(weight(x, coeffs or k_weighting(sample_rate)), G, S, lengths)[0]


def coverage(mask, G, S, L):
    """n(t): the J2 blocks covering each sample t < L."""
    n = np.zeros(L)
    for j in np.nonzero(mask)[0]:
        n[j * S:j * S + G] += 1
    return n


def grad_y(y, gl, G, S, lengths=None):
    """dLKFS / dy times gl per item: gl (20 / ln 10) g_c y n(t) / (E2 |J2| G); 0 for empty J2 items."""
    B, C, L = y.shape
    _, E2, masks, _ = gated(y, G, S, lengths)
    gy = np.zeros((B, C, L))
    for b in range(B):
        k = int(masks[b].sum())
        if k:
            n = coverage(masks[b], G, S, L)
            gy[b] = gl[b] * 2 * DB * WEIGHTS[:C, None] * y[b] * n / (E2[b] * k * G)
    return gy


def vjp(x, gl, sample_rate, lengths=None, coeffs=None):
    """The gradient of ``loudness`` with respect to x at output gradient gl (B,): gy back through each clamp (1 where
    the unclamped value lies in [-1, 1], as torch.clamp) and each filter's adjoint (the filter run in reverse time)."""
    coeffs = coeffs or k_weighting(sample_rate)
    G, S = geometry(sample_rate)
    x = np.asarray(x, np.float64)
    pre, ys = [], [x]
    for b, a in coeffs:
        u = IR.lfilter_fast(ys[-1], b, a)
        pre.append(u)
        ys.append(np.clip(u, -1, 1))
    g = grad_y(ys[-1], np.asarray(gl, np.float64), G, S, lengths)
    for (b, a), u in zip(coeffs[::-1], pre[::-1]):
        g = g * (np.abs(u) <= 1)
        g = scipy.signal.lfilter(np.asarray(b, np.float64), np.asarray(a, np.float64), g[..., ::-1], axis=-1)[..., ::-1]
    return g


def impulse_l1_full(b, a):
    """||h||_1 of the whole filter b / A(z)."""
    imp = np.zeros(1 << 16)
    imp[0] = 1.0
    return float(np.abs(scipy.signal.lfilter(np.asarray(b, np.float64), np.asarray(a, np.float64), imp)).sum())


def weighting_error(x, coeffs32):
    """Bound on max |y_kernel - y| of the two float32 lfilter launches with float32 coefficients coeffs32: each
    filter's own bound (iir_ref.error_bound) plus the previous error carried through the filter (||h||_1 times it); the
    clamps are 1-Lipschitz."""
    x = np.asarray(x, np.float64)
    d, u = 0.0, x
    for b, a in coeffs32:
        b64, a64 = np.asarray(b, np.float64), np.asarray(a, np.float64)
        y = IR.lfilter_fast(u, b64, a64)
        own = IR.error_bound(b64, a64, float(np.abs(u).max()) + d, float(np.abs(y).max()), IR.local_max(u, b64, a64))
        d = impulse_l1_full(b64, a64) * d + own
        u = np.clip(y, -1, 1)
    return d


def lkfs_bound(y, G, S, delta, lengths=None):
    """Bound on |LKFS_kernel - LKFS| per item when every sample of y (B, C, L) is off by at most delta and the gate
    decisions agree: |d(y^2)| <= 2 |y| delta + delta^2 and mean |y| <= sqrt(mean y^2) give
    |dE_j| <= sum_c g_c (2 sqrt(e_cj) delta + delta^2); then |dLKFS| <= (10 / ln 10) mean_J2 |dE_j| / (E2 - that), with
    a relative 1e-12 for the float64 sums and one float32 rounding of the result."""
    out, E2, masks, es = gated(y, G, S, lengths)
    bound = np.zeros(len(out))
    for b in range(len(out)):
        if not masks[b].any():
            continue
        e = es[b]
        dE = (WEIGHTS[:len(e), None] * (2 * np.sqrt(e) * delta + delta ** 2)).sum(axis=0)[masks[b]].mean()
        dE += 1e-12 * E2[b]
        bound[b] = DB * dE / max(E2[b] - dE, 1e-300) + abs(out[b]) * EPS32 + 1e-30
    return bound


def gate_margin(y, G, S, lengths=None):
    """Per item the smallest distance (LU) of a block's loudness from either gate."""
    out, _, _, es = gated(y, G, S, lengths)
    m = np.full(len(out), np.inf)
    for b, e in enumerate(es):
        E = (WEIGHTS[:len(e), None] * e).sum(axis=0)
        if not E.size:
            continue
        with np.errstate(divide='ignore'):
            l = -0.691 + 10 * np.log10(E)
            j1 = l > -70
            rel = -0.691 + 10 * np.log10(E[j1].mean()) - 10 if j1.any() else -np.inf
        m[b] = min(np.abs(l + 70).min(), np.abs(l - rel).min() if j1.any() else np.inf)
    return m
