"""Float64 restatement of YIN / pYIN as kapre_b200 defines them (signal.yin / signal.pyin), with the elementwise
error bound of the float32 CMNDF and the bound on a float32 Viterbi decode's path score.

Everything here is numpy in float64 and written from the definitions, independently of pitch_core.cuh's order of
operations: the framing, d(tau) in the difference form, the CMNDF, YIN's trough choice and parabolic shift, pYIN's
trough probabilities and observations, the dense transition matrix and a dense Viterbi."""
import numpy as np

TINY = 2.0 ** -126
U = 2.0 ** -24


def gamma(n):
    n = np.asarray(n, dtype=np.float64)
    return n * U / (1.0 - n * U)


def frames(x, g):
    """(M, F) float64 frames of one row x (L,) under pitch_geometry g (zeros outside the signal)."""
    F, h, pad = g['frame_length'], g['hop_length'], g['pad']
    x = np.asarray(x, dtype=np.float64)
    xp = np.concatenate([np.zeros(pad), x, np.zeros(pad)])
    M = 0 if xp.size < F else 1 + (xp.size - F) // h
    idx = np.arange(M)[:, None] * h + np.arange(F)[None, :]
    return xp[idx] if M else np.zeros((0, F))


def difference(fr, g):
    """d[m, tau - 1] = sum_{j=1..W} (x[j] - x[j + tau])^2 for tau = 1 .. max_period."""
    W, P = g['win_length'], g['max_period']
    d = np.empty((fr.shape[0], P))
    a = fr[:, 1:W + 1]
    for tau in range(1, P + 1):
        d[:, tau - 1] = ((a - fr[:, 1 + tau:W + 1 + tau]) ** 2).sum(axis=1)
    return d


def cmndf_from_d(d, g):
    """c[m, k] = d(tau) / (mean_{k<=tau} d + 2^-126), tau = min_period + k."""
    tau = np.arange(1, d.shape[1] + 1, dtype=np.float64)
    c = d / (np.cumsum(d, axis=1) / tau + TINY)
    return c[:, g['min_period'] - 1:]


def cmndf(x, g):
    return cmndf_from_d(difference(frames(x, g), g), g)


def cmndf_bound(x, g):
    """Elementwise bound on |c32 - c| for the kernel's float32 CMNDF.  Every term of d is >= 0, so each step's
    rounding is relative: a segment partial is a chain of G fmaf of squared differences (gamma_{G + 2}); a frame adds
    W / G partials, in all gamma_{W + 2}.  Any order of summing tau values of d adds gamma_tau to S(tau); the mean,
    the denominator's 2^-126 and the quotient round once each.  c's relative error is then at most
    2 gamma_{W + 2} + gamma_tau + 3u, to first order; 1 % covers the higher orders."""
    c = cmndf(x, g)
    tau = np.arange(g['min_period'], g['max_period'] + 1, dtype=np.float64)
    rel = (2 * gamma(g['win_length'] + 2) + gamma(tau) + 3 * U) * 1.01
    return c, rel[None, :] * c + 1e-30


def is_trough(c):
    n = c.size
    t = np.zeros(n, bool)
    t[0] = c[0] < c[1]
    t[n - 1] = c[n - 1] < c[n - 2]
    t[1:n - 1] = (c[1:n - 1] < c[:n - 2]) & (c[1:n - 1] <= c[2:])
    return t


def refined_period(c, k, min_p):
    n = c.size
    shift = 0.0
    if 0 < k < n - 1:
        a = c[k + 1] + c[k - 1] - 2 * c[k]
        b = (c[k + 1] - c[k - 1]) / 2
        if abs(b) < abs(a):
            shift = -b / a
    return min_p + k + shift


def yin_decide(c, g, thresh, sr):
    """(trough index k, f0) of one frame's CMNDF c (float64 values)."""
    c = np.asarray(c, dtype=np.float64)
    tr = np.nonzero(is_trough(c) & (c < thresh))[0]
    k = int(tr[0]) if tr.size else int(np.argmin(c))
    return k, sr / refined_period(c, k, g['min_period'])


def pyin_observe(c, g, q, tab):
    """pYIN's observations of one frame's CMNDF c: ({bin: summed probability}, voiced_prob, [(k, P)] per trough)."""
    c = np.asarray(c, dtype=np.float64)
    nt = q['n_thresholds']
    beta = tab['beta_probs']
    lam = q['boltzmann_parameter']
    ks = np.nonzero(is_trough(c))[0]
    obs, per = {}, []
    if ks.size == 0:
        return obs, 0.0, per
    i = np.arange(1, nt + 1)
    below = c[ks][:, None] * nt < i[None, :]             # c < s_i, s_i = i / n_thresholds (exact)
    rank = np.cumsum(below, axis=0) - 1
    N = below.sum(axis=0)
    prior = np.where(below, (1 - np.exp(-lam)) * np.exp(-lam * rank) / (1 - np.exp(-lam * np.maximum(N, 1))), 0.0)
    P = prior @ beta
    gmin = int(np.argmin(c[ks]))
    P[gmin] += q['no_trough_prob'] * beta[~below[gmin]].sum()
    B = 12 * q['bins_per_semitone']
    for k, p in zip(ks, P):
        per.append((int(k), float(p)))
        if p > 0:
            f = g['sample_rate'] / refined_period(c, int(k), g['min_period'])
            b = int(np.clip(np.round(B * np.log2(f / g['fmin'])), 0, q['n_pitch'] - 1))
            obs[b] = obs.get(b, 0.0) + p
    return obs, min(sum(obs.values()), 1.0), per


def transition(q, tab):
    """Dense (2 n_pitch, 2 n_pitch) transition matrix kron([[1-p, p], [p, 1-p]], T) with T's row i the triangle
    centred on i (tap w // 2 on the diagonal), cut at the edges and normalised."""
    from scipy.signal.windows import triang
    n, w, p = q['n_pitch'], q['band_width'], q['switch_prob']
    tri = triang(w)
    T = np.zeros((n, n))
    for i in range(n):
        for qq in range(w):
            j = i + qq - w // 2
            if 0 <= j < n:
                T[i, j] = tri[qq]
    T /= T.sum(axis=1, keepdims=True)
    return np.kron(np.array([[1 - p, p], [p, 1 - p]]), T), T > 0


def log_obs(obs_list, vps, q):
    """(M, 2 n_pitch) log(observation + 2^-126)."""
    n = q['n_pitch']
    L = np.empty((len(obs_list), 2 * n))
    for t, (obs, vp) in enumerate(zip(obs_list, vps)):
        o = np.zeros(2 * n)
        for b, p in obs.items():
            o[b] = p
        o[n:] = (1 - vp) / n
        L[t] = np.log(o + TINY)
    return L


def viterbi(lobs, A, band):
    """Float64 Viterbi over log(A + 2^-126) inside the band (-inf outside), p_init 1 / n_pitch on each unvoiced state;
    ties to the smallest index.  Returns (path, its score)."""
    S = A.shape[0]
    n = S // 2
    la = np.where(np.kron(np.ones((2, 2), bool), band), np.log(A + TINY), -np.inf)
    init = np.log(np.concatenate([np.zeros(n), np.full(n, 1.0 / n)]) + TINY)
    M = lobs.shape[0]
    sc = init + lobs[0]
    bp = np.zeros((M, S), np.int64)
    for t in range(1, M):
        cand = sc[:, None] + la
        bp[t] = np.argmax(cand, axis=0)
        sc = cand[bp[t], np.arange(S)] + lobs[t]
        sc = sc - sc.max()
    path = np.empty(M, np.int64)
    path[-1] = int(np.argmax(sc))
    for t in range(M - 1, 0, -1):
        path[t - 1] = bp[t, path[t]]
    return path, path_score(path, lobs, la, init)


def path_score(path, lobs, la, init):
    s = init[path[0]] + lobs[0, path[0]]
    for t in range(1, len(path)):
        s += la[path[t - 1], path[t]] + lobs[t, path[t]]
    return s


def log_transition(A, band):
    return np.where(np.kron(np.ones((2, 2), bool), band), np.log(A + TINY), -np.inf)


def path_bound(M, lobs, la):
    """How far below the float64 optimum the float32 decode's path may score.  Each step's terms (a score, a
    log-weight and a log-observation, each within a few hundred of 0 after the per-step normalisation) are formed and
    compared in float32 with a handful of roundings, and the log tables are rounded once: per step at most 16 u times
    the largest magnitude involved.  A path that wins in float32 is within twice the sum of those errors of the best."""
    finite = np.abs(la[np.isfinite(la)]).max()
    mag = finite + np.abs(lobs).max() + 2 * np.abs(lobs).max()
    return 2.0 * M * 16 * U * mag
