"""Float64 numpy/scipy restatement of the rhythm definitions (onset strength, tempogram, tempo, peak picking, beat
tracking) as DESIGN.md §4 states them, restated from librosa 0.10's definitions, not checked against librosa.  Every
function works on one row (a 1-D envelope, or a (frames, bins) spectrogram)."""
import numpy as np
import scipy.ndimage

FLT_MIN = np.float32(np.finfo(np.float32).tiny)


def onset_strength_row(S, lag=1, max_size=1, aggregate='mean', pad_frames=0):
    """S: (T, K) float32.  The envelope (T,) float32, the kernel's rounding: D in float32, the mean of float64 sums
    rounded once, the median numpy's on float32."""
    S = np.asarray(S, np.float32)
    T, K = S.shape
    R = scipy.ndimage.maximum_filter1d(S, max_size, axis=1, mode='reflect') if max_size > 1 else S
    D = np.maximum(np.float32(0), S[lag:] - R[:-lag]) if lag < T else np.zeros((0, K), np.float32)
    nan = np.isnan(S[lag:] - R[:-lag]).any(axis=1) if lag < T else np.zeros(0, bool)
    if aggregate == 'mean':
        A = np.array([np.float32(np.sum(d.astype(np.float64)) / K) for d in D], np.float32)
    else:
        A = np.median(D, axis=1).astype(np.float32)
    A = np.where(nan, np.float32(np.nan), A)
    P = lag + pad_frames
    out = np.zeros(T, np.float32)
    n = max(0, T - P)
    out[P:] = A[:n]
    return out


def onset_strength_torch(S, lag=1, max_size=1, aggregate='mean', pad_frames=0):
    """The same in float64 torch with autograd (tie-free inputs): S a (T, K) float64 tensor requiring grad."""
    import torch
    T, K = S.shape
    if max_size > 1:
        h = max_size // 2
        pad = torch.full((T, h), -float('inf'), dtype=S.dtype)
        padr = torch.full((T, max_size - 1 - h), -float('inf'), dtype=S.dtype)
        Sp = torch.cat([pad, S, padr], 1)
        R = Sp.unfold(1, max_size, 1).max(dim=2).values
    else:
        R = S
    D = torch.relu(S[lag:] - R[:-lag])
    A = D.mean(1) if aggregate == 'mean' else _torch_median(D)
    P = lag + pad_frames
    n = max(0, T - P)
    return torch.cat([torch.zeros(P, dtype=S.dtype), A[:n]])


def _torch_median(D):
    K = D.shape[1]
    s = D.sort(dim=1).values
    if K % 2:
        return s[:, (K - 1) // 2]
    return 0.5 * (s[:, K // 2 - 1] + s[:, K // 2])


def hann(W):
    return 0.5 - 0.5 * np.cos(2 * np.pi * np.arange(W) / W)


def tempogram_row(e, W, center=True, norm=True):
    """(frames, W) float64 autocorrelation tempogram of a float32 envelope."""
    e = np.asarray(e, np.float64)
    T = e.size
    if center:
        c = W // 2
        ep = np.pad(e, (c, c), mode='linear_ramp', end_values=(0, 0))
        n = T
    else:
        ep = e
        n = T - W + 1
    frames = np.lib.stride_tricks.sliding_window_view(ep, W)[:n] * hann(W)
    F = np.fft.rfft(frames, n=2 * W, axis=1)
    ac = np.fft.irfft(np.abs(F) ** 2, axis=1)[:, :W]
    if norm:
        mx = np.abs(ac).max(axis=1, keepdims=True)
        ac = np.where(mx >= FLT_MIN, ac / np.where(mx >= FLT_MIN, mx, 1), ac)
    return ac


def tempo_prior(W, sr, hop, start_bpm=120.0, std_bpm=1.0, max_tempo=320.0):
    """(bpm, logprior) over lags 0 .. W - 1, float64 (lag 0: inf and -inf)."""
    with np.errstate(divide='ignore'):
        bpm = 60.0 * sr / (hop * np.arange(W, dtype=np.float64))
        logprior = -0.5 * ((np.log2(bpm) - np.log2(start_bpm)) / std_bpm) ** 2
    if max_tempo is not None:
        logprior[:int(np.argmax(bpm < max_tempo))] = -np.inf
    return bpm, logprior


def tempo_scores(g, logprior):
    return np.log1p(1e6 * np.asarray(g, np.float64)) + logprior


def _pick(g, logprior, bpm):
    """bpm at the first maximum of the scores, NaN scores skipped (g < -1e-6); NaN when g is non-finite or no score
    is left."""
    if not np.isfinite(g).all():
        return np.nan
    with np.errstate(invalid='ignore'):
        sc = tempo_scores(g, logprior)
    if np.isnan(sc).all():
        return np.nan
    return bpm[np.nanargmax(sc)]


def tempo_row(tg, logprior, bpm, per_frame=False):
    """The tempo of a (frames, W) tempogram: one value, or one per frame."""
    tg = np.asarray(tg, np.float64)
    if per_frame:
        return np.array([_pick(r, logprior, bpm) for r in tg])
    return _pick(tg.mean(axis=0), logprior, bpm)


def detect_defaults(sr, hop):
    pre_max = int(0.03 * sr // hop)
    pre_avg = int(0.10 * sr // hop)
    return dict(pre_max=pre_max, post_max=1, pre_avg=pre_avg, post_avg=pre_avg + 1, wait=int(0.03 * sr // hop))


def peak_inputs(e, normalize=True):
    """The float32 x the kernel thresholds."""
    e = np.asarray(e, np.float32)
    if not normalize:
        return e
    x = e - e.min()
    return x / (x.max() + FLT_MIN)


def peak_pick_row(e, pre_max, post_max, pre_avg, post_avg, wait, delta=0.07, normalize=True, return_scores=False):
    """Boolean onset mask of one envelope; with ``return_scores`` also x - (av + delta) per frame (the margin)."""
    x = peak_inputs(e, normalize)
    T = x.size
    mask = np.zeros(T, bool)
    margin = np.zeros(T)
    if not np.isfinite(x).all() or not (x != 0).any():
        return (mask, margin) if return_scores else mask
    xd = x.astype(np.float64)
    cands = []
    for n in range(T):
        a0, a1 = max(0, n - pre_max), min(T, n + post_max)
        b0, b1 = max(0, n - pre_avg), min(T, n + post_avg)
        av = xd[b0:b1].sum() / (b1 - b0)
        margin[n] = xd[n] - (av + delta)
        if x[n] == x[a0:a1].max() and x[n] != 0 and xd[n] >= av + delta:
            cands.append(n)
    last = -np.inf
    for n in cands:
        if n > last + wait:
            mask[n] = True
            last = n
    return (mask, margin) if return_scores else mask


def local_score(e, p):
    e = np.asarray(e, np.float64)
    sd = e.std(ddof=1) if e.size > 1 else np.nan
    o = e / sd if sd > 0 else e
    d = np.arange(-p, p + 1)
    w = np.exp(-0.5 * (32.0 * d / p) ** 2)
    return np.convolve(o, w, 'same') if o.size >= w.size else np.convolve(o, w, 'full')[p:p + o.size]


def beat_dp(ls, p, tightness=100.0):
    """Serial float64 loop: (cs, back)."""
    T = ls.size
    half = int(np.rint(p / 2))
    ds = np.arange(-2 * p, -half + 1)
    with np.errstate(divide='ignore'):
        txwt = -tightness * np.log(-ds / p) ** 2
    above = np.nonzero(ls >= 0.01 * ls.max())[0]
    i0 = int(above[0]) if above.size else T          # no frame passes: every backlink is -1 (librosa's first_beat)
    cs = np.zeros(T)
    back = np.zeros(T, np.int64)
    for i in range(T):
        best, bd = 0.0, 0
        for q, d in enumerate(ds):
            j = i + d
            c = txwt[q] + (cs[j] if (j >= 0 and d != 0) else 0.0)
            if q == 0 or c > best:
                best, bd = c, d
        cs[i] = ls[i] + best
        back[i] = -1 if i < i0 else i + bd
    return cs, back


def beats_from(ls, cs, back, trim=True):
    """The beat frames (ascending) from the DP's output."""
    T = cs.size
    L = np.array([i >= 1 and cs[i] > cs[i - 1] and (i == T - 1 or cs[i] >= cs[i + 1]) for i in range(T)])
    if not L.any():
        return np.zeros(0, np.int64)
    med = np.median(cs[L])
    q = np.nonzero(2 * cs * L > med)[0]
    if q.size == 0:
        return np.zeros(0, np.int64)
    beats = [int(q[-1])]
    while back[beats[-1]] >= 0:
        beats.append(int(back[beats[-1]]))
    beats = np.array(beats[::-1])
    v = ls[beats]
    s = np.convolve(v, [0.5, 1.0, 0.5], 'same') if v.size >= 3 else np.array(
        [0.5 * (v[j - 1] if j > 0 else 0) + v[j] + 0.5 * (v[j + 1] if j + 1 < v.size else 0) for j in range(v.size)])
    thr = 0.5 * np.sqrt(np.mean(s ** 2)) if trim else 0.0
    J = np.nonzero(s > thr)[0]
    if J.size == 0:
        return np.zeros(0, np.int64)
    return beats[J.min():J.max()]


def period(bpm, sr, hop):
    return int(np.rint(60.0 * (sr / hop) / bpm))


def beat_track_row(e, bpm, sr, hop, tightness=100.0, trim=True):
    """(tempo, beat frames) of one float32 envelope given its bpm, or (tempo, None) when no tracking happens."""
    e = np.asarray(e, np.float32)
    if not np.isfinite(e).all():
        return np.nan, np.zeros(0, np.int64)
    if not (e != 0).any():
        return 0.0, np.zeros(0, np.int64)
    p = period(bpm, sr, hop)
    ls = local_score(e, p)
    cs, back = beat_dp(ls, p, tightness)
    return bpm, beats_from(ls, cs, back, trim)


def beat_margin(e, bpm, sr, hop, tightness=100.0, trim=True):
    """The smallest relative gap behind the beat decisions of one envelope: each frame's best DP candidate against
    its runner-up, the last-beat test ``2 cs [L] > med``, the ``i0`` threshold and the trim threshold.  Below a
    rounding-sized margin a device that rounds exp, log and fma differently may decide otherwise."""
    e = np.asarray(e, np.float32)
    p = period(bpm, sr, hop)
    ls = local_score(e, p)
    cs, back = beat_dp(ls, p, tightness)
    T = ls.size
    half = int(np.rint(p / 2))
    ds = np.arange(-2 * p, -half + 1)
    with np.errstate(divide='ignore'):
        txwt = -tightness * np.log(-ds / p) ** 2
    gaps = []
    scale = max(1.0, np.abs(cs).max())
    for i in range(T):
        j = i + ds
        c = txwt + np.where((j >= 0) & (ds != 0), cs[np.clip(j, 0, T - 1)], 0.0)
        c = np.sort(c[np.isfinite(c)])
        if c.size >= 2:
            gaps.append((c[-1] - c[-2]) / scale)
    gaps.append(np.abs(ls - 0.01 * ls.max()).min() / max(1.0, np.abs(ls).max()))
    L = np.array([i >= 1 and cs[i] > cs[i - 1] and (i == T - 1 or cs[i] >= cs[i + 1]) for i in range(T)])
    if L.any():
        med = np.median(cs[L])
        gaps.append(np.abs(2 * cs[L] - med).min() / scale)
        beats = beats_from(ls, cs, back, trim=False)
        if trim and beats.size:
            v = ls[beats]
            s = np.convolve(np.r_[0.0, v, 0.0], [0.5, 1.0, 0.5], 'valid')
            thr = 0.5 * np.sqrt(np.mean(s ** 2))
            gaps.append(np.abs(s - thr).min() / max(1.0, np.abs(s).max()))
    return min(gaps)
