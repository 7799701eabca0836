"""Float64 restatement of the chroma features (kapre_b200.signal.chroma_stft / chroma_cqt / chroma_cens /
estimate_tuning), independent of the kernels, with elementwise error bounds derived from the code.

The definitions are those DESIGN.md states (modelled on librosa 0.10's feature.chroma_stft, chroma_cqt, chroma_cens,
core.piptrack, estimate_tuning and pitch_tuning); they were not checked against librosa, which is not a dependency.

Bounds.  The projection y_j = sum_k W_jk s_k is one float32 fmaf chain of K non-negative terms, so its rounding error
is relative: |y32 - y| <= gamma_K y over the float32 operands, and W's rounding to float32 and the square of a
magnitude add a unit each: gamma_(K+2) y against float64 W and the float32 magnitude.  The length of a frame adds
NC units (a sum of NC such values) and the square root one more; the division adds one.  Every quantity is
non-negative, so the output's bound stays relative and elementwise:
    |out32 - out| <= gamma_(2 K + 2 NC + 16) |out| + 2^-149.
The gradient's bound is taken over the absolute values of every term (the same formulas with |.|), as the terms may
cancel: |g32 - g| <= gamma_(3 K + 4 NC + 32) G_abs."""
import numpy as np

U32 = 2.0 ** -24
TINY32 = float(np.finfo(np.float32).tiny)


def gamma(n):
    return n * U32 / (1 - n * U32)


def threshold(y, thr):
    return y if thr is None else np.where(y < thr, 0.0, y)


def length(v, norm):
    """(..., NC) -> (..., 1): librosa's normalize length, 1 where it is below FLT_MIN."""
    a = np.abs(v)
    if norm is None:
        return np.ones(v.shape[:-1] + (1,))
    if norm == np.inf:
        n = a.max(axis=-1, keepdims=True)
    elif norm == 1:
        n = a.sum(axis=-1, keepdims=True)
    else:
        n = np.sqrt((a ** 2).sum(axis=-1, keepdims=True))
    return np.where(n < TINY32, 1.0, n)


def normalize(v, norm):
    return v / length(v, norm)


def project(s, W, norm, thr=None):
    """s: (..., K) float64 input, W: (NC, K).  Returns (out, bound) of normalize(threshold(W s), norm)."""
    K, NC = s.shape[-1], W.shape[0]
    y = s @ W.T
    out = normalize(threshold(y, thr), norm)
    return out, gamma(2 * K + 2 * NC + 16) * np.abs(out) + 2.0 ** -149


def project_grad(s, W, norm, g, thr=None, mode='linear', x=None):
    """Gradient of sum(g * project(s)) to the input x of ``mode`` ('linear': s = x; 'square': s = x^2; 'complex':
    s = |x|) in float64, and its bound (the same chain over absolute values)."""
    K, NC = s.shape[-1], W.shape[0]
    y = s @ W.T
    v = threshold(y, thr)
    keep = np.ones_like(y) if thr is None else (y >= thr).astype(np.float64)
    if norm is None:
        gv, gabs = g, np.abs(g)
    else:
        a = np.abs(v)
        raw = a.max(axis=-1, keepdims=True) if norm == np.inf else a.sum(axis=-1, keepdims=True) if norm == 1 \
            else np.sqrt((a ** 2).sum(axis=-1, keepdims=True))
        small = raw < TINY32
        n = np.where(small, 1.0, raw)
        dot = (g * v).sum(axis=-1, keepdims=True)
        dabs = (np.abs(g) * np.abs(v)).sum(axis=-1, keepdims=True)
        sg = np.sign(v)
        if norm == 1:
            gv = g / n - sg * dot / n ** 2
            gabs = np.abs(g) / n + np.abs(sg) * dabs / n ** 2
        elif norm == 2:
            gv = g / n - v * dot / n ** 3
            gabs = np.abs(g) / n + np.abs(v) * dabs / n ** 3
        else:
            first = np.zeros_like(v)
            np.put_along_axis(first, np.abs(v).argmax(axis=-1)[..., None], 1.0, axis=-1)
            gv = g / n - first * sg * dot / n ** 2
            gabs = np.abs(g) / n + first * dabs / n ** 2
        gv = np.where(small, g, gv)
        gabs = np.where(small, np.abs(g), gabs)
    gy, gyabs = gv * keep, gabs * keep
    gs, gsabs = gy @ W, gyabs @ np.abs(W)
    if mode == 'square':
        gs, gsabs = 2 * x * gs, 2 * np.abs(x) * gsabs
    elif mode == 'complex':
        a = np.abs(x)
        r = np.where(a > 0, x / np.where(a > 0, a, 1), 0)
        gs, gsabs = r * gs, gsabs
    return gs, gamma(3 * K + 4 * NC + 32) * gsabs + 2.0 ** -140


def piptrack32(S, sr, n_fft, lo, hi):
    """float32 restatement of the peak pass on one (frames, K) float32 power spectrogram: a list per frame of (bin,
    mag, pitch) float32 triples, ascending."""
    S = np.asarray(S, np.float32)
    out = []
    f32 = np.float32
    for s in S:
        if not np.isfinite(s).all():
            out.append([])
            continue
        ref = f32(0.1) * s.max()
        sp = np.where(s > ref, s, f32(0))
        peaks = []
        for k in range(lo, hi):
            if not (s[k] > ref and sp[k] > sp[k - 1] and sp[k] >= sp[k + 1]):
                continue
            a = f32(0.5) * (s[k + 1] - s[k - 1])
            d = (f32(2) * s[k] - s[k + 1]) - s[k - 1]
            sh = f32(0) if abs(d) < np.finfo(np.float32).tiny else a / d
            pitch = ((f32(k) + sh) * f32(sr)) / f32(n_fft)
            mag = s[k] + (f32(0.5) * a) * sh
            peaks.append((k, mag, pitch))
        out.append(peaks)
    return out


def median32(mags):
    """numpy's median of float32 values, with an even count's mean taken as 0.5f (a + b) in float32."""
    m = np.sort(np.asarray(mags, np.float32))
    n = m.size
    if n % 2:
        return m[n // 2]
    return np.float32(0.5) * (m[n // 2 - 1] + m[n // 2])


def pitch_tuning(pitches, resolution, bins_per_octave):
    """(tuning, index) of the residual histogram (index = number of bins when there are no pitches)."""
    edges = np.linspace(-0.5, 0.5, int(np.ceil(1.0 / resolution)) + 1)
    p = np.asarray(pitches, np.float64)
    if p.size == 0:
        return 0.0, edges.size - 1
    r = np.mod(bins_per_octave * np.log2(p / 27.5), 1.0)
    r[r >= 0.5] -= 1.0
    counts, _ = np.histogram(r, edges)
    i = int(np.argmax(counts))
    return float(edges[i]), i


def estimate_tuning(S_item, sr, n_fft, lo, hi, resolution=0.01, bins_per_octave=12):
    """One item's tuning from its (channels, frames, K) float32 spectrogram: (tuning, index, median, n peaks)."""
    peaks = [p for ch in S_item for fr in piptrack32(ch, sr, n_fft, lo, hi) for p in fr]
    if not peaks:
        return 0.0, int(np.ceil(1.0 / resolution)), None, 0
    mags = np.array([p[1] for p in peaks], np.float32)
    pitches = np.array([p[2] for p in peaks], np.float32)
    m = median32(mags)
    t, i = pitch_tuning(pitches[mags >= m], resolution, bins_per_octave)
    return t, i, m, len(peaks)


def quantize(v):
    """CENS quantisation of the L1-normalised chroma (float64 rule on float32 thresholds)."""
    v = np.asarray(v, np.float64)
    q = sum((v > float(np.float32(s))).astype(np.float64) for s in (0.4, 0.2, 0.1, 0.05)) * 0.25
    return np.where(np.isnan(v), np.nan, q)


def smooth(q, taps):
    """(..., M, NC): out[m] = sum_i w_i q[m + N // 2 - i], zeros outside, and its bound before normalisation."""
    q = np.asarray(q, np.float64)
    N, M = len(taps), q.shape[-2]
    out = np.zeros_like(q)
    for i, w in enumerate(taps):
        sh = N // 2 - i
        src = np.arange(M) + sh
        ok = (src >= 0) & (src < M)
        out[..., ok, :] += w * q[..., src[ok], :]
    return out


def cens_from_q(q, taps):
    """CENS output from the kernel's quantised q, and its relative bound."""
    y = smooth(q, taps)
    out = normalize(y, 2)
    NC = q.shape[-1]
    return out, gamma(len(taps) + 2 * NC + 16) * np.abs(out) + 2.0 ** -149
