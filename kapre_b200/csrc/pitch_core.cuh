// Kernel bodies of YIN / probabilistic YIN pitch tracking: the difference function, the CMNDF and the per-frame
// decisions (one launch), and pYIN's Viterbi decode (a second launch).
//
// Frame m of a (item, channel) row covers the samples [m h - pad, m h - pad + F) (pad = F / 2 with centring, zeros
// outside the signal).  With x its samples (0-based) and W the window,
//   d(tau) = sum_{j=1..W} (x[j] - x[j + tau])^2,   1 <= tau <= max_period
//   c(tau) = d(tau) / (S(tau) / tau + 2^-126),   S(tau) = sum_{k<=tau} d(k),   min_period <= tau <= max_period
// d is summed in the difference form (every term >= 0), never as E0 + E_tau - 2 r(tau).
//
// Segments.  d is built from partial sums over segments of G samples: with sharing (h < W, g = gcd(W, h) >= 32 and
// two or more frames per tile fit the budget) G = g and the segments sit on a grid of stride g anchored to the frames'
// window starts, so a segment is computed once for the W / g frames whose windows hold it; otherwise G = W and every
// frame has its own segment.  A segment's partial is one float32 fmaf chain over its samples in ascending order, and
// d(tau) adds a frame's partials in segment order; S is summed in chunks of 32 lags with the chunk sums carried in
// order.  So every value's bits depend on (item, channel, frame, lag) alone: not on the tile, the batch position, the
// strides or the grid.
//
// Partial pass: a warp takes one (segment, lag group); lane l holds KB lags tau0 + KB l + k in registers and slides a
// window of the KB samples x[a + i + tau] along i (two shared loads per step: x[a + i], the same for every lane, and
// the sample entering lane 31's window; the other lanes take theirs from the next lane by a shuffle).  The emulation
// reads that sample from the staged buffer instead: the same value.
//
// Decisions, per frame, by one thread (the CMNDF is already in shared memory): YIN's trough choice and parabolic
// shift, or pYIN's trough probabilities, pitch bins and voiced probability, written as a sparse list of (bin, P)
// candidates per frame (adjacent troughs that land in one bin merged, in lag order).
//
// Viterbi: one CTA per (item, channel) row; thread j takes pitch bin j's voiced and unvoiced destination states.
// The scores (with the source row's log-normaliser folded in) are double-buffered in shared memory next to the
// w-tap triangle log-weights; backpointers (uint16) go to the workspace and one thread backtracks.
//
// Like the other bodies these are barrier-free phases: under nvcc each phase runs once per thread, separated by CTA
// barriers; the CPU emulation (tests/emu, KB_HOST_EMU) runs each phase as a loop over the CTA's threads.
#pragma once
#include <vector>
#include "stft_core.cuh"

#define KB_PITCH_THREADS 256
#define KB_PITCH_WARPS (KB_PITCH_THREADS / 32)
#define KB_PITCH_MAX_TF 32                  // frames per tile
#define KB_PITCH_MAX_FRAME 8192             // KAPRE_PITCH_MAX_FRAME
#define KB_PITCH_MAX_THRESHOLDS 1024        // KAPRE_PITCH_MAX_THRESHOLDS
#define KB_PITCH_SMEM_BUDGET (100 * 1024)   // two CTAs per SM
#define KB_PITCH_SMEM_MAX (220 * 1024)
#define KB_PITCH_MIN_SHARE 32               // smallest shared segment
#define KB_VIT_THREADS 1024
#define KB_VIT_MAX_PITCH 8192               // KAPRE_PITCH_MAX_BINS
#define KB_VIT_MAX_BAND 8192

struct KbPitchParams {
    // plan geometry
    int F, W, h, pad;                     // frame, window, hop, leading zero padding
    int min_p, max_p, n;                  // lag range of the CMNDF, n = max_p - min_p + 1
    int share, G, SS, R, SPF;             // sharing; segment length; segment stride; segments per hop (h / SS); per frame
    int KB, NLG;                          // lags per lane (template), lag groups of 32 KB lags
    int TF, NSEG, NQ, SPAN;               // frames per tile, segments per tile, 32-lag chunks, staged floats
    int smem;                             // bytes of dynamic shared memory
    float sr;
    double thresh;                        // YIN trough threshold
    int pyin;                             // 1: pYIN epilogue
    int n_thr, n_pitch, cmax;             // thresholds, pitch bins, most troughs per frame ((n + 1) / 2)
    const float* beta;                    // [n_thr]: beta_probs[1 .. n_thr]
    const float* bpow;                    // [cmax + 1]: e^{-lambda r}
    const float* bnorm;                   // [cmax + 1]: (1 - e^-lambda) / (1 - e^{-lambda N})
    const float* bonus;                   // [n_thr + 1]: no_trough_prob * (beta_1 + ... + beta_k)
    const double* edges;                  // [n_pitch - 1]: period at the upper edge of bin m, descending
    // per call
    int B, C, L, M;
    long long tiles, jobs;                // tiles per row, jobs
    const float* x;
    long long x_sb, x_sc, x_sl;
    float* out;                           // YIN f0, or pYIN voiced probability; element strides (b, c, frame)
    long long o_sb, o_sc, o_st;
    float* cm;                            // optional CMNDF (b, c, frame, lag - min_p)
    long long c_sb, c_sc, c_st, c_sk;
    int* cand_n;                          // pYIN candidates of frame (row, m): cand_n[row M + m] entries of
    unsigned short* cand_bin;             //   cand_bin / cand_p[(row M + m) cmax + e]
    float* cand_p;
};

// ---- host side: tiling shared by the library and the CPU emulation ----
inline int kb_pitch_gcd(int a, int b) { while (b) { const int t = a % b; a = b; b = t; } return a; }

inline int kb_pitch_span(const KbPitchParams& p, int TF, int NSEG) {
    const int frames = (TF - 1) * p.h + p.F;
    const int comp = 1 + (NSEG - 1) * p.SS + p.G + p.NLG * 32 * p.KB + 1;
    return frames > comp ? frames : comp;
}

// Shared memory (floats): staged samples, partials [NSEG][max_p], CMNDF rows [TF][max_p], chunk sums and non-finite
// flags [TF][NQ], and for pYIN per frame a trough list (lag, count) [2 cmax] and per-threshold ranks and weights
// [2 n_thr].
inline long long kb_pitch_smem_floats(const KbPitchParams& p, int TF, int NSEG) {
    long long f = kb_pitch_span(p, TF, NSEG);
    f = (f + 3) & ~3LL;
    f += (long long)NSEG * p.max_p + (long long)TF * p.max_p + 2LL * TF * p.NQ;
    if (p.pyin) f += (long long)TF * (2LL * p.cmax + 2LL * p.n_thr);
    return f;
}

// Lags per lane: the choice among 4, 8, 11 and 16 with the fewest issue slots per useful lag (two FP32 instructions
// per lag and about six others per step, over the lag groups the lane count rounds up to).
inline int kb_pitch_pick_kb(int max_p) {
    const int opts[4] = {4, 8, 11, 16};
    int best = 4;
    double bc = 1e300;
    for (int o : opts) {
        const int nlg = (max_p + 32 * o - 1) / (32 * o);
        const double cost = (double)nlg * 32 * o * (2.0 * o + 6.0) / (2.0 * o);
        if (cost < bc) { bc = cost; best = o; }
    }
    return best;
}

// Fills the tiling fields from F, W, h, pad, min_p, max_p, pyin, n_thr.  Returns false when even one frame per tile
// does not fit in shared memory (kapre_b200.backend.pitch_geometry's limits rule that out).
inline bool kb_pitch_tiling(KbPitchParams& p) {
    p.n = p.max_p - p.min_p + 1;
    p.cmax = (p.n + 1) / 2;
    p.NQ = (p.max_p + 31) / 32;
    p.KB = kb_pitch_pick_kb(p.max_p);
    p.NLG = (p.max_p + 32 * p.KB - 1) / (32 * p.KB);
    const int g = kb_pitch_gcd(p.W, p.h);
    for (int share = (p.h < p.W && g >= KB_PITCH_MIN_SHARE) ? 1 : 0; share >= 0; --share) {
        p.share = share;
        p.G = share ? g : p.W;
        p.SS = share ? g : p.h;
        p.R = p.h / p.SS;
        p.SPF = p.W / p.G;
        int tf = 0;
        for (int t = 1; t <= KB_PITCH_MAX_TF; ++t) {
            const int nseg = (t - 1) * p.R + p.SPF;
            if (kb_pitch_smem_floats(p, t, nseg) * 4 <= KB_PITCH_SMEM_BUDGET) tf = t;
        }
        if (share && tf < 2) continue;
        if (tf == 0) {
            if (kb_pitch_smem_floats(p, 1, p.SPF) * 4 > KB_PITCH_SMEM_MAX) return false;
            tf = 1;
        }
        p.TF = tf;
        p.NSEG = (tf - 1) * p.R + p.SPF;
        p.SPAN = kb_pitch_span(p, tf, p.NSEG);
        p.smem = (int)(kb_pitch_smem_floats(p, tf, p.NSEG) * 4);
        return true;
    }
    return false;
}

// Per-call sizes; false when the job count overflows.
inline bool kb_pitch_setup(KbPitchParams& p) {
    p.tiles = ((long long)p.M + p.TF - 1) / p.TF;
    p.jobs = (long long)p.B * p.C * p.tiles;
    return p.jobs < (1LL << 40);
}

#if defined(KB_HOST_EMU)
#define KB_PI_THREADS_BEGIN(NT) for (int tid = 0; tid < (NT); ++tid) {
#define KB_PI_THREADS_END }
#define KB_PI_FN inline
inline float kb_pitch_nan() { return std::nanf(""); }
#else
#define KB_PI_THREADS_BEGIN(NT) { const int tid = threadIdx.x;
#define KB_PI_THREADS_END }
#define KB_PI_FN __device__ __forceinline__
KB_D float kb_pitch_nan() { return __int_as_float(0x7fc00000); }
#endif

// The sample entering the window of lane `lane` at the next step: the next lane's first window sample, or for lane 31
// xs[tail] (the same address for every lane).  The emulation reads xs[own] (the same value).
KB_PI_FN float kb_pitch_next(float v0, const float* xs, int own, int tail, int lane) {
#if defined(KB_HOST_EMU)
    (void)v0; (void)tail; (void)lane;
    return xs[own];
#else
    (void)own;
    const float s = __shfl_down_sync(0xffffffffu, v0, 1);
    const float t = xs[tail];
    return lane == 31 ? t : s;
#endif
}

// Partials of segment `a` (staged offset of its first sample) for lags tau0 .. tau0 + KB - 1, written to prow[tau - 1]
// for tau <= max_p.  tail0: staged offset of the sample entering lane 31's window at step 0.
template <int KB>
KB_PI_FN void kb_pitch_partial(const KbPitchParams& p, const float* xs, float* prow, int a, int tau0, int tail0,
                               int lane) {
    float v[KB], acc[KB];
#pragma unroll
    for (int k = 0; k < KB; ++k) { v[k] = xs[a + tau0 + k]; acc[k] = 0.0f; }
    int i = 0;
    for (; i + KB <= p.G; i += KB) {
#pragma unroll
        for (int r = 0; r < KB; ++r) {
            const float xa = xs[a + i + r];
            const float nx = kb_pitch_next(v[r], xs, a + i + r + tau0 + KB, tail0 + i + r, lane);
#pragma unroll
            for (int k = 0; k < KB; ++k) {
                const float dlt = xa - v[(r + k) % KB];
                acc[k] = fmaf(dlt, dlt, acc[k]);
            }
            v[r] = nx;
        }
    }
    for (; i < p.G; ++i) {
        const float xa = xs[a + i];
        const float nx = kb_pitch_next(v[0], xs, a + i + tau0 + KB, tail0 + i, lane);
#pragma unroll
        for (int k = 0; k < KB; ++k) {
            const float dlt = xa - v[k];
            acc[k] = fmaf(dlt, dlt, acc[k]);
        }
#pragma unroll
        for (int k = 0; k + 1 < KB; ++k) v[k] = v[k + 1];
        v[KB - 1] = nx;
    }
#pragma unroll
    for (int k = 0; k < KB; ++k)
        if (tau0 + k <= p.max_p) prow[tau0 + k - 1] = acc[k];
}

KB_PI_FN void kb_pitch_partials(const KbPitchParams& p, const float* xs, float* P, int tid) {
    const int warp = tid >> 5, lane = tid & 31;
    for (int u = warp; u < p.NSEG * p.NLG; u += KB_PITCH_WARPS) {
        const int seg = u / p.NLG, lg = u - seg * p.NLG;
        const int a = 1 + seg * p.SS;
        const int tau0 = 1 + lg * 32 * p.KB + lane * p.KB;
        const int tail0 = a + 1 + lg * 32 * p.KB + 32 * p.KB;
        float* prow = P + (long long)seg * p.max_p;
        switch (p.KB) {
            case 4: kb_pitch_partial<4>(p, xs, prow, a, tau0, tail0, lane); break;
            case 8: kb_pitch_partial<8>(p, xs, prow, a, tau0, tail0, lane); break;
            case 11: kb_pitch_partial<11>(p, xs, prow, a, tau0, tail0, lane); break;
            default: kb_pitch_partial<16>(p, xs, prow, a, tau0, tail0, lane); break;
        }
    }
}

KB_HD bool kb_pitch_trough(const float* c, int k, int n) {
    if (k == 0) return c[0] < c[1];
    if (k == n - 1) return c[n - 1] < c[n - 2];
    return c[k] < c[k - 1] && c[k] <= c[k + 1];
}

// Refined period min_p + k + shift of lag index k (the parabolic shift is 0 at the ends and where |b| >= |a|).
KB_HD float kb_pitch_period(const float* c, int k, int n, int min_p) {
    float shift = 0.0f;
    if (k > 0 && k < n - 1) {
        const float a = (c[k + 1] + c[k - 1]) - (c[k] + c[k]);
        const float b = (c[k + 1] - c[k - 1]) * 0.5f;
        if (fabsf(b) < fabsf(a)) shift = -b / a;
    }
    return (float)(min_p + k) + shift;
}

// Pitch bin of a period: the number of bin edges (descending periods) at or above it.
KB_HD int kb_pitch_bin(const double* edges, int n_pitch, float period) {
    int lo = 0, hi = n_pitch - 1;        // answer in [lo, hi]
    const double pd = (double)period;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;  // is bin > mid, i.e. period <= edges[mid]?
        if (pd <= edges[mid]) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}

// YIN: f0 of one frame from its CMNDF c[0 .. n-1] (lags min_p .. max_p).
KB_HD float kb_yin_f0(const float* c, int n, int min_p, double thresh, float sr) {
    int kk = -1;
    for (int k = 0; k < n; ++k)
        if (kb_pitch_trough(c, k, n) && (double)c[k] < thresh) { kk = k; break; }
    if (kk < 0) {
        kk = 0;
        for (int k = 1; k < n; ++k)
            if (c[k] < c[kk]) kk = k;
    }
    return sr / kb_pitch_period(c, kk, n, min_p);
}

// pYIN: candidates of one frame.  lk / lc / rk / aw: scratch of cmax, cmax, n_thr, n_thr entries.  Writes the merged
// (bin, P) list and returns the voiced probability.
KB_PI_FN float kb_pyin_frame(const KbPitchParams& p, const float* c, int* lk, int* lc, int* rk, float* aw,
                             long long fi) {
    const int n = p.n, nt = p.n_thr;
    int T = 0, gm = -1;
    for (int k = 0; k < n; ++k) {
        if (!kb_pitch_trough(c, k, n)) continue;
        const double s = (double)c[k] * nt;   // exact: thresholds i with i / n_thr <= c[k]
        lk[T] = k;
        lc[T] = s >= (double)nt ? nt : (int)floor(s);
        if (gm < 0 || c[k] < c[lk[gm]]) gm = T;
        ++T;
    }
    // N_i (troughs below threshold i) into rk, then the weights A_i = bnorm[N_i] beta_i
    for (int i = 0; i < nt; ++i) rk[i] = 0;
    for (int t = 0; t < T; ++t)
        for (int i = lc[t]; i < nt; ++i) ++rk[i];
    for (int i = 0; i < nt; ++i) { aw[i] = p.bnorm[rk[i]] * p.beta[i]; rk[i] = 0; }
    int nc = 0, last = -1;
    float acc = 0.0f, vsum = 0.0f;
    int* cn = p.cand_n + fi;
    unsigned short* cb = p.cand_bin + fi * p.cmax;
    float* cp = p.cand_p + fi * p.cmax;
    for (int t = 0; t < T; ++t) {
        float P = 0.0f;
        for (int i = lc[t]; i < nt; ++i) {       // threshold i + 1: rank rk[i] among the troughs below it
            P = fmaf(p.bpow[rk[i]], aw[i], P);
            ++rk[i];
        }
        if (t == gm) P += p.bonus[lc[t]];
        if (!(P > 0.0f)) continue;
        const int bin = kb_pitch_bin(p.edges, p.n_pitch, kb_pitch_period(c, lk[t], n, p.min_p));
        if (bin == last) { acc += P; continue; }
        if (last >= 0) { cb[nc] = (unsigned short)last; cp[nc] = acc; vsum += acc; ++nc; }
        last = bin; acc = P;
    }
    if (last >= 0) { cb[nc] = (unsigned short)last; cp[nc] = acc; vsum += acc; ++nc; }
    *cn = nc;
    return fminf(vsum, 1.0f);
}

KB_PI_FN void kb_pitch_cta(const KbPitchParams& p, char* smem, long long cta, long long n_cta) {
    float* xs = reinterpret_cast<float*>(smem);
    float* P = xs + ((p.SPAN + 3) & ~3);
    float* crow = P + (long long)p.NSEG * p.max_p;
    float* csum = crow + (long long)p.TF * p.max_p;
    int* bad = reinterpret_cast<int*>(csum + p.TF * p.NQ);
    int* scr = bad + p.TF * p.NQ;
    const float tiny = 1.17549435e-38f;  // 2^-126
    for (long long job = cta; job < p.jobs; job += n_cta) {
        const long long row = job / p.tiles;
        const int tile = (int)(job - row * p.tiles);
        const int b = (int)(row / p.C), ch = (int)(row - (long long)b * p.C);
        const int t0 = tile * p.TF;
        const int nf = p.M - t0 < p.TF ? p.M - t0 : p.TF;
        const long long base = (long long)t0 * p.h - p.pad;
        const float* xr = p.x + (long long)b * p.x_sb + (long long)ch * p.x_sc;
        // phase 1: stage the tile's samples (zeros outside the signal)
        KB_PI_THREADS_BEGIN(KB_PITCH_THREADS)
            for (int e = tid; e < p.SPAN; e += KB_PITCH_THREADS) {
                const long long s = base + e;
                xs[e] = (s >= 0 && s < p.L) ? xr[s * p.x_sl] : 0.0f;
            }
        KB_PI_THREADS_END
        KB_SYNC_CTA;
        // phase 2: segment partials
        KB_PI_THREADS_BEGIN(KB_PITCH_THREADS)
            kb_pitch_partials(p, xs, P, tid);
        KB_PI_THREADS_END
        KB_SYNC_CTA;
        // phase 3: d per (frame, 32-lag chunk), chunk sums, non-finite samples of the frame
        KB_PI_THREADS_BEGIN(KB_PITCH_THREADS)
            for (int u = tid; u < nf * p.NQ; u += KB_PITCH_THREADS) {
                const int f = u / p.NQ, q = u - f * p.NQ;
                const float* pr = P + (long long)f * p.R * p.max_p;
                float* dr = crow + (long long)f * p.max_p;
                const int t1 = 32 * q + 32 < p.max_p ? 32 * q + 32 : p.max_p;
                float s = 0.0f;
                for (int tau = 32 * q + 1; tau <= t1; ++tau) {
                    float d = pr[tau - 1];
                    for (int r = 1; r < p.SPF; ++r) d += pr[(long long)r * p.max_p + tau - 1];
                    dr[tau - 1] = d;
                    s += d;
                }
                csum[f * p.NQ + q] = s;
                int nb = 0;
                const int j1 = (int)((long long)(q + 1) * p.F / p.NQ);
                for (int j = (int)((long long)q * p.F / p.NQ); j < j1; ++j) nb |= !(fabsf(xs[f * p.h + j]) < INFINITY);
                bad[f * p.NQ + q] = nb;
            }
        KB_PI_THREADS_END
        KB_SYNC_CTA;
        // phase 4: S(tau) = (chunk sums before q) + the running sum in the chunk; c(tau) in place of d(tau)
        KB_PI_THREADS_BEGIN(KB_PITCH_THREADS)
            for (int u = tid; u < nf * p.NQ; u += KB_PITCH_THREADS) {
                const int f = u / p.NQ, q = u - f * p.NQ;
                float carry = 0.0f;
                for (int e = 0; e < q; ++e) carry += csum[f * p.NQ + e];
                float* dr = crow + (long long)f * p.max_p;
                const int t1 = 32 * q + 32 < p.max_p ? 32 * q + 32 : p.max_p;
                float run = 0.0f;
                for (int tau = 32 * q + 1; tau <= t1; ++tau) {
                    const float d = dr[tau - 1];
                    run += d;
                    const float mean = (carry + run) / (float)tau;
                    dr[tau - 1] = d / (mean + tiny);
                }
                if (p.cm) {
                    float* co = p.cm + (long long)b * p.c_sb + (long long)ch * p.c_sc + (long long)(t0 + f) * p.c_st;
                    const int ta = 32 * q + 1 > p.min_p ? 32 * q + 1 : p.min_p;
                    for (int tau = ta; tau <= t1; ++tau) co[(long long)(tau - p.min_p) * p.c_sk] = dr[tau - 1];
                }
            }
        KB_PI_THREADS_END
        KB_SYNC_CTA;
        // phase 5: one thread per frame: YIN's f0, or pYIN's candidates and voiced probability
        KB_PI_THREADS_BEGIN(KB_PITCH_THREADS)
            if (tid < nf) {
                const int f = tid;
                int nb = 0;
                for (int q = 0; q < p.NQ; ++q) nb |= bad[f * p.NQ + q];
                const float* c = crow + (long long)f * p.max_p + (p.min_p - 1);
                float* o = p.out + (long long)b * p.o_sb + (long long)ch * p.o_sc + (long long)(t0 + f) * p.o_st;
                if (!p.pyin) {
                    *o = nb ? kb_pitch_nan() : kb_yin_f0(c, p.n, p.min_p, p.thresh, p.sr);
                } else {
                    const long long fi = row * p.M + t0 + f;
                    if (nb) {
                        p.cand_n[fi] = 0;
                        *o = kb_pitch_nan();
                    } else {
                        int* sf = scr + (long long)f * (2 * p.cmax + 2 * p.n_thr);
                        *o = kb_pyin_frame(p, c, sf, sf + p.cmax, sf + 2 * p.cmax,
                                           reinterpret_cast<float*>(sf + 2 * p.cmax + p.n_thr), fi);
                    }
                }
            }
        KB_PI_THREADS_END
        KB_SYNC_CTA;
    }
}

// ---- Viterbi ----
struct KbVitParams {
    int n, w, half;                       // pitch bins, band taps, w / 2
    int M, C, nt;                         // frames, channels, threads
    long long rows;                       // B C
    int cmax;
    float ls, lw;                         // log(1 - switch_prob), log(switch_prob)
    float lpv, lpu;                       // log of the initial probabilities (voiced, unvoiced)
    float fill;
    const float* ltri;                    // [w]
    const float* lnorm;                   // [n]: -log(row sum of the cut triangle)
    const float* freq;                    // [n]
    const int* cand_n;
    const unsigned short* cand_bin;
    const float* cand_p;
    float* vp;                            // voiced probability (read; NaN rows rewritten), element strides (b, c, t)
    float* f0;
    unsigned char* flag;
    long long o_sb, o_sc, o_st;
    unsigned short* bp;                   // [row][t][2 n]
};

KB_HD int kb_vit_smem(int n, int w) { return (6 * n + w + 2 * 64) * 4; }

#if defined(KB_HOST_EMU)
// Block max: each emulated thread keeps its own slot.
#define KB_VIT_RED_SLOTS(nt) (nt)
inline void kb_vit_red_put(float* red, float v, int tid) { red[tid] = v; }
#else
#define KB_VIT_RED_SLOTS(nt) (((nt) + 31) / 32)
KB_D void kb_vit_red_put(float* red, float v, int tid) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    if ((tid & 31) == 0) red[tid >> 5] = v;
}
#endif

KB_PI_FN void kb_vit_cta(const KbVitParams& p, char* smem, float* red, long long cta, long long n_cta) {
    const int n = p.n, S = 2 * n;
    float* buf0 = reinterpret_cast<float*>(smem);
    float* buf1 = buf0 + S;
    float* lnorm = buf1 + S;
    float* ltri = lnorm + n;
    float* lov = ltri + p.w;
    int* flag = reinterpret_cast<int*>(lov + n);
    const float tiny = 1.17549435e-38f;
    const float lt = logf(tiny);
    const int nred = KB_VIT_RED_SLOTS(p.nt);
    KB_PI_THREADS_BEGIN(p.nt)
        for (int j = tid; j < n; j += p.nt) { lnorm[j] = p.lnorm[j]; lov[j] = lt; }
        for (int q = tid; q < p.w; q += p.nt) ltri[q] = p.ltri[q];
    KB_PI_THREADS_END
    for (long long row = cta; row < p.rows; row += n_cta) {
        const int b = (int)(row / p.C), ch = (int)(row - (long long)b * p.C);
        const long long ob = (long long)b * p.o_sb + (long long)ch * p.o_sc;
        const long long fr0 = row * p.M;
        KB_PI_THREADS_BEGIN(p.nt)
            if (tid == 0) *flag = 0;
        KB_PI_THREADS_END
        KB_SYNC_CTA;
        // a NaN voiced probability marks a frame with a non-finite sample: the whole row is unvoiced and NaN
        KB_PI_THREADS_BEGIN(p.nt)
            for (int t = tid; t < p.M; t += p.nt)
                if (p.vp[ob + (long long)t * p.o_st] != p.vp[ob + (long long)t * p.o_st]) *flag = 1;
        KB_PI_THREADS_END
        KB_SYNC_CTA;
        if (*flag) {
            KB_PI_THREADS_BEGIN(p.nt)
                for (int t = tid; t < p.M; t += p.nt) {
                    const long long e = ob + (long long)t * p.o_st;
                    p.f0[e] = p.fill; p.flag[e] = 0; p.vp[e] = kb_pitch_nan();
                }
            KB_PI_THREADS_END
            KB_SYNC_CTA;
            continue;
        }
        if (p.M == 0) continue;
        // frame 0: scatter its observations, then the initial scores
        KB_PI_THREADS_BEGIN(p.nt)
            for (int k = tid; k < p.cand_n[fr0]; k += p.nt)
                lov[p.cand_bin[fr0 * p.cmax + k]] = logf(p.cand_p[fr0 * p.cmax + k] + tiny);
        KB_PI_THREADS_END
        KB_SYNC_CTA;
        float* cur = buf0;
        float* nxt = buf1;
        KB_PI_THREADS_BEGIN(p.nt)
            const float lou = logf((1.0f - p.vp[ob]) / (float)n + tiny);
            float mx = -INFINITY;
            for (int j = tid; j < n; j += p.nt) {
                const float v = p.lpv + lov[j], u = p.lpu + lou;
                nxt[j] = v; nxt[n + j] = u;
                mx = fmaxf(mx, fmaxf(v, u));
            }
            kb_vit_red_put(red, mx, tid);
        KB_PI_THREADS_END
        for (int t = 1;; ++t) {
            KB_SYNC_CTA;
            // clear the last frame's observations; unless that was the final frame, normalise its scores (subtract
            // their maximum, fold in the source rows' normalisers)
            KB_PI_THREADS_BEGIN(p.nt)
                const long long pf = fr0 + t - 1;
                for (int k = tid; k < p.cand_n[pf]; k += p.nt) lov[p.cand_bin[pf * p.cmax + k]] = lt;
                if (t < p.M) {
                    float mx = red[0];
                    for (int e = 1; e < nred; ++e) mx = fmaxf(mx, red[e]);
                    for (int j = tid; j < n; j += p.nt) {
                        nxt[j] = (nxt[j] - mx) + lnorm[j];
                        nxt[n + j] = (nxt[n + j] - mx) + lnorm[j];
                    }
                }
            KB_PI_THREADS_END
            KB_SYNC_CTA;
            if (t == p.M) break;
            { float* tmp = cur; cur = nxt; nxt = tmp; }
            const long long fi = fr0 + t;
            KB_PI_THREADS_BEGIN(p.nt)
                for (int k = tid; k < p.cand_n[fi]; k += p.nt)
                    lov[p.cand_bin[fi * p.cmax + k]] = logf(p.cand_p[fi * p.cmax + k] + tiny);
            KB_PI_THREADS_END
            KB_SYNC_CTA;
            // one step: for destination bin j, the best voiced and unvoiced sources in its band (smallest index on
            // ties), then the switch / stay weights
            KB_PI_THREADS_BEGIN(p.nt)
                const float lou = logf((1.0f - p.vp[ob + (long long)t * p.o_st]) / (float)n + tiny);
                unsigned short* bpt = p.bp + (size_t)fi * S;
                float mx = -INFINITY;
                for (int j = tid; j < n; j += p.nt) {
                    const int lo = j + p.half - p.w + 1 > 0 ? j + p.half - p.w + 1 : 0;
                    const int hi = j + p.half < n - 1 ? j + p.half : n - 1;
                    float ba = -INFINITY, bb = -INFINITY;
                    int ia = lo, ib = lo;
                    for (int i = lo; i <= hi; ++i) {
                        const float tw = ltri[j - i + p.half];
                        const float va = cur[i] + tw, vb = cur[n + i] + tw;
                        if (va > ba) { ba = va; ia = i; }
                        if (vb > bb) { bb = vb; ib = i; }
                    }
                    const float x1 = ba + p.ls, x2 = bb + p.lw;
                    const float y1 = ba + p.lw, y2 = bb + p.ls;
                    const float v = (x1 >= x2 ? x1 : x2) + lov[j];
                    const float u = (y1 >= y2 ? y1 : y2) + lou;
                    bpt[j] = (unsigned short)(x1 >= x2 ? ia : n + ib);
                    bpt[n + j] = (unsigned short)(y1 >= y2 ? ia : n + ib);
                    nxt[j] = v; nxt[n + j] = u;
                    mx = fmaxf(mx, fmaxf(v, u));
                }
                kb_vit_red_put(red, mx, tid);
            KB_PI_THREADS_END
        }
        // backtrace from the best final state (raw scores, first on ties)
        KB_PI_THREADS_BEGIN(p.nt)
            if (tid == 0) {
                int s = 0;
                for (int e = 1; e < S; ++e)
                    if (nxt[e] > nxt[s]) s = e;
                for (int t = p.M - 1; t >= 0; --t) {
                    const long long e = ob + (long long)t * p.o_st;
                    const bool voiced = s < n;
                    p.f0[e] = voiced ? p.freq[s] : p.fill;
                    p.flag[e] = voiced ? 1 : 0;
                    if (t > 0) s = p.bp[(size_t)(fr0 + t) * S + s];
                }
            }
        KB_PI_THREADS_END
        KB_SYNC_CTA;
    }
}
