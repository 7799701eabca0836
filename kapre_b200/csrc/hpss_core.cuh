// Kernel bodies of the harmonic/percussive separation (Fitzgerald's median filtering, as librosa.decompose.hpss):
// the forward (medians, soft masks and the requested outputs in one launch) and the two passes of its gradient.
//
// Medians.  For a (item, channel) row of magnitudes S[t][b] (t < T frames, b < K bins), H[t][b] is the element of rank
// k_h / 2 of S[t - k_h/2 .. t - k_h/2 + k_h - 1][b] and P[t][b] that of S[t][b - k_p/2 .. b - k_p/2 + k_p - 1], indices
// reflected with period 2n, edge included (scipy.ndimage.median_filter(mode='reflect')).  A window holding a NaN gives
// NaN.  A job is a tile of KB_HS_TT frames x KB_HS_TK bins of one row; it stages the tile's magnitudes with a cross-
// shaped halo, reflections resolved at staging: A = frames [t0 - k_h/2, t0 + TT + k_h - 1 - k_h/2) of the tile's bins and
// Bp = bins [b0 - k_p/2, b0 + TK + k_p - 1 - k_p/2) of the tile's frames (its centre copied from A, not read again).
//
// Selection.  Each thread walks a run of KB_HS_RUN consecutive outputs along its filter axis and keeps its window
// sorted in NS registers (NS = 32 or 64 >= k, the unused slots +inf): a step deletes the outgoing value and inserts the
// incoming one in one unrolled pass over the slots (compare, select, min, max per slot), and the median is slot k / 2.
// So a median costs O(NS) instructions, not O(k^2).  NaN cannot be ordered, so the window keeps a count of its NaNs and
// holds +inf in their place; -0 is kept as +0.
//
// Masks (librosa.util.softmask): m(a, b) = NaN if a or b is NaN; with power inf, a > b as 1 / 0; else Z = max(a, b),
// 0.5 (split_zeros: both margins 1) or 0 when Z < FLT_MIN, else (a/Z)^p / ((a/Z)^p + (b/Z)^p), each step one correctly
// rounded float32 operation (powf only for p other than 1 and 2).  M_H = m(H, margin_h P), M_P = m(P, margin_p H).  The
// outputs are S M (float input), M X (complex input) or the masks.
//
// Gradient, two launches over a workspace of 16 bytes per element (kb_hs_w [row][t][b], one array per median):
//   1. per tile, the medians again and, for each, the element it selected: rank k/2 under the order (value, position
//      in the reflected window), mapped back to the index that position copies (a window holding NaN: its first NaN).
//      The gradient of each median (the mask term) goes to the workspace with that index; the direct term
//      M_H g_H + M_P g_P goes to the input gradient.
//   2. per element, the median gradients whose index names it, in ascending order of the output along frames then
//      along bins (an element can only be selected by outputs less than k away, reflections included), added to the
//      direct term; complex input then goes through |X| (g X / |X|, 0 at X = 0).
// So every output's bits depend only on its row's data and its (frame, bin), and there are no floating-point atomics.
//
// Like the other bodies these are barrier-free phases: under nvcc each phase runs once per thread, separated by CTA
// barriers; the CPU emulation (tests/emu, KB_HOST_EMU) runs each phase as a loop over the CTA's threads.
#pragma once
#include "stft_core.cuh"

#define KB_HS_THREADS 128
#define KB_HS_TT 64                 // frames per tile
#define KB_HS_TK 64                 // bins per tile
#define KB_HS_RUN 32                // outputs per thread and walk
#define KB_HS_KMAX 64               // KAPRE_HPSS_MAX_KERNEL
#define KB_HS_TINY 1.17549435e-38f  // FLT_MIN
#define KB_HS_INF __int_as_float(0x7f800000)

enum { KB_HS_POW_GENERIC = 0, KB_HS_POW_1 = 1, KB_HS_POW_2 = 2, KB_HS_POW_INF = 3 };

#if defined(KB_HOST_EMU)
#undef KB_HS_INF
#define KB_HS_INF INFINITY
#define KB_HS_THREADS_BEGIN for (int tid = 0; tid < KB_HS_THREADS; ++tid) {
#define KB_HS_THREADS_END }
#define KB_HS_FN inline
inline float kb_hs_nan() { return std::nanf(""); }
inline float kb_hs_mul(float a, float b) { return a * b; }
inline float kb_hs_add(float a, float b) { return a + b; }
inline float kb_hs_div(float a, float b) { return a / b; }
inline float kb_hs_pow(float a, float b) { return std::pow(a, b); }
#else
#define KB_HS_THREADS_BEGIN { const int tid = threadIdx.x;
#define KB_HS_THREADS_END }
#define KB_HS_FN __device__ __forceinline__
KB_D float kb_hs_nan() { return __int_as_float(0x7fc00000); }
KB_D float kb_hs_mul(float a, float b) { return __fmul_rn(a, b); }
KB_D float kb_hs_add(float a, float b) { return __fadd_rn(a, b); }
KB_D float kb_hs_div(float a, float b) { return __fdiv_rn(a, b); }
KB_D float kb_hs_pow(float a, float b) { return powf(a, b); }
#endif

struct alignas(8) kb_hs_w { float g; int src; };

struct KbHpssParams {
    int B, C, T, K;
    int kh, kp;                           // median lengths along frames and bins
    float mh, mp;                         // margins
    float power;
    int pmode;                            // KB_HS_POW_*
    int split;                            // both margins 1: a mask over Z < FLT_MIN is 0.5
    int cplx;                             // input complex64 (magnitude |X| = kb_cabs, outputs M X)
    int mask;                             // write the masks (float32) instead of the components
    long long tiles_t, tiles_k, jobs;
    const void* x;                        // float or float2, element strides (b, c, t, k)
    long long x_sb, x_sc, x_st, x_sk;
    void* oh;                             // harmonic output (nullable), element strides (b, c, t, k)
    long long oh_sb, oh_sc, oh_st, oh_sk;
    void* op;                             // percussive output (nullable)
    long long op_sb, op_sc, op_st, op_sk;
    // backward
    const void* gh;                       // gradient of the harmonic output or mask (nullable)
    long long gh_sb, gh_sc, gh_st, gh_sk;
    const void* gp;                       // gradient of the percussive output or mask (nullable)
    long long gp_sb, gp_sc, gp_st, gp_sk;
    void* gx;                             // gradient of the input (float or float2)
    long long gx_sb, gx_sc, gx_st, gx_sk;
    kb_hs_w* wh;                          // workspace [row][t][b]: gradient of H and the index (frame) it selected
    kb_hs_w* wp;                          //                        gradient of P and the index (bin) it selected
};

inline bool kb_hpss_setup(KbHpssParams& p) {
    p.tiles_t = ((long long)p.T + KB_HS_TT - 1) / KB_HS_TT;
    p.tiles_k = ((long long)p.K + KB_HS_TK - 1) / KB_HS_TK;
    p.jobs = (long long)p.B * p.C * p.tiles_t * p.tiles_k;
    return p.jobs < (1LL << 40);
}

// Slots of the sorted window for a median of length k.
KB_HD int kb_hs_slots(int k) { return k <= 32 ? 32 : 64; }

// Row stride of Bp: odd, so that the percussive walk (one thread per frame) reads without bank conflicts.
KB_HD int kb_hs_bstride(int kp) { return (KB_HS_TK + kp - 1) | 1; }

// Shared memory (floats): U = A (TT + k_h - 1 rows of TK), later Ps [TT][TK + 1]; Bp [TT][bstride]; Hs [TT][TK]; the
// backward adds the selected indices sH [TT][TK] and sP [TT][TK + 1].
KB_HD int kb_hs_ufloats(int kh) {
    const int a = (KB_HS_TT + kh - 1) * KB_HS_TK, b = KB_HS_TT * (KB_HS_TK + 1);
    return a > b ? a : b;
}
KB_HD int kb_hpss_smem(int kh, int kp, int bwd) {
    int n = kb_hs_ufloats(kh) + KB_HS_TT * kb_hs_bstride(kp) + KB_HS_TT * KB_HS_TK;
    if (bwd) n += KB_HS_TT * KB_HS_TK + KB_HS_TT * (KB_HS_TK + 1);
    return n * 4;
}

// Index of position i of a row of n under reflection with period 2n, edge included (d c b a | a b c d | d c b a).
KB_HD int kb_hs_reflect(int i, int n) {
    const int n2 = 2 * n;
    int m = i % n2;
    if (m < 0) m += n2;
    return m < n ? m : n2 - 1 - m;
}

KB_HD long long kb_hs_off(long long row, int C, long long sb, long long sc, long long st, long long sk, int t, int b) {
    return (row / C) * sb + (row % C) * sc + (long long)t * st + (long long)b * sk;
}

KB_HS_FN float kb_hs_mag(const KbHpssParams& p, long long o) {
    if (p.cplx) {
        const float2 c = reinterpret_cast<const float2*>(p.x)[o];
        return kb_cabs(c.x, c.y);
    }
    return reinterpret_cast<const float*>(p.x)[o];
}

// The key a value takes in the sorted window: NaN as +inf (counted apart), -0 as +0.
KB_HS_FN float kb_hs_key(float v) { return v != v ? KB_HS_INF : kb_hs_add(v, 0.0f); }

template <int NS>
KB_HS_FN void kb_hs_insert(float (&a)[NS], float v) {
#pragma unroll
    for (int j = NS - 1; j > 0; --j) a[j] = fmaxf(a[j - 1], fminf(a[j], v));
    a[0] = fminf(a[0], v);
}

// Delete o (present) and insert v, in one ascending pass.
template <int NS>
KB_HS_FN void kb_hs_replace(float (&a)[NS], float o, float v) {
    bool passed = false;
    float prev = -KB_HS_INF;
#pragma unroll
    for (int j = 0; j < NS; ++j) {
        passed = passed || a[j] == o;
        const float b = passed ? (j + 1 < NS ? a[j + 1] : KB_HS_INF) : a[j];
        a[j] = fmaxf(prev, fminf(b, v));
        prev = b;
    }
}

template <int NS>
KB_HS_FN float kb_hs_pick(const float (&a)[NS], int r) {
    float m = a[0];
#pragma unroll
    for (int j = 1; j < NS; ++j) m = j == r ? a[j] : m;
    return m;
}

// Walk n consecutive outputs: output i's window is w[(i + j) es], j < k.  out(i, median) gets NaN for a window holding
// NaN.
template <int NS, typename Out>
KB_HS_FN void kb_hs_walk(const float* w, int es, int k, int n, Out out) {
    float a[NS];
#pragma unroll
    for (int j = 0; j < NS; ++j) a[j] = KB_HS_INF;
    int nanc = 0;
    for (int j = 0; j < k; ++j) {
        const float v = w[j * es];
        nanc += v != v;
        kb_hs_insert<NS>(a, kb_hs_key(v));
    }
    const int r = k / 2;
    for (int i = 0;; ++i) {
        out(i, nanc ? kb_hs_nan() : kb_hs_pick<NS>(a, r));
        if (i + 1 >= n) break;
        const float o = w[i * es], v = w[(i + k) * es];
        nanc += (v != v) - (o != o);
        kb_hs_replace<NS>(a, kb_hs_key(o), kb_hs_key(v));
    }
}

// Window position (0 .. k - 1) of the element a median m selected: rank k/2 under (value, position); the first NaN of
// a window holding one.
KB_HS_FN int kb_hs_select(const float* w, int es, int k, float m) {
    if (m != m) {
        for (int j = 0; j < k; ++j)
            if (w[j * es] != w[j * es]) return j;
        return 0;
    }
    int less = 0;
    for (int j = 0; j < k; ++j) less += w[j * es] < m;
    int skip = k / 2 - less;
    for (int j = 0; j < k; ++j) {
        if (w[j * es] == m) {
            if (skip == 0) return j;
            --skip;
        }
    }
    return 0;
}

KB_HS_FN float kb_hs_powf(const KbHpssParams& p, float v) {
    if (p.pmode == KB_HS_POW_1) return v;
    if (p.pmode == KB_HS_POW_2) return kb_hs_mul(v, v);
    return kb_hs_pow(v, p.power);
}

// librosa.util.softmask(a, b, power, split_zeros)
KB_HS_FN float kb_hs_softmask(const KbHpssParams& p, float a, float b) {
    if (a != a || b != b) return kb_hs_nan();
    if (p.pmode == KB_HS_POW_INF) return a > b ? 1.0f : 0.0f;
    const float z = fmaxf(a, b);
    if (z < KB_HS_TINY) return p.split ? 0.5f : 0.0f;
    const float pa = kb_hs_powf(p, kb_hs_div(a, z)), pb = kb_hs_powf(p, kb_hs_div(b, z));
    return kb_hs_div(pa, kb_hs_add(pa, pb));
}

// (dm/da, dm/db) of the soft mask, evaluated on a / Z and b / Z; 0 where the derivative is infinite or undefined
// (Z < FLT_MIN, power inf, a zero argument with p < 1).
KB_HS_FN void kb_hs_dmask(const KbHpssParams& p, float a, float b, float* da, float* db) {
    if (a != a || b != b) { *da = *db = kb_hs_nan(); return; }
    const float z = fmaxf(a, b);
    if (p.pmode == KB_HS_POW_INF || z < KB_HS_TINY) { *da = *db = 0.0f; return; }
    const float a1 = a / z, b1 = b / z;
    const float pa = kb_hs_powf(p, a1), pb = kb_hs_powf(p, b1);
    const float den = pa + pb;                 // >= 1: max(a1, b1) = 1
    float ga, gb;                              // p x^(p - 1)
    if (p.pmode == KB_HS_POW_1) { ga = 1.0f; gb = 1.0f; }
    else if (p.pmode == KB_HS_POW_2) { ga = 2.0f * a1; gb = 2.0f * b1; }
    else {
        ga = (a1 == 0.0f && p.power < 1.0f) ? 0.0f : p.power * kb_hs_pow(a1, p.power - 1.0f);
        gb = (b1 == 0.0f && p.power < 1.0f) ? 0.0f : p.power * kb_hs_pow(b1, p.power - 1.0f);
    }
    *da = ((ga * pb) / den / den) / z;
    *db = -((pa * gb) / den / den) / z;
}

// The forward (BWD = 0) or the first gradient pass (BWD = 1) over one tile per job.
template <int NSH, int NSP, int BWD>
KB_HS_FN void kb_hpss_cta(const KbHpssParams& p, char* smem, long long cta, long long n_cta) {
    const int TT = KB_HS_TT, TK = KB_HS_TK, kh = p.kh, kp = p.kp, hh = kh / 2, hp = kp / 2;
    const int BS = kb_hs_bstride(kp), PS = TK + 1;
    float* U = reinterpret_cast<float*>(smem);          // A, then Ps
    float* Bp = U + kb_hs_ufloats(kh);
    float* Hs = Bp + TT * BS;
    int* sH = reinterpret_cast<int*>(Hs + TT * TK);     // backward only
    int* sP = sH + TT * TK;
    for (long long job = cta; job < p.jobs; job += n_cta) {
        const long long row = job / (p.tiles_t * p.tiles_k);
        const long long rem = job % (p.tiles_t * p.tiles_k);
        const int t0 = (int)(rem / p.tiles_k) * TT, b0 = (int)(rem % p.tiles_k) * TK;
        // stage A and the bin halo of Bp
        KB_HS_THREADS_BEGIN
        for (int i = tid; i < (TT + kh - 1) * TK; i += KB_HS_THREADS) {
            const int r = i / TK, c = i % TK, b = b0 + c;
            U[i] = b < p.K ? kb_hs_mag(p, kb_hs_off(row, p.C, p.x_sb, p.x_sc, p.x_st, p.x_sk,
                                                   kb_hs_reflect(t0 - hh + r, p.T), b))
                           : 0.0f;
        }
        const int halo = kp - 1;
        for (int i = tid; i < TT * halo; i += KB_HS_THREADS) {
            const int f = i / halo, j = i % halo, c = j < hp ? j : TK + j;   // left halo [0, hp), right [hp + TK, ..)
            const int t = t0 + f;
            Bp[f * BS + c] = t < p.T ? kb_hs_mag(p, kb_hs_off(row, p.C, p.x_sb, p.x_sc, p.x_st, p.x_sk, t,
                                                              kb_hs_reflect(b0 - hp + c, p.K)))
                                     : 0.0f;
        }
        KB_HS_THREADS_END
        KB_SYNC_CTA;
        KB_HS_THREADS_BEGIN
        for (int i = tid; i < TT * TK; i += KB_HS_THREADS) {
            const int f = i / TK, c = i % TK, t = t0 + f;
            // past the row's last bin the percussive windows read reflected bins, which A does not hold
            Bp[f * BS + hp + c] = b0 + c < p.K ? U[(f + hh) * TK + c]
                                : t < p.T ? kb_hs_mag(p, kb_hs_off(row, p.C, p.x_sb, p.x_sc, p.x_st, p.x_sk, t,
                                                                   kb_hs_reflect(b0 + c, p.K)))
                                          : 0.0f;
        }
        KB_HS_THREADS_END
        KB_SYNC_CTA;
        // harmonic medians: thread (column c, run) walks frames run RUN .. run RUN + RUN - 1 of the tile
        KB_HS_THREADS_BEGIN
        const int c = tid % TK, f0 = (tid / TK) * KB_HS_RUN;
        const int n = p.T - t0 - f0 < KB_HS_RUN ? p.T - t0 - f0 : KB_HS_RUN;
        if (b0 + c < p.K && n > 0) {
            const float* w = U + f0 * TK + c;
            kb_hs_walk<NSH>(w, TK, kh, n, [&](int i, float m) {
                Hs[(f0 + i) * TK + c] = m;
                if (BWD) sH[(f0 + i) * TK + c] = kb_hs_reflect(t0 + f0 + i - hh + kb_hs_select(w + i * TK, TK, kh, m),
                                                               p.T);
            });
        }
        KB_HS_THREADS_END
        KB_SYNC_CTA;
        // percussive medians: thread (frame f, run) walks bins run RUN .. run RUN + RUN - 1 of the tile; Ps replaces A
        float* Ps = U;
        KB_HS_THREADS_BEGIN
        const int f = tid % TT, c0 = (tid / TT) * KB_HS_RUN;
        const int n = p.K - b0 - c0 < KB_HS_RUN ? p.K - b0 - c0 : KB_HS_RUN;
        if (t0 + f < p.T && n > 0) {
            const float* w = Bp + f * BS + c0;
            kb_hs_walk<NSP>(w, 1, kp, n, [&](int i, float m) {
                Ps[f * PS + c0 + i] = m;
                if (BWD) sP[f * PS + c0 + i] = kb_hs_reflect(b0 + c0 + i - hp + kb_hs_select(w + i, 1, kp, m), p.K);
            });
        }
        KB_HS_THREADS_END
        KB_SYNC_CTA;
        // masks and outputs (forward), or the direct term and the median gradients (backward)
        KB_HS_THREADS_BEGIN
        for (int i = tid; i < TT * TK; i += KB_HS_THREADS) {
            const int f = i / TK, c = i % TK, t = t0 + f, b = b0 + c;
            if (t >= p.T || b >= p.K) continue;
            const float s = Bp[f * BS + hp + c], hv = Hs[f * TK + c], pv = Ps[f * PS + c];
            const float mhv = kb_hs_softmask(p, hv, kb_hs_mul(p.mh, pv));
            const float mpv = kb_hs_softmask(p, pv, kb_hs_mul(p.mp, hv));
            float2 X = make_float2(0.0f, 0.0f);
            if (p.cplx && (BWD || !p.mask))
                X = reinterpret_cast<const float2*>(p.x)[kb_hs_off(row, p.C, p.x_sb, p.x_sc, p.x_st, p.x_sk, t, b)];
            if (!BWD) {
                const float ms[2] = {mhv, mpv};
                for (int q = 0; q < 2; ++q) {
                    void* o = q ? p.op : p.oh;
                    if (!o) continue;
                    const long long oo = q ? kb_hs_off(row, p.C, p.op_sb, p.op_sc, p.op_st, p.op_sk, t, b)
                                           : kb_hs_off(row, p.C, p.oh_sb, p.oh_sc, p.oh_st, p.oh_sk, t, b);
                    if (p.mask) reinterpret_cast<float*>(o)[oo] = ms[q];
                    else if (p.cplx) reinterpret_cast<float2*>(o)[oo] = make_float2(kb_hs_mul(ms[q], X.x),
                                                                                    kb_hs_mul(ms[q], X.y));
                    else reinterpret_cast<float*>(o)[oo] = kb_hs_mul(s, ms[q]);
                }
            } else {
                // output gradients: float, or float2 for the components of a complex input
                float2 g[2] = {make_float2(0.0f, 0.0f), make_float2(0.0f, 0.0f)};
                for (int q = 0; q < 2; ++q) {
                    const void* gq = q ? p.gp : p.gh;
                    if (!gq) continue;
                    const long long go = q ? kb_hs_off(row, p.C, p.gp_sb, p.gp_sc, p.gp_st, p.gp_sk, t, b)
                                           : kb_hs_off(row, p.C, p.gh_sb, p.gh_sc, p.gh_st, p.gh_sk, t, b);
                    g[q] = (p.cplx && !p.mask) ? reinterpret_cast<const float2*>(gq)[go]
                                               : make_float2(reinterpret_cast<const float*>(gq)[go], 0.0f);
                }
                float gm[2];                                    // gradients of the masks
                for (int q = 0; q < 2; ++q)
                    gm[q] = p.mask ? g[q].x : p.cplx ? g[q].x * X.x + g[q].y * X.y : g[q].x * s;
                float dh = 0.0f, dp = 0.0f, da, db;
                kb_hs_dmask(p, hv, p.mh * pv, &da, &db);
                if (gm[0] != 0.0f) { dh += gm[0] * da; dp += gm[0] * db * p.mh; }
                kb_hs_dmask(p, pv, p.mp * hv, &da, &db);
                if (gm[1] != 0.0f) { dp += gm[1] * da; dh += gm[1] * db * p.mp; }
                const long long e = ((row * p.T) + t) * (long long)p.K + b;
                kb_hs_w wv;
                wv.g = dh; wv.src = sH[f * TK + c]; p.wh[e] = wv;
                wv.g = dp; wv.src = sP[f * PS + c]; p.wp[e] = wv;
                const long long xo = kb_hs_off(row, p.C, p.gx_sb, p.gx_sc, p.gx_st, p.gx_sk, t, b);
                if (p.cplx) {
                    const float2 d = p.mask ? make_float2(0.0f, 0.0f)
                                            : make_float2(mhv * g[0].x + mpv * g[1].x, mhv * g[0].y + mpv * g[1].y);
                    reinterpret_cast<float2*>(p.gx)[xo] = d;
                } else {
                    reinterpret_cast<float*>(p.gx)[xo] = p.mask ? 0.0f : mhv * g[0].x + mpv * g[1].x;
                }
            }
        }
        KB_HS_THREADS_END
        KB_SYNC_CTA;
    }
}

// Second gradient pass: element e = (row, t, b) of block `cta` (KB_HS_THREADS elements each) gathers the median
// gradients that selected it and adds them to the direct term.
KB_HS_FN void kb_hpss_gather_cta(const KbHpssParams& p, char*, long long cta, long long n_cta) {
    const long long n = (long long)p.B * p.C * p.T * p.K;
    for (long long e0 = cta * KB_HS_THREADS; e0 < n; e0 += n_cta * KB_HS_THREADS) {
        KB_HS_THREADS_BEGIN
        const long long e = e0 + tid;
        if (e < n) {
            const int b = (int)(e % p.K), t = (int)((e / p.K) % p.T);
            const long long row = e / ((long long)p.T * p.K);
            float acc = 0.0f;
            const int tl = t - p.kh + 1 > 0 ? t - p.kh + 1 : 0, th = t + p.kh - 1 < p.T - 1 ? t + p.kh - 1 : p.T - 1;
            for (int u = tl; u <= th; ++u) {
                const kb_hs_w w = p.wh[e + (long long)(u - t) * p.K];
                if (w.src == t) acc += w.g;
            }
            const int bl = b - p.kp + 1 > 0 ? b - p.kp + 1 : 0, bh = b + p.kp - 1 < p.K - 1 ? b + p.kp - 1 : p.K - 1;
            for (int v = bl; v <= bh; ++v) {
                const kb_hs_w w = p.wp[e + (v - b)];
                if (w.src == b) acc += w.g;
            }
            const long long xo = kb_hs_off(row, p.C, p.gx_sb, p.gx_sc, p.gx_st, p.gx_sk, t, b);
            if (p.cplx) {
                const float2 X = reinterpret_cast<const float2*>(p.x)[kb_hs_off(row, p.C, p.x_sb, p.x_sc, p.x_st,
                                                                                p.x_sk, t, b)];
                const float a = kb_cabs(X.x, X.y);
                const float sa = a > 0.0f ? acc : 0.0f, r = a > 0.0f ? a : 1.0f;
                float2* g = reinterpret_cast<float2*>(p.gx) + xo;
                *g = make_float2(g->x + sa * (X.x / r), g->y + sa * (X.y / r));
            } else {
                float* g = reinterpret_cast<float*>(p.gx) + xo;
                *g = *g + acc;
            }
        }
        KB_HS_THREADS_END
    }
}
