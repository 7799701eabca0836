// Kernel bodies of the chroma features: the projection of a spectrogram onto pitch classes with its per-frame
// threshold and normalisation (forward and backward), librosa's tuning estimate (piptrack peaks, an exact per-item
// median and the residual histogram) and the CENS smoothing.
//
// Projection.  For each frame of a (item, channel) row, y_j = sum_k W[j][k] s_k with s_k the input as it is (a power
// spectrogram or |C|), its square (|X| -> |X|^2) or the modulus of a complex input, each y_j one float32 fmaf chain in
// ascending k.  Then entries below the threshold are set to 0 and the frame is normalised (max |v|, sum |v| or the
// root of the sum of squares; a frame whose length is below FLT_MIN is left as it is).  A CTA takes TF frames of one
// row; thread (f, g) keeps frame f's chroma g CPT .. g CPT + CPT - 1, whose partial sums live in shared memory between
// chunks of KC bins.  So an output's bits depend on (item, channel, frame, chroma) alone, never on the tile, the grid,
// the batch or the strides, and there are no floating-point atomics.  The CENS mode writes the L1-normalised frame
// quantised to q = 0.25 #{s in (0.4, 0.2, 0.1, 0.05) : v > s} instead (NaN stays NaN).
//
// Tuning estimate, per item over all its channels, in a fixed number of launches whatever the data:
//   1. peaks: per frame, ref = 0.1 max_k S_k; bin k in [lo, hi) is a peak when S_k > ref and S' = S (S > ref) has a
//      local maximum there (S'_k > S'_{k-1}, S'_k >= S'_{k+1}).  Two peaks are never adjacent, so peak k goes to slot
//      (k - lo) / 2 of its frame; empty slots hold -1.  A frame holding a non-finite bin has no peaks.  The pass also
//      counts the peaks' top mag byte into the item's first radix histogram (integer atomics, order-free).
//   2-4. radix select of the median's lower rank over the mags' float bits (they are positive): each CTA redoes the
//      item's selection from the finished histograms and counts the next byte of the peaks that still match;
//   5. the smallest mag above that value (integer atomicMin), for the upper rank of an even count;
//   6. the residual histogram of the peaks with mag >= median: r = mod(bpo log2(pitch / 27.5), 1) in [-0.5, 0.5),
//      binned against the plan's float64 edges exactly as numpy.histogram bins;
//   7. per item, the left edge of the first fullest bin (0.0 without peaks) and the index of its filterbank table.
//
// CENS smoothing: out[m] = normalise_2(sum_i w_i q[m + N / 2 - i]) over the N taps (zeros outside the row), one fmaf
// chain in ascending i.
//
// Like the other bodies these are barrier-free phases: under nvcc each phase runs once per thread, separated by CTA
// barriers; the CPU emulation (tests/emu, KB_HOST_EMU) runs each phase as a loop over the CTA's threads.
#pragma once
#include "stft_core.cuh"

#define KB_CH_THREADS 256
#define KB_CH_KC 32                 // bins per staged chunk
#define KB_CH_CPT 16                // chroma per thread
#define KB_CH_MAX_CHROMA 64         // KAPRE_CHROMA_MAX_CHROMA
#define KB_CH_PEAK_TF 8             // frames per peak tile (32 threads each)
#define KB_CH_SEL_TF 32             // frames per selection tile
#define KB_CH_SMOOTH_TF 64          // frames per CENS smoothing tile
#define KB_CH_TINY 1.17549435e-38f  // FLT_MIN

enum { KB_CH_IN_LINEAR = 0, KB_CH_IN_SQUARE = 1, KB_CH_IN_COMPLEX = 2 };
enum { KB_CH_NORM_NONE = 0, KB_CH_NORM_INF = 1, KB_CH_NORM_L1 = 2, KB_CH_NORM_L2 = 3 };

#if defined(KB_HOST_EMU)
#define KB_CH_THREADS_BEGIN for (int tid = 0; tid < KB_CH_THREADS; ++tid) {
#define KB_CH_THREADS_END }
#define KB_CH_FN inline
inline float kb_ch_nan() { return std::nanf(""); }
inline float kb_ch_mul(float a, float b) { return a * b; }
inline float kb_ch_add(float a, float b) { return a + b; }
inline float kb_ch_sub(float a, float b) { return a - b; }
inline float kb_ch_div(float a, float b) { return a / b; }
inline unsigned kb_ch_f2u(float f) { unsigned u; std::memcpy(&u, &f, 4); return u; }
inline float kb_ch_u2f(unsigned u) { float f; std::memcpy(&f, &u, 4); return f; }
inline bool kb_ch_finite(float v) { return std::isfinite(v); }
inline void kb_ch_atomic_add(unsigned* p, unsigned v) { *p += v; }
inline void kb_ch_atomic_min(unsigned* p, unsigned v) { if (v < *p) *p = v; }
#else
#define KB_CH_THREADS_BEGIN { const int tid = threadIdx.x;
#define KB_CH_THREADS_END }
#define KB_CH_FN __device__ __forceinline__
KB_D float kb_ch_nan() { return __int_as_float(0x7fc00000); }
KB_D float kb_ch_mul(float a, float b) { return __fmul_rn(a, b); }
KB_D float kb_ch_add(float a, float b) { return __fadd_rn(a, b); }
KB_D float kb_ch_sub(float a, float b) { return __fsub_rn(a, b); }
KB_D float kb_ch_div(float a, float b) { return __fdiv_rn(a, b); }
KB_D unsigned kb_ch_f2u(float f) { return __float_as_uint(f); }
KB_D float kb_ch_u2f(unsigned u) { return __uint_as_float(u); }
KB_D bool kb_ch_finite(float v) { return isfinite(v); }
KB_D void kb_ch_atomic_add(unsigned* p, unsigned v) { atomicAdd(p, v); }
KB_D void kb_ch_atomic_min(unsigned* p, unsigned v) { atomicMin(p, v); }
#endif

// ---- projection ---------------------------------------------------------------------------------------------------
struct KbChromaParams {
    int NC, K;                            // chroma, input bins
    int in_mode, norm, cens;              // cens: write the quantised L1-normalised frame
    int has_thr;
    float thr;
    const float* W;                       // [table][NC][K]
    const int* tab;                       // per item table index (device), or null: table 0
    int G, TF;                            // chroma groups of CPT, frames per tile (KB_CH_THREADS / G)
    int B, C, M;
    long long tiles, jobs;
    const void* x;                        // float, or float2 for KB_CH_IN_COMPLEX; element strides (b, c, t, k)
    long long x_sb, x_sc, x_st, x_sk;
    float* out;                           // element strides (b, c, t, j)
    long long o_sb, o_sc, o_st, o_sk;
    // backward
    const float* g;                       // gradient of the output, element strides (b, c, t, j)
    long long g_sb, g_sc, g_st, g_sk;
    void* gx;                             // gradient of the input (float, or float2), element strides (b, c, t, k)
    long long gx_sb, gx_sc, gx_st, gx_sk;
};

inline void kb_chroma_tiling(KbChromaParams& p) {
    p.G = (p.NC + KB_CH_CPT - 1) / KB_CH_CPT;
    p.TF = KB_CH_THREADS / p.G;
}

inline bool kb_chroma_setup(KbChromaParams& p) {
    p.tiles = ((long long)p.M + p.TF - 1) / p.TF;
    p.jobs = (long long)p.B * p.C * p.tiles;
    return p.jobs < (1LL << 40);
}

// Shared memory: staged input [TF][KC + 1], the chunk's table [KC][G CPT] (forward) or [NC][KC + 1] (backward), and
// per-frame chroma [TF][G CPT].
KB_HD int kb_chroma_wfloats(int NC, int G) {
    const int a = KB_CH_KC * G * KB_CH_CPT, b = NC * (KB_CH_KC + 1);
    return a > b ? a : b;
}
KB_HD int kb_chroma_smem(int NC, int G, int TF) {
    return (TF * (KB_CH_KC + 1) + kb_chroma_wfloats(NC, G) + TF * G * KB_CH_CPT) * 4;
}

// The input value s_k of element offset o.
KB_CH_FN float kb_chroma_in(const KbChromaParams& p, long long o) {
    if (p.in_mode == KB_CH_IN_COMPLEX) {
        const float2 c = reinterpret_cast<const float2*>(p.x)[o];
        return kb_cabs<true>(c.x, c.y);
    }
    const float v = reinterpret_cast<const float*>(p.x)[o];
    return p.in_mode == KB_CH_IN_SQUARE ? kb_ch_mul(v, v) : v;
}

// The thresholded value of y (entries below the threshold set to 0).
KB_HD float kb_chroma_thr(float y, int has_thr, float thr) { return (has_thr && y < thr) ? 0.0f : y; }

// Length of a frame's thresholded chroma y[0 .. n) under `norm` (1 when it is below FLT_MIN), in ascending order;
// *imax: the first index of the maximum (norm inf).
KB_HD float kb_chroma_length(const float* y, int n, int norm, int has_thr, float thr, int* imax) {
    float len = 0.0f;
    *imax = 0;
    if (norm == KB_CH_NORM_INF) {
        for (int j = 0; j < n; ++j) {
            const float a = fabsf(kb_chroma_thr(y[j], has_thr, thr));
            if (a > len || (a != a && len == len)) { len = a; *imax = j; }
        }
    } else if (norm == KB_CH_NORM_L1) {
        for (int j = 0; j < n; ++j) len = len + fabsf(kb_chroma_thr(y[j], has_thr, thr));
    } else if (norm == KB_CH_NORM_L2) {
        for (int j = 0; j < n; ++j) {
            const float v = kb_chroma_thr(y[j], has_thr, thr);
            len = fmaf(v, v, len);
        }
        len = sqrtf(len);
    } else {
        return 1.0f;
    }
    return len < KB_CH_TINY ? 1.0f : len;
}

KB_HD float kb_chroma_quant(float v) {
    if (v != v) return v;
    return 0.25f * (float)((v > 0.4f) + (v > 0.2f) + (v > 0.1f) + (v > 0.05f));
}

// y_j of the tile's frames into ys[f][G CPT] (partial sums staged between chunks).  Shared by forward and backward.
KB_CH_FN void kb_chroma_project(const KbChromaParams& p, float* xs, float* ws, float* ys, long long row, int m0,
                                const float* W) {
    const int TF = p.TF, NCP = p.G * KB_CH_CPT, KS = KB_CH_KC + 1;
    const long long xb = (row / p.C) * p.x_sb + (row % p.C) * p.x_sc;
    KB_CH_THREADS_BEGIN
    for (int i = tid; i < TF * NCP; i += KB_CH_THREADS) ys[i] = 0.0f;
    KB_CH_THREADS_END
    for (int k0 = 0; k0 < p.K; k0 += KB_CH_KC) {
        const int kn = p.K - k0 < KB_CH_KC ? p.K - k0 : KB_CH_KC;
        KB_SYNC_CTA;
        KB_CH_THREADS_BEGIN
        for (int i = tid; i < TF * KB_CH_KC; i += KB_CH_THREADS) {
            const int f = i / KB_CH_KC, kk = i % KB_CH_KC, m = m0 + f;
            xs[f * KS + kk] = (m < p.M && kk < kn) ? kb_chroma_in(p, xb + m * p.x_st + (long long)(k0 + kk) * p.x_sk)
                                                   : 0.0f;
        }
        for (int i = tid; i < KB_CH_KC * NCP; i += KB_CH_THREADS) {
            const int j = i / KB_CH_KC, kk = i % KB_CH_KC;
            ws[kk * NCP + j] = (j < p.NC && kk < kn) ? W[(long long)j * p.K + k0 + kk] : 0.0f;
        }
        KB_CH_THREADS_END
        KB_SYNC_CTA;
        KB_CH_THREADS_BEGIN
        const int f = tid % TF, g = tid / TF;       // the last tid % G threads idle when G does not divide it
        float acc[KB_CH_CPT];
        if (g < p.G) {
#pragma unroll
            for (int j = 0; j < KB_CH_CPT; ++j) acc[j] = ys[f * NCP + g * KB_CH_CPT + j];
            for (int kk = 0; kk < kn; ++kk) {
                const float s = xs[f * KS + kk];
                const float* wr = ws + kk * NCP + g * KB_CH_CPT;
#pragma unroll
                for (int j = 0; j < KB_CH_CPT; ++j) acc[j] = fmaf(wr[j], s, acc[j]);
            }
#pragma unroll
            for (int j = 0; j < KB_CH_CPT; ++j) ys[f * NCP + g * KB_CH_CPT + j] = acc[j];
        }
        KB_CH_THREADS_END
    }
    KB_SYNC_CTA;
}

KB_CH_FN const float* kb_chroma_table(const KbChromaParams& p, long long row) {
    const long long t = p.tab ? p.tab[row / p.C] : 0;
    return p.W + t * p.NC * (long long)p.K;
}

KB_CH_FN void kb_chroma_cta(const KbChromaParams& p, char* smem, long long cta, long long n_cta) {
    const int TF = p.TF, NCP = p.G * KB_CH_CPT, NC = p.NC;
    float* xs = reinterpret_cast<float*>(smem);
    float* ws = xs + TF * (KB_CH_KC + 1);
    float* ys = ws + kb_chroma_wfloats(NC, p.G);
    for (long long job = cta; job < p.jobs; job += n_cta) {
        const long long row = job / p.tiles;
        const int m0 = (int)(job % p.tiles) * TF;
        kb_chroma_project(p, xs, ws, ys, row, m0, kb_chroma_table(p, row));
        KB_CH_THREADS_BEGIN
        const int f = tid % TF, g = tid / TF, m = m0 + f;
        if (m < p.M) {
            const float* yr = ys + f * NCP;
            int imax;
            const float len = kb_chroma_length(yr, NC, p.cens ? KB_CH_NORM_L1 : p.norm, p.has_thr, p.thr, &imax);
            const long long ob = (row / p.C) * p.o_sb + (row % p.C) * p.o_sc + m * p.o_st;
            for (int j = g * KB_CH_CPT; j < NC && j < (g + 1) * KB_CH_CPT; ++j) {
                const float o = kb_ch_div(kb_chroma_thr(yr[j], p.has_thr, p.thr), len);
                p.out[ob + j * p.o_sk] = p.cens ? kb_chroma_quant(o) : o;
            }
        }
        KB_CH_THREADS_END
        KB_SYNC_CTA;
    }
}

// Backward: recompute y, take the output gradient back through the normalisation and the threshold (in place in ys),
// then through W (sum over j ascending) and the input mode.
KB_CH_FN void kb_chroma_bwd_cta(const KbChromaParams& p, char* smem, long long cta, long long n_cta) {
    const int TF = p.TF, NCP = p.G * KB_CH_CPT, NC = p.NC, KS = KB_CH_KC + 1;
    float* xs = reinterpret_cast<float*>(smem);
    float* ws = xs + TF * KS;
    float* ys = ws + kb_chroma_wfloats(NC, p.G);
    for (long long job = cta; job < p.jobs; job += n_cta) {
        const long long row = job / p.tiles;
        const int m0 = (int)(job % p.tiles) * TF;
        const float* W = kb_chroma_table(p, row);
        kb_chroma_project(p, xs, ws, ys, row, m0, W);
        KB_CH_THREADS_BEGIN
        const int f = tid;
        if (f < TF) {
            float* yr = ys + f * NCP;
            const int m = m0 + f;
            if (m < p.M) {
                int imax;
                const float len = kb_chroma_length(yr, NC, p.norm, p.has_thr, p.thr, &imax);
                const bool small = p.norm == KB_CH_NORM_NONE || len < KB_CH_TINY;
                const long long gb = (row / p.C) * p.g_sb + (row % p.C) * p.g_sc + m * p.g_st;
                float dot = 0.0f;
                for (int j = 0; j < NC; ++j) dot = fmaf(p.g[gb + j * p.g_sk], kb_chroma_thr(yr[j], p.has_thr, p.thr), dot);
                const float dl = (dot / len) / len;   // dot / len^2: len^2 itself leaves the float range below 2^-63
                for (int j = 0; j < NC; ++j) {
                    const float gj = p.g[gb + j * p.g_sk];
                    const float v = kb_chroma_thr(yr[j], p.has_thr, p.thr);
                    float gv;
                    if (small) {
                        gv = gj;
                    } else {
                        const float sg = v > 0.0f ? 1.0f : (v < 0.0f ? -1.0f : 0.0f);
                        gv = gj / len;
                        if (p.norm == KB_CH_NORM_L1) gv = gv - sg * dl;
                        else if (p.norm == KB_CH_NORM_L2) gv = gv - v * (dl / len);
                        else if (j == imax) gv = gv - sg * dl;
                    }
                    yr[j] = (p.has_thr && yr[j] < p.thr) ? 0.0f : gv;
                }
            } else {
                for (int j = 0; j < NC; ++j) yr[j] = 0.0f;
            }
        }
        KB_CH_THREADS_END
        const long long xb = (row / p.C) * p.x_sb + (row % p.C) * p.x_sc;
        const long long gxb = (row / p.C) * p.gx_sb + (row % p.C) * p.gx_sc;
        for (int k0 = 0; k0 < p.K; k0 += KB_CH_KC) {
            const int kn = p.K - k0 < KB_CH_KC ? p.K - k0 : KB_CH_KC;
            KB_SYNC_CTA;
            KB_CH_THREADS_BEGIN
            for (int i = tid; i < NC * KB_CH_KC; i += KB_CH_THREADS) {
                const int j = i / KB_CH_KC, kk = i % KB_CH_KC;
                ws[j * KS + kk] = kk < kn ? W[(long long)j * p.K + k0 + kk] : 0.0f;
            }
            KB_CH_THREADS_END
            KB_SYNC_CTA;
            KB_CH_THREADS_BEGIN
            for (int i = tid; i < TF * KB_CH_KC; i += KB_CH_THREADS) {
                const int f = i / KB_CH_KC, kk = i % KB_CH_KC, m = m0 + f;
                if (m >= p.M || kk >= kn) continue;
                const float* gy = ys + f * NCP;
                float s = 0.0f;
                for (int j = 0; j < NC; ++j) s = fmaf(ws[j * KS + kk], gy[j], s);
                const long long xo = xb + m * p.x_st + (long long)(k0 + kk) * p.x_sk;
                const long long go = gxb + m * p.gx_st + (long long)(k0 + kk) * p.gx_sk;
                if (p.in_mode == KB_CH_IN_COMPLEX) {
                    const float2 c = reinterpret_cast<const float2*>(p.x)[xo];
                    // s (C / |C|): s / |C| overflows for a tiny C whose s scales as 1 / |C|
                    const float a = kb_cabs<true>(c.x, c.y);
                    const float sa = a > 0.0f ? s : 0.0f, r = a > 0.0f ? a : 1.0f;
                    reinterpret_cast<float2*>(p.gx)[go] = make_float2(sa * (c.x / r), sa * (c.y / r));
                } else if (p.in_mode == KB_CH_IN_SQUARE) {
                    const float a = reinterpret_cast<const float*>(p.x)[xo];
                    reinterpret_cast<float*>(p.gx)[go] = (2.0f * a) * s;
                } else {
                    reinterpret_cast<float*>(p.gx)[go] = s;
                }
            }
            KB_CH_THREADS_END
        }
        KB_SYNC_CTA;
    }
}

// ---- tuning estimate --------------------------------------------------------------------------------------------------
struct KbTuneParams {
    int K, lo, hi, cap;                   // bins, peak range [lo, hi), slots per frame ((hi - lo + 1) / 2)
    int in_mode;                          // KB_CH_IN_LINEAR or KB_CH_IN_SQUARE
    float sr, nfft;
    double bpo;
    int nres;                             // residual histogram bins
    const double* edges;                  // [nres + 1]
    int pass;                             // selection launches: 1 .. 3 radix bytes, 4 min above, 5 residual histogram
    int B, C, M;
    long long tiles, jobs;
    const float* x;
    long long x_sb, x_sc, x_st, x_sk;
    float* mag;                           // [row][M][cap]
    float* pitch;
    unsigned* hist;                       // [item][4][256]
    unsigned* above;                      // [item]
    unsigned* res;                        // [item][nres]
    double* tuning;                       // [item]
    int* tab;                             // [item]: the filterbank table of the estimate (nres without peaks)
};

KB_HD int kb_tune_peak_smem() { return (2 * KB_CH_THREADS + 2 * KB_CH_PEAK_TF + 256) * 4; }
KB_HD int kb_tune_sel_smem() { return (1024 + 8) * 4; }

// The median's state from the item's finished histograms of bytes 0 .. d - 1: sel[0] = matched prefix, sel[1] =
// remaining rank, sel[2] = count, sel[3] = elements equal to the prefix after the last byte (d = 4).
KB_HD void kb_tune_select(const unsigned* h, int d, unsigned* sel) {
    unsigned n = 0;
    for (int b = 0; b < 256; ++b) n += h[b];
    unsigned r = n ? (n - 1) / 2 : 0, pre = 0, eq = 0;
    for (int i = 0; i < d; ++i) {
        unsigned cum = 0;
        int b = 0;
        for (; b < 255; ++b) {
            if (cum + h[i * 256 + b] > r) break;
            cum += h[i * 256 + b];
        }
        r -= cum;
        pre = (pre << 8) | (unsigned)b;
        eq = h[i * 256 + b];
    }
    sel[0] = pre; sel[1] = r; sel[2] = n; sel[3] = eq;
}

KB_CH_FN float kb_tune_in(const KbTuneParams& p, long long o) {
    const float v = p.x[o];
    return p.in_mode == KB_CH_IN_SQUARE ? kb_ch_mul(v, v) : v;
}

// Pass 0: peaks of KB_CH_PEAK_TF frames of one row, 32 threads per frame.
KB_CH_FN void kb_tune_peak_cta(const KbTuneParams& p, char* smem, long long cta, long long n_cta) {
    float* red = reinterpret_cast<float*>(smem);
    int* bad = reinterpret_cast<int*>(red + KB_CH_THREADS);
    float* ref = reinterpret_cast<float*>(bad + KB_CH_THREADS);
    int* fbad = reinterpret_cast<int*>(ref + KB_CH_PEAK_TF);
    unsigned* hs = reinterpret_cast<unsigned*>(fbad + KB_CH_PEAK_TF);
    for (long long job = cta; job < p.jobs; job += n_cta) {
        const long long row = job / p.tiles;
        const int m0 = (int)(job % p.tiles) * KB_CH_PEAK_TF;
        const long long xb = (row / p.C) * p.x_sb + (row % p.C) * p.x_sc;
        KB_CH_THREADS_BEGIN
        hs[tid] = 0u;
        const int f = tid / 32, l = tid % 32, m = m0 + f;
        float mx = 0.0f;
        int nf = 0;
        if (m < p.M) {
            for (int k = l; k < p.K; k += 32) {
                const float s = kb_tune_in(p, xb + m * p.x_st + k * p.x_sk);
                if (!kb_ch_finite(s)) nf = 1;
                else if (s > mx) mx = s;
            }
        }
        red[tid] = mx;
        bad[tid] = nf;
        KB_CH_THREADS_END
        KB_SYNC_CTA;
        KB_CH_THREADS_BEGIN
        if (tid < KB_CH_PEAK_TF) {
            float mx = 0.0f;
            int nf = 0;
            for (int l = 0; l < 32; ++l) {
                if (red[tid * 32 + l] > mx) mx = red[tid * 32 + l];
                nf |= bad[tid * 32 + l];
            }
            ref[tid] = kb_ch_mul(0.1f, mx);
            fbad[tid] = nf;
        }
        KB_CH_THREADS_END
        KB_SYNC_CTA;
        KB_CH_THREADS_BEGIN
        const int f = tid / 32, l = tid % 32, m = m0 + f;
        if (m < p.M) {
            const long long fo = (row * p.M + m) * (long long)p.cap;
            const float rf = ref[f];
            for (int s = l; s < p.cap; s += 32) {
                float mg = -1.0f, pt = -1.0f;
                if (!fbad[f]) {
                    for (int k = p.lo + 2 * s; k < p.lo + 2 * s + 2 && k < p.hi; ++k) {
                        const long long o = xb + m * p.x_st;
                        const float sm = kb_tune_in(p, o + (k - 1) * p.x_sk);
                        const float s0 = kb_tune_in(p, o + k * p.x_sk);
                        const float sp = kb_tune_in(p, o + (k + 1) * p.x_sk);
                        if (!(s0 > rf)) continue;
                        const float tm = sm > rf ? sm : 0.0f, tp = sp > rf ? sp : 0.0f;
                        if (!(s0 > tm && s0 >= tp)) continue;
                        const float a = kb_ch_mul(0.5f, kb_ch_sub(sp, sm));
                        const float d = kb_ch_sub(kb_ch_sub(kb_ch_mul(2.0f, s0), sp), sm);
                        const float sh = fabsf(d) < KB_CH_TINY ? 0.0f : kb_ch_div(a, d);
                        pt = kb_ch_div(kb_ch_mul(kb_ch_add((float)k, sh), p.sr), p.nfft);
                        mg = kb_ch_add(s0, kb_ch_mul(kb_ch_mul(0.5f, a), sh));
                    }
                }
                p.mag[fo + s] = mg;
                p.pitch[fo + s] = pt;
                if (mg >= 0.0f) kb_ch_atomic_add(hs + (kb_ch_f2u(mg) >> 24), 1u);
            }
        }
        KB_CH_THREADS_END
        KB_SYNC_CTA;
        KB_CH_THREADS_BEGIN
        if (hs[tid]) kb_ch_atomic_add(p.hist + (row / p.C) * 1024 + tid, hs[tid]);
        KB_CH_THREADS_END
        KB_SYNC_CTA;
    }
}

// numpy.histogram's bin of x over uniform float64 edges e[0 .. n] (the last bin closed), or -1 outside them.
KB_HD int kb_tune_bin(double x, const double* e, int n) {
    if (!(x >= e[0] && x <= e[n])) return -1;
    int i = (int)((x - e[0]) * ((double)n / (e[n] - e[0])));
    if (i >= n) i = n - 1;
    if (i < 0) i = 0;
    if (x < e[i]) --i;
    else if (i != n - 1 && x >= e[i + 1]) ++i;
    return i;
}

// Passes 1 .. 5 over the slots of KB_CH_SEL_TF frames of one row.
KB_CH_FN void kb_tune_sel_cta(const KbTuneParams& p, char* smem, long long cta, long long n_cta) {
    unsigned* hs = reinterpret_cast<unsigned*>(smem);           // 1024: the item's histograms, then this pass's counts
    unsigned* sel = hs + 1024;                                  // 8: selection state
    const int d = p.pass < 4 ? p.pass : 4;
    for (long long job = cta; job < p.jobs; job += n_cta) {
        const long long row = job / p.tiles, item = row / p.C;
        const int m0 = (int)(job % p.tiles) * KB_CH_SEL_TF;
        KB_CH_THREADS_BEGIN
        for (int i = tid; i < 1024; i += KB_CH_THREADS) hs[i] = p.hist[item * 1024 + i];
        KB_CH_THREADS_END
        KB_SYNC_CTA;
        KB_CH_THREADS_BEGIN
        if (tid == 0) {
            kb_tune_select(hs, d, sel);
            // the median: the lower rank's value, or for an even count the mean with the next larger order statistic
            float med = kb_ch_u2f(sel[0]);
            if (p.pass == 5 && sel[2] % 2 == 0) {
                const unsigned le = (sel[2] - 1) / 2 - sel[1] + sel[3];   // elements <= the lower rank's value
                const float hi = le > sel[2] / 2 ? med : kb_ch_u2f(p.above[item]);
                med = kb_ch_mul(0.5f, kb_ch_add(med, hi));
            }
            sel[4] = kb_ch_f2u(med);
            sel[5] = 0xffffffffu;
        }
        KB_CH_THREADS_END
        KB_SYNC_CTA;
        KB_CH_THREADS_BEGIN
        for (int i = tid; i < 1024; i += KB_CH_THREADS) hs[i] = 0u;
        KB_CH_THREADS_END
        KB_SYNC_CTA;
        const unsigned pre = sel[0], n = sel[2];
        const float med = kb_ch_u2f(sel[4]);
        KB_CH_THREADS_BEGIN
        const int nf = (p.M - m0 < KB_CH_SEL_TF ? p.M - m0 : KB_CH_SEL_TF) * p.cap;
        const long long base = (row * p.M + m0) * (long long)p.cap;
        if (n) {
            for (int i = tid; i < nf; i += KB_CH_THREADS) {
                const float mg = p.mag[base + i];
                if (!(mg >= 0.0f)) continue;
                const unsigned key = kb_ch_f2u(mg);
                if (p.pass < 4) {
                    if ((key >> (32 - 8 * d)) == pre) kb_ch_atomic_add(hs + ((key >> (24 - 8 * d)) & 255u), 1u);
                } else if (p.pass == 4) {
                    if (key > pre) kb_ch_atomic_min(sel + 5, key);
                } else if (mg >= med) {
                    double r = p.bpo * log2((double)p.pitch[base + i] / 27.5);
                    r = fmod(r, 1.0);
                    if (r < 0.0) r += 1.0;
                    if (r >= 0.5) r -= 1.0;
                    const int b = kb_tune_bin(r, p.edges, p.nres);
                    if (b >= 0) kb_ch_atomic_add(hs + b, 1u);
                }
            }
        }
        KB_CH_THREADS_END
        KB_SYNC_CTA;
        KB_CH_THREADS_BEGIN
        if (p.pass < 4) {
            if (hs[tid]) kb_ch_atomic_add(p.hist + item * 1024 + d * 256 + tid, hs[tid]);
        } else if (p.pass == 4) {
            if (tid == 0 && sel[5] != 0xffffffffu) kb_ch_atomic_min(p.above + item, sel[5]);
        } else {
            for (int b = tid; b < p.nres && b < 1024; b += KB_CH_THREADS)
                if (hs[b]) kb_ch_atomic_add(p.res + item * (long long)p.nres + b, hs[b]);
        }
        KB_CH_THREADS_END
        KB_SYNC_CTA;
    }
}

// Pass 6: per item the first fullest residual bin; its left edge is the tuning.
KB_CH_FN void kb_tune_argmax_cta(const KbTuneParams& p, char* smem, long long cta, long long n_cta) {
    unsigned* bc = reinterpret_cast<unsigned*>(smem);
    int* bi = reinterpret_cast<int*>(bc + KB_CH_THREADS);
    for (long long item = cta; item < p.B; item += n_cta) {
        const unsigned* h = p.res + item * (long long)p.nres;
        KB_CH_THREADS_BEGIN
        unsigned best = 0;
        int at = p.nres;
        for (int b = tid; b < p.nres; b += KB_CH_THREADS)
            if (h[b] > best) { best = h[b]; at = b; }
        bc[tid] = best;
        bi[tid] = at;
        KB_CH_THREADS_END
        KB_SYNC_CTA;
        KB_CH_THREADS_BEGIN
        if (tid == 0) {
            unsigned best = 0;
            int at = p.nres;
            for (int t = 0; t < KB_CH_THREADS; ++t)
                if (bc[t] > best || (bc[t] == best && best > 0 && bi[t] < at)) { best = bc[t]; at = bi[t]; }
            p.tuning[item] = at < p.nres ? p.edges[at] : 0.0;
            p.tab[item] = at;
        }
        KB_CH_THREADS_END
        KB_SYNC_CTA;
    }
}

// ---- CENS smoothing ---------------------------------------------------------------------------------------------------
struct KbCensParams {
    int NC, N;                            // chroma, taps
    const float* w;                       // [N]
    int B, C, M;
    long long tiles, jobs;
    const float* q;                       // [row][M][NC]
    float* out;                           // element strides (b, c, t, j)
    long long o_sb, o_sc, o_st, o_sk;
};

KB_HD int kb_cens_smem(int NC, int N) {
    return ((KB_CH_SMOOTH_TF + N) * NC + N + KB_CH_SMOOTH_TF * NC) * 4;
}

KB_CH_FN void kb_cens_cta(const KbCensParams& p, char* smem, long long cta, long long n_cta) {
    const int NC = p.NC, N = p.N, TF = KB_CH_SMOOTH_TF, H = N / 2, SPAN = TF + N - 1;
    float* qs = reinterpret_cast<float*>(smem);                 // [SPAN][NC]: frames m0 - (N - 1 - H) ..
    float* ws = qs + (TF + N) * NC;
    float* ys = ws + N;                                         // [TF][NC]
    for (long long job = cta; job < p.jobs; job += n_cta) {
        const long long row = job / p.tiles;
        const int m0 = (int)(job % p.tiles) * TF;
        const int a0 = m0 - (N - 1 - H);
        KB_CH_THREADS_BEGIN
        for (int i = tid; i < SPAN * NC; i += KB_CH_THREADS) {
            const int m = a0 + i / NC;
            qs[i] = (m >= 0 && m < p.M) ? p.q[(row * p.M + m) * NC + i % NC] : 0.0f;
        }
        for (int i = tid; i < N; i += KB_CH_THREADS) ws[i] = p.w[i];
        KB_CH_THREADS_END
        KB_SYNC_CTA;
        KB_CH_THREADS_BEGIN
        for (int i = tid; i < TF * NC; i += KB_CH_THREADS) {
            const int f = i / NC, j = i % NC;
            // q[m + H - t] sits at staged frame f + H - t + (N - 1 - H) = f + N - 1 - t
            float s = 0.0f;
            for (int t = 0; t < N; ++t) s = fmaf(ws[t], qs[(f + N - 1 - t) * NC + j], s);
            ys[i] = s;
        }
        KB_CH_THREADS_END
        KB_SYNC_CTA;
        KB_CH_THREADS_BEGIN
        for (int i = tid; i < TF * NC; i += KB_CH_THREADS) {
            const int f = i / NC, j = i % NC, m = m0 + f;
            if (m >= p.M) continue;
            int imax;
            const float len = kb_chroma_length(ys + f * NC, NC, KB_CH_NORM_L2, 0, 0.0f, &imax);
            p.out[(row / p.C) * p.o_sb + (row % p.C) * p.o_sc + m * p.o_st + j * p.o_sk] = kb_ch_div(ys[i], len);
        }
        KB_CH_THREADS_END
        KB_SYNC_CTA;
    }
}
