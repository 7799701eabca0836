// Kernel bodies of onset detection and beat tracking (modelled on librosa 0.10's onset.onset_strength,
// feature.tempogram, feature.tempo, onset.onset_detect and beat.beat_track): onset strength and its gradient, the
// autocorrelation tempogram, the tempo decision, peak picking and the dynamic-programming beat tracker.
//
// A row is one (item, channel) pair; every output's bits depend only on its row's data (onset strength: its row of S).
//
// Onset strength.  A job is a tile of KbOnsetParams::F output frames of one row.  Output frame t >= P reads frame
// u = t - P + lag of S and frame u - lag; it stages S[u] and the frame u - lag padded with -inf to K + m - 1 bins
// (m = max_size), takes the window maximum R[b] = max S[u - lag][b - m/2 .. b - m/2 + m - 1] by doubling (log2 m
// passes over ping-pong buffers; a tie goes to the lower bin, a NaN wins), forms D = max(0, S[u] - R) (NaN kept) and
// aggregates: 'mean' as a float64 sum in ascending bin order divided by K, 'median' by an exact radix selection over
// the float bits of D (D >= +0, so the bits order as the values; four 8-bit passes per selected rank, integer shared
// atomics for the histograms).  The gradient is two launches over a workspace of 8 bytes per element: the first
// recomputes the tile and writes, per (u, b), the gradient reaching D[u][b] and the bin R[u - lag][b] came from;
// the second gathers per element of S its own term and the terms of frame v + lag whose maximum it was, in
// ascending bin order.  No floating-point atomics.
//
// Tempogram.  A job is a tile of frames of one row: it stages the padded envelope span (ramps computed at staging),
// applies the periodic Hann window, and each thread accumulates 8 consecutive lags of one frame as float32 fma
// chains in ascending j, then the frame is divided by its largest |ac| (norm = inf).
//
// Tempo, peak picking and beat tracking run one CTA per row (tempo with aggregate None: per (row, frame)).  The beat
// tracker's dynamic programme advances S = max(1, rint(p / 2)) frames per step: frame i reads cumulative scores at
// i - 2p .. i - rint(p / 2) only, so the S frames of a step are independent.
//
// Like the other bodies these are barrier-free phases: under nvcc each phase runs once per thread, separated by CTA
// barriers; the CPU emulation (tests/emu, KB_HOST_EMU) runs each phase as a loop over the CTA's threads.  Where a
// product feeds a sum the code writes the fma or keeps them apart, so both builds round alike.
#pragma once
#include <climits>
#include "stft_core.cuh"

#define KB_RH_THREADS 128
#define KB_RH_MAX_BINS 4097          // KAPRE_ONSET_MAX_BINS
#define KB_RH_MAX_WIN 4096           // KAPRE_TEMPOGRAM_MAX_WIN
#define KB_RH_MAX_PERIOD 4096        // KAPRE_BEAT_MAX_PERIOD
#define KB_RH_TINY 1.17549435e-38f   // FLT_MIN
#define KB_RH_LAGS 8                 // lags per tempogram task
#define KB_RH_SMEM_BUDGET (96 * 1024)

enum { KB_RH_AGG_MEAN = 0, KB_RH_AGG_MEDIAN = 1 };

#if defined(KB_HOST_EMU)
#include <cstring>
#define KB_RH_THREADS_BEGIN for (int tid = 0; tid < KB_RH_THREADS; ++tid) {
#define KB_RH_THREADS_END }
#define KB_RH_FN inline
inline float kb_rh_nanf() { return std::nanf(""); }
inline double kb_rh_nan() { return std::nan(""); }
inline float kb_rh_inff() { return INFINITY; }
inline double kb_rh_inf() { return INFINITY; }
inline unsigned kb_rh_fbits(float v) { unsigned u; std::memcpy(&u, &v, 4); return u; }
inline float kb_rh_bitsf(unsigned u) { float v; std::memcpy(&v, &u, 4); return v; }
inline unsigned long long kb_rh_dbits(double v) { unsigned long long u; std::memcpy(&u, &v, 8); return u; }
inline double kb_rh_bitsd(unsigned long long u) { double v; std::memcpy(&v, &u, 8); return v; }
inline void kb_rh_atomic_add(int* p, int v) { *p += v; }
inline double kb_rh_rint(double x) { return std::nearbyint(x); }
inline double kb_rh_cospi(double x) { return std::cos(3.141592653589793 * x); }
#else
#define KB_RH_THREADS_BEGIN { const int tid = threadIdx.x;
#define KB_RH_THREADS_END }
#define KB_RH_FN __device__ __forceinline__
KB_D float kb_rh_nanf() { return __int_as_float(0x7fc00000); }
KB_D double kb_rh_nan() { return __longlong_as_double(0x7ff8000000000000LL); }
KB_D float kb_rh_inff() { return __int_as_float(0x7f800000); }
KB_D double kb_rh_inf() { return __longlong_as_double(0x7ff0000000000000LL); }
KB_D unsigned kb_rh_fbits(float v) { return __float_as_uint(v); }
KB_D float kb_rh_bitsf(unsigned u) { return __uint_as_float(u); }
KB_D unsigned long long kb_rh_dbits(double v) { return (unsigned long long)__double_as_longlong(v); }
KB_D double kb_rh_bitsd(unsigned long long u) { return __longlong_as_double((long long)u); }
KB_D void kb_rh_atomic_add(int* p, int v) { atomicAdd(p, v); }
KB_D double kb_rh_rint(double x) { return rint(x); }
KB_D double kb_rh_cospi(double x) { return cospi(x); }
#endif

KB_HD long long kb_rh_off3(long long row, int C, long long sb, long long sc, long long st, int t) {
    return (row / C) * sb + (row % C) * sc + (long long)t * st;
}

// ---------------------------------------------------------------------------------------------------- onset strength
struct alignas(8) kb_on_w { float g; int src; };

struct KbOnsetParams {
    int B, C, T, K;
    int lag, m, agg, P;                   // P = lag + (n_fft / (2 hop) when centred)
    int F, levels;                        // frames per tile, floor(log2 m)
    long long tiles, jobs;
    const float* x;                       // S, element strides (b, c, t, k)
    long long x_sb, x_sc, x_st, x_sk;
    float* out;                           // envelope, strides (b, c, t)
    long long o_sb, o_sc, o_st;
    // backward
    const float* g;                       // gradient of the envelope, strides (b, c, t)
    long long g_sb, g_sc, g_st;
    float* gx;                            // gradient of S, strides (b, c, t, k)
    long long gx_sb, gx_sc, gx_st, gx_sk;
    kb_on_w* ws;                          // [row][u][b]
};

// Shared memory per frame (4-byte words): D row K, two padded value rows and (backward) two index rows of
// K + m - 1, a 256-bin histogram and 8 + 4 scalars.
KB_HD int kb_onset_frame_words(int K, int m, int bwd) {
    const int n = K + m - 1;
    return K + 2 * n + (bwd ? 2 * n : 0) + 256 + 12;
}
KB_HD int kb_onset_tile_frames(int K, int m, int bwd) {
    int f = (KB_RH_SMEM_BUDGET / 4) / kb_onset_frame_words(K, m, bwd);
    if (f > 32) f = 32;
    return f < 1 ? 1 : f;
}
KB_HD int kb_onset_smem(int K, int m, int F, int bwd) { return F * kb_onset_frame_words(K, m, bwd) * 4; }

inline bool kb_onset_setup(KbOnsetParams& p, int bwd) {
    p.F = kb_onset_tile_frames(p.K, p.m, bwd);
    p.levels = 0;
    while ((2 << p.levels) <= p.m) ++p.levels;
    p.tiles = ((long long)p.T + p.F - 1) / p.F;
    p.jobs = (long long)p.B * p.C * p.tiles;
    return p.jobs < (1LL << 40);
}

// (a, ia) vs (b, ib): the larger value, a NaN first, the lower index on a tie.
KB_RH_FN void kb_rh_pick(float a, int ia, float b, int ib, float* v, int* i) {
    bool ta;
    if (a != a) ta = !(b != b) || ia <= ib;
    else if (b != b) ta = false;
    else ta = a > b || (a == b && ia <= ib);
    *v = ta ? a : b;
    *i = ta ? ia : ib;
}

// Forward (BWD = 0) or first gradient pass (BWD = 1) over one tile of output frames per job.
template <int BWD>
KB_RH_FN void kb_onset_cta(const KbOnsetParams& p, char* smem, long long cta, long long n_cta) {
    const int K = p.K, m = p.m, F = p.F, n = K + m - 1, hm = m / 2, lag = p.lag, P = p.P;
    const int W = kb_onset_frame_words(K, m, BWD);
    float* base = reinterpret_cast<float*>(smem);
    // per frame f: D [K], V0 [n], V1 [n], (I0 [n], I1 [n]), hist [256], ints [8], floats [4]
#define KB_ON_D(f) (base + (long long)(f) * W)
#define KB_ON_V(f, q) (KB_ON_D(f) + K + (q) * n)
#define KB_ON_I(f, q) (reinterpret_cast<int*>(KB_ON_D(f) + K + 2 * n) + (q) * n)
#define KB_ON_H(f) (reinterpret_cast<int*>(KB_ON_D(f) + K + (BWD ? 4 : 2) * n))
#define KB_ON_S(f) (KB_ON_H(f) + 256)
#define KB_ON_F(f) (reinterpret_cast<float*>(KB_ON_S(f) + 8))
    // ints: 0 prefix, 1 rank, 2 NaN seen, 3 first selected bin, 4 second selected bin; floats: 0 aggregate, 1 a, 2 b,
    // 3 incoming gradient
    const int last = p.levels & 1;
    for (long long job = cta; job < p.jobs; job += n_cta) {
        const long long row = job / p.tiles;
        const int t0 = (int)(job % p.tiles) * F;
        KB_RH_THREADS_BEGIN
        for (int i = tid; i < F * K; i += KB_RH_THREADS) {
            const int f = i / K, b = i % K, t = t0 + f;
            float v = 0.0f;
            if (t >= P && t < p.T)
                v = p.x[(row / p.C) * p.x_sb + (row % p.C) * p.x_sc + (long long)(t - P + lag) * p.x_st +
                        (long long)b * p.x_sk];
            KB_ON_D(f)[b] = v;
        }
        for (int i = tid; i < F * n; i += KB_RH_THREADS) {
            const int f = i / n, j = i % n, t = t0 + f, b = j - hm;
            const bool in = b >= 0 && b < K && t >= P && t < p.T;
            KB_ON_V(f, 0)[j] = in ? p.x[(row / p.C) * p.x_sb + (row % p.C) * p.x_sc + (long long)(t - P) * p.x_st +
                                        (long long)b * p.x_sk]
                                  : -kb_rh_inff();
            if (BWD) KB_ON_I(f, 0)[j] = in ? b : INT_MAX;
        }
        for (int f = tid; f < F; f += KB_RH_THREADS) KB_ON_S(f)[2] = 0;
        KB_RH_THREADS_END
        KB_SYNC_CTA;
        // window maximum by doubling: level q holds the maximum of 2^q padded bins from j
        for (int q = 1; q <= p.levels; ++q) {
            const int h = 1 << (q - 1), s = (q - 1) & 1, d = q & 1;
            KB_RH_THREADS_BEGIN
            for (int i = tid; i < F * n; i += KB_RH_THREADS) {
                const int f = i / n, j = i % n;
                const float a = KB_ON_V(f, s)[j];
                if (j + h < n) {
                    float v;
                    int ix;
                    kb_rh_pick(a, BWD ? KB_ON_I(f, s)[j] : j, KB_ON_V(f, s)[j + h], BWD ? KB_ON_I(f, s)[j + h] : j + h,
                               &v, &ix);
                    KB_ON_V(f, d)[j] = v;
                    if (BWD) KB_ON_I(f, d)[j] = ix;
                } else {
                    KB_ON_V(f, d)[j] = a;
                    if (BWD) KB_ON_I(f, d)[j] = KB_ON_I(f, s)[j];
                }
            }
            KB_RH_THREADS_END
            KB_SYNC_CTA;
        }
        // D = max(0, S[u] - R), NaN kept; the backward keeps R's bin in the other index buffer
        KB_RH_THREADS_BEGIN
        const int span = m - (1 << p.levels);
        for (int i = tid; i < F * K; i += KB_RH_THREADS) {
            const int f = i / K, b = i % K;
            float r;
            int ix;
            kb_rh_pick(KB_ON_V(f, last)[b], BWD ? KB_ON_I(f, last)[b] : b, KB_ON_V(f, last)[b + span],
                       BWD ? KB_ON_I(f, last)[b + span] : b + span, &r, &ix);
            const float dv = KB_ON_D(f)[b] - r;
            const float dd = dv != dv ? dv : (dv > 0.0f ? dv : 0.0f);
            KB_ON_D(f)[b] = dd;
            if (dd != dd) KB_ON_S(f)[2] = 1;
            if (BWD) KB_ON_I(f, 1 - last)[b] = ix;
        }
        KB_RH_THREADS_END
        KB_SYNC_CTA;
        if (p.agg == KB_RH_AGG_MEAN) {
            KB_RH_THREADS_BEGIN
            for (int f = tid; f < F; f += KB_RH_THREADS) {
                double s = 0.0;
                for (int b = 0; b < K; ++b) s += (double)KB_ON_D(f)[b];
                KB_ON_F(f)[0] = (float)(s / (double)K);
            }
            KB_RH_THREADS_END
            KB_SYNC_CTA;
        } else {
            // exact selection of rank (K - 1) / 2 (odd K) or K / 2 - 1 and K / 2 (even K)
            const int nsel = (K & 1) ? 1 : 2;
            for (int q = 0; q < nsel; ++q) {
                KB_RH_THREADS_BEGIN
                for (int i = tid; i < F * 256; i += KB_RH_THREADS) KB_ON_H(i / 256)[i % 256] = 0;
                for (int f = tid; f < F; f += KB_RH_THREADS) {
                    KB_ON_S(f)[0] = 0;
                    KB_ON_S(f)[1] = (K & 1) ? (K - 1) / 2 : K / 2 - 1 + q;
                }
                KB_RH_THREADS_END
                KB_SYNC_CTA;
                for (int sh = 24; sh >= 0; sh -= 8) {
                    KB_RH_THREADS_BEGIN
                    for (int i = tid; i < F * K; i += KB_RH_THREADS) {
                        const int f = i / K, b = i % K;
                        const unsigned key = kb_rh_fbits(KB_ON_D(f)[b]);
                        if (sh == 24 || (key >> (sh + 8)) == ((unsigned)KB_ON_S(f)[0] >> (sh + 8)))
                            kb_rh_atomic_add(&KB_ON_H(f)[(key >> sh) & 255], 1);
                    }
                    KB_RH_THREADS_END
                    KB_SYNC_CTA;
                    KB_RH_THREADS_BEGIN
                    for (int f = tid; f < F; f += KB_RH_THREADS) {
                        int* h = KB_ON_H(f);
                        int r = KB_ON_S(f)[1], dgt = 0;
                        for (; dgt < 255 && r >= h[dgt]; ++dgt) r -= h[dgt];
                        KB_ON_S(f)[1] = r;
                        KB_ON_S(f)[0] = (int)((unsigned)KB_ON_S(f)[0] | ((unsigned)dgt << sh));
                        for (int j = 0; j < 256; ++j) h[j] = 0;
                    }
                    KB_RH_THREADS_END
                    KB_SYNC_CTA;
                }
                KB_RH_THREADS_BEGIN
                for (int f = tid; f < F; f += KB_RH_THREADS) KB_ON_F(f)[1 + q] = kb_rh_bitsf((unsigned)KB_ON_S(f)[0]);
                KB_RH_THREADS_END
                KB_SYNC_CTA;
            }
            KB_RH_THREADS_BEGIN
            for (int f = tid; f < F; f += KB_RH_THREADS) {
                const float a = KB_ON_F(f)[1];
                KB_ON_F(f)[0] = KB_ON_S(f)[2] ? kb_rh_nanf() : (K & 1) ? a : 0.5f * (a + KB_ON_F(f)[2]);
            }
            KB_RH_THREADS_END
            KB_SYNC_CTA;
        }
        if (!BWD) {
            KB_RH_THREADS_BEGIN
            for (int f = tid; f < F; f += KB_RH_THREADS) {
                const int t = t0 + f;
                if (t < p.T) p.out[kb_rh_off3(row, p.C, p.o_sb, p.o_sc, p.o_st, t)] = t < P ? 0.0f : KB_ON_F(f)[0];
            }
            KB_RH_THREADS_END
            KB_SYNC_CTA;
        } else {
            // the incoming gradient and, for the median, the bins selected under the order (value, bin)
            KB_RH_THREADS_BEGIN
            for (int f = tid; f < F; f += KB_RH_THREADS) {
                const int t = t0 + f;
                KB_ON_F(f)[3] = (t >= P && t < p.T) ? p.g[kb_rh_off3(row, p.C, p.g_sb, p.g_sc, p.g_st, t)] : 0.0f;
                KB_ON_S(f)[3] = KB_ON_S(f)[4] = -1;
                if (p.agg != KB_RH_AGG_MEDIAN || KB_ON_S(f)[2]) continue;
                for (int q = 0; q < ((K & 1) ? 1 : 2); ++q) {
                    const float v = KB_ON_F(f)[1 + q];
                    const int r = (K & 1) ? (K - 1) / 2 : K / 2 - 1 + q;
                    int less = 0;
                    for (int b = 0; b < K; ++b) less += KB_ON_D(f)[b] < v;
                    int skip = r - less, sel = -1;
                    for (int b = 0; b < K && sel < 0; ++b)
                        if (KB_ON_D(f)[b] == v) { if (skip == 0) sel = b; else --skip; }
                    KB_ON_S(f)[3 + q] = sel;
                }
            }
            KB_RH_THREADS_END
            KB_SYNC_CTA;
            KB_RH_THREADS_BEGIN
            for (int i = tid; i < F * K; i += KB_RH_THREADS) {
                const int f = i / K, b = i % K, t = t0 + f;
                if (t < P || t >= p.T) continue;
                const float g = KB_ON_F(f)[3];
                float c = 0.0f;
                if (KB_ON_D(f)[b] > 0.0f) {
                    if (p.agg == KB_RH_AGG_MEAN) c = g / (float)K;
                    else if (K & 1) c = b == KB_ON_S(f)[3] ? g : 0.0f;
                    else c = (b == KB_ON_S(f)[3] || b == KB_ON_S(f)[4]) ? 0.5f * g : 0.0f;
                }
                kb_on_w w;
                w.g = c;
                w.src = KB_ON_I(f, 1 - last)[b];
                p.ws[((row * p.T) + (t - P + lag)) * (long long)K + b] = w;
            }
            KB_RH_THREADS_END
            KB_SYNC_CTA;
        }
    }
#undef KB_ON_D
#undef KB_ON_V
#undef KB_ON_I
#undef KB_ON_H
#undef KB_ON_S
#undef KB_ON_F
}

// Second gradient pass: element (row, v, b') of block `cta` gathers the gradient of D[v][b'] and subtracts those of
// D[v + lag][b] whose window maximum came from b', in ascending b.
KB_RH_FN void kb_onset_gather_cta(const KbOnsetParams& p, char*, long long cta, long long n_cta) {
    const long long n = (long long)p.B * p.C * p.T * p.K;
    const int K = p.K, m = p.m, hm = m / 2, ulo = p.lag, uhi = p.T - p.P + p.lag;
    for (long long e0 = cta * KB_RH_THREADS; e0 < n; e0 += n_cta * KB_RH_THREADS) {
        KB_RH_THREADS_BEGIN
        const long long e = e0 + tid;
        if (e < n) {
            const int b = (int)(e % K), v = (int)((e / K) % p.T);
            const long long row = e / ((long long)p.T * K);
            float acc = 0.0f;
            if (v >= ulo && v < uhi) acc = p.ws[e].g;
            if (v + p.lag >= ulo && v + p.lag < uhi) {
                const int lo = b + hm - m + 1 > 0 ? b + hm - m + 1 : 0, hi = b + hm < K - 1 ? b + hm : K - 1;
                const kb_on_w* w = p.ws + e + (long long)p.lag * K - b;
                for (int c = lo; c <= hi; ++c)
                    if (w[c].src == b) acc = acc - w[c].g;
            }
            p.gx[(row / p.C) * p.gx_sb + (row % p.C) * p.gx_sc + (long long)v * p.gx_st + (long long)b * p.gx_sk] = acc;
        }
        KB_RH_THREADS_END
    }
}

// ---------------------------------------------------------------------------------------------------------- tempogram
struct KbTempogramParams {
    int B, C, T, W, center, norm;
    int n_out, F;                         // frames out, frames per tile
    long long tiles, jobs;
    const float* e;                       // envelope, strides (b, c, t)
    long long e_sb, e_sc, e_st;
    float* out;                           // (b, c, t, lag) strides
    long long o_sb, o_sc, o_st, o_sk;
};

KB_HD int kb_tg_blocks(int W) { return (W + KB_RH_LAGS - 1) / KB_RH_LAGS; }
// words: window W, span F + W - 1, y F (W + LAGS), ac F W, block maxima F blocks, frame maxima F
KB_HD int kb_tg_words(int W, int F) {
    return W + (F + W - 1) + F * (W + KB_RH_LAGS) + F * W + F * kb_tg_blocks(W) + F;
}
KB_HD int kb_tg_tile_frames(int W) {
    int f = 16;
    while (f > 1 && kb_tg_words(W, f) * 4 > KB_RH_SMEM_BUDGET + 8 * 1024) --f;
    return f;
}

inline bool kb_tempogram_setup(KbTempogramParams& p) {
    p.n_out = p.center ? p.T : p.T - p.W + 1;
    if (p.n_out < 0) p.n_out = 0;
    p.F = kb_tg_tile_frames(p.W);
    p.tiles = ((long long)p.n_out + p.F - 1) / p.F;
    p.jobs = (long long)p.B * p.C * p.tiles;
    return p.jobs < (1LL << 40);
}

KB_RH_FN void kb_tempogram_cta(const KbTempogramParams& p, char* smem, long long cta, long long n_cta) {
    const int W = p.W, F = p.F, c = W / 2, NB = kb_tg_blocks(W), YS = W + KB_RH_LAGS;
    const int plen = p.center ? p.T + 2 * c : p.T;
    float* win = reinterpret_cast<float*>(smem);
    float* span = win + W;
    float* y = span + (F + W - 1);
    float* ac = y + F * YS;
    float* bm = ac + F * W;
    float* fm = bm + F * NB;
    for (long long job = cta; job < p.jobs; job += n_cta) {
        const long long row = job / p.tiles;
        const int t0 = (int)(job % p.tiles) * F;
        const long long eb = (row / p.C) * p.e_sb + (row % p.C) * p.e_sc;
        KB_RH_THREADS_BEGIN
        for (int j = tid; j < W; j += KB_RH_THREADS)
            win[j] = (float)(0.5 - 0.5 * kb_rh_cospi(2.0 * (double)j / (double)W));
        for (int i = tid; i < F + W - 1; i += KB_RH_THREADS) {
            const int q = t0 + i;
            float v = 0.0f;
            if (q < plen) {
                if (!p.center) v = p.e[eb + (long long)q * p.e_st];
                else if (q < c) v = (float)((double)p.e[eb] * (double)q / (double)c);
                else if (q >= c + p.T) {
                    const int k = q - c - p.T + 1;
                    v = (float)((double)p.e[eb + (long long)(p.T - 1) * p.e_st] * (double)(c - k) / (double)c);
                } else v = p.e[eb + (long long)(q - c) * p.e_st];
            }
            span[i] = v;
        }
        KB_RH_THREADS_END
        KB_SYNC_CTA;
        KB_RH_THREADS_BEGIN
        for (int i = tid; i < F * YS; i += KB_RH_THREADS) {
            const int f = i / YS, j = i % YS;
            y[i] = j < W ? win[j] * span[f + j] : 0.0f;
        }
        KB_RH_THREADS_END
        KB_SYNC_CTA;
        // ac[l] = sum_{j <= W-1-l} y[j] y[j + l]: lags l0 .. l0 + 7 of one frame per task, a register window over y
        KB_RH_THREADS_BEGIN
        for (int task = tid; task < F * NB; task += KB_RH_THREADS) {
            const int f = task / NB, l0 = (task % NB) * KB_RH_LAGS;
            if (t0 + f >= p.n_out) continue;
            const float* yf = y + f * YS;
            float acc[KB_RH_LAGS], yw[KB_RH_LAGS];
#pragma unroll
            for (int r = 0; r < KB_RH_LAGS; ++r) {
                acc[r] = 0.0f;
                yw[r] = l0 + r < YS ? yf[l0 + r] : 0.0f;
            }
            for (int j = 0; j < W - l0; ++j) {
                const float a = yf[j];
#pragma unroll
                for (int r = 0; r < KB_RH_LAGS; ++r) acc[r] = fmaf(a, yw[r], acc[r]);
#pragma unroll
                for (int r = 0; r < KB_RH_LAGS - 1; ++r) yw[r] = yw[r + 1];
                const int nx = j + l0 + KB_RH_LAGS;
                yw[KB_RH_LAGS - 1] = nx < YS ? yf[nx] : 0.0f;
            }
            float mx = 0.0f;
#pragma unroll
            for (int r = 0; r < KB_RH_LAGS; ++r)
                if (l0 + r < W) {
                    ac[f * W + l0 + r] = acc[r];
                    mx = fmaxf(mx, fabsf(acc[r]));
                }
            bm[f * NB + task % NB] = mx;
        }
        KB_RH_THREADS_END
        KB_SYNC_CTA;
        KB_RH_THREADS_BEGIN
        for (int f = tid; f < F; f += KB_RH_THREADS) {
            float mx = 0.0f;
            for (int k = 0; k < NB; ++k) mx = fmaxf(mx, bm[f * NB + k]);
            fm[f] = mx;
        }
        KB_RH_THREADS_END
        KB_SYNC_CTA;
        KB_RH_THREADS_BEGIN
        for (int i = tid; i < F * W; i += KB_RH_THREADS) {
            const int f = i / W, l = i % W, t = t0 + f;
            if (t >= p.n_out) continue;
            const float v = ac[i], mx = fm[f];
            p.out[(row / p.C) * p.o_sb + (row % p.C) * p.o_sc + (long long)t * p.o_st + (long long)l * p.o_sk] =
                (p.norm && mx >= KB_RH_TINY) ? v / mx : v;
        }
        KB_RH_THREADS_END
        KB_SYNC_CTA;
    }
}

// -------------------------------------------------------------------------------------------------------------- tempo
#define KB_RH_TEMPO_CHUNK 64         // frames per partial sum of the mean

struct KbTempoParams {
    int B, C, T, W, per_frame;
    long long chunks, jobs;               // chunks of KB_RH_TEMPO_CHUNK frames per row (mean)
    const float* tg;                      // (b, c, t, lag) strides
    long long g_sb, g_sc, g_st, g_sk;
    double* part;                         // mean: [row][chunk][lag] float64 partial sums
    const double* logprior;               // W values (lag 0: -inf)
    double bpm_scale;                     // 60 sr / hop: bpm[l] = bpm_scale / l
    float* out;                           // per row (contiguous (b, c)) or per frame ((b, c, t) strides)
    long long o_sb, o_sc, o_st;
};

inline void kb_tempo_setup(KbTempoParams& p) {
    p.chunks = ((long long)p.T + KB_RH_TEMPO_CHUNK - 1) / KB_RH_TEMPO_CHUNK;
    p.jobs = (long long)p.B * p.C * (p.per_frame ? p.T : 1);
}
KB_HD long long kb_tempo_ws_bytes(int B, int C, int T, int W) {
    return (long long)B * C * ((T + KB_RH_TEMPO_CHUNK - 1) / KB_RH_TEMPO_CHUNK) * W * 8;
}
KB_HD int kb_tempo_smem(int W) { return W * 8 + 16; }

// Mean, first launch: job (row, chunk) sums its frames of every lag in ascending frame order.  A non-finite value
// makes the sum non-finite: float32 values cannot overflow a float64 sum of fewer than 2^31 terms.
KB_RH_FN void kb_tempo_part_cta(const KbTempoParams& p, char*, long long cta, long long n_cta) {
    const long long njobs = (long long)p.B * p.C * p.chunks;
    for (long long job = cta; job < njobs; job += n_cta) {
        const long long row = job / p.chunks, ch = job % p.chunks;
        const long long gb = (row / p.C) * p.g_sb + (row % p.C) * p.g_sc;
        const int u0 = (int)(ch * KB_RH_TEMPO_CHUNK);
        const int u1 = u0 + KB_RH_TEMPO_CHUNK < p.T ? u0 + KB_RH_TEMPO_CHUNK : p.T;
        KB_RH_THREADS_BEGIN
        for (int l = tid; l < p.W; l += KB_RH_THREADS) {
            double s = 0.0;
            for (int u = u0; u < u1; ++u) s += (double)p.tg[gb + (long long)u * p.g_st + (long long)l * p.g_sk];
            p.part[job * p.W + l] = s;
        }
        KB_RH_THREADS_END
    }
}

// The decision: per row, g = (sum of the chunk sums in ascending order) / T; per frame, g = tg.  A non-finite g
// gives NaN; a lag whose score is NaN (g < -1e-6) is skipped, and a row with none left gives NaN.
KB_RH_FN void kb_tempo_cta(const KbTempoParams& p, char* smem, long long cta, long long n_cta) {
    const int W = p.W;
    double* score = reinterpret_cast<double*>(smem);
    int* bad = reinterpret_cast<int*>(score + W);
    for (long long job = cta; job < p.jobs; job += n_cta) {
        const long long row = p.per_frame ? job / p.T : job;
        const int t = p.per_frame ? (int)(job % p.T) : 0;
        const long long gb = (row / p.C) * p.g_sb + (row % p.C) * p.g_sc;
        KB_RH_THREADS_BEGIN
        if (tid == 0) *bad = 0;
        KB_RH_THREADS_END
        KB_SYNC_CTA;
        KB_RH_THREADS_BEGIN
        for (int l = tid; l < W; l += KB_RH_THREADS) {
            double g;
            if (p.per_frame) {
                g = (double)p.tg[gb + (long long)t * p.g_st + (long long)l * p.g_sk];
            } else {
                double s = 0.0;
                for (long long c = 0; c < p.chunks; ++c) s += p.part[(row * p.chunks + c) * W + l];
                g = s / (double)p.T;
            }
            if (!(g - g == 0.0)) *bad = 1;
            score[l] = log1p(1.0e6 * g) + p.logprior[l];
        }
        KB_RH_THREADS_END
        KB_SYNC_CTA;
        KB_RH_THREADS_BEGIN
        if (tid == 0) {
            int best = -1;
            for (int l = 0; l < W; ++l)
                if (score[l] == score[l] && (best < 0 || score[l] > score[best])) best = l;
            const float bpm = (*bad || best < 0) ? kb_rh_nanf() : (float)(p.bpm_scale / (double)best);
            if (p.per_frame) p.out[kb_rh_off3(row, p.C, p.o_sb, p.o_sc, p.o_st, t)] = bpm;
            else p.out[row] = bpm;
        }
        KB_RH_THREADS_END
        KB_SYNC_CTA;
    }
}

// ------------------------------------------------------------------------------------------------------- peak picking
struct KbPeakParams {
    int B, C, T;
    int pre_max, post_max, pre_avg, post_avg, wait, normalize;
    double delta;
    long long jobs;
    const float* e;                       // envelope, strides (b, c, t)
    long long e_sb, e_sc, e_st;
    unsigned char* mask;                  // strides (b, c, t)
    long long m_sb, m_sc, m_st;
};

// words: per-thread min and max, then scalars (min, scale, non-finite, any nonzero)
KB_HD int kb_peak_smem() { return (2 * KB_RH_THREADS + 4) * 4; }

KB_RH_FN float kb_pk_x(const KbPeakParams& p, const float* e, long long eb, int n, float mn, float den) {
    const float v = e[eb + (long long)n * p.e_st];
    return p.normalize ? (v - mn) / den : v;
}

KB_RH_FN void kb_peak_cta(const KbPeakParams& p, char* smem, long long cta, long long n_cta) {
    float* pmin = reinterpret_cast<float*>(smem);
    float* pmax = pmin + KB_RH_THREADS;
    float* sc = pmax + KB_RH_THREADS;        // 0 min, 1 max x + FLT_MIN
    int* fl = reinterpret_cast<int*>(sc + 2); // 0 non-finite, 1 any nonzero
    const int T = p.T;
    for (long long row = cta; row < p.jobs; row += n_cta) {
        const long long eb = (row / p.C) * p.e_sb + (row % p.C) * p.e_sc;
        const long long mb = (row / p.C) * p.m_sb + (row % p.C) * p.m_sc;
        KB_RH_THREADS_BEGIN
        float lo = kb_rh_inff(), hi = -kb_rh_inff();
        int bad = 0;
        for (int n = tid; n < T; n += KB_RH_THREADS) {
            const float v = p.e[eb + (long long)n * p.e_st];
            bad |= !(v - v == 0.0f);
            lo = fminf(lo, v);
            hi = fmaxf(hi, v);
        }
        pmin[tid] = lo;
        pmax[tid] = hi;
        if (tid == 0) { fl[0] = 0; fl[1] = 0; }
        KB_RH_THREADS_END
        KB_SYNC_CTA;
        KB_RH_THREADS_BEGIN
        for (int n = tid; n < T; n += KB_RH_THREADS) {
            const float v = p.e[eb + (long long)n * p.e_st];
            if (!(v - v == 0.0f)) fl[0] = 1;
        }
        if (tid == 0) {
            float lo2 = pmin[0], hi2 = pmax[0];
            for (int k = 1; k < KB_RH_THREADS; ++k) { lo2 = fminf(lo2, pmin[k]); hi2 = fmaxf(hi2, pmax[k]); }
            sc[0] = lo2;
            sc[1] = (hi2 - lo2) + KB_RH_TINY;   // max(e - min e) = fl(max e - min e): rounding is monotonic
        }
        KB_RH_THREADS_END
        KB_SYNC_CTA;
        // candidates
        KB_RH_THREADS_BEGIN
        const float mn = sc[0], den = sc[1];
        for (int n = tid; n < T; n += KB_RH_THREADS) {
            const float x = kb_pk_x(p, p.e, eb, n, mn, den);
            if (x != 0.0f) fl[1] = 1;
            const long long nn = n;
            const int a0 = (int)(nn - p.pre_max > 0 ? nn - p.pre_max : 0);
            const int a1 = (int)(nn + p.post_max < T ? nn + p.post_max : T);
            float mx = -kb_rh_inff();
            for (int k = a0; k < a1; ++k) mx = fmaxf(mx, kb_pk_x(p, p.e, eb, k, mn, den));
            const int b0 = (int)(nn - p.pre_avg > 0 ? nn - p.pre_avg : 0);
            const int b1 = (int)(nn + p.post_avg < T ? nn + p.post_avg : T);
            double s = 0.0;
            for (int k = b0; k < b1; ++k) s += (double)kb_pk_x(p, p.e, eb, k, mn, den);
            const double av = s / (double)(b1 - b0);
            const bool cand = x == mx && x != 0.0f && (double)x >= av + p.delta;
            p.mask[mb + (long long)n * p.m_st] = cand ? 1 : 0;
        }
        KB_RH_THREADS_END
        KB_SYNC_CTA;
        // the wait walk over the candidates, or no onsets at all
        KB_RH_THREADS_BEGIN
        if (tid == 0) {
            const bool none = fl[0] || !fl[1];
            long long last = -(1LL << 40);
            for (int n = 0; n < T; ++n) {
                unsigned char* mk = p.mask + mb + (long long)n * p.m_st;
                if (!*mk) continue;
                if (!none && n > last + (long long)p.wait) last = n;
                else *mk = 0;
            }
        }
        KB_RH_THREADS_END
        KB_SYNC_CTA;
    }
}

// ------------------------------------------------------------------------------------------------------ beat tracking
struct KbBeatParams {
    int B, C, T, trim;
    double fps;                           // sr / hop
    double tightness;
    const float* bpm;                     // per row (contiguous (b, c)), or null: bpm_const for every row
    float bpm_const;
    long long jobs;
    const float* e;                       // envelope, strides (b, c, t)
    long long e_sb, e_sc, e_st;
    float* tempo;                         // per row, contiguous (b, c)
    unsigned char* mask;                  // strides (b, c, t)
    long long m_sb, m_sc, m_st;
    void* ws;                             // per row: ls, cs (double T), back, beats (int T)
};

KB_HD long long kb_beat_ws_bytes_row(int T) { return (long long)T * 24; }

// words (4 bytes): Gaussian window p + 1 doubles, txwt 2p + 1 doubles, per-thread doubles and ints, histogram 256,
// scalars
#define KB_BT_SCAL 32
KB_HD int kb_beat_smem() {
    return (KB_RH_MAX_PERIOD + 1) * 8 + (2 * KB_RH_MAX_PERIOD + 1) * 8 + KB_RH_THREADS * 8 + KB_RH_THREADS * 4 + 256 * 4 +
           KB_BT_SCAL * 8;
}

// Ordered 64-bit key of a double (ascending keys for ascending values).
KB_RH_FN unsigned long long kb_rh_dkey(double v) {
    const unsigned long long u = kb_rh_dbits(v);
    return (u >> 63) ? ~u : (u | 0x8000000000000000ULL);
}
KB_RH_FN double kb_rh_unkey(unsigned long long k) {
    return kb_rh_bitsd((k >> 63) ? (k & 0x7fffffffffffffffULL) : ~k);
}

KB_RH_FN bool kb_bt_in_l(const double* cs, int T, int i) {
    return i >= 1 && cs[i] > cs[i - 1] && (i == T - 1 || cs[i] >= cs[i + 1]);
}

KB_RH_FN void kb_beat_cta(const KbBeatParams& p, char* smem, long long cta, long long n_cta) {
    const int T = p.T;
    double* win = reinterpret_cast<double*>(smem);
    double* txw = win + (KB_RH_MAX_PERIOD + 1);
    double* pd = txw + (2 * KB_RH_MAX_PERIOD + 1);
    int* pi = reinterpret_cast<int*>(pd + KB_RH_THREADS);
    int* hist = pi + KB_RH_THREADS;
    double* sd = reinterpret_cast<double*>(hist + 256);   // 0 mean, 1 std, 2 max ls, 3 median, 4 sel a
    long long* si = reinterpret_cast<long long*>(sd + 8);  // 0 state, 1 p, 2 i0, 3 |L|, 4 prefix, 5 rank, 6 last
    for (long long row = cta; row < p.jobs; row += n_cta) {
        const long long eb = (row / p.C) * p.e_sb + (row % p.C) * p.e_sc;
        const long long mb = (row / p.C) * p.m_sb + (row % p.C) * p.m_sc;
        double* ls = reinterpret_cast<double*>(static_cast<char*>(p.ws) + row * kb_beat_ws_bytes_row(T));
        double* cs = ls + T;
        int* back = reinterpret_cast<int*>(cs + T);
        int* beats = back + T;
        // sum, non-finite and nonzero flags; the mask cleared
        KB_RH_THREADS_BEGIN
        double s = 0.0;
        int fl = 0;
        for (int n = tid; n < T; n += KB_RH_THREADS) {
            const float v = p.e[eb + (long long)n * p.e_st];
            s += (double)v;
            fl |= (v - v == 0.0f ? 0 : 1) | (v != 0.0f ? 2 : 0);
            p.mask[mb + (long long)n * p.m_st] = 0;
        }
        pd[tid] = s;
        pi[tid] = fl;
        KB_RH_THREADS_END
        KB_SYNC_CTA;
        KB_RH_THREADS_BEGIN
        if (tid == 0) {
            double a = 0.0;
            int f = 0;
            for (int k = 0; k < KB_RH_THREADS; ++k) { a += pd[k]; f |= pi[k]; }
            sd[0] = a / (double)T;
            // state: 0 track, 1 non-finite (tempo NaN), 2 all zero (tempo 0), 3 period out of range
            si[0] = (f & 1) ? 1 : !(f & 2) ? 2 : 0;
        }
        KB_RH_THREADS_END
        KB_SYNC_CTA;
        KB_RH_THREADS_BEGIN
        double s2 = 0.0;
        for (int n = tid; n < T; n += KB_RH_THREADS) {
            const double d = (double)p.e[eb + (long long)n * p.e_st] - sd[0];
            s2 = fma(d, d, s2);
        }
        pd[tid] = s2;
        KB_RH_THREADS_END
        KB_SYNC_CTA;
        KB_RH_THREADS_BEGIN
        if (tid == 0) {
            double a = 0.0;
            for (int k = 0; k < KB_RH_THREADS; ++k) a += pd[k];
            const double sdv = sqrt(a / (double)(T - 1));
            sd[1] = sdv > 0.0 ? sdv : 1.0;
            const float bpm = p.bpm ? p.bpm[row] : p.bpm_const;
            long long per = 0;
            if (si[0] == 0) {
                const double q = kb_rh_rint(60.0 * p.fps / (double)bpm);
                if (q >= 1.0 && q <= (double)KB_RH_MAX_PERIOD) per = (long long)q;
                else si[0] = 3;
            }
            si[1] = per;
            p.tempo[row] = si[0] == 1 ? kb_rh_nanf() : si[0] == 2 ? 0.0f : bpm;
        }
        KB_RH_THREADS_END
        KB_SYNC_CTA;
        if (si[0] != 0) continue;
        const int per = (int)si[1], half = (int)kb_rh_rint(0.5 * per), nd = 2 * per - half + 1;
        KB_RH_THREADS_BEGIN
        for (int d = tid; d <= per; d += KB_RH_THREADS) {
            const double x = 32.0 * (double)d / (double)per;
            win[d] = exp(-0.5 * (x * x));
        }
        for (int k = tid; k < nd; k += KB_RH_THREADS) {
            const double r = log((double)(2 * per - k) / (double)per);   // d = -2p + k
            txw[k] = -p.tightness * (r * r);
        }
        KB_RH_THREADS_END
        KB_SYNC_CTA;
        // local score, its per-thread maxima
        KB_RH_THREADS_BEGIN
        const double sdv = sd[1];
        double mx = -kb_rh_inf();
        for (int i = tid; i < T; i += KB_RH_THREADS) {
            double a = 0.0;
            for (int d = -per; d <= per; ++d) {
                const int j = i - d;
                if (j < 0 || j >= T) continue;
                a = fma((double)p.e[eb + (long long)j * p.e_st] / sdv, win[d < 0 ? -d : d], a);
            }
            ls[i] = a;
            mx = a > mx ? a : mx;
        }
        pd[tid] = mx;
        KB_RH_THREADS_END
        KB_SYNC_CTA;
        KB_RH_THREADS_BEGIN
        if (tid == 0) {
            double a = pd[0];
            for (int k = 1; k < KB_RH_THREADS; ++k) a = pd[k] > a ? pd[k] : a;
            sd[2] = a;
        }
        KB_RH_THREADS_END
        KB_SYNC_CTA;
        KB_RH_THREADS_BEGIN
        int first = T;
        for (int i = tid; i < T && first == T; i += KB_RH_THREADS)
            if (ls[i] >= 0.01 * sd[2]) first = i;
        pi[tid] = first;
        KB_RH_THREADS_END
        KB_SYNC_CTA;
        KB_RH_THREADS_BEGIN
        if (tid == 0) {
            int a = T;
            for (int k = 0; k < KB_RH_THREADS; ++k) a = pi[k] < a ? pi[k] : a;
            si[2] = a;
        }
        KB_RH_THREADS_END
        KB_SYNC_CTA;
        // the dynamic programme, S independent frames per step
        const int S = half > 1 ? half : 1, i0 = (int)si[2];
        for (int base = 0; base < T; base += S) {
            KB_RH_THREADS_BEGIN
            for (int k = tid; k < S && base + k < T; k += KB_RH_THREADS) {
                const int i = base + k;
                double best = 0.0;
                int bd = 0;
                for (int q = 0; q < nd; ++q) {
                    const int d = q - 2 * per, j = i + d;
                    const double c = txw[q] + ((j >= 0 && d != 0) ? cs[j] : 0.0);
                    if (q == 0 || c > best) { best = c; bd = d; }
                }
                cs[i] = ls[i] + best;
                back[i] = i < i0 ? -1 : i + bd;
            }
            KB_RH_THREADS_END
            KB_SYNC_CTA;
        }
        // |L|, then the median of cs over L by radix selection on ordered 64-bit keys
        KB_RH_THREADS_BEGIN
        int cnt = 0;
        for (int i = tid; i < T; i += KB_RH_THREADS) cnt += kb_bt_in_l(cs, T, i);
        pi[tid] = cnt;
        KB_RH_THREADS_END
        KB_SYNC_CTA;
        KB_RH_THREADS_BEGIN
        if (tid == 0) {
            long long a = 0;
            for (int k = 0; k < KB_RH_THREADS; ++k) a += pi[k];
            si[3] = a;
        }
        KB_RH_THREADS_END
        KB_SYNC_CTA;
        const long long nl = si[3];
        if (nl == 0) continue;
        const int nsel = (nl & 1) ? 1 : 2;
        for (int q = 0; q < nsel; ++q) {
            KB_RH_THREADS_BEGIN
            for (int j = tid; j < 256; j += KB_RH_THREADS) hist[j] = 0;
            if (tid == 0) { si[4] = 0; si[5] = (nl & 1) ? (nl - 1) / 2 : nl / 2 - 1 + q; }
            KB_RH_THREADS_END
            KB_SYNC_CTA;
            for (int sh = 56; sh >= 0; sh -= 8) {
                KB_RH_THREADS_BEGIN
                const unsigned long long pre = (unsigned long long)si[4];
                for (int i = tid; i < T; i += KB_RH_THREADS) {
                    if (!kb_bt_in_l(cs, T, i)) continue;
                    const unsigned long long key = kb_rh_dkey(cs[i]);
                    if (sh == 56 || (key >> (sh + 8)) == (pre >> (sh + 8)))
                        kb_rh_atomic_add(&hist[(key >> sh) & 255], 1);
                }
                KB_RH_THREADS_END
                KB_SYNC_CTA;
                KB_RH_THREADS_BEGIN
                if (tid == 0) {
                    long long r = si[5];
                    int dgt = 0;
                    for (; dgt < 255 && r >= hist[dgt]; ++dgt) r -= hist[dgt];
                    si[5] = r;
                    si[4] = (long long)((unsigned long long)si[4] | ((unsigned long long)dgt << sh));
                    for (int j = 0; j < 256; ++j) hist[j] = 0;
                }
                KB_RH_THREADS_END
                KB_SYNC_CTA;
            }
            KB_RH_THREADS_BEGIN
            if (tid == 0) {
                const double v = kb_rh_unkey((unsigned long long)si[4]);
                if (q == 0) sd[4] = v;
                sd[3] = q == 0 ? v : 0.5 * (sd[4] + v);
            }
            KB_RH_THREADS_END
            KB_SYNC_CTA;
        }
        // the last beat: the largest i with 2 cs[i] [i in L] > med
        KB_RH_THREADS_BEGIN
        const double med = sd[3];
        int lastb = -1;
        for (int i = tid; i < T; i += KB_RH_THREADS) {
            const double v = kb_bt_in_l(cs, T, i) ? 2.0 * cs[i] : 0.0;
            if (v > med) lastb = i;
        }
        pi[tid] = lastb;
        KB_RH_THREADS_END
        KB_SYNC_CTA;
        // backtrack, trim and write the mask
        KB_RH_THREADS_BEGIN
        if (tid == 0) {
            int b = -1;
            for (int k = 0; k < KB_RH_THREADS; ++k) b = pi[k] > b ? pi[k] : b;
            int nb = 0;
            if (b >= 0) {
                beats[nb++] = b;
                while (back[b] >= 0) { b = back[b]; beats[nb++] = b; }
            }
            // beats[nb - 1 - j] is beat j in ascending order
            double ss = 0.0;
            for (int j = 0; j < nb; ++j) {
                const double vl = j > 0 ? ls[beats[nb - j]] : 0.0, vr = j + 1 < nb ? ls[beats[nb - 2 - j]] : 0.0;
                const double sj = fma(0.5, vr, fma(0.5, vl, ls[beats[nb - 1 - j]]));
                ss = fma(sj, sj, ss);
            }
            const double thr = (p.trim && nb > 0) ? 0.5 * sqrt(ss / (double)nb) : 0.0;
            int jlo = -1, jhi = -1;
            for (int j = 0; j < nb; ++j) {
                const double vl = j > 0 ? ls[beats[nb - j]] : 0.0, vr = j + 1 < nb ? ls[beats[nb - 2 - j]] : 0.0;
                const double sj = fma(0.5, vr, fma(0.5, vl, ls[beats[nb - 1 - j]]));
                if (sj > thr) { if (jlo < 0) jlo = j; jhi = j; }
            }
            for (int j = jlo; jlo >= 0 && j < jhi; ++j) p.mask[mb + (long long)beats[nb - 1 - j] * p.m_st] = 1;
        }
        KB_RH_THREADS_END
        KB_SYNC_CTA;
    }
}
