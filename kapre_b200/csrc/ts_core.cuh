// Kernel bodies of the phase-vocoder time stretch (torchaudio.functional.phase_vocoder) and its gradient.  For each
// column (b, c, f) of a complex spectrogram X with T frames, output frame u < T' = ceil(T / rate) is
//   ts_u = (double)u * rate,  k_u = floor(ts_u),  alpha_u = ts_u - k_u        (X[T] = X[T + 1] = 0)
//   m[u] = alpha_u |X[k_u + 1]| + (1 - alpha_u) |X[k_u]|
//   phi[u] = q(X[0]) + sum_{v < u} (q(X[k_v + 1]) - q(X[k_v]))                  (uint32 arithmetic, mod 2^32)
//   Y[u] = m[u] (cospi(s), sinpi(s)),  s = (int32)phi[u] 2^-31
// with the fixed-point angle q(z) = rint(kb_atan2(z) 2^31 / pi) mod 2^32, a count of 2^-32 turns.  torchaudio's phase
// recurrence wraps a(k+1) - a(k) - adv and adds adv back; modulo 2 pi that is a(k+1) - a(k) for any phase advance,
// which is what the sum above accumulates.  Integer addition is exact and associative: the phase does not drift
// with u, and any cut of the sum into chunks gives the same bits.
//
// Gradient (torch's convention G = dL/dRe + i dL/dIm), from Y and G only:
//   gm[u] = Re(conj(Y) G) / |Y|,  gphi[u] = Im(conj(Y) G)   (0 where Y = 0),  lam_u = sum_{v > u} gphi[v]
//   frame j:  g|X| += (1 - alpha_u) gm[u] where k_u = j, += alpha_u gm[u] where k_u + 1 = j
//             gth  -= lam_u where k_u = j,  += lam_u where k_u + 1 = j,  frame 0 also += sum_u gphi[u]
//   gX = X / |X| (g|X| + i gth / |X|), 0 where |X| = 0.
//
// Work split: one thread per (chunk, column), columns numbered as in pcen_core.cuh (c fastest when the channel axis
// is innermost), so a warp's 32 columns are neighbours in memory at every frame.  Every thread of a launch has the
// same rate and chunk bounds, so the data-dependent loops below take the same trip counts across a warp.
//
// Chunks partition the INPUT frames: chunk c owns frames [c Tc, min((c + 1) Tc, T)) and the outputs whose k_u lies
// there (the last chunk also the outputs with k_u >= T).  Forward: a thread walks its frames in increasing order,
// with register tiles of KB_TS_U frames loaded one tile ahead, keeps |X| and q of the previous frame, and emits the
// outputs with k_u = f - 1 when frame f arrives, so each input element is loaded and its angle taken once.  Pass 1
// (chunked only) writes each chunk's uint32 phase sum; pass 2 starts chunk c from q(X[0]) plus the sums of the
// chunks before it.  Backward: a thread walks its frames in decreasing order with the same tiles, carrying lam and
// the accumulators of the two open frames; it processes the outputs with k_u in [c Tc - 1, end) and writes gX of
// its own frames, every one exactly once (zeros included).  The outputs with k_u = c Tc - 1 belong to the chunk
// below and are recomputed.  Pass 1 writes each chunk's float sum of gphi; pass 2 starts lam from the sums of the
// chunks above.
//
// Like the other bodies these are barrier-free per-thread functions: the CUDA wrappers call them with the global
// thread index, the CPU emulation (tests/emu, KB_HOST_EMU) calls them for every index in turn.
#pragma once
#include "stft_core.cuh"
#include "pcen_core.cuh"

#define KB_TS_THREADS 128
#define KB_TS_U 8              // frames per register tile

struct KbTsParams {
    const float2* X;  long long x_sb, x_sc, x_st, x_sf;    // input spectrogram (complex64 element strides)
    float2* Y;        long long y_sb, y_sc, y_st, y_sf;    // forward output; read by the backward
    const float2* G;  long long g_sb, g_sc, g_st, g_sf;    // backward: gradient of Y
    float2* gX;       long long o_sb, o_sc, o_st, o_sf;    // backward: gradient of X
    double rate, inv_rate;                                 // inv_rate = 1 / rate (a first guess only)
    int B, C, T, F, T_out;
    int c_inner;                                           // column index runs over c fastest
    long long n_cols;                                      // B C F
    int K, Tc;                                             // chunks, frames per chunk (K = ceil(T / Tc))
    void* state;                                           // (K, n_cols) chunk sums: uint32 forward, float backward
};

struct KbTsCol {
    long long x, y, g, o;      // element offsets of the column's frame 0 in X, Y, G, gX
};

// Thread i -> (chunk, column) and the column's (b, c, f), in 32-bit arithmetic (the host keeps K n_cols < 2^32).
KB_FN KbTsCol kb_ts_col(const KbTsParams& p, long long i, int* chunk, long long* column) {
    const unsigned ui = (unsigned)i, n = (unsigned)p.n_cols, C = (unsigned)p.C, F = (unsigned)p.F;
    const unsigned k = ui / n, col = ui - k * n;
    unsigned b, c, f;
    if (p.c_inner) { c = col % C; const unsigned r = col / C; f = r % F; b = r / F; }
    else { f = col % F; const unsigned r = col / F; c = r % C; b = r / C; }
    *chunk = (int)k;
    *column = col;
    KbTsCol o;
    o.x = (long long)b * p.x_sb + (long long)c * p.x_sc + (long long)f * p.x_sf;
    o.y = (long long)b * p.y_sb + (long long)c * p.y_sc + (long long)f * p.y_sf;
    o.g = (long long)b * p.g_sb + (long long)c * p.g_sc + (long long)f * p.g_sf;
    o.o = (long long)b * p.o_sb + (long long)c * p.o_sc + (long long)f * p.o_sf;
    return o;
}

// k_u = floor(u rate) with u rate one float64 product.  torch's float64 arange, formed blockwise, agrees on the floor
// except at exact-integer points of some rates (DESIGN.md, time stretch).
KB_FN int kb_ts_k(double rate, int u) { return (int)floor((double)u * rate); }
KB_FN float kb_ts_alpha(double rate, int u) {
    const double ts = (double)u * rate;
    return (float)(ts - floor(ts));
}

// The smallest output u in [0, T_out] with k_u >= f.
KB_FN int kb_ts_first(const KbTsParams& p, int f) {
    if (f <= 0) return 0;
    const double e = ceil((double)f * p.inv_rate);
    int u = e < (double)p.T_out ? (int)e : p.T_out;
    while (u > 0 && kb_ts_k(p.rate, u - 1) >= f) --u;
    while (u < p.T_out && kb_ts_k(p.rate, u) < f) ++u;
    return u;
}

// Chunk k's frames [f0, f1) and outputs [u0, u1).
KB_FN void kb_ts_chunk(const KbTsParams& p, int k, int* f0, int* f1, int* u0, int* u1) {
    *f0 = k * p.Tc;
    *f1 = *f0 + p.Tc < p.T ? *f0 + p.Tc : p.T;
    *u0 = kb_ts_first(p, *f0);
    *u1 = k == p.K - 1 ? p.T_out : kb_ts_first(p, *f1);
}

// Fixed-point angle: rint(atan2 2^31 / pi) mod 2^32.  The product is formed in float64, so the only rounding after
// kb_atan2 is the final one to an integer (at most 2^-32 turn = 7.3e-10 rad).
KB_FN unsigned kb_ts_q(float2 z) {
    const float a = kb_atan2(z.y, z.x);
    return (unsigned)(long long)rint((double)a * 683565275.5764316);     // 2^31 / pi
}

KB_FN float kb_ts_abs(float2 z) { return kb_cabs<true>(z.x, z.y); }

// (cos, sin) of pi s.  The device computes sincospif; the emulation rounds the float64 values.
#if defined(KB_HOST_EMU)
inline void kb_ts_cispi(float s, float* c, float* sn) {
    const double a = 3.14159265358979323846 * (double)s;
    *c = (float)std::cos(a);
    *sn = (float)std::sin(a);
}
#else
KB_D void kb_ts_cispi(float s, float* c, float* sn) { sincospif(s, sn, c); }
#endif

KB_FN float2 kb_ts_ld(const float2* x, long long off) {
#if defined(__CUDA_ARCH__)
    return __ldg(x + off);
#else
    return x[off];
#endif
}

// ------------------------------------------------------------------------------------------ forward
// OUT = false: pass 1 (chunked only), thread i < (K - 1) n_cols writes the phase sum of chunk i / n_cols.
// OUT = true: pass 2 (the only pass when K = 1), thread i < K n_cols writes the outputs of chunk i / n_cols.
template <bool OUT>
KB_FN void kb_ts_fwd(const KbTsParams& p, long long i) {
    int k;
    long long col;
    const KbTsCol cl = kb_ts_col(p, i, &k, &col);
    int f0, f1, u, u1;
    kb_ts_chunk(p, k, &f0, &f1, &u, &u1);
    unsigned phi = 0u;
    if (OUT) {
        phi = kb_ts_q(kb_ts_ld(p.X, cl.x));
        const unsigned* st = (const unsigned*)p.state;
        for (int j = 0; j < k; ++j) phi += st[(long long)j * p.n_cols + col];
    }
    if (u < u1) {
        const float2* x = p.X + cl.x;
        float2* y = OUT ? p.Y + cl.y : nullptr;
        const int f_last = kb_ts_k(p.rate, u1 - 1) + 1;      // the last frame any output of the chunk reads
        const int f_ld = f_last < p.T - 1 ? f_last : p.T - 1;  // frames past T - 1 are the zero padding
        int ku = kb_ts_k(p.rate, u);
        float pm = 0.0f;
        unsigned pq = 0u;
        float2 cur[KB_TS_U], nxt[KB_TS_U];
#pragma unroll
        for (int j = 0; j < KB_TS_U; ++j)
            cur[j] = f0 + j <= f_ld ? kb_ts_ld(x, (long long)(f0 + j) * p.x_st) : make_float2(0.0f, 0.0f);
        for (int t = f0; t <= f_last; t += KB_TS_U) {
#pragma unroll
            for (int j = 0; j < KB_TS_U; ++j) {
                const int tn = t + KB_TS_U + j;
                nxt[j] = tn <= f_ld ? kb_ts_ld(x, (long long)tn * p.x_st) : make_float2(0.0f, 0.0f);
            }
#pragma unroll
            for (int j = 0; j < KB_TS_U; ++j) {
                const int f = t + j;
                if (f <= f_last) {
                    const unsigned q = kb_ts_q(cur[j]);
                    const float m = OUT ? kb_ts_abs(cur[j]) : 0.0f;
                    while (u < u1 && ku == f - 1) {       // outputs between frames f - 1 and f
                        if (OUT) {
                            const float a = kb_ts_alpha(p.rate, u);
                            const float mag = fmaf(a, m, (1.0f - a) * pm);
                            float c, s;
                            kb_ts_cispi((float)(int)phi * 0x1p-31f, &c, &s);
                            y[(long long)u * p.y_st] = make_float2(mag * c, mag * s);
                        }
                        phi += q - pq;
                        ku = kb_ts_k(p.rate, ++u);
                    }
                    pm = m;
                    pq = q;
                }
            }
#pragma unroll
            for (int j = 0; j < KB_TS_U; ++j) cur[j] = nxt[j];
        }
    }
    if (!OUT) ((unsigned*)p.state)[(long long)k * p.n_cols + col] = phi;
}

// ------------------------------------------------------------------------------------------ backward
// gm and gphi of output u.
KB_FN void kb_ts_out_grad(const KbTsParams& p, const KbTsCol& cl, int u, float* gm, float* gphi) {
    const float2 yv = kb_ts_ld(p.Y, cl.y + (long long)u * p.y_st);
    const float2 gv = kb_ts_ld(p.G, cl.g + (long long)u * p.g_st);
    const float r = kb_ts_abs(yv);
    const float re = fmaf(yv.x, gv.x, yv.y * gv.y);
    const float im = fmaf(yv.x, gv.y, -yv.y * gv.x);
    *gm = r > 0.0f ? re / r : 0.0f;
    *gphi = r > 0.0f ? im : 0.0f;
}

// Pass 1 (chunked only): thread i < (K - 1) n_cols writes the sum of gphi over the outputs of chunk 1 + i / n_cols.
KB_FN void kb_ts_bwd_state(const KbTsParams& p, long long i) {
    int k;
    long long col;
    const KbTsCol cl = kb_ts_col(p, i, &k, &col);
    ++k;
    int f0, f1, u0, u1;
    kb_ts_chunk(p, k, &f0, &f1, &u0, &u1);
    float lam = 0.0f;
#pragma unroll 4
    for (int u = u1 - 1; u >= u0; --u) {
        float gm, gphi;
        kb_ts_out_grad(p, cl, u, &gm, &gphi);
        lam += gphi;
    }
    ((float*)p.state)[(long long)k * p.n_cols + col] = lam;
}

// gX of one frame from its accumulators.
KB_FN float2 kb_ts_gx(float2 xv, float gmag, float gth) {
    const float r = kb_ts_abs(xv);
    if (!(r > 0.0f)) return make_float2(0.0f, 0.0f);
    const float inv = 1.0f / r;
    const float a = gmag * inv, b = gth * inv * inv;          // gX = X (a + i b)
    return make_float2(fmaf(xv.x, a, -xv.y * b), fmaf(xv.y, a, xv.x * b));
}

// Pass 2 (the only pass when K = 1): thread i < K n_cols writes gX of the frames of chunk i / n_cols.
KB_FN void kb_ts_bwd_out(const KbTsParams& p, long long i) {
    int k;
    long long col;
    const KbTsCol cl = kb_ts_col(p, i, &k, &col);
    int f0, f1, u0, u1;
    kb_ts_chunk(p, k, &f0, &f1, &u0, &u1);
    float lam = 0.0f;                                          // sum of gphi over the outputs after u
    {
        const float* st = (const float*)p.state;
        for (int j = p.K - 1; j > k; --j) lam += st[(long long)j * p.n_cols + col];
    }
    int u = u1 - 1;
    int ku = u >= 0 ? kb_ts_k(p.rate, u) : -2;
    // frame w's accumulators; the outputs with k_u >= f1 - 1 come first (only their lower frame can be ours)
    float am = 0.0f, at = 0.0f;
    while (u >= 0 && ku >= f1 - 1) {
        float gm, gphi;
        kb_ts_out_grad(p, cl, u, &gm, &gphi);
        if (ku == f1 - 1) {
            am = fmaf(1.0f - kb_ts_alpha(p.rate, u), gm, am);
            at -= lam;
        }
        lam += gphi;
        ku = --u >= 0 ? kb_ts_k(p.rate, u) : -2;
    }
    const float2* x = p.X + cl.x;
    float2* gx = p.gX + cl.o;
    float2 cur[KB_TS_U], nxt[KB_TS_U];                         // X[t - j]
#pragma unroll
    for (int j = 0; j < KB_TS_U; ++j)
        cur[j] = f1 - 1 - j >= f0 ? kb_ts_ld(x, (long long)(f1 - 1 - j) * p.x_st) : make_float2(0.0f, 0.0f);
    for (int t = f1 - 1; t >= f0; t -= KB_TS_U) {
#pragma unroll
        for (int j = 0; j < KB_TS_U; ++j) {
            const int tn = t - KB_TS_U - j;
            nxt[j] = tn >= f0 ? kb_ts_ld(x, (long long)tn * p.x_st) : make_float2(0.0f, 0.0f);
        }
#pragma unroll
        for (int j = 0; j < KB_TS_U; ++j) {
            const int w = t - j;
            if (w >= f0) {
                float nm = 0.0f, nt = 0.0f;                    // frame w - 1
                while (u >= 0 && ku == w - 1) {                // outputs between frames w - 1 and w
                    float gm, gphi;
                    kb_ts_out_grad(p, cl, u, &gm, &gphi);
                    const float a = kb_ts_alpha(p.rate, u);
                    am = fmaf(a, gm, am);
                    at += lam;
                    nm = fmaf(1.0f - a, gm, nm);
                    nt -= lam;
                    lam += gphi;
                    ku = --u >= 0 ? kb_ts_k(p.rate, u) : -2;
                }
                if (w == 0) at += lam;                         // phi[u] contains q(X[0]) for every u
                gx[(long long)w * p.o_st] = kb_ts_gx(cur[j], am, at);
                am = nm;
                at = nt;
            }
        }
#pragma unroll
        for (int j = 0; j < KB_TS_U; ++j) cur[j] = nxt[j];
    }
}

// ------------------------------------------------------------------------------------------ host side
// Chunk count for n_cols columns of T input frames on a GPU that holds `resident` threads at once: PCEN's rule (one
// chunk while the columns fill a sixteenth of the GPU, else up to 32 chunks of at least 64 frames).
inline int kb_ts_chunks(long long n_cols, int T, long long resident) { return kb_pcen_chunks(n_cols, T, resident); }

// Frames per chunk and the resulting chunk count for a requested count K (Tc = ceil(T / K), K = ceil(T / Tc)).
inline void kb_ts_set_chunks(KbTsParams& p, int K) {
    if (K < 1 || p.T <= 0) K = 1;
    p.Tc = p.T > 0 ? (p.T + K - 1) / K : 1;
    p.K = p.T > 0 ? (p.T + p.Tc - 1) / p.Tc : 1;
}
