// Kernel bodies of per-channel energy normalisation (PCEN) and its gradient.  Every column (b, c, f) of a
// non-negative spectrogram E is processed independently along time:
//   M[-1] = E[0],  M[t] = (1 - s) M[t-1] + s E[t],  A = eps + M,
//   u = E A^-a,    y = d^r expm1(r log1p(u / d))        (= (u + d)^r - d^r without cancellation)
// with a = gain, d = bias, r = power, s = smooth_coef per band (a parameter pointer with element stride 0 is one
// value for every band).  The backward pass is the reverse-time scan
//   lam[t] = gM[t] + (1 - s) lam[t+1],  gE[t] = gy D A^-a + s lam[t]  (lam[0] in full at t = 0)
// with D = dy/du and gM = -gy D a u / A, plus per-column sums of the four parameter gradients.
//
// Work split: one thread per (chunk, column).  A warp's 32 columns are neighbours in memory at every frame (the
// column index runs over c fastest when the channel axis is the innermost one, as in channels_last, else over f
// fastest), so each frame is one coalesced 128 B access per warp.  The recurrence is serial in time, so a
// thread keeps a tile of U frames of its inputs in registers and loads the next tile before it works through the
// current one: U to 2U loads per input stream stay in flight behind the dependent arithmetic.
//
// Chunks: M is linear in its start state, M[t] = M_local[t] + (1 - s)^(t - t0 + 1) M[t0 - 1], so time can be cut
// into K chunks of Tc frames when there are too few columns to fill the GPU.  Pass 1 writes each chunk's end
// state from a zero start (chunk 0 from E[0]); pass 2 folds the states of the chunks before its own with Horner's
// rule in q = (1 - s)^Tc (at most K - 1 terms) and then runs the full recurrence.  The backward pass chunks the
// same way in reverse: lam is linear in its end state.
//
// Like the other bodies these are barrier-free per-thread functions: the CUDA wrappers call them with the global
// thread index, the CPU emulation (tests/emu, KB_HOST_EMU) calls them for every index in turn.
#pragma once
#include "stft_core.cuh"

#define KB_PCEN_THREADS 128
#define KB_PCEN_U 16            // forward: frames per register tile
#define KB_PCEN_UB 8            // backward: frames per register tile (three input streams)
#define KB_PCEN_MAX_CHUNKS 32   // pass 2 folds at most 31 chunk states

struct KbPcenParams {
    const float* E;   long long e_sb, e_sc, e_st, e_sf;
    float* y;         long long y_sb, y_sc, y_st, y_sf;    // forward output
    float* M;         long long m_sb, m_sc, m_st, m_sf;    // smoother state: written by the forward when non-null,
                                                           // read by the backward
    const float* gy;  long long g_sb, g_sc, g_st, g_sf;    // backward
    float* gE;        long long o_sb, o_sc, o_st, o_sf;
    const float* gain; const float* bias; const float* power; const float* smooth;
    int gain_st, bias_st, power_st, smooth_st;             // 0: one value for every band, 1: one per band
    float eps;
    int B, C, T, F;
    int c_inner;                                           // column index runs over c fastest
    long long n_cols;                                      // B C F
    int K, Tc;                                             // chunks, frames per chunk (K = ceil(T / Tc))
    float* state;                                          // (K, n_cols) chunk end states (K > 1)
    float* part;                                           // backward: (4, K, B, C, F) parameter partial sums
};

struct KbPcenCol {
    long long e, y, m, g, o;    // element offsets of the column's frame 0 in E, y, M, gy, gE
    long long bcf;              // (b C + c) F + f: the column's place in the parameter partial sums
    int f;
};

KB_HD KbPcenCol kb_pcen_col(const KbPcenParams& p, long long col) {
    long long b, c, f;
    if (p.c_inner) { c = col % p.C; const long long r = col / p.C; f = r % p.F; b = r / p.F; }
    else { f = col % p.F; const long long r = col / p.F; c = r % p.C; b = r / p.C; }
    KbPcenCol o;
    o.e = b * p.e_sb + c * p.e_sc + f * p.e_sf;
    o.y = b * p.y_sb + c * p.y_sc + f * p.y_sf;
    o.m = b * p.m_sb + c * p.m_sc + f * p.m_sf;
    o.g = b * p.g_sb + c * p.g_sc + f * p.g_sf;
    o.o = b * p.o_sb + c * p.o_sc + f * p.o_sf;
    o.bcf = (b * p.C + c) * p.F + f;
    o.f = (int)f;
    return o;
}

// One band's parameters and the constants derived from them.
struct KbPcenBand {
    float a, d, r, s, s1, inv_d, dr;    // s1 = 1 - s, dr = d^r
};

KB_HD KbPcenBand kb_pcen_band(const KbPcenParams& p, int f) {
    KbPcenBand q;
    q.a = p.gain[f * p.gain_st];
    q.d = p.bias[f * p.bias_st];
    q.r = p.power[f * p.power_st];
    q.s = p.smooth[f * p.smooth_st];
    q.s1 = 1.0f - q.s;
    q.inv_d = 1.0f / q.d;
    q.dr = powf(q.d, q.r);
    return q;
}

// Decay across one full chunk, (1 - s)^Tc.  powf keeps a negative 1 - s (s > 1 after a training step) exact in sign.
KB_HD float kb_pcen_decay(const KbPcenBand& q, int Tc) { return powf(q.s1, (float)Tc); }

KB_HD float kb_pcen_out(const KbPcenBand& q, float e, float m, float eps) {
    const float u = e * expf(-q.a * logf(eps + m));
    return q.dr * expm1f(q.r * log1pf(u * q.inv_d));
}

// ------------------------------------------------------------------------------------------ forward
// Pass 1 (chunked only): thread i < (K - 1) n_cols writes the end state of chunk k = i / n_cols.
KB_FN void kb_pcen_fwd_state(const KbPcenParams& p, long long i) {
    const int k = (int)(i / p.n_cols);
    const long long col = i - (long long)k * p.n_cols;
    const KbPcenCol cl = kb_pcen_col(p, col);
    const KbPcenBand q = kb_pcen_band(p, cl.f);
    const float* e = p.E + cl.e;
    const int t0 = k * p.Tc, t1 = t0 + p.Tc;        // never the last chunk: t1 <= T
    float m = k == 0 ? e[0] : 0.0f;
    float cur[KB_PCEN_U], nxt[KB_PCEN_U];
#pragma unroll
    for (int j = 0; j < KB_PCEN_U; ++j) cur[j] = t0 + j < t1 ? e[(long long)(t0 + j) * p.e_st] : 0.0f;
    for (int t = t0; t < t1; t += KB_PCEN_U) {
#pragma unroll
        for (int j = 0; j < KB_PCEN_U; ++j) {
            const int tn = t + KB_PCEN_U + j;
            nxt[j] = tn < t1 ? e[(long long)tn * p.e_st] : 0.0f;
        }
#pragma unroll
        for (int j = 0; j < KB_PCEN_U; ++j)
            if (t + j < t1) m = fmaf(q.s1, m, q.s * cur[j]);
#pragma unroll
        for (int j = 0; j < KB_PCEN_U; ++j) cur[j] = nxt[j];
    }
    p.state[(long long)k * p.n_cols + col] = m;
}

// Pass 2 (the only pass when K = 1): thread i < K n_cols runs chunk k = i / n_cols from its true start state and
// writes y (and M when p.M is non-null).  y does not depend on whether M is written.
KB_FN void kb_pcen_fwd_out(const KbPcenParams& p, long long i) {
    const int k = (int)(i / p.n_cols);
    const long long col = i - (long long)k * p.n_cols;
    const KbPcenCol cl = kb_pcen_col(p, col);
    const KbPcenBand q = kb_pcen_band(p, cl.f);
    const float* e = p.E + cl.e;
    float* y = p.y + cl.y;
    float* M = p.M ? p.M + cl.m : nullptr;
    const int t0 = k * p.Tc, t1 = t0 + p.Tc < p.T ? t0 + p.Tc : p.T;
    float m;
    if (k == 0) {
        m = e[0];
    } else {
        const float dq = kb_pcen_decay(q, p.Tc);
        m = 0.0f;
        for (int j = 0; j < k; ++j) m = fmaf(m, dq, p.state[(long long)j * p.n_cols + col]);
    }
    float cur[KB_PCEN_U], nxt[KB_PCEN_U];
#pragma unroll
    for (int j = 0; j < KB_PCEN_U; ++j) cur[j] = t0 + j < t1 ? e[(long long)(t0 + j) * p.e_st] : 0.0f;
    for (int t = t0; t < t1; t += KB_PCEN_U) {
#pragma unroll
        for (int j = 0; j < KB_PCEN_U; ++j) {
            const int tn = t + KB_PCEN_U + j;
            nxt[j] = tn < t1 ? e[(long long)tn * p.e_st] : 0.0f;
        }
#pragma unroll
        for (int j = 0; j < KB_PCEN_U; ++j) {
            if (t + j < t1) {
                m = fmaf(q.s1, m, q.s * cur[j]);
                y[(long long)(t + j) * p.y_st] = kb_pcen_out(q, cur[j], m, p.eps);
                if (M) M[(long long)(t + j) * p.m_st] = m;
            }
        }
#pragma unroll
        for (int j = 0; j < KB_PCEN_U; ++j) cur[j] = nxt[j];
    }
}

// ------------------------------------------------------------------------------------------ backward
// The per-frame quantities of the backward pass at one frame.
struct KbPcenBwdTerms {
    float gEd, gM, g_gain, g_bias, g_power;
};

KB_HD KbPcenBwdTerms kb_pcen_bwd_terms(const KbPcenBand& q, float e, float m, float gy, float eps, float log_d) {
    const float A = eps + m;
    const float lA = logf(A);
    const float Aa = expf(-q.a * lA);                  // A^-a
    const float u = e * Aa;
    const float L = log1pf(u * q.inv_d);
    const float x1 = expm1f((q.r - 1.0f) * L);         // (1 + u/d)^(r-1) - 1
    const float xr = expm1f(q.r * L);                  // (1 + u/d)^r - 1
    const float rdr1 = q.r * q.dr * q.inv_d;           // r d^(r-1)
    const float gyD = gy * rdr1 * (1.0f + x1);         // gy dy/du
    KbPcenBwdTerms o;
    o.gEd = gyD * Aa;
    o.gM = -gyD * q.a * u / A;
    o.g_gain = -gyD * u * lA;
    o.g_bias = gy * rdr1 * x1;
    o.g_power = gy * q.dr * (log_d * xr + (1.0f + xr) * L);
    return o;
}

// Loads one backward tile: frames t - j for j = 0..UB-1 that lie in [t0, t), zeros elsewhere.
KB_HD void kb_pcen_bwd_load(const KbPcenParams& p, const KbPcenCol& cl, int t, int t0, float* e, float* m, float* g) {
#pragma unroll
    for (int j = 0; j < KB_PCEN_UB; ++j) {
        const int tt = t - j;
        const bool in = tt >= t0;
        e[j] = in ? p.E[cl.e + (long long)tt * p.e_st] : 0.0f;
        m[j] = in ? p.M[cl.m + (long long)tt * p.m_st] : 0.0f;
        g[j] = in ? p.gy[cl.g + (long long)tt * p.g_st] : 0.0f;
    }
}

// Pass 1 (chunked only): thread i < (K - 1) n_cols writes lam at the first frame of chunk k = 1 + i / n_cols,
// scanned from a zero end state.
KB_FN void kb_pcen_bwd_state(const KbPcenParams& p, long long i) {
    const int k = 1 + (int)(i / p.n_cols);
    const long long col = i - (long long)(k - 1) * p.n_cols;
    const KbPcenCol cl = kb_pcen_col(p, col);
    const KbPcenBand q = kb_pcen_band(p, cl.f);
    const float log_d = logf(q.d);
    const int t0 = k * p.Tc, t1 = t0 + p.Tc < p.T ? t0 + p.Tc : p.T;
    float lam = 0.0f;
    float ce[KB_PCEN_UB], cm[KB_PCEN_UB], cg[KB_PCEN_UB], ne[KB_PCEN_UB], nm[KB_PCEN_UB], ng[KB_PCEN_UB];
    kb_pcen_bwd_load(p, cl, t1 - 1, t0, ce, cm, cg);
    for (int t = t1 - 1; t >= t0; t -= KB_PCEN_UB) {
        kb_pcen_bwd_load(p, cl, t - KB_PCEN_UB, t0, ne, nm, ng);
#pragma unroll
        for (int j = 0; j < KB_PCEN_UB; ++j) {
            if (t - j >= t0) {
                const KbPcenBwdTerms w = kb_pcen_bwd_terms(q, ce[j], cm[j], cg[j], p.eps, log_d);
                lam = fmaf(q.s1, lam, w.gM);
            }
        }
#pragma unroll
        for (int j = 0; j < KB_PCEN_UB; ++j) { ce[j] = ne[j]; cm[j] = nm[j]; cg[j] = ng[j]; }
    }
    p.state[(long long)k * p.n_cols + col] = lam;
}

// Pass 2 (the only pass when K = 1): thread i < K n_cols scans chunk k = i / n_cols from its true end state,
// writes gE and the chunk's four parameter partial sums part[j][k][b][c][f] (j: gain, bias, power, smooth_coef).
KB_FN void kb_pcen_bwd_out(const KbPcenParams& p, long long i) {
    const int k = (int)(i / p.n_cols);
    const long long col = i - (long long)k * p.n_cols;
    const KbPcenCol cl = kb_pcen_col(p, col);
    const KbPcenBand q = kb_pcen_band(p, cl.f);
    const float log_d = logf(q.d);
    const int t0 = k * p.Tc, t1 = t0 + p.Tc < p.T ? t0 + p.Tc : p.T;
    float lam = 0.0f;               // lam[t1]
    if (k + 1 < p.K) {
        const float dq = kb_pcen_decay(q, p.Tc);
        for (int j = p.K - 1; j > k; --j) lam = fmaf(lam, dq, p.state[(long long)j * p.n_cols + col]);
    }
    // M[t0 - 1]: the state before the chunk's first frame (E[0] before frame 0, whose term below is zero)
    const float m_before = t0 > 0 ? p.M[cl.m + (long long)(t0 - 1) * p.m_st] : p.E[cl.e];
    float s_gain = 0.0f, s_bias = 0.0f, s_power = 0.0f, s_smooth = 0.0f;
    float ce[KB_PCEN_UB], cm[KB_PCEN_UB], cg[KB_PCEN_UB], ne[KB_PCEN_UB], nm[KB_PCEN_UB], ng[KB_PCEN_UB];
    kb_pcen_bwd_load(p, cl, t1 - 1, t0, ce, cm, cg);
    for (int t = t1 - 1; t >= t0; t -= KB_PCEN_UB) {
        kb_pcen_bwd_load(p, cl, t - KB_PCEN_UB, t0, ne, nm, ng);
#pragma unroll
        for (int j = 0; j < KB_PCEN_UB; ++j) {
            const int tt = t - j;
            if (tt >= t0) {
                const KbPcenBwdTerms w = kb_pcen_bwd_terms(q, ce[j], cm[j], cg[j], p.eps, log_d);
                lam = fmaf(q.s1, lam, w.gM);
                const float m_prev = tt - 1 < t0 ? m_before : (j + 1 < KB_PCEN_UB ? cm[j + 1] : nm[0]);
                p.gE[cl.o + (long long)tt * p.o_st] = fmaf(tt > 0 ? q.s : 1.0f, lam, w.gEd);
                s_gain += w.g_gain;
                s_bias += w.g_bias;
                s_power += w.g_power;
                s_smooth = fmaf(lam, ce[j] - m_prev, s_smooth);
            }
        }
#pragma unroll
        for (int j = 0; j < KB_PCEN_UB; ++j) { ce[j] = ne[j]; cm[j] = nm[j]; cg[j] = ng[j]; }
    }
    const long long n = (long long)p.K * p.n_cols, o = (long long)k * p.n_cols + cl.bcf;
    p.part[o] = s_gain;
    p.part[n + o] = s_bias;
    p.part[2 * n + o] = s_power;
    p.part[3 * n + o] = s_smooth;
}

// ------------------------------------------------------------------------------------------ host side
// Chunk count for n_cols columns of T frames on a GPU that holds `resident` threads at once: one chunk while the
// columns alone fill a sixteenth of the GPU (chunking costs a second read of the inputs), else enough chunks to
// reach a quarter of it, at most KB_PCEN_MAX_CHUNKS and none shorter than 64 frames.
inline int kb_pcen_chunks(long long n_cols, int T, long long resident) {
    if (n_cols <= 0 || T <= 0 || n_cols * 16 >= resident) return 1;
    long long K = (resident / 4 + n_cols - 1) / n_cols;
    if (K > KB_PCEN_MAX_CHUNKS) K = KB_PCEN_MAX_CHUNKS;
    if (K > T / 64) K = T / 64;
    return K < 2 ? 1 : (int)K;
}

// Frames per chunk and the resulting chunk count for a requested count K (Tc = ceil(T / K), K = ceil(T / Tc)).
inline void kb_pcen_set_chunks(KbPcenParams& p, int K) {
    if (K < 1 || p.T <= 0) K = 1;
    p.Tc = p.T > 0 ? (p.T + K - 1) / K : 1;
    p.K = p.T > 0 ? (p.T + p.Tc - 1) / p.Tc : 1;
}
