// Bodies of the backward passes of the layers next to the hot path: Phase, get_stft_mag_phase's fused mode,
// Delta, Frame, Energy and ConcatenateFrequencyMap.  (SpecAugment needs no pass of its own: its gradient is the
// forward launch over the gradient with mask value 0 and the same masks.)
//
// As in grad_core.cuh, every body is one barrier-free element function of a single thread: the CUDA wrappers call
// it with the global thread index, the CPU emulation (tests/emu, KB_HOST_EMU) calls it for every index in turn.
// Each output element is written exactly once (gathers, no atomics).  Gradients of complex tensors follow
// PyTorch's convention, dL/dRe + i dL/dIm.
#pragma once
#include "stft_core.cuh"

// tf.pad's SYMMETRIC (0) / REFLECT (1) extension of a length-T axis: the index in [0, T) that position t reads,
// or -1 for a zero (CONSTANT (2), or a position more than one reflection away).  Integer-only: Delta's forward
// and backward share it.
KB_FN long long kb_pad_index(long long t, long long T, int mode) {
    if (t >= 0 && t < T) return t;
    if (mode == 2) return -1;
    if (t < 0) t = (mode == 0) ? (-t - 1) : (-t);
    else t = (mode == 0) ? (2 * T - 1 - t) : (2 * T - 2 - t);
    return (t >= 0 && t < T) ? t : -1;
}

// ------------------------------------------------------------------------------------------ Phase
// d angle(X) / dX: gX = g i X / |X|^2 (torch.angle's rule), 0 where |X| = 0.
KB_FN void kb_phase_bwd_elem(const float2* __restrict__ X, const float* __restrict__ g, float2* __restrict__ gX,
                             long long i) {
    const float2 v = X[i];
    const float m = kb_sqrt(v.x * v.x + v.y * v.y);
    const float s = m > 0.0f ? (g[i] / m) / m : 0.0f;
    gX[i] = make_float2(-s * v.y, s * v.x);
}

// ------------------------------------------------------------------------------------------ magnitude + phase
// Fused mode 5 (|X| in channels [0, C), angle(X) in [C, 2C)): gX = X / |X| (g_mag + i g_phase / |X|), 0 where
// |X| = 0.  g_mag is the magnitude half's gradient after the decibel backward, if any.  Every tensor is addressed
// through its own (batch, channel, frame, bin) element strides; a NULL gm or gp stands for zeros.  The thread
// index walks (b, c, t, f) with f fastest, or (b, t, f, c) with c fastest when `c_inner` (channels_last gX).
struct KbMagPhaseBwdParams {
    const float2* X;  long long x_sb, x_sc, x_st, x_sf;
    const float* gm;  long long m_sb, m_sc, m_st, m_sf;
    const float* gp;  long long p_sb, p_sc, p_st, p_sf;
    float2* gX;       long long o_sb, o_sc, o_st, o_sf;
    long long C, T, F;
    int c_inner;
};

KB_FN void kb_mag_phase_bwd_elem(const KbMagPhaseBwdParams& p, long long i) {
    long long b, c, t, f;
    if (p.c_inner) { c = i % p.C; const long long r = i / p.C; f = r % p.F; t = (r / p.F) % p.T; b = r / (p.F * p.T); }
    else { f = i % p.F; const long long r = i / p.F; t = r % p.T; c = (r / p.T) % p.C; b = r / (p.T * p.C); }
    const float2 v = p.X[b * p.x_sb + c * p.x_sc + t * p.x_st + f * p.x_sf];
    const float gm = p.gm ? p.gm[b * p.m_sb + c * p.m_sc + t * p.m_st + f * p.m_sf] : 0.0f;
    const float gp = p.gp ? p.gp[b * p.p_sb + c * p.p_sc + t * p.p_st + f * p.p_sf] : 0.0f;
    const float m = kb_sqrt(v.x * v.x + v.y * v.y);
    float a = 0.0f, q = 0.0f;           // gX = a X + q i X
    if (m > 0.0f) { a = gm / m; q = (gp / m) / m; }
    p.gX[b * p.o_sb + c * p.o_sc + t * p.o_st + f * p.o_sf] = make_float2(a * v.x - q * v.y, a * v.y + q * v.x);
}

// ------------------------------------------------------------------------------------------ Delta
// Forward: y[t] = inv_denom sum_{m=1..n} m (x[P(t+m)] - x[P(t-m)]), P = kb_pad_index (a -1 reads zero), on a
// contiguous (outer, T, inner) tensor.  Adjoint, gathered per input position s:
//   gx[s] = inv_denom sum_{u: P(u) = s} sum_{m=1..n} m (g[u - m] - g[u + m]),   terms with frames outside [0, T) dropped,
// where u runs over s itself and its mirror images (symmetric: -s-1, 2T-1-s; reflect: -s, 2T-2-s).  A mirror image
// counts only if P really maps it back to s, which keeps short axes (T <= n) exact.
KB_FN float kb_delta_bwd_tap(const float* gb, long long u, long long T, long long inner, int n) {
    float acc = 0.0f;
    for (int m = 1; m <= n; ++m) {
        const long long tp = u - m, tm = u + m;
        const float a = (tp >= 0 && tp < T) ? gb[tp * inner] : 0.0f;
        const float b = (tm >= 0 && tm < T) ? gb[tm * inner] : 0.0f;
        acc += (float)m * (a - b);
    }
    return acc;
}

KB_FN void kb_delta_bwd_elem(const float* __restrict__ g, float* __restrict__ gx, long long T, long long inner, int n,
                             float inv_denom, int mode, long long i) {
    const long long in = i % inner;
    const long long s = (i / inner) % T;
    const long long o = i / (inner * T);
    const float* gb = g + o * T * inner + in;
    float acc = kb_delta_bwd_tap(gb, s, T, inner, n);
    if (mode != 2) {
        const long long u0 = (mode == 0) ? (-s - 1) : (-s);
        const long long u1 = (mode == 0) ? (2 * T - 1 - s) : (2 * T - 2 - s);
        if (u0 < 0 && u0 >= -n && kb_pad_index(u0, T, mode) == s) acc += kb_delta_bwd_tap(gb, u0, T, inner, n);
        if (u1 >= T && u1 < T + n && kb_pad_index(u1, T, mode) == s) acc += kb_delta_bwd_tap(gb, u1, T, inner, n);
    }
    gx[i] = acc * inv_denom;
}

// ------------------------------------------------------------------------------------------ Frame / Energy
// Frames t = 0..T-1 start at t hop and hold frame_length samples; positions past the signal hold a constant, so
// only samples s < L receive gradient.  Both passes walk the frames covering s: t from min(s / hop, T - 1) down
// while s - t hop < frame_length; a sample no frame covers gets 0.
struct KbFrameBwdParams {
    const float* g;               // Frame: (b, c, frame, n) element strides; Energy: (b, c, frame), g_sn unused
    long long g_sb, g_sc, g_st, g_sn;
    const float* x;               // Energy only: the forward's input
    long long x_sb, x_sc, x_sl;
    float* gx;
    long long o_sb, o_sc, o_sl;
    int C, L, T, fl, hop;
    float scale2;                 // Energy only: 2 * scale
};

// Frame: gx[s] = sum_t g[t, s - t hop]
KB_FN void kb_frame_bwd_elem(const KbFrameBwdParams& p, long long i) {
    const long long s = i % p.L, bc = i / p.L;
    const long long c = bc % p.C, b = bc / p.C;
    const float* gb = p.g + b * p.g_sb + c * p.g_sc;
    long long t = s / p.hop;
    if (t > p.T - 1) t = p.T - 1;
    float acc = 0.0f;
    for (; t >= 0; --t) {
        const long long n = s - t * p.hop;
        if (n >= p.fl) break;
        acc += gb[t * p.g_st + n * p.g_sn];
    }
    p.gx[b * p.o_sb + c * p.o_sc + s * p.o_sl] = acc;
}

// Energy: y[t] = scale sum_n frame_t[n]^2, so gx[s] = 2 scale x[s] sum_t g[t]
KB_FN void kb_energy_bwd_elem(const KbFrameBwdParams& p, long long i) {
    const long long s = i % p.L, bc = i / p.L;
    const long long c = bc % p.C, b = bc / p.C;
    const float* gb = p.g + b * p.g_sb + c * p.g_sc;
    long long t = s / p.hop;
    if (t > p.T - 1) t = p.T - 1;
    float acc = 0.0f;
    bool covered = false;
    for (; t >= 0 && s - t * p.hop < p.fl; --t) { acc += gb[t * p.g_st]; covered = true; }
    const float xv = p.x[b * p.x_sb + c * p.x_sc + s * p.x_sl];
    p.gx[b * p.o_sb + c * p.o_sc + s * p.o_sl] = covered ? p.scale2 * xv * acc : 0.0f;
}

// ------------------------------------------------------------------------------------------ ConcatenateFrequencyMap
// The appended channel is a constant, so gx is the first C channels of the (C + 1)-channel gradient: contiguous
// (b, t, f, c) [channels_last] or (b, c, t, f) tensors, gx indexed by i.
KB_FN void kb_concat_fm_bwd_elem(const float* __restrict__ g, float* __restrict__ gx, long long C, long long T,
                                 long long F, int channels_last, long long i) {
    long long src;
    if (channels_last) {
        const long long c = i % C, r = i / C;              // r = (b T + t) F + f
        src = r * (C + 1) + c;
    } else {
        const long long tf = i % (T * F), bc = i / (T * F);
        const long long c = bc % C, b = bc / C;
        src = (b * (C + 1) + c) * (T * F) + tf;
    }
    gx[i] = g[src];
}
