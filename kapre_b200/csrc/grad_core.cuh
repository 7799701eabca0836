// Bodies of the passes the backward entry points need on top of the existing transform kernels.
//
// Every linear adjoint of the hot path is an existing launch with another constant table:
//   * STFT^T      = the inverse-STFT kernel with the dual window w * n_fft / 2, plus kb_stft_adj_cta (below);
//   * ISTFT^T     = the forward STFT kernel with the window dual * 2 / n_fft, plus kb_istft_adj_cta;
//   * filterbank^T = the filterbank kernel with the transposed (n_bands, n_freq) matrix.
// The non-linear layers get their own passes: kb_mag_bwd_elem (Magnitude) and kb_dbb_* (MagnitudeToDecibel).
//
// Each body is one barrier-free phase of a single thread: the CUDA wrappers call it with the global thread index,
// the CPU emulation (tests/emu, KB_HOST_EMU) calls it for every index in turn.  Atomics on the per-item workspace
// become plain read-modify-writes there, and the warp reductions in front of them are the identity.
#pragma once
#include "stft_core.cuh"

#if defined(KB_HOST_EMU)
inline unsigned kb_grad_wmax_u32(unsigned v) { return v; }
inline float kb_grad_wsum(float v) { return v; }
inline unsigned kb_grad_wsum_u32(unsigned v) { return v; }
inline bool kb_grad_lead(long long) { return true; }
inline void kb_grad_atomic_max(unsigned* a, unsigned v) { if (v > *a) *a = v; }
inline void kb_grad_atomic_add(float* a, float v) { *a += v; }
inline void kb_grad_atomic_add(unsigned* a, unsigned v) { *a += v; }
#else
KB_D unsigned kb_grad_wmax_u32(unsigned v) { return __reduce_max_sync(0xffffffffu, v); }
KB_D unsigned kb_grad_wsum_u32(unsigned v) { return __reduce_add_sync(0xffffffffu, v); }
KB_D float kb_grad_wsum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
KB_D bool kb_grad_lead(long long tid) { return (tid & 31) == 0; }
KB_D void kb_grad_atomic_max(unsigned* a, unsigned v) { if (v) atomicMax(a, v); }
KB_D void kb_grad_atomic_add(float* a, float v) { if (v != 0.0f) atomicAdd(a, v); }
KB_D void kb_grad_atomic_add(unsigned* a, unsigned v) { if (v) atomicAdd(a, v); }
#endif

// ---------------------------------------------------------------------------------------------- STFT adjoint
// The inverse-STFT launch with dual window w * N/2 leaves, at padded sample u,
//   ola[u] = sum_t w[m] (Re G_t0 / 2 + (-1)^m Re G_tP / 2 + sum_{0<k<N/2} Re(G_tk e^{2 pi i k m / N})),  m = u - t hop,
// i.e. the gradient with its DC and Nyquist terms counted half (irfft weighs them 1 against 2).  This pass adds the
// other half, crops the window [pad_left, pad_left + L) of the padded signal and writes 0 wherever no frame's first
// win_eff samples reach (the tail without pad_end, gaps when hop > win_eff): those samples do not enter the STFT.
struct KbStftAdjParams {
    const float2* G;                  // incoming gradient, complex (batch, channel, frame, bin) element strides
    long long g_sb, g_sc, g_st, g_sk;
    const float* ola;                 // overlap-add of the inverse launch, padded samples [0, ola_len)
    long long a_sb, a_sc, a_sl;
    float* gx;                        // gradient of the waveform, (batch, channel, sample) element strides
    long long x_sb, x_sc, x_sl;
    int B, C, L, T;
    int n_fft, hop, win_eff, pad_left;
    const float* w;                   // analysis window, win_eff samples
};

KB_FN void kb_stft_adj_elem(const KbStftAdjParams& p, long long i) {
    const long long s = i % p.L, bc = i / p.L;
    const int c = (int)(bc % p.C), b = (int)(bc / p.C);
    const long long u = s + p.pad_left;
    long long t = u / p.hop;
    if (t > p.T - 1) t = p.T - 1;
    float acc = 0.0f;
    if (t >= 0 && u - t * p.hop < p.win_eff) {
        acc = p.ola[b * p.a_sb + c * p.a_sc + u * p.a_sl];
        const float2* Gs = p.G + b * p.g_sb + c * p.g_sc;
        const bool nyq = (p.n_fft & 1) == 0;
        float edge = 0.0f;
        for (; t >= 0; --t) {
            const int m = (int)(u - t * p.hop);
            if (m >= p.win_eff) break;
            const float2* Gt = Gs + t * p.g_st;
            float e = Gt[0].x;
            if (nyq) {
                const float ny = Gt[(long long)(p.n_fft / 2) * p.g_sk].x;
                e += (m & 1) ? -ny : ny;
            }
            edge += p.w[m] * e;
        }
        acc += 0.5f * edge;
    }
    p.gx[b * p.x_sb + c * p.x_sc + s * p.x_sl] = acc;
}

// ------------------------------------------------------------------------------------------ ISTFT adjoint
// The forward launch with window dual * 2/N over the output gradient gives (2/N) rfft(dual * gy_frame) in every bin;
// the inverse weighs Re X_0 and Re X_{N/2} by 1/N (and ignores their imaginary parts), so those two bins are halved
// and their imaginary parts zeroed, in place.  Odd N has no Nyquist bin.
struct KbIstftAdjParams {
    float2* gX;
    long long sb, sc, st, sk;
    int B, C, T, n_fft;
};

KB_FN void kb_istft_adj_elem(const KbIstftAdjParams& p, long long i) {
    const int nb = (p.n_fft & 1) ? 1 : 2;
    const int e = (int)(i % nb);
    const long long r = i / nb;
    const long long t = r % p.T, bc = r / p.T;
    const long long c = bc % p.C, b = bc / p.C;
    float2* v = p.gX + b * p.sb + c * p.sc + t * p.st + (e ? (long long)(p.n_fft / 2) * p.sk : 0LL);
    *v = make_float2(0.5f * v->x, 0.0f);
}

// ------------------------------------------------------------------------------------------ Magnitude
// d|X| / dX in PyTorch's convention for complex inputs: g X / |X|, 0 where |X| = 0 (tf.math.divide_no_nan,
// torch.sgn).  |X| is formed exactly as the forward kernels form it.
KB_FN void kb_mag_bwd_elem(const float2* __restrict__ X, const float* __restrict__ g, float2* __restrict__ gX,
                           long long i) {
    const float2 v = X[i];
    const float m = kb_sqrt(v.x * v.x + v.y * v.y);
    const float s = m > 0.0f ? g[i] / m : 0.0f;
    gX[i] = make_float2(s * v.x, s * v.y);
}

// ------------------------------------------------------------------------------------------ MagnitudeToDecibel
// y = max(D(x), max_item D(x) - dynamic_range), D(x) = db_mul log2(max(x, amin)) - db_sub, with TensorFlow's gradient
// rules (kapre/backend.py:178-192):
//   * tf.maximum(a, b) passes the gradient to a where a >= b (ties included), else to b;
//   * the threshold's gradient (the sum over the clamped elements) goes to the item's maximum through reduce_max,
//     split equally among tied maxima;
//   * d D / dx = 10 / (ln 10 x) where x >= amin, else 0.
// Three passes over (n_items, item_size), `chunks` CTAs per item, per-item workspace words: [0, n) maximum of
// max(x, amin) (uint view, as the forward keeps it), [n, 2n) sum of the clamped elements' gradients (float),
// [2n, 3n) number of elements equal to the maximum.  The clamp decision repeats the forward's device arithmetic
// (the same D and threshold, and no clamp at all when the threshold is not above D(amin), where the forward's
// clamp pass returns early), so both sides agree on which elements were clamped.
struct KbDbBwdParams {
    const float* x;
    const float* g;
    float* gx;
    long long item_size;
    unsigned int* ws;
    long long n_items;
    float amin, db_mul, db_sub, dyn_range, dscale;   // dscale = 10 / ln 10
};

// pass 1: per-item maximum of max(x, amin); the thread walks elements i0, i0 + step, ... of item `item`
KB_FN void kb_dbb_max(const KbDbBwdParams& p, long long item, long long i0, long long step, long long tid) {
    const float* xi = p.x + item * p.item_size;
    unsigned mx = 0u;
    for (long long i = i0; i < p.item_size; i += step) {
        const float v = kb_floor_keepnan(xi[i], p.amin);
        uint32_t u;
#if defined(KB_HOST_EMU)
        std::memcpy(&u, &v, 4);
#else
        u = __float_as_uint(v);
#endif
        mx = u > mx ? u : mx;
    }
    mx = kb_grad_wmax_u32(mx);
    if (kb_grad_lead(tid)) kb_grad_atomic_max(p.ws + item, mx);
}

KB_FN float kb_dbb_from_bits(unsigned u) {
    float f;
#if defined(KB_HOST_EMU)
    std::memcpy(&f, &u, 4);
#else
    f = __uint_as_float(u);
#endif
    return f;
}

KB_FN float kb_dbb_thr(const KbDbBwdParams& p, float mx, bool* binds) {
    const float thr = (p.db_mul * kb_log2(fmaxf(mx, p.amin)) - p.db_sub) - p.dyn_range;
    const float floor_db = p.db_mul * kb_log2(p.amin) - p.db_sub;
    *binds = thr > floor_db;
    return thr;
}

// pass 2: gradient of the elements that kept their value; per-item sum of the clamped ones' and tie count
KB_FN void kb_dbb_pass(const KbDbBwdParams& p, long long item, long long i0, long long step, long long tid) {
    const float mx = kb_dbb_from_bits(p.ws[item]);
    bool binds;
    const float thr = kb_dbb_thr(p, mx, &binds);
    const float* xi = p.x + item * p.item_size;
    const float* gi = p.g + item * p.item_size;
    float* gxi = p.gx + item * p.item_size;
    float clamped = 0.0f;
    unsigned ties = 0u;
    for (long long i = i0; i < p.item_size; i += step) {
        const float xv = xi[i], gv = gi[i];
        const float v = kb_floor_keepnan(xv, p.amin);
        const float y = p.db_mul * kb_log2(v) - p.db_sub;
        const bool keep = !binds || y >= thr;
        if (!keep) clamped += gv;
        if (v == mx) ties += 1u;
        gxi[i] = (keep && xv >= p.amin) ? gv * (p.dscale / xv) : 0.0f;
    }
    clamped = kb_grad_wsum(clamped);
    ties = kb_grad_wsum_u32(ties);
    if (kb_grad_lead(tid)) {
        kb_grad_atomic_add(reinterpret_cast<float*>(p.ws + p.n_items + item), clamped);
        kb_grad_atomic_add(p.ws + 2 * p.n_items + item, ties);
    }
}

// pass 3: the maxima take an equal share of the threshold's gradient
KB_FN void kb_dbb_share(const KbDbBwdParams& p, long long item, long long i0, long long step) {
    const float mx = kb_dbb_from_bits(p.ws[item]);
    const float sum = kb_dbb_from_bits(p.ws[p.n_items + item]);
    const unsigned ties = p.ws[2 * p.n_items + item];
    if (sum == 0.0f || ties == 0u) return;
    const float share = sum / (float)ties;
    const float* xi = p.x + item * p.item_size;
    float* gxi = p.gx + item * p.item_size;
    for (long long i = i0; i < p.item_size; i += step) {
        const float xv = xi[i];
        if (kb_floor_keepnan(xv, p.amin) == mx && xv >= p.amin) gxi[i] += share * (p.dscale / xv);
    }
}
