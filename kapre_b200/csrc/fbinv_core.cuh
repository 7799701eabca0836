// Kernel body of the filterbank inversion (kapre_filterbank_invert in kapre_b200.cu launches it): per frame, the
// non-negative least-squares problem  min ||A s - m||^2  subject to s >= 0, with A the (n_bands x n_freq) transpose of
// the filterbank matrix, solved by projected accelerated gradient (FISTA) with a fixed number of iterations:
//   s_0 = max(A^T (m / d), 0),  d = A A^T 1 (m / d = 0 where d = 0);  y_0 = s_0,  t_0 = 1
//   s_{k+1} = max(y_k - step A^T (A y_k - m), 0),  t_{k+1} = (1 + sqrt(1 + 4 t_k^2)) / 2,
//   y_{k+1} = s_{k+1} + ((t_k - 1) / t_{k+1}) (s_{k+1} - s_k);   the output is s_n.
// step = 1 / ||A||_2^2 and 1 / d are computed in float64 when the plan is made and stored as float32.  t_k runs in
// float64 inside the kernel (one uniform scalar per iteration), so no per-call host table is needed.
//
// Organisation (as kb_fb_cta): persistent CTAs over tiles of R frames of one (item, channel).  The tile's state
// lives in shared memory as [row][frame] with row stride R + 1: s and y over the n_freq bins (+3 zero rows that the
// 4-wide band dots may read), m and the residual r over the bands.  A lane owns a frame; warps walk bands in the
// residual phase (banded row dots, kb_make_bands lists) and bins in the update phase (the bin's column list: at most 2
// entries for a mel bank).  Each frame's arithmetic is a fixed sequence of explicitly rounded operations that does not
// depend on R, the CTA count, the frame's place in the batch or the strides, so neither does its output.  No atomics.
//
// The projection max(v, 0) is written v < 0 ? 0 : v, so a NaN input is not hidden: it reaches the bins its bands
// touch, in its own frame only.
//
// Like the other bodies the phases are barrier-free; the CPU emulation (tests/emu, KB_HOST_EMU) runs each phase as a
// loop over the CTA's threads.
#pragma once
#include "kb_tables.h"
#include "stft_core.cuh"

#define KB_FBI_WARPS 32

struct KbFbiCol { int band; float w; };   // one nonzero of A^T's row (= the filterbank's row) for a bin

struct KbFbiParams {
    const float* x;                       // (batch, channel, frame, band) element strides
    long long x_sb, x_sc, x_st, x_sk;
    int B, C, T, F, M;                    // F = n_freq bins, M = n_bands
    const KbBand* bands;                  // A's rows: band m covers bins [lo, hi) with weights fbw[off + k - lo]
    const float* fbw;
    const int* cptr;                      // A's columns: bin k has entries cols[cptr[k] .. cptr[k + 1])
    const KbFbiCol* cols;
    const float* inv_d;                   // 1 / (A A^T 1)_m, 0 where that is 0
    float step;
    int n_iter;
    int from_db;                          // 1: x is in decibels, m = 10^(x / 10) db_scale
    double db_scale;                      // max(amin, ref_value)
    float* out;                           // (batch, channel, frame, bin) element strides
    long long o_sb, o_sc, o_st, o_sk;
    int n_tiles_t;                        // ceil(T / R)
    int n_warps;
    int R;                                // frames per tile: 32, 16, ..., 1
};

// Shared-memory layout (bytes) of a tile of R frames.
struct KbFbiSmem { int s, y, m, r, total; };
KB_HD KbFbiSmem kb_fbi_smem_layout(int F, int M, int R) {
    const int RS = R + 1;
    KbFbiSmem L;
    L.s = 0;
    L.y = L.s + kb_align16(F * RS * 4);
    L.m = L.y + kb_align16((F + 3) * RS * 4);
    L.r = L.m + kb_align16(M * RS * 4);
    L.total = L.r + kb_align16(M * RS * 4);
    return L;
}

// The largest R in {32, ..., 1} whose tile fits `smem_limit` bytes, or 0 when not even one frame's state fits.
static inline int kb_fbi_pick_r(int F, int M, int smem_limit) {
    for (int R = 32; R >= 1; R >>= 1)
        if (kb_fbi_smem_layout(F, M, R).total <= smem_limit) return R;
    return 0;
}

#if defined(KB_HOST_EMU)
static inline float kb_fbi_fma(float a, float b, float c) { return std::fmaf(a, b, c); }
static inline float kb_fbi_mul(float a, float b) { return a * b; }
static inline float kb_fbi_add(float a, float b) { return a + b; }
static inline float kb_fbi_sub(float a, float b) { return a - b; }
#else
KB_D float kb_fbi_fma(float a, float b, float c) { return __fmaf_rn(a, b, c); }
KB_D float kb_fbi_mul(float a, float b) { return __fmul_rn(a, b); }
KB_D float kb_fbi_add(float a, float b) { return __fadd_rn(a, b); }
KB_D float kb_fbi_sub(float a, float b) { return __fsub_rn(a, b); }
#endif
KB_HD float kb_fbi_relu(float v) { return v < 0.0f ? 0.0f : v; }   // keeps NaN

// (A^T v)_k for one frame column: v rows are RS floats apart.
KB_FN float kb_fbi_col_dot(const KbFbiParams& p, int k, const float* vcol, int RS) {
    float g = 0.0f;
    const int j1 = p.cptr[k + 1];
    for (int j = p.cptr[k]; j < j1; ++j) {
        const KbFbiCol e = p.cols[j];
        g = kb_fbi_fma(e.w, vcol[e.band * RS], g);
    }
    return g;
}

// (A y)_m for one frame column: four interleaved partial sums over the 4-padded band (as kb_band_dot).
KB_FN float kb_fbi_row_dot(const float* w, const float* ycol, int len4, int RS) {
    float a0 = 0.0f, a1 = 0.0f, a2 = 0.0f, a3 = 0.0f;
    for (int i = 0; i < len4; ++i) {
        const kb_f4 wv = reinterpret_cast<const kb_f4*>(w)[i];
        a0 = kb_fbi_fma(wv.x, ycol[0], a0);
        a1 = kb_fbi_fma(wv.y, ycol[RS], a1);
        a2 = kb_fbi_fma(wv.z, ycol[2 * RS], a2);
        a3 = kb_fbi_fma(wv.w, ycol[3 * RS], a3);
        ycol += 4 * RS;
    }
    return kb_fbi_add(kb_fbi_add(a0, a1), kb_fbi_add(a2, a3));
}

KB_FN float kb_fbi_from_db(float v, double scale) {
#if defined(KB_HOST_EMU)
    return (float)(std::pow(10.0, (double)v * 0.1) * scale);
#else
    return (float)(exp10((double)v * 0.1) * scale);
#endif
}

template <int FRT>
#if defined(KB_HOST_EMU)
inline void kb_fbi_cta_r(const KbFbiParams& p, char* smem, int cta, int n_cta)
#else
__device__ __forceinline__ void kb_fbi_cta_r(const KbFbiParams& p, char* smem, int cta, int n_cta)
#endif
{
    constexpr int RS = FRT + 1;
    const int NW = p.n_warps;
    const int kb_nt = NW * 32;
    (void)kb_nt;
    const KbFbiSmem L = kb_fbi_smem_layout(p.F, p.M, FRT);
    float* s_s = reinterpret_cast<float*>(smem + L.s);
    float* y_s = reinterpret_cast<float*>(smem + L.y);
    float* m_s = reinterpret_cast<float*>(smem + L.m);
    float* r_s = reinterpret_cast<float*>(smem + L.r);
    const int n_tiles = p.B * p.C * p.n_tiles_t;
    const int F = p.F, M = p.M;
#if defined(KB_HOST_EMU)
    std::vector<KbThreadRegs> kb_regs(kb_nt);
#else
    KbThreadRegs kb_regs;
#endif
    for (int tile = cta; tile < n_tiles; tile += n_cta) {
        const int sig = tile / p.n_tiles_t;
        const int tt = tile - sig * p.n_tiles_t;
        const int b = sig / p.C, c = sig - b * p.C;
        const int t0 = tt * FRT;
        const float* xs = p.x + (long long)b * p.x_sb + (long long)c * p.x_sc;
        // load m (frames past T read as 0 and stay 0) and the back-projection weights m / d into r
        KB_PHASE_BEGIN
            (void)R;
            for (int idx = tid; idx < 3 * RS; idx += kb_nt) y_s[F * RS + idx] = 0.0f;
            const int tot = FRT * M;
            for (int idx = tid; idx < tot; idx += kb_nt) {
                const int r = idx / M, m = idx - r * M;
                const int t = t0 + r;
                float v = 0.0f;
                if (t < p.T) {
                    v = xs[(long long)t * p.x_st + (long long)m * p.x_sk];
                    if (p.from_db) v = kb_fbi_from_db(v, p.db_scale);
                }
                m_s[m * RS + r] = v;
                const float id = p.inv_d[m];
                r_s[m * RS + r] = id != 0.0f ? kb_fbi_mul(v, id) : 0.0f;
            }
        KB_PHASE_END
        KB_SYNC_CTA;
        // s_0 = y_0 = max(A^T (m / d), 0)
        KB_PHASE_BEGIN
            (void)R;
            const int warp = tid >> 5, lane = tid & 31;
            if (lane < FRT)
                for (int k = warp; k < F; k += NW) {
                    const float v = kb_fbi_relu(kb_fbi_col_dot(p, k, r_s + lane, RS));
                    s_s[k * RS + lane] = v;
                    y_s[k * RS + lane] = v;
                }
        KB_PHASE_END
        KB_SYNC_CTA;
        double tk = 1.0;
        for (int it = 0; it < p.n_iter; ++it) {
            const double tn = 0.5 * (1.0 + sqrt(1.0 + 4.0 * tk * tk));
            const float coef = (float)((tk - 1.0) / tn);
            tk = tn;
            // r = A y - m
            KB_PHASE_BEGIN
                (void)R;
                const int warp = tid >> 5, lane = tid & 31;
                if (lane < FRT)
                    for (int m = warp; m < M; m += NW) {
                        const KbBand bd = p.bands[m];
                        const float ay = kb_fbi_row_dot(p.fbw + bd.off, y_s + bd.lo * RS + lane, (bd.hi - bd.lo) >> 2, RS);
                        r_s[m * RS + lane] = kb_fbi_sub(ay, m_s[m * RS + lane]);
                    }
            KB_PHASE_END
            KB_SYNC_CTA;
            // s' = max(y - step A^T r, 0);  y' = s' + coef (s' - s)
            KB_PHASE_BEGIN
                (void)R;
                const int warp = tid >> 5, lane = tid & 31;
                if (lane < FRT)
                    for (int k = warp; k < F; k += NW) {
                        const float g = kb_fbi_col_dot(p, k, r_s + lane, RS);
                        const int e = k * RS + lane;
                        const float sn = kb_fbi_relu(kb_fbi_fma(-p.step, g, y_s[e]));
                        const float so = s_s[e];
                        s_s[e] = sn;
                        y_s[e] = kb_fbi_fma(coef, kb_fbi_sub(sn, so), sn);
                    }
            KB_PHASE_END
            KB_SYNC_CTA;
        }
        KB_PHASE_BEGIN
            (void)R;
            const long long obase = (long long)b * p.o_sb + (long long)c * p.o_sc;
            const int tot = FRT * F;
            for (int idx = tid; idx < tot; idx += kb_nt) {
                const int r = idx / F, k = idx - r * F;
                const int t = t0 + r;
                if (t < p.T) p.out[obase + (long long)t * p.o_st + (long long)k * p.o_sk] = s_s[k * RS + r];
            }
        KB_PHASE_END
        KB_SYNC_CTA;
    }
}

#if defined(KB_HOST_EMU)
inline void kb_fbi_cta(const KbFbiParams& p, char* smem, int cta, int n_cta)
#else
__device__ __forceinline__ void kb_fbi_cta(const KbFbiParams& p, char* smem, int cta, int n_cta)
#endif
{
    switch (p.R) {
        case 32: kb_fbi_cta_r<32>(p, smem, cta, n_cta); break;
        case 16: kb_fbi_cta_r<16>(p, smem, cta, n_cta); break;
        case 8: kb_fbi_cta_r<8>(p, smem, cta, n_cta); break;
        case 4: kb_fbi_cta_r<4>(p, smem, cta, n_cta); break;
        case 2: kb_fbi_cta_r<2>(p, smem, cta, n_cta); break;
        default: kb_fbi_cta_r<1>(p, smem, cta, n_cta); break;
    }
}

// ---- plan tables (host) -----------------------------------------------------------------------------------------
// From a row-major (n_freq x n_bands) filterbank: A's row bands (kb_make_bands), A's column lists (the nonzeros of
// each filterbank row, in band order), 1 / d with d = A A^T 1, and step = 1 / ||A||_2^2.  d and ||A||_2 are computed in
// float64 from the float32 weights; ||A||_2^2 is the largest eigenvalue of A A^T by power iteration from the all-ones
// vector (A A^T is non-negative, so that start is not orthogonal to the top eigenvector), run until the Rayleigh
// quotient settles to 1e-15 relative (a few thousand iterations at most for kapre's mel and log banks; the result
// is then within 1e-9 of the largest eigenvalue, from below).
struct KbFbiTables {
    std::vector<KbBand> bands;
    std::vector<float> w;
    std::vector<int> cptr;
    std::vector<KbFbiCol> cols;
    std::vector<float> inv_d;
    double norm2;   // ||A||_2^2
    float step;
};

static inline void kb_fbi_make_tables(const float* fb, int n_freq, int n_bands, KbFbiTables& t) {
    kb_make_bands(fb, n_freq, n_bands, t.bands, t.w);
    t.cptr.assign((size_t)n_freq + 1, 0);
    t.cols.clear();
    for (int k = 0; k < n_freq; ++k) {
        for (int m = 0; m < n_bands; ++m) {
            const float w = fb[(size_t)k * n_bands + m];
            if (w != 0.0f) t.cols.push_back(KbFbiCol{m, w});
        }
        t.cptr[k + 1] = (int)t.cols.size();
    }
    if (t.cols.empty()) t.cols.push_back(KbFbiCol{0, 0.0f});   // a valid device allocation; never read
    // A A^T v = sum over bins k of (row k of the filterbank) (row k . v)
    auto aat = [&](const std::vector<double>& v, std::vector<double>& out) {
        out.assign(n_bands, 0.0);
        for (int k = 0; k < n_freq; ++k) {
            double dot = 0.0;
            for (int j = t.cptr[k]; j < t.cptr[k + 1]; ++j) dot += (double)t.cols[j].w * v[t.cols[j].band];
            for (int j = t.cptr[k]; j < t.cptr[k + 1]; ++j) out[t.cols[j].band] += (double)t.cols[j].w * dot;
        }
    };
    std::vector<double> v(n_bands, 1.0), u;
    aat(v, u);
    t.inv_d.resize(n_bands);
    for (int m = 0; m < n_bands; ++m) t.inv_d[m] = u[m] > 0.0 ? (float)(1.0 / u[m]) : 0.0f;
    double lam = 0.0;
    for (int it = 0; it < 20000; ++it) {
        double nv = 0.0, vu = 0.0;
        for (int m = 0; m < n_bands; ++m) { nv += v[m] * v[m]; vu += v[m] * u[m]; }
        const double q = nv > 0.0 ? vu / nv : 0.0;     // Rayleigh quotient of v
        const bool done = it > 0 && std::fabs(q - lam) <= 1e-15 * q;
        lam = q;
        if (done || q == 0.0) break;
        double nu = 0.0;
        for (int m = 0; m < n_bands; ++m) nu += u[m] * u[m];
        nu = std::sqrt(nu);
        for (int m = 0; m < n_bands; ++m) v[m] = u[m] / nu;
        aat(v, u);
    }
    t.norm2 = lam;
    t.step = lam > 0.0 ? (float)(1.0 / lam) : 0.0f;
}
