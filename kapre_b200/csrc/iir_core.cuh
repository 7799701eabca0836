// Kernel bodies of the IIR filter (kapre_lfilter, torchaudio.functional.lfilter) and its gradient.  With
// coefficients normalised by a0 (b, a below are b / a0, a / a0, zero-padded to order KB_IIR_N):
//
//   u[t] = sum_{k=0..N} b_k x[t-k],   y[t] = u[t] - sum_{k=1..N} a_k y[t-k],   x, y = 0 before t = 0.
//
// The recursion is linear in its state s_t = (y[t], y[t-1], ..., y[t-N+1]) with the companion matrix Phi
// (Phi[0][k] = -a_{k+1}, Phi[i][i-1] = 1), so time is cut into chunks of Tc samples per (item, channel) column:
//
//   1. powers  (kb_iir_powers_cta)  Phi^Tc and Phi^(2^j Tc), j = 1..5, in float64 per distinct filter;
//   2. state   (kb_iir_state_cta)   each chunk's end state e_c from a zero start (FIR part from the true input),
//                                   and each block of 32 chunks' aggregate A_b (a scan of the e_c from zero);
//   3. carry   (kb_iir_carry_col)   C_b = Phi^(32 Tc) C_(b-1) + A_b, serially over the blocks of a column;
//   4. output  (kb_iir_out_cta)     the block's scan again with C_(b-1) folded into its first chunk, which gives
//                                   every chunk's start state, then the chunk is rerun from it (rounded to float32).
//
// The scans are Kogge-Stone over the 32 chunks of an aligned block: in round j chunk l adds Phi^(2^j Tc) times
// the partial sum of chunk l - 2^j.  The carries are float64.  Tc, the blocks and the tree are fixed by the
// absolute chunk index, so y[t] depends on x[0..t] and the coefficients alone: not on the length, the batch, the
// grid, the strides, broadcasting or the data format.
//
// Every body runs in its own logical time tau with the physical sample tau (forward) or L-1-tau (`reverse`).
// The gradient is the same machinery run in the other direction on gy with the all-pole part only:
//   v[t] = gy[t] - sum_k a_k v[t+k],  gx[t] = sum_k b_k v[t+k],  gb_k = sum_t v[t] x[t-k],  ga_k = -sum_t v[t] y[t-k]
// (`bwd`).  gx is formed from v and the recursion's own state, so it needs no halo; the coefficient sums are
// written per (chunk, column) when `part` is set, and reduced by the caller.
//
// Work split: one warp per block of 32 chunks of one column, lane l owning chunk l.  The block's input span
// (32 Tc samples plus 8 on either side) is staged in shared memory by a TMA bulk copy when it lies inside the signal
// and is contiguous (stride 1 along time), else by a cooperative loader (any strides, zeros outside the signal), so
// that global loads coalesce.  Tc = 65 is 1 mod 32: lane l reads sample l Tc + t, so the 32 lanes hit 32 banks.
// The output is staged the same way and stored cooperatively.
//
// Like the other bodies these are barrier-free phases: under nvcc each phase runs once per lane and the phases are
// separated by __syncwarp(); the CPU emulation (tests/emu, KB_HOST_EMU) runs each phase as a loop over the lanes.
#pragma once
#include "stft_core.cuh"

#define KB_IIR_N 8                                  // largest order; lower orders run with zero coefficients
#define KB_IIR_NC (KB_IIR_N + 1)
#define KB_IIR_TC 65                                // samples per chunk (1 mod 32: conflict-free staging)
#define KB_IIR_W 32                                 // chunks per block (one warp)
#define KB_IIR_SPAN (KB_IIR_W * KB_IIR_TC)          // samples per block
#define KB_IIR_HALO 8
#define KB_IIR_STAGE (KB_IIR_SPAN + 2 * KB_IIR_HALO)   // staged samples per block
#define KB_IIR_NPOW 6                               // Phi^(2^j Tc), j = 0..5
#define KB_IIR_FLAG_CLAMP 1
#define KB_IIR_FLAG_REVERSE 2

struct KbIirParams {
    const float* x;  long long x_sb, x_sc, x_sl;    // input: x (forward) or gy (backward)
    long long x_numel;                              // elements addressable from x (max element offset + 1)
    unsigned x_align;                               // ((uintptr_t)x >> 2) & 3
    float* y;        long long y_sb, y_sc, y_sl;    // output: y or gx
    const float* xr; long long xr_sb, xr_sc, xr_sl; // backward with `part`: the forward's input
    const float* yr; long long yr_sb, yr_sc, yr_sl; // and its unclamped output
    const float* bc; long long b_sb, b_sc;          // normalised b (order + 1 per filter, unit stride)
    const float* ac; long long a_sb, a_sc;          // normalised a (a[0] is not read)
    int order;
    int B, C, L;
    int K, nblk;                                    // chunks and blocks per column
    long long n_cols;                               // B C
    int n_fb, n_fc;                                 // distinct denominators along batch and channels
    int reverse, clamp, bwd;
    double* pw;                                     // (n_fb n_fc, KB_IIR_NPOW, N, N)
    float* e;                                       // (n_cols, K, N) chunk end states from a zero start
    double* blk;                                    // (n_cols, nblk, N) block aggregates, then block carries
    float* part;                                    // (2 order + 1, n_cols, K) coefficient partial sums, or null:
                                                    // rows 0..order gb_k, rows order + k ga_k (k >= 1)
};

// Shared memory of one block body (one warp): mbarrier, staged input, staged output, scan ping-pong, and in the
// backward with coefficient sums the staged forward input and output.
struct KbIirSmem {
    int bar, xs, ys, sc, xr, yr, total;
};
KB_HD KbIirSmem kb_iir_smem(int with_refs) {
    KbIirSmem s;
    int off = 0;
    s.bar = off; off += 16;
    s.xs = off; off += kb_align16((KB_IIR_STAGE + 8) * 4);     // + 4 either side: the 16 B-rounded bulk copy
    s.ys = off; off += kb_align16(KB_IIR_SPAN * 4);
    s.sc = off; off += 2 * KB_IIR_W * KB_IIR_N * 8;
    s.xr = off; if (with_refs) off += kb_align16(KB_IIR_STAGE * 4);
    s.yr = off; if (with_refs) off += kb_align16(KB_IIR_STAGE * 4);
    s.total = off;
    return s;
}

// ---- host side: geometry (shared by the library and the CPU emulation) ----
// Chunks, blocks and the distinct-filter counts once B, C, L and the coefficient strides are set.
inline void kb_iir_setup(KbIirParams& p) {
    p.K = (int)(((long long)p.L + KB_IIR_TC - 1) / KB_IIR_TC);
    p.nblk = (p.K + KB_IIR_W - 1) / KB_IIR_W;
    p.n_cols = (long long)p.B * p.C;
    p.n_fb = p.a_sb ? p.B : 1;
    p.n_fc = p.a_sc ? p.C : 1;
}

KB_HD long long kb_iir_filter(const KbIirParams& p, long long col) {
    const long long b = col / p.C, c = col - b * p.C;
    return (p.n_fb > 1 ? b : 0) * p.n_fc + (p.n_fc > 1 ? c : 0);
}

// ---- the per-lane arithmetic ----
struct KbIirCoef {
    float b[KB_IIR_NC], a[KB_IIR_NC];               // zero past the order; a[0] unused
};

KB_HD void kb_iir_coef(const KbIirParams& p, long long col, KbIirCoef& q) {
    const long long bi = col / p.C, ci = col - bi * p.C;
    const float* bp = p.bc + bi * p.b_sb + ci * p.b_sc;
    const float* ap = p.ac + bi * p.a_sb + ci * p.a_sc;
#pragma unroll
    for (int k = 0; k < KB_IIR_NC; ++k) {
        q.b[k] = k <= p.order ? bp[k] : 0.0f;
        q.a[k] = k >= 1 && k <= p.order ? ap[k] : 0.0f;
    }
}

// y = u - a_N w[N-1] - ... - a_2 w[1] - a_1 w[0]: the term on the previous output last, so that the dependency
// chain through the recursion is one FMA per sample.
KB_HD float kb_iir_pole(const KbIirCoef& q, float u, const float* w) {
    float acc = u;
#pragma unroll
    for (int k = KB_IIR_N; k >= 1; --k) acc = fmaf(-q.a[k], w[k - 1], acc);
    return acc;
}

// sum_k b_k (cur, w[0], ..., w[N-1]) in the order b_N .. b_0.
KB_HD float kb_iir_zero(const KbIirCoef& q, float cur, const float* w) {
    float acc = q.b[KB_IIR_N] * w[KB_IIR_N - 1];
#pragma unroll
    for (int k = KB_IIR_N - 1; k >= 1; --k) acc = fmaf(q.b[k], w[k - 1], acc);
    return fmaf(q.b[0], cur, acc);
}

KB_HD void kb_iir_push(float* w, float v) {
#pragma unroll
    for (int k = KB_IIR_N - 1; k >= 1; --k) w[k] = w[k - 1];
    w[0] = v;
}

KB_HD float kb_iir_clamp(float v) { return v < -1.0f ? -1.0f : (v > 1.0f ? 1.0f : v); }   // NaN passes, as torch.clamp

// Staged span of a block: logical samples [t0 - HALO, t0 + SPAN + HALO).  Sample u sits at slot(u) = base + (u - s0)
// forward, base + (STAGE - 1 - (u - s0)) in reverse (the buffer holds the span in physical order).
struct KbIirTile {
    long long col;
    int blk, t0, n;                                 // first logical sample, samples in the block
    int bulk, head, bytes;                          // bulk copy: slot 0 at buf[head]
    const float* src;
};

KB_HD KbIirTile kb_iir_tile(const KbIirParams& p, long long tile) {
    KbIirTile t;
    t.col = tile / p.nblk;
    t.blk = (int)(tile - t.col * p.nblk);
    t.t0 = t.blk * KB_IIR_SPAN;
    t.n = p.L - t.t0 < KB_IIR_SPAN ? p.L - t.t0 : KB_IIR_SPAN;
    t.bulk = 0; t.head = 0; t.bytes = 0; t.src = nullptr;
    const long long s0 = (long long)t.t0 - KB_IIR_HALO, s1 = s0 + KB_IIR_STAGE;
    if (p.x_sl == 1 && s0 >= 0 && s1 <= p.L) {
        const long long bi = t.col / p.C, ci = t.col - bi * p.C;
        const long long p0 = p.reverse ? (long long)p.L - s1 : s0;          // first physical sample
        const long long off0 = bi * p.x_sb + ci * p.x_sc + p0;
        const int head = (int)((p.x_align + (unsigned)off0) & 3u);
        const int tail = (int)((0u - (p.x_align + (unsigned)off0 + (unsigned)KB_IIR_STAGE)) & 3u);
        if (off0 - head >= 0 && off0 + KB_IIR_STAGE + tail <= p.x_numel) {
            t.bulk = 1; t.head = head; t.src = p.x + (off0 - head); t.bytes = (head + KB_IIR_STAGE + tail) * 4;
        }
    }
    return t;
}

KB_HD long long kb_iir_phys(const KbIirParams& p, long long u) { return p.reverse ? (long long)p.L - 1 - u : u; }

// The cooperative loader: element e of the staged span of column `col` from a (batch, channel, sample)-strided
// signal, zero outside [0, L), laid out as kb_iir_tile describes.
KB_HD float kb_iir_load(const KbIirParams& p, const float* base, long long sb, long long sc, long long sl, long long col,
                        int t0, int e) {
    const long long bi = col / p.C, ci = col - bi * p.C;
    const long long u = (long long)t0 - KB_IIR_HALO + (p.reverse ? KB_IIR_STAGE - 1 - e : e);
    if (u < 0 || u >= p.L) return 0.0f;
    return base[bi * sb + ci * sc + kb_iir_phys(p, u) * sl];
}

// A lane's view of a staged span: v(u) for logical u = t0 - HALO + i is at ptr[i * step].
struct KbIirView {
    const float* ptr;
    int step;
};
KB_HD KbIirView kb_iir_view(const KbIirParams& p, const float* buf) {
    KbIirView v;
    v.ptr = p.reverse ? buf + (KB_IIR_STAGE - 1) : buf;
    v.step = p.reverse ? -1 : 1;
    return v;
}

// s' = P s (+ acc) for one 8 x 8 float64 matrix, rows in a fixed order.
KB_HD void kb_iir_matvec(const double* P, const double* s, double* out) {
#pragma unroll
    for (int r = 0; r < KB_IIR_N; ++r) {
        double acc = out[r];
#pragma unroll
        for (int k = 0; k < KB_IIR_N; ++k) acc = fma(P[r * KB_IIR_N + k], s[k], acc);
        out[r] = acc;
    }
}

#if defined(KB_HOST_EMU)
#define KB_IIR_LANES_BEGIN for (int lane = 0; lane < 32; ++lane) {
#define KB_IIR_LANES_END }
#define KB_IIR_FN inline
#else
#define KB_IIR_LANES_BEGIN { const int lane = (int)(threadIdx.x & 31);
#define KB_IIR_LANES_END }
#define KB_IIR_FN __device__ __forceinline__
#endif

// ------------------------------------------------------------------------------------------ 1. powers
// One warp per distinct denominator f: Phi^Tc = Phi^64 Phi by squaring, then its five squares, into p.pw[f].
// `m`: 3 x 64 doubles of shared memory.  Lane l computes elements l and l + 32 of each product.
KB_IIR_FN void kb_iir_powers_cta(const KbIirParams& p, double* m, long long f) {
    double* phi = m;
    double* cur = m + 64;
    double* nxt = m + 128;
    double* out = p.pw + f * (KB_IIR_NPOW * 64);
    KB_IIR_LANES_BEGIN
        const long long fb = f / p.n_fc, fc = f - fb * p.n_fc;
        const float* ap = p.ac + fb * p.a_sb + fc * p.a_sc;
        for (int e = lane; e < 64; e += 32) {
            const int r = e >> 3, k = e & 7;
            double v = 0.0;
            if (r == 0) v = k + 1 <= p.order ? -(double)ap[k + 1] : 0.0;
            else v = k == r - 1 ? 1.0 : 0.0;
            phi[e] = v;
            cur[e] = v;
        }
    KB_IIR_LANES_END
    KB_SYNC_WARP;
    // 6 squarings (Phi^64), one product with Phi (Phi^65 = Phi^Tc), 5 squarings: 12 products, the j-th power
    // written after products 7 .. 12
    for (int s = 0; s < 12; ++s) {
        const double* rhs = s == 6 ? phi : cur;
        KB_IIR_LANES_BEGIN
            for (int e = lane; e < 64; e += 32) {
                const int r = e >> 3, c = e & 7;
                double acc = 0.0;
                for (int k = 0; k < KB_IIR_N; ++k) acc = fma(cur[r * 8 + k], rhs[k * 8 + c], acc);
                nxt[e] = acc;
                if (s >= 6) out[(s - 6) * 64 + e] = acc;
            }
        KB_IIR_LANES_END
        KB_SYNC_WARP;
        KB_IIR_LANES_BEGIN
            for (int e = lane; e < 64; e += 32) cur[e] = nxt[e];
        KB_IIR_LANES_END
        KB_SYNC_WARP;
    }
}

// Kogge-Stone scan of the block's 32 states in sc[0 .. 256) (ping-pong with sc[256 .. 512)); the result in sc[0 ..).
KB_IIR_FN void kb_iir_scan(const double* pw, double* sc) {
    double* a = sc;
    double* b = sc + KB_IIR_W * KB_IIR_N;
    for (int j = 0; j < 5; ++j) {
        const int d = 1 << j;
        KB_IIR_LANES_BEGIN
            double v[KB_IIR_N];
#pragma unroll
            for (int r = 0; r < KB_IIR_N; ++r) v[r] = a[lane * KB_IIR_N + r];
            if (lane >= d) kb_iir_matvec(pw + j * 64, a + (lane - d) * KB_IIR_N, v);
#pragma unroll
            for (int r = 0; r < KB_IIR_N; ++r) b[lane * KB_IIR_N + r] = v[r];
        KB_IIR_LANES_END
        KB_SYNC_WARP;
        double* t = a; a = b; b = t;
    }
    // five rounds: the result is in b's original buffer; copy it back
    KB_IIR_LANES_BEGIN
#pragma unroll
        for (int r = 0; r < KB_IIR_N; ++r) b[lane * KB_IIR_N + r] = a[lane * KB_IIR_N + r];
    KB_IIR_LANES_END
    KB_SYNC_WARP;
}

// Stage the block's span of the input (bulk copy or cooperative loader).
KB_IIR_FN void kb_iir_stage(const KbIirParams& p, const KbIirTile& t, float* xs, KbBar* bar) {
    KB_IIR_LANES_BEGIN
        if (t.bulk) {
            if (lane == 0) { kb_bar_init(bar, 1); kb_bulk_g2s(xs, t.src, t.bytes, bar); }
        } else {
#pragma unroll 4
            for (int e = lane; e < KB_IIR_STAGE; e += 32) xs[e] = kb_iir_load(p, p.x, p.x_sb, p.x_sc, p.x_sl, t.col, t.t0, e);
        }
    KB_IIR_LANES_END
    KB_SYNC_WARP;
}

// Run chunk `lane` of the tile from start state w (y[c0-1], ..., y[c0-N]).  Forward: FIR from the staged input,
// outputs to `ys` (when non-null), end state back into w.  Backward: the all-pole recursion on the staged gy, the
// outputs gx = sum_k b_k v[t+k] from the recursion's state, and (with `refs`, from the staged forward input and
// output xrv, yrv) the coefficient sums into g: g[k] = sum v x[t-k], g[N + k] = sum v y[t-k].
KB_HD int kb_iir_run(const KbIirParams& p, const KbIirCoef& q, const KbIirView& xv, int lane, int n_tile, float* w,
                     float* ys, int refs, const KbIirView& xrv, const KbIirView& yrv, float* g) {
    const int c0 = lane * KB_IIR_TC;                // chunk start, relative to the tile
    const int n = n_tile - c0 < KB_IIR_TC ? n_tile - c0 : KB_IIR_TC;
    if (n <= 0) return 0;
    const float* xp = xv.ptr + (KB_IIR_HALO + c0) * xv.step;
    float xw[KB_IIR_N];
#pragma unroll
    for (int k = 0; k < KB_IIR_N; ++k) xw[k] = p.bwd ? 0.0f : xp[-(k + 1) * xv.step];
    for (int t = 0; t < n; ++t) {
        const float cur = xp[t * xv.step];
        if (!p.bwd) {
            const float y = kb_iir_pole(q, kb_iir_zero(q, cur, xw), w);
            kb_iir_push(xw, cur);
            kb_iir_push(w, y);
            if (ys) ys[c0 + t] = y;
        } else {
            const float v = kb_iir_pole(q, cur, w);
            const float gx = kb_iir_zero(q, v, w);
            if (refs) {
                // x[t-k], y[t-k] of the forward are logical samples c0 + t + k of this (reversed) scan
                const float* xr = xrv.ptr + (KB_IIR_HALO + c0 + t) * xrv.step;
                const float* yr = yrv.ptr + (KB_IIR_HALO + c0 + t) * yrv.step;
#pragma unroll
                for (int k = 0; k <= KB_IIR_N; ++k) {
                    if (k <= p.order) g[k] = fmaf(v, xr[k * xrv.step], g[k]);
                    if (k >= 1 && k <= p.order) g[KB_IIR_N + k] = fmaf(v, yr[k * yrv.step], g[KB_IIR_N + k]);
                }
            }
            kb_iir_push(w, v);
            if (ys) ys[c0 + t] = gx;
        }
    }
    return n;
}

// ------------------------------------------------------------------------------------------ 2. state
KB_IIR_FN void kb_iir_state_cta(const KbIirParams& p, char* smem, long long tile) {
    const KbIirSmem S = kb_iir_smem(0);
    KbBar* bar = reinterpret_cast<KbBar*>(smem + S.bar);
    float* xs = reinterpret_cast<float*>(smem + S.xs);
    double* sc = reinterpret_cast<double*>(smem + S.sc);
    const KbIirTile t = kb_iir_tile(p, tile);
    kb_iir_stage(p, t, xs, bar);
    KB_IIR_LANES_BEGIN
        if (t.bulk) kb_bar_wait(bar, 0);
        KbIirCoef q;
        kb_iir_coef(p, t.col, q);
        float w[KB_IIR_N];
#pragma unroll
        for (int k = 0; k < KB_IIR_N; ++k) w[k] = 0.0f;
        float g[1];
        const KbIirView none = kb_iir_view(p, xs);
        const int ran = kb_iir_run(p, q, kb_iir_view(p, xs + t.head), lane, t.n, w, nullptr, 0, none, none, g);
        const int c = t.blk * KB_IIR_W + lane;
        if (ran) {
            float* e = p.e + ((size_t)t.col * p.K + c) * KB_IIR_N;
#pragma unroll
            for (int k = 0; k < KB_IIR_N; ++k) e[k] = w[k];
        }
#pragma unroll
        for (int k = 0; k < KB_IIR_N; ++k) sc[lane * KB_IIR_N + k] = ran ? (double)w[k] : 0.0;
    KB_IIR_LANES_END
    KB_SYNC_WARP;
    kb_iir_scan(p.pw + kb_iir_filter(p, t.col) * (KB_IIR_NPOW * 64), sc);
    KB_IIR_LANES_BEGIN
        if (lane < KB_IIR_N) p.blk[((size_t)t.col * p.nblk + t.blk) * KB_IIR_N + lane] = sc[(KB_IIR_W - 1) * KB_IIR_N + lane];
    KB_IIR_LANES_END
}

// ------------------------------------------------------------------------------------------ 3. carry
// One thread per column: C_b = Phi^(32 Tc) C_(b-1) + A_b for the blocks whose carry a later block reads.
KB_HD void kb_iir_carry_col(const KbIirParams& p, long long col) {
    const double* P = p.pw + kb_iir_filter(p, col) * (KB_IIR_NPOW * 64) + 5 * 64;
    double* blk = p.blk + (size_t)col * p.nblk * KB_IIR_N;
    double c[KB_IIR_N], nxt[KB_IIR_N];
#pragma unroll
    for (int r = 0; r < KB_IIR_N; ++r) c[r] = blk[r];
    for (int b = 1; b + 1 < p.nblk; ++b) {
#pragma unroll
        for (int r = 0; r < KB_IIR_N; ++r) nxt[r] = blk[b * KB_IIR_N + r];
        kb_iir_matvec(P, c, nxt);
#pragma unroll
        for (int r = 0; r < KB_IIR_N; ++r) { c[r] = nxt[r]; blk[b * KB_IIR_N + r] = nxt[r]; }
    }
}

// ------------------------------------------------------------------------------------------ 4. output
KB_IIR_FN void kb_iir_out_cta(const KbIirParams& p, char* smem, long long tile) {
    const int refs = p.bwd && p.part != nullptr;
    const KbIirSmem S = kb_iir_smem(refs);
    KbBar* bar = reinterpret_cast<KbBar*>(smem + S.bar);
    float* xs = reinterpret_cast<float*>(smem + S.xs);
    float* ys = reinterpret_cast<float*>(smem + S.ys);
    double* sc = reinterpret_cast<double*>(smem + S.sc);
    float* xrs = reinterpret_cast<float*>(smem + S.xr);
    float* yrs = reinterpret_cast<float*>(smem + S.yr);
    const KbIirTile t = kb_iir_tile(p, tile);
    const double* pw = p.pw + kb_iir_filter(p, t.col) * (KB_IIR_NPOW * 64);
    const double* carry = t.blk > 0 ? p.blk + ((size_t)t.col * p.nblk + t.blk - 1) * KB_IIR_N : nullptr;
    kb_iir_stage(p, t, xs, bar);
    // the chunk end states, C_(b-1) folded into the first one
    KB_IIR_LANES_BEGIN
        const int c = t.blk * KB_IIR_W + lane;
        double v[KB_IIR_N];
#pragma unroll
        for (int k = 0; k < KB_IIR_N; ++k) v[k] = c < p.K ? (double)p.e[((size_t)t.col * p.K + c) * KB_IIR_N + k] : 0.0;
        if (lane == 0 && carry) kb_iir_matvec(pw, carry, v);
#pragma unroll
        for (int k = 0; k < KB_IIR_N; ++k) sc[lane * KB_IIR_N + k] = v[k];
        if (refs) {
#pragma unroll 4
            for (int e = lane; e < KB_IIR_STAGE; e += 32) {
                xrs[e] = kb_iir_load(p, p.xr, p.xr_sb, p.xr_sc, p.xr_sl, t.col, t.t0, e);
                yrs[e] = kb_iir_load(p, p.yr, p.yr_sb, p.yr_sc, p.yr_sl, t.col, t.t0, e);
            }
        }
    KB_IIR_LANES_END
    KB_SYNC_WARP;
    kb_iir_scan(pw, sc);
    // rerun each chunk from its start state
    KB_IIR_LANES_BEGIN
        if (t.bulk) kb_bar_wait(bar, 0);
        KbIirCoef q;
        kb_iir_coef(p, t.col, q);
        float w[KB_IIR_N];
#pragma unroll
        for (int k = 0; k < KB_IIR_N; ++k)
            w[k] = lane > 0 ? (float)sc[(lane - 1) * KB_IIR_N + k] : (carry ? (float)carry[k] : 0.0f);
        float g[2 * KB_IIR_N + 1];
#pragma unroll
        for (int k = 0; k < 2 * KB_IIR_N + 1; ++k) g[k] = 0.0f;
        const int ran = kb_iir_run(p, q, kb_iir_view(p, xs + t.head), lane, t.n, w, ys, refs, kb_iir_view(p, xrs),
                                   kb_iir_view(p, yrs), g);
        if (refs && ran) {
            const long long c = (long long)t.blk * KB_IIR_W + lane, stride = p.n_cols * p.K;
            float* o = p.part + t.col * p.K + c;
#pragma unroll
            for (int k = 0; k <= KB_IIR_N; ++k) {
                if (k <= p.order) o[k * stride] = g[k];
                if (k >= 1 && k <= p.order) o[(p.order + k) * stride] = -g[KB_IIR_N + k];
            }
        }
    KB_IIR_LANES_END
    KB_SYNC_WARP;
    // coalesced store of the staged outputs
    KB_IIR_LANES_BEGIN
        const long long bi = t.col / p.C, ci = t.col - bi * p.C;
        float* yo = p.y + bi * p.y_sb + ci * p.y_sc;
        for (int e = lane; e < t.n; e += 32) {
            const float v = ys[e];
            yo[kb_iir_phys(p, (long long)t.t0 + e) * p.y_sl] = p.clamp ? kb_iir_clamp(v) : v;
        }
    KB_IIR_LANES_END
}
