// Kernel bodies of the second-order-section cascade (kapre_sosfilt, scipy.signal.sosfilt).  Filter rows
// [b0, b1, b2, a0, a1, a2] with a0 = 1 (not read), sections s = 0 .. S-1 in row order, each in direct form II
// transposed with state (z1, z2):
//
//   y_s = b0 x_s + z1,   z1' = b1 x_s - a1 y_s + z2,   z2' = b2 x_s - a2 y_s,   x_0 = x[t],  x_(s+1) = y_s,  y[t] = y_(S-1)
//
// The cascade is a linear recurrence in the 2S-dimensional state (z1_0, z2_0, z1_1, ...) with a state matrix Phi that
// is block lower-triangular (section s feeds section s + 1), so it runs on the chunked scan of iir_core.cuh with Phi in
// place of the companion matrix:
//
//   1. powers  (kb_sos_powers_cta)  Phi^Tc and Phi^(2^j Tc), j = 1..5, in float64 per distinct filter;
//   2. state   (kb_sos_state_cta)   each chunk's end state from a zero start, and each block's aggregate (a scan);
//   3. carry   (kb_sos_carry_col)   C_b = Phi^(32 Tc) C_(b-1) + A_b, serially over the blocks of a column, from
//                                   C_(-1) = zi (the caller's initial state, float64);
//   4. output  (kb_sos_out_cta)     the block's scan again with C_(b-1) folded into its first chunk, then each chunk
//                                   rerun from its start state rounded to float32; the lane that ends the column
//                                   writes its end state, zf.
//
// Chunks, blocks, staging, the loaders, the reverse flag and the coalesced store are iir_core.cuh's (KbIirParams holds
// the geometry), so y[t] depends on x[0..t], the coefficients and zi alone, as there.  Everything is instantiated per
// section count S <= KB_SOS_MAX, so a lane's state and coefficients are registers and the scan is 2S wide.
#pragma once
#include "iir_core.cuh"

#define KB_SOS_MAX 8                                // sections (order 16)
#define KB_SOS_ROW 6                                // floats per section row

struct KbSosParams {
    KbIirParams g;      // x, y and their strides, B, C, L, K, nblk, n_cols, reverse, and the workspace pw / e / blk.
                        // g.ac, g.a_sb, g.a_sc: the sos rows (S x 6 floats per filter, unit stride inside a filter);
                        // g.pw is (n_f, KB_IIR_NPOW, 2S, 2S), g.e (n_cols, K, 2S), g.blk (n_cols, nblk, 2S)
    int S;
    const float* zi; long long zi_sb, zi_sc, zi_ss; // (z1, z2) of section s at zi + b zi_sb + c zi_sc + s zi_ss, or null
    float* zf; long long zf_sb, zf_sc, zf_ss;       // the same for the final state, or null
};

// Shared memory of one block body (one warp): mbarrier, staged input, staged output, scan ping-pong (2S wide).
struct KbSosSmem {
    int bar, xs, ys, sc, total;
};
KB_HD KbSosSmem kb_sos_smem(int S) {
    KbSosSmem s;
    int off = 0;
    s.bar = off; off += 16;
    s.xs = off; off += kb_align16((KB_IIR_STAGE + 8) * 4);     // + 4 either side: the 16 B-rounded bulk copy
    s.ys = off; off += kb_align16(KB_IIR_SPAN * 4);
    s.sc = off; off += 2 * KB_IIR_W * 2 * S * 8;
    s.total = off;
    return s;
}

// b0, b1, b2 and the negated a1, a2 of every section, in registers.
template <int S>
struct KbSosCoef {
    float b0[S], b1[S], b2[S], na1[S], na2[S];
};

template <int S>
KB_HD void kb_sos_coef(const KbSosParams& p, long long col, KbSosCoef<S>& q) {
    const long long bi = col / p.g.C, ci = col - bi * p.g.C;
    const float* r = p.g.ac + bi * p.g.a_sb + ci * p.g.a_sc;
#pragma unroll
    for (int s = 0; s < S; ++s) {
        q.b0[s] = r[s * KB_SOS_ROW + 0];
        q.b1[s] = r[s * KB_SOS_ROW + 1];
        q.b2[s] = r[s * KB_SOS_ROW + 2];
        q.na1[s] = -r[s * KB_SOS_ROW + 4];
        q.na2[s] = -r[s * KB_SOS_ROW + 5];
    }
}

// Run chunk `lane` of the tile through every section from state w (z1, z2 per section), outputs to `ys` when non-null,
// the end state back into w.  Five fmaf per section and sample: y = b0 x + z1, z1' = -a1 y + (b1 x + z2),
// z2' = -a2 y + b2 x.
template <int S>
KB_HD int kb_sos_run(const KbSosCoef<S>& q, const KbIirView& xv, int lane, int n_tile, float* w, float* ys) {
    const int c0 = lane * KB_IIR_TC;                // chunk start, relative to the tile
    const int n = n_tile - c0 < KB_IIR_TC ? n_tile - c0 : KB_IIR_TC;
    if (n <= 0) return 0;
    const float* xp = xv.ptr + (KB_IIR_HALO + c0) * xv.step;
    for (int t = 0; t < n; ++t) {
        float v = xp[t * xv.step];
#pragma unroll
        for (int s = 0; s < S; ++s) {
            const float y = fmaf(q.b0[s], v, w[2 * s]);
            w[2 * s] = fmaf(q.na1[s], y, fmaf(q.b1[s], v, w[2 * s + 1]));
            w[2 * s + 1] = fmaf(q.na2[s], y, q.b2[s] * v);
            v = y;
        }
        if (ys) ys[c0 + t] = v;
    }
    return n;
}

// out += P s for one D x D float64 matrix, rows in a fixed order.
template <int D>
KB_HD void kb_sos_matvec(const double* P, const double* s, double* out) {
#pragma unroll
    for (int r = 0; r < D; ++r) {
        double acc = out[r];
#pragma unroll
        for (int k = 0; k < D; ++k) acc = fma(P[r * D + k], s[k], acc);
        out[r] = acc;
    }
}

// ------------------------------------------------------------------------------------------ 1. powers
// One warp per distinct filter f: Phi (column k is one zero-input step of the cascade from the unit state e_k, in
// float64), Phi^Tc = Phi^64 Phi by squaring, then its five squares, into g.pw[f].  `m`: 3 (2S)^2 doubles of shared
// memory.
template <int S>
KB_IIR_FN void kb_sos_powers_cta(const KbSosParams& p, double* m, long long f) {
    constexpr int D = 2 * S, DD = D * D;
    double* phi = m;
    double* cur = m + DD;
    double* nxt = m + 2 * DD;
    double* out = p.g.pw + f * (KB_IIR_NPOW * DD);
    KB_IIR_LANES_BEGIN
        if (lane < D) {
            const long long fb = f / p.g.n_fc, fc = f - fb * p.g.n_fc;
            const float* r = p.g.ac + fb * p.g.a_sb + fc * p.g.a_sc;
            double z[D];
#pragma unroll
            for (int k = 0; k < D; ++k) z[k] = k == lane ? 1.0 : 0.0;
            double x = 0.0;
#pragma unroll
            for (int s = 0; s < S; ++s) {
                const double y = (double)r[s * KB_SOS_ROW] * x + z[2 * s];
                const double z1 = (double)r[s * KB_SOS_ROW + 1] * x - (double)r[s * KB_SOS_ROW + 4] * y + z[2 * s + 1];
                z[2 * s + 1] = (double)r[s * KB_SOS_ROW + 2] * x - (double)r[s * KB_SOS_ROW + 5] * y;
                z[2 * s] = z1;
                x = y;
            }
#pragma unroll
            for (int k = 0; k < D; ++k) {
                phi[k * D + lane] = z[k];
                cur[k * D + lane] = z[k];
            }
        }
    KB_IIR_LANES_END
    KB_SYNC_WARP;
    // 6 squarings (Phi^64), one product with Phi (Phi^65 = Phi^Tc), 5 squarings: 12 products, the j-th power
    // written after products 7 .. 12
    for (int s = 0; s < 12; ++s) {
        const double* rhs = s == 6 ? phi : cur;
        KB_IIR_LANES_BEGIN
            for (int e = lane; e < DD; e += 32) {
                const int r = e / D, c = e - r * D;
                double acc = 0.0;
                for (int k = 0; k < D; ++k) acc = fma(cur[r * D + k], rhs[k * D + c], acc);
                nxt[e] = acc;
                if (s >= 6) out[(s - 6) * DD + e] = acc;
            }
        KB_IIR_LANES_END
        KB_SYNC_WARP;
        KB_IIR_LANES_BEGIN
            for (int e = lane; e < DD; e += 32) cur[e] = nxt[e];
        KB_IIR_LANES_END
        KB_SYNC_WARP;
    }
}

// Kogge-Stone scan of the block's 32 states in sc[0 .. 32 D) (ping-pong with sc[32 D .. 64 D)); the result in sc[0 ..).
template <int S>
KB_IIR_FN void kb_sos_scan(const double* pw, double* sc) {
    constexpr int D = 2 * S;
    double* a = sc;
    double* b = sc + KB_IIR_W * D;
    for (int j = 0; j < 5; ++j) {
        const int d = 1 << j;
        KB_IIR_LANES_BEGIN
            double v[D];
#pragma unroll
            for (int r = 0; r < D; ++r) v[r] = a[lane * D + r];
            if (lane >= d) kb_sos_matvec<D>(pw + j * D * D, a + (lane - d) * D, v);
#pragma unroll
            for (int r = 0; r < D; ++r) b[lane * D + r] = v[r];
        KB_IIR_LANES_END
        KB_SYNC_WARP;
        double* t = a; a = b; b = t;
    }
    // five rounds: the result is in b's original buffer; copy it back
    KB_IIR_LANES_BEGIN
#pragma unroll
        for (int r = 0; r < D; ++r) b[lane * D + r] = a[lane * D + r];
    KB_IIR_LANES_END
    KB_SYNC_WARP;
}

KB_HD const float* kb_sos_zi(const KbSosParams& p, long long col) {
    const long long bi = col / p.g.C, ci = col - bi * p.g.C;
    return p.zi + bi * p.zi_sb + ci * p.zi_sc;
}

// ------------------------------------------------------------------------------------------ 2. state
template <int S>
KB_IIR_FN void kb_sos_state_cta(const KbSosParams& p, char* smem, long long tile) {
    constexpr int D = 2 * S;
    const KbSosSmem M = kb_sos_smem(S);
    KbBar* bar = reinterpret_cast<KbBar*>(smem + M.bar);
    float* xs = reinterpret_cast<float*>(smem + M.xs);
    double* sc = reinterpret_cast<double*>(smem + M.sc);
    const KbIirTile t = kb_iir_tile(p.g, tile);
    kb_iir_stage(p.g, t, xs, bar);
    KB_IIR_LANES_BEGIN
        if (t.bulk) kb_bar_wait(bar, 0);
        KbSosCoef<S> q;
        kb_sos_coef<S>(p, t.col, q);
        float w[D];
#pragma unroll
        for (int k = 0; k < D; ++k) w[k] = 0.0f;
        const int ran = kb_sos_run<S>(q, kb_iir_view(p.g, xs + t.head), lane, t.n, w, nullptr);
        const int c = t.blk * KB_IIR_W + lane;
        if (ran) {
            float* e = p.g.e + ((size_t)t.col * p.g.K + c) * D;
#pragma unroll
            for (int k = 0; k < D; ++k) e[k] = w[k];
        }
#pragma unroll
        for (int k = 0; k < D; ++k) sc[lane * D + k] = ran ? (double)w[k] : 0.0;
    KB_IIR_LANES_END
    KB_SYNC_WARP;
    kb_sos_scan<S>(p.g.pw + kb_iir_filter(p.g, t.col) * (KB_IIR_NPOW * D * D), sc);
    KB_IIR_LANES_BEGIN
        if (lane < D) p.g.blk[((size_t)t.col * p.g.nblk + t.blk) * D + lane] = sc[(KB_IIR_W - 1) * D + lane];
    KB_IIR_LANES_END
}

// ------------------------------------------------------------------------------------------ 3. carry
// One thread per column: C_b = Phi^(32 Tc) C_(b-1) + A_b for the blocks whose carry a later block reads, from
// C_(-1) = zi (zero without zi, when C_0 = A_0 is left as the state pass wrote it).
template <int S>
KB_HD void kb_sos_carry_col(const KbSosParams& p, long long col) {
    constexpr int D = 2 * S;
    const double* P = p.g.pw + kb_iir_filter(p.g, col) * (KB_IIR_NPOW * D * D) + 5 * D * D;
    double* blk = p.g.blk + (size_t)col * p.g.nblk * D;
    const float* zi = p.zi ? kb_sos_zi(p, col) : nullptr;
    double c[D], nxt[D];
#pragma unroll
    for (int r = 0; r < D; ++r) c[r] = zi ? (double)zi[(r >> 1) * p.zi_ss + (r & 1)] : 0.0;
    for (int b = 0; b + 1 < p.g.nblk; ++b) {
#pragma unroll
        for (int r = 0; r < D; ++r) nxt[r] = blk[b * D + r];
        if (b > 0 || zi) kb_sos_matvec<D>(P, c, nxt);
#pragma unroll
        for (int r = 0; r < D; ++r) { c[r] = nxt[r]; blk[b * D + r] = nxt[r]; }
    }
}

// ------------------------------------------------------------------------------------------ 4. output
template <int S>
KB_IIR_FN void kb_sos_out_cta(const KbSosParams& p, char* smem, long long tile) {
    constexpr int D = 2 * S;
    const KbSosSmem M = kb_sos_smem(S);
    KbBar* bar = reinterpret_cast<KbBar*>(smem + M.bar);
    float* xs = reinterpret_cast<float*>(smem + M.xs);
    float* ys = reinterpret_cast<float*>(smem + M.ys);
    double* sc = reinterpret_cast<double*>(smem + M.sc);
    const KbIirTile t = kb_iir_tile(p.g, tile);
    const double* pw = p.g.pw + kb_iir_filter(p.g, t.col) * (KB_IIR_NPOW * D * D);
    const double* carry = t.blk > 0 ? p.g.blk + ((size_t)t.col * p.g.nblk + t.blk - 1) * D : nullptr;
    const float* zi = t.blk == 0 && p.zi ? kb_sos_zi(p, t.col) : nullptr;
    kb_iir_stage(p.g, t, xs, bar);
    // the chunk end states, the block's start state (C_(b-1), or zi) folded into the first one
    KB_IIR_LANES_BEGIN
        const int c = t.blk * KB_IIR_W + lane;
        double v[D];
#pragma unroll
        for (int k = 0; k < D; ++k) v[k] = c < p.g.K ? (double)p.g.e[((size_t)t.col * p.g.K + c) * D + k] : 0.0;
        if (lane == 0 && (carry || zi)) {
            double s0[D];
#pragma unroll
            for (int k = 0; k < D; ++k) s0[k] = carry ? carry[k] : (double)zi[(k >> 1) * p.zi_ss + (k & 1)];
            kb_sos_matvec<D>(pw, s0, v);
        }
#pragma unroll
        for (int k = 0; k < D; ++k) sc[lane * D + k] = v[k];
    KB_IIR_LANES_END
    KB_SYNC_WARP;
    kb_sos_scan<S>(pw, sc);
    // rerun each chunk from its start state
    KB_IIR_LANES_BEGIN
        if (t.bulk) kb_bar_wait(bar, 0);
        KbSosCoef<S> q;
        kb_sos_coef<S>(p, t.col, q);
        float w[D];
#pragma unroll
        for (int k = 0; k < D; ++k)
            w[k] = lane > 0 ? (float)sc[(lane - 1) * D + k]
                            : carry ? (float)carry[k] : (zi ? zi[(k >> 1) * p.zi_ss + (k & 1)] : 0.0f);
        const int ran = kb_sos_run<S>(q, kb_iir_view(p.g, xs + t.head), lane, t.n, w, ys);
        if (ran && p.zf && t.blk * KB_IIR_W + lane == p.g.K - 1) {
            const long long bi = t.col / p.g.C, ci = t.col - bi * p.g.C;
            float* zf = p.zf + bi * p.zf_sb + ci * p.zf_sc;
#pragma unroll
            for (int k = 0; k < D; ++k) zf[(k >> 1) * p.zf_ss + (k & 1)] = w[k];
        }
    KB_IIR_LANES_END
    KB_SYNC_WARP;
    // coalesced store of the staged outputs
    KB_IIR_LANES_BEGIN
        const long long bi = t.col / p.g.C, ci = t.col - bi * p.g.C;
        float* yo = p.g.y + bi * p.g.y_sb + ci * p.g.y_sc;
        for (int e = lane; e < t.n; e += 32) yo[kb_iir_phys(p.g, (long long)t.t0 + e) * p.g.y_sl] = ys[e];
    KB_IIR_LANES_END
}
