// Kernel bodies of gated loudness (kapre_loudness, torchaudio.functional.loudness, ITU-R BS.1770-4) and its gradient.
// They run on the K-weighted signal y (the two kapre_lfilter calls come first).  For an item of C <= 5 channels and
// valid length len, with gate G and step S samples:
//
//   blocks [jS, jS + G) for j < J = (len - G) / S + 1 (J = 0 when len < G),   e_cj = mean over block j of y_c^2,
//   E_j = sum_c g_c e_cj,  l_j = -0.691 + 10 log10(E_j),  g = (1, 1, 1, 1.41, 1.41),
//   J1 = {j : l_j > -70},  Gamma = -0.691 + 10 log10(mean_{J1} E_j) - 10,  J2 = {j in J1 : l_j > Gamma},
//   LKFS = -0.691 + 10 log10(E2),  E2 = mean_{J2} E_j   (-inf when J2 is empty, NaN when a block is not finite).
//
// Geometry: with m = G / S and rho = G mod S, every step interval [kS, (k+1)S) holds at most one interior block
// boundary, at kS + rho, so it is two pieces, [kS, kS + rho) and [kS + rho, (k+1)S) (the first empty when rho = 0).
// Block j is both pieces of intervals j .. j + m - 1 and the first piece of interval j + m.
//
// Three passes, each a warp per tile and barrier-free (phases separated by __syncwarp(); the CPU emulation under
// KB_HOST_EMU runs each phase as a loop over the lanes):
//   1. energy   (kb_loud_energy_tile, one tile per (item, interval)): the float64 sums of y^2 of both pieces of the
//               interval per channel, into `part`.  A piece is staged in rounds of KB_NOISE_R samples through shared
//               memory by noise_core.cuh's cursors, so loads coalesce in both data formats; lane l adds samples
//               a + l, a + l + 32, ... of a piece [a, e) in order and a fixed tree (strides 16 .. 1) adds the lanes.
//               The order depends on the column and the absolute sample index alone.  Intervals that no block of the
//               item touches are skipped.
//   2. gate     (kb_loud_gate_tile, one tile per item): the block energies from the pieces in ascending order, both
//               gates in float64 with fixed-order reductions, LKFS rounded once to float32, and the stats the
//               gradient reads: (E2, |J2|) and one J2 decision per block.
//   3. backward (kb_loud_bwd_tile, one tile per (item, interval) over the whole length):
//                 gy[t] = gL (20 / ln 10) g_c y[t] n(t) / (E2 |J2| G),  n(t) = the number of J2 blocks covering t,
//               constant on a piece; exactly 0 where n(t) = 0 and for items with an empty J2.
#pragma once
#include "noise_core.cuh"

#define KB_LOUD_MAXC 5                              // channels of an item (BS.1770's weights)
#define KB_LOUD_WARPS 4                             // tiles (warps) per CTA
#define KB_LOUD_BIAS -0.691
#define KB_LOUD_ABS_GATE -70.0
#define KB_LOUD_DB_LN10 4.3429448190325182          // 10 / ln(10)

KB_HD double kb_loud_weight(int c) { return c < 3 ? 1.0 : 1.41; }

struct KbLoudParams {
    const float* y; long long y_sb, y_sc, y_sl;     // K-weighted signal, element strides (batch, channel, sample)
    const int* len;                                 // per item valid length (null: L), clamped to [0, L] here
    float* out;                                     // forward: LKFS per item
    double* part;                                   // (B, K, 2, C) piece sums
    double* stats;                                  // (B, 2): E2, |J2|
    unsigned char* mask;                            // (B, Jmax) J2 decisions
    const float* gl;                                // backward: output gradient per item
    float* gy; long long g_sb, g_sc, g_sl;          // backward: gradient of y
    int B, C, L, G, S, rho, m;
    int K;                                          // intervals an L-sample item's blocks touch
    int Jmax;                                       // blocks of an L-sample item
    int Kb;                                         // backward intervals: ceil(L / S)
    long long tiles;
};

// Blocks of an item of len samples, and the intervals they touch.
KB_HD int kb_loud_blocks(const KbLoudParams& p, int len) { return len >= p.G ? (len - p.G) / p.S + 1 : 0; }
KB_HD int kb_loud_intervals(const KbLoudParams& p, int J) { return J ? J - 1 + p.m + (p.rho > 0) : 0; }

// ---- host side: geometry (shared by the library and the CPU emulation) ----
inline void kb_loud_setup(KbLoudParams& p) {
    p.rho = p.G % p.S;
    p.m = p.G / p.S;
    p.Jmax = kb_loud_blocks(p, p.L);
    p.K = kb_loud_intervals(p, p.Jmax);
    p.Kb = (int)(((long long)p.L + p.S - 1) / p.S);
}

KB_HD int kb_loud_len(const KbLoudParams& p, long long b) {
    if (!p.len) return p.L;
    const int l = p.len[b];
    return l < 0 ? 0 : (l > p.L ? p.L : l);
}

// Shared memory of one tile: the staged block (C rows of KB_NOISE_R samples), the lane sums for the tree and the
// per-row limits the cursors read.
struct KbLoudSmem {
    int xs, red, cnt, lim, total;
};
KB_HD KbLoudSmem kb_loud_smem() {
    KbLoudSmem s;
    int off = 0;
    s.xs = off; off += KB_LOUD_MAXC * KB_NOISE_R * 4;
    s.red = off; off += KB_LOUD_MAXC * 32 * 8;
    s.cnt = off; off += 32 * 4;
    s.lim = off; off += KB_NOISE_G * 4;
    s.total = kb_align16(off);
    return s;
}

struct KbLoudPtrs {
    float* xs;
    double* red;
    int *cnt, *lim;
};
KB_HD KbLoudPtrs kb_loud_ptrs(char* smem) {
    const KbLoudSmem S = kb_loud_smem();
    KbLoudPtrs P;
    P.xs = reinterpret_cast<float*>(smem + S.xs);
    P.red = reinterpret_cast<double*>(smem + S.red);
    P.cnt = reinterpret_cast<int*>(smem + S.cnt);
    P.lim = reinterpret_cast<int*>(smem + S.lim);
    return P;
}

// Piece pc of interval k clipped to [0, end): [*a, *e), empty when *a >= *e.
KB_HD void kb_loud_piece(const KbLoudParams& p, int k, int pc, int end, int* a, int* e) {
    const long long s = (long long)k * p.S + (pc ? p.rho : 0);
    long long f = pc ? (long long)(k + 1) * p.S : s + p.rho;
    if (f > end) f = end;
    *a = (int)(s < end ? s : end);
    *e = (int)(f > *a ? f : *a);
}

// Sets every row's limit to e for the cursors (kb_noise_fetch masks samples at or past it).
KB_NOISE_FN void kb_loud_set_lim(const KbLoudPtrs& P, int e) {
    KB_NOISE_LANES_BEGIN
        if (lane < KB_NOISE_G) P.lim[lane] = e;
    KB_NOISE_LANES_END
    KB_SYNC_WARP;
}

// Stages the (C x R) block of y at [t0, t0 + R) (0 at or past the limits) into P.xs.
KB_NOISE_FN void kb_loud_stage(const KbLoudParams& p, const KbLoudPtrs& P, long long b, int t0) {
    KB_NOISE_LANES_BEGIN
        KbNoiseCur ky = kb_noise_cur(p.y, p.y_sb, p.y_sc, p.y_sl, b, 0, p.C, lane);
        for (int bt = 0; bt < p.C; ++bt) {
            float v[KB_NOISE_PL];
            const KbNoiseCur k0 = ky;
            kb_noise_fetch(ky, t0, P.lim, bt, lane, v);
            kb_noise_put(k0, bt, lane, v, P.xs);
        }
    KB_NOISE_LANES_END
    KB_SYNC_WARP;
}

// ------------------------------------------------------------------------------------------ 1. piece sums
KB_NOISE_FN void kb_loud_energy_tile(const KbLoudParams& p, char* smem, long long tile) {
    const long long b = tile / p.K;
    const int k = (int)(tile - b * p.K);
    const int J = kb_loud_blocks(p, kb_loud_len(p, b));
    if (k >= kb_loud_intervals(p, J)) return;
    const int end = (J - 1) * p.S + p.G;
    const KbLoudPtrs P = kb_loud_ptrs(smem);
    for (int pc = 0; pc < 2; ++pc) {
        int a, e;
        kb_loud_piece(p, k, pc, end, &a, &e);
        kb_loud_set_lim(P, e);
        KB_NOISE_LANE_ARR(double, acc, KB_LOUD_MAXC);
        KB_NOISE_LANES_BEGIN
#pragma unroll
            for (int c = 0; c < KB_LOUD_MAXC; ++c) KB_NOISE_LV(acc)[c] = 0.0;
        KB_NOISE_LANES_END
        for (int t0 = a; t0 < e; t0 += KB_NOISE_R) {
            kb_loud_stage(p, P, b, t0);
            KB_NOISE_LANES_BEGIN
#pragma unroll
                for (int c = 0; c < KB_LOUD_MAXC; ++c) {
                    if (c < p.C) {
                        double s = KB_NOISE_LV(acc)[c];
#pragma unroll
                        for (int i = 0; i < KB_NOISE_PL; ++i) {
                            const double v = (double)P.xs[c * KB_NOISE_R + lane + 32 * i];
                            s += v * v;                 // samples at or past e were staged as 0: s + 0 == s
                        }
                        KB_NOISE_LV(acc)[c] = s;
                    }
                }
            KB_NOISE_LANES_END
            KB_SYNC_WARP;
        }
        KB_NOISE_LANES_BEGIN
#pragma unroll
            for (int c = 0; c < KB_LOUD_MAXC; ++c)
                if (c < p.C) P.red[c * 32 + lane] = KB_NOISE_LV(acc)[c];
        KB_NOISE_LANES_END
        KB_SYNC_WARP;
        for (int d = 16; d >= 1; d >>= 1) {
            KB_NOISE_LANES_BEGIN
                if (lane < d)
                    for (int c = 0; c < p.C; ++c) P.red[c * 32 + lane] += P.red[c * 32 + lane + d];
            KB_NOISE_LANES_END
            KB_SYNC_WARP;
        }
        KB_NOISE_LANES_BEGIN
            if (lane < p.C) p.part[((b * p.K + k) * 2 + pc) * p.C + lane] = P.red[lane * 32];
        KB_NOISE_LANES_END
        KB_SYNC_WARP;
    }
}

// ------------------------------------------------------------------------------------------ 2. gates
// E_j from the pieces in ascending order: per channel p0[j] + p1[j] + ... + p1[j + m - 1] (+ p0[j + m]), over G, then
// weighted in channel order.
KB_HD double kb_loud_block(const KbLoudParams& p, long long b, int j) {
    const double* q = p.part + b * p.K * 2 * p.C;
    double E = 0.0;
    for (int c = 0; c < p.C; ++c) {
        double s = 0.0;
        for (int k = j; k < j + p.m; ++k) {
            s += q[(2 * k) * p.C + c];
            s += q[(2 * k + 1) * p.C + c];
        }
        if (p.rho > 0) s += q[(2 * (j + p.m)) * p.C + c];
        E += kb_loud_weight(c) * (s / p.G);
    }
    return E;
}

// The fixed tree over the lanes' values in P.red[0 .. 64) (two sums) and P.cnt[0 .. 32): the totals land in P.red[0],
// P.red[32] and P.cnt[0].
KB_NOISE_FN void kb_loud_tree(const KbLoudPtrs& P) {
    for (int d = 16; d >= 1; d >>= 1) {
        KB_NOISE_LANES_BEGIN
            if (lane < d) {
                P.red[lane] += P.red[lane + d];
                P.red[32 + lane] += P.red[32 + lane + d];
                P.cnt[lane] += P.cnt[lane + d];
            }
        KB_NOISE_LANES_END
        KB_SYNC_WARP;
    }
}

KB_NOISE_FN void kb_loud_gate_tile(const KbLoudParams& p, char* smem, long long b) {
    const KbLoudPtrs P = kb_loud_ptrs(smem);
    const int J = kb_loud_blocks(p, kb_loud_len(p, b));
    // pass 1: the absolute gate (sum and count of J1), and the count of non-finite block energies
    KB_NOISE_LANES_BEGIN
        double s = 0.0, nf = 0.0;
        int n = 0;
        for (int j = lane; j < J; j += 32) {
            const double E = kb_loud_block(p, b, j);
            if (!(E - E == 0.0)) nf += 1.0;
            if (KB_LOUD_BIAS + 10.0 * log10(E) > KB_LOUD_ABS_GATE) { s += E; ++n; }
        }
        P.red[lane] = s; P.red[32 + lane] = nf; P.cnt[lane] = n;
    KB_NOISE_LANES_END
    KB_SYNC_WARP;
    kb_loud_tree(P);
    const double s1 = P.red[0];
    const int n1 = P.cnt[0];
    const bool nan = P.red[32] != 0.0;
    KB_SYNC_WARP;
    // pass 2: the relative gate, its decisions, and the sum and count of J2
    const double rel = KB_LOUD_BIAS + 10.0 * log10(s1 / (double)n1) - 10.0;
    KB_NOISE_LANES_BEGIN
        double s = 0.0;
        int n = 0;
        for (int j = lane; j < J; j += 32) {
            const double E = kb_loud_block(p, b, j);
            const double l = KB_LOUD_BIAS + 10.0 * log10(E);
            const bool in = n1 > 0 && l > KB_LOUD_ABS_GATE && l > rel;
            if (in) { s += E; ++n; }
            p.mask[b * p.Jmax + j] = in ? 1 : 0;
        }
        P.red[lane] = s; P.red[32 + lane] = 0.0; P.cnt[lane] = n;
    KB_NOISE_LANES_END
    KB_SYNC_WARP;
    kb_loud_tree(P);
    KB_NOISE_LANES_BEGIN
        if (lane == 0) {
            const int n = P.cnt[0];
            const double E2 = nan ? (double)NAN : (n ? P.red[0] / (double)n : 0.0);
            p.out[b] = nan ? NAN : (n ? (float)(KB_LOUD_BIAS + 10.0 * log10(E2)) : -INFINITY);
            p.stats[2 * b] = E2;
            p.stats[2 * b + 1] = (double)n;
        }
    KB_NOISE_LANES_END
}

// ------------------------------------------------------------------------------------------ 3. gradient
// J2 blocks covering piece pc of interval k: blocks max(0, k - m + pc) .. min(k, J - 1).
KB_HD int kb_loud_cover(const KbLoudParams& p, long long b, int J, int k, int pc) {
    int lo = k - p.m + pc, hi = k < J - 1 ? k : J - 1, n = 0;
    if (lo < 0) lo = 0;
    for (int j = lo; j <= hi; ++j) n += p.mask[b * p.Jmax + j];
    return n;
}

KB_NOISE_FN void kb_loud_bwd_tile(const KbLoudParams& p, char* smem, long long tile) {
    const long long b = tile / p.Kb;
    const int k = (int)(tile - b * p.Kb);
    const int J = kb_loud_blocks(p, kb_loud_len(p, b));
    const KbLoudPtrs P = kb_loud_ptrs(smem);
    const double n2 = p.stats[2 * b + 1];
    // gL (20 / ln 10) / (E2 |J2| G); the channel weight and n(t) come per piece
    const double scale = n2 > 0.0 ? (double)p.gl[b] * 2.0 * KB_LOUD_DB_LN10 / (p.stats[2 * b] * n2 * p.G) : 0.0;
    for (int pc = 0; pc < 2; ++pc) {
        int a, e;
        kb_loud_piece(p, k, pc, p.L, &a, &e);
        const int n = n2 > 0.0 ? kb_loud_cover(p, b, J, k, pc) : 0;
        kb_loud_set_lim(P, e);
        for (int t0 = a; t0 < e; t0 += KB_NOISE_R) {
            if (n) kb_loud_stage(p, P, b, t0);              // nothing is read where the gradient is 0
            KB_NOISE_LANES_BEGIN
#pragma unroll
                for (int c = 0; c < KB_LOUD_MAXC; ++c) {
                    if (c >= p.C) break;
                    const double f = scale * kb_loud_weight(c) * n;
#pragma unroll
                    for (int i = 0; i < KB_NOISE_PL; ++i) {
                        float* v = P.xs + c * KB_NOISE_R + lane + 32 * i;
                        *v = n ? (float)(f * (double)*v) : 0.0f;
                    }
                }
            KB_NOISE_LANES_END
            KB_SYNC_WARP;
            KB_NOISE_LANES_BEGIN
                KbNoiseCur kg = kb_noise_cur(p.gy, p.g_sb, p.g_sc, p.g_sl, b, 0, p.C, lane);
                for (int bt = 0; bt < p.C; ++bt) kb_noise_emit(kg, t0, e, bt, lane, P.xs);
            KB_NOISE_LANES_END
            KB_SYNC_WARP;
        }
    }
}
