// Kernel bodies of the loudness meter: true peak (kapre_true_peak) and its gradient, and the loudness series and
// loudness range (kapre_loudness_stats).  They sit beside gated loudness (loudness_core.cuh), whose energy and gate
// passes kapre_loudness_stats launches unchanged, and whose piece sums the series pass reads.
//
// True peak (BS.1770-4 Annex 2 with scipy's resample_poly filter instead of the annex's 48-tap example), per (item,
// channel) column x of valid length len:
//
//   z[4n + r] = sum_{m=0}^{20} w_r[m] x[n - 10 + m],   w_r[m] = 4 h[80 + r - 4m]  (0 outside h),   0 <= t < 4 len,
//   TP = 20 log10 max_t |z[t]|,   x = 0 outside [0, len),
//
// with h the 81 taps of signal.resample_filter(4, 1).  Each output is formed exactly as resample_core.cuh forms it
// (four fmaf chains over m mod 4, then (a0 + a1) + (a2 + a3)), so z is bit for bit what kapre_resample(4, 1) writes.
// Two barrier-free passes, a warp per tile (the CPU emulation under KB_HOST_EMU runs each phase as a loop over lanes):
//   1. peak (kb_tp_peak_tile, one tile per (item, channel, KB_TP_SEG input samples)): the segment's span staged in
//      shared memory, the 4 KB_TP_SEG outputs formed in registers and never written; each lane keeps the largest key
//      (|z| bits << 32) | ~t, a fixed tree takes the warp's largest and the tile writes it.  Key order is |z| order with
//      ties to the lowest t, and a NaN's bits exceed every finite |z|'s, so NaN propagates.
//   2. fold (kb_tp_fold_tile, one tile per column): the largest of the column's keys, TP rounded once to float32, and
//      the stats the gradient reads: (z[t*], t*), z[t*] recomputed with the same arithmetic for its sign.
// Gradient (kb_tp_bwd, one thread per input sample): dTP / dx[n] = (20 / ln 10) w[t* - 4n + 40] / z[t*] (w = 4 h),
// 0 outside h's support, at n >= len, and for silent columns (z[t*] = 0).
//
// Loudness series and range, on the window energies E_j = sum_c g_c e_cj of loudness_core.cuh's blocks:
//   series (kb_meter_series, one thread per (item, window)): s_j = -0.691 + 10 log10 E_j for j < J(len), else -inf;
//          with `e` set, E_j is also kept for the range pass.
//   range  (kb_meter_lra_tile, one tile per item, EBU Tech 3342 on the 3 s windows): J1 = {s_j > -70}, Gamma =
//          -0.691 + 10 log10(mean_J1 E_j) - 20, J2 = {j in J1 : s_j > Gamma}, n = |J2|; with v the ascending s_j of J2,
//          LRA = v[((n-1) 95 + 50) / 100] - v[((n-1) 10 + 50) / 100] (0 when n = 0, NaN when an E_j is not finite).
//          s is monotone in E, so the two order statistics are selected on E's float64 bits (positive, so ordered as
//          integers) by a radix select of 16 four-bit digits: no sort and no length limit.
#pragma once
#include "loudness_core.cuh"

#define KB_TP_TAPS 81                               // signal.resample_filter(4, 1): 2 * 10 * 4 + 1
#define KB_TP_M 21                                  // taps per phase (m = 0 .. 20)
#define KB_TP_SEG 2048                              // input samples per peak tile
#define KB_TP_SPAN (KB_TP_SEG + KB_TP_M - 1)        // staged samples of a tile: [n0 - 10, n0 + SEG + 10)
#define KB_TP_WARPS 4                               // tiles (warps) per CTA
#define KB_TP_MAX_LEN (1 << 30)                     // 4 len output indices fit the key's 32 bits
#define KB_TP_DB20 8.6858896380650366               // 20 / ln(10)

struct KbTpParams {
    const float* x; long long x_sb, x_sc, x_sl;     // waveform, element strides (batch, channel, sample)
    const int* len;                                 // per item valid length (null: L), clamped to [0, L] here
    float* out;                                     // (B, C) dBTP
    unsigned long long* key;                        // (B, C, nseg) tile maxima
    float* zs; unsigned* ts;                        // stats: (B, C) z[t*] and t*
    const float* g;                                 // backward: (B, C) output gradient
    float* gx; long long g_sb, g_sc, g_sl;          // backward: gradient of x
    int B, C, L, nseg;
    long long tiles;
    float w[4][KB_TP_M];                            // w[r][m] = 4 h[80 + r - 4m]
    float w4[KB_TP_TAPS];                           // 4 h
};

// ---- host side: taps and geometry (shared by the library and the CPU emulation) ----
inline void kb_tp_setup(KbTpParams& p, const float* taps) {
    for (int r = 0; r < 4; ++r)
        for (int m = 0; m < KB_TP_M; ++m) {
            const int i = 80 + r - 4 * m;
            p.w[r][m] = i >= 0 && i < KB_TP_TAPS ? 4.0f * taps[i] : 0.0f;
        }
    for (int i = 0; i < KB_TP_TAPS; ++i) p.w4[i] = 4.0f * taps[i];
    p.nseg = (int)(((long long)p.L + KB_TP_SEG - 1) / KB_TP_SEG);
}

KB_HD int kb_tp_len(const KbTpParams& p, long long b) {
    if (!p.len) return p.L;
    const int l = p.len[b];
    return l < 0 ? 0 : (l > p.L ? p.L : l);
}

// Output 4n + r from the 21 samples s[0 .. 20] = x[n - 10 .. n + 10], in resample_core.cuh's order.
KB_HD float kb_tp_z(const KbTpParams& p, const float* s, int r) {
    float a[4] = {0.0f, 0.0f, 0.0f, 0.0f};
#pragma unroll
    for (int m = 0; m < KB_TP_M; ++m)
        if (r == 0 || m > 0) a[m & 3] = fmaf(p.w[r][m], s[m], a[m & 3]);
    return (a[0] + a[1]) + (a[2] + a[3]);
}

KB_D unsigned long long kb_tp_key(float z, unsigned t) {
    return ((unsigned long long)kb_f2u(fabsf(z)) << 32) | (unsigned long long)(0xffffffffu - t);
}

// Shared memory of one peak or fold tile: the staged span, and the lanes' keys for the tree.
struct KbTpSmem {
    int xs, key, total;
};
KB_HD KbTpSmem kb_tp_smem() {
    KbTpSmem s;
    int off = 0;
    s.key = off; off += 32 * 8;
    s.xs = off; off += (KB_TP_SPAN + 3) * 4;
    s.total = kb_align16(off);
    return s;
}

// The largest of the 32 lane keys in K[0 .. 32), by a fixed tree; lands in K[0].
KB_NOISE_FN void kb_tp_tree(unsigned long long* K) {
    for (int d = 16; d >= 1; d >>= 1) {
        KB_NOISE_LANES_BEGIN
            if (lane < d && K[lane + d] > K[lane]) K[lane] = K[lane + d];
        KB_NOISE_LANES_END
        KB_SYNC_WARP;
    }
}

// ------------------------------------------------------------------------------------------ 1. peak per tile
KB_NOISE_FN void kb_tp_peak_tile(const KbTpParams& p, char* smem, long long tile) {
    const KbTpSmem S = kb_tp_smem();
    unsigned long long* K = reinterpret_cast<unsigned long long*>(smem + S.key);
    float* xs = reinterpret_cast<float*>(smem + S.xs);
    const long long col = tile / p.nseg;
    const int seg = (int)(tile - col * p.nseg);
    const long long b = col / p.C;
    const int c = (int)(col - b * p.C);
    const int len = kb_tp_len(p, b);
    const int n0 = seg * KB_TP_SEG;
    const int n1 = n0 + KB_TP_SEG < len ? n0 + KB_TP_SEG : len;
    const float* xc = p.x + b * p.x_sb + (long long)c * p.x_sc;
    // phase 1: stage x[n0 - 10, n1 + 10), zeros outside [0, len)
    KB_NOISE_LANES_BEGIN
        if (n0 < n1)
            for (int e = lane; e < n1 - n0 + KB_TP_M - 1; e += 32) {
                const long long t = (long long)n0 - 10 + e;
                xs[e] = t >= 0 && t < len ? xc[t * p.x_sl] : 0.0f;
            }
    KB_NOISE_LANES_END
    KB_SYNC_WARP;
    // phase 2: each lane's largest key over its samples n0 + lane + 32 i
    KB_NOISE_LANES_BEGIN
        unsigned long long best = 0;
        for (int n = n0 + lane; n < n1; n += 32) {
            const float* s = xs + (n - n0);
#pragma unroll
            for (int r = 0; r < 4; ++r) {
                const unsigned long long k = kb_tp_key(kb_tp_z(p, s, r), 4u * (unsigned)n + (unsigned)r);
                best = k > best ? k : best;
            }
        }
        K[lane] = best;
    KB_NOISE_LANES_END
    KB_SYNC_WARP;
    kb_tp_tree(K);
    KB_NOISE_LANES_BEGIN
        if (lane == 0) p.key[tile] = K[0];
    KB_NOISE_LANES_END
    KB_SYNC_WARP;
}

// ------------------------------------------------------------------------------------------ 2. fold per column
KB_NOISE_FN void kb_tp_fold_tile(const KbTpParams& p, char* smem, long long col) {
    const KbTpSmem S = kb_tp_smem();
    unsigned long long* K = reinterpret_cast<unsigned long long*>(smem + S.key);
    const long long b = col / p.C;
    const int c = (int)(col - b * p.C);
    const int len = kb_tp_len(p, b);
    const int ns = (int)(((long long)len + KB_TP_SEG - 1) / KB_TP_SEG);
    KB_NOISE_LANES_BEGIN
        unsigned long long best = 0;
        for (int s = lane; s < ns; s += 32) {
            const unsigned long long k = p.key[col * p.nseg + s];
            best = k > best ? k : best;
        }
        K[lane] = best;
    KB_NOISE_LANES_END
    KB_SYNC_WARP;
    kb_tp_tree(K);
    KB_NOISE_LANES_BEGIN
        if (lane == 0) {
            const unsigned long long k = K[0];
            const unsigned t = 0xffffffffu - (unsigned)(k & 0xffffffffu);
            float z = 0.0f;
            if (k >> 32) {                                  // recompute z[t*] for its sign
                const float* xc = p.x + b * p.x_sb + (long long)c * p.x_sc;
                const long long n = t >> 2;
                float s[KB_TP_M];
#pragma unroll
                for (int m = 0; m < KB_TP_M; ++m) {
                    const long long i = n - 10 + m;
                    s[m] = i >= 0 && i < len ? xc[i * p.x_sl] : 0.0f;
                }
                z = kb_tp_z(p, s, (int)(t & 3u));
            }
            p.zs[col] = z;
            p.ts[col] = t;
            p.out[col] = (float)(20.0 * log10((double)fabsf(z)));
        }
    KB_NOISE_LANES_END
}

// ------------------------------------------------------------------------------------------ 3. gradient
KB_HD void kb_tp_bwd(const KbTpParams& p, long long i) {
    const long long col = i / p.L;
    const int n = (int)(i - col * p.L);
    const long long b = col / p.C;
    const int c = (int)(col - b * p.C);
    const float z = p.zs[col];
    const long long d = (long long)p.ts[col] + 40 - 4LL * n;
    float v = 0.0f;
    if (z != 0.0f && d >= 0 && d < KB_TP_TAPS && n < kb_tp_len(p, b))
        v = (float)((double)p.g[col] * KB_TP_DB20 * (double)p.w4[d] / (double)z);
    p.gx[b * p.g_sb + (long long)c * p.g_sc + (long long)n * p.g_sl] = v;
}

// ------------------------------------------------------------------------------------------ 4. loudness series
// lo: kapre_loudness's parameters for the window (piece sums in p.part); out (B, Jmax); e (B, Jmax) or null.
KB_HD void kb_meter_series(const KbLoudParams& p, float* out, double* e, long long i) {
    const long long b = i / p.Jmax;
    const int j = (int)(i - b * p.Jmax);
    float v = -INFINITY;
    if (j < kb_loud_blocks(p, kb_loud_len(p, b))) {
        const double E = kb_loud_block(p, b, j);
        v = (float)(KB_LOUD_BIAS + 10.0 * log10(E));
        if (e) e[i] = E;
    }
    out[i] = v;
}

// ------------------------------------------------------------------------------------------ 5. loudness range
#define KB_LRA_REL_GATE -20.0

struct KbLraSmem {
    int cnt, red, n, tot, total;
};
KB_HD KbLraSmem kb_lra_smem() {
    KbLraSmem s;
    int off = 0;
    s.red = off; off += 64 * 8;                     // lane sums (E, non-finite count)
    s.cnt = off; off += 2 * 16 * 32 * 4;            // digit counts [target][digit][lane]
    s.n = off; off += 32 * 4;                       // lane counts
    s.tot = off; off += 2 * 16 * 4;                 // digit totals [target][digit]
    s.total = kb_align16(off);
    return s;
}

// Sums P.red[0 .. 64) pairwise and P.n[0 .. 32) by a fixed tree: totals in red[0], red[32], n[0].
KB_NOISE_FN void kb_lra_tree(double* red, int* n) {
    for (int d = 16; d >= 1; d >>= 1) {
        KB_NOISE_LANES_BEGIN
            if (lane < d) {
                red[lane] += red[lane + d];
                red[32 + lane] += red[32 + lane + d];
                n[lane] += n[lane + d];
            }
        KB_NOISE_LANES_END
        KB_SYNC_WARP;
    }
}

KB_D unsigned long long kb_d2u(double v) {
#if defined(KB_HOST_EMU)
    unsigned long long u;
    std::memcpy(&u, &v, 8);
    return u;
#else
    return (unsigned long long)__double_as_longlong(v);
#endif
}
KB_D double kb_u2d(unsigned long long u) {
#if defined(KB_HOST_EMU)
    double v;
    std::memcpy(&v, &u, 8);
    return v;
#else
    return __longlong_as_double((long long)u);
#endif
}

// p: the 3 s windows' geometry; e (B, Jmax): their E_j, rewritten here to E_j on J2 and 0 elsewhere; out: LRA per item.
KB_NOISE_FN void kb_meter_lra_tile(const KbLoudParams& p, double* e, float* out, char* smem, long long b) {
    const KbLraSmem S = kb_lra_smem();
    double* red = reinterpret_cast<double*>(smem + S.red);
    int* cnt = reinterpret_cast<int*>(smem + S.cnt);
    int* nn = reinterpret_cast<int*>(smem + S.n);
    int* tot = reinterpret_cast<int*>(smem + S.tot);
    const int J = kb_loud_blocks(p, kb_loud_len(p, b));
    double* eb = e + b * p.Jmax;
    // pass 1: the absolute gate (sum and count of J1) and the count of non-finite energies
    KB_NOISE_LANES_BEGIN
        double s = 0.0, nf = 0.0;
        int n = 0;
        for (int j = lane; j < J; j += 32) {
            const double E = eb[j];
            if (!(E - E == 0.0)) nf += 1.0;
            if (KB_LOUD_BIAS + 10.0 * log10(E) > KB_LOUD_ABS_GATE) { s += E; ++n; }
        }
        red[lane] = s; red[32 + lane] = nf; nn[lane] = n;
    KB_NOISE_LANES_END
    KB_SYNC_WARP;
    kb_lra_tree(red, nn);
    const double s1 = red[0];
    const int n1 = nn[0];
    const bool nan = red[32] != 0.0;
    KB_SYNC_WARP;
    // pass 2: the relative gate; E_j stays on J2 and becomes 0 elsewhere
    const double rel = KB_LOUD_BIAS + 10.0 * log10(s1 / (double)n1) + KB_LRA_REL_GATE;
    KB_NOISE_LANES_BEGIN
        int n = 0;
        for (int j = lane; j < J; j += 32) {
            const double E = eb[j];
            const double l = KB_LOUD_BIAS + 10.0 * log10(E);
            const bool in = n1 > 0 && l > KB_LOUD_ABS_GATE && l > rel;
            n += in;
            eb[j] = in ? E : 0.0;
        }
        red[lane] = 0.0; red[32 + lane] = 0.0; nn[lane] = n;
    KB_NOISE_LANES_END
    KB_SYNC_WARP;
    kb_lra_tree(red, nn);
    const int n2 = nn[0];
    KB_SYNC_WARP;
    if (nan || n2 == 0) {
        KB_NOISE_LANES_BEGIN
            if (lane == 0) out[b] = nan ? NAN : 0.0f;
        KB_NOISE_LANES_END
        return;
    }
    // pass 3: radix select of ranks lo and hi among the nonzero keys, four bits a round from the top
    int rank[2] = {((n2 - 1) * 10 + 50) / 100, ((n2 - 1) * 95 + 50) / 100};
    unsigned long long pre[2] = {0, 0}, msk = 0;
    for (int sh = 60; sh >= 0; sh -= 4) {
        KB_NOISE_LANES_BEGIN
            for (int q = 0; q < 32; ++q) cnt[q * 32 + lane] = 0;
            for (int j = lane; j < J; j += 32) {
                const unsigned long long k = kb_d2u(eb[j]);
                if (k == 0) continue;
                const int dg = (int)((k >> sh) & 15u);
                if ((k & msk) == pre[0]) ++cnt[dg * 32 + lane];
                if ((k & msk) == pre[1]) ++cnt[(16 + dg) * 32 + lane];
            }
        KB_NOISE_LANES_END
        KB_SYNC_WARP;
        KB_NOISE_LANES_BEGIN
            int t = 0;
            for (int l = 0; l < 32; ++l) t += cnt[lane * 32 + l];
            tot[lane] = t;
        KB_NOISE_LANES_END
        KB_SYNC_WARP;
        for (int q = 0; q < 2; ++q) {
            int dg = 0;
            while (dg < 15 && rank[q] >= tot[16 * q + dg]) rank[q] -= tot[16 * q + dg++];
            pre[q] |= (unsigned long long)dg << sh;
        }
        msk |= 15ull << sh;
        KB_SYNC_WARP;
    }
    KB_NOISE_LANES_BEGIN
        if (lane == 0)
            out[b] = (float)((KB_LOUD_BIAS + 10.0 * log10(kb_u2d(pre[1]))) - (KB_LOUD_BIAS + 10.0 * log10(kb_u2d(pre[0]))));
    KB_NOISE_LANES_END
}
