// Kernel bodies of additive noise at a target SNR (kapre_add_noise, torchaudio.functional.add_noise) and its gradient.
// For every (item, channel) column of x with L samples, noise n, snr in dB and valid length len:
//
//   Ex = sum_{t < len} x[t]^2,   En = sum_{t < len} n[t]^2,   s = sqrt(Ex / En) 10^(-snr / 20)   (s = 0 where Ex or En is 0)
//   y[t] = fmaf((float)s, n[t], x[t])   for every t < L
//
// and with g the output gradient and D = sum_{t < L} g[t] n[t]:
//
//   gx[t] = g[t] + [t < len] (D s / Ex) x[t],   gn[t] = s g[t] - [t < len] (D s / En) n[t],   gsnr = -D s ln(10) / 20.
//
// Ex, En, D and s are float64: the product of two float32 values is exact in float64, so only the additions round.
// The summation order is a function of the column and the absolute sample index alone: a column is cut into segments
// of KB_NOISE_SEG samples; in a segment, lane j of a warp sums samples j, j + 32, j + 64, ... in ascending order, the
// 32 lane sums are added by a fixed tree (halving strides 16, 8, 4, 2, 1), and the segment sums are folded in segment
// order.  No atomics: an output's bits do not depend on the grid, the batch, the strides, the data format, whether a
// broadcast noise is materialised, or whether the noise comes from a tensor or from a bank.
//
// Work split: one warp per tile of (item, group of up to KB_NOISE_G channels, segment).  A tile runs in rounds of
// KB_NOISE_R samples: each operand's (channels x samples) block is staged in shared memory, read by the lanes in the
// order of its layout (consecutive samples of a column when time is contiguous, consecutive (sample, channel) pairs
// when channels are interleaved), so global loads and stores coalesce in both formats while every lane reduces its
// own samples.  Two launches each way:
//   forward   1. energy (kb_noise_sum_tile):  per tile the segment sums of x^2 and n^2 over t < len, into `part`;
//             2. mix    (kb_noise_out_tile):  fold the column's segment sums in order, s, and y; the tile of segment 0
//                                             writes (Ex, En) to `stats`;
//   backward  1. D      (kb_noise_sum_tile):  per tile the segment sum of g n, into `part`;
//             2. grads  (kb_noise_out_tile):  fold D, then gx (and gn, gsnr when asked for) from the saved stats.
//
// Noise: a (batch, channel, sample)-strided tensor (strides 0 broadcast), or a bank of mono clips, where item b reads
// n[b, c, t] = bank[start_b + (offset_b + t) mod clip_b] for every channel; the wrap is kept incrementally per lane.
//
// Like the other bodies these are barrier-free phases: under nvcc each phase runs once per lane and the phases are
// separated by __syncwarp(); the CPU emulation (tests/emu, KB_HOST_EMU) runs each phase as a loop over the lanes.
#pragma once
#include "stft_core.cuh"

#define KB_NOISE_SEG 4096                           // samples per segment (fixes the summation tree)
#define KB_NOISE_R 256                              // samples per staged round
#define KB_NOISE_PL (KB_NOISE_R / 32)               // samples of a round per lane and row
#define KB_NOISE_G 8                                // channels per tile
#define KB_NOISE_WARPS 4                            // tiles (warps) per CTA

struct KbNoiseWave {
    const float* p;
    long long sb, sc, sl;                           // element strides (batch, channel, sample)
};

struct KbNoiseParams {
    KbNoiseWave x;                                  // forward: x; backward: the output gradient g
    KbNoiseWave xr;                                 // backward: the forward's x
    KbNoiseWave n;                                  // tensor noise (n.p null in bank mode)
    const float* bank; long long bank_numel;        // bank mode: concatenated mono clips
    const long long* start;                         // per item: first sample of the clip in the bank
    const long long* clip;                          // per item: clip length
    const long long* offset;                        // per item: clip sample at t = 0
    const float* snr; long long snr_sb, snr_sc;     // dB, per (item, channel) by strides (0 broadcasts)
    const int* len; long long len_sb, len_sc;       // valid lengths (null: L)
    float* y; long long y_sb, y_sc, y_sl;           // forward: y; backward: gx
    float* gn; long long gn_sb, gn_sc, gn_sl;       // backward, optional
    float* gsnr;                                    // backward, optional: (B, C) contiguous
    double* stats;                                  // (B C, 2) (Ex, En): written by the forward (optional), read back
    double* part;                                   // (B C, nseg, 2) segment sums
    int B, C, L;
    int G, nseg;                                    // channel groups per item, segments per column
    long long tiles;                                // B G nseg
    int bwd;
};

// Shared memory of one tile (one warp) whose groups have at most cg channels: the lane sums for the tree (two per
// channel), the staged blocks of x (or g), the noise and, in the backward, the forward's x; per channel the mask limit,
// the limit L, and the scales.
struct KbNoiseSmem {
    int red, xs, ns, rs, lim, sv, total;
};
KB_HD KbNoiseSmem kb_noise_smem(int cg) {
    KbNoiseSmem s;
    int off = 0;
    s.red = off; off += 2 * cg * 32 * 8;
    s.xs = off; off += cg * KB_NOISE_R * 4;
    s.ns = off; off += cg * KB_NOISE_R * 4;
    s.rs = off; off += cg * KB_NOISE_R * 4;
    s.lim = off; off += (2 * KB_NOISE_G + 2) * 4;
    s.sv = off; off += 4 * KB_NOISE_G * 8;
    s.total = kb_align16(off);
    return s;
}

// ---- host side: geometry (shared by the library and the CPU emulation) ----
inline void kb_noise_setup(KbNoiseParams& p) {
    p.G = (p.C + KB_NOISE_G - 1) / KB_NOISE_G;
    p.nseg = (int)(((long long)p.L + KB_NOISE_SEG - 1) / KB_NOISE_SEG);
    p.tiles = (long long)p.B * p.G * p.nseg;
}

#define KB_NOISE_LN10_20 0.11512925464970229         // ln(10) / 20

// s in float64; 0 where either energy is 0 (a silent noise excerpt leaves the signal as it is).  10^(-snr / 20) is
// exp(-snr ln(10) / 20): exp needs no stack on the device, pow does.
KB_HD double kb_noise_scale(double ex, double en, float snr) {
    if (ex == 0.0 || en == 0.0) return 0.0;
    return sqrt(ex / en) * exp(-(double)snr * KB_NOISE_LN10_20);
}

struct KbNoiseTile {
    long long b;
    int c0, cg, seg;
};

KB_HD KbNoiseTile kb_noise_tile(const KbNoiseParams& p, long long tile) {
    KbNoiseTile t;
    const long long bg = tile / p.nseg;
    t.seg = (int)(tile - bg * p.nseg);
    t.b = bg / p.G;
    t.c0 = (int)(bg - t.b * p.G) * KB_NOISE_G;
    t.cg = p.C - t.c0 < KB_NOISE_G ? p.C - t.c0 : KB_NOISE_G;
    return t;
}

KB_HD long long kb_noise_abs(long long v) { return v < 0 ? -v : v; }

// A lane's walk over one operand's (rows x R) block of a round.  Element e = lane + 32 j of the block is read in the
// order of the operand's layout: channel-major (row e / R, sample e mod R: lanes read consecutive samples of a row) when
// time is contiguous, sample-major (sample e / rows, row e mod rows: lanes read consecutive (sample, channel) pairs)
// when channels are interleaved.  rows == 1 with a channel stride of 0 is a broadcast noise, staged once for every
// channel.  The block lands in shared memory as dst[row * R + sample] either way.
struct KbNoiseCur {
    const float* base;
    long long sc, sl;
    int rows, sm;                                   // sm: sample-major
    int s, c, q, r;                                 // sample-major: position of the lane's next element, and its step
};

KB_HD KbNoiseCur kb_noise_cur(const float* p, long long sb, long long sc, long long sl, long long b, int c0, int rows,
                              int lane) {
    KbNoiseCur k;
    k.base = p + b * sb + (long long)c0 * sc;
    k.sc = sc; k.sl = sl; k.rows = rows;
    k.sm = rows > 1 && kb_noise_abs(sc) < kb_noise_abs(sl);
    k.q = 32 / rows; k.r = 32 - k.q * rows;
    k.s = lane / rows; k.c = lane - k.s * rows;
    return k;
}

// Steps a sample-major cursor to the lane's next element.
KB_HD void kb_noise_step(KbNoiseCur& k) {
    k.s += k.q; k.c += k.r;
    if (k.c >= k.rows) { k.c -= k.rows; ++k.s; }
}

// Batch bt of a block (elements lane + 32 j, 8 bt <= j < 8 bt + 8): the lane's values, 0 at or past lim[row].  The
// caller issues every operand's fetch of a batch before it stores any of them (kb_noise_put), so a lane has all those
// loads in flight together.
KB_HD void kb_noise_fetch(KbNoiseCur& k, int t0, const int* lim, int bt, int lane, float* v) {
    if (k.sm) {
#pragma unroll
        for (int i = 0; i < KB_NOISE_PL; ++i) {
            const int t = t0 + k.s;
            v[i] = t < lim[k.c] ? k.base[k.c * k.sc + (long long)t * k.sl] : 0.0f;
            kb_noise_step(k);
        }
    } else {
        const int lc = lim[bt];
        const float* row = k.base + bt * k.sc;
#pragma unroll
        for (int i = 0; i < KB_NOISE_PL; ++i) {
            const int t = t0 + lane + 32 * i;
            v[i] = t < lc ? row[(long long)t * k.sl] : 0.0f;
        }
    }
}

// Stores a fetched batch into dst[row * R + sample]; k is the cursor as it was before the fetch.
KB_HD void kb_noise_put(KbNoiseCur k, int bt, int lane, const float* v, float* dst) {
#pragma unroll
    for (int i = 0; i < KB_NOISE_PL; ++i) {
        if (k.sm) {
            dst[k.c * KB_NOISE_R + k.s] = v[i];
            kb_noise_step(k);
        } else {
            dst[bt * KB_NOISE_R + lane + 32 * i] = v[i];
        }
    }
}

// The mirror for an output (a cursor made from the output pointer): batch bt of the block in src goes to
// [t0, min(t0 + R, L)) through the cursor's strides, the shared-memory reads first, then the global stores.
KB_HD void kb_noise_emit(KbNoiseCur& k, int t0, int L, int bt, int lane, const float* src) {
    float v[KB_NOISE_PL];
    KbNoiseCur k0 = k;
#pragma unroll
    for (int i = 0; i < KB_NOISE_PL; ++i) {
        if (k.sm) {
            v[i] = src[k.c * KB_NOISE_R + k.s];
            kb_noise_step(k);
        } else {
            v[i] = src[bt * KB_NOISE_R + lane + 32 * i];
        }
    }
    float* out = const_cast<float*>(k0.base);
#pragma unroll
    for (int i = 0; i < KB_NOISE_PL; ++i) {
        const int s = k0.sm ? k0.s : lane + 32 * i, c = k0.sm ? k0.c : bt;
        if (t0 + s < L) out[c * k0.sc + (long long)(t0 + s) * k0.sl] = v[i];
        if (k0.sm) kb_noise_step(k0);
    }
}

// A lane's position in its item's bank clip for samples lane + 32 i (i < KB_NOISE_PL) of the round at t0; clip <= 0 or
// a clip outside the bank reads no samples (the noise is 0, so y = x).
struct KbNoiseBankPos {
    const float* clip_p;                            // null: no samples
    long long clip, step;                           // step = R mod clip
    long long u[KB_NOISE_PL];
};

KB_HD KbNoiseBankPos kb_noise_bank_pos(const KbNoiseParams& p, long long b, int t0, int lane) {
    KbNoiseBankPos q;
    const long long st = p.start[b], cl = p.clip[b];
    q.clip_p = nullptr; q.clip = 1; q.step = 0;
#pragma unroll
    for (int i = 0; i < KB_NOISE_PL; ++i) q.u[i] = 0;
    if (cl <= 0 || st < 0 || st > p.bank_numel - cl) return q;
    q.clip_p = p.bank + st;
    q.clip = cl;
    q.step = KB_NOISE_R % cl;
    long long o = p.offset[b] % cl;
    if (o < 0) o += cl;
#pragma unroll
    for (int i = 0; i < KB_NOISE_PL; ++i) q.u[i] = (o + t0 + lane + 32 * i) % cl;
    return q;
}

// The bank's samples of the round at t0 (0 at or past lim), as one batch of a one-row block; advances the positions.
KB_HD void kb_noise_fetch_bank(KbNoiseBankPos& q, int t0, int lim, int lane, float* v) {
#pragma unroll
    for (int i = 0; i < KB_NOISE_PL; ++i) {
        const int s = lane + 32 * i;
        v[i] = q.clip_p && t0 + s < lim ? q.clip_p[q.u[i]] : 0.0f;
        const long long u = q.u[i] + q.step;
        q.u[i] = u >= q.clip ? u - q.clip : u;
    }
}

#if defined(KB_HOST_EMU)
#define KB_NOISE_LANES_BEGIN for (int lane = 0; lane < 32; ++lane) {
#define KB_NOISE_LANES_END }
#define KB_NOISE_FN inline
#define KB_NOISE_LANE_VAR(T, v) T v##_lanes[32]        // a per-lane value that lives across phases
#define KB_NOISE_LANE_ARR(T, v, n) T v##_lanes[32][n]
#define KB_NOISE_LV(v) v##_lanes[lane]
#else
#define KB_NOISE_LANES_BEGIN { const int lane = (int)(threadIdx.x & 31);
#define KB_NOISE_LANES_END }
#define KB_NOISE_FN __device__ __forceinline__
#define KB_NOISE_LANE_VAR(T, v) T v
#define KB_NOISE_LANE_ARR(T, v, n) T v[n]
#define KB_NOISE_LV(v) v
#endif

struct KbNoisePtrs {
    double *red, *red1;                             // [cg][32] lane sums of the first and the second sum
    float *xs, *ns, *rs;                            // staged blocks [cg][R]
    int *lim, *full;                                // per channel: min(max(len, 0), L), and L
    int* one;                                       // the largest limit and L (a channel-broadcast noise's limits)
    double* dv;                                     // [3][KB_NOISE_G]: s, D s / Ex, D s / En
    float* sv;                                      // [KB_NOISE_G]: (float)s
};

KB_HD KbNoisePtrs kb_noise_ptrs(char* smem, int cg) {
    const KbNoiseSmem S = kb_noise_smem(cg);
    KbNoisePtrs P;
    P.red = reinterpret_cast<double*>(smem + S.red);
    P.red1 = P.red + cg * 32;
    P.xs = reinterpret_cast<float*>(smem + S.xs);
    P.ns = reinterpret_cast<float*>(smem + S.ns);
    P.rs = reinterpret_cast<float*>(smem + S.rs);
    P.lim = reinterpret_cast<int*>(smem + S.lim);
    P.full = P.lim + KB_NOISE_G;
    P.one = P.lim + 2 * KB_NOISE_G;
    P.dv = reinterpret_cast<double*>(smem + S.sv);
    P.sv = reinterpret_cast<float*>(smem + S.sv + 3 * KB_NOISE_G * 8);
    return P;
}

// Largest channel count of a tile: the shared-memory layout every tile of a launch uses.
KB_HD int kb_noise_cg_max(const KbNoiseParams& p) { return p.C < KB_NOISE_G ? p.C : KB_NOISE_G; }

// Per channel of the tile the mask limit min(max(len, 0), L) (L without lengths) and L; returns the largest limit.
KB_NOISE_FN int kb_noise_limits(const KbNoiseParams& p, const KbNoiseTile& t, const KbNoisePtrs& P) {
    KB_NOISE_LANES_BEGIN
        if (lane < t.cg) {
            int v = p.L;
            if (p.len) {
                const int l = p.len[t.b * p.len_sb + (long long)(t.c0 + lane) * p.len_sc];
                v = l < 0 ? 0 : (l > p.L ? p.L : l);
            }
            P.lim[lane] = v;
            P.full[lane] = p.L;
        }
    KB_NOISE_LANES_END
    KB_SYNC_WARP;
    int m = 0;
    for (int c = 0; c < t.cg; ++c) m = P.lim[c] > m ? P.lim[c] : m;
    KB_NOISE_LANES_BEGIN
        if (lane == 0) { P.one[0] = m; P.one[1] = p.L; }
    KB_NOISE_LANES_END
    KB_SYNC_WARP;
    return m;
}

// Rows of the staged noise: one for a bank or a channel-broadcast tensor, else the tile's channels.
KB_HD int kb_noise_rows(const KbNoiseParams& p, const KbNoiseTile& t) {
    return (p.n.p == nullptr || p.n.sc == 0) ? 1 : t.cg;
}

// Batch bt of the round's noise block: a tensor through its cursor, or the bank (a one-row block: bt == 0).
KB_HD void kb_noise_fetch_noise(const KbNoiseParams& p, KbNoiseCur& k, KbNoiseBankPos& bp, int t0, const int* lim,
                                int bt, int lane, float* v) {
    if (p.n.p) kb_noise_fetch(k, t0, lim, bt, lane, v);
    else kb_noise_fetch_bank(bp, t0, lim[0], lane, v);
}

// ------------------------------------------------------------------------------------------ 1. segment sums
// Forward: x^2 and n^2 over t < len.  Backward: g n over t < L.  part[(col, seg)] = (first sum, second sum).
KB_NOISE_FN void kb_noise_sum_tile(const KbNoiseParams& p, char* smem, long long tile) {
    const KbNoiseTile t = kb_noise_tile(p, tile);
    const KbNoisePtrs P = kb_noise_ptrs(smem, kb_noise_cg_max(p));
    const int lim_max = p.bwd ? p.L : kb_noise_limits(p, t, P);
    if (p.bwd) kb_noise_limits(p, t, P);                 // fills P.full
    const int* lim = p.bwd ? P.full : P.lim;
    const int rows = kb_noise_rows(p, t);
    const int t_seg = t.seg * KB_NOISE_SEG;
    const int t_end = p.L - t_seg < KB_NOISE_SEG ? p.L : t_seg + KB_NOISE_SEG;
    KB_NOISE_LANE_ARR(double, a0, KB_NOISE_G);
    KB_NOISE_LANE_ARR(double, a1, KB_NOISE_G);
    KB_NOISE_LANE_VAR(KbNoiseBankPos, bp);
    KB_NOISE_LANES_BEGIN
#pragma unroll
        for (int c = 0; c < KB_NOISE_G; ++c) { KB_NOISE_LV(a0)[c] = 0.0; KB_NOISE_LV(a1)[c] = 0.0; }
        if (!p.n.p) KB_NOISE_LV(bp) = kb_noise_bank_pos(p, t.b, t_seg, lane);
    KB_NOISE_LANES_END
    for (int t0 = t_seg; t0 < t_end && t0 < lim_max; t0 += KB_NOISE_R) {
        KB_NOISE_LANES_BEGIN
            KbNoiseCur kx = kb_noise_cur(p.x.p, p.x.sb, p.x.sc, p.x.sl, t.b, t.c0, t.cg, lane);
            KbNoiseCur kn = kb_noise_cur(p.n.p, p.n.sb, p.n.sc, p.n.sl, t.b, t.c0, rows, lane);
            const int* nlim = rows == 1 ? (p.bwd ? P.one + 1 : P.one) : lim;
            for (int bt = 0; bt < t.cg; ++bt) {
                float vx[KB_NOISE_PL], vn[KB_NOISE_PL];
                const KbNoiseCur kx0 = kx, kn0 = kn;
                kb_noise_fetch(kx, t0, lim, bt, lane, vx);
                if (bt < rows) kb_noise_fetch_noise(p, kn, KB_NOISE_LV(bp), t0, nlim, bt, lane, vn);
                kb_noise_put(kx0, bt, lane, vx, P.xs);
                if (bt < rows) kb_noise_put(kn0, bt, lane, vn, P.ns);
            }
        KB_NOISE_LANES_END
        KB_SYNC_WARP;
        KB_NOISE_LANES_BEGIN
#pragma unroll
            for (int c = 0; c < KB_NOISE_G; ++c) {
                if (c < t.cg) {
                    const float* nr = P.ns + (rows > 1 ? c : 0) * KB_NOISE_R;
                    const int lc = lim[c];
                    double s0 = KB_NOISE_LV(a0)[c], s1 = KB_NOISE_LV(a1)[c];
#pragma unroll
                    for (int i = 0; i < KB_NOISE_PL; ++i) {
                        const int s = lane + 32 * i;
                        const double xv = (double)P.xs[c * KB_NOISE_R + s], nv = (double)nr[s];
                        if (t0 + s < lc) {
                            if (p.bwd) {
                                s0 += xv * nv;
                            } else {
                                s0 += xv * xv;
                                s1 += nv * nv;
                            }
                        }
                    }
                    KB_NOISE_LV(a0)[c] = s0;
                    KB_NOISE_LV(a1)[c] = s1;
                }
            }
        KB_NOISE_LANES_END
        KB_SYNC_WARP;
    }
    // the fixed tree over the 32 lane sums
    KB_NOISE_LANES_BEGIN
#pragma unroll
        for (int c = 0; c < KB_NOISE_G; ++c) {
            if (c < t.cg) {
                P.red[c * 32 + lane] = KB_NOISE_LV(a0)[c];
                P.red1[c * 32 + lane] = KB_NOISE_LV(a1)[c];
            }
        }
    KB_NOISE_LANES_END
    KB_SYNC_WARP;
    for (int d = 16; d >= 1; d >>= 1) {
        KB_NOISE_LANES_BEGIN
            if (lane < d) {
                for (int c = 0; c < t.cg; ++c) {
                    P.red[c * 32 + lane] += P.red[c * 32 + lane + d];
                    P.red1[c * 32 + lane] += P.red1[c * 32 + lane + d];
                }
            }
        KB_NOISE_LANES_END
        KB_SYNC_WARP;
    }
    KB_NOISE_LANES_BEGIN
        if (lane < t.cg) {
            const long long col = t.b * p.C + t.c0 + lane;
            double* o = p.part + (col * p.nseg + t.seg) * 2;
            o[0] = P.red[lane * 32];
            o[1] = P.red1[lane * 32];
        }
    KB_NOISE_LANES_END
}

// ------------------------------------------------------------------------------------------ 2. output
// Forward: y = fmaf(s, n, x).  Backward: gx, and gn and gsnr when their pointers are set.
KB_NOISE_FN void kb_noise_out_tile(const KbNoiseParams& p, char* smem, long long tile) {
    const KbNoiseTile t = kb_noise_tile(p, tile);
    const KbNoisePtrs P = kb_noise_ptrs(smem, kb_noise_cg_max(p));
    kb_noise_limits(p, t, P);
    const int rows = kb_noise_rows(p, t);
    const int t_seg = t.seg * KB_NOISE_SEG;
    const int t_end = p.L - t_seg < KB_NOISE_SEG ? p.L : t_seg + KB_NOISE_SEG;
    // lane c folds channel c's segment sums in segment order
    KB_NOISE_LANES_BEGIN
        if (lane < t.cg) {
            const long long col = t.b * p.C + t.c0 + lane;
            const double* q = p.part + col * p.nseg * 2;
            double e0 = 0.0, e1 = 0.0;
            for (int k = 0; k < p.nseg; ++k) { e0 += q[2 * k]; e1 += q[2 * k + 1]; }
            const float snr = p.snr[t.b * p.snr_sb + (long long)(t.c0 + lane) * p.snr_sc];
            if (!p.bwd) {
                P.sv[lane] = (float)kb_noise_scale(e0, e1, snr);
                if (t.seg == 0 && p.stats) { p.stats[col * 2] = e0; p.stats[col * 2 + 1] = e1; }
            } else {
                const double ex = p.stats[col * 2], en = p.stats[col * 2 + 1];
                const double s = kb_noise_scale(ex, en, snr), ds = e0 * s;
                P.dv[lane] = s;
                P.dv[KB_NOISE_G + lane] = s != 0.0 ? ds / ex : 0.0;
                P.dv[2 * KB_NOISE_G + lane] = s != 0.0 ? ds / en : 0.0;
                if (t.seg == 0 && p.gsnr) p.gsnr[col] = (float)(-ds * KB_NOISE_LN10_20);
            }
        }
    KB_NOISE_LANES_END
    KB_SYNC_WARP;
    KB_NOISE_LANE_VAR(KbNoiseBankPos, bp);
    if (!p.n.p && !p.bwd) {
        KB_NOISE_LANES_BEGIN
            KB_NOISE_LV(bp) = kb_noise_bank_pos(p, t.b, t_seg, lane);
        KB_NOISE_LANES_END
    }
    const int want_n = !p.bwd || p.gn;
    for (int t0 = t_seg; t0 < t_end; t0 += KB_NOISE_R) {
        KB_NOISE_LANES_BEGIN
            KbNoiseCur kx = kb_noise_cur(p.x.p, p.x.sb, p.x.sc, p.x.sl, t.b, t.c0, t.cg, lane);
            KbNoiseCur kr = kb_noise_cur(p.xr.p, p.xr.sb, p.xr.sc, p.xr.sl, t.b, t.c0, t.cg, lane);
            KbNoiseCur kn = kb_noise_cur(p.n.p, p.n.sb, p.n.sc, p.n.sl, t.b, t.c0, rows, lane);
            const int* nlim = rows == 1 ? (p.bwd ? P.one : P.one + 1) : (p.bwd ? P.lim : P.full);
            for (int bt = 0; bt < t.cg; ++bt) {
                float vx[KB_NOISE_PL], vr[KB_NOISE_PL], vn[KB_NOISE_PL];
                const KbNoiseCur kx0 = kx, kr0 = kr, kn0 = kn;
                kb_noise_fetch(kx, t0, P.full, bt, lane, vx);
                if (p.bwd) kb_noise_fetch(kr, t0, P.lim, bt, lane, vr);
                if (want_n && bt < rows) kb_noise_fetch_noise(p, kn, KB_NOISE_LV(bp), t0, nlim, bt, lane, vn);
                kb_noise_put(kx0, bt, lane, vx, P.xs);
                if (p.bwd) kb_noise_put(kr0, bt, lane, vr, P.rs);
                if (want_n && bt < rows) kb_noise_put(kn0, bt, lane, vn, P.ns);
            }
        KB_NOISE_LANES_END
        KB_SYNC_WARP;
        KB_NOISE_LANES_BEGIN
            for (int c = 0; c < t.cg; ++c) {
                float* xr = P.xs + c * KB_NOISE_R;
                float* rr = P.rs + c * KB_NOISE_R;
                const float* nr = P.ns + (rows > 1 ? c : 0) * KB_NOISE_R;
                if (!p.bwd) {
                    const float s = P.sv[c];
#pragma unroll
                    for (int i = 0; i < KB_NOISE_PL; ++i) {
                        const int e = lane + 32 * i;
                        xr[e] = fmaf(s, nr[e], xr[e]);
                    }
                } else {
                    const double s = P.dv[c], cx = P.dv[KB_NOISE_G + c], cn = P.dv[2 * KB_NOISE_G + c];
                    const int lc = P.lim[c];
#pragma unroll
                    for (int i = 0; i < KB_NOISE_PL; ++i) {
                        const int e = lane + 32 * i;
                        const bool in = t0 + e < lc;
                        const double g = (double)xr[e], xv = (double)rr[e];
                        if (p.gn) rr[e] = (float)(s * g - (in ? cn * (double)nr[e] : 0.0));
                        xr[e] = (float)(g + (in ? cx * xv : 0.0));
                    }
                }
            }
        KB_NOISE_LANES_END
        KB_SYNC_WARP;
        KB_NOISE_LANES_BEGIN
            KbNoiseCur ky = kb_noise_cur(p.y, p.y_sb, p.y_sc, p.y_sl, t.b, t.c0, t.cg, lane);
            for (int bt = 0; bt < t.cg; ++bt) kb_noise_emit(ky, t0, p.L, bt, lane, P.xs);
            if (p.bwd && p.gn) {
                KbNoiseCur kg = kb_noise_cur(p.gn, p.gn_sb, p.gn_sc, p.gn_sl, t.b, t.c0, t.cg, lane);
                for (int bt = 0; bt < t.cg; ++bt) kb_noise_emit(kg, t0, p.L, bt, lane, P.rs);
            }
        KB_NOISE_LANES_END
        KB_SYNC_WARP;
    }
}
