// Kernel body of the band-limited interpolator (J. O. Smith's algorithm, as in resampy): resampling by any real
// ratio with one filter table that does not depend on the ratio.
//
//   h(u) = sinc(u) I0(beta sqrt(1 - (u / Z)^2)) / I0(beta) for |u| < Z, else 0   (Z = 10 zero crossings, beta = 5)
//   I    = integral of h over [-Z, Z]
//   y[m] = (gain / I) sum_j x[j] h(s (pos(m) - j)),   pos(m) = offset + m step,   x[j] = 0 outside [0, L)
//
// Forward, ratio rho = output rate / input rate: step = 1 / rho, s = gain = min(1, rho).  Adjoint (h is even): the
// same sum over the output gradient with step' = rho, offset' = -offset rho, s' = s / rho, gain' = gain
// (kb_sinc_args).  Both are this one body with other numbers.
//
// Table: (h(k / Q), h((k + 1) / Q) - h(k / Q)) for k = 0 .. Z Q, float32 pairs, so that a tap weight is one 8 B
// shared-memory load and one FMA: h(t / Q) ~ tab[k].x + (t - k) tab[k].y with k = floor(t).  The linear
// interpolation is off by at most max|h''| / (8 Q^2) = 4.0e-7 per tap at Q = 1024 (max|h''| = 3.33 at u = 0).
//
// Per output m: pos(m) is one float64 multiply-add, split into n = floor(pos) and frac = pos - n.  The taps are
// walked in two wings of nw = ceil(Z / s) taps each: x[n - i] at u = s (frac + i) and x[n + 1 + i] at
// u = s (1 - frac + i), i = 0 .. nw - 1.  The table position of tap i is fma(i, s Q, frac s Q) in float32, formed
// from the integer tap counter, so it carries three roundings whatever i is: a relative error of 1.8e-7 in u, i.e.
// at most 1.8e-7 |u h'(u)| <= 2e-7 in the weight.  Positions past the table's end are clamped to its last entry,
// which is (0, 0).  Everything an output depends on is computed from m alone, so an output does not depend on the
// tile it fell in, the grid, the batch position, the data format or the strides.
//
// Data movement is that of resample_core.cuh: a persistent CTA walks tiles of NT consecutive outputs of one
// (item, channel group); a group is one channel or all C channels of a channel-interleaved waveform, staged as
// [sample][channel]; the tile's input span comes in by one TMA bulk copy when it lies inside the signal and is
// contiguous in memory, else through the cooperative loader (any strides, zeros outside the signal).  Each thread
// owns one channel of the group and every S-th output of the tile (S = threads / G).
//
// Written as barrier-free phases like the other bodies (KB_HOST_EMU runs each phase as a loop over the threads).
#pragma once
#include <cmath>
#include <vector>
#include "resample_core.cuh"

#define KB_SINC_THREADS 512
#define KB_SINC_Z 10                                    // zero crossings on either side
#define KB_SINC_Q 1024                                  // table entries per zero crossing
#define KB_SINC_BETA 5.0                                // Kaiser beta, the family of signal.resample_filter
#define KB_SINC_NTAB (KB_SINC_Z * KB_SINC_Q + 1)
#define KB_SINC_RATIO_MIN 0.25                          // two octaves either way: at most 80 taps per output
#define KB_SINC_RATIO_MAX 4.0

struct KbSincParams {
    const float* x;                 // input, element strides (batch, channel, sample)
    long long x_sb, x_sc, x_sl;
    long long x_numel;              // elements addressable from x (max element offset + 1)
    unsigned x_align;               // ((uintptr_t)x >> 2) & 3
    int bulk_ok;                    // a tile's span is one contiguous run of memory
    int B, C, L;
    float* y;                       // output, element strides (batch, channel, sample)
    long long y_sb, y_sc, y_sl;
    int L_out;
    const float2* tab;              // KB_SINC_NTAB pairs (device)
    double step, offset;            // pos(m) = offset + m step, in input samples
    float sQ;                       // s Q: table entries per input sample
    float scale;                    // gain / I
    int nw;                         // taps per wing
    int G, n_groups;                // channels per tile, channel groups per item (C / G)
    int NT, n_tiles_t, n_tiles;     // outputs per tile, tiles per (item, group), all tiles
    int S;                          // thread's output stride
    int n_threads;
};

// ---- host side: the filter, its table, and the numbers of a call (shared by the library and the CPU emulation) ----
inline double kb_sinc_i0(double x) {
    const double t = 0.25 * x * x;
    double term = 1.0, sum = 1.0;
    for (int k = 1; k < 200; ++k) {
        term *= t / ((double)k * (double)k);
        sum += term;
        if (term < 1e-18 * sum) break;
    }
    return sum;
}

inline double kb_sinc_h(double u) {
    const double a = std::fabs(u) / KB_SINC_Z;
    if (a >= 1.0) return 0.0;
    const double pu = 3.14159265358979323846 * u;
    const double sc = u == 0.0 ? 1.0 : std::sin(pu) / pu;
    return sc * kb_sinc_i0(KB_SINC_BETA * std::sqrt(1.0 - a * a)) / kb_sinc_i0(KB_SINC_BETA);
}

// I: composite Simpson over [0, Z] with 4096 intervals per zero crossing, doubled (h is even).
inline double kb_sinc_integral() {
    const int n = KB_SINC_Z * 4096;
    const double dx = (double)KB_SINC_Z / n;
    double sum = kb_sinc_h(0.0) + kb_sinc_h((double)KB_SINC_Z);
    for (int k = 1; k < n; ++k) sum += ((k & 1) ? 4.0 : 2.0) * kb_sinc_h(k * dx);
    return 2.0 * sum * dx / 3.0;
}

inline void kb_sinc_table(std::vector<float2>& tab) {
    tab.resize(KB_SINC_NTAB);
    double h0 = kb_sinc_h(0.0);
    for (int k = 0; k < KB_SINC_NTAB; ++k) {
        const double h1 = k + 1 < KB_SINC_NTAB ? kb_sinc_h((double)(k + 1) / KB_SINC_Q) : 0.0;
        tab[k].x = (float)h0;
        tab[k].y = k + 1 < KB_SINC_NTAB ? (float)(h1 - h0) : 0.0f;
        h0 = h1;
    }
}

// The four numbers of a call from (ratio, offset): the forward sum, or its adjoint.
inline void kb_sinc_args(double ratio, double offset, int adjoint, double* step, double* off, double* s, double* gain) {
    const double s_fwd = ratio < 1.0 ? ratio : 1.0;
    *gain = s_fwd;
    if (!adjoint) { *step = 1.0 / ratio; *off = offset; *s = s_fwd; }
    else { *step = ratio; *off = -offset * ratio; *s = s_fwd / ratio; }
}

KB_HD int kb_sinc_span(int NT, double step, int nw) { return (int)ceil((double)(NT - 1) * step) + 2 + 2 * nw; }
KB_HD int kb_sinc_smem(int NT, double step, int nw, int G) {
    return 16 + kb_align16(KB_SINC_NTAB * 8) + kb_align16((kb_sinc_span(NT, step, nw) * G + 8) * 4);
}

// Stepping and tiling constants once x, y, B, C, L, L_out, G and NT are set; false: too many tiles.
inline bool kb_sinc_setup(KbSincParams& p, double step, double offset, double s, double gain, double integral, int n_threads) {
    p.step = step; p.offset = offset;
    p.sQ = (float)(s * KB_SINC_Q);
    p.scale = (float)(gain / integral);
    p.nw = (int)std::ceil((double)KB_SINC_Z / s);
    p.n_groups = p.C / p.G;
    p.n_tiles_t = (int)((p.L_out + (long long)p.NT - 1) / p.NT);
    const long long tiles = (long long)p.B * p.n_groups * p.n_tiles_t;
    if (tiles > 0x7fffffffLL) return false;
    p.n_tiles = (int)tiles;
    p.n_threads = n_threads;
    p.S = n_threads / p.G;
    return true;
}

KB_HD double kb_sinc_pos(const KbSincParams& p, long long m) { return fma((double)m, p.step, p.offset); }

struct KbSincTile {
    int b, g, nt;                   // item, channel group, outputs in this tile
    long long m0, i0;               // first output, first staged input sample
    int count;                      // staged floats (samples x G)
    int bulk, head, bytes;          // bulk copy: element i0 lands at buf[head]; bytes copied from src
    const float* src;
};

KB_HD KbSincTile kb_sinc_tile(const KbSincParams& p, int tile) {
    KbSincTile t;
    const int sig = tile / p.n_tiles_t, tt = tile - sig * p.n_tiles_t;
    t.b = sig / p.n_groups;
    t.g = sig - t.b * p.n_groups;
    t.m0 = (long long)tt * p.NT;
    t.nt = (int)((long long)p.L_out - t.m0 < p.NT ? (long long)p.L_out - t.m0 : p.NT);
    // pos is non-decreasing in m, so the first and the last output bound the span
    t.i0 = (long long)floor(kb_sinc_pos(p, t.m0)) - (p.nw - 1);
    const long long i_end = (long long)floor(kb_sinc_pos(p, t.m0 + t.nt - 1)) + p.nw + 1;      // one past the last sample read
    t.count = (int)(i_end - t.i0) * p.G;
    t.bulk = 0; t.head = 0; t.bytes = 0; t.src = nullptr;
    if (p.bulk_ok && t.i0 >= 0 && i_end <= p.L) {
        const long long off0 = (long long)t.b * p.x_sb + (long long)t.g * p.G * p.x_sc + t.i0 * p.x_sl;
        const int head = (int)((p.x_align + (unsigned)off0) & 3u);
        const int tail = (int)((0u - (p.x_align + (unsigned)off0 + (unsigned)t.count)) & 3u);
        if (off0 - head >= 0 && off0 + t.count + tail <= p.x_numel) {
            t.bulk = 1; t.head = head; t.src = p.x + (off0 - head); t.bytes = (head + t.count + tail) * 4;
        }
    }
    return t;
}

KB_RS_FN void kb_sinc_cta(const KbSincParams& p, char* smem, int cta, int n_cta) {
    KbBar* bar = reinterpret_cast<KbBar*>(smem);
    float2* tab = reinterpret_cast<float2*>(smem + 16);
    float* buf = reinterpret_cast<float*>(smem + 16 + kb_align16(KB_SINC_NTAB * 8));
    KB_RS_THREADS_BEGIN
        for (int i = tid; i < KB_SINC_NTAB; i += p.n_threads) tab[i] = p.tab[i];
        if (tid == 0) kb_bar_init(bar, 1);
    KB_RS_THREADS_END
    KB_SYNC_CTA;
    const float t_end = (float)(KB_SINC_Z * KB_SINC_Q);
    unsigned par = 0;
    for (int tile = cta; tile < p.n_tiles; tile += n_cta) {
        const KbSincTile t = kb_sinc_tile(p, tile);
        // phase 1: stage the span
        KB_RS_THREADS_BEGIN
            if (t.bulk) {
                if (tid == 0) kb_bulk_g2s(buf, t.src, t.bytes, bar);
            } else {
                const float* xs = p.x + (long long)t.b * p.x_sb + (long long)t.g * p.G * p.x_sc;
                for (int e = tid; e < t.count; e += p.n_threads) {
                    int i = e, c = 0;
                    if (p.G > 1) { i = e / p.G; c = e - i * p.G; }
                    const long long si = t.i0 + i;
                    buf[e] = (si >= 0 && si < p.L) ? xs[si * p.x_sl + (long long)c * p.x_sc] : 0.0f;
                }
            }
        KB_RS_THREADS_END
        KB_SYNC_CTA;
        // phase 2: the outputs
        KB_RS_THREADS_BEGIN
            if (t.bulk) kb_bar_wait(bar, par);
            const float* sp = buf + t.head;
            int j = tid / p.G;
            const int c = tid - j * p.G;
            if (j < p.S) {
                const int ch = t.g * p.G + c;
                float* yo = p.y + (long long)t.b * p.y_sb + (long long)ch * p.y_sc + (t.m0 + j) * p.y_sl;
                const long long ystep = (long long)p.S * p.y_sl;
                for (; j < t.nt; j += p.S) {
                    const double pos = kb_sinc_pos(p, t.m0 + j);
                    const double fl = floor(pos);
                    const double frac = pos - fl;
                    const float tl0 = (float)frac * p.sQ, tr0 = (float)(1.0 - frac) * p.sQ;
                    const float* xl = sp + (int)((long long)fl - t.i0) * p.G + c;      // x[n], n = floor(pos)
                    const float* xr = xl + p.G;
                    float a0 = 0.0f, a1 = 0.0f;
                    for (int i = 0; i < p.nw; ++i) {
                        const float fi = (float)i;
                        const float tl = fminf(fmaf(fi, p.sQ, tl0), t_end);
                        const float tr = fminf(fmaf(fi, p.sQ, tr0), t_end);
                        const int kl = (int)tl, kr = (int)tr;
                        const float2 el = tab[kl], er = tab[kr];
                        a0 = fmaf(fmaf(tl - (float)kl, el.y, el.x), xl[-i * p.G], a0);
                        a1 = fmaf(fmaf(tr - (float)kr, er.y, er.x), xr[i * p.G], a1);
                    }
                    *yo = (a0 + a1) * p.scale;
                    yo += ystep;
                }
            }
            kb_rs_fence_proxy_async();
        KB_RS_THREADS_END
        if (t.bulk) par ^= 1u;
        KB_SYNC_CTA;
    }
}
