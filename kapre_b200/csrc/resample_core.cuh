// Kernel body of the polyphase resampler (scipy.signal.resample_poly with zeros outside the signal):
//   y[n] = gain * sum_i x[i] h[hl + n down - i up],   h of odd length 2 hl + 1, terms outside h dropped.
// With t = n down, phase t mod up and first input base(n) = floor(t / up) - f (f = floor(hl / up)), this is a
// K-tap dot product y[n] = sum_m w[row(n)][m] x[base(n) + m] with w[.][m] = gain h[hl + phase + (f - m) up].
//
// Table layout: row r holds the taps of the outputs n = r (mod up), so neighbouring outputs read neighbouring
// rows.  Rows are Kp floats apart, Kp = K rounded up to a multiple of 4 with Kp / 4 odd: a lane reads its taps as
// 16 B vectors and the 8 lanes of a quarter-warp, whose rows are consecutive, hit 8 distinct 16 B bank groups.
//
// Data movement: a persistent CTA walks tiles of NT consecutive outputs of one (item, channel group).  A channel
// group is one channel, or all C channels of a channel-interleaved (channels_last) waveform, whose samples then
// sit side by side in shared memory ([sample][channel]) as in memory, so loads and stores stay coalesced.  The
// tile's input span is staged with one TMA bulk copy when it lies inside the signal and is contiguous in memory,
// else by the cooperative loader (any strides, zeros outside the signal).
//
// Each thread owns one channel of the group and every S-th output of the tile (S = threads / G).  Its phase,
// table row and first input index are set once per tile and then stepped by constants, so the inner loop has no
// division and no 64-bit index arithmetic.
//
// Like the other bodies, it is written as barrier-free phases: under nvcc each phase runs once per thread and the
// phases are separated by CTA barriers; the CPU emulation (tests/emu, KB_HOST_EMU) runs each phase as a loop over
// the CTA's threads.
#pragma once
#include <vector>
#include "stft_core.cuh"

#define KB_RESAMPLE_THREADS 256
#define KB_RESAMPLE_MAX_M 1280      // max(up, down): covers every pair of the common rates from 8 to 96 kHz

struct KbResampleParams {
    const float* x;                 // input, element strides (batch, channel, sample)
    long long x_sb, x_sc, x_sl;
    long long x_numel;              // elements addressable from x (max element offset + 1)
    unsigned x_align;               // ((uintptr_t)x >> 2) & 3
    int bulk_ok;                    // a tile's span is one contiguous run of memory (G == 1: x_sl == 1; G == C: x_sc == 1, x_sl == C)
    int B, C, L;
    float* y;                       // output, element strides (batch, channel, sample)
    long long y_sb, y_sc, y_sl;
    int L_out;
    const float* tab;               // up rows of Kp taps (device)
    int up, down, f, Kp;
    int G, n_groups;                // channels per tile, channel groups per item (C / G)
    int NT, n_tiles_t, n_tiles;     // outputs per tile, tiles per (item, group), all tiles
    int S, S_r, dS_q, dS_r;         // thread's output stride, S mod up, (S down) div / mod up
    int n_threads;
};

// Shared memory: mbarrier (16 B), the table, the staged span ([sample][channel], 4 floats of slack on either side
// for the 16 B-rounded bulk copy).
KB_HD int kb_resample_span(int NT, int up, int down, int Kp) { return (int)(((long long)(NT - 1) * down) / up) + 2 + Kp; }
KB_HD int kb_resample_smem(int up, int Kp, int NT, int down, int G) {
    return 16 + kb_align16(up * Kp * 4) + kb_align16((kb_resample_span(NT, up, down, Kp) * G + 8) * 4);
}

// ---- host side: table and launch geometry (shared by the library and the CPU emulation) ----
// Taps per phase K = 2 f + 2 (the support of h seen from any phase), padded to Kp.
inline int kb_resample_kp(int up, int n_taps) {
    const int K = 2 * (((n_taps - 1) / 2) / up) + 2;
    int Kp = (K + 3) & ~3;
    if (up > 1 && ((Kp / 4) & 1) == 0) Kp += 4;     // odd 16 B row stride: the rows of a quarter-warp in distinct banks
    return Kp;
}

// Row r serves the outputs n = r (mod up), whose phase is r down mod up.
inline void kb_resample_table(int up, int down, const float* taps, int n_taps, double gain, std::vector<float>& tab) {
    const int hl = (n_taps - 1) / 2, f = hl / up, Kp = kb_resample_kp(up, n_taps);
    tab.assign((size_t)up * Kp, 0.0f);
    for (int r = 0; r < up; ++r) {
        const long long ph = ((long long)r * down) % up;
        for (int m = 0; m < Kp; ++m) {
            const long long idx = hl + ph + (long long)(f - m) * up;
            if (idx >= 0 && idx < n_taps) tab[(size_t)r * Kp + m] = (float)(gain * (double)taps[idx]);
        }
    }
}

// Tiling and stepping constants once x, y, L_out, C, up, down, f, Kp, G and NT are set; false: too many tiles.
inline bool kb_resample_setup(KbResampleParams& p, int n_threads) {
    p.n_groups = p.C / p.G;
    p.n_tiles_t = (int)((p.L_out + (long long)p.NT - 1) / p.NT);
    const long long tiles = (long long)p.B * p.n_groups * p.n_tiles_t;
    if (tiles > 0x7fffffffLL) return false;
    p.n_tiles = (int)tiles;
    p.n_threads = n_threads;
    p.S = n_threads / p.G;
    p.S_r = p.S % p.up;
    p.dS_q = (int)(((long long)p.S * p.down) / p.up);
    p.dS_r = (int)(((long long)p.S * p.down) % p.up);
    return true;
}

struct KbRsTile {
    int b, g, nt;                   // item, channel group, outputs in this tile
    long long n0, i0;               // first output, first staged input sample
    int count;                      // staged floats (samples x G)
    int bulk, head, bytes;          // bulk copy: element i0 lands at buf[head]; bytes copied from src
    const float* src;
};

KB_HD KbRsTile kb_resample_tile(const KbResampleParams& p, int tile) {
    KbRsTile t;
    const int sig = tile / p.n_tiles_t, tt = tile - sig * p.n_tiles_t;
    t.b = sig / p.n_groups;
    t.g = sig - t.b * p.n_groups;
    t.n0 = (long long)tt * p.NT;
    t.nt = (int)((long long)p.L_out - t.n0 < p.NT ? (long long)p.L_out - t.n0 : p.NT);
    t.i0 = t.n0 * p.down / p.up - p.f;
    const long long i_end = (t.n0 + t.nt - 1) * p.down / p.up - p.f + p.Kp;    // one past the last sample read
    const int span = (int)(i_end - t.i0);
    t.count = span * p.G;
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

#if defined(KB_HOST_EMU)
#define KB_RS_THREADS_BEGIN for (int tid = 0; tid < p.n_threads; ++tid) {
#define KB_RS_THREADS_END }
static inline void kb_rs_fence_proxy_async() {}
#define KB_RS_FN inline
#else
#define KB_RS_THREADS_BEGIN { const int tid = threadIdx.x;
#define KB_RS_THREADS_END }
// generic-proxy writes / reads of the staging buffer are ordered before the next tile's bulk copy into it
KB_D void kb_rs_fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
#define KB_RS_FN __device__ __forceinline__
#endif

KB_RS_FN void kb_resample_cta(const KbResampleParams& p, char* smem, int cta, int n_cta) {
    KbBar* bar = reinterpret_cast<KbBar*>(smem);
    float* tab = reinterpret_cast<float*>(smem + 16);
    float* buf = reinterpret_cast<float*>(smem + 16 + kb_align16(p.up * p.Kp * 4));
    const int n_tab = p.up * p.Kp;
    KB_RS_THREADS_BEGIN
        for (int i = tid; i < n_tab; i += p.n_threads) tab[i] = p.tab[i];
        if (tid == 0) kb_bar_init(bar, 1);
    KB_RS_THREADS_END
    KB_SYNC_CTA;
    unsigned par = 0;
    for (int tile = cta; tile < p.n_tiles; tile += n_cta) {
        const KbRsTile t = kb_resample_tile(p, tile);
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
            const float* s = buf + t.head;
            int j = tid / p.G;
            const int c = tid - j * p.G;
            if (j < p.S) {
                const long long n = t.n0 + j;
                const long long tq = n * p.down;
                int ph = (int)(tq % p.up);                      // phase of output n
                int r = (int)(n % p.up);                        // its table row
                int rel = (int)(tq / p.up - p.f - t.i0);        // its first input, relative to the span
                const int ch = t.g * p.G + c;
                float* yo = p.y + (long long)t.b * p.y_sb + (long long)ch * p.y_sc + n * p.y_sl;
                const long long ystep = (long long)p.S * p.y_sl;
                for (; j < t.nt; j += p.S) {
                    const float* xs = s + rel * p.G + c;
                    const kb_f4* w = reinterpret_cast<const kb_f4*>(tab + r * p.Kp);
                    float a0 = 0.0f, a1 = 0.0f, a2 = 0.0f, a3 = 0.0f;
                    for (int q = 0; q < p.Kp / 4; ++q) {
                        const kb_f4 wv = w[q];
                        const float* xq = xs + 4 * q * p.G;
                        a0 = fmaf(wv.x, xq[0], a0);
                        a1 = fmaf(wv.y, xq[p.G], a1);
                        a2 = fmaf(wv.z, xq[2 * p.G], a2);
                        a3 = fmaf(wv.w, xq[3 * p.G], a3);
                    }
                    *yo = (a0 + a1) + (a2 + a3);
                    yo += ystep;
                    rel += p.dS_q;
                    ph += p.dS_r;
                    if (ph >= p.up) { ph -= p.up; ++rel; }
                    r += p.S_r;
                    if (r >= p.up) r -= p.up;
                }
            }
            kb_rs_fence_proxy_async();
        KB_RS_THREADS_END
        if (t.bulk) par ^= 1u;
        KB_SYNC_CTA;
    }
}
