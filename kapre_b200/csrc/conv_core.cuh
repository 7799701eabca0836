// Kernel body of the per-bin spectral multiply-accumulate of the partitioned convolution (kapre_convolve): complex64
// sequences along the frame axis, one per (item, channel, bin), in two modes
//
//   convolve:  out[i] = sum_{s < S} a[s] b[i - s]
//   correlate: out[i] = sum_{s < S} conj(a[s]) b[i + s]          (terms with b's index outside [0, Tb) are dropped)
//
// The forward is convolve with a = H (the filter's P block spectra), b = X (the signal's J block spectra); the
// adjoints are correlate with a = H, b = G (gradient of the signal spectra) and with a = X, b = G (gradient of H).
//
// Every operand is a base pointer and (batch, channel, frame, bin) element strides; a batch or channel stride of 0
// broadcasts the operand (one filter for the whole batch, no copy).
//
// Order of the sum: s ascending, one fmaf per real product, each output accumulated in registers of one thread.
// Whether a term is dropped depends on (i, s) only, so an output's bits depend on nothing but its operands: not on
// the tile it falls in, the grid, the batch position, the strides or broadcasting.
//
// Data movement: a persistent CTA walks tiles of KB_CONV_FB consecutive bins (the contiguous axis of every spectrum
// the library writes, so loads and stores coalesce) x up to KB_CONV_NO consecutive outputs of one (item, channel).
// The sum runs in chunks of KB_CONV_SC terms: each chunk stages its a rows and the b rows its outputs read (zeros
// outside b) in shared memory.  Lane l of warp w owns bin l and outputs w R .. w R + R - 1 of the tile.
//
// Written as barrier-free phases like the other bodies (KB_HOST_EMU runs each phase as a loop over the threads, and
// keeps each thread's accumulators in an array).
#pragma once
#include <vector>
#include "resample_core.cuh"       // KB_RS_THREADS_BEGIN / _END

#define KB_CONV_THREADS 256
#define KB_CONV_FB 32                                   // bins per tile: one warp's lanes
#define KB_CONV_R 8                                     // outputs per thread
#define KB_CONV_NO (KB_CONV_THREADS / 32 * KB_CONV_R)   // outputs per tile (64)
#define KB_CONV_SC 32                                   // terms per staged chunk
#define KB_CONV_SPAN (KB_CONV_NO + KB_CONV_SC - 1)      // b rows a chunk can read
#define KB_CONV_SMEM ((KB_CONV_SC + KB_CONV_SPAN) * KB_CONV_FB * 8)

struct KbConvParams {
    const float2* a;                // S frames
    long long a_sb, a_sc, a_st, a_sf;
    const float2* b;                // Tb frames
    long long b_sb, b_sc, b_st, b_sf;
    float2* out;                    // To frames
    long long o_sb, o_sc, o_st, o_sf;
    int Bn, C, F;                   // items, channels, bins
    int S, Tb, To;
    int correlate;
    int n_fg, n_og, n_tiles;        // bin groups, output groups, all tiles
    int n_threads;
};

// Block size B of the partition for a filter of K taps (the STFT runs at n_fft = 2 B).  It depends on K alone, so
// that an output's bits depend on the inputs alone.  The smallest B whose P = ceil(K / B) stays <= 8 terms, else
// the largest: see DESIGN.md for the measurements behind it.
inline int kb_conv_block_size(long long K) {
    for (int b = 128; b < 1024; b *= 2)
        if ((K + b - 1) / b <= 8) return b;
    return 1024;
}

// Tiling once the operands, sizes and mode are set; false: too many tiles.
inline bool kb_conv_setup(KbConvParams& p, int n_threads) {
    p.n_fg = (p.F + KB_CONV_FB - 1) / KB_CONV_FB;
    p.n_og = (p.To + KB_CONV_NO - 1) / KB_CONV_NO;
    const long long tiles = (long long)p.Bn * p.C * p.n_og * p.n_fg;
    if (tiles > 0x7fffffffLL) return false;
    p.n_tiles = (int)tiles;
    p.n_threads = n_threads;
    return true;
}

#if defined(KB_HOST_EMU)
#define KB_CONV_ACC_DECL std::vector<float2> kb_conv_accv((size_t)p.n_threads * KB_CONV_R);
#define KB_CONV_ACC (kb_conv_accv.data() + (size_t)tid * KB_CONV_R)
#define KB_CONV_FN inline
#else
#define KB_CONV_ACC_DECL float2 kb_conv_acc[KB_CONV_R];
#define KB_CONV_ACC kb_conv_acc
#define KB_CONV_FN __device__ __forceinline__
#endif

KB_CONV_FN void kb_conv_cta(const KbConvParams& p, char* smem, int cta, int n_cta) {
    float2* as = reinterpret_cast<float2*>(smem);                  // [KB_CONV_SC][KB_CONV_FB]
    float2* bs = as + KB_CONV_SC * KB_CONV_FB;                      // [KB_CONV_SPAN][KB_CONV_FB]
    KB_CONV_ACC_DECL
    for (int tile = cta; tile < p.n_tiles; tile += n_cta) {
        int r = tile;
        const int fg = r % p.n_fg; r /= p.n_fg;
        const int og = r % p.n_og; r /= p.n_og;
        const int c = r % p.C;
        const int item = r / p.C;
        const int f0 = fg * KB_CONV_FB, o0 = og * KB_CONV_NO;
        const int nt = p.To - o0 < KB_CONV_NO ? p.To - o0 : KB_CONV_NO;
        const float2* ap = p.a + (long long)item * p.a_sb + (long long)c * p.a_sc;
        const float2* bp = p.b + (long long)item * p.b_sb + (long long)c * p.b_sc;
        KB_RS_THREADS_BEGIN
            float2* acc = KB_CONV_ACC;
#pragma unroll
            for (int k = 0; k < KB_CONV_R; ++k) acc[k] = make_float2(0.0f, 0.0f);
        KB_RS_THREADS_END
        for (int s0 = 0; s0 < p.S; s0 += KB_CONV_SC) {
            const int sc = p.S - s0 < KB_CONV_SC ? p.S - s0 : KB_CONV_SC;
            const int span = nt + sc - 1;
            // first b frame staged: convolve reads b[i - s], correlate b[i + s]
            const int kb0 = p.correlate ? o0 + s0 : o0 - s0 - (sc - 1);
            // phase 1: stage a (conjugated for correlate) and the b rows, zeros past the bins and outside b
            KB_RS_THREADS_BEGIN
                for (int e = tid; e < sc * KB_CONV_FB; e += p.n_threads) {
                    const int row = e / KB_CONV_FB, f = f0 + (e - row * KB_CONV_FB);
                    float2 v = make_float2(0.0f, 0.0f);
                    if (f < p.F) v = ap[(long long)(s0 + row) * p.a_st + (long long)f * p.a_sf];
                    if (p.correlate) v.y = -v.y;
                    as[e] = v;
                }
                for (int e = tid; e < span * KB_CONV_FB; e += p.n_threads) {
                    const int row = e / KB_CONV_FB, f = f0 + (e - row * KB_CONV_FB);
                    const int k = kb0 + row;
                    float2 v = make_float2(0.0f, 0.0f);
                    if (f < p.F && k >= 0 && k < p.Tb) v = bp[(long long)k * p.b_st + (long long)f * p.b_sf];
                    bs[e] = v;
                }
            KB_RS_THREADS_END
            KB_SYNC_CTA;
            // phase 2: the chunk's terms, s ascending, into each thread's accumulators
            KB_RS_THREADS_BEGIN
                float2* acc = KB_CONV_ACC;
                const int lane = tid & 31, io0 = (tid >> 5) * KB_CONV_R;
                for (int js = 0; js < sc; ++js) {
                    const float2 av = as[js * KB_CONV_FB + lane];
                    const int s = s0 + js;
#pragma unroll
                    for (int k = 0; k < KB_CONV_R; ++k) {
                        const int io = io0 + k;
                        const int i = o0 + io;
                        const int kk = p.correlate ? i + s : i - s;          // b's frame
                        if (io < nt && kk >= 0 && kk < p.Tb) {
                            const int row = p.correlate ? io + js : io - js + sc - 1;
                            const float2 bv = bs[row * KB_CONV_FB + lane];
                            acc[k].x = fmaf(-av.y, bv.y, fmaf(av.x, bv.x, acc[k].x));
                            acc[k].y = fmaf(av.y, bv.x, fmaf(av.x, bv.y, acc[k].y));
                        }
                    }
                }
            KB_RS_THREADS_END
            KB_SYNC_CTA;
        }
        // phase 3: store
        KB_RS_THREADS_BEGIN
            const float2* acc = KB_CONV_ACC;
            const int lane = tid & 31, io0 = (tid >> 5) * KB_CONV_R, f = f0 + lane;
            if (f < p.F) {
                float2* op = p.out + (long long)item * p.o_sb + (long long)c * p.o_sc + (long long)f * p.o_sf;
#pragma unroll
                for (int k = 0; k < KB_CONV_R; ++k)
                    if (io0 + k < nt) op[(long long)(o0 + io0 + k) * p.o_st] = acc[k];
            }
        KB_RS_THREADS_END
    }
}
