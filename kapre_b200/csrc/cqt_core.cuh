// Kernel bodies of the multirate constant-Q transform and its adjoint.
//
// Octave i (0 = top) reads pyramid level y_i (y_0 = x, y_{i+1} = resample_poly(y_i, 1, 2), made by the resampling
// kernel) with hop h_i = h / 2^i.  Its bins share one tap table of N_i = (longest filter) taps per bin, centred on
// j = N_i / 2 and zero outside each bin's own filter, with the scale and the conjugate folded in (float64 on the host,
// rounded once to float32):
//   C[k, m] = sum_{j < N_i} y_i[m h_i + j - N_i / 2] T_k[j],    y_i = 0 outside [0, L_i)
// Every output is one float32 dot product with j ascending (re and im accumulated separately with fmaf), whatever
// the tile, the thread, the batch, the strides or the grid, so its bits depend on (item, channel, octave, frame,
// bin) alone.  The adjoint's recomputation of C (magnitude mode) runs the same sequence and gets the same bits.
//
// Forward job = (segment, item-channel, tile of TF frames), segment = (octave, group of bins whose table fits the
// table budget).  The job stages the group's table ([j][bin], two bins per float4) when it changes and the span
// [t0 h - N/2, (t0 + TF - 1) h + N - N/2) of samples, zero-filled outside the level, with coalesced loads.  Thread
// = (bin pair, frame slot): it accumulates 2 bins x FR frames (frames slot + NSu r) in registers, so per tap it
// loads one float4 of taps and FR samples for 4 FR multiply-adds.  FR (1, 2 or 4) and the slots in use NSu are sized
// from the segment's frames per tile TF, so that where the span budget caps TF (the top octaves) threads do not
// compute frames past the tile and throw them away.  The lanes of a warp
// read the same taps (broadcast) and samples of up to 32 / NP + 1 frames that lie h apart; when h is even the staged
// span gets one skew word every h samples (frame stride h + 1, odd), so those reads hit distinct banks whatever h is.
//
// Adjoint job = (item-channel, tile of TS samples) of one octave (one launch per octave):
//   g_i[t] = sum_groups sum_m sum_k (T_k[j].re G[k, m].re + T_k[j].im G[k, m].im) + add[t],   j = t - m h + N / 2
// with G the complex output gradient, or in magnitude mode G = g C / |C| (0 where |C| = 0) from C recomputed here.
// Lane = sample; it reads the [bin][j] table at consecutive j (conflict-free) and G rows that are the same for most
// lanes (broadcast).  `add` is the resampling adjoint of g_{i+1}, so the chain needs no separate add.
//
// Like the other bodies, these are written as barrier-free phases: under nvcc each phase runs once per thread and the
// phases are separated by CTA barriers; the CPU emulation (tests/emu, KB_HOST_EMU) runs each phase as a loop over the
// CTA's threads.
#pragma once
#include <vector>
#include "stft_core.cuh"

#define KB_CQT_THREADS 128
#define KB_CQT_FR 4                       // most frames per thread
#define KB_CQT_MAX_OCT 12                 // KAPRE_CQT_MAX_OCTAVES
#define KB_CQT_MAX_TAPS 2048              // KAPRE_CQT_MAX_TAPS: a bin pair's row of taps fits the table budget
#define KB_CQT_MAX_SEGS 256
#define KB_CQT_TAB_BYTES (32 * 1024)      // staged taps of one bin group
#define KB_CQT_SPAN_FLOATS (8 * 1024)     // staged samples of one tile (skew words included)
#define KB_CQT_BWD_THREADS 256
#define KB_CQT_BWD_SR 4                   // samples per adjoint thread
#define KB_CQT_GC_BYTES (32 * 1024)       // staged output gradient of one adjoint tile and bin group

struct KbCqtSeg {
    int oct, k0, nk, nkp;                 // octave, first bin of the group (within the octave), bins, bins rounded to even
    int NP, NS, TF;                       // bin pairs, frame slots, frames per tile
    int FR, NSu;                          // frames per thread (1, 2 or 4), slots in use: NSu FR >= TF
    int n_tiles;                          // ceil(M / TF) (per call)
    long long tab_off;                    // float2 offset of the group's [j][nkp] table
    long long job0;                       // first job of the segment (per call)
};

struct KbCqtOct {
    int L, h, N, half, pad;               // level length, hop, taps per bin, N / 2, skew (1 when h is even)
    int k0, nk;                           // first output bin and bins of the octave
    int bgk, n_bgroups, TS;               // adjoint: bins per group, groups, samples per tile
    long long btab_off;                   // float2 offset of the octave's [bin][j] table
    const float* y;                       // level samples, element strides (batch, channel, sample)
    long long y_sb, y_sc, y_sl;
};

struct KbCqtParams {
    int B, C, M, n_bins, n_oct, n_threads;
    KbCqtOct oct[KB_CQT_MAX_OCT];
    const float2* tab;                    // forward tables (device)
    const float2* btab;                   // adjoint tables (device)
    int mag;                              // 1: |C| (float32), 0: C (complex64)
    // forward
    int n_segs;
    long long jobs;
    void* out;                            // element strides (batch, channel, frame, bin)
    long long o_sb, o_sc, o_st, o_sk;
    KbCqtSeg seg[KB_CQT_MAX_SEGS];
    // adjoint of octave bo
    int bo;
    const void* g;                        // output gradient: complex64, or float32 in magnitude mode
    long long g_sb, g_sc, g_st, g_sk;
    const float* add;                     // addend (level bo, contiguous (B, C, L)), or null
    float* gy;                            // result, element strides (batch, channel, sample)
    long long gy_sb, gy_sc, gy_sl;
};

// ---- host side: geometry shared by the library and the CPU emulation ----
KB_HD int kb_cqt_staged(int span, int h, int pad) { return span + pad * ((span - 1) / h) + 1; }

// Bins per forward group: the table budget's worth (even), at most the octave's bins and 2 KB_CQT_THREADS.
inline int kb_cqt_fwd_group(int N, int nk) {
    int gk = (KB_CQT_TAB_BYTES / (8 * N)) & ~1;
    const int nk_even = (nk + 1) & ~1;
    if (gk > nk_even) gk = nk_even;
    if (gk > 2 * KB_CQT_THREADS) gk = 2 * KB_CQT_THREADS;
    return gk;
}

// Frames per tile of a segment: the most that fit the span budget, at most NS x KB_CQT_FR.
inline int kb_cqt_pick_tf(int NS, int h, int N, int pad) {
    int tf = NS * KB_CQT_FR;
    while (tf > 1 && kb_cqt_staged((tf - 1) * h + N, h, pad) > KB_CQT_SPAN_FLOATS) --tf;
    return tf;
}

// Samples per adjoint tile: as many as the threads cover, fewer when the staged gradient rows or (magnitude mode)
// samples would not fit.  0: not even one sample fits (kb_cqt_build then takes fewer bins per group; with one bin
// every h >= 1 and N <= KB_CQT_MAX_TAPS fits, which tests/test_cqt_emu.py checks exhaustively).
inline int kb_cqt_pick_ts(int h, int N, int bgk, int pad) {
    for (int ts = KB_CQT_BWD_THREADS * KB_CQT_BWD_SR; ts >= 1; ts /= 2) {
        const int nfr = (ts + N - 2) / h + 1;      // frames m with u0 + N/2 - N < m h <= u0 + ts - 1 + N/2
        if ((long long)nfr * bgk * 8 <= KB_CQT_GC_BYTES && kb_cqt_staged((nfr - 1) * h + N, h, pad) <= KB_CQT_SPAN_FLOATS)
            return ts;
    }
    return 0;
}

// Octave geometry and both tables from the per-octave [bin][N_i] complex tables (float pairs, top octave first).
// Returns 0, or 1 + the octave that does not fit: a filter over KB_CQT_MAX_TAPS, or more than KB_CQT_MAX_SEGS
// (octave, bin group) segments in all (kapre_b200.backend.cqt_geometry checks both first).
inline int kb_cqt_build(int n_bins, int bpo, int hop, const int* taps, const float* tab_host, KbCqtParams& p,
                        std::vector<float2>& tab, std::vector<float2>& btab) {
    p.n_bins = n_bins;
    p.n_oct = (n_bins + bpo - 1) / bpo;
    tab.clear(); btab.clear();
    p.n_segs = 0;
    long long src = 0;
    for (int i = 0; i < p.n_oct; ++i) {
        KbCqtOct& o = p.oct[i];
        const int k1 = n_bins - i * bpo, k0 = k1 - bpo > 0 ? k1 - bpo : 0;
        o.k0 = k0; o.nk = k1 - k0;
        o.h = hop >> i; o.N = taps[i]; o.half = o.N / 2; o.pad = (o.h & 1) ? 0 : 1;
        if (o.N < 1 || o.N > KB_CQT_MAX_TAPS) return i + 1;
        const float2* T = reinterpret_cast<const float2*>(tab_host) + src;
        // adjoint table: the octave's rows as given
        o.btab_off = (long long)btab.size();
        btab.insert(btab.end(), T, T + (size_t)o.nk * o.N);
        // adjoint bin groups: the table budget's worth, fewer while a sample tile's gradient rows do not fit
        o.bgk = KB_CQT_TAB_BYTES / (8 * o.N);
        if (o.bgk > o.nk) o.bgk = o.nk;
        while ((o.TS = kb_cqt_pick_ts(o.h, o.N, o.bgk, o.pad)) == 0 && o.bgk > 1) --o.bgk;
        if (o.TS == 0) return i + 1;
        o.n_bgroups = (o.nk + o.bgk - 1) / o.bgk;
        // forward tables: groups of an even number of bins, [j][nkp], at most one bin pair per thread
        const int gk = kb_cqt_fwd_group(o.N, o.nk);
        for (int g0 = 0; g0 < o.nk; g0 += gk) {
            if (p.n_segs == KB_CQT_MAX_SEGS) return i + 1;
            KbCqtSeg& s = p.seg[p.n_segs++];
            s.oct = i; s.k0 = g0; s.nk = o.nk - g0 < gk ? o.nk - g0 : gk; s.nkp = (s.nk + 1) & ~1;
            s.NP = s.nkp / 2;
            s.NS = KB_CQT_THREADS / s.NP;
            s.TF = kb_cqt_pick_tf(s.NS, o.h, o.N, o.pad);
            s.FR = s.NS >= s.TF ? 1 : 2 * s.NS >= s.TF ? 2 : 4;
            s.NSu = (s.TF + s.FR - 1) / s.FR;
            s.tab_off = (long long)tab.size();
            tab.resize(tab.size() + (size_t)o.N * s.nkp, make_float2(0.0f, 0.0f));
            for (int j = 0; j < o.N; ++j)
                for (int kk = 0; kk < s.nk; ++kk)
                    tab[(size_t)s.tab_off + (size_t)j * s.nkp + kk] = T[(size_t)(g0 + kk) * o.N + j];
        }
        src += (long long)o.nk * o.N;
    }
    return 0;
}

// Per-call tiling of the forward; false when the job count overflows.
inline bool kb_cqt_setup(KbCqtParams& p) {
    long long job = 0;
    const long long bc = (long long)p.B * p.C;
    for (int s = 0; s < p.n_segs; ++s) {
        KbCqtSeg& sg = p.seg[s];
        sg.n_tiles = (p.M + sg.TF - 1) / sg.TF;
        sg.job0 = job;
        job += bc * sg.n_tiles;
    }
    p.jobs = job;
    return job < (1LL << 40);
}

#if defined(KB_HOST_EMU)
#define KB_CQ_THREADS_BEGIN for (int tid = 0; tid < p.n_threads; ++tid) {
#define KB_CQ_THREADS_END }
#define KB_CQ_FN inline
#else
#define KB_CQ_THREADS_BEGIN { const int tid = threadIdx.x;
#define KB_CQ_THREADS_END }
#define KB_CQ_FN __device__ __forceinline__
#endif

KB_HD long long kb_cqt_floordiv(long long a, long long b) { return a >= 0 ? a / b : -((-a + b - 1) / b); }

// Stage samples [base, base + span) of one level row into the skewed layout (zeros outside [0, L)).
KB_CQ_FN void kb_cqt_stage(const KbCqtOct& o, const float* ys, long long base, int span, float* buf, int tid, int nt) {
    for (int e = tid; e < span; e += nt) {
        const long long n = base + e;
        buf[e + o.pad * (e / o.h)] = (n >= 0 && n < o.L) ? ys[n * o.y_sl] : 0.0f;
    }
}

// One thread's outputs: bins 2 pi and 2 pi + 1 of the group at frames slot + NSu q (q < FR) of the tile.
template <int FR>
KB_CQ_FN void kb_cqt_fwd_block(const KbCqtParams& p, const KbCqtSeg& sg, const KbCqtOct& o, const float2* tab,
                               const float* buf, int b, int c, int t0, int nt, int pi, int slot) {
    const int hs = o.h + o.pad;
    int off[FR];
    float a0r[FR], a0i[FR], a1r[FR], a1i[FR];
#pragma unroll
    for (int q = 0; q < FR; ++q) {
        const int m = slot + sg.NSu * q;
        off[q] = (m < nt ? m : nt - 1) * hs;
        a0r[q] = a0i[q] = a1r[q] = a1i[q] = 0.0f;
    }
    const kb_f4* w4 = reinterpret_cast<const kb_f4*>(tab) + pi;
    const int row = sg.NP;
    int jj = 0, ph = 0;
    for (int j = 0; j < o.N; ++j) {
        const kb_f4 w = w4[j * row];
#pragma unroll
        for (int q = 0; q < FR; ++q) {
            const float v = buf[off[q] + jj];
            a0r[q] = fmaf(v, w.x, a0r[q]);
            a0i[q] = fmaf(v, w.y, a0i[q]);
            a1r[q] = fmaf(v, w.z, a1r[q]);
            a1i[q] = fmaf(v, w.w, a1i[q]);
        }
        ++jj;
        if (++ph == o.h) { ph = 0; jj += o.pad; }
    }
    const int kk0 = sg.k0 + 2 * pi;
    const long long ob = (long long)b * p.o_sb + (long long)c * p.o_sc;
    const bool two = 2 * pi + 1 < sg.nk;
#pragma unroll
    for (int q = 0; q < FR; ++q) {
        const int m = slot + sg.NSu * q;
        if (m >= nt) continue;
        const long long e = ob + (long long)(t0 + m) * p.o_st + (long long)(o.k0 + kk0) * p.o_sk;
        if (p.mag) {
            float* y = static_cast<float*>(p.out);
            y[e] = kb_cabs<true>(a0r[q], a0i[q]);
            if (two) y[e + p.o_sk] = kb_cabs<true>(a1r[q], a1i[q]);
        } else {
            float2* y = static_cast<float2*>(p.out);
            y[e] = make_float2(a0r[q], a0i[q]);
            if (two) y[e + p.o_sk] = make_float2(a1r[q], a1i[q]);
        }
    }
}

KB_CQ_FN void kb_cqt_fwd_cta(const KbCqtParams& p, char* smem, long long cta, long long n_cta) {
    float2* tab = reinterpret_cast<float2*>(smem);
    float* buf = reinterpret_cast<float*>(smem + KB_CQT_TAB_BYTES);
    int cur = -1, s = 0;
    for (long long job = cta; job < p.jobs; job += n_cta) {
        while (s > 0 && p.seg[s].job0 > job) --s;
        while (s + 1 < p.n_segs && p.seg[s + 1].job0 <= job) ++s;
        const KbCqtSeg& sg = p.seg[s];
        const KbCqtOct& o = p.oct[sg.oct];
        const long long r = job - sg.job0;
        const long long bc = r / sg.n_tiles;
        const int tile = (int)(r - bc * sg.n_tiles);
        const int b = (int)(bc / p.C), c = (int)(bc - (long long)b * p.C);
        const int t0 = tile * sg.TF;
        const int nt = p.M - t0 < sg.TF ? p.M - t0 : sg.TF;
        const long long base = (long long)t0 * o.h - o.half;
        const int span = (nt - 1) * o.h + o.N;
        // phase 1: the group's taps (when they change) and the tile's samples
        KB_CQ_THREADS_BEGIN
            if (s != cur) {
                const float2* src = p.tab + sg.tab_off;
                for (int e = tid; e < o.N * sg.nkp; e += p.n_threads) tab[e] = src[e];
            }
            kb_cqt_stage(o, o.y + (long long)b * o.y_sb + (long long)c * o.y_sc, base, span, buf, tid, p.n_threads);
        KB_CQ_THREADS_END
        cur = s;
        KB_SYNC_CTA;
        // phase 2: 2 bins x FR frames per thread
        KB_CQ_THREADS_BEGIN
            const int pi = tid % sg.NP, slot = tid / sg.NP;
            if (slot < sg.NSu && slot < nt) {
                if (sg.FR == 1) kb_cqt_fwd_block<1>(p, sg, o, tab, buf, b, c, t0, nt, pi, slot);
                else if (sg.FR == 2) kb_cqt_fwd_block<2>(p, sg, o, tab, buf, b, c, t0, nt, pi, slot);
                else kb_cqt_fwd_block<4>(p, sg, o, tab, buf, b, c, t0, nt, pi, slot);
            }
        KB_CQ_THREADS_END
        KB_SYNC_CTA;
    }
}

// Shared memory of the adjoint: the bin group's [bin][j] taps, the tile's output-gradient rows, the staged samples.
KB_HD int kb_cqt_bwd_smem() { return KB_CQT_TAB_BYTES + KB_CQT_GC_BYTES + KB_CQT_SPAN_FLOATS * 4; }

KB_CQ_FN void kb_cqt_bwd_cta(const KbCqtParams& p, char* smem, long long cta, long long n_cta) {
    const KbCqtOct& o = p.oct[p.bo];
    float2* tab = reinterpret_cast<float2*>(smem);
    float2* gc = reinterpret_cast<float2*>(smem + KB_CQT_TAB_BYTES);
    float* buf = reinterpret_cast<float*>(smem + KB_CQT_TAB_BYTES + KB_CQT_GC_BYTES);
    const long long tiles_t = (o.L + o.TS - 1) / o.TS;
    const long long jobs = (long long)p.B * p.C * tiles_t;
    for (long long job = cta; job < jobs; job += n_cta) {
        const long long bc = job / tiles_t;
        const int tile = (int)(job - bc * tiles_t);
        const int b = (int)(bc / p.C), c = (int)(bc - (long long)b * p.C);
        const int u0 = tile * o.TS, u1 = o.L - u0 < o.TS ? o.L : u0 + o.TS;
        long long mlo = kb_cqt_floordiv((long long)u0 + o.half - o.N, o.h) + 1;
        long long mhi = ((long long)u1 - 1 + o.half) / o.h + 1;
        if (mlo < 0) mlo = 0;
        if (mhi > p.M) mhi = p.M;
        const int nfr = mhi > mlo ? (int)(mhi - mlo) : 0;
        float acc[KB_CQT_BWD_SR];
        for (int q = 0; q < KB_CQT_BWD_SR; ++q) acc[q] = 0.0f;    // per-thread state (the emulation's loop reuses it)
        // the samples of frames [mlo, mhi), for the magnitude mode's recomputation of C
        if (p.mag && nfr > 0) {
            KB_CQ_THREADS_BEGIN
                kb_cqt_stage(o, o.y + (long long)b * o.y_sb + (long long)c * o.y_sc, mlo * o.h - o.half,
                             (nfr - 1) * o.h + o.N, buf, tid, p.n_threads);
            KB_CQ_THREADS_END
        }
#if defined(KB_HOST_EMU)
        std::vector<float> acc_t((size_t)p.n_threads * KB_CQT_BWD_SR, 0.0f);
#endif
        for (int g = 0; g < (nfr > 0 ? o.n_bgroups : 0); ++g) {
            const int kg0 = g * o.bgk, nkg = o.nk - kg0 < o.bgk ? o.nk - kg0 : o.bgk;
            KB_SYNC_CTA;
            // phase 1: the group's taps and output-gradient rows
            KB_CQ_THREADS_BEGIN
                const float2* src = p.btab + o.btab_off + (long long)kg0 * o.N;
                for (int e = tid; e < nkg * o.N; e += p.n_threads) tab[e] = src[e];
                const long long gb = (long long)b * p.g_sb + (long long)c * p.g_sc;
                for (int e = tid; e < nfr * nkg; e += p.n_threads) {
                    const int f = e / nkg, kk = e - f * nkg;
                    const long long ge = gb + (mlo + f) * p.g_st + (long long)(o.k0 + kg0 + kk) * p.g_sk;
                    if (p.mag) gc[e] = make_float2(static_cast<const float*>(p.g)[ge], 0.0f);
                    else gc[e] = static_cast<const float2*>(p.g)[ge];
                }
            KB_CQ_THREADS_END
            KB_SYNC_CTA;
            // phase 2 (magnitude mode): G = g C / |C| with C recomputed exactly as the forward computes it
            if (p.mag) {
                KB_CQ_THREADS_BEGIN
                    const int hs = o.h + o.pad;
                    for (int e = tid; e < nfr * nkg; e += p.n_threads) {
                        const int f = e / nkg, kk = e - f * nkg;
                        const float2* w = tab + kk * o.N;
                        const float* sv = buf + f * hs;
                        float cr = 0.0f, ci = 0.0f;
                        int jj = 0, ph = 0;
                        for (int j = 0; j < o.N; ++j) {
                            const float v = sv[jj];
                            cr = fmaf(v, w[j].x, cr);
                            ci = fmaf(v, w[j].y, ci);
                            ++jj;
                            if (++ph == o.h) { ph = 0; jj += o.pad; }
                        }
                        const float m = kb_cabs<true>(cr, ci);
                        const float sc = m > 0.0f ? gc[e].x / m : 0.0f;
                        gc[e] = make_float2(sc * cr, sc * ci);
                    }
                KB_CQ_THREADS_END
                KB_SYNC_CTA;
            }
            // phase 3: each sample gathers the frames whose filters cover it
            KB_CQ_THREADS_BEGIN
#if defined(KB_HOST_EMU)
                for (int q = 0; q < KB_CQT_BWD_SR; ++q) acc[q] = acc_t[(size_t)tid * KB_CQT_BWD_SR + q];
#endif
                for (int q = 0; q < KB_CQT_BWD_SR; ++q) {
                    const int t = u0 + tid + q * p.n_threads;
                    if (t >= u1) continue;
                    long long a = kb_cqt_floordiv((long long)t + o.half - o.N, o.h) + 1;
                    long long z = ((long long)t + o.half) / o.h + 1;
                    if (a < mlo) a = mlo;
                    if (z > mhi) z = mhi;
                    float s = acc[q];
                    for (long long m = a; m < z; ++m) {
                        const int j = (int)(t - m * o.h + o.half);
                        const float2* gr = gc + (m - mlo) * nkg;
                        for (int kk = 0; kk < nkg; ++kk) {
                            const float2 w = tab[kk * o.N + j], gv = gr[kk];
                            s = fmaf(w.x, gv.x, s);
                            s = fmaf(w.y, gv.y, s);
                        }
                    }
                    acc[q] = s;
                }
#if defined(KB_HOST_EMU)
                for (int q = 0; q < KB_CQT_BWD_SR; ++q) acc_t[(size_t)tid * KB_CQT_BWD_SR + q] = acc[q];
#endif
            KB_CQ_THREADS_END
        }
        // phase 4: g_i = the gather + the resampling adjoint of g_{i+1}
        KB_CQ_THREADS_BEGIN
#if defined(KB_HOST_EMU)
            for (int q = 0; q < KB_CQT_BWD_SR; ++q) acc[q] = acc_t[(size_t)tid * KB_CQT_BWD_SR + q];
#endif
            for (int q = 0; q < KB_CQT_BWD_SR; ++q) {
                const int t = u0 + tid + q * p.n_threads;
                if (t >= u1) continue;
                float v = acc[q];
                if (p.add) v += p.add[((long long)b * p.C + c) * o.L + t];
                p.gy[(long long)b * p.gy_sb + (long long)c * p.gy_sc + (long long)t * p.gy_sl] = v;
            }
        KB_CQ_THREADS_END
        KB_SYNC_CTA;
    }
}
