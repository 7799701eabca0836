// Host-side builders for the constant tables the kernels read (window, twiddles, banded
// filterbank, dual window).  Pure C++ (no CUDA) so the CPU emulation harness in tests/emu
// shares them with the CUDA library.
#pragma once
#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>
#include "kb_common.h"
#include "fft_regs.cuh"

static inline int kb_q_for_nfft(int n_fft) {
    // supported fast-path sizes: n_fft = 64 * Q, Q in {4, 8, 16, 32}
    switch (n_fft) {
        case 256: return 4;
        case 512: return 8;
        case 1024: return 16;
        case 2048: return 32;
        default: return 0;
    }
}

// exp(-2 pi i q k1 / P), row stride 33 (bank-conflict padding).
// Entry [q][0] is 1 mathematically and no kernel multiplies by it in the ordinary transpose (ex[0] = v[0]); the
// paired-column variant of the fused kernel (kb_col_dftq_pair_mag) does: it holds exp(-2 pi i s q / Q), s = Q/2 + 1,
// which shifts the spectrum of column k1 = 0 cyclically by s so that lane 0's self-paired column lines up with the
// register pattern of the other lanes.
static inline void kb_make_twp(int Q, std::vector<float2>& out) {
    const int P = 32 * Q;
    out.assign((size_t)Q * 33, make_float2(1.0f, 0.0f));
    for (int q = 0; q < Q; ++q) {
        for (int k1 = 1; k1 < 32; ++k1) {
            const int r = (q * k1) % P;
            const double a = -2.0 * M_PI * (double)r / (double)P;
            out[(size_t)q * 33 + k1] = make_float2((float)std::cos(a), (float)std::sin(a));
        }
        const int r0 = ((Q / 2 + 1) * q) % Q;
        const double a0 = -2.0 * M_PI * (double)r0 / (double)Q;
        out[(size_t)q * 33] = make_float2((float)std::cos(a0), (float)std::sin(a0));
    }
}

// exp(-2 pi i k / n_fft), k = 0 .. n_fft/4 - 1
static inline void kb_make_twn(int n_fft, std::vector<float2>& out) {
    const int n = n_fft / 4;
    out.resize(n);
    for (int k = 0; k < n; ++k) {
        const double a = -2.0 * M_PI * (double)k / (double)n_fft;
        out[k] = make_float2((float)std::cos(a), (float)std::sin(a));
    }
}

// The same table for the paired-column pair step: entries k = 0 (mod 32) are only read by lane 0's self-paired
// column k1 = 0, through the code path that multiplies by -i (bins >= P/2 of the other lanes), so they hold i W^k.
static inline void kb_make_twn2(int n_fft, std::vector<float2>& out) {
    kb_make_twn(n_fft, out);
    for (size_t k = 0; k < out.size(); k += 32) out[k] = make_float2(-out[k].y, out[k].x);
}

// 0.5 * analysis window, right zero-padded (win < n_fft) or cropped (win > n_fft) to n_fft:
// tf.signal.stft's rfft(fft_length) semantics, kapre/time_frequency.py:174-182.  The 0.5 is
// the (Z[k] +- conj Z[P-k]) / 2 of the packed real FFT, folded in here (exact in binary fp).
static inline void kb_make_wh(const float* window, int win_length, int n_fft, std::vector<float>& out) {
    out.assign(n_fft, 0.0f);
    const int n = win_length < n_fft ? win_length : n_fft;
    for (int i = 0; i < n; ++i) out[i] = 0.5f * window[i];
}

// Is the analysis window a cosine-sum window a - b cos(2 pi n / n_fft) over exactly n_fft samples?
// (tf.signal.hann_window / hamming_window with win_length == n_fft, n_fft even.)  tol: the table
// passed in is float32, so 3e-7 covers its rounding.
static inline bool kb_fit_cosine_window(const float* window, int win_length, int n_fft, double* a, double* b) {
    if (win_length != n_fft || (n_fft & 1)) return false;
    const double w0 = window[0], wm = window[n_fft / 2];
    *a = 0.5 * (w0 + wm);
    *b = 0.5 * (wm - w0);
    for (int n = 0; n < n_fft; ++n) {
        const double fit = *a - *b * cos(2.0 * M_PI * (double)n / (double)n_fft);
        if (fabs(fit - (double)window[n]) > 3e-7) return false;
    }
    return true;
}

// Per-lane factors of the in-register window (KbStftParams::cwq), pre-scaled by 0.5 * b.
static inline void kb_make_cwq(int Q, int n_fft, double b, std::vector<kb_f4>& out) {
    out.resize(Q);
    for (int q = 0; q < Q; ++q) {
        const double ae = 2.0 * M_PI * (double)(2 * q) / (double)n_fft;
        const double ao = 2.0 * M_PI * (double)(2 * q + 1) / (double)n_fft;
        kb_f4 v;
        v.x = (float)(0.5 * b * cos(ae)); v.y = (float)(0.5 * b * cos(ao));
        v.z = (float)(0.5 * b * sin(ae)); v.w = (float)(0.5 * b * sin(ao));
        out[q] = v;
    }
}

// Window table of a cosine-sum window holding exactly what the in-register form of kb_col_window_dft32 computes
// (a0, then fma(cc, -cos(2 pi j / 32), .), then fma(ss, sin(2 pi j / 32), .), each rounded once like __fmaf_rn):
// frames read through the table (odd sample offset, cooperative staging, odd hop) then get the same bits as frames
// windowed in registers, so an item's output does not depend on its alignment, its place in the batch or the tile shape.
static inline void kb_make_wh_cosw(int Q, float a0, const std::vector<kb_f4>& cwq, std::vector<float>& out) {
    out.assign((size_t)64 * Q, 0.0f);
    for (int q = 0; q < Q; ++q) {
        const float cc[2] = {cwq[q].x, cwq[q].y}, ss[2] = {cwq[q].z, cwq[q].w};
        for (int j = 0; j < 32; ++j) {
            const float cj = j <= 16 ? kb_cos32(j) : kb_cos32(32 - j);
            const float sj = j <= 16 ? kb_sin32(j) : -kb_sin32(32 - j);
            for (int e = 0; e < 2; ++e) {
                float wv = a0;
                if (cj != 0.0f) wv = std::fmaf(cc[e], -cj, wv);
                if (sj != 0.0f) wv = std::fmaf(ss[e], sj, wv);
                out[(size_t)2 * (q + Q * j) + e] = wv;
            }
        }
    }
}

// Banded form of a (n_freq x n_bands) row-major filterbank: per band the tight support
// [lo, hi) of its non-zero weights (interior zeros kept), zero-padded so that both the offset
// into the weight array and hi - lo are multiples of 4 (hi may exceed n_freq by up to 3: the
// kernels keep three zero rows behind the magnitudes).
static inline void kb_make_bands(const float* fb, int n_freq, int n_bands,
                                 std::vector<KbBand>& bands, std::vector<float>& w) {
    bands.resize(n_bands);
    w.clear();
    for (int m = 0; m < n_bands; ++m) {
        int lo = n_freq, hi = 0;
        for (int k = 0; k < n_freq; ++k)
            if (fb[(size_t)k * n_bands + m] != 0.0f) {
                if (k < lo) lo = k;
                hi = k + 1;
            }
        if (hi <= lo) { lo = 0; hi = 0; }
        const int len4 = (hi - lo + 3) & ~3;
        KbBand b;
        b.lo = lo; b.hi = lo + len4; b.off = (int)w.size(); b.pad = 0;
        for (int k = lo; k < lo + len4; ++k) w.push_back(k < hi ? fb[(size_t)k * n_bands + m] : 0.0f);
        bands[m] = b;
    }
    if (w.empty()) w.assign(4, 0.0f);
}

// Chunk-list form for the fused kernel's filterbank phase: each band becomes ceil(len/4) chunks of 4
// consecutive bins (an all-zero band still gets one zero chunk so that its output is written) and the
// bands are dealt to `groups` lane groups so that the groups' chunk counts are balanced (longest band
// first onto the least-loaded group): the phase ends with a CTA barrier, so its time is the longest
// list.  Mel bands grow with frequency -- round-robin dealing left 13 chunks against a mean of 9.8 for
// the 128-band / 513-bin bank.
static inline void kb_make_fb_chunks(const float* fb, int n_freq, int n_bands, int groups,
                                     std::vector<kb_f4>& cw, std::vector<kb_i2>& cm, std::vector<int>& cg) {
    std::vector<int> lo_of(n_bands), hi_of(n_bands), cnt(n_bands), order(n_bands);
    for (int m = 0; m < n_bands; ++m) {
        int lo = n_freq, hi = 0;
        for (int k = 0; k < n_freq; ++k)
            if (fb[(size_t)k * n_bands + m] != 0.0f) {
                if (k < lo) lo = k;
                hi = k + 1;
            }
        if (hi <= lo) { lo = 0; hi = 1; }
        lo &= ~1;   // chunks start on even bins: the kernel loads bin pairs as aligned vectors
        lo_of[m] = lo; hi_of[m] = hi; cnt[m] = (hi - lo + 3) / 4; order[m] = m;
    }
    std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return cnt[a] > cnt[b]; });
    std::vector<int> load(groups, 0);
    std::vector<std::vector<int>> members(groups);
    for (int idx = 0; idx < n_bands; ++idx) {
        const int m = order[idx];
        int best = 0;
        for (int g = 1; g < groups; ++g) if (load[g] < load[best]) best = g;
        load[best] += cnt[m];
        members[best].push_back(m);
    }
    cw.clear(); cm.clear(); cg.assign(groups + 1, 0);
    for (int g = 0; g < groups; ++g) {
        cg[g] = (int)cw.size();
        std::sort(members[g].begin(), members[g].end());
        for (int m : members[g]) {
            const int lo = lo_of[m], hi = hi_of[m];
            for (int k0 = lo; k0 < hi; k0 += 4) {
                kb_f4 w;
                float* wp = &w.x;
                for (int j = 0; j < 4; ++j) {
                    const int k = k0 + j;
                    wp[j] = (k < hi && k < n_freq) ? fb[(size_t)k * n_bands + m] : 0.0f;   // zero outside the band
                }
                kb_i2 mt;
                mt.x = k0;
                mt.y = (k0 + 4 >= hi) ? m : -1;
                cw.push_back(w);
                cm.push_back(mt);
            }
        }
    }
    cg[groups] = (int)cw.size();
}

// Band descriptors for the two-level form of the same chunk lists (the chunks of a band are consecutive in cw): group g
// owns descriptors [bg[g], bg[g+1]); descriptor = (first bin | chunks << 16, band | first chunk << 16).  The fused kernel's
// filterbank phase then runs an inner loop without the per-chunk "last chunk of the band?" test.
static inline void kb_make_fb_band_desc(const std::vector<kb_i2>& cm, const std::vector<int>& cg, int groups,
                                        std::vector<kb_i2>& bd, std::vector<int>& bg) {
    bd.clear(); bg.assign(groups + 1, 0);
    for (int g = 0; g < groups; ++g) {
        bg[g] = (int)bd.size();
        int first = cg[g];
        for (int i = cg[g]; i < cg[g + 1]; ++i) {
            if (cm[i].y >= 0) {                       // last chunk of a band
                kb_i2 d;
                d.x = cm[first].x | ((i - first + 1) << 16);
                d.y = cm[i].y | (first << 16);
                bd.push_back(d);
                first = i + 1;
            }
        }
    }
    bg[groups] = (int)bd.size();
}

// Tensor-core form of the filterbank for the fused kernel (mma.sync m16n8k8, 3xTF32 split): the
// (frames x bins) . (bins x bands) product is tiled into 8-band column tiles; tile j only needs the
// k-steps (8 bins each) its bands' supports touch (block-banded GEMM: ~17 % of the dense tile grid for a
// 128-band Slaney mel bank).  A job = one column tile and a run of consecutive k-steps; a tile with
// many k-steps is cut into two jobs so that the 16 job slots (dealt longest-first) stay balanced --
// both halves then add their partial sums into the zeroed output tile (two addends: order-independent).
//   mw[step*32 + lane] = B fragment of the step for that lane, pre-split: (b0_hi, b1_hi, b0_lo, b1_lo)
//                        b0 = fb[k0 + t][8j + g], b1 = fb[k0 + t + 4][8j + g], g = lane / 4, t = lane % 4
//   ms[step] = (k0, j if this is the job's last step else -1);  slot s owns steps [mg[s], mg[s+1])
#define KB_MMA_SLOTS 16
static inline float kb_tf32_hi(float v) {
    uint32_t u;
    std::memcpy(&u, &v, 4);
    u &= 0xffffe000u;
    float r;
    std::memcpy(&r, &u, 4);
    return r;
}
// nearest TF32 value (ties away from zero, like cvt.rna.tf32.f32); v - kb_tf32_rn(v) is exact in fp32
static inline float kb_tf32_rn(float v) {
    uint32_t u;
    std::memcpy(&u, &v, 4);
    u = (u + 0x1000u) & 0xffffe000u;
    float r;
    std::memcpy(&r, &u, 4);
    return r;
}
static inline void kb_make_fb_mma(const float* fb, int n_freq, int n_bands, std::vector<kb_f4>& mw,
                                  std::vector<kb_i2>& ms, std::vector<int>& mg) {
    struct Job { int j, s0, s1; };   // column tile, k-steps [s0, s1)
    const int n_tiles = (n_bands + 7) / 8;
    std::vector<Job> jobs;
    int total = 0;
    std::vector<Job> whole;
    for (int j = 0; j < n_tiles; ++j) {
        int lo = n_freq, hi = 0;
        for (int k = 0; k < n_freq; ++k)
            for (int m = 8 * j; m < 8 * j + 8 && m < n_bands; ++m)
                if (fb[(size_t)k * n_bands + m] != 0.0f) {
                    if (k < lo) lo = k;
                    hi = k + 1;
                }
        if (hi <= lo) { lo = 0; hi = 1; }   // all-zero tile: one step so that its outputs are written
        Job w{j, lo / 8, (hi + 7) / 8};
        whole.push_back(w);
        total += w.s1 - w.s0;
    }
    const int target = (total + KB_MMA_SLOTS - 1) / KB_MMA_SLOTS;
    for (const Job& w : whole) {
        const int n = w.s1 - w.s0;
        if (n > target && n >= 2) {
            const int mid = w.s0 + (n + 1) / 2;
            jobs.push_back(Job{w.j, w.s0, mid});
            jobs.push_back(Job{w.j, mid, w.s1});
        } else {
            jobs.push_back(w);
        }
    }
    std::stable_sort(jobs.begin(), jobs.end(), [](const Job& a, const Job& b) { return (a.s1 - a.s0) > (b.s1 - b.s0); });
    std::vector<int> load(KB_MMA_SLOTS, 0);
    std::vector<std::vector<Job>> members(KB_MMA_SLOTS);
    for (const Job& jb : jobs) {
        int best = 0;
        for (int s = 1; s < KB_MMA_SLOTS; ++s) if (load[s] < load[best]) best = s;
        load[best] += jb.s1 - jb.s0;
        members[best].push_back(jb);
    }
    // A warp of an NW-warp CTA walks slots w, w + NW, ...: place the slots so that position i (heavy,
    // descending) pairs with position i + 8 (light, ascending).
    std::vector<int> order(KB_MMA_SLOTS);
    for (int s = 0; s < KB_MMA_SLOTS; ++s) order[s] = s;
    std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return load[a] > load[b]; });
    std::vector<int> place(KB_MMA_SLOTS);
    for (int i = 0; i < KB_MMA_SLOTS / 2; ++i) {
        place[i] = order[i];
        place[KB_MMA_SLOTS / 2 + i] = order[KB_MMA_SLOTS - 1 - i];
    }
    mw.clear(); ms.clear(); mg.assign(KB_MMA_SLOTS + 1, 0);
    for (int pos = 0; pos < KB_MMA_SLOTS; ++pos) {
        mg[pos] = (int)ms.size();
        for (const Job& jb : members[place[pos]]) {
            for (int s = jb.s0; s < jb.s1; ++s) {
                const int k0 = 8 * s;
                kb_i2 d;
                d.x = k0;
                d.y = (s == jb.s1 - 1) ? jb.j : -1;
                ms.push_back(d);
                for (int lane = 0; lane < 32; ++lane) {
                    const int g = lane >> 2, t = lane & 3;
                    const int m = 8 * jb.j + g;
                    float b[2];
                    for (int h = 0; h < 2; ++h) {
                        const int k = k0 + t + 4 * h;
                        b[h] = (k < n_freq && m < n_bands) ? fb[(size_t)k * n_bands + m] : 0.0f;
                    }
                    kb_f4 v;
                    v.x = kb_tf32_hi(b[0]); v.y = kb_tf32_hi(b[1]);
                    v.z = b[0] - v.x;       v.w = b[1] - v.y;
                    mw.push_back(v);
                }
            }
        }
    }
    mg[KB_MMA_SLOTS] = (int)ms.size();
}

// Synthesis-window table for the inverse kernel: dual[m] = w~[m] / n_fft, negated for odd m
// (x[2n+1] = -Im FFT(conj Z)[n] / N); w~ is tf.signal.inverse_stft_window_fn's window,
// kapre/time_frequency.py:278-280, truncated to the samples irfft(n_fft) actually provides.
static inline void kb_make_dual(const float* dual_window, int win, int n_fft, std::vector<float>& out) {
    out.assign(win + 2, 0.0f);
    for (int m = 0; m < win; ++m) {
        const double v = (double)dual_window[m] / (double)n_fft;
        out[m] = (float)((m & 1) ? -v : v);
    }
}
