// Kernel bodies of Kaldi-compatible features (kapre_kaldi_features: torchaudio.compliance.kaldi.fbank / mfcc /
// spectrogram over a batch of items and channels) and of their gradient to the waveform.
//
// Per (item b, channel c, frame f) with W samples per frame, shift H and padded size N = 2P in {256, 512, 1024, 2048}:
//   1. x[i] = wave[src(f H + i)] + dither d(seed, b, c, f, i), i < W  (src: identity, or torchaudio's reflection at
//      both ends of the item's own length when snip_edges is off)
//   2. x -= mean(x)                                    (remove_dc_offset)
//   3. raw_energy: e = log(max(sum x^2, eps)), then max(e, log(energy_floor)) when energy_floor != 0
//   4. x[i] -= p x[max(i - 1, 0)]                       (pre-emphasis, in descending i)
//   5. x *= window, zero-padded to N; without raw_energy the log energy is taken here
//   6. X = rfft(x); S[k] = |X[k]|^2 (use_power) or |X[k]|, k <= P
// then fbank: mel[m] = sum_k banks[m][k] S[k], log(max(mel, eps)) when use_log_fbank, energy column first or last;
// mfcc: the log mel through the DCT (lifter folded in), c0 replaced by the energy, htk_compat reordering;
// spectrogram: log(max(S, eps)) with bin 0 replaced by the log energy.
//
// The real FFT is the register FFT of stft_core.cuh: N real samples as P = 32 Q complex ones, Q lanes of a warp per
// frame and 32 / Q frames per warp (kb_col_window_dft32 -> kb_col_gather -> kb_col_dftq_store), then the pair step
// below.  The window table holds 0.5 w, which the pair step's (Z[k] +- conj Z[P-k]) doubles back (exact).
//
// Work split: one warp per job of FPW = 32 / Q consecutive frames of one (item, channel); CTAs of KB_KALDI_WARPS
// warps walk the jobs persistently, and no warp waits for another.  Frame means and energies are float64 sums in a
// fixed order (lane j takes samples j, j + 32, ... in order, then a fixed 32-lane tree), bands are summed in
// ascending bins and the DCT in ascending bands, so a frame's bits depend only on its samples and the options: not
// on the batch, the position, the strides, the data format or the grid.  No atomics anywhere.
//
// Gradient (waveform only): per frame the forward is recomputed (with the same dither), the incoming gradient goes
// back through the log floors, the DCT, the banks (a transposed band list, ascending bands per bin), power or
// magnitude, the adjoint of the zero-padded rfft (a c2r transform done as a forward FFT of the conjugated packed
// spectrum), the window, pre-emphasis (P^T), the energies and DC removal; the frame's W gradients go to a workspace,
// and a second pass gathers, for every sample, its frames' contributions in ascending (padded position, frame)
// order, reflected positions included.  Samples at or past an item's length get exactly 0.  subtract_mean adds a
// per-column pass over the valid frames in both directions (kb_kaldi_cmn_col).
//
// Under nvcc each phase runs once per lane and the phases are separated by __syncwarp(); the CPU emulation
// (tests/emu/kb_emu_kaldi.cpp, KB_HOST_EMU) runs each phase as a loop over the 32 lanes.
#pragma once
#include <vector>
#include "kb_tables.h"
#include "stft_core.cuh"

#define KB_KALDI_WARPS 4                             // warps (independent jobs) per CTA
#define KB_KALDI_MAX_MEL 256                         // mel bands: FPW x n_mel floats fit a warp's exchange region
#define KB_KALDI_EPS 1.1920928955078125e-07f         // float32 machine epsilon, torchaudio's floor
#define KB_KALDI_LOG_EPS -15.942384719848633f        // float32(log(eps)): the value wherever the floor binds

enum { KB_KALDI_FBANK = 0, KB_KALDI_MFCC = 1, KB_KALDI_SPECTROGRAM = 2 };

struct KbKaldiParams {
    const float* x; long long x_sb, x_sc, x_sl;      // waveform (forward and backward)
    const int* len;                                  // per item valid length (device), null: L
    int B, C, L;
    int W, H, N, Q;                                  // window, shift, padded size, lanes per frame
    int snip, min_len;                               // snip_edges; items shorter than min_len have no frames
    int T;                                           // frames per item in the output
    int kind, n_mel, n_ceps, K;                      // K: output columns per frame
    int use_energy, htk, raw_energy, use_power, use_log, remove_dc;
    float preemph, dither, log_floor;                // log_floor: log(energy_floor), or -inf when it is 0
    unsigned long long seed;
    const float* wh;                                 // N: 0.5 window, 0 past W
    const float* half;                               // N: 0.5 (the adjoint FFT's unwindowed input)
    const float2* twp;                               // kb_make_twp(Q)
    const float2* twn;                               // kb_make_twn(N)
    const int* mlo; const int* mlen; const int* moff; const float* mw;   // band m: bins [mlo, mlo + mlen)
    const int* klo; const int* klen; const int* kidx; const float* kw;   // bin k: bands kidx[klo .. klo + klen)
    const float* dct;                                // n_mel x n_ceps, lifter (and htk's sqrt 2) folded in
    float* y; long long y_sb, y_sc, y_st, y_sk;      // forward output (B, C, T, K) by strides
    const float* g; long long g_sb, g_sc, g_st, g_sk;   // backward: output gradient
    float* gf;                                       // backward: per-frame gradients (B C T W)
    float* gx; long long gx_sb, gx_sc, gx_sl;        // backward: waveform gradient
    long long jobs;                                  // B C ceil(T / FPW)
    int bwd;
};

KB_HD int kb_kaldi_frames(int len, int W, int H, int snip, int min_len) {
    if (len < W || len < min_len || len <= 0) return 0;
    return snip ? 1 + (len - W) / H : (len + H / 2) / H;
}

// Sample of the item (length len) at padded position j: snip_edges reads it as it is; otherwise torchaudio pads
// W / 2 - H / 2 samples on the left reflected as [2, 1, 0 | 0, 1, 2 ...] and the whole reversed item on the right.
KB_HD int kb_kaldi_src(int j, int len, int pad) {
    const int s = j - pad;
    return s < 0 ? -1 - s : (s < len ? s : 2 * len - 1 - s);
}

KB_HD int kb_kaldi_pad(int W, int H, int snip) { return snip ? 0 : W / 2 - H / 2; }

// ---- dither: Irwin-Hall sum of twelve 24-bit hashes, exact in integers ----
KB_HD unsigned long long kb_kaldi_mix(unsigned long long z) {
    z += 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}
KB_HD unsigned long long kb_kaldi_frame_key(unsigned long long seed, long long b, int c, int f) {
    unsigned long long h = kb_kaldi_mix(seed);
    h = kb_kaldi_mix(h ^ (unsigned long long)b);
    h = kb_kaldi_mix(h ^ (unsigned long long)c);
    return kb_kaldi_mix(h ^ (unsigned long long)f);
}
// A standard normal-like value with mean 0 and variance 1 - 2^-48: n = 2 S - 12 (2^24 - 1) with S the sum of twelve
// uniform 24-bit integers, returned as float(n) 2^-25 (one rounding, the same on the device and in NumPy).
KB_HD float kb_kaldi_gauss(unsigned long long key, int i) {
    int s = 0;
#pragma unroll
    for (int r = 0; r < 6; ++r) {
        const unsigned long long u = kb_kaldi_mix(key ^ (unsigned long long)(6 * i + r));
        s += (int)(u >> 40) + (int)((u >> 16) & 0xFFFFFFu);
    }
    const int n = 2 * s - 12 * 0xFFFFFF;
    return (float)n * 2.98023223876953125e-08f;      // 2^-25
}

KB_HD float kb_kaldi_mul_rn(float a, float b) {
#if defined(__CUDA_ARCH__)
    return __fmul_rn(a, b);
#else
    return a * b;
#endif
}

// log(max(v, eps)) keeping NaN; exactly float32(log(eps)) where the floor binds
KB_HD float kb_kaldi_log_floor(float v) {
    if (v != v) return v;
    return v > KB_KALDI_EPS ? logf(v) : KB_KALDI_LOG_EPS;
}

// ---- host side: the plan's tables (shared by the library and the CPU emulation) ----
struct KbKaldiTables {
    std::vector<float> wh, half, mw, kw, dct;
    std::vector<float2> twp, twn;
    std::vector<int> mlo, mlen, moff, klo, klen, kidx;
};

inline bool kb_kaldi_finite(float v) { return v == v && v - v == 0.0f; }

// 0.5 window, 0.5, twiddles, the M bands of banks ((M, N / 2 + 1) row-major) as bin runs and as per-bin band lists
// (ascending bands), and the DCT.  Returns the first non-finite input's kind (1 window, 2 banks, 3 DCT) or 0.
inline int kb_kaldi_tables(int W, int N, int M, int n_dct, const float* window, const float* banks, const float* dct,
                           KbKaldiTables& t) {
    const int P = N / 2;
    for (int i = 0; i < W; ++i)
        if (!kb_kaldi_finite(window[i])) return 1;
    kb_make_wh(window, W, N, t.wh);
    t.half.assign((size_t)N, 0.5f);
    kb_make_twp(P / 32, t.twp);
    kb_make_twn(N, t.twn);
    t.mlo.assign(M > 0 ? M : 1, 0); t.mlen.assign(M > 0 ? M : 1, 0); t.moff.assign(M > 0 ? M : 1, 0);
    t.mw.clear(); t.kw.clear(); t.kidx.clear();
    t.klo.assign(P + 1, 0); t.klen.assign(P + 1, 0);
    for (int m = 0; m < M; ++m) {
        const float* row = banks + (size_t)m * (P + 1);
        int lo = -1, hi = -1;
        for (int k = 0; k <= P; ++k) {
            if (!kb_kaldi_finite(row[k])) return 2;
            if (row[k] != 0.0f) { if (lo < 0) lo = k; hi = k + 1; }
        }
        if (lo < 0) lo = hi = 0;
        t.mlo[m] = lo; t.mlen[m] = hi - lo; t.moff[m] = (int)t.mw.size();
        for (int k = lo; k < hi; ++k) t.mw.push_back(row[k]);
    }
    for (int k = 0; k <= P; ++k) {
        t.klo[k] = (int)t.kidx.size();
        for (int m = 0; m < M; ++m)
            if (k >= t.mlo[m] && k < t.mlo[m] + t.mlen[m]) {
                t.kidx.push_back(m);
                t.kw.push_back(banks[(size_t)m * (P + 1) + k]);
            }
        t.klen[k] = (int)t.kidx.size() - t.klo[k];
    }
    t.dct.assign(dct ? dct : nullptr, dct ? dct + (size_t)n_dct : nullptr);
    for (float v : t.dct)
        if (!kb_kaldi_finite(v)) return 3;
    if (t.mw.empty()) t.mw.push_back(0.0f);
    if (t.kidx.empty()) { t.kidx.push_back(0); t.kw.push_back(0.0f); }
    if (t.dct.empty()) t.dct.push_back(0.0f);
    return 0;
}

// ---- shared memory of one warp ----
struct KbKaldiSmem {
    int fr, ex, red, st, xs, xsp, gm, total;
};
KB_HD KbKaldiSmem kb_kaldi_smem(int N, int Q, int n_mel, int bwd) {
    const int FPW = 32 / Q, P = N / 2;
    KbKaldiSmem s;
    int off = 0;
    s.fr = off; off += kb_align16(FPW * N * 4);                   // frames; then power (FPW x (P + 1)); bwd: FFT input
    s.ex = off; off += kb_align16(32 * 33 * 8);                   // FFT exchange; then mel values (FPW x n_mel)
    s.red = off; off += kb_align16(FPW * 32 * 8);                 // lane partial sums
    s.st = off; off += kb_align16(FPW * 4 * 8);                   // per frame: mean, E_raw, E_win, log energy
    s.xs = s.xsp = s.gm = off;
    if (bwd) {
        s.xs = off; off += kb_align16(FPW * N * 4);               // frames after DC removal
        s.xsp = off; off += kb_align16(FPW * (P + 1) * 8);        // spectrum X, then its gradient
        s.gm = off; off += kb_align16(FPW * (n_mel > 0 ? n_mel : 1) * 4);   // gradient of the mel values
    }
    s.total = off;
    return s;
}

#if defined(KB_HOST_EMU)
#define KB_KL_BEGIN for (int lane = 0; lane < 32; ++lane) {
#define KB_KL_END }
#define KB_KALDI_FN inline
#define KB_KL_REGS KbThreadRegs& R = kb_lregs[lane];
#define KB_KL_NREGS 32
#define KB_KL_ARR(T, v, n) T v##_lanes[32][n]           // a per-lane array that lives across phases
#define KB_KL_LV(v) v##_lanes[lane]
#else
#define KB_KL_BEGIN { const int lane = (int)(threadIdx.x & 31);
#define KB_KL_END }
#define KB_KALDI_FN __device__ __forceinline__
#define KB_KL_REGS KbThreadRegs& R = kb_lregs[0];
#define KB_KL_NREGS 1
#define KB_KL_ARR(T, v, n) T v[n]
#define KB_KL_LV(v) v
#endif

struct KbKaldiJob {
    long long b;
    int c, f0, len, Tb;
};

KB_HD KbKaldiJob kb_kaldi_job(const KbKaldiParams& p, long long job) {
    const int FPW = 32 / p.Q;
    const long long nfg = (p.T + FPW - 1) / FPW;
    const long long bc = job / nfg;
    KbKaldiJob j;
    j.f0 = (int)(job - bc * nfg) * FPW;
    j.b = bc / p.C;
    j.c = (int)(bc - j.b * p.C);
    int l = p.L;
    if (p.len) {
        l = p.len[j.b];
        l = l < 0 ? 0 : (l > p.L ? p.L : l);
    }
    j.len = l;
    j.Tb = kb_kaldi_frames(l, p.W, p.H, p.snip, p.min_len);
    return j;
}

// 32-lane fixed tree over red[g * 32 + lane] for every frame g of the job
KB_KALDI_FN void kb_kaldi_tree(double* red, int FPW) {
    for (int d = 16; d >= 1; d >>= 1) {
        KB_KL_BEGIN
            if (lane < d)
                for (int g = 0; g < FPW; ++g) red[g * 32 + lane] += red[g * 32 + lane + d];
        KB_KL_END
        KB_SYNC_WARP;
    }
}

KB_HD float kb_kaldi_log_energy(const KbKaldiParams& p, double e) {
    const float v = kb_kaldi_log_floor((float)e);
    return (v != v || v > p.log_floor) ? v : p.log_floor;
}

// Steps 1-5 for the job's frames: fr[g N + i] holds the pre-emphasised frame (0 from W to N), st[g] the mean, raw
// energy, window energy and log energy; with xs the frames after DC removal are kept too.
template <int Q>
KB_KALDI_FN void kb_kaldi_frames_in(const KbKaldiParams& p, const KbKaldiJob& j, float* fr, double* red, double* st,
                                    float* xs) {
    constexpr int FPW = 32 / Q;
    const int N = p.N, W = p.W;
    const int pad = kb_kaldi_pad(W, p.H, p.snip);
    const float* xb = p.x + j.b * p.x_sb + (long long)j.c * p.x_sc;
    KB_KL_BEGIN
        for (int g = 0; g < FPW; ++g) {
            const int f = j.f0 + g;
            float* fg = fr + g * N;
            if (f < j.Tb) {
                const unsigned long long key = kb_kaldi_frame_key(p.seed, j.b, j.c, f);
                for (int i = lane; i < N; i += 32) {
                    float v = 0.0f;
                    if (i < W) {
                        v = xb[(long long)kb_kaldi_src(f * p.H + i, j.len, pad) * p.x_sl];
                        if (p.dither != 0.0f) v += kb_kaldi_mul_rn(p.dither, kb_kaldi_gauss(key, i));
                    }
                    fg[i] = v;
                }
            } else {
                for (int i = lane; i < N; i += 32) fg[i] = 0.0f;
            }
        }
    KB_KL_END
    KB_SYNC_WARP;
    // frame means
    KB_KL_BEGIN
        for (int g = 0; g < FPW; ++g) {
            double s = 0.0;
            for (int i = lane; i < W; i += 32) s += (double)fr[g * N + i];
            red[g * 32 + lane] = s;
        }
    KB_KL_END
    KB_SYNC_WARP;
    kb_kaldi_tree(red, FPW);
    KB_KL_BEGIN
        if (lane < FPW) st[lane * 4] = p.remove_dc ? (double)(float)(red[lane * 32] / (double)W) : 0.0;
    KB_KL_END
    KB_SYNC_WARP;
    KB_KL_BEGIN
        for (int g = 0; g < FPW; ++g) {
            const float mean = (float)st[g * 4];
            double s = 0.0;
            for (int i = lane; i < W; i += 32) {
                const float v = fr[g * N + i] - mean;
                fr[g * N + i] = v;
                if (xs) xs[g * N + i] = v;
                s += (double)v * (double)v;
            }
            red[g * 32 + lane] = s;
        }
    KB_KL_END
    KB_SYNC_WARP;
    kb_kaldi_tree(red, FPW);
    KB_KL_BEGIN
        if (lane < FPW) st[lane * 4 + 1] = red[lane * 32];
    KB_KL_END
    KB_SYNC_WARP;
    // pre-emphasis, descending 32-sample chunks: every read sees the value before this step
    if (p.preemph != 0.0f) {
        for (int k0 = ((W - 1) / 32) * 32; k0 >= 0; k0 -= 32) {
            KB_KL_ARR(float, nv, FPW);
            KB_KL_BEGIN
                const int i = k0 + lane;
#pragma unroll
                for (int g = 0; g < FPW; ++g) {
                    float v = 0.0f;
                    if (i < W) {
                        const float a = fr[g * N + i], b = fr[g * N + (i > 0 ? i - 1 : 0)];
                        v = a - kb_kaldi_mul_rn(p.preemph, b);
                    }
                    KB_KL_LV(nv)[g] = v;
                }
            KB_KL_END
            KB_SYNC_WARP;
            KB_KL_BEGIN
                const int i = k0 + lane;
                if (i < W) {
#pragma unroll
                    for (int g = 0; g < FPW; ++g) fr[g * N + i] = KB_KL_LV(nv)[g];
                }
            KB_KL_END
            KB_SYNC_WARP;
        }
    }
    // window energy
    KB_KL_BEGIN
        for (int g = 0; g < FPW; ++g) {
            double s = 0.0;
            if (!p.raw_energy)
                for (int i = lane; i < W; i += 32) {
                    const float v = kb_kaldi_mul_rn(fr[g * N + i], 2.0f * p.wh[i]);
                    s += (double)v * (double)v;
                }
            red[g * 32 + lane] = s;
        }
    KB_KL_END
    KB_SYNC_WARP;
    kb_kaldi_tree(red, FPW);
    KB_KL_BEGIN
        if (lane < FPW) {
            st[lane * 4 + 2] = red[lane * 32];
            st[lane * 4 + 3] = (double)kb_kaldi_log_energy(p, p.raw_energy ? st[lane * 4 + 1] : red[lane * 32]);
        }
    KB_KL_END
    KB_SYNC_WARP;
}

// The register FFT of the job's frames (fr, times the table tw) into the exchange region, Z in natural order
// (frame g at ex + g (P + Q)).
template <int Q>
KB_KALDI_FN void kb_kaldi_fft(const KbKaldiParams& p, KbThreadRegs* kb_lregs, const float* fr, const float* tw,
                              cpx* ex, int nfr) {
    constexpr int FPW = 32 / Q, P = 32 * Q;
    KB_KL_BEGIN
        KB_KL_REGS
        const int g = lane / Q, q = lane % Q;
        if (g < nfr) kb_col_window_dft32<Q>(R, fr + g * p.N, tw, nullptr, 0.0f, reinterpret_cast<const cpx*>(p.twp), ex,
                                            g, q, 1);
    KB_KL_END
    KB_SYNC_WARP;
    KB_KL_BEGIN
        KB_KL_REGS
        const int g = lane / Q, q = lane % Q;
        if (g < nfr) kb_col_gather<Q>(R, ex, g, q);
    KB_KL_END
    KB_SYNC_WARP;
    KB_KL_BEGIN
        KB_KL_REGS
        const int g = lane / Q, q = lane % Q;
        if (g < nfr) kb_col_dftq_store<Q>(R, ex, g, q, P + Q);
    KB_KL_END
    KB_SYNC_WARP;
    (void)FPW;
}

// The real-FFT pair step: X[k] for k <= P from Z; S[k] to pw[g (P + 1) + k], and X to xsp when given.
template <int Q>
KB_KALDI_FN void kb_kaldi_pair(const KbKaldiParams& p, const cpx* ex, float* pw, cpx* xsp, int nfr) {
    constexpr int P = 32 * Q;
    const cpx* twn = reinterpret_cast<const cpx*>(p.twn);
    KB_KL_BEGIN
        for (int g = 0; g < nfr; ++g) {
            const cpx* zf = ex + g * (P + Q);
            float* pg = pw + g * (P + 1);
            for (int i = 0; i <= Q / 2; ++i) {
                int k, kk;
                cpx X1, X2;
                if (i < Q / 2) {
                    k = lane + 32 * i;
                    kk = P - k;
                    const cpx A = zf[k], Bv = zf[kk & (P - 1)];
                    const cpx E = cadd_conj(A, Bv), D = csub_conj(A, Bv);
                    const cpx T = cmul(cmake(D.im, -D.re), twn[k]);
                    X1 = cadd(E, T);
                    X2 = csub(E, T);
                    X2.im = -X2.im;
                } else {
                    if (lane != 0) continue;
                    k = P / 2;
                    kk = -1;
                    const cpx A = zf[P / 2];
                    X1 = cmake(2.0f * A.re, -2.0f * A.im);
                    X2 = X1;
                }
                const float n1 = cnorm(X1), n2 = cnorm(X2);
                pg[k] = p.use_power ? n1 : kb_cabs<true>(X1.re, X1.im);
                if (kk >= 0) pg[kk] = p.use_power ? n2 : kb_cabs<true>(X2.re, X2.im);
                if (xsp) {
                    xsp[g * (P + 1) + k] = X1;
                    if (kk >= 0) xsp[g * (P + 1) + kk] = X2;
                }
            }
        }
    KB_KL_END
    KB_SYNC_WARP;
}

// Column of output feature c (mfcc: cepstrum c; fbank: band c; the energy is c = -1)
KB_HD int kb_kaldi_col(const KbKaldiParams& p, int c) {
    if (p.kind == KB_KALDI_FBANK) {
        if (c < 0) return p.htk ? p.n_mel : 0;
        return c + (p.use_energy && !p.htk ? 1 : 0);
    }
    if (p.kind == KB_KALDI_MFCC) return p.htk ? (c == 0 ? p.n_ceps - 1 : c - 1) : c;
    return c;
}

// Mel values of the job's frames from pw into mel[g n_mel + m] (log when asked, always for mfcc)
KB_KALDI_FN void kb_kaldi_mel(const KbKaldiParams& p, const float* pw, float* mel, int nfr, bool logit) {
    const int P = p.N / 2;
    KB_KL_BEGIN
        for (int g = 0; g < nfr; ++g)
            for (int m = lane; m < p.n_mel; m += 32) {
                const float* s = pw + g * (P + 1) + p.mlo[m];
                const float* w = p.mw + p.moff[m];
                float a = 0.0f;
                for (int t = 0; t < p.mlen[m]; ++t) a = fmaf(w[t], s[t], a);
                mel[g * p.n_mel + m] = logit ? kb_kaldi_log_floor(a) : a;
            }
    KB_KL_END
    KB_SYNC_WARP;
}

// ------------------------------------------------------------------------------------------ forward
template <int Q>
KB_KALDI_FN void kb_kaldi_fwd_job(const KbKaldiParams& p, char* smem, long long job) {
    constexpr int FPW = 32 / Q, P = 32 * Q;
    const KbKaldiSmem S = kb_kaldi_smem(p.N, Q, p.n_mel, 0);
    float* fr = reinterpret_cast<float*>(smem + S.fr);
    cpx* ex = reinterpret_cast<cpx*>(smem + S.ex);
    double* red = reinterpret_cast<double*>(smem + S.red);
    double* st = reinterpret_cast<double*>(smem + S.st);
    KbThreadRegs kb_lregs[KB_KL_NREGS];
    const KbKaldiJob j = kb_kaldi_job(p, job);
    int nfr = j.Tb - j.f0;
    nfr = nfr < 0 ? 0 : (nfr > FPW ? FPW : nfr);
    if (nfr > 0) {
        kb_kaldi_frames_in<Q>(p, j, fr, red, st, nullptr);
        kb_kaldi_fft<Q>(p, kb_lregs, fr, p.wh, ex, nfr);
        kb_kaldi_pair<Q>(p, ex, fr, nullptr, nfr);     // fr is dead after the first FFT step: power goes there
        if (p.kind != KB_KALDI_SPECTROGRAM)
            kb_kaldi_mel(p, fr, reinterpret_cast<float*>(ex), nfr, p.use_log || p.kind == KB_KALDI_MFCC);
    }
    const float* mel = reinterpret_cast<const float*>(ex);
    float* yb = p.y + j.b * p.y_sb + (long long)j.c * p.y_sc;
    KB_KL_BEGIN
        for (int g = 0; g < FPW; ++g) {
            const int f = j.f0 + g;
            if (f >= p.T) break;
            float* yf = yb + (long long)f * p.y_st;
            if (g >= nfr) {
                for (int k = lane; k < p.K; k += 32) yf[(long long)k * p.y_sk] = 0.0f;
                continue;
            }
            const float le = (float)st[g * 4 + 3];
            if (p.kind == KB_KALDI_SPECTROGRAM) {
                for (int k = lane; k <= P; k += 32)
                    yf[(long long)k * p.y_sk] = k == 0 ? le : kb_kaldi_log_floor(fr[g * (P + 1) + k]);
            } else if (p.kind == KB_KALDI_FBANK) {
                for (int m = lane; m < p.n_mel; m += 32)
                    yf[(long long)kb_kaldi_col(p, m) * p.y_sk] = mel[g * p.n_mel + m];
                if (p.use_energy && lane == 0) yf[(long long)kb_kaldi_col(p, -1) * p.y_sk] = le;
            } else {
                for (int c = lane; c < p.n_ceps; c += 32) {
                    float a = 0.0f;
                    for (int m = 0; m < p.n_mel; ++m) a = fmaf(mel[g * p.n_mel + m], p.dct[m * p.n_ceps + c], a);
                    if (c == 0 && p.use_energy) a = le;
                    yf[(long long)kb_kaldi_col(p, c) * p.y_sk] = a;
                }
            }
        }
    KB_KL_END
    KB_SYNC_WARP;
}

// ------------------------------------------------------------------------------------------ backward, per frame
template <int Q>
KB_KALDI_FN void kb_kaldi_bwd_job(const KbKaldiParams& p, char* smem, long long job) {
    constexpr int P = 32 * Q, FPW = 32 / Q;
    const KbKaldiSmem S = kb_kaldi_smem(p.N, Q, p.n_mel, 1);
    float* fr = reinterpret_cast<float*>(smem + S.fr);
    cpx* ex = reinterpret_cast<cpx*>(smem + S.ex);
    double* red = reinterpret_cast<double*>(smem + S.red);
    double* st = reinterpret_cast<double*>(smem + S.st);
    float* xs = reinterpret_cast<float*>(smem + S.xs);
    cpx* xsp = reinterpret_cast<cpx*>(smem + S.xsp);
    float* gm = reinterpret_cast<float*>(smem + S.gm);
    float* mel = reinterpret_cast<float*>(ex);
    KbThreadRegs kb_lregs[KB_KL_NREGS];
    const KbKaldiJob j = kb_kaldi_job(p, job);
    int nfr = j.Tb - j.f0;
    nfr = nfr < 0 ? 0 : (nfr > FPW ? FPW : nfr);
    if (nfr <= 0) return;
    const int N = p.N, W = p.W;
    kb_kaldi_frames_in<Q>(p, j, fr, red, st, xs);
    kb_kaldi_fft<Q>(p, kb_lregs, fr, p.wh, ex, nfr);
    kb_kaldi_pair<Q>(p, ex, fr, xsp, nfr);
    const bool has_mel = p.kind != KB_KALDI_SPECTROGRAM;
    const bool logm = p.use_log || p.kind == KB_KALDI_MFCC;
    if (has_mel) kb_kaldi_mel(p, fr, mel, nfr, false);
    const float* gb = p.g + j.b * p.g_sb + (long long)j.c * p.g_sc;
    // gradient of the log energy (st[g 4]) and of the mel values (gm)
    KB_KL_BEGIN
        for (int g = 0; g < nfr; ++g) {
            const float* gf = gb + (long long)(j.f0 + g) * p.g_st;
            if (lane == 0) {
                float ge = 0.0f;
                if (p.kind == KB_KALDI_SPECTROGRAM) ge = gf[0];
                else if (p.use_energy) ge = gf[(long long)kb_kaldi_col(p, p.kind == KB_KALDI_FBANK ? -1 : 0) * p.g_sk];
                // through log(max(E, eps)) and the energy floor: zero where either binds
                const double E = p.raw_energy ? st[g * 4 + 1] : st[g * 4 + 2];
                const float le = (float)st[g * 4 + 3];
                const bool live = (float)E > KB_KALDI_EPS && le > p.log_floor;
                st[g * 4] = live ? (double)ge / E : 0.0;
            }
            if (has_mel)
                for (int m = lane; m < p.n_mel; m += 32) {
                    float gl;
                    if (p.kind == KB_KALDI_FBANK) {
                        gl = gf[(long long)kb_kaldi_col(p, m) * p.g_sk];
                    } else {
                        gl = 0.0f;
                        for (int c = p.use_energy ? 1 : 0; c < p.n_ceps; ++c)
                            gl = fmaf(p.dct[m * p.n_ceps + c], gf[(long long)kb_kaldi_col(p, c) * p.g_sk], gl);
                    }
                    const float v = mel[g * p.n_mel + m];
                    gm[g * p.n_mel + m] = logm ? (v > KB_KALDI_EPS || v != v ? gl / v : 0.0f) : gl;
                }
        }
    KB_KL_END
    KB_SYNC_WARP;
    // gradient of the spectrum X[k], in place of X
    KB_KL_BEGIN
        for (int g = 0; g < nfr; ++g) {
            const float* gf = gb + (long long)(j.f0 + g) * p.g_st;
            for (int k = lane; k <= P; k += 32) {
                const float s = fr[g * (P + 1) + k];
                float gs = 0.0f;
                if (p.kind == KB_KALDI_SPECTROGRAM) {
                    if (k > 0 && (s > KB_KALDI_EPS || s != s)) gs = gf[(long long)k * p.g_sk] / s;
                } else {
                    for (int t = 0; t < p.klen[k]; ++t)
                        gs = fmaf(p.kw[p.klo[k] + t], gm[g * p.n_mel + p.kidx[p.klo[k] + t]], gs);
                }
                const cpx X = xsp[g * (P + 1) + k];
                float sc;
                if (p.use_power || p.kind == KB_KALDI_SPECTROGRAM) sc = 2.0f * gs;
                else sc = s > 0.0f ? gs / s : 0.0f;
                xsp[g * (P + 1) + k] = cmake(sc * X.re, sc * X.im);
            }
        }
    KB_KL_END
    KB_SYNC_WARP;
    // The windowed frame's gradient is Re(sum_{k <= P} gX[k] e^{+2 pi i k n / N}): the c2r transform of the Hermitian
    // H (H[0] = Re gX[0], H[P] = Re gX[P], H[k] = gX[k] / 2).  With z[m] = g[2m] + i g[2m + 1],
    // z = IDFT_P(Z2), Z2[m] = (H[m] + conj H[P - m]) + i (H[m] - conj H[P - m]) W_N^-m, and IDFT_P(Z2) =
    // conj(DFT_P(conj Z2)): conj Z2 goes through the forward FFT (the input table is 0.5, so it is halved: the 1/2 of
    // H's interior is taken there and H[0], H[P] enter doubled).
    const cpx* twn = reinterpret_cast<const cpx*>(p.twn);
    KB_KL_BEGIN
        for (int g = 0; g < nfr; ++g) {
            const cpx* gX = xsp + g * (P + 1);
            cpx* c = reinterpret_cast<cpx*>(fr + g * N);
            for (int m = lane; m <= P / 2; m += 32) {
                // 2 H[k]: 2 Re gX at k = 0 and P, gX elsewhere
                const int mm = P - m;
                cpx Hm = gX[m], Hmm = gX[mm];
                if (m == 0) { Hm = cmake(2.0f * Hm.re, 0.0f); Hmm = cmake(2.0f * Hmm.re, 0.0f); }
                // W_N^-m = conj(twn[m]) for m < P/2; W_N^-(P/2) = i; W_N^-(P-m) = -W_N^m
                const cpx E = cadd_conj(Hm, Hmm), D = csub_conj(Hm, Hmm);            // H[m] +- conj H[P-m]
                cpx wm;
                if (m < P / 2) wm = cmake(twn[m].re, -twn[m].im); else wm = cmake(0.0f, 1.0f);
                const cpx iD = cmake(-D.im, D.re);
                const cpx Z2m = cadd(E, cmul(iD, wm));
                c[m] = cmake(Z2m.re, -Z2m.im);
                if (m > 0 && m < P / 2) {
                    // Z2[P - m] = (H[P-m] + conj H[m]) + i (H[P-m] - conj H[m]) (-W_N^m)
                    const cpx E2 = cadd_conj(Hmm, Hm), D2 = csub_conj(Hmm, Hm);
                    const cpx iD2 = cmake(-D2.im, D2.re);
                    const cpx wmm = cmake(-twn[m].re, -twn[m].im);
                    const cpx Z2mm = cadd(E2, cmul(iD2, wmm));
                    c[mm] = cmake(Z2mm.re, -Z2mm.im);
                }
            }
        }
    KB_KL_END
    KB_SYNC_WARP;
    kb_kaldi_fft<Q>(p, kb_lregs, fr, p.half, ex, nfr);
    // windowed-frame gradient -> pre-emphasised frame gradient (fr), with the window-energy term
    KB_KL_BEGIN
        for (int g = 0; g < nfr; ++g) {
            const cpx* r = ex + g * (P + Q);
            const float ge = p.raw_energy ? 0.0f : (float)st[g * 4];
            const float* xg = xs + g * N;
            for (int i = lane; i < N; i += 32) {
                float v = 0.0f;
                if (i < W) {
                    const cpx z = r[i >> 1];
                    float gw = (i & 1) ? -z.im : z.re;
                    const float w = 2.0f * p.wh[i];
                    if (ge != 0.0f) {
                        const float xp = p.preemph != 0.0f ? xg[i] - kb_kaldi_mul_rn(p.preemph, xg[i > 0 ? i - 1 : 0])
                                                           : xg[i];
                        gw = fmaf(2.0f * ge, xp * w, gw);
                    }
                    v = gw * w;
                }
                fr[g * N + i] = v;
            }
        }
    KB_KL_END
    KB_SYNC_WARP;
    // P^T (ascending chunks: every read sees the value before this step), the raw-energy term, the DC-removal
    // adjoint, out to the per-frame workspace
    if (p.preemph != 0.0f) {
        for (int k0 = 0; k0 < W; k0 += 32) {
            KB_KL_ARR(float, nv, FPW);
            KB_KL_BEGIN
                const int i = k0 + lane;
#pragma unroll
                for (int g = 0; g < FPW; ++g) {
                    float v = 0.0f;
                    if (g < nfr && i < W) {
                        const float a = fr[g * N + i], nx = i + 1 < W ? fr[g * N + i + 1] : 0.0f;
                        v = (i == 0 ? a - kb_kaldi_mul_rn(p.preemph, a) : a) - kb_kaldi_mul_rn(p.preemph, nx);
                    }
                    KB_KL_LV(nv)[g] = v;
                }
            KB_KL_END
            KB_SYNC_WARP;
            KB_KL_BEGIN
                const int i = k0 + lane;
                if (i < W) {
#pragma unroll
                    for (int g = 0; g < FPW; ++g)
                        if (g < nfr) fr[g * N + i] = KB_KL_LV(nv)[g];
                }
            KB_KL_END
            KB_SYNC_WARP;
        }
    }
    KB_KL_BEGIN
        for (int g = 0; g < nfr; ++g) {
            const float ge = p.raw_energy ? (float)st[g * 4] : 0.0f;
            double s = 0.0;
            for (int i = lane; i < W; i += 32) {
                float v = fr[g * N + i];
                if (ge != 0.0f) v = fmaf(2.0f * ge, xs[g * N + i], v);
                fr[g * N + i] = v;
                s += (double)v;
            }
            red[g * 32 + lane] = s;
        }
    KB_KL_END
    KB_SYNC_WARP;
    kb_kaldi_tree(red, FPW);
    KB_KL_BEGIN
        for (int g = 0; g < nfr; ++g) {
            const float mean = p.remove_dc ? (float)(red[g * 32] / (double)W) : 0.0f;
            float* o = p.gf + (((j.b * p.C + j.c) * (long long)p.T) + j.f0 + g) * W;
            for (int i = lane; i < W; i += 32) o[i] = fr[g * N + i] - mean;
        }
    KB_KL_END
    KB_SYNC_WARP;
}

// ------------------------------------------------------------------------------------------ backward, gather
// a + the contributions of the frames (ascending) that cover padded position jp
KB_HD float kb_kaldi_gather_pos(const KbKaldiParams& p, const float* gfc, int jp, int Tb, float a) {
    if (jp < 0) return a;
    const int flo = jp - p.W + 1 <= 0 ? 0 : (jp - p.W + p.H) / p.H;
    int fhi = jp / p.H;
    if (fhi > Tb - 1) fhi = Tb - 1;
    for (int f = flo; f <= fhi; ++f) a += gfc[(long long)f * p.W + (jp - f * p.H)];
    return a;
}

// gx[b, c, s]: the frames' gradients at every padded position that reads sample s, in ascending (position, frame)
// order; 0 at or past the item's length.
KB_HD void kb_kaldi_gather_elem(const KbKaldiParams& p, long long e) {
    const long long bc = e / p.L;
    const int s = (int)(e - bc * p.L);
    const long long b = bc / p.C;
    const int c = (int)(bc - b * p.C);
    int len = p.L;
    if (p.len) {
        len = p.len[b];
        len = len < 0 ? 0 : (len > p.L ? p.L : len);
    }
    const int Tb = kb_kaldi_frames(len, p.W, p.H, p.snip, p.min_len);
    float a = 0.0f;
    if (s < len && Tb > 0) {
        const int pad = kb_kaldi_pad(p.W, p.H, p.snip);
        const float* gfc = p.gf + bc * (long long)p.T * p.W;
        if (!p.snip && s < pad) a = kb_kaldi_gather_pos(p, gfc, pad - 1 - s, Tb, a);
        a = kb_kaldi_gather_pos(p, gfc, s + pad, Tb, a);
        if (!p.snip) a = kb_kaldi_gather_pos(p, gfc, pad + 2 * len - 1 - s, Tb, a);
    }
    p.gx[b * p.gx_sb + (long long)c * p.gx_sc + (long long)s * p.gx_sl] = a;
}

// ------------------------------------------------------------------------------------------ subtract_mean
// Column (b, c, k): out = in - mean over the item's valid frames (float64, ascending frames); 0 past them.
KB_HD void kb_kaldi_cmn_col(const KbKaldiParams& p, const float* in, long long i_sb, long long i_sc, long long i_st,
                            long long i_sk, float* out, long long o_sb, long long o_sc, long long o_st, long long o_sk,
                            long long e) {
    const long long bc = e / p.K;
    const int k = (int)(e - bc * p.K);
    const long long b = bc / p.C;
    const int c = (int)(bc - b * p.C);
    int len = p.L;
    if (p.len) {
        len = p.len[b];
        len = len < 0 ? 0 : (len > p.L ? p.L : len);
    }
    const int Tb = kb_kaldi_frames(len, p.W, p.H, p.snip, p.min_len);
    const float* ic = in + b * i_sb + (long long)c * i_sc + (long long)k * i_sk;
    float* oc = out + b * o_sb + (long long)c * o_sc + (long long)k * o_sk;
    double s = 0.0;
    for (int t = 0; t < Tb; ++t) s += (double)ic[(long long)t * i_st];
    const float mean = Tb > 0 ? (float)(s / (double)Tb) : 0.0f;
    for (int t = 0; t < p.T; ++t) oc[(long long)t * o_st] = t < Tb ? ic[(long long)t * i_st] - mean : 0.0f;
}
