// CPU emulation of the Kaldi feature bodies (kapre_b200/csrc/kaldi_core.cuh; tests only, never shipped).  Compiled
// with KB_HOST_EMU: each phase of a job runs as a loop over its 32 lanes, jobs one after another in the order `order`
// gives (the result must not depend on it), and the passes in the order the library launches them.
#define KB_HOST_EMU 1
#include <cmath>
#include <cstdint>
#include <vector>
#include "../../kapre_b200/csrc/kb_tables.h"
#include "../../kapre_b200/csrc/kaldi_core.cuh"

template <int Q>
static void run_jobs(const KbKaldiParams& p, int bwd, int order) {
    const KbKaldiSmem S = kb_kaldi_smem(p.N, Q, p.n_mel, bwd);
    std::vector<kb_f4> smem(S.total / 16 + 1);
    char* sm = reinterpret_cast<char*>(smem.data());
    for (long long i = 0; i < p.jobs; ++i) {
        long long job = i;
        if (order == 1) job = p.jobs - 1 - i;
        if (order == 2) { const long long h = p.jobs / 2; job = i < h ? 2 * i + 1 : 2 * (i - h); }
        if (bwd) kb_kaldi_bwd_job<Q>(p, sm, job);
        else kb_kaldi_fwd_job<Q>(p, sm, job);
    }
}

static void run(const KbKaldiParams& p, int bwd, int order) {
    switch (p.Q) {
        case 4: run_jobs<4>(p, bwd, order); break;
        case 8: run_jobs<8>(p, bwd, order); break;
        case 16: run_jobs<16>(p, bwd, order); break;
        default: run_jobs<32>(p, bwd, order); break;
    }
}

extern "C" {

// ic: kind, W, H, N, snip, min_len, n_mel, n_ceps, use_energy, htk, raw_energy, use_power, use_log, remove_dc,
//     subtract_mean, B, C, L, T (19 ints).  fc: preemph, energy_floor, dither (3 floats).
// xs: x strides (b, c, l); ys: y (or gy) strides (b, c, t, k); gxs: gx strides (b, c, l).  len: per item or null.
// bwd = 0: y = features(x).  bwd = 1: gx = gradient at gy (y holds gy and is read).
// order: 0 ascending jobs, 1 descending, 2 a fixed permutation.
int kb_emu_kaldi(const int* ic, const float* fc, unsigned long long seed, const float* window, const float* banks,
                 const float* dct, const float* x, const long long* xs, const int* len, float* y, const long long* ys,
                 int bwd, float* gx, const long long* gxs, int order) {
    KbKaldiParams p{};
    p.kind = ic[0]; p.W = ic[1]; p.H = ic[2]; p.N = ic[3]; p.snip = ic[4]; p.min_len = ic[5];
    p.n_mel = p.kind == KB_KALDI_SPECTROGRAM ? 0 : ic[6]; p.n_ceps = ic[7];
    p.use_energy = ic[8]; p.htk = ic[9]; p.raw_energy = ic[10]; p.use_power = ic[11]; p.use_log = ic[12];
    p.remove_dc = ic[13];
    const int subtract_mean = ic[14];
    p.B = ic[15]; p.C = ic[16]; p.L = ic[17]; p.T = ic[18];
    p.Q = p.N / 64;
    p.K = p.kind == KB_KALDI_FBANK ? p.n_mel + p.use_energy : p.kind == KB_KALDI_MFCC ? p.n_ceps : p.N / 2 + 1;
    p.preemph = fc[0];
    p.log_floor = fc[1] == 0.0f ? -INFINITY : (float)std::log((double)fc[1]);
    p.dither = fc[2];
    p.seed = seed;
    KbKaldiTables t;
    if (kb_kaldi_tables(p.W, p.N, p.n_mel, p.kind == KB_KALDI_MFCC ? p.n_mel * p.n_ceps : 0, window, banks, dct, t))
        return -1;
    p.wh = t.wh.data(); p.half = t.half.data(); p.twp = t.twp.data(); p.twn = t.twn.data();
    p.mlo = t.mlo.data(); p.mlen = t.mlen.data(); p.moff = t.moff.data(); p.mw = t.mw.data();
    p.klo = t.klo.data(); p.klen = t.klen.data(); p.kidx = t.kidx.data(); p.kw = t.kw.data();
    p.dct = t.dct.data();
    p.x = x; p.x_sb = xs[0]; p.x_sc = xs[1]; p.x_sl = xs[2];
    p.len = len;
    const int FPW = 32 / p.Q;
    p.jobs = (long long)p.B * p.C * ((p.T + FPW - 1) / FPW);
    if (!bwd) {
        p.y = y; p.y_sb = ys[0]; p.y_sc = ys[1]; p.y_st = ys[2]; p.y_sk = ys[3];
        run(p, 0, order);
        if (subtract_mean)
            for (long long e = 0; e < (long long)p.B * p.C * p.K; ++e)
                kb_kaldi_cmn_col(p, y, ys[0], ys[1], ys[2], ys[3], y, ys[0], ys[1], ys[2], ys[3], e);
        return 0;
    }
    std::vector<float> gf((size_t)p.B * p.C * p.T * p.W + 1, 0.0f);
    std::vector<float> gc;
    p.g = y; p.g_sb = ys[0]; p.g_sc = ys[1]; p.g_st = ys[2]; p.g_sk = ys[3];
    if (subtract_mean) {
        gc.assign((size_t)p.B * p.C * p.T * p.K + 1, 0.0f);
        const long long cs = (long long)p.T * p.K;
        for (long long e = 0; e < (long long)p.B * p.C * p.K; ++e)
            kb_kaldi_cmn_col(p, y, ys[0], ys[1], ys[2], ys[3], gc.data(), cs * p.C, cs, p.K, 1, e);
        p.g = gc.data(); p.g_sb = cs * p.C; p.g_sc = cs; p.g_st = p.K; p.g_sk = 1;
    }
    p.gf = gf.data();
    p.gx = gx; p.gx_sb = gxs[0]; p.gx_sc = gxs[1]; p.gx_sl = gxs[2];
    p.bwd = 1;
    run(p, 1, order);
    for (long long e = 0; e < (long long)p.B * p.C * p.L; ++e) kb_kaldi_gather_elem(p, e);
    return 0;
}

// The dither values d(seed, b, c, f, i), i < n, of one frame (unit variance; the kernel scales them by dither).
int kb_emu_kaldi_gauss(unsigned long long seed, long long b, int c, int f, int n, float* out) {
    const unsigned long long key = kb_kaldi_frame_key(seed, b, c, f);
    for (int i = 0; i < n; ++i) out[i] = kb_kaldi_gauss(key, i);
    return 0;
}

int kb_emu_kaldi_frames(int len, int W, int H, int snip, int min_len) {
    return kb_kaldi_frames(len, W, H, snip, min_len);
}

}  // extern "C"
