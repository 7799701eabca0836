// CPU emulation of the rhythm bodies (kapre_b200/csrc/rhythm_core.cuh; tests only, never shipped).  Compiled with
// KB_HOST_EMU: each phase of a CTA body runs as a loop over its threads.  Jobs are run one CTA at a time in the order
// `order` gives (0 ascending, 1 descending, 2 a fixed permutation), or with n_cta > 0 by that many CTAs walking the
// jobs grid-stride; the result must not depend on either.
#define KB_HOST_EMU 1
#include <cmath>
#include <cstdint>
#include <vector>
#include "../../kapre_b200/csrc/kb_tables.h"
#include "../../kapre_b200/csrc/rhythm_core.cuh"

static long long perm(long long i, long long n, int order) {
    if (order == 1) return n - 1 - i;
    if (order == 2) { const long long h = n / 2; return i < h ? 2 * i + 1 : 2 * (i - h); }
    return i;
}

template <typename P, typename F>
static void run(const P& p, long long jobs, long long smem, int order, int n_cta, F body) {
    std::vector<kb_f4> buf(smem / 16 + 1);
    char* sm = reinterpret_cast<char*>(buf.data());
    const long long n = n_cta > 0 ? n_cta : jobs;
    for (long long i = 0; i < n; ++i) body(p, sm, perm(i, n, order), n);
}

extern "C" {

// ic: B, C, T, K, lag, m, agg, pad.  xs: S strides (b, c, t, k); os: envelope strides (b, c, t).
static int onset_setup(KbOnsetParams& p, const int* ic, const float* x, const long long* xs, int bwd) {
    p.B = ic[0]; p.C = ic[1]; p.T = ic[2]; p.K = ic[3]; p.lag = ic[4]; p.m = ic[5]; p.agg = ic[6];
    p.P = ic[4] + ic[7];
    p.x = x; p.x_sb = xs[0]; p.x_sc = xs[1]; p.x_st = xs[2]; p.x_sk = xs[3];
    return kb_onset_setup(p, bwd) ? 0 : -1;
}

int kb_emu_onset(const int* ic, const float* x, const long long* xs, float* out, const long long* os, int order,
                 int n_cta) {
    KbOnsetParams p{};
    if (onset_setup(p, ic, x, xs, 0)) return -1;
    p.out = out; p.o_sb = os[0]; p.o_sc = os[1]; p.o_st = os[2];
    run(p, p.jobs, kb_onset_smem(p.K, p.m, p.F, 0), order, n_cta, kb_onset_cta<0>);
    return 0;
}

// ws: B C T K kb_on_w.
int kb_emu_onset_bwd(const int* ic, const float* x, const long long* xs, const float* g, const long long* gs,
                     float* gx, const long long* gxs, kb_on_w* ws, int order, int n_cta) {
    KbOnsetParams p{};
    if (onset_setup(p, ic, x, xs, 1)) return -1;
    p.g = g; p.g_sb = gs[0]; p.g_sc = gs[1]; p.g_st = gs[2];
    p.gx = gx; p.gx_sb = gxs[0]; p.gx_sc = gxs[1]; p.gx_st = gxs[2]; p.gx_sk = gxs[3];
    p.ws = ws;
    run(p, p.jobs, kb_onset_smem(p.K, p.m, p.F, 1), order, n_cta, kb_onset_cta<1>);
    const long long n = (long long)p.B * p.C * p.T * p.K;
    run(p, (n + KB_RH_THREADS - 1) / KB_RH_THREADS, 16, order, n_cta, kb_onset_gather_cta);
    return 0;
}

// ic: B, C, T, W, center, norm.  es: (b, c, t); os: (b, c, t, lag).  Returns the frames written.
int kb_emu_tempogram(const int* ic, const float* e, const long long* es, float* out, const long long* os, int order,
                     int n_cta) {
    KbTempogramParams p{};
    p.B = ic[0]; p.C = ic[1]; p.T = ic[2]; p.W = ic[3]; p.center = ic[4]; p.norm = ic[5];
    p.e = e; p.e_sb = es[0]; p.e_sc = es[1]; p.e_st = es[2];
    p.out = out; p.o_sb = os[0]; p.o_sc = os[1]; p.o_st = os[2]; p.o_sk = os[3];
    if (!kb_tempogram_setup(p)) return -1;
    run(p, p.jobs, (long long)kb_tg_words(p.W, p.F) * 4, order, n_cta, kb_tempogram_cta);
    return p.n_out;
}

// ic: B, C, T, W, per_frame.  gs: (b, c, t, lag); os: (b, c, t) (per frame) or null.  Both launches of the mean.
int kb_emu_tempo(const int* ic, const float* tg, const long long* gs, const double* logprior, double bpm_scale,
                 float* out, const long long* os, int order, int n_cta) {
    KbTempoParams p{};
    p.B = ic[0]; p.C = ic[1]; p.T = ic[2]; p.W = ic[3]; p.per_frame = ic[4];
    p.tg = tg; p.g_sb = gs[0]; p.g_sc = gs[1]; p.g_st = gs[2]; p.g_sk = gs[3];
    p.logprior = logprior; p.bpm_scale = bpm_scale; p.out = out;
    if (os) { p.o_sb = os[0]; p.o_sc = os[1]; p.o_st = os[2]; }
    kb_tempo_setup(p);
    std::vector<double> part(kb_tempo_ws_bytes(p.B, p.C, p.T, p.W) / 8 + 1);
    p.part = part.data();
    if (!p.per_frame) run(p, (long long)p.B * p.C * p.chunks, 16, order, n_cta, kb_tempo_part_cta);
    run(p, p.jobs, kb_tempo_smem(p.W), order, n_cta, kb_tempo_cta);
    return 0;
}

// ic: B, C, T, pre_max, post_max, pre_avg, post_avg, wait, normalize.
int kb_emu_peak(const int* ic, double delta, const float* e, const long long* es, unsigned char* mask,
                const long long* ms, int order, int n_cta) {
    KbPeakParams p{};
    p.B = ic[0]; p.C = ic[1]; p.T = ic[2]; p.pre_max = ic[3]; p.post_max = ic[4]; p.pre_avg = ic[5];
    p.post_avg = ic[6]; p.wait = ic[7]; p.normalize = ic[8]; p.delta = delta;
    p.e = e; p.e_sb = es[0]; p.e_sc = es[1]; p.e_st = es[2];
    p.mask = mask; p.m_sb = ms[0]; p.m_sc = ms[1]; p.m_st = ms[2];
    p.jobs = p.T ? (long long)p.B * p.C : 0;
    run(p, p.jobs, kb_peak_smem(), order, n_cta, kb_peak_cta);
    return 0;
}

// ic: B, C, T, trim.  dc: fps, tightness.  bpm: per row or null (bpm_const).  ws: B C T 24 bytes.
int kb_emu_beat(const int* ic, const double* dc, const float* bpm, float bpm_const, const float* e,
                const long long* es, float* tempo, unsigned char* mask, const long long* ms, void* ws, int order,
                int n_cta) {
    KbBeatParams p{};
    p.B = ic[0]; p.C = ic[1]; p.T = ic[2]; p.trim = ic[3]; p.fps = dc[0]; p.tightness = dc[1];
    p.bpm = bpm; p.bpm_const = bpm_const;
    p.e = e; p.e_sb = es[0]; p.e_sc = es[1]; p.e_st = es[2];
    p.tempo = tempo; p.mask = mask; p.m_sb = ms[0]; p.m_sc = ms[1]; p.m_st = ms[2];
    p.ws = ws;
    p.jobs = (long long)p.B * p.C;
    run(p, p.jobs, kb_beat_smem(), order, n_cta, kb_beat_cta);
    return 0;
}

}  // extern "C"
