// CPU emulation of the chroma bodies (kapre_b200/csrc/chroma_core.cuh; tests only, never shipped).  Compiled with
// KB_HOST_EMU: each phase of a CTA body runs as a loop over its threads.  Jobs are run one CTA at a time in the order
// `order` gives (0 ascending, 1 descending, 2 a fixed permutation), or with n_cta > 0 by that many CTAs walking the
// jobs grid-stride; the result must not depend on either.
#define KB_HOST_EMU 1
#include <cmath>
#include <cstdint>
#include <vector>
#include "../../kapre_b200/csrc/kb_tables.h"
#include "../../kapre_b200/csrc/chroma_core.cuh"

static long long perm(long long i, long long n, int order) {
    if (order == 1) return n - 1 - i;
    if (order == 2) { const long long h = n / 2; return i < h ? 2 * i + 1 : 2 * (i - h); }
    return i;
}

template <typename P, typename F>
static void run(const P& p, long long jobs, int smem, int order, int n_cta, F body) {
    std::vector<kb_f4> buf(smem / 16 + 1);
    char* sm = reinterpret_cast<char*>(buf.data());
    const long long n = n_cta > 0 ? n_cta : jobs;
    for (long long i = 0; i < n; ++i) body(p, sm, perm(i, n, order), n);
}

extern "C" {

// The projection body, forward (g == null) or backward.  ic: NC, K, in_mode, norm, cens, has_thr, B, C, M.  W: float32
// tables [t][NC][K]; tab: per item table (nullable).  xs / os / gs / gxs: element strides (b, c, t, k).
int kb_emu_chroma(const int* ic, float thr, const float* W, const int* tab, const void* x, const long long* xs,
                  float* out, const long long* os, const float* g, const long long* gs, void* gx,
                  const long long* gxs, int order, int n_cta) {
    KbChromaParams p{};
    p.NC = ic[0]; p.K = ic[1]; p.in_mode = ic[2]; p.norm = ic[3]; p.cens = ic[4]; p.has_thr = ic[5]; p.thr = thr;
    p.B = ic[6]; p.C = ic[7]; p.M = ic[8];
    p.W = W; p.tab = tab;
    kb_chroma_tiling(p);
    if (!kb_chroma_setup(p)) return -1;
    p.x = x; p.x_sb = xs[0]; p.x_sc = xs[1]; p.x_st = xs[2]; p.x_sk = xs[3];
    const int smem = kb_chroma_smem(p.NC, p.G, p.TF);
    if (!g) {
        p.out = out; p.o_sb = os[0]; p.o_sc = os[1]; p.o_st = os[2]; p.o_sk = os[3];
        run(p, p.jobs, smem, order, n_cta, kb_chroma_cta);
    } else {
        p.g = g; p.g_sb = gs[0]; p.g_sc = gs[1]; p.g_st = gs[2]; p.g_sk = gs[3];
        p.gx = gx; p.gx_sb = gxs[0]; p.gx_sc = gxs[1]; p.gx_st = gxs[2]; p.gx_sk = gxs[3];
        run(p, p.jobs, smem, order, n_cta, kb_chroma_bwd_cta);
    }
    return 0;
}

// The tuning estimate's seven passes.  ic: K, lo, hi, in_mode, nres, B, C, M.  ws: scratch the caller zeroed except
// `above` (0xff bytes).  mag / pitch: rows M cap slots.
int kb_emu_tuning(const int* ic, float sr, float nfft, double bpo, const double* edges, const float* x,
                  const long long* xs, float* mag, float* pitch, unsigned* hist, unsigned* above, unsigned* res,
                  double* tuning, int* tab, int order, int n_cta) {
    KbTuneParams p{};
    p.K = ic[0]; p.lo = ic[1]; p.hi = ic[2]; p.cap = (p.hi - p.lo + 1) / 2; p.in_mode = ic[3]; p.nres = ic[4];
    p.B = ic[5]; p.C = ic[6]; p.M = ic[7];
    p.sr = sr; p.nfft = nfft; p.bpo = bpo; p.edges = edges;
    p.x = x; p.x_sb = xs[0]; p.x_sc = xs[1]; p.x_st = xs[2]; p.x_sk = xs[3];
    p.mag = mag; p.pitch = pitch; p.hist = hist; p.above = above; p.res = res; p.tuning = tuning; p.tab = tab;
    const long long rows = (long long)p.B * p.C;
    if (p.M > 0) {
        p.tiles = ((long long)p.M + KB_CH_PEAK_TF - 1) / KB_CH_PEAK_TF;
        p.jobs = rows * p.tiles;
        run(p, p.jobs, kb_tune_peak_smem(), order, n_cta, kb_tune_peak_cta);
        p.tiles = ((long long)p.M + KB_CH_SEL_TF - 1) / KB_CH_SEL_TF;
        p.jobs = rows * p.tiles;
        for (p.pass = 1; p.pass <= 5; ++p.pass) run(p, p.jobs, kb_tune_sel_smem(), order, n_cta, kb_tune_sel_cta);
    }
    run(p, p.B, 2 * KB_CH_THREADS * 4, order, n_cta, kb_tune_argmax_cta);
    return 0;
}

// The CENS smoothing body over q [row][M][NC].  w: float32 taps.
int kb_emu_cens(int NC, int N, const float* w, int B, int C, int M, const float* q, float* out, const long long* os,
                int order, int n_cta) {
    KbCensParams p{};
    p.NC = NC; p.N = N; p.w = w; p.B = B; p.C = C; p.M = M; p.q = q;
    p.out = out; p.o_sb = os[0]; p.o_sc = os[1]; p.o_st = os[2]; p.o_sk = os[3];
    p.tiles = ((long long)M + KB_CH_SMOOTH_TF - 1) / KB_CH_SMOOTH_TF;
    p.jobs = (long long)B * C * p.tiles;
    run(p, p.jobs, kb_cens_smem(NC, N), order, n_cta, kb_cens_cta);
    return 0;
}

}  // extern "C"
