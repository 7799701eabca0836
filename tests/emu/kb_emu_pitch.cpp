// CPU emulation of the pitch-tracking bodies (kapre_b200/csrc/pitch_core.cuh; tests only, never shipped).
// Compiled with KB_HOST_EMU: each phase of a CTA body runs as a loop over its threads.  Jobs (tiles, or rows for the
// Viterbi) are run one CTA at a time in the order `order` gives (0 ascending, 1 descending, 2 a fixed permutation),
// or with n_cta > 0 by that many CTAs walking the jobs grid-stride; the result must not depend on either.
#define KB_HOST_EMU 1
#include <cmath>
#include <cstdint>
#include <vector>
#include "../../kapre_b200/csrc/kb_tables.h"
#include "../../kapre_b200/csrc/pitch_core.cuh"

static long long perm(long long i, long long n, int order) {
    if (order == 1) return n - 1 - i;
    if (order == 2) { const long long h = n / 2; return i < h ? 2 * i + 1 : 2 * (i - h); }
    return i;
}

// ic: F, W, h, center, min_p, max_p, pyin, n_thr, n_pitch
static bool geometry(KbPitchParams& p, const int* ic, float sr, double thresh) {
    p = KbPitchParams{};
    p.F = ic[0]; p.W = ic[1]; p.h = ic[2]; p.pad = ic[3] ? ic[0] / 2 : 0;
    p.min_p = ic[4]; p.max_p = ic[5]; p.pyin = ic[6]; p.n_thr = ic[7]; p.n_pitch = ic[8];
    p.sr = sr; p.thresh = thresh;
    return kb_pitch_tiling(p);
}

static std::vector<float> to_f(const double* v, size_t n) {
    std::vector<float> r(n);
    for (size_t i = 0; i < n; ++i) r[i] = (float)v[i];
    return r;
}

extern "C" {

// Tiling the plan picks: share, G, KB, TF, NSEG, SPAN, smem bytes.
int kb_emu_pitch_tiling(const int* ic, int* out) {
    KbPitchParams p;
    if (!geometry(p, ic, 1.0f, 0.1)) return -1;
    out[0] = p.share; out[1] = p.G; out[2] = p.KB; out[3] = p.TF; out[4] = p.NSEG; out[5] = p.SPAN; out[6] = p.smem;
    return 0;
}

// The difference-function body.  dims: B, C, L, M.  xs / os / cs: element strides of x (b, c, l), out (b, c, t) and
// cm (b, c, t, k).  tabs (pYIN): beta, bpow, bnorm, bonus (float64, rounded here as the plan rounds them) and edges.
int kb_emu_pitch(const int* ic, float sr, double thresh, const int* dims, const float* x, const long long* xs,
                 float* out, const long long* os, float* cm, const long long* cs, const double* const* tabs,
                 int* cand_n, unsigned short* cand_bin, float* cand_p, int order, int n_cta) {
    KbPitchParams p;
    if (!geometry(p, ic, sr, thresh)) return -1;
    std::vector<float> beta, bpow, bnorm, bonus;
    if (p.pyin) {
        beta = to_f(tabs[0], p.n_thr); bpow = to_f(tabs[1], p.cmax + 1); bnorm = to_f(tabs[2], p.cmax + 1);
        bonus = to_f(tabs[3], p.n_thr + 1);
        p.beta = beta.data(); p.bpow = bpow.data(); p.bnorm = bnorm.data(); p.bonus = bonus.data();
        p.edges = tabs[4];
        p.cand_n = cand_n; p.cand_bin = cand_bin; p.cand_p = cand_p;
    }
    p.B = dims[0]; p.C = dims[1]; p.L = dims[2]; p.M = dims[3];
    p.x = x; p.x_sb = xs[0]; p.x_sc = xs[1]; p.x_sl = xs[2];
    p.out = out; p.o_sb = os[0]; p.o_sc = os[1]; p.o_st = os[2];
    p.cm = cm;
    if (cm) { p.c_sb = cs[0]; p.c_sc = cs[1]; p.c_st = cs[2]; p.c_sk = cs[3]; }
    if (!kb_pitch_setup(p)) return -2;
    std::vector<kb_f4> smem(p.smem / 16 + 1);
    char* sm = reinterpret_cast<char*>(smem.data());
    if (n_cta > 0) {
        for (long long i = 0; i < n_cta; ++i) kb_pitch_cta(p, sm, perm(i, n_cta, order), n_cta);
        return 0;
    }
    for (long long i = 0; i < p.jobs; ++i) kb_pitch_cta(p, sm, perm(i, p.jobs, order), p.jobs);
    return 0;
}

// The Viterbi body.  vi: n_pitch, band_width, M, C, rows, cmax.  vf: log_stay, log_switch, log_init_voiced,
// log_init_unvoiced, fill_na.  tabs: log_triangle, log_row_norm, freqs (float64).  bp: rows M 2 n_pitch entries.
int kb_emu_viterbi(const int* vi, const float* vf, const double* const* tabs, const int* cand_n,
                   const unsigned short* cand_bin, const float* cand_p, float* vp, float* f0, unsigned char* flag,
                   const long long* os, unsigned short* bp, int nt, int order, int n_cta) {
    KbVitParams p{};
    p.n = vi[0]; p.w = vi[1]; p.half = vi[1] / 2; p.M = vi[2]; p.C = vi[3]; p.rows = vi[4]; p.cmax = vi[5];
    p.nt = nt;
    p.ls = vf[0]; p.lw = vf[1]; p.lpv = vf[2]; p.lpu = vf[3]; p.fill = vf[4];
    std::vector<float> ltri = to_f(tabs[0], p.w), lnorm = to_f(tabs[1], p.n), freq = to_f(tabs[2], p.n);
    p.ltri = ltri.data(); p.lnorm = lnorm.data(); p.freq = freq.data();
    p.cand_n = cand_n; p.cand_bin = cand_bin; p.cand_p = cand_p;
    p.vp = vp; p.f0 = f0; p.flag = flag; p.o_sb = os[0]; p.o_sc = os[1]; p.o_st = os[2];
    p.bp = bp;
    std::vector<kb_f4> smem(kb_vit_smem(p.n, p.w) / 16 + 1);
    std::vector<float> red(nt);
    char* sm = reinterpret_cast<char*>(smem.data());
    const long long jobs = n_cta > 0 ? n_cta : p.rows;
    for (long long i = 0; i < jobs; ++i) kb_vit_cta(p, sm, red.data(), perm(i, jobs, order), jobs);
    return 0;
}

}  // extern "C"
