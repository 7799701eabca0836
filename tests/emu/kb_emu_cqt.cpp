// CPU emulation of the constant-Q transform bodies (kapre_b200/csrc/cqt_core.cuh; tests only, never shipped).
// Compiled with KB_HOST_EMU: each phase of a CTA body runs as a loop over its threads.  Jobs are run one CTA at a
// time in the order `order` gives (0 ascending, 1 descending, 2 a fixed permutation); the result must not depend on
// it.  The pyramid levels come from the caller (the resampling body has its own emulation and tests).
#define KB_HOST_EMU 1
#include <cmath>
#include <cstdint>
#include <vector>
#include "../../kapre_b200/csrc/kb_tables.h"
#include "../../kapre_b200/csrc/cqt_core.cuh"

static long long perm(long long i, long long n, int order) {
    if (order == 1) return n - 1 - i;
    if (order == 2) { const long long h = n / 2; return i < h ? 2 * i + 1 : 2 * (i - h); }
    return i;
}

static int setup(KbCqtParams& p, std::vector<float2>& tab, std::vector<float2>& btab, const int* ic, const float* taps,
                 const float* const* lv, const long long* ls) {
    // ic: n_bins, bpo, hop, B, C, L, taps[n_oct]
    if (kb_cqt_build(ic[0], ic[1], ic[2], ic + 6, taps, p, tab, btab)) return -1;
    p.B = ic[3]; p.C = ic[4];
    p.M = 1 + ic[5] / ic[2];
    p.tab = tab.data(); p.btab = btab.data();
    long long L = ic[5];
    for (int i = 0; i < p.n_oct; ++i) {
        KbCqtOct& o = p.oct[i];
        o.L = (int)L;
        L = (L + 1) / 2;
        o.y = lv[i]; o.y_sb = ls[3 * i]; o.y_sc = ls[3 * i + 1]; o.y_sl = ls[3 * i + 2];
    }
    return 0;
}

extern "C" {

// lv[i] / ls[3i..3i+2]: level i and its (batch, channel, sample) strides.  out / os: (b, c, t, k) element strides.
// n_cta = 0: one CTA per job; n_cta > 0: that many CTAs walk the jobs grid-stride (tables kept across jobs).
int kb_emu_cqt(const int* ic, const float* taps, const float* const* lv, const long long* ls, int mag, void* out,
               const long long* os, int order, int n_cta) {
    KbCqtParams p{};
    std::vector<float2> tab, btab;
    if (setup(p, tab, btab, ic, taps, lv, ls)) return -1;
    p.n_threads = KB_CQT_THREADS;
    p.mag = mag;
    p.out = out; p.o_sb = os[0]; p.o_sc = os[1]; p.o_st = os[2]; p.o_sk = os[3];
    if (!kb_cqt_setup(p)) return -2;
    std::vector<kb_f4> smem((KB_CQT_TAB_BYTES + KB_CQT_SPAN_FLOATS * 4) / 16 + 1);
    if (n_cta > 0) {
        for (long long i = 0; i < n_cta; ++i)
            kb_cqt_fwd_cta(p, reinterpret_cast<char*>(smem.data()), perm(i, n_cta, order), n_cta);
        return 0;
    }
    for (long long i = 0; i < p.jobs; ++i)
        kb_cqt_fwd_cta(p, reinterpret_cast<char*>(smem.data()), perm(i, p.jobs, order), p.jobs);
    return 0;
}

// One octave's adjoint: gy = adjoint_bo(g) + add (add: contiguous (B, C, L_bo) or null).  gs: g's (b, c, t, k)
// strides; gys: gy's (b, c, l).
int kb_emu_cqt_adjoint(const int* ic, const float* taps, const float* const* lv, const long long* ls, int mag,
                       int bo, const void* g, const long long* gs, const float* add, float* gy, const long long* gys,
                       int order) {
    KbCqtParams p{};
    std::vector<float2> tab, btab;
    if (setup(p, tab, btab, ic, taps, lv, ls)) return -1;
    p.n_threads = KB_CQT_BWD_THREADS;
    p.mag = mag;
    p.bo = bo;
    p.g = g; p.g_sb = gs[0]; p.g_sc = gs[1]; p.g_st = gs[2]; p.g_sk = gs[3];
    p.add = add;
    p.gy = gy; p.gy_sb = gys[0]; p.gy_sc = gys[1]; p.gy_sl = gys[2];
    const KbCqtOct& o = p.oct[bo];
    const long long jobs = (long long)p.B * p.C * ((o.L + o.TS - 1) / o.TS);
    std::vector<kb_f4> smem(kb_cqt_bwd_smem() / 16 + 1);
    for (long long i = 0; i < jobs; ++i)
        kb_cqt_bwd_cta(p, reinterpret_cast<char*>(smem.data()), perm(i, jobs, order), jobs);
    return 0;
}

// Pairs (h, N), 1 <= h <= h_max, 1 <= N <= n_max, where one bin per adjoint group still finds no sample tile, or a
// one-frame forward tile does not fit the span budget.  Past h = 1024 + n_max a tile's frames no longer overlap, so
// larger hops behave like that one.
long long kb_emu_cqt_unfit(int h_max, int n_max) {
    long long bad = 0;
    for (int h = 1; h <= h_max; ++h)
        for (int N = 1; N <= n_max; ++N) {
            const int pad = (h & 1) ? 0 : 1;
            if (kb_cqt_pick_ts(h, N, 1, pad) == 0 || kb_cqt_pick_tf(1, h, N, pad) < 1 ||
                kb_cqt_staged(N, h, pad) > KB_CQT_SPAN_FLOATS)
                ++bad;
        }
    return bad;
}

// Geometry the plan picks: per segment (octave, k0, nk, TF); per octave (bgk, TS).  Returns the segment count.
int kb_emu_cqt_geometry(const int* ic, const float* taps, int* seg_out, int* oct_out) {
    KbCqtParams p{};
    std::vector<float2> tab, btab;
    const float* lv[KB_CQT_MAX_OCT] = {};
    long long ls[3 * KB_CQT_MAX_OCT] = {};
    if (setup(p, tab, btab, ic, taps, lv, ls)) return -1;
    for (int s = 0; s < p.n_segs; ++s) {
        seg_out[4 * s] = p.seg[s].oct; seg_out[4 * s + 1] = p.seg[s].k0; seg_out[4 * s + 2] = p.seg[s].nk;
        seg_out[4 * s + 3] = p.seg[s].TF;
        if (p.seg[s].NSu * p.seg[s].FR < p.seg[s].TF || p.seg[s].NSu > p.seg[s].NS || p.seg[s].NS < 1) return -3;
    }
    for (int i = 0; i < p.n_oct; ++i) { oct_out[2 * i] = p.oct[i].bgk; oct_out[2 * i + 1] = p.oct[i].TS; }
    return p.n_segs;
}

}  // extern "C"
