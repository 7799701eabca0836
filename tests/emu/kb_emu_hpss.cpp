// CPU emulation of the HPSS bodies (kapre_b200/csrc/hpss_core.cuh; tests only, never shipped).  Compiled with
// KB_HOST_EMU: each phase of a CTA body runs as a loop over its threads.  Jobs are run one CTA at a time in the order
// `order` gives (0 ascending, 1 descending, 2 a fixed permutation), or with n_cta > 0 by that many CTAs walking the
// jobs grid-stride; the result must not depend on either.
#define KB_HOST_EMU 1
#include <cmath>
#include <cstdint>
#include <vector>
#include "../../kapre_b200/csrc/kb_tables.h"
#include "../../kapre_b200/csrc/hpss_core.cuh"

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

template <int BWD>
static void run_tiles(const KbHpssParams& p, int order, int n_cta) {
    const int smem = kb_hpss_smem(p.kh, p.kp, BWD);
    const int sh = kb_hs_slots(p.kh), sp = kb_hs_slots(p.kp);
    if (sh == 32 && sp == 32) run(p, p.jobs, smem, order, n_cta, kb_hpss_cta<32, 32, BWD>);
    else if (sh == 32) run(p, p.jobs, smem, order, n_cta, kb_hpss_cta<32, 64, BWD>);
    else if (sp == 32) run(p, p.jobs, smem, order, n_cta, kb_hpss_cta<64, 32, BWD>);
    else run(p, p.jobs, smem, order, n_cta, kb_hpss_cta<64, 64, BWD>);
}

static void set4(long long* d, const long long* s) { d[0] = s[0]; d[1] = s[1]; d[2] = s[2]; d[3] = s[3]; }

extern "C" {

// ic: B, C, T, K, kh, kp, pmode, split, cplx, mask.  fc: mh, mp, power.  Strides (b, c, t, k) in elements.
static int setup(KbHpssParams& p, const int* ic, const float* fc, const void* x, const long long* xs) {
    p.B = ic[0]; p.C = ic[1]; p.T = ic[2]; p.K = ic[3]; p.kh = ic[4]; p.kp = ic[5];
    p.pmode = ic[6]; p.split = ic[7]; p.cplx = ic[8]; p.mask = ic[9];
    p.mh = fc[0]; p.mp = fc[1]; p.power = fc[2];
    p.x = x; set4(&p.x_sb, xs);
    return kb_hpss_setup(p) ? 0 : -1;
}

int kb_emu_hpss(const int* ic, const float* fc, const void* x, const long long* xs, void* oh, const long long* ohs,
                void* op, const long long* ops, int order, int n_cta) {
    KbHpssParams p{};
    if (setup(p, ic, fc, x, xs)) return -1;
    p.oh = oh; if (oh) set4(&p.oh_sb, ohs);
    p.op = op; if (op) set4(&p.op_sb, ops);
    run_tiles<0>(p, order, n_cta);
    return 0;
}

// Both gradient passes.  ws: 2 x B C T K kb_hs_w.
int kb_emu_hpss_bwd(const int* ic, const float* fc, const void* x, const long long* xs, const void* gh,
                    const long long* ghs, const void* gp, const long long* gps, void* gx, const long long* gxs,
                    kb_hs_w* ws, int order, int n_cta) {
    KbHpssParams p{};
    if (setup(p, ic, fc, x, xs)) return -1;
    p.gh = gh; if (gh) set4(&p.gh_sb, ghs);
    p.gp = gp; if (gp) set4(&p.gp_sb, gps);
    p.gx = gx; set4(&p.gx_sb, gxs);
    const long long n = (long long)p.B * p.C * p.T * p.K;
    p.wh = ws; p.wp = ws + n;
    run_tiles<1>(p, order, n_cta);
    run(p, (n + KB_HS_THREADS - 1) / KB_HS_THREADS, 16, order, n_cta, kb_hpss_gather_cta);
    return 0;
}

}  // extern "C"
