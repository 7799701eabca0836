// CPU emulation of the filterbank-inversion kernel (kapre_b200/csrc/fbinv_core.cuh; tests only, never shipped).
// Compiled with KB_HOST_EMU: the CTA body runs for every CTA in turn, each phase as a loop over its threads.
#define KB_HOST_EMU 1
#include <cmath>
#include <cstdint>
#include <vector>
#include "../../kapre_b200/csrc/fbinv_core.cuh"

extern "C" {

// The plan's host tables for a row-major (n_freq x n_bands) filterbank: step, ||A||_2^2 and 1 / d (n_bands floats).
void kb_emu_fbi_tables(const float* fb, int n_freq, int n_bands, float* step, double* norm2, float* inv_d) {
    KbFbiTables t;
    kb_fbi_make_tables(fb, n_freq, n_bands, t);
    *step = t.step;
    *norm2 = t.norm2;
    for (int m = 0; m < n_bands; ++m) inv_d[m] = t.inv_d[m];
}

int kb_emu_fbi_pick_r(int n_freq, int n_bands, int smem_limit) { return kb_fbi_pick_r(n_freq, n_bands, smem_limit); }

// xs / os: (batch, channel, frame, bin) element strides of x (n_bands bins) and out (n_freq bins).  R: frames per tile,
// n_cta: CTAs of the persistent grid.
int kb_emu_fbi(const float* fb, int n_freq, int n_bands, const float* x, const long long* xs, int B, int C, int T,
               int n_iter, int from_db, float ref_value, float amin, float* out, const long long* os, int R, int n_cta) {
    KbFbiTables t;
    kb_fbi_make_tables(fb, n_freq, n_bands, t);
    KbFbiParams p{};
    p.x = x; p.x_sb = xs[0]; p.x_sc = xs[1]; p.x_st = xs[2]; p.x_sk = xs[3];
    p.B = B; p.C = C; p.T = T; p.F = n_freq; p.M = n_bands;
    p.bands = t.bands.data(); p.fbw = t.w.data(); p.cptr = t.cptr.data(); p.cols = t.cols.data(); p.inv_d = t.inv_d.data();
    p.step = t.step;
    p.n_iter = n_iter;
    p.from_db = from_db;
    p.db_scale = amin > ref_value ? (double)amin : (double)ref_value;
    p.out = out; p.o_sb = os[0]; p.o_sc = os[1]; p.o_st = os[2]; p.o_sk = os[3];
    p.R = R;
    p.n_tiles_t = (T + R - 1) / R;
    p.n_warps = KB_FBI_WARPS;
    std::vector<float> smem((size_t)kb_fbi_smem_layout(n_freq, n_bands, R).total / 4, std::nanf(""));
    for (int cta = 0; cta < n_cta; ++cta) kb_fbi_cta(p, reinterpret_cast<char*>(smem.data()), cta, n_cta);
    return 0;
}

}  // extern "C"
