// CPU emulation of the band-limited interpolator body (kapre_b200/csrc/sinc_core.cuh; tests only, never shipped).
// Compiled with KB_HOST_EMU: each phase of the CTA body runs as a loop over its threads, CTAs one after another.
#define KB_HOST_EMU 1
#include <cmath>
#include <cstdint>
#include <vector>
#include "../../kapre_b200/csrc/kb_tables.h"
#include "../../kapre_b200/csrc/sinc_core.cuh"

extern "C" {

// xs / ys: (batch, channel, sample) element strides.  adjoint = 0: the forward sum of (ratio, offset) from x (L
// samples) to y (L_out samples); adjoint = 1: its transpose, from the output gradient x to the input gradient y.
int kb_emu_sinc(const float* x, const long long* xs, long long x_numel, int B, int C, int L, float* y, const long long* ys,
                int L_out, double ratio, double offset, int adjoint, int G, int NT, int n_threads, int n_cta, int bulk_ok) {
    static std::vector<float2> tab;
    static double integral = 0.0;
    if (tab.empty()) { kb_sinc_table(tab); integral = kb_sinc_integral(); }
    double step, off, s, gain;
    kb_sinc_args(ratio, offset, adjoint, &step, &off, &s, &gain);
    KbSincParams p{};
    p.x = x; p.x_sb = xs[0]; p.x_sc = xs[1]; p.x_sl = xs[2]; p.x_numel = x_numel;
    p.x_align = (unsigned)(((uintptr_t)x >> 2) & 3u);
    p.bulk_ok = bulk_ok;
    p.B = B; p.C = C; p.L = L;
    p.y = y; p.y_sb = ys[0]; p.y_sc = ys[1]; p.y_sl = ys[2]; p.L_out = L_out;
    p.tab = tab.data();
    p.G = G; p.NT = NT;
    if (!kb_sinc_setup(p, step, off, s, gain, integral, n_threads)) return -2;
    std::vector<kb_f4> smem(kb_sinc_smem(NT, step, p.nw, G) / 16 + 1);
    for (int cta = 0; cta < n_cta; ++cta) kb_sinc_cta(p, reinterpret_cast<char*>(smem.data()), cta, n_cta);
    return 0;
}

double kb_emu_sinc_integral() { return kb_sinc_integral(); }
double kb_emu_sinc_h(double u) { return kb_sinc_h(u); }
// entry k of the shared-memory table: (h(k / Q), h((k + 1) / Q) - h(k / Q))
void kb_emu_sinc_table(float* out) {
    std::vector<float2> tab;
    kb_sinc_table(tab);
    for (int k = 0; k < KB_SINC_NTAB; ++k) { out[2 * k] = tab[k].x; out[2 * k + 1] = tab[k].y; }
}
int kb_emu_sinc_smem(int NT, double ratio, int adjoint, int G) {
    double step, off, s, gain;
    kb_sinc_args(ratio, 0.0, adjoint, &step, &off, &s, &gain);
    return kb_sinc_smem(NT, step, (int)std::ceil((double)KB_SINC_Z / s), G);
}

}  // extern "C"
