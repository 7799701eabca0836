// CPU emulation of the polyphase resampler body (kapre_b200/csrc/resample_core.cuh; tests only, never shipped).
// Compiled with KB_HOST_EMU: each phase of the CTA body runs as a loop over its threads, CTAs one after another.
#define KB_HOST_EMU 1
#include <cmath>
#include <cstdint>
#include <vector>
#include "../../kapre_b200/csrc/kb_tables.h"
#include "../../kapre_b200/csrc/resample_core.cuh"

extern "C" {

// xs / ys: (batch, channel, sample) element strides.  gain: up for the forward, the forward's up for the adjoint.
int kb_emu_resample(const float* x, const long long* xs, long long x_numel, int B, int C, int L, float* y,
                    const long long* ys, int L_out, int up, int down, const float* taps, int n_taps, double gain, int G,
                    int NT, int n_threads, int n_cta, int bulk_ok) {
    std::vector<float> tab;
    kb_resample_table(up, down, taps, n_taps, gain, tab);
    KbResampleParams p{};
    p.x = x; p.x_sb = xs[0]; p.x_sc = xs[1]; p.x_sl = xs[2]; p.x_numel = x_numel;
    p.x_align = (unsigned)(((uintptr_t)x >> 2) & 3u);
    p.bulk_ok = bulk_ok;
    p.B = B; p.C = C; p.L = L;
    p.y = y; p.y_sb = ys[0]; p.y_sc = ys[1]; p.y_sl = ys[2]; p.L_out = L_out;
    p.tab = tab.data(); p.up = up; p.down = down; p.f = ((n_taps - 1) / 2) / up; p.Kp = kb_resample_kp(up, n_taps);
    p.G = G; p.NT = NT;
    if (!kb_resample_setup(p, n_threads)) return -2;
    std::vector<kb_f4> smem(kb_resample_smem(up, p.Kp, NT, down, G) / 16 + 1);
    for (int cta = 0; cta < n_cta; ++cta) kb_resample_cta(p, reinterpret_cast<char*>(smem.data()), cta, n_cta);
    return 0;
}

int kb_emu_resample_kp(int up, int n_taps) { return kb_resample_kp(up, n_taps); }

}  // extern "C"
