// CPU emulation of the second-order-section bodies (kapre_b200/csrc/sos_core.cuh; tests only, never shipped).
// Compiled with KB_HOST_EMU: each phase of a block body runs as a loop over its 32 lanes, blocks one after another, in
// the order the library launches them (powers, state, carry, output).
#define KB_HOST_EMU 1
#include <cmath>
#include <cstdint>
#include <vector>
#include "../../kapre_b200/csrc/kb_tables.h"
#include "../../kapre_b200/csrc/sos_core.cuh"

template <int S>
static void kb_emu_sos_run(KbSosParams& p, int tile_order) {
    constexpr int D = 2 * S;
    const long long n_f = (long long)p.g.n_fb * p.g.n_fc, tiles = p.g.n_cols * p.g.nblk;
    std::vector<double> pw((size_t)n_f * KB_IIR_NPOW * D * D);
    std::vector<float> e((size_t)p.g.n_cols * p.g.K * D);
    std::vector<double> blk((size_t)p.g.n_cols * p.g.nblk * D);
    p.g.pw = pw.data(); p.g.e = e.data(); p.g.blk = blk.data();
    std::vector<double> m(3 * D * D);
    for (long long f = 0; f < n_f; ++f) kb_sos_powers_cta<S>(p, m.data(), f);
    std::vector<kb_f4> smem(kb_sos_smem(S).total / 16 + 1);
    char* sm = reinterpret_cast<char*>(smem.data());
    for (long long i = 0; i < tiles; ++i) kb_sos_state_cta<S>(p, sm, tile_order ? tiles - 1 - i : i);
    for (long long c = 0; c < p.g.n_cols; ++c) kb_sos_carry_col<S>(p, tile_order ? p.g.n_cols - 1 - c : c);
    for (long long i = 0; i < tiles; ++i) kb_sos_out_cta<S>(p, sm, tile_order ? tiles - 1 - i : i);
}

extern "C" {

// x, y: (batch, channel, sample) element strides xs / ys; sos: S x 6 floats per filter at strides cs = (sb, sc);
// zi / zf (either may be null): (z1, z2) per section at strides zis / zfs = (sb, sc, ss).  flags: 2 reverse.
// tile_order = 1 runs the blocks of each pass in reverse order (the result must not depend on it).  bulk = 0 forces
// the cooperative loader.
int kb_emu_sosfilt(const float* x, const long long* xs, float* y, const long long* ys, const float* sos,
                   const long long* cs, int S, int B, int C, int L, int flags, const float* zi, const long long* zis,
                   float* zf, const long long* zfs, int tile_order, int bulk, long long x_numel) {
    KbSosParams p{};
    p.g.x = x; p.g.x_sb = xs[0]; p.g.x_sc = xs[1]; p.g.x_sl = xs[2];
    p.g.x_numel = bulk ? x_numel : 0;       // 0: no block qualifies for the bulk copy
    p.g.x_align = (unsigned)(((uintptr_t)x >> 2) & 3u);
    p.g.y = y; p.g.y_sb = ys[0]; p.g.y_sc = ys[1]; p.g.y_sl = ys[2];
    p.g.ac = sos; p.g.a_sb = cs[0]; p.g.a_sc = cs[1];
    p.g.B = B; p.g.C = C; p.g.L = L;
    p.g.reverse = (flags & KB_IIR_FLAG_REVERSE) ? 1 : 0;
    p.S = S;
    if (zi) { p.zi = zi; p.zi_sb = zis[0]; p.zi_sc = zis[1]; p.zi_ss = zis[2]; }
    if (zf) { p.zf = zf; p.zf_sb = zfs[0]; p.zf_sc = zfs[1]; p.zf_ss = zfs[2]; }
    kb_iir_setup(p.g);
    if (p.g.n_cols == 0 || L == 0) return 0;
    switch (S) {
    case 1: kb_emu_sos_run<1>(p, tile_order); return 0;
    case 2: kb_emu_sos_run<2>(p, tile_order); return 0;
    case 3: kb_emu_sos_run<3>(p, tile_order); return 0;
    case 4: kb_emu_sos_run<4>(p, tile_order); return 0;
    case 5: kb_emu_sos_run<5>(p, tile_order); return 0;
    case 6: kb_emu_sos_run<6>(p, tile_order); return 0;
    case 7: kb_emu_sos_run<7>(p, tile_order); return 0;
    case 8: kb_emu_sos_run<8>(p, tile_order); return 0;
    }
    return -1;
}

// The powers Phi^(2^j Tc) of one filter (sos: S x 6 floats), (KB_IIR_NPOW, 2S, 2S) float64.
int kb_emu_sos_powers(const float* sos, int S, double* out) {
    KbSosParams p{};
    p.g.ac = sos; p.g.B = 1; p.g.C = 1; p.g.L = 1;
    p.S = S;
    kb_iir_setup(p.g);
    p.g.pw = out;
    std::vector<double> m(3 * 4 * KB_SOS_MAX * KB_SOS_MAX);
    switch (S) {
    case 1: kb_sos_powers_cta<1>(p, m.data(), 0); return 0;
    case 2: kb_sos_powers_cta<2>(p, m.data(), 0); return 0;
    case 3: kb_sos_powers_cta<3>(p, m.data(), 0); return 0;
    case 4: kb_sos_powers_cta<4>(p, m.data(), 0); return 0;
    case 5: kb_sos_powers_cta<5>(p, m.data(), 0); return 0;
    case 6: kb_sos_powers_cta<6>(p, m.data(), 0); return 0;
    case 7: kb_sos_powers_cta<7>(p, m.data(), 0); return 0;
    case 8: kb_sos_powers_cta<8>(p, m.data(), 0); return 0;
    }
    return -1;
}

}  // extern "C"
