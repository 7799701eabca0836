// CPU emulation of the IIR filter bodies (kapre_b200/csrc/iir_core.cuh; tests only, never shipped).  Compiled with
// KB_HOST_EMU: each phase of a block body runs as a loop over its 32 lanes, blocks one after another, in the order
// the library launches them (powers, state, carry, output).
#define KB_HOST_EMU 1
#include <cmath>
#include <cstdint>
#include <vector>
#include "../../kapre_b200/csrc/kb_tables.h"
#include "../../kapre_b200/csrc/iir_core.cuh"

extern "C" {

// x, y: (batch, channel, sample) element strides xs / ys; b, a: order + 1 floats per filter at strides cs =
// (b_sb, b_sc, a_sb, a_sc).  bwd = 0: y = lfilter(x) (flags: 1 clamp, 2 reverse).  bwd = 1: x is gy, y receives gx,
// and with xr / yr (strides rs) part receives the (2 order + 1, B C, K) coefficient sums.  tile_order = 1 runs the
// blocks of each pass in reverse order (the result must not depend on it).  x_align: the bulk copies' alignment
// phase; bulk = 0 forces the cooperative loader.
int kb_emu_lfilter(const float* x, const long long* xs, float* y, const long long* ys, const float* b, const float* a,
                   const long long* cs, int order, int B, int C, int L, int flags, int bwd, const float* xr,
                   const float* yr, const long long* rs, float* part, int tile_order, int bulk, long long x_numel) {
    KbIirParams p{};
    p.x = x; p.x_sb = xs[0]; p.x_sc = xs[1]; p.x_sl = xs[2];
    p.x_numel = bulk ? x_numel : 0;         // 0: no block qualifies for the bulk copy
    p.x_align = (unsigned)(((uintptr_t)x >> 2) & 3u);
    p.y = y; p.y_sb = ys[0]; p.y_sc = ys[1]; p.y_sl = ys[2];
    p.bc = b; p.b_sb = cs[0]; p.b_sc = cs[1];
    p.ac = a; p.a_sb = cs[2]; p.a_sc = cs[3];
    p.order = order; p.B = B; p.C = C; p.L = L;
    p.reverse = (flags & KB_IIR_FLAG_REVERSE) ? 1 : 0;
    p.clamp = (flags & KB_IIR_FLAG_CLAMP) ? 1 : 0;
    p.bwd = bwd;
    if (bwd) { p.reverse ^= 1; p.clamp = 0; }
    if (order < 0 || order > KB_IIR_N) return -1;
    kb_iir_setup(p);
    if (p.n_cols == 0 || L == 0) return 0;
    if (part) {
        p.part = part;
        p.xr = xr; p.xr_sb = rs[0]; p.xr_sc = rs[1]; p.xr_sl = rs[2];
        p.yr = yr; p.yr_sb = rs[3]; p.yr_sc = rs[4]; p.yr_sl = rs[5];
    }
    const long long n_f = (long long)p.n_fb * p.n_fc, tiles = p.n_cols * p.nblk;
    std::vector<double> pw((size_t)n_f * KB_IIR_NPOW * 64);
    std::vector<float> e((size_t)p.n_cols * p.K * KB_IIR_N);
    std::vector<double> blk((size_t)p.n_cols * p.nblk * KB_IIR_N);
    p.pw = pw.data(); p.e = e.data(); p.blk = blk.data();
    std::vector<double> m(192);
    for (long long f = 0; f < n_f; ++f) kb_iir_powers_cta(p, m.data(), f);
    std::vector<kb_f4> smem(kb_iir_smem(1).total / 16 + 1);
    char* sm = reinterpret_cast<char*>(smem.data());
    for (long long i = 0; i < tiles; ++i) kb_iir_state_cta(p, sm, tile_order ? tiles - 1 - i : i);
    for (long long c = 0; c < p.n_cols; ++c) kb_iir_carry_col(p, tile_order ? p.n_cols - 1 - c : c);
    for (long long i = 0; i < tiles; ++i) kb_iir_out_cta(p, sm, tile_order ? tiles - 1 - i : i);
    return 0;
}

int kb_emu_iir_consts(int* out) {
    out[0] = KB_IIR_N; out[1] = KB_IIR_TC; out[2] = KB_IIR_W;
    return 0;
}

// The powers Phi^(2^j Tc) of one denominator (a: order + 1 floats), (KB_IIR_NPOW, 8, 8) float64.
int kb_emu_iir_powers(const float* a, int order, double* out) {
    KbIirParams p{};
    p.ac = a; p.order = order; p.B = 1; p.C = 1; p.L = 1;
    kb_iir_setup(p);
    p.pw = out;
    std::vector<double> m(192);
    kb_iir_powers_cta(p, m.data(), 0);
    return 0;
}

}  // extern "C"
