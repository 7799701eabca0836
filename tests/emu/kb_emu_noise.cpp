// CPU emulation of the additive-noise bodies (kapre_b200/csrc/noise_core.cuh; tests only, never shipped).  Compiled with
// KB_HOST_EMU: each phase of a tile runs as a loop over its 32 lanes, tiles one after another in the order `order`
// gives (the result must not depend on it), the segment-sum pass before the output pass, as the library launches them.
#define KB_HOST_EMU 1
#include <cmath>
#include <cstdint>
#include <vector>
#include "../../kapre_b200/csrc/kb_tables.h"
#include "../../kapre_b200/csrc/noise_core.cuh"

extern "C" {

// st: element strides (b, c, l) of x, the noise, y, xr and gn (15 values); a batch or channel of 1 in the noise is
// broadcast by the caller through stride 0.  noise == null: bank mode (bank, bank_numel, start, clip, offset).
// ss: snr strides (b, c) and length strides (b, c).  bwd = 0: y = add_noise(x), stats (optional) receives (Ex, En).
// bwd = 1: x is g, y receives gx, xr is the forward's x, stats is read, gn and gsnr are optional.
// order: 0 ascending tiles, 1 descending, 2 a fixed permutation (odd tiles first).
int kb_emu_add_noise(const float* x, const float* noise, const float* bank, long long bank_numel, const long long* start,
                     const long long* clip, const long long* offset, const float* snr, const int* len,
                     const long long* st, const long long* ss, float* y, double* stats, int B, int C, int L, int bwd,
                     const float* xr, float* gn, float* gsnr, int order) {
    KbNoiseParams p{};
    p.x = {x, st[0], st[1], st[2]};
    p.n = {noise, st[3], st[4], st[5]};
    p.bank = bank; p.bank_numel = bank_numel; p.start = start; p.clip = clip; p.offset = offset;
    p.y = y; p.y_sb = st[6]; p.y_sc = st[7]; p.y_sl = st[8];
    p.xr = {xr, st[9], st[10], st[11]};
    p.gn = gn; p.gn_sb = st[12]; p.gn_sc = st[13]; p.gn_sl = st[14];
    p.gsnr = gsnr;
    p.snr = snr; p.snr_sb = ss[0]; p.snr_sc = ss[1];
    p.len = len; p.len_sb = ss[2]; p.len_sc = ss[3];
    p.stats = stats;
    p.B = B; p.C = C; p.L = L; p.bwd = bwd;
    kb_noise_setup(p);
    if (p.tiles == 0) return 0;
    std::vector<double> part((size_t)B * C * p.nseg * 2);
    p.part = part.data();
    std::vector<kb_f4> smem(kb_noise_smem(kb_noise_cg_max(p)).total / 16 + 1);
    char* sm = reinterpret_cast<char*>(smem.data());
    auto tile_at = [&](long long i) -> long long {
        if (order == 1) return p.tiles - 1 - i;
        if (order == 2) {
            const long long half = p.tiles / 2;
            return i < half ? 2 * i + 1 : 2 * (i - half);
        }
        return i;
    };
    for (long long i = 0; i < p.tiles; ++i) kb_noise_sum_tile(p, sm, tile_at(i));
    for (long long i = 0; i < p.tiles; ++i) kb_noise_out_tile(p, sm, tile_at(i));
    return 0;
}

int kb_emu_noise_consts(int* out) {
    out[0] = KB_NOISE_SEG; out[1] = KB_NOISE_R; out[2] = KB_NOISE_G;
    return 0;
}

}  // extern "C"
