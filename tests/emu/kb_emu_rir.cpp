// CPU emulation of the image-source RIR body (kapre_b200/csrc/rir_core.cuh; tests only, never shipped).  Compiled with
// KB_HOST_EMU: each phase of a CTA runs as a loop over its threads, tiles one after another.
#define KB_HOST_EMU 1
#include <cmath>
#include <cstdint>
#include <vector>
#include "../../kapre_b200/csrc/rir_core.cuh"

extern "C" {

// rec: (B, 14) float64 item records; mic: (B, M, 3); ws: the signed window (W floats); out: (B, M, L) at element
// strides os = (sb, sm, st).  nw: warps per tile (1 .. 8); tile_order = 1 runs the tiles in reverse order.
int kb_emu_rir_ism(const double* rec, const double* mic, int B, int M, int L, int W, double fs, double c,
                   const float* ws, float* out, const long long* os, int nw, int tile_order) {
    if (nw < 1 || nw > KB_RIR_MAX_NW || W < 1 || W > KB_RIR_MAX_W) return -1;
    KbRirParams p{};
    p.rec = rec; p.mic = mic; p.out = out;
    p.o_sb = os[0]; p.o_sm = os[1]; p.o_st = os[2];
    p.B = B; p.M = M; p.L = L; p.W = W; p.nw = nw;
    p.n_tt = (L + 32 * nw - 1) / (32 * nw);
    p.fs = fs; p.c = c;
    for (int k = 0; k < W; ++k) p.ws[k] = ws[k];
    std::vector<kb_f4> smem(kb_rir_smem(32 * nw).total / 16 + 1);
    const long long tiles = (long long)B * M * p.n_tt;
    for (long long i = 0; i < tiles; ++i)
        kb_rir_tile(p, reinterpret_cast<char*>(smem.data()), tile_order ? tiles - 1 - i : i);
    return 0;
}

}  // extern "C"
