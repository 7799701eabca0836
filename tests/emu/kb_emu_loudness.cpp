// CPU emulation of the gated-loudness bodies (kapre_b200/csrc/loudness_core.cuh; tests only, never shipped).  Compiled
// with KB_HOST_EMU: each phase of a tile runs as a loop over its 32 lanes, tiles one after another in the order `order`
// gives (the result must not depend on it), the energy pass before the gate pass, as the library launches them.
#define KB_HOST_EMU 1
#include <cmath>
#include <cstdint>
#include <vector>
#include "../../kapre_b200/csrc/kb_tables.h"
#include "../../kapre_b200/csrc/loudness_core.cuh"

static long long kb_emu_loud_tile(long long i, long long n, int order) {
    if (order == 1) return n - 1 - i;
    if (order == 2) {
        const long long half = n / 2;
        return i < half ? 2 * i + 1 : 2 * (i - half);
    }
    return i;
}

static KbLoudParams kb_emu_loud_params(const float* y, const long long* st, const int* len, int B, int C, int L, int G,
                                       int S) {
    KbLoudParams p{};
    p.y = y; p.y_sb = st[0]; p.y_sc = st[1]; p.y_sl = st[2];
    p.len = len;
    p.B = B; p.C = C; p.L = L; p.G = G; p.S = S;
    kb_loud_setup(p);
    return p;
}

extern "C" {

// y: the K-weighted signal at element strides st = (b, c, l); len: per-item lengths or null.  out: B LKFS values;
// stats: B (E2, |J2|) pairs; mask: B x Jmax decisions (Jmax from kb_emu_loudness_geometry); part (optional, B x K x 2
// x C) receives the piece sums.  order: 0 ascending tiles, 1 descending, 2 a fixed permutation (odd tiles first).
int kb_emu_loudness(const float* y, const long long* st, const int* len, int B, int C, int L, int G, int S, float* out,
                    double* stats, unsigned char* mask, double* part_out, int order) {
    KbLoudParams p = kb_emu_loud_params(y, st, len, B, C, L, G, S);
    std::vector<double> part((size_t)B * p.K * 2 * C + 1);
    p.part = part.data(); p.out = out; p.stats = stats; p.mask = mask;
    std::vector<kb_f4> smem(kb_loud_smem().total / 16 + 1);
    char* sm = reinterpret_cast<char*>(smem.data());
    p.tiles = (long long)B * p.K;
    for (long long i = 0; i < p.tiles; ++i) kb_loud_energy_tile(p, sm, kb_emu_loud_tile(i, p.tiles, order));
    for (long long i = 0; i < B; ++i) kb_loud_gate_tile(p, sm, kb_emu_loud_tile(i, B, order));
    if (part_out)
        for (size_t i = 0; i + 1 < part.size(); ++i) part_out[i] = part[i];
    return 0;
}

// gy at strides gst from the forward's stats and mask and the per-item output gradient gl.
int kb_emu_loudness_backward(const float* gl, const float* y, const long long* st, const int* len, int B, int C, int L,
                             int G, int S, const double* stats, const unsigned char* mask, float* gy,
                             const long long* gst, int order) {
    KbLoudParams p = kb_emu_loud_params(y, st, len, B, C, L, G, S);
    p.gl = gl; p.gy = gy; p.g_sb = gst[0]; p.g_sc = gst[1]; p.g_sl = gst[2];
    p.stats = const_cast<double*>(stats);
    p.mask = const_cast<unsigned char*>(mask);
    std::vector<kb_f4> smem(kb_loud_smem().total / 16 + 1);
    char* sm = reinterpret_cast<char*>(smem.data());
    p.tiles = (long long)B * p.Kb;
    for (long long i = 0; i < p.tiles; ++i) kb_loud_bwd_tile(p, sm, kb_emu_loud_tile(i, p.tiles, order));
    return 0;
}

// (rho, m, Jmax, K, Kb) of a shape.
int kb_emu_loudness_geometry(int L, int G, int S, int* out) {
    KbLoudParams p{};
    p.B = 1; p.C = 1; p.L = L; p.G = G; p.S = S;
    kb_loud_setup(p);
    out[0] = p.rho; out[1] = p.m; out[2] = p.Jmax; out[3] = p.K; out[4] = p.Kb;
    return 0;
}

}  // extern "C"
