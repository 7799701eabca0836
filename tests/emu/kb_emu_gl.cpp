// CPU emulation of the Griffin-Lim element passes (kapre_b200/csrc/gl_core.cuh; tests only, never shipped).
// Compiled with KB_HOST_EMU: each pass runs its element function for every index in turn.
#define KB_HOST_EMU 1
#include <cmath>
#include <cstdint>
#include <vector>
#include "../../kapre_b200/csrc/kb_tables.h"
#include "../../kapre_b200/csrc/gl_core.cuh"

namespace {

// ss: (batch, channel, frame, bin) element strides of S.
KbGlParams kb_emu_gl_params(const float* S, const long long* ss, int B, int C, int T, int F) {
    KbGlParams p{};
    p.S = S; p.s_sb = ss[0]; p.s_sc = ss[1]; p.s_st = ss[2]; p.s_sf = ss[3];
    p.C = C; p.T = T; p.F = F;
    p.n = (long long)B * C * T * F;
    return p;
}

}  // namespace

extern "C" {

// X: contiguous (B, C, T, F) complex64 (interleaved float pairs).
void kb_emu_gl_init(const float* S, const long long* ss, int B, int C, int T, int F, int init, unsigned long long seed,
                    float* X) {
    KbGlParams p = kb_emu_gl_params(S, ss, B, C, T, F);
    p.init = init; p.seed = seed; p.X = (float2*)X;
    for (long long i = 0; i < p.n; ++i) kb_gl_init_elem(p, i);
}

// Yprev may be null, and X may be Yprev (the in-place update the library runs).
void kb_emu_gl_project(const float* S, const long long* ss, int B, int C, int T, int F, const float* Y,
                       const float* Yprev, float beta, float* X) {
    KbGlParams p = kb_emu_gl_params(S, ss, B, C, T, F);
    p.Y = (const float2*)Y; p.Yprev = (const float2*)Yprev; p.beta = beta; p.X = (float2*)X;
    for (long long i = 0; i < p.n; ++i) kb_gl_project_elem(p, i);
}

float kb_emu_gl_u(unsigned long long seed, long long i) { return kb_gl_u(seed, i); }

void kb_emu_gl_phasor(float u, float* s, float* c) { kb_gl_phasor(u, s, c); }

}  // extern "C"
