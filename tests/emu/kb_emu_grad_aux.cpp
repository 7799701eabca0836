// CPU emulation of the adjacent layers' backward bodies (kapre_b200/csrc/grad_aux_core.cuh; tests only, never shipped).
// Compiled with KB_HOST_EMU like kb_emu_grad.cpp: each body runs once per global thread index.
#define KB_HOST_EMU 1
#include <cmath>
#include <cstdlib>
#include <vector>
#include "../../kapre_b200/csrc/kb_tables.h"
#include "../../kapre_b200/csrc/grad_aux_core.cuh"

extern "C" {

long long kb_emu_pad_index(long long t, long long T, int mode) { return kb_pad_index(t, T, mode); }

int kb_emu_phase_bwd(const float* X, const float* g, float* gX, long long n) {
    for (long long i = 0; i < n; ++i)
        kb_phase_bwd_elem(reinterpret_cast<const float2*>(X), g, reinterpret_cast<float2*>(gX), i);
    return 0;
}

// strides: 4 (batch, channel, frame, bin) element strides per tensor; gm / gp may be NULL
int kb_emu_mag_phase_bwd(const float* X, const long long* xs, const float* gm, const long long* ms, const float* gp,
                         const long long* ps, float* gX, const long long* os, long long B, long long C, long long T,
                         long long F, int c_inner) {
    KbMagPhaseBwdParams p{};
    p.X = reinterpret_cast<const float2*>(X); p.x_sb = xs[0]; p.x_sc = xs[1]; p.x_st = xs[2]; p.x_sf = xs[3];
    p.gm = gm; if (gm) { p.m_sb = ms[0]; p.m_sc = ms[1]; p.m_st = ms[2]; p.m_sf = ms[3]; }
    p.gp = gp; if (gp) { p.p_sb = ps[0]; p.p_sc = ps[1]; p.p_st = ps[2]; p.p_sf = ps[3]; }
    p.gX = reinterpret_cast<float2*>(gX); p.o_sb = os[0]; p.o_sc = os[1]; p.o_st = os[2]; p.o_sf = os[3];
    p.C = C; p.T = T; p.F = F; p.c_inner = c_inner;
    const long long n = B * C * T * F;
    for (long long i = 0; i < n; ++i) kb_mag_phase_bwd_elem(p, i);
    return 0;
}

int kb_emu_delta_bwd(const float* g, float* gx, long long outer, long long T, long long inner, int n, float inv_denom,
                     int mode) {
    const long long total = outer * T * inner;
    for (long long i = 0; i < total; ++i) kb_delta_bwd_elem(g, gx, T, inner, n, inv_denom, mode, i);
    return 0;
}

// gs: (b, c, frame, n) strides of g; os: (b, c, sample) strides of gx
int kb_emu_frame_bwd(const float* g, const long long* gs, float* gx, const long long* os, int B, int C, int L, int T,
                     int fl, int hop) {
    KbFrameBwdParams p{};
    p.g = g; p.g_sb = gs[0]; p.g_sc = gs[1]; p.g_st = gs[2]; p.g_sn = gs[3];
    p.gx = gx; p.o_sb = os[0]; p.o_sc = os[1]; p.o_sl = os[2];
    p.C = C; p.L = L; p.T = T; p.fl = fl; p.hop = hop;
    const long long n = (long long)B * C * L;
    for (long long i = 0; i < n; ++i) kb_frame_bwd_elem(p, i);
    return 0;
}

// xs, os: (b, c, sample) strides; gs: (b, c, frame) strides
int kb_emu_energy_bwd(const float* x, const long long* xs, const float* g, const long long* gs, float* gx,
                      const long long* os, int B, int C, int L, int T, int fl, int hop, float scale) {
    KbFrameBwdParams p{};
    p.g = g; p.g_sb = gs[0]; p.g_sc = gs[1]; p.g_st = gs[2];
    p.x = x; p.x_sb = xs[0]; p.x_sc = xs[1]; p.x_sl = xs[2];
    p.gx = gx; p.o_sb = os[0]; p.o_sc = os[1]; p.o_sl = os[2];
    p.C = C; p.L = L; p.T = T; p.fl = fl; p.hop = hop; p.scale2 = 2.0f * scale;
    const long long n = (long long)B * C * L;
    for (long long i = 0; i < n; ++i) kb_energy_bwd_elem(p, i);
    return 0;
}

int kb_emu_concat_fm_bwd(const float* g, float* gx, long long B, long long C, long long T, long long F, int channels_last) {
    const long long n = B * C * T * F;
    for (long long i = 0; i < n; ++i) kb_concat_fm_bwd_elem(g, gx, C, T, F, channels_last, i);
    return 0;
}

}  // extern "C"
