// CPU emulation of the PCEN bodies (kapre_b200/csrc/pcen_core.cuh; tests only, never shipped).
// Compiled with KB_HOST_EMU: every pass runs its thread function for each thread index in turn.
#define KB_HOST_EMU 1
#include <cmath>
#include <cstdint>
#include <vector>
#include "../../kapre_b200/csrc/kb_tables.h"
#include "../../kapre_b200/csrc/pcen_core.cuh"

namespace {

// es / ys / ms / gs / os: (batch, channel, frame, band) element strides.  prm: gain, bias, power, smooth_coef
// (host arrays), pst: their element strides (0 or 1).  Tc: frames per chunk (0: the library's unchunked choice).
KbPcenParams kb_emu_pcen_params(const float* E, const long long* es, int B, int C, int T, int F,
                                const float* const* prm, const int* pst, float eps, int Tc) {
    KbPcenParams p{};
    p.E = E; p.e_sb = es[0]; p.e_sc = es[1]; p.e_st = es[2]; p.e_sf = es[3];
    p.gain = prm[0]; p.bias = prm[1]; p.power = prm[2]; p.smooth = prm[3];
    p.gain_st = pst[0]; p.bias_st = pst[1]; p.power_st = pst[2]; p.smooth_st = pst[3];
    p.eps = eps;
    p.B = B; p.C = C; p.T = T; p.F = F;
    p.n_cols = (long long)B * C * F;
    p.c_inner = C > 1 && std::llabs(es[1]) < std::llabs(es[3]) ? 1 : 0;
    kb_pcen_set_chunks(p, 1);
    if (Tc > 0 && T > 0) { p.Tc = Tc; p.K = (T + Tc - 1) / Tc; }
    return p;
}

}  // namespace

extern "C" {

int kb_emu_pcen(const float* E, const long long* es, int B, int C, int T, int F, const float* const* prm,
                const int* pst, float eps, int Tc, float* y, const long long* ys, float* M, const long long* ms) {
    KbPcenParams p = kb_emu_pcen_params(E, es, B, C, T, F, prm, pst, eps, Tc);
    p.y = y; p.y_sb = ys[0]; p.y_sc = ys[1]; p.y_st = ys[2]; p.y_sf = ys[3];
    p.M = M;
    if (M) { p.m_sb = ms[0]; p.m_sc = ms[1]; p.m_st = ms[2]; p.m_sf = ms[3]; }
    if (p.n_cols * T == 0) return 0;
    std::vector<float> state((size_t)p.K * p.n_cols, NAN);
    p.state = state.data();
    for (long long i = 0; i < (long long)(p.K - 1) * p.n_cols; ++i) kb_pcen_fwd_state(p, i);
    for (long long i = 0; i < (long long)p.K * p.n_cols; ++i) kb_pcen_fwd_out(p, i);
    return p.K;
}

// part: (4, K, n_cols) partial sums, K = the returned chunk count (the caller sizes it for ceil(T / Tc) chunks).
int kb_emu_pcen_backward(const float* E, const long long* es, const float* M, const long long* ms, const float* gy,
                         const long long* gs, int B, int C, int T, int F, const float* const* prm, const int* pst,
                         float eps, int Tc, float* gE, const long long* os, float* part) {
    KbPcenParams p = kb_emu_pcen_params(E, es, B, C, T, F, prm, pst, eps, Tc);
    p.M = const_cast<float*>(M); p.m_sb = ms[0]; p.m_sc = ms[1]; p.m_st = ms[2]; p.m_sf = ms[3];
    p.gy = gy; p.g_sb = gs[0]; p.g_sc = gs[1]; p.g_st = gs[2]; p.g_sf = gs[3];
    p.gE = gE; p.o_sb = os[0]; p.o_sc = os[1]; p.o_st = os[2]; p.o_sf = os[3];
    p.part = part;
    if (p.n_cols * T == 0) return 0;
    std::vector<float> state((size_t)p.K * p.n_cols, NAN);
    p.state = state.data();
    for (long long i = 0; i < (long long)(p.K - 1) * p.n_cols; ++i) kb_pcen_bwd_state(p, i);
    for (long long i = 0; i < (long long)p.K * p.n_cols; ++i) kb_pcen_bwd_out(p, i);
    return p.K;
}

int kb_emu_pcen_chunks(long long n_cols, int T, long long resident) { return kb_pcen_chunks(n_cols, T, resident); }

}  // extern "C"
