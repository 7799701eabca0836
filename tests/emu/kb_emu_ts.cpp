// CPU emulation of the time-stretch bodies (kapre_b200/csrc/ts_core.cuh; tests only, never shipped).
// Compiled with KB_HOST_EMU: every pass runs its thread function for each thread index in turn.
#define KB_HOST_EMU 1
#include <cmath>
#include <cstdint>
#include <vector>
#include "../../kapre_b200/csrc/kb_tables.h"
#include "../../kapre_b200/csrc/ts_core.cuh"

namespace {

// xs: (batch, channel, frame, bin) element strides of X (complex elements).  Tc: frames per chunk (0: one chunk).
KbTsParams kb_emu_ts_params(const float* X, const long long* xs, int B, int C, int T, int F, double rate, int Tc) {
    KbTsParams p{};
    p.X = (const float2*)X; p.x_sb = xs[0]; p.x_sc = xs[1]; p.x_st = xs[2]; p.x_sf = xs[3];
    p.rate = rate; p.inv_rate = 1.0 / rate;
    p.B = B; p.C = C; p.T = T; p.F = F;
    p.T_out = (int)std::ceil((double)T / rate);
    p.n_cols = (long long)B * C * F;
    p.c_inner = C > 1 && std::llabs(xs[1]) < std::llabs(xs[3]) ? 1 : 0;
    kb_ts_set_chunks(p, 1);
    if (Tc > 0 && T > 0) { p.Tc = Tc; p.K = (T + Tc - 1) / Tc; }
    return p;
}

}  // namespace

extern "C" {

// Returns the chunk count used (0 when there is nothing to do).
int kb_emu_ts(const float* X, const long long* xs, int B, int C, int T, int F, double rate, int Tc, float* Y,
              const long long* ys) {
    KbTsParams p = kb_emu_ts_params(X, xs, B, C, T, F, rate, Tc);
    p.Y = (float2*)Y; p.y_sb = ys[0]; p.y_sc = ys[1]; p.y_st = ys[2]; p.y_sf = ys[3];
    if (p.n_cols * p.T_out == 0) return 0;
    std::vector<unsigned> state((size_t)p.K * p.n_cols, 0xdeadbeefu);
    p.state = state.data();
    for (long long i = 0; i < (long long)(p.K - 1) * p.n_cols; ++i) kb_ts_fwd<false>(p, i);
    for (long long i = 0; i < (long long)p.K * p.n_cols; ++i) kb_ts_fwd<true>(p, i);
    return p.K;
}

int kb_emu_ts_backward(const float* X, const long long* xs, const float* Y, const long long* ys, const float* G,
                       const long long* gs, int B, int C, int T, int F, double rate, int Tc, float* gX,
                       const long long* os) {
    KbTsParams p = kb_emu_ts_params(X, xs, B, C, T, F, rate, Tc);
    p.Y = (float2*)const_cast<float*>(Y); p.y_sb = ys[0]; p.y_sc = ys[1]; p.y_st = ys[2]; p.y_sf = ys[3];
    p.G = (const float2*)G; p.g_sb = gs[0]; p.g_sc = gs[1]; p.g_st = gs[2]; p.g_sf = gs[3];
    p.gX = (float2*)gX; p.o_sb = os[0]; p.o_sc = os[1]; p.o_st = os[2]; p.o_sf = os[3];
    if (p.n_cols * T == 0) return 0;
    std::vector<float> state((size_t)p.K * p.n_cols, NAN);
    p.state = state.data();
    for (long long i = 0; i < (long long)(p.K - 1) * p.n_cols; ++i) kb_ts_bwd_state(p, i);
    for (long long i = 0; i < (long long)p.K * p.n_cols; ++i) kb_ts_bwd_out(p, i);
    return p.K;
}

int kb_emu_ts_chunks(long long n_cols, int T, long long resident) { return kb_ts_chunks(n_cols, T, resident); }

}  // extern "C"
