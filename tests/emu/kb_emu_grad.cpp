// CPU emulation of the backward passes' kernel bodies (kapre_b200/csrc/grad_core.cuh; tests only, never shipped).
// Compiled with KB_HOST_EMU like kb_emu.cpp: each body runs once per global thread index, atomics become plain
// read-modify-writes.  The transform launches the backward passes reuse are emulated by kb_emu.cpp.
#define KB_HOST_EMU 1
#include <cmath>
#include <cstdlib>
#include <vector>
#include "../../kapre_b200/csrc/kb_tables.h"
#include "../../kapre_b200/csrc/grad_core.cuh"

extern "C" {

// STFT adjoint edge/crop pass over an overlap-add `ola` (B, C, ola_len) contiguous; gx (B, C, L) with the given strides
int kb_emu_stft_adj(const float* G, long long g_sb, long long g_sc, long long g_st, long long g_sk, const float* ola,
                    long long ola_len, float* gx, long long x_sb, long long x_sc, long long x_sl, int B, int C, int L,
                    int T, int n_fft, int hop, int win_eff, int pad_left, const float* w) {
    KbStftAdjParams p{};
    p.G = reinterpret_cast<const float2*>(G); p.g_sb = g_sb; p.g_sc = g_sc; p.g_st = g_st; p.g_sk = g_sk;
    p.ola = ola; p.a_sb = (long long)C * ola_len; p.a_sc = ola_len; p.a_sl = 1;
    p.gx = gx; p.x_sb = x_sb; p.x_sc = x_sc; p.x_sl = x_sl;
    p.B = B; p.C = C; p.L = L; p.T = T; p.n_fft = n_fft; p.hop = hop; p.win_eff = win_eff; p.pad_left = pad_left; p.w = w;
    const long long n = (long long)B * C * L;
    for (long long i = 0; i < n; ++i) kb_stft_adj_elem(p, i);
    return 0;
}

int kb_emu_istft_adj(float* gX, long long sb, long long sc, long long st, long long sk, int B, int C, int T, int n_fft) {
    KbIstftAdjParams p{};
    p.gX = reinterpret_cast<float2*>(gX); p.sb = sb; p.sc = sc; p.st = st; p.sk = sk;
    p.B = B; p.C = C; p.T = T; p.n_fft = n_fft;
    const long long n = (long long)B * C * T * ((n_fft & 1) ? 1 : 2);
    for (long long i = 0; i < n; ++i) kb_istft_adj_elem(p, i);
    return 0;
}

int kb_emu_mag_bwd(const float* X, const float* g, float* gX, long long n) {
    for (long long i = 0; i < n; ++i)
        kb_mag_bwd_elem(reinterpret_cast<const float2*>(X), g, reinterpret_cast<float2*>(gX), i);
    return 0;
}

// the three decibel-backward passes with `chunks` CTAs of `nt` threads per item; ws: 3 * n_items words, zero on entry
int kb_emu_db_bwd(const float* x, const float* g, float* gx, long long n_items, long long item_size, float amin,
                  float db_mul, float db_sub, float dyn_range, float dscale, unsigned int* ws, int chunks, int nt) {
    KbDbBwdParams p{};
    p.x = x; p.g = g; p.gx = gx; p.item_size = item_size; p.ws = ws; p.n_items = n_items;
    p.amin = amin; p.db_mul = db_mul; p.db_sub = db_sub; p.dyn_range = dyn_range; p.dscale = dscale;
    const long long step = (long long)chunks * nt;
    for (int pass = 0; pass < 3; ++pass)
        for (long long item = 0; item < n_items; ++item)
            for (int ch = 0; ch < chunks; ++ch)
                for (int t = 0; t < nt; ++t) {
                    const long long i0 = (long long)ch * nt + t;
                    if (pass == 0) kb_dbb_max(p, item, i0, step, t);
                    else if (pass == 1) kb_dbb_pass(p, item, i0, step, t);
                    else kb_dbb_share(p, item, i0, step);
                }
    return 0;
}

}  // extern "C"
