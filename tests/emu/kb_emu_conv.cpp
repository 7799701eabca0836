// CPU emulation of the spectral multiply-accumulate body (kapre_b200/csrc/conv_core.cuh; tests only, never shipped).
// Compiled with KB_HOST_EMU: each phase of the CTA body runs as a loop over its threads, CTAs one after another.
#define KB_HOST_EMU 1
#include <cmath>
#include <cstdint>
#include <vector>
#include "../../kapre_b200/csrc/kb_tables.h"
#include "../../kapre_b200/csrc/conv_core.cuh"

extern "C" {

// a, b, out: complex64 (interleaved float pairs) with (batch, channel, frame, bin) element strides as / bs / os.
// correlate = 0: out[i] = sum_s a[s] b[i - s]; 1: out[i] = sum_s conj(a[s]) b[i + s].
int kb_emu_spec_conv(const float* a, const long long* as, int S, const float* b, const long long* bs, int Tb, float* out,
                     const long long* os, int Bn, int C, int F, int To, int correlate, int n_threads, int n_cta) {
    KbConvParams p{};
    p.a = reinterpret_cast<const float2*>(a); p.a_sb = as[0]; p.a_sc = as[1]; p.a_st = as[2]; p.a_sf = as[3];
    p.b = reinterpret_cast<const float2*>(b); p.b_sb = bs[0]; p.b_sc = bs[1]; p.b_st = bs[2]; p.b_sf = bs[3];
    p.out = reinterpret_cast<float2*>(out); p.o_sb = os[0]; p.o_sc = os[1]; p.o_st = os[2]; p.o_sf = os[3];
    p.Bn = Bn; p.C = C; p.F = F; p.S = S; p.Tb = Tb; p.To = To; p.correlate = correlate;
    if (n_threads % 32 || n_threads / 32 * KB_CONV_R != KB_CONV_NO) return -1;     // the body assumes its CTA shape
    if (!kb_conv_setup(p, n_threads)) return -2;
    std::vector<kb_f4> smem(KB_CONV_SMEM / 16 + 1);
    for (int cta = 0; cta < n_cta; ++cta) kb_conv_cta(p, reinterpret_cast<char*>(smem.data()), cta, n_cta);
    return 0;
}

long long kb_emu_conv_block_size(long long K) { return kb_conv_block_size(K); }

}  // extern "C"
