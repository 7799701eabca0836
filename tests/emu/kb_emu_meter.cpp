// CPU emulation of the loudness-meter bodies (kapre_b200/csrc/meter_core.cuh) and of the gated-loudness passes they
// follow (loudness_core.cuh; tests only, never shipped).  Compiled with KB_HOST_EMU: each phase of a tile runs as a
// loop over its 32 lanes, tiles one after another in the order `order` gives (the result must not depend on it), and
// the passes in the order the library launches them.
#define KB_HOST_EMU 1
#include <cmath>
#include <cstdint>
#include <vector>
#include "../../kapre_b200/csrc/kb_tables.h"
#include "../../kapre_b200/csrc/meter_core.cuh"

static long long kb_emu_meter_tile(long long i, long long n, int order) {
    if (order == 1) return n - 1 - i;
    if (order == 2) {
        const long long half = n / 2;
        return i < half ? 2 * i + 1 : 2 * (i - half);
    }
    return i;
}

static KbLoudParams kb_emu_meter_loud(const float* y, const long long* st, const int* len, int B, int C, int L, int G,
                                      int S) {
    KbLoudParams p{};
    p.y = y;
    if (st) { p.y_sb = st[0]; p.y_sc = st[1]; p.y_sl = st[2]; }
    p.len = len;
    p.B = B; p.C = C; p.L = L; p.G = G; p.S = S;
    kb_loud_setup(p);
    return p;
}

static KbTpParams kb_emu_tp_params(const int* len, int B, int C, int L, const float* taps) {
    KbTpParams p{};
    p.len = len;
    p.B = B; p.C = C; p.L = L;
    kb_tp_setup(p, taps);
    p.tiles = (long long)B * C * p.nseg;
    return p;
}

extern "C" {

// Window counts (Jm, Js) of a shape.
int kb_emu_meter_geometry(int L, int G, int S, int G3, int* out) {
    KbLoudParams p = kb_emu_meter_loud(nullptr, nullptr, nullptr, 1, 1, L, G, S);
    KbLoudParams q = kb_emu_meter_loud(nullptr, nullptr, nullptr, 1, 1, L, G3, S);
    out[0] = p.Jmax; out[1] = q.Jmax;
    return 0;
}

// kapre_loudness_stats on the K-weighted y at element strides st = (b, c, l): integrated (B), momentary (B, Jm),
// short_term (B, Js), lra (B).
int kb_emu_loudness_stats(const float* y, const long long* st, const int* len, int B, int C, int L, int G, int S,
                          int G3, float* integrated, float* momentary, float* short_term, float* lra, int order) {
    KbLoudParams pm = kb_emu_meter_loud(y, st, len, B, C, L, G, S);
    KbLoudParams ps = kb_emu_meter_loud(y, st, len, B, C, L, G3, S);
    std::vector<double> part((size_t)B * pm.K * 2 * C + 1), part3((size_t)B * ps.K * 2 * C + 1);
    std::vector<double> stats((size_t)2 * B + 1), e((size_t)B * ps.Jmax + 1);
    std::vector<unsigned char> mask((size_t)B * pm.Jmax + 1);
    pm.part = part.data(); pm.stats = stats.data(); pm.mask = mask.data(); pm.out = integrated;
    ps.part = part3.data();
    std::vector<kb_f4> smem(kb_loud_smem().total / 16 + kb_lra_smem().total / 16 + 1);
    char* sm = reinterpret_cast<char*>(smem.data());
    pm.tiles = (long long)B * pm.K;
    for (long long i = 0; i < pm.tiles; ++i) kb_loud_energy_tile(pm, sm, kb_emu_meter_tile(i, pm.tiles, order));
    for (long long i = 0; i < B; ++i) kb_loud_gate_tile(pm, sm, kb_emu_meter_tile(i, B, order));
    const long long nm = (long long)B * pm.Jmax;
    for (long long i = 0; i < nm; ++i) kb_meter_series(pm, momentary, nullptr, kb_emu_meter_tile(i, nm, order));
    ps.tiles = (long long)B * ps.K;
    for (long long i = 0; i < ps.tiles; ++i) kb_loud_energy_tile(ps, sm, kb_emu_meter_tile(i, ps.tiles, order));
    const long long ns = (long long)B * ps.Jmax;
    for (long long i = 0; i < ns; ++i) kb_meter_series(ps, short_term, e.data(), kb_emu_meter_tile(i, ns, order));
    for (long long i = 0; i < B; ++i) kb_meter_lra_tile(ps, e.data(), lra, sm, kb_emu_meter_tile(i, B, order));
    return 0;
}

// The range pass alone on given window energies e (B, J) with per-item counts n (null: J): LRA per item.
int kb_emu_lra(const double* e, const int* n, int B, int J, float* lra) {
    KbLoudParams p = kb_emu_meter_loud(nullptr, nullptr, n, B, 1, J, 1, 1);
    std::vector<double> w(e, e + (size_t)B * J);
    std::vector<kb_f4> smem(kb_lra_smem().total / 16 + 1);
    for (long long b = 0; b < B; ++b) kb_meter_lra_tile(p, w.data(), lra, reinterpret_cast<char*>(smem.data()), b);
    return 0;
}

// kapre_true_peak on x at strides st: out (B, C) dBTP; zs, ts (B, C): z[t*] and t*.
int kb_emu_true_peak(const float* x, const long long* st, const int* len, int B, int C, int L, const float* taps,
                     float* out, float* zs, unsigned* ts, int order) {
    KbTpParams p = kb_emu_tp_params(len, B, C, L, taps);
    p.x = x; p.x_sb = st[0]; p.x_sc = st[1]; p.x_sl = st[2];
    std::vector<unsigned long long> key((size_t)p.tiles + 1);
    p.key = key.data(); p.out = out; p.zs = zs; p.ts = ts;
    std::vector<kb_f4> smem(kb_tp_smem().total / 16 + 1);
    char* sm = reinterpret_cast<char*>(smem.data());
    for (long long i = 0; i < p.tiles; ++i) kb_tp_peak_tile(p, sm, kb_emu_meter_tile(i, p.tiles, order));
    const long long cols = (long long)B * C;
    for (long long i = 0; i < cols; ++i) kb_tp_fold_tile(p, sm, kb_emu_meter_tile(i, cols, order));
    return 0;
}

// kapre_true_peak_backward: gx at strides gst from g (B, C) and the forward's zs, ts.
int kb_emu_true_peak_backward(const float* g, const int* len, int B, int C, int L, const float* taps, const float* zs,
                              const unsigned* ts, float* gx, const long long* gst) {
    KbTpParams p = kb_emu_tp_params(len, B, C, L, taps);
    p.g = g; p.zs = const_cast<float*>(zs); p.ts = const_cast<unsigned*>(ts);
    p.gx = gx; p.g_sb = gst[0]; p.g_sc = gst[1]; p.g_sl = gst[2];
    for (long long i = 0; i < (long long)B * C * L; ++i) kb_tp_bwd(p, i);
    return 0;
}

}  // extern "C"
