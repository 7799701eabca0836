// CPU emulation harness for the CUDA kernel bodies (tests only, never shipped).
// Compiles kapre_b200/csrc/*_core.cuh with KB_HOST_EMU so every barrier-free phase runs as a
// loop over the CTA's threads; lets `pytest -m "not gpu"` validate the index arithmetic of
// the fused kernels against the oracle in a container that has no GPU.
#define KB_HOST_EMU 1
#include <cmath>
#include <cstdlib>
#include <cstdio>
#include <vector>
#include "../../kapre_b200/csrc/kb_tables.h"
#include "../../kapre_b200/csrc/stft_core.cuh"
#include "../../kapre_b200/csrc/stft_mc_core.cuh"
#include "../../kapre_b200/csrc/istft_core.cuh"
#include "../../kapre_b200/csrc/aux_core.cuh"
#include "../../kapre_b200/csrc/mr_core.cuh"

template <int Q, int MODE>
static void run_stft_qm(const KbStftParams& p, int n_cta) {
    const bool fbm = (p.mode == KB_OUT_FB || p.mode == KB_OUT_FB_DB) && p.fb_mma;
    const KbStftSmem L = kb_stft_smem_layout(Q, p.n_fft, p.hop, p.TF, p.n_warps, p.mode, p.n_bands,
                                             fbm ? p.n_msteps : p.n_chunks, fbm ? 1 : 0);
    std::vector<char> raw(L.total + 64 + 16);
    char* smem = raw.data() + ((16 - ((uintptr_t)raw.data() & 15)) & 15);
    for (int cta = 0; cta < n_cta; ++cta) {
        std::fill(raw.begin(), raw.end(), (char)0x7f);  // poison: catches reads of unwritten smem
        if constexpr (MODE == KB_OUT_FB || MODE == KB_OUT_FB_DB) {
            if (fbm) { kb_stft_cta<Q, MODE, 1>(p, smem, cta, n_cta); continue; }
        }
        if (p.variant & 2) { kb_stft_cta<Q, MODE, 2>(p, smem, cta, n_cta); continue; }
        kb_stft_cta<Q, MODE>(p, smem, cta, n_cta);
    }
}

template <int Q>
static void run_stft(const KbStftParams& p, int n_cta) {
    switch (p.mode) {
        case KB_OUT_COMPLEX: run_stft_qm<Q, KB_OUT_COMPLEX>(p, n_cta); break;
        case KB_OUT_MAG: run_stft_qm<Q, KB_OUT_MAG>(p, n_cta); break;
        case KB_OUT_MAG_DB: run_stft_qm<Q, KB_OUT_MAG_DB>(p, n_cta); break;
        case KB_OUT_FB: run_stft_qm<Q, KB_OUT_FB>(p, n_cta); break;
        case KB_OUT_FB_DB: run_stft_qm<Q, KB_OUT_FB_DB>(p, n_cta); break;
        case KB_OUT_MAG_PHASE: run_stft_qm<Q, KB_OUT_MAG_PHASE>(p, n_cta); break;
    }
}

template <int Q, int MODE>
static void run_stft_mc_qm(const KbStftParams& p, int n_cta) {
    const KbStftMcSmem L = kb_stft_mc_smem_layout(Q, p.n_fft, p.hop, p.TF, p.C, p.n_warps, p.mc_wh);
    std::vector<char> raw(L.total + 64 + 16);
    char* smem = raw.data() + ((16 - ((uintptr_t)raw.data() & 15)) & 15);
    for (int cta = 0; cta < n_cta; ++cta) {
        std::fill(raw.begin(), raw.end(), (char)0x7f);
        kb_stft_mc_cta<Q, MODE>(p, smem, cta, n_cta);
    }
}

template <int Q, int MODE>
static void run_stft_mcfb_qm(const KbStftParams& p, int n_cta) {
    const KbStftMcFbSmem L = kb_stft_mcfb_smem_layout(Q, p.n_fft, p.hop, p.TF, p.C, p.n_warps, p.mc_wh, p.n_bands,
                                                      p.n_chunks);
    std::vector<char> raw(L.total + 64 + 16);
    char* smem = raw.data() + ((16 - ((uintptr_t)raw.data() & 15)) & 15);
    for (int cta = 0; cta < n_cta; ++cta) {
        std::fill(raw.begin(), raw.end(), (char)0x7f);
        kb_stft_mcfb_cta<Q, MODE>(p, smem, cta, n_cta);
    }
}

template <int Q>
static void run_stft_mc(const KbStftParams& p, int n_cta) {
    switch (p.mode) {
        case KB_OUT_FB: run_stft_mcfb_qm<Q, KB_OUT_FB>(p, n_cta); break;
        case KB_OUT_FB_DB: run_stft_mcfb_qm<Q, KB_OUT_FB_DB>(p, n_cta); break;
        case KB_OUT_COMPLEX: run_stft_mc_qm<Q, KB_OUT_COMPLEX>(p, n_cta); break;
        case KB_OUT_MAG: run_stft_mc_qm<Q, KB_OUT_MAG>(p, n_cta); break;
        case KB_OUT_MAG_DB: run_stft_mc_qm<Q, KB_OUT_MAG_DB>(p, n_cta); break;
        case KB_OUT_MAG_PHASE: run_stft_mc_qm<Q, KB_OUT_MAG_PHASE>(p, n_cta); break;
    }
}

template <int Q>
static void run_istft(const KbIstftParams& p, int n_cta) {
    const KbIstftSmem L = kb_istft_smem_layout(Q, p.n_fft, p.hop, p.win, p.TFc, p.n_warps);
    std::vector<char> smem(L.total + 64);
    for (int cta = 0; cta < n_cta; ++cta) {
        std::fill(smem.begin(), smem.end(), (char)0x7f);
        kb_istft_cta<Q>(p, smem.data(), cta, n_cta);
    }
}

template <int Q>
static void run_istft2(const KbIstftParams& p, int n_cta) {
    const KbIstft2Smem L = kb_istft2_smem_layout(Q, p.n_fft, p.hop, p.win, p.n_warps);
    std::vector<char> smem(L.total + 64);
    for (int cta = 0; cta < n_cta; ++cta) {
        std::fill(smem.begin(), smem.end(), (char)0x7f);
        kb_istft2_cta<Q>(p, smem.data(), cta, n_cta);
    }
}

// The plan's window table (kapre_stft_plan_create): the register form's values for a cosine-sum window, else 0.5 * window.
static void kb_emu_make_wh(const float* window, int win_length, int n_fft, int Q, KbStftParams& p,
                           const std::vector<kb_f4>& cwq, std::vector<float>& wh) {
    if (p.cosw) kb_make_wh_cosw(Q, p.cw_a0, cwq, wh);
    else kb_make_wh(window, win_length, n_fft, wh);
    p.wh = wh.data();
}

extern "C" {

int kb_emu_stft(const float* x, long long x_sb, long long x_sc, long long x_sl, int B, int C, int L,
                int n_fft, int win_length, int hop, int pad_left, int T, const float* window,
                int mode, void* out, long long o_sb, long long o_sc, long long o_st, long long o_sk,
                const float* fb, int n_freq, int n_bands, float amin, float db_mul, float db_sub,
                unsigned int* item_max, int TF, int n_warps, int n_cta, int dbuf, int bulk, long long x_numel,
                int db_on, long long ph_off, int fb_mma) {
    const int Q = kb_q_for_nfft(n_fft);
    if (!Q) return -1;
    if ((mode == KB_OUT_FB || mode == KB_OUT_FB_DB) && TF != n_warps * (32 / Q)) return -2;  // kernel contract
    if (TF % (32 / Q)) return -2;
    std::vector<float> wh;
    std::vector<float2> twp, twn, twn2;
    std::vector<KbBand> bands;
    std::vector<float> fbw;
    std::vector<kb_f4> cw; std::vector<kb_i2> cm; std::vector<int> cg;
    kb_make_twp(Q, twp);
    kb_make_twn(n_fft, twn);
    kb_make_twn2(n_fft, twn2);
    // fb_mma argument: bit 0 tensor-core filterbank, bit 1 band descriptors, bit 2 natural-order pair step (kernel variant 2;
    // the default is the paired-column form)
    const int variant = (fb_mma >> 1) & 2;
    if (fb) { kb_make_bands(fb, n_freq, n_bands, bands, fbw); kb_make_fb_chunks(fb, n_freq, n_bands, 32, cw, cm, cg); }
    KbStftParams p{};
    p.x = x; p.x_sb = x_sb; p.x_sc = x_sc; p.x_sl = x_sl; p.B = B; p.C = C; p.L = L;
    p.n_fft = n_fft; p.hop = hop; p.T = T; p.pad_left = pad_left;
    p.twp = twp.data(); p.twn = twn.data(); p.twn2 = twn2.data();
    std::vector<kb_f4> cwq;
    {
        double ca = 0.0, cb = 0.0;
        if (kb_fit_cosine_window(window, win_length, n_fft, &ca, &cb) && !getenv("KAPRE_B200_NOCOSW")) {
            kb_make_cwq(Q, n_fft, cb, cwq);
            p.cosw = 1; p.cw_a0 = (float)(0.5 * ca); p.cwq = cwq.data();
        }
    }
    kb_emu_make_wh(window, win_length, n_fft, Q, p, cwq, wh);
    p.out = out; p.o_sb = o_sb; p.o_sc = o_sc; p.o_st = o_st; p.o_sk = o_sk; p.mode = mode;
    p.bands = fb ? bands.data() : nullptr; p.fbw = fb ? fbw.data() : nullptr; p.n_bands = fb ? n_bands : 0;
    p.n_fbw = fb ? (int)fbw.size() : 0;
    if (fb) { p.cw = cw.data(); p.cm = cm.data(); p.cg = cg.data(); p.n_chunks = (int)cm.size(); }
    std::vector<kb_i2> bd; std::vector<int> bg;
    if (fb && (fb_mma & 2)) {          // bit 1: two-level band-descriptor walk of the chunk lists
        kb_make_fb_band_desc(cm, cg, 32, bd, bg);
        p.fb_bands = 1; p.bd = bd.data(); p.bg = bg.data(); p.n_bd = (int)bd.size();
    }
    p.variant = variant;
    fb_mma &= 1;
    std::vector<kb_f4> mw; std::vector<kb_i2> ms; std::vector<int> mg;
    if (fb && fb_mma) {
        kb_make_fb_mma(fb, n_freq, n_bands, mw, ms, mg);
        p.fb_mma = 1; p.mw = mw.data(); p.ms = ms.data(); p.mg = mg.data(); p.n_msteps = (int)ms.size();
    }
    p.x_lo = x; p.x_hi = x + x_numel; p.x_numel = x_numel; p.x_align = (unsigned)(((uintptr_t)x >> 2) & 3);
    p.bulk_ok = (bulk && x_sl == 1) ? 1 : 0; p.dbuf = dbuf;
    p.amin = amin; p.db_mul = db_mul; p.db_sub = db_sub; p.item_max = item_max; p.db_on = db_on; p.ph_off = ph_off;
    p.db_ftz = (amin >= 1.17549435e-38f) ? 1 : 0;
    p.TF = TF; p.n_tiles_t = (T + TF - 1) / TF; p.n_warps = n_warps;
    switch (Q) {
        case 4: run_stft<4>(p, n_cta); break;
        case 8: run_stft<8>(p, n_cta); break;
        case 16: run_stft<16>(p, n_cta); break;
        case 32: run_stft<32>(p, n_cta); break;
    }
    return 0;
}

// Multi-channel tiles (stft_mc_core.cuh): TF = time frames per tile, every tile holds all C channels.
int kb_emu_stft_mc(const float* x, long long x_sb, long long x_sc, long long x_sl, int B, int C, int L,
                   int n_fft, int win_length, int hop, int pad_left, int T, const float* window,
                   int mode, void* out, long long o_sb, long long o_sc, long long o_st, long long o_sk,
                   float amin, float db_mul, float db_sub, unsigned int* item_max, int TF, int n_warps, int n_cta,
                   int db_on, long long ph_off, const float* fb, int n_freq, int n_bands) {
    const int Q = kb_q_for_nfft(n_fft);
    if (!Q) return -1;
    const bool fbm = (mode == KB_OUT_FB || mode == KB_OUT_FB_DB);
    if (fbm && (!fb || TF * C > n_warps * (32 / Q) || (32 % n_warps) != 0)) return -2;   // kernel contract
    if (n_warps * (32 / Q) > 32) return -2;
    std::vector<float> wh; std::vector<float2> twp, twn, twn2;
    std::vector<kb_f4> cw; std::vector<kb_i2> cm; std::vector<int> cg;
    if (fbm) kb_make_fb_chunks(fb, n_freq, n_bands, 32, cw, cm, cg);
    kb_make_twp(Q, twp);
    kb_make_twn(n_fft, twn);
    kb_make_twn2(n_fft, twn2);
    KbStftParams p{};
    p.x = x; p.x_sb = x_sb; p.x_sc = x_sc; p.x_sl = x_sl; p.B = B; p.C = C; p.L = L;
    p.n_fft = n_fft; p.hop = hop; p.T = T; p.pad_left = pad_left;
    p.twp = twp.data(); p.twn = twn.data(); p.twn2 = twn2.data();
    std::vector<kb_f4> cwq;
    {
        double ca = 0.0, cb = 0.0;
        if (kb_fit_cosine_window(window, win_length, n_fft, &ca, &cb) && !getenv("KAPRE_B200_NOCOSW")) {
            kb_make_cwq(Q, n_fft, cb, cwq);
            p.cosw = 1; p.cw_a0 = (float)(0.5 * ca); p.cwq = cwq.data();
        }
    }
    kb_emu_make_wh(window, win_length, n_fft, Q, p, cwq, wh);
    p.out = out; p.o_sb = o_sb; p.o_sc = o_sc; p.o_st = o_st; p.o_sk = o_sk; p.mode = mode;
    p.amin = amin; p.db_mul = db_mul; p.db_sub = db_sub; p.item_max = item_max; p.db_on = db_on; p.ph_off = ph_off;
    p.db_ftz = (amin >= 1.17549435e-38f) ? 1 : 0;
    if (fbm) { p.n_bands = n_bands; p.cw = cw.data(); p.cm = cm.data(); p.cg = cg.data(); p.n_chunks = (int)cw.size(); }
    p.TF = TF; p.n_tiles_t = (T + TF - 1) / TF; p.n_warps = n_warps;
    p.mc_wh = (!p.cosw || (hop & 1)) ? 1 : 0;
    p.mc_cl_in = (x_sc < x_sl) ? 1 : 0;
    p.mc_out = (o_sc == 1) ? 1 : 0;
    const int FR = n_warps * (32 / Q), ncol = TF * C;
    const int last = ncol - ((ncol - 1) / FR) * FR;
    p.mc_magic_c = kb_magic((unsigned)C);
    p.mc_magic_g = kb_magic((unsigned)((n_warps * 32) / C));
    p.mc_magic_fr = kb_magic((unsigned)(FR < ncol ? FR : ncol));
    p.mc_magic_last = kb_magic((unsigned)last);
    switch (Q) {
        case 4: run_stft_mc<4>(p, n_cta); break;
        case 8: run_stft_mc<8>(p, n_cta); break;
        case 16: run_stft_mc<16>(p, n_cta); break;
        case 32: run_stft_mc<32>(p, n_cta); break;
    }
    return 0;
}

int kb_emu_istft(const float* X, long long x_sb, long long x_sc, long long x_st, long long x_sk,
                 int B, int C, int T, int n_fft, int win_length, int hop, const float* dual_window,
                 float* y, long long y_sb, long long y_sc, long long y_sl, int TFc, int n_warps, int n_cta) {
    const int Q = kb_q_for_nfft(n_fft);
    if (!Q) return -1;
    std::vector<float> dual;
    std::vector<float2> twp, twn;
    const int win = win_length < n_fft ? win_length : n_fft;
    kb_make_dual(dual_window, win, n_fft, dual);
    kb_make_twp(Q, twp);
    kb_make_twn(n_fft, twn);
    KbIstftParams p{};
    p.X = reinterpret_cast<const float2*>(X); p.x_sb = x_sb; p.x_sc = x_sc; p.x_st = x_st; p.x_sk = x_sk;
    p.B = B; p.C = C; p.T = T; p.n_fft = n_fft; p.hop = hop; p.win = win;
    p.out_len = (T - 1) * hop + win_length;
    p.dual = dual.data(); p.twp = twp.data(); p.twn = twn.data();
    p.y = y; p.y_sb = y_sb; p.y_sc = y_sc; p.y_sl = y_sl;
    p.TFc = TFc; p.R = (win + hop - 1) / hop; p.hops_out = TFc - (p.R - 1);
    p.n_tiles_t = kb_istft_tiles(T, hop, win_length, p.hops_out);
    p.n_warps = n_warps;
    switch (Q) {
        case 4: run_istft<4>(p, n_cta); break;
        case 8: run_istft<8>(p, n_cta); break;
        case 16: run_istft<16>(p, n_cta); break;
        case 32: run_istft<32>(p, n_cta); break;
    }
    return 0;
}


int kb_emu_istft2(const float* X, long long x_sb, long long x_sc, long long x_st, long long x_sk,
                  int B, int C, int T, int n_fft, int win_length, int hop, const float* dual_window,
                  float* y, long long y_sb, long long y_sc, long long y_sl, int seg, int n_warps, int n_cta) {
    const int Q = kb_q_for_nfft(n_fft);
    if (!Q) return -1;
    std::vector<float> dual;
    std::vector<float2> twp, twn;
    const int win = win_length < n_fft ? win_length : n_fft;
    kb_make_dual(dual_window, win, n_fft, dual);
    kb_make_twp(Q, twp);
    kb_make_twn(n_fft, twn);
    KbIstftParams p{};
    p.X = reinterpret_cast<const float2*>(X); p.x_sb = x_sb; p.x_sc = x_sc; p.x_st = x_st; p.x_sk = x_sk;
    p.B = B; p.C = C; p.T = T; p.n_fft = n_fft; p.hop = hop; p.win = win;
    p.out_len = (T - 1) * hop + win_length;
    p.dual = dual.data(); p.twp = twp.data(); p.twn = twn.data();
    p.y = y; p.y_sb = y_sb; p.y_sc = y_sc; p.y_sl = y_sl;
    p.R = (win + hop - 1) / hop; p.seg = seg;
    p.n_tiles_t = kb_istft2_tiles(T, hop, win_length, seg);
    p.n_warps = n_warps;
    switch (Q) {
        case 4: run_istft2<4>(p, n_cta); break;
        case 8: run_istft2<8>(p, n_cta); break;
        case 16: run_istft2<16>(p, n_cta); break;
        case 32: run_istft2<32>(p, n_cta); break;
    }
    return 0;
}


// ---- stand-alone / generic-n_fft kernel bodies (aux_core.cuh) -----------------------------------
int kb_emu_dft(const float* x, long long x_sb, long long x_sc, long long x_sl, int B, int C, int L,
               int n_fft, int win_length, int hop, int pad_left, int T, const float* window, int mode,
               void* out, long long o_sb, long long o_sc, long long o_st, long long o_sk, int n_cta) {
    const int win_eff = win_length < n_fft ? win_length : n_fft;
    std::vector<float2> tw(n_fft);
    for (int r = 0; r < n_fft; ++r) {
        const double a = -2.0 * M_PI * (double)r / (double)n_fft;
        tw[r] = make_float2((float)cos(a), (float)sin(a));
    }
    KbDftParams p{};
    p.x = x; p.x_sb = x_sb; p.x_sc = x_sc; p.x_sl = x_sl; p.B = B; p.C = C; p.L = L;
    p.n_fft = n_fft; p.hop = hop; p.T = T; p.pad_left = pad_left; p.win_eff = win_eff; p.w = window; p.tw = tw.data();
    p.out = out; p.o_sb = o_sb; p.o_sc = o_sc; p.o_st = o_st; p.o_sk = o_sk; p.mode = mode;
    p.n_tiles_t = (T + KB_DFT_TF - 1) / KB_DFT_TF; p.n_warps = 8;
    const KbDftSmem L_ = kb_dft_smem_layout(n_fft, win_eff);
    std::vector<char> smem(L_.total + 64);
    for (int cta = 0; cta < n_cta; ++cta) {
        std::fill(smem.begin(), smem.end(), (char)0x7f);
        kb_dft_cta(p, smem.data(), cta, n_cta);
    }
    return 0;
}

// Mixed-radix Stockham kernel (mr_core.cuh).  Returns -3 when n_fft has a prime factor > 5.
int kb_emu_mr(const float* x, long long x_sb, long long x_sc, long long x_sl, int B, int C, int L,
              int n_fft, int win_length, int hop, int pad_left, int T, const float* window, int mode,
              void* out, long long o_sb, long long o_sc, long long o_st, long long o_sk, int n_warps, int fpw, int n_cta, int group,
              const float* fb, int n_freq, int n_bands, float amin, float db_mul, float db_sub, unsigned int* item_max, int frt) {
    const int win_eff = win_length < n_fft ? win_length : n_fft;
    std::vector<float2> tw(n_fft);
    for (int r = 0; r < n_fft; ++r) {
        const double a = -2.0 * M_PI * (double)r / (double)n_fft;
        tw[r] = make_float2((float)cos(a), (float)sin(a));
    }
    KbMrParams q{};
    KbDftParams& p = q.d;
    p.x = x; p.x_sb = x_sb; p.x_sc = x_sc; p.x_sl = x_sl; p.B = B; p.C = C; p.L = L;
    p.n_fft = n_fft; p.hop = hop; p.T = T; p.pad_left = pad_left; p.win_eff = win_eff; p.w = window; p.tw = tw.data();
    p.out = out; p.o_sb = o_sb; p.o_sc = o_sc; p.o_st = o_st; p.o_sk = o_sk; p.mode = mode; p.n_warps = n_warps;
    q.half = (n_fft & 1) ? 0 : 1;
    q.P = q.half ? n_fft / 2 : n_fft;
    q.n_pass = kb_mr_factor(q.P, q.radix);
    if (q.n_pass < 0) return -3;
    if (group < 1 || n_warps % group) return -4;
    q.G = group;
    q.pad1 = (q.n_pass > 0 && q.radix[0] % 2 == 0) ? 1 : 0;
    q.TF = fpw * (n_warps / group);
    std::vector<KbBand> bands; std::vector<float> fbw;
    const bool fbm = (mode == KB_OUT_FB || mode == KB_OUT_FB_DB);
    if (fbm) {
        if (!fb || n_freq != n_fft / 2 + 1 || frt < 1 || frt % (n_warps / group) || n_warps / group > frt) return -5;
        kb_make_bands(fb, n_freq, n_bands, bands, fbw);
        q.FRT = frt; q.TF = frt; q.bands = bands.data(); q.fbw = fbw.data(); q.n_bands = n_bands;
    }
    q.amin = amin; q.db_mul = db_mul; q.db_sub = db_sub; q.item_max = item_max;
    q.db_ftz = (amin >= 1.17549435e-38f) ? 1 : 0;
    kb_mr_finish(q);
    const KbMrSmem L_ = kb_mr_smem_layout(q.P, n_warps / group, n_fft / 2 + 1, q.n_bands, q.FRT);
    std::vector<char> smem(L_.total + 64);
    for (int cta = 0; cta < n_cta; ++cta) {
        std::fill(smem.begin(), smem.end(), (char)0x7f);
        kb_mr_cta(q, smem.data(), cta, n_cta);
    }
    return 0;
}

int kb_emu_idft(const float* X, long long x_sb, long long x_sc, long long x_st, long long x_sk, int B, int C, int T,
                int n_fft, int win_length, int hop, const float* dual_window, float* y, long long y_sb,
                long long y_sc, long long y_sl, int n_cta) {
    const int win = win_length < n_fft ? win_length : n_fft;
    std::vector<float> dn(win);
    for (int m = 0; m < win; ++m) dn[m] = (float)((double)dual_window[m] / (double)n_fft);
    std::vector<float2> tw(n_fft);
    for (int r = 0; r < n_fft; ++r) {
        const double a = 2.0 * M_PI * (double)r / (double)n_fft;
        tw[r] = make_float2((float)cos(a), (float)sin(a));
    }
    KbIdftParams p{};
    p.X = (const float2*)X; p.x_sb = x_sb; p.x_sc = x_sc; p.x_st = x_st; p.x_sk = x_sk;
    p.B = B; p.C = C; p.T = T; p.n_fft = n_fft; p.hop = hop; p.win = win;
    p.out_len = (T - 1) * hop + win_length; p.dualn = dn.data(); p.tw = tw.data();
    p.y = y; p.y_sb = y_sb; p.y_sc = y_sc; p.y_sl = y_sl;
    p.n_warps = 8; p.n_tiles_s = (p.out_len + 255) / 256;
    std::vector<char> smem((size_t)n_fft * 8 + 64);
    for (int cta = 0; cta < n_cta; ++cta) {
        std::fill(smem.begin(), smem.end(), (char)0x7f);
        kb_idft_cta(p, smem.data(), cta, n_cta);
    }
    return 0;
}

int kb_emu_fb(const float* x, long long x_sb, long long x_sc, long long x_st, long long x_sk, int B, int C, int T,
              const float* fb, int n_freq, int n_bands, float* out, long long o_sb, long long o_sc, long long o_st,
              long long o_sk, int n_cta, int R) {
    std::vector<KbBand> bands; std::vector<float> fbw;
    kb_make_bands(fb, n_freq, n_bands, bands, fbw);
    KbFbParams p{};
    p.x = x; p.x_sb = x_sb; p.x_sc = x_sc; p.x_st = x_st; p.x_sk = x_sk; p.B = B; p.C = C; p.T = T; p.F = n_freq;
    p.bands = bands.data(); p.fbw = fbw.data(); p.n_bands = n_bands;
    p.out = out; p.o_sb = o_sb; p.o_sc = o_sc; p.o_st = o_st; p.o_sk = o_sk;
    p.R = R; p.n_tiles_t = (T + R - 1) / R; p.n_warps = 8;
    const KbFbSmem L_ = kb_fb_smem_layout(n_freq, n_bands, R);
    std::vector<char> smem(L_.total + 64);
    for (int cta = 0; cta < n_cta; ++cta) {
        std::fill(smem.begin(), smem.end(), (char)0x7f);
        kb_fb_cta(p, smem.data(), cta, n_cta);
    }
    return 0;
}

// The plan's window tables: wh (n_fft floats), and for a cosine-sum window cwq (4 * Q floats) and a0.  Returns cosw.
int kb_emu_window_tables(const float* window, int win_length, int n_fft, float* wh_out, float* cwq_out, float* a0_out) {
    const int Q = kb_q_for_nfft(n_fft);
    if (!Q) return -1;
    KbStftParams p{};
    std::vector<kb_f4> cwq;
    std::vector<float> wh;
    double ca = 0.0, cb = 0.0;
    if (kb_fit_cosine_window(window, win_length, n_fft, &ca, &cb)) {
        kb_make_cwq(Q, n_fft, cb, cwq);
        p.cosw = 1; p.cw_a0 = (float)(0.5 * ca);
        for (int q = 0; q < Q; ++q) std::memcpy(cwq_out + 4 * q, &cwq[q], 16);
        *a0_out = p.cw_a0;
    }
    kb_emu_make_wh(window, win_length, n_fft, Q, p, cwq, wh);
    std::memcpy(wh_out, wh.data(), (size_t)n_fft * 4);
    return p.cosw;
}

// Shared memory of the single-channel kernel at a tile shape (kb_stft_smem_layout), for enumerating the shapes the
// launcher may pick; n_chunks is the filterbank's chunk count (kb_make_fb_chunks over 32 lane groups).
int kb_emu_stft_smem(int n_fft, int hop, int TF, int n_warps, int mode, int n_bands, int n_chunks) {
    const int Q = kb_q_for_nfft(n_fft);
    if (!Q) return -1;
    return kb_stft_smem_layout(Q, n_fft, hop, TF, n_warps, mode, n_bands, n_chunks, 0).total;
}

int kb_emu_fb_chunks(const float* fb, int n_freq, int n_bands) {
    std::vector<kb_f4> cw; std::vector<kb_i2> cm; std::vector<int> cg;
    kb_make_fb_chunks(fb, n_freq, n_bands, 32, cw, cm, cg);
    return (int)cm.size();
}

// The fused kernels' decibel tail on an array: db_mul * log2(max(x, amin)) - db_sub, with the same host stand-in for
// the device log2 as the kernel bodies, so MODE_*_DB can be compared bit for bit with the tail applied to MODE_MAG / MODE_FB.
void kb_emu_db_tail(const float* x, float* out, long long n, float amin, float db_mul, float db_sub) {
    for (long long i = 0; i < n; ++i) out[i] = db_mul * kb_log2(kb_floor_keepnan(x[i], amin)) - db_sub;
}

// The host model of the async staging primitives (stft_core.cuh) against known misuses, each on a private buffer.
// Returns a bit per case that the model caught: 0 wrong parity, 1 read before the wait (the read sees the NaN fill),
// 2 second arrive.expect_tx in one phase, 3 misaligned destination, source or size, 4 size 0 or >= 2^20, 5 wait that
// would hang, 6 re-initialisation with a copy in flight, 7 exit with a copy in flight; bit 8: three phases of the
// correct protocol land their data with no violation.  Leaves the model reset.
int kb_emu_async_selftest() {
    alignas(16) static float src[64];
    alignas(16) static float dst[68];
    alignas(16) static KbBar bar;
    for (int i = 0; i < 64; ++i) src[i] = (float)i;
    int flagged = 0;
    auto after = [&](int bit, auto&& play) {
        kb_emu_async_reset();
        play();
        if (kb_emu_async_violations() > 0) flagged |= 1 << bit;
        kb_emu_async_reset();
    };
    after(0, [&] { kb_bar_init(&bar, 1); kb_bulk_g2s(dst, src, 64, &bar); kb_bar_wait(&bar, 1); kb_bar_wait(&bar, 0); });
    {
        kb_emu_async_reset();
        kb_bar_init(&bar, 1);
        kb_bulk_g2s(dst, src, 64, &bar);
        const float early = dst[3];
        kb_bar_wait(&bar, 0);
        if (std::isnan(early) && dst[3] == 3.0f && kb_emu_async_violations() == 0) flagged |= 1 << 1;
        kb_emu_async_reset();
    }
    after(2, [&] { kb_bar_init(&bar, 1); kb_bulk_g2s(dst, src, 32, &bar); kb_bulk_g2s(dst + 8, src + 8, 32, &bar);
                   kb_bar_wait(&bar, 0); });
    {
        int caught = 0;
        after(3, [&] { kb_bar_init(&bar, 1); kb_bulk_g2s(dst + 1, src, 64, &bar); kb_bar_wait(&bar, 0); });
        caught += (flagged >> 3) & 1; flagged &= ~(1 << 3);
        after(3, [&] { kb_bar_init(&bar, 1); kb_bulk_g2s(dst, src + 2, 64, &bar); kb_bar_wait(&bar, 0); });
        caught += (flagged >> 3) & 1; flagged &= ~(1 << 3);
        after(3, [&] { kb_bar_init(&bar, 1); kb_bulk_g2s(dst, src, 60, &bar); kb_bar_wait(&bar, 0); });
        caught += (flagged >> 3) & 1; flagged &= ~(1 << 3);
        if (caught == 3) flagged |= 1 << 3;
    }
    {
        int caught = 0;
        after(4, [&] { kb_bar_init(&bar, 1); kb_bulk_g2s(dst, src, 0, &bar); });
        caught += (flagged >> 4) & 1; flagged &= ~(1 << 4);
        after(4, [&] { kb_bar_init(&bar, 1); kb_bulk_g2s(dst, src, 1 << 20, &bar); });
        caught += (flagged >> 4) & 1; flagged &= ~(1 << 4);
        if (caught == 2) flagged |= 1 << 4;
    }
    after(5, [&] { kb_bar_init(&bar, 1); kb_bulk_g2s(dst, src, 64, &bar); kb_bar_wait(&bar, 0); kb_bar_wait(&bar, 1);
                   kb_bar_wait(&bar, 1); });
    after(6, [&] { kb_bar_init(&bar, 1); kb_bulk_g2s(dst, src, 64, &bar); kb_bar_init(&bar, 1); kb_bulk_g2s(dst, src, 64, &bar);
                   kb_bar_wait(&bar, 0); });
    after(7, [&] { kb_bar_init(&bar, 1); kb_bulk_g2s(dst, src, 64, &bar); });
    {
        kb_emu_async_reset();
        kb_bar_init(&bar, 1);
        bool ok = true;
        for (int k = 0; k < 3; ++k) {
            kb_bulk_g2s(dst + 4 * k, src + 16 * k, 64, &bar);
            for (unsigned w = 0; w < 4; ++w) kb_bar_wait(&bar, (unsigned)k & 1u);   // every thread of a phase waits
            for (int i = 0; i < 16; ++i) ok = ok && dst[4 * k + i] == src[16 * k + i];
        }
        if (ok && kb_emu_async_violations() == 0) flagged |= 1 << 8;
        kb_emu_async_reset();
    }
    return flagged;
}

// kb_cabs (|X| over the whole float range) on arrays: rn = 1 the correctly rounded form, 0 the kb_sqrt(cnorm) form
void kb_emu_cabs(const float* re, const float* im, float* out, long long n, int rn) {
    for (long long i = 0; i < n; ++i) out[i] = rn ? kb_cabs<true>(re[i], im[i]) : kb_cabs<false>(re[i], im[i]);
}

// kb_atan2 (the Phase outputs' polynomial atan2) on arrays, for the accuracy test
void kb_emu_atan2(const float* y, const float* x, float* out, long long n) {
    for (long long i = 0; i < n; ++i) out[i] = kb_atan2(y[i], x[i]);
}

}  // extern "C"
