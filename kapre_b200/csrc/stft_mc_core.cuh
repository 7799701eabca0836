// Multi-channel variant of the fused forward kernel for interleaved ("channels_last") tensors.
//
// kapre's default data format keeps the channel axis innermost: waveforms (batch, time, ch)
// and spectrograms (batch, time, freq, ch)  (kapre/time_frequency.py:164-187 transposes around
// tf.signal.stft).  With one (batch, channel) signal per tile (stft_core.cuh) such a tensor is
// read with a stride of C floats and -- worse -- written 4 bytes at a time C floats apart, so
// every 32-byte sector is touched C times.  Here a tile is TF time frames of ALL C channels of
// one batch item:
//   * the interleaved sample span is read once, fully coalesced, and de-interleaved into planar
//     shared memory [channel][sample]; every (frame, channel) "column" then runs the same
//     register FFT as the single-channel kernel;
//   * for interleaved outputs the real-FFT pair step is done cooperatively by the whole CTA
//     with the lanes running over (channel fastest, bin) so that stores are contiguous
//     (bin, channel) rows; planar outputs keep the per-warp epilogue.
// Modes: complex, magnitude, magnitude dB, magnitude+phase (the filterbank modes stay on the
// single-channel kernel).
#pragma once
#include "stft_core.cuh"

struct KbStftMcSmem {
    int wh, twp, twn, cwq, ci, samples, ex, total;   // byte offsets
    int span, spanp, exw;
};

struct KbColInfo {        // one per column of the current round, written in phase 1
    long long ooff;       // element offset of (batch, frame, bin 0, channel) in the output
    int zoff;             // complex offset of the column's natural-order spectrum in the exchange buffer
    int valid;
};

// Exchange-region geometry of this kernel.  The cooperative pair step reads the natural-order spectra
// of consecutive columns at (almost) the same bin from consecutive lanes, so column c's spectrum is
// placed 3*c (mod 16) complex slots into the banks: frame stride P + 3 inside a region, region stride
// 32*33 + (3*FPW mod 16 ...).  Both still hold the 32 x 33 transpose and FPW natural-order spectra.
KB_HD int kb_mc_zstr(int Q) { return 32 * Q + 3; }
KB_HD int kb_mc_exw(int Q) {
    const int FPW = 32 / Q;
    int e = (3 * FPW) % 16;
    while (32 * 33 + e < FPW * kb_mc_zstr(Q)) e += 16;
    return 32 * 33 + e;
}

KB_HD KbStftMcSmem kb_stft_mc_smem_layout(int Q, int n_fft, int hop, int TFt, int C, int n_warps, int with_wh) {
    KbStftMcSmem s;
    const int P = 32 * Q;
    int off = 0;
    s.wh = off;  if (with_wh) off += kb_align16(n_fft * 4);
    s.twp = off; off += kb_align16(Q * 33 * 8);
    s.twn = off; off += kb_align16((P / 2) * 8);
    s.cwq = off; off += Q * 16;
    s.ci = off;  off += 32 * (int)sizeof(KbColInfo);
    s.span = (TFt - 1) * hop + n_fft;
    // plane stride: even (8 B-aligned planes) and == 2*round(16/C) mod 32, so that the de-interleaving
    // stores of 32 consecutive (sample, channel) pairs spread over the banks
    {
        int want = 2 * ((16 + C / 2) / C);
        if (want < 2) want = 2;
        int sp = (s.span + 1) & ~1;
        sp += ((want - sp) % 32 + 32) % 32;
        s.spanp = sp;
    }
    s.samples = off; off += kb_align16(C * s.spanp * 4);
    s.exw = kb_mc_exw(Q);
    s.ex = off;  off += kb_align16(n_warps * s.exw * 8);
    s.total = off;
    return s;
}

// x / d for x * d < 2^32 with magic = ceil(2^32 / d) (d > 1)
KB_HD unsigned kb_magic(unsigned d) { return d > 1 ? (unsigned)((0x100000000ULL + d - 1) / d) : 0u; }
#if defined(KB_HOST_EMU)
static inline unsigned kb_mulhi(unsigned a, unsigned b) { return (unsigned)(((unsigned long long)a * b) >> 32); }
#else
KB_D unsigned kb_mulhi(unsigned a, unsigned b) { return __umulhi(a, b); }
#endif
#if defined(KB_HOST_EMU)
static inline int kb_fdiv(int x, int d, unsigned magic) { return d == 1 ? x : (int)kb_mulhi((unsigned)x, magic); }
#else
KB_D int kb_fdiv(int x, int d, unsigned magic) { return d == 1 ? x : (int)kb_mulhi((unsigned)x, magic); }
#endif

// 4-byte asynchronous global -> shared copy (LDGSTS); !ok writes a zero without reading.
#if defined(KB_HOST_EMU)
static inline void kb_cp_async4(float* dst, const float* src, bool ok) { *dst = ok ? *src : 0.0f; }
static inline void kb_cp_async_wait() {}
#else
KB_D void kb_cp_async4(float* dst, const float* src, bool ok) {
    const int sz = ok ? 4 : 0;
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(kb_smem_u32(dst)), "l"(src), "r"(sz) : "memory");
}
KB_D void kb_cp_async_wait() { asm volatile("cp.async.wait_all;" ::: "memory"); }
#endif

// De-interleaving loads of one tile (all threads).  Every thread owns ONE channel and walks its samples
// with a fixed step, so the loop body is a compare, two pointer bumps and the copy:
//   interleaved input: thread -> (channel = tid % C, first sample tid / C), step S / C with S the largest
//                      multiple of C below the CTA size  (consecutive threads = consecutive addresses);
//   planar input:      thread -> (channel = tid / G, first sample tid % G), step G = CTA size / C.
// Samples outside the signal (pad_begin / pad_end / tails) are stored as zeros.
#if defined(KB_HOST_EMU)
inline void kb_mc_issue_loads(const KbStftParams& p, float* smp, int b, int t0, int span, int spanp, int tid, int nt)
#else
__device__ __forceinline__ void kb_mc_issue_loads(const KbStftParams& p, float* smp, int b, int t0, int span,
                                                  int spanp, int tid, int nt)
#endif
{
    const int C = p.C;
    const int G = kb_fdiv(nt, C, p.mc_magic_c);          // threads per channel
    int c, i0;
    if (p.mc_cl_in) { i0 = kb_fdiv(tid, C, p.mc_magic_c); c = tid - i0 * C; if (i0 >= G) return; }
    else { c = kb_fdiv(tid, G, p.mc_magic_g); i0 = tid - c * G; if (c >= C) return; }
    const int s_first = t0 * p.hop - p.pad_left;
    int v0 = -s_first, v1 = p.L - s_first;               // valid samples of the tile: [v0, v1)
    if (v0 < 0) v0 = 0;
    if (v1 > span) v1 = span;
    const unsigned vr = v1 > v0 ? (unsigned)(v1 - v0) : 0u;
    const float* src = p.x + (long long)b * p.x_sb + (long long)c * p.x_sc + (long long)(s_first + i0) * p.x_sl;
    const long long sstep = (long long)G * p.x_sl;
    float* dst = smp + c * spanp;
    if (v0 == 0 && v1 >= span) {
        // whole tile inside the signal (all but the first / last tiles of an item): no per-sample bounds test, the shared
        // address is stepped as a 32-bit offset -- 4 instructions per sample instead of 13 (ncu on cfg3: the loader was
        // 29 % of the kernel's instructions)
#if defined(KB_HOST_EMU)
        for (int i = i0; i < span; i += G) { dst[i] = *src; src += sstep; }
#else
        unsigned d = kb_smem_u32(dst + i0);
        const unsigned dstep = (unsigned)G * 4u;
#pragma unroll 8
        for (int i = i0; i < span; i += G) {
            asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(d), "l"(src) : "memory");
            d += dstep;
            src += sstep;
        }
#endif
        return;
    }
#pragma unroll 4
    for (int i = i0; i < span; i += G) {
        if ((unsigned)(i - v0) < vr) kb_cp_async4(dst + i, src, true);
        else dst[i] = 0.0f;
        src += sstep;
    }
}

// One output pair (bins k and P - k, or the self-paired bin P / 2) of one column.
// X2 arrives as conj(X[P - k]).  `o` is the output base, `off` the element offset of (frame, bin 0, channel).
template <int MODE>
#if defined(KB_HOST_EMU)
inline void kb_mc_emit(const KbStftParams& p, bool dbany, void* o, long long off, int k, int kk, cpx X1, cpx X2,
                       float& runmax)
#else
__device__ __forceinline__ void kb_mc_emit(const KbStftParams& p, bool dbany, void* o, long long off, int k, int kk,
                                           cpx X1, cpx X2, float& runmax)
#endif
{
    const long long sk = p.o_sk;
    if (MODE == KB_OUT_COMPLEX) {
        float2* oc = reinterpret_cast<float2*>(o) + off;
        oc[k * sk] = make_float2(X1.re, X1.im);
        if (kk >= 0) oc[kk * sk] = make_float2(X2.re, -X2.im);
    } else {
        float* orl = reinterpret_cast<float*>(o) + off;
        float m1 = kb_cabs(X1);
        float m2 = kb_cabs(X2);
        if (MODE == KB_OUT_MAG_PHASE) {   // tf.math.angle, kapre/time_frequency.py:402
            orl[k * sk + p.ph_off] = kb_atan2(X1.im, X1.re);
            if (kk >= 0) orl[kk * sk + p.ph_off] = kb_atan2(-X2.im, X2.re);
        }
        if (dbany) {
            m1 = kb_floor_keepnan(m1, p.amin);
            m2 = kb_floor_keepnan(m2, p.amin);
            runmax = kb_max_keepnan(runmax, m1);
            if (kk >= 0) runmax = kb_max_keepnan(runmax, m2);
            m1 = p.db_mul * kb_log2(m1) - p.db_sub;
            m2 = p.db_mul * kb_log2(m2) - p.db_sub;
        }
        orl[k * sk] = m1;
        if (kk >= 0) orl[kk * sk] = m2;
    }
}

// (The three FFT steps are written out in this body rather than calling the kb_col_* helpers of
// stft_core.cuh: with the helpers ptxas schedules the Q = 32 instantiations 11 % slower -- measured on cfg3.)
template <int Q, int MODE>
#if defined(KB_HOST_EMU)
inline void kb_stft_mc_cta(const KbStftParams& p, char* smem, int cta, int n_cta)
#else
__device__ __forceinline__ void kb_stft_mc_cta(const KbStftParams& p, char* smem, int cta, int n_cta)
#endif
{
    constexpr int P = 32 * Q;
    constexpr int FPW = 32 / Q;
    constexpr int ZSTR = P + 3;          // kb_mc_zstr(Q)
    const bool dbany = (MODE == KB_OUT_MAG_DB) || (MODE == KB_OUT_MAG_PHASE && p.db_on);
    const int NW = p.n_warps;
    const int kb_nt = NW * 32;
    (void)kb_nt;
    const int H = p.hop, N = p.n_fft, C = p.C, TFt = p.TF;
    const int NCOL = TFt * C;                       // columns = (frame, channel) pairs, channel fastest
    const KbStftMcSmem L = kb_stft_mc_smem_layout(Q, N, H, TFt, C, NW, p.mc_wh);
    float* __restrict__ wh_s = reinterpret_cast<float*>(smem + L.wh);
    cpx* __restrict__ twp_s = reinterpret_cast<cpx*>(smem + L.twp);
    cpx* __restrict__ twn_s = reinterpret_cast<cpx*>(smem + L.twn);
    kb_f4* __restrict__ cwq_s = reinterpret_cast<kb_f4*>(smem + L.cwq);
    KbColInfo* ci_s = reinterpret_cast<KbColInfo*>(smem + L.ci);
    float* smp = reinterpret_cast<float*>(smem + L.samples);
    cpx* ex_s = reinterpret_cast<cpx*>(smem + L.ex);
    const int EXS = L.exw;
    const int FR = NW * FPW;                        // columns per round
    const int n_rounds = (NCOL + FR - 1) / FR;
    const int n_tiles = p.B * p.n_tiles_t;
    const int span = L.span, spanp = L.spanp;
    const bool even_base = (H & 1) == 0;
    const bool use_cosw = even_base && p.cosw;

#if defined(KB_HOST_EMU)
    std::vector<KbThreadRegs> kb_regs(kb_nt);
#else
    KbThreadRegs kb_regs;
#endif

    KB_PHASE_BEGIN
        (void)R;
        if (p.mc_wh) { for (int i = tid; i < N; i += kb_nt) wh_s[i] = p.wh[i]; }
        for (int i = tid; i < Q * 33; i += kb_nt) { float2 t = p.twp[i]; twp_s[i] = cmake(t.x, t.y); }
        for (int i = tid; i < P / 2; i += kb_nt) { float2 t = p.twn[i]; twn_s[i] = cmake(t.x, t.y); }
        if (p.cosw) { for (int i = tid; i < Q; i += kb_nt) cwq_s[i] = p.cwq[i]; }
    KB_PHASE_END
    KB_SYNC_CTA;
    if (cta < n_tiles) {
        const int b0 = cta / p.n_tiles_t;
        KB_PHASE_BEGIN
            (void)R;
            kb_mc_issue_loads(p, smp, b0, (cta - b0 * p.n_tiles_t) * TFt, span, spanp, tid, kb_nt);
        KB_PHASE_END
    }

    for (int tile = cta; tile < n_tiles; tile += n_cta) {
        const int b = tile / p.n_tiles_t;
        const int t0 = (tile - b * p.n_tiles_t) * TFt;
        const bool has_next = (tile + n_cta) < n_tiles;
        const int nb = (tile + n_cta) / p.n_tiles_t;
        const int nt0 = ((tile + n_cta) - nb * p.n_tiles_t) * TFt;

        // ---- this tile's samples were requested during the previous tile (or before the loop) ---
        KB_PHASE_BEGIN
            (void)tid;
            R.runmax = 0.0f;
            kb_cp_async_wait();
        KB_PHASE_END
        KB_SYNC_CTA;

        for (int round = 0; round < n_rounds; ++round) {
            // ---- phase 1: window, 32-point DFTs, twiddle, transpose-store; column bookkeeping ---
            KB_PHASE_BEGIN
                const int warp = tid >> 5, lane = tid & 31;
                const int g = lane / Q, q = lane % Q;
                const int col = round * FR + warp * FPW + g;
                if (tid < FR) {
                    const int cc = round * FR + tid;
                    const int fl = kb_fdiv(cc, C, p.mc_magic_c), ch = cc - fl * C;
                    KbColInfo ci;
                    ci.valid = (cc < NCOL && t0 + fl < p.T) ? 1 : 0;
                    ci.ooff = (long long)b * p.o_sb + (long long)ch * p.o_sc + (long long)(t0 + fl) * p.o_st;
                    ci.zoff = (tid / FPW) * EXS + (tid % FPW) * ZSTR;
                    ci_s[tid] = ci;
                }
                if (col < NCOL) {
                    const int fl = kb_fdiv(col, C, p.mc_magic_c), ch = col - fl * C;
                    const float* fr = smp + ch * spanp + fl * H;
                    if (use_cosw) {
                        const kb_f4 cq = cwq_s[q];
                        const cpx cc = cmake(cq.x, cq.y), ss = cmake(cq.z, cq.w);
                        const cpx a0 = cmake(p.cw_a0, p.cw_a0);
#pragma unroll
                        for (int j = 0; j < 32; ++j) {
                            const int n2 = 2 * (q + Q * j);
                            const cpx xv = *reinterpret_cast<const cpx*>(fr + n2);
                            const float cj = j <= 16 ? kb_cos32(j) : kb_cos32(32 - j);
                            const float sj = j <= 16 ? kb_sin32(j) : -kb_sin32(32 - j);
                            cpx wv = a0;
                            if (cj != 0.0f) wv = cfma_s(cc, -cj, wv);
                            if (sj != 0.0f) wv = cfma_s(ss, sj, wv);
                            R.v[j] = cmul_elem(xv, wv);
                        }
                    } else if (even_base) {
#pragma unroll
                        for (int j = 0; j < 32; ++j) {
                            const int n2 = 2 * (q + Q * j);
                            const cpx xv = *reinterpret_cast<const cpx*>(fr + n2);
                            const cpx wv = *reinterpret_cast<const cpx*>(wh_s + n2);
                            R.v[j] = cmul_elem(xv, wv);
                        }
                    } else {
#pragma unroll
                        for (int j = 0; j < 32; ++j) {
                            const int n2 = 2 * (q + Q * j);
                            R.v[j] = cmake(fr[n2] * wh_s[n2], fr[n2 + 1] * wh_s[n2 + 1]);
                        }
                    }
                    kb_fft_dif<32>(R.v);
                    cpx* ex = ex_s + warp * EXS + (g * Q + q) * 33;
                    const cpx* tw = twp_s + q * 33;
                    ex[0] = R.v[0];
#pragma unroll
                    for (int k1 = 1; k1 < 32; ++k1) ex[k1] = cmul(R.v[kb_brev<32>(k1)], tw[k1]);
                }
            KB_PHASE_END
            if (!p.mc_out && round == n_rounds - 1) {
                // every warp has consumed the sample planes: fetch the next tile behind phases 2-4
                KB_SYNC_CTA;
                if (has_next) {
                    KB_PHASE_BEGIN
                        (void)R;
                        kb_mc_issue_loads(p, smp, nb, nt0, span, spanp, tid, kb_nt);
                    KB_PHASE_END
                }
            } else {
                KB_SYNC_WARP;
            }
            // ---- phase 2: gather this lane's columns --------------------------------------
            KB_PHASE_BEGIN
                const int warp = tid >> 5, lane = tid & 31;
                const int g = lane / Q, q = lane % Q;
                const int col = round * FR + warp * FPW + g;
                if (col < NCOL) {
                    const cpx* ex = ex_s + warp * EXS + (g * Q) * 33;
#pragma unroll
                    for (int i = 0; i < FPW; ++i) {
                        const int k1 = q + Q * i;
#pragma unroll
                        for (int q2 = 0; q2 < Q; ++q2) R.v[i * Q + q2] = ex[q2 * 33 + k1];
                    }
                }
            KB_PHASE_END
            KB_SYNC_WARP;
            // ---- phase 3: Q-point DFTs, natural-order store (aliases the exchange buffer) ---
            KB_PHASE_BEGIN
                const int warp = tid >> 5, lane = tid & 31;
                const int g = lane / Q, q = lane % Q;
                const int col = round * FR + warp * FPW + g;
                if (col < NCOL) {
                    cpx* zs = ex_s + warp * EXS + g * ZSTR;
#pragma unroll
                    for (int i = 0; i < FPW; ++i) {
                        kb_fft_dif<Q>(R.v + i * Q);
                        const int k1 = q + Q * i;
#pragma unroll
                        for (int k2 = 0; k2 < Q; ++k2) zs[k1 + 32 * k2] = R.v[i * Q + kb_brev<Q>(k2)];
                    }
                }
            KB_PHASE_END
            // ---- phase 4: real-FFT pair step + epilogue ------------------------------------
            if (p.mc_out) {
                // interleaved output: the whole CTA walks (bin, column) with the column (= channel) fastest
                KB_SYNC_CTA;
                if (has_next && round == n_rounds - 1) {   // sample planes are free: prefetch behind the pair step
                    KB_PHASE_BEGIN
                        (void)R;
                        kb_mc_issue_loads(p, smp, nb, nt0, span, spanp, tid, kb_nt);
                    KB_PHASE_END
                }
                KB_PHASE_BEGIN
                    const int left = NCOL - round * FR;
                    const int ncol_r = left < FR ? left : FR;
                    const unsigned mg = (ncol_r == FR) ? p.mc_magic_fr : p.mc_magic_last;
                    // thread -> (column = tid % ncol_r, first bin tid / ncol_r), bin step = threads / ncol_r
                    const int k0 = kb_fdiv(tid, ncol_r, mg);
                    const int dk = kb_fdiv(kb_nt, ncol_r, mg);
                    const KbColInfo ci = ci_s[tid - k0 * ncol_r];
                    float rmax = R.runmax;
                    if (k0 < dk && ci.valid) {
                        const cpx* zf = ex_s + ci.zoff;
                        for (int k = k0; k <= P / 2; k += dk) {
                            cpx X1, X2;
                            int kk;
                            if (k < P / 2) {
                                kk = P - k;
                                const cpx A = zf[k];
                                const cpx Bv = zf[kk & (P - 1)];
                                const cpx W = twn_s[k];
                                const cpx E = cadd_conj(A, Bv);
                                const cpx D = csub_conj(A, Bv);
                                const cpx T = cmul(cmake(D.im, -D.re), W);
                                X1 = cadd(E, T);
                                X2 = csub(E, T);
                            } else {
                                kk = -1;
                                const cpx A = zf[P / 2];
                                X1 = cmake(2.0f * A.re, -2.0f * A.im);
                                X2 = X1;
                            }
                            kb_mc_emit<MODE>(p, dbany, p.out, ci.ooff, k, kk, X1, X2, rmax);
                        }
                    }
                    R.runmax = rmax;
                KB_PHASE_END
                KB_SYNC_CTA;
            } else {
                // planar output: each warp finishes its own columns, lanes along the bin axis
                KB_SYNC_WARP;
                KB_PHASE_BEGIN
                    const int warp = tid >> 5, lane = tid & 31;
                    float rmax = R.runmax;
#pragma unroll
                    for (int gg = 0; gg < FPW; ++gg) {
                        const int col = round * FR + warp * FPW + gg;
                        const int fl = kb_fdiv(col, C, p.mc_magic_c), ch = col - fl * C;
                        if (col >= NCOL || t0 + fl >= p.T) continue;
                        const long long ooff = (long long)b * p.o_sb + (long long)ch * p.o_sc + (long long)(t0 + fl) * p.o_st;
                        const cpx* zf = ex_s + warp * EXS + gg * ZSTR;
#pragma unroll
                        for (int i = 0; i <= Q / 2; ++i) {
                            cpx X1, X2;
                            int k, kk;
                            if (i < Q / 2) {
                                k = lane + 32 * i;
                                kk = P - k;
                                const cpx A = zf[k];
                                const cpx Bv = zf[kk & (P - 1)];
                                const cpx W = twn_s[k];
                                const cpx E = cadd_conj(A, Bv);
                                const cpx D = csub_conj(A, Bv);
                                const cpx T = cmul(cmake(D.im, -D.re), W);
                                X1 = cadd(E, T);
                                X2 = csub(E, T);
                            } else {
                                if (lane != 0) continue;
                                k = P / 2;
                                kk = -1;
                                const cpx A = zf[P / 2];
                                X1 = cmake(2.0f * A.re, -2.0f * A.im);
                                X2 = X1;
                            }
                            kb_mc_emit<MODE>(p, dbany, p.out, ooff, k, kk, X1, X2, rmax);
                        }
                    }
                    R.runmax = rmax;
                KB_PHASE_END
                KB_SYNC_WARP;   // the warp's exchange region is rewritten by its next round
            }
        }  // rounds

        if (dbany) {
#if defined(KB_HOST_EMU)
            for (int tid = 0; tid < kb_nt; ++tid)
                kb_atomic_max_u32(p.item_max + b, kb_f2u(kb_regs[tid].runmax));
#else
            const unsigned int wm = __reduce_max_sync(0xffffffffu, kb_f2u(kb_regs.runmax));
            if ((threadIdx.x & 31) == 0 && wm != 0u) kb_atomic_max_u32(p.item_max + b, wm);
#endif
        }
    }
}

// ==========================================================================================
// Filterbank modes (mel / log-frequency, optional dB) on all-channel tiles.
//
// Same tile decomposition and loader as above; one round per tile (NCOL = TF * C <= NW * FPW columns),
// then the filterbank epilogue of stft_core.cuh: magnitudes parked in the warps' exchange regions as
// [bin][frame-in-warp], 32 lane groups walk the chunk lists, results staged in out_s[column][band].
// The copy-out is what changes: for interleaved outputs a warp writes one time frame's (band, channel)
// block, which is contiguous in memory, instead of one channel's bands C floats apart.
// ==========================================================================================
struct KbStftMcFbSmem {
    int wh, twp, twn, cwq, cw, cm, cg, samples, outs, ex, total;
    int span, spanp, exw, Mp;
};

KB_HD KbStftMcFbSmem kb_stft_mcfb_smem_layout(int Q, int n_fft, int hop, int TFt, int C, int n_warps, int with_wh,
                                              int n_bands, int n_chunks) {
    KbStftMcFbSmem s;
    const int P = 32 * Q, FPW = 32 / Q;
    const KbStftMcSmem base = kb_stft_mc_smem_layout(Q, n_fft, hop, TFt, C, n_warps, with_wh);
    int off = 0;
    s.wh = off;  if (with_wh) off += kb_align16(n_fft * 4);
    s.twp = off; off += kb_align16(Q * 33 * 8);
    s.twn = off; off += kb_align16((P / 2) * 8);
    s.cwq = off; off += Q * 16;
    s.cw = off;  off += n_chunks * 16;
    s.cm = off;  off += kb_align16(n_chunks * 8);
    s.cg = off;  off += kb_align16(33 * 4);
    s.span = base.span; s.spanp = base.spanp;
    s.samples = off; off += kb_align16(C * s.spanp * 4);
    s.Mp = n_bands | 1;
    s.outs = off; off += kb_align16(n_warps * FPW * s.Mp * 4);
    s.exw = kb_exw(Q);            // geometry of stft_core.cuh: its filterbank phase is reused unchanged
    s.ex = off;  off += kb_align16(n_warps * s.exw * 8);
    s.total = off;
    return s;
}

template <int Q, int MODE>
#if defined(KB_HOST_EMU)
inline void kb_stft_mcfb_cta(const KbStftParams& p, char* smem, int cta, int n_cta)
#else
__device__ __forceinline__ void kb_stft_mcfb_cta(const KbStftParams& p, char* smem, int cta, int n_cta)
#endif
{
    constexpr int P = 32 * Q;
    constexpr int FPW = 32 / Q;
    constexpr int ZSTR = P + Q;
    constexpr bool dbmode = (MODE == KB_OUT_FB_DB);
    constexpr bool paired = FPW >= 2;          // paired-column pair step (stft_core.cuh) whenever a lane owns two or more columns
    const int NW = p.n_warps;
    const int kb_nt = NW * 32;
    (void)kb_nt;
    const int H = p.hop, N = p.n_fft, C = p.C, TFt = p.TF;
    const int NCOL = TFt * C;                       // <= NW * FPW (host guarantees)
    const KbStftMcFbSmem L = kb_stft_mcfb_smem_layout(Q, N, H, TFt, C, NW, p.mc_wh, p.n_bands, p.n_chunks);
    float* __restrict__ wh_s = reinterpret_cast<float*>(smem + L.wh);
    cpx* __restrict__ twp_s = reinterpret_cast<cpx*>(smem + L.twp);
    cpx* __restrict__ twn_s = reinterpret_cast<cpx*>(smem + L.twn);
    kb_f4* __restrict__ cwq_s = reinterpret_cast<kb_f4*>(smem + L.cwq);
    kb_f4* __restrict__ cw_s = reinterpret_cast<kb_f4*>(smem + L.cw);
    kb_i2* __restrict__ cm_s = reinterpret_cast<kb_i2*>(smem + L.cm);
    int* __restrict__ cg_s = reinterpret_cast<int*>(smem + L.cg);
    float* smp = reinterpret_cast<float*>(smem + L.samples);
    float* __restrict__ out_s = reinterpret_cast<float*>(smem + L.outs);
    cpx* ex_s = reinterpret_cast<cpx*>(smem + L.ex);
    const int EXS = L.exw;
    const int n_tiles = p.B * p.n_tiles_t;
    const int span = L.span, spanp = L.spanp;
    const bool even_base = (H & 1) == 0;
    const int wmode = even_base ? (p.cosw ? 2 : 1) : 0;   // see kb_col_window_dft32

#if defined(KB_HOST_EMU)
    std::vector<KbThreadRegs> kb_regs(kb_nt);
#else
    KbThreadRegs kb_regs;
#endif

    KB_PHASE_BEGIN
        (void)R;
        if (p.mc_wh) { for (int i = tid; i < N; i += kb_nt) wh_s[i] = p.wh[i]; }
        for (int i = tid; i < Q * 33; i += kb_nt) { float2 t = p.twp[i]; twp_s[i] = cmake(t.x, t.y); }
        for (int i = tid; i < P / 2; i += kb_nt) { float2 t = paired ? p.twn2[i] : p.twn[i]; twn_s[i] = cmake(t.x, t.y); }
        if (p.cosw) { for (int i = tid; i < Q; i += kb_nt) cwq_s[i] = p.cwq[i]; }
        for (int i = tid; i < p.n_chunks; i += kb_nt) { cw_s[i] = p.cw[i]; cm_s[i] = p.cm[i]; }
        for (int i = tid; i <= 32; i += kb_nt) cg_s[i] = p.cg[i];
    KB_PHASE_END
    KB_SYNC_CTA;
    if (cta < n_tiles) {
        const int b0 = cta / p.n_tiles_t;
        KB_PHASE_BEGIN
            (void)R;
            kb_mc_issue_loads(p, smp, b0, (cta - b0 * p.n_tiles_t) * TFt, span, spanp, tid, kb_nt);
        KB_PHASE_END
    }

    for (int tile = cta; tile < n_tiles; tile += n_cta) {
        const int b = tile / p.n_tiles_t;
        const int t0 = (tile - b * p.n_tiles_t) * TFt;
        const bool has_next = (tile + n_cta) < n_tiles;
        const int nb = (tile + n_cta) / p.n_tiles_t;
        const int nt0 = ((tile + n_cta) - nb * p.n_tiles_t) * TFt;

        KB_PHASE_BEGIN
            (void)tid;
            R.runmax = 0.0f;
            kb_cp_async_wait();
        KB_PHASE_END
        KB_SYNC_CTA;      // samples visible; the previous tile's copy-out is done with out_s

        // ---- phase 1: window, 32-point DFTs, twiddle, transpose-store ---------------------------
        KB_PHASE_BEGIN
            const int warp = tid >> 5, lane = tid & 31;
            const int g = lane / Q, q = lane % Q;
            const int col = warp * FPW + g;
            if (col < NCOL) {
                const int fl = kb_fdiv(col, C, p.mc_magic_c), ch = col - fl * C;
                kb_col_window_dft32<Q, paired>(R, smp + ch * spanp + fl * H, wh_s, cwq_s, p.cw_a0, twp_s, ex_s + warp * EXS, g, q,
                                               wmode);
            }
        KB_PHASE_END
        if constexpr (paired) {
        // ---- phases 2-4, paired-column form (stft_core.cuh: kb_col_gather_paired / kb_col_dftq_pair_mag) ----
        KB_SYNC_WARP;
        KB_PHASE_BEGIN
            const int warp = tid >> 5, lane = tid & 31;
            const int g = lane / Q, q = lane % Q;
            if (warp * FPW + g < NCOL) {
                kb_col_gather_paired<Q>(R, ex_s + warp * EXS, g, q);
            } else {   // column past the tile: its magnitudes must read as zeros in the filterbank phase
#pragma unroll
                for (int i = 0; i < 32; ++i) R.v[i] = cmake(0.0f, 0.0f);
            }
        KB_PHASE_END
        KB_SYNC_WARP;
        KB_PHASE_BEGIN
            const int warp = tid >> 5, lane = tid & 31;
            const int g = lane / Q, q = lane % Q;
            float* mw = reinterpret_cast<float*>(ex_s + warp * EXS);
            kb_col_dftq_pair_mag<Q>(R, twn_s, mw, g, q);
            if (lane < 3) {
#pragma unroll
                for (int gg = 0; gg < FPW; ++gg) mw[(P + 1 + lane) * FPW + gg] = 0.0f;   // pad bins
            }
        KB_PHASE_END
        } else {
        KB_SYNC_WARP;
        // ---- phase 2: gather this lane's columns ----------------------------------------------
        KB_PHASE_BEGIN
            const int warp = tid >> 5, lane = tid & 31;
            const int g = lane / Q, q = lane % Q;
            if (warp * FPW + g < NCOL) kb_col_gather<Q>(R, ex_s + warp * EXS, g, q);
        KB_PHASE_END
        KB_SYNC_WARP;
        // ---- phase 3: Q-point DFTs, natural-order store ---------------------------------------
        KB_PHASE_BEGIN
            const int warp = tid >> 5, lane = tid & 31;
            const int g = lane / Q, q = lane % Q;
            if (warp * FPW + g < NCOL) kb_col_dftq_store<Q>(R, ex_s + warp * EXS, g, q, ZSTR);
        KB_PHASE_END
        KB_SYNC_WARP;
        // ---- phase 4: pair step, magnitudes parked in registers (R.v is dead) -------------------
        KB_PHASE_BEGIN
            const int warp = tid >> 5, lane = tid & 31;
            float* magr = reinterpret_cast<float*>(R.v);
#pragma unroll
            for (int gg = 0; gg < FPW; ++gg) {
                const bool active = (warp * FPW + gg) < NCOL;
                const cpx* zf = ex_s + warp * EXS + gg * ZSTR;
#pragma unroll
                for (int i = 0; i <= Q / 2; ++i) {
                    float m1 = 0.0f, m2 = 0.0f;
                    if (active) {
                        cpx X1, X2;
                        if (i < Q / 2) {
                            const int k = lane + 32 * i;
                            const cpx A = zf[k];
                            const cpx Bv = zf[(P - k) & (P - 1)];
                            const cpx W = twn_s[k];
                            const cpx E = cadd_conj(A, Bv);
                            const cpx D = csub_conj(A, Bv);
                            const cpx T = cmul(cmake(D.im, -D.re), W);
                            X1 = cadd(E, T);
                            X2 = csub(E, T);
                        } else {
                            const cpx A = zf[P / 2];
                            X1 = cmake(2.0f * A.re, -2.0f * A.im);
                            X2 = X1;
                        }
                        m1 = kb_sqrt(cnorm(X1));
                        m2 = kb_sqrt(cnorm(X2));
                    }
                    magr[(gg * (Q / 2 + 1) + i) * 2 + 0] = m1;
                    magr[(gg * (Q / 2 + 1) + i) * 2 + 1] = m2;
                }
            }
        KB_PHASE_END
        KB_SYNC_WARP;
        // ---- phase 4b: magnitudes -> own exchange region, layout [bin][frame-in-warp] -----------
        KB_PHASE_BEGIN
            const int warp = tid >> 5, lane = tid & 31;
            const float* magr = reinterpret_cast<const float*>(R.v);
            float* mw = reinterpret_cast<float*>(ex_s + warp * EXS);
#pragma unroll
            for (int i = 0; i < Q / 2; ++i) {
                const int k = lane + 32 * i;
                float lo[FPW], hi[FPW];
#pragma unroll
                for (int gg = 0; gg < FPW; ++gg) {
                    lo[gg] = magr[(gg * (Q / 2 + 1) + i) * 2 + 0];
                    hi[gg] = magr[(gg * (Q / 2 + 1) + i) * 2 + 1];
                }
                kb_store_vec<FPW>(mw + k * FPW, lo);
                kb_store_vec<FPW>(mw + (P - k) * FPW, hi);
            }
            if (lane == 0) {
                float mid[FPW];
#pragma unroll
                for (int gg = 0; gg < FPW; ++gg) mid[gg] = magr[(gg * (Q / 2 + 1) + Q / 2) * 2 + 0];
                kb_store_vec<FPW>(mw + (P / 2) * FPW, mid);
            }
            if (lane < 3) {
#pragma unroll
                for (int gg = 0; gg < FPW; ++gg) mw[(P + 1 + lane) * FPW + gg] = 0.0f;   // pad bins
            }
        KB_PHASE_END
        }
        KB_SYNC_CTA;      // all magnitudes visible; the sample planes are free
        if (has_next) {
            KB_PHASE_BEGIN
                (void)R;
                kb_mc_issue_loads(p, smp, nb, nt0, span, spanp, tid, kb_nt);
            KB_PHASE_END
        }
        // ---- phase 5: filterbank (as in stft_core.cuh) ---------------------------------------------
        KB_PHASE_BEGIN
            (void)R;
            // NW is a power of two (kb_pick_mcfb_cfg): lane group = tid / NW, lane within the group = tid % NW
            const int w = tid & (NW - 1);
            const int grp = tid >> kb_ilog2(NW);                    // 0..31
            const float* __restrict__ mw = reinterpret_cast<const float*>(ex_s + w * EXS);
            float* __restrict__ ocol = out_s + (w * FPW) * L.Mp;
            float a0[FPW], a1[FPW];
#pragma unroll
            for (int g = 0; g < FPW; ++g) { a0[g] = 0.0f; a1[g] = 0.0f; }
            const int ce = cg_s[grp + 1];
            for (int i = cg_s[grp]; i < ce; ++i) {
                const kb_f4 wv = cw_s[i];
                const kb_i2 mt = cm_s[i];
                const float* mp = mw + mt.x * FPW;
                float m01[2 * FPW], m23[2 * FPW];
                kb_load_vec<2 * FPW>(m01, mp);
                kb_load_vec<2 * FPW>(m23, mp + 2 * FPW);
#pragma unroll
                for (int g = 0; g < FPW; ++g) {
                    a0[g] += wv.x * m01[g];
                    a1[g] += wv.y * m01[FPW + g];
                    a0[g] += wv.z * m23[g];
                    a1[g] += wv.w * m23[FPW + g];
                }
                if (mt.y >= 0) {
#pragma unroll
                    for (int g = 0; g < FPW; ++g) {
                        ocol[g * L.Mp + mt.y] = a0[g] + a1[g];
                        a0[g] = 0.0f;
                        a1[g] = 0.0f;
                    }
                }
            }
        KB_PHASE_END
        KB_SYNC_CTA;
        // ---- phase 6: decibel + copy-out ------------------------------------------------------------
        KB_PHASE_BEGIN
            const int warp = tid >> 5, lane = tid & 31;
            float* o = reinterpret_cast<float*>(p.out) + (long long)b * p.o_sb;
            const int M = p.n_bands;
            const float amin = p.amin, dmul = p.db_mul, dsub = p.db_sub;
            float rmax = R.runmax;
            if (p.mc_out) {
                // interleaved output: one time frame's (band, channel) block is contiguous
                const int MC = M * C;
                for (int fl = warp; fl < TFt; fl += NW) {
                    const int t = t0 + fl;
                    if (t >= p.T) break;
                    float* __restrict__ orow = o + (long long)t * p.o_st;
                    const float* __restrict__ srow = out_s + (fl * C) * L.Mp;
                    for (int e = lane; e < MC; e += 32) {
                        const int m = kb_fdiv(e, C, p.mc_magic_c), c = e - m * C;
                        float v = srow[c * L.Mp + m];
                        if (dbmode) {
                            v = kb_floor_keepnan(v, amin);
                            rmax = kb_max_keepnan(rmax, v);
                            v = dmul * kb_log2(v) - dsub;
                        }
                        orow[e] = v;
                    }
                }
            } else {
                const int sk = (int)p.o_sk;
                for (int col = warp; col < NCOL; col += NW) {
                    const int fl = kb_fdiv(col, C, p.mc_magic_c), c = col - fl * C;
                    const int t = t0 + fl;
                    if (t >= p.T) break;
                    float* __restrict__ orow = o + (long long)c * p.o_sc + (long long)t * p.o_st;
                    const float* __restrict__ srow = out_s + col * L.Mp;
                    for (int m = lane; m < M; m += 32) {
                        float v = srow[m];
                        if (dbmode) {
                            v = kb_floor_keepnan(v, amin);
                            rmax = kb_max_keepnan(rmax, v);
                            v = dmul * kb_log2(v) - dsub;
                        }
                        orow[(long long)m * sk] = v;
                    }
                }
            }
            R.runmax = rmax;
        KB_PHASE_END

        if (dbmode) {
#if defined(KB_HOST_EMU)
            for (int tid = 0; tid < kb_nt; ++tid)
                kb_atomic_max_u32(p.item_max + b, kb_f2u(kb_regs[tid].runmax));
#else
            const unsigned int wm = __reduce_max_sync(0xffffffffu, kb_f2u(kb_regs.runmax));
            if ((threadIdx.x & 31) == 0 && wm != 0u) kb_atomic_max_u32(p.item_max + b, wm);
#endif
        }
    }
}
