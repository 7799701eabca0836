// Mixed-radix (2, 3, 4, 5) Stockham FFT for every n_fft the register kernel (n_fft = 64 * {4, 8, 16, 32}) does not
// take: the reference's own tests use n_fft = 1000 = 2^3 5^3 (tests/test_time_frequency.py:72-125), speech front
// ends 400, music 4096 / 8192.  Same semantics as kapre/time_frequency.py:169-182 (pad_begin, right zero-pad of a
// short window to n_fft, rfft).
//
// A group of G warps (G = 1, 2, 4, 8, 16; picked by the host so that ~32 warps are resident per SM whatever the
// size of the two P-point buffers) transforms one frame at a time in shared memory:
//   even n_fft: packed real FFT -- complex FFT of length P = n_fft / 2 of z[n] = x[2n] + i x[2n+1], then the pair step
//               X[k], X[P-k] from Z[k], Z[P-k] (as in stft_core.cuh);   odd n_fft: complex FFT of length P = n_fft.
//   Stockham autosort passes (ping-pong between two P-point buffers, natural order in and out), pass with radix r
//   after radices of product Ns:   lane j < P / r:  k = j mod Ns,
//       v[t] = in[j + t P / r] * exp(-2 pi i t k / (Ns r)),  V = DFT_r(v),  out[(j - k) r + k + t Ns] = V[t]
//   twiddles from one shared table exp(-2 pi i m / P).  The first pass writes with a lane stride of r elements; when r is
//   even that hand-off buffer is indexed as i + (i >> 4) (one spare element per 16), which spreads the 16 lanes of a
//   half-warp over all banks; later passes (Ns >= r) are at most 2-way conflicted and stay unpadded.
// Everything a pass needs that involves a division (twiddle step, j mod Ns at the group's first butterfly, ...) is
// precomputed on the host per pass (KbMrPass, kb_mr_finish).  Throughput is about 2.2x below the register kernel at the
// neighbouring power of two (3-5 passes over shared memory instead of 1 transpose: ~1090 warp instructions per n_fft 400
// frame, 340 of them butterflies), against ~100x for the direct O(N^2) DFT it replaces (kb_dft_cta stays for sizes
// with a prime factor > 5).
#pragma once
#include "aux_core.cuh"
#include "stft_mc_core.cuh"   // kb_magic / kb_fdiv

#define KB_MR_MAX_PASS 12

// one Stockham pass: radix r after radices of product ns
struct alignas(16) KbMrPass {
    int r, ns;
    int tstep;        // P / (ns r): exp(-2 pi i t k / (ns r)) = tw_s[t k tstep]
    int kinc;         // (32 G) mod ns: step of k = j mod ns when j advances by the group size
    unsigned magic;   // kb_magic(ns)
    int nb;           // P / r butterflies
    int pad0, pad1;
};

struct KbMrParams {
    KbDftParams d;            // tensors, sizes, window (w[0, win_eff)), tw = exp(-2 pi i r / n_fft), mode, n_warps
    int P;                    // complex FFT length: n_fft / 2 (even n_fft) or n_fft
    int half;                 // 1: packed real FFT (even n_fft)
    int n_pass;
    int radix[KB_MR_MAX_PASS];
    int TF;                   // frames per tile (= frames per group per tile * n_warps / G)
    int G;                    // warps per frame
    int pad1;                 // the buffer between pass 0 and pass 1 is indexed i + (i >> 4)
    // constants the host precomputes (kb_mr_finish) so that the kernel's loops contain no division and do not
    // re-derive the shared-memory layout
    KbMrPass pass[KB_MR_MAX_PASS];
    int bufsz;                    // kb_mr_bufsz(P)
    int off_buf, off_mag, off_outs, Mp;   // kb_mr_smem_layout
    int sk1;                      // output bins are contiguous (o_sk == 1)
    int p0g;                      // first pass reads interior frames straight from global memory (kb_mr_pass0_global)
    // fused tail (modes KB_OUT_MAG_DB, KB_OUT_FB, KB_OUT_FB_DB; kapre/time_frequency.py:535-548, kapre/backend.py:186-192)
    int FRT;                  // filterbank modes: frames per tile (32 / 16 / 8) = columns of the magnitude tile; else 0
    const KbBand* bands;
    const float* fbw;
    int n_bands;
    float amin, db_mul, db_sub;
    int db_ftz;
    unsigned int* item_max;   // per batch item: bits of max(max(x, amin)) for the clamp pass
};

// radices of P in {8, 4, 2, 3, 5} order (large radices first: fewest passes over shared memory); returns -1 if P has
// another prime factor
static inline int kb_mr_factor(int P, int* radix) {
    int n = 0;
    while (P % 8 == 0 && n < KB_MR_MAX_PASS) { radix[n++] = 8; P /= 8; }
    while (P % 4 == 0 && n < KB_MR_MAX_PASS) { radix[n++] = 4; P /= 4; }
    while (P % 2 == 0 && n < KB_MR_MAX_PASS) { radix[n++] = 2; P /= 2; }
    while (P % 3 == 0 && n < KB_MR_MAX_PASS) { radix[n++] = 3; P /= 3; }
    while (P % 5 == 0 && n < KB_MR_MAX_PASS) { radix[n++] = 5; P /= 5; }
    return P == 1 ? n : -1;
}

struct KbMrSmem { int tw, buf, mag, outs, total, Mp; };
KB_HD int kb_mr_bufsz(int P) { return kb_align16((P + (P >> 4) + 1) * 8); }
// FRT > 0 adds the filterbank tile: magnitudes [bin][frame] (row stride FRT + 1, three zero pad rows for the 4-bin
// groups of kb_band_dot) and the (frame x band) result block
KB_HD KbMrSmem kb_mr_smem_layout(int P, int n_groups, int F = 0, int n_bands = 0, int FRT = 0) {
    KbMrSmem s;
    s.tw = 0;
    s.buf = kb_align16(P * 8);
    s.mag = s.buf + n_groups * 2 * kb_mr_bufsz(P);
    s.Mp = n_bands | 1;
    s.outs = s.mag + (FRT > 0 ? kb_align16((F + 3) * (FRT + 1) * 4) : 0);
    s.total = s.outs + (FRT > 0 ? kb_align16(FRT * s.Mp * 4) : 0);
    return s;
}

// launch shape: warps per frame (G) and per CTA (NW) that keep the most warps resident per SM (64 registers per thread:
// `want` = 32), given tw + 2 buffers per group (+ the filterbank tile).  A group may not be wider than twice the
// butterflies of its narrowest pass (P / largest radix) -- wider groups are resident but idle; among equals the smaller
// G wins (loop order).  Returns warps per SM, 0 if nothing fits.
static inline int kb_mr_pick(int P, int smem_optin, int smem_sm, int want, int* NW_out, int* G_out, int* bps_out,
                             int F = 0, int n_bands = 0, int FRT = 0) {
    int radix[KB_MR_MAX_PASS];
    const int np = kb_mr_factor(P, radix);
    int rmax = 2;
    for (int i = 0; i < np; ++i) if (radix[i] > rmax) rmax = radix[i];
    const int gs_max = 2 * (P / rmax) > 32 ? 2 * (P / rmax) : 32;
    int best = 0;
    for (int NW = 8; NW <= 16; NW += 8)
        for (int G = 1; G <= NW; G *= 2) {
            if (G * 32 > gs_max) continue;
            if (FRT > 0 && (NW / G > FRT || FRT % (NW / G))) continue;     // whole frames per group and tile
            const int smem = kb_mr_smem_layout(P, NW / G, F, n_bands, FRT).total;
            if (smem > smem_optin) continue;
            int bps = smem_sm / (smem + 1024);
            if (bps * NW > want) bps = want / NW;
            if (bps < 1) continue;
            if (bps * NW > best) { best = bps * NW; *NW_out = NW; *G_out = G; *bps_out = bps; }
        }
    return best;
}

// host-side constants of a launch; call once G, n_warps, FRT and the tensors are set
static inline void kb_mr_finish(KbMrParams& q) {
    int Ns = 1;
    const int GS = 32 * q.G;
    for (int ps = 0; ps < q.n_pass; ++ps) {
        KbMrPass& w = q.pass[ps];
        w.r = q.radix[ps];
        w.ns = Ns;
        w.tstep = q.P / (Ns * w.r);
        w.kinc = GS % Ns;
        w.magic = kb_magic((unsigned)Ns);
        w.nb = q.P / w.r;
        w.pad0 = w.pad1 = 0;
        Ns *= w.r;
    }
    q.bufsz = kb_mr_bufsz(q.P);
    const KbMrSmem L = kb_mr_smem_layout(q.P, q.d.n_warps / q.G, q.d.n_fft / 2 + 1, q.n_bands, q.FRT);
    q.off_buf = L.buf; q.off_mag = L.mag; q.off_outs = L.outs; q.Mp = L.Mp;
    q.sk1 = q.d.o_sk == 1 ? 1 : 0;
    // first pass from global memory: only the threads that own a butterfly load, so with ONE frame in flight per CTA
    // (a single group: n_fft 4096 with the fused tail, measured -7 %) the staged load with every thread loading wins
    q.p0g = (q.half && q.n_pass > 0 && q.d.n_warps / q.G >= 2) ? 1 : 0;
}

KB_HD cpx kb_mul_mi(cpx a) { return cmake(a.im, -a.re); }   // a * (-i)

// forward DFTs of size r on v[0..r)
KB_HD void kb_dft_r2(cpx* v) { const cpx a = v[0], b = v[1]; v[0] = cadd(a, b); v[1] = csub(a, b); }
KB_HD void kb_dft_r4(cpx* v) {
    const cpx a = cadd(v[0], v[2]), b = csub(v[0], v[2]), c = cadd(v[1], v[3]), d = kb_mul_mi(csub(v[1], v[3]));
    v[0] = cadd(a, c); v[2] = csub(a, c); v[1] = cadd(b, d); v[3] = csub(b, d);
}
KB_HD void kb_dft_r8(cpx* v) {
    // two radix-4 butterflies on the even / odd inputs, then the radix-2 combination with W_8^k
    cpx e[4] = {v[0], v[2], v[4], v[6]}, o[4] = {v[1], v[3], v[5], v[7]};
    kb_dft_r4(e);
    kb_dft_r4(o);
    const float h = 0.70710678118654752440f;
    const cpx o1 = cscale(cadd(o[1], kb_mul_mi(o[1])), h);            // o1 * (1 - i) / sqrt2
    const cpx o2 = kb_mul_mi(o[2]);                                    // o2 * (-i)
    const cpx o3 = cscale(csub(kb_mul_mi(o[3]), o[3]), h);            // o3 * (-1 - i) / sqrt2
    v[0] = cadd(e[0], o[0]); v[4] = csub(e[0], o[0]);
    v[1] = cadd(e[1], o1);   v[5] = csub(e[1], o1);
    v[2] = cadd(e[2], o2);   v[6] = csub(e[2], o2);
    v[3] = cadd(e[3], o3);   v[7] = csub(e[3], o3);
}
KB_HD void kb_dft_r3(cpx* v) {
    const cpx t1 = cadd(v[1], v[2]);
    const cpx m1 = cfma_s(t1, -0.5f, v[0]);
    const cpx m2 = kb_mul_mi(cscale(csub(v[1], v[2]), 0.86602540378443864676f));
    v[0] = cadd(v[0], t1); v[1] = cadd(m1, m2); v[2] = csub(m1, m2);
}
KB_HD void kb_dft_r5(cpx* v) {
    const float c1 = 0.30901699437494742410f, c2 = -0.80901699437494742410f;
    const float s1 = 0.95105651629515357212f, s2 = 0.58778525229247312917f;
    const cpx a1 = cadd(v[1], v[4]), a2 = cadd(v[2], v[3]), b1 = csub(v[1], v[4]), b2 = csub(v[2], v[3]);
    const cpx r1 = cfma_s(a2, c2, cfma_s(a1, c1, v[0])), r2 = cfma_s(a2, c1, cfma_s(a1, c2, v[0]));
    const cpx q1 = kb_mul_mi(cfma_s(b2, s2, cscale(b1, s1))), q2 = kb_mul_mi(cfma_s(b2, -s1, cscale(b1, s2)));
    v[0] = cadd(v[0], cadd(a1, a2));
    v[1] = cadd(r1, q1); v[4] = csub(r1, q1);
    v[2] = cadd(r2, q2); v[3] = csub(r2, q2);
}

// one Stockham pass of radix RDX for thread gl of a group of GS threads (butterflies j = gl, gl + GS, ...);
// k = gl mod Ns on entry, stepped with j
template <int RDX, bool PIN, bool POUT>
KB_FN void kb_mr_pass(const cpx* __restrict__ in, cpx* __restrict__ out, const cpx* __restrict__ tw_s, int nb, int Ns,
                      int tstep, int kinc, int k, int gl, int GS) {
    for (int j = gl; j < nb; j += GS) {
        cpx v[RDX];
        if (PIN) {
            int i = j;
#pragma unroll
            for (int t = 0; t < RDX; ++t) { v[t] = in[i + (i >> 4)]; i += nb; }
        } else {
            const cpx* pi = in + j;
#pragma unroll
            for (int t = 0; t < RDX; ++t) { v[t] = *pi; pi += nb; }
        }
        if (Ns > 1) {
            const int kt = k * tstep;
            const cpx* tp = tw_s + kt;
#pragma unroll
            for (int t = 1; t < RDX; ++t) { v[t] = cmul(v[t], *tp); tp += kt; }
        }
        if (RDX == 2) kb_dft_r2(v);
        else if (RDX == 3) kb_dft_r3(v);
        else if (RDX == 4) kb_dft_r4(v);
        else if (RDX == 8) kb_dft_r8(v);
        else kb_dft_r5(v);
        if (POUT) {
            int i = (j - k) * RDX + k;
#pragma unroll
            for (int t = 0; t < RDX; ++t) { out[i + (i >> 4)] = v[t]; i += Ns; }
        } else {
            cpx* po = out + ((j - k) * RDX + k);
#pragma unroll
            for (int t = 0; t < RDX; ++t) { *po = v[t]; po += Ns; }
        }
        k += kinc;
        if (k >= Ns) k -= Ns;
    }
}
// first pass (Ns = 1: no twiddles) of a frame that lies wholly inside the signal: the butterfly inputs are the windowed
// sample pairs straight from global memory (v[t] = (x[2i] w[2i], x[2i+1] w[2i+1]), i = j + t nb) -- no staging buffer trip
template <int RDX, bool POUT>
KB_FN void kb_mr_pass0_global(const float2* __restrict__ xp, const float2* __restrict__ wp, cpx* __restrict__ out, int nb,
                              int gl, int GS) {
    for (int j = gl; j < nb; j += GS) {
        float2 xv[RDX], wv[RDX];
        {
            const float2* px = xp + j;
            const float2* pw = wp + j;
#pragma unroll
            for (int t = 0; t < RDX; ++t) {
#if defined(KB_HOST_EMU)
                xv[t] = *px; wv[t] = *pw;
#else
                xv[t] = __ldg(px); wv[t] = __ldg(pw);
#endif
                px += nb; pw += nb;
            }
        }
        cpx v[RDX];
#pragma unroll
        for (int t = 0; t < RDX; ++t) v[t] = cmake(xv[t].x * wv[t].x, xv[t].y * wv[t].y);
        if (RDX == 2) kb_dft_r2(v);
        else if (RDX == 3) kb_dft_r3(v);
        else if (RDX == 4) kb_dft_r4(v);
        else if (RDX == 8) kb_dft_r8(v);
        else kb_dft_r5(v);
        if (POUT) {
            int i = j * RDX;
#pragma unroll
            for (int t = 0; t < RDX; ++t) { out[i + (i >> 4)] = v[t]; ++i; }
        } else {
            cpx* po = out + j * RDX;
#pragma unroll
            for (int t = 0; t < RDX; ++t) po[t] = v[t];
        }
    }
}
template <bool POUT>
KB_FN void kb_mr_pass0_global_r(int r, const float2* xp, const float2* wp, cpx* out, int nb, int gl, int GS) {
    if (r == 8) kb_mr_pass0_global<8, POUT>(xp, wp, out, nb, gl, GS);
    else if (r == 4) kb_mr_pass0_global<4, POUT>(xp, wp, out, nb, gl, GS);
    else if (r == 2) kb_mr_pass0_global<2, POUT>(xp, wp, out, nb, gl, GS);
    else if (r == 3) kb_mr_pass0_global<3, POUT>(xp, wp, out, nb, gl, GS);
    else kb_mr_pass0_global<5, POUT>(xp, wp, out, nb, gl, GS);
}

template <bool PIN, bool POUT>
KB_FN void kb_mr_pass_r(int r, const cpx* in, cpx* out, const cpx* tw_s, int nb, int Ns, int tstep, int kinc, int k, int gl,
                        int GS) {
    if (r == 8) kb_mr_pass<8, PIN, POUT>(in, out, tw_s, nb, Ns, tstep, kinc, k, gl, GS);
    else if (r == 4) kb_mr_pass<4, PIN, POUT>(in, out, tw_s, nb, Ns, tstep, kinc, k, gl, GS);
    else if (r == 2) kb_mr_pass<2, PIN, POUT>(in, out, tw_s, nb, Ns, tstep, kinc, k, gl, GS);
    else if (r == 3) kb_mr_pass<3, PIN, POUT>(in, out, tw_s, nb, Ns, tstep, kinc, k, gl, GS);
    else kb_mr_pass<5, PIN, POUT>(in, out, tw_s, nb, Ns, tstep, kinc, k, gl, GS);
}

// synchronisation of one frame group: a warp barrier when G == 1, else a named barrier (ids 1 .. 15) over its G warps
#if defined(KB_HOST_EMU)
#define KB_MR_SYNC
#else
#define KB_MR_SYNC do { if (q.G == 1) __syncwarp(); else asm volatile("bar.sync %0, %1;" :: "r"(1 + (int)(threadIdx.x >> gsh)), "r"(GS) : "memory"); } while (0)
#endif

template <int FRT>
#if defined(KB_HOST_EMU)
inline void kb_mr_cta_t(const KbMrParams& q, char* smem, int cta, int n_cta)
#else
__device__ __forceinline__ void kb_mr_cta_t(const KbMrParams& q, char* smem, int cta, int n_cta)
#endif
{
    constexpr int RS = FRT + 1;
    const KbDftParams& p = q.d;
    const int NW = p.n_warps;
    const int kb_nt = NW * 32;
    (void)kb_nt;
    const int N = p.n_fft, We = p.win_eff, F = N / 2 + 1, P = q.P;
    const int G = q.G, GS = G * 32, NG = NW / G;
    const int gsh = 5 + kb_ilog2(G);         // G is a power of two: group = tid >> gsh, thread in group = tid & (GS - 1)
    struct { int buf, Mp; } L;                 // kb_mr_smem_layout, precomputed by kb_mr_finish
    L.buf = q.off_buf; L.Mp = q.Mp;
    cpx* tw_s = reinterpret_cast<cpx*>(smem);
    float* mag_s = reinterpret_cast<float*>(smem + q.off_mag);
    float* out_s = reinterpret_cast<float*>(smem + q.off_outs);
    (void)NG;
    const bool dbmode = p.mode == KB_OUT_MAG_DB || p.mode == KB_OUT_FB_DB;
    (void)mag_s; (void)out_s;
    const int bufsz = q.bufsz;
    const int n_tiles_t = (p.T + q.TF - 1) / q.TF;
    const int n_tiles = p.B * p.C * n_tiles_t;
    const int fpw = q.TF / NG;               // frames per group and tile
#if defined(KB_HOST_EMU)
    std::vector<KbThreadRegs> kb_regs(kb_nt);
#else
    KbThreadRegs kb_regs;
#endif
    KB_PHASE_BEGIN
        (void)R;
        const int st = q.half ? 2 : 1;
        for (int i = tid; i < P; i += kb_nt) { float2 t = p.tw[i * st]; tw_s[i] = cmake(t.x, t.y); }
        if (FRT > 0) for (int i = tid; i < 3 * RS; i += kb_nt) mag_s[F * RS + i] = 0.0f;   // pad rows, never written again
    KB_PHASE_END
    KB_SYNC_CTA;
    for (int tile = cta; tile < n_tiles; tile += n_cta) {
        const int sig = tile / n_tiles_t;
        const int tt = tile - sig * n_tiles_t;
        const int b = sig / p.C, c = sig - b * p.C;
        const float* xsig = p.x + (long long)b * p.x_sb + (long long)c * p.x_sc;
        const long long obase = (long long)b * p.o_sb + (long long)c * p.o_sc;
        KB_PHASE_BEGIN
            R.runmax = 0.0f;
        KB_PHASE_END
        for (int fi = 0; fi < fpw; ++fi) {
            // every step below is private to one group of G warps (its own two buffers): group-level synchronisation only
            KB_PHASE_BEGIN
                (void)R;
                const int grp = tid >> gsh, gl = tid & (GS - 1);
                const int t = tt * q.TF + grp * fpw + fi;
                cpx* A = reinterpret_cast<cpx*>(smem + L.buf + (grp * 2) * bufsz);
                if (t < p.T) {
                    const long long s0 = (long long)t * p.hop - p.pad_left;
                    const bool interior = s0 >= 0 && s0 + N <= p.L && We == N && p.x_sl == 1 &&
                                          (((reinterpret_cast<uintptr_t>(xsig) >> 2) + (uintptr_t)s0) & 1u) == 0;
                    if (q.p0g && interior) {
                        // whole frame inside the signal, 8-byte aligned: the first pass reads the windowed sample pairs
                        // straight from global memory (kb_mr_pass0_global), nothing to stage
                    } else if (q.half && interior) {
                        // the same frame staged by every thread of the group: vector loads of (x[2n], x[2n+1]) and of the
                        // window pair, four trips' loads in flight before the first multiply
                        const float2* xp = reinterpret_cast<const float2*>(xsig + s0);
                        const float2* wp = reinterpret_cast<const float2*>(p.w);
                        for (int n0 = gl; n0 < P; n0 += 4 * GS) {
                            float2 xv[4], wv[4];
#pragma unroll
                            for (int u = 0; u < 4; ++u) {
                                const int n = n0 + u * GS;
                                if (n < P) {
#if defined(KB_HOST_EMU)
                                    xv[u] = xp[n]; wv[u] = wp[n];
#else
                                    xv[u] = __ldg(xp + n); wv[u] = __ldg(wp + n);
#endif
                                }
                            }
#pragma unroll
                            for (int u = 0; u < 4; ++u) {
                                const int n = n0 + u * GS;
                                if (n < P) A[n] = cmake(xv[u].x * wv[u].x, xv[u].y * wv[u].y);
                            }
                        }
                    } else if (q.half) {
                        for (int n = gl; n < P; n += GS) {
                            float v[2];
#pragma unroll
                            for (int h = 0; h < 2; ++h) {
                                const int m = 2 * n + h;
                                const long long s = s0 + m;
                                v[h] = (m < We && s >= 0 && s < p.L) ? kb_ldg(xsig + s * p.x_sl) * kb_ldg(p.w + m) : 0.0f;
                            }
                            A[n] = cmake(v[0], v[1]);
                        }
                    } else {
                        for (int n = gl; n < P; n += GS) {
                            const long long s = s0 + n;
                            const float v = (n < We && s >= 0 && s < p.L) ? kb_ldg(xsig + s * p.x_sl) * kb_ldg(p.w + n) : 0.0f;
                            A[n] = cmake(v, 0.0f);
                        }
                    }
                }
            KB_PHASE_END
            KB_MR_SYNC;
            for (int ps = 0; ps < q.n_pass; ++ps) {
                const KbMrPass w = q.pass[ps];
                const int r = w.r, Ns = w.ns;
                KB_PHASE_BEGIN
                    (void)R;
                    const int grp = tid >> gsh, gl = tid & (GS - 1);
                    const int t = tt * q.TF + grp * fpw + fi;
                    cpx* b0 = reinterpret_cast<cpx*>(smem + L.buf + (grp * 2) * bufsz);
                    cpx* b1 = reinterpret_cast<cpx*>(smem + L.buf + (grp * 2 + 1) * bufsz);
                    const cpx* in = (ps & 1) ? b1 : b0;
                    cpx* out = (ps & 1) ? b0 : b1;
                    bool from_global = false;
                    if (ps == 0 && q.p0g && t < p.T) {
                        const long long s0 = (long long)t * p.hop - p.pad_left;
                        from_global = s0 >= 0 && s0 + N <= p.L && We == N && p.x_sl == 1 &&
                                      (((reinterpret_cast<uintptr_t>(xsig) >> 2) + (uintptr_t)s0) & 1u) == 0;   // "interior" of the load phase
                        if (from_global) {
                            const float2* xp = reinterpret_cast<const float2*>(xsig + s0);
                            const float2* wp = reinterpret_cast<const float2*>(p.w);
                            if (q.pad1) kb_mr_pass0_global_r<true>(r, xp, wp, out, w.nb, gl, GS);
                            else kb_mr_pass0_global_r<false>(r, xp, wp, out, w.nb, gl, GS);
                        }
                    }
                    if (t < p.T && !from_global) {
                        const int k = gl - Ns * kb_fdiv(gl, Ns, w.magic);   // gl mod Ns
                        if (ps > 1 || !q.pad1) kb_mr_pass_r<false, false>(r, in, out, tw_s, w.nb, Ns, w.tstep, w.kinc, k, gl, GS);
                        else if (ps == 0) kb_mr_pass_r<false, true>(r, in, out, tw_s, w.nb, Ns, w.tstep, w.kinc, k, gl, GS);
                        else kb_mr_pass_r<true, false>(r, in, out, tw_s, w.nb, Ns, w.tstep, w.kinc, k, gl, GS);
                    }
                KB_PHASE_END
                KB_MR_SYNC;
            }
            KB_PHASE_BEGIN
                const int grp = tid >> gsh, gl = tid & (GS - 1);
                const int t = tt * q.TF + grp * fpw + fi;
                const cpx* Z = reinterpret_cast<const cpx*>(smem + L.buf + (grp * 2 + (q.n_pass & 1)) * bufsz);
                const bool zp = q.pad1 && q.n_pass == 1;   // a single pass leaves its (padded) output as the spectrum
                if (t < p.T) {
                    const long long o = obase + (long long)t * p.o_st;
                    float2* oc = reinterpret_cast<float2*>(p.out) + o;
                    float* orl = reinterpret_cast<float*>(p.out) + o;
                    float* mcol = mag_s + (grp * fpw + fi);          // FRT > 0: this frame's column of the magnitude tile
                    (void)mcol;
                    float rmax = R.runmax;
                    const long long sk = p.o_sk;
                    // all bins of the frame through emit(k, X[k]); the output form is picked once per frame, not per bin
                    auto bins = [&](auto emit) {
                        if (q.half) {
                            // X[k]   = (Z[k] + conj Z[P-k]) / 2 - i/2 exp(-2 pi i k / N) (Z[k] - conj Z[P-k]),  k = 0 .. P/2,  and from
                            // the same operands its mirror image X[P-k] = conj((Z[k] + conj Z[P-k]) / 2 + i/2 exp(..) (Z[k] - conj Z[P-k]))
                            const int hk = P >> 1;
                            for (int k = gl; k <= hk; k += GS) {
                                const int km = P - k, ib = k == 0 ? 0 : km;
                                const cpx a = Z[zp ? k + (k >> 4) : k];
                                const cpx bq = Z[zp ? ib + (ib >> 4) : ib];
                                const cpx e = cadd_conj(a, bq), dd = csub_conj(a, bq);
#if defined(KB_HOST_EMU)
                                const float2 w2 = p.tw[k];
#else
                                const float2 w2 = __ldg(p.tw + k);
#endif
                                const cpx tq = cmul(cmake(dd.im, -dd.re), cmake(w2.x, w2.y));
                                emit(k, cscale(cadd(e, tq), 0.5f));
                                if (km != k) {
                                    const cpx xm = cscale(csub(e, tq), 0.5f);
                                    emit(km, cmake(xm.re, -xm.im));
                                }
                            }
                        } else {
                            for (int k = gl; k < F; k += GS) emit(k, Z[zp ? k + (k >> 4) : k]);
                        }
                    };
                    auto db = [&](float v) {
                        v = kb_floor_keepnan(v, q.amin);
                        rmax = kb_max_keepnan(rmax, v);
                        return q.db_mul * (q.db_ftz ? kb_lg2_ftz(v) : kb_log2(v)) - q.db_sub;
                    };
                    if (FRT > 0) bins([&](int k, cpx X) { mcol[k * RS] = kb_sqrt(cnorm(X)); });
                    else if (p.mode == KB_OUT_COMPLEX) {
                        if (q.sk1) bins([&](int k, cpx X) { oc[k] = make_float2(X.re, X.im); });
                        else bins([&](int k, cpx X) { oc[k * sk] = make_float2(X.re, X.im); });
                    } else if (p.mode == KB_OUT_MAG_DB) {
                        if (q.sk1) bins([&](int k, cpx X) { orl[k] = db(kb_cabs(X)); });
                        else bins([&](int k, cpx X) { orl[k * sk] = db(kb_cabs(X)); });
                    } else {
                        if (q.sk1) bins([&](int k, cpx X) { orl[k] = kb_cabs(X); });
                        else bins([&](int k, cpx X) { orl[k * sk] = kb_cabs(X); });
                    }
                    R.runmax = rmax;
                }
            KB_PHASE_END
            KB_MR_SYNC;
        }
        if (FRT > 0) {
            // ---- filterbank over the tile: lane = frame column, warps stride over the bands (as kb_fb_cta_r) ----
            KB_SYNC_CTA;
            KB_PHASE_BEGIN
                (void)R;
                const int warp = tid >> 5, lane = tid & 31;
                // a tile narrower than a warp (FRT 16 / 8): 32 / FRT bands per trip, so that no lane idles
                constexpr int FW = FRT > 0 ? FRT : 32, BPT = 32 / FW;
                const int f = lane & (FW - 1), sub = lane / FW;
                const float* mcol = mag_s + f;
                for (int m = warp * BPT + sub; m < q.n_bands; m += NW * BPT) {
                    const KbBand bd = q.bands[m];
                    out_s[f * L.Mp + m] = kb_band_dot<RS>(q.fbw + bd.off, mcol + bd.lo * RS, (bd.hi - bd.lo) >> 2);
                }
            KB_PHASE_END
            KB_SYNC_CTA;
            // ---- decibel + coalesced copy-out of the (FRT x n_bands) block ----
            KB_PHASE_BEGIN
                const int warp = tid >> 5, lane = tid & 31;
                float* o = reinterpret_cast<float*>(p.out) + obase;
                const int M = q.n_bands;
                float rmax = R.runmax;
                for (int r = warp; r < FRT; r += NW) {
                    const int t = tt * q.TF + r;
                    if (t >= p.T) continue;
                    const float* srow = out_s + r * L.Mp;
                    float* orow = o + (long long)t * p.o_st;
                    for (int m = lane; m < M; m += 32) {
                        float v = srow[m];
                        if (dbmode) {
                            v = kb_floor_keepnan(v, q.amin);
                            rmax = kb_max_keepnan(rmax, v);
                            v = q.db_mul * (q.db_ftz ? kb_lg2_ftz(v) : kb_log2(v)) - q.db_sub;
                        }
                        orow[(long long)m * p.o_sk] = v;
                    }
                }
                R.runmax = rmax;
            KB_PHASE_END
            KB_SYNC_CTA;      // the next tile's frames overwrite the magnitude tile
        }
        // ---- per-item maximum for the decibel clamp (kapre/backend.py:190-192) ----
        if (dbmode) {
#if defined(KB_HOST_EMU)
            for (int tid = 0; tid < kb_nt; ++tid)
                kb_atomic_max_u32(q.item_max + b, kb_f2u(kb_regs[tid].runmax));
#else
            const unsigned int wm = __reduce_max_sync(0xffffffffu, kb_f2u(kb_regs.runmax));
            if ((threadIdx.x & 31) == 0 && wm != 0u) kb_atomic_max_u32(q.item_max + b, wm);
#endif
        }
    }
}

#if defined(KB_HOST_EMU)
inline void kb_mr_cta(const KbMrParams& q, char* smem, int cta, int n_cta)
#else
__device__ __forceinline__ void kb_mr_cta(const KbMrParams& q, char* smem, int cta, int n_cta)
#endif
{
    switch (q.FRT) {
        case 32: kb_mr_cta_t<32>(q, smem, cta, n_cta); break;
        case 16: kb_mr_cta_t<16>(q, smem, cta, n_cta); break;
        case 8: kb_mr_cta_t<8>(q, smem, cta, n_cta); break;
        default: kb_mr_cta_t<0>(q, smem, cta, n_cta); break;
    }
}
