// Fused forward kernel body: frame + window + real FFT (+ |.| + filterbank + dB).
//
// Replaces, in one pass over the waveform, the reference op chain
//   kapre/time_frequency.py:164-187  (transpose, pad_begin, tf.signal.stft, transpose)
//   kapre/time_frequency.py:351-359  (tf.abs)
//   kapre/time_frequency.py:535-548  (tf.tensordot with the filterbank, transpose)
//   kapre/backend.py:186-188         (10*log10(max(x, amin)) - 10*log10(max(amin, ref)))
// The per-item clamp of kapre/backend.py:190-192 needs the item-wide maximum, so this
// kernel only reduces that maximum (atomicMax) and a second tiny kernel applies the clamp.
//
// Data movement: a persistent CTA walks tiles of TF consecutive frames of one (batch,
// channel) signal.  The hop-overlapped sample span of the NEXT tile is fetched with one TMA
// bulk copy (cp.async.bulk + mbarrier) into the other half of a double buffer while the
// current tile is transformed, so every sample is read from HBM/L2 once per tile and the
// load latency is off the critical path.  Strided (interleaved-channel) inputs use a
// cooperative fallback loader.
//
// Real FFT of length N as one complex FFT of length P = N/2 = 32*Q on the packed signal
// z[n] = x[2n] + i x[2n+1]; Q lanes of a warp cooperate on one frame (32/Q frames per warp):
//   pass 1  lane q: 32-point DFT over j of z[q + Q j]        (registers)
//           twiddle exp(-2 pi i q k1 / P), transpose through the warp's shared buffer
//   pass 2  lane q: Q-point DFTs over its columns (registers)
//   pair    X[k], X[P-k] from Z[k], Z[P-k] and exp(-2 pi i k / N)  -> output epilogue
//           paired-column form (n_fft <= 1024, most modes): the lane's columns are k1 = r and 32 - r, so both members of
//             every pair sit in its own registers (kb_col_gather_paired / kb_col_dftq_pair)
//           natural-order form (n_fft 2048, complex output at n_fft 512 / 256): columns k1 = q + Q i, Z written back
//             in natural order and re-read (kb_col_gather / kb_col_dftq_store + phase 4)
// Filterbank epilogue: magnitudes of the tile stay in shared memory ([bin][frame]); one lane
// per frame column accumulates a band with warp-uniform weights (vector loads from smem).
#pragma once
#include "fft_regs.cuh"

struct KbStftSmem {
    int wh, twp, twn, cwq, cw, cm, cg, bar, plan, samples, outs, ex, total;  // byte offsets
    int span;       // samples staged per tile
    int exw;        // complex elements per warp in the exchange buffer (incl. bank skew)
    int Mp;         // padded band stride of out_s
};

// Per-warp exchange region: 32 x 33 complex for the FFT transpose, plus a skew so that the
// magnitudes the filterbank phase reads from all warps' regions ([bin][frame-in-warp]) land in
// distinct banks for distinct frame columns.
KB_HD int kb_exw(int Q, int fbmma = 0) {
    const int FPW = 32 / Q;
    // region stride = 2112 + 2*FPW floats: the CUDA-core filterbank phase reads 2 bins x FPW frames per lane.
    // Tensor-core filterbank: stride = 2112 + 4*FPW floats, so that the A-fragment loads (8 frame rows x 4 bins
    // per instruction, kb_mma_a_off) hit 32 distinct banks for every Q.
    return 32 * 33 + (fbmma ? 2 * FPW : FPW);
}

// Shared-memory carve-up; used by the host launcher (size) and by the kernel (offsets).
KB_HD KbStftSmem kb_stft_smem_layout(int Q, int n_fft, int hop, int TF, int n_warps, int mode,
                                     int n_bands, int n_chunks, int fbmma = 0) {
    KbStftSmem s;
    const int P = 32 * Q;
    const bool fb = (mode == KB_OUT_FB || mode == KB_OUT_FB_DB);
    int off = 0;
    s.wh = off;  off += kb_align16(n_fft * 4);
    s.twp = off; off += kb_align16(Q * 33 * 8);
    s.twn = off; off += kb_align16((P / 2) * 8);
    s.cwq = off; off += Q * 16;
    s.cw = off; if (fb && !fbmma) off += n_chunks * 16;   // fbmma: n_chunks = number of k-steps, cm holds their descriptors
    s.cm = off; if (fb) off += kb_align16(n_chunks * 8);
    s.cg = off; if (fb) off += kb_align16(33 * 4);
    s.bar = off; off += 16;
    s.plan = off; off += 64;
    s.span = (TF - 1) * hop + n_fft;
    s.Mp = n_bands | 1;
    s.samples = off; off += kb_align16((s.span + 8) * 4);  // +4 front (alignment shift) +4 back (rounded copy)
    s.outs = off; if (fb) off += kb_align16(TF * s.Mp * 4);
    s.exw = kb_exw(Q, fbmma);
    s.ex = off;  off += kb_align16(n_warps * s.exw * 8);
    s.total = off;
    return s;
}

struct KbThreadRegs {
    cpx v[32];
    float runmax;
    cpx aux;          // inverse kernel: prefetched middle bin (lane 0)
};

#if defined(KB_HOST_EMU)
#include <vector>
#include <algorithm>
#define KB_PHASE_BEGIN for (int tid = 0; tid < kb_nt; ++tid) { KbThreadRegs& R = kb_regs[tid];
#define KB_PHASE_END }
#define KB_SYNC_WARP
#define KB_SYNC_CTA
static inline float kb_sqrt(float v) { return std::sqrt(v); }
static inline float kb_log2(float v) { return std::log2(v); }
static inline float kb_lg2_ftz(float v) { return std::log2(v); }
static inline float kb_fdividef(float a, float b) { return a / b; }
static inline float kb_ldg(const float* p) { return *p; }
static inline void kb_atomic_max_u32(unsigned int* p, unsigned int v) { if (v > *p) *p = v; }
static inline unsigned int kb_f2u(float f) { unsigned int u; std::memcpy(&u, &f, 4); return u; }
// Async staging primitives: a host model of the mbarrier protocol that checks how a body uses it.  An 8-byte KbBar in
// emulated shared memory cannot hold the model's state, so it lives in a table keyed by the barrier's address.  A bulk
// copy fills its destination with NaN and is performed only by the wait that completes its phase, so a read of the
// buffer before that wait, or a new copy into a buffer still being read, changes the output.  Every misuse the
// hardware would turn into a fault, a hang or a silent race counts as a violation (kb_emu_async_violations).  The
// model checks one ordering only, a copy that lands late: a copy landing early, so that a generic store into its
// destination before the wait would be lost, is not modelled, and neither is fence.proxy.async.
#include <map>
typedef unsigned long long KbBar;
struct KbEmuCopy { void* dst; const void* src; int bytes; };
struct KbEmuBar {
    unsigned long long phase = 0;           // completed phases
    int count = 0;                          // arrivals per phase (mbarrier.init)
    int arrived = 0;                        // arrivals in the current phase
    std::vector<KbEmuCopy> pending;         // bulk copies of the current phase
};
struct KbEmuAsync {
    std::map<const KbBar*, KbEmuBar> bars;
    long long violations = 0;
};
inline KbEmuAsync& kb_emu_async() { static KbEmuAsync s; return s; }
static inline void kb_bar_init(KbBar* b, int count) {
    KbEmuAsync& s = kb_emu_async();
    KbEmuBar& m = s.bars[b];
    if (!m.pending.empty()) ++s.violations;     // re-initialised while a copy into shared memory is in flight
    m = KbEmuBar{};
    m.count = count;
}
static inline void kb_bulk_g2s(void* dst, const void* src, int bytes, KbBar* bar) {
    KbEmuAsync& s = kb_emu_async();
    const auto it = s.bars.find(bar);
    const bool aligned = ((uintptr_t)dst & 15u) == 0 && ((uintptr_t)src & 15u) == 0 && (bytes & 15) == 0;
    const bool sized = bytes > 0 && bytes < (1 << 20);
    // with count arrivals per phase, one more arrive.expect_tx would complete a phase nobody waits for
    const bool accepts = it != s.bars.end() && it->second.arrived < it->second.count;
    if (!aligned || !sized || !accepts) ++s.violations;
    if (!sized || it == s.bars.end()) return;
    ++it->second.arrived;
    it->second.pending.push_back({dst, src, bytes});
    const unsigned nan = 0x7fc0deadu;
    for (int i = 0; i + 4 <= bytes; i += 4) std::memcpy(static_cast<char*>(dst) + i, &nan, 4);
}
// mbarrier.try_wait.parity: returns once the phase with parity `parity` has completed.  The body's phases run one
// after another for all threads, so a wait never has to wait for a copy issued after it: a wait that finds its phase
// current with copies pending completes it (performs the copies), one that finds it current with nothing pending
// would hang, and one that finds it complete while copies of the current phase are pending, or that names the phase
// before the first (which the hardware reports as complete; no body here relies on that), has the wrong parity.
static inline void kb_bar_wait(KbBar* bar, unsigned parity) {
    KbEmuAsync& s = kb_emu_async();
    const auto it = s.bars.find(bar);
    if (it == s.bars.end()) { ++s.violations; return; }
    KbEmuBar& m = it->second;
    if ((m.phase & 1u) != (parity & 1u)) {
        if (m.phase == 0 || !m.pending.empty()) ++s.violations;
        return;
    }
    if (m.pending.empty() || m.arrived < m.count) { ++s.violations; return; }
    for (const KbEmuCopy& c : m.pending) std::memcpy(c.dst, c.src, (size_t)c.bytes);
    m.pending.clear();
    m.arrived = 0;
    ++m.phase;
}
// Exported by every emulation library (each is one translation unit that includes this header): the violations since
// the last reset, plus one per barrier that still has copies in flight (a CTA that exits before its copies land).
extern "C" __attribute__((used)) inline long long kb_emu_async_violations(void) {
    const KbEmuAsync& s = kb_emu_async();
    long long n = s.violations;
    for (const auto& kv : s.bars) n += kv.second.pending.empty() ? 0 : 1;
    return n;
}
extern "C" __attribute__((used)) inline void kb_emu_async_reset(void) {
    KbEmuAsync& s = kb_emu_async();
    s.bars.clear();
    s.violations = 0;
}
#else
#define KB_PHASE_BEGIN { const int tid = threadIdx.x; KbThreadRegs& R = kb_regs;
#define KB_PHASE_END }
#define KB_SYNC_WARP __syncwarp()
#define KB_SYNC_CTA __syncthreads()
KB_D float kb_sqrt(float v) { float r; asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(v)); return r; }
KB_D float kb_log2(float v) { return __log2f(v); }
KB_D float kb_lg2_ftz(float v) { float r; asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(v)); return r; }
KB_D float kb_fdividef(float a, float b) { return __fdividef(a, b); }
KB_D float kb_ldg(const float* p) { return __ldg(p); }
KB_D void kb_atomic_max_u32(unsigned int* p, unsigned int v) { atomicMax(p, v); }
KB_D unsigned int kb_f2u(float f) { return __float_as_uint(f); }
typedef unsigned long long KbBar;
KB_D unsigned int kb_smem_u32(const void* p) { return (unsigned int)__cvta_generic_to_shared(p); }
KB_D void kb_bar_init(KbBar* b, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(kb_smem_u32(b)), "r"(count) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
// One TMA bulk copy global -> shared (SASS: UBLKCP), completion signalled on the mbarrier.
KB_D void kb_bulk_g2s(void* dst, const void* src, int bytes, KbBar* bar) {
    const unsigned int b = kb_smem_u32(bar);
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(b), "r"(bytes) : "memory");
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(kb_smem_u32(dst)), "l"(src), "r"(bytes), "r"(b) : "memory");
}
KB_D void kb_bar_wait(KbBar* bar, unsigned parity) {
    const unsigned int b = kb_smem_u32(bar);
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "KB_WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra KB_DONE_%=;\n\t"
        "bra KB_WAIT_%=;\n\t"
        "KB_DONE_%=:\n\t}"
        ::"r"(b), "r"(parity) : "memory");
}
#endif

// |re + i im| over the whole float range.  The squared norm underflows below |X| ~ 2^-63 (sqrt.approx.ftz flushes it
// to 0) and overflows above 2^64, so outside n in [2^-64, 2^64] both parts are first scaled by a power of two that
// brings max(|re|, |im|) to [1, 4).  The scale is exact and even in the squared norm, so the rescaled form gives the
// bits the plain form would give on the scaled input, and |2^k X| = 2^k |X| bit for bit while the result is normal.
// Inside the range both squares are normal floats unless one part is below 2^-31 of the other.  RN selects the form
// of the sites that round correctly, sqrtf(fmaf(re, re, im im)); otherwise kb_sqrt(cnorm(X)).  Zero, inf and NaN take
// the plain form.  The scales are built from their exponent bits (ldexpf is a library routine with branches).
KB_HD float kb_pow2(int e) {   // 2^e, -126 <= e <= 127
#if defined(__CUDA_ARCH__)
    return __uint_as_float((unsigned)(e + 127) << 23);
#else
    const uint32_t u = (uint32_t)(e + 127) << 23;
    float r;
    std::memcpy(&r, &u, 4);
    return r;
#endif
}
// The rescaled branch is rare; the STFT family's form keeps it out of line (__noinline__), so that the unrolled
// epilogues carry one compare per bin.  The correctly rounded form stays inline: its kernels use no stack.
template <bool RN>
#if defined(KB_HOST_EMU)
static inline float kb_cabs_rescaled(float re, float im)
#else
__device__ __forceinline__ float kb_cabs_rescaled(float re, float im)
#endif
{
    auto plain = [](float x, float y) { return RN ? sqrtf(fmaf(x, x, y * y)) : kb_sqrt(cnorm(cmake(x, y))); };
    const float a = fmaxf(fabsf(re), fabsf(im));
    if (!(a > 0.0f) || a > 3.40282347e38f) return plain(re, im);
    const int f = (int)(kb_f2u(a) >> 23);                          // biased exponent of a
    const int e = (f < 1 ? 1 : f > 253 ? 253 : f) - 127;           // a in [2^e, 2^(e+1)) unless subnormal / top
    const float down = kb_pow2(-e);
    return plain(re * down, im * down) * kb_pow2(e);
}
#if !defined(KB_HOST_EMU)
__device__ __noinline__ float kb_cabs_rescaled_approx(float re, float im) { return kb_cabs_rescaled<false>(re, im); }
#endif
template <bool RN = false>
#if defined(KB_HOST_EMU)
static inline float kb_cabs(float re, float im)
#else
KB_D float kb_cabs(float re, float im)
#endif
{
    const float n = RN ? fmaf(re, re, im * im) : cnorm(cmake(re, im));
    if (kb_f2u(n) - 0x1f800000u <= 0x40000000u) return RN ? sqrtf(n) : kb_sqrt(n);   // n in [2^-64, 2^64]
#if defined(KB_HOST_EMU)
    return kb_cabs_rescaled<RN>(re, im);
#else
    return RN ? kb_cabs_rescaled<true>(re, im) : kb_cabs_rescaled_approx(re, im);
#endif
}
#if defined(KB_HOST_EMU)
static inline float kb_cabs(cpx X) { return kb_cabs<false>(X.re, X.im); }
#else
KB_D float kb_cabs(cpx X) { return kb_cabs<false>(X.re, X.im); }
#endif

// atan2 for the Phase outputs (tf.math.angle, kapre/time_frequency.py:402): octant reduction to t = min / max in [0, 1],
// atan(t) = t + t s q(s), s = t^2, q a degree-7 minimax fit (weighted least squares on Chebyshev nodes): max error 2.8e-7 rad
// over random float32 arguments, the same as a correctly rounded float32 atan2 within 1 ulp of pi -- and ~20 instructions
// instead of the ~45 of atan2f (the magnitude + phase mode spends most of its time here).  Signed zeros and the quadrants
// follow atan2f; atan2(0, 0) = 0.
#if defined(KB_HOST_EMU)
static inline float kb_atan2(float y, float x)
#else
KB_D float kb_atan2(float y, float x)
#endif
{
    const float ax = fabsf(x), ay = fabsf(y);
    const float mx = fmaxf(ax, ay), mn = fminf(ax, ay);
    // __fdividef (mn times an approximate 1 / mx) returns 0 for 2^126 < mx < 2^128, and 1 / mx overflows for a
    // subnormal mx: scale both operands by a power of two first (exact, and 1 in between, where the quotient keeps
    // the bits of the unscaled division)
    const float sc = mx > 0x1p126f ? 0x1p-4f : mx < 0x1p-100f ? 0x1p24f : 1.0f;
    const float t = mx == 0.0f ? 0.0f : kb_fdividef(mn * sc, mx * sc);
    const float s = t * t;
    float r = 0.0026222908826366536f;
    r = fmaf(r, s, -0.015132737140170525f);
    r = fmaf(r, s, 0.04112221452660872f);
    r = fmaf(r, s, -0.07366738638336225f);
    r = fmaf(r, s, 0.10573948441726781f);
    r = fmaf(r, s, -0.14185979604290994f);
    r = fmaf(r, s, 0.199903971231639f);
    r = fmaf(r, s, -0.3333298707427664f);
    r = fmaf(r * s, t, t);
    if (ay > ax) r = 1.57079632679489662f - r;
    if (kb_f2u(x) >> 31) r = 3.14159265358979324f - r;   // incl. x = -0: atan2(+-0, -0) = +-pi
    return copysignf(r, y);
}

// ---- tensor-core filterbank primitives ------------------------------------------------------
// A-fragment element (frame f, bin k) of the tile's magnitudes: region of warp f / FPW, [bin][frame-in-warp].
template <int FPW>
KB_HD int kb_mma_a_off(int f, int RS) { return (f / FPW) * RS + (f % FPW); }
KB_HD float kb_tf32_trunc(float v) {
#if defined(__CUDA_ARCH__)
    return __uint_as_float(__float_as_uint(v) & 0xffffe000u);
#else
    uint32_t u; std::memcpy(&u, &v, 4); u &= 0xffffe000u; float r; std::memcpy(&r, &u, 4); return r;
#endif
}
#if !defined(KB_HOST_EMU)
// D += A (16x8, row) . B (8x8, col), TF32 inputs, fp32 accumulate (SASS: HMMA.1688.F32.TF32)
KB_D void kb_mma_tf32(float* d, const float* a, float b0, float b1) {
    asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(__float_as_uint(a[0])), "r"(__float_as_uint(a[1])), "r"(__float_as_uint(a[2])),
                   "r"(__float_as_uint(a[3])), "r"(__float_as_uint(b0)), "r"(__float_as_uint(b1)));
}
#endif

// Where a tile's samples come from.  Everything here is a pure function of the tile index,
// so every thread computes the same plan (no broadcast needed).
struct KbTilePlan {
    int b, c, t0;
    int s_first;         // first padded-signal sample of the tile (may be negative: pad_begin)
    int v0, v1;          // valid (non-pad) range in tile coordinates [v0, v1), v0 == v1: all pad
    int shift;           // smem index of tile sample i is i + shift
    int bulk;            // 1: one TMA bulk copy, 0: cooperative loads
    const float* src;    // 16 B-aligned source of the bulk copy
    int dst;             // smem float index (multiple of 4) of the bulk copy
    int bytes;           // multiple of 16
};

// Plan of the tile `tt` (index along time) of signal `sig` = b * C + c.
KB_HD KbTilePlan kb_plan_tile_at(const KbStftParams& p, int span, unsigned sig, int tt) {
    // Executed by every thread once or twice per tile, so it is kept to 32-bit arithmetic
    // except for the final pointer.
    KbTilePlan t;
    if (p.C == 1) { t.b = (int)sig; t.c = 0; }
    else { t.b = (int)(sig / (unsigned)p.C); t.c = (int)sig - t.b * p.C; }
    t.t0 = tt * p.TF;
    const int s_first = t.t0 * p.hop - p.pad_left;      // host guarantees T*hop + n_fft < 2^31
    t.s_first = s_first;
    int a = -s_first, e = p.L - s_first;
    if (a < 0) a = 0;
    if (e > span) e = span;
    if (e < a) e = a;
    t.v0 = a; t.v1 = e;
    t.shift = 0; t.bulk = 0; t.src = nullptr; t.dst = 0; t.bytes = 0;
    if (p.bulk_ok && e > a) {
        // element offsets of the first / one-past-last valid sample inside the waveform tensor
        const long long off0 = (long long)t.b * p.x_sb + (long long)t.c * p.x_sc + (s_first + a);
        const int head = (int)((p.x_align + (unsigned)off0) & 3u);           // floats before v0 in its 16 B line
        const int tail = (int)((0u - (p.x_align + (unsigned)off0 + (unsigned)(e - a))) & 3u);
        const long long lo = off0 - head, hi = off0 + (e - a) + tail;        // rounded range, in elements
        if (lo >= 0 && hi <= p.x_numel) {
            t.shift = (head - a) & 3;                                       // (v0 + shift - head) % 4 == 0
            t.bulk = 1;
            t.src = p.x + lo;
            t.dst = a + t.shift - head;
            t.bytes = (int)(hi - lo) * 4;
        }
    }
    return t;
}

KB_HD KbTilePlan kb_plan_tile(const KbStftParams& p, int span, int tile) {
    const unsigned sig = (unsigned)tile / (unsigned)p.n_tiles_t;
    return kb_plan_tile_at(p, span, sig, tile - (int)sig * p.n_tiles_t);
}

// Issue the loads of one tile into sample buffer `buf` (all threads call this).
// Pad regions are zero-filled with plain stores; the <= 3 floats on either side of the valid
// range that the 16 B-rounded bulk copy may overwrite are re-zeroed by kb_finish_tile_loads.
#if defined(KB_HOST_EMU)
inline void kb_issue_tile_loads(const KbStftParams& p, const KbTilePlan& t, float* buf, int span, KbBar* bar,
                                int tid, int nt)
#else
__device__ __forceinline__ void kb_issue_tile_loads(const KbStftParams& p, const KbTilePlan& t, float* buf,
                                                    int span, KbBar* bar, int tid, int nt)
#endif
{
    float* s = buf + t.shift;
    if (t.bulk) {
        if (tid == 0) kb_bulk_g2s(buf + t.dst, t.src, t.bytes, bar);
        for (int i = tid; i < t.v0 - 4; i += nt) s[i] = 0.0f;
        for (int i = t.v1 + 4 + tid; i < span; i += nt) s[i] = 0.0f;
    } else {
        const float* xsig = p.x + (long long)t.b * p.x_sb + (long long)t.c * p.x_sc + (long long)t.s_first * p.x_sl;
        int i = tid;
        for (; i + 3 * nt < span; i += 4 * nt) {   // 4 independent loads in flight per thread
            float v[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const int ii = i + u * nt;
                v[u] = (ii >= t.v0 && ii < t.v1) ? xsig[(long long)ii * p.x_sl] : 0.0f;
            }
#pragma unroll
            for (int u = 0; u < 4; ++u) s[i + u * nt] = v[u];
        }
        for (; i < span; i += nt) s[i] = (i >= t.v0 && i < t.v1) ? xsig[(long long)i * p.x_sl] : 0.0f;
    }
}

// After the bulk copy has landed: restore the zeros next to the valid range.  Returns
// whether anything was (possibly) written, i.e. whether a CTA barrier is needed.
#if defined(KB_HOST_EMU)
inline bool kb_finish_tile_loads(const KbTilePlan& t, float* buf, int span, int tid)
#else
__device__ __forceinline__ bool kb_finish_tile_loads(const KbTilePlan& t, float* buf, int span, int tid)
#endif
{
    if (!t.bulk) return false;
    const bool edge = (t.v0 > 0) || (t.v1 < span);
    if (edge && tid < 8) {
        float* s = buf + t.shift;
        const int i = (tid < 4) ? (t.v0 - 1 - tid) : (t.v1 + (tid - 4));
        if (i >= 0 && i < span && (i < t.v0 || i >= t.v1)) s[i] = 0.0f;
    }
    return edge;
}

// Filterbank accumulation for one band: warp-uniform weights (16 B vectors from smem), one
// frame column per lane; `mc` points at the column's magnitude for bin lo, consecutive bins are
// FPW floats apart ([bin][frame-in-warp] layout inside the owning warp's exchange region).
template <int FPW>
KB_HD float kb_band_dot(const float* __restrict__ w, const float* __restrict__ mc, int len4) {
    float a0 = 0.0f, a1 = 0.0f, a2 = 0.0f, a3 = 0.0f;
    for (int i = 0; i < len4; ++i) {
        const kb_f4 wv = reinterpret_cast<const kb_f4*>(w)[i];   // 16 B, warp-uniform address
        a0 += wv.x * mc[0];
        a1 += wv.y * mc[FPW];
        a2 += wv.z * mc[2 * FPW];
        a3 += wv.w * mc[3 * FPW];
        mc += 4 * FPW;
    }
    return (a0 + a1) + (a2 + a3);
}

// FPW consecutive floats (FPW in {1,2,4,8}) from a FPW*4-byte aligned shared address.
template <int FPW>
KB_HD void kb_load_vec(float* dst, const float* src) {
    if constexpr (FPW == 1) {
        dst[0] = src[0];
    } else if constexpr (FPW == 2) {
        const float2 v = *reinterpret_cast<const float2*>(src);
        dst[0] = v.x; dst[1] = v.y;
    } else {
#pragma unroll
        for (int j = 0; j < FPW / 4; ++j) {
            const kb_f4 v = reinterpret_cast<const kb_f4*>(src)[j];
            dst[4 * j] = v.x; dst[4 * j + 1] = v.y; dst[4 * j + 2] = v.z; dst[4 * j + 3] = v.w;
        }
    }
}

template <int FPW>
KB_HD void kb_store_vec(float* dst, const float* src) {
    if constexpr (FPW == 1) {
        dst[0] = src[0];
    } else if constexpr (FPW == 2) {
        float2 v; v.x = src[0]; v.y = src[1];
        *reinterpret_cast<float2*>(dst) = v;
    } else {
#pragma unroll
        for (int j = 0; j < FPW / 4; ++j) {
            kb_f4 v; v.x = src[4 * j]; v.y = src[4 * j + 1]; v.z = src[4 * j + 2]; v.w = src[4 * j + 3];
            reinterpret_cast<kb_f4*>(dst)[j] = v;
        }
    }
}

// ------------------------------------------------------------------------------------------
// The register FFT of one frame column, shared by the single-channel kernel below and the
// all-channel kernels of stft_mc_core.cuh.  A column is owned by the Q lanes (g, q = 0..Q-1) of a
// warp; `region` is the warp's exchange buffer.  Between the three steps the warp synchronises.
// ------------------------------------------------------------------------------------------
#if defined(KB_HOST_EMU)
#define KB_FN inline
#else
#define KB_FN __device__ __forceinline__
#endif

// Step 1: window the frame at `fr`, 32-point DFTs over z[q + Q j], twiddle, store transposed (32 x 33).
//   wmode 2: cosine-sum window evaluated in registers (KbStftParams::cwq), samples read as aligned pairs
//   wmode 1: window table, aligned pairs;  wmode 0: window table, scalar loads (odd sample offset)
template <int Q, bool TW0 = false>
KB_FN void kb_col_window_dft32(KbThreadRegs& R, const float* fr, const float* __restrict__ wh_s,
                               const kb_f4* __restrict__ cwq_s, float cw_a0, const cpx* __restrict__ twp_s,
                               cpx* region, int g, int q, int wmode) {
    if (wmode == 2) {
        // 0.5 w[2(q + Q j) + {0,1}] = a0 - cc * cos(2 pi j / 32) + ss * sin(2 pi j / 32)
        const kb_f4 cq = cwq_s[q];
        const cpx cc = cmake(cq.x, cq.y), ss = cmake(cq.z, cq.w);
        const cpx a0 = cmake(cw_a0, cw_a0);
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
    } else if (wmode == 1) {
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
    cpx* ex = region + (g * Q + q) * 33;
    const cpx* tw = twp_s + q * 33;
    ex[0] = TW0 ? cmul(R.v[0], tw[0]) : R.v[0];   // TW0: spectrum shift of column 0 for the paired-column form (kb_make_twp)
#pragma unroll
    for (int k1 = 1; k1 < 32; ++k1) ex[k1] = cmul(R.v[kb_brev<32>(k1)], tw[k1]);
}

// Step 2: gather the lane's columns k1 = q + Q i of the transposed buffer.
template <int Q>
KB_FN void kb_col_gather(KbThreadRegs& R, const cpx* region, int g, int q) {
    constexpr int FPW = 32 / Q;
    const cpx* ex = region + (g * Q) * 33;
#pragma unroll
    for (int i = 0; i < FPW; ++i) {
        const int k1 = q + Q * i;
#pragma unroll
        for (int q2 = 0; q2 < Q; ++q2) R.v[i * Q + q2] = ex[q2 * 33 + k1];
    }
}

// Step 3: Q-point DFTs, natural-order store Z[k1 + 32 k2] at region + g * zstr (aliases the transpose buffer).
template <int Q>
KB_FN void kb_col_dftq_store(KbThreadRegs& R, cpx* region, int g, int q, int zstr) {
    constexpr int FPW = 32 / Q;
    cpx* zs = region + g * zstr;
#pragma unroll
    for (int i = 0; i < FPW; ++i) {
        kb_fft_dif<Q>(R.v + i * Q);
        const int k1 = q + Q * i;
#pragma unroll
        for (int k2 = 0; k2 < Q; ++k2) zs[k1 + 32 * k2] = R.v[i * Q + kb_brev<Q>(k2)];
    }
}

// ------------------------------------------------------------------------------------------
// Paired-column form of steps 2-4 for the fused filterbank modes (Q <= 16, i.e. two or more columns per lane).
// The real-FFT pair step combines Z[k] with Z[P - k]; with k = k1 + 32 k2 the partner of column k1 is column
// 32 - k1.  Dealing the columns so that lane q owns BOTH k1 = r and k1 = 32 - r (r = q + Q u, u < 16 / Q) keeps every
// pair inside one lane: the natural-order store, its re-read and the register parking of the magnitudes disappear
// (2 of the 5 trips of a spectrum through shared memory), and the magnitudes go straight to [bin][frame].
// The two self-paired columns k1 = 0 and k1 = 16 form lane 0's first pair; there the partners sit inside one column,
// which costs Q complex selects: column 16 is loaded as `a`, column 0 as `b`, pre-shifted cyclically by s = Q/2 + 1
// (a modulation folded into the twiddle table, kb_make_twp) so that slot i pairs
//     i <  Q/2:  A = a[i]      (bin 16 + 32 i),      B = a[Q-1-i]   (instead of b[Q-1-i])
//     i >= Q/2:  A = b'[i-1]   (bin 32 (i - Q/2)),   B = b'[Q-1-i]  (the generic register)
// and b'[Q-1] is the middle bin P/2.  Slots i >= Q/2 are bins >= P/2: W^k = -i W^(k - P/2), table twn2 (kb_make_twn2).
// ------------------------------------------------------------------------------------------
KB_HD cpx csel(bool c, cpx a, cpx b) { return cmake(c ? a.re : b.re, c ? a.im : b.im); }

template <int Q>
KB_FN void kb_col_gather_paired(KbThreadRegs& R, const cpx* region, int g, int q) {
    constexpr int CP = 16 / Q;   // column pairs per lane
    const cpx* ex = region + (g * Q) * 33;
#pragma unroll
    for (int u = 0; u < CP; ++u) {
        const int r = q + Q * u;
        const int kA = (r == 0) ? 16 : r, kB = (r == 0) ? 0 : 32 - r;
#pragma unroll
        for (int q2 = 0; q2 < Q; ++q2) {
            R.v[(2 * u) * Q + q2] = ex[q2 * 33 + kA];
            R.v[(2 * u + 1) * Q + q2] = ex[q2 * 33 + kB];
        }
    }
}

// Q-point DFTs of the lane's column pairs and the pair step; emit(k, X, cj) receives bin k of the frame: X[k] = X, or
// conj(X) when cj (the mirror image P - k of a slot).
template <int Q, class Emit>
KB_FN void kb_col_dftq_pair(KbThreadRegs& R, const cpx* __restrict__ twn2_s, int q, Emit emit) {
    constexpr int CP = 16 / Q, P = 32 * Q, H = Q / 2;
#pragma unroll
    for (int u = 0; u < CP; ++u) {
        cpx* a = R.v + (2 * u) * Q;
        cpx* b = R.v + (2 * u + 1) * Q;
        kb_fft_dif<Q>(a);
        kb_fft_dif<Q>(b);
        const int r = q + Q * u;
        const bool sp = (u == 0) && (q == 0);      // the self-paired columns
        const int kLo = sp ? 16 : r;               // slot i < H:  bin kLo + 32 i
        const int kHi = sp ? -(P / 2) : r;         // slot i >= H: bin kHi + 32 i
        const int tHi = sp ? 0 : r;                // twiddle index of slot i >= H: tHi + 32 i - P/2
#pragma unroll
        for (int i = 0; i < Q; ++i) {
            cpx A, Bv;
            if (i < H) {
                A = a[kb_brev<Q>(i)];
                Bv = (u == 0) ? csel(sp, a[kb_brev<Q>(Q - 1 - i)], b[kb_brev<Q>(Q - 1 - i)]) : b[kb_brev<Q>(Q - 1 - i)];
            } else {
                A = (u == 0) ? csel(sp, b[kb_brev<Q>(i - 1)], a[kb_brev<Q>(i)]) : a[kb_brev<Q>(i)];
                Bv = b[kb_brev<Q>(Q - 1 - i)];
            }
            const cpx E = cadd_conj(A, Bv);            // A + conj(B)
            const cpx D = csub_conj(A, Bv);            // A - conj(B)
            cpx X1, X2;
            if (i < H) {
                const cpx T = cmul(cmake(D.im, -D.re), twn2_s[kLo + 32 * i]);   // W^k (-i D)
                X1 = cadd(E, T);
                X2 = csub(E, T);
            } else {
                const cpx G = cmul(D, twn2_s[tHi + (32 * i - P / 2)]);          // W^k (-i D) = -W^(k - P/2) D
                X1 = csub(E, G);
                X2 = cadd(E, G);
            }
            const int k = (i < H ? kLo : kHi) + 32 * i;
            emit(k, X1, false);
            emit(P - k, X2, true);                     // X2 = conj(X[P - k])
        }
        if (u == 0) {
            if (sp) {   // bin P/2 pairs with itself
                const cpx A = b[kb_brev<Q>(Q - 1)];
                emit(P / 2, cmake(2.0f * A.re, -2.0f * A.im), false);
            }
        }
    }
}

// fused filterbank modes: magnitudes -> mw[bin * FPW + g] (the warp's own exchange region, layout [bin][frame-in-warp])
template <int Q>
KB_FN void kb_col_dftq_pair_mag(KbThreadRegs& R, const cpx* __restrict__ twn2_s, float* mw, int g, int q) {
    constexpr int FPW = 32 / Q;
    float* mg = mw + g;
    kb_col_dftq_pair<Q>(R, twn2_s, q, [&](int k, cpx X, bool) { mg[k * FPW] = kb_sqrt(cnorm(X)); });
}

// ------------------------------------------------------------------------------------------
// Filterbank phase on the tensor pipe: out[frame][band] += mag[frame][bin] . fb[bin][band] as a
// block-banded GEMM of mma.sync m16n8k8 tiles (frames x 8 bins) . (8 bins x 8 bands), fp32-grade through the
// 3xTF32 split (A_lo.B_hi + A_hi.B_lo + A_hi.B_hi; the lo parts are exact differences).  Replaces
// tf.tensordot of kapre/time_frequency.py:544.  A warp walks the job slots w, w + NW, ... of
// kb_make_fb_mma; B fragments come pre-split from global memory (one 16 B load per lane and k-step,
// prefetched one step ahead), A fragments are read from the warps' exchange regions and split in registers.
// ------------------------------------------------------------------------------------------
template <int Q>
KB_FN void kb_fb_mma_load_a(const float* __restrict__ exf, int RS, int FR, int mt, int lane, int k0, float* a) {
    constexpr int FPW = 32 / Q;
    const int g = lane >> 2, t = lane & 3;
    const int f0 = 16 * mt + g, f1 = f0 + 8;
    const float* ap = exf + (k0 + t) * FPW;
    if (f0 < FR) {
        const float* r = ap + kb_mma_a_off<FPW>(f0, RS);
        a[0] = r[0]; a[2] = r[4 * FPW];
    } else { a[0] = 0.0f; a[2] = 0.0f; }
    if (f1 < FR) {
        const float* r = ap + kb_mma_a_off<FPW>(f1, RS);
        a[1] = r[0]; a[3] = r[4 * FPW];
    } else { a[1] = 0.0f; a[3] = 0.0f; }
}

// accumulator fragment -> out_s[frame][band] (added: a column tile may be split over two jobs)
KB_FN void kb_fb_mma_flush(float* out_s, int Mp, int n_bands, int FR, int mt, int lane, int j, const float* acc) {
    const int g = lane >> 2, t = lane & 3;
    const int col = 8 * j + 2 * t;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int f = 16 * mt + g + 8 * h;
        if (f < FR) {
            float* o = out_s + f * Mp + col;
#if defined(KB_HOST_EMU)
            if (col < n_bands) o[0] += acc[2 * h];
            if (col + 1 < n_bands) o[1] += acc[2 * h + 1];
#else
            if (col < n_bands) atomicAdd(o, acc[2 * h]);
            if (col + 1 < n_bands) atomicAdd(o + 1, acc[2 * h + 1]);
#endif
        }
    }
}

#if defined(KB_HOST_EMU)
// Emulation of the whole phase: the fragments are gathered with the device code's per-lane addressing
// (kb_fb_mma_load_a / the mw table / kb_fb_mma_flush) and multiplied as dense tiles per the PTX layouts
// of mma.m16n8k8: A row g(+8) col t(+4); B row t(+4) col g; D row g(+8) cols 2t, 2t+1.
template <int Q>
inline void kb_fb_mma_phase(const float* exf, int RS, int FR, const kb_f4* mw, const kb_i2* ms_s, const int* mg_s,
                            float* out_s, int Mp, int n_bands, int NW) {
    const int MT = (FR + 15) >> 4;
    for (int warp = 0; warp < NW; ++warp)
        for (int slot = warp; slot < KB_MMA_SLOTS; slot += NW) {
            std::vector<float> acc(2 * 32 * 4, 0.0f);
            for (int i = mg_s[slot]; i < mg_s[slot + 1]; ++i) {
                const kb_i2 sd = ms_s[i];
                for (int mt = 0; mt < MT; ++mt) {
                    float Ah[16][8], Al[16][8], Bh[8][8], Bl[8][8];
                    for (int lane = 0; lane < 32; ++lane) {
                        const int g = lane >> 2, t = lane & 3;
                        float a[4];
                        kb_fb_mma_load_a<Q>(exf, RS, FR, mt, lane, sd.x, a);
                        const int rr[4] = {g, g + 8, g, g + 8}, cc[4] = {t, t, t + 4, t + 4};
                        for (int e = 0; e < 4; ++e) {
                            const float hi = kb_tf32_trunc(a[e]);
                            Ah[rr[e]][cc[e]] = hi;
                            Al[rr[e]][cc[e]] = kb_tf32_trunc(a[e] - hi);
                        }
                        const kb_f4 b = mw[(size_t)i * 32 + lane];
                        Bh[t][g] = b.x; Bh[t + 4][g] = b.y;
                        Bl[t][g] = kb_tf32_trunc(b.z); Bl[t + 4][g] = kb_tf32_trunc(b.w);
                    }
                    for (int lane = 0; lane < 32; ++lane) {
                        const int g = lane >> 2, t = lane & 3;
                        for (int e = 0; e < 4; ++e) {
                            const int r = g + 8 * (e >> 1), c = 2 * t + (e & 1);
                            float d = acc[(mt * 32 + lane) * 4 + e];
                            float s1 = 0.0f, s2 = 0.0f, s3 = 0.0f;
                            for (int k = 0; k < 8; ++k) { s1 += Al[r][k] * Bh[k][c]; s2 += Ah[r][k] * Bl[k][c]; s3 += Ah[r][k] * Bh[k][c]; }
                            d += s1; d += s2; d += s3;
                            acc[(mt * 32 + lane) * 4 + e] = d;
                        }
                    }
                }
                if (sd.y >= 0) {
                    for (int mt = 0; mt < MT; ++mt)
                        for (int lane = 0; lane < 32; ++lane) {
                            kb_fb_mma_flush(out_s, Mp, n_bands, FR, mt, lane, sd.y, &acc[(mt * 32 + lane) * 4]);
                            for (int e = 0; e < 4; ++e) acc[(mt * 32 + lane) * 4 + e] = 0.0f;
                        }
                }
            }
        }
}
#else
template <int Q>
__device__ __forceinline__ void kb_fb_mma_phase(const float* __restrict__ exf, int RS, int FR,
                                                const kb_f4* __restrict__ mw, const kb_i2* __restrict__ ms_s,
                                                const int* __restrict__ mg_s, float* out_s, int Mp, int n_bands,
                                                int NW) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int MT = (FR + 15) >> 4;
    for (int slot = warp; slot < KB_MMA_SLOTS; slot += NW) {
        int i = mg_s[slot];
        const int e = mg_s[slot + 1];
        if (i >= e) continue;
        float acc[2][4];
#pragma unroll
        for (int mt = 0; mt < 2; ++mt)
#pragma unroll
            for (int q = 0; q < 4; ++q) acc[mt][q] = 0.0f;
        const float4* __restrict__ mw4 = reinterpret_cast<const float4*>(mw);
        float4 bn = __ldg(mw4 + (size_t)i * 32 + lane);
        for (; i < e; ++i) {
            const kb_i2 sd = ms_s[i];
            const float4 b = bn;
            if (i + 1 < e) bn = __ldg(mw4 + (size_t)(i + 1) * 32 + lane);
#pragma unroll
            for (int mt = 0; mt < 2; ++mt) {
                if (mt < MT) {
                    float a[4], ah[4], al[4];
                    kb_fb_mma_load_a<Q>(exf, RS, FR, mt, lane, sd.x, a);
#pragma unroll
                    for (int q = 0; q < 4; ++q) { ah[q] = kb_tf32_trunc(a[q]); al[q] = a[q] - ah[q]; }
                    kb_mma_tf32(acc[mt], al, b.x, b.y);
                    kb_mma_tf32(acc[mt], ah, b.z, b.w);
                    kb_mma_tf32(acc[mt], ah, b.x, b.y);
                }
            }
            if (sd.y >= 0) {
#pragma unroll
                for (int mt = 0; mt < 2; ++mt) {
                    if (mt < MT) {
                        kb_fb_mma_flush(out_s, Mp, n_bands, FR, mt, lane, sd.y, acc[mt]);
#pragma unroll
                        for (int q = 0; q < 4; ++q) acc[mt][q] = 0.0f;
                    }
                }
            }
        }
    }
}
#endif

// One CTA's share of the work: tiles cta, cta + n_cta, ...
template <int Q, int MODE, int FBMMA = 0>
#if defined(KB_HOST_EMU)
inline void kb_stft_cta(const KbStftParams& p, char* smem, int cta, int n_cta)
#else
__device__ __forceinline__ void kb_stft_cta(const KbStftParams& p, char* smem, int cta, int n_cta)
#endif
{
    constexpr int P = 32 * Q;        // complex FFT length
    constexpr int FPW = 32 / Q;      // frames per warp per round
    constexpr int ZSTR = P + Q;      // frame stride (complex) of the natural-order buffer
    constexpr bool fbmode = (MODE == KB_OUT_FB || MODE == KB_OUT_FB_DB);
    constexpr bool dbmode = (MODE == KB_OUT_MAG_DB || MODE == KB_OUT_FB_DB);
    const bool dbany = dbmode || (MODE == KB_OUT_MAG_PHASE && p.db_on);   // per-item maximum needed
    const int NW = p.n_warps;
    const int kb_nt = NW * 32;
    (void)kb_nt;
    const int H = p.hop, N = p.n_fft, TF = p.TF;
    // filterbank phase on the tensor pipe (kb_fb_mma_phase): a separate instantiation, kept selectable for the A/B
    // against the CUDA-core chunk lists (the default; chosen on the previous GPU target, not yet re-measured on H100)
    constexpr bool fbmma = fbmode && (FBMMA & 1) != 0;
    // Pair step: the paired-column form (kb_col_dftq_pair) whenever a lane owns two or more columns (n_fft <= 1024), except
    // where its output pattern costs more than the shared-memory trips it saves: a lane then writes bins q + 32 i, i.e. runs
    // of Q consecutive bins per frame instead of 32, which matters in the store-bound modes (complex output, magnitude +
    // phase) at small n_fft.  This selection is carried over from the previous GPU target, not yet re-measured on H100.
    // FBMMA bit 1 selects the other form (the A/B alternative).
    constexpr bool prefer_natural = (MODE == KB_OUT_COMPLEX && Q < 16) || (MODE == KB_OUT_MAG_PHASE && Q <= 8);
    constexpr bool paired = FPW >= 2 && !fbmma && (((FBMMA & 2) != 0) == prefer_natural);
    const KbStftSmem L = kb_stft_smem_layout(Q, N, H, TF, NW, MODE, p.n_bands, fbmma ? p.n_msteps : p.n_chunks,
                                             fbmma ? 1 : 0);
    float* __restrict__ wh_s = reinterpret_cast<float*>(smem + L.wh);
    cpx* __restrict__ twp_s = reinterpret_cast<cpx*>(smem + L.twp);
    cpx* __restrict__ twn_s = reinterpret_cast<cpx*>(smem + L.twn);
    kb_f4* __restrict__ cwq_s = reinterpret_cast<kb_f4*>(smem + L.cwq);
    kb_f4* __restrict__ cw_s = reinterpret_cast<kb_f4*>(smem + L.cw);
    kb_i2* __restrict__ cm_s = reinterpret_cast<kb_i2*>(smem + L.cm);
    int* __restrict__ cg_s = reinterpret_cast<int*>(smem + L.cg);
    KbBar* bar = reinterpret_cast<KbBar*>(smem + L.bar);
    KbTilePlan* plan_s = reinterpret_cast<KbTilePlan*>(smem + L.plan);   // next tile's plan (filterbank modes)
    float* smp0 = reinterpret_cast<float*>(smem + L.samples);
    float* __restrict__ out_s = reinterpret_cast<float*>(smem + L.outs);
    cpx* ex_s = reinterpret_cast<cpx*>(smem + L.ex);
    const int EXS = L.exw;                         // per-warp stride (complex) incl. bank skew
    const int FR = NW * FPW;                       // frames per round
    const int n_rounds = fbmode ? 1 : (TF + FR - 1) / FR;   // filterbank modes: TF == FR (host guarantees)
    const int n_tiles = p.B * p.C * p.n_tiles_t;
    const int span = L.span;

#if defined(KB_HOST_EMU)
    std::vector<KbThreadRegs> kb_regs(kb_nt);
#else
    KbThreadRegs kb_regs;
#endif

    // ---- one-time: tables to shared memory, barrier, first tile's loads ----------------------
    KB_PHASE_BEGIN
        (void)R;
        if (tid == 0) kb_bar_init(bar, 1);
        for (int i = tid; i < N; i += kb_nt) wh_s[i] = p.wh[i];
        for (int i = tid; i < Q * 33; i += kb_nt) { float2 t = p.twp[i]; twp_s[i] = cmake(t.x, t.y); }
        for (int i = tid; i < P / 2; i += kb_nt) { float2 t = paired ? p.twn2[i] : p.twn[i]; twn_s[i] = cmake(t.x, t.y); }
        if (p.cosw) { for (int i = tid; i < Q; i += kb_nt) cwq_s[i] = p.cwq[i]; }
        if (fbmma) {
            for (int i = tid; i < p.n_msteps; i += kb_nt) cm_s[i] = p.ms[i];
            for (int i = tid; i <= KB_MMA_SLOTS; i += kb_nt) cg_s[i] = p.mg[i];
            for (int i = tid; i < TF * L.Mp; i += kb_nt) out_s[i] = 0.0f;   // the phase accumulates into a zeroed tile
        } else if (fbmode && p.fb_bands) {   // band descriptors live where the per-chunk descriptors would (n_bd <= n_chunks)
            for (int i = tid; i < p.n_chunks; i += kb_nt) cw_s[i] = p.cw[i];
            for (int i = tid; i < p.n_bd; i += kb_nt) cm_s[i] = p.bd[i];
            for (int i = tid; i <= 32; i += kb_nt) cg_s[i] = p.bg[i];
        } else if (fbmode) {
            // chunk descriptors as byte offsets (first bin -> its magnitudes inside a warp's region, band -> its slot in an
            // out_s row): the loop's dependent load -> address -> load chain is one add long
            for (int i = tid; i < p.n_chunks; i += kb_nt) {
                cw_s[i] = p.cw[i];
                kb_i2 d = p.cm[i];
                d.x *= FPW * 4;
                d.y = d.y >= 0 ? d.y * 4 : -1;
                cm_s[i] = d;
            }
            for (int i = tid; i <= 32; i += kb_nt) cg_s[i] = p.cg[i];
        }
    KB_PHASE_END
    KB_SYNC_CTA;
#if !defined(KB_HOST_EMU)
    // Programmatic dependent launch: everything above only touched the plan's constant tables, so it
    // overlaps the tail of the previous kernel in the stream; data (waveform, output, item maxima)
    // is touched only after the predecessor has completed.  No-op without the launch attribute.
    asm volatile("griddepcontrol.wait;" ::: "memory");
    asm volatile("griddepcontrol.launch_dependents;");
#endif
    unsigned par = 0;   // mbarrier phase parity (uniform across the CTA)
    if (cta < n_tiles) {
        const KbTilePlan tp = kb_plan_tile(p, span, cta);
        KB_PHASE_BEGIN
            (void)R;
            kb_issue_tile_loads(p, tp, smp0, span, bar, tid, kb_nt);
        KB_PHASE_END
    }

    // filterbank modes step (signal, tile-in-signal) by n_cta tiles per iteration
    const unsigned step_sig = (unsigned)n_cta / (unsigned)p.n_tiles_t;
    const int step_tt = n_cta - (int)step_sig * p.n_tiles_t;
    unsigned nx_sig = (unsigned)cta / (unsigned)p.n_tiles_t;
    int nx_tt = cta - (int)nx_sig * p.n_tiles_t;
    for (int tile = cta; tile < n_tiles; tile += n_cta) {
        // filterbank modes: the plan was computed once when the tile's loads were issued and parked
        // in shared memory (a CTA barrier lies in between); otherwise recompute it (cheap per frame
        // there, tiles are larger)
        const KbTilePlan tp = (fbmode && tile != cta) ? *plan_s : kb_plan_tile(p, span, tile);
        const int b = tp.b, c = tp.c, t0 = tp.t0;
        const long long obase = (long long)b * p.o_sb + (long long)c * p.o_sc;
        const float* __restrict__ smp_s = smp0 + tp.shift;
        const bool has_next = (tile + n_cta) < n_tiles;

        // ---- wait for this tile's samples -----------------------------------------------------
        if (tp.bulk) {
            kb_bar_wait(bar, par);
            par ^= 1u;
        }
        {
            bool need = false;
            KB_PHASE_BEGIN
                R.runmax = 0.0f;
                need = kb_finish_tile_loads(tp, smp0, span, tid);
            KB_PHASE_END
            if (need || !tp.bulk) { KB_SYNC_CTA; }
        }
        const bool even_base = (((tp.shift & 1) == 0) && ((H & 1) == 0));

        for (int round = 0; round < n_rounds; ++round) {
            // ---- phase 1: window, 32-point DFTs, twiddle, transpose-store ------------------
            KB_PHASE_BEGIN
                const int warp = tid >> 5, lane = tid & 31;
                const int g = lane / Q, q = lane % Q;
                const int col = round * FR + warp * FPW + g;
                if (col < TF)
                    kb_col_window_dft32<Q, paired>(R, smp_s + col * H, wh_s, cwq_s, p.cw_a0, twp_s, ex_s + warp * EXS, g, q,
                                                   even_base ? (p.cosw ? 2 : 1) : 0);
            KB_PHASE_END
            if (round == n_rounds - 1 && !fbmode) {
                // every warp has consumed the sample buffer: fetch the next tile behind phases 2-4
                KB_SYNC_CTA;
                if (has_next) {
                    const KbTilePlan tn = kb_plan_tile(p, span, tile + n_cta);
                    KB_PHASE_BEGIN
                        (void)R;
                        kb_issue_tile_loads(p, tn, smp0, span, bar, tid, kb_nt);
                    KB_PHASE_END
                }
            } else {
                KB_SYNC_WARP;
            }
            if constexpr (paired) {
                // ---- phases 2-4, paired-column form: both members of every pair (k, P - k) in one lane --------
                KB_PHASE_BEGIN
                    const int warp = tid >> 5, lane = tid & 31;
                    const int g = lane / Q, q = lane % Q;
                    const int col = round * FR + warp * FPW + g;
                    if (col < TF) kb_col_gather_paired<Q>(R, ex_s + warp * EXS, g, q);
                KB_PHASE_END
                KB_SYNC_WARP;   // every lane has its columns: the region may be overwritten (magnitudes / next round)
                KB_PHASE_BEGIN
                    const int warp = tid >> 5, lane = tid & 31;
                    const int g = lane / Q, q = lane % Q;
                    const int col = round * FR + warp * FPW + g;
                    if constexpr (fbmode) {
                        float* mw = reinterpret_cast<float*>(ex_s + warp * EXS);
                        if (col < TF) kb_col_dftq_pair_mag<Q>(R, twn_s, mw, g, q);
                        if (lane < 3) {   // pad bins: chunks of 4 bins read past bin P
#pragma unroll
                            for (int gg = 0; gg < FPW; ++gg) mw[(P + 1 + lane) * FPW + gg] = 0.0f;
                        }
                    } else {
                        const int t = t0 + col;
                        if (col < TF && t < p.T) {
                            const long long ofr = obase + (long long)t * p.o_st;
                            const int sk = (int)p.o_sk;
                            float2* oc = reinterpret_cast<float2*>(p.out) + ofr;
                            float* orl = reinterpret_cast<float*>(p.out) + ofr;
                            float rmax = R.runmax;
                            kb_col_dftq_pair<Q>(R, twn_s, q, [&](int k, cpx X, bool cj) {
                                if (MODE == KB_OUT_COMPLEX) {
                                    const float2 v = make_float2(X.re, cj ? -X.im : X.im);
                                    if (sk == 1) oc[k] = v; else oc[k * sk] = v;
                                } else {
                                    float m = kb_cabs(X);
                                    if (MODE == KB_OUT_MAG_PHASE)   // tf.math.angle, kapre/time_frequency.py:402
                                        orl[(long long)k * sk + p.ph_off] = kb_atan2(cj ? -X.im : X.im, X.re);
                                    if (dbany) {
                                        m = kb_floor_keepnan(m, p.amin);
                                        rmax = kb_max_keepnan(rmax, m);
                                        m = p.db_mul * kb_log2(m) - p.db_sub;
                                    }
                                    if (sk == 1) orl[k] = m; else orl[k * sk] = m;
                                }
                            });
                            R.runmax = rmax;
                        }
                    }
                KB_PHASE_END
                if (!fbmode) { KB_SYNC_WARP; }
            } else {
            // ---- phase 2: gather this lane's columns --------------------------------------
            KB_PHASE_BEGIN
                const int warp = tid >> 5, lane = tid & 31;
                const int g = lane / Q, q = lane % Q;
                const int col = round * FR + warp * FPW + g;
                if (col < TF) kb_col_gather<Q>(R, ex_s + warp * EXS, g, q);
            KB_PHASE_END
            KB_SYNC_WARP;
            // ---- phase 3: Q-point DFTs, natural-order store (aliases the exchange buffer) ---
            KB_PHASE_BEGIN
                const int warp = tid >> 5, lane = tid & 31;
                const int g = lane / Q, q = lane % Q;
                const int col = round * FR + warp * FPW + g;
                if (col < TF) kb_col_dftq_store<Q>(R, ex_s + warp * EXS, g, q, ZSTR);
            KB_PHASE_END
            KB_SYNC_WARP;
            // ---- phase 4: real-FFT pair post-processing + epilogue -------------------------
            // Filterbank modes park the magnitudes in registers (R.v is dead) and store them in
            // phase 4b, because they overwrite the warp's natural-order buffer in place.
            KB_PHASE_BEGIN
                const int warp = tid >> 5, lane = tid & 31;
                float* magr = reinterpret_cast<float*>(R.v);
#pragma unroll
                for (int gg = 0; gg < FPW; ++gg) {
                    const int col = round * FR + warp * FPW + gg;
                    const int t = t0 + col;
                    if (col >= TF) break;
                    const bool valid = t < p.T;
                    const cpx* zf = ex_s + warp * EXS + gg * ZSTR;
                    const long long ofr = obase + (long long)t * p.o_st;
                    const int sk = (int)p.o_sk;
                    float2* oc = reinterpret_cast<float2*>(p.out) + ofr;
                    float* orl = reinterpret_cast<float*>(p.out) + ofr;
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
                            const cpx E = cadd_conj(A, Bv);            // A + conj(B)
                            const cpx D = csub_conj(A, Bv);            // A - conj(B)
                            const cpx T = cmul(cmake(D.im, -D.re), W); // W * (-i D)
                            X1 = cadd(E, T);
                            X2 = csub(E, T);                           // conj(X[P-k]); sign of Im fixed on store
                        } else {  // bin P/2 pairs with itself; only lane 0's value is used
                            k = P / 2;
                            kk = -1;
                            const cpx A = zf[P / 2];
                            X1 = cmake(2.0f * A.re, -2.0f * A.im);
                            X2 = X1;
                            if (!fbmode && lane != 0) continue;
                        }
                        if (MODE == KB_OUT_COMPLEX) {
                            if (valid) {
                                if (sk == 1) {
                                    oc[k] = make_float2(X1.re, X1.im);
                                    if (kk >= 0) oc[kk] = make_float2(X2.re, -X2.im);
                                } else {
                                    oc[k * sk] = make_float2(X1.re, X1.im);
                                    if (kk >= 0) oc[kk * sk] = make_float2(X2.re, -X2.im);
                                }
                            }
                        } else {
                            float m1 = fbmode ? kb_sqrt(cnorm(X1)) : kb_cabs(X1);
                            float m2 = fbmode ? kb_sqrt(cnorm(X2)) : kb_cabs(X2);
                            if (fbmode) {
                                magr[(gg * (Q / 2 + 1) + i) * 2 + 0] = m1;
                                magr[(gg * (Q / 2 + 1) + i) * 2 + 1] = m2;
                            } else if (valid) {
                                if (MODE == KB_OUT_MAG_PHASE) {   // tf.math.angle, kapre/time_frequency.py:402
                                    orl[(long long)k * sk + p.ph_off] = kb_atan2(X1.im, X1.re);
                                    if (kk >= 0) orl[(long long)kk * sk + p.ph_off] = kb_atan2(-X2.im, X2.re);
                                }
                                if (dbany) {
                                    m1 = kb_floor_keepnan(m1, p.amin);
                                    m2 = kb_floor_keepnan(m2, p.amin);
                                    R.runmax = kb_max_keepnan(R.runmax, m1);
                                    if (kk >= 0) R.runmax = kb_max_keepnan(R.runmax, m2);
                                    m1 = p.db_mul * kb_log2(m1) - p.db_sub;
                                    m2 = p.db_mul * kb_log2(m2) - p.db_sub;
                                }
                                if (sk == 1) {
                                    orl[k] = m1;
                                    if (kk >= 0) orl[kk] = m2;
                                } else {
                                    orl[k * sk] = m1;
                                    if (kk >= 0) orl[kk * sk] = m2;
                                }
                            }
                        }
                    }
                }
            KB_PHASE_END
            KB_SYNC_WARP;
            if (fbmode) {
                // ---- phase 4b: magnitudes -> own exchange region, layout [bin][frame-in-warp] ---
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
                    if (lane < (fbmma ? 7 : 3)) {   // pad bins: chunks of 4 bins / k-steps of 8 bins read past bin P
#pragma unroll
                        for (int gg = 0; gg < FPW; ++gg) mw[(P + 1 + lane) * FPW + gg] = 0.0f;
                    }
                KB_PHASE_END
            }
            }
        }  // rounds

        if (fbmode) {
            KB_SYNC_CTA;   // all magnitudes visible; sample buffer and out_s are free
            if (has_next) {
                // (signal, tile-in-signal) of the next tile, stepped without a division
                nx_sig += step_sig; nx_tt += step_tt;
                if (nx_tt >= p.n_tiles_t) { nx_tt -= p.n_tiles_t; ++nx_sig; }
                const KbTilePlan tn = kb_plan_tile_at(p, span, nx_sig, nx_tt);
                KB_PHASE_BEGIN
                    (void)R;
                    if (tid == 0) *plan_s = tn;
                    kb_issue_tile_loads(p, tn, smp0, span, bar, tid, kb_nt);
                KB_PHASE_END
            }
            // ---- phase 5: filterbank ------------------------------------------------------------
            // 32 lane groups of NW lanes; lane w of a group owns the FPW frame columns held in warp
            // w's exchange region (one vector load per bin), the group walks its list of 4-bin chunks.
            if (fbmma) {
                kb_fb_mma_phase<Q>(reinterpret_cast<const float*>(ex_s), 2 * EXS, FR, p.mw, cm_s, cg_s, out_s, L.Mp,
                                   p.n_bands, NW);
            } else if (p.fb_bands) {
            // two-level walk: bands of the lane group, then the band's 4-bin chunks (same sums in the same order as the
            // flat chunk list below, without the per-chunk flush test)
            KB_PHASE_BEGIN
                (void)R;
                const int warp = tid >> 5, lane = tid & 31;
                const int w = lane % NW;
                const int grp = warp * (32 / NW) + lane / NW;           // 0..31
                const float* __restrict__ mw = reinterpret_cast<const float*>(ex_s + w * EXS);
                float* __restrict__ ocol = out_s + (w * FPW) * L.Mp;
                const int be = cg_s[grp + 1];
                for (int bi = cg_s[grp]; bi < be; ++bi) {
                    const kb_i2 d = cm_s[bi];
                    const float* mp = mw + (d.x & 0xffff) * FPW;
                    const kb_f4* __restrict__ wp = cw_s + (d.y >> 16);
                    const int nch = d.x >> 16;
                    float a0[FPW], a1[FPW];
#pragma unroll
                    for (int g = 0; g < FPW; ++g) { a0[g] = 0.0f; a1[g] = 0.0f; }
                    for (int c = 0; c < nch; ++c) {
                        const kb_f4 wv = wp[c];
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
                        mp += 4 * FPW;
                    }
                    const int m = d.y & 0xffff;
#pragma unroll
                    for (int g = 0; g < FPW; ++g) ocol[g * L.Mp + m] = a0[g] + a1[g];
                }
            KB_PHASE_END
            } else {
            KB_PHASE_BEGIN
                (void)R;
                // NW is a power of two (kb_pick_fwd_cfg): lane group = tid / NW, lane within the group = tid % NW
                const int w = tid & (NW - 1);
                const int grp = tid >> kb_ilog2(NW);                    // 0..31
                const float* __restrict__ mw = reinterpret_cast<const float*>(ex_s + w * EXS);
                float* __restrict__ ocol = out_s + (w * FPW) * L.Mp;
                float a0[FPW], a1[FPW];
#pragma unroll
                for (int g = 0; g < FPW; ++g) { a0[g] = 0.0f; a1[g] = 0.0f; }
                const int ce = cg_s[grp + 1];
                for (int i = cg_s[grp]; i < ce; ++i) {
                    const kb_f4 wv = cw_s[i];                             // 16 B, uniform within the group
                    const kb_i2 mt = cm_s[i];                             // byte offsets (see the table prologue)
                    const float* mp = reinterpret_cast<const float*>(reinterpret_cast<const char*>(mw) + mt.x);
                    float m01[2 * FPW], m23[2 * FPW];          // bins (k, k+1) and (k+2, k+3), k even
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
                        float* ob = reinterpret_cast<float*>(reinterpret_cast<char*>(ocol) + mt.y);
#pragma unroll
                        for (int g = 0; g < FPW; ++g) {
                            ob[g * L.Mp] = a0[g] + a1[g];
                            a0[g] = 0.0f;
                            a1[g] = 0.0f;
                        }
                    }
                }
            KB_PHASE_END
            }
            KB_SYNC_CTA;
            // ---- phase 6: decibel + coalesced copy-out of the (TF x n_bands) block ----------
            KB_PHASE_BEGIN
                const int warp = tid >> 5, lane = tid & 31;
                float* o = reinterpret_cast<float*>(p.out) + obase;
                const int M = p.n_bands;
                const int sk = (int)p.o_sk;
                const float amin = p.amin, dmul = p.db_mul, dsub = p.db_sub;
                const bool ftz = p.db_ftz != 0;      // amin is a normal float: the bare MUFU.LG2 is exact enough
                float rmax = R.runmax;
                for (int colm = warp; colm < TF; colm += NW) {
                    const int t = t0 + colm;
                    float* srow = out_s + colm * L.Mp;
                    if (t >= p.T) {                  // frames past the end of the signal: nothing to write
                        if (fbmma) { for (int m = lane; m < M; m += 32) srow[m] = 0.0f; }
                        continue;
                    }
                    if (sk == 1) {
                        // contiguous rows: four values per lane and trip, immediate offsets
                        float* __restrict__ orow = o + (long long)t * p.o_st;
                        int m = lane;
                        for (; m + 96 < M; m += 128) {
                            float v[4];
#pragma unroll
                            for (int u = 0; u < 4; ++u) v[u] = srow[m + 32 * u];
                            if (fbmma) {             // the tensor-core phase accumulates into a zeroed tile
#pragma unroll
                                for (int u = 0; u < 4; ++u) srow[m + 32 * u] = 0.0f;
                            }
                            if (dbmode) {
#pragma unroll
                                for (int u = 0; u < 4; ++u) {
                                    v[u] = kb_floor_keepnan(v[u], amin);
                                    rmax = kb_max_keepnan(rmax, v[u]);
                                    v[u] = dmul * (ftz ? kb_lg2_ftz(v[u]) : kb_log2(v[u])) - dsub;
                                }
                            }
#pragma unroll
                            for (int u = 0; u < 4; ++u) orow[m + 32 * u] = v[u];
                        }
                        for (; m < M; m += 32) {
                            float v = srow[m];
                            if (fbmma) srow[m] = 0.0f;
                            if (dbmode) {
                                v = kb_floor_keepnan(v, amin);
                                rmax = kb_max_keepnan(rmax, v);
                                v = dmul * (ftz ? kb_lg2_ftz(v) : kb_log2(v)) - dsub;
                            }
                            orow[m] = v;
                        }
                    } else {
                        float* __restrict__ orow = o + (long long)t * p.o_st + lane * sk;
                        const int step = 32 * sk;
                        for (int m = lane; m < M; m += 32) {
                            float v = srow[m];
                            if (fbmma) srow[m] = 0.0f;
                            if (dbmode) {
                                v = kb_floor_keepnan(v, amin);
                                rmax = kb_max_keepnan(rmax, v);
                                v = dmul * (ftz ? kb_lg2_ftz(v) : kb_log2(v)) - dsub;
                            }
                            *orow = v;
                            orow += step;
                        }
                    }
                }
                R.runmax = rmax;
            KB_PHASE_END
        }

        // ---- per-item maximum for the decibel clamp (kapre/backend.py:190-192) --------------
        if (dbany) {
#if defined(KB_HOST_EMU)
            for (int tid = 0; tid < kb_nt; ++tid)
                kb_atomic_max_u32(p.item_max + b, kb_f2u(kb_regs[tid].runmax));
#else
            const unsigned int wm = __reduce_max_sync(0xffffffffu, kb_f2u(kb_regs.runmax));
            if ((threadIdx.x & 31) == 0 && wm != 0u) kb_atomic_max_u32(p.item_max + b, wm);
#endif
        }
        if (!fbmode) { KB_SYNC_WARP; }
    }
}
