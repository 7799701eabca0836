// kapre_b200 -- CUDA kernels (sm_90a) and the C ABI declared in include/kapre_b200.h.
//
// Kernel bodies live in stft_core.cuh / istft_core.cuh / aux_core.cuh (shared with the CPU
// emulation harness under tests/emu); this file holds the __global__ wrappers, the
// element-wise kernels, launch-configuration logic and the extern "C" entry points.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <atomic>
#include <functional>
#include <string>
#include <type_traits>
#include <utility>
#include <vector>

#include "../../include/kapre_b200.h"
#include "kb_tables.h"
#include "stft_core.cuh"
#include "stft_mc_core.cuh"
#include "istft_core.cuh"
#include "aux_core.cuh"
#include "mr_core.cuh"
#include "tc_dft.cuh"
#include "tc_mel.cuh"
#include "grad_core.cuh"
#include "grad_aux_core.cuh"
#include "resample_core.cuh"
#include "sinc_core.cuh"
#include "conv_core.cuh"
#include "pcen_core.cuh"
#include "gl_core.cuh"
#include "ts_core.cuh"
#include "fbinv_core.cuh"
#include "iir_core.cuh"
#include "sos_core.cuh"
#include "noise_core.cuh"
#include "kaldi_core.cuh"
#include "loudness_core.cuh"
#include "meter_core.cuh"
#include "cqt_core.cuh"
#include "pitch_core.cuh"
#include "chroma_core.cuh"
#include "hpss_core.cuh"
#include "rhythm_core.cuh"
#include "rir_core.cuh"

// ------------------------------------------------------------------------------------------
// error handling
// ------------------------------------------------------------------------------------------
static thread_local std::string g_err;
static thread_local std::string g_launch_info;
static std::atomic<uint64_t> g_launches{0};

// optional kernel timing (bench.py roofline): event pairs around the dominant kernels
#include <mutex>
static std::mutex g_prof_mu;
static int g_prof_on = 0;             // 0: off, n: every n-th dominant-kernel launch is bracketed by events
static std::atomic<uint64_t> g_prof_seq{0};
static std::vector<std::pair<cudaEvent_t, cudaEvent_t>> g_prof_events;

struct KbProfScope {
    cudaStream_t st;
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    KbProfScope(cudaStream_t s, bool timed) : st(s) {
        const int every = g_prof_on;
        if (!timed || !every) return;
        // sampling: an event record between two kernels serialises them (no programmatic dependent
        // launch across it), so a stride > 1 leaves most launches of a timed loop undisturbed
        if ((g_prof_seq++ % (uint64_t)every) != 0) return;
        if (cudaEventCreate(&e0) != cudaSuccess || cudaEventCreate(&e1) != cudaSuccess) { e0 = e1 = nullptr; return; }
        cudaEventRecord(e0, st);
    }
    ~KbProfScope() {
        if (!e0) return;
        cudaEventRecord(e1, st);
        std::lock_guard<std::mutex> lk(g_prof_mu);
        g_prof_events.emplace_back(e0, e1);
    }
};

static int kb_fail(int code, const char* fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    g_err = buf;
    return code;
}
#define KB_CUDA(expr)                                                                         \
    do {                                                                                      \
        cudaError_t e_ = (expr);                                                              \
        if (e_ != cudaSuccess)                                                                \
            return kb_fail(KAPRE_E_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e_), \
                           __FILE__, __LINE__);                                               \
    } while (0)

template <typename K>
static int kb_set_smem(K kernel, int smem) {
    if (smem > 48 * 1024)
        KB_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    return 0;
}

// One kernel launch.  Every launch of the library goes through kb_launch, which fixes two policies:
// - kapre_launch_count() counts each successful launch once;
// - `timed` launches are the ones kapre_profile_read() (bench.py's kernel time) brackets with events.
// `pdl`: programmatic dependent launch, so that the kernel is scheduled while the previous one in the stream drains.
// Only kernels whose body waits for the grid dependency (griddepcontrol.wait) may be launched that way.
// Call sites name the fields ({.grid = ..., .timed = true}; nvcc and its host compilers accept designated
// initializers in C++17 mode), so which launches are timed reads off each call.
struct KbLaunch {
    int grid, block, smem = 0;
    cudaStream_t st;
    bool pdl = false, timed = false;
};

template <typename... P, typename... A>
static int kb_launch(void (*kernel)(P...), const KbLaunch& l, A&&... args) {
    int rc = kb_set_smem(kernel, l.smem);
    if (rc) return rc;
    KbProfScope prof(l.st, l.timed);
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3((unsigned)l.grid);
    cfg.blockDim = dim3((unsigned)l.block);
    cfg.dynamicSmemBytes = (size_t)l.smem;
    cfg.stream = l.st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = l.pdl ? 1 : 0;
    KB_CUDA(cudaLaunchKernelEx(&cfg, kernel, std::forward<A>(args)...));
    g_launches++;
    return 0;
}

// Regions of one scratch buffer, each starting on a 256-byte boundary; with a null base it only measures.  Each
// operation's regions are described once, in a layout function that both its sizing function and the operation call,
// so the size a caller allocates and the regions the kernels write cannot drift apart.  take<T>(d0, d1, ...) reserves
// d0 d1 ... elements of T; a negative count, or a count or total beyond int64, sets `overflow` instead of wrapping.
struct KbLayout {
    char* base = nullptr;
    int64_t end = 0;
    bool overflow = false;
    void pad() {
        overflow |= __builtin_add_overflow(end, (int64_t)255, &end);
        end &= ~(int64_t)255;
    }
    template <typename T, typename... N>
    T* take(N... dims) {
        pad();
        const int64_t at = end;
        int64_t bytes = sizeof(T);
        for (const long long d : {(long long)dims...}) overflow |= d < 0 || __builtin_mul_overflow(bytes, (int64_t)d, &bytes);
        overflow |= __builtin_add_overflow(end, bytes, &end);
        return base && !overflow ? (T*)(base + at) : nullptr;
    }
    // what a sizing function returns: the total, or KAPRE_E_INVALID when it does not fit in int64
    int64_t bytes(const char* what) const {
        return overflow ? kb_fail(KAPRE_E_INVALID, "%s workspace overflows", what) : end;
    }
};

// SMs x resident threads per SM of the current device: the thread count the time-scan kernels (PCEN, time stretch)
// size their time chunks against.
static int kb_resident_threads(long long* threads) {
    int dev = 0, sms = 0, per_sm = 0;
    KB_CUDA(cudaGetDevice(&dev));
    KB_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    KB_CUDA(cudaDeviceGetAttribute(&per_sm, cudaDevAttrMaxThreadsPerMultiProcessor, dev));
    *threads = (long long)sms * per_sm;
    return 0;
}

// Grid of a persistent kernel whose CTAs loop over `tiles`: what fits on the device at once (a CTA that waited for a
// slot would start its share of the tiles late), and no more CTAs than tiles.  The shared-memory attribute is set
// first because the occupancy query needs it above 48 KiB.  The launch is reported as "<name> grid=G tiles=T"
// (kapre_last_launch_info), which tells whether a CTA walks more than one tile.
template <typename K>
static int kb_resident_grid(K kernel, const char* name, int block, int smem, long long tiles, int sm_count, int* grid) {
    int rc = kb_set_smem(kernel, smem);
    if (rc) return rc;
    int per_sm = 0;
    KB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, block, smem));
    if (per_sm < 1) per_sm = 1;
    const long long cap = (long long)sm_count * per_sm;
    *grid = (int)(tiles < cap ? tiles : cap);
    char buf[96];
    snprintf(buf, sizeof(buf), "%s grid=%d tiles=%lld", name, *grid, tiles);
    g_launch_info = buf;
    return 0;
}

// The launch report of a call that makes several persistent launches: add() after each launch keeps its report, and
// at the end of the call the report is all of them in launch order, joined with "; ", so that the grid of every
// launch can be read (kb_resident_grid alone would leave only the last).
struct KbLaunchReports {
    std::string all;
    void add() { all += (all.empty() ? "" : "; ") + g_launch_info; }
    ~KbLaunchReports() {
        if (!all.empty()) g_launch_info = all;
    }
};

// ------------------------------------------------------------------------------------------
// __global__ wrappers
// ------------------------------------------------------------------------------------------
template <int Q, int MODE>
__global__ void __launch_bounds__(KB_MAX_WARPS * 32, 2) kb_stft_kernel(const __grid_constant__ KbStftParams p) {
    extern __shared__ __align__(16) char kb_smem[];
    kb_stft_cta<Q, MODE>(p, kb_smem, (int)blockIdx.x, (int)gridDim.x);
}

// variant with the filterbank phase on the tensor pipe (mma.sync 3xTF32), selected by KAPRE_B200_FBMMA=1
template <int Q, int MODE>
__global__ void __launch_bounds__(KB_MAX_WARPS * 32, 2) kb_stft_kernel_mma(const __grid_constant__ KbStftParams p) {
    extern __shared__ __align__(16) char kb_smem[];
    kb_stft_cta<Q, MODE, 1>(p, kb_smem, (int)blockIdx.x, (int)gridDim.x);
}

// the A/B alternative of the pair step (template bit 1: natural-order pair step instead of the paired-column form)
template <int Q, int MODE, int V>
__global__ void __launch_bounds__(KB_MAX_WARPS * 32, 2) kb_stft_kernel_v(const __grid_constant__ KbStftParams p) {
    extern __shared__ __align__(16) char kb_smem[];
    kb_stft_cta<Q, MODE, V>(p, kb_smem, (int)blockIdx.x, (int)gridDim.x);
}

// 16-warp CTAs, one per SM: n_fft = 2048 in the filterbank modes, where an 8-warp CTA already needs more than
// half of the SM's shared memory (8.4 KB of exchange buffer per warp), so two CTAs never fit
template <int Q, int MODE>
__global__ void __launch_bounds__(512, 1) kb_stft_kernel_w16(const __grid_constant__ KbStftParams p) {
    extern __shared__ __align__(16) char kb_smem[];
    kb_stft_cta<Q, MODE>(p, kb_smem, (int)blockIdx.x, (int)gridDim.x);
}

template <int Q, int MODE>
__global__ void __launch_bounds__(KB_MAX_WARPS * 32, 2) kb_stft_mcfb_kernel(const __grid_constant__ KbStftParams p) {
    extern __shared__ __align__(16) char kb_smem[];
    kb_stft_mcfb_cta<Q, MODE>(p, kb_smem, blockIdx.x, gridDim.x);
}

// multi-channel tiles (interleaved tensors): up to 16 warps, one or two CTAs per SM
template <int Q, int MODE>
__global__ void __launch_bounds__(512, 1) kb_stft_mc_kernel(const __grid_constant__ KbStftParams p) {
    extern __shared__ __align__(16) char kb_smem[];
    kb_stft_mc_cta<Q, MODE>(p, kb_smem, blockIdx.x, gridDim.x);
}

// 4 warps per CTA (one FFT round per overlap class), two or three CTAs per SM: the register file is not the
// limit here, so the kernel may use up to 168 registers and keeps the round's global loads in flight.
#define KB_ISTFT_MAX_WARPS 4
template <int Q>
__global__ void __launch_bounds__(KB_ISTFT_MAX_WARPS * 32, 3) kb_istft_kernel(const __grid_constant__ KbIstftParams p) {
    extern __shared__ __align__(16) char kb_smem[];
    kb_istft_cta<Q>(p, kb_smem, (int)blockIdx.x, (int)gridDim.x);
}

__global__ void __launch_bounds__(KB_MAX_WARPS * 32) kb_fb_kernel(const __grid_constant__ KbFbParams p) {
    extern __shared__ __align__(16) char kb_smem[];
    kb_fb_cta(p, kb_smem, (int)blockIdx.x, (int)gridDim.x);
}

__global__ void __launch_bounds__(KB_MAX_WARPS * 32) kb_dft_kernel(const __grid_constant__ KbDftParams p) {
    extern __shared__ __align__(16) char kb_smem[];
    kb_dft_cta(p, kb_smem, (int)blockIdx.x, (int)gridDim.x);
}

__global__ void __launch_bounds__(512) kb_mr_kernel(const __grid_constant__ KbMrParams p) {
    extern __shared__ __align__(16) char kb_smem[];
    kb_mr_cta(p, kb_smem, (int)blockIdx.x, (int)gridDim.x);
}

__global__ void __launch_bounds__(KB_MAX_WARPS * 32) kb_idft_kernel(const __grid_constant__ KbIdftParams p) {
    extern __shared__ __align__(16) char kb_smem[];
    kb_idft_cta(p, kb_smem, (int)blockIdx.x, (int)gridDim.x);
}

// Dynamic-range clamp, kapre/backend.py:190-192: y = max(y, max_item(y) - dynamic_range).
// item_max holds max(x, amin) per item (uint view); log is monotone, so the item maximum in
// dB is dB(item_max).  `chunks` CTAs per item (so that one long item is rewritten by many CTAs when the
// clamp binds): each reads the maximum and returns immediately when the clamp cannot bind (threshold <=
// dB(amin)), which is the common case, so no output byte is re-read.  The workspace is
// SELF-CLEANING: words [0, n_items) are the maxima, words [n_items, 2 n_items) count the CTAs of an item that
// have read its maximum; the last one resets both to zero.  A NaN anywhere in an item makes its maximum NaN
// (the producers keep NaN through their max()), and tf.maximum(y, NaN) is NaN for the whole item.
// Launched with programmatic dependent launch: the grid is scheduled while the producer kernel drains.
__global__ void kb_db_clamp_kernel(float* __restrict__ y, long long item_size, long long run, long long period,
                                   unsigned int* __restrict__ item_max, unsigned int n_items, int chunks, float amin,
                                   float db_mul, float db_sub, float dyn_range) {
#if __CUDA_ARCH__ >= 900
    asm volatile("griddepcontrol.launch_dependents;");   // the next fused kernel may start its table prologue
    cudaGridDependencySynchronize();
#endif
    const long long item = blockIdx.x / chunks;
    const int chunk = (int)(blockIdx.x - item * chunks);
    __shared__ unsigned int s_mx;
    if (threadIdx.x == 0) s_mx = item_max[item];
    __syncthreads();
    if (threadIdx.x == 0) {
        // every CTA of the item has its copy of the maximum before the last arrival clears it
        unsigned int* cnt = item_max + n_items + item;
        if (chunks == 1 || atomicAdd(cnt, 1u) == (unsigned int)(chunks - 1)) {
            item_max[item] = 0u;
            if (chunks > 1) *cnt = 0u;
        }
    }
    const float mx = __uint_as_float(s_mx);
    float thr = (db_mul * __log2f(fmaxf(mx, amin)) - db_sub) - dyn_range;
    const float floor_db = db_mul * __log2f(amin) - db_sub;
    const bool nan_item = mx != mx;
    if (!nan_item && !(thr > floor_db)) return;
    if (nan_item) thr = mx;
    float* yi = y + item * item_size;
    const long long step = (long long)chunks * blockDim.x;
    // only elements with (i mod period) < run are decibel values (magnitude half of a mag+phase tensor)
    for (long long i = (long long)chunk * blockDim.x + threadIdx.x; i < item_size; i += step) {
        if (run >= period || i % period < run) yi[i] = nan_item ? thr : fmaxf(yi[i], thr);
    }
}

// Stand-alone MagnitudeToDecibel pass 1: y = db(max(x, amin)), per-item max of max(x, amin).
__global__ void kb_db_kernel(const float* __restrict__ x, float* __restrict__ y, long long item_size,
                             int chunks, unsigned int* __restrict__ item_max, float amin,
                             float db_mul, float db_sub) {
    const long long item = blockIdx.x / chunks;
    const int chunk = blockIdx.x - (int)(item * chunks);
    const float* xi = x + item * item_size;
    float* yi = y + item * item_size;
    unsigned int mxu = 0u;
    for (long long i = (long long)chunk * blockDim.x + threadIdx.x; i < item_size;
         i += (long long)chunks * blockDim.x) {
        const float xv = xi[i];
        const float v = xv < amin ? amin : xv;               // max that keeps NaN (tf.maximum propagates it)
        mxu = max(mxu, __float_as_uint(v));                    // v > 0 or NaN: the uint order is the float order, NaN on top
        yi[i] = db_mul * __log2f(v) - db_sub;
    }
    const unsigned int wm = __reduce_max_sync(0xffffffffu, mxu);
    if ((threadIdx.x & 31) == 0 && wm != 0u) atomicMax(item_max + item, wm);
}

__global__ void kb_magnitude_kernel(const float2* __restrict__ x, float* __restrict__ y, long long n) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n;
         i += (long long)gridDim.x * blockDim.x) {
        const float2 v = x[i];
        y[i] = kb_cabs(v.x, v.y);
    }
}

__global__ void kb_phase_kernel(const float2* __restrict__ x, float* __restrict__ y, long long n) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n;
         i += (long long)gridDim.x * blockDim.x) {
        const float2 v = x[i];
        y[i] = atan2f(v.y, v.x);
    }
}

// kapre.ConcatenateFrequencyMap (kapre/time_frequency.py:648-744): out = concat(x, linspace(0, 1, F) broadcast over
// (batch, time)) along the channel axis.  One pass: every output element is either a copy or the map value.
__global__ void kb_concat_freq_map_kernel(const float* __restrict__ x, float* __restrict__ y, long long B, long long C,
                                          long long T, long long F, int channels_last) {
    const long long Co = C + 1;
    const long long total = B * Co * T * F;
    const float step = F > 1 ? 1.0f / (float)(F - 1) : 0.0f;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        long long b, c, t, f;
        if (channels_last) { c = i % Co; f = (i / Co) % F; t = (i / (Co * F)) % T; b = i / (Co * F * T); }
        else { f = i % F; t = (i / F) % T; c = (i / (F * T)) % Co; b = i / (F * T * Co); }
        float v;
        if (c == C) v = (f == F - 1 && F > 1) ? 1.0f : (float)f * step;      // tf.linspace: exact end point
        else v = channels_last ? x[((b * T + t) * F + f) * C + c] : x[((b * C + c) * T + t) * F + f];
        y[i] = v;
    }
}

// kapre.SpecAugment (kapre/augmentation.py:116-326): per item, every element whose time index lies in one of the item's time
// masks [start, start + width] or whose frequency index lies in one of its frequency masks is replaced by mask_value
// (tf.where(mask, mask_value, x) after reduce_any over the masks).  The (start, width) pairs are drawn on the host
// (the reference draws them with tf.random.uniform per item and mask); depth is 1, so both data formats are (b, t, f).
__global__ void kb_spec_augment_kernel(const float* __restrict__ x, float* __restrict__ y, long long B, long long T, long long F,
                                       const int* __restrict__ tmask, int n_t, const int* __restrict__ fmask, int n_f,
                                       float mask_value) {
    const long long total = B * T * F;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const long long f = i % F, t = (i / F) % T, b = i / (F * T);
        bool m = false;
        for (int j = 0; j < n_t; ++j) {
            const int s0 = tmask[(b * n_t + j) * 2], w = tmask[(b * n_t + j) * 2 + 1];
            m = m || (t >= s0 && t <= s0 + w);
        }
        for (int j = 0; j < n_f; ++j) {
            const int s0 = fmask[(b * n_f + j) * 2], w = fmask[(b * n_f + j) * 2 + 1];
            m = m || (f >= s0 && f <= s0 + w);
        }
        y[i] = m ? mask_value : x[i];
    }
}

// ---- adjacent layers: Delta / Frame / Energy (element-wise or small-window kernels, HBM-bound) ----
// kb_pad_index (tf.pad's extension of the time axis) lives in grad_aux_core.cuh: Delta's backward uses it too.
__global__ void kb_delta_kernel(const float* __restrict__ x, float* __restrict__ y, long long outer, long long T,
                                long long inner, int n, float inv_denom, int mode) {
    const long long total = outer * T * inner;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const long long in = i % inner;
        const long long t = (i / inner) % T;
        const long long o = i / (inner * T);
        const float* base = x + o * T * inner + in;
        float acc = 0.0f;
        for (int m = 1; m <= n; ++m) {
            const long long tp = kb_pad_index(t + m, T, mode), tm = kb_pad_index(t - m, T, mode);
            const float a = tp >= 0 ? base[tp * inner] : 0.0f;
            const float b = tm >= 0 ? base[tm * inner] : 0.0f;
            acc += (float)m * (a - b);
        }
        y[i] = acc * inv_denom;
    }
}

__global__ void kb_frame_kernel(const float* __restrict__ x, long long x_sb, long long x_sc, long long x_sl, int B, int C,
                                int L, int fl, int hop, int T, float pad_value, float* __restrict__ out, long long o_sb,
                                long long o_sc, long long o_st, long long o_sk) {
    const long long total = (long long)B * C * T * fl;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int n = (int)(i % fl);
        const long long r = i / fl;
        const int t = (int)(r % T);
        const long long bc = r / T;
        const int c = (int)(bc % C), b = (int)(bc / C);
        const long long s = (long long)t * hop + n;
        const float v = s < L ? x[b * x_sb + c * x_sc + s * x_sl] : pad_value;
        out[b * o_sb + c * o_sc + t * o_st + n * o_sk] = v;
    }
}

__global__ void kb_energy_kernel(const float* __restrict__ x, long long x_sb, long long x_sc, long long x_sl, int B, int C,
                                 int L, int fl, int hop, int T, float pad_value, float scale, float* __restrict__ out,
                                 long long o_sb, long long o_sc, long long o_st) {
    const long long n_frames = (long long)B * C * T;
    const int lane = threadIdx.x & 31;
    const long long warp0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const long long n_warps = ((long long)gridDim.x * blockDim.x) >> 5;
    for (long long f = warp0; f < n_frames; f += n_warps) {
        const int t = (int)(f % T);
        const long long bc = f / T;
        const int c = (int)(bc % C), b = (int)(bc / C);
        const float* xs = x + b * x_sb + c * x_sc;
        float acc = 0.0f;
        for (int n = lane; n < fl; n += 32) {
            const long long s = (long long)t * hop + n;
            const float v = s < L ? xs[s * x_sl] : pad_value;
            acc += v * v;
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
        if (lane == 0) out[b * o_sb + c * o_sc + t * o_st] = scale * acc;
    }
}

// ------------------------------------------------------------------------------------------
// plans
// ------------------------------------------------------------------------------------------
struct DevInfo {
    int device = -1;
    int sm_count = 0;
    int smem_optin = 0;
};

static int kb_dev_info(DevInfo* d) {
    KB_CUDA(cudaGetDevice(&d->device));
    KB_CUDA(cudaDeviceGetAttribute(&d->sm_count, cudaDevAttrMultiProcessorCount, d->device));
    KB_CUDA(cudaDeviceGetAttribute(&d->smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, d->device));
    return 0;
}

// A plan's constant device tables: one allocation, freed when the plan is deleted.
struct KbTables {
    void* block = nullptr;
    KbTables() = default;
    KbTables(const KbTables&) = delete;
    KbTables& operator=(const KbTables&) = delete;
    ~KbTables() { cudaFree(block); }
};

// Builds a plan's KbTables.  add() copies a host array into a staging buffer, at the offset KbLayout gives it (each
// region on a 256-byte boundary), and keeps the plan field that is to point at it; the field of an empty array is set
// null.  upload() pads the end to 256 bytes, so that a bulk copy which rounds a table's size up stays inside the
// block, makes one allocation and one copy, and sets the fields.  A failed upload leaves `t` and the fields unset.
class KbTableUpload {
    KbLayout L;
    std::vector<char> host;
    std::vector<std::function<void(char*)>> fields;

  public:
    template <typename T, typename P>   // P: T or const T
    void add(const std::vector<T>& v, P** field) {
        static_assert(std::is_same<std::remove_const_t<P>, T>::value, "a table field points at the table's type");
        *field = nullptr;
        if (v.empty()) return;
        L.pad();
        const int64_t at = L.end;
        L.take<T>(v.size());
        host.resize(L.end);
        memcpy(host.data() + at, v.data(), v.size() * sizeof(T));
        fields.push_back([field, at](char* base) { *field = (P*)(base + at); });
    }
    int upload(KbTables& t, const char* what) {
        if (host.empty()) return 0;
        L.pad();
        host.resize(L.end);
        KbTables made;
        if (cudaMalloc(&made.block, L.end) != cudaSuccess) return kb_fail(KAPRE_E_NOMEM, "%s: plan allocation", what);
        if (cudaMemcpy(made.block, host.data(), L.end, cudaMemcpyHostToDevice) != cudaSuccess)
            return kb_fail(KAPRE_E_CUDA, "%s: plan upload", what);
        std::swap(t.block, made.block);
        for (auto& set : fields) set((char*)t.block);
        return 0;
    }
};

struct kapre_stft_plan {
    int n_fft, win_length, hop, Q;
    DevInfo dev;
    KbTables tables;
    float* wh = nullptr;      // fused path: 0.5 * window padded to n_fft
    kb_f4* cwq = nullptr;     // cosine-sum window factors (cosw), see KbStftParams
    int cosw = 0;
    float cw_a0 = 0.0f;
    float2* twp = nullptr;
    float2* twn = nullptr;
    float2* twn2 = nullptr;   // kb_make_twn2 (paired-column pair step)
    float* w = nullptr;       // generic path: window[0, win_eff)
    float2* tw = nullptr;     // generic path: exp(-2 pi i r / n_fft)
    int win_eff;
    // tensor-core path (tc_mel.cuh; n_fft = win_length = 1024, cosine-sum window a - b cos): constant operands
    double win_a = 0.0, win_b = 0.0;
    float* tc_f1 = nullptr;   // stage-1 matrix hi/lo
    float* tc_cs = nullptr;   // stage-2 C / S matrices hi/lo
    float2* tc_tw = nullptr;  // a e^{-2 pi i n2 k1 / 1024}
    float2* tc_w32 = nullptr; // e^{-2 pi i j / 32}
    // adjoint (kapre_stft_backward): the inverse plan with dual window w * n_fft / 2, made on first use
    std::vector<float> window_host;
    std::mutex adj_mu;
    kapre_istft_plan* adj = nullptr;
};

// (K = 32 rows, N = 32 columns) matrix -> the K-major (8 kchunk, 32 col, 4) layout of the wgmma B operand, TF32 hi / lo
static void kb_tc_pack_b(const double* M, float* hi, float* lo) {
    for (int kc = 0; kc < 8; ++kc)
        for (int c = 0; c < 32; ++c)
            for (int e = 0; e < 4; ++e) {
                const float w = (float)M[(4 * kc + e) * 32 + c], h = kb_tf32_rn(w);
                hi[(kc * 32 + c) * 4 + e] = h;
                lo[(kc * 32 + c) * 4 + e] = w - h;
            }
}

static void kb_tc_tables(kapre_stft_plan* p, KbTableUpload& tb) {
    std::vector<double> M(1024);
    std::vector<float> f1(2048), cs(4096);
    for (int n1 = 0; n1 < 32; ++n1)
        for (int c = 0; c < 32; ++c) {
            const int k1 = c >> 1;
            const double a = -2.0 * M_PI * (double)((n1 * k1) % 32) / 32.0;
            M[n1 * 32 + c] = (c == 1) ? ((n1 & 1) ? -1.0 : 1.0) : ((c & 1) ? sin(a) : cos(a));
        }
    kb_tc_pack_b(M.data(), f1.data(), f1.data() + 1024);
    for (int n2 = 0; n2 < 32; ++n2)
        for (int k2 = 0; k2 < 32; ++k2) M[n2 * 32 + k2] = cos(2.0 * M_PI * (double)((n2 * k2) % 32) / 32.0);
    kb_tc_pack_b(M.data(), cs.data(), cs.data() + 1024);
    for (int n2 = 0; n2 < 32; ++n2)
        for (int k2 = 0; k2 < 32; ++k2) M[n2 * 32 + k2] = sin(2.0 * M_PI * (double)((n2 * k2) % 32) / 32.0);
    kb_tc_pack_b(M.data(), cs.data() + 2048, cs.data() + 3072);
    std::vector<float2> tw(18 * 32), w32(16);
    for (int k1 = 0; k1 < 18; ++k1)
        for (int n2 = 0; n2 < 32; ++n2) {
            const double a = -2.0 * M_PI * (double)(n2 * k1) / 1024.0;
            tw[k1 * 32 + n2] = make_float2((float)(p->win_a * cos(a)), (float)(p->win_a * sin(a)));
        }
    for (int j = 0; j < 16; ++j) {
        const double a = -2.0 * M_PI * (double)j / 32.0;
        w32[j] = make_float2((float)cos(a), (float)sin(a));
    }
    tb.add(f1, &p->tc_f1); tb.add(cs, &p->tc_cs); tb.add(tw, &p->tc_tw); tb.add(w32, &p->tc_w32);
}

struct kapre_istft_plan {
    int n_fft, win_length, hop, Q, win;
    DevInfo dev;
    KbTables tables;
    float* dual = nullptr;    // fused path (kb_make_dual)
    float2* twp = nullptr;
    float2* twn = nullptr;
    float* dualn = nullptr;   // generic path: dual / n_fft
    float2* tw = nullptr;     // generic path: exp(+2 pi i r / n_fft)
    // adjoint (kapre_istft_backward): the forward plan with window dual * 2 / n_fft, made on first use
    std::vector<float> dual_host;
    std::mutex adj_mu;
    kapre_stft_plan* adj = nullptr;
};

struct kapre_filterbank {
    int n_freq, n_bands, n_w;
    DevInfo dev;
    KbTables tables;
    KbBand* bands = nullptr;   // band-major form (stand-alone ApplyFilterbank kernel)
    float* w = nullptr;
    int Q = 0;                 // chunk-list form for the fused kernel (n_freq == 32*Q + 1), else 0
    int n_chunks = 0;
    kb_f4* cw = nullptr;
    kb_i2* cm = nullptr;
    int* cg = nullptr;
    int n_bd = 0;              // band descriptors of the two-level walk (kb_make_fb_band_desc)
    kb_i2* bd = nullptr;
    int* bg = nullptr;
    int n_msteps = 0;          // tensor-core form (kb_make_fb_mma) for the fused kernel
    kb_f4* mw = nullptr;
    kb_i2* ms = nullptr;
    int* mg = nullptr;
};

static float2* g_tc_dbg = nullptr;   // experimental: complex-spectrum dump of the next tensor-core launch (kapre_tc_set_debug)

static int kb_env_int(const char* name, int dflt) {
    const char* v = getenv(name);
    return (v && *v) ? atoi(v) : dflt;
}

// ------------------------------------------------------------------------------------------
// launch configuration of the fused forward kernel
// ------------------------------------------------------------------------------------------
struct FwdCfg { int TF, NW, smem, bps; };
#ifndef KB_PAIRED_DEFAULT
#define KB_PAIRED_DEFAULT 1
#endif
#ifndef KB_FBMMA_DEFAULT
#define KB_FBMMA_DEFAULT 0
#endif
#ifndef KB_TC_DEFAULT
#define KB_TC_DEFAULT 0
#endif
// Tile shape of the fused forward kernel.  The kernel is
// latency-bound, so resident warps per SM (up to the 16 the 128-register kernel allows) matter
// most, then larger tiles (less re-staging of the hop overlap).  Filterbank modes keep the
// tile's magnitudes in the warps' exchange regions, which needs TF == frames per round.
// `n_sig` signals of `T` frames each: small batches (BASELINE cfg1 is 244 frames) that cannot fill the machine are
// latency-bound and get their own choice (see below); everything else maximises resident warps.
static bool kb_pick_fwd_cfg(const DevInfo& dev, int Q, int n_fft, int hop, int mode, int n_bands, int n_chunks,
                            int fbmma, long long n_sig, int T, FwdCfg* out) {
    const int FPW = 32 / Q;
    const bool fb = (mode == KB_OUT_FB || mode == KB_OUT_FB_DB);
    const int force_tf = kb_env_int("KAPRE_B200_TF", 0);
    const int force_nw = kb_env_int("KAPRE_B200_NW", 0);
    const int sm_smem = 228 * 1024;
    bool found = false;
    FwdCfg best{};
    double best_score = -1.0;
    const int nws[5] = {1, 2, 4, 8, 16};
    for (int a = 0; a < 5; ++a) {
        const int NW = nws[a];
        if (force_nw && NW != force_nw) continue;
        if (NW == 16 && !(Q == 32 && fb && !fbmma)) continue;      // only kb_stft_kernel_w16's instantiations
        const int FR = NW * FPW;
        if (FR > 32) continue;
        for (int TF = 32; TF >= 1; TF >>= 1) {
            if (fb ? (TF != FR) : (TF % FR != 0)) continue;
            if (!fb && force_tf && TF != force_tf) continue;
            const KbStftSmem L = kb_stft_smem_layout(Q, n_fft, hop, TF, NW, mode, n_bands, n_chunks, fbmma);
            if (L.total > dev.smem_optin) continue;
            int bps = sm_smem / (L.total + 1024);
            if (bps > 16 / NW) bps = 16 / NW;                 // 128 registers per thread: 16 warps per SM
            if (bps < 1) continue;
            const int warps = bps * NW;
            // throughput score (large problems): resident warps first, then longer tiles (less re-staging of the overlap)
            double score = (double)warps * 1000.0 + TF * 10.0 + NW;
            if (n_sig > 0 && T > 0) {
                const double tiles = (double)n_sig * (double)((T + TF - 1) / TF);
                const double slots = (double)dev.sm_count * bps;
                if (tiles < slots) {
                    // latency regime: all tiles run at once and the call costs one tile (table prologue, one FFT round,
                    // filterbank, copy-out): prefer 4-warp CTAs, then one round per tile, then more tiles.  (Preference carried
                    // over from measurements on the previous GPU target; not yet re-measured on H100.)
                    const double rounds = (double)((TF + FR - 1) / FR);
                    score = 1.0e6 - (NW == 4 ? 0.0 : 500.0) - rounds * 200.0 - (double)TF;
                } else {
                    score += 2.0e6;                               // any shape that fills the machine beats one that does not
                }
            }
            if (score > best_score) {
                best_score = score;
                best = FwdCfg{TF, NW, L.total, bps};
                found = true;
            }
        }
    }
    *out = best;
    return found;
}

// The fused forward kernels start with griddepcontrol.wait (kb_stft_cta), so they are launched with programmatic
// dependent launch: their table prologue overlaps the tail of the previous kernel in the stream (the clamp of the
// previous call).
template <int Q, int MODE>
static int kb_launch_stft_qm(const KbStftParams& p, int grid, int smem, cudaStream_t st) {
    constexpr bool FB = MODE == KB_OUT_FB || MODE == KB_OUT_FB_DB;
    void (*kernel)(KbStftParams) = kb_stft_kernel<Q, MODE>;
    if (p.n_warps > KB_MAX_WARPS) {
        if constexpr (Q == 32 && FB) kernel = kb_stft_kernel_w16<Q, MODE>;
        else return kb_fail(KAPRE_E_UNSUPPORTED, "no 16-warp instantiation for Q=%d mode=%d", Q, MODE);
    } else if (Q == 16 && (p.variant & 2)) {
        // the other form of the pair step (KAPRE_B200_PAIRED=0): the A/B alternative, n_fft 1024 only
        kernel = kb_stft_kernel_v<16, MODE, 2>;
    } else if constexpr (FB) {
        if (p.fb_mma) kernel = kb_stft_kernel_mma<Q, MODE>;
    }
    return kb_launch(kernel, {.grid = grid, .block = p.n_warps * 32, .smem = smem, .st = st,
                              .pdl = kb_env_int("KAPRE_B200_PDL_FWD", 1) != 0, .timed = true}, p);
}

template <int Q>
static int kb_launch_stft(const KbStftParams& p, int grid, int smem, cudaStream_t st) {
    switch (p.mode) {
        case KB_OUT_COMPLEX: return kb_launch_stft_qm<Q, KB_OUT_COMPLEX>(p, grid, smem, st);
        case KB_OUT_MAG: return kb_launch_stft_qm<Q, KB_OUT_MAG>(p, grid, smem, st);
        case KB_OUT_MAG_DB: return kb_launch_stft_qm<Q, KB_OUT_MAG_DB>(p, grid, smem, st);
        case KB_OUT_FB: return kb_launch_stft_qm<Q, KB_OUT_FB>(p, grid, smem, st);
        case KB_OUT_FB_DB: return kb_launch_stft_qm<Q, KB_OUT_FB_DB>(p, grid, smem, st);
        case KB_OUT_MAG_PHASE: return kb_launch_stft_qm<Q, KB_OUT_MAG_PHASE>(p, grid, smem, st);
    }
    return kb_fail(KAPRE_E_INVALID, "bad mode");
}

template <int Q>
__global__ void __launch_bounds__(KB_ISTFT_MAX_WARPS * 32, 4) kb_istft2_kernel(const __grid_constant__ KbIstftParams p) {
    extern __shared__ __align__(128) char kb_smem[];
    kb_istft2_cta<Q>(p, kb_smem, (int)blockIdx.x, (int)gridDim.x);
}


// Tile shape of the multi-channel kernel: TF time frames x C channels = columns, FR = NW * FPW of
// them per round.  Prefer many resident warps, full rounds, two CTAs per SM (their barriers
// overlap), then longer tiles (less re-staging of the frame overlap).
static bool kb_pick_mc_cfg(const DevInfo& dev, int Q, int n_fft, int hop, int C, int with_wh, FwdCfg* out) {
    const int FPW = 32 / Q;
    const int sm_smem = 228 * 1024;
    const int force_tf = kb_env_int("KAPRE_B200_MC_TF", 0);
    const int force_nw = kb_env_int("KAPRE_B200_MC_NW", 0);
    bool found = false;
    FwdCfg best{};
    double best_score = -1.0;
    for (int NW = 1; NW <= 16; ++NW) {
        if (force_nw && NW != force_nw) continue;
        const int FR = NW * FPW;
        if (FR > 32) continue;
        for (int TF = 1; TF <= 32; ++TF) {
            if (force_tf && TF != force_tf) continue;
            const int ncol = TF * C;
            const int rounds = (ncol + FR - 1) / FR;
            if (rounds > 8) break;
            const KbStftMcSmem L = kb_stft_mc_smem_layout(Q, n_fft, hop, TF, C, NW, with_wh);
            if (L.total > dev.smem_optin) break;
            if (NW * 32 < C) continue;                                // the loader gives every channel >= 1 thread
            int bps = sm_smem / (L.total + 1024);
            if (bps > 16 / NW) bps = 16 / NW;                         // 128 registers per thread
            if (bps < 1) continue;
            int warps = bps * NW;
            const double eff = (double)ncol / (double)(rounds * FR);
            const double score = warps * eff * 1000.0 + (bps >= 2 ? 400.0 : 0.0) + TF * 5.0 - rounds * 20.0;
            if (score > best_score) {
                best_score = score;
                best = FwdCfg{TF, NW, L.total, bps};
                found = true;
            }
        }
    }
    *out = best;
    return found;
}

// Filterbank modes on all-channel tiles: one round per tile, TF = floor(NW * FPW / C) time frames.
static bool kb_pick_mcfb_cfg(const DevInfo& dev, int Q, int n_fft, int hop, int C, int with_wh, int n_bands,
                             int n_chunks, FwdCfg* out) {
    const int FPW = 32 / Q;
    const int sm_smem = 228 * 1024;
    bool found = false;
    FwdCfg best{};
    double best_score = -1.0;
    const int nws[3] = {2, 4, 8};
    for (int a = 0; a < 3; ++a) {
        const int NW = nws[a];
        const int FR = NW * FPW;
        if (FR > 32 || FR < C || NW * 32 < C) continue;
        const int TF = FR / C;
        const KbStftMcFbSmem L = kb_stft_mcfb_smem_layout(Q, n_fft, hop, TF, C, NW, with_wh, n_bands, n_chunks);
        if (L.total > dev.smem_optin) continue;
        int bps = sm_smem / (L.total + 1024);
        if (bps > 16 / NW) bps = 16 / NW;
        if (bps < 1) continue;
        const double eff = (double)(TF * C) / (double)FR;
        const double score = bps * NW * eff * 1000.0 + TF * 10.0 + NW;
        if (score > best_score) { best_score = score; best = FwdCfg{TF, NW, L.total, bps}; found = true; }
    }
    *out = best;
    return found;
}

template <int Q>
static int kb_launch_stft_mcfb(const KbStftParams& p, int grid, int smem, cudaStream_t st) {
    void (*kernel)(KbStftParams);
    if (p.mode == KB_OUT_FB) kernel = kb_stft_mcfb_kernel<Q, KB_OUT_FB>;
    else if (p.mode == KB_OUT_FB_DB) kernel = kb_stft_mcfb_kernel<Q, KB_OUT_FB_DB>;
    else return kb_fail(KAPRE_E_INVALID, "bad mode for the multi-channel filterbank kernel");
    return kb_launch(kernel, {.grid = grid, .block = p.n_warps * 32, .smem = smem, .st = st, .timed = true}, p);
}

template <int Q>
static int kb_launch_stft_mc(const KbStftParams& p, int grid, int smem, cudaStream_t st) {
    void (*kernel)(KbStftParams);
    switch (p.mode) {
        case KB_OUT_COMPLEX: kernel = kb_stft_mc_kernel<Q, KB_OUT_COMPLEX>; break;
        case KB_OUT_MAG: kernel = kb_stft_mc_kernel<Q, KB_OUT_MAG>; break;
        case KB_OUT_MAG_DB: kernel = kb_stft_mc_kernel<Q, KB_OUT_MAG_DB>; break;
        case KB_OUT_MAG_PHASE: kernel = kb_stft_mc_kernel<Q, KB_OUT_MAG_PHASE>; break;
        default: return kb_fail(KAPRE_E_INVALID, "bad mode for the multi-channel kernel");
    }
    return kb_launch(kernel, {.grid = grid, .block = p.n_warps * 32, .smem = smem, .st = st, .timed = true}, p);
}

static int kb_check_device(const DevInfo& d) {
    int cur = -1;
    KB_CUDA(cudaGetDevice(&cur));
    if (cur != d.device)
        return kb_fail(KAPRE_E_INVALID, "plan was created on device %d but device %d is current", d.device, cur);
    return 0;
}

static int kb_launch_clamp(float* y, long long n_items, long long item_size, unsigned int* item_max,
                           float amin, float db_mul, float db_sub, float dr, cudaStream_t st,
                           long long run = 1, long long period = 1) {
    if (n_items <= 0 || item_size <= 0) return 0;
    // one CTA per 32 Ki elements of an item (at most 64): a binding clamp on a long item is rewritten in parallel
    long long chunks = (item_size + 32767) / 32768;
    if (chunks > 64) chunks = 64;
    if (chunks < 1) chunks = 1;
    if (n_items * chunks > 0x7fffffffLL) return kb_fail(KAPRE_E_UNSUPPORTED, "too many items for the clamp kernel");
    return kb_launch(kb_db_clamp_kernel, {.grid = (int)(n_items * chunks), .block = 256, .st = st,
                                          .pdl = kb_env_int("KAPRE_B200_PDL", 1) != 0},
                     y, item_size, run, period, item_max, (unsigned int)n_items, (int)chunks, amin, db_mul, db_sub, dr);
}

static void kb_db_consts(const kapre_db_cfg* db, float* db_mul, float* db_sub) {
    // 10*log10(v) = (10*log10(2)) * log2(v);  kapre/backend.py:187-188
    *db_mul = (float)(10.0 * log10(2.0));
    const double m = db->amin > db->ref_value ? db->amin : db->ref_value;
    *db_sub = (float)(10.0 * log10(m));
}

static int kb_check_db(const kapre_db_cfg* db) {
    if (!db) return kb_fail(KAPRE_E_INVALID, "decibel configuration required");
    // kapre/backend.py:168-173
    if (!(db->ref_value > 0)) return kb_fail(KAPRE_E_INVALID, "ref_value must be positive, got: %g", db->ref_value);
    if (!(db->amin > 0)) return kb_fail(KAPRE_E_INVALID, "amin must be positive, got: %g", db->amin);
    if (!(db->dynamic_range > 0)) return kb_fail(KAPRE_E_INVALID, "dynamic_range must be positive, got: %g", db->dynamic_range);
    return 0;
}

// ------------------------------------------------------------------------------------------
// C ABI
// ------------------------------------------------------------------------------------------
extern "C" {

const char* kapre_last_error(void) { return g_err.c_str(); }
int kapre_version(void) { return KAPRE_B200_VERSION; }
uint64_t kapre_launch_count(void) { return g_launches.load(); }
const char* kapre_last_launch_info(void) { return g_launch_info.c_str(); }

int kapre_profile_enable(int enable) {
    std::lock_guard<std::mutex> lk(g_prof_mu);
    g_prof_on = enable > 0 ? enable : 0;
    g_prof_seq = 0;
    return 0;
}

int kapre_profile_read(double* total_ms, uint64_t* launches) {
    std::vector<std::pair<cudaEvent_t, cudaEvent_t>> evs;
    {
        std::lock_guard<std::mutex> lk(g_prof_mu);
        evs.swap(g_prof_events);
    }
    double tot = 0.0;
    uint64_t n = 0;
    for (auto& pr : evs) {
        float ms = 0.0f;
        if (cudaEventSynchronize(pr.second) == cudaSuccess && cudaEventElapsedTime(&ms, pr.first, pr.second) == cudaSuccess) {
            tot += ms;
            ++n;
        }
        cudaEventDestroy(pr.first);
        cudaEventDestroy(pr.second);
    }
    if (total_ms) *total_ms = tot;
    if (launches) *launches = n;
    return 0;
}

int kapre_stft_plan_create(int n_fft, int win_length, int hop_length, const float* window_host,
                           kapre_stft_plan** out) {
    if (!out || !window_host) return kb_fail(KAPRE_E_INVALID, "null argument");
    if (n_fft < 2 || win_length < 1 || hop_length < 1)
        return kb_fail(KAPRE_E_INVALID, "n_fft=%d win_length=%d hop_length=%d out of range", n_fft, win_length, hop_length);
    if (n_fft > 16384) return kb_fail(KAPRE_E_UNSUPPORTED, "n_fft=%d > 16384 is not supported", n_fft);
    kapre_stft_plan* p = new kapre_stft_plan();
    p->n_fft = n_fft; p->win_length = win_length; p->hop = hop_length;
    p->Q = kb_q_for_nfft(n_fft);
    p->win_eff = win_length < n_fft ? win_length : n_fft;
    p->window_host.assign(window_host, window_host + win_length);
    int rc = kb_dev_info(&p->dev);
    if (rc) { delete p; return rc; }
    KbTableUpload tb;
    if (p->Q) {
        std::vector<float> wh; std::vector<float2> twp, twn, twn2;
        double ca = 0.0, cb = 0.0;
        if (kb_fit_cosine_window(window_host, win_length, n_fft, &ca, &cb) && kb_env_int("KAPRE_B200_NOCOSW", 0) == 0) {
            std::vector<kb_f4> cwq;
            kb_make_cwq(p->Q, n_fft, cb, cwq);
            tb.add(cwq, &p->cwq);
            p->cosw = 1;
            p->cw_a0 = (float)(0.5 * ca);
            kb_make_wh_cosw(p->Q, p->cw_a0, cwq, wh);   // the table frames read when not windowed in registers
        } else {
            kb_make_wh(window_host, win_length, n_fft, wh);
        }
        kb_make_twp(p->Q, twp);
        kb_make_twn(n_fft, twn);
        kb_make_twn2(n_fft, twn2);
        tb.add(wh, &p->wh); tb.add(twp, &p->twp); tb.add(twn, &p->twn); tb.add(twn2, &p->twn2);
        if (n_fft == 1024 && win_length == 1024 && kb_fit_cosine_window(window_host, win_length, n_fft, &ca, &cb) && ca > 0.0) {
            p->win_a = ca; p->win_b = cb;
            kb_tc_tables(p, tb);
        }
    }
    {   // generic tables are always built: they also serve sizes the fused kernel cannot take
        std::vector<float> w(window_host, window_host + p->win_eff);
        std::vector<float2> tw(n_fft);
        for (int r = 0; r < n_fft; ++r) {
            const double a = -2.0 * M_PI * (double)r / (double)n_fft;
            tw[r] = make_float2((float)cos(a), (float)sin(a));
        }
        tb.add(w, &p->w); tb.add(tw, &p->tw);
    }
    if ((rc = tb.upload(p->tables, "stft"))) { delete p; return rc; }
    *out = p;
    return 0;
}

void kapre_stft_plan_destroy(kapre_stft_plan* p) {
    if (!p) return;
    kapre_istft_plan_destroy(p->adj);
    delete p;
}

int kapre_stft_num_frames(const kapre_stft_plan* p, int length, int pad_begin, int pad_end) {
    if (!p || length < 0) return kb_fail(KAPRE_E_INVALID, "bad argument");
    const long long Lp = (long long)length + (pad_begin ? (p->n_fft - p->hop) : 0);
    if (pad_end) return (int)((Lp + p->hop - 1) / p->hop);
    if (Lp < p->win_length) return 0;
    return (int)(1 + (Lp - p->win_length) / p->hop);
}

int kapre_stft_supports_mode(const kapre_stft_plan* p, int mode) {
    if (!p) return 0;
    if (mode < KAPRE_OUT_COMPLEX || mode > KAPRE_OUT_MAG_PHASE) return 0;
    if (p->Q) return 1;
    if (mode == KAPRE_OUT_COMPLEX || mode == KAPRE_OUT_MAG) return 1;
    if (mode == KAPRE_OUT_MAG_PHASE) return 0;
    // fused filterbank / decibel tail of the mixed-radix kernel: 5-smooth transform length whose buffers fit
    int radix[KB_MR_MAX_PASS];
    const int P = (p->n_fft & 1) ? p->n_fft : p->n_fft / 2;
    if (kb_mr_factor(P, radix) < 0 || kb_env_int("KAPRE_B200_NOMR", 0)) return 0;
    int nw, g, b;
    if (mode == KAPRE_OUT_MAG_DB) return kb_mr_pick(P, p->dev.smem_optin, 228 * 1024, 32, &nw, &g, &b) > 0 ? 1 : 0;
    // 128 bands as the sizing assumption for the filterbank tile (the launch re-picks with the real count and fails loudly)
    return kb_mr_pick(P, p->dev.smem_optin, 228 * 1024, 32, &nw, &g, &b, p->n_fft / 2 + 1, 128, 8) > 0 ? 1 : 0;
}

int kapre_stft_forward(const kapre_stft_plan* plan, const float* x_dev, const kapre_wave_desc* xd,
                       int pad_begin, int pad_end, int mode, void* out_dev, const kapre_spec_desc* od,
                       const kapre_filterbank* fb, const kapre_db_cfg* db, void* workspace_dev, void* stream) {
    if (!plan || !xd || !od) return kb_fail(KAPRE_E_INVALID, "null argument");
    if (mode < KAPRE_OUT_COMPLEX || mode > KAPRE_OUT_MAG_PHASE) return kb_fail(KAPRE_E_INVALID, "bad mode %d", mode);
    int rc = kb_check_device(plan->dev);
    if (rc) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    const int B = xd->batch, C = xd->channels, Ln = xd->length;
    if (B < 0 || C < 0 || Ln < 0) return kb_fail(KAPRE_E_INVALID, "negative size");
    if (pad_begin && plan->hop > plan->n_fft)
        return kb_fail(KAPRE_E_INVALID, "pad_begin needs hop_length <= n_fft (the padding is n_fft - hop_length = %d)",
                       plan->n_fft - plan->hop);
    const int T = kapre_stft_num_frames(plan, Ln, pad_begin, pad_end);
    if (B == 0 || C == 0 || T <= 0) return 0;
    if (!x_dev || !out_dev) return kb_fail(KAPRE_E_INVALID, "null data pointer");
    if ((long long)T * plan->hop + plan->n_fft > 0x7fffffffLL)
        return kb_fail(KAPRE_E_UNSUPPORTED, "signal too long");
    const bool fbmode = (mode == KAPRE_OUT_FB || mode == KAPRE_OUT_FB_DB);
    const bool dbmode = (mode == KAPRE_OUT_MAG_DB || mode == KAPRE_OUT_FB_DB || (mode == KAPRE_OUT_MAG_PHASE && db != nullptr));
    if (fbmode) {
        if (!fb) return kb_fail(KAPRE_E_INVALID, "filterbank required for mode %d", mode);
        if (fb->n_freq != plan->n_fft / 2 + 1)
            return kb_fail(KAPRE_E_INVALID, "filterbank has %d rows but n_fft/2+1 = %d", fb->n_freq, plan->n_fft / 2 + 1);
        if (fb->dev.device != plan->dev.device) return kb_fail(KAPRE_E_INVALID, "filterbank lives on another device");
        if (plan->Q && fb->Q != plan->Q) return kb_fail(KAPRE_E_INVALID, "filterbank was not prepared for n_fft=%d", plan->n_fft);
    }
    float db_mul = 0, db_sub = 0;
    long long db_item_size = 0, db_run = 1, db_period = 1;
    if (dbmode) {
        if ((rc = kb_check_db(db))) return rc;
        if (!workspace_dev) return kb_fail(KAPRE_E_INVALID, "workspace required for decibel modes");
        kb_db_consts(db, &db_mul, &db_sub);
        // Output layout of the clamp pass, checked BEFORE anything is launched (a late failure would leave
        // per-item maxima in the self-cleaning workspace).  Items are contiguous blocks of stride_b elements
        // in both data formats.
        const long long K = fbmode ? fb->n_bands : (plan->n_fft / 2 + 1);
        const long long chans = (mode == KAPRE_OUT_MAG_PHASE) ? 2LL * C : C;
        db_item_size = chans * T * K;
        if (od->stride_b != db_item_size)
            return kb_fail(KAPRE_E_UNSUPPORTED, "decibel modes need a batch-contiguous output (stride_b=%lld, item=%lld)",
                           (long long)od->stride_b, db_item_size);
        if (mode == KAPRE_OUT_MAG_PHASE) {   // clamp only the magnitude channels [0, C) of the 2C-channel item
            if (od->stride_c == 1 && od->stride_f == chans && od->stride_t == K * chans) { db_run = C; db_period = chans; }
            else if (od->stride_f == 1 && od->stride_t == K && od->stride_c == (long long)T * K) { db_run = (long long)C * T * K; db_period = db_item_size; }
            else return kb_fail(KAPRE_E_UNSUPPORTED, "mag+phase decibel output must be a contiguous channels_first or channels_last tensor");
        }
    }
    const int pad_left = pad_begin ? (plan->n_fft - plan->hop) : 0;

    if (!plan->Q) {
        if (mode == KAPRE_OUT_MAG_PHASE)
            return kb_fail(KAPRE_E_UNSUPPORTED, "n_fft=%d has no fused magnitude+phase path; chain the stand-alone ops", plan->n_fft);
        KbDftParams p{};
        p.x = x_dev; p.x_sb = xd->stride_b; p.x_sc = xd->stride_c; p.x_sl = xd->stride_l;
        p.B = B; p.C = C; p.L = Ln; p.n_fft = plan->n_fft; p.hop = plan->hop; p.T = T; p.pad_left = pad_left;
        p.win_eff = plan->win_eff; p.w = plan->w; p.tw = plan->tw;
        p.out = out_dev; p.o_sb = od->stride_b; p.o_sc = od->stride_c; p.o_st = od->stride_t; p.o_sk = od->stride_f;
        p.mode = mode; p.n_tiles_t = (T + KB_DFT_TF - 1) / KB_DFT_TF; p.n_warps = 8;
        {   // mixed-radix Stockham FFT when n_fft/2 (even) or n_fft (odd) is 5-smooth and the buffers fit
            KbMrParams q{};
            q.half = (plan->n_fft & 1) ? 0 : 1;
            q.P = q.half ? plan->n_fft / 2 : plan->n_fft;
            q.n_pass = kb_mr_factor(q.P, q.radix);
            int NW = 8, G = 1, bps = 1, FRT = 0, fit = 0;
            const int want = kb_env_int("KAPRE_B200_MR_WARPS", 32);
            const int F = plan->n_fft / 2 + 1, nb = fbmode ? fb->n_bands : 0;
            if (q.n_pass >= 0 && kb_env_int("KAPRE_B200_NOMR", 0) == 0) {
                if (!fbmode) fit = kb_mr_pick(q.P, plan->dev.smem_optin, 228 * 1024, want, &NW, &G, &bps);
                else {
                    // filterbank tile of 32 frames unless a smaller one keeps clearly more warps resident
                    for (int frt = 32; frt >= 8; frt >>= 1) {
                        int nw = 8, g = 1, b2 = 1;
                        const int f2 = kb_mr_pick(q.P, plan->dev.smem_optin, 228 * 1024, want, &nw, &g, &b2, F, nb, frt);
                        if (f2 > fit + fit / 2) { fit = f2; NW = nw; G = g; bps = b2; FRT = frt; }
                    }
                }
            }
            if (fit > 0) {
                const int smem = kb_mr_smem_layout(q.P, NW / G, F, nb, FRT).total;
                q.d = p; q.d.n_warps = NW;
                q.G = G;
                q.pad1 = (q.n_pass > 0 && q.radix[0] % 2 == 0) ? 1 : 0;
                q.FRT = FRT;
                if (fbmode) { q.bands = fb->bands; q.fbw = fb->w; q.n_bands = fb->n_bands; }
                kb_mr_finish(q);
                // frames per group and tile: 16 amortises the per-tile bookkeeping (two divisions, 64-bit bases) unless the
                // batch is small -- keep at least ~8 tiles per resident CTA for the tail
                int fpg = 16;
                while (fpg > 4 && (long long)B * C * ((T + fpg * (NW / G) - 1) / (fpg * (NW / G))) < 8LL * plan->dev.sm_count * bps)
                    fpg >>= 1;
                q.TF = FRT > 0 ? FRT : fpg * (NW / G);
                if (dbmode) {
                    q.amin = db->amin; q.db_mul = db_mul; q.db_sub = db_sub; q.item_max = (unsigned int*)workspace_dev;
                    q.db_ftz = (db->amin >= 1.17549435e-38f) ? 1 : 0;
                }
                const long long tiles = (long long)B * C * ((T + q.TF - 1) / q.TF);
                const long long gmax = (long long)plan->dev.sm_count * bps;
                const int grid = (int)(tiles < gmax ? tiles : gmax);
                if ((rc = kb_launch(kb_mr_kernel, {.grid = grid, .block = NW * 32, .smem = smem, .st = st, .timed = true}, q)))
                    return rc;
                char buf[160];
                snprintf(buf, sizeof(buf), "MR P%d passes%d NW%d G%d grid%d smem%d bps%d frt%d", q.P, q.n_pass, NW, G, grid, smem, bps, FRT);
                g_launch_info = buf;
                if (dbmode)
                    rc = kb_launch_clamp((float*)out_dev, B, db_item_size, (unsigned int*)workspace_dev, db->amin, db_mul, db_sub,
                                         db->dynamic_range, st, db_run, db_period);
                return rc;
            }
        }
        if (!(mode == KAPRE_OUT_COMPLEX || mode == KAPRE_OUT_MAG))
            return kb_fail(KAPRE_E_UNSUPPORTED, "n_fft=%d (prime factor above 5) has no fused filterbank/decibel path; chain the stand-alone ops", plan->n_fft);
        const KbDftSmem L = kb_dft_smem_layout(plan->n_fft, plan->win_eff);
        if (L.total > plan->dev.smem_optin) return kb_fail(KAPRE_E_UNSUPPORTED, "n_fft=%d has a prime factor above 5 and is too large for the direct-DFT kernel (%d B of shared memory needed)", plan->n_fft, L.total);
        long long tiles = (long long)B * C * p.n_tiles_t;
        int grid = (int)(tiles < plan->dev.sm_count * 4LL ? tiles : plan->dev.sm_count * 4LL);
        if ((rc = kb_launch(kb_dft_kernel, {.grid = grid, .block = 256, .smem = L.total, .st = st}, p))) return rc;
        {
            char buf[96];
            snprintf(buf, sizeof(buf), "DFT n_fft%d grid%d smem%d (direct O(N^2): prime factor > 5)", plan->n_fft, grid, L.total);
            g_launch_info = buf;
        }
        return 0;
    }

    // address range of the waveform tensor (non-negative strides): the rounded bulk copies stay inside
    const long long max_off = (long long)(B - 1) * xd->stride_b + (long long)(C - 1) * xd->stride_c +
                              (long long)(Ln - 1) * xd->stride_l;
    const bool bulk = (xd->stride_l == 1) && (((uintptr_t)x_dev & 3) == 0) && xd->stride_b >= 0 && xd->stride_c >= 0 &&
                      kb_env_int("KAPRE_B200_NOBULK", 0) == 0;
    // ---- tensor-core FFT path (tc_mel.cuh): n_fft = win_length = 1024, cosine-sum window, hop 128 / 256, planar signals ----
    if (fbmode && plan->tc_f1 && (plan->hop == 256 || plan->hop == 128) && xd->stride_l == 1 && fb->n_bands <= 128 &&
        fb->cw && kb_env_int("KAPRE_B200_TC", KB_TC_DEFAULT)) {
        const KbTcMelSmem TL = kb_tcm_smem_layout(fb->n_chunks);
        if (TL.total <= plan->dev.smem_optin) {
            KbTcMelParams q{};
            q.x = x_dev; q.x_sb = xd->stride_b; q.x_sc = xd->stride_c;
            q.B = B; q.C = C; q.L = Ln; q.T = T; q.hop = plan->hop; q.pad_left = pad_left;
            q.wc = (float)(plan->win_b / (2.0 * plan->win_a));
            q.f1 = plan->tc_f1; q.cs = plan->tc_cs; q.tw = plan->tc_tw; q.w32 = plan->tc_w32;
            q.cw = fb->cw; q.cm = fb->cm; q.cg = fb->cg; q.n_chunks = fb->n_chunks; q.n_bands = fb->n_bands;
            q.out = (float*)out_dev; q.o_sb = od->stride_b; q.o_sc = od->stride_c; q.o_st = od->stride_t; q.o_sk = od->stride_f;
            q.db = dbmode ? 1 : 0;
            if (dbmode) { q.amin = db->amin; q.db_mul = db_mul; q.db_sub = db_sub; q.item_max = (unsigned int*)workspace_dev; }
            q.dbg = g_tc_dbg; g_tc_dbg = nullptr;
            q.n_tiles_t = (T + TCM_TF - 1) / TCM_TF;
            const long long tiles = (long long)B * C * q.n_tiles_t;
            if (tiles > 0x7fffffffLL) return kb_fail(KAPRE_E_UNSUPPORTED, "too many tiles");
            const int grid = (int)(tiles < plan->dev.sm_count ? tiles : plan->dev.sm_count);
            if ((rc = kb_launch(kb_tc_mel_kernel, {.grid = grid, .block = TCM_THREADS, .smem = TL.total, .st = st,
                                                   .pdl = kb_env_int("KAPRE_B200_PDL_FWD", 1) != 0, .timed = true}, q)))
                return rc;
            char buf[160];
            snprintf(buf, sizeof(buf), "TC wgmma n_fft1024 hop%d grid%d smem%d tiles%lld", plan->hop, grid, TL.total, tiles);
            g_launch_info = buf;
            if (dbmode)
                rc = kb_launch_clamp((float*)out_dev, B, db_item_size, (unsigned int*)workspace_dev, db->amin, db_mul, db_sub,
                                     db->dynamic_range, st, db_run, db_period);
            return rc;
        }
    }
    FwdCfg cfg;
    // filterbank phase on the tensor pipe (mma.sync 3xTF32) or on the CUDA cores (chunk lists)
    const int fbmma = (fbmode && fb->mw && kb_env_int("KAPRE_B200_FBMMA", KB_FBMMA_DEFAULT)) ? 1 : 0;
    // Pair step of the register kernel: kb_stft_cta picks the paired-column or the natural-order form per (n_fft, mode)
    // (choice carried over from the previous GPU target, not yet re-measured on H100);
    // KAPRE_B200_PAIRED=0 runs the other form (variant bit 1,
    // instantiated for n_fft 1024 only: the A/B alternative).
    const int variant = (!fbmma && plan->Q == 16 && kb_env_int("KAPRE_B200_PAIRED", KB_PAIRED_DEFAULT) == 0) ? 2 : 0;
    if (!kb_pick_fwd_cfg(plan->dev, plan->Q, plan->n_fft, plan->hop, mode, fbmode ? fb->n_bands : 0,
                         fbmode ? (fbmma ? fb->n_msteps : fb->n_chunks) : 0, fbmma, (long long)B * C, T, &cfg))
        return kb_fail(KAPRE_E_UNSUPPORTED, "no launch configuration fits shared memory (n_fft=%d hop=%d bands=%d)",
                       plan->n_fft, plan->hop, fbmode ? fb->n_bands : 0);
    KbStftParams p{};
    p.x = x_dev; p.x_sb = xd->stride_b; p.x_sc = xd->stride_c; p.x_sl = xd->stride_l;
    p.B = B; p.C = C; p.L = Ln; p.n_fft = plan->n_fft; p.hop = plan->hop; p.T = T; p.pad_left = pad_left;
    p.x_lo = x_dev; p.x_hi = x_dev + max_off + 1; p.x_numel = max_off + 1;
    p.x_align = (unsigned)(((uintptr_t)x_dev >> 2) & 3); p.bulk_ok = bulk ? 1 : 0; p.dbuf = 0;
    p.wh = plan->wh; p.twp = plan->twp; p.twn = plan->twn; p.twn2 = plan->twn2;
    p.cosw = plan->cosw; p.cw_a0 = plan->cw_a0; p.cwq = plan->cwq;
    p.out = out_dev; p.o_sb = od->stride_b; p.o_sc = od->stride_c; p.o_st = od->stride_t; p.o_sk = od->stride_f;
    p.mode = mode;
    if (fbmode) {
        p.bands = fb->bands; p.fbw = fb->w; p.n_bands = fb->n_bands; p.n_fbw = fb->n_w;
        p.cw = fb->cw; p.cm = fb->cm; p.cg = fb->cg; p.n_chunks = fb->n_chunks;
        p.mw = fb->mw; p.ms = fb->ms; p.mg = fb->mg; p.n_msteps = fb->n_msteps;
        p.bd = fb->bd; p.bg = fb->bg; p.n_bd = fb->n_bd;
        // the groups of a warp walk bands of different lengths; the flat predicated chunk list is balanced per group and
        // is the default (chosen on the previous GPU target, not yet re-measured on H100).
        p.fb_bands = (fb->bd && kb_env_int("KAPRE_B200_FBBANDS", 0)) ? 1 : 0;
    }
    if (dbmode) {
        p.amin = db->amin; p.db_mul = db_mul; p.db_sub = db_sub; p.item_max = (unsigned int*)workspace_dev;
        p.db_ftz = (db->amin >= 1.17549435e-38f) ? 1 : 0;
    }
    if (mode == KAPRE_OUT_MAG_PHASE) { p.db_on = dbmode ? 1 : 0; p.ph_off = (long long)C * od->stride_c; }
    // interleaved (channels_last) tensors with several channels: tiles that hold all channels
    const bool strided_in = xd->stride_l != 1, strided_out = od->stride_f != 1;
    const bool mc_ok = C > 1 && C <= 32 && (strided_in || strided_out) && xd->stride_b >= 0 &&
                       xd->stride_c >= 0 && xd->stride_l >= 0 && kb_env_int("KAPRE_B200_NOMC", 0) == 0;
    FwdCfg mcfg{};
    const int mc_wh = (!plan->cosw || (plan->hop & 1)) ? 1 : 0;
    const bool use_mc = mc_ok && (fbmode ? kb_pick_mcfb_cfg(plan->dev, plan->Q, plan->n_fft, plan->hop, C, mc_wh,
                                                            fb->n_bands, fb->n_chunks, &mcfg)
                                         : kb_pick_mc_cfg(plan->dev, plan->Q, plan->n_fft, plan->hop, C, mc_wh, &mcfg));
    long long tiles;
    int grid;
    if (use_mc) {
        cfg = mcfg;
        p.TF = cfg.TF; p.n_tiles_t = (T + cfg.TF - 1) / cfg.TF; p.n_warps = cfg.NW;
        p.mc_wh = mc_wh;
        p.mc_cl_in = (xd->stride_c < xd->stride_l) ? 1 : 0;
        p.mc_out = (od->stride_c == 1) ? 1 : 0;
        const int FR = cfg.NW * (32 / plan->Q), ncol = cfg.TF * C;
        const int last = ncol - ((ncol - 1) / FR) * FR;
        p.mc_magic_c = kb_magic((unsigned)C);
        p.mc_magic_g = kb_magic((unsigned)((cfg.NW * 32) / C));
        p.mc_magic_fr = kb_magic((unsigned)(FR < ncol ? FR : ncol));
        p.mc_magic_last = kb_magic((unsigned)last);
        tiles = (long long)B * p.n_tiles_t;
        if (tiles > 0x7fffffffLL) return kb_fail(KAPRE_E_UNSUPPORTED, "too many tiles");
        const long long gmax = (long long)plan->dev.sm_count * cfg.bps;
        grid = (int)(tiles < gmax ? tiles : gmax);
        if (fbmode) {
            switch (plan->Q) {
                case 4: rc = kb_launch_stft_mcfb<4>(p, grid, cfg.smem, st); break;
                case 8: rc = kb_launch_stft_mcfb<8>(p, grid, cfg.smem, st); break;
                case 16: rc = kb_launch_stft_mcfb<16>(p, grid, cfg.smem, st); break;
                case 32: rc = kb_launch_stft_mcfb<32>(p, grid, cfg.smem, st); break;
                default: rc = kb_fail(KAPRE_E_UNSUPPORTED, "bad Q");
            }
        } else {
            switch (plan->Q) {
                case 4: rc = kb_launch_stft_mc<4>(p, grid, cfg.smem, st); break;
                case 8: rc = kb_launch_stft_mc<8>(p, grid, cfg.smem, st); break;
                case 16: rc = kb_launch_stft_mc<16>(p, grid, cfg.smem, st); break;
                case 32: rc = kb_launch_stft_mc<32>(p, grid, cfg.smem, st); break;
                default: rc = kb_fail(KAPRE_E_UNSUPPORTED, "bad Q");
            }
        }
    } else {
        p.TF = cfg.TF; p.n_tiles_t = (T + cfg.TF - 1) / cfg.TF; p.n_warps = cfg.NW;
        p.fb_mma = fbmma;
        p.variant = variant;

        tiles = (long long)B * C * p.n_tiles_t;
        if (tiles > 0x7fffffffLL) return kb_fail(KAPRE_E_UNSUPPORTED, "too many tiles");
        const long long gmax = (long long)plan->dev.sm_count * cfg.bps;
        grid = (int)(tiles < gmax ? tiles : gmax);
        switch (plan->Q) {
            case 4: rc = kb_launch_stft<4>(p, grid, cfg.smem, st); break;
            case 8: rc = kb_launch_stft<8>(p, grid, cfg.smem, st); break;
            case 16: rc = kb_launch_stft<16>(p, grid, cfg.smem, st); break;
            case 32: rc = kb_launch_stft<32>(p, grid, cfg.smem, st); break;
            default: rc = kb_fail(KAPRE_E_UNSUPPORTED, "bad Q");
        }
    }
    if (rc) return rc;
    {
        char buf[160];
        snprintf(buf, sizeof(buf), "%sQ%d TF%d NW%d bulk%d grid%d smem%d bps%d tiles%lld fbmma%d v%d", use_mc ? "MC " : "", plan->Q,
                 cfg.TF, cfg.NW, use_mc ? 0 : (int)bulk, grid, cfg.smem, cfg.bps, tiles, use_mc ? 0 : fbmma,
                 use_mc ? 0 : p.variant);
        g_launch_info = buf;
    }
    if (dbmode)
        rc = kb_launch_clamp((float*)out_dev, B, db_item_size, (unsigned int*)workspace_dev, db->amin, db_mul, db_sub,
                             db->dynamic_range, st, db_run, db_period);
    return rc;
}

int kapre_istft_plan_create(int n_fft, int win_length, int hop_length, const float* dual_window_host,
                            kapre_istft_plan** out) {
    if (!out || !dual_window_host) return kb_fail(KAPRE_E_INVALID, "null argument");
    if (n_fft < 2 || win_length < 1 || hop_length < 1)
        return kb_fail(KAPRE_E_INVALID, "n_fft=%d win_length=%d hop_length=%d out of range", n_fft, win_length, hop_length);
    if (n_fft > 16384) return kb_fail(KAPRE_E_UNSUPPORTED, "n_fft=%d > 16384 is not supported", n_fft);
    kapre_istft_plan* p = new kapre_istft_plan();
    p->n_fft = n_fft; p->win_length = win_length; p->hop = hop_length;
    p->Q = kb_q_for_nfft(n_fft);
    p->win = win_length < n_fft ? win_length : n_fft;
    p->dual_host.assign(dual_window_host, dual_window_host + win_length);
    int rc = kb_dev_info(&p->dev);
    if (rc) { delete p; return rc; }
    KbTableUpload tb;
    if (p->Q) {
        std::vector<float> dual; std::vector<float2> twp, twn;
        kb_make_dual(dual_window_host, p->win, n_fft, dual);
        kb_make_twp(p->Q, twp);
        kb_make_twn(n_fft, twn);
        tb.add(dual, &p->dual); tb.add(twp, &p->twp); tb.add(twn, &p->twn);
    }
    {
        std::vector<float> dn(p->win);
        for (int m = 0; m < p->win; ++m) dn[m] = (float)((double)dual_window_host[m] / (double)n_fft);
        std::vector<float2> tw(n_fft);
        for (int r = 0; r < n_fft; ++r) {
            const double a = 2.0 * M_PI * (double)r / (double)n_fft;
            tw[r] = make_float2((float)cos(a), (float)sin(a));
        }
        tb.add(dn, &p->dualn); tb.add(tw, &p->tw);
    }
    if ((rc = tb.upload(p->tables, "istft"))) { delete p; return rc; }
    *out = p;
    return 0;
}

void kapre_istft_plan_destroy(kapre_istft_plan* p) {
    if (!p) return;
    kapre_stft_plan_destroy(p->adj);
    delete p;
}

int kapre_istft_inverse(const kapre_istft_plan* plan, const void* stft_dev, int batch, int channels, int frames,
                        const kapre_spec_desc* sd, float* y_dev, const kapre_wave_desc* yd, void* stream) {
    if (!plan || !sd || !yd) return kb_fail(KAPRE_E_INVALID, "null argument");
    int rc = kb_check_device(plan->dev);
    if (rc) return rc;
    if (batch < 0 || channels < 0 || frames < 0) return kb_fail(KAPRE_E_INVALID, "negative size");
    if (batch == 0 || channels == 0 || frames == 0) return 0;
    if (!stft_dev || !y_dev) return kb_fail(KAPRE_E_INVALID, "null data pointer");
    cudaStream_t st = (cudaStream_t)stream;
    const long long out_len = (long long)(frames - 1) * plan->hop + plan->win_length;
    if (out_len > 0x7fffffffLL) return kb_fail(KAPRE_E_UNSUPPORTED, "signal too long");
    if (yd->length != (int)out_len)
        return kb_fail(KAPRE_E_INVALID, "output length must be (frames-1)*hop+win_length = %lld, got %d", out_len, yd->length);

    if (!plan->Q) {
        KbIdftParams p{};
        p.X = (const float2*)stft_dev; p.x_sb = sd->stride_b; p.x_sc = sd->stride_c; p.x_st = sd->stride_t; p.x_sk = sd->stride_f;
        p.B = batch; p.C = channels; p.T = frames; p.n_fft = plan->n_fft; p.hop = plan->hop; p.win = plan->win;
        p.out_len = (int)out_len; p.dualn = plan->dualn; p.tw = plan->tw;
        p.y = y_dev; p.y_sb = yd->stride_b; p.y_sc = yd->stride_c; p.y_sl = yd->stride_l;
        p.n_warps = 8; p.n_tiles_s = (int)((out_len + 255) / 256);
        const int smem = plan->n_fft * 8;
        if (smem > plan->dev.smem_optin) return kb_fail(KAPRE_E_UNSUPPORTED, "n_fft too large");
        long long tiles = (long long)batch * channels * p.n_tiles_s;
        int grid = (int)(tiles < plan->dev.sm_count * 8LL ? tiles : plan->dev.sm_count * 8LL);
        return kb_launch(kb_idft_kernel, {.grid = grid, .block = 256, .smem = smem, .st = st}, p);
    }

    const int Q = plan->Q, FPW = 32 / Q;
    const int R = (plan->win + plan->hop - 1) / plan->hop;
    if (kb_env_int("KAPRE_B200_ISTFT2", 1)) {
        // streaming kernel: tiles of seg = m * FR - (R - 1) output hops, m rounds of FR = NW * FPW frames each.  m is the
        // round count that minimises (waves of tiles over the resident CTAs) x (rounds per tile).
        const int NW = KB_ISTFT_MAX_WARPS, FR = NW * FPW;
        const KbIstft2Smem L2 = kb_istft2_smem_layout(Q, plan->n_fft, plan->hop, plan->win, NW);
        if (L2.total <= plan->dev.smem_optin) {
            int bps = (228 * 1024) / (L2.total + 1024);
            if (bps > 4) bps = 4;              // __launch_bounds__(128, 4)
            if (bps < 1) bps = 1;
            const long long slots = (long long)plan->dev.sm_count * bps;
            const long long hops = (out_len + plan->hop - 1) / plan->hop;
            // rounds per tile: the most (<= 6: R - 1 halo frames per tile cost <= 6 %) that still leave about one tile per
            // resident CTA (the static tile walk balances per SM, not per CTA).  The 6-round cap and the 85 % fill target
            // are carried over from the previous GPU target and not yet re-measured on H100.
            // Floor: tiles long enough that the halo stays under ~20 % of the frames (hop << win: R is large).
            int m_lo = (5 * (R - 1) + FR - 1) / FR;
            if (m_lo < 1) m_lo = 1;
            const int m_hi = m_lo > 6 ? m_lo : 6;
            int best_m = m_lo, best_seg = m_lo * FR - (R - 1);
            for (int m = m_hi; m >= m_lo; --m) {
                const int seg = m * FR - (R - 1);
                const long long nt = (long long)batch * channels * ((hops + seg - 1) / seg);
                best_m = m; best_seg = seg;
                if (nt * 100 >= slots * 85) break;
            }
            const int m_env = kb_env_int("KAPRE_B200_ISTFT2_M", 0);
            if (m_env > 0 && m_env * FR - (R - 1) >= 1) { best_m = m_env; best_seg = m_env * FR - (R - 1); }
            KbIstftParams p{};
            p.X = (const float2*)stft_dev; p.x_sb = sd->stride_b; p.x_sc = sd->stride_c; p.x_st = sd->stride_t; p.x_sk = sd->stride_f;
            p.B = batch; p.C = channels; p.T = frames; p.n_fft = plan->n_fft; p.hop = plan->hop; p.win = plan->win;
            p.out_len = (int)out_len; p.dual = plan->dual; p.twp = plan->twp; p.twn = plan->twn;
            p.y = y_dev; p.y_sb = yd->stride_b; p.y_sc = yd->stride_c; p.y_sl = yd->stride_l;
            p.R = R; p.seg = best_seg; p.n_warps = NW;
            p.n_tiles_t = kb_istft2_tiles(frames, plan->hop, plan->win_length, best_seg);
            const long long tiles = (long long)batch * channels * p.n_tiles_t;
            if (tiles > 0x7fffffffLL) return kb_fail(KAPRE_E_UNSUPPORTED, "too many tiles");
            const int grid = (int)(tiles < slots ? tiles : slots);
            {
                char buf[160];
                snprintf(buf, sizeof(buf), "ISTFT2 Q%d NW%d seg%d rounds%d tiles%lld grid%d smem%d bps%d", Q, NW, best_seg, best_m, tiles, grid, L2.total, bps);
                g_launch_info = buf;
            }
            void (*kernel)(KbIstftParams);
            switch (Q) {
                case 4: kernel = kb_istft2_kernel<4>; break;
                case 8: kernel = kb_istft2_kernel<8>; break;
                case 16: kernel = kb_istft2_kernel<16>; break;
                case 32: kernel = kb_istft2_kernel<32>; break;
                default: return kb_fail(KAPRE_E_UNSUPPORTED, "bad Q");
            }
            return kb_launch(kernel, {.grid = grid, .block = NW * 32, .smem = L2.total, .st = st, .timed = true}, p);
        }
    }
    // one FFT round per overlap class: TFc = R * NW * FPW frames per tile
    int NW = kb_env_int("KAPRE_B200_INW", KB_ISTFT_MAX_WARPS), TFc = 0, smem = 0, bps = 0;
    if (NW > KB_ISTFT_MAX_WARPS || NW < 1) NW = KB_ISTFT_MAX_WARPS;
    for (;; NW >>= 1) {
        if (NW < 1) return kb_fail(KAPRE_E_UNSUPPORTED, "inverse STFT tile does not fit shared memory (n_fft=%d hop=%d)", plan->n_fft, plan->hop);
        TFc = R * NW * FPW;
        if (TFc < R) TFc = R;
        const KbIstftSmem L = kb_istft_smem_layout(Q, plan->n_fft, plan->hop, plan->win, TFc, NW);
        smem = L.total;
        if (smem <= plan->dev.smem_optin) break;
    }
    bps = (228 * 1024) / (smem + 1024);
    if (bps > 3) bps = 3;              // __launch_bounds__(128, 3): 168 registers per thread
    if (bps < 1) bps = 1;
    KbIstftParams p{};
    p.X = (const float2*)stft_dev; p.x_sb = sd->stride_b; p.x_sc = sd->stride_c; p.x_st = sd->stride_t; p.x_sk = sd->stride_f;
    p.B = batch; p.C = channels; p.T = frames; p.n_fft = plan->n_fft; p.hop = plan->hop; p.win = plan->win;
    p.out_len = (int)out_len; p.dual = plan->dual; p.twp = plan->twp; p.twn = plan->twn;
    p.y = y_dev; p.y_sb = yd->stride_b; p.y_sc = yd->stride_c; p.y_sl = yd->stride_l;
    p.TFc = TFc; p.R = R; p.hops_out = TFc - (R - 1);
    p.n_tiles_t = kb_istft_tiles(frames, plan->hop, plan->win_length, p.hops_out);
    p.n_warps = NW;
    const long long tiles = (long long)batch * channels * p.n_tiles_t;
    if (tiles > 0x7fffffffLL) return kb_fail(KAPRE_E_UNSUPPORTED, "too many tiles");
    const long long gmax = (long long)plan->dev.sm_count * bps;
    const int grid = (int)(tiles < gmax ? tiles : gmax);
    void (*kernel)(KbIstftParams);
    switch (Q) {
        case 4: kernel = kb_istft_kernel<4>; break;
        case 8: kernel = kb_istft_kernel<8>; break;
        case 16: kernel = kb_istft_kernel<16>; break;
        case 32: kernel = kb_istft_kernel<32>; break;
        default: return kb_fail(KAPRE_E_UNSUPPORTED, "bad Q");
    }
    return kb_launch(kernel, {.grid = grid, .block = NW * 32, .smem = smem, .st = st, .timed = true}, p);
}

int kapre_filterbank_create(const float* fb_host, int n_freq, int n_bands, kapre_filterbank** out) {
    if (!out || !fb_host) return kb_fail(KAPRE_E_INVALID, "null argument");
    if (n_freq < 1 || n_bands < 1) return kb_fail(KAPRE_E_INVALID, "empty filterbank");
    kapre_filterbank* f = new kapre_filterbank();
    f->n_freq = n_freq; f->n_bands = n_bands;
    int rc = kb_dev_info(&f->dev);
    if (rc) { delete f; return rc; }
    std::vector<KbBand> bands; std::vector<float> w;
    kb_make_bands(fb_host, n_freq, n_bands, bands, w);
    f->n_w = (int)w.size();
    KbTableUpload tb;
    tb.add(bands, &f->bands); tb.add(w, &f->w);
    f->Q = kb_q_for_nfft((n_freq - 1) * 2);
    if (f->Q) {
        std::vector<kb_f4> cw; std::vector<kb_i2> cm; std::vector<int> cg;
        kb_make_fb_chunks(fb_host, n_freq, n_bands, 32, cw, cm, cg);
        f->n_chunks = (int)cw.size();
        tb.add(cw, &f->cw); tb.add(cm, &f->cm); tb.add(cg, &f->cg);
        std::vector<kb_i2> bd; std::vector<int> bg;
        kb_make_fb_band_desc(cm, cg, 32, bd, bg);
        f->n_bd = (int)bd.size();
        tb.add(bd, &f->bd); tb.add(bg, &f->bg);
        std::vector<kb_f4> mw; std::vector<kb_i2> ms; std::vector<int> mg;
        kb_make_fb_mma(fb_host, n_freq, n_bands, mw, ms, mg);
        f->n_msteps = (int)ms.size();
        tb.add(mw, &f->mw); tb.add(ms, &f->ms); tb.add(mg, &f->mg);
    }
    if ((rc = tb.upload(f->tables, "filterbank"))) { delete f; return rc; }
    *out = f;
    return 0;
}

void kapre_filterbank_destroy(kapre_filterbank* f) { delete f; }

int kapre_apply_filterbank(const kapre_filterbank* fb, const float* x_dev, int batch, int channels, int frames,
                           const kapre_spec_desc* xd, float* out_dev, const kapre_spec_desc* od, void* stream) {
    if (!fb || !xd || !od) return kb_fail(KAPRE_E_INVALID, "null argument");
    int rc = kb_check_device(fb->dev);
    if (rc) return rc;
    if (batch < 0 || channels < 0 || frames < 0) return kb_fail(KAPRE_E_INVALID, "negative size");
    if (batch == 0 || channels == 0 || frames == 0) return 0;
    if (!x_dev || !out_dev) return kb_fail(KAPRE_E_INVALID, "null data pointer");
    KbFbParams p{};
    p.x = x_dev; p.x_sb = xd->stride_b; p.x_sc = xd->stride_c; p.x_st = xd->stride_t; p.x_sk = xd->stride_f;
    p.B = batch; p.C = channels; p.T = frames; p.F = fb->n_freq;
    p.bands = fb->bands; p.fbw = fb->w; p.n_bands = fb->n_bands;
    p.out = out_dev; p.o_sb = od->stride_b; p.o_sc = od->stride_c; p.o_st = od->stride_t; p.o_sk = od->stride_f;
    p.R = kb_fb_pick_r(fb->n_freq, fb->n_bands, fb->dev.smem_optin);
    if (p.R == 0)
        return kb_fail(KAPRE_E_UNSUPPORTED, "filterbank %dx%d does not fit shared memory", fb->n_freq, fb->n_bands);
    p.n_tiles_t = (frames + p.R - 1) / p.R; p.n_warps = 8;
    const KbFbSmem L = kb_fb_smem_layout(fb->n_freq, fb->n_bands, p.R);
    int bps = (228 * 1024) / (L.total + 1024);
    if (bps > 8) bps = 8;
    if (bps < 1) bps = 1;
    const long long tiles = (long long)batch * channels * p.n_tiles_t;
    const long long gmax = (long long)fb->dev.sm_count * bps;
    const int grid = (int)(tiles < gmax ? tiles : gmax);
    return kb_launch(kb_fb_kernel, {.grid = grid, .block = 256, .smem = L.total, .st = (cudaStream_t)stream}, p);
}

static int kb_ew_grid(int64_t n, int* grid) {
    int dev = 0, sms = 0;
    KB_CUDA(cudaGetDevice(&dev));
    KB_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    long long g = (n + 255) / 256;
    const long long cap = (long long)sms * 16;
    *grid = (int)(g < cap ? g : cap);
    if (*grid < 1) *grid = 1;
    return 0;
}

int kapre_magnitude(const void* x_complex_dev, float* out_dev, int64_t n, void* stream) {
    if (n < 0) return kb_fail(KAPRE_E_INVALID, "negative size");
    if (n == 0) return 0;
    if (!x_complex_dev || !out_dev) return kb_fail(KAPRE_E_INVALID, "null data pointer");
    int grid, rc;
    if ((rc = kb_ew_grid(n, &grid))) return rc;
    return kb_launch(kb_magnitude_kernel, {.grid = grid, .block = 256, .st = (cudaStream_t)stream},
                     (const float2*)x_complex_dev, out_dev, n);
}

int kapre_phase(const void* x_complex_dev, float* out_dev, int64_t n, void* stream) {
    if (n < 0) return kb_fail(KAPRE_E_INVALID, "negative size");
    if (n == 0) return 0;
    if (!x_complex_dev || !out_dev) return kb_fail(KAPRE_E_INVALID, "null data pointer");
    int grid, rc;
    if ((rc = kb_ew_grid(n, &grid))) return rc;
    return kb_launch(kb_phase_kernel, {.grid = grid, .block = 256, .st = (cudaStream_t)stream},
                     (const float2*)x_complex_dev, out_dev, n);
}

int kapre_concat_frequency_map(const float* x_dev, float* out_dev, int64_t batch, int64_t channels, int64_t frames,
                               int64_t n_freq, int channels_last, void* stream) {
    if (batch < 0 || channels < 0 || frames < 0 || n_freq < 0) return kb_fail(KAPRE_E_INVALID, "negative size");
    const long long total = (long long)batch * (channels + 1) * frames * n_freq;
    if (total == 0) return 0;
    if (!out_dev || (!x_dev && channels > 0)) return kb_fail(KAPRE_E_INVALID, "null data pointer");
    int grid, rc;
    if ((rc = kb_ew_grid(total, &grid))) return rc;
    return kb_launch(kb_concat_freq_map_kernel, {.grid = grid, .block = 256, .st = (cudaStream_t)stream}, x_dev, out_dev,
                     batch, channels, frames, n_freq, channels_last ? 1 : 0);
}

int kapre_spec_augment(const float* x_dev, float* out_dev, int64_t batch, int64_t frames, int64_t n_freq,
                       const int* time_masks_dev, int n_time_masks, const int* freq_masks_dev, int n_freq_masks,
                       float mask_value, void* stream) {
    if (batch < 0 || frames < 0 || n_freq < 0 || n_time_masks < 0 || n_freq_masks < 0) return kb_fail(KAPRE_E_INVALID, "negative size");
    const long long total = (long long)batch * frames * n_freq;
    if (total == 0) return 0;
    if (!x_dev || !out_dev || (n_time_masks && !time_masks_dev) || (n_freq_masks && !freq_masks_dev))
        return kb_fail(KAPRE_E_INVALID, "null data pointer");
    int grid, rc;
    if ((rc = kb_ew_grid(total, &grid))) return rc;
    return kb_launch(kb_spec_augment_kernel, {.grid = grid, .block = 256, .st = (cudaStream_t)stream}, x_dev, out_dev,
                     batch, frames, n_freq, time_masks_dev, n_time_masks, freq_masks_dev, n_freq_masks, mask_value);
}

static int kb_frames_for(int L, int fl, int hop, int pad_end) {
    if (pad_end) return (L + hop - 1) / hop;
    return L < fl ? 0 : 1 + (L - fl) / hop;
}

int kapre_delta(const float* x_dev, float* out_dev, int64_t outer, int64_t frames, int64_t inner, int win_length,
                int pad_mode, void* stream) {
    if (win_length < 3 || (win_length & 1) == 0) return kb_fail(KAPRE_E_INVALID, "win_length must be odd and >= 3, got %d", win_length);
    if (pad_mode < 0 || pad_mode > 2) return kb_fail(KAPRE_E_INVALID, "bad pad_mode %d", pad_mode);
    if (outer < 0 || frames < 0 || inner < 0) return kb_fail(KAPRE_E_INVALID, "negative size");
    const long long total = (long long)outer * frames * inner;
    if (total == 0) return 0;
    if (!x_dev || !out_dev) return kb_fail(KAPRE_E_INVALID, "null data pointer");
    if (x_dev == out_dev) return kb_fail(KAPRE_E_INVALID, "delta cannot run in place");
    const int n = (win_length - 1) / 2;
    double denom = 0;
    for (int m = 1; m <= n; ++m) denom += 2.0 * m * m;
    int grid, rc;
    if ((rc = kb_ew_grid(total, &grid))) return rc;
    return kb_launch(kb_delta_kernel, {.grid = grid, .block = 256, .st = (cudaStream_t)stream}, x_dev, out_dev, outer,
                     frames, inner, n, (float)(1.0 / denom), pad_mode);
}

int kapre_frame(const float* x_dev, const kapre_wave_desc* xd, int frame_length, int hop_length, int pad_end, float pad_value,
                float* out_dev, const kapre_spec_desc* od, void* stream) {
    if (!xd || !od) return kb_fail(KAPRE_E_INVALID, "null argument");
    if (frame_length <= 0 || hop_length <= 0) return kb_fail(KAPRE_E_INVALID, "frame_length and hop_length must be positive");
    const int T = kb_frames_for(xd->length, frame_length, hop_length, pad_end);
    const long long total = (long long)xd->batch * xd->channels * T * frame_length;
    if (total <= 0) return 0;
    if (!x_dev || !out_dev) return kb_fail(KAPRE_E_INVALID, "null data pointer");
    int grid, rc;
    if ((rc = kb_ew_grid(total, &grid))) return rc;
    return kb_launch(kb_frame_kernel, {.grid = grid, .block = 256, .st = (cudaStream_t)stream}, x_dev, xd->stride_b,
                     xd->stride_c, xd->stride_l, xd->batch, xd->channels, xd->length, frame_length, hop_length, T,
                     pad_value, out_dev, od->stride_b, od->stride_c, od->stride_t, od->stride_f);
}

int kapre_energy(const float* x_dev, const kapre_wave_desc* xd, int frame_length, int hop_length, int pad_end, float pad_value,
                 float scale, float* out_dev, const kapre_wave_desc* od, void* stream) {
    if (!xd || !od) return kb_fail(KAPRE_E_INVALID, "null argument");
    if (frame_length <= 0 || hop_length <= 0) return kb_fail(KAPRE_E_INVALID, "frame_length and hop_length must be positive");
    const int T = kb_frames_for(xd->length, frame_length, hop_length, pad_end);
    const long long n_frames = (long long)xd->batch * xd->channels * T;
    if (n_frames <= 0) return 0;
    if (!x_dev || !out_dev) return kb_fail(KAPRE_E_INVALID, "null data pointer");
    if (od->length != T) return kb_fail(KAPRE_E_INVALID, "output must have %d frames, got %d", T, od->length);
    int grid, rc;
    if ((rc = kb_ew_grid(n_frames * 32, &grid))) return rc;
    return kb_launch(kb_energy_kernel, {.grid = grid, .block = 256, .st = (cudaStream_t)stream}, x_dev, xd->stride_b,
                     xd->stride_c, xd->stride_l, xd->batch, xd->channels, xd->length, frame_length, hop_length, T,
                     pad_value, scale, out_dev, od->stride_b, od->stride_c, od->stride_l);
}

int kapre_magnitude_to_decibel(const float* x_dev, float* out_dev, int64_t n_items, int64_t item_size,
                               const kapre_db_cfg* db, void* workspace_dev, void* stream) {
    int rc = kb_check_db(db);
    if (rc) return rc;
    if (n_items < 0 || item_size < 0) return kb_fail(KAPRE_E_INVALID, "negative size");
    if (n_items == 0 || item_size == 0) return 0;
    if (!x_dev || !out_dev || !workspace_dev) return kb_fail(KAPRE_E_INVALID, "null data pointer");
    cudaStream_t st = (cudaStream_t)stream;
    float db_mul, db_sub;
    kb_db_consts(db, &db_mul, &db_sub);
    long long chunks = (item_size + 256 * 8 - 1) / (256 * 8);
    if (chunks > 64) chunks = 64;
    if (chunks < 1) chunks = 1;
    const long long grid = n_items * chunks;
    if (grid > 0x7fffffffLL) return kb_fail(KAPRE_E_UNSUPPORTED, "too many items");
    if ((rc = kb_launch(kb_db_kernel, {.grid = (int)grid, .block = 256, .st = st}, x_dev, out_dev, item_size, (int)chunks,
                        (unsigned int*)workspace_dev, db->amin, db_mul, db_sub)))
        return rc;
    return kb_launch_clamp(out_dev, n_items, item_size, (unsigned int*)workspace_dev, db->amin, db_mul, db_sub,
                           db->dynamic_range, st);
}

// Experimental: the next tensor-core log-mel launch also dumps its complex spectrum (signals, T, 513) float2 to dbg_dev.
int kapre_tc_set_debug(void* dbg_dev) { g_tc_dbg = (float2*)dbg_dev; return 0; }

// ---- experimental: tensor-core (wgmma) DFT stage, see tc_dft.cuh -----------------------------------
// Stage 1 of the 32 x 32 factorisation of the n_fft = 1024 / hop = 256 real FFT over `n_items` waveforms of
// `length` samples (`item_stride` floats apart).  store != 0: out = (items, T, 32, 32) floats with
// out[i, f, n2, 2 k1 + {0,1}] = Re / Im of sum_n1 x[256 f + 32 n1 + n2] exp(-2 pi i n1 k1 / 32), k1 = 0..15, except
// column 1 (Im of k1 = 0, identically zero), which carries the real k1 = 16 sum.  store == 0 (timing): out must
// hold grid * 256 floats of checksums; *grid_out receives the grid size.  T = 1 + (length - 1024) / 256.
int kapre_tc_dft_stage1(const float* x_dev, int n_items, long long item_stride, int length, float* out_dev, int store,
                        int* grid_out, const float* fmat_override_dev, void* stream) {
    if (!x_dev || !out_dev) return kb_fail(KAPRE_E_INVALID, "null data pointer");
    if (n_items < 1 || length < KB_TC_NFFT) return kb_fail(KAPRE_E_INVALID, "need n_items >= 1 and length >= 1024");
    DevInfo dev;
    int rc = kb_dev_info(&dev);
    if (rc) return rc;
    // one matrix per device, kept for the life of the process (never freed: a static KbTables would call cudaFree
    // at exit, when the CUDA runtime may already be gone)
    static KbTables* const fmat = new KbTables[64];
    if (dev.device < 0 || dev.device >= 64) return kb_fail(KAPRE_E_UNSUPPORTED, "device index");
    KbTables& t = fmat[dev.device];
    if (!t.block) {
        std::vector<float> f(2048);
        for (int kc = 0; kc < 8; ++kc)
            for (int c = 0; c < 32; ++c)
                for (int e = 0; e < 4; ++e) {
                    const int n1 = 4 * kc + e, k1 = c >> 1;
                    double v;
                    if (c == 1) v = (n1 & 1) ? -1.0 : 1.0;                       // k1 = 16: (-1)^n1
                    else {
                        const double a = -2.0 * M_PI * (double)((n1 * k1) % 32) / 32.0;
                        v = (c & 1) ? sin(a) : cos(a);
                    }
                    const float w = (float)v, hi = kb_tf32_hi(w);
                    f[(size_t)(kc * 32 + c) * 4 + e] = hi;
                    f[1024 + (size_t)(kc * 32 + c) * 4 + e] = w - hi;
                }
        KbTableUpload tb;
        const float* m;   // the block's one table, at its start
        tb.add(f, &m);
        if ((rc = tb.upload(t, "tc_dft"))) return rc;
    }
    KbTcParams p{};
    p.x = x_dev; p.item_stride = item_stride; p.n_items = n_items; p.length = length;
    p.T = 1 + (length - KB_TC_NFFT) / KB_TC_HOP;
    p.out = out_dev; p.store = store;
    p.fmat = fmat_override_dev ? fmat_override_dev : (const float*)t.block;   // override: layout debugging (2048 floats)
    p.n_tiles_t = (p.T + KB_TC_TILE_F - 1) / KB_TC_TILE_F;
    const long long tiles = (long long)n_items * p.n_tiles_t;
    const long long gmax = (long long)dev.sm_count * 2;
    const int grid = (int)(tiles < gmax ? tiles : gmax);
    if (grid_out) *grid_out = grid;
    return kb_launch(kb_tc_dft_stage1_kernel, {.grid = grid, .block = KB_TC_THREADS, .smem = KB_TC_SMEM,
                                               .st = (cudaStream_t)stream, .timed = true}, p);
}

}  // extern "C"

// ---- backward passes (grad_core.cuh) ---------------------------------------------------------------
// Adjoint plans are constants of their owner: made on first use under the owner's lock, freed with it.
static int kb_stft_adjoint_plan(const kapre_stft_plan* cp, kapre_istft_plan** out) {
    kapre_stft_plan* p = const_cast<kapre_stft_plan*>(cp);
    std::lock_guard<std::mutex> lk(p->adj_mu);
    if (!p->adj) {
        // dual window w * N/2: the inverse kernel's irfft carries 1/N and weighs interior bins 2
        std::vector<float> d(p->win_length, 0.0f);
        for (int m = 0; m < p->win_eff; ++m) d[m] = (float)((double)p->window_host[m] * (double)p->n_fft * 0.5);
        int rc = kapre_istft_plan_create(p->n_fft, p->win_length, p->hop, d.data(), &p->adj);
        if (rc) { p->adj = nullptr; return rc; }
    }
    *out = p->adj;
    return 0;
}

static int kb_istft_adjoint_plan(const kapre_istft_plan* cp, kapre_stft_plan** out) {
    kapre_istft_plan* p = const_cast<kapre_istft_plan*>(cp);
    std::lock_guard<std::mutex> lk(p->adj_mu);
    if (!p->adj) {
        // window dual * 2/N over the first min(win_length, n_fft) samples (the only ones the inverse produces)
        std::vector<float> w(p->win_length, 0.0f);
        for (int m = 0; m < p->win; ++m) w[m] = (float)((double)p->dual_host[m] * 2.0 / (double)p->n_fft);
        int rc = kapre_stft_plan_create(p->n_fft, p->win_length, p->hop, w.data(), &p->adj);
        if (rc) { p->adj = nullptr; return rc; }
    }
    *out = p->adj;
    return 0;
}

__global__ void kb_stft_adj_kernel(const __grid_constant__ KbStftAdjParams p, long long n) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        kb_stft_adj_elem(p, i);
}

__global__ void kb_istft_adj_kernel(const __grid_constant__ KbIstftAdjParams p, long long n) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        kb_istft_adj_elem(p, i);
}

__global__ void kb_mag_bwd_kernel(const float2* __restrict__ X, const float* __restrict__ g, float2* __restrict__ gX,
                                  long long n) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        kb_mag_bwd_elem(X, g, gX, i);
}

// one decibel-backward pass: `chunks` CTAs per item, each walking a strided share of the item
template <int PASS>
__global__ void __launch_bounds__(256) kb_dbb_kernel(const __grid_constant__ KbDbBwdParams p, int chunks) {
    const long long item = blockIdx.x / chunks;
    const int chunk = (int)(blockIdx.x - item * chunks);
    const long long i0 = (long long)chunk * blockDim.x + threadIdx.x, step = (long long)chunks * blockDim.x;
    if (PASS == 0) kb_dbb_max(p, item, i0, step, threadIdx.x);
    else if (PASS == 1) kb_dbb_pass(p, item, i0, step, threadIdx.x);
    else kb_dbb_share(p, item, i0, step);
}

// adjacent layers' backward passes (grad_aux_core.cuh): grid-stride loops over the gradient they write
__global__ void kb_phase_bwd_kernel(const float2* __restrict__ X, const float* __restrict__ g, float2* __restrict__ gX,
                                    long long n) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        kb_phase_bwd_elem(X, g, gX, i);
}

__global__ void kb_mag_phase_bwd_kernel(const __grid_constant__ KbMagPhaseBwdParams p, long long n) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        kb_mag_phase_bwd_elem(p, i);
}

__global__ void kb_delta_bwd_kernel(const float* __restrict__ g, float* __restrict__ gx, long long T, long long inner,
                                    int n, float inv_denom, int mode, long long total) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x)
        kb_delta_bwd_elem(g, gx, T, inner, n, inv_denom, mode, i);
}

__global__ void kb_frame_bwd_kernel(const __grid_constant__ KbFrameBwdParams p, long long n) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        kb_frame_bwd_elem(p, i);
}

__global__ void kb_energy_bwd_kernel(const __grid_constant__ KbFrameBwdParams p, long long n) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        kb_energy_bwd_elem(p, i);
}

__global__ void kb_concat_fm_bwd_kernel(const float* __restrict__ g, float* __restrict__ gx, long long C, long long T,
                                        long long F, int channels_last, long long n) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        kb_concat_fm_bwd_elem(g, gx, C, T, F, channels_last, i);
}

// padded-signal geometry of the STFT adjoint: frames, overlap-add length, and whether the overlap-add can be
// written straight into gx (no pad in front and no sample past the signal's end)
static void kb_stft_adj_geom(const kapre_stft_plan* p, int length, int pad_begin, int pad_end, int* T, long long* ola_len,
                             bool* direct) {
    *T = kapre_stft_num_frames(p, length, pad_begin, pad_end);
    *ola_len = *T > 0 ? (long long)(*T - 1) * p->hop + p->win_length : 0;
    *direct = !pad_begin && *ola_len <= length;
}

// the workspace of the STFT adjoint: the (B, C, ola_len) overlap-add, unless it goes straight into gx
static float* kb_stft_adj_layout(KbLayout& L, int batch, int channels, int T, long long ola_len, bool direct) {
    return direct || T <= 0 ? nullptr : L.take<float>(batch, channels, ola_len);
}

extern "C" {

int64_t kapre_stft_backward_workspace_bytes(const kapre_stft_plan* plan, int batch, int channels, int length,
                                            int pad_begin, int pad_end) {
    if (!plan || batch < 0 || channels < 0 || length < 0) return kb_fail(KAPRE_E_INVALID, "bad argument");
    int T;
    long long ola_len;
    bool direct;
    kb_stft_adj_geom(plan, length, pad_begin, pad_end, &T, &ola_len, &direct);
    KbLayout L;
    kb_stft_adj_layout(L, batch, channels, T, ola_len, direct);
    return L.bytes("stft_backward");
}

int kapre_stft_backward(const kapre_stft_plan* plan, const void* g_dev, const kapre_spec_desc* gd, int batch,
                        int channels, int frames, int pad_begin, int pad_end, float* gx_dev, const kapre_wave_desc* xd,
                        void* workspace_dev, void* stream) {
    if (!plan || !gd || !xd) return kb_fail(KAPRE_E_INVALID, "null argument");
    int rc = kb_check_device(plan->dev);
    if (rc) return rc;
    if (xd->batch != batch || xd->channels != channels || batch < 0 || channels < 0 || xd->length < 0)
        return kb_fail(KAPRE_E_INVALID, "gx descriptor (%d, %d) does not match batch=%d channels=%d", xd->batch,
                       xd->channels, batch, channels);
    if (pad_begin && plan->hop > plan->n_fft)
        return kb_fail(KAPRE_E_INVALID, "pad_begin needs hop_length <= n_fft");
    const int L = xd->length;
    int T;
    long long ola_len;
    bool direct;
    kb_stft_adj_geom(plan, L, pad_begin, pad_end, &T, &ola_len, &direct);
    if (frames != T) return kb_fail(KAPRE_E_INVALID, "%d samples give %d frames, got frames=%d", L, T, frames);
    const long long n = (long long)batch * channels * L;
    if (n == 0) return 0;
    if (!gx_dev || (T > 0 && !g_dev)) return kb_fail(KAPRE_E_INVALID, "null data pointer");
    if (T > 0 && !direct && !workspace_dev)
        return kb_fail(KAPRE_E_INVALID, "workspace of kapre_stft_backward_workspace_bytes() bytes required");
    cudaStream_t st = (cudaStream_t)stream;
    KbStftAdjParams q{};
    q.G = (const float2*)g_dev; q.g_sb = gd->stride_b; q.g_sc = gd->stride_c; q.g_st = gd->stride_t; q.g_sk = gd->stride_f;
    q.gx = gx_dev; q.x_sb = xd->stride_b; q.x_sc = xd->stride_c; q.x_sl = xd->stride_l;
    q.B = batch; q.C = channels; q.L = L; q.T = T;
    q.n_fft = plan->n_fft; q.hop = plan->hop; q.win_eff = plan->win_eff; q.pad_left = pad_begin ? plan->n_fft - plan->hop : 0;
    q.w = plan->w;
    if (T > 0) {
        kapre_istft_plan* adj;
        if ((rc = kb_stft_adjoint_plan(plan, &adj))) return rc;
        kapre_wave_desc od;
        od.batch = batch; od.channels = channels; od.length = (int)ola_len;
        if (direct) {   // in place: the pass below reads and writes the same sample
            od.stride_b = xd->stride_b; od.stride_c = xd->stride_c; od.stride_l = xd->stride_l;
            q.ola = gx_dev;
        } else {
            od.stride_b = (long long)channels * ola_len; od.stride_c = ola_len; od.stride_l = 1;
            KbLayout L{(char*)workspace_dev};
            q.ola = kb_stft_adj_layout(L, batch, channels, T, ola_len, direct);
        }
        q.a_sb = od.stride_b; q.a_sc = od.stride_c; q.a_sl = od.stride_l;
        if ((rc = kapre_istft_inverse(adj, g_dev, batch, channels, T, gd, (float*)q.ola, &od, stream))) return rc;
    }
    int grid;
    if ((rc = kb_ew_grid(n, &grid))) return rc;
    return kb_launch(kb_stft_adj_kernel, {.grid = grid, .block = 256, .st = st}, q, n);
}

int kapre_istft_backward(const kapre_istft_plan* plan, const float* gy_dev, const kapre_wave_desc* yd, int batch,
                         int channels, int frames, void* gX_dev, const kapre_spec_desc* sd, void* stream) {
    if (!plan || !yd || !sd) return kb_fail(KAPRE_E_INVALID, "null argument");
    int rc = kb_check_device(plan->dev);
    if (rc) return rc;
    if (batch < 0 || channels < 0 || frames < 0) return kb_fail(KAPRE_E_INVALID, "negative size");
    if (yd->batch != batch || yd->channels != channels)
        return kb_fail(KAPRE_E_INVALID, "gy descriptor (%d, %d) does not match batch=%d channels=%d", yd->batch,
                       yd->channels, batch, channels);
    if (batch == 0 || channels == 0 || frames == 0) return 0;
    const long long out_len = (long long)(frames - 1) * plan->hop + plan->win_length;
    if (yd->length != out_len)
        return kb_fail(KAPRE_E_INVALID, "gy length must be (frames-1)*hop+win_length = %lld, got %d", out_len, yd->length);
    if (!gy_dev || !gX_dev) return kb_fail(KAPRE_E_INVALID, "null data pointer");
    kapre_stft_plan* adj;
    if ((rc = kb_istft_adjoint_plan(plan, &adj))) return rc;
    if ((rc = kapre_stft_forward(adj, gy_dev, yd, 0, 0, KAPRE_OUT_COMPLEX, gX_dev, sd, nullptr, nullptr, nullptr, stream)))
        return rc;
    KbIstftAdjParams q{};
    q.gX = (float2*)gX_dev; q.sb = sd->stride_b; q.sc = sd->stride_c; q.st = sd->stride_t; q.sk = sd->stride_f;
    q.B = batch; q.C = channels; q.T = frames; q.n_fft = plan->n_fft;
    const long long n = (long long)batch * channels * frames * ((plan->n_fft & 1) ? 1 : 2);
    int grid;
    if ((rc = kb_ew_grid(n, &grid))) return rc;
    return kb_launch(kb_istft_adj_kernel, {.grid = grid, .block = 256, .st = (cudaStream_t)stream}, q, n);
}

int kapre_magnitude_backward(const void* x_complex_dev, const float* g_dev, void* gx_complex_dev, int64_t n, void* stream) {
    if (n < 0) return kb_fail(KAPRE_E_INVALID, "negative size");
    if (n == 0) return 0;
    if (!x_complex_dev || !g_dev || !gx_complex_dev) return kb_fail(KAPRE_E_INVALID, "null data pointer");
    int grid, rc;
    if ((rc = kb_ew_grid(n, &grid))) return rc;
    return kb_launch(kb_mag_bwd_kernel, {.grid = grid, .block = 256, .st = (cudaStream_t)stream},
                     (const float2*)x_complex_dev, g_dev, (float2*)gx_complex_dev, n);
}

int kapre_magnitude_to_decibel_backward(const float* x_dev, const float* g_dev, float* gx_dev, int64_t n_items,
                                        int64_t item_size, const kapre_db_cfg* db, void* workspace_dev, void* stream) {
    int rc = kb_check_db(db);
    if (rc) return rc;
    if (n_items < 0 || item_size < 0) return kb_fail(KAPRE_E_INVALID, "negative size");
    if (n_items == 0 || item_size == 0) return 0;
    if (!x_dev || !g_dev || !gx_dev || !workspace_dev) return kb_fail(KAPRE_E_INVALID, "null data pointer");
    if (gx_dev == x_dev) return kb_fail(KAPRE_E_INVALID, "gx must not alias x (the last pass re-reads x)");
    cudaStream_t st = (cudaStream_t)stream;
    KbDbBwdParams p{};
    p.x = x_dev; p.g = g_dev; p.gx = gx_dev; p.item_size = item_size; p.ws = (unsigned int*)workspace_dev;
    p.n_items = n_items; p.amin = db->amin; p.dyn_range = db->dynamic_range;
    p.dscale = (float)(10.0 / log(10.0));
    kb_db_consts(db, &p.db_mul, &p.db_sub);
    long long chunks = (item_size + 256 * 8 - 1) / (256 * 8);
    if (chunks > 64) chunks = 64;
    if (chunks < 1) chunks = 1;
    const long long grid = n_items * chunks;
    if (grid > 0x7fffffffLL) return kb_fail(KAPRE_E_UNSUPPORTED, "too many items");
    const KbLaunch l{.grid = (int)grid, .block = 256, .st = st};
    if ((rc = kb_launch(kb_dbb_kernel<0>, l, p, (int)chunks)) || (rc = kb_launch(kb_dbb_kernel<1>, l, p, (int)chunks)) ||
        (rc = kb_launch(kb_dbb_kernel<2>, l, p, (int)chunks)))
        return rc;
    KB_CUDA(cudaMemsetAsync(workspace_dev, 0, (size_t)n_items * 3 * sizeof(unsigned int), st));   // self-cleaning
    return 0;
}

int kapre_phase_backward(const void* x_complex_dev, const float* g_dev, void* gx_complex_dev, int64_t n, void* stream) {
    if (n < 0) return kb_fail(KAPRE_E_INVALID, "negative size");
    if (n == 0) return 0;
    if (!x_complex_dev || !g_dev || !gx_complex_dev) return kb_fail(KAPRE_E_INVALID, "null data pointer");
    int grid, rc;
    if ((rc = kb_ew_grid(n, &grid))) return rc;
    return kb_launch(kb_phase_bwd_kernel, {.grid = grid, .block = 256, .st = (cudaStream_t)stream},
                     (const float2*)x_complex_dev, g_dev, (float2*)gx_complex_dev, n);
}

int kapre_mag_phase_backward(const void* x_complex_dev, const kapre_spec_desc* x_desc, const float* g_mag_dev,
                             const kapre_spec_desc* gm_desc, const float* g_phase_dev, const kapre_spec_desc* gp_desc,
                             void* gx_complex_dev, const kapre_spec_desc* gx_desc, int batch, int channels, int frames,
                             int n_freq, void* stream) {
    if (!x_desc || !gx_desc || (g_mag_dev && !gm_desc) || (g_phase_dev && !gp_desc))
        return kb_fail(KAPRE_E_INVALID, "null argument");
    if (batch < 0 || channels < 0 || frames < 0 || n_freq < 0) return kb_fail(KAPRE_E_INVALID, "negative size");
    const long long n = (long long)batch * channels * frames * n_freq;
    if (n == 0) return 0;
    if (!x_complex_dev || !gx_complex_dev) return kb_fail(KAPRE_E_INVALID, "null data pointer");
    if (gx_complex_dev == x_complex_dev) return kb_fail(KAPRE_E_INVALID, "gX must not alias X");
    KbMagPhaseBwdParams p{};
    p.X = (const float2*)x_complex_dev;
    p.x_sb = x_desc->stride_b; p.x_sc = x_desc->stride_c; p.x_st = x_desc->stride_t; p.x_sf = x_desc->stride_f;
    p.gm = g_mag_dev;
    if (gm_desc) { p.m_sb = gm_desc->stride_b; p.m_sc = gm_desc->stride_c; p.m_st = gm_desc->stride_t; p.m_sf = gm_desc->stride_f; }
    p.gp = g_phase_dev;
    if (gp_desc) { p.p_sb = gp_desc->stride_b; p.p_sc = gp_desc->stride_c; p.p_st = gp_desc->stride_t; p.p_sf = gp_desc->stride_f; }
    p.gX = (float2*)gx_complex_dev;
    p.o_sb = gx_desc->stride_b; p.o_sc = gx_desc->stride_c; p.o_st = gx_desc->stride_t; p.o_sf = gx_desc->stride_f;
    p.C = channels; p.T = frames; p.F = n_freq;
    p.c_inner = (channels > 1 && gx_desc->stride_c < gx_desc->stride_f) ? 1 : 0;   // channels_last: walk c fastest
    int grid, rc;
    if ((rc = kb_ew_grid(n, &grid))) return rc;
    return kb_launch(kb_mag_phase_bwd_kernel, {.grid = grid, .block = 256, .st = (cudaStream_t)stream}, p, n);
}

int kapre_delta_backward(const float* g_dev, float* gx_dev, int64_t outer, int64_t frames, int64_t inner, int win_length,
                         int pad_mode, void* stream) {
    if (win_length < 3 || (win_length & 1) == 0) return kb_fail(KAPRE_E_INVALID, "win_length must be odd and >= 3, got %d", win_length);
    if (pad_mode < 0 || pad_mode > 2) return kb_fail(KAPRE_E_INVALID, "bad pad_mode %d", pad_mode);
    if (outer < 0 || frames < 0 || inner < 0) return kb_fail(KAPRE_E_INVALID, "negative size");
    const long long total = (long long)outer * frames * inner;
    if (total == 0) return 0;
    if (!g_dev || !gx_dev) return kb_fail(KAPRE_E_INVALID, "null data pointer");
    if (g_dev == gx_dev) return kb_fail(KAPRE_E_INVALID, "delta backward cannot run in place");
    const int n = (win_length - 1) / 2;
    double denom = 0;
    for (int m = 1; m <= n; ++m) denom += 2.0 * m * m;
    int grid, rc;
    if ((rc = kb_ew_grid(total, &grid))) return rc;
    return kb_launch(kb_delta_bwd_kernel, {.grid = grid, .block = 256, .st = (cudaStream_t)stream}, g_dev, gx_dev, frames,
                     inner, n, (float)(1.0 / denom), pad_mode, total);
}

// the frame counts kapre_frame / kapre_energy give `length` samples (pad_end off, on): the gradient must have one of them
static bool kb_frames_match(int length, int fl, int hop, int frames) {
    return frames == kb_frames_for(length, fl, hop, 0) || frames == kb_frames_for(length, fl, hop, 1);
}

int kapre_frame_backward(const float* g_dev, const kapre_spec_desc* g_desc, int frames, int frame_length, int hop_length,
                         float* gx_dev, const kapre_wave_desc* gx_desc, void* stream) {
    if (!g_desc || !gx_desc) return kb_fail(KAPRE_E_INVALID, "null argument");
    if (frame_length <= 0 || hop_length <= 0) return kb_fail(KAPRE_E_INVALID, "frame_length and hop_length must be positive");
    if (gx_desc->batch < 0 || gx_desc->channels < 0 || gx_desc->length < 0 || frames < 0)
        return kb_fail(KAPRE_E_INVALID, "negative size");
    if (!kb_frames_match(gx_desc->length, frame_length, hop_length, frames))
        return kb_fail(KAPRE_E_INVALID, "%d samples do not give %d frames of %d every %d", gx_desc->length, frames,
                       frame_length, hop_length);
    const long long n = (long long)gx_desc->batch * gx_desc->channels * gx_desc->length;
    if (n == 0) return 0;
    if (!gx_dev || (frames > 0 && !g_dev)) return kb_fail(KAPRE_E_INVALID, "null data pointer");
    KbFrameBwdParams p{};
    p.g = g_dev; p.g_sb = g_desc->stride_b; p.g_sc = g_desc->stride_c; p.g_st = g_desc->stride_t; p.g_sn = g_desc->stride_f;
    p.gx = gx_dev; p.o_sb = gx_desc->stride_b; p.o_sc = gx_desc->stride_c; p.o_sl = gx_desc->stride_l;
    p.C = gx_desc->channels; p.L = gx_desc->length; p.T = frames; p.fl = frame_length; p.hop = hop_length;
    int grid, rc;
    if ((rc = kb_ew_grid(n, &grid))) return rc;
    return kb_launch(kb_frame_bwd_kernel, {.grid = grid, .block = 256, .st = (cudaStream_t)stream}, p, n);
}

int kapre_energy_backward(const float* x_dev, const kapre_wave_desc* x_desc, const float* g_dev,
                          const kapre_wave_desc* g_desc, int frame_length, int hop_length, float scale, float* gx_dev,
                          const kapre_wave_desc* gx_desc, void* stream) {
    if (!x_desc || !g_desc || !gx_desc) return kb_fail(KAPRE_E_INVALID, "null argument");
    if (frame_length <= 0 || hop_length <= 0) return kb_fail(KAPRE_E_INVALID, "frame_length and hop_length must be positive");
    if (x_desc->batch < 0 || x_desc->channels < 0 || x_desc->length < 0 || g_desc->length < 0)
        return kb_fail(KAPRE_E_INVALID, "negative size");
    if (gx_desc->batch != x_desc->batch || gx_desc->channels != x_desc->channels || gx_desc->length != x_desc->length ||
        g_desc->batch != x_desc->batch || g_desc->channels != x_desc->channels)
        return kb_fail(KAPRE_E_INVALID, "x, g and gx descriptors disagree on batch / channels / length");
    const int T = g_desc->length;
    if (!kb_frames_match(x_desc->length, frame_length, hop_length, T))
        return kb_fail(KAPRE_E_INVALID, "%d samples do not give %d frames of %d every %d", x_desc->length, T,
                       frame_length, hop_length);
    const long long n = (long long)x_desc->batch * x_desc->channels * x_desc->length;
    if (n == 0) return 0;
    if (!x_dev || !gx_dev || (T > 0 && !g_dev)) return kb_fail(KAPRE_E_INVALID, "null data pointer");
    KbFrameBwdParams p{};
    p.g = g_dev; p.g_sb = g_desc->stride_b; p.g_sc = g_desc->stride_c; p.g_st = g_desc->stride_l;
    p.x = x_dev; p.x_sb = x_desc->stride_b; p.x_sc = x_desc->stride_c; p.x_sl = x_desc->stride_l;
    p.gx = gx_dev; p.o_sb = gx_desc->stride_b; p.o_sc = gx_desc->stride_c; p.o_sl = gx_desc->stride_l;
    p.C = x_desc->channels; p.L = x_desc->length; p.T = T; p.fl = frame_length; p.hop = hop_length;
    p.scale2 = 2.0f * scale;
    int grid, rc;
    if ((rc = kb_ew_grid(n, &grid))) return rc;
    return kb_launch(kb_energy_bwd_kernel, {.grid = grid, .block = 256, .st = (cudaStream_t)stream}, p, n);
}

int kapre_concat_frequency_map_backward(const float* g_dev, float* gx_dev, int64_t batch, int64_t channels,
                                        int64_t frames, int64_t n_freq, int channels_last, void* stream) {
    if (batch < 0 || channels < 0 || frames < 0 || n_freq < 0) return kb_fail(KAPRE_E_INVALID, "negative size");
    const long long n = (long long)batch * channels * frames * n_freq;
    if (n == 0) return 0;
    if (!g_dev || !gx_dev) return kb_fail(KAPRE_E_INVALID, "null data pointer");
    int grid, rc;
    if ((rc = kb_ew_grid(n, &grid))) return rc;
    return kb_launch(kb_concat_fm_bwd_kernel, {.grid = grid, .block = 256, .st = (cudaStream_t)stream}, g_dev, gx_dev,
                     channels, frames, n_freq, channels_last ? 1 : 0, n);
}

}  // extern "C"

// ---- polyphase resampler (resample_core.cuh) ------------------------------------------------------
__global__ void __launch_bounds__(KB_RESAMPLE_THREADS) kb_resample_kernel(const __grid_constant__ KbResampleParams p) {
    extern __shared__ __align__(16) char kb_smem[];
    kb_resample_cta(p, kb_smem, (int)blockIdx.x, (int)gridDim.x);
}

struct kapre_resample_plan {
    int up, down, n_taps, hl, f, Kp;
    int symmetric;
    DevInfo dev;
    KbTables tables;
    float* tab = nullptr;       // up rows of Kp taps, gain folded in (resample_core.cuh)
    std::vector<float> taps_host;
    // adjoint (kapre_resample_backward): up and down exchanged, gain up; made on first use
    std::mutex adj_mu;
    kapre_resample_plan* adj = nullptr;
};

static long long kb_gcd(long long a, long long b) {
    while (b) { const long long t = a % b; a = b; b = t; }
    return a;
}

static int kb_resample_plan_build(int up, int down, const float* taps, int n_taps, double gain, kapre_resample_plan** out) {
    kapre_resample_plan* p = new kapre_resample_plan();
    p->up = up; p->down = down; p->n_taps = n_taps;
    p->hl = (n_taps - 1) / 2;
    p->f = p->hl / up;
    p->Kp = kb_resample_kp(up, n_taps);
    p->taps_host.assign(taps, taps + n_taps);
    p->symmetric = 1;
    for (int k = 0; k < n_taps; ++k)
        if (taps[k] != taps[n_taps - 1 - k]) p->symmetric = 0;
    int rc = kb_dev_info(&p->dev);
    if (rc) { delete p; return rc; }
    if (kb_resample_smem(up, p->Kp, 1, down, 1) > p->dev.smem_optin) {
        const int need = up * p->Kp * 4;
        delete p;
        return kb_fail(KAPRE_E_UNSUPPORTED, "resampling table of %d x %d taps (%d B) does not fit in shared memory", up,
                       need / 4 / up, need);
    }
    std::vector<float> tab;
    kb_resample_table(up, down, taps, n_taps, gain, tab);
    KbTableUpload tb;
    tb.add(tab, &p->tab);
    if ((rc = tb.upload(p->tables, "resample"))) { delete p; return rc; }
    *out = p;
    return 0;
}

// Largest tile (outputs, a power of two <= 2048) whose staged span fits beside the table: in half of the opt-in
// shared memory when possible, so that two CTAs share an SM, else in all of it.
static int kb_resample_pick_nt(const kapre_resample_plan* p, int G) {
    for (int budget : {p->dev.smem_optin / 2 - 1024, p->dev.smem_optin})
        for (int nt = 2048; nt >= 1; nt /= 2)
            if (kb_resample_smem(p->up, p->Kp, nt, p->down, G) <= budget) return nt;
    return 0;
}

static int kb_resample_launch(const kapre_resample_plan* plan, const float* x_dev, const kapre_wave_desc* xd, float* y_dev,
                              const kapre_wave_desc* yd, void* stream) {
    if (!plan || !xd || !yd) return kb_fail(KAPRE_E_INVALID, "null argument");
    if (xd->batch < 0 || xd->channels < 0 || xd->length < 0 || yd->length < 0) return kb_fail(KAPRE_E_INVALID, "negative size");
    if (yd->batch != xd->batch || yd->channels != xd->channels)
        return kb_fail(KAPRE_E_INVALID, "input and output descriptors disagree on batch / channels");
    if ((long long)yd->batch * yd->channels * yd->length == 0) return 0;
    if (!x_dev || !y_dev) return kb_fail(KAPRE_E_INVALID, "null data pointer");
    if ((const void*)x_dev == (const void*)y_dev) return kb_fail(KAPRE_E_INVALID, "resampling cannot run in place");
    int rc = kb_check_device(plan->dev);
    if (rc) return rc;
    KbResampleParams p{};
    const int B = xd->batch, C = xd->channels;
    p.x = x_dev; p.x_sb = xd->stride_b; p.x_sc = xd->stride_c; p.x_sl = xd->stride_l;
    p.B = B; p.C = C; p.L = xd->length;
    p.y = y_dev; p.y_sb = yd->stride_b; p.y_sc = yd->stride_c; p.y_sl = yd->stride_l;
    p.L_out = yd->length;
    p.tab = plan->tab; p.up = plan->up; p.down = plan->down; p.f = plan->f; p.Kp = plan->Kp;
    // channel-interleaved input: all channels in one tile
    const bool interleaved = C > 1 && C <= KB_RESAMPLE_THREADS && llabs(xd->stride_c) < llabs(xd->stride_l);
    p.G = interleaved ? C : 1;
    const bool nonneg = xd->stride_b >= 0 && xd->stride_c >= 0 && xd->stride_l >= 0;
    p.x_numel = (B > 0 && C > 0 && p.L > 0)
        ? (long long)(B - 1) * xd->stride_b + (long long)(C - 1) * xd->stride_c + (long long)(p.L - 1) * xd->stride_l + 1 : 0;
    p.x_align = (unsigned)(((uintptr_t)x_dev >> 2) & 3u);
    p.bulk_ok = nonneg && (((uintptr_t)x_dev & 3u) == 0) &&
                (p.G == 1 ? xd->stride_l == 1 : (xd->stride_c == 1 && xd->stride_l == C)) ? 1 : 0;
    p.NT = kb_resample_pick_nt(plan, p.G);
    if (p.NT == 0)
        return kb_fail(KAPRE_E_UNSUPPORTED, "%d channels of a %d:%d resampler do not fit in shared memory", p.G, plan->up, plan->down);
    if (!kb_resample_setup(p, KB_RESAMPLE_THREADS)) return kb_fail(KAPRE_E_UNSUPPORTED, "too many tiles");
    const int smem = kb_resample_smem(p.up, p.Kp, p.NT, p.down, p.G);
    int grid;
    if ((rc = kb_resident_grid(kb_resample_kernel, "resample", KB_RESAMPLE_THREADS, smem, p.n_tiles, plan->dev.sm_count, &grid)))
        return rc;
    return kb_launch(kb_resample_kernel, {.grid = grid, .block = KB_RESAMPLE_THREADS, .smem = smem,
                                          .st = (cudaStream_t)stream, .timed = true}, p);
}

extern "C" {

int kapre_resample_plan_create(int up, int down, const float* taps_host, int n_taps, kapre_resample_plan** out) {
    if (!out || !taps_host) return kb_fail(KAPRE_E_INVALID, "null argument");
    if (up < 1 || down < 1) return kb_fail(KAPRE_E_INVALID, "up=%d and down=%d must be positive", up, down);
    if (kb_gcd(up, down) != 1) return kb_fail(KAPRE_E_INVALID, "up=%d and down=%d must be coprime (divide both by their gcd)", up, down);
    if (n_taps < 1 || (n_taps & 1) == 0) return kb_fail(KAPRE_E_INVALID, "n_taps=%d must be odd", n_taps);
    const int M = up > down ? up : down;
    if (M > KB_RESAMPLE_MAX_M)
        return kb_fail(KAPRE_E_UNSUPPORTED, "resampling by %d/%d is not supported: max(up, down) = %d exceeds %d (the "
                       "anti-aliasing filter of %d taps would not fit in shared memory)", up, down, M, KB_RESAMPLE_MAX_M,
                       20 * M + 1);
    return kb_resample_plan_build(up, down, taps_host, n_taps, (double)up, out);
}

void kapre_resample_plan_destroy(kapre_resample_plan* p) {
    if (!p) return;
    kapre_resample_plan_destroy(p->adj);
    delete p;
}

int64_t kapre_resample_output_length(const kapre_resample_plan* plan, int64_t length) {
    if (!plan || length < 0) return kb_fail(KAPRE_E_INVALID, "bad argument");
    return (length * plan->up + plan->down - 1) / plan->down;
}

int kapre_resample(const kapre_resample_plan* plan, const float* x_dev, const kapre_wave_desc* x_desc, float* y_dev,
                   const kapre_wave_desc* y_desc, void* stream) {
    return kb_resample_launch(plan, x_dev, x_desc, y_dev, y_desc, stream);
}

int kapre_resample_backward(const kapre_resample_plan* plan, const float* g_dev, const kapre_wave_desc* g_desc,
                            float* gx_dev, const kapre_wave_desc* gx_desc, void* stream) {
    if (!plan) return kb_fail(KAPRE_E_INVALID, "null argument");
    // before the adjoint is made: it is made on the current device
    int rc = kb_check_device(plan->dev);
    if (rc) return rc;
    if (!plan->symmetric) return kb_fail(KAPRE_E_UNSUPPORTED, "the resampling backward pass needs a symmetric filter");
    kapre_resample_plan* p = const_cast<kapre_resample_plan*>(plan);
    kapre_resample_plan* adj;
    {
        std::lock_guard<std::mutex> lk(p->adj_mu);
        if (!p->adj) {
            // A^T g = (up / down) resample(g; down, up): gain down of the exchanged plan times up / down
            rc = kb_resample_plan_build(p->down, p->up, p->taps_host.data(), p->n_taps, (double)p->up, &p->adj);
            if (rc) { p->adj = nullptr; return rc; }
        }
        adj = p->adj;
    }
    return kb_resample_launch(adj, g_dev, g_desc, gx_dev, gx_desc, stream);
}

}  // extern "C"

// ---- band-limited interpolation (sinc_core.cuh) ---------------------------------------------------
__global__ void __launch_bounds__(KB_SINC_THREADS, 2) kb_sinc_resample_kernel(const __grid_constant__ KbSincParams p) {
    extern __shared__ __align__(16) char kb_smem[];
    kb_sinc_cta(p, kb_smem, (int)blockIdx.x, (int)gridDim.x);
}

struct kapre_sinc_plan {
    DevInfo dev;
    KbTables tables;
    float2* tab = nullptr;      // KB_SINC_NTAB pairs (h, forward difference)
    double integral = 1.0;      // I
};

// Largest tile (outputs, a power of two <= 2048) whose staged span fits beside the table: in half of the opt-in
// shared memory when possible (less the 1 KB the system reserves per CTA and 1 KB of static shared memory), so that
// two CTAs share an SM, else in all of it.
static int kb_sinc_pick_nt(const kapre_sinc_plan* p, double step, int nw, int G) {
    for (int budget : {p->dev.smem_optin / 2 - 2048, p->dev.smem_optin - 1024})
        for (int nt = 2048; nt >= 1; nt /= 2)
            if (kb_sinc_smem(nt, step, nw, G) <= budget) return nt;
    return 0;
}

// One launch of y[m] = (gain / I) sum_j x[j] h(s (offset + m step - j)): the forward and the adjoint differ only in
// the four numbers kb_sinc_args makes.
static int kb_sinc_launch(const kapre_sinc_plan* plan, const float* x_dev, const kapre_wave_desc* xd, float* y_dev,
                          const kapre_wave_desc* yd, double ratio, double offset, int adjoint, void* stream) {
    if (!plan || !xd || !yd) return kb_fail(KAPRE_E_INVALID, "null argument");
    if (!(ratio >= KB_SINC_RATIO_MIN && ratio <= KB_SINC_RATIO_MAX))
        return kb_fail(KAPRE_E_INVALID, "ratio must lie in [%g, %g], got: %g", KB_SINC_RATIO_MIN, KB_SINC_RATIO_MAX, ratio);
    if (!(fabs(offset) <= 1099511627776.0)) return kb_fail(KAPRE_E_INVALID, "offset must be finite and at most 2^40 in size, got: %g", offset);
    if (xd->batch < 0 || xd->channels < 0 || xd->length < 0 || yd->length < 0) return kb_fail(KAPRE_E_INVALID, "negative size");
    if (yd->batch != xd->batch || yd->channels != xd->channels)
        return kb_fail(KAPRE_E_INVALID, "input and output descriptors disagree on batch / channels");
    if ((long long)yd->batch * yd->channels * yd->length == 0) return 0;
    if ((!x_dev && xd->length > 0) || !y_dev) return kb_fail(KAPRE_E_INVALID, "null data pointer");
    if ((const void*)x_dev == (const void*)y_dev) return kb_fail(KAPRE_E_INVALID, "interpolation cannot run in place");
    int rc = kb_check_device(plan->dev);
    if (rc) return rc;
    double step, off, s, gain;
    kb_sinc_args(ratio, offset, adjoint, &step, &off, &s, &gain);
    KbSincParams p{};
    const int B = xd->batch, C = xd->channels;
    p.x = x_dev; p.x_sb = xd->stride_b; p.x_sc = xd->stride_c; p.x_sl = xd->stride_l;
    p.B = B; p.C = C; p.L = xd->length;
    p.y = y_dev; p.y_sb = yd->stride_b; p.y_sc = yd->stride_c; p.y_sl = yd->stride_l;
    p.L_out = yd->length;
    p.tab = plan->tab;
    // channel-interleaved input: all channels in one tile
    const bool interleaved = C > 1 && C <= KB_SINC_THREADS && llabs(xd->stride_c) < llabs(xd->stride_l);
    p.G = interleaved ? C : 1;
    const bool nonneg = xd->stride_b >= 0 && xd->stride_c >= 0 && xd->stride_l >= 0;
    p.x_numel = (B > 0 && C > 0 && p.L > 0)
        ? (long long)(B - 1) * xd->stride_b + (long long)(C - 1) * xd->stride_c + (long long)(p.L - 1) * xd->stride_l + 1 : 0;
    p.x_align = (unsigned)(((uintptr_t)x_dev >> 2) & 3u);
    p.bulk_ok = nonneg && (((uintptr_t)x_dev & 3u) == 0) &&
                (p.G == 1 ? xd->stride_l == 1 : (xd->stride_c == 1 && xd->stride_l == C)) ? 1 : 0;
    const int nw = (int)ceil((double)KB_SINC_Z / s);
    p.NT = kb_sinc_pick_nt(plan, step, nw, p.G);
    if (p.NT == 0)
        return kb_fail(KAPRE_E_UNSUPPORTED, "%d interleaved channels at ratio %g do not fit in shared memory", p.G, ratio);
    if (!kb_sinc_setup(p, step, off, s, gain, plan->integral, KB_SINC_THREADS)) return kb_fail(KAPRE_E_UNSUPPORTED, "too many tiles");
    const int smem = kb_sinc_smem(p.NT, step, p.nw, p.G);
    int grid;
    if ((rc = kb_resident_grid(kb_sinc_resample_kernel, "sinc", KB_SINC_THREADS, smem, p.n_tiles, plan->dev.sm_count, &grid)))
        return rc;
    return kb_launch(kb_sinc_resample_kernel, {.grid = grid, .block = KB_SINC_THREADS, .smem = smem,
                                               .st = (cudaStream_t)stream, .timed = true}, p);
}

extern "C" {

int kapre_sinc_plan_create(kapre_sinc_plan** out) {
    if (!out) return kb_fail(KAPRE_E_INVALID, "null argument");
    kapre_sinc_plan* p = new kapre_sinc_plan();
    int rc = kb_dev_info(&p->dev);
    if (rc) { delete p; return rc; }
    if (kb_sinc_smem(1, 1.0 / KB_SINC_RATIO_MIN, (int)(KB_SINC_Z / KB_SINC_RATIO_MIN), 1) > p->dev.smem_optin) {
        delete p;
        return kb_fail(KAPRE_E_UNSUPPORTED, "the interpolation table (%d B) does not fit in shared memory", KB_SINC_NTAB * 8);
    }
    std::vector<float2> tab;
    kb_sinc_table(tab);
    p->integral = kb_sinc_integral();
    KbTableUpload tb;
    tb.add(tab, &p->tab);
    if ((rc = tb.upload(p->tables, "sinc"))) { delete p; return rc; }
    *out = p;
    return 0;
}

void kapre_sinc_plan_destroy(kapre_sinc_plan* p) { delete p; }

int kapre_sinc_resample(const kapre_sinc_plan* plan, const float* x_dev, const kapre_wave_desc* x_desc, float* y_dev,
                        const kapre_wave_desc* y_desc, double ratio, double offset, void* stream) {
    return kb_sinc_launch(plan, x_dev, x_desc, y_dev, y_desc, ratio, offset, 0, stream);
}

int kapre_sinc_resample_backward(const kapre_sinc_plan* plan, const float* g_dev, const kapre_wave_desc* g_desc,
                                 float* gx_dev, const kapre_wave_desc* gx_desc, double ratio, double offset, void* stream) {
    return kb_sinc_launch(plan, g_dev, g_desc, gx_dev, gx_desc, ratio, offset, 1, stream);
}

}  // extern "C"

// ---- partitioned FFT convolution (conv_core.cuh) ---------------------------------------------------------
__global__ void __launch_bounds__(KB_CONV_THREADS) kb_spec_conv_kernel(const __grid_constant__ KbConvParams p) {
    extern __shared__ __align__(16) char kb_smem[];
    kb_conv_cta(p, kb_smem, (int)blockIdx.x, (int)gridDim.x);
}

struct kapre_convolve_plan {
    int B;                              // block size: STFT at n_fft 2B, window ones(B), hop B
    DevInfo dev;
    kapre_stft_plan* stft = nullptr;
    kapre_istft_plan* istft = nullptr;  // n_fft = win_length = 2B, hop B, dual window ones(2B)
};

// Frames of a call: J = ceil(L / B) signal blocks, T = J + P - 1 output blocks, (T + 1) B untrimmed samples.
static int kb_conv_geom(const kapre_convolve_plan* plan, long long L, long long P, int* J, int* T, int* out_len) {
    if (L < 1) return kb_fail(KAPRE_E_INVALID, "signal length must be >= 1, got %lld", L);
    if (P < 1) return kb_fail(KAPRE_E_INVALID, "filter spectrum must have >= 1 block, got P=%lld", P);
    const long long j = (L + plan->B - 1) / plan->B, t = j + P - 1, n = (t + 1) * plan->B;
    if (n > 0x7fffffffLL)
        return kb_fail(KAPRE_E_INVALID, "%lld samples and %lld filter blocks of %d give %lld output samples, more than "
                       "int32 holds", L, P, plan->B, n);
    *J = (int)j; *T = (int)t; *out_len = (int)n;
    return 0;
}

// The forward workspace: the signal's spectra X, first because kapre_convolve_backward reads them at offset 0, then
// the output's spectra Y.
static void kb_conv_layout(KbLayout& L, int batch, int channels, int J, int T, int B, float2** X, float2** Y) {
    *X = L.take<float2>(batch, channels, J, B + 1);
    *Y = L.take<float2>(batch, channels, T, B + 1);
    L.pad();
}

// The backward workspace: the output gradient's spectra G, the signal gradient's spectra gX, and the STFT adjoint's
// overlap-add, which it needs only when the length is not a multiple of the block.
static void kb_conv_backward_layout(KbLayout& L, int batch, int channels, int length, int J, int T, int B, float2** G,
                                    float2** gX, float** ola) {
    *G = L.take<float2>(batch, channels, T, B + 1);
    *gX = L.take<float2>(batch, channels, J, B + 1);
    *ola = length % B ? L.take<float>(batch, channels, J, B) : nullptr;
    L.pad();
}

static kapre_spec_desc kb_conv_spec_desc(int C, int frames, int B) {
    const long long F = B + 1;
    return {(int64_t)C * frames * F, (int64_t)frames * F, F, 1};
}

// One launch of the per-bin multiply-accumulate over Bn x C sequences: To outputs from S a-frames and Tb b-frames.
static int kb_conv_mac(const kapre_convolve_plan* plan, const void* a, const kapre_spec_desc* ad, int S, const void* b,
                       const kapre_spec_desc* bd, int Tb, void* out, const kapre_spec_desc* od, int Bn, int C, int To,
                       int correlate, cudaStream_t st) {
    KbConvParams p{};
    p.a = (const float2*)a; p.a_sb = ad->stride_b; p.a_sc = ad->stride_c; p.a_st = ad->stride_t; p.a_sf = ad->stride_f;
    p.b = (const float2*)b; p.b_sb = bd->stride_b; p.b_sc = bd->stride_c; p.b_st = bd->stride_t; p.b_sf = bd->stride_f;
    p.out = (float2*)out; p.o_sb = od->stride_b; p.o_sc = od->stride_c; p.o_st = od->stride_t; p.o_sf = od->stride_f;
    p.Bn = Bn; p.C = C; p.F = plan->B + 1;
    p.S = S; p.Tb = Tb; p.To = To;
    p.correlate = correlate;
    if (!kb_conv_setup(p, KB_CONV_THREADS)) return kb_fail(KAPRE_E_UNSUPPORTED, "too many tiles");
    int grid, rc;
    if ((rc = kb_resident_grid(kb_spec_conv_kernel, "spec_conv", KB_CONV_THREADS, KB_CONV_SMEM, p.n_tiles, plan->dev.sm_count, &grid)))
        return rc;
    return kb_launch(kb_spec_conv_kernel, {.grid = grid, .block = KB_CONV_THREADS, .smem = KB_CONV_SMEM, .st = st,
                                           .timed = true}, p);
}

static int kb_conv_check_wave(const kapre_wave_desc* d, const char* what) {
    if (d->batch < 0 || d->channels < 0) return kb_fail(KAPRE_E_INVALID, "%s: negative size", what);
    return 0;
}

extern "C" {

int64_t kapre_convolve_block_size(int64_t ir_length) {
    if (ir_length < 1) return kb_fail(KAPRE_E_INVALID, "filter length must be >= 1, got %lld", (long long)ir_length);
    return kb_conv_block_size(ir_length);
}

int kapre_convolve_plan_create(int block, kapre_convolve_plan** out) {
    if (!out) return kb_fail(KAPRE_E_INVALID, "null argument");
    if (block != 128 && block != 256 && block != 512 && block != 1024)
        return kb_fail(KAPRE_E_INVALID, "block size must be 128, 256, 512 or 1024, got %d", block);
    kapre_convolve_plan* p = new kapre_convolve_plan();
    p->B = block;
    int rc = kb_dev_info(&p->dev);
    if (rc) { delete p; return rc; }
    const std::vector<float> ones(2 * block, 1.0f);
    if ((rc = kapre_stft_plan_create(2 * block, block, block, ones.data(), &p->stft)) ||
        (rc = kapre_istft_plan_create(2 * block, 2 * block, block, ones.data(), &p->istft))) {
        kapre_convolve_plan_destroy(p);
        return rc;
    }
    *out = p;
    return 0;
}

void kapre_convolve_plan_destroy(kapre_convolve_plan* p) {
    if (!p) return;
    kapre_stft_plan_destroy(p->stft);
    kapre_istft_plan_destroy(p->istft);
    delete p;
}

int kapre_convolve_ir_spectrum(const kapre_convolve_plan* plan, const float* h_dev, const kapre_wave_desc* h_desc,
                               void* H_dev, const kapre_spec_desc* H_desc, void* stream) {
    if (!plan || !h_desc || !H_desc) return kb_fail(KAPRE_E_INVALID, "null argument");
    if (h_desc->length < 1) return kb_fail(KAPRE_E_INVALID, "filter length must be >= 1, got %d", h_desc->length);
    int rc = kb_conv_check_wave(h_desc, "filter");
    if (rc) return rc;
    return kapre_stft_forward(plan->stft, h_dev, h_desc, 0, 1, KAPRE_OUT_COMPLEX, H_dev, H_desc, nullptr, nullptr,
                              nullptr, stream);
}

int64_t kapre_convolve_workspace_bytes(const kapre_convolve_plan* plan, int batch, int channels, int length, int P) {
    if (!plan) return kb_fail(KAPRE_E_INVALID, "null argument");
    if (batch < 0 || channels < 0) return kb_fail(KAPRE_E_INVALID, "negative size");
    int J, T, n, rc;
    if ((rc = kb_conv_geom(plan, length, P, &J, &T, &n))) return rc;
    KbLayout L;
    float2 *X, *Y;
    kb_conv_layout(L, batch, channels, J, T, plan->B, &X, &Y);
    return L.bytes("convolve");
}

int kapre_convolve(const kapre_convolve_plan* plan, const float* x_dev, const kapre_wave_desc* x_desc, const void* H_dev,
                   const kapre_spec_desc* H_desc, int P, float* y_dev, const kapre_wave_desc* y_desc, void* workspace_dev,
                   void* stream) {
    if (!plan || !x_desc || !H_desc || !y_desc) return kb_fail(KAPRE_E_INVALID, "null argument");
    int rc = kb_check_device(plan->dev);
    if (rc) return rc;
    if ((rc = kb_conv_check_wave(x_desc, "signal"))) return rc;
    int J, T, n;
    if ((rc = kb_conv_geom(plan, x_desc->length, P, &J, &T, &n))) return rc;
    if (y_desc->batch != x_desc->batch || y_desc->channels != x_desc->channels || y_desc->length != n)
        return kb_fail(KAPRE_E_INVALID, "output must be %d x %d x %d samples, got %d x %d x %d", x_desc->batch,
                       x_desc->channels, n, y_desc->batch, y_desc->channels, y_desc->length);
    const int Bn = x_desc->batch, C = x_desc->channels;
    if (Bn == 0 || C == 0) return 0;
    if (!x_dev || !H_dev || !y_dev || !workspace_dev) return kb_fail(KAPRE_E_INVALID, "null data pointer");
    KbLayout L{(char*)workspace_dev};
    float2 *X, *Y;
    kb_conv_layout(L, Bn, C, J, T, plan->B, &X, &Y);
    const kapre_spec_desc Xd = kb_conv_spec_desc(C, J, plan->B), Yd = kb_conv_spec_desc(C, T, plan->B);
    cudaStream_t st = (cudaStream_t)stream;
    if ((rc = kapre_stft_forward(plan->stft, x_dev, x_desc, 0, 1, KAPRE_OUT_COMPLEX, X, &Xd, nullptr, nullptr, nullptr,
                                 stream)))
        return rc;
    if ((rc = kb_conv_mac(plan, H_dev, H_desc, P, X, &Xd, J, Y, &Yd, Bn, C, T, 0, st))) return rc;
    // the launch report names the multiply-accumulate (the persistent launch) before the inverse STFT's
    const std::string mac = g_launch_info;
    if ((rc = kapre_istft_inverse(plan->istft, Y, Bn, C, T, &Yd, y_dev, y_desc, stream))) return rc;
    g_launch_info = mac + "; " + g_launch_info;
    return 0;
}

int64_t kapre_convolve_backward_workspace_bytes(const kapre_convolve_plan* plan, int batch, int channels, int length,
                                                int P) {
    if (!plan) return kb_fail(KAPRE_E_INVALID, "null argument");
    if (batch < 0 || channels < 0) return kb_fail(KAPRE_E_INVALID, "negative size");
    int J, T, n, rc;
    if ((rc = kb_conv_geom(plan, length, P, &J, &T, &n))) return rc;
    KbLayout L;
    float2 *G, *gX;
    float* ola;
    kb_conv_backward_layout(L, batch, channels, length, J, T, plan->B, &G, &gX, &ola);
    return L.bytes("convolve_backward");
}

int kapre_convolve_backward(const kapre_convolve_plan* plan, const float* gy_dev, const kapre_wave_desc* gy_desc,
                            const void* H_dev, const kapre_spec_desc* H_desc, const void* X_dev,
                            const kapre_spec_desc* X_desc, int P, float* gx_dev, const kapre_wave_desc* gx_desc,
                            void* gH_dev, const kapre_spec_desc* gH_desc, void* workspace_dev, void* stream) {
    if (!plan || !gy_desc || !gx_desc) return kb_fail(KAPRE_E_INVALID, "null argument");
    if (gx_dev && !H_desc) return kb_fail(KAPRE_E_INVALID, "the signal gradient needs H and its descriptor");
    if (gH_dev && (!X_desc || !gH_desc)) return kb_fail(KAPRE_E_INVALID, "the filter gradient needs X and gH descriptors");
    int rc = kb_check_device(plan->dev);
    if (rc) return rc;
    if ((rc = kb_conv_check_wave(gx_desc, "signal gradient"))) return rc;
    int J, T, n;
    if ((rc = kb_conv_geom(plan, gx_desc->length, P, &J, &T, &n))) return rc;
    if (gy_desc->batch != gx_desc->batch || gy_desc->channels != gx_desc->channels || gy_desc->length != n)
        return kb_fail(KAPRE_E_INVALID, "output gradient must be %d x %d x %d samples, got %d x %d x %d", gx_desc->batch,
                       gx_desc->channels, n, gy_desc->batch, gy_desc->channels, gy_desc->length);
    const int Bn = gx_desc->batch, C = gx_desc->channels;
    if (Bn == 0 || C == 0 || (!gx_dev && !gH_dev)) return 0;
    if (!gy_dev || !workspace_dev || (gx_dev && !H_dev) || (gH_dev && !X_dev))
        return kb_fail(KAPRE_E_INVALID, "null data pointer");
    KbLayout L{(char*)workspace_dev};
    float2 *G, *gX;
    float* ola;
    kb_conv_backward_layout(L, Bn, C, gx_desc->length, J, T, plan->B, &G, &gX, &ola);
    const kapre_spec_desc Gd = kb_conv_spec_desc(C, T, plan->B), gXd = kb_conv_spec_desc(C, J, plan->B);
    cudaStream_t st = (cudaStream_t)stream;
    if ((rc = kapre_istft_backward(plan->istft, gy_dev, gy_desc, Bn, C, T, G, &Gd, stream))) return rc;
    std::string macs;   // the launch report: the multiply-accumulates, signal gradient's first
    if (gx_dev) {
        if ((rc = kb_conv_mac(plan, H_dev, H_desc, P, G, &Gd, T, gX, &gXd, Bn, C, J, 1, st))) return rc;
        macs = g_launch_info;
        if ((rc = kapre_stft_backward(plan->stft, gX, &gXd, Bn, C, J, 0, 1, gx_dev, gx_desc, ola, stream))) return rc;
    }
    if (gH_dev) {
        if ((rc = kb_conv_mac(plan, X_dev, X_desc, J, G, &Gd, T, gH_dev, gH_desc, Bn, C, P, 1, st))) return rc;
        macs += (macs.empty() ? "" : "; ") + g_launch_info;
    }
    g_launch_info = macs;
    return 0;
}

int kapre_convolve_ir_spectrum_backward(const kapre_convolve_plan* plan, const void* gH_dev, const kapre_spec_desc* gH_desc,
                                        int P, float* gh_dev, const kapre_wave_desc* gh_desc, void* workspace_dev,
                                        void* stream) {
    if (!plan || !gH_desc || !gh_desc) return kb_fail(KAPRE_E_INVALID, "null argument");
    if (gh_desc->length < 1) return kb_fail(KAPRE_E_INVALID, "filter length must be >= 1, got %d", gh_desc->length);
    int rc = kb_conv_check_wave(gh_desc, "filter gradient");
    if (rc) return rc;
    if ((gh_desc->length + (long long)plan->B - 1) / plan->B != P)
        return kb_fail(KAPRE_E_INVALID, "a filter of %d taps has %d blocks of %d, got P=%d", gh_desc->length,
                       (gh_desc->length + plan->B - 1) / plan->B, plan->B, P);
    return kapre_stft_backward(plan->stft, gH_dev, gH_desc, gh_desc->batch, gh_desc->channels, P, 0, 1, gh_dev, gh_desc,
                               workspace_dev, stream);
}

}  // extern "C"

// ---- per-channel energy normalisation (pcen_core.cuh) ------------------------------------------------
__global__ void __launch_bounds__(KB_PCEN_THREADS) kb_pcen_state_kernel(const __grid_constant__ KbPcenParams p, long long n) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) kb_pcen_fwd_state(p, i);
}
__global__ void __launch_bounds__(KB_PCEN_THREADS) kb_pcen_kernel(const __grid_constant__ KbPcenParams p, long long n) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) kb_pcen_fwd_out(p, i);
}
__global__ void __launch_bounds__(KB_PCEN_THREADS) kb_pcen_bwd_state_kernel(const __grid_constant__ KbPcenParams p, long long n) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) kb_pcen_bwd_state(p, i);
}
__global__ void __launch_bounds__(KB_PCEN_THREADS) kb_pcen_bwd_kernel(const __grid_constant__ KbPcenParams p, long long n) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) kb_pcen_bwd_out(p, i);
}

// Chunking of n_cols columns of `frames` frames against the current device's resident-thread capacity.
static int kb_pcen_pick_chunks(long long n_cols, int frames, int* chunks) {
    long long threads = 0;
    int rc = kb_resident_threads(&threads);
    if (rc) return rc;
    *chunks = kb_pcen_chunks(n_cols, frames, threads);
    return 0;
}

static int kb_pcen_setup(KbPcenParams& p, const kapre_spec_desc* E_desc, int batch, int channels, int frames, int bands,
                         const kapre_pcen_params* prm) {
    if (!E_desc || !prm) return kb_fail(KAPRE_E_INVALID, "null argument");
    if (batch < 0 || channels < 0 || frames < 0 || bands < 0) return kb_fail(KAPRE_E_INVALID, "negative size");
    if (!prm->gain || !prm->bias || !prm->power || !prm->smooth) return kb_fail(KAPRE_E_INVALID, "null parameter pointer");
    for (int st : {prm->gain_stride, prm->bias_stride, prm->power_stride, prm->smooth_stride})
        if (st != 0 && st != 1) return kb_fail(KAPRE_E_INVALID, "parameter strides must be 0 (shared) or 1 (per band), got %d", st);
    if (!(prm->eps > 0.0f)) return kb_fail(KAPRE_E_INVALID, "eps must be positive, got %g", prm->eps);
    p.B = batch; p.C = channels; p.T = frames; p.F = bands;
    p.n_cols = (long long)batch * channels * bands;
    p.E = nullptr;
    p.e_sb = E_desc->stride_b; p.e_sc = E_desc->stride_c; p.e_st = E_desc->stride_t; p.e_sf = E_desc->stride_f;
    p.c_inner = channels > 1 && llabs(E_desc->stride_c) < llabs(E_desc->stride_f) ? 1 : 0;
    p.gain = prm->gain; p.bias = prm->bias; p.power = prm->power; p.smooth = prm->smooth;
    p.gain_st = prm->gain_stride; p.bias_st = prm->bias_stride; p.power_st = prm->power_stride;
    p.smooth_st = prm->smooth_stride;
    p.eps = prm->eps;
    int K = 1, rc;
    if (p.n_cols * frames > 0 && (rc = kb_pcen_pick_chunks(p.n_cols, frames, &K))) return rc;
    kb_pcen_set_chunks(p, K);
    return 0;
}

// the workspace of a chunked scan: the (K, n_cols) chunk end states
static void kb_pcen_layout(KbLayout& L, KbPcenParams& p) { p.state = p.K > 1 ? L.take<float>(p.K, p.n_cols) : nullptr; }

extern "C" {

int kapre_pcen_workspace(int batch, int channels, int frames, int bands, int* chunks, int64_t* workspace_bytes) {
    if (!chunks || !workspace_bytes) return kb_fail(KAPRE_E_INVALID, "null argument");
    if (batch < 0 || channels < 0 || frames < 0 || bands < 0) return kb_fail(KAPRE_E_INVALID, "negative size");
    KbPcenParams p{};
    p.T = frames;
    p.n_cols = (long long)batch * channels * bands;
    int K = 1, rc;
    if (p.n_cols * frames > 0 && (rc = kb_pcen_pick_chunks(p.n_cols, frames, &K))) return rc;
    kb_pcen_set_chunks(p, K);
    KbLayout L;
    kb_pcen_layout(L, p);
    if ((*workspace_bytes = L.bytes("pcen")) < 0) return (int)*workspace_bytes;
    *chunks = p.K;
    return 0;
}

int kapre_pcen(const float* E_dev, const kapre_spec_desc* E_desc, int batch, int channels, int frames, int bands,
               const kapre_pcen_params* params, float* y_dev, const kapre_spec_desc* y_desc, float* M_dev,
               const kapre_spec_desc* M_desc, void* workspace_dev, void* stream) {
    KbPcenParams p{};
    int rc = kb_pcen_setup(p, E_desc, batch, channels, frames, bands, params);
    if (rc) return rc;
    if (!y_desc || (M_dev && !M_desc)) return kb_fail(KAPRE_E_INVALID, "null argument");
    if (p.n_cols * frames == 0) return 0;
    if (!E_dev || !y_dev) return kb_fail(KAPRE_E_INVALID, "null data pointer");
    if ((const void*)E_dev == (const void*)y_dev || (const void*)E_dev == (const void*)M_dev)
        return kb_fail(KAPRE_E_INVALID, "PCEN cannot run in place");
    if (p.K > 1 && !workspace_dev) return kb_fail(KAPRE_E_INVALID, "PCEN over %d time chunks needs a workspace", p.K);
    p.E = E_dev;
    p.y = y_dev; p.y_sb = y_desc->stride_b; p.y_sc = y_desc->stride_c; p.y_st = y_desc->stride_t; p.y_sf = y_desc->stride_f;
    p.M = M_dev;
    if (M_dev) { p.m_sb = M_desc->stride_b; p.m_sc = M_desc->stride_c; p.m_st = M_desc->stride_t; p.m_sf = M_desc->stride_f; }
    KbLayout L{(char*)workspace_dev};
    kb_pcen_layout(L, p);
    // one thread per (chunk, column): the state pass covers chunks 0 .. K - 2, the output pass all K
    const long long ns = (long long)(p.K - 1) * p.n_cols, n = ns + p.n_cols;
    const long long grid = (n + KB_PCEN_THREADS - 1) / KB_PCEN_THREADS;
    if (grid > 0x7fffffffLL) return kb_fail(KAPRE_E_UNSUPPORTED, "too many PCEN columns");
    const KbLaunch l{.grid = (int)grid, .block = KB_PCEN_THREADS, .st = (cudaStream_t)stream, .timed = true};
    if (p.K > 1 && (rc = kb_launch(kb_pcen_state_kernel, {.grid = (int)((ns + KB_PCEN_THREADS - 1) / KB_PCEN_THREADS),
                                                          .block = KB_PCEN_THREADS, .st = l.st, .timed = true}, p, ns)))
        return rc;
    return kb_launch(kb_pcen_kernel, l, p, n);
}

int kapre_pcen_backward(const float* E_dev, const kapre_spec_desc* E_desc, const float* M_dev,
                        const kapre_spec_desc* M_desc, const float* gy_dev, const kapre_spec_desc* gy_desc, int batch,
                        int channels, int frames, int bands, const kapre_pcen_params* params, float* gE_dev,
                        const kapre_spec_desc* gE_desc, float* param_partials_dev, void* workspace_dev, void* stream) {
    KbPcenParams p{};
    int rc = kb_pcen_setup(p, E_desc, batch, channels, frames, bands, params);
    if (rc) return rc;
    if (!M_desc || !gy_desc || !gE_desc) return kb_fail(KAPRE_E_INVALID, "null argument");
    if (p.n_cols == 0) return 0;
    if (!param_partials_dev) return kb_fail(KAPRE_E_INVALID, "null data pointer");
    if (frames == 0) {
        KB_CUDA(cudaMemsetAsync(param_partials_dev, 0, (size_t)4 * p.n_cols * sizeof(float), (cudaStream_t)stream));
        return 0;
    }
    if (!E_dev || !M_dev || !gy_dev || !gE_dev) return kb_fail(KAPRE_E_INVALID, "null data pointer");
    if ((const void*)gE_dev == (const void*)E_dev || (const void*)gE_dev == (const void*)M_dev ||
        (const void*)gE_dev == (const void*)gy_dev)
        return kb_fail(KAPRE_E_INVALID, "PCEN backward cannot run in place");
    if (p.K > 1 && !workspace_dev) return kb_fail(KAPRE_E_INVALID, "PCEN over %d time chunks needs a workspace", p.K);
    p.E = E_dev;
    p.M = const_cast<float*>(M_dev);
    p.m_sb = M_desc->stride_b; p.m_sc = M_desc->stride_c; p.m_st = M_desc->stride_t; p.m_sf = M_desc->stride_f;
    p.gy = gy_dev; p.g_sb = gy_desc->stride_b; p.g_sc = gy_desc->stride_c; p.g_st = gy_desc->stride_t; p.g_sf = gy_desc->stride_f;
    p.gE = gE_dev; p.o_sb = gE_desc->stride_b; p.o_sc = gE_desc->stride_c; p.o_st = gE_desc->stride_t; p.o_sf = gE_desc->stride_f;
    KbLayout L{(char*)workspace_dev};
    kb_pcen_layout(L, p);
    p.part = param_partials_dev;
    const long long ns = (long long)(p.K - 1) * p.n_cols, n = ns + p.n_cols;
    const long long grid = (n + KB_PCEN_THREADS - 1) / KB_PCEN_THREADS;
    if (grid > 0x7fffffffLL) return kb_fail(KAPRE_E_UNSUPPORTED, "too many PCEN columns");
    const KbLaunch l{.grid = (int)grid, .block = KB_PCEN_THREADS, .st = (cudaStream_t)stream, .timed = true};
    if (p.K > 1 && (rc = kb_launch(kb_pcen_bwd_state_kernel, {.grid = (int)((ns + KB_PCEN_THREADS - 1) / KB_PCEN_THREADS),
                                                              .block = KB_PCEN_THREADS, .st = l.st, .timed = true}, p, ns)))
        return rc;
    return kb_launch(kb_pcen_bwd_kernel, l, p, n);
}

}  // extern "C"

// ---- Griffin-Lim (gl_core.cuh) -------------------------------------------------------------------------
__global__ void __launch_bounds__(KB_GL_THREADS) kb_gl_init_kernel(const __grid_constant__ KbGlParams p) {
    const long long step = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < p.n; i += step) kb_gl_init_elem(p, i);
}
__global__ void __launch_bounds__(KB_GL_THREADS) kb_gl_project_kernel(const __grid_constant__ KbGlParams p) {
    const long long step = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < p.n; i += step) kb_gl_project_elem(p, i);
}

// Workspace: spectrum buffers 0 and 1 (each (B, C, frames, F) complex64), then the (B, C, len) waveform.
static void kb_gl_layout(KbLayout& L, int batch, int channels, int frames, int F, long long len, float2** X, float** wave) {
    X[0] = L.take<float2>(batch, channels, frames, F);
    X[1] = L.take<float2>(batch, channels, frames, F);
    *wave = L.take<float>(batch, channels, len);
}

extern "C" {

int64_t kapre_griffin_lim_workspace_bytes(const kapre_stft_plan* plan, int batch, int channels, int frames) {
    if (!plan) return kb_fail(KAPRE_E_INVALID, "null argument");
    if (batch < 0 || channels < 0 || frames < 0) return kb_fail(KAPRE_E_INVALID, "negative size");
    const long long len = frames > 0 ? (long long)(frames - 1) * plan->hop + plan->win_length : 0;
    KbLayout L;
    float2* X[2];
    float* wave;
    kb_gl_layout(L, batch, channels, frames, plan->n_fft / 2 + 1, len, X, &wave);
    return L.bytes("griffin_lim");
}

int kapre_griffin_lim(const kapre_stft_plan* stft, const kapre_istft_plan* istft, const float* S_dev,
                      const kapre_spec_desc* S_desc, int batch, int channels, int frames,
                      const kapre_griffin_lim_cfg* cfg, float* y_dev, const kapre_wave_desc* y_desc,
                      void* workspace_dev, void* stream) {
    if (!stft || !istft || !S_desc || !cfg || !y_desc) return kb_fail(KAPRE_E_INVALID, "null argument");
    if (stft->n_fft != istft->n_fft || stft->win_length != istft->win_length || stft->hop != istft->hop)
        return kb_fail(KAPRE_E_INVALID, "STFT plan (n_fft=%d win_length=%d hop=%d) and inverse plan (n_fft=%d win_length=%d "
                       "hop=%d) disagree", stft->n_fft, stft->win_length, stft->hop, istft->n_fft, istft->win_length, istft->hop);
    if (stft->dev.device != istft->dev.device)
        return kb_fail(KAPRE_E_INVALID, "STFT plan lives on device %d, inverse plan on device %d", stft->dev.device,
                       istft->dev.device);
    int rc = kb_check_device(stft->dev);
    if (rc) return rc;
    if (cfg->n_iter < 0) return kb_fail(KAPRE_E_INVALID, "n_iter must be >= 0, got %d", cfg->n_iter);
    if (!(cfg->momentum >= 0.0f && cfg->momentum < 1.0f))
        return kb_fail(KAPRE_E_INVALID, "momentum must be in [0, 1), got %g", cfg->momentum);
    if (cfg->init != KAPRE_GL_INIT_ONES && cfg->init != KAPRE_GL_INIT_RANDOM)
        return kb_fail(KAPRE_E_INVALID, "init must be KAPRE_GL_INIT_ONES or KAPRE_GL_INIT_RANDOM, got %d", cfg->init);
    if (batch < 0 || channels < 0 || frames < 0) return kb_fail(KAPRE_E_INVALID, "negative size");
    const long long L = frames > 0 ? (long long)(frames - 1) * stft->hop + stft->win_length : 0;
    if (L > 0x7fffffffLL) return kb_fail(KAPRE_E_UNSUPPORTED, "signal too long");
    if (y_desc->batch != batch || y_desc->channels != channels || y_desc->length != (int)L)
        return kb_fail(KAPRE_E_INVALID, "output must be %d x %d x %lld samples, got %d x %d x %d", batch, channels, L,
                       y_desc->batch, y_desc->channels, y_desc->length);
    if (batch == 0 || channels == 0 || frames == 0) return 0;
    if (!S_dev || !y_dev || !workspace_dev) return kb_fail(KAPRE_E_INVALID, "null data pointer");

    const int F = stft->n_fft / 2 + 1;
    KbGlParams p{};
    p.S = S_dev; p.s_sb = S_desc->stride_b; p.s_sc = S_desc->stride_c; p.s_st = S_desc->stride_t; p.s_sf = S_desc->stride_f;
    p.C = channels; p.T = frames; p.F = F;
    p.n = (long long)batch * channels * frames * F;
    p.beta = cfg->momentum / (1.0f + cfg->momentum);
    p.init = cfg->init;
    p.seed = (unsigned long long)cfg->seed;
    KbLayout ws{(char*)workspace_dev};
    float2* X[2];
    float* wave;
    kb_gl_layout(ws, batch, channels, frames, F, L, X, &wave);
    const kapre_spec_desc sd = {(int64_t)channels * frames * F, (int64_t)frames * F, F, 1};
    const kapre_wave_desc wd = {batch, channels, (int32_t)L, (int64_t)channels * L, L, 1};
    int grid;
    if ((rc = kb_ew_grid(p.n, &grid))) return rc;
    const KbLaunch l{.grid = grid, .block = KB_GL_THREADS, .st = (cudaStream_t)stream};

    p.X = X[0];
    if ((rc = kb_launch(kb_gl_init_kernel, l, p))) return rc;
    int cur = 0;
    for (int it = 0; it < cfg->n_iter; ++it) {
        // X (buffer cur) -> waveform -> Y over X in buffer cur; the new X goes over Yprev in the other buffer
        if ((rc = kapre_istft_inverse(istft, X[cur], batch, channels, frames, &sd, wave, &wd, stream))) return rc;
        if ((rc = kapre_stft_forward(stft, wave, &wd, 0, 0, KAPRE_OUT_COMPLEX, X[cur], &sd, nullptr, nullptr, nullptr,
                                     stream)))
            return rc;
        p.Y = X[cur];
        p.Yprev = (it > 0 && p.beta != 0.0f) ? X[1 - cur] : nullptr;
        p.X = X[1 - cur];
        if ((rc = kb_launch(kb_gl_project_kernel, l, p))) return rc;
        cur = 1 - cur;
    }
    return kapre_istft_inverse(istft, X[cur], batch, channels, frames, &sd, y_dev, y_desc, stream);
}

}  // extern "C"

// ---- phase-vocoder time stretch (ts_core.cuh) ----------------------------------------------------------
__global__ void __launch_bounds__(KB_TS_THREADS) kb_ts_state_kernel(const __grid_constant__ KbTsParams p, long long n) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) kb_ts_fwd<false>(p, i);
}
__global__ void __launch_bounds__(KB_TS_THREADS) kb_ts_kernel(const __grid_constant__ KbTsParams p, long long n) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) kb_ts_fwd<true>(p, i);
}
__global__ void __launch_bounds__(KB_TS_THREADS) kb_ts_bwd_state_kernel(const __grid_constant__ KbTsParams p, long long n) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) kb_ts_bwd_state(p, i);
}
__global__ void __launch_bounds__(KB_TS_THREADS) kb_ts_bwd_kernel(const __grid_constant__ KbTsParams p, long long n) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) kb_ts_bwd_out(p, i);
}

// Output frames of a time stretch, ceil(frames / rate) as torch.arange counts them; negative on a bad argument.
static long long kb_ts_out_frames(int frames, double rate) {
    if (!std::isfinite(rate) || !(rate > 0.0)) return kb_fail(KAPRE_E_INVALID, "rate must be finite and positive, got %g", rate);
    if (frames < 0) return kb_fail(KAPRE_E_INVALID, "negative size");
    const double n = std::ceil((double)frames / rate);
    if (!(n <= 2147483647.0))
        return kb_fail(KAPRE_E_INVALID, "%d frames at rate %g give %.0f output frames, more than 2^31 - 1", frames, rate, n);
    return (long long)n;
}

static int kb_ts_setup(KbTsParams& p, const kapre_spec_desc* X_desc, int batch, int channels, int frames, int bins,
                       double rate) {
    if (!X_desc) return kb_fail(KAPRE_E_INVALID, "null argument");
    if (batch < 0 || channels < 0 || frames < 0 || bins < 0) return kb_fail(KAPRE_E_INVALID, "negative size");
    const long long n_out = kb_ts_out_frames(frames, rate);
    if (n_out < 0) return (int)n_out;
    p.B = batch; p.C = channels; p.T = frames; p.F = bins; p.T_out = (int)n_out;
    p.rate = rate;
    p.inv_rate = 1.0 / rate;
    p.n_cols = (long long)batch * channels * bins;
    p.x_sb = X_desc->stride_b; p.x_sc = X_desc->stride_c; p.x_st = X_desc->stride_t; p.x_sf = X_desc->stride_f;
    p.c_inner = channels > 1 && llabs(X_desc->stride_c) < llabs(X_desc->stride_f) ? 1 : 0;
    int K = 1;
    if (p.n_cols * frames > 0) {
        long long threads = 0;
        int rc = kb_resident_threads(&threads);
        if (rc) return rc;
        K = kb_ts_chunks(p.n_cols, frames, threads);
    }
    kb_ts_set_chunks(p, K);
    return 0;
}

// Byte range [lo, hi) of a (batch, channels, frames, bins) complex64 tensor with these element strides.
static void kb_ts_span(const void* base, const kapre_spec_desc* d, int B, int C, int T, int F, uintptr_t* lo, uintptr_t* hi) {
    long long a = 0, b = 0;
    const long long n[4] = {B, C, T, F}, s[4] = {d->stride_b, d->stride_c, d->stride_t, d->stride_f};
    for (int j = 0; j < 4; ++j) {
        const long long e = (n[j] - 1) * s[j];
        if (e < 0) a += e; else b += e;
    }
    *lo = (uintptr_t)base + (uintptr_t)(a * 8);
    *hi = (uintptr_t)base + (uintptr_t)(b * 8 + 8);
}

static bool kb_ts_overlap(const void* p, const kapre_spec_desc* pd, int pt, const void* q, const kapre_spec_desc* qd, int qt,
                          int B, int C, int F) {
    uintptr_t a0, a1, b0, b1;
    kb_ts_span(p, pd, B, C, pt, F, &a0, &a1);
    kb_ts_span(q, qd, B, C, qt, F, &b0, &b1);
    return a0 < b1 && b0 < a1;
}

// the workspace of a chunked scan: the (K, n_cols) chunk sums
static void kb_ts_layout(KbLayout& L, KbTsParams& p) { p.state = p.K > 1 ? L.take<float>(p.K, p.n_cols) : nullptr; }

extern "C" {

int kapre_time_stretch_workspace(int batch, int channels, int frames, int bins, double rate, int* chunks,
                                 int64_t* workspace_bytes) {
    if (!chunks || !workspace_bytes) return kb_fail(KAPRE_E_INVALID, "null argument");
    const kapre_spec_desc d = {0, 0, 0, 0};
    KbTsParams p{};
    int rc = kb_ts_setup(p, &d, batch, channels, frames, bins, rate);
    if (rc) return rc;
    KbLayout L;
    kb_ts_layout(L, p);
    if ((*workspace_bytes = L.bytes("time_stretch")) < 0) return (int)*workspace_bytes;
    *chunks = p.K;
    return 0;
}

int kapre_time_stretch(const void* X_dev, const kapre_spec_desc* X_desc, int batch, int channels, int frames, int bins,
                       double rate, void* Y_dev, const kapre_spec_desc* Y_desc, void* workspace_dev, void* stream) {
    KbTsParams p{};
    int rc = kb_ts_setup(p, X_desc, batch, channels, frames, bins, rate);
    if (rc) return rc;
    if (!Y_desc) return kb_fail(KAPRE_E_INVALID, "null argument");
    if (p.n_cols * p.T_out == 0) return 0;
    if (!X_dev || !Y_dev) return kb_fail(KAPRE_E_INVALID, "null data pointer");
    if (kb_ts_overlap(X_dev, X_desc, frames, Y_dev, Y_desc, p.T_out, batch, channels, bins))
        return kb_fail(KAPRE_E_INVALID, "the time-stretch output overlaps its input");
    if (p.K > 1 && !workspace_dev)
        return kb_fail(KAPRE_E_INVALID, "a time stretch over %d time chunks needs a workspace", p.K);
    p.X = (const float2*)X_dev;
    p.Y = (float2*)Y_dev; p.y_sb = Y_desc->stride_b; p.y_sc = Y_desc->stride_c; p.y_st = Y_desc->stride_t; p.y_sf = Y_desc->stride_f;
    KbLayout L{(char*)workspace_dev};
    kb_ts_layout(L, p);
    // one thread per (chunk, column): the state pass covers chunks 0 .. K - 2, the output pass all K
    const long long ns = (long long)(p.K - 1) * p.n_cols, n = ns + p.n_cols;
    if (n > 0xffffffffLL) return kb_fail(KAPRE_E_UNSUPPORTED, "too many time-stretch columns");
    const cudaStream_t st = (cudaStream_t)stream;
    if (p.K > 1 && (rc = kb_launch(kb_ts_state_kernel, {.grid = (int)((ns + KB_TS_THREADS - 1) / KB_TS_THREADS),
                                                        .block = KB_TS_THREADS, .st = st, .timed = true}, p, ns)))
        return rc;
    return kb_launch(kb_ts_kernel, {.grid = (int)((n + KB_TS_THREADS - 1) / KB_TS_THREADS), .block = KB_TS_THREADS,
                                    .st = st, .timed = true}, p, n);
}

int kapre_time_stretch_backward(const void* X_dev, const kapre_spec_desc* X_desc, const void* Y_dev,
                                const kapre_spec_desc* Y_desc, const void* G_dev, const kapre_spec_desc* G_desc,
                                int batch, int channels, int frames, int bins, double rate, void* gX_dev,
                                const kapre_spec_desc* gX_desc, void* workspace_dev, void* stream) {
    KbTsParams p{};
    int rc = kb_ts_setup(p, X_desc, batch, channels, frames, bins, rate);
    if (rc) return rc;
    if (!Y_desc || !G_desc || !gX_desc) return kb_fail(KAPRE_E_INVALID, "null argument");
    if (p.n_cols * frames == 0) return 0;
    if (!X_dev || !Y_dev || !G_dev || !gX_dev) return kb_fail(KAPRE_E_INVALID, "null data pointer");
    if (kb_ts_overlap(gX_dev, gX_desc, frames, X_dev, X_desc, frames, batch, channels, bins) ||
        kb_ts_overlap(gX_dev, gX_desc, frames, Y_dev, Y_desc, p.T_out, batch, channels, bins) ||
        kb_ts_overlap(gX_dev, gX_desc, frames, G_dev, G_desc, p.T_out, batch, channels, bins))
        return kb_fail(KAPRE_E_INVALID, "the time-stretch input gradient overlaps X, Y or the output gradient");
    if (p.K > 1 && !workspace_dev)
        return kb_fail(KAPRE_E_INVALID, "a time stretch over %d time chunks needs a workspace", p.K);
    p.X = (const float2*)X_dev;
    p.Y = (float2*)const_cast<void*>(Y_dev);
    p.y_sb = Y_desc->stride_b; p.y_sc = Y_desc->stride_c; p.y_st = Y_desc->stride_t; p.y_sf = Y_desc->stride_f;
    p.G = (const float2*)G_dev;
    p.g_sb = G_desc->stride_b; p.g_sc = G_desc->stride_c; p.g_st = G_desc->stride_t; p.g_sf = G_desc->stride_f;
    p.gX = (float2*)gX_dev;
    p.o_sb = gX_desc->stride_b; p.o_sc = gX_desc->stride_c; p.o_st = gX_desc->stride_t; p.o_sf = gX_desc->stride_f;
    KbLayout L{(char*)workspace_dev};
    kb_ts_layout(L, p);
    const long long ns = (long long)(p.K - 1) * p.n_cols, n = ns + p.n_cols;
    if (n > 0xffffffffLL) return kb_fail(KAPRE_E_UNSUPPORTED, "too many time-stretch columns");
    const cudaStream_t st = (cudaStream_t)stream;
    if (p.K > 1 && (rc = kb_launch(kb_ts_bwd_state_kernel, {.grid = (int)((ns + KB_TS_THREADS - 1) / KB_TS_THREADS),
                                                            .block = KB_TS_THREADS, .st = st, .timed = true}, p, ns)))
        return rc;
    return kb_launch(kb_ts_bwd_kernel, {.grid = (int)((n + KB_TS_THREADS - 1) / KB_TS_THREADS), .block = KB_TS_THREADS,
                                        .st = st, .timed = true}, p, n);
}

}  // extern "C"

// ---- filterbank inversion (fbinv_core.cuh) ----------------------------------------------------------------------
__global__ void __launch_bounds__(KB_FBI_WARPS * 32, 1) kb_fbi_kernel(const __grid_constant__ KbFbiParams p) {
    extern __shared__ __align__(16) char kb_smem[];
    kb_fbi_cta(p, kb_smem, (int)blockIdx.x, (int)gridDim.x);
}

struct kapre_fb_inverse_plan {
    int n_freq, n_bands;
    DevInfo dev;
    KbTables tables;
    float step = 0.0f;
    KbBand* bands = nullptr;
    float* w = nullptr;
    int* cptr = nullptr;
    KbFbiCol* cols = nullptr;
    float* inv_d = nullptr;
};

extern "C" {

int kapre_fb_inverse_plan_create(const float* fb_host, int n_freq, int n_bands, kapre_fb_inverse_plan** out) {
    if (!out || !fb_host) return kb_fail(KAPRE_E_INVALID, "null argument");
    if (n_freq < 1 || n_bands < 1) return kb_fail(KAPRE_E_INVALID, "empty filterbank");
    kapre_fb_inverse_plan* f = new kapre_fb_inverse_plan();
    f->n_freq = n_freq; f->n_bands = n_bands;
    int rc = kb_dev_info(&f->dev);
    if (rc) { delete f; return rc; }
    KbFbiTables t;
    kb_fbi_make_tables(fb_host, n_freq, n_bands, t);
    f->step = t.step;
    KbTableUpload tb;
    tb.add(t.bands, &f->bands); tb.add(t.w, &f->w); tb.add(t.cptr, &f->cptr); tb.add(t.cols, &f->cols);
    tb.add(t.inv_d, &f->inv_d);
    if ((rc = tb.upload(f->tables, "fb_inverse"))) { delete f; return rc; }
    *out = f;
    return 0;
}

void kapre_fb_inverse_plan_destroy(kapre_fb_inverse_plan* f) { delete f; }

int kapre_filterbank_invert(const kapre_fb_inverse_plan* plan, const kapre_fb_inverse_cfg* cfg, const float* x_dev,
                            int batch, int channels, int frames, const kapre_spec_desc* x_desc, float* out_dev,
                            const kapre_spec_desc* out_desc, void* stream) {
    if (!plan || !cfg || !x_desc || !out_desc) return kb_fail(KAPRE_E_INVALID, "null argument");
    int rc = kb_check_device(plan->dev);
    if (rc) return rc;
    if (cfg->n_iter < 0) return kb_fail(KAPRE_E_INVALID, "n_iter must be >= 0, got %d", cfg->n_iter);
    if (cfg->from_decibel != 0 && cfg->from_decibel != 1)
        return kb_fail(KAPRE_E_INVALID, "from_decibel must be 0 or 1, got %d", cfg->from_decibel);
    if (cfg->from_decibel && !(cfg->ref_value > 0.0f && cfg->ref_value <= 3.402823466e38f))
        return kb_fail(KAPRE_E_INVALID, "ref_value must be positive and finite, got %g", cfg->ref_value);
    if (cfg->from_decibel && !(cfg->amin > 0.0f && cfg->amin <= 3.402823466e38f))
        return kb_fail(KAPRE_E_INVALID, "amin must be positive and finite, got %g", cfg->amin);
    if (batch < 0 || channels < 0 || frames < 0) return kb_fail(KAPRE_E_INVALID, "negative size");
    if (batch == 0 || channels == 0 || frames == 0) return 0;
    if (!x_dev || !out_dev) return kb_fail(KAPRE_E_INVALID, "null data pointer");
    KbFbiParams p{};
    p.x = x_dev; p.x_sb = x_desc->stride_b; p.x_sc = x_desc->stride_c; p.x_st = x_desc->stride_t; p.x_sk = x_desc->stride_f;
    p.B = batch; p.C = channels; p.T = frames; p.F = plan->n_freq; p.M = plan->n_bands;
    p.bands = plan->bands; p.fbw = plan->w; p.cptr = plan->cptr; p.cols = plan->cols; p.inv_d = plan->inv_d;
    p.step = plan->step;
    p.n_iter = cfg->n_iter;
    p.from_db = cfg->from_decibel;
    p.db_scale = cfg->amin > cfg->ref_value ? (double)cfg->amin : (double)cfg->ref_value;
    p.out = out_dev; p.o_sb = out_desc->stride_b; p.o_sc = out_desc->stride_c; p.o_st = out_desc->stride_t;
    p.o_sk = out_desc->stride_f;
    p.R = kb_fbi_pick_r(plan->n_freq, plan->n_bands, plan->dev.smem_optin);
    if (p.R == 0)
        return kb_fail(KAPRE_E_UNSUPPORTED, "filterbank inversion: one frame of a %dx%d filterbank does not fit shared memory",
                       plan->n_freq, plan->n_bands);
    p.n_tiles_t = (frames + p.R - 1) / p.R;
    p.n_warps = KB_FBI_WARPS;
    const long long tiles = (long long)batch * channels * p.n_tiles_t;
    if (tiles > 0x7fffffffLL) return kb_fail(KAPRE_E_UNSUPPORTED, "too many frames");
    const int smem = kb_fbi_smem_layout(plan->n_freq, plan->n_bands, p.R).total;
    int grid;
    if ((rc = kb_resident_grid(kb_fbi_kernel, "fbinv", KB_FBI_WARPS * 32, smem, tiles, plan->dev.sm_count, &grid))) return rc;
    return kb_launch(kb_fbi_kernel, {.grid = grid, .block = KB_FBI_WARPS * 32, .smem = smem, .st = (cudaStream_t)stream}, p);
}

}  // extern "C"

// ---- IIR filters (iir_core.cuh) -------------------------------------------------------------------------------------
__global__ void __launch_bounds__(32) kb_iir_powers_kernel(const __grid_constant__ KbIirParams p) {
    __shared__ double m[192];
    kb_iir_powers_cta(p, m, (long long)blockIdx.x);
}
__global__ void __launch_bounds__(32) kb_iir_state_kernel(const __grid_constant__ KbIirParams p) {
    extern __shared__ __align__(16) char kb_smem[];
    kb_iir_state_cta(p, kb_smem, (long long)blockIdx.x);
}
__global__ void __launch_bounds__(128) kb_iir_carry_kernel(const __grid_constant__ KbIirParams p) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < p.n_cols) kb_iir_carry_col(p, i);
}
__global__ void __launch_bounds__(32) kb_iir_out_kernel(const __grid_constant__ KbIirParams p) {
    extern __shared__ __align__(16) char kb_smem[];
    kb_iir_out_cta(p, kb_smem, (long long)blockIdx.x);
}

// Workspace sections: powers (one set per column at most), chunk end states, block carries.  More than 4e18 bytes
// counts as an overflow.
static void kb_iir_layout(KbLayout& L, KbIirParams& p) {
    const double total = (double)p.n_cols * (KB_IIR_NPOW * 64 * 8 + (double)p.K * KB_IIR_N * 4 + (double)p.nblk * KB_IIR_N * 8);
    L.overflow |= total > 4.0e18;
    p.pw = L.take<double>(p.n_cols, KB_IIR_NPOW * 64);
    p.e = L.take<float>(p.n_cols, p.K, KB_IIR_N);
    p.blk = L.take<double>(p.n_cols, p.nblk, KB_IIR_N);
    L.pad();
}

static int kb_iir_check_sizes(int batch, int channels, int length, int order) {
    if (batch < 0 || channels < 0 || length < 0) return kb_fail(KAPRE_E_INVALID, "negative size");
    if (order < 0) return kb_fail(KAPRE_E_INVALID, "order must be >= 0, got %d", order);
    if (order > KB_IIR_N) return kb_fail(KAPRE_E_UNSUPPORTED, "IIR order %d is above the supported %d", order, KB_IIR_N);
    const long long K = ((long long)length + KB_IIR_TC - 1) / KB_IIR_TC;
    const long long nblk = (K + KB_IIR_W - 1) / KB_IIR_W;
    if ((long long)batch * channels * nblk > 0x7fffffffLL || (long long)batch * channels > 0x7fffffffLL)
        return kb_fail(KAPRE_E_INVALID, "too many IIR columns or blocks");
    return 0;
}

static bool kb_iir_same_shape(const kapre_wave_desc* a, const kapre_wave_desc* b) {
    return a->batch == b->batch && a->channels == b->channels && a->length == b->length;
}

// Fills everything but the data pointers; 1: nothing to do.
static int kb_iir_prepare(KbIirParams& p, const kapre_wave_desc* xd, const kapre_iir_coeffs* cf, int flags,
                          void* workspace_dev) {
    if (!xd || !cf) return kb_fail(KAPRE_E_INVALID, "null argument");
    if (flags & ~(KAPRE_IIR_CLAMP | KAPRE_IIR_REVERSE)) return kb_fail(KAPRE_E_INVALID, "unknown flags 0x%x", flags);
    int rc = kb_iir_check_sizes(xd->batch, xd->channels, xd->length, cf->order);
    if (rc) return rc;
    if (cf->b_stride_b < 0 || cf->b_stride_c < 0 || cf->a_stride_b < 0 || cf->a_stride_c < 0)
        return kb_fail(KAPRE_E_INVALID, "coefficient strides must be >= 0");
    p.B = xd->batch; p.C = xd->channels; p.L = xd->length;
    p.x_sb = xd->stride_b; p.x_sc = xd->stride_c; p.x_sl = xd->stride_l;
    p.bc = cf->b; p.b_sb = cf->b_stride_b; p.b_sc = cf->b_stride_c;
    p.ac = cf->a; p.a_sb = cf->a_stride_b; p.a_sc = cf->a_stride_c;
    p.order = cf->order;
    kb_iir_setup(p);
    if (p.n_cols == 0 || p.L == 0) return 1;
    if (!cf->b || !cf->a) return kb_fail(KAPRE_E_INVALID, "null coefficient pointer");
    if (!workspace_dev) return kb_fail(KAPRE_E_INVALID, "null workspace");
    KbLayout L{(char*)workspace_dev};
    kb_iir_layout(L, p);
    return L.overflow ? kb_fail(KAPRE_E_INVALID, "IIR workspace overflows") : 0;
}

// The largest element offset + 1 of a wave descriptor (the bulk copies' bound), strides assumed >= 0 where they matter.
static long long kb_iir_numel(const kapre_wave_desc* d) {
    long long n = 1;
    n += (long long)(d->batch - 1) * (d->stride_b > 0 ? d->stride_b : 0);
    n += (long long)(d->channels - 1) * (d->stride_c > 0 ? d->stride_c : 0);
    n += (long long)(d->length - 1) * (d->stride_l > 0 ? d->stride_l : 0);
    return n;
}

static int kb_iir_launch(KbIirParams& p, const float* in, const kapre_wave_desc* in_d, cudaStream_t st) {
    p.x = in;
    p.x_numel = kb_iir_numel(in_d);
    p.x_align = (unsigned)(((uintptr_t)in >> 2) & 3u);
    const long long n_f = (long long)p.n_fb * p.n_fc, tiles = p.n_cols * p.nblk;
    int rc;
    if ((rc = kb_launch(kb_iir_powers_kernel, {.grid = (int)n_f, .block = 32, .st = st}, p))) return rc;
    if ((rc = kb_launch(kb_iir_state_kernel, {.grid = (int)tiles, .block = 32, .smem = kb_iir_smem(0).total, .st = st,
                                              .timed = true}, p)))
        return rc;
    if ((rc = kb_launch(kb_iir_carry_kernel, {.grid = (int)((p.n_cols + 127) / 128), .block = 128, .st = st}, p)))
        return rc;
    const int refs = p.bwd && p.part != nullptr;
    return kb_launch(kb_iir_out_kernel, {.grid = (int)tiles, .block = 32, .smem = kb_iir_smem(refs).total, .st = st,
                                         .timed = true}, p);
}

extern "C" {

int64_t kapre_lfilter_workspace_bytes(int batch, int channels, int length, int order) {
    int rc = kb_iir_check_sizes(batch, channels, length, order);
    if (rc) return rc;
    KbIirParams p{};
    p.B = batch; p.C = channels; p.L = length;
    kb_iir_setup(p);
    KbLayout L;
    kb_iir_layout(L, p);
    return L.bytes("IIR");
}

int kapre_lfilter(const float* x_dev, const kapre_wave_desc* x_desc, const kapre_iir_coeffs* coeffs, int flags,
                  float* y_dev, const kapre_wave_desc* y_desc, void* workspace_dev, void* stream) {
    if (!y_desc) return kb_fail(KAPRE_E_INVALID, "null argument");
    KbIirParams p{};
    int rc = kb_iir_prepare(p, x_desc, coeffs, flags, workspace_dev);
    if (rc < 0) return rc;
    if (!kb_iir_same_shape(x_desc, y_desc)) return kb_fail(KAPRE_E_INVALID, "input and output shapes differ");
    if (rc == 1) return 0;
    if (!x_dev || !y_dev) return kb_fail(KAPRE_E_INVALID, "null data pointer");
    if ((const void*)x_dev == (const void*)y_dev) return kb_fail(KAPRE_E_INVALID, "lfilter cannot run in place");
    p.y = y_dev; p.y_sb = y_desc->stride_b; p.y_sc = y_desc->stride_c; p.y_sl = y_desc->stride_l;
    p.reverse = (flags & KAPRE_IIR_REVERSE) ? 1 : 0;
    p.clamp = (flags & KAPRE_IIR_CLAMP) ? 1 : 0;
    p.bwd = 0;
    return kb_iir_launch(p, x_dev, x_desc, (cudaStream_t)stream);
}

int kapre_lfilter_backward(const float* gy_dev, const kapre_wave_desc* gy_desc, const float* x_dev,
                           const kapre_wave_desc* x_desc, const float* y_dev, const kapre_wave_desc* y_desc,
                           const kapre_iir_coeffs* coeffs, int flags, float* gx_dev, const kapre_wave_desc* gx_desc,
                           float* partials_dev, void* workspace_dev, void* stream) {
    if (!gx_desc) return kb_fail(KAPRE_E_INVALID, "null argument");
    KbIirParams p{};
    int rc = kb_iir_prepare(p, gy_desc, coeffs, flags, workspace_dev);
    if (rc < 0) return rc;
    if (!kb_iir_same_shape(gy_desc, gx_desc)) return kb_fail(KAPRE_E_INVALID, "gradient shapes differ");
    if (partials_dev) {
        if (!x_desc || !y_desc) return kb_fail(KAPRE_E_INVALID, "coefficient gradients need x and y");
        if (!kb_iir_same_shape(gy_desc, x_desc) || !kb_iir_same_shape(gy_desc, y_desc))
            return kb_fail(KAPRE_E_INVALID, "x and y must have the gradient's shape");
    }
    if (rc == 1) return 0;      // no chunks: the partial sums are empty too
    if (!gy_dev || !gx_dev) return kb_fail(KAPRE_E_INVALID, "null data pointer");
    if ((const void*)gy_dev == (const void*)gx_dev) return kb_fail(KAPRE_E_INVALID, "lfilter backward cannot run in place");
    if (partials_dev && (!x_dev || !y_dev)) return kb_fail(KAPRE_E_INVALID, "coefficient gradients need x and y");
    p.y = gx_dev; p.y_sb = gx_desc->stride_b; p.y_sc = gx_desc->stride_c; p.y_sl = gx_desc->stride_l;
    p.reverse = (flags & KAPRE_IIR_REVERSE) ? 0 : 1;       // the adjoint runs the other way
    p.clamp = 0;
    p.bwd = 1;
    if (partials_dev) {
        p.part = partials_dev;
        p.xr = x_dev; p.xr_sb = x_desc->stride_b; p.xr_sc = x_desc->stride_c; p.xr_sl = x_desc->stride_l;
        p.yr = y_dev; p.yr_sb = y_desc->stride_b; p.yr_sc = y_desc->stride_c; p.yr_sl = y_desc->stride_l;
    }
    return kb_iir_launch(p, gy_dev, gy_desc, (cudaStream_t)stream);
}

}  // extern "C"

// ---- second-order sections (sos_core.cuh) ---------------------------------------------------------------------------
template <int S>
__global__ void __launch_bounds__(32) kb_sos_powers_kernel(const __grid_constant__ KbSosParams p) {
    __shared__ double m[3 * 4 * S * S];
    kb_sos_powers_cta<S>(p, m, (long long)blockIdx.x);
}
template <int S>
__global__ void __launch_bounds__(32) kb_sos_state_kernel(const __grid_constant__ KbSosParams p) {
    extern __shared__ __align__(16) char kb_smem[];
    kb_sos_state_cta<S>(p, kb_smem, (long long)blockIdx.x);
}
template <int S>
__global__ void __launch_bounds__(128) kb_sos_carry_kernel(const __grid_constant__ KbSosParams p) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < p.g.n_cols) kb_sos_carry_col<S>(p, i);
}
template <int S>
__global__ void __launch_bounds__(32) kb_sos_out_kernel(const __grid_constant__ KbSosParams p) {
    extern __shared__ __align__(16) char kb_smem[];
    kb_sos_out_cta<S>(p, kb_smem, (long long)blockIdx.x);
}

// Workspace sections: powers (one set per column at most), chunk end states, block carries, each 2S wide.
static void kb_sos_layout(KbLayout& L, KbSosParams& p) {
    const int D = 2 * p.S;
    p.g.pw = L.take<double>(p.g.n_cols, KB_IIR_NPOW * D * D);
    p.g.e = L.take<float>(p.g.n_cols, p.g.K, D);
    p.g.blk = L.take<double>(p.g.n_cols, p.g.nblk, D);
    L.pad();
}

static int kb_sos_check_sizes(int batch, int channels, int length, int n_sections) {
    if (batch < 0 || channels < 0 || length < 0) return kb_fail(KAPRE_E_INVALID, "negative size");
    if (n_sections < 1 || n_sections > KB_SOS_MAX)
        return kb_fail(KAPRE_E_UNSUPPORTED, "%d sections: 1 to %d are supported", n_sections, KB_SOS_MAX);
    return kb_iir_check_sizes(batch, channels, length, 0);
}

// Fills the geometry and the workspace pointers; 1: nothing to do.
static int kb_sos_prepare(KbSosParams& p, const kapre_wave_desc* xd, const kapre_sos_coeffs* cf, void* workspace_dev) {
    if (!xd || !cf) return kb_fail(KAPRE_E_INVALID, "null argument");
    int rc = kb_sos_check_sizes(xd->batch, xd->channels, xd->length, cf->n_sections);
    if (rc) return rc;
    if (cf->stride_b < 0 || cf->stride_c < 0) return kb_fail(KAPRE_E_INVALID, "coefficient strides must be >= 0");
    p.g.B = xd->batch; p.g.C = xd->channels; p.g.L = xd->length;
    p.g.x_sb = xd->stride_b; p.g.x_sc = xd->stride_c; p.g.x_sl = xd->stride_l;
    p.g.ac = cf->sos; p.g.a_sb = cf->stride_b; p.g.a_sc = cf->stride_c;
    p.S = cf->n_sections;
    kb_iir_setup(p.g);
    if (p.g.n_cols == 0 || p.g.L == 0) return 1;
    if (!cf->sos) return kb_fail(KAPRE_E_INVALID, "null coefficient pointer");
    if (!workspace_dev) return kb_fail(KAPRE_E_INVALID, "null workspace");
    KbLayout L{(char*)workspace_dev};
    kb_sos_layout(L, p);
    return L.overflow ? kb_fail(KAPRE_E_INVALID, "SOS workspace overflows") : 0;
}

template <int S>
static int kb_sos_launch_s(const KbSosParams& p, cudaStream_t st) {
    const long long n_f = (long long)p.g.n_fb * p.g.n_fc, tiles = p.g.n_cols * p.g.nblk;
    const int smem = kb_sos_smem(S).total;
    int rc;
    if ((rc = kb_launch(kb_sos_powers_kernel<S>, {.grid = (int)n_f, .block = 32, .st = st}, p))) return rc;
    if ((rc = kb_launch(kb_sos_state_kernel<S>, {.grid = (int)tiles, .block = 32, .smem = smem, .st = st, .timed = true},
                        p)))
        return rc;
    if ((rc = kb_launch(kb_sos_carry_kernel<S>, {.grid = (int)((p.g.n_cols + 127) / 128), .block = 128, .st = st}, p)))
        return rc;
    return kb_launch(kb_sos_out_kernel<S>, {.grid = (int)tiles, .block = 32, .smem = smem, .st = st, .timed = true}, p);
}

static int kb_sos_launch(const KbSosParams& p, cudaStream_t st) {
    switch (p.S) {
    case 1: return kb_sos_launch_s<1>(p, st);
    case 2: return kb_sos_launch_s<2>(p, st);
    case 3: return kb_sos_launch_s<3>(p, st);
    case 4: return kb_sos_launch_s<4>(p, st);
    case 5: return kb_sos_launch_s<5>(p, st);
    case 6: return kb_sos_launch_s<6>(p, st);
    case 7: return kb_sos_launch_s<7>(p, st);
    case 8: return kb_sos_launch_s<8>(p, st);
    }
    return kb_fail(KAPRE_E_UNSUPPORTED, "%d sections", p.S);
}

extern "C" {

int64_t kapre_sosfilt_workspace_bytes(int batch, int channels, int length, int n_sections) {
    int rc = kb_sos_check_sizes(batch, channels, length, n_sections);
    if (rc) return rc;
    KbSosParams p{};
    p.g.B = batch; p.g.C = channels; p.g.L = length;
    p.S = n_sections;
    kb_iir_setup(p.g);
    KbLayout L;
    kb_sos_layout(L, p);
    return L.bytes("SOS");
}

int kapre_sosfilt(const float* x_dev, const kapre_wave_desc* x_desc, const kapre_sos_coeffs* sos, const float* zi_dev,
                  const kapre_sos_state_desc* zi_desc, int flags, float* y_dev, const kapre_wave_desc* y_desc,
                  float* zf_dev, const kapre_sos_state_desc* zf_desc, void* workspace_dev, void* stream) {
    if (!y_desc) return kb_fail(KAPRE_E_INVALID, "null argument");
    if (flags & ~KAPRE_IIR_REVERSE) return kb_fail(KAPRE_E_INVALID, "unknown flags 0x%x", flags);
    if ((zi_dev && !zi_desc) || (zf_dev && !zf_desc)) return kb_fail(KAPRE_E_INVALID, "a state needs its descriptor");
    if (zi_dev && (zi_desc->stride_b < 0 || zi_desc->stride_c < 0 || zi_desc->stride_s < 0))
        return kb_fail(KAPRE_E_INVALID, "zi strides must be >= 0");
    KbSosParams p{};
    int rc = kb_sos_prepare(p, x_desc, sos, workspace_dev);
    if (rc < 0) return rc;
    if (!kb_iir_same_shape(x_desc, y_desc)) return kb_fail(KAPRE_E_INVALID, "input and output shapes differ");
    if (rc == 1) return 0;
    if (!x_dev || !y_dev) return kb_fail(KAPRE_E_INVALID, "null data pointer");
    if ((const void*)x_dev == (const void*)y_dev) return kb_fail(KAPRE_E_INVALID, "sosfilt cannot run in place");
    p.g.x = x_dev;
    p.g.x_numel = kb_iir_numel(x_desc);
    p.g.x_align = (unsigned)(((uintptr_t)x_dev >> 2) & 3u);
    p.g.y = y_dev; p.g.y_sb = y_desc->stride_b; p.g.y_sc = y_desc->stride_c; p.g.y_sl = y_desc->stride_l;
    p.g.reverse = (flags & KAPRE_IIR_REVERSE) ? 1 : 0;
    if (zi_dev) { p.zi = zi_dev; p.zi_sb = zi_desc->stride_b; p.zi_sc = zi_desc->stride_c; p.zi_ss = zi_desc->stride_s; }
    if (zf_dev) { p.zf = zf_dev; p.zf_sb = zf_desc->stride_b; p.zf_sc = zf_desc->stride_c; p.zf_ss = zf_desc->stride_s; }
    return kb_sos_launch(p, (cudaStream_t)stream);
}

}  // extern "C"

// ---- additive noise (noise_core.cuh) -------------------------------------------------------------------------------
// Both passes wait for the previous kernel in the stream before touching data, so they may be launched with PDL.  Four
// CTAs of four warps per SM: 128 registers, which hold a lane's batches of loads of every operand in flight at once.
__global__ void __launch_bounds__(KB_NOISE_WARPS * 32, 4) kb_noise_sum_kernel(const __grid_constant__ KbNoiseParams p) {
    extern __shared__ __align__(16) char kb_smem[];
    asm volatile("griddepcontrol.wait;" ::: "memory");
    const int w = (int)(threadIdx.x >> 5);
    const long long tile = (long long)blockIdx.x * KB_NOISE_WARPS + w;
    if (tile < p.tiles) kb_noise_sum_tile(p, kb_smem + w * kb_noise_smem(kb_noise_cg_max(p)).total, tile);
}
__global__ void __launch_bounds__(KB_NOISE_WARPS * 32, 4) kb_noise_out_kernel(const __grid_constant__ KbNoiseParams p) {
    extern __shared__ __align__(16) char kb_smem[];
    asm volatile("griddepcontrol.wait;" ::: "memory");
    const int w = (int)(threadIdx.x >> 5);
    const long long tile = (long long)blockIdx.x * KB_NOISE_WARPS + w;
    if (tile < p.tiles) kb_noise_out_tile(p, kb_smem + w * kb_noise_smem(kb_noise_cg_max(p)).total, tile);
}

// The workspace of a shape: the (B C, nseg, 2) segment sums.  -1: a negative size or an overflow.
static int kb_noise_layout(KbLayout& L, int batch, int channels, int length, double** part) {
    if (batch < 0 || channels < 0 || length < 0) return -1;
    const long long nseg = ((long long)length + KB_NOISE_SEG - 1) / KB_NOISE_SEG;
    const long long groups = ((long long)channels + KB_NOISE_G - 1) / KB_NOISE_G;
    const double total = (double)batch * channels * nseg * 16.0;
    if (total > 4.0e18 || (double)batch * groups * nseg / KB_NOISE_WARPS > 2147483647.0) return -1;
    *part = L.take<double>(batch, channels, nseg, 2);
    L.pad();
    return L.overflow ? -1 : 0;
}

static bool kb_noise_same_shape(const kapre_wave_desc* a, const kapre_wave_desc* b) {
    return a->batch == b->batch && a->channels == b->channels && a->length == b->length;
}

static KbNoiseWave kb_noise_wave(const float* p, const kapre_wave_desc* d) {
    KbNoiseWave w;
    w.p = p;
    w.sb = d->batch == 1 ? 0 : d->stride_b;
    w.sc = d->channels == 1 ? 0 : d->stride_c;
    w.sl = d->stride_l;
    return w;
}

// Checks and fills everything the two directions share; 1: nothing to launch.
static int kb_noise_prepare(KbNoiseParams& p, const kapre_wave_desc* xd, const kapre_noise_source* ns,
                            const kapre_snr_desc* sd, void* workspace_dev) {
    if (!xd || !ns || !sd) return kb_fail(KAPRE_E_INVALID, "null argument");
    KbLayout L{(char*)workspace_dev};
    if (kb_noise_layout(L, xd->batch, xd->channels, xd->length, &p.part) < 0)
        return kb_fail(KAPRE_E_INVALID, "add_noise: negative size or too many samples (%d, %d, %d)", xd->batch,
                       xd->channels, xd->length);
    if (ns->mode == KAPRE_NOISE_TENSOR) {
        const kapre_wave_desc& nd = ns->noise_desc;
        if ((nd.batch != 1 && nd.batch != xd->batch) || (nd.channels != 1 && nd.channels != xd->channels) ||
            nd.length != xd->length)
            return kb_fail(KAPRE_E_INVALID, "noise shape (%d, %d, %d) does not broadcast to (%d, %d, %d)", nd.batch,
                           nd.channels, nd.length, xd->batch, xd->channels, xd->length);
    } else if (ns->mode == KAPRE_NOISE_BANK) {
        if (ns->bank_length < 0) return kb_fail(KAPRE_E_INVALID, "negative bank length");
    } else {
        return kb_fail(KAPRE_E_INVALID, "unknown noise mode %d", ns->mode);
    }
    p.B = xd->batch; p.C = xd->channels; p.L = xd->length;
    kb_noise_setup(p);
    if (p.tiles == 0) return 1;
    if (!sd->snr) return kb_fail(KAPRE_E_INVALID, "null snr pointer");
    if (ns->mode == KAPRE_NOISE_TENSOR && !ns->noise) return kb_fail(KAPRE_E_INVALID, "null noise pointer");
    if (ns->mode == KAPRE_NOISE_BANK && (!ns->bank || !ns->start || !ns->clip_len || !ns->offset))
        return kb_fail(KAPRE_E_INVALID, "null bank pointer");
    if (!workspace_dev) return kb_fail(KAPRE_E_INVALID, "null workspace");
    if (ns->mode == KAPRE_NOISE_TENSOR) {
        p.n = kb_noise_wave(ns->noise, &ns->noise_desc);
    } else {
        p.bank = ns->bank; p.bank_numel = ns->bank_length;
        p.start = (const long long*)ns->start; p.clip = (const long long*)ns->clip_len;
        p.offset = (const long long*)ns->offset;
    }
    p.snr = sd->snr; p.snr_sb = sd->snr_stride_b; p.snr_sc = sd->snr_stride_c;
    p.len = sd->lengths; p.len_sb = sd->lengths_stride_b; p.len_sc = sd->lengths_stride_c;
    return 0;
}

static int kb_noise_launch(const KbNoiseParams& p, cudaStream_t st) {
    const int grid = (int)((p.tiles + KB_NOISE_WARPS - 1) / KB_NOISE_WARPS);
    const int smem = KB_NOISE_WARPS * kb_noise_smem(kb_noise_cg_max(p)).total;
    int rc;
    if ((rc = kb_launch(kb_noise_sum_kernel, {.grid = grid, .block = KB_NOISE_WARPS * 32, .smem = smem, .st = st,
                                              .pdl = true}, p)))
        return rc;
    return kb_launch(kb_noise_out_kernel, {.grid = grid, .block = KB_NOISE_WARPS * 32, .smem = smem, .st = st,
                                           .pdl = true}, p);
}

extern "C" {

int64_t kapre_add_noise_workspace_bytes(int batch, int channels, int length) {
    KbLayout L;
    double* part;
    if (kb_noise_layout(L, batch, channels, length, &part) < 0)
        return kb_fail(KAPRE_E_INVALID, "add_noise: negative size or too many samples");
    return L.end;
}

int kapre_add_noise(const float* x_dev, const kapre_wave_desc* x_desc, const kapre_noise_source* noise,
                    const kapre_snr_desc* snr, float* y_dev, const kapre_wave_desc* y_desc, double* stats_dev,
                    void* workspace_dev, void* stream) {
    if (!y_desc) return kb_fail(KAPRE_E_INVALID, "null argument");
    KbNoiseParams p{};
    int rc = kb_noise_prepare(p, x_desc, noise, snr, workspace_dev);
    if (rc < 0) return rc;
    if (!kb_noise_same_shape(x_desc, y_desc)) return kb_fail(KAPRE_E_INVALID, "input and output shapes differ");
    if (rc == 1) return 0;
    if (!x_dev || !y_dev) return kb_fail(KAPRE_E_INVALID, "null data pointer");
    if ((const void*)y_dev == (const void*)x_dev || (const void*)y_dev == (const void*)p.n.p)
        return kb_fail(KAPRE_E_INVALID, "add_noise cannot run in place");
    p.x = kb_noise_wave(x_dev, x_desc);
    p.x.sb = x_desc->stride_b; p.x.sc = x_desc->stride_c;
    p.y = y_dev; p.y_sb = y_desc->stride_b; p.y_sc = y_desc->stride_c; p.y_sl = y_desc->stride_l;
    p.stats = stats_dev;
    p.bwd = 0;
    return kb_noise_launch(p, (cudaStream_t)stream);
}

int kapre_add_noise_backward(const float* g_dev, const kapre_wave_desc* g_desc, const float* x_dev,
                             const kapre_wave_desc* x_desc, const kapre_noise_source* noise, const kapre_snr_desc* snr,
                             const double* stats_dev, float* gx_dev, const kapre_wave_desc* gx_desc, float* gn_dev,
                             const kapre_wave_desc* gn_desc, float* gsnr_dev, void* workspace_dev, void* stream) {
    if (!x_desc || !gx_desc) return kb_fail(KAPRE_E_INVALID, "null argument");
    KbNoiseParams p{};
    int rc = kb_noise_prepare(p, g_desc, noise, snr, workspace_dev);
    if (rc < 0) return rc;
    if (!kb_noise_same_shape(g_desc, x_desc) || !kb_noise_same_shape(g_desc, gx_desc))
        return kb_fail(KAPRE_E_INVALID, "gradient and input shapes differ");
    if (gn_dev) {
        if (noise->mode != KAPRE_NOISE_TENSOR) return kb_fail(KAPRE_E_INVALID, "a noise bank has no gradient");
        if (!gn_desc || !kb_noise_same_shape(g_desc, gn_desc))
            return kb_fail(KAPRE_E_INVALID, "the noise gradient needs the input's shape");
    }
    if (rc == 1) return 0;
    if (!g_dev || !x_dev || !gx_dev || !stats_dev) return kb_fail(KAPRE_E_INVALID, "null data pointer");
    if ((const void*)gx_dev == (const void*)g_dev || (gn_dev && (const void*)gn_dev == (const void*)g_dev))
        return kb_fail(KAPRE_E_INVALID, "add_noise backward cannot run in place");
    p.x = kb_noise_wave(g_dev, g_desc);
    p.x.sb = g_desc->stride_b; p.x.sc = g_desc->stride_c;
    p.xr = kb_noise_wave(x_dev, x_desc);
    p.xr.sb = x_desc->stride_b; p.xr.sc = x_desc->stride_c;
    p.y = gx_dev; p.y_sb = gx_desc->stride_b; p.y_sc = gx_desc->stride_c; p.y_sl = gx_desc->stride_l;
    if (gn_dev) { p.gn = gn_dev; p.gn_sb = gn_desc->stride_b; p.gn_sc = gn_desc->stride_c; p.gn_sl = gn_desc->stride_l; }
    p.gsnr = gsnr_dev;
    p.stats = const_cast<double*>(stats_dev);
    p.bwd = 1;
    return kb_noise_launch(p, (cudaStream_t)stream);
}

}  // extern "C"

// ---- Kaldi-compatible features (kaldi_core.cuh) ----------------------------------------------------------------------
// Persistent CTAs of four independent warps; one warp per job of 32 / Q frames.  The forward needs about 19 KB of
// shared memory per warp (two CTAs per SM), the backward about 45 KB (one CTA per SM).
template <int Q>
__global__ void __launch_bounds__(KB_KALDI_WARPS * 32, 2) kb_kaldi_fwd_kernel(const __grid_constant__ KbKaldiParams p) {
    extern __shared__ __align__(16) char kb_smem[];
    const int w = (int)(threadIdx.x >> 5);
    const int per = kb_kaldi_smem(p.N, Q, p.n_mel, 0).total;
    for (long long job = (long long)blockIdx.x * KB_KALDI_WARPS + w; job < p.jobs;
         job += (long long)gridDim.x * KB_KALDI_WARPS)
        kb_kaldi_fwd_job<Q>(p, kb_smem + w * per, job);
}
template <int Q>
__global__ void __launch_bounds__(KB_KALDI_WARPS * 32, 1) kb_kaldi_bwd_kernel(const __grid_constant__ KbKaldiParams p) {
    extern __shared__ __align__(16) char kb_smem[];
    const int w = (int)(threadIdx.x >> 5);
    const int per = kb_kaldi_smem(p.N, Q, p.n_mel, 1).total;
    for (long long job = (long long)blockIdx.x * KB_KALDI_WARPS + w; job < p.jobs;
         job += (long long)gridDim.x * KB_KALDI_WARPS)
        kb_kaldi_bwd_job<Q>(p, kb_smem + w * per, job);
}
__global__ void kb_kaldi_gather_kernel(const __grid_constant__ KbKaldiParams p, long long n) {
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e < n) kb_kaldi_gather_elem(p, e);
}
__global__ void kb_kaldi_cmn_kernel(const __grid_constant__ KbKaldiParams p, const float* in, kapre_spec_desc id,
                                    float* out, kapre_spec_desc od, long long n) {
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e < n)
        kb_kaldi_cmn_col(p, in, id.stride_b, id.stride_c, id.stride_t, id.stride_f, out, od.stride_b, od.stride_c,
                         od.stride_t, od.stride_f, e);
}

struct kapre_kaldi_plan {
    kapre_kaldi_config cfg;
    int Q, K, P;
    DevInfo dev;
    KbTables tables;
    const float* wh; const float* half; const float2* twp; const float2* twn;
    const int* mlo; const int* mlen; const int* moff; const float* mw;
    const int* klo; const int* klen; const int* kidx; const float* kw;
    const float* dct;
};

// The backward workspace: the per-frame gradients gf, then the mean-subtracted output gradient gc (empty without mean
// subtraction).
static void kb_kaldi_layout(KbLayout& L, const kapre_kaldi_plan* plan, int batch, int channels, int frames, float** gf,
                            float** gc) {
    *gf = L.take<float>(batch, channels, frames, plan->cfg.window_size);
    *gc = L.take<float>(batch, channels, frames, plan->cfg.subtract_mean ? plan->K : 0);
}

static bool kb_finite(float v) { return kb_kaldi_finite(v); }

static int kb_kaldi_check_cfg(const kapre_kaldi_config* c) {
    if (c->kind < KAPRE_KALDI_FBANK || c->kind > KAPRE_KALDI_SPECTROGRAM)
        return kb_fail(KAPRE_E_INVALID, "kaldi: unknown feature kind %d", c->kind);
    if (c->window_size < 2 || c->window_shift < 1 || c->min_length < 0)
        return kb_fail(KAPRE_E_INVALID, "kaldi: window size %d must be >= 2 and the shift %d >= 1", c->window_size,
                       c->window_shift);
    if (c->padded_window_size < c->window_size || (c->padded_window_size & 1))
        return kb_fail(KAPRE_E_INVALID, "kaldi: padded window size %d must be even and >= the window size %d",
                       c->padded_window_size, c->window_size);
    const int n = c->padded_window_size;
    if (n != 256 && n != 512 && n != 1024 && n != 2048)
        return kb_fail(KAPRE_E_UNSUPPORTED, "kaldi: padded window size %d is not supported (256, 512, 1024 or 2048)", n);
    if (!kb_finite(c->preemphasis_coefficient) || c->preemphasis_coefficient < 0.0f ||
        c->preemphasis_coefficient > 1.0f)
        return kb_fail(KAPRE_E_INVALID, "kaldi: preemphasis_coefficient must be in [0, 1]");
    if (!kb_finite(c->energy_floor) || c->energy_floor < 0.0f)
        return kb_fail(KAPRE_E_INVALID, "kaldi: energy_floor must be finite and >= 0");
    const int flags[] = {c->snip_edges, c->use_energy, c->htk_compat, c->raw_energy, c->use_power, c->use_log_fbank,
                         c->remove_dc_offset, c->subtract_mean};
    for (int f : flags)
        if (f != 0 && f != 1) return kb_fail(KAPRE_E_INVALID, "kaldi: flags must be 0 or 1");
    if (c->kind != KAPRE_KALDI_SPECTROGRAM && (c->num_mel_bins < 1 || c->num_mel_bins > KB_KALDI_MAX_MEL))
        return kb_fail(KAPRE_E_INVALID, "kaldi: num_mel_bins %d must be in [1, %d]", c->num_mel_bins, KB_KALDI_MAX_MEL);
    if (c->kind == KAPRE_KALDI_MFCC && (c->num_ceps < 1 || c->num_ceps > c->num_mel_bins))
        return kb_fail(KAPRE_E_INVALID, "kaldi: num_ceps %d must be in [1, num_mel_bins]", c->num_ceps);
    if (c->kind != KAPRE_KALDI_FBANK && !c->use_power)
        return kb_fail(KAPRE_E_INVALID, "kaldi: mfcc and spectrogram use the power spectrum");
    if (c->kind == KAPRE_KALDI_MFCC && !c->use_log_fbank)
        return kb_fail(KAPRE_E_INVALID, "kaldi: mfcc takes the log mel energies");
    return 0;
}

static KbKaldiParams kb_kaldi_params(const kapre_kaldi_plan* pl) {
    const kapre_kaldi_config& c = pl->cfg;
    KbKaldiParams p{};
    p.W = c.window_size; p.H = c.window_shift; p.N = c.padded_window_size; p.Q = pl->Q;
    p.snip = c.snip_edges; p.min_len = c.min_length;
    p.kind = c.kind; p.n_mel = c.kind == KAPRE_KALDI_SPECTROGRAM ? 0 : c.num_mel_bins; p.n_ceps = c.num_ceps;
    p.K = pl->K;
    p.use_energy = c.use_energy; p.htk = c.htk_compat; p.raw_energy = c.raw_energy; p.use_power = c.use_power;
    p.use_log = c.use_log_fbank; p.remove_dc = c.remove_dc_offset;
    p.preemph = c.preemphasis_coefficient;
    p.log_floor = c.energy_floor == 0.0f ? -INFINITY : (float)log((double)c.energy_floor);
    p.wh = pl->wh; p.half = pl->half; p.twp = pl->twp; p.twn = pl->twn;
    p.mlo = pl->mlo; p.mlen = pl->mlen; p.moff = pl->moff; p.mw = pl->mw;
    p.klo = pl->klo; p.klen = pl->klen; p.kidx = pl->kidx; p.kw = pl->kw;
    p.dct = pl->dct;
    return p;
}

// Shape checks and per-call fields shared by both directions; 1: nothing to launch.
static int kb_kaldi_prepare(KbKaldiParams& p, const kapre_kaldi_plan* pl, const kapre_wave_desc* xd,
                            const int32_t* len_h, const int32_t* len_d, int frames, float dither, uint64_t seed) {
    if (!pl || !xd) return kb_fail(KAPRE_E_INVALID, "null argument");
    int rc = kb_check_device(pl->dev);
    if (rc) return rc;
    if (xd->batch < 0 || xd->channels < 0 || xd->length < 0)
        return kb_fail(KAPRE_E_INVALID, "kaldi: negative size (%d, %d, %d)", xd->batch, xd->channels, xd->length);
    if (!kb_finite(dither) || dither < 0.0f) return kb_fail(KAPRE_E_INVALID, "kaldi: dither must be finite and >= 0");
    if (len_h && !len_d) return kb_fail(KAPRE_E_INVALID, "kaldi: lengths need their device copy");
    p = kb_kaldi_params(pl);
    p.B = xd->batch; p.C = xd->channels; p.L = xd->length;
    int tmax = 0;
    for (int b = 0; b < (len_h ? p.B : 1); ++b) {
        const int l = len_h ? len_h[b] : p.L;
        if (l < 0 || l > p.L) return kb_fail(KAPRE_E_INVALID, "kaldi: length %d of item %d is outside [0, %d]", l, b, p.L);
        const int t = kb_kaldi_frames(l, p.W, p.H, p.snip, p.min_len);
        tmax = t > tmax ? t : tmax;
    }
    if (p.B == 0) tmax = 0;
    if (frames != tmax) return kb_fail(KAPRE_E_INVALID, "kaldi: frames %d, the batch has %d", frames, tmax);
    if ((long long)frames * p.K > 2147483647LL || (long long)frames * p.W > 2147483647LL)
        return kb_fail(KAPRE_E_INVALID, "kaldi: frames x bins overflows int32");
    p.T = frames;
    p.len = len_h ? len_d : nullptr;
    p.dither = dither; p.seed = (unsigned long long)seed;
    const int FPW = 32 / p.Q;
    p.jobs = (long long)p.B * p.C * ((p.T + FPW - 1) / FPW);
    return p.jobs == 0 ? 1 : 0;
}

template <int Q>
static int kb_kaldi_launch_q(const KbKaldiParams& p, int sm_count, cudaStream_t st) {
    const int bwd = p.bwd;
    const int smem = KB_KALDI_WARPS * kb_kaldi_smem(p.N, Q, p.n_mel, bwd).total;
    const long long ctas = (p.jobs + KB_KALDI_WARPS - 1) / KB_KALDI_WARPS;
    int grid = 0, rc;
    if (bwd) {
        if ((rc = kb_resident_grid(kb_kaldi_bwd_kernel<Q>, "kaldi_bwd", KB_KALDI_WARPS * 32, smem, ctas, sm_count, &grid))) return rc;
        return kb_launch(kb_kaldi_bwd_kernel<Q>, {.grid = grid, .block = KB_KALDI_WARPS * 32, .smem = smem, .st = st}, p);
    }
    if ((rc = kb_resident_grid(kb_kaldi_fwd_kernel<Q>, "kaldi_fwd", KB_KALDI_WARPS * 32, smem, ctas, sm_count, &grid))) return rc;
    return kb_launch(kb_kaldi_fwd_kernel<Q>, {.grid = grid, .block = KB_KALDI_WARPS * 32, .smem = smem, .st = st,
                                              .timed = true}, p);
}

static int kb_kaldi_launch(const KbKaldiParams& p, int sm_count, cudaStream_t st) {
    switch (p.Q) {
        case 4: return kb_kaldi_launch_q<4>(p, sm_count, st);
        case 8: return kb_kaldi_launch_q<8>(p, sm_count, st);
        case 16: return kb_kaldi_launch_q<16>(p, sm_count, st);
        default: return kb_kaldi_launch_q<32>(p, sm_count, st);
    }
}

static int kb_kaldi_cmn(const KbKaldiParams& p, const float* in, const kapre_spec_desc& id, float* out,
                        const kapre_spec_desc& od, cudaStream_t st) {
    const long long n = (long long)p.B * p.C * p.K;
    return kb_launch(kb_kaldi_cmn_kernel, {.grid = (int)((n + 255) / 256), .block = 256, .st = st}, p, in, id, out, od, n);
}

extern "C" {

int kapre_kaldi_plan_create(const kapre_kaldi_config* cfg, const float* window_host, const float* banks_host,
                            const float* dct_host, kapre_kaldi_plan** out) {
    if (!cfg || !out || !window_host) return kb_fail(KAPRE_E_INVALID, "null argument");
    *out = nullptr;
    int rc = kb_kaldi_check_cfg(cfg);
    if (rc) return rc;
    const int W = cfg->window_size, N = cfg->padded_window_size, P = N / 2, Q = P / 32;
    const bool mel = cfg->kind != KAPRE_KALDI_SPECTROGRAM;
    const int M = mel ? cfg->num_mel_bins : 0;
    if (mel && !banks_host) return kb_fail(KAPRE_E_INVALID, "kaldi: null mel banks");
    if (cfg->kind == KAPRE_KALDI_MFCC && !dct_host) return kb_fail(KAPRE_E_INVALID, "kaldi: null DCT matrix");
    KbKaldiTables t;
    const int bad = kb_kaldi_tables(W, N, M, cfg->kind == KAPRE_KALDI_MFCC ? M * cfg->num_ceps : 0, window_host,
                                    banks_host, dct_host, t);
    if (bad) return kb_fail(KAPRE_E_INVALID, "kaldi: non-finite %s", bad == 1 ? "window" : bad == 2 ? "mel weight" : "DCT");
    kapre_kaldi_plan* pl = new kapre_kaldi_plan();
    pl->cfg = *cfg;
    pl->Q = Q; pl->P = P;
    pl->K = cfg->kind == KAPRE_KALDI_FBANK ? M + cfg->use_energy
          : cfg->kind == KAPRE_KALDI_MFCC ? cfg->num_ceps : P + 1;
    if ((rc = kb_dev_info(&pl->dev))) { delete pl; return rc; }
    KbTableUpload tb;
    tb.add(t.wh, &pl->wh); tb.add(t.half, &pl->half); tb.add(t.twp, &pl->twp); tb.add(t.twn, &pl->twn);
    tb.add(t.mlo, &pl->mlo); tb.add(t.mlen, &pl->mlen); tb.add(t.moff, &pl->moff); tb.add(t.mw, &pl->mw);
    tb.add(t.klo, &pl->klo); tb.add(t.klen, &pl->klen); tb.add(t.kidx, &pl->kidx); tb.add(t.kw, &pl->kw);
    tb.add(t.dct, &pl->dct);
    if ((rc = tb.upload(pl->tables, "kaldi"))) { delete pl; return rc; }
    *out = pl;
    return 0;
}

void kapre_kaldi_plan_destroy(kapre_kaldi_plan* plan) { delete plan; }

int kapre_kaldi_num_frames(const kapre_kaldi_plan* plan, int length) {
    if (!plan) return kb_fail(KAPRE_E_INVALID, "null plan");
    if (length < 0) return kb_fail(KAPRE_E_INVALID, "negative length");
    const kapre_kaldi_config& c = plan->cfg;
    return kb_kaldi_frames(length, c.window_size, c.window_shift, c.snip_edges, c.min_length);
}

int kapre_kaldi_num_bins(const kapre_kaldi_plan* plan) {
    if (!plan) return kb_fail(KAPRE_E_INVALID, "null plan");
    return plan->K;
}

int64_t kapre_kaldi_workspace_bytes(const kapre_kaldi_plan* plan, int batch, int channels, int frames, int backward) {
    if (!plan) return kb_fail(KAPRE_E_INVALID, "null plan");
    if (batch < 0 || channels < 0 || frames < 0) return kb_fail(KAPRE_E_INVALID, "kaldi: negative size");
    if ((long long)frames * plan->K > 2147483647LL || (long long)frames * plan->cfg.window_size > 2147483647LL)
        return kb_fail(KAPRE_E_INVALID, "kaldi: frames x bins overflows int32");
    if (!backward) return 0;
    const double cols = (double)batch * channels * frames;
    const double bytes = cols * plan->cfg.window_size * 4.0 + (plan->cfg.subtract_mean ? cols * plan->K * 4.0 : 0.0);
    if (bytes > 4.0e18) return kb_fail(KAPRE_E_INVALID, "kaldi: workspace overflow");
    KbLayout L;
    float *gf, *gc;
    kb_kaldi_layout(L, plan, batch, channels, frames, &gf, &gc);
    return L.bytes("kaldi");
}

int kapre_kaldi_features(const kapre_kaldi_plan* plan, const float* x_dev, const kapre_wave_desc* x_desc,
                         const int32_t* lengths_host, const int32_t* lengths_dev, int frames, float dither,
                         uint64_t seed, float* y_dev, const kapre_spec_desc* y_desc, void* workspace_dev,
                         void* stream) {
    (void)workspace_dev;
    if (!y_desc) return kb_fail(KAPRE_E_INVALID, "null argument");
    KbKaldiParams p;
    int rc = kb_kaldi_prepare(p, plan, x_desc, lengths_host, lengths_dev, frames, dither, seed);
    if (rc < 0) return rc;
    if (rc == 1) return 0;
    if (!x_dev || !y_dev) return kb_fail(KAPRE_E_INVALID, "null data pointer");
    p.x = x_dev; p.x_sb = x_desc->stride_b; p.x_sc = x_desc->stride_c; p.x_sl = x_desc->stride_l;
    p.y = y_dev; p.y_sb = y_desc->stride_b; p.y_sc = y_desc->stride_c; p.y_st = y_desc->stride_t;
    p.y_sk = y_desc->stride_f;
    p.bwd = 0;
    const cudaStream_t st = (cudaStream_t)stream;
    if ((rc = kb_kaldi_launch(p, plan->dev.sm_count, st))) return rc;
    if (plan->cfg.subtract_mean) return kb_kaldi_cmn(p, y_dev, *y_desc, y_dev, *y_desc, st);
    return 0;
}

int kapre_kaldi_features_backward(const kapre_kaldi_plan* plan, const float* gy_dev, const kapre_spec_desc* gy_desc,
                                  const float* x_dev, const kapre_wave_desc* x_desc, const int32_t* lengths_host,
                                  const int32_t* lengths_dev, int frames, float dither, uint64_t seed, float* gx_dev,
                                  const kapre_wave_desc* gx_desc, void* workspace_dev, void* stream) {
    if (!gy_desc || !gx_desc) return kb_fail(KAPRE_E_INVALID, "null argument");
    KbKaldiParams p;
    int rc = kb_kaldi_prepare(p, plan, x_desc, lengths_host, lengths_dev, frames, dither, seed);
    if (rc < 0) return rc;
    if (gx_desc->batch != x_desc->batch || gx_desc->channels != x_desc->channels || gx_desc->length != x_desc->length)
        return kb_fail(KAPRE_E_INVALID, "kaldi: the gradient needs the waveform's shape");
    const long long n = (long long)p.B * p.C * p.L;
    if (n == 0) return 0;
    if (!x_dev || !gx_dev || (p.jobs > 0 && (!gy_dev || !workspace_dev)))
        return kb_fail(KAPRE_E_INVALID, "null data pointer");
    p.x = x_dev; p.x_sb = x_desc->stride_b; p.x_sc = x_desc->stride_c; p.x_sl = x_desc->stride_l;
    p.gx = gx_dev; p.gx_sb = gx_desc->stride_b; p.gx_sc = gx_desc->stride_c; p.gx_sl = gx_desc->stride_l;
    KbLayout L{(char*)workspace_dev};
    float* gc;
    kb_kaldi_layout(L, plan, p.B, p.C, p.T, &p.gf, &gc);
    p.bwd = 1;
    const cudaStream_t st = (cudaStream_t)stream;
    if (p.jobs > 0) {
        p.g = gy_dev; p.g_sb = gy_desc->stride_b; p.g_sc = gy_desc->stride_c; p.g_st = gy_desc->stride_t;
        p.g_sk = gy_desc->stride_f;
        if (plan->cfg.subtract_mean) {
            kapre_spec_desc cd;
            cd.stride_f = 1; cd.stride_t = p.K; cd.stride_c = (int64_t)p.T * p.K; cd.stride_b = cd.stride_c * p.C;
            if ((rc = kb_kaldi_cmn(p, gy_dev, *gy_desc, gc, cd, st))) return rc;
            p.g = gc; p.g_sb = cd.stride_b; p.g_sc = cd.stride_c; p.g_st = cd.stride_t; p.g_sk = cd.stride_f;
        }
        if ((rc = kb_kaldi_launch(p, plan->dev.sm_count, st))) return rc;
    }
    return kb_launch(kb_kaldi_gather_kernel, {.grid = (int)((n + 255) / 256), .block = 256, .st = st}, p, n);
}

}  // extern "C"

// ---- gated loudness (loudness_core.cuh) ----------------------------------------------------------------------------
// Every pass waits for the previous kernel in the stream before touching data, so all three may be launched with PDL.
__global__ void __launch_bounds__(KB_LOUD_WARPS * 32) kb_loud_energy_kernel(const __grid_constant__ KbLoudParams p) {
    extern __shared__ __align__(16) char kb_smem[];
    asm volatile("griddepcontrol.wait;" ::: "memory");
    const int w = (int)(threadIdx.x >> 5);
    const long long tile = (long long)blockIdx.x * KB_LOUD_WARPS + w;
    if (tile < p.tiles) kb_loud_energy_tile(p, kb_smem + w * kb_loud_smem().total, tile);
}
__global__ void __launch_bounds__(KB_LOUD_WARPS * 32) kb_loud_gate_kernel(const __grid_constant__ KbLoudParams p) {
    extern __shared__ __align__(16) char kb_smem[];
    asm volatile("griddepcontrol.wait;" ::: "memory");
    const int w = (int)(threadIdx.x >> 5);
    const long long b = (long long)blockIdx.x * KB_LOUD_WARPS + w;
    if (b < p.B) kb_loud_gate_tile(p, kb_smem + w * kb_loud_smem().total, b);
}
__global__ void __launch_bounds__(KB_LOUD_WARPS * 32) kb_loud_bwd_kernel(const __grid_constant__ KbLoudParams p) {
    extern __shared__ __align__(16) char kb_smem[];
    asm volatile("griddepcontrol.wait;" ::: "memory");
    const int w = (int)(threadIdx.x >> 5);
    const long long tile = (long long)blockIdx.x * KB_LOUD_WARPS + w;
    if (tile < p.tiles) kb_loud_bwd_tile(p, kb_smem + w * kb_loud_smem().total, tile);
}

// Checks a shape, fills the geometry and lays out the two buffers: the workspace (the (B, K, 2C) piece sums) and the
// stats record ((E2, |J2|) per item, then one decision byte per block, in one region).  -1 on a bad argument or an
// overflow.
static int kb_loud_geometry(KbLoudParams& p, int batch, int channels, int length, int gate, int step, KbLayout& ws,
                            KbLayout& rec) {
    if (batch < 0 || channels < 1 || channels > KB_LOUD_MAXC || length < 0 || gate < 1 || step < 1 || step > gate)
        return -1;
    p.B = batch; p.C = channels; p.L = length; p.G = gate; p.S = step;
    kb_loud_setup(p);
    const double w = (double)batch * p.K * 2 * channels * 8.0, s = (double)batch * (16.0 + p.Jmax);
    const double tiles = (double)batch * (p.Kb > p.K ? p.Kb : p.K);
    if (w > 4.0e18 || s > 4.0e18 || tiles / KB_LOUD_WARPS > 2147483647.0) return -1;
    p.part = ws.take<double>(batch, p.K, 2 * channels);
    ws.pad();
    unsigned char* r = rec.take<unsigned char>(batch, 16 + p.Jmax);
    rec.pad();
    p.stats = (double*)r;
    p.mask = r ? r + (int64_t)batch * 16 : nullptr;
    return ws.overflow || rec.overflow ? -1 : 0;
}

static int kb_loud_launch(void (*kernel)(KbLoudParams), long long work, const KbLoudParams& p, cudaStream_t st) {
    return kb_launch(kernel, {.grid = (int)((work + KB_LOUD_WARPS - 1) / KB_LOUD_WARPS), .block = KB_LOUD_WARPS * 32,
                              .smem = KB_LOUD_WARPS * kb_loud_smem().total, .st = st, .pdl = true}, p);
}

extern "C" {

int64_t kapre_loudness_workspace_bytes(int batch, int channels, int length, int gate, int step, int64_t* stats_bytes) {
    KbLoudParams p{};
    KbLayout ws, rec;
    if (kb_loud_geometry(p, batch, channels, length, gate, step, ws, rec) < 0)
        return kb_fail(KAPRE_E_INVALID, "loudness: bad size (%d, %d, %d), gate %d or step %d, or an overflow", batch,
                       channels, length, gate, step);
    if (stats_bytes) *stats_bytes = rec.end;
    return ws.end;
}

int kapre_loudness(const float* y_dev, const kapre_wave_desc* y_desc, const int32_t* lengths_dev, int gate, int step,
                   float* out_dev, void* stats_dev, void* workspace_dev, void* stream) {
    if (!y_desc) return kb_fail(KAPRE_E_INVALID, "null argument");
    KbLoudParams p{};
    KbLayout ws{(char*)workspace_dev}, rec{(char*)stats_dev};
    if (kb_loud_geometry(p, y_desc->batch, y_desc->channels, y_desc->length, gate, step, ws, rec) < 0)
        return kb_fail(KAPRE_E_INVALID, "loudness: bad size (%d, %d, %d), gate %d or step %d, or an overflow",
                       y_desc->batch, y_desc->channels, y_desc->length, gate, step);
    if (p.B == 0) return 0;
    if (!out_dev || !stats_dev || (p.K && (!y_dev || !workspace_dev)))
        return kb_fail(KAPRE_E_INVALID, "null data pointer");
    p.y = y_dev; p.y_sb = y_desc->stride_b; p.y_sc = y_desc->stride_c; p.y_sl = y_desc->stride_l;
    p.len = lengths_dev;
    p.out = out_dev;
    p.tiles = (long long)p.B * p.K;
    const cudaStream_t st = (cudaStream_t)stream;
    int rc;
    if (p.tiles && (rc = kb_loud_launch(kb_loud_energy_kernel, p.tiles, p, st))) return rc;
    return kb_loud_launch(kb_loud_gate_kernel, p.B, p, st);
}

int kapre_loudness_backward(const float* gl_dev, const float* y_dev, const kapre_wave_desc* y_desc,
                            const int32_t* lengths_dev, int gate, int step, const void* stats_dev, float* gy_dev,
                            const kapre_wave_desc* gy_desc, void* stream) {
    if (!y_desc || !gy_desc) return kb_fail(KAPRE_E_INVALID, "null argument");
    KbLoudParams p{};
    KbLayout ws, rec{(char*)const_cast<void*>(stats_dev)};
    if (kb_loud_geometry(p, y_desc->batch, y_desc->channels, y_desc->length, gate, step, ws, rec) < 0)
        return kb_fail(KAPRE_E_INVALID, "loudness: bad size (%d, %d, %d), gate %d or step %d, or an overflow",
                       y_desc->batch, y_desc->channels, y_desc->length, gate, step);
    if (gy_desc->batch != p.B || gy_desc->channels != p.C || gy_desc->length != p.L)
        return kb_fail(KAPRE_E_INVALID, "gradient and signal shapes differ");
    p.tiles = (long long)p.B * p.Kb;
    if (p.tiles == 0) return 0;
    if (!gl_dev || !y_dev || !stats_dev || !gy_dev) return kb_fail(KAPRE_E_INVALID, "null data pointer");
    if ((const void*)gy_dev == (const void*)y_dev) return kb_fail(KAPRE_E_INVALID, "loudness backward cannot run in place");
    p.y = y_dev; p.y_sb = y_desc->stride_b; p.y_sc = y_desc->stride_c; p.y_sl = y_desc->stride_l;
    p.len = lengths_dev;
    p.gl = gl_dev;
    p.gy = gy_dev; p.g_sb = gy_desc->stride_b; p.g_sc = gy_desc->stride_c; p.g_sl = gy_desc->stride_l;
    return kb_loud_launch(kb_loud_bwd_kernel, p.tiles, p, (cudaStream_t)stream);
}

}  // extern "C"

// ---- loudness meter: true peak, loudness series and range (meter_core.cuh) ------------------------------------------
// Every kernel waits for the previous kernel in the stream before touching data, so all may be launched with PDL.
__global__ void __launch_bounds__(KB_TP_WARPS * 32) kb_tp_peak_kernel(const __grid_constant__ KbTpParams p) {
    extern __shared__ __align__(16) char kb_smem[];
    asm volatile("griddepcontrol.wait;" ::: "memory");
    const int w = (int)(threadIdx.x >> 5);
    const long long tile = (long long)blockIdx.x * KB_TP_WARPS + w;
    if (tile < p.tiles) kb_tp_peak_tile(p, kb_smem + w * kb_tp_smem().total, tile);
}
__global__ void __launch_bounds__(KB_TP_WARPS * 32) kb_tp_fold_kernel(const __grid_constant__ KbTpParams p) {
    extern __shared__ __align__(16) char kb_smem[];
    asm volatile("griddepcontrol.wait;" ::: "memory");
    const int w = (int)(threadIdx.x >> 5);
    const long long col = (long long)blockIdx.x * KB_TP_WARPS + w;
    if (col < (long long)p.B * p.C) kb_tp_fold_tile(p, kb_smem + w * kb_tp_smem().total, col);
}
__global__ void __launch_bounds__(256) kb_tp_bwd_kernel(const __grid_constant__ KbTpParams p) {
    asm volatile("griddepcontrol.wait;" ::: "memory");
    const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
    if (i < (long long)p.B * p.C * p.L) kb_tp_bwd(p, i);
}
__global__ void __launch_bounds__(256) kb_meter_series_kernel(const __grid_constant__ KbLoudParams p, float* out,
                                                              double* e) {
    asm volatile("griddepcontrol.wait;" ::: "memory");
    const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
    if (i < (long long)p.B * p.Jmax) kb_meter_series(p, out, e, i);
}
__global__ void __launch_bounds__(KB_LOUD_WARPS * 32) kb_meter_lra_kernel(const __grid_constant__ KbLoudParams p,
                                                                          double* e, float* out) {
    extern __shared__ __align__(16) char kb_smem[];
    asm volatile("griddepcontrol.wait;" ::: "memory");
    const int w = (int)(threadIdx.x >> 5);
    const long long b = (long long)blockIdx.x * KB_LOUD_WARPS + w;
    if (b < p.B) kb_meter_lra_tile(p, e, out, kb_smem + w * kb_lra_smem().total, b);
}

// Checks a shape, fills the geometry (taps may be null when only sizing) and lays out the workspace (the (B, C, nseg)
// tile keys) and the stats record ((B, C) z[t*], then (B, C) t*).  -1 on a bad argument or an overflow.
static int kb_tp_geometry(KbTpParams& p, int batch, int channels, int length, const float* taps, KbLayout& ws,
                          KbLayout& rec) {
    if (batch < 0 || channels < 1 || length < 0 || length > KB_TP_MAX_LEN) return -1;
    p.B = batch; p.C = channels; p.L = length;
    float zero[KB_TP_TAPS] = {};
    kb_tp_setup(p, taps ? taps : zero);
    const double cols = (double)batch * channels;
    if (cols * p.nseg / KB_TP_WARPS > 2147483647.0 || cols * length / 256.0 > 2147483647.0) return -1;
    p.tiles = (long long)batch * channels * p.nseg;
    p.key = ws.take<unsigned long long>(batch, channels, p.nseg);
    ws.pad();
    p.zs = rec.take<float>(batch, channels);
    p.ts = rec.take<unsigned>(batch, channels);
    rec.pad();
    return ws.overflow || rec.overflow ? -1 : 0;
}

static int kb_tp_launch(void (*kernel)(KbTpParams), long long work, const KbTpParams& p, cudaStream_t st) {
    return kb_launch(kernel, {.grid = (int)((work + KB_TP_WARPS - 1) / KB_TP_WARPS), .block = KB_TP_WARPS * 32,
                              .smem = KB_TP_WARPS * kb_tp_smem().total, .st = st, .pdl = true}, p);
}

// The loudness-stats workspace: kapre_loudness's piece sums and stats record for the 400 ms blocks, the same for the
// 3 s windows, and the (B, J_S) float64 window energies the range pass reads.
static int kb_meter_geometry(KbLoudParams& pm, KbLoudParams& ps, int batch, int channels, int length, int gate,
                             int step, int gate3, KbLayout& ws, double** e) {
    if (gate3 < gate) return -1;
    if (kb_loud_geometry(pm, batch, channels, length, gate, step, ws, ws) < 0) return -1;
    if (kb_loud_geometry(ps, batch, channels, length, gate3, step, ws, ws) < 0) return -1;
    *e = ws.take<double>(batch, ps.Jmax);
    ws.pad();
    if ((double)batch * (pm.Jmax > ps.Jmax ? pm.Jmax : ps.Jmax) / 256.0 > 2147483647.0) return -1;
    return ws.overflow ? -1 : 0;
}

extern "C" {

int64_t kapre_true_peak_workspace_bytes(int batch, int channels, int length, int64_t* stats_bytes) {
    KbTpParams p{};
    KbLayout ws, rec;
    if (kb_tp_geometry(p, batch, channels, length, nullptr, ws, rec) < 0)
        return kb_fail(KAPRE_E_INVALID, "true_peak: bad size (%d, %d, %d) or an overflow", batch, channels, length);
    if (stats_bytes) *stats_bytes = rec.end;
    return ws.end;
}

int kapre_true_peak(const float* x_dev, const kapre_wave_desc* x_desc, const int32_t* lengths_dev,
                    const float* taps_host, float* out_dev, void* stats_dev, void* workspace_dev, void* stream) {
    if (!x_desc || !taps_host) return kb_fail(KAPRE_E_INVALID, "null argument");
    KbTpParams p{};
    KbLayout ws{(char*)workspace_dev}, rec{(char*)stats_dev};
    if (kb_tp_geometry(p, x_desc->batch, x_desc->channels, x_desc->length, taps_host, ws, rec) < 0)
        return kb_fail(KAPRE_E_INVALID, "true_peak: bad size (%d, %d, %d) or an overflow", x_desc->batch,
                       x_desc->channels, x_desc->length);
    if (p.B == 0) return 0;
    if (!out_dev || !stats_dev || (p.tiles && (!x_dev || !workspace_dev)))
        return kb_fail(KAPRE_E_INVALID, "null data pointer");
    p.x = x_dev; p.x_sb = x_desc->stride_b; p.x_sc = x_desc->stride_c; p.x_sl = x_desc->stride_l;
    p.len = lengths_dev;
    p.out = out_dev;
    const cudaStream_t st = (cudaStream_t)stream;
    int rc;
    if (p.tiles && (rc = kb_tp_launch(kb_tp_peak_kernel, p.tiles, p, st))) return rc;
    return kb_tp_launch(kb_tp_fold_kernel, (long long)p.B * p.C, p, st);
}

int kapre_true_peak_backward(const float* g_dev, const int32_t* lengths_dev, const float* taps_host,
                             const void* stats_dev, float* gx_dev, const kapre_wave_desc* gx_desc, void* stream) {
    if (!gx_desc || !taps_host) return kb_fail(KAPRE_E_INVALID, "null argument");
    KbTpParams p{};
    KbLayout ws, rec{(char*)const_cast<void*>(stats_dev)};
    if (kb_tp_geometry(p, gx_desc->batch, gx_desc->channels, gx_desc->length, taps_host, ws, rec) < 0)
        return kb_fail(KAPRE_E_INVALID, "true_peak: bad size (%d, %d, %d) or an overflow", gx_desc->batch,
                       gx_desc->channels, gx_desc->length);
    const long long n = (long long)p.B * p.C * p.L;
    if (n == 0) return 0;
    if (!g_dev || !stats_dev || !gx_dev) return kb_fail(KAPRE_E_INVALID, "null data pointer");
    p.len = lengths_dev;
    p.g = g_dev;
    p.gx = gx_dev; p.g_sb = gx_desc->stride_b; p.g_sc = gx_desc->stride_c; p.g_sl = gx_desc->stride_l;
    return kb_launch(kb_tp_bwd_kernel, {.grid = (int)((n + 255) / 256), .block = 256, .st = (cudaStream_t)stream,
                                        .pdl = true}, p);
}

int64_t kapre_loudness_stats_workspace_bytes(int batch, int channels, int length, int gate, int step, int gate3) {
    KbLoudParams pm{}, ps{};
    KbLayout ws;
    double* e;
    if (kb_meter_geometry(pm, ps, batch, channels, length, gate, step, gate3, ws, &e) < 0)
        return kb_fail(KAPRE_E_INVALID, "loudness_stats: bad size (%d, %d, %d), gate %d, step %d or gate3 %d, or an "
                       "overflow", batch, channels, length, gate, step, gate3);
    return ws.end;
}

int kapre_loudness_stats(const float* y_dev, const kapre_wave_desc* y_desc, const int32_t* lengths_dev, int gate,
                         int step, int gate3, float* integrated_dev, float* momentary_dev, float* short_term_dev,
                         float* lra_dev, void* workspace_dev, void* stream) {
    if (!y_desc) return kb_fail(KAPRE_E_INVALID, "null argument");
    KbLoudParams pm{}, ps{};
    KbLayout ws{(char*)workspace_dev};
    double* e;
    if (kb_meter_geometry(pm, ps, y_desc->batch, y_desc->channels, y_desc->length, gate, step, gate3, ws, &e) < 0)
        return kb_fail(KAPRE_E_INVALID, "loudness_stats: bad size (%d, %d, %d), gate %d, step %d or gate3 %d, or an "
                       "overflow", y_desc->batch, y_desc->channels, y_desc->length, gate, step, gate3);
    if (pm.B == 0) return 0;
    if (!integrated_dev || !lra_dev || !workspace_dev || (pm.Jmax && !momentary_dev) || (ps.Jmax && !short_term_dev) ||
        (pm.K && !y_dev))
        return kb_fail(KAPRE_E_INVALID, "null data pointer");
    for (KbLoudParams* p : {&pm, &ps}) {
        p->y = y_dev; p->y_sb = y_desc->stride_b; p->y_sc = y_desc->stride_c; p->y_sl = y_desc->stride_l;
        p->len = lengths_dev;
        p->tiles = (long long)p->B * p->K;
    }
    pm.out = integrated_dev;
    const cudaStream_t st = (cudaStream_t)stream;
    int rc;
    // integrated loudness: kapre_loudness's two passes as they are
    if (pm.tiles && (rc = kb_loud_launch(kb_loud_energy_kernel, pm.tiles, pm, st))) return rc;
    if ((rc = kb_loud_launch(kb_loud_gate_kernel, pm.B, pm, st))) return rc;
    const long long nm = (long long)pm.B * pm.Jmax, ns = (long long)ps.B * ps.Jmax;
    if (nm && (rc = kb_launch(kb_meter_series_kernel, {.grid = (int)((nm + 255) / 256), .block = 256, .st = st,
                                                       .pdl = true}, pm, momentary_dev, (double*)nullptr)))
        return rc;
    if (ps.tiles && (rc = kb_loud_launch(kb_loud_energy_kernel, ps.tiles, ps, st))) return rc;
    if (ns && (rc = kb_launch(kb_meter_series_kernel, {.grid = (int)((ns + 255) / 256), .block = 256, .st = st,
                                                       .pdl = true}, ps, short_term_dev, e)))
        return rc;
    return kb_launch(kb_meter_lra_kernel, {.grid = (int)((ps.B + KB_LOUD_WARPS - 1) / KB_LOUD_WARPS),
                                           .block = KB_LOUD_WARPS * 32, .smem = KB_LOUD_WARPS * kb_lra_smem().total,
                                           .st = st, .pdl = true}, ps, e, lra_dev);
}

}  // extern "C"

// ---- constant-Q transform (cqt_core.cuh) ------------------------------------------------------------------------------
__global__ void __launch_bounds__(KB_CQT_THREADS) kb_cqt_fwd_kernel(const __grid_constant__ KbCqtParams p) {
    extern __shared__ __align__(16) char kb_smem[];
    kb_cqt_fwd_cta(p, kb_smem, blockIdx.x, gridDim.x);
}
__global__ void __launch_bounds__(KB_CQT_BWD_THREADS) kb_cqt_bwd_kernel(const __grid_constant__ KbCqtParams p) {
    extern __shared__ __align__(16) char kb_smem[];
    kb_cqt_bwd_cta(p, kb_smem, blockIdx.x, gridDim.x);
}

struct kapre_cqt_plan {
    kapre_cqt_config cfg;
    KbCqtParams geo;                        // octaves and segments (per-call fields unset)
    DevInfo dev;
    KbTables tables;
    float2* tab = nullptr;
    float2* btab = nullptr;
    kapre_resample_plan* rs = nullptr;      // the 2:1 decimator
};

static const int KB_CQT_FWD_SMEM = KB_CQT_TAB_BYTES + KB_CQT_SPAN_FLOATS * 4;

// Level i's length: L_0 = length, L_{i+1} = ceil(L_i / 2).
static long long kb_cqt_level_len(long long L, int i) {
    for (int k = 0; k < i; ++k) L = (L + 1) / 2;
    return L;
}

// The forward workspace: the (B, C, L_i) pyramid levels 1 .. n_oct-1, which the backward reads too.
static void kb_cqt_layout(KbLayout& L, int n_oct, int batch, int channels, int length, float** lvl) {
    for (int i = 1; i < n_oct; ++i) lvl[i] = L.take<float>(batch, channels, kb_cqt_level_len(length, i));
    L.pad();
}

// The backward workspace: the adjoint's levels 1 .. n_oct-1, then its resampling adjoints at levels 0 .. n_oct-2.
static void kb_cqt_backward_layout(KbLayout& L, int n_oct, int batch, int channels, int length, float** glvl,
                                   float** rlvl) {
    for (int i = 1; i < n_oct; ++i) glvl[i] = L.take<float>(batch, channels, kb_cqt_level_len(length, i));
    for (int i = 0; i + 1 < n_oct; ++i) rlvl[i] = L.take<float>(batch, channels, kb_cqt_level_len(length, i));
    L.pad();
}

static int kb_cqt_check_shape(const kapre_cqt_plan* plan, const kapre_wave_desc* xd) {
    if (!plan || !xd) return kb_fail(KAPRE_E_INVALID, "null argument");
    if (xd->batch < 0 || xd->channels < 0 || xd->length < 0)
        return kb_fail(KAPRE_E_INVALID, "cqt: negative size (%d, %d, %d)", xd->batch, xd->channels, xd->length);
    if ((double)xd->batch * xd->channels * (xd->length + 1.0) * 3.0 > 4.0e18)
        return kb_fail(KAPRE_E_INVALID, "cqt: size overflow");
    return kb_check_device(plan->dev);
}

// Common fields: levels (level 0 = x, the others contiguous (B, C, L_i) in the workspace) and sizes.
static KbCqtParams kb_cqt_params(const kapre_cqt_plan* plan, const float* x, const kapre_wave_desc* xd, const void* ws) {
    KbCqtParams p = plan->geo;
    p.B = xd->batch; p.C = xd->channels;
    p.M = 1 + xd->length / plan->cfg.hop_length;
    p.tab = plan->tab; p.btab = plan->btab;
    KbLayout L{(char*)const_cast<void*>(ws)};
    float* lvl[KB_CQT_MAX_OCT];
    kb_cqt_layout(L, p.n_oct, p.B, p.C, xd->length, lvl);
    for (int i = 0; i < p.n_oct; ++i) {
        KbCqtOct& o = p.oct[i];
        o.L = (int)kb_cqt_level_len(xd->length, i);
        if (i == 0) { o.y = x; o.y_sb = xd->stride_b; o.y_sc = xd->stride_c; o.y_sl = xd->stride_l; }
        else { o.y = lvl[i]; o.y_sb = (long long)p.C * o.L; o.y_sc = o.L; o.y_sl = 1; }
    }
    return p;
}

static kapre_wave_desc kb_cqt_level_desc(int B, int C, int L) {
    kapre_wave_desc d;
    d.batch = B; d.channels = C; d.length = L;
    d.stride_b = (int64_t)C * L; d.stride_c = L; d.stride_l = 1;
    return d;
}

extern "C" {

int kapre_cqt_plan_create(const kapre_cqt_config* cfg, const float* taps_host, const float* decim_taps_host,
                          int n_decim_taps, kapre_cqt_plan** out) {
    if (!cfg || !taps_host || !decim_taps_host || !out) return kb_fail(KAPRE_E_INVALID, "null argument");
    *out = nullptr;
    if (cfg->n_bins < 1 || cfg->bins_per_octave < 1 || cfg->hop_length < 1)
        return kb_fail(KAPRE_E_INVALID, "cqt: n_bins %d, bins_per_octave %d and hop_length %d must be positive",
                       cfg->n_bins, cfg->bins_per_octave, cfg->hop_length);
    const int n_oct = (cfg->n_bins + cfg->bins_per_octave - 1) / cfg->bins_per_octave;
    if (n_oct > KAPRE_CQT_MAX_OCTAVES)
        return kb_fail(KAPRE_E_UNSUPPORTED, "cqt: %d octaves exceed the limit of %d", n_oct, KAPRE_CQT_MAX_OCTAVES);
    if (cfg->hop_length % (1 << (n_oct - 1)))
        return kb_fail(KAPRE_E_INVALID, "cqt: hop_length %d must be a multiple of 2^(octaves - 1) = %d",
                       cfg->hop_length, 1 << (n_oct - 1));
    for (int i = 0; i < n_oct; ++i)
        if (cfg->taps[i] < 1 || cfg->taps[i] > KAPRE_CQT_MAX_TAPS)
            return kb_fail(cfg->taps[i] < 1 ? KAPRE_E_INVALID : KAPRE_E_UNSUPPORTED,
                           "cqt: octave %d's filters of %d taps exceed the limit of %d taps", i, cfg->taps[i],
                           KAPRE_CQT_MAX_TAPS);
    kapre_cqt_plan* pl = new kapre_cqt_plan();
    pl->cfg = *cfg;
    std::vector<float2> tab, btab;
    const int bad = kb_cqt_build(cfg->n_bins, cfg->bins_per_octave, cfg->hop_length, cfg->taps, taps_host, pl->geo,
                                 tab, btab);
    int rc = 0;
    if (bad) {
        delete pl;
        return kb_fail(KAPRE_E_UNSUPPORTED, "cqt: octave %d takes the transform past the kernel's limit of %d (octave, bin "
                       "group) segments (a group holds the bins whose taps fit %d B)", bad - 1, KB_CQT_MAX_SEGS,
                       KB_CQT_TAB_BYTES);
    }
    for (const float2& v : tab)
        if (!std::isfinite(v.x) || !std::isfinite(v.y)) { delete pl; return kb_fail(KAPRE_E_INVALID, "cqt: non-finite tap"); }
    KbTableUpload tb;
    tb.add(tab, &pl->tab); tb.add(btab, &pl->btab);
    if ((rc = kb_dev_info(&pl->dev)) || (rc = tb.upload(pl->tables, "cqt")) ||
        (rc = kapre_resample_plan_create(1, 2, decim_taps_host, n_decim_taps, &pl->rs))) {
        delete pl;
        return rc;
    }
    *out = pl;
    return 0;
}

void kapre_cqt_plan_destroy(kapre_cqt_plan* plan) {
    if (!plan) return;
    kapre_resample_plan_destroy(plan->rs);
    delete plan;
}

int kapre_cqt_num_frames(const kapre_cqt_plan* plan, int length) {
    if (!plan) return kb_fail(KAPRE_E_INVALID, "null plan");
    if (length < 0) return kb_fail(KAPRE_E_INVALID, "negative length");
    return 1 + length / plan->cfg.hop_length;
}

int64_t kapre_cqt_workspace_bytes(const kapre_cqt_plan* plan, int batch, int channels, int length, int backward) {
    if (!plan) return kb_fail(KAPRE_E_INVALID, "null plan");
    if (batch < 0 || channels < 0 || length < 0) return kb_fail(KAPRE_E_INVALID, "cqt: negative size");
    if ((double)batch * channels * (length + 1.0) * 3.0 > 4.0e18) return kb_fail(KAPRE_E_INVALID, "cqt: size overflow");
    KbLayout L;
    float *a[KB_CQT_MAX_OCT], *b[KB_CQT_MAX_OCT];
    if (backward) kb_cqt_backward_layout(L, plan->geo.n_oct, batch, channels, length, a, b);
    else kb_cqt_layout(L, plan->geo.n_oct, batch, channels, length, a);
    return L.bytes("cqt");
}

int kapre_cqt(const kapre_cqt_plan* plan, const float* x_dev, const kapre_wave_desc* x_desc, int magnitude,
              void* out_dev, const kapre_spec_desc* out_desc, void* workspace_dev, void* stream) {
    int rc = kb_cqt_check_shape(plan, x_desc);
    if (rc) return rc;
    if (!out_desc) return kb_fail(KAPRE_E_INVALID, "null argument");
    if (magnitude != 0 && magnitude != 1) return kb_fail(KAPRE_E_INVALID, "cqt: magnitude must be 0 or 1");
    if ((long long)x_desc->batch * x_desc->channels == 0) return 0;
    if (!x_dev || !out_dev || (plan->geo.n_oct > 1 && !workspace_dev)) return kb_fail(KAPRE_E_INVALID, "null data pointer");
    KbCqtParams p = kb_cqt_params(plan, x_dev, x_desc, workspace_dev);
    p.n_threads = KB_CQT_THREADS;
    p.mag = magnitude;
    p.out = out_dev; p.o_sb = out_desc->stride_b; p.o_sc = out_desc->stride_c; p.o_st = out_desc->stride_t;
    p.o_sk = out_desc->stride_f;
    if (!kb_cqt_setup(p)) return kb_fail(KAPRE_E_INVALID, "cqt: too many tiles");
    const cudaStream_t st = (cudaStream_t)stream;
    for (int i = 1; i < p.n_oct; ++i) {
        const KbCqtOct& a = p.oct[i - 1];
        const kapre_wave_desc ad = i == 1 ? *x_desc : kb_cqt_level_desc(p.B, p.C, a.L);
        const kapre_wave_desc yd = kb_cqt_level_desc(p.B, p.C, p.oct[i].L);
        if (yd.length == 0) continue;
        if ((rc = kb_resample_launch(plan->rs, a.y, &ad, const_cast<float*>(p.oct[i].y), &yd, stream))) return rc;
    }
    int grid;
    if ((rc = kb_resident_grid(kb_cqt_fwd_kernel, "cqt_fwd", KB_CQT_THREADS, KB_CQT_FWD_SMEM, p.jobs,
                               plan->dev.sm_count, &grid)))
        return rc;
    return kb_launch(kb_cqt_fwd_kernel, {.grid = grid, .block = KB_CQT_THREADS, .smem = KB_CQT_FWD_SMEM, .st = st,
                                         .timed = true}, p);
}

int kapre_cqt_backward(const kapre_cqt_plan* plan, const float* x_dev, const kapre_wave_desc* x_desc,
                       const void* fwd_workspace_dev, const void* g_dev, const kapre_spec_desc* g_desc, int magnitude,
                       float* gx_dev, const kapre_wave_desc* gx_desc, void* workspace_dev, void* stream) {
    int rc = kb_cqt_check_shape(plan, x_desc);
    if (rc) return rc;
    if (!g_desc || !gx_desc) return kb_fail(KAPRE_E_INVALID, "null argument");
    if (magnitude != 0 && magnitude != 1) return kb_fail(KAPRE_E_INVALID, "cqt: magnitude must be 0 or 1");
    if (gx_desc->batch != x_desc->batch || gx_desc->channels != x_desc->channels || gx_desc->length != x_desc->length)
        return kb_fail(KAPRE_E_INVALID, "cqt: the gradient needs the waveform's shape");
    const long long bc = (long long)x_desc->batch * x_desc->channels;
    if (bc * x_desc->length == 0) return 0;
    const int n_oct = plan->geo.n_oct;
    if (!g_dev || !gx_dev || (n_oct > 1 && !workspace_dev) || (magnitude && (!x_dev || (n_oct > 1 && !fwd_workspace_dev))))
        return kb_fail(KAPRE_E_INVALID, "null data pointer");
    KbCqtParams p = kb_cqt_params(plan, x_dev, x_desc, fwd_workspace_dev);
    p.n_threads = KB_CQT_BWD_THREADS;
    p.mag = magnitude;
    p.g = g_dev; p.g_sb = g_desc->stride_b; p.g_sc = g_desc->stride_c; p.g_st = g_desc->stride_t;
    p.g_sk = g_desc->stride_f;
    KbLayout L{(char*)workspace_dev};
    float *glvl[KB_CQT_MAX_OCT], *rlvl[KB_CQT_MAX_OCT];
    kb_cqt_backward_layout(L, n_oct, p.B, p.C, x_desc->length, glvl, rlvl);
    const cudaStream_t st = (cudaStream_t)stream;
    const int smem = kb_cqt_bwd_smem();
    KbLaunchReports reports;    // every octave's launch and the resampling launches between them
    // lowest octave first: g_i = adjoint_i(G) + R^T g_{i+1}
    for (int i = n_oct - 1; i >= 0; --i) {
        const KbCqtOct& o = p.oct[i];
        if (o.L == 0) continue;
        p.bo = i;
        p.add = nullptr;
        if (i + 1 < n_oct && p.oct[i + 1].L > 0) {
            const kapre_wave_desc gd = kb_cqt_level_desc(p.B, p.C, p.oct[i + 1].L);
            const kapre_wave_desc rd = kb_cqt_level_desc(p.B, p.C, o.L);
            if ((rc = kapre_resample_backward(plan->rs, glvl[i + 1], &gd, rlvl[i], &rd, stream))) return rc;
            reports.add();
            p.add = rlvl[i];
        }
        if (i == 0) { p.gy = gx_dev; p.gy_sb = gx_desc->stride_b; p.gy_sc = gx_desc->stride_c; p.gy_sl = gx_desc->stride_l; }
        else { p.gy = glvl[i]; p.gy_sb = (long long)p.C * o.L; p.gy_sc = o.L; p.gy_sl = 1; }
        const long long tiles = bc * ((o.L + o.TS - 1) / o.TS);
        int grid;
        if ((rc = kb_resident_grid(kb_cqt_bwd_kernel, "cqt_bwd", KB_CQT_BWD_THREADS, smem, tiles, plan->dev.sm_count,
                                   &grid)))
            return rc;
        if ((rc = kb_launch(kb_cqt_bwd_kernel, {.grid = grid, .block = KB_CQT_BWD_THREADS, .smem = smem, .st = st}, p)))
            return rc;
        reports.add();
    }
    return 0;
}

}  // extern "C"

// ---- pitch tracking (pitch_core.cuh) ------------------------------------------------------------------------------
__global__ void __launch_bounds__(KB_PITCH_THREADS) kb_pitch_kernel(const __grid_constant__ KbPitchParams p) {
    extern __shared__ __align__(16) char kb_smem[];
    kb_pitch_cta(p, kb_smem, blockIdx.x, gridDim.x);
}
__global__ void __launch_bounds__(KB_VIT_THREADS) kb_viterbi_kernel(const __grid_constant__ KbVitParams p) {
    extern __shared__ __align__(16) char kb_smem[];
    kb_vit_cta(p, kb_smem, reinterpret_cast<float*>(kb_smem) + 6 * p.n + p.w + 4, blockIdx.x, gridDim.x);
}

struct kapre_pitch_plan {
    kapre_pitch_config cfg;
    KbPitchParams geo;                      // tiling and tables (per-call fields unset)
    KbVitParams vit;
    DevInfo dev;
    KbTables tables;
};

// One pYIN table, converted to T and checked finite after the conversion.
template <typename T>
static int kb_pitch_table(KbTableUpload& tb, const double* src, size_t n, const T** dst) {
    std::vector<T> h(n);
    for (size_t i = 0; i < n; ++i) {
        h[i] = (T)src[i];
        if (!std::isfinite((double)h[i])) return kb_fail(KAPRE_E_INVALID, "pitch: non-finite table entry");
    }
    tb.add(h, dst);
    return 0;
}

static int kb_pitch_frames(const kapre_pitch_config& c, long long length) {
    const long long lp = length + (c.center ? 2LL * (c.frame_length / 2) : 0);
    return lp < c.frame_length ? 0 : (int)(1 + (lp - c.frame_length) / c.hop_length);
}

static int kb_pitch_check_shape(const kapre_pitch_plan* plan, const kapre_wave_desc* xd) {
    if (!plan || !xd) return kb_fail(KAPRE_E_INVALID, "null argument");
    if (xd->batch < 0 || xd->channels < 0 || xd->length < 0)
        return kb_fail(KAPRE_E_INVALID, "pitch: negative size (%d, %d, %d)", xd->batch, xd->channels, xd->length);
    return kb_check_device(plan->dev);
}

// The pYIN workspace: per frame the candidate count, probabilities and pitch bins, then the Viterbi back-pointers.
struct KbPyinWs {
    int* cand_n;
    float* cand_p;
    unsigned short *cand_bin, *bp;
};

static KbPyinWs kb_pyin_layout(KbLayout& L, const kapre_pitch_plan* plan, int batch, int channels, int M) {
    KbPyinWs w;
    w.cand_n = L.take<int>(batch, channels, M);
    w.cand_p = L.take<float>(batch, channels, M, plan->geo.cmax);
    w.cand_bin = L.take<unsigned short>(batch, channels, M, plan->geo.cmax);
    w.bp = L.take<unsigned short>(batch, channels, M, 2 * plan->cfg.n_pitch);
    return w;
}

// The difference-function launch of kapre_yin (pyin = 0) and kapre_pyin.
static int kb_pitch_launch(const kapre_pitch_plan* plan, const float* x, const kapre_wave_desc* xd, float* out,
                           const kapre_frames_desc* od, float* cm, const kapre_spec_desc* cd, void* ws, cudaStream_t st) {
    KbPitchParams p = plan->geo;
    p.B = xd->batch; p.C = xd->channels; p.L = xd->length;
    p.M = kb_pitch_frames(plan->cfg, xd->length);
    p.x = x; p.x_sb = xd->stride_b; p.x_sc = xd->stride_c; p.x_sl = xd->stride_l;
    p.out = out; p.o_sb = od->stride_b; p.o_sc = od->stride_c; p.o_st = od->stride_t;
    p.cm = cm;
    if (cm) { p.c_sb = cd->stride_b; p.c_sc = cd->stride_c; p.c_st = cd->stride_t; p.c_sk = cd->stride_f; }
    if (p.pyin) {
        KbLayout L{(char*)ws};
        const KbPyinWs w = kb_pyin_layout(L, plan, p.B, p.C, p.M);
        p.cand_n = w.cand_n; p.cand_p = w.cand_p; p.cand_bin = w.cand_bin;
    }
    if (!kb_pitch_setup(p)) return kb_fail(KAPRE_E_INVALID, "pitch: too many tiles");
    int grid, rc;
    if ((rc = kb_resident_grid(kb_pitch_kernel, "pitch", KB_PITCH_THREADS, p.smem, p.jobs, plan->dev.sm_count, &grid)))
        return rc;
    return kb_launch(kb_pitch_kernel, {.grid = grid, .block = KB_PITCH_THREADS, .smem = p.smem, .st = st,
                                       .timed = true}, p);
}

extern "C" {

int kapre_pitch_plan_create(const kapre_pitch_config* cfg, const kapre_pitch_tables* tab, kapre_pitch_plan** out) {
    if (!cfg || !out) return kb_fail(KAPRE_E_INVALID, "null argument");
    *out = nullptr;
    const kapre_pitch_config& c = *cfg;
    if (!(c.sample_rate > 0.0f) || c.frame_length < 2 || c.win_length < 1 || c.hop_length < 1 ||
        c.win_length >= c.frame_length || c.min_period < 1 || c.max_period < c.min_period + 2 ||
        c.max_period > c.frame_length - c.win_length - 1)
        return kb_fail(KAPRE_E_INVALID, "pitch: bad geometry (frame %d, window %d, hop %d, periods %d .. %d)",
                       c.frame_length, c.win_length, c.hop_length, c.min_period, c.max_period);
    if (c.frame_length > KAPRE_PITCH_MAX_FRAME)
        return kb_fail(KAPRE_E_UNSUPPORTED, "pitch: frame_length %d exceeds the limit of %d", c.frame_length,
                       KAPRE_PITCH_MAX_FRAME);
    if (tab) {
        if (c.n_thresholds < 1 || c.n_pitch < 1 || c.band_width < 1)
            return kb_fail(KAPRE_E_INVALID, "pyin: n_thresholds, n_pitch and band_width must be positive");
        if (c.n_thresholds > KAPRE_PITCH_MAX_THRESHOLDS || c.n_pitch > KAPRE_PITCH_MAX_BINS ||
            c.band_width > KAPRE_PITCH_MAX_BAND)
            return kb_fail(KAPRE_E_UNSUPPORTED, "pyin: %d thresholds, %d pitch bins or a band of %d exceed the limits "
                           "(%d, %d, %d)", c.n_thresholds, c.n_pitch, c.band_width, KAPRE_PITCH_MAX_THRESHOLDS,
                           KAPRE_PITCH_MAX_BINS, KAPRE_PITCH_MAX_BAND);
        if (!tab->beta_probs || !tab->boltzmann_pow || !tab->boltzmann_norm || !tab->no_trough_bonus ||
            (c.n_pitch > 1 && !tab->period_edges) || !tab->freqs || !tab->log_triangle || !tab->log_row_norm)
            return kb_fail(KAPRE_E_INVALID, "pyin: null table");
    }
    kapre_pitch_plan* pl = new kapre_pitch_plan();
    pl->cfg = c;
    KbPitchParams& g = pl->geo;
    g = KbPitchParams{};
    g.F = c.frame_length; g.W = c.win_length; g.h = c.hop_length; g.pad = c.center ? c.frame_length / 2 : 0;
    g.min_p = c.min_period; g.max_p = c.max_period;
    g.sr = c.sample_rate; g.thresh = c.trough_threshold;
    g.pyin = tab ? 1 : 0;
    g.n_thr = tab ? c.n_thresholds : 0;
    g.n_pitch = tab ? c.n_pitch : 0;
    if (!kb_pitch_tiling(g)) {
        delete pl;
        return kb_fail(KAPRE_E_UNSUPPORTED, "pitch: one frame does not fit the kernel's shared memory");
    }
    KbTableUpload tb;
    int rc = kb_dev_info(&pl->dev);
    if (!rc && g.smem > pl->dev.smem_optin) rc = kb_fail(KAPRE_E_UNSUPPORTED, "pitch: %d B of shared memory", g.smem);
    if (!rc && tab) {
        KbVitParams& v = pl->vit;
        v = KbVitParams{};
        v.n = c.n_pitch; v.w = c.band_width; v.half = c.band_width / 2;
        v.cmax = g.cmax;
        v.ls = c.log_stay; v.lw = c.log_switch; v.lpv = c.log_init_voiced; v.lpu = c.log_init_unvoiced;
        v.fill = c.fill_na;
        v.nt = (c.n_pitch + 31) / 32 * 32;
        if (v.nt > KB_VIT_THREADS) v.nt = KB_VIT_THREADS;
        if (kb_vit_smem(v.n, v.w) > pl->dev.smem_optin)
            rc = kb_fail(KAPRE_E_UNSUPPORTED, "pyin: %d pitch bins and a band of %d need %d B of shared memory", v.n,
                         v.w, kb_vit_smem(v.n, v.w));
        const double* edges = tab->period_edges;
        std::vector<double> one(1, 0.0);
        if (c.n_pitch == 1) edges = one.data();
        if (!rc) rc = kb_pitch_table<float>(tb, tab->beta_probs, c.n_thresholds, &g.beta);
        if (!rc) rc = kb_pitch_table<float>(tb, tab->boltzmann_pow, g.cmax + 1, &g.bpow);
        if (!rc) rc = kb_pitch_table<float>(tb, tab->boltzmann_norm, g.cmax + 1, &g.bnorm);
        if (!rc) rc = kb_pitch_table<float>(tb, tab->no_trough_bonus, c.n_thresholds + 1, &g.bonus);
        if (!rc) rc = kb_pitch_table<double>(tb, edges, c.n_pitch > 1 ? c.n_pitch - 1 : 1, &g.edges);
        if (!rc) rc = kb_pitch_table<float>(tb, tab->freqs, c.n_pitch, &v.freq);
        if (!rc) rc = kb_pitch_table<float>(tb, tab->log_triangle, c.band_width, &v.ltri);
        if (!rc) rc = kb_pitch_table<float>(tb, tab->log_row_norm, c.n_pitch, &v.lnorm);
    }
    if (!rc) rc = tb.upload(pl->tables, "pitch");
    if (rc) {
        delete pl;
        return rc;
    }
    *out = pl;
    return 0;
}

void kapre_pitch_plan_destroy(kapre_pitch_plan* plan) { delete plan; }

int kapre_pitch_num_frames(const kapre_pitch_plan* plan, int length) {
    if (!plan) return kb_fail(KAPRE_E_INVALID, "null plan");
    if (length < 0) return kb_fail(KAPRE_E_INVALID, "negative length");
    return kb_pitch_frames(plan->cfg, length);
}

int64_t kapre_pitch_workspace_bytes(const kapre_pitch_plan* plan, int batch, int channels, int length) {
    if (!plan) return kb_fail(KAPRE_E_INVALID, "null plan");
    if (batch < 0 || channels < 0 || length < 0) return kb_fail(KAPRE_E_INVALID, "pitch: negative size");
    if (!plan->geo.pyin) return 0;
    KbLayout L;
    kb_pyin_layout(L, plan, batch, channels, kb_pitch_frames(plan->cfg, length));
    return L.bytes("pyin");
}

int kapre_yin(const kapre_pitch_plan* plan, const float* x_dev, const kapre_wave_desc* x_desc, float* f0_dev,
              const kapre_frames_desc* f0_desc, float* cmndf_dev, const kapre_spec_desc* cmndf_desc, void* stream) {
    int rc = kb_pitch_check_shape(plan, x_desc);
    if (rc) return rc;
    if (!f0_desc || (cmndf_dev && !cmndf_desc)) return kb_fail(KAPRE_E_INVALID, "null argument");
    if ((long long)x_desc->batch * x_desc->channels * kb_pitch_frames(plan->cfg, x_desc->length) == 0) return 0;
    if (!x_dev || !f0_dev) return kb_fail(KAPRE_E_INVALID, "null data pointer");
    KbPitchParams geo = plan->geo;
    if (geo.pyin) {   // a pYIN plan also serves YIN: the same tiling without the pYIN scratch
        kapre_pitch_plan tmp;
        tmp.cfg = plan->cfg; tmp.dev = plan->dev; tmp.geo = geo;
        tmp.geo.pyin = 0;
        tmp.geo.n_thr = 0;
        kb_pitch_tiling(tmp.geo);
        return kb_pitch_launch(&tmp, x_dev, x_desc, f0_dev, f0_desc, cmndf_dev, cmndf_desc, nullptr,
                               (cudaStream_t)stream);
    }
    return kb_pitch_launch(plan, x_dev, x_desc, f0_dev, f0_desc, cmndf_dev, cmndf_desc, nullptr, (cudaStream_t)stream);
}

int kapre_pyin(const kapre_pitch_plan* plan, const float* x_dev, const kapre_wave_desc* x_desc, float* f0_dev,
               uint8_t* voiced_flag_dev, float* voiced_prob_dev, const kapre_frames_desc* out_desc, float* cmndf_dev,
               const kapre_spec_desc* cmndf_desc, void* workspace_dev, void* stream) {
    int rc = kb_pitch_check_shape(plan, x_desc);
    if (rc) return rc;
    if (!plan->geo.pyin) return kb_fail(KAPRE_E_INVALID, "pyin: the plan was created without pYIN tables");
    if (!out_desc || (cmndf_dev && !cmndf_desc)) return kb_fail(KAPRE_E_INVALID, "null argument");
    const int M = kb_pitch_frames(plan->cfg, x_desc->length);
    const long long rows = (long long)x_desc->batch * x_desc->channels;
    if (rows * M == 0) return 0;
    if (!x_dev || !f0_dev || !voiced_flag_dev || !voiced_prob_dev || !workspace_dev)
        return kb_fail(KAPRE_E_INVALID, "null data pointer");
    const cudaStream_t st = (cudaStream_t)stream;
    KbLaunchReports reports;
    if ((rc = kb_pitch_launch(plan, x_dev, x_desc, voiced_prob_dev, out_desc, cmndf_dev, cmndf_desc, workspace_dev, st)))
        return rc;
    reports.add();
    KbVitParams v = plan->vit;
    KbLayout L{(char*)workspace_dev};
    const KbPyinWs w = kb_pyin_layout(L, plan, x_desc->batch, x_desc->channels, M);
    v.M = M; v.C = x_desc->channels; v.rows = rows;
    v.cand_n = w.cand_n; v.cand_p = w.cand_p; v.cand_bin = w.cand_bin; v.bp = w.bp;
    v.vp = voiced_prob_dev; v.f0 = f0_dev; v.flag = voiced_flag_dev;
    v.o_sb = out_desc->stride_b; v.o_sc = out_desc->stride_c; v.o_st = out_desc->stride_t;
    const int smem = kb_vit_smem(v.n, v.w);
    int grid;
    if ((rc = kb_resident_grid(kb_viterbi_kernel, "viterbi", v.nt, smem, rows, plan->dev.sm_count, &grid))) return rc;
    reports.add();
    return kb_launch(kb_viterbi_kernel, {.grid = grid, .block = v.nt, .smem = smem, .st = st, .timed = true}, v);
}

}  // extern "C"

// ---- chroma features (chroma_core.cuh) ----------------------------------------------------------------------------
__global__ void __launch_bounds__(KB_CH_THREADS) kb_chroma_kernel(const __grid_constant__ KbChromaParams p) {
    extern __shared__ __align__(16) char kb_smem[];
    kb_chroma_cta(p, kb_smem, blockIdx.x, gridDim.x);
}
__global__ void __launch_bounds__(KB_CH_THREADS) kb_chroma_bwd_kernel(const __grid_constant__ KbChromaParams p) {
    extern __shared__ __align__(16) char kb_smem[];
    kb_chroma_bwd_cta(p, kb_smem, blockIdx.x, gridDim.x);
}
__global__ void __launch_bounds__(KB_CH_THREADS) kb_tune_peak_kernel(const __grid_constant__ KbTuneParams p) {
    extern __shared__ __align__(16) char kb_smem[];
    kb_tune_peak_cta(p, kb_smem, blockIdx.x, gridDim.x);
}
__global__ void __launch_bounds__(KB_CH_THREADS) kb_tune_sel_kernel(const __grid_constant__ KbTuneParams p) {
    extern __shared__ __align__(16) char kb_smem[];
    kb_tune_sel_cta(p, kb_smem, blockIdx.x, gridDim.x);
}
__global__ void __launch_bounds__(KB_CH_THREADS) kb_tune_argmax_kernel(const __grid_constant__ KbTuneParams p) {
    extern __shared__ __align__(16) char kb_smem[];
    kb_tune_argmax_cta(p, kb_smem, blockIdx.x, gridDim.x);
}
__global__ void __launch_bounds__(KB_CH_THREADS) kb_cens_kernel(const __grid_constant__ KbCensParams p) {
    extern __shared__ __align__(16) char kb_smem[];
    kb_cens_cta(p, kb_smem, blockIdx.x, gridDim.x);
}

struct kapre_chroma_plan {
    kapre_chroma_plan_desc d;
    DevInfo dev;
    KbTables tables;
    float* W = nullptr;                   // n_tables x n_chroma x n_bins
    float* smooth = nullptr;
    double* edges = nullptr;
};

static int kb_chroma_check(const kapre_chroma_plan* plan, const void* x, const kapre_spec_desc* xd, int B, int C, int M,
                           const void* out, const kapre_spec_desc* od) {
    if (!plan || !xd || !od) return kb_fail(KAPRE_E_INVALID, "null argument");
    if (B < 0 || C < 0 || M < 0) return kb_fail(KAPRE_E_INVALID, "chroma: negative size (%d, %d, %d)", B, C, M);
    const int rc = kb_check_device(plan->dev);
    if (rc) return rc;
    if ((long long)B * C * M && (!x || !out)) return kb_fail(KAPRE_E_INVALID, "null data pointer");
    return 0;
}

static int kb_chroma_params(const kapre_chroma_plan* plan, const kapre_chroma_config* cfg, const void* x,
                            const kapre_spec_desc* xd, int B, int C, int M, const int* tab, KbChromaParams* out) {
    if (!cfg) return kb_fail(KAPRE_E_INVALID, "null argument");
    if (plan->d.n_tables < 1) return kb_fail(KAPRE_E_INVALID, "chroma: the plan has no filterbank table");
    if (cfg->in_mode < 0 || cfg->in_mode > 2 || cfg->norm < 0 || cfg->norm > 3)
        return kb_fail(KAPRE_E_INVALID, "chroma: bad input mode %d or norm %d", cfg->in_mode, cfg->norm);
    KbChromaParams p{};
    p.NC = plan->d.n_chroma; p.K = plan->d.n_bins;
    p.in_mode = cfg->in_mode; p.norm = cfg->norm; p.has_thr = cfg->has_threshold; p.thr = cfg->threshold;
    p.W = plan->W; p.tab = tab;
    kb_chroma_tiling(p);
    p.B = B; p.C = C; p.M = M;
    p.x = x; p.x_sb = xd->stride_b; p.x_sc = xd->stride_c; p.x_st = xd->stride_t; p.x_sk = xd->stride_f;
    if (!kb_chroma_setup(p)) return kb_fail(KAPRE_E_INVALID, "chroma: too many tiles");
    *out = p;
    return 0;
}

static int kb_chroma_fwd_launch(const kapre_chroma_plan* plan, const KbChromaParams& p, cudaStream_t st) {
    const int smem = kb_chroma_smem(p.NC, p.G, p.TF);
    int grid, rc;
    if ((rc = kb_resident_grid(kb_chroma_kernel, "chroma", KB_CH_THREADS, smem, p.jobs, plan->dev.sm_count, &grid)))
        return rc;
    return kb_launch(kb_chroma_kernel, {.grid = grid, .block = KB_CH_THREADS, .smem = smem, .st = st, .timed = true}, p);
}

// The chroma_cens workspace: the (B, C, frames, n_chroma) chroma that the smoothing pass reads.
static float* kb_cens_layout(KbLayout& L, const kapre_chroma_plan* plan, int batch, int channels, int frames) {
    return L.take<float>(batch, channels, frames, plan->d.n_chroma);
}

// The tuning workspace: per item the radix and residual histograms and the smallest magnitude above the lower rank,
// then per frame the peak magnitudes and pitches.
static void kb_tune_layout(KbLayout& L, const kapre_chroma_plan* plan, int batch, int channels, int frames,
                           KbTuneParams& p) {
    const int cap = (plan->d.peak_hi - plan->d.peak_lo + 1) / 2;
    p.hist = L.take<unsigned>(batch, 1024);
    p.res = L.take<unsigned>(batch, plan->d.n_tuning_bins);
    p.above = L.take<unsigned>(batch);
    p.mag = L.take<float>(batch, channels, frames, cap);
    p.pitch = L.take<float>(batch, channels, frames, cap);
    L.pad();
}

extern "C" {

int kapre_chroma_plan_create(const kapre_chroma_plan_desc* desc, kapre_chroma_plan** out) {
    if (!desc || !out) return kb_fail(KAPRE_E_INVALID, "null argument");
    *out = nullptr;
    const kapre_chroma_plan_desc& d = *desc;
    if (d.n_chroma < 1 || d.n_chroma > KAPRE_CHROMA_MAX_CHROMA)
        return kb_fail(KAPRE_E_UNSUPPORTED, "chroma: n_chroma %d outside [1, %d]", d.n_chroma, KAPRE_CHROMA_MAX_CHROMA);
    if (d.n_bins < 1 || d.n_bins > KAPRE_CHROMA_MAX_BINS || d.n_tables < 0 || (d.n_tables && !d.tables))
        return kb_fail(KAPRE_E_INVALID, "chroma: bad table (%d bins, %d tables)", d.n_bins, d.n_tables);
    if (d.n_smooth < 0 || d.n_smooth > KAPRE_CHROMA_MAX_SMOOTH || (d.n_smooth && !d.smooth))
        return kb_fail(KAPRE_E_INVALID, "chroma: bad smoothing window of %d taps", d.n_smooth);
    if (d.n_tuning_bins < 0 || d.n_tuning_bins > KAPRE_CHROMA_MAX_TUNING_BINS || (d.n_tuning_bins && !d.tuning_edges))
        return kb_fail(KAPRE_E_INVALID, "chroma: bad tuning histogram of %d bins", d.n_tuning_bins);
    if (d.n_tuning_bins && (d.peak_lo < 1 || d.peak_hi > d.n_bins - 1 || d.peak_hi <= d.peak_lo ||
                            !(d.sample_rate > 0.0f) || !(d.n_fft > 0.0f) || !(d.bins_per_octave > 0.0)))
        return kb_fail(KAPRE_E_INVALID, "chroma: bad peak range [%d, %d) of %d bins", d.peak_lo, d.peak_hi, d.n_bins);
    kapre_chroma_plan* pl = new kapre_chroma_plan();
    pl->d = d;
    pl->d.tables = nullptr; pl->d.smooth = nullptr; pl->d.tuning_edges = nullptr;
    KbTableUpload tb;
    if (d.n_tables) {
        const size_t n = (size_t)d.n_tables * d.n_chroma * d.n_bins;
        std::vector<float> h(n);
        for (size_t i = 0; i < n; ++i) h[i] = (float)d.tables[i];
        tb.add(h, &pl->W);
    }
    if (d.n_smooth) tb.add(std::vector<float>(d.smooth, d.smooth + d.n_smooth), &pl->smooth);
    if (d.n_tuning_bins) tb.add(std::vector<double>(d.tuning_edges, d.tuning_edges + d.n_tuning_bins + 1), &pl->edges);
    int rc;
    if ((rc = kb_dev_info(&pl->dev)) || (rc = tb.upload(pl->tables, "chroma"))) {
        delete pl;
        return rc;
    }
    *out = pl;
    return 0;
}

void kapre_chroma_plan_destroy(kapre_chroma_plan* plan) { delete plan; }

int kapre_chroma(const kapre_chroma_plan* plan, const kapre_chroma_config* cfg, const void* x_dev,
                 const kapre_spec_desc* x_desc, int batch, int channels, int frames, const int* table_dev, float* out_dev,
                 const kapre_spec_desc* out_desc, void* stream) {
    int rc = kb_chroma_check(plan, x_dev, x_desc, batch, channels, frames, out_dev, out_desc);
    if (rc) return rc;
    KbChromaParams p;
    if ((rc = kb_chroma_params(plan, cfg, x_dev, x_desc, batch, channels, frames, table_dev, &p))) return rc;
    if (!p.jobs) return 0;
    p.out = out_dev; p.o_sb = out_desc->stride_b; p.o_sc = out_desc->stride_c; p.o_st = out_desc->stride_t;
    p.o_sk = out_desc->stride_f;
    return kb_chroma_fwd_launch(plan, p, (cudaStream_t)stream);
}

int kapre_chroma_backward(const kapre_chroma_plan* plan, const kapre_chroma_config* cfg, const void* x_dev,
                          const kapre_spec_desc* x_desc, int batch, int channels, int frames, const int* table_dev,
                          const float* g_dev, const kapre_spec_desc* g_desc, void* gx_dev, const kapre_spec_desc* gx_desc,
                          void* stream) {
    int rc = kb_chroma_check(plan, x_dev, x_desc, batch, channels, frames, gx_dev, gx_desc);
    if (rc) return rc;
    if (!g_desc) return kb_fail(KAPRE_E_INVALID, "null argument");
    KbChromaParams p;
    if ((rc = kb_chroma_params(plan, cfg, x_dev, x_desc, batch, channels, frames, table_dev, &p))) return rc;
    if (!p.jobs) return 0;
    if (!g_dev) return kb_fail(KAPRE_E_INVALID, "null data pointer");
    p.g = g_dev; p.g_sb = g_desc->stride_b; p.g_sc = g_desc->stride_c; p.g_st = g_desc->stride_t;
    p.g_sk = g_desc->stride_f;
    p.gx = gx_dev; p.gx_sb = gx_desc->stride_b; p.gx_sc = gx_desc->stride_c; p.gx_st = gx_desc->stride_t;
    p.gx_sk = gx_desc->stride_f;
    const int smem = kb_chroma_smem(p.NC, p.G, p.TF);
    int grid;
    if ((rc = kb_resident_grid(kb_chroma_bwd_kernel, "chroma_bwd", KB_CH_THREADS, smem, p.jobs, plan->dev.sm_count,
                               &grid)))
        return rc;
    return kb_launch(kb_chroma_bwd_kernel, {.grid = grid, .block = KB_CH_THREADS, .smem = smem,
                                            .st = (cudaStream_t)stream}, p);
}

int64_t kapre_chroma_cens_workspace_bytes(const kapre_chroma_plan* plan, int batch, int channels, int frames) {
    if (!plan) return kb_fail(KAPRE_E_INVALID, "null plan");
    if (batch < 0 || channels < 0 || frames < 0) return kb_fail(KAPRE_E_INVALID, "chroma: negative size");
    KbLayout L;
    kb_cens_layout(L, plan, batch, channels, frames);
    return L.bytes("chroma_cens");
}

int kapre_chroma_cens(const kapre_chroma_plan* plan, int in_mode, const void* x_dev, const kapre_spec_desc* x_desc,
                      int batch, int channels, int frames, float* out_dev, const kapre_spec_desc* out_desc,
                      void* workspace_dev, void* stream) {
    int rc = kb_chroma_check(plan, x_dev, x_desc, batch, channels, frames, out_dev, out_desc);
    if (rc) return rc;
    if (plan->d.n_smooth < 1) return kb_fail(KAPRE_E_INVALID, "chroma_cens: the plan has no smoothing window");
    const kapre_chroma_config cfg = {in_mode, KAPRE_CHROMA_NORM_L1, 1, 0.0f};
    KbChromaParams p;
    if ((rc = kb_chroma_params(plan, &cfg, x_dev, x_desc, batch, channels, frames, nullptr, &p))) return rc;
    if (!p.jobs) return 0;
    if (!workspace_dev) return kb_fail(KAPRE_E_INVALID, "null workspace");
    const int NC = plan->d.n_chroma;
    KbLayout L{(char*)workspace_dev};
    float* q = kb_cens_layout(L, plan, batch, channels, frames);
    p.cens = 1;
    p.out = q;
    p.o_sc = (long long)frames * NC; p.o_sb = channels * p.o_sc; p.o_st = NC; p.o_sk = 1;
    const cudaStream_t st = (cudaStream_t)stream;
    KbLaunchReports reports;
    if ((rc = kb_chroma_fwd_launch(plan, p, st))) return rc;
    reports.add();
    KbCensParams c{};
    c.NC = NC; c.N = plan->d.n_smooth; c.w = plan->smooth;
    c.B = batch; c.C = channels; c.M = frames;
    c.tiles = ((long long)frames + KB_CH_SMOOTH_TF - 1) / KB_CH_SMOOTH_TF;
    c.jobs = (long long)batch * channels * c.tiles;
    c.q = q;
    c.out = out_dev; c.o_sb = out_desc->stride_b; c.o_sc = out_desc->stride_c; c.o_st = out_desc->stride_t;
    c.o_sk = out_desc->stride_f;
    const int smem = kb_cens_smem(NC, c.N);
    if (smem > plan->dev.smem_optin) return kb_fail(KAPRE_E_UNSUPPORTED, "chroma_cens: %d B of shared memory", smem);
    int grid;
    if ((rc = kb_resident_grid(kb_cens_kernel, "cens", KB_CH_THREADS, smem, c.jobs, plan->dev.sm_count, &grid)))
        return rc;
    reports.add();
    return kb_launch(kb_cens_kernel, {.grid = grid, .block = KB_CH_THREADS, .smem = smem, .st = st}, c);
}

int64_t kapre_chroma_tuning_workspace_bytes(const kapre_chroma_plan* plan, int batch, int channels, int frames) {
    if (!plan) return kb_fail(KAPRE_E_INVALID, "null plan");
    if (batch < 0 || channels < 0 || frames < 0) return kb_fail(KAPRE_E_INVALID, "chroma: negative size");
    if (!plan->d.n_tuning_bins) return kb_fail(KAPRE_E_INVALID, "chroma: the plan has no tuning estimate");
    KbLayout L;
    KbTuneParams p{};
    kb_tune_layout(L, plan, batch, channels, frames, p);
    return L.bytes("chroma_tuning");
}

int kapre_chroma_tuning(const kapre_chroma_plan* plan, int in_mode, const float* x_dev, const kapre_spec_desc* x_desc,
                        int batch, int channels, int frames, double* tuning_dev, int* table_dev, void* workspace_dev,
                        void* stream) {
    int rc = kb_chroma_check(plan, x_dev, x_desc, batch, channels, frames, tuning_dev, x_desc);
    if (rc) return rc;
    if (!plan->d.n_tuning_bins) return kb_fail(KAPRE_E_INVALID, "chroma: the plan has no tuning estimate");
    if (in_mode != KAPRE_CHROMA_IN_LINEAR && in_mode != KAPRE_CHROMA_IN_SQUARE)
        return kb_fail(KAPRE_E_INVALID, "estimate_tuning: bad input mode %d", in_mode);
    if (batch == 0) return 0;
    if (!tuning_dev || !table_dev || !workspace_dev) return kb_fail(KAPRE_E_INVALID, "null data pointer");
    const cudaStream_t st = (cudaStream_t)stream;
    KbTuneParams p{};
    const kapre_chroma_plan_desc& d = plan->d;
    p.K = d.n_bins; p.lo = d.peak_lo; p.hi = d.peak_hi; p.cap = (d.peak_hi - d.peak_lo + 1) / 2;
    p.in_mode = in_mode; p.sr = d.sample_rate; p.nfft = d.n_fft; p.bpo = d.bins_per_octave;
    p.nres = d.n_tuning_bins; p.edges = plan->edges;
    p.B = batch; p.C = channels; p.M = frames;
    p.x = x_dev; p.x_sb = x_desc->stride_b; p.x_sc = x_desc->stride_c; p.x_st = x_desc->stride_t;
    p.x_sk = x_desc->stride_f;
    KbLayout L{(char*)workspace_dev};
    kb_tune_layout(L, plan, batch, channels, frames, p);
    p.tuning = tuning_dev; p.tab = table_dev;
    // both histograms, which the layout puts next to each other, start at zero; the minima start at the largest value
    KB_CUDA(cudaMemsetAsync(p.hist, 0, (size_t)((char*)p.above - (char*)p.hist), st));
    KB_CUDA(cudaMemsetAsync(p.above, 0xff, (size_t)batch * 4, st));
    const long long rows = (long long)batch * channels;
    int grid;
    KbLaunchReports reports;
    if (frames > 0) {
        p.tiles = ((long long)frames + KB_CH_PEAK_TF - 1) / KB_CH_PEAK_TF;
        p.jobs = rows * p.tiles;
        if ((rc = kb_resident_grid(kb_tune_peak_kernel, "tune_peak", KB_CH_THREADS, kb_tune_peak_smem(), p.jobs,
                                   plan->dev.sm_count, &grid)))
            return rc;
        if ((rc = kb_launch(kb_tune_peak_kernel, {.grid = grid, .block = KB_CH_THREADS, .smem = kb_tune_peak_smem(),
                                                  .st = st}, p)))
            return rc;
        reports.add();
        p.tiles = ((long long)frames + KB_CH_SEL_TF - 1) / KB_CH_SEL_TF;
        p.jobs = rows * p.tiles;
        if ((rc = kb_resident_grid(kb_tune_sel_kernel, "tune_select", KB_CH_THREADS, kb_tune_sel_smem(), p.jobs,
                                   plan->dev.sm_count, &grid)))
            return rc;
        for (p.pass = 1; p.pass <= 5; ++p.pass)
            if ((rc = kb_launch(kb_tune_sel_kernel, {.grid = grid, .block = KB_CH_THREADS, .smem = kb_tune_sel_smem(),
                                                     .st = st}, p)))
                return rc;
        reports.add();
    }
    if ((rc = kb_resident_grid(kb_tune_argmax_kernel, "tune_argmax", KB_CH_THREADS, 2 * KB_CH_THREADS * 4, batch,
                               plan->dev.sm_count, &grid)))
        return rc;
    reports.add();
    return kb_launch(kb_tune_argmax_kernel, {.grid = grid, .block = KB_CH_THREADS, .smem = 2 * KB_CH_THREADS * 4,
                                             .st = st}, p);
}

}  // extern "C"

// ---- harmonic/percussive separation (hpss_core.cuh) ---------------------------------------------------------------
template <int NSH, int NSP, int BWD>
__global__ void __launch_bounds__(KB_HS_THREADS) kb_hpss_kernel(const __grid_constant__ KbHpssParams p) {
    extern __shared__ __align__(16) char kb_smem[];
    kb_hpss_cta<NSH, NSP, BWD>(p, kb_smem, blockIdx.x, gridDim.x);
}
__global__ void __launch_bounds__(KB_HS_THREADS) kb_hpss_gather_kernel(const __grid_constant__ KbHpssParams p) {
    kb_hpss_gather_cta(p, nullptr, blockIdx.x, gridDim.x);
}

template <int BWD>
static int kb_hpss_tiles_launch(const KbHpssParams& p, cudaStream_t st) {
    const int sh = kb_hs_slots(p.kh), sp = kb_hs_slots(p.kp);
    void (*k)(const KbHpssParams) = sh == 32 ? (sp == 32 ? kb_hpss_kernel<32, 32, BWD> : kb_hpss_kernel<32, 64, BWD>)
                                             : (sp == 32 ? kb_hpss_kernel<64, 32, BWD> : kb_hpss_kernel<64, 64, BWD>);
    DevInfo dev;
    int rc, grid;
    if ((rc = kb_dev_info(&dev))) return rc;
    const int smem = kb_hpss_smem(p.kh, p.kp, BWD);
    if ((rc = kb_resident_grid(k, BWD ? "hpss_bwd" : "hpss", KB_HS_THREADS, smem, p.jobs, dev.sm_count, &grid)))
        return rc;
    return kb_launch(k, {.grid = grid, .block = KB_HS_THREADS, .smem = smem, .st = st, .timed = !BWD}, p);
}

// The backward workspace: one region of 2n weights, the harmonic median's n and then the percussive median's n.
static void kb_hpss_layout(KbLayout& L, int batch, int channels, int frames, int bins, KbHpssParams& p) {
    p.wh = L.take<kb_hs_w>(batch, channels, frames, bins, 2);
    p.wp = p.wh ? p.wh + (long long)batch * channels * frames * bins : nullptr;
}

static int kb_hpss_params(const kapre_hpss_config* cfg, const void* S, int is_complex, const kapre_spec_desc* sd,
                          int B, int C, int T, int K, KbHpssParams* out) {
    if (!cfg || !sd) return kb_fail(KAPRE_E_INVALID, "null argument");
    if (B < 0 || C < 0 || T < 0 || K < 0) return kb_fail(KAPRE_E_INVALID, "hpss: negative size (%d, %d, %d, %d)", B, C, T, K);
    if (cfg->kernel_h < 1 || cfg->kernel_h > KAPRE_HPSS_MAX_KERNEL || cfg->kernel_p < 1 ||
        cfg->kernel_p > KAPRE_HPSS_MAX_KERNEL)
        return kb_fail(KAPRE_E_INVALID, "hpss: kernel sizes (%d, %d) outside [1, %d]", cfg->kernel_h, cfg->kernel_p,
                       KAPRE_HPSS_MAX_KERNEL);
    if (!(cfg->margin_h >= 1.0f) || !(cfg->margin_p >= 1.0f) || !isfinite(cfg->margin_h) || !isfinite(cfg->margin_p))
        return kb_fail(KAPRE_E_INVALID, "hpss: margins must be finite and >= 1");
    if (!(cfg->power > 0.0f)) return kb_fail(KAPRE_E_INVALID, "hpss: power must be > 0");
    KbHpssParams p{};
    p.B = B; p.C = C; p.T = T; p.K = K;
    p.kh = cfg->kernel_h; p.kp = cfg->kernel_p; p.mh = cfg->margin_h; p.mp = cfg->margin_p; p.power = cfg->power;
    p.pmode = isinf(cfg->power) ? KB_HS_POW_INF : cfg->power == 1.0f ? KB_HS_POW_1
                                : cfg->power == 2.0f ? KB_HS_POW_2 : KB_HS_POW_GENERIC;
    p.split = cfg->margin_h == 1.0f && cfg->margin_p == 1.0f;
    p.cplx = is_complex != 0; p.mask = cfg->mask != 0;
    p.x = S; p.x_sb = sd->stride_b; p.x_sc = sd->stride_c; p.x_st = sd->stride_t; p.x_sk = sd->stride_f;
    if (!kb_hpss_setup(p)) return kb_fail(KAPRE_E_INVALID, "hpss: too many tiles");
    if (p.jobs && !S) return kb_fail(KAPRE_E_INVALID, "null data pointer");
    *out = p;
    return 0;
}

extern "C" {

int kapre_hpss(const kapre_hpss_config* cfg, const void* S_dev, int is_complex, const kapre_spec_desc* S_desc, int batch,
               int channels, int frames, int bins, void* h_dev, const kapre_spec_desc* h_desc, void* p_dev,
               const kapre_spec_desc* p_desc, void* stream) {
    KbHpssParams p;
    int rc = kb_hpss_params(cfg, S_dev, is_complex, S_desc, batch, channels, frames, bins, &p);
    if (rc) return rc;
    if ((h_dev && !h_desc) || (p_dev && !p_desc)) return kb_fail(KAPRE_E_INVALID, "null argument");
    if (!p.jobs || (!h_dev && !p_dev)) return 0;
    p.oh = h_dev;
    if (h_dev) { p.oh_sb = h_desc->stride_b; p.oh_sc = h_desc->stride_c; p.oh_st = h_desc->stride_t; p.oh_sk = h_desc->stride_f; }
    p.op = p_dev;
    if (p_dev) { p.op_sb = p_desc->stride_b; p.op_sc = p_desc->stride_c; p.op_st = p_desc->stride_t; p.op_sk = p_desc->stride_f; }
    return kb_hpss_tiles_launch<0>(p, (cudaStream_t)stream);
}

int64_t kapre_hpss_workspace_bytes(int batch, int channels, int frames, int bins) {
    if (batch < 0 || channels < 0 || frames < 0 || bins < 0) return kb_fail(KAPRE_E_INVALID, "hpss: negative size");
    KbLayout L;
    KbHpssParams p{};
    kb_hpss_layout(L, batch, channels, frames, bins, p);
    return L.bytes("hpss");
}

int kapre_hpss_backward(const kapre_hpss_config* cfg, const void* S_dev, int is_complex, const kapre_spec_desc* S_desc,
                        int batch, int channels, int frames, int bins, const void* gh_dev, const kapre_spec_desc* gh_desc,
                        const void* gp_dev, const kapre_spec_desc* gp_desc, void* gS_dev,
                        const kapre_spec_desc* gS_desc, void* workspace_dev, void* stream) {
    KbHpssParams p;
    int rc = kb_hpss_params(cfg, S_dev, is_complex, S_desc, batch, channels, frames, bins, &p);
    if (rc) return rc;
    if (!gS_desc || (gh_dev && !gh_desc) || (gp_dev && !gp_desc)) return kb_fail(KAPRE_E_INVALID, "null argument");
    if (!p.jobs) return 0;
    if (!gS_dev || !workspace_dev) return kb_fail(KAPRE_E_INVALID, "null data pointer");
    p.gh = gh_dev;
    if (gh_dev) { p.gh_sb = gh_desc->stride_b; p.gh_sc = gh_desc->stride_c; p.gh_st = gh_desc->stride_t; p.gh_sk = gh_desc->stride_f; }
    p.gp = gp_dev;
    if (gp_dev) { p.gp_sb = gp_desc->stride_b; p.gp_sc = gp_desc->stride_c; p.gp_st = gp_desc->stride_t; p.gp_sk = gp_desc->stride_f; }
    p.gx = gS_dev; p.gx_sb = gS_desc->stride_b; p.gx_sc = gS_desc->stride_c; p.gx_st = gS_desc->stride_t;
    p.gx_sk = gS_desc->stride_f;
    KbLayout L{(char*)workspace_dev};
    kb_hpss_layout(L, batch, channels, frames, bins, p);
    const long long n = (long long)batch * channels * frames * bins;
    cudaStream_t st = (cudaStream_t)stream;
    KbLaunchReports reports;
    if ((rc = kb_hpss_tiles_launch<1>(p, st))) return rc;
    reports.add();
    DevInfo dev;
    if ((rc = kb_dev_info(&dev))) return rc;
    int grid;
    if ((rc = kb_resident_grid(kb_hpss_gather_kernel, "hpss_gather", KB_HS_THREADS, 0,
                               (n + KB_HS_THREADS - 1) / KB_HS_THREADS, dev.sm_count, &grid)))
        return rc;
    reports.add();
    return kb_launch(kb_hpss_gather_kernel, {.grid = grid, .block = KB_HS_THREADS, .st = st}, p);
}

}  // extern "C"

// ---- onset strength, tempogram, tempo, peak picking, beat tracking (rhythm_core.cuh) --------------------------------
template <int BWD>
__global__ void __launch_bounds__(KB_RH_THREADS, 1) kb_onset_kernel(const __grid_constant__ KbOnsetParams p) {
    extern __shared__ __align__(16) char kb_smem[];
    kb_onset_cta<BWD>(p, kb_smem, blockIdx.x, gridDim.x);
}
__global__ void __launch_bounds__(KB_RH_THREADS) kb_onset_gather_kernel(const __grid_constant__ KbOnsetParams p) {
    kb_onset_gather_cta(p, nullptr, blockIdx.x, gridDim.x);
}
__global__ void __launch_bounds__(KB_RH_THREADS) kb_tempogram_kernel(const __grid_constant__ KbTempogramParams p) {
    extern __shared__ __align__(16) char kb_smem[];
    kb_tempogram_cta(p, kb_smem, blockIdx.x, gridDim.x);
}
__global__ void __launch_bounds__(KB_RH_THREADS) kb_tempo_part_kernel(const __grid_constant__ KbTempoParams p) {
    kb_tempo_part_cta(p, nullptr, blockIdx.x, gridDim.x);
}
__global__ void __launch_bounds__(KB_RH_THREADS) kb_tempo_kernel(const __grid_constant__ KbTempoParams p) {
    extern __shared__ __align__(16) char kb_smem[];
    kb_tempo_cta(p, kb_smem, blockIdx.x, gridDim.x);
}
__global__ void __launch_bounds__(KB_RH_THREADS) kb_peak_kernel(const __grid_constant__ KbPeakParams p) {
    extern __shared__ __align__(16) char kb_smem[];
    kb_peak_cta(p, kb_smem, blockIdx.x, gridDim.x);
}
__global__ void __launch_bounds__(KB_RH_THREADS, 1) kb_beat_kernel(const __grid_constant__ KbBeatParams p) {
    extern __shared__ __align__(16) char kb_smem[];
    kb_beat_cta(p, kb_smem, blockIdx.x, gridDim.x);
}

// A persistent launch of `kernel` over `jobs` jobs.
template <typename K, typename P>
static int kb_rh_launch(K kernel, const char* name, int smem, long long jobs, const P& p, cudaStream_t st, bool timed) {
    DevInfo dev;
    int rc, grid;
    if ((rc = kb_dev_info(&dev))) return rc;
    if ((rc = kb_resident_grid(kernel, name, KB_RH_THREADS, smem, jobs, dev.sm_count, &grid))) return rc;
    return kb_launch(kernel, {.grid = grid, .block = KB_RH_THREADS, .smem = smem, .st = st, .timed = timed}, p);
}

static int kb_rh_rows(int B, int C, int T, const char* what) {
    if (B < 0 || C < 0 || T < 0) return kb_fail(KAPRE_E_INVALID, "%s: negative size (%d, %d, %d)", what, B, C, T);
    return 0;
}

static int kb_onset_params(const kapre_onset_config* cfg, const float* S, const kapre_spec_desc* sd, int B, int C,
                           int T, int K, int bwd, KbOnsetParams* out) {
    if (!cfg || !sd) return kb_fail(KAPRE_E_INVALID, "null argument");
    int rc = kb_rh_rows(B, C, T, "onset_strength");
    if (rc) return rc;
    if (K < 1 || K > KAPRE_ONSET_MAX_BINS)
        return kb_fail(KAPRE_E_INVALID, "onset_strength: bins %d outside [1, %d]", K, KAPRE_ONSET_MAX_BINS);
    if (cfg->max_size < 1 || cfg->max_size > K)
        return kb_fail(KAPRE_E_INVALID, "onset_strength: max_size %d outside [1, %d]", cfg->max_size, K);
    if (cfg->lag < 1 || (T > 0 && cfg->lag >= T))
        return kb_fail(KAPRE_E_INVALID, "onset_strength: lag %d outside [1, frames)", cfg->lag);
    if (cfg->pad_frames < 0 || cfg->pad_frames > (1 << 28))
        return kb_fail(KAPRE_E_INVALID, "onset_strength: pad_frames %d out of range", cfg->pad_frames);
    if (cfg->aggregate != KAPRE_ONSET_MEAN && cfg->aggregate != KAPRE_ONSET_MEDIAN)
        return kb_fail(KAPRE_E_INVALID, "onset_strength: unknown aggregate %d", cfg->aggregate);
    KbOnsetParams p{};
    p.B = B; p.C = C; p.T = T; p.K = K;
    p.lag = cfg->lag; p.m = cfg->max_size; p.agg = cfg->aggregate; p.P = cfg->lag + cfg->pad_frames;
    p.x = S; p.x_sb = sd->stride_b; p.x_sc = sd->stride_c; p.x_st = sd->stride_t; p.x_sk = sd->stride_f;
    if (!kb_onset_setup(p, bwd)) return kb_fail(KAPRE_E_INVALID, "onset_strength: too many tiles");
    if (p.jobs && !S) return kb_fail(KAPRE_E_INVALID, "null data pointer");
    *out = p;
    return 0;
}

// The onset strength backward's workspace: the (B, C, frames, bins) weights the gather pass reads.
static kb_on_w* kb_onset_layout(KbLayout& L, int B, int C, int T, int K) { return L.take<kb_on_w>(B, C, T, K); }

// The tempo workspace: the mean's float64 partial sums per row, chunk and lag.
static double* kb_tempo_layout(KbLayout& L, int B, int C, int T, int W) {
    return (double*)L.take<char>(kb_tempo_ws_bytes(B, C, T, W));
}

// Checks a shape and lays out the beat tracker's workspace: per row ls, cs (double T), back and beats (int T).
static int kb_beat_layout(KbLayout& L, int B, int C, int T, void** ws) {
    int rc = kb_rh_rows(B, C, T, "beat_track");
    if (rc) return rc;
    const long long rows = (long long)B * C;
    if (rows && kb_beat_ws_bytes_row(T) > (1LL << 46) / rows) return kb_fail(KAPRE_E_INVALID, "beat_track: too large");
    *ws = L.take<char>(B, C, kb_beat_ws_bytes_row(T));
    return 0;
}

extern "C" {

int kapre_onset_strength(const kapre_onset_config* cfg, const float* S_dev, const kapre_spec_desc* S_desc, int batch,
                         int channels, int frames, int bins, float* out_dev, const kapre_frames_desc* out_desc,
                         void* stream) {
    KbOnsetParams p;
    int rc = kb_onset_params(cfg, S_dev, S_desc, batch, channels, frames, bins, 0, &p);
    if (rc) return rc;
    if (!out_desc) return kb_fail(KAPRE_E_INVALID, "null argument");
    if (!p.jobs) return 0;
    if (!out_dev) return kb_fail(KAPRE_E_INVALID, "null data pointer");
    p.out = out_dev; p.o_sb = out_desc->stride_b; p.o_sc = out_desc->stride_c; p.o_st = out_desc->stride_t;
    return kb_rh_launch(kb_onset_kernel<0>, "onset", kb_onset_smem(p.K, p.m, p.F, 0), p.jobs, p, (cudaStream_t)stream,
                        true);
}

int64_t kapre_onset_strength_workspace_bytes(int batch, int channels, int frames, int bins) {
    if (batch < 0 || channels < 0 || frames < 0 || bins < 0) return kb_fail(KAPRE_E_INVALID, "onset_strength: negative size");
    KbLayout L;
    kb_onset_layout(L, batch, channels, frames, bins);
    return L.bytes("onset_strength");
}

int kapre_onset_strength_backward(const kapre_onset_config* cfg, const float* S_dev, const kapre_spec_desc* S_desc,
                                  int batch, int channels, int frames, int bins, const float* g_dev,
                                  const kapre_frames_desc* g_desc, float* gS_dev, const kapre_spec_desc* gS_desc,
                                  void* workspace_dev, void* stream) {
    KbOnsetParams p;
    int rc = kb_onset_params(cfg, S_dev, S_desc, batch, channels, frames, bins, 1, &p);
    if (rc) return rc;
    if (!g_desc || !gS_desc) return kb_fail(KAPRE_E_INVALID, "null argument");
    if (!p.jobs) return 0;
    if (!g_dev || !gS_dev || !workspace_dev) return kb_fail(KAPRE_E_INVALID, "null data pointer");
    p.g = g_dev; p.g_sb = g_desc->stride_b; p.g_sc = g_desc->stride_c; p.g_st = g_desc->stride_t;
    p.gx = gS_dev; p.gx_sb = gS_desc->stride_b; p.gx_sc = gS_desc->stride_c; p.gx_st = gS_desc->stride_t;
    p.gx_sk = gS_desc->stride_f;
    KbLayout L{(char*)workspace_dev};
    p.ws = kb_onset_layout(L, batch, channels, frames, bins);
    cudaStream_t st = (cudaStream_t)stream;
    KbLaunchReports reports;
    if ((rc = kb_rh_launch(kb_onset_kernel<1>, "onset_bwd", kb_onset_smem(p.K, p.m, p.F, 1), p.jobs, p, st, false)))
        return rc;
    reports.add();
    const long long n = (long long)batch * channels * frames * bins;
    rc = kb_rh_launch(kb_onset_gather_kernel, "onset_gather", 0, (n + KB_RH_THREADS - 1) / KB_RH_THREADS, p, st,
                      false);
    reports.add();
    return rc;
}

int kapre_tempogram(const float* e_dev, const kapre_frames_desc* e_desc, int batch, int channels, int frames,
                    int win_length, int center, int norm_inf, float* out_dev, const kapre_spec_desc* out_desc,
                    void* stream) {
    if (!e_desc || !out_desc) return kb_fail(KAPRE_E_INVALID, "null argument");
    int rc = kb_rh_rows(batch, channels, frames, "tempogram");
    if (rc) return rc;
    if (win_length < 2 || win_length > KAPRE_TEMPOGRAM_MAX_WIN)
        return kb_fail(KAPRE_E_INVALID, "tempogram: win_length %d outside [2, %d]", win_length, KAPRE_TEMPOGRAM_MAX_WIN);
    if (!center && frames < win_length)
        return kb_fail(KAPRE_E_INVALID, "tempogram: %d frames < win_length %d without center", frames, win_length);
    KbTempogramParams p{};
    p.B = batch; p.C = channels; p.T = frames; p.W = win_length; p.center = center != 0; p.norm = norm_inf != 0;
    p.e = e_dev; p.e_sb = e_desc->stride_b; p.e_sc = e_desc->stride_c; p.e_st = e_desc->stride_t;
    p.out = out_dev; p.o_sb = out_desc->stride_b; p.o_sc = out_desc->stride_c; p.o_st = out_desc->stride_t;
    p.o_sk = out_desc->stride_f;
    if (!kb_tempogram_setup(p)) return kb_fail(KAPRE_E_INVALID, "tempogram: too many tiles");
    if (!p.jobs) return 0;
    if (!e_dev || !out_dev) return kb_fail(KAPRE_E_INVALID, "null data pointer");
    return kb_rh_launch(kb_tempogram_kernel, "tempogram", kb_tg_words(p.W, p.F) * 4, p.jobs, p, (cudaStream_t)stream,
                        true);
}

int64_t kapre_tempo_workspace_bytes(int batch, int channels, int frames, int win_length) {
    int rc = kb_rh_rows(batch, channels, frames, "tempo");
    if (rc) return rc;
    if (win_length < 2 || win_length > KAPRE_TEMPOGRAM_MAX_WIN)
        return kb_fail(KAPRE_E_INVALID, "tempo: win_length %d outside [2, %d]", win_length, KAPRE_TEMPOGRAM_MAX_WIN);
    KbLayout L;
    kb_tempo_layout(L, batch, channels, frames, win_length);
    return L.bytes("tempo");
}

int kapre_tempo(const float* tg_dev, const kapre_spec_desc* tg_desc, int batch, int channels, int frames, int win_length,
                const double* logprior_dev, double bpm_scale, int per_frame, float* out_dev,
                const kapre_frames_desc* out_desc, void* workspace_dev, void* stream) {
    if (!tg_desc || (per_frame && !out_desc)) return kb_fail(KAPRE_E_INVALID, "null argument");
    int rc = kb_rh_rows(batch, channels, frames, "tempo");
    if (rc) return rc;
    if (win_length < 2 || win_length > KAPRE_TEMPOGRAM_MAX_WIN)
        return kb_fail(KAPRE_E_INVALID, "tempo: win_length %d outside [2, %d]", win_length, KAPRE_TEMPOGRAM_MAX_WIN);
    if (!per_frame && batch && channels && frames < 1) return kb_fail(KAPRE_E_INVALID, "tempo: no frames");
    if (!(bpm_scale > 0.0) || !isfinite(bpm_scale)) return kb_fail(KAPRE_E_INVALID, "tempo: bpm_scale must be > 0");
    KbTempoParams p{};
    p.B = batch; p.C = channels; p.T = frames; p.W = win_length; p.per_frame = per_frame != 0;
    p.tg = tg_dev; p.g_sb = tg_desc->stride_b; p.g_sc = tg_desc->stride_c; p.g_st = tg_desc->stride_t;
    p.g_sk = tg_desc->stride_f;
    p.logprior = logprior_dev; p.bpm_scale = bpm_scale; p.out = out_dev;
    KbLayout L{(char*)workspace_dev};
    p.part = kb_tempo_layout(L, batch, channels, frames, win_length);
    if (per_frame) { p.o_sb = out_desc->stride_b; p.o_sc = out_desc->stride_c; p.o_st = out_desc->stride_t; }
    kb_tempo_setup(p);
    if (!p.jobs) return 0;
    if (!tg_dev || !logprior_dev || !out_dev || (!per_frame && !workspace_dev))
        return kb_fail(KAPRE_E_INVALID, "null data pointer");
    cudaStream_t st = (cudaStream_t)stream;
    KbLaunchReports reports;
    if (!per_frame) {
        if ((rc = kb_rh_launch(kb_tempo_part_kernel, "tempo_part", 0, (long long)batch * channels * p.chunks, p, st,
                               false)))
            return rc;
        reports.add();
    }
    rc = kb_rh_launch(kb_tempo_kernel, "tempo", kb_tempo_smem(p.W), p.jobs, p, st, false);
    reports.add();
    return rc;
}

int kapre_onset_detect(const float* e_dev, const kapre_frames_desc* e_desc, int batch, int channels, int frames,
                       const kapre_onset_detect_config* cfg, uint8_t* mask_dev, const kapre_frames_desc* mask_desc,
                       void* stream) {
    if (!e_desc || !cfg || !mask_desc) return kb_fail(KAPRE_E_INVALID, "null argument");
    int rc = kb_rh_rows(batch, channels, frames, "onset_detect");
    if (rc) return rc;
    if (cfg->pre_max < 0 || cfg->pre_avg < 0 || cfg->wait < 0 || cfg->post_max < 1 || cfg->post_avg < 1)
        return kb_fail(KAPRE_E_INVALID, "onset_detect: pre_* and wait must be >= 0, post_* >= 1");
    if (cfg->pre_max > KAPRE_PEAK_MAX_WINDOW || cfg->post_max > KAPRE_PEAK_MAX_WINDOW ||
        cfg->pre_avg > KAPRE_PEAK_MAX_WINDOW || cfg->post_avg > KAPRE_PEAK_MAX_WINDOW || cfg->wait > KAPRE_PEAK_MAX_WINDOW)
        return kb_fail(KAPRE_E_INVALID, "onset_detect: pre_*, post_* and wait must be <= %d", KAPRE_PEAK_MAX_WINDOW);
    if (!isfinite(cfg->delta)) return kb_fail(KAPRE_E_INVALID, "onset_detect: delta must be finite");
    KbPeakParams p{};
    p.B = batch; p.C = channels; p.T = frames;
    p.pre_max = cfg->pre_max; p.post_max = cfg->post_max; p.pre_avg = cfg->pre_avg; p.post_avg = cfg->post_avg;
    p.wait = cfg->wait; p.normalize = cfg->normalize != 0; p.delta = cfg->delta;
    p.e = e_dev; p.e_sb = e_desc->stride_b; p.e_sc = e_desc->stride_c; p.e_st = e_desc->stride_t;
    p.mask = mask_dev; p.m_sb = mask_desc->stride_b; p.m_sc = mask_desc->stride_c; p.m_st = mask_desc->stride_t;
    p.jobs = frames ? (long long)batch * channels : 0;
    if (!p.jobs) return 0;
    if (!e_dev || !mask_dev) return kb_fail(KAPRE_E_INVALID, "null data pointer");
    return kb_rh_launch(kb_peak_kernel, "onset_detect", kb_peak_smem(), p.jobs, p, (cudaStream_t)stream, false);
}

int64_t kapre_beat_track_workspace_bytes(int batch, int channels, int frames) {
    KbLayout L;
    void* ws;
    int rc = kb_beat_layout(L, batch, channels, frames, &ws);
    return rc ? rc : L.bytes("beat_track");
}

int kapre_beat_track(const float* e_dev, const kapre_frames_desc* e_desc, int batch, int channels, int frames,
                     const kapre_beat_config* cfg, const float* bpm_dev, float bpm, float* tempo_dev, uint8_t* mask_dev,
                     const kapre_frames_desc* mask_desc, void* workspace_dev, void* stream) {
    if (!e_desc || !cfg || !mask_desc) return kb_fail(KAPRE_E_INVALID, "null argument");
    KbBeatParams p{};
    KbLayout L{(char*)workspace_dev};
    int rc = kb_beat_layout(L, batch, channels, frames, &p.ws);
    if (rc) return rc;
    if (!(cfg->fps > 0.0) || !isfinite(cfg->fps)) return kb_fail(KAPRE_E_INVALID, "beat_track: fps must be > 0");
    if (!(cfg->tightness > 0.0) || !isfinite(cfg->tightness))
        return kb_fail(KAPRE_E_INVALID, "beat_track: tightness must be > 0");
    if (!bpm_dev && !(bpm > 0.0f && isfinite(bpm))) return kb_fail(KAPRE_E_INVALID, "beat_track: bpm must be > 0");
    p.B = batch; p.C = channels; p.T = frames; p.trim = cfg->trim != 0; p.fps = cfg->fps; p.tightness = cfg->tightness;
    p.bpm = bpm_dev; p.bpm_const = bpm;
    p.e = e_dev; p.e_sb = e_desc->stride_b; p.e_sc = e_desc->stride_c; p.e_st = e_desc->stride_t;
    p.tempo = tempo_dev; p.mask = mask_dev;
    p.m_sb = mask_desc->stride_b; p.m_sc = mask_desc->stride_c; p.m_st = mask_desc->stride_t;
    p.jobs = (long long)batch * channels;
    if (!p.jobs) return 0;
    if (!frames) return kb_fail(KAPRE_E_INVALID, "beat_track: no frames");
    if (!e_dev || !tempo_dev || !mask_dev || !workspace_dev) return kb_fail(KAPRE_E_INVALID, "null data pointer");
    return kb_rh_launch(kb_beat_kernel, "beat_track", kb_beat_smem(), p.jobs, p, (cudaStream_t)stream, false);
}

}  // extern "C"

// ---- image-source room impulse responses (rir_core.cuh) -------------------------------------------------------------
__global__ void __launch_bounds__(KB_RIR_MAX_NW * 32, 1) kb_rir_kernel(const __grid_constant__ KbRirParams p) {
    extern __shared__ __align__(16) char kb_smem[];
    asm volatile("griddepcontrol.wait;" ::: "memory");
    kb_rir_tile(p, kb_smem, (long long)blockIdx.x);
}

// In place, per (item, mic) row of L samples: h *= 1 / sqrt(sum h^2), the sum in float64 in a fixed order (lane l
// adds samples l, l + 32, ... in turn; then the 32 lane sums are added in lane order).  One warp per row.
__global__ void __launch_bounds__(256) kb_rir_norm_kernel(float* out, long long sb, long long sm, long long st, int B,
                                                          int M, int L) {
    asm volatile("griddepcontrol.wait;" ::: "memory");
    const long long row = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
    const int lane = (int)(threadIdx.x & 31);
    if (row >= (long long)B * M) return;
    float* h = out + (row / M) * sb + (row % M) * sm;
    double part = 0.0;
    for (int t = lane; t < L; t += 32) {
        const double v = (double)h[t * st];
        part = __dadd_rn(part, __dmul_rn(v, v));
    }
    double s = 0.0;
    for (int i = 0; i < 32; ++i) s = __dadd_rn(s, __shfl_sync(0xffffffffu, part, i));
    if (!(s > 0.0)) return;
    const double inv = __ddiv_rn(1.0, __dsqrt_rn(s));
    for (int t = lane; t < L; t += 32) h[t * st] = (float)__dmul_rn((double)h[t * st], inv);
}

static bool kb_rir_inside(double v, double L) { return std::isfinite(v) && v > 0.0 && v < L; }

// The analytic bound on one response's image count: the lattice boxes [(2n - 1) L, (2n + 1) L] meeting the ball of
// radius R around the mic, times 8.  It bounds the kernel's work even with a max_order: the tiles enumerate every
// candidate in the ball and drop the images of higher order one by one.  Below the cap every axis has at most 2^21
// boxes, so the row, column and image counts and their prefix sums stay far inside int32.
static double kb_rir_image_bound(const double* rec, const double* mic, double R) {
    double boxes = 8.0;
    for (int d = 0; d < 3; ++d) {
        const double L = rec[d];
        boxes *= floor((mic[d] + R + L) / (2.0 * L)) - ceil((mic[d] - R - L) / (2.0 * L)) + 1.0;
    }
    return boxes;
}

extern "C" {

int kapre_rir_ism(const double* records_host, const double* records_dev, int batch, int n_mics, int output_length,
                  int filter_length, double sample_rate, double sound_speed, int flags, float* out_dev,
                  int64_t stride_b, int64_t stride_m, int64_t stride_t, void* stream) {
    const int W = filter_length, L = output_length;
    if (batch < 0 || n_mics < 1 || L < 1)
        return kb_fail(KAPRE_E_INVALID, "rir_ism: bad size: batch %d, %d mics, output_length %d", batch, n_mics, L);
    if (W < 1 || W > KB_RIR_MAX_W || !(W & 1))
        return kb_fail(KAPRE_E_INVALID, "rir_ism: delay_filter_length must be odd, 1 to %d, got %d", KB_RIR_MAX_W, W);
    if (!(std::isfinite(sample_rate) && sample_rate > 0) || !(std::isfinite(sound_speed) && sound_speed > 0))
        return kb_fail(KAPRE_E_INVALID, "rir_ism: sample_rate and sound_speed must be finite and positive");
    if (flags & ~KAPRE_RIR_UNIT_NORM) return kb_fail(KAPRE_E_INVALID, "rir_ism: unknown flags %d", flags);
    if (batch == 0) return 0;
    if (!records_host || !records_dev != !out_dev) return kb_fail(KAPRE_E_INVALID, "null argument");
    const double* mics = records_host + (size_t)batch * KB_RIR_REC;
    for (int b = 0; b < batch; ++b) {
        const double* r = records_host + (size_t)b * KB_RIR_REC;
        for (int d = 0; d < 3; ++d) {
            if (!(std::isfinite(r[d]) && r[d] > 0))
                return kb_fail(KAPRE_E_INVALID, "rir_ism: item %d: room sides must be finite and positive", b);
            if (!kb_rir_inside(r[3 + d], r[d]))
                return kb_fail(KAPRE_E_INVALID, "rir_ism: item %d: the source must lie strictly inside the room", b);
        }
        for (int w = 0; w < 6; ++w)
            if (!(r[6 + w] >= 0.0 && r[6 + w] <= 1.0))
                return kb_fail(KAPRE_E_INVALID, "rir_ism: item %d: reflection coefficients must lie in [0, 1]", b);
        if (!(r[12] == -1.0 || (r[12] >= 0 && r[12] <= 1e6 && r[12] == floor(r[12]))))
            return kb_fail(KAPRE_E_INVALID, "rir_ism: item %d: max_order must be -1 or a non-negative integer", b);
        if (!(r[13] >= 0 && r[13] == floor(r[13]) && r[13] + L <= 2147483647.0))
            return kb_fail(KAPRE_E_INVALID, "rir_ism: item %d: start must be an integer >= 0 with start + "
                           "output_length < 2^31", b);
        const double R = (r[13] + L) * sound_speed / sample_rate;
        for (int m = 0; m < n_mics; ++m) {
            const double* q = mics + ((size_t)b * n_mics + m) * 3;
            for (int d = 0; d < 3; ++d)
                if (!kb_rir_inside(q[d], r[d]))
                    return kb_fail(KAPRE_E_INVALID, "rir_ism: item %d mic %d must lie strictly inside the room", b, m);
            const double dist = sqrt((q[0] - r[3]) * (q[0] - r[3]) + (q[1] - r[4]) * (q[1] - r[4]) +
                                     (q[2] - r[5]) * (q[2] - r[5]));
            if (!(dist >= 1e-3))
                return kb_fail(KAPRE_E_INVALID, "rir_ism: item %d mic %d is closer than 1 mm to the source", b, m);
            const double n_img = kb_rir_image_bound(r, q, R);
            if (!(n_img <= (double)KB_RIR_MAX_IMAGES))
                return kb_fail(KAPRE_E_INVALID, "rir_ism: item %d mic %d: up to %.3g images, above the cap of %lld "
                               "(a shorter response or a larger room)", b, m, n_img,
                               (long long)KB_RIR_MAX_IMAGES);
        }
    }
    if (!records_dev) return 0;                             // validation only
    KbRirParams p{};
    p.nw = KB_RIR_MAX_NW;
    p.n_tt = (L + 32 * p.nw - 1) / (32 * p.nw);
    const long long tiles = (long long)batch * n_mics * p.n_tt;
    if (tiles > 2147483647LL || (double)batch * n_mics / 8.0 > 2147483647.0)
        return kb_fail(KAPRE_E_INVALID, "rir_ism: %lld tiles exceed the grid", tiles);
    p.rec = records_dev;
    p.mic = records_dev + (size_t)batch * KB_RIR_REC;
    p.out = out_dev; p.o_sb = stride_b; p.o_sm = stride_m; p.o_st = stride_t;
    p.B = batch; p.M = n_mics; p.L = L; p.W = W;
    p.fs = sample_rate; p.c = sound_speed;
    const int half = (W - 1) / 2;
    for (int k = 0; k < W; ++k) {
        const double w = W == 1 ? 1.0 : 0.5 - 0.5 * cos(2.0 * 3.14159265358979323846 * k / (W - 1));
        p.ws[k] = (float)(((k + 1 - half) & 1) ? -w : w);
    }
    const cudaStream_t st = (cudaStream_t)stream;
    int rc = kb_launch(kb_rir_kernel, {.grid = (int)tiles, .block = 32 * p.nw, .smem = kb_rir_smem(32 * p.nw).total,
                                       .st = st, .pdl = true, .timed = true}, p);
    if (rc || !(flags & KAPRE_RIR_UNIT_NORM)) return rc;
    const long long rows = (long long)batch * n_mics;
    return kb_launch(kb_rir_norm_kernel, {.grid = (int)((rows + 7) / 8), .block = 256, .st = st, .pdl = true}, out_dev,
                     (long long)stride_b, (long long)stride_m, (long long)stride_t, batch, n_mics, L);
}

}  // extern "C"
