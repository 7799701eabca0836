/*
 * kapre_b200 -- C ABI of the GPU-native STFT -> |.| -> filterbank -> dB hot path (+ inverse STFT).
 *
 * This is the drop-in boundary of the repo: everything the reference computes inside
 * TensorFlow for the five hot-path layers is reachable through these entry points, with
 * plain pointers and sizes only (no torch / CUDA types in the signatures).  The Python
 * layer classes in kapre_b200/ (mirrors of kapre.STFT / InverseSTFT / Magnitude /
 * ApplyFilterbank / MagnitudeToDecibel) bind them with ctypes; INTEGRATION.md shows the
 * stub a kapre maintainer would add.
 *
 * Conventions
 *   - every function returns 0 on success or a negative KAPRE_E_* code; the message is
 *     available from kapre_last_error() (thread-local).  Nothing throws across the ABI.
 *   - `*_dev` pointers are device pointers on the CUDA device that was current when the plan
 *     was created; the caller owns every data buffer.  The library allocates only the small
 *     constant tables held by plans (window, twiddles, banded filterbank).
 *   - every call only enqueues work on `stream` (a cudaStream_t passed as void*; NULL = the
 *     legacy default stream) and returns; nothing synchronises.
 *   - tensors are described by element strides, so both of kapre's data formats
 *     ('channels_first' (B,C,T,F) / 'channels_last' (B,T,F,C); waveforms (B,C,L) / (B,L,C))
 *     are served without transposes (replaces kapre/time_frequency.py:164-167,184-185,
 *     304-305,316-317,546-547).
 */
#ifndef KAPRE_B200_H_
#define KAPRE_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define KAPRE_B200_VERSION 200

enum {
    KAPRE_OK = 0,
    KAPRE_E_INVALID = -1,      /* bad argument */
    KAPRE_E_UNSUPPORTED = -2,  /* valid in the reference but not implemented here */
    KAPRE_E_CUDA = -3,         /* CUDA runtime error (see kapre_last_error) */
    KAPRE_E_NOMEM = -4
};

/* What kapre_stft_forward writes.  One launch replaces the layer chain named on the right. */
enum {
    KAPRE_OUT_COMPLEX = 0, /* complex64   kapre.STFT                         time_frequency.py:146-187 */
    KAPRE_OUT_MAG = 1,     /* float32     STFT -> Magnitude                  time_frequency.py:351-359 */
    KAPRE_OUT_MAG_DB = 2,  /* float32     STFT -> Magnitude -> MagnitudeToDecibel      composed.py:32-135 */
    KAPRE_OUT_FB = 3,      /* float32     STFT -> Magnitude -> ApplyFilterbank         composed.py:138-261 */
    KAPRE_OUT_FB_DB = 4,   /* float32     ... -> ApplyFilterbank -> MagnitudeToDecibel composed.py:254-261 */
    KAPRE_OUT_MAG_PHASE = 5 /* float32    get_stft_mag_phase (composed.py:420-511): the output tensor has 2*channels
                             *             channels, magnitudes (dB-scaled if `db` is given) in channels [0, C) and
                             *             tf.math.angle phases in channels [C, 2C) */
};

/* Waveform tensor: element strides of (batch, channel, sample). */
typedef struct {
    int32_t batch, channels, length;
    int64_t stride_b, stride_c, stride_l;
} kapre_wave_desc;

/* Spectrogram tensor: element strides of (batch, channel, frame, bin).  Elements are
 * float32, or complex64 (one element = 8 bytes) for complex STFTs. */
typedef struct {
    int64_t stride_b, stride_c, stride_t, stride_f;
} kapre_spec_desc;

/* kapre.MagnitudeToDecibel(ref_value, amin, dynamic_range), kapre/backend.py:126-194. */
typedef struct {
    float ref_value, amin, dynamic_range;
} kapre_db_cfg;

typedef struct kapre_stft_plan kapre_stft_plan;
typedef struct kapre_istft_plan kapre_istft_plan;
typedef struct kapre_filterbank kapre_filterbank;

/* ---- forward STFT (kapre.STFT.__init__/call, kapre/time_frequency.py:101-187) -------------
 * `window_host`: win_length analysis-window samples (host memory), i.e. what
 * backend.get_window_fn(window_name)(win_length) returns (kapre/backend.py:58-100).
 * n_fft in {256,512,1024,2048} runs the fused FFT kernel; any other n_fft >= 2 runs the
 * direct-DFT kernel (same results, slower). */
int kapre_stft_plan_create(int n_fft, int win_length, int hop_length, const float* window_host,
                           kapre_stft_plan** out);
void kapre_stft_plan_destroy(kapre_stft_plan* plan);

/* Frames produced for `length` samples: tf.signal.frame semantics after kapre's pad_begin
 * (n_fft - hop zeros in front, kapre/time_frequency.py:169-172). */
int kapre_stft_num_frames(const kapre_stft_plan* plan, int length, int pad_begin, int pad_end);

/* 1 if kapre_stft_forward can produce `mode` in one fused launch for this plan. */
int kapre_stft_supports_mode(const kapre_stft_plan* plan, int mode);

/* Enqueue the transform.  `fb` is required for KAPRE_OUT_FB / _FB_DB, `db` for *_DB.
 * `workspace_dev`: at least 8 * batch bytes, needed for *_DB (per-item maxima for the
 * dynamic-range clamp of kapre/backend.py:190-192 + per-item arrival counters of the clamp pass, which
 * runs several CTAs per long item); may be NULL otherwise.  The workspace is
 * SELF-CLEANING: it must be all-zero when first passed in (cudaMemset once after allocation)
 * and every call leaves it all-zero again, so it can be reused by later calls on the same
 * stream without further memsets. */
int kapre_stft_forward(const kapre_stft_plan* plan, const float* x_dev, const kapre_wave_desc* x_desc,
                       int pad_begin, int pad_end, int mode, void* out_dev,
                       const kapre_spec_desc* out_desc, const kapre_filterbank* fb,
                       const kapre_db_cfg* db, void* workspace_dev, void* stream);

/* ---- inverse STFT (kapre.InverseSTFT, kapre/time_frequency.py:246-319) ---------------------
 * `dual_window_host`: win_length samples of tf.signal.inverse_stft_window_fn(hop, forward
 * window) (kapre/time_frequency.py:278-280).  Output length is (frames-1)*hop + win_length. */
int kapre_istft_plan_create(int n_fft, int win_length, int hop_length, const float* dual_window_host,
                            kapre_istft_plan** out);
void kapre_istft_plan_destroy(kapre_istft_plan* plan);
int kapre_istft_inverse(const kapre_istft_plan* plan, const void* stft_dev, int batch, int channels,
                        int frames, const kapre_spec_desc* stft_desc, float* y_dev,
                        const kapre_wave_desc* y_desc, void* stream);

/* ---- filterbank (kapre.ApplyFilterbank, kapre/time_frequency.py:501-548) --------------------
 * `fb_host`: row-major (n_freq, n_bands) float32 matrix, e.g. backend.filterbank_mel(...)
 * (kapre/backend.py:197-231) or backend.filterbank_log(...) (kapre/backend.py:234-299).
 * Gradient: the layer is linear, so its vector-Jacobian product is kapre_apply_filterbank with a
 * second filterbank made from the TRANSPOSED (n_bands, n_freq) matrix, applied to the gradient of
 * the output (n_bands bins in, n_freq bins out).  A mel or log bank is banded and so is its transpose. */
int kapre_filterbank_create(const float* fb_host, int n_freq, int n_bands, kapre_filterbank** out);
void kapre_filterbank_destroy(kapre_filterbank* fb);
int kapre_apply_filterbank(const kapre_filterbank* fb, const float* x_dev, int batch, int channels,
                           int frames, const kapre_spec_desc* x_desc, float* out_dev,
                           const kapre_spec_desc* out_desc, void* stream);

/* ---- element-wise layers ------------------------------------------------------------------- */
/* kapre.Magnitude (tf.abs of complex64), kapre/time_frequency.py:351-359; n complex elements. */
int kapre_magnitude(const void* x_complex_dev, float* out_dev, int64_t n, void* stream);
/* kapre.Phase (tf.math.angle), kapre/time_frequency.py:391-402; n complex elements. */
int kapre_phase(const void* x_complex_dev, float* out_dev, int64_t n, void* stream);
/* backend.magnitude_to_decibel on a contiguous (n_items, item_size) tensor: the maximum for the
 * dynamic-range clamp is taken per item (kapre/backend.py:178-192); pass n_items = 1 for a
 * 1-D input (global maximum).  workspace_dev: >= 8 * n_items bytes, zero on entry, left zero
 * (self-cleaning, see kapre_stft_forward).  In-place is allowed. */
int kapre_magnitude_to_decibel(const float* x_dev, float* out_dev, int64_t n_items, int64_t item_size,
                               const kapre_db_cfg* db, void* workspace_dev, void* stream);

/* kapre.ConcatenateFrequencyMap (kapre/time_frequency.py:648-744): contiguous (b, t, f, ch) [channels_last != 0] or
 * (b, ch, t, f) float32 input -> the same with one more channel holding linspace(0, 1, n_freq) along the frequency axis. */
int kapre_concat_frequency_map(const float* x_dev, float* out_dev, int64_t batch, int64_t channels, int64_t frames,
                               int64_t n_freq, int channels_last, void* stream);

/* kapre.SpecAugment (kapre/augmentation.py:116-326) on a contiguous (batch, frames, n_freq) float32 tensor (depth 1: both data
 * formats have this memory layout).  `time_masks_dev` / `freq_masks_dev`: (batch, n_masks, 2) int32 (start, width) pairs; an element
 * whose time (frequency) index lies in [start, start + width] of any mask of its item becomes mask_value.  The pairs are drawn by the
 * caller (width ~ U{0..param-1}, start ~ U{0..limit-width-1}, as the reference does per item and mask). */
int kapre_spec_augment(const float* x_dev, float* out_dev, int64_t batch, int64_t frames, int64_t n_freq,
                       const int* time_masks_dev, int n_time_masks, const int* freq_masks_dev, int n_freq_masks,
                       float mask_value, void* stream);

/* ---- backward passes (vector-Jacobian products) ----------------------------------------------
 * Gradients follow PyTorch's convention for complex tensors: dL/dRe + i dL/dIm.  Same stream and
 * ownership rules as the forward calls; the library allocates no data buffers.
 *
 * Gradient of kapre_stft_forward(KAPRE_OUT_COMPLEX): g (complex64, `frames` frames of n_fft/2+1 bins)
 * -> gx (float32 waveform of gx_desc->length samples, the length the forward call saw).  Runs the
 * inverse-STFT kernel of an adjoint plan (made on first use, freed with `plan`) and one small pass.
 * `workspace_dev`: kapre_stft_backward_workspace_bytes() bytes of scratch for the overlap-add of the
 * padded signal (contents ignored); that size is 0, and NULL may be passed, when the overlap-add can be
 * written straight into gx (no pad_begin and no frame past the signal's end). */
int64_t kapre_stft_backward_workspace_bytes(const kapre_stft_plan* plan, int batch, int channels, int length,
                                            int pad_begin, int pad_end);
int kapre_stft_backward(const kapre_stft_plan* plan, const void* g_dev, const kapre_spec_desc* g_desc, int batch,
                        int channels, int frames, int pad_begin, int pad_end, float* gx_dev,
                        const kapre_wave_desc* gx_desc, void* workspace_dev, void* stream);
/* Gradient of kapre_istft_inverse: gy (float32, (frames-1)*hop + win_length samples) -> gX (complex64,
 * `frames` frames of n_fft/2+1 bins).  Runs the forward STFT kernel of an adjoint plan (made on first
 * use, freed with `plan`) and one small pass over the DC and Nyquist bins. */
int kapre_istft_backward(const kapre_istft_plan* plan, const float* gy_dev, const kapre_wave_desc* gy_desc, int batch,
                         int channels, int frames, void* gX_dev, const kapre_spec_desc* gX_desc, void* stream);
/* Gradient of kapre_magnitude: gX = g X / |X|, 0 where |X| = 0; n complex elements. */
int kapre_magnitude_backward(const void* x_complex_dev, const float* g_dev, void* gx_complex_dev, int64_t n,
                             void* stream);
/* Gradient of kapre_magnitude_to_decibel (and of the decibel tail of the fused modes) with respect to its
 * input x, given the gradient g of its output; TensorFlow's rules: tf.maximum passes the gradient to its
 * first argument on ties, the threshold's gradient goes to the item's maximum (split among tied maxima).
 * workspace_dev: >= 12 * n_items bytes, zero on entry, left zero (self-cleaning).  gx may alias g, not x. */
int kapre_magnitude_to_decibel_backward(const float* x_dev, const float* g_dev, float* gx_dev, int64_t n_items,
                                        int64_t item_size, const kapre_db_cfg* db, void* workspace_dev, void* stream);
/* Gradient of kapre_phase: gX = g i X / |X|^2 (torch.angle's rule), 0 where |X| = 0; n complex elements. */
int kapre_phase_backward(const void* x_complex_dev, const float* g_dev, void* gx_complex_dev, int64_t n, void* stream);
/* Gradient of kapre_stft_forward(KAPRE_OUT_MAG_PHASE) with respect to the complex spectrum X (recomputed by the
 * caller with KAPRE_OUT_COMPLEX): gX = X / |X| (g_mag + i g_phase / |X|), 0 where |X| = 0.  g_mag is the magnitude
 * half's gradient, taken through kapre_magnitude_to_decibel_backward first when the forward was decibel-scaled;
 * g_phase the phase half's.  Every tensor is (batch, channels, frames, n_freq) with its own element strides, so
 * both halves can be read where they lie in the 2C-channel gradient; a NULL g_mag or g_phase (and its descriptor)
 * means zero.  gX must not alias X. */
int kapre_mag_phase_backward(const void* x_complex_dev, const kapre_spec_desc* x_desc, const float* g_mag_dev,
                             const kapre_spec_desc* g_mag_desc, const float* g_phase_dev,
                             const kapre_spec_desc* g_phase_desc, void* gx_complex_dev, const kapre_spec_desc* gx_desc,
                             int batch, int channels, int frames, int n_freq, void* stream);
/* Gradient of kapre_delta on the same contiguous (outer, frames, inner) layout:
 *   gx[s] = sum_t sum_{m=1..n} m ([P(t+m) = s] - [P(t-m) = s]) g[t] / (2 sum m^2),
 * P the pad_mode extension of the time axis (a position P sends to zero contributes nothing); in the interior
 * gx[s] = sum_m m (g[s-m] - g[s+m]) / (2 sum m^2).  One gather per element, no atomics; not in place. */
int kapre_delta_backward(const float* g_dev, float* gx_dev, int64_t outer, int64_t frames, int64_t inner,
                         int win_length, int pad_mode, void* stream);
/* Gradient of kapre_frame: g (frames frames of frame_length samples, g_desc strides as kapre_frame's out_desc)
 * -> gx[s] = sum over frames t with 0 <= s - t*hop < frame_length of g[t, s - t*hop], for the gx_desc->length
 * samples of the signal (pad_value positions are constants and drop out); samples no frame covers get 0. */
int kapre_frame_backward(const float* g_dev, const kapre_spec_desc* g_desc, int frames, int frame_length,
                         int hop_length, float* gx_dev, const kapre_wave_desc* gx_desc, void* stream);
/* Gradient of kapre_energy: g (g_desc->length = frames) and the forward's input x ->
 * gx[s] = 2 * scale * x[s] * sum over frames t covering s of g[t]; 0 for samples no frame covers (the gaps when
 * hop_length > frame_length). */
int kapre_energy_backward(const float* x_dev, const kapre_wave_desc* x_desc, const float* g_dev,
                          const kapre_wave_desc* g_desc, int frame_length, int hop_length, float scale, float* gx_dev,
                          const kapre_wave_desc* gx_desc, void* stream);
/* Gradient of kapre_concat_frequency_map: gx = the first `channels` channels of the contiguous (channels + 1)-channel
 * gradient g, in either data format; gx contiguous with `channels` channels. */
int kapre_concat_frequency_map_backward(const float* g_dev, float* gx_dev, int64_t batch, int64_t channels,
                                        int64_t frames, int64_t n_freq, int channels_last, void* stream);
/* SpecAugment has no entry of its own: its gradient is kapre_spec_augment over the gradient with mask_value = 0
 * and the same device masks. */

/* ---- adjacent layers ------------------------------------------------------------------------ */
/* kapre.Delta (kapre/time_frequency.py:563-644): y[t] = sum_{m=-n..n} m * x[t+m] / (2 sum m^2) along the
 * time axis of a contiguous tensor viewed as (outer, frames, inner); x is extended beyond its ends by
 * `pad_mode` (0 = symmetric, 1 = reflect, 2 = constant zero -- tf.pad's modes).  win_length = 2n+1. */
int kapre_delta(const float* x_dev, float* out_dev, int64_t outer, int64_t frames, int64_t inner,
                int win_length, int pad_mode, void* stream);
/* kapre.Frame (kapre/signal.py:22-119, tf.signal.frame): out[b, c, t, n] = x[b, c, t*hop + n], or
 * pad_value beyond the signal when pad_end.  out_desc strides are (batch, channel, frame, sample-in-frame). */
int kapre_frame(const float* x_dev, const kapre_wave_desc* x_desc, int frame_length, int hop_length, int pad_end,
                float pad_value, float* out_dev, const kapre_spec_desc* out_desc, void* stream);
/* kapre.Energy (kapre/signal.py:123-233): scale * sum_n frame[n]^2 per frame; out_desc.length = frames. */
int kapre_energy(const float* x_dev, const kapre_wave_desc* x_desc, int frame_length, int hop_length, int pad_end,
                 float pad_value, float scale, float* out_dev, const kapre_wave_desc* out_desc, void* stream);

/* ---- resampling ------------------------------------------------------------------------------
 * Polyphase resampler, scipy.signal.resample_poly(x, up, down) with zeros outside the signal:
 *   y[n] = up * sum_i x[i] h[hl + n*down - i*up]   (h: n_taps = 2*hl + 1 taps, terms outside h are zero).
 * `taps_host`: the n_taps float32 filter taps (host memory), e.g. kapre_b200.signal.resample_filter(up, down), the
 * windowed sinc firwin(20 max(up, down) + 1, 1 / max(up, down), window=('kaiser', 5.0)).  up and down must be
 * coprime and max(up, down) <= 1280 (every pair of 8, 11.025, 16, 22.05, 24, 32, 44.1, 48, 88.2 and 96 kHz);
 * larger ratios return KAPRE_E_UNSUPPORTED, because the polyphase table (up to 143 KB) must fit in shared memory. */
typedef struct kapre_resample_plan kapre_resample_plan;
int kapre_resample_plan_create(int up, int down, const float* taps_host, int n_taps, kapre_resample_plan** out);
void kapre_resample_plan_destroy(kapre_resample_plan* plan);
/* ceil(length * up / down): the output length of scipy.signal.resample_poly. */
int64_t kapre_resample_output_length(const kapre_resample_plan* plan, int64_t length);
/* Resample along the sample axis.  y_desc has x_desc's batch and channels; y_desc->length outputs are written
 * (normally kapre_resample_output_length(x_desc->length)).  Any strides; y must not overlap x. */
int kapre_resample(const kapre_resample_plan* plan, const float* x_dev, const kapre_wave_desc* x_desc, float* y_dev,
                   const kapre_wave_desc* y_desc, void* stream);
/* Gradient of kapre_resample: gx = (up / down) * resample(g; down, up), cropped to gx_desc->length samples (the
 * length the forward call saw).  This is the adjoint because the filter is symmetric (KAPRE_E_UNSUPPORTED
 * otherwise).  Runs the forward kernel of an adjoint plan (made on first use, freed with `plan`). */
int kapre_resample_backward(const kapre_resample_plan* plan, const float* g_dev, const kapre_wave_desc* g_desc,
                            float* gx_dev, const kapre_wave_desc* gx_desc, void* stream);

/* ---- band-limited interpolation: resampling by any real ratio ------------------------------------
 * J. O. Smith's algorithm (what resampy / librosa's kaiser_best do) with a table that does not depend on the
 * ratio.  With Z = 10 zero crossings and Kaiser beta 5 (the family of the polyphase filter above):
 *   h(u) = sinc(u) I0(5 sqrt(1 - (u/Z)^2)) / I0(5) for |u| < Z, else 0;      I = integral of h over [-Z, Z]
 *   y[m] = (g / I) sum_j x[j] h(s (offset + m / ratio - j)),   s = g = min(1, ratio),   x[j] = 0 outside the signal.
 * `ratio` = output rate / input rate; the cutoff is the lower of the two Nyquist rates.  `offset` is the position of
 * output sample 0 in input samples (0: the two signals start together).  A ratio outside [0.25, 4] (two octaves
 * either way, at most 80 taps per output), a non-finite ratio or offset, or |offset| > 2^40 returns KAPRE_E_INVALID
 * before anything is launched.  The filter is tabulated at 1024 points per zero crossing and read by linear
 * interpolation: an output is within 1.7e-5 max|x| of the sum above (1e-6 typical).  At rational ratios this is
 * scipy.signal.resample_poly up to its normalisation (scipy divides by the tap sum): 1e-4 .. 6e-4 of unit-variance
 * input at 1:3, 3:2 and 2:1.
 * The plan is the device table of h for the current device; it takes no arguments, and one plan serves every ratio. */
typedef struct kapre_sinc_plan kapre_sinc_plan;
int kapre_sinc_plan_create(kapre_sinc_plan** out);
void kapre_sinc_plan_destroy(kapre_sinc_plan* plan);
/* Interpolate along the sample axis in one launch.  y_desc has x_desc's batch and channels; y_desc->length outputs are
 * written whatever the ratio (ceil(x_desc->length * ratio) covers the input): outputs whose support lies past the
 * signal are exactly 0, so cropping or zero-padding to a given length costs nothing.  Any strides; y must not overlap
 * x.  An output sample does not depend on the batch size, the data layout or the strides. */
int kapre_sinc_resample(const kapre_sinc_plan* plan, const float* x_dev, const kapre_wave_desc* x_desc, float* y_dev,
                        const kapre_wave_desc* y_desc, double ratio, double offset, void* stream);
/* Gradient of kapre_sinc_resample called with the same (ratio, offset): gx = A^T g, written for gx_desc->length
 * samples (the length the forward call saw).  Because h is even this is the same sum with step ratio instead of
 * 1 / ratio, offset -offset * ratio and s / ratio instead of s: the same kernel, one launch. */
int kapre_sinc_resample_backward(const kapre_sinc_plan* plan, const float* g_dev, const kapre_wave_desc* g_desc,
                                 float* gx_dev, const kapre_wave_desc* gx_desc, double ratio, double offset, void* stream);

/* ---- convolution with long filters (uniformly partitioned overlap-add) ---------------------------
 * y = x * h (full linear convolution along the sample axis) through this library's transform pair: with a block size
 * B in {128, 256, 512, 1024},
 *   X = STFT(x; n_fft 2B, window ones(B), hop B, pad_end): J = ceil(L / B) blocks, block j = x[jB, jB + B) zero-padded
 *   H = the same transform of h: P = ceil(K / B) blocks
 *   Y_i = sum_{p < P} H_p X_{i - p}   (X_j = 0 outside [0, J)),  i < T = J + P - 1
 *   y = InverseSTFT(Y; n_fft 2B, hop B, dual window ones(2B)): (T + 1) B samples, of which the first L + K - 1 are
 *       the convolution and the rest are zero up to rounding.
 * The per-bin sum runs in a fixed order (p ascending), so an output sample does not depend on the batch size, the
 * item's position, the strides or broadcasting.  Across data layouts it agrees to float32 rounding: an interleaved
 * multi-channel waveform is transformed by kapre_stft_forward's all-channel kernel.  An output is within a few 1e-6 of rms(x) ||h||_2
 * (DESIGN.md §4 gives the bound).  Spectra (H, X, their gradients) are (batch, channels, blocks, B + 1 bins)
 * complex64 with kapre_spec_desc strides; a batch or channel stride of 0 in H_desc broadcasts one filter over the
 * batch or the channels, without a copy. */
typedef struct kapre_convolve_plan kapre_convolve_plan;
/* The block size B for a filter of ir_length taps: a function of the length alone (so an output's bits depend on the
 * inputs alone), the one kapre_b200's layers use.  KAPRE_E_INVALID for ir_length < 1. */
int64_t kapre_convolve_block_size(int64_t ir_length);
/* The transform pair of one block size (128, 256, 512 or 1024, else KAPRE_E_INVALID) on the current device. */
int kapre_convolve_plan_create(int block, kapre_convolve_plan** out);
void kapre_convolve_plan_destroy(kapre_convolve_plan* plan);
/* H = the block spectra of h (h_desc->length = K >= 1 taps, any batch and channels, any strides): P = ceil(K / B)
 * blocks written through H_desc.  One launch; callers keep H, so a filter bank is transformed once. */
int kapre_convolve_ir_spectrum(const kapre_convolve_plan* plan, const float* h_dev, const kapre_wave_desc* h_desc,
                               void* H_dev, const kapre_spec_desc* H_desc, void* stream);
/* Scratch of kapre_convolve: X (J blocks) and Y (T blocks) for batch x channels signals of `length` samples, each
 * rounded up to 256 B.  < 0 on error (length < 1, P < 1, or (T + 1) B beyond int32). */
int64_t kapre_convolve_workspace_bytes(const kapre_convolve_plan* plan, int batch, int channels, int length, int P);
/* y = x * h given H (P blocks, batch and channels as x's or broadcast through zero strides).  y_desc: x's batch and
 * channels and exactly (T + 1) B samples, any strides; crop it for torchaudio's 'full' / 'same' / 'valid'.  Three
 * launches: STFT, the per-bin multiply-accumulate, the inverse.  `workspace_dev`: kapre_convolve_workspace_bytes
 * bytes; on return it begins with X, (batch, channels, J, B + 1) complex64 contiguous, which
 * kapre_convolve_backward reads for the filter's gradient.  Sizes that are invalid for kapre_convolve_workspace_bytes
 * return KAPRE_E_INVALID here before anything is launched. */
int kapre_convolve(const kapre_convolve_plan* plan, const float* x_dev, const kapre_wave_desc* x_desc, const void* H_dev,
                   const kapre_spec_desc* H_desc, int P, float* y_dev, const kapre_wave_desc* y_desc, void* workspace_dev,
                   void* stream);
/* Scratch of kapre_convolve_backward: G (T blocks), the signal spectra's gradient (J blocks) and, when length is not a
 * multiple of B, batch x channels x J B floats of overlap-add scratch. */
int64_t kapre_convolve_backward_workspace_bytes(const kapre_convolve_plan* plan, int batch, int channels, int length,
                                                int P);
/* Gradients of kapre_convolve given the gradient gy of its untrimmed (T + 1) B-sample output (zero where the caller
 * cropped it away).  G = InverseSTFT^T(gy); then
 *   gx = STFT^T(gX),  gX_j = sum_{p < P} conj(H_p) G_{j + p}    (j < J; written when gx_dev is not NULL)
 *   gH_p = sum_{j < J} conj(X_j) G_{j + p}                      (p < P; per (item, channel), written when gH_dev is
 *                                                               not NULL, from the X kapre_convolve left in its workspace)
 * gx_desc is required in both cases: its batch, channels and length (the forward's L) fix the geometry.  Sum gH
 * over a broadcast filter's batch or channels before kapre_convolve_ir_spectrum_backward. */
int kapre_convolve_backward(const kapre_convolve_plan* plan, const float* gy_dev, const kapre_wave_desc* gy_desc,
                            const void* H_dev, const kapre_spec_desc* H_desc, const void* X_dev,
                            const kapre_spec_desc* X_desc, int P, float* gx_dev, const kapre_wave_desc* gx_desc,
                            void* gH_dev, const kapre_spec_desc* gH_desc, void* workspace_dev, void* stream);
/* gh = the gradient of kapre_convolve_ir_spectrum given gH (P blocks), for gh_desc->length = K taps with
 * ceil(K / B) = P.  `workspace_dev`: batch x channels x P B floats of scratch when K is not a multiple of B, else it
 * may be NULL. */
int kapre_convolve_ir_spectrum_backward(const kapre_convolve_plan* plan, const void* gH_dev, const kapre_spec_desc* gH_desc,
                                        int P, float* gh_dev, const kapre_wave_desc* gh_desc, void* workspace_dev,
                                        void* stream);

/* ---- IIR filters (torchaudio.functional.lfilter) ---------------------------------------------------
 * Along the time axis of every (item, channel) column, with normalised coefficients (b / a0, a / a0):
 *   y[t] = sum_{k=0..N} b[k] x[t-k] - sum_{k=1..N} a[k] y[t-k],   x, y = 0 before t = 0,
 * then clamped to [-1, 1] with KAPRE_IIR_CLAMP.  KAPRE_IIR_REVERSE runs the filter in reverse time (sample t is
 * read and written at L-1-t), which is filtfilt's second pass without a flip.  Order N <= 8
 * (KAPRE_E_UNSUPPORTED above).  Coefficients: N + 1 consecutive floats per filter at b + i stride_b + c stride_c
 * (a[0] is not read); a stride of 0 shares one filter over the batch or the channels.
 * The kernel cuts time into chunks of 65 samples and carries the chunk states in float64 (DESIGN.md §IIR), so that
 * y[t] depends on x[0..t] and the coefficients alone: not on the length, the batch, the strides or broadcasting.
 * Four launches: the state-transition powers, the chunk states, the carry across blocks of 32 chunks, the output. */
typedef struct {
    const float* b;
    const float* a;
    int64_t b_stride_b, b_stride_c, a_stride_b, a_stride_c;
    int order;
} kapre_iir_coeffs;
#define KAPRE_IIR_CLAMP 1
#define KAPRE_IIR_REVERSE 2
/* Scratch of kapre_lfilter and kapre_lfilter_backward.  < 0 on error: a negative size, an order outside [0, 8], or a
 * workspace or chunk count beyond int64 / int32. */
int64_t kapre_lfilter_workspace_bytes(int batch, int channels, int length, int order);
/* y = lfilter(x).  x_desc and y_desc: same batch, channels and length, any strides; y must not alias x. */
int kapre_lfilter(const float* x_dev, const kapre_wave_desc* x_desc, const kapre_iir_coeffs* coeffs, int flags,
                  float* y_dev, const kapre_wave_desc* y_desc, void* workspace_dev, void* stream);
/* Gradients of kapre_lfilter (called with the forward's flags; KAPRE_IIR_CLAMP is ignored: the gradient is that of
 * the unclamped output).  With v the all-pole recursion run the other way on gy,
 *   gx[t] = sum_k b[k] v[t+k],   gb[k] = sum_t v[t] x[t-k],   ga[k] = -sum_t v[t] y[t-k]  (k >= 1, y unclamped).
 * partials_dev (optional; needs x_dev and y_dev): (2 N + 1, batch, channels, ceil(length / 65)) float32, row k <= N
 * the gb[k] sums per chunk, row N + k the ga[k] sums; the caller sums them (over broadcast axes too).  Four
 * launches. */
int kapre_lfilter_backward(const float* gy_dev, const kapre_wave_desc* gy_desc, const float* x_dev,
                           const kapre_wave_desc* x_desc, const float* y_dev, const kapre_wave_desc* y_desc,
                           const kapre_iir_coeffs* coeffs, int flags, float* gx_dev, const kapre_wave_desc* gx_desc,
                           float* partials_dev, void* workspace_dev, void* stream);

/* ---- second-order-section cascades (scipy.signal.sosfilt) -------------------------------------------------------
 * Along the time axis of every (item, channel) column, S sections in row order, each row [b0, b1, b2, a0, a1, a2]
 * in direct form II transposed with state (z1, z2) (a0 is taken to be 1 and not read):
 *   y_s[t] = b0 x_s[t] + z1,   z1 <- b1 x_s[t] - a1 y_s[t] + z2,   z2 <- b2 x_s[t] - a2 y_s[t],
 * x_0 = x, x_(s+1) = y_s, y = y_(S-1).  1 <= S <= 8 (KAPRE_E_UNSUPPORTED otherwise).  Coefficients: S rows of 6
 * consecutive floats per filter at sos + i stride_b + c stride_c; a stride of 0 shares one filter over the batch or
 * the channels.  KAPRE_IIR_REVERSE runs the cascade in reverse time (sample t is read and written at L-1-t).
 * The kernel is lfilter's chunked scan over the cascade's 2S-dimensional state (DESIGN.md §SOS): y[t] depends on
 * x[0..t], the coefficients and zi alone, not on the length, the batch, the strides or broadcasting.  Four launches. */
typedef struct {
    const float* sos;
    int64_t stride_b, stride_c;
    int n_sections;
} kapre_sos_coeffs;
/* A (batch, channels, S, 2) float32 state in scipy's convention: (z1, z2) of section s of column (i, c) are the two
 * consecutive floats at i stride_b + c stride_c + s stride_s.  Strides of 0 broadcast an initial state. */
typedef struct {
    int64_t stride_b, stride_c, stride_s;
} kapre_sos_state_desc;
/* Scratch of kapre_sosfilt.  < 0 on error: a negative size, n_sections outside [1, 8], or a workspace or chunk count
 * beyond int64 / int32. */
int64_t kapre_sosfilt_workspace_bytes(int batch, int channels, int length, int n_sections);
/* y = sosfilt(x) from the initial state zi (NULL: zero), writing the final state to zf when zf_dev is not NULL (the
 * state after the last sample processed, which is sample 0 with KAPRE_IIR_REVERSE; not written when length is 0).
 * flags: 0 or KAPRE_IIR_REVERSE.  x_desc and y_desc: same batch, channels and length, any strides; y must not alias
 * x. */
int kapre_sosfilt(const float* x_dev, const kapre_wave_desc* x_desc, const kapre_sos_coeffs* sos, const float* zi_dev,
                  const kapre_sos_state_desc* zi_desc, int flags, float* y_dev, const kapre_wave_desc* y_desc,
                  float* zf_dev, const kapre_sos_state_desc* zf_desc, void* workspace_dev, void* stream);

/* ---- image-source room impulse responses (DESIGN.md §RIR) -----------------------------------------------------------
 * Shoebox room [0, Lx] x [0, Ly] x [0, Lz], walls (x=0, x=Lx, y=0, y=Ly, z=0, z=Lz) with pressure reflection
 * coefficients beta_w.  Image (n, p), n in Z^3, p in {0,1}^3: i_d = 2 n_d L_d + (1 - 2 p_d) s_d, r = |i - m|,
 * tau = r fs / c, g = prod_d beta_(d,lo)^|n_d - p_d| beta_(d,hi)^|n_d| / (4 pi r), and
 *   h[floor(tau) + k] += g w[k] sinc(k - half - frac(tau)),  k < W,  w = np.hanning(W),
 * over the images of order <= max_order (all, when it is -1).  Output samples [start, start + output_length) of every
 * (item, mic) response, float32 at element strides (stride_b, stride_m, stride_t).  A sample's bits depend only on
 * its item's record, its mic and its index, not on the batch, the strides or start.  One launch.
 * records: batch records of 14 float64 (room[3], source[3], beta[6], max_order, start), then (batch, n_mics, 3)
 * float64 mic positions; records_host is validated before anything is launched and records_dev (the same values on
 * the device) is what the kernel reads.  KAPRE_E_INVALID for a side that is not finite and positive, a source or mic
 * not strictly inside its room, a mic within 1 mm of the source, beta outside [0, 1], a max_order that is not -1 or a
 * non-negative integer, a start that is not a non-negative integer or with start + output_length >= 2^31, an even
 * filter_length or one outside [1, 255], output_length < 1, and a response whose image bound (lattice boxes meeting
 * the arrival ball of radius (start + output_length) c / fs, times 8) exceeds 2^24, whatever its max_order: the
 * kernel's enumeration walks the whole ball.
 * With records_dev and out_dev both NULL the call only validates records_host.
 * KAPRE_RIR_UNIT_NORM: a second launch scales each response to unit L2 norm (a float64 sum in a fixed order). */
#define KAPRE_RIR_UNIT_NORM 1
int kapre_rir_ism(const double* records_host, const double* records_dev, int batch, int n_mics, int output_length,
                  int filter_length, double sample_rate, double sound_speed, int flags, float* out_dev,
                  int64_t stride_b, int64_t stride_m, int64_t stride_t, void* stream);

/* ---- additive noise at a target SNR (torchaudio.functional.add_noise) -------------------------------------------
 * For every (item, channel) column of x (L samples), noise n, snr in dB and valid length len:
 *   Ex = sum_{t < len} x[t]^2,  En = sum_{t < len} n[t]^2,  s = sqrt(Ex / En) 10^(-snr / 20),  y[t] = x[t] + s n[t]
 * for every t < L (noise is added past len too, as torchaudio does).  The mask is t < len, so len <= 0 counts no
 * sample and len >= L every sample.  Ex, En and s are float64, s is rounded to float32 once and y = fmaf(s, n, x).
 * One deviation from torchaudio: where En == 0 (or Ex == 0) s = 0 and y = x bit for bit, where torchaudio gives NaN
 * for En == 0.  A NaN or inf in x or n makes that column non-finite.  The summation order depends on the column and
 * the absolute sample index alone (segments of 4096 samples, a fixed tree per segment, the segments folded in order;
 * no atomics), so an output's bits do not depend on the batch, the strides, the data format, broadcasting, or
 * whether the noise comes from a tensor or a bank.  Two launches each way. */
#define KAPRE_NOISE_TENSOR 0
#define KAPRE_NOISE_BANK 1
typedef struct {
    int mode;                   /* KAPRE_NOISE_TENSOR or KAPRE_NOISE_BANK */
    /* TENSOR: (batch, channels, length) with batch 1 or x's, channels 1 or x's and x's length; a batch or channel of 1
     * (or a stride of 0) broadcasts without a copy. */
    const float* noise;
    kapre_wave_desc noise_desc;
    /* BANK: bank_length floats of concatenated mono clips; per item (device arrays of batch int64) the clip's first
     * sample `start`, its length `clip_len` and `offset`: n[b, c, t] = bank[start[b] + (offset[b] + t) mod clip_len[b]]
     * for every channel, so short clips loop.  An item whose clip is empty or does not lie inside the bank reads
     * zeros (so its output is its input). */
    const float* bank;
    int64_t bank_length;
    const int64_t* start;
    const int64_t* clip_len;
    const int64_t* offset;
} kapre_noise_source;
/* snr (float32, required) and lengths (int32, optional: NULL means every sample counts) at
 * ptr + b stride_b + c stride_c; a stride of 0 broadcasts. */
typedef struct {
    const float* snr;
    int64_t snr_stride_b, snr_stride_c;
    const int32_t* lengths;
    int64_t lengths_stride_b, lengths_stride_c;
} kapre_snr_desc;
/* Scratch of kapre_add_noise and kapre_add_noise_backward: 16 bytes per (item, channel, 4096-sample segment), rounded
 * up to 256.  < 0 on a negative size or an overflow. */
int64_t kapre_add_noise_workspace_bytes(int batch, int channels, int length);
/* y = x + s n.  y_desc: x's batch, channels and length, any strides; y must not be x or the noise.  stats_dev
 * (optional): (batch, channels, 2) float64 (Ex, En) per column, which kapre_add_noise_backward reads. */
int kapre_add_noise(const float* x_dev, const kapre_wave_desc* x_desc, const kapre_noise_source* noise,
                    const kapre_snr_desc* snr, float* y_dev, const kapre_wave_desc* y_desc, double* stats_dev,
                    void* workspace_dev, void* stream);
/* Gradients of kapre_add_noise given the output gradient g, x, the same noise, snr and lengths, and the stats the
 * forward wrote.  With D = sum_{t < L} g[t] n[t] per column:
 *   gx[t] = g[t] + [t < len] (D s / Ex) x[t],  gn[t] = s g[t] - [t < len] (D s / En) n[t],  gsnr = -D s ln(10) / 20,
 * where every term through s is 0 where Ex == 0 or En == 0.  gx is required; gn (tensor noise only, x's full shape)
 * and gsnr ((batch, channels) float32, contiguous) are written when not NULL.  Sum gn and gsnr over broadcast axes. */
int kapre_add_noise_backward(const float* g_dev, const kapre_wave_desc* g_desc, const float* x_dev,
                             const kapre_wave_desc* x_desc, const kapre_noise_source* noise, const kapre_snr_desc* snr,
                             const double* stats_dev, float* gx_dev, const kapre_wave_desc* gx_desc, float* gn_dev,
                             const kapre_wave_desc* gn_desc, float* gsnr_dev, void* workspace_dev, void* stream);

/* ---- gated loudness (torchaudio.functional.loudness, ITU-R BS.1770-4) -------------------------------------------
 * On the K-weighted signal y (batch, channels <= 5, length): per item of valid length len (lengths_dev, int32 per
 * item on the device, clamped to [0, length]; NULL: every sample counts), blocks [j step, j step + gate) for
 * j <= (len - gate) / step (none when len < gate), e_cj = mean of y_c^2 over block j, E_j = sum_c g_c e_cj with
 * g = (1, 1, 1, 1.41, 1.41), l_j = -0.691 + 10 log10(E_j); J1 = {j : l_j > -70}; Gamma = -0.691 +
 * 10 log10(mean_{J1} E_j) - 10; J2 = {j in J1 : l_j > Gamma}; LKFS = -0.691 + 10 log10(mean_{J2} E_j), float64
 * throughout and rounded once to float32.  An empty J2 gives -inf (torchaudio gives NaN); a non-finite block energy
 * gives NaN.  Sums run in a fixed order that depends on the item and the absolute sample index alone, so an item's
 * result does not depend on the batch, its position, the strides, the data format or its samples past len.  K-weight
 * with two kapre_lfilter calls first (see INTEGRATION.md). */
/* Scratch of kapre_loudness (the return value) and, in *stats_bytes (may be NULL), the size of its stats buffer, which
 * kapre_loudness_backward reads.  < 0 on a bad size (channels outside [1, 5], gate < 1, step outside [1, gate]) or an
 * overflow. */
int64_t kapre_loudness_workspace_bytes(int batch, int channels, int length, int gate, int step, int64_t* stats_bytes);
/* out_dev: batch float32 LKFS.  Two launches (one when length < gate). */
int kapre_loudness(const float* y_dev, const kapre_wave_desc* y_desc, const int32_t* lengths_dev, int gate, int step,
                   float* out_dev, void* stats_dev, void* workspace_dev, void* stream);
/* gy = the gradient of kapre_loudness with respect to y at output gradient gl_dev (batch float32), given the stats
 * the forward wrote:  gy[t] = gl (20 / ln 10) g_c y[t] n(t) / (E2 |J2| gate), n(t) the J2 blocks covering t; exactly 0
 * where n(t) = 0 and for -inf items.  gy_desc: y's shape, any strides, not y.  One launch. */
int kapre_loudness_backward(const float* gl_dev, const float* y_dev, const kapre_wave_desc* y_desc,
                            const int32_t* lengths_dev, int gate, int step, const void* stats_dev, float* gy_dev,
                            const kapre_wave_desc* gy_desc, void* stream);

/* ---- loudness meter: series, loudness range and true peak (EBU R128, EBU Tech 3341 / 3342, ITU-R BS.1770-4) -----
 * kapre_loudness_stats runs on the K-weighted signal y as kapre_loudness does (same lengths rule, channels <= 5), and
 * writes per item: the integrated loudness (kapre_loudness's two passes, so bit for bit its result); the momentary
 * series (batch, Jm) with Jm = (length - gate) / step + 1 (0 when length < gate) and the short-term series
 * (batch, Js) with gate3 in place of gate, both row-major: entry j is -0.691 + 10 log10(E_j) over the window
 * [j step, j step + window), E_j the channel-weighted mean square, and -inf for j at or past the item's own window
 * count; and the loudness range (EBU Tech 3342) of the short-term windows: J1 = {s_j > -70}, Gamma = -0.691 +
 * 10 log10(mean_J1 E_j) - 20, J2 = {j in J1 : s_j > Gamma}, n = |J2|, v the ascending s of J2,
 * LRA = v[((n-1) 95 + 50) / 100] - v[((n-1) 10 + 50) / 100] (0 when n = 0), float64 and rounded once.  A non-finite
 * window energy makes that item's entries and LRA NaN.  Six launches (two when length < gate). */
/* Scratch of kapre_loudness_stats; < 0 on a bad size (as kapre_loudness, and gate3 < gate) or an overflow. */
int64_t kapre_loudness_stats_workspace_bytes(int batch, int channels, int length, int gate, int step, int gate3);
int kapre_loudness_stats(const float* y_dev, const kapre_wave_desc* y_desc, const int32_t* lengths_dev, int gate,
                         int step, int gate3, float* integrated_dev, float* momentary_dev, float* short_term_dev,
                         float* lra_dev, void* workspace_dev, void* stream);
/* True peak per (item, channel) column of a waveform x (any channel count, lengths as kapre_loudness, length <= 2^30):
 * TP = 20 log10 max_t |z[t]|, z = scipy.signal.resample_poly(x[:len], 4, 1) with taps_host the 81 float32 taps of its
 * filter (kapre_b200.signal.resample_filter(4, 1)); z is formed as kapre_resample forms it, in registers, and never
 * written.  -inf for a silent column, NaN when a NaN reaches z.  out_dev: (batch, channels) float32 row-major;
 * stats_dev (its size in *stats_bytes): z[t*] and the first argmax t*, which kapre_true_peak_backward reads. */
int64_t kapre_true_peak_workspace_bytes(int batch, int channels, int length, int64_t* stats_bytes);
/* Two launches. */
int kapre_true_peak(const float* x_dev, const kapre_wave_desc* x_desc, const int32_t* lengths_dev,
                    const float* taps_host, float* out_dev, void* stats_dev, void* workspace_dev, void* stream);
/* gx = the gradient of kapre_true_peak at output gradient g_dev ((batch, channels) float32 row-major):
 * gx[n] = g (20 / ln 10) 4 h[t* - 4n + 40] / z[t*] inside h's support and n < len, else exactly 0 (also for -inf
 * columns).  gx_desc: x's shape, any strides.  One launch. */
int kapre_true_peak_backward(const float* g_dev, const int32_t* lengths_dev, const float* taps_host,
                             const void* stats_dev, float* gx_dev, const kapre_wave_desc* gx_desc, void* stream);

/* ---- Kaldi-compatible features (torchaudio.compliance.kaldi.fbank / mfcc / spectrogram) -------------------
 * Every (item, channel) column of a float32 waveform is framed, dithered, DC-removed, pre-emphasised, windowed,
 * zero-padded to padded_window_size and transformed as torchaudio 2.11's functions do (one frame set per channel
 * instead of one selected channel).  Output: (batch, channels, frames, bins) by element strides, with
 *   fbank:        bins = num_mel_bins + use_energy   (energy first, or last with htk_compat)
 *   mfcc:         bins = num_ceps
 *   spectrogram:  bins = padded_window_size / 2 + 1
 * Item b is computed as if cut to lengths[b] samples: its frame count is
 *   snip_edges: 1 + (len - W) / shift, 0 when len < W;   otherwise (len + shift / 2) / shift, 0 when len < W,
 * and 0 when len < min_length; frames past an item's count are written as 0.  padded_window_size must be one of
 * 256, 512, 1024, 2048 (KAPRE_E_UNSUPPORTED otherwise).  Dither adds `dither` times a deterministic unit-variance
 * value keyed by (seed, item, channel, frame, sample).  An item's output bits do not depend on the batch, its
 * position, the strides, the data format or the launch shape. */
enum { KAPRE_KALDI_FBANK = 0, KAPRE_KALDI_MFCC = 1, KAPRE_KALDI_SPECTROGRAM = 2 };
typedef struct {
    int kind;                           /* KAPRE_KALDI_* */
    int window_size, window_shift;      /* samples: W >= 2, shift >= 1 */
    int padded_window_size;             /* N >= W, a power of two in [256, 2048] */
    int snip_edges;                     /* 0 or 1 */
    int min_length;                     /* samples; shorter items have no frames */
    int num_mel_bins;                   /* fbank / mfcc: 1 .. 256 */
    int num_ceps;                       /* mfcc: 1 .. num_mel_bins */
    int use_energy, htk_compat, raw_energy, use_power, use_log_fbank, remove_dc_offset, subtract_mean;
    float preemphasis_coefficient;      /* [0, 1] */
    float energy_floor;                 /* >= 0 */
} kapre_kaldi_config;
typedef struct kapre_kaldi_plan kapre_kaldi_plan;
/* window_host: W floats.  banks_host (fbank / mfcc): num_mel_bins x (N / 2 + 1) row-major mel weights.  dct_host
 * (mfcc): num_mel_bins x num_ceps, lifter applied (and c0's column scaled by sqrt 2 under htk_compat without
 * use_energy).  Options must be finite; mfcc and spectrogram need use_power and mfcc use_log_fbank. */
int kapre_kaldi_plan_create(const kapre_kaldi_config* cfg, const float* window_host, const float* banks_host,
                            const float* dct_host, kapre_kaldi_plan** out);
void kapre_kaldi_plan_destroy(kapre_kaldi_plan* plan);
/* Frames of an item of `length` samples (< 0 on a negative length); bins per frame. */
int kapre_kaldi_num_frames(const kapre_kaldi_plan* plan, int length);
int kapre_kaldi_num_bins(const kapre_kaldi_plan* plan);
/* Scratch of kapre_kaldi_features (backward = 0: none) or of kapre_kaldi_features_backward (the per-frame gradients
 * and, with subtract_mean, the centred output gradient).  < 0 on a bad size or an overflow. */
int64_t kapre_kaldi_workspace_bytes(const kapre_kaldi_plan* plan, int batch, int channels, int frames, int backward);
/* y = features(x).  lengths_host (NULL: every item is x_desc->length long) holds each item's length in [0, length];
 * lengths_dev holds the same values on the device.  frames must be the largest frame count of the batch.  One
 * launch, two with subtract_mean. */
int kapre_kaldi_features(const kapre_kaldi_plan* plan, const float* x_dev, const kapre_wave_desc* x_desc,
                         const int32_t* lengths_host, const int32_t* lengths_dev, int frames, float dither,
                         uint64_t seed, float* y_dev, const kapre_spec_desc* y_desc, void* workspace_dev,
                         void* stream);
/* gx = the gradient of features(x) to x at output gradient gy, with the forward's dither (same dither and seed).
 * Samples at or past an item's length get 0.  Two launches, three with subtract_mean. */
int kapre_kaldi_features_backward(const kapre_kaldi_plan* plan, const float* gy_dev, const kapre_spec_desc* gy_desc,
                                  const float* x_dev, const kapre_wave_desc* x_desc, const int32_t* lengths_host,
                                  const int32_t* lengths_dev, int frames, float dither, uint64_t seed, float* gx_dev,
                                  const kapre_wave_desc* gx_desc, void* workspace_dev, void* stream);

/* ---- constant-Q transform (multirate, modelled on librosa's cqt / vqt) ------------------------------------------
 * Octave i = 0 .. n_oct - 1 (n_oct = ceil(n_bins / bins_per_octave), octave 0 the top one) holds the bins
 * [max(0, n_bins - (i + 1) B), n_bins - i B) and reads pyramid level y_i: y_0 = x, y_{i+1} = resample_poly(y_i, 1, 2)
 * with the decimation filter given to the plan (L_{i+1} = ceil(L_i / 2)), hop h_i = hop_length / 2^i.  With octave i's
 * table T (one row of taps[i] complex taps per bin, the scale and the conjugate folded in),
 *   C[k, m] = sum_{j < taps[i]} y_i[m h_i + j - taps[i] / 2] T_k[j],   y_i = 0 outside [0, L_i),  m < 1 + length / hop
 * as one float32 dot product per output with j ascending, so an output's bits depend on (item, channel, octave,
 * frame, bin) alone: not on the batch, its position, the strides or the launch shape. */
#define KAPRE_CQT_MAX_OCTAVES 12
#define KAPRE_CQT_MAX_TAPS 2048
typedef struct {
    int n_bins, bins_per_octave;
    int hop_length;                       /* a multiple of 2^(n_oct - 1) */
    int taps[KAPRE_CQT_MAX_OCTAVES];      /* row length of octave i's table, 1 .. KAPRE_CQT_MAX_TAPS */
} kapre_cqt_config;
typedef struct kapre_cqt_plan kapre_cqt_plan;
/* taps_host: octave 0's table, then octave 1's, ..., each (bins of the octave) x taps[i] complex64 (float pairs),
 * bins ascending.  decim_taps_host: the odd, symmetric 2:1 decimation filter (kapre_resample_plan_create(1, 2, ...)).
 * Every octave with taps[i] <= KAPRE_CQT_MAX_TAPS fits the kernel's shared-memory staging at any hop;
 * KAPRE_E_UNSUPPORTED when the octaves need more than 256 (octave, bin group) segments, a group being the bins whose
 * taps fit 32 KB (kapre_b200.backend.cqt_geometry computes the count). */
int kapre_cqt_plan_create(const kapre_cqt_config* cfg, const float* taps_host, const float* decim_taps_host,
                          int n_decim_taps, kapre_cqt_plan** out);
void kapre_cqt_plan_destroy(kapre_cqt_plan* plan);
/* 1 + length / hop_length (< 0 on a negative length). */
int kapre_cqt_num_frames(const kapre_cqt_plan* plan, int length);
/* Device scratch of kapre_cqt (backward = 0: pyramid levels 1 .. n_oct - 1) or of kapre_cqt_backward (backward = 1:
 * the adjoint's levels and their decimation adjoints).  < 0 on a bad size or an overflow. */
int64_t kapre_cqt_workspace_bytes(const kapre_cqt_plan* plan, int batch, int channels, int length, int backward);
/* out = C (complex64, magnitude = 0) or |C| (float32, magnitude = 1), (batch, channels, frames, n_bins) by element
 * strides.  The pyramid is left in workspace_dev (kapre_cqt_workspace_bytes(..., 0) bytes).  n_oct - 1 resampling
 * launches and one transform launch. */
int kapre_cqt(const kapre_cqt_plan* plan, const float* x_dev, const kapre_wave_desc* x_desc, int magnitude,
              void* out_dev, const kapre_spec_desc* out_desc, void* workspace_dev, void* stream);
/* gx = the gradient of kapre_cqt to x at output gradient g: Re(A^H g) for complex g (torch's dL/dRe + i dL/dIm), or
 * in magnitude mode the same at g C / |C| (0 where |C| = 0), C recomputed from x and the pyramid the forward left in
 * fwd_workspace_dev (unused in complex mode).  workspace_dev: kapre_cqt_workspace_bytes(..., 1) bytes.  Lowest
 * octave first, 2 n_oct - 1 launches: n_oct adjoint gathers and n_oct - 1 resampling adjoints. */
int kapre_cqt_backward(const kapre_cqt_plan* plan, const float* x_dev, const kapre_wave_desc* x_desc,
                       const void* fwd_workspace_dev, const void* g_dev, const kapre_spec_desc* g_desc, int magnitude,
                       float* gx_dev, const kapre_wave_desc* gx_desc, void* workspace_dev, void* stream);

/* ---- pitch tracking: YIN and probabilistic YIN (modelled on librosa's yin / pyin) -----------------------------------
 * Frame m of each (item, channel) row holds the samples [m hop - pad, m hop - pad + frame_length), pad =
 * frame_length / 2 with `center` (zeros outside the signal), m < kapre_pitch_num_frames.  With x the frame and W the
 * window, d(tau) = sum_{j=1..W} (x[j] - x[j + tau])^2 and the CMNDF c(tau) = d(tau) / (mean_{k<=tau} d(k) + 2^-126)
 * for min_period <= tau <= max_period.  Every output's bits depend on (item, channel, frame) alone. */
#define KAPRE_PITCH_MAX_FRAME 8192
#define KAPRE_PITCH_MAX_THRESHOLDS 1024
#define KAPRE_PITCH_MAX_BINS 8192
#define KAPRE_PITCH_MAX_BAND 8192
typedef struct {
    float sample_rate;
    int frame_length, win_length, hop_length, center;
    int min_period, max_period;           /* 1 <= min_period, min_period + 2 <= max_period < frame_length - win_length */
    double trough_threshold;              /* YIN */
    /* pYIN (kapre_pyin only) */
    int n_thresholds, n_pitch, band_width;
    float log_stay, log_switch;           /* log(1 - switch_prob), log(switch_prob) */
    float log_init_voiced, log_init_unvoiced;
    float fill_na;
} kapre_pitch_config;
/* float64 host tables of pYIN (rounded to float32 on upload, except the edges).  cmax = (n + 1) / 2, n =
 * max_period - min_period + 1, is the most troughs a frame can hold. */
typedef struct {
    const double* beta_probs;             /* n_thresholds: Bcdf(i / n) - Bcdf((i - 1) / n), i = 1 .. n */
    const double* boltzmann_pow;          /* cmax + 1: e^{-lambda r} */
    const double* boltzmann_norm;         /* cmax + 1: (1 - e^{-lambda}) / (1 - e^{-lambda N}) (entry 0 unused) */
    const double* no_trough_bonus;        /* n_thresholds + 1: no_trough_prob (beta_1 + ... + beta_k) */
    const double* period_edges;           /* n_pitch - 1: the period at the upper edge of bin m (descending) */
    const double* freqs;                  /* n_pitch: the bins' frequencies */
    const double* log_triangle;           /* band_width: log of the triangle taps */
    const double* log_row_norm;           /* n_pitch: -log(sum of row i's taps inside [0, n_pitch)) */
} kapre_pitch_tables;
/* Element strides (batch, channel, frame) of a per-frame output. */
typedef struct {
    int64_t stride_b, stride_c, stride_t;
} kapre_frames_desc;
typedef struct kapre_pitch_plan kapre_pitch_plan;
/* tables = NULL: a YIN-only plan.  KAPRE_E_UNSUPPORTED past the KAPRE_PITCH_MAX_* limits. */
int kapre_pitch_plan_create(const kapre_pitch_config* cfg, const kapre_pitch_tables* tables, kapre_pitch_plan** out);
void kapre_pitch_plan_destroy(kapre_pitch_plan* plan);
/* max(0, 1 + (length + 2 pad - frame_length) / hop_length) (< 0 on a negative length). */
int kapre_pitch_num_frames(const kapre_pitch_plan* plan, int length);
/* Device scratch of kapre_pyin: the candidate lists and the Viterbi backpointers (2 n_pitch uint16 per frame). */
int64_t kapre_pitch_workspace_bytes(const kapre_pitch_plan* plan, int batch, int channels, int length);
/* f0 = sr / (min_period + k + shift) of YIN's trough k (first below trough_threshold, else the first global minimum),
 * NaN on frames holding a non-finite sample.  cmndf_dev (nullable): c(min_period + k) at (b, c, frame, k).  One launch. */
int kapre_yin(const kapre_pitch_plan* plan, const float* x_dev, const kapre_wave_desc* x_desc, float* f0_dev,
              const kapre_frames_desc* f0_desc, float* cmndf_dev, const kapre_spec_desc* cmndf_desc, void* stream);
/* pYIN's Viterbi-decoded f0 (fill_na on unvoiced frames), voiced flag (uint8) and voiced probability, all three with
 * the strides of out_desc.  A row with a non-finite sample in any frame gives fill_na, 0 and NaN throughout.  Two
 * launches. */
int kapre_pyin(const kapre_pitch_plan* plan, const float* x_dev, const kapre_wave_desc* x_desc, float* f0_dev,
               uint8_t* voiced_flag_dev, float* voiced_prob_dev, const kapre_frames_desc* out_desc, float* cmndf_dev,
               const kapre_spec_desc* cmndf_desc, void* workspace_dev, void* stream);

/* ---- chroma features (modelled on librosa's chroma_stft, chroma_cqt, chroma_cens and estimate_tuning) -------------
 * A chroma plan holds n_tables filterbank tables W (n_chroma x n_bins each), optionally the CENS smoothing taps and
 * optionally the tuning estimate's geometry.  For every frame of a (item, channel) row of a spectrogram s (any element
 * strides (b, c, t, k)), y_j = sum_k W[j][k] s_k in ascending k (float32), entries below the threshold are set to 0
 * and the frame is normalised; a frame whose length is below FLT_MIN is left as it is.  An output's bits depend on
 * (item, channel, frame, chroma) and the item's table alone. */
#define KAPRE_CHROMA_MAX_CHROMA 64
#define KAPRE_CHROMA_MAX_BINS 4097
#define KAPRE_CHROMA_MAX_TUNING_BINS 1000
#define KAPRE_CHROMA_MAX_SMOOTH 514
enum { KAPRE_CHROMA_IN_LINEAR = 0, KAPRE_CHROMA_IN_SQUARE = 1, KAPRE_CHROMA_IN_COMPLEX = 2 };
enum { KAPRE_CHROMA_NORM_NONE = 0, KAPRE_CHROMA_NORM_INF = 1, KAPRE_CHROMA_NORM_L1 = 2, KAPRE_CHROMA_NORM_L2 = 3 };
typedef struct {
    int n_chroma, n_bins, n_tables;       /* n_tables = 0: a plan for the tuning estimate alone */
    const double* tables;                 /* n_tables x n_chroma x n_bins, rounded to float32 on upload */
    int n_smooth;                         /* CENS smoothing taps (0: no CENS) */
    const double* smooth;
    int n_tuning_bins;                    /* residual histogram bins (0: no tuning estimate) */
    const double* tuning_edges;           /* n_tuning_bins + 1, ascending */
    int peak_lo, peak_hi;                 /* piptrack's bins [peak_lo, peak_hi), 1 <= peak_lo, peak_hi < n_bins */
    float sample_rate, n_fft;             /* pitch = (k + shift) sample_rate / n_fft */
    double bins_per_octave;               /* of the residual */
} kapre_chroma_plan_desc;
typedef struct {
    int in_mode;                          /* KAPRE_CHROMA_IN_*: s = x, x^2 (float x) or |x| (complex64 x) */
    int norm;                             /* KAPRE_CHROMA_NORM_* */
    int has_threshold;
    float threshold;
} kapre_chroma_config;
typedef struct kapre_chroma_plan kapre_chroma_plan;
int kapre_chroma_plan_create(const kapre_chroma_plan_desc* desc, kapre_chroma_plan** out);
void kapre_chroma_plan_destroy(kapre_chroma_plan* plan);
/* The chroma (batch, channels, frames, n_chroma) at out_desc's strides.  table_dev (nullable, device int per item):
 * the table of each item, else table 0.  One launch. */
int kapre_chroma(const kapre_chroma_plan* plan, const kapre_chroma_config* cfg, const void* x_dev,
                 const kapre_spec_desc* x_desc, int batch, int channels, int frames, const int* table_dev, float* out_dev,
                 const kapre_spec_desc* out_desc, void* stream);
/* Gradient of kapre_chroma to x (float, or complex64 for KAPRE_CHROMA_IN_COMPLEX) at gx_desc's strides, given the
 * output gradient g.  Through the normalisation (norm inf: to the first index of the maximum), the threshold, W and the
 * input mode (2 x g, or g x / |x| with 0 at x = 0).  One launch. */
int kapre_chroma_backward(const kapre_chroma_plan* plan, const kapre_chroma_config* cfg, const void* x_dev,
                          const kapre_spec_desc* x_desc, int batch, int channels, int frames, const int* table_dev,
                          const float* g_dev, const kapre_spec_desc* g_desc, void* gx_dev, const kapre_spec_desc* gx_desc,
                          void* stream);
int64_t kapre_chroma_cens_workspace_bytes(const kapre_chroma_plan* plan, int batch, int channels, int frames);
/* CENS: threshold 0, L1 normalisation and quantisation (one launch), then the smoothing along time with zeros outside
 * the row and the L2 normalisation (a second launch). */
int kapre_chroma_cens(const kapre_chroma_plan* plan, int in_mode, const void* x_dev, const kapre_spec_desc* x_desc,
                      int batch, int channels, int frames, float* out_dev, const kapre_spec_desc* out_desc,
                      void* workspace_dev, void* stream);
int64_t kapre_chroma_tuning_workspace_bytes(const kapre_chroma_plan* plan, int batch, int channels, int frames);
/* librosa's estimate_tuning per item over all its channels from a power (KAPRE_CHROMA_IN_SQUARE of |X|) or given
 * (KAPRE_CHROMA_IN_LINEAR) spectrogram: tuning_dev (double per item) and table_dev (int per item: the index of the
 * tuning's edge, n_tuning_bins for an item without peaks).  Seven launches and two memsets whatever the data; nothing
 * is read back to the host. */
int kapre_chroma_tuning(const kapre_chroma_plan* plan, int in_mode, const float* x_dev, const kapre_spec_desc* x_desc,
                        int batch, int channels, int frames, double* tuning_dev, int* table_dev, void* workspace_dev,
                        void* stream);

/* ---- harmonic/percussive separation (modelled on librosa.decompose.hpss) ------------------------------------------
 * S (batch x channels x frames x bins, any element strides) is float32 magnitudes, used as given, or complex64, whose
 * magnitude |X| is formed as kapre_magnitude forms it; S must be non-negative (not checked).  Per (item, channel) row:
 *   H = median over kernel_h frames, P = median over kernel_p bins, each the element of rank k/2 of its window with
 *   indices reflected with period 2n, edge included (scipy.ndimage.median_filter(mode='reflect')); a window holding NaN
 *   gives NaN;
 *   M_H = softmask(H, margin_h P), M_P = softmask(P, margin_p H) (librosa.util.softmask: a > b as 1/0 for power inf;
 *   else 0.5 when both margins are 1 and max(a, b) < FLT_MIN, 0 otherwise, else (a/Z)^p / ((a/Z)^p + (b/Z)^p) with
 *   Z = max(a, b));
 *   outputs S M_H and S M_P (float S), M_H X and M_P X (complex64 S), or the masks themselves (float32).
 * Every output's bits depend only on its row's data and its (frame, bin). */
#define KAPRE_HPSS_MAX_KERNEL 64
typedef struct {
    int kernel_h, kernel_p;       /* 1 .. KAPRE_HPSS_MAX_KERNEL */
    float power;                  /* > 0, may be +inf */
    float margin_h, margin_p;     /* finite, >= 1 */
    int mask;                     /* 1: write the masks instead of the components */
} kapre_hpss_config;
/* Either output may be NULL (not written).  Outputs must not overlap S.  One launch. */
int kapre_hpss(const kapre_hpss_config* cfg, const void* S_dev, int is_complex, const kapre_spec_desc* S_desc, int batch,
               int channels, int frames, int bins, void* h_dev, const kapre_spec_desc* h_desc, void* p_dev,
               const kapre_spec_desc* p_desc, void* stream);
/* Device scratch of kapre_hpss_backward: 16 bytes per element of S (a gradient and the index of the element it goes to,
 * for each median). */
int64_t kapre_hpss_workspace_bytes(int batch, int channels, int frames, int bins);
/* Gradient of kapre_hpss to S (float32, or complex64 in torch's convention) at gS_desc's strides, given the gradients
 * of its outputs (same dtype as the outputs: float32 masks, or the components in S's dtype); either may be NULL (zero).
 * The direct term M_H g_H + M_P g_P plus the mask term through each median, which goes to the one element the median
 * selected (rank k/2 under (value, position in the reflected window)); complex S then through |X| (g X / |X|, 0 at
 * X = 0).  Infinite or undefined mask derivatives (max(a, b) < FLT_MIN, power inf, a zero median with power < 1)
 * contribute 0.  Two launches; gS must not overlap the other buffers. */
int kapre_hpss_backward(const kapre_hpss_config* cfg, const void* S_dev, int is_complex, const kapre_spec_desc* S_desc,
                        int batch, int channels, int frames, int bins, const void* gh_dev, const kapre_spec_desc* gh_desc,
                        const void* gp_dev, const kapre_spec_desc* gp_desc, void* gS_dev,
                        const kapre_spec_desc* gS_desc, void* workspace_dev, void* stream);

/* ---- onset strength, tempogram, tempo, onset detection, beat tracking (modelled on librosa 0.10) ------------------
 * A row is one (item, channel) pair; every output's bits depend only on its row's data.  Per-frame signals (envelopes,
 * masks) use kapre_frames_desc; masks are uint8 0 / 1.
 *
 * Onset strength of S (batch x channels x frames x bins, float32, any strides), per row with m = max_size and P =
 * lag + pad_frames:  R[t][b] = max S[t][b - m/2 .. b - m/2 + m - 1] (bins outside [0, K) skipped),
 * D[t][b] = max(0, S[t][b] - R[t - lag][b]) (NaN kept), A[t] = mean over b (float64 sum in ascending b, / K, rounded
 * once) or median (numpy's; NaN in the frame gives NaN), out[t] = 0 for t < P, A[t - P + lag] otherwise. */
#define KAPRE_ONSET_MAX_BINS 4097
#define KAPRE_TEMPOGRAM_MAX_WIN 4096
#define KAPRE_BEAT_MAX_PERIOD 4096
enum { KAPRE_ONSET_MEAN = 0, KAPRE_ONSET_MEDIAN = 1 };
typedef struct {
    int lag;                      /* >= 1, < frames */
    int max_size;                 /* 1 .. bins */
    int aggregate;                /* KAPRE_ONSET_MEAN or KAPRE_ONSET_MEDIAN */
    int pad_frames;               /* n_fft / (2 hop_length) for a centred S, else 0 */
} kapre_onset_config;
/* bins <= KAPRE_ONSET_MAX_BINS.  One launch. */
int kapre_onset_strength(const kapre_onset_config* cfg, const float* S_dev, const kapre_spec_desc* S_desc, int batch,
                         int channels, int frames, int bins, float* out_dev, const kapre_frames_desc* out_desc,
                         void* stream);
/* Device scratch of kapre_onset_strength_backward: 8 bytes per element of S. */
int64_t kapre_onset_strength_workspace_bytes(int batch, int channels, int frames, int bins);
/* Gradient of kapre_onset_strength to S given g, the envelope's gradient: relu'(0) = 0, each window maximum's
 * gradient to the lowest of its tied bins, the median's to the element(s) it selected under (value, bin) (0.5 each
 * for even bins).  Two launches, no floating-point atomics; gS must not overlap the other buffers. */
int kapre_onset_strength_backward(const kapre_onset_config* cfg, const float* S_dev, const kapre_spec_desc* S_desc,
                                  int batch, int channels, int frames, int bins, const float* g_dev,
                                  const kapre_frames_desc* g_desc, float* gS_dev, const kapre_spec_desc* gS_desc,
                                  void* workspace_dev, void* stream);
/* Autocorrelation tempogram of envelopes e (batch x channels x frames): frame t is y = w * padded[t .. t + W) with w
 * the periodic Hann window of W = win_length (2 .. KAPRE_TEMPOGRAM_MAX_WIN) and, with center, e padded by W/2 linear
 * ramps to zero on each side (np.pad(mode='linear_ramp')), frames 0 .. frames - 1; without center frames
 * 0 .. frames - W.  out[t][l] = sum_{j <= W-1-l} y[j] y[j + l] (float32 fma chain in ascending j), divided by
 * max_l |out[t][l]| when norm_inf and that maximum is >= FLT_MIN.  out_desc: strides (b, c, t, lag).  One launch. */
int kapre_tempogram(const float* e_dev, const kapre_frames_desc* e_desc, int batch, int channels, int frames,
                    int win_length, int center, int norm_inf, float* out_dev, const kapre_spec_desc* out_desc,
                    void* stream);
/* Tempo from a tempogram tg (batch x channels x frames x W, strides (b, c, t, lag)).  per_frame = 0: g is the
 * float64 mean of tg over the frames (sums of 64-frame chunks added in ascending order, / frames), out holds
 * batch x channels floats (contiguous), two launches over the workspace of kapre_tempo_workspace_bytes.
 * per_frame = 1: g is tg per frame, out at out_desc's strides, one launch, no workspace.  The tempo is
 * bpm_scale / argmax_l (log1p(1e6 g[l]) + logprior[l]) (first maximum, float64; a NaN score is skipped), with
 * logprior a device array of W doubles.  A non-finite g, or no lag with a score, gives NaN. */
int64_t kapre_tempo_workspace_bytes(int batch, int channels, int frames, int win_length);
int kapre_tempo(const float* tg_dev, const kapre_spec_desc* tg_desc, int batch, int channels, int frames, int win_length,
                const double* logprior_dev, double bpm_scale, int per_frame, float* out_dev,
                const kapre_frames_desc* out_desc, void* workspace_dev, void* stream);
#define KAPRE_PEAK_MAX_WINDOW (1 << 30)
typedef struct {
    int pre_max, post_max, pre_avg, post_avg, wait;   /* 0 .. KAPRE_PEAK_MAX_WINDOW; post_max, post_avg >= 1 */
    int normalize;
    double delta;
} kapre_onset_detect_config;
/* librosa's peak picking per row of e: x = e - min e, x / (max x + FLT_MIN) with normalize (float32); n is a
 * candidate iff x[n] == max x[n - pre_max .. n + post_max), x[n] != 0 and x[n] >= mean x[n - pre_avg .. n + post_avg)
 * + delta (float64; windows clipped to the row); candidates closer than wait + 1 to the last accepted one are dropped.
 * A row whose x has no nonzero or a non-finite value has no onsets.  One launch. */
int kapre_onset_detect(const float* e_dev, const kapre_frames_desc* e_desc, int batch, int channels, int frames,
                       const kapre_onset_detect_config* cfg, uint8_t* mask_dev, const kapre_frames_desc* mask_desc,
                       void* stream);
typedef struct {
    double fps;                   /* sample_rate / hop_length, > 0 */
    double tightness;             /* > 0 */
    int trim;
} kapre_beat_config;
/* Device scratch of kapre_beat_track: the local score, cumulative score, backlinks and beats of every row
 * (24 bytes per frame). */
int64_t kapre_beat_track_workspace_bytes(int batch, int channels, int frames);
/* librosa's dynamic-programming beat tracker per row of e.  bpm_dev: batch x channels floats (contiguous), or NULL to
 * use bpm for every row; period p = rint(60 fps / bpm) (half to even).  tempo_dev (batch x channels, contiguous)
 * receives the bpm used, 0 for an all-zero row and NaN for a non-finite one; mask_dev the beats.  A row with no
 * beats, an all-zero or non-finite row, or a p outside [1, KAPRE_BEAT_MAX_PERIOD] has an empty mask.  One launch. */
int kapre_beat_track(const float* e_dev, const kapre_frames_desc* e_desc, int batch, int channels, int frames,
                     const kapre_beat_config* cfg, const float* bpm_dev, float bpm, float* tempo_dev, uint8_t* mask_dev,
                     const kapre_frames_desc* mask_desc, void* workspace_dev, void* stream);

/* ---- per-channel energy normalisation (PCEN) ---------------------------------------------------
 * Each column (b, c, f) of a non-negative spectrogram E (batch x channels x frames x bands, any strides) is
 * processed along time:
 *   M[-1] = E[0],  M[t] = (1 - s) M[t-1] + s E[t],  y[t] = d^r expm1(r log1p(E[t] (eps + M[t])^-a / d))
 * with a = gain, d = bias, r = power, s = smooth_coef.  Each parameter is a device pointer with an element
 * stride of 0 (one value for every band) or 1 (one value per band); values are used as given (no clamping). */
typedef struct {
    const float *gain, *bias, *power, *smooth;
    int gain_stride, bias_stride, power_stride, smooth_stride;
    float eps;
} kapre_pcen_params;
/* The time chunking a call on the current device uses for this shape (`*chunks`, >= 1) and the device scratch it
 * needs (`*workspace_bytes`: chunks x batch x channels x bands floats when chunks > 1, else 0).  The same shape
 * gives the same chunking on the same device, so the numbers hold for both kapre_pcen and kapre_pcen_backward. */
int kapre_pcen_workspace(int batch, int channels, int frames, int bands, int* chunks, int64_t* workspace_bytes);
/* y = PCEN(E).  `M_dev` (nullable): also write the smoother state M, which kapre_pcen_backward reads.  y and M must
 * not overlap E.  `workspace_dev`: kapre_pcen_workspace's bytes (NULL when 0). */
int kapre_pcen(const float* E_dev, const kapre_spec_desc* E_desc, int batch, int channels, int frames, int bands,
               const kapre_pcen_params* params, float* y_dev, const kapre_spec_desc* y_desc, float* M_dev,
               const kapre_spec_desc* M_desc, void* workspace_dev, void* stream);
/* Gradient of kapre_pcen given E, the M it wrote and the output gradient gy: writes gE (every element once) and
 * the parameter partial sums `param_partials_dev`, a contiguous (4, chunks, batch, channels, bands) float array
 * (gain, bias, power, smooth_coef; chunks from kapre_pcen_workspace).  Summed over chunks, batch and channels they
 * give the per-band gradients, summed over bands as well the gradient of a shared parameter. */
int kapre_pcen_backward(const float* E_dev, const kapre_spec_desc* E_desc, const float* M_dev,
                        const kapre_spec_desc* M_desc, const float* gy_dev, const kapre_spec_desc* gy_desc, int batch,
                        int channels, int frames, int bands, const kapre_pcen_params* params, float* gE_dev,
                        const kapre_spec_desc* gE_desc, float* param_partials_dev, void* workspace_dev, void* stream);

/* ---- Griffin-Lim phase reconstruction ------------------------------------------------------------
 * Fast Griffin-Lim (the momentum form librosa and torchaudio use) over this library's transform pair: given a
 * magnitude spectrogram S (batch x channels x frames x (n_fft/2 + 1) bins, any strides),
 *   X = S A_0;  repeat n_iter times: y = ISTFT(X); Y = STFT(y) (no padding: `frames` frames again);
 *               A = Y - beta Yprev (A = Y the first time); X = S A / (|A| + 1e-16); Yprev = Y
 *   then y = ISTFT(X): (frames - 1) * hop + win_length samples, untrimmed, as kapre_istft_inverse writes them,
 * with beta = momentum / (1 + momentum).  A_0 = 1 (KAPRE_GL_INIT_ONES) or exp(2 pi i u) (KAPRE_GL_INIT_RANDOM) with
 *   u = (mix(seed ^ mix(i)) >> 40) * 2^-24,  i = ((b * channels + c) * frames + t) * (n_fft/2 + 1) + f,
 *   mix(z): z += 0x9E3779B97F4A7C15; z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9; z = (z ^ (z >> 27)) * 0x94D049BB133111EB;
 *           return z ^ (z >> 31)          (splitmix64, uint64 arithmetic)
 * so the phases depend on the seed and the canonical index only, not on S's strides.
 * `stft` and `istft` must agree on n_fft, win_length and hop and live on the same device; pair the STFT window with
 * its dual in the inverse plan, as InverseSTFT does (tf.signal.inverse_stft_window_fn), or the loop does not
 * reconstruct.  One call enqueues the whole loop: 2 + 3 n_iter launches where the STFT and the inverse are one
 * launch each (n_fft 256 / 512 / 1024 / 2048).  Not differentiable. */
enum { KAPRE_GL_INIT_ONES = 0, KAPRE_GL_INIT_RANDOM = 1 };
typedef struct {
    int n_iter;        /* >= 0 */
    float momentum;    /* in [0, 1) */
    int init;          /* KAPRE_GL_INIT_* */
    uint64_t seed;     /* KAPRE_GL_INIT_RANDOM only */
} kapre_griffin_lim_cfg;
/* Device scratch of kapre_griffin_lim: two (batch, channels, frames, n_fft/2 + 1) complex64 spectra and one
 * (batch, channels, (frames - 1) * hop + win_length) float32 waveform.  0 for an empty batch; < 0 on error. */
int64_t kapre_griffin_lim_workspace_bytes(const kapre_stft_plan* plan, int batch, int channels, int frames);
/* y = GriffinLim(S).  `y_desc`: batch, channels and (frames - 1) * hop + win_length samples, any strides.
 * `workspace_dev`: kapre_griffin_lim_workspace_bytes bytes (contents ignored); S and y must not overlap it. */
int kapre_griffin_lim(const kapre_stft_plan* stft, const kapre_istft_plan* istft, const float* S_dev,
                      const kapre_spec_desc* S_desc, int batch, int channels, int frames,
                      const kapre_griffin_lim_cfg* cfg, float* y_dev, const kapre_wave_desc* y_desc,
                      void* workspace_dev, void* stream);

/* ---- phase-vocoder time stretch ----------------------------------------------------------------
 * torchaudio.functional.phase_vocoder on a complex64 spectrogram X (batch x channels x frames x bins, any strides):
 * frames' = ceil(frames / rate) output frames; for output u, ts = (double)u * rate, k = floor(ts), alpha = ts - k and
 * (X[frames] = X[frames + 1] = 0)
 *   m[u] = alpha |X[k + 1]| + (1 - alpha) |X[k]|
 *   phi[u] = q(X[0]) + sum_{v < u} (q(X[k_v + 1]) - q(X[k_v]))    in uint32 arithmetic (mod 2^32)
 *   Y[u] = m[u] (cospi(s), sinpi(s)),  s = (int32)phi[u] * 2^-31
 * with q(z) = rint(atan2(z) * 2^31 / pi) mod 2^32, each angle a count of 2^-32 turns.  Modulo 2 pi, torchaudio's
 * wrapped phase advance cancels, so the result does not depend on hop length or phase advance and none is taken.  The
 * integer phase sum does not drift, and the output does not depend on the time chunking below.  rate must be finite
 * and positive and frames' must fit in int32 (KAPRE_E_INVALID otherwise, before anything is launched). */
/* The time chunking a call on the current device uses for this shape (`*chunks`, >= 1) and the device scratch it needs
 * (`*workspace_bytes`: 4 x chunks x batch x channels x bins when chunks > 1, else 0); the same for the backward. */
int kapre_time_stretch_workspace(int batch, int channels, int frames, int bins, double rate, int* chunks,
                                 int64_t* workspace_bytes);
/* Y = stretch(X): frames' output frames with Y_desc's strides.  Y must not overlap X.  `workspace_dev`:
 * kapre_time_stretch_workspace's bytes (NULL when 0). */
int kapre_time_stretch(const void* X_dev, const kapre_spec_desc* X_desc, int batch, int channels, int frames, int bins,
                       double rate, void* Y_dev, const kapre_spec_desc* Y_desc, void* workspace_dev, void* stream);
/* Gradient of kapre_time_stretch given X, the Y it wrote and the output gradient G (torch's convention dL/dRe +
 * i dL/dIm): with gm = Re(conj(Y) G) / |Y|, gphi = Im(conj(Y) G) (0 where Y = 0) and lam_u = sum_{v > u} gphi[v],
 * input frame j collects g|X| (the (1 - alpha) and alpha shares of gm of the outputs that read it) and gth (+lam_u
 * where it is frame k_u + 1, -lam_u where it is frame k_u, and the sum of all gphi at frame 0), and
 * gX = X / |X| (g|X| + i gth / |X|), 0 where |X| = 0.  Every gX element is written once (frames no output reads get
 * 0); gX must not overlap X, Y or G. */
int kapre_time_stretch_backward(const void* X_dev, const kapre_spec_desc* X_desc, const void* Y_dev,
                                const kapre_spec_desc* Y_desc, const void* G_dev, const kapre_spec_desc* G_desc,
                                int batch, int channels, int frames, int bins, double rate, void* gX_dev,
                                const kapre_spec_desc* gX_desc, void* workspace_dev, void* stream);

/* ---- filterbank inversion (mel / log spectrogram -> linear magnitudes) ----------------------------------------
 * With A the (n_bands x n_freq) transpose of a row-major (n_freq x n_bands) filterbank `fb_host` (as given to
 * kapre_filterbank_create), each frame's n_bands values m are mapped to the n_freq values s that a fixed number of
 * projected accelerated gradient (FISTA) steps take towards  min ||A s - m||^2  subject to s >= 0:
 *   s_0 = max(A^T (m / d), 0) with d = A A^T 1 (m / d = 0 where d = 0);  y_0 = s_0;  t_0 = 1;
 *   s_{k+1} = max(y_k - step A^T (A y_k - m), 0);  t_{k+1} = (1 + sqrt(1 + 4 t_k^2)) / 2;
 *   y_{k+1} = s_{k+1} + ((t_k - 1) / t_{k+1}) (s_{k+1} - s_k);   output s_{n_iter}.
 * step = 1 / ||A||_2^2 (float64 power iteration when the plan is made).  Bins no band touches come out 0.  The
 * minimiser is not unique (n_freq > n_bands); the output is this iteration's result.  With from_decibel the input is
 * dB and is converted on load: m = 10^(x / 10) max(amin, ref_value), the inverse of kapre_magnitude_to_decibel where
 * its dynamic-range clamp did not bind.  One launch; each input element is read once and each output element written
 * once, and a frame's output does not depend on its place in the batch, the strides or the data format.  Not
 * differentiable. */
typedef struct kapre_fb_inverse_plan kapre_fb_inverse_plan;
int kapre_fb_inverse_plan_create(const float* fb_host, int n_freq, int n_bands, kapre_fb_inverse_plan** out);
void kapre_fb_inverse_plan_destroy(kapre_fb_inverse_plan* plan);
typedef struct {
    int n_iter;          /* >= 0 */
    int from_decibel;    /* 0 or 1 */
    float ref_value;     /* from_decibel only: > 0 */
    float amin;          /* from_decibel only: > 0 */
} kapre_fb_inverse_cfg;
/* out = invert(x).  x: (batch, channels, frames) x n_bands, out: ... x n_freq, any strides; out must not overlap x.
 * KAPRE_E_UNSUPPORTED when one frame's state (2 n_freq + 2 n_bands floats, doubled for the padded tile) does not fit
 * the device's shared memory. */
int kapre_filterbank_invert(const kapre_fb_inverse_plan* plan, const kapre_fb_inverse_cfg* cfg, const float* x_dev,
                            int batch, int channels, int frames, const kapre_spec_desc* x_desc, float* out_dev,
                            const kapre_spec_desc* out_desc, void* stream);

/* ---- misc ---------------------------------------------------------------------------------- */
const char* kapre_last_error(void);
int kapre_version(void);
/* Number of kernels this library has launched in this process (for bench.py's gpu_launches). */
uint64_t kapre_launch_count(void);
/* Name of the last fused-forward launch configuration, e.g. "Q16 TF16 NW4 grid296 smem98304", or of the last
 * persistent launch, "<kernel> grid=G tiles=T".  A call that makes several persistent launches (the CQT, HPSS and
 * onset-strength gradients, pYIN, CENS, the tuning estimate, tempo) reports all of them in launch order, joined
 * with "; ". */
const char* kapre_last_launch_info(void);
/* Kernel timing for bench.py's roofline: enable = n > 0 brackets every n-th fused forward / inverse
 * kernel launch by CUDA events on its own stream (n = 1: every launch; a stride leaves the other
 * launches free to overlap their predecessor through programmatic dependent launch); 0 = off.  kapre_profile_read synchronises with
 * the recorded events, adds their durations to *total_ms / *launches and clears the list. */
int kapre_profile_enable(int enable);
int kapre_profile_read(double* total_ms, uint64_t* launches);

/* Experimental (measured prototype, not on the product path): stage 1 of the 32 x 32 factorisation of the
 * n_fft = 1024 / hop = 256 real FFT as a wgmma (Hopper tensor core) GEMM with register accumulators, fp32-grade
 * via the 3xTF32 split.  Layout of `out_dev` and the meaning of `store` are documented at the definition
 * (kapre_b200/csrc/kapre_b200.cu). */
/* Experimental: the next tensor-core (KAPRE_B200_TC=1) fused launch also writes its complex spectrum, (signals, frames, 513)
 * complex64, to dbg_dev -- used by the parity tests of the tensor-core FFT stages. */
int kapre_tc_set_debug(void* dbg_dev);
int kapre_tc_dft_stage1(const float* x_dev, int n_items, long long item_stride, int length, float* out_dev, int store,
                        int* grid_out, const float* fmat_override_dev, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* KAPRE_B200_H_ */
