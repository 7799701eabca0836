"""Mirrors of the waveform-side layers of ``kapre/signal.py`` that sit next to the hot path
``Frame`` (reference :22-119), ``Energy`` (:123-233) and ``LogmelToMFCC``
(:365-447).  Same constructor arguments, validation and ``get_config`` keys; ``call`` runs CUDA
kernels through the C ABI.  ``Resample`` (polyphase sample-rate conversion) has no counterpart in the
reference, which expects audio to be resampled before it reaches the model; neither has ``Speed`` (speed perturbation by any
real factor, band-limited interpolation), ``Convolve`` (convolution with long filters, partitioned FFT) or the IIR
filters ``lfilter``, ``filtfilt``, ``IIRFilter`` and ``Biquad`` (torchaudio's, on a chunked linear-recurrence scan), or
the second-order-section cascades ``sosfilt``, ``sosfiltfilt`` and ``SOSFilter`` (scipy's, on the same scan), or
``add_noise`` (torchaudio's, with deterministic float64 energies), or ``loudness`` and ``Loudness`` (torchaudio's
BS.1770 gated loudness, with per-item lengths), or the loudness meter ``loudness_stats`` and ``true_peak`` (EBU R128's
momentary and short-term loudness, loudness range and true peak), or the pitch trackers ``yin``, ``pyin``, ``YIN`` and ``PYIN``
(librosa's), or the chroma features ``chroma_stft``, ``chroma_cqt``, ``chroma_cens`` and ``estimate_tuning``
(librosa's), or the harmonic/percussive separation ``hpss``, ``harmonic`` and ``percussive`` (librosa's), or the
rhythm features ``onset_strength``, ``onset_detect``, ``tempogram``, ``tempo`` and ``beat_track`` (librosa's)."""
from __future__ import annotations

import math

import numpy as np
import torch

from . import backend, ops
from .backend import _CH_DEFAULT_STR, _CH_FIRST_STR, _CH_LAST_STR
from .time_frequency import Layer, _unwrap_format, register_keras_serializable

__all__ = ['Frame', 'Energy', 'LogmelToMFCC', 'Resample', 'Speed', 'Convolve', 'lfilter', 'filtfilt', 'IIRFilter',
           'Biquad', 'sosfilt', 'sosfiltfilt', 'SOSFilter', 'add_noise', 'loudness', 'Loudness', 'loudness_stats', 'true_peak',
           'LoudnessStats', 'kaldi_fbank', 'kaldi_mfcc', 'kaldi_spectrogram', 'yin', 'pyin',
           'YIN', 'PYIN', 'chroma_stft', 'chroma_cqt', 'chroma_cens', 'estimate_tuning', 'hpss', 'harmonic',
           'percussive', 'onset_strength', 'onset_detect', 'tempogram', 'tempo', 'beat_track', 'simulate_rir_ism']


def _resolve(fmt):
    return backend.image_data_format() if fmt == _CH_DEFAULT_STR else fmt


@register_keras_serializable(package='Kapre')
class Frame(Layer):
    """``tf.signal.frame`` along the time axis (reference kapre/signal.py:22-119):
    ``(batch, time, ch)`` -> ``(batch, frames, frame_length, ch)`` or
    ``(batch, ch, time)`` -> ``(batch, ch, frames, frame_length)``."""

    def __init__(self, frame_length, hop_length, pad_end=False, pad_value=0, data_format='default', **kwargs):
        super().__init__(**kwargs)
        backend.validate_data_format_str(data_format)
        if frame_length <= 0:
            raise ValueError('frame_length must be positive, got: %s' % (frame_length,))
        if hop_length <= 0:
            raise ValueError('hop_length must be positive, got: %s' % (hop_length,))
        if frame_length < hop_length:
            raise ValueError('frame_length (%s) must be >= hop_length (%s)' % (frame_length, hop_length))
        self.frame_length, self.hop_length = frame_length, hop_length
        self.pad_end, self.pad_value = pad_end, pad_value
        self.data_format_str = data_format
        self.data_format = _resolve(data_format)
        self.time_axis = 2 if self.data_format == _CH_FIRST_STR else 1

    def call(self, x):
        return ops.frame(x, self.frame_length, self.hop_length, self.pad_end, self.pad_value, self.data_format)

    _config_fields = (
        ('frame_length', 'frame_length'),
        ('hop_length', 'hop_length'),
        ('pad_end', 'pad_end'),
        ('pad_value', 'pad_value'),
        ('data_format', 'data_format_str'),
    )


@register_keras_serializable(package='Kapre')
class Energy(Layer):
    """Energy per frame, normalised to ``ref_duration`` (reference kapre/signal.py:123-233):
    ``ref_duration / (frame_length / sample_rate) * sum(frame ** 2)``.  Output ``(batch, frames, ch)`` or
    ``(batch, ch, frames)``.  (The reference's stray ``tf.print`` debugging, :191-207, is not reproduced.)"""

    def __init__(self, sample_rate=22050, ref_duration=0.1, frame_length=2205, hop_length=1102, pad_end=False,
                 pad_value=0, data_format='default', **kwargs):
        super().__init__(**kwargs)
        backend.validate_data_format_str(data_format)
        self.sample_rate, self.ref_duration = sample_rate, ref_duration
        self.frame_length, self.hop_length = frame_length, hop_length
        self.pad_end, self.pad_value = pad_end, pad_value
        self.data_format_str = data_format
        self.data_format = _resolve(data_format)
        self.time_axis = 2 if self.data_format == _CH_FIRST_STR else 1

    def call(self, x):
        nor_coeff = self.ref_duration / (self.frame_length / self.sample_rate)
        return ops.energy(x, self.frame_length, self.hop_length, self.pad_end, self.pad_value, nor_coeff,
                          self.data_format)

    _config_fields = (
        ('sample_rate', 'sample_rate'),
        ('ref_duration', 'ref_duration'),
        ('frame_length', 'frame_length'),
        ('hop_length', 'hop_length'),
        ('pad_end', 'pad_end'),
        ('pad_value', 'pad_value'),
        ('data_format', 'data_format_str'),
    )


def resample_filter(up: int, down: int) -> np.ndarray:
    """The anti-aliasing filter of ``scipy.signal.resample_poly`` with its default window:
    ``firwin(2 hl + 1, 1 / M, window=('kaiser', 5.0))`` with ``M = max(up, down)``, ``hl = 10 M``, i.e. the
    Kaiser-windowed ``sinc((k - hl) / M) / M`` normalised to unit sum.  Computed in float64, returned as float32."""
    M = max(int(up), int(down))
    hl = 10 * M
    n = 2 * hl + 1
    k = np.arange(n, dtype=np.float64)
    h = np.sinc((k - hl) / M) / M * np.kaiser(n, 5.0)
    h = 0.5 * (h + h[::-1])         # exactly symmetric: the backward pass relies on it
    return (h / h.sum()).astype(np.float32)


def _positive_int(name, v):
    if isinstance(v, bool) or not isinstance(v, (int, np.integer)) or v <= 0:
        raise ValueError('%s must be a positive integer, got: %r' % (name, v))
    return int(v)


@register_keras_serializable(package='Kapre')
class Resample(Layer):
    """Sample-rate conversion along the time axis: ``scipy.signal.resample_poly(x, up, down)`` with its default
    Kaiser (beta 5) filter and zeros outside the signal, ``up / down = target_sample_rate / orig_sample_rate``
    reduced.  ``(batch, time, ch)`` -> ``(batch, ceil(time * up / down), ch)`` or the same with ``(batch, ch, time)``.
    Equal rates return the input unchanged.  Supports every ratio with ``max(up, down) <= 1280``, which includes
    every pair of 8, 11.025, 16, 22.05, 24, 32, 44.1, 48, 88.2 and 96 kHz."""

    def __init__(self, orig_sample_rate, target_sample_rate, data_format='default', **kwargs):
        super().__init__(**kwargs)
        backend.validate_data_format_str(data_format)
        self.orig_sample_rate = _positive_int('orig_sample_rate', orig_sample_rate)
        self.target_sample_rate = _positive_int('target_sample_rate', target_sample_rate)
        g = math.gcd(self.orig_sample_rate, self.target_sample_rate)
        self.up, self.down = self.target_sample_rate // g, self.orig_sample_rate // g
        self.data_format_str = data_format
        self.data_format = _resolve(data_format)
        self.plan = None if self.up == self.down else ops.ResamplePlan(self.up, self.down,
                                                                      resample_filter(self.up, self.down))

    def call(self, x):
        if x.dim() != 3:
            raise ValueError('Resample expects a 3-D batch, got shape %s' % (tuple(x.shape),))
        if self.plan is None:
            return x
        return ops.resample(x, self.plan, self.data_format)

    _config_fields = (
        ('orig_sample_rate', 'orig_sample_rate'),
        ('target_sample_rate', 'target_sample_rate'),
        ('data_format', 'data_format_str'),
    )


@register_keras_serializable(package='Kapre')
class Speed(Layer):
    """Speed perturbation (``torchaudio.transforms.Speed``, Kaldi's 0.9 / 1.0 / 1.1 and the continuous variants):
    the waveform played ``factor`` times faster, hence ``factor`` times higher.  ``(batch, time, ch)`` ->
    ``(batch, ceil(time / factor), ch)`` or the same with ``(batch, ch, time)``.  ``factor`` is any number in
    [0.25, 4]; ``call(x, factor=...)`` overrides it for one call, and ``factor == 1`` returns the input itself.

    One launch of the band-limited interpolation kernel (``kapre_sinc_resample`` with ratio ``1 / factor``) whose
    filter table does not depend on the factor, so a new factor per step costs nothing: no plan, no table, no cache
    entry.  The gradient with respect to the input is available when the CUDA input requires grad."""

    def __init__(self, factor, data_format='default', **kwargs):
        super().__init__(**kwargs)
        backend.validate_data_format_str(data_format)
        self.factor = self._check(factor)
        self.data_format_str = data_format
        self.data_format = _resolve(data_format)

    @staticmethod
    def _check(factor):
        # the interpolation ratio is 1 / factor, and [0.25, 4] is its own reciprocal
        return ops._check_ratio(factor, 'factor')

    def output_length(self, length, factor=None):
        return math.ceil(int(length) / (self.factor if factor is None else factor))

    def call(self, x, factor=None):
        if x.dim() != 3:
            raise ValueError('Speed expects a 3-D batch, got shape %s' % (tuple(x.shape),))
        factor = self.factor if factor is None else self._check(factor)
        if factor == 1.0:
            return x
        length = x.shape[2] if self.data_format == _CH_FIRST_STR else x.shape[1]
        return ops.sinc_resample(x, 1.0 / factor, self.output_length(length, factor), 0.0, self.data_format)

    _config_fields = (
        ('factor', 'factor'),
        ('data_format', 'data_format_str'),
    )


@register_keras_serializable(package='Kapre')
class Convolve(Layer):
    """Convolution of waveforms with filters along the time axis (``torchaudio.transforms.Convolve``, i.e.
    ``torchaudio.functional.fftconvolve``): ``call(x, h)`` with ``x`` ``(batch, time, ch)`` / ``(batch, ch, time)`` and
    ``h`` either ``(K,)``, one filter for every item and channel, or 3-D in the same data format with batch 1 or
    ``batch`` and channels 1 or ``ch`` (1 broadcasts).  ``mode``: 'full' (``time + K - 1`` samples), 'same' (``time``)
    or 'valid' (``max(time, K) - min(time, K) + 1``), cropped from the full convolution as torchaudio does.

    A uniformly partitioned overlap-add (``kapre_convolve``): the filter's block spectra, then the STFT of the signal,
    one per-bin multiply-accumulate along the blocks and the inverse STFT, four launches in all.  The block size is a
    function of ``K`` alone, so an output does not depend on the batch it came in.  Differentiable with respect to
    ``x`` and ``h``."""

    def __init__(self, mode='full', data_format='default', **kwargs):
        super().__init__(**kwargs)
        backend.validate_data_format_str(data_format)
        data_format = _unwrap_format(data_format)
        if mode not in ops.CONVOLVE_MODES:
            raise ValueError('mode must be one of %s, got: %r' % (ops.CONVOLVE_MODES, mode))
        self.mode = mode
        self.data_format_str = data_format
        self.data_format = _resolve(data_format)

    def call(self, x, h):
        if not (isinstance(h, torch.Tensor) and h.is_cuda):
            h, _ = ops.to_device(h)
        return ops.convolve(x, h, self.mode, self.data_format)

    _config_fields = (
        ('mode', 'mode'),
        ('data_format', 'data_format_str'),
    )


def _coeff_tensor(c, name):
    """A coefficient argument as a tensor (CPU or CUDA, autograd kept)."""
    if isinstance(c, torch.Tensor):
        return c
    arr = np.asarray(c, np.float64)
    if arr.dtype.kind not in 'fiu':
        raise ValueError('%s must be numeric, got: %r' % (name, c))
    return torch.from_numpy(np.ascontiguousarray(arr))


def _normalised(x, a_coeffs, b_coeffs, data_format):
    """(b / a0, a / a0) as 3-D float32 tensors on x's device, after every check: shapes (``ops.iir_check``) and, for
    host coefficients, a0 != 0.  The division is a torch op, so autograd carries the gradient to raw a, b and a0."""
    if not (isinstance(x, torch.Tensor) and x.is_cuda):
        raise ops.N.KapreNativeError('lfilter needs a CUDA waveform')
    a = _coeff_tensor(a_coeffs, 'a_coeffs')
    b = _coeff_tensor(b_coeffs, 'b_coeffs')
    _, (Bc, Cc, n) = ops.iir_check(x, b, a, data_format)
    for t in (a, b):
        if t.is_cuda and t.device != x.device:
            raise ValueError('coefficients on %s, the waveform on %s' % (t.device, x.device))
    if not a.is_cuda:
        a0 = a.detach().reshape(-1, n)[:, 0]
        if bool((a0 == 0).any()):
            raise ValueError('a_coeffs[..., 0] must not be 0')
        if not bool(torch.isfinite(a.detach()).all() and torch.isfinite(b.detach()).all()):
            raise ValueError('coefficients must be finite')
    a = a.to(device=x.device, dtype=torch.float32)
    b = b.to(device=x.device, dtype=torch.float32)
    a0 = a[..., :1]
    return (b / a0).reshape(Bc, Cc, n), (a / a0).reshape(Bc, Cc, n)


def lfilter(waveform, a_coeffs, b_coeffs, clamp=True, data_format='default'):
    """``torchaudio.functional.lfilter`` along the time axis of ``waveform`` ``(batch, time, ch)`` /
    ``(batch, ch, time)`` (a CUDA tensor), with torchaudio's argument order:

        y[t] = (sum_{k=0..N} b[k] x[t-k] - sum_{k=1..N} a[k] y[t-k]) / a[0],   zero initial state,

    then clamped to [-1, 1] when ``clamp``.  ``a_coeffs`` and ``b_coeffs`` have one shape: ``(N + 1,)`` (one filter),
    ``(ch, N + 1)`` (one per channel, torchaudio's ``batching=True`` form) or ``(batch, ch, N + 1)`` with batch and
    channels 1 or the waveform's (one per item and channel).  Order N <= 8.

    The coefficients are divided by ``a[0]`` in float32 on the device, as torchaudio does, so the kernel sees
    normalised float32 coefficients; ``a[0] == 0`` raises for host coefficients but is not checked for CUDA tensors
    (that would synchronise), where it gives inf or NaN as in torchaudio.  Only stable filters are meaningful.  High
    orders in direct form are fragile in float32 (rounding the denominator of an 8th-order Butterworth at 0.05 of
    Nyquist makes it unstable), so prefer biquads or low orders for sharp filters.

    Four launches (``kapre_lfilter``).  Differentiable with respect to the waveform and both coefficient tensors."""
    fmt = _resolve(_unwrap_format(data_format))
    b, a = _normalised(waveform, a_coeffs, b_coeffs, fmt)
    return ops.lfilter(waveform, b, a, clamp=clamp, reverse=False, data_format=fmt)


def filtfilt(waveform, a_coeffs, b_coeffs, clamp=True, data_format='default'):
    """``torchaudio.functional.filtfilt``: ``lfilter`` without clamping, then ``lfilter`` in reverse time, then the
    clamp; zero-phase, with no edge padding (unlike scipy's ``filtfilt``).  Arguments as ``lfilter``.  The reverse pass
    runs the kernel backwards in time, so nothing is flipped or copied.  Eight launches."""
    fmt = _resolve(_unwrap_format(data_format))
    b, a = _normalised(waveform, a_coeffs, b_coeffs, fmt)
    y = ops.lfilter(waveform, b, a, clamp=False, reverse=False, data_format=fmt)
    return ops.lfilter(y, b, a, clamp=clamp, reverse=True, data_format=fmt)


def add_noise(waveform, noise, snr, lengths=None, data_format='default'):
    """``torchaudio.functional.add_noise`` on the GPU: per (item, channel) column,

        y = x + s n,   s = sqrt(Ex / En) 10^(-snr / 20),   Ex = sum_{t < len} x[t]^2,   En = sum_{t < len} n[t]^2,

    with noise added past ``len`` too, as torchaudio does.  ``waveform``: ``(batch, time, ch)`` / ``(batch, ch, time)``
    (a CUDA tensor); ``noise``: the same shape, or batch and / or channels of 1 (broadcast without a copy); ``snr``
    (dB) and ``lengths``: numbers or tensors broadcastable to ``(batch, ch)`` by torch's rules (``(batch, 1)`` for
    one value per item).  The SNR is measured per channel, as torchaudio does.

    The energies and ``s`` are float64 and summed in a fixed order (segments of 4096 samples, a fixed tree in each,
    the segments in order), so an item's output does not depend on the batch, its position, the strides or the data
    format.  One deliberate deviation: where the noise (or the signal) has zero energy over the valid samples, ``s`` is
    0 and the output is the input bit for bit; torchaudio returns NaN there for silent noise.  Two launches;
    differentiable with respect to ``waveform``, ``noise`` and ``snr`` (every term through ``s`` is 0 where an
    energy is 0)."""
    return ops.add_noise(waveform, noise, snr, lengths, _resolve(_unwrap_format(data_format)))


def loudness(waveform, sample_rate, lengths=None, data_format='default'):
    """``torchaudio.functional.loudness`` (ITU-R BS.1770-4 gated loudness, LKFS) per item of ``waveform``
    ``(batch, time, ch)`` / ``(batch, ch, time)`` (a CUDA tensor, ch <= 5), as a ``(batch,)`` float32 tensor.

    The K-weighting is torchaudio's: ``treble_biquad(sample_rate, 4.0, 1500.0, 1 / sqrt(2))`` then
    ``highpass_biquad(sample_rate, 38.0, 0.5)``, each clamped to [-1, 1] as torchaudio's biquads do.  The 400 ms
    blocks step by 100 ms (rounded as torchaudio rounds them), with the absolute gate at -70 LKFS and the relative
    gate 10 LU below, and the channel weights (1, 1, 1, 1.41, 1.41).  ``sample_rate`` must be above 3000 Hz.
    ``lengths``: a number or ``(batch,)`` integers; item b is measured as if cut to ``lengths[b]`` samples (clamped to
    [0, time] on the device, without a sync).

    The block energies and gates are float64 in a fixed order, so an item's result does not depend on the batch, its
    position, the strides or the data format.  Deliberate deviations from torchaudio: an item whose blocks are all
    gated out (silence, fewer samples than one block, or no samples) gives ``-inf`` and a gradient of 0, where
    torchaudio gives NaN or raises; a non-finite sample that reaches a block makes that item NaN and no other.

    Ten launches: two ``kapre_lfilter`` calls of four, then ``kapre_loudness``'s energy and gate passes.  The filter
    coefficients are uploaded once per device and rate, so a call can be captured in a CUDA graph.  Differentiable
    with respect to ``waveform``."""
    return ops.loudness(waveform, sample_rate, lengths, _resolve(_unwrap_format(data_format)))


LoudnessStats = ops.LoudnessStats
LoudnessStats.__doc__ = """What ``loudness_stats`` returns: ``integrated`` (batch,) LKFS, ``momentary`` (batch, J_M) and
``short_term`` (batch, J_S) LUFS series, ``loudness_range`` (batch,) LU and ``true_peak`` (batch, ch) dBTP."""


def loudness_stats(waveform, sample_rate, lengths=None, data_format='default'):
    """The EBU R128 loudness meter per item of ``waveform`` ``(batch, time, ch)`` / ``(batch, ch, time)`` (a CUDA
    tensor, ch <= 5), as a ``LoudnessStats`` of float32 tensors.  ``lengths`` as in ``loudness``.

    With ``G = round(0.4 sample_rate)``, ``S = round(G / 4)`` and ``G3 = round(3 sample_rate)``:

    - ``integrated`` ``(batch,)``: ``loudness`` of the same input, bit for bit (the same passes run).
    - ``momentary`` ``(batch, J_M)``, ``J_M = (time - G) // S + 1`` (0 when ``time < G``): entry j is
      ``-0.691 + 10 log10(sum_c g_c e_cj)``, e_cj the mean square of channel c of the K-weighted signal over
      ``[jS, jS + G)``, ungated.  Entries at or past the item's own count ``(len - G) // S + 1`` are ``-inf``, as is a
      silent window, so ``amax`` over a row is the item's maximum momentary loudness.
    - ``short_term`` ``(batch, J_S)``: the same with the 3 s window ``G3`` and the same step.
    - ``loudness_range`` ``(batch,)`` LU, EBU Tech 3342 on the short-term windows: the absolute gate at -70 LUFS, the
      relative gate 20 LU below the mean energy of the windows above it (strict comparisons), then the 95th minus the
      10th percentile of the remaining loudnesses by the nearest-rank rule ``v[((n - 1) p + 50) // 100]``; 0 when no
      window remains.  Float64 throughout, rounded once; selected on the device without a sort or a length limit.
    - ``true_peak`` ``(batch, ch)``: ``true_peak`` of the waveform.

    A non-finite sample makes that item's results NaN (true peak: that channel's) and no other item's.  The
    K-weighting runs once and feeds every output.  Sixteen launches: two ``kapre_lfilter`` calls of four,
    ``kapre_loudness_stats``'s six passes and ``kapre_true_peak``'s two.  No host sync and output sizes from ``time``
    alone, so a call can be captured in a CUDA graph.  No gradient: called under grad mode on an input that requires
    grad it raises; ``loudness`` and ``true_peak`` are differentiable."""
    return ops.loudness_stats(waveform, sample_rate, lengths, _resolve(_unwrap_format(data_format)))


def true_peak(waveform, lengths=None, data_format='default'):
    """True peak in dBTP per (item, channel) of ``waveform`` ``(batch, time, ch)`` / ``(batch, ch, time)`` (a CUDA
    tensor, any channel count, time <= 2^30), as a ``(batch, ch)`` float32 tensor:
    ``20 log10 max_t |z_c[t]|`` with ``z_c = scipy.signal.resample_poly(x_c[:len], 4, 1)``, 4x oversampling with
    ``resample_filter(4, 1)``, scipy's default Kaiser design.  ITU-R BS.1770-4 Annex 2 gives a 48-tap filter as an
    example that any compliant filter may replace; using scipy's makes ``resample_poly`` in float64 an exact oracle.
    No K-weighting and no sample rate.  ``lengths`` as in ``loudness``.

    z is formed in registers exactly as ``Resample`` forms it and never written; the maximum and its first argmax are
    exact and do not depend on the batch, the strides or the data format.  A silent channel gives ``-inf``; a NaN that
    reaches z gives NaN.  Two launches; differentiable with respect to ``waveform`` (one launch): the gradient is
    ``torch.amax``'s through the fixed linear map x -> z at the first argmax, and exactly 0 for ``-inf`` channels."""
    return ops.true_peak(waveform, lengths, _resolve(_unwrap_format(data_format)))


@register_keras_serializable(package='Kapre')
class Loudness(Layer):
    """``torchaudio.transforms.Loudness`` as a layer: ``(batch, time, ch)`` / ``(batch, ch, time)`` in (ch <= 5), the
    ``(batch,)`` loudness in LKFS out (``loudness``).  ``call(x, lengths=None)``."""

    def __init__(self, sample_rate, data_format='default', **kwargs):
        super().__init__(**kwargs)
        backend.validate_data_format_str(data_format)
        data_format = _unwrap_format(data_format)
        backend.k_weighting_coefficients(sample_rate)           # validates the rate
        self.sample_rate = sample_rate
        self.data_format_str = data_format
        self.data_format = _resolve(data_format)

    def call(self, x, lengths=None):
        return ops.loudness(x, self.sample_rate, lengths, self.data_format)

    _config_fields = (
        ('sample_rate', 'sample_rate'),
        ('data_format', 'data_format_str'),
    )


def _host_coeffs(b, a):
    """Validated float64 host copies of a layer's coefficients (same shape, order <= 8, a0 != 0, finite)."""
    b = np.asarray(b, np.float64)
    a = np.asarray(a, np.float64)
    if b.shape != a.shape or b.ndim not in (1, 2, 3) or b.shape[-1] < 1:
        raise ValueError('b and a must have one 1-D, 2-D or 3-D shape, got %s and %s' % (b.shape, a.shape))
    if b.shape[-1] - 1 > ops.IIR_MAX_ORDER:
        raise ValueError('IIR order %d is above the supported %d' % (b.shape[-1] - 1, ops.IIR_MAX_ORDER))
    if np.any(a[..., 0] == 0):
        raise ValueError('a[..., 0] must not be 0')
    if not (np.all(np.isfinite(a)) and np.all(np.isfinite(b))):
        raise ValueError('coefficients must be finite')
    return b, a


@register_keras_serializable(package='Kapre')
class IIRFilter(Layer):
    """An IIR filter (``lfilter``) with fixed or trainable coefficients: ``(batch, time, ch)`` / ``(batch, ch, time)``
    in, the same shape out.  ``b`` and ``a``: one shape, ``(N + 1,)``, ``(ch, N + 1)`` or ``(batch, ch, N + 1)`` as for
    ``lfilter``, N <= 8, ``a[..., 0] != 0``.  They become the layer's weights on the first call: float32 tensors on
    the input's device, raw (not normalised; the division by ``a[0]`` is part of every call), with
    ``requires_grad = trainable``, so a learnable front end trains all of b and a.  Nothing keeps a trained filter
    stable."""

    def __init__(self, b, a, clamp=True, trainable=False, data_format='default', **kwargs):
        super().__init__(trainable=trainable, **kwargs)
        backend.validate_data_format_str(data_format)
        data_format = _unwrap_format(data_format)
        self.b, self.a = _host_coeffs(b, a)
        self.clamp = bool(clamp)
        self.data_format_str = data_format
        self.data_format = _resolve(data_format)
        self.built = False
        self._weights = []

    def build(self, device):
        self._weights = [torch.tensor(v, dtype=torch.float32, device=device).requires_grad_(bool(self.trainable))
                         for v in (self.b, self.a)]
        self.built = True

    @property
    def weights(self):
        """[b, a] once built (the first call), else []."""
        return list(self._weights)

    def count_params(self):
        if not self.built:
            raise ValueError('You tried to call `count_params` on layer %s, but the layer isn\'t built.' % self.name)
        return sum(int(w.numel()) for w in self._weights)

    def call(self, x):
        if not self.built:
            self.build(x.device)
        elif self._weights[0].device != x.device:
            raise ValueError('IIRFilter %s was built on %s and cannot run on %s' % (self.name, self._weights[0].device,
                                                                                   x.device))
        b, a = self._weights
        return lfilter(x, a, b, clamp=self.clamp, data_format=self.data_format)

    def get_config(self):
        config = super().get_config()
        config.update({'b': self.b.tolist(), 'a': self.a.tolist(), 'clamp': self.clamp,
                       'data_format': self.data_format_str})
        return config


@register_keras_serializable(package='Kapre')
class Biquad(Layer):
    """A second-order filter of torchaudio's biquad family (``lowpass_biquad``, ``highpass_biquad``,
    ``bandpass_biquad``, ``bandreject_biquad``, ``allpass_biquad``, ``equalizer_biquad``): ``kind`` one of
    ``backend.BIQUAD_KINDS``, centre or cutoff ``freq`` in Hz at ``sample_rate``, quality factor ``Q`` and, for the
    equalizer, ``gain`` in dB.  The coefficients are designed and normalised in float64 on the host
    (``backend.biquad_coefficients``) and applied with ``lfilter`` (clamped to [-1, 1] when ``clamp``, as torchaudio's
    helpers do).  ``(batch, time, ch)`` / ``(batch, ch, time)`` in, the same shape out; differentiable with respect to
    the input."""

    def __init__(self, kind, sample_rate, freq, Q=0.707, gain=0.0, clamp=True, data_format='default', **kwargs):
        super().__init__(**kwargs)
        backend.validate_data_format_str(data_format)
        data_format = _unwrap_format(data_format)
        b, a = backend.biquad_coefficients(kind, sample_rate, freq, Q, gain)
        if b.ndim != 1:
            raise ValueError('freq, Q and gain must be numbers')
        self.kind, self.sample_rate, self.freq, self.Q, self.gain = kind, sample_rate, freq, Q, gain
        self.clamp = bool(clamp)
        self.b, self.a = b / a[0], a / a[0]
        self.data_format_str = data_format
        self.data_format = _resolve(data_format)
        self._coeffs = {}

    def coefficients(self, device):
        """(b, a) as float32 tensors on ``device`` (a[0] = 1), made on first use there."""
        key = device.index if device.index is not None else torch.cuda.current_device()
        c = self._coeffs.get(key)
        if c is None:
            c = self._coeffs[key] = tuple(torch.tensor(v, dtype=torch.float32, device=device) for v in (self.b, self.a))
        return c

    def call(self, x):
        b, a = self.coefficients(x.device)
        return lfilter(x, a, b, clamp=self.clamp, data_format=self.data_format)

    _config_fields = (
        ('kind', 'kind'),
        ('sample_rate', 'sample_rate'),
        ('freq', 'freq'),
        ('Q', 'Q'),
        ('gain', 'gain'),
        ('clamp', 'clamp'),
        ('data_format', 'data_format_str'),
    )


def _host_sos(sos):
    """Validated float64 host copy of second-order sections: (S, 6), (ch, S, 6) or (batch, ch, S, 6), 1 <= S <= 8,
    finite, every a0 == 1 (as ``scipy.signal.sosfilt`` requires)."""
    sos = np.asarray(sos, np.float64)
    if sos.ndim not in (2, 3, 4) or sos.shape[-1] != 6:
        raise ValueError('sos must be (S, 6), (ch, S, 6) or (batch, ch, S, 6), got shape %s' % (sos.shape,))
    if not 1 <= sos.shape[-2] <= ops.SOS_MAX_SECTIONS:
        raise ValueError('%d sections: 1 to %d are supported' % (sos.shape[-2], ops.SOS_MAX_SECTIONS))
    if not np.all(np.isfinite(sos)):
        raise ValueError('sos must be finite')
    if np.any(sos[..., 3] != 1):
        raise ValueError('every section must have a0 == 1 (sos[..., 3])')
    return sos


def _sos_tensor(x, sos, data_format):
    """sos as a (Bc, Cc, S, 6) float32 tensor on x's device after every check (``ops.sos_check``; a0 == 1 and finite
    values for host coefficients).  The coefficients are rounded to float32 once."""
    if not (isinstance(x, torch.Tensor) and x.is_cuda):
        raise ops.N.KapreNativeError('sosfilt needs a CUDA waveform')
    if isinstance(sos, torch.Tensor) and sos.requires_grad and torch.is_grad_enabled():
        raise ValueError('sosfilt has no gradient with respect to sos; detach it')
    if isinstance(sos, torch.Tensor) and sos.is_cuda:
        if sos.device != x.device:
            raise ValueError('sos on %s, the waveform on %s' % (sos.device, x.device))
        t = sos
    else:
        t = torch.from_numpy(_host_sos(sos.detach().cpu().numpy() if isinstance(sos, torch.Tensor) else sos))
    _, (Bc, Cc, S) = ops.sos_check(x, t, data_format)
    return t.to(device=x.device, dtype=torch.float32).reshape(Bc, Cc, S, 6)


def sosfilt(waveform, sos, zi=None, data_format='default'):
    """``scipy.signal.sosfilt`` along the time axis of ``waveform`` ``(batch, time, ch)`` / ``(batch, ch, time)`` (a CUDA
    tensor): S second-order sections in row order, each row ``[b0, b1, b2, a0, a1, a2]`` run in direct form II
    transposed,

        y = b0 x + z1,   z1 <- b1 x - a1 y + z2,   z2 <- b2 x - a2 y,

    the output of one section the input of the next.  ``sos``: ``(S, 6)`` (one filter), ``(ch, S, 6)`` or
    ``(batch, ch, S, 6)`` with axes of 1 shared, 1 <= S <= 8 (order 16); scipy's ``output='sos'`` designs.  a0 must be
    1: host coefficients with another a0 raise, and a0 of a CUDA tensor is not read (a check would synchronise).  The
    coefficients are rounded to float32 once.

    ``zi``: the initial state, ``(S, 2)``, ``(ch, S, 2)`` or ``(batch, ch, S, 2)`` in scipy's convention (for example
    ``backend.sosfilt_zi(sos) * x0``); with it the call returns ``(y, zf)``, zf the ``(batch, ch, S, 2)`` float32 final
    state, which continues the filter when passed as the next piece's ``zi``.  Without it the state starts at zero and
    only y is returned.

    Four launches (``kapre_sosfilt``): the chunked scan of ``lfilter`` over the cascade's 2S-dimensional state, so
    sharp filters that direct form cannot hold in float32 (``butter(8, 0.05)``) stay stable, and an output depends
    only on the input up to it, the coefficients and zi.  Differentiable with respect to the waveform (the backward is
    the same four launches in reverse time); zf carries no gradient, and a ``sos`` or ``zi`` that requires grad
    raises under grad mode."""
    fmt = _resolve(_unwrap_format(data_format))
    s = _sos_tensor(waveform, sos, fmt)
    z = None
    if zi is not None:
        z = zi if isinstance(zi, torch.Tensor) else torch.from_numpy(np.asarray(zi, np.float32))
        if torch.is_grad_enabled() and z.requires_grad:
            raise ValueError('sosfilt has no gradient with respect to zi; detach it')
        if z.is_cuda and z.device != waveform.device:
            raise ValueError('zi on %s, the waveform on %s' % (z.device, waveform.device))
        B, C = waveform.shape[0], waveform.shape[2 if fmt == _CH_LAST_STR else 1]
        Bz, Cz = ops.sos_state_check(z, B, C, s.shape[2], 'zi')
        z = z.to(device=waveform.device, dtype=torch.float32).reshape(Bz, Cz, s.shape[2], 2)
    y, zf = ops.sosfilt(waveform, s, z, reverse=False, data_format=fmt, want_zf=zi is not None)
    return (y, zf) if zi is not None else y


SOS_PADTYPES = ('odd', 'even', 'constant', None)


def _extend(x, n, padtype, t):
    """scipy's odd / even / constant extension of axis t by n samples on either side, with torch ops."""
    L = x.shape[t]
    first, last = x.narrow(t, 0, 1), x.narrow(t, L - 1, 1)
    left, right = x.narrow(t, 1, n).flip(t), x.narrow(t, L - 1 - n, n).flip(t)
    if padtype == 'odd':
        left, right = 2 * first - left, 2 * last - right
    elif padtype == 'constant':
        left, right = first.expand_as(left), last.expand_as(right)
    return torch.cat([left, x, right], t)


def sosfiltfilt(waveform, sos, padtype='odd', padlen=None, data_format='default'):
    """``scipy.signal.sosfiltfilt``: zero-phase filtering by ``sosfilt`` forward and then in reverse time, on the
    waveform extended at both ends.  ``padtype``: 'odd', 'even', 'constant' or None (no extension); ``padlen``
    defaults to ``3 (2 S + 1 - min(#(b2 == 0), #(a2 == 0)))`` (for per-item or per-channel coefficients, the largest
    over the filters; for CUDA coefficients counting reads them back, so pass ``padlen`` to avoid the
    synchronisation).  The forward pass starts from ``sosfilt_zi(sos) * x_ext[0]``, the reverse pass from
    ``sosfilt_zi(sos) * y[-1]``, and the extension is trimmed.  ``time <= padlen`` raises.  Arguments otherwise as
    ``sosfilt``.

    Eight launches; the reverse pass runs the kernel backwards in time, so nothing is flipped.  Differentiable with
    respect to the waveform, through both data-dependent initial states."""
    fmt = _resolve(_unwrap_format(data_format))
    s = _sos_tensor(waveform, sos, fmt)
    if padtype not in SOS_PADTYPES:
        raise ValueError('padtype must be one of %s, got: %r' % (SOS_PADTYPES, padtype))
    t = 1 if fmt == _CH_LAST_STR else 2
    L = waveform.shape[t]
    if padtype is None:
        edge = 0
    elif padlen is None:
        h = s.detach().cpu() if isinstance(sos, torch.Tensor) and sos.is_cuda else np.asarray(_host_sos(
            sos.detach().numpy() if isinstance(sos, torch.Tensor) else sos), np.float32)
        h = np.asarray(h).reshape(-1, s.shape[2], 6)
        taps = 2 * s.shape[2] + 1 - np.minimum((h[..., 2] == 0).sum(-1), (h[..., 5] == 0).sum(-1))
        edge = 3 * int(taps.max())
    else:
        if isinstance(padlen, bool) or not isinstance(padlen, (int, np.integer)) or padlen < 0:
            raise ValueError('padlen must be a non-negative integer, got: %r' % (padlen,))
        edge = int(padlen)
    if L <= edge:
        raise ValueError('the waveform\'s length %d must be greater than padlen, which is %d' % (L, edge))
    B, C = waveform.shape[0], waveform.shape[3 - t]
    ops.sosfilt_workspace(B, C, L + 2 * edge, s.shape[2], waveform.device)     # size checks before any launch
    ext = _extend(waveform, edge, padtype, t) if edge else waveform
    zi, gain = backend.sos_steady_state(s)
    y, _ = ops.sosfilt(ext, s, zi, scale=ext.select(t, 0), dc_gain=gain, reverse=False, data_format=fmt)
    y, _ = ops.sosfilt(y, s, zi, scale=y.select(t, y.shape[t] - 1), dc_gain=gain, reverse=True, data_format=fmt)
    return y.narrow(t, edge, L) if edge else y


@register_keras_serializable(package='Kapre')
class SOSFilter(Layer):
    """A fixed second-order-section cascade (``sosfilt`` from a zero state): ``(batch, time, ch)`` /
    ``(batch, ch, time)`` in, the same shape out.  ``sos``: ``(S, 6)``, ``(ch, S, 6)`` or ``(batch, ch, S, 6)`` as for
    ``sosfilt``, 1 <= S <= 8, a0 == 1 (scipy's ``output='sos'`` designs).  The coefficients are uploaded once per
    device as float32, so a call can be captured in a CUDA graph.  Differentiable with respect to the input."""

    def __init__(self, sos, data_format='default', **kwargs):
        super().__init__(**kwargs)
        backend.validate_data_format_str(data_format)
        data_format = _unwrap_format(data_format)
        self.sos = _host_sos(sos)
        self.data_format_str = data_format
        self.data_format = _resolve(data_format)
        self._coeffs = {}

    def coefficients(self, device):
        """sos as a float32 tensor on ``device``, made on first use there."""
        key = device.index if device.index is not None else torch.cuda.current_device()
        c = self._coeffs.get(key)
        if c is None:
            c = self._coeffs[key] = torch.tensor(self.sos, dtype=torch.float32, device=device)
        return c

    def call(self, x):
        if not (isinstance(x, torch.Tensor) and x.is_cuda):
            raise ops.N.KapreNativeError('SOSFilter needs a CUDA waveform')
        return sosfilt(x, self.coefficients(x.device), data_format=self.data_format)

    def get_config(self):
        config = super().get_config()
        config.update({'sos': self.sos.tolist(), 'data_format': self.data_format_str})
        return config


def dct2_htk_matrix(n_mels: int, n_mfccs: int) -> np.ndarray:
    """``tf.signal.mfccs_from_log_mel_spectrograms`` as a matrix: unnormalised DCT-II
    ``2 sum_n x[n] cos(pi k (2n+1) / (2N))`` scaled by ``1/sqrt(2N)`` (HTK convention), first
    ``n_mfccs`` coefficients.  Shape ``(n_mels, n_mfccs)`` so that it plugs into the filterbank kernel."""
    n = np.arange(n_mels, dtype=np.float64)[:, None]
    k = np.arange(n_mfccs, dtype=np.float64)[None, :]
    return (np.sqrt(2.0 / n_mels) * np.cos(np.pi * k * (2.0 * n + 1.0) / (2.0 * n_mels))).astype(np.float32)


@register_keras_serializable(package='Kapre')
class LogmelToMFCC(Layer):
    """MFCC from a log-mel spectrogram (reference kapre/signal.py:365-447): HTK-scaled DCT-II along the
    mel axis, first ``n_mfccs`` coefficients.  ``(b, time, mel, ch)`` -> ``(b, time, n_mfccs, ch)`` or
    ``(b, ch, time, mel)`` -> ``(b, ch, time, n_mfccs)``.  The DCT is a dense matrix on the mel axis, so it
    runs on the same kernel as ``ApplyFilterbank``."""

    def __init__(self, n_mfccs=20, data_format='default', **kwargs):
        super().__init__(**kwargs)
        backend.validate_data_format_str(data_format)
        self.n_mfccs = n_mfccs
        self.data_format_str = data_format
        self.data_format = _resolve(data_format)
        self.permutation = (0, 1, 3, 2) if self.data_format == _CH_LAST_STR else None
        self._fb = {}

    def call(self, log_melgrams):
        n_mels = log_melgrams.shape[2] if self.data_format == _CH_LAST_STR else log_melgrams.shape[3]
        fb = self._fb.get(n_mels)
        if fb is None:
            fb = self._fb[n_mels] = ops.Filterbank(dct2_htk_matrix(n_mels, min(self.n_mfccs, n_mels)))
        return ops.apply_filterbank(log_melgrams, fb, self.data_format)

    _config_fields = (('n_mfccs', 'n_mfccs'), ('data_format', 'data_format_str'))


def _kaldi(kind, waveform, lengths, data_format, seed, kwargs):
    o = ops.kaldi_options(kind, **kwargs)
    fmt = _resolve(_unwrap_format(data_format))
    if fmt not in (_CH_FIRST_STR, _CH_LAST_STR):
        raise ValueError('Unknown data_format: %r' % (data_format,))
    return ops.kaldi_features(waveform, ops.kaldi_plan(kind, o), lengths, fmt, o['dither'], seed)


def kaldi_fbank(waveform, lengths=None, data_format='default', seed=0, **kwargs):
    """``torchaudio.compliance.kaldi.fbank`` on the GPU for a batch: every keyword of torchaudio's function with its
    default, except ``channel`` (every channel is computed).  ``waveform``: float32 ``(batch, time, ch)`` /
    ``(batch, ch, time)`` CUDA tensor; returns ``(batch, frames, bins, ch)`` / ``(batch, ch, frames, bins)`` with
    ``bins = num_mel_bins + use_energy``.  ``lengths`` (``(batch,)`` integers, samples): item b is computed as if cut
    to ``lengths[b]`` and its frames past its own count are 0; ``frames`` is the largest count.  Dither is a
    deterministic function of ``(seed, item, channel, frame, sample)``.  The padded window must be 256, 512, 1024 or
    2048 samples.  One launch (two with ``subtract_mean``); differentiable with respect to ``waveform``."""
    return _kaldi('fbank', waveform, lengths, data_format, seed, kwargs)


def kaldi_mfcc(waveform, lengths=None, data_format='default', seed=0, **kwargs):
    """``torchaudio.compliance.kaldi.mfcc`` on the GPU for a batch (``num_ceps`` bins); see ``kaldi_fbank``."""
    return _kaldi('mfcc', waveform, lengths, data_format, seed, kwargs)


def kaldi_spectrogram(waveform, lengths=None, data_format='default', seed=0, **kwargs):
    """``torchaudio.compliance.kaldi.spectrogram`` on the GPU for a batch (``padded_window_size // 2 + 1`` bins);
    see ``kaldi_fbank``."""
    return _kaldi('spectrogram', waveform, lengths, data_format, seed, kwargs)


# ---- pitch tracking -------------------------------------------------------------------------------------------
_PYIN_DEFAULTS = dict(n_thresholds=100, beta_parameters=(2, 18), boltzmann_parameter=2, resolution=0.1,
                      max_transition_rate=35.92, switch_prob=0.01, no_trough_prob=0.01)
_pitch_plans = {}


def _pitch_plan(sample_rate, fmin, fmax, frame_length, win_length, hop_length, center, trough_threshold, pyin=None,
                fill_na=float('nan')):
    """One PitchPlan per configuration (so a call uploads nothing after the first and can be captured)."""
    key = (float(sample_rate), float(fmin), float(fmax), frame_length, win_length, hop_length, bool(center),
           float(trough_threshold), None if pyin is None else tuple(sorted((k, v if not isinstance(v, list) else
                                                                            tuple(v)) for k, v in pyin.items())),
           repr(float(fill_na)))
    plan = _pitch_plans.get(key)
    if plan is None:
        plan = ops.PitchPlan(sample_rate, fmin, fmax, frame_length, win_length, hop_length, center, trough_threshold,
                             pyin, fill_na)
        _pitch_plans[key] = plan
    return plan


def yin(waveform, sample_rate, fmin, fmax, frame_length=2048, win_length=None, hop_length=None, trough_threshold=0.1,
        center=True, data_format='default'):
    """YIN fundamental frequency (Hz) per frame of ``waveform`` ``(batch, time, ch)`` / ``(batch, ch, time)`` (a
    float32 CUDA tensor), as ``(batch, frames, ch)`` / ``(batch, ch, frames)`` float32; modelled on ``librosa.yin``.

    Frame m holds samples [m h - F / 2, m h + F / 2) with ``center`` (zeros outside the signal; librosa 0.10's
    ``pad_mode='constant'``, the only pad mode), else [m h, m h + F); frames = 1 + (L_pad - F) // h.  With W =
    ``win_length`` (default F // 2), h = ``hop_length`` (default F // 4) and x the frame,

        d(tau) = sum_{j=1..W} (x[j] - x[j + tau])^2,   c(tau) = d(tau) / (mean_{k<=tau} d(k) + 2^-126)

    for tau in [floor(sr / fmax), min(ceil(sr / fmin), F - W - 1)].  The first trough of c below
    ``trough_threshold`` is chosen, else the first global minimum, refined by a parabolic shift; f0 = sr / period.
    Unlike librosa, no autocorrelation or energy term is flushed to zero below 1e-6, so quiet signals behave as loud
    ones.  A frame holding a non-finite sample gives NaN; no other frame changes.  An output's bits depend on its
    (item, channel, frame) alone.

    One launch.  f0 comes from a discrete choice, so it has no gradient: an input that requires grad is accepted
    and the output carries no ``grad_fn``."""
    fmt = _resolve(_unwrap_format(data_format))
    plan = _pitch_plan(sample_rate, fmin, fmax, frame_length, win_length, hop_length, center, trough_threshold)
    return ops.yin(waveform, plan, fmt)


def pyin(waveform, sample_rate, fmin, fmax, frame_length=2048, win_length=None, hop_length=None, n_thresholds=100,
         beta_parameters=(2, 18), boltzmann_parameter=2, resolution=0.1, max_transition_rate=35.92, switch_prob=0.01,
         no_trough_prob=0.01, fill_na=float('nan'), center=True, data_format='default'):
    """Probabilistic YIN (modelled on ``librosa.pyin``): ``(f0, voiced_flag, voiced_prob)``, each ``(batch, frames,
    ch)`` / ``(batch, ch, frames)`` (float32, bool, float32).  Framing and CMNDF as ``yin``.

    Each trough of the CMNDF gets the probability sum_i Boltzmann(rank among the troughs below s_i) beta_i over the
    thresholds s_i = i / n_thresholds with beta_i the Beta(``beta_parameters``) mass of (s_{i-1}, s_i]; the first
    global-minimum trough also gets ``no_trough_prob`` times the mass of the thresholds at or below it.  Troughs map
    to pitch bins of ``resolution`` semitones from ``fmin``; the voiced observation of a bin is the **sum** of its
    troughs' probabilities (librosa keeps the last one), ``voiced_prob = min(sum, 1)``, and each unvoiced state
    observes (1 - voiced_prob) / n_pitch.  A Viterbi decode over 2 n_pitch states (voiced, then unvoiced) with a
    triangular transition band of ``max_transition_rate`` semitones per second and ``switch_prob`` gives the path;
    f0 is the bin frequency on voiced frames and ``fill_na`` elsewhere.  Log probabilities are log(p + 2^-126) and
    transitions outside the band are excluded (librosa gives them log(tiny)).  A non-finite sample makes its whole
    (item, channel) row ``fill_na``, unvoiced and NaN; no other row changes.

    Two launches: the CMNDF with the trough probabilities, then the Viterbi decode.  No gradient: an input that
    requires grad is accepted and the outputs carry no ``grad_fn``."""
    fmt = _resolve(_unwrap_format(data_format))
    q = dict(n_thresholds=n_thresholds, beta_parameters=tuple(beta_parameters), boltzmann_parameter=boltzmann_parameter,
             resolution=resolution, max_transition_rate=max_transition_rate, switch_prob=switch_prob,
             no_trough_prob=no_trough_prob)
    plan = _pitch_plan(sample_rate, fmin, fmax, frame_length, win_length, hop_length, center, 0.1, q, fill_na)
    return ops.pyin(waveform, plan, fmt)


@register_keras_serializable(package='Kapre')
class YIN(Layer):
    """``yin`` as a layer: ``(batch, time, ch)`` / ``(batch, ch, time)`` in, ``(batch, frames, ch)`` / ``(batch, ch,
    frames)`` f0 out.  Same arguments as ``yin`` (without the waveform)."""

    def __init__(self, sample_rate, fmin, fmax, frame_length=2048, win_length=None, hop_length=None,
                 trough_threshold=0.1, center=True, data_format='default', **kwargs):
        super().__init__(**kwargs)
        backend.validate_data_format_str(data_format)
        data_format = _unwrap_format(data_format)
        self.sample_rate, self.fmin, self.fmax = sample_rate, fmin, fmax
        self.frame_length, self.win_length, self.hop_length = frame_length, win_length, hop_length
        self.trough_threshold, self.center = trough_threshold, center
        self.data_format_str = data_format
        self.data_format = _resolve(data_format)
        self.plan = _pitch_plan(sample_rate, fmin, fmax, frame_length, win_length, hop_length, center,
                                trough_threshold)

    def call(self, x):
        return ops.yin(x, self.plan, self.data_format)

    _config_fields = (
        ('sample_rate', 'sample_rate'), ('fmin', 'fmin'), ('fmax', 'fmax'), ('frame_length', 'frame_length'),
        ('win_length', 'win_length'), ('hop_length', 'hop_length'), ('trough_threshold', 'trough_threshold'),
        ('center', 'center'), ('data_format', 'data_format_str'),
    )


@register_keras_serializable(package='Kapre')
class PYIN(Layer):
    """``pyin`` as a layer: the waveform in, ``(f0, voiced_flag, voiced_prob)`` out.  Same arguments as ``pyin``."""

    def __init__(self, sample_rate, fmin, fmax, frame_length=2048, win_length=None, hop_length=None, n_thresholds=100,
                 beta_parameters=(2, 18), boltzmann_parameter=2, resolution=0.1, max_transition_rate=35.92,
                 switch_prob=0.01, no_trough_prob=0.01, fill_na=float('nan'), center=True, data_format='default',
                 **kwargs):
        super().__init__(**kwargs)
        backend.validate_data_format_str(data_format)
        data_format = _unwrap_format(data_format)
        self.sample_rate, self.fmin, self.fmax = sample_rate, fmin, fmax
        self.frame_length, self.win_length, self.hop_length = frame_length, win_length, hop_length
        self.n_thresholds, self.beta_parameters = n_thresholds, tuple(beta_parameters)
        self.boltzmann_parameter, self.resolution = boltzmann_parameter, resolution
        self.max_transition_rate, self.switch_prob = max_transition_rate, switch_prob
        self.no_trough_prob, self.fill_na, self.center = no_trough_prob, fill_na, center
        self.data_format_str = data_format
        self.data_format = _resolve(data_format)
        q = dict(n_thresholds=n_thresholds, beta_parameters=self.beta_parameters,
                 boltzmann_parameter=boltzmann_parameter, resolution=resolution,
                 max_transition_rate=max_transition_rate, switch_prob=switch_prob, no_trough_prob=no_trough_prob)
        self.plan = _pitch_plan(sample_rate, fmin, fmax, frame_length, win_length, hop_length, center, 0.1, q, fill_na)

    def call(self, x):
        return ops.pyin(x, self.plan, self.data_format)

    _config_fields = (
        ('sample_rate', 'sample_rate'), ('fmin', 'fmin'), ('fmax', 'fmax'), ('frame_length', 'frame_length'),
        ('win_length', 'win_length'), ('hop_length', 'hop_length'), ('n_thresholds', 'n_thresholds'),
        ('beta_parameters', 'beta_parameters'), ('boltzmann_parameter', 'boltzmann_parameter'),
        ('resolution', 'resolution'), ('max_transition_rate', 'max_transition_rate'), ('switch_prob', 'switch_prob'),
        ('no_trough_prob', 'no_trough_prob'), ('fill_na', 'fill_na'), ('center', 'center'),
        ('data_format', 'data_format_str'),
    )


# ---- chroma ------------------------------------------------------------------------------------------------------------
_chroma_plans = {}


def _cached(key, make):
    plan = _chroma_plans.get(key)
    if plan is None:
        plan = make()
        _chroma_plans[key] = plan
    return plan


def _stft_chroma_plans(sample_rate, n_fft, hop_length, window_name, n_chroma, tuning, ctroct, octwidth, base_c,
                       bins_per_octave=None, resolution=0.01, tables=True):
    """(StftPlan, ChromaPlan) of one chroma_stft / estimate_tuning configuration.  ``tuning=None``: one table per
    left edge of the tuning grid plus one for 0.0 (items without peaks), and the tuning estimate."""
    n_fft = backend._check_n_fft(n_fft)
    n_chroma = backend._check_n_chroma(n_chroma)
    if isinstance(hop_length, bool) or int(hop_length) != hop_length or int(hop_length) < 1:
        raise ValueError('hop_length must be a positive integer, got %r' % (hop_length,))
    hop_length = int(hop_length)
    sr = float(sample_rate)
    if not (np.isfinite(sr) and sr > 0):
        raise ValueError('sample_rate must be positive, got %r' % (sample_rate,))
    stft = _cached(('stft', n_fft, hop_length, window_name),
                   lambda: ops.StftPlan(n_fft, n_fft, hop_length, backend.get_window_fn(window_name)(n_fft)))
    fb = dict(ctroct=ctroct, octwidth=octwidth, base_c=bool(base_c))
    if tuning is not None:
        t = float(tuning)
        key = ('chroma', sr, n_fft, n_chroma, t, ctroct, octwidth, bool(base_c))
        return stft, _cached(key, lambda: ops.ChromaPlan(
            backend.chroma_filterbank(sr, n_fft, n_chroma, t, **fb)[None]))
    bpo = n_chroma if bins_per_octave is None else bins_per_octave
    if isinstance(bpo, bool) or not (np.isfinite(float(bpo)) and float(bpo) > 0):
        raise ValueError('bins_per_octave must be positive, got %r' % (bins_per_octave,))
    edges = backend.tuning_edges(resolution)
    lo, hi = backend.piptrack_bins(sr, n_fft)
    est = dict(edges=edges, lo=lo, hi=hi, sample_rate=sr, n_fft=float(n_fft), bins_per_octave=float(bpo))
    if not tables:
        key = ('tuning', sr, n_fft, float(bpo), float(resolution))
        return stft, _cached(key, lambda: ops.ChromaPlan(None, tuning=est, n_chroma=1, n_bins=n_fft // 2 + 1))
    key = ('chroma_est', sr, n_fft, n_chroma, float(resolution), ctroct, octwidth, bool(base_c))

    def make():
        grid = [backend.chroma_filterbank(sr, n_fft, n_chroma, e, **fb) for e in edges[:-1]]
        grid.append(backend.chroma_filterbank(sr, n_fft, n_chroma, 0.0, **fb))
        return ops.ChromaPlan(np.stack(grid), tuning=est)
    return stft, _cached(key, make)


def _centred_magnitude(waveform, stft, fmt, center):
    """|STFT| of ``waveform`` with ``n_fft // 2`` zeros on each side when ``center``: a pad in front of the fused
    STFT-magnitude launch, differentiable through both."""
    if not (isinstance(waveform, torch.Tensor) and waveform.is_cuda):
        raise ops.N.KapreNativeError('chroma needs a CUDA waveform')
    if waveform.dim() != 3:
        raise ValueError('expected a 3-D waveform batch, got shape %s' % (tuple(waveform.shape),))
    x = waveform.to(torch.float32)
    if center:
        h = stft.n_fft // 2
        x = torch.nn.functional.pad(x, (0, 0, h, h) if fmt == _CH_LAST_STR else (h, h))
    return ops.stft_forward(x, stft, fmt, fmt, False, False, ops.N.OUT_MAG)


def _spectrogram_arg(S, name, fmt, bins, allow_complex=False):
    if not (isinstance(S, torch.Tensor) and S.is_cuda):
        raise ops.N.KapreNativeError('%s must be a CUDA tensor' % name)
    if S.dim() != 4:
        raise ValueError('%s must be 4-D, got shape %s' % (name, tuple(S.shape)))
    K = S.shape[2] if fmt == _CH_LAST_STR else S.shape[3]
    if K != bins:
        raise ValueError('%s has %d bins, expected %d' % (name, K, bins))
    if not (S.dtype == torch.float32 or (allow_complex and S.dtype == torch.complex64)):
        raise ValueError('%s must be float32%s, got %s' % (name, ' or complex64' if allow_complex else '', S.dtype))
    return S


def chroma_stft(waveform=None, sample_rate=22050, S=None, norm=np.inf, n_fft=2048, hop_length=512, win_length=None,
                window_name=None, center=True, tuning=None, n_chroma=12, ctroct=5.0, octwidth=2.0, base_c=True,
                data_format='default'):
    """Chroma of a power spectrogram (modelled on ``librosa.feature.chroma_stft``): float32 ``(batch, frames,
    n_chroma, ch)`` / ``(batch, ch, frames, n_chroma)``.

    From ``waveform`` (``(batch, time, ch)`` / ``(batch, ch, time)`` float32 CUDA), S = |STFT|^2 with the periodic
    Hann window (``window_name``) of ``n_fft`` samples every ``hop_length``, unnormalised; with ``center`` the signal
    first gets ``n_fft // 2`` zeros on each side (librosa's ``pad_mode='constant'``), giving ``1 + time // hop``
    frames.  ``win_length`` must be None or ``n_fft``.  ``S`` (instead of a waveform): a power spectrogram in this
    library's layout, used as given.  The chroma is ``normalize(W @ S, norm)`` with W =
    ``backend.chroma_filterbank(sample_rate, n_fft, n_chroma, tuning, ctroct, octwidth, base_c)``; ``norm`` is inf,
    1, 2 or None, and a frame whose length is below FLT_MIN is left as it is.

    ``tuning=None`` estimates each item's tuning from S (``estimate_tuning`` with ``bins_per_octave=n_chroma``) on
    the device: the plan holds a table per edge of the tuning grid and the projection reads each item's index, so
    nothing is synchronised with the host and the call can be captured in a CUDA graph; the result equals
    ``chroma_stft(tuning=t_i)`` item by item, bit for bit.

    Launches: the STFT magnitude and the projection (2), plus 7 with ``tuning=None``; from ``S`` only the chroma
    launches.  Differentiable with respect to the waveform and ``S``; the tuning estimate is a constant."""
    fmt = _resolve(_unwrap_format(data_format))
    code = backend.chroma_norm_code(norm)
    if win_length is not None and win_length != n_fft:
        raise ValueError('win_length must be None or n_fft=%r, got %r: the STFT does not centre a shorter window'
                         % (n_fft, win_length))
    if (waveform is None) == (S is None):
        raise ValueError('pass exactly one of waveform and S')
    stft, plan = _stft_chroma_plans(sample_rate, n_fft, hop_length, window_name, n_chroma, tuning, ctroct, octwidth,
                                    base_c)
    if S is None:
        X = _centred_magnitude(waveform, stft, fmt, center)
        mode = ops.N.CHROMA_IN_SQUARE
    else:
        X = _spectrogram_arg(S, 'S', fmt, n_fft // 2 + 1)
        mode = ops.N.CHROMA_IN_LINEAR
    table = None
    if tuning is None:
        table = ops.chroma_tuning(X, plan, mode, fmt)[1]
    return ops.chroma(X, plan, mode, code, None, fmt, table)


def estimate_tuning(waveform=None, sample_rate=22050, S=None, n_fft=2048, hop_length=None, resolution=0.01,
                    bins_per_octave=12, data_format='default'):
    """librosa's ``estimate_tuning`` per item (over all its channels) on the device: a float64 ``(batch,)`` CUDA
    tensor of tunings in fractions of a bin of ``bins_per_octave``, in [-0.5, 0.5).

    piptrack's peaks (``fmin=150``, ``fmax=min(4000, sr / 2)``, ``threshold=0.1``) of S, from ``waveform`` the
    centred |STFT| (``power=1``, hop ``n_fft // 4`` by default) or the given ``S`` (the library's layout); the peaks
    with magnitude at or above their exact median; the residual ``mod(bins_per_octave log2(pitch / 27.5), 1)`` in
    [-0.5, 0.5) binned over ``linspace(-0.5, 0.5, ceil(1 / resolution) + 1)``; the left edge of the first fullest
    bin.  An item without peaks gives 0.0, and a frame holding a non-finite bin has no peaks.  Launches: the STFT
    magnitude (from a waveform) and 7, whatever the data; nothing is read back.  No gradient: an input that requires
    grad is accepted and the output carries no ``grad_fn``."""
    fmt = _resolve(_unwrap_format(data_format))
    if (waveform is None) == (S is None):
        raise ValueError('pass exactly one of waveform and S')
    n_fft = backend._check_n_fft(n_fft)
    hop = n_fft // 4 if hop_length is None else hop_length
    stft, plan = _stft_chroma_plans(sample_rate, n_fft, hop, None, 1, None, 5.0, 2.0, True, bins_per_octave,
                                    resolution, tables=False)
    with torch.no_grad():
        if S is None:
            X = _centred_magnitude(waveform.detach(), stft, fmt, True)
        else:
            X = _spectrogram_arg(S, 'S', fmt, n_fft // 2 + 1).detach()
        return ops.chroma_tuning(X, plan, ops.N.CHROMA_IN_LINEAR, fmt)[0]


def _cqt_chroma_plans(sample_rate, hop_length, f_min, tuning, n_chroma, n_octaves, bins_per_octave, base_c, smooth):
    n_chroma = backend._check_n_chroma(n_chroma)
    for name, v in (('n_octaves', n_octaves), ('bins_per_octave', bins_per_octave)):
        if isinstance(v, bool) or int(v) != v or int(v) < 1:
            raise ValueError('%s must be a positive integer, got %r' % (name, v))
    if isinstance(tuning, bool) or tuning is None or not np.isfinite(float(tuning)):
        raise ValueError('tuning must be a finite number (per-item tuning needs a CQT plan per item), got %r'
                         % (tuning,))
    bpo, n_bins = int(bins_per_octave), int(n_octaves) * int(bins_per_octave)
    fmin = backend.CQT_C1 if f_min is None else float(f_min)
    m = backend.cq_to_chroma(n_bins, bpo, n_chroma, fmin, base_c)
    ftuned = fmin * 2.0 ** (float(tuning) / bpo)
    cqt = _cached(('cqt', float(sample_rate), int(hop_length), ftuned, n_bins, bpo),
                  lambda: ops.CqtPlan(sample_rate, hop_length, ftuned, n_bins, bpo))
    taps = None if smooth is False else backend.cens_window(smooth)
    key = ('cq_chroma', n_bins, bpo, n_chroma, fmin, bool(base_c), None if taps is None else tuple(taps))
    return cqt, _cached(key, lambda: ops.ChromaPlan(m[None], smooth=taps))


def _cq_magnitude(waveform, C, cqt, fmt):
    if (waveform is None) == (C is None):
        raise ValueError('pass exactly one of waveform and C')
    if C is None:
        return ops.cqt(waveform, cqt, fmt, fmt, True), ops.N.CHROMA_IN_LINEAR
    C = _spectrogram_arg(C, 'C', fmt, cqt.n_bins, allow_complex=True)
    return C, ops.N.CHROMA_IN_COMPLEX if C.dtype == torch.complex64 else ops.N.CHROMA_IN_LINEAR


def chroma_cqt(waveform=None, sample_rate=22050, C=None, hop_length=512, f_min=None, norm=np.inf, threshold=0.0,
               tuning=0.0, n_chroma=12, n_octaves=7, bins_per_octave=36, base_c=True, data_format='default'):
    """Constant-Q chroma (modelled on ``librosa.feature.chroma_cqt``): float32 ``(batch, frames, n_chroma, ch)`` /
    ``(batch, ch, frames, n_chroma)``.

    C = |CQT| of ``n_octaves * bins_per_octave`` bins from ``f_min 2^(tuning / bins_per_octave)`` (``f_min`` default
    C1; see ``time_frequency.CQT``), or the given ``C`` (complex64, or float32 |C|, in the CQT's layout).  The chroma
    is ``normalize(threshold(M @ C), norm)`` with M = ``backend.cq_to_chroma`` (``bins_per_octave`` a multiple of
    ``n_chroma``), entries below ``threshold`` set to 0 (None: no threshold).  ``tuning`` is a number: librosa's
    ``None`` would need a CQT plan per item.  Launches: the CQT's (7 at the defaults) and 1; from ``C`` only the
    chroma launch.  Differentiable with respect to the waveform and ``C``."""
    fmt = _resolve(_unwrap_format(data_format))
    code = backend.chroma_norm_code(norm)
    if threshold is not None and not np.isfinite(float(threshold)):
        raise ValueError('threshold must be finite or None, got %r' % (threshold,))
    cqt, plan = _cqt_chroma_plans(sample_rate, hop_length, f_min, tuning, n_chroma, n_octaves, bins_per_octave,
                                  base_c, False)
    X, mode = _cq_magnitude(waveform, C, cqt, fmt)
    return ops.chroma(X, plan, mode, code, threshold, fmt)


def chroma_cens(waveform=None, sample_rate=22050, C=None, hop_length=512, f_min=None, tuning=0.0, n_chroma=12,
                n_octaves=7, bins_per_octave=36, base_c=True, norm=2, win_len_smooth=41, data_format='default'):
    """Chroma energy normalised statistics (modelled on ``librosa.feature.chroma_cens``): ``chroma_cqt`` with no
    normalisation, L1-normalised per frame, quantised to ``0.25 #{s in (0.4, 0.2, 0.1, 0.05) : v > s}``, smoothed
    along time by ``hann(win_len_smooth + 2, symmetric) / sum`` centred with zeros outside the signal
    (``scipy.ndimage.convolve(mode='constant')``; None or 0: no smoothing) and normalised with ``norm`` (2).  A NaN
    chroma stays NaN through the quantisation (librosa's would become 0), so it reaches only the frames whose smoothing
    window holds it.  Launches: the CQT's and 2.  No gradient: an input that requires grad is accepted and the output
    carries no ``grad_fn``."""
    fmt = _resolve(_unwrap_format(data_format))
    if backend.chroma_norm_code(norm) != 3:
        raise ValueError('chroma_cens supports norm=2 only, got %r' % (norm,))
    cqt, plan = _cqt_chroma_plans(sample_rate, hop_length, f_min, tuning, n_chroma, n_octaves, bins_per_octave,
                                  base_c, win_len_smooth)
    with torch.no_grad():
        X, mode = _cq_magnitude(None if waveform is None else waveform.detach(),
                                None if C is None else C.detach(), cqt, fmt)
        return ops.chroma_cens(X, plan, mode, fmt)


# ---- harmonic/percussive separation ------------------------------------------------------------------------------------
def hpss(S, kernel_size=31, power=2.0, mask=False, margin=1.0, data_format='default'):
    """Harmonic/percussive separation by median filtering (``librosa.decompose.hpss``, Fitzgerald 2010) of a CUDA
    spectrogram batch ``(batch, frames, bins, ch)`` / ``(batch, ch, frames, bins)``: float32 magnitudes (or power),
    used as given, or complex64 (``STFT``'s output), whose magnitude is formed as ``Magnitude`` forms it.  S must be
    non-negative; this is not checked.

    ``H`` and ``P`` are the medians of ``kernel_size`` values along frames and along bins, exactly as
    ``scipy.ndimage.median_filter(mode='reflect')`` computes them (an even size takes the upper median); a window
    holding NaN gives NaN.  The masks are ``softmask(H, margin_h P)`` and ``softmask(P, margin_p H)`` with librosa's
    ``util.softmask``.  Returns ``(harmonic, percussive)``: ``S M`` for float input, ``M X`` for complex input, or the
    masks with ``mask=True``; each shaped like S.  ``kernel_size`` (1 .. 64) and ``margin`` (finite, >= 1) are a
    number or a pair (harmonic, percussive); ``power > 0`` may be ``inf``.  One launch; differentiable with respect
    to S."""
    backend.validate_data_format_str(data_format)
    cfg = ops.hpss_config(kernel_size, power, mask, margin)
    return ops.hpss(S, cfg, _resolve(_unwrap_format(data_format)))


_hpss_transforms = {}


def _hpss_component(waveform, component, kernel_size, power, margin, n_fft, win_length, hop_length, window_name,
                    data_format):
    from .time_frequency import STFT, InverseSTFT
    backend.validate_data_format_str(data_format)
    fmt = _resolve(_unwrap_format(data_format))
    cfg = ops.hpss_config(kernel_size, power, False, margin)
    win = n_fft if win_length is None else win_length
    hop = win // 4 if hop_length is None else hop_length
    if hop > win:
        raise ValueError('hop_length (%r) must not exceed win_length (%r)' % (hop, win))
    if not isinstance(waveform, torch.Tensor) or waveform.dim() != 3:
        raise ValueError('%s expects a 3-D waveform batch' % (component,))
    key = (n_fft, win_length, hop_length, window_name, fmt)
    pair = _hpss_transforms.get(key)
    if pair is None:
        pair = (STFT(n_fft=n_fft, win_length=win_length, hop_length=hop_length, window_name=window_name,
                     pad_begin=True, pad_end=True, input_data_format=fmt, output_data_format=_CH_LAST_STR),
                InverseSTFT(n_fft=n_fft, win_length=win_length, hop_length=hop_length, forward_window_name=window_name,
                            input_data_format=_CH_LAST_STR, output_data_format=fmt))
        _hpss_transforms[key] = pair
    stft, istft = pair
    length = waveform.shape[2] if fmt == _CH_FIRST_STR else waveform.shape[1]
    h, p = ops.hpss(stft.call(waveform), cfg, _CH_LAST_STR, want_h=component == 'harmonic',
                    want_p=component == 'percussive')
    y = istft.call(h if component == 'harmonic' else p)
    start = stft.n_fft - stft.hop_length
    return y[:, :, start:start + length] if fmt == _CH_FIRST_STR else y[:, start:start + length, :]


def harmonic(waveform, kernel_size=31, power=2.0, margin=1.0, n_fft=2048, win_length=None, hop_length=None,
             window_name=None, data_format='default'):
    """The harmonic part of a CUDA waveform batch ``(batch, time, ch)`` / ``(batch, ch, time)``, the same shape out
    (``librosa.effects.harmonic``): ``STFT`` with ``pad_begin`` and ``pad_end``, ``hpss`` writing the harmonic
    component alone, ``InverseSTFT`` with the dual window, then ``time`` samples from ``n_fft - hop_length`` on, which
    is where input sample 0 lands, so the output is time-aligned with the input.  With margins of 1 and a finite power
    the masks sum to 1 and ``harmonic(y) + percussive(y)`` reproduces ``y`` to rounding.

    Departure from librosa: the framing is kapre's (``pad_begin``/``pad_end`` and the dual window), not librosa's
    centred frames and envelope-normalised ``istft``, so samples near the ends differ.  ``hop_length > win_length``
    raises ``ValueError``.  Three launches; differentiable with respect to the waveform."""
    return _hpss_component(waveform, 'harmonic', kernel_size, power, margin, n_fft, win_length, hop_length,
                           window_name, data_format)


def percussive(waveform, kernel_size=31, power=2.0, margin=1.0, n_fft=2048, win_length=None, hop_length=None,
               window_name=None, data_format='default'):
    """The percussive part of a CUDA waveform batch (``librosa.effects.percussive``); see ``harmonic``."""
    return _hpss_component(waveform, 'percussive', kernel_size, power, margin, n_fft, win_length, hop_length,
                           window_name, data_format)


# ---- onsets, tempo and beats -------------------------------------------------------------------------------------------
def _rhythm_frontend(sample_rate, n_fft, hop_length, n_mels, fmin, fmax):
    """(StftPlan, Filterbank) of librosa's default onset feature: the periodic Hann STFT and the slaney mel bank."""
    n_fft = backend._check_n_fft(n_fft)
    if isinstance(hop_length, bool) or int(hop_length) != hop_length or int(hop_length) < 1:
        raise ValueError('hop_length must be a positive integer, got %r' % (hop_length,))
    sr = float(sample_rate)
    if not (np.isfinite(sr) and sr > 0):
        raise ValueError('sample_rate must be positive, got %r' % (sample_rate,))
    n_mels = ops._check_int('n_mels', n_mels, 1)
    stft = _cached(('stft', n_fft, int(hop_length), None),
                   lambda: ops.StftPlan(n_fft, n_fft, int(hop_length), backend.get_window_fn(None)(n_fft)))
    key = ('onset_mel', sr, n_fft, n_mels, float(fmin), None if fmax is None else float(fmax))
    fb = _cached(key, lambda: ops.Filterbank(backend.filterbank_mel(sr, n_fft // 2 + 1, n_mels, fmin, fmax)))
    return stft, fb


def _onset_feature(waveform, sample_rate, n_fft, hop_length, n_mels, fmin, fmax, fmt):
    """librosa's default onset feature of a waveform batch: the centred |STFT|^2, the mel bank and
    ``MagnitudeToDecibel(1.0, 1e-10, 80)`` (the clamp reference is each item's maximum)."""
    stft, fb = _rhythm_frontend(sample_rate, n_fft, hop_length, n_mels, fmin, fmax)
    X = _centred_magnitude(waveform, stft, fmt, True)
    return backend.magnitude_to_decibel(ops.apply_filterbank(X * X, fb, fmt), ref_value=1.0, amin=1e-10,
                                        dynamic_range=80.0)


def _one_source(a, b, names):
    if (a is None) == (b is None):
        raise ValueError('pass exactly one of %s and %s' % names)


def onset_strength(waveform=None, sample_rate=22050, S=None, lag=1, max_size=1, detrend=False, center=True,
                   aggregate='mean', n_fft=2048, hop_length=512, n_mels=128, fmin=0.0, fmax=None,
                   data_format='default'):
    """Spectral-flux onset strength (modelled on ``librosa.onset.onset_strength``): float32 ``(batch, frames, ch)`` /
    ``(batch, ch, frames)``, one value per frame of S.

    From ``waveform`` (``(batch, time, ch)`` / ``(batch, ch, time)`` float32 CUDA), S is librosa's default feature:
    the centred periodic-Hann STFT (``n_fft // 2`` zeros on each side, ``1 + time // hop_length`` frames), squared,
    ``backend.filterbank_mel(sample_rate, n_fft // 2 + 1, n_mels, fmin, fmax)`` and ``MagnitudeToDecibel(1.0,
    1e-10, 80)``, whose clamp reference is each item's maximum (librosa: the whole array's).  ``S`` (instead): any
    float32 spectrogram in this library's layout, 1 to 4097 bins, used as given.

    With m = ``max_size`` and K bins: ``R[t][b]`` = max of S[t] over bins ``b - m//2 .. b - m//2 + m - 1`` inside
    the row, ``D = max(0, S[t] - R[t - lag])`` (NaN kept), the mean (float64 sum / K, rounded once) or numpy's
    median over bins, then ``lag + n_fft // (2 hop_length)`` (with ``center``, else ``lag``) zeros in front and the
    row cut to its frames; ``detrend`` then runs ``lfilter(b=[1, -1], a=[1, -0.99])``.  Restated from librosa's
    definitions, not checked against librosa.

    One launch from S (plus four for ``detrend``), four more from a waveform.  Differentiable with respect to S and
    the waveform: relu'(0) = 0, a window maximum's gradient to the lowest of its tied bins, the median's to the
    element(s) it selected."""
    fmt = _resolve(_unwrap_format(data_format))
    _one_source(waveform, S, ('waveform', 'S'))
    n_fft = backend._check_n_fft(n_fft)
    hop_length = ops._check_int('hop_length', hop_length, 1)
    cfg = ops.onset_config(lag, max_size, aggregate, n_fft // (2 * hop_length) if center else 0)
    if S is None:
        if not (isinstance(waveform, torch.Tensor) and waveform.dim() == 3):
            raise ValueError('waveform must be a 3-D (batch, time, ch) / (batch, ch, time) tensor')
        length = waveform.shape[1] if fmt == _CH_LAST_STR else waveform.shape[2]
        ops.onset_limits(cfg, ops._check_int('n_mels', n_mels, 1), 1 + length // hop_length)
        S = _onset_feature(waveform, sample_rate, n_fft, hop_length, n_mels, fmin, fmax, fmt)
    elif not (isinstance(S, torch.Tensor) and S.is_cuda):
        raise ops.N.KapreNativeError('S must be a CUDA tensor')
    e = ops.onset_strength(S, cfg, fmt)
    if detrend:
        b = torch.tensor([[[1.0, -1.0]]], dtype=torch.float32, device=e.device)
        a = torch.tensor([[[1.0, -0.99]]], dtype=torch.float32, device=e.device)
        e = ops.lfilter(e, b, a, clamp=False, data_format=fmt)
    return e


def _envelope(waveform, onset_envelope, sample_rate, hop_length, fmt, aggregate='mean'):
    _one_source(waveform, onset_envelope, ('waveform', 'onset_envelope'))
    if onset_envelope is not None:
        return onset_envelope
    with torch.no_grad():
        return onset_strength(waveform.detach(), sample_rate=sample_rate, hop_length=hop_length, aggregate=aggregate,
                              data_format=fmt)


def tempogram(waveform=None, sample_rate=22050, onset_envelope=None, hop_length=512, win_length=384, center=True,
              norm=np.inf, data_format='default'):
    """Autocorrelation tempogram (modelled on ``librosa.feature.tempogram``): float32 ``(batch, frames,
    win_length, ch)`` / ``(batch, ch, frames, win_length)``.

    With W = ``win_length`` (2 .. 4096) and ``center``, the envelope gets ``W // 2`` linear ramps to zero on each
    side (``np.pad(mode='linear_ramp')``) and there is one frame per envelope frame; without it the frames are
    0 .. T - W.  Each frame is windowed by the periodic Hann window of W, autocorrelated (``ac[l] = sum y[j]
    y[j + l]``, a float32 fma chain in ascending j) and, with ``norm=np.inf``, divided by its largest ``|ac|`` unless
    that is below FLT_MIN; ``norm=None`` leaves it.  From a waveform the envelope is ``onset_strength`` at its defaults
    with this ``hop_length``.  Restated from librosa's definitions, not checked against librosa.

    One launch from the envelope.  No gradient: under grad mode an input that requires grad raises."""
    fmt = _resolve(_unwrap_format(data_format))
    if norm is not None and norm != np.inf:
        raise ValueError('norm must be np.inf or None, got %r' % (norm,))
    for x in (waveform, onset_envelope):
        if ops._wants_grad(x):
            raise ValueError('tempogram has no gradient: call it under torch.no_grad() or on a detached input')
    ops.tempogram_check(win_length)
    e = _envelope(waveform, onset_envelope, sample_rate, hop_length, fmt)
    return ops.tempogram(e, win_length, center, norm is not None, fmt)


_tempo_plans = {}


def _tempo_plan(sample_rate, hop_length, ac_size, start_bpm, std_bpm, max_tempo, win_length=None):
    """The TempoPlan of one configuration: W lags from ``ac_size`` (librosa's ``time_to_frames``), or ``win_length``
    (a given tempogram's own lag count) when that is not None."""
    for name, v in (('start_bpm', start_bpm), ('std_bpm', std_bpm)):
        if isinstance(v, bool) or not (np.isfinite(float(v)) and float(v) > 0):
            raise ValueError('%s must be positive, got %r' % (name, v))
    sr = float(sample_rate)
    if not (np.isfinite(sr) and sr > 0):
        raise ValueError('sample_rate must be positive, got %r' % (sample_rate,))
    hop = ops._check_int('hop_length', hop_length, 1)
    if win_length is None:
        W = int(math.floor(math.floor(float(ac_size) * sr) / hop))
        if not 2 <= W <= ops.N.TEMPOGRAM_MAX_WIN:
            raise ValueError('ac_size=%r gives a window of %d frames, outside [2, %d]'
                             % (ac_size, W, ops.N.TEMPOGRAM_MAX_WIN))
    else:
        W = ops.tempogram_check(win_length)
    key = (sr, hop, W, float(start_bpm), float(std_bpm), None if max_tempo is None else float(max_tempo))
    plan = _tempo_plans.get(key)
    if plan is None:
        plan = ops.TempoPlan(W, sr, hop, start_bpm, std_bpm, max_tempo)
        _tempo_plans[key] = plan
    return plan


def tempo(waveform=None, sample_rate=22050, onset_envelope=None, tg=None, hop_length=512, start_bpm=120.0,
          std_bpm=1.0, ac_size=8.0, max_tempo=320.0, aggregate='mean', data_format='default'):
    """Tempo in bpm (modelled on ``librosa.feature.tempo``): float32 ``(batch, ch)``, or per frame ``(batch, frames,
    ch)`` / ``(batch, ch, frames)`` with ``aggregate=None``.

    From a waveform or an envelope, tg is the centred ``norm=inf`` tempogram of W = floor(floor(ac_size sr) / hop)
    lags (2 .. 4096).  A given ``tg`` (``(batch, frames, W, ch)`` / ``(batch, ch, frames, W)`` float32) is used with
    its own W, as librosa does, and ``ac_size`` is not used.  g is the float64 mean of tg over its frames (or each
    frame with ``aggregate=None``).  With ``bpm[l] = 60 sr / (hop l)`` and a log-normal prior around ``start_bpm``
    (``std_bpm`` octaves; lags below the first one under ``max_tempo`` excluded), the tempo is ``bpm[first argmax
    (log1p(1e6 g) + logprior)]`` in float64.  Restated from librosa's definitions, not checked against librosa.

    Departures: a row (or frame) holding a non-finite value gives NaN.  A lag whose score is NaN (g below -1e-6,
    which a detrended or user-made envelope can give) is skipped, as ``np.nanargmax`` skips it, where numpy's argmax
    would pick it; a row with no lag left gives NaN.

    Launches: two from ``tg`` (one with ``aggregate=None``), one more from an envelope, five more from a waveform.
    No gradient: an input that requires grad is accepted and the output carries no ``grad_fn``."""
    fmt = _resolve(_unwrap_format(data_format))
    if aggregate not in ('mean', None):
        raise ValueError("aggregate must be 'mean' or None, got %r" % (aggregate,))
    if sum(x is not None for x in (waveform, onset_envelope, tg)) != 1:
        raise ValueError('pass exactly one of waveform, onset_envelope and tg')
    W = None
    if tg is not None:
        if not isinstance(tg, torch.Tensor) or tg.dim() != 4:
            raise ValueError('tg must be a 4-D tempogram tensor')
        W = int(tg.shape[2] if fmt == _CH_LAST_STR else tg.shape[3])
    plan = _tempo_plan(sample_rate, hop_length, ac_size, start_bpm, std_bpm, max_tempo, W)
    with torch.no_grad():
        if tg is None:
            e = _envelope(waveform, onset_envelope, sample_rate, hop_length, fmt)
            tg = ops.tempogram(e.detach(), plan.W, True, True, fmt)
        return ops.tempo(tg, plan, aggregate is None, fmt)


def onset_detect(waveform=None, sample_rate=22050, onset_envelope=None, hop_length=512, normalize=True, pre_max=None,
                 post_max=None, pre_avg=None, post_avg=None, delta=0.07, wait=None, data_format='default'):
    """Onsets by peak picking (modelled on ``librosa.onset.onset_detect`` with ``sparse=False``): a bool mask shaped
    like the envelope.

    Defaults: ``pre_max = wait = floor(0.03 sr / hop)``, ``post_max = 1``, ``pre_avg = floor(0.1 sr / hop)``,
    ``post_avg = pre_avg + 1``.  With ``normalize`` x = (e - min e) / (max(e - min e) + FLT_MIN) in float32; frame n
    is a candidate when x[n] is the maximum of x[n - pre_max .. n + post_max), is nonzero and is at least the
    float64 mean of x[n - pre_avg .. n + post_avg) plus ``delta`` (windows clipped to the row); candidates within
    ``wait`` frames of the last accepted one are dropped.  A row with no nonzero x or a non-finite value has no
    onsets.  Restated from librosa's definitions, not checked against librosa.

    One launch from the envelope (five more from a waveform).  No gradient."""
    fmt = _resolve(_unwrap_format(data_format))
    sr = float(sample_rate)
    hop = ops._check_int('hop_length', hop_length, 1)
    d_pre_max = int(0.03 * sr // hop)
    d_pre_avg = int(0.10 * sr // hop)
    cfg = ops.onset_detect_config(d_pre_max if pre_max is None else pre_max, 1 if post_max is None else post_max,
                                  d_pre_avg if pre_avg is None else pre_avg,
                                  d_pre_avg + 1 if post_avg is None else post_avg,
                                  d_pre_max if wait is None else wait, delta, normalize)
    with torch.no_grad():
        e = _envelope(waveform, onset_envelope, sample_rate, hop, fmt)
        return ops.onset_detect(e, cfg, fmt)


def beat_track(waveform=None, sample_rate=22050, onset_envelope=None, hop_length=512, start_bpm=120.0,
               tightness=100.0, trim=True, bpm=None, data_format='default'):
    """Dynamic-programming beat tracking (modelled on ``librosa.beat.beat_track``): ``(tempo, beats)``, tempo float32
    ``(batch, ch)`` and beats a bool mask shaped like the envelope.

    From a waveform the envelope is ``onset_strength(aggregate='median')``.  ``bpm=None`` takes each row's
    ``tempo(onset_envelope=e, start_bpm=start_bpm)`` on the device; a given ``bpm`` is used for every row.  The
    period is p = rint(60 (sr / hop) / bpm), 1 .. 4096.  The local score is the envelope over its standard deviation
    (ddof=1) convolved with exp(-0.5 (32 d / p)^2), d = -p .. p; the float64 dynamic programme scores each frame
    from offsets -2p .. -rint(p / 2) with ``-tightness ln(-d / p)^2``, the last beat is the last frame whose doubled
    cumulative score (at local maxima) exceeds their median, backlinks give the rest, and with ``trim`` the weak
    beats at both ends are dropped (keeping librosa's slice, which drops the last strong one too).  An all-zero row
    gives tempo 0 and no beats, a non-finite one tempo NaN and no beats.  Restated from librosa's definitions, not
    checked against librosa.

    Nothing is synchronised with the host, so the call can be captured in a CUDA graph.  Launches: one, plus three for
    the tempo and five for a waveform's envelope.  No gradient."""
    fmt = _resolve(_unwrap_format(data_format))
    cfg = ops.beat_config(sample_rate, ops._check_int('hop_length', hop_length, 1), tightness, trim)
    if bpm is None:
        plan = _tempo_plan(sample_rate, hop_length, 8.0, start_bpm, 1.0, 320.0)
    else:
        if isinstance(bpm, bool) or not (np.isfinite(float(bpm)) and float(bpm) > 0):
            raise ValueError('bpm must be positive, got %r' % (bpm,))
        p = int(np.rint(60.0 * cfg.fps / float(bpm)))
        if not 1 <= p <= ops.N.BEAT_MAX_PERIOD:
            raise ValueError('bpm=%r gives a beat period of %d frames, outside [1, %d]'
                             % (bpm, p, ops.N.BEAT_MAX_PERIOD))
    with torch.no_grad():
        e = _envelope(waveform, onset_envelope, sample_rate, hop_length, fmt, aggregate='median')
        if bpm is None:
            bpm = ops.tempo(ops.tempogram(e.detach(), plan.W, True, True, fmt), plan, False, fmt)
        return ops.beat_track(e, cfg, bpm, fmt)


def _host64(v, name, shapes):
    """A host value (number, NumPy array or CPU tensor) as float64 whose shape, or shape without its leading batch
    axis, is one of ``shapes`` (None: any length)."""
    if isinstance(v, torch.Tensor):
        if v.is_cuda:
            raise ValueError('%s must be a host value (geometry is read on the host), got a CUDA tensor' % name)
        v = v.detach().numpy()
    a = np.asarray(v, np.float64)

    def fits(shape):
        return any(len(shape) == len(t) and all(x is None or x == y for x, y in zip(t, shape)) for t in shapes)
    if not (fits(a.shape) or (a.ndim and fits(a.shape[1:]))):
        raise ValueError('%s must have shape %s, or a batch of them, got %s' % (name, ' or '.join(map(str, shapes)),
                                                                              a.shape))
    return a


def simulate_rir_ism(room, source, mic_array, max_order, absorption, output_length, delay_filter_length=81,
                     sound_speed=343.0, sample_rate=16000.0, data_format='default'):
    """Room impulse responses of a shoebox room by the image-source method (named and shaped after torchaudio's old
    prototype ``simulate_rir_ism``; the maths is this library's own, modelled on pyroomacoustics' shoebox ISM and not
    checked against either, DESIGN.md §RIR).

    ``room`` (sides, metres) and ``source`` are ``(3,)`` or ``(B, 3)``, ``mic_array`` ``(M, 3)`` or ``(B, M, 3)``,
    ``absorption`` (energy absorption in [0, 1]) a float, ``(6,)`` or ``(B, 6)`` for the walls
    ``(x=0, x=Lx, y=0, y=Ly, z=0, z=Lz)``: host values (floats, NumPy arrays or CPU tensors).  Each image adds its
    gain times a Hann-windowed sinc of ``delay_filter_length`` (odd, 1 to 255) taps centred on its delay plus half the
    filter; ``max_order`` (None or an int >= 0) keeps the images of at most that many reflections.  Returns the first
    ``output_length`` samples of every response, float32 ``(B, output_length, M)`` / ``(B, M, output_length)`` in
    waveform layout, so that ``Convolve()(x.expand(...), h)`` gives the array's signals.  One launch, no gradient.
    Each sample's bits depend on its item's geometry and its index alone.  Out-of-range values raise ValueError
    before anything is launched."""
    if max_order is not None and (isinstance(max_order, (bool, np.bool_)) or not isinstance(max_order, (int, np.integer))
                                  or max_order < 0):
        raise ValueError('max_order must be None or a non-negative int, got: %r' % (max_order,))
    if isinstance(output_length, (bool, np.bool_)) or not isinstance(output_length, (int, np.integer)) \
            or output_length < 1:
        raise ValueError('output_length must be an int >= 1, got: %r' % (output_length,))
    if isinstance(delay_filter_length, (bool, np.bool_)) or not isinstance(delay_filter_length, (int, np.integer)):
        raise ValueError('delay_filter_length must be an odd int from 1 to 255, got: %r' % (delay_filter_length,))
    backend.validate_data_format_str(data_format)
    fmt = _resolve(_unwrap_format(data_format))
    room = _host64(room, 'room', [(3,)])
    source = _host64(source, 'source', [(3,)])
    mics = _host64(mic_array, 'mic_array', [(None, 3)])
    if mics.shape[-2] < 1:
        raise ValueError('mic_array needs at least one mic, got shape %s' % (mics.shape,))
    absorption = _host64(absorption, 'absorption', [(), (6,)])
    B = max(a.shape[0] if a.ndim == nd else 1 for a, nd in ((room, 2), (source, 2), (mics, 3), (absorption, 2)))
    for a, nd, name in ((room, 2, 'room'), (source, 2, 'source'), (mics, 3, 'mic_array'), (absorption, 2, 'absorption')):
        if a.ndim == nd and a.shape[0] not in (1, B):
            raise ValueError('%s has batch %d, expected 1 or %d' % (name, a.shape[0], B))
    room = np.broadcast_to(room.reshape(-1, 3), (B, 3))
    source = np.broadcast_to(source.reshape(-1, 3), (B, 3))
    mics = np.broadcast_to(mics.reshape((-1,) + mics.shape[-2:]), (B,) + mics.shape[-2:])
    absorption = np.broadcast_to(absorption.reshape(-1, 6) if absorption.ndim else absorption.reshape(1, 1), (B, 6))
    if not np.all((absorption >= 0) & (absorption <= 1)):
        raise ValueError('absorption must lie in [0, 1]')
    records = np.zeros((B, ops.RIR_RECORD), np.float64)
    records[:, 0:3], records[:, 3:6], records[:, 6:12] = room, source, np.sqrt(1.0 - absorption)
    records[:, 12] = -1.0 if max_order is None else float(max_order)
    return ops.rir_ism(records, mics, int(output_length), int(delay_filter_length), float(sample_rate),
                       float(sound_speed), fmt)
