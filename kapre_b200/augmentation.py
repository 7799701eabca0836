"""Augmentation layers (reference: kapre/augmentation.py).  ``SpecAugment``: the masks are drawn on the host, the
masking is one CUDA pass (``kapre_spec_augment``).  ``TimeStretch``: a phase vocoder, one CUDA scan over time
(``kapre_time_stretch``).  ``PitchShift``: STFT, that phase vocoder, the inverse STFT and one band-limited
interpolation (``kapre_sinc_resample``) back to the input length."""
from __future__ import annotations

import numpy as np

from . import backend, ops
from .backend import _CH_DEFAULT_STR, _CH_FIRST_STR, _CH_LAST_STR
from .time_frequency import STFT, InverseSTFT, Layer, _resolve, _unwrap_format, register_keras_serializable


def draw_masks(rng: np.random.Generator, batch: int, n_masks: int, mask_param: int, axis_limit: int) -> np.ndarray:
    """(batch, n_masks, 2) int32 (start, width) pairs, distributed as kapre/augmentation.py:205-208 draws them:
    ``width ~ U{0 .. mask_param - 1}``, ``start ~ U{0 .. axis_limit - width - 1}`` (tf.random.uniform with integer maxval is
    exclusive); the masked indices are ``start <= i <= start + width``."""
    if axis_limit < mask_param:
        raise ValueError('Time and freq axis shapes must be greater than time_mask_param '
                         'and freq_mask_param respectively')
    width = rng.integers(0, mask_param, size=(batch, n_masks))
    start = (rng.random(size=(batch, n_masks)) * (axis_limit - width)).astype(np.int64)
    start = np.minimum(start, axis_limit - width - 1)
    return np.stack([start, width], axis=-1).astype(np.int32)


@register_keras_serializable(package='Kapre')
class SpecAugment(Layer):
    """SpecAugment (reference: kapre/augmentation.py:116-326): ``n_time_masks`` / ``n_freq_masks`` random masks per batch item
    on the time / frequency axis of a depth-1 spectrogram, applied only when called with ``training=True``."""

    def __init__(self, freq_mask_param, time_mask_param, n_freq_masks=1, n_time_masks=1, mask_value=0.0,
                 data_format='default', seed=None, **kwargs):
        super().__init__(**kwargs)
        backend.validate_data_format_str(data_format)
        data_format = _unwrap_format(data_format)
        self.freq_mask_param = freq_mask_param
        self.time_mask_param = time_mask_param
        self.n_freq_masks = n_freq_masks
        self.n_time_masks = n_time_masks
        self.mask_value = mask_value
        if not self.freq_mask_param or not self.time_mask_param:
            raise RuntimeError('Both freq_mask_param and time_mask_param must be defined and different '
                               'than zero')
        self.data_format = _resolve(data_format)
        self._rng = np.random.default_rng(seed)

    def call(self, x, training=None, **kwargs):
        if training in (None, False):
            return x
        if x.dim() != 4:
            raise ValueError('ndim of input tensor x should be 4 (batch spectrogram),' 'but it is %d' % x.dim())
        if self.data_format == _CH_FIRST_STR:
            B, C, T, F = x.shape
        else:
            B, T, F, C = x.shape
        if C != 1:
            raise RuntimeError('SpecAugment does not support spectrograms with depth greater than 1')
        tm = draw_masks(self._rng, B, max(int(self.n_time_masks), 0), self.time_mask_param, T) \
            if self.n_time_masks >= 1 else np.zeros((B, 0, 2), np.int32)
        fm = draw_masks(self._rng, B, max(int(self.n_freq_masks), 0), self.freq_mask_param, F) \
            if self.n_freq_masks >= 1 else np.zeros((B, 0, 2), np.int32)
        self.last_masks = (tm, fm)          # what was applied (tests, debugging)
        return ops.spec_augment(x, tm, fm, float(self.mask_value), self.data_format)

    def __call__(self, x, training=None, **kwargs):
        if training in (None, False):
            return x                                       # inference: identity, like the reference
        t, was_host = ops.to_device(x)
        y = self.call(t, training=training)
        return ops.to_host(y) if was_host else y

    def get_config(self):
        config = super().get_config()
        config.update({'freq_mask_param': self.freq_mask_param, 'time_mask_param': self.time_mask_param,
                       'n_freq_masks': self.n_freq_masks, 'n_time_masks': self.n_time_masks,
                       'mask_value': self.mask_value,
                       'data_format': self.data_format if self.data_format in (_CH_FIRST_STR, _CH_LAST_STR) else _CH_DEFAULT_STR})
        return config


@register_keras_serializable(package='Kapre')
class TimeStretch(Layer):
    """Stretches a complex spectrogram in time without changing its pitch: ``torchaudio.transforms.TimeStretch`` /
    ``torchaudio.functional.phase_vocoder``.  ``(batch, time, freq, ch)`` / ``(batch, ch, time, freq)`` complex in,
    ``ceil(time / rate)`` frames out in the same data format (complex64; complex128 input is cast).  ``rate > 1``
    speeds up, ``rate < 1`` slows down; ``rate == 1`` returns the input itself.  ``call(x, rate=...)`` overrides the
    rate for one call, like torchaudio's ``overriding_rate``.

    Output frame ``u`` reads frames ``k = floor(u * rate)`` and ``k + 1`` (zeros past the end), with
    ``alpha = u * rate - k`` in float64: its magnitude is ``alpha |X[k + 1]| + (1 - alpha) |X[k]|`` and its phase is
    ``angle(X[0])`` plus the sum of ``angle(X[k_v + 1]) - angle(X[k_v])`` over the outputs ``v < u``.  torchaudio adds
    and removes a ``phase_advance`` inside a wrap to 2 pi; modulo 2 pi that cancels exactly, so the result does not
    depend on the hop length and the layer takes none.  The phase sum is kept as a 32-bit fixed-point count of
    turns, so it does not drift over long inputs (torchaudio's float32 ``cumsum`` does) and the output does not depend
    on the batch size or data format.  The gradient with respect to the input is available when the CUDA input
    requires grad."""

    def __init__(self, rate, data_format='default', **kwargs):
        super().__init__(**kwargs)
        backend.validate_data_format_str(data_format)
        data_format = _unwrap_format(data_format)
        self.rate = ops._check_rate(rate)
        self.data_format_original = data_format
        self.data_format = _resolve(data_format)

    def call(self, x, rate=None):
        if x.dim() != 4:
            raise ValueError('TimeStretch expects a 4-D complex batch, got shape %s' % (tuple(x.shape),))
        return ops.time_stretch(x, self.rate if rate is None else ops._check_rate(rate), self.data_format)

    _config_fields = (
        ('rate', 'rate'),
        ('data_format', 'data_format_original'),
    )


@register_keras_serializable(package='Kapre')
class PitchShift(Layer):
    """Shifts the pitch of a waveform by ``n_steps`` steps of an octave divided into ``bins_per_octave`` without
    changing its length (``torchaudio.transforms.PitchShift``): ``(batch, time, ch)`` / ``(batch, ch, time)`` in, the
    same shape out.  ``n_steps`` is any number with ``|n_steps| <= 2 * bins_per_octave``; ``call(x, n_steps=...)``
    overrides it for one call, and 0 returns the input itself.

    With ``rate = 2 ** (-n_steps / bins_per_octave)`` the layer runs four steps: ``STFT``
    (``pad_begin`` and ``pad_end``, so that frames cover every input sample), ``TimeStretch(rate)``, ``InverseSTFT``
    with the dual window, and the band-limited interpolation ``ops.sinc_resample`` by the ratio ``rate`` to the input
    length.  Two differences from torchaudio: the ratio is ``rate`` itself, not ``int(sample_rate / rate) /
    sample_rate``, so the layer takes no sample rate; and the output is time-aligned with the input.

    Alignment.  ``pad_begin`` prepends ``pad = n_fft - hop_length`` zeros, so input sample ``t`` is the centre of the
    (fractional) frame ``k = (t + pad - win_length / 2) / hop_length``.  The stretch moves frame ``k`` to frame
    ``k / rate``, and the inverse puts the centre of that frame at ``k / rate * hop_length + win_length / 2`` of its
    untrimmed output.  Output sample ``m`` of the interpolation reads position ``offset + m / rate``, so it reads input
    time ``m`` when ``offset = win_length / 2 + (pad - win_length / 2) / rate``.  That aligns the frames exactly; what
    a phase vocoder does to the position of an event inside a frame (it keeps each bin's phase advance, not the
    relation between bins) stays, so a tone burst comes out within ``hop_length`` of where it was and a click within
    half a window.

    Differentiable with respect to the input, because each of the four steps is."""

    def __init__(self, n_steps, bins_per_octave=12, n_fft=2048, win_length=None, hop_length=None, window_name=None,
                 data_format='default', **kwargs):
        super().__init__(**kwargs)
        backend.validate_data_format_str(data_format)
        data_format = _unwrap_format(data_format)
        if isinstance(bins_per_octave, bool) or not isinstance(bins_per_octave, (int, np.integer)) or bins_per_octave <= 0:
            raise ValueError('bins_per_octave must be a positive integer, got: %r' % (bins_per_octave,))
        self.bins_per_octave = int(bins_per_octave)
        self.n_steps = self._check(n_steps)
        self.data_format_original = data_format
        self.data_format = _resolve(data_format)
        self.stft = STFT(n_fft=n_fft, win_length=win_length, hop_length=hop_length, window_name=window_name,
                         pad_begin=True, pad_end=True, input_data_format=self.data_format,
                         output_data_format=_CH_LAST_STR)
        self.n_fft, self.win_length, self.hop_length = self.stft.n_fft, self.stft.win_length, self.stft.hop_length
        self.window_name = window_name
        self.stretch = TimeStretch(self.rate(self.n_steps), data_format=_CH_LAST_STR)
        self.istft = InverseSTFT(n_fft=n_fft, win_length=win_length, hop_length=hop_length,
                                 forward_window_name=window_name, input_data_format=_CH_LAST_STR,
                                 output_data_format=self.data_format)

    def _check(self, n_steps):
        if isinstance(n_steps, (bool, np.bool_)) or not isinstance(n_steps, (int, float, np.integer, np.floating)) \
                or not abs(float(n_steps)) <= 2 * self.bins_per_octave:
            raise ValueError('n_steps must be a number with |n_steps| <= 2 * bins_per_octave = %d, got: %r'
                             % (2 * self.bins_per_octave, n_steps))
        return float(n_steps)

    def rate(self, n_steps):
        """The time-stretch rate and the interpolation ratio of a shift by ``n_steps``."""
        return 2.0 ** (-float(n_steps) / self.bins_per_octave)

    def offset(self, rate):
        """Where input sample 0 lands in the untrimmed inverse STFT of the stretched frames (see the class docstring)."""
        return self.win_length / 2.0 + ((self.n_fft - self.hop_length) - self.win_length / 2.0) / rate

    def call(self, x, n_steps=None):
        if x.dim() != 3:
            raise ValueError('PitchShift expects a 3-D batch, got shape %s' % (tuple(x.shape),))
        n_steps = self.n_steps if n_steps is None else self._check(n_steps)
        if n_steps == 0.0:
            return x
        rate = self.rate(n_steps)
        length = x.shape[2] if self.data_format == _CH_FIRST_STR else x.shape[1]
        y = self.istft.call(self.stretch.call(self.stft.call(x), rate=rate))
        return ops.sinc_resample(y, rate, length, self.offset(rate), self.data_format)

    _config_fields = (
        ('n_steps', 'n_steps'),
        ('bins_per_octave', 'bins_per_octave'),
        ('n_fft', 'n_fft'),
        ('win_length', 'win_length'),
        ('hop_length', 'hop_length'),
        ('window_name', 'window_name'),
        ('data_format', 'data_format_original'),
    )
