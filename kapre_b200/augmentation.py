"""Augmentation layers (reference: kapre/augmentation.py).  ``SpecAugment``: the masks are drawn on the host, the
masking is one CUDA pass (``kapre_spec_augment``).  ``TimeStretch``: a phase vocoder, one CUDA scan over time
(``kapre_time_stretch``)."""
from __future__ import annotations

import numpy as np

from . import backend, ops
from .backend import _CH_DEFAULT_STR, _CH_FIRST_STR, _CH_LAST_STR
from .time_frequency import Layer, _resolve, _unwrap_format, register_keras_serializable


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
