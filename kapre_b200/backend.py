"""Host-side mirror of ``kapre/backend.py`` for the hot path.

Same public names, argument meaning and error behaviour as the reference
(``kapre/backend.py``), but the constants are built with NumPy on the host
(the reference calls ``tf.signal.*_window`` / ``librosa.filters.mel``) and the tensor op
``magnitude_to_decibel`` runs as CUDA kernels through the C ABI.
"""
from __future__ import annotations

from typing import Callable, Optional, Union

import numpy as np

_CH_FIRST_STR = 'channels_first'   # kapre/backend.py:53
_CH_LAST_STR = 'channels_last'     # kapre/backend.py:54
_CH_DEFAULT_STR = 'default'        # kapre/backend.py:55

_IMAGE_DATA_FORMAT = _CH_LAST_STR  # Keras' default K.image_data_format()
_FLOATX = 'float32'                # Keras' default K.floatx()


def image_data_format() -> str:
    """What ``'default'`` resolves to (``K.image_data_format()``, kapre/time_frequency.py:142-144)."""
    return _IMAGE_DATA_FORMAT


def set_image_data_format(data_format: str) -> None:
    """Equivalent of ``keras.backend.set_image_data_format`` for the ``'default'`` resolution."""
    global _IMAGE_DATA_FORMAT
    if data_format not in (_CH_FIRST_STR, _CH_LAST_STR):
        raise ValueError('Unknown data_format: %r' % (data_format,))
    _IMAGE_DATA_FORMAT = data_format


def _get_floatx() -> str:
    return _FLOATX


# ------------------------------------------------------------------------------- windows
def _raised_cosine(length: int, a: float, b: float, dtype) -> np.ndarray:
    # tf.signal's "periodic" raised cosine: periodic for even lengths, symmetric for odd ones
    # (denominator W + even - 1), ones for W == 1.
    length = int(length)
    if length == 1:
        return np.ones(1, dtype=dtype)
    denom = length + (1 - length % 2) - 1
    phase = (2.0 * np.pi / denom) * np.arange(length, dtype=np.float64)
    return (a - b * np.cos(phase)).astype(dtype)


def hann_window(window_length, dtype=np.float32):
    return _raised_cosine(window_length, 0.5, 0.5, dtype)


def hamming_window(window_length, dtype=np.float32):
    return _raised_cosine(window_length, 0.54, 0.46, dtype)


def kaiser_window(window_length, beta=12.0, dtype=np.float32):
    return np.kaiser(int(window_length), beta).astype(dtype)


def kaiser_bessel_derived_window(window_length, beta=12.0, dtype=np.float32):
    half = int(window_length) // 2
    cs = np.cumsum(np.kaiser(half + 1, beta))
    half_w = np.sqrt(cs[:-1] / cs[-1])
    return np.concatenate([half_w, half_w[::-1]]).astype(dtype)


def vorbis_window(window_length, dtype=np.float32):
    n = np.arange(int(window_length), dtype=np.float64) + 0.5
    return np.sin(np.pi / 2.0 * np.sin(np.pi * n / int(window_length)) ** 2).astype(dtype)


_WINDOWS = {
    'hamming_window': hamming_window,
    'hann_window': hann_window,
    'kaiser_bessel_derived_window': kaiser_bessel_derived_window,
    'kaiser_window': kaiser_window,
    'vorbis_window': vorbis_window,
}


def get_window_fn(window_name: Optional[str] = None) -> Callable[..., np.ndarray]:
    """Return a window function given its name (kapre/backend.py:58-100).

    ``None`` means ``'hann_window'``.  The returned callable takes the window length and
    returns a float32 NumPy array with ``tf.signal``'s values.  Unknown names raise
    ``NotImplementedError`` like the reference.
    """
    if window_name is None:
        return hann_window
    if window_name not in _WINDOWS:
        raise NotImplementedError(
            'Window name %s is not supported now. Currently, %d windows are'
            'supported - %s' % (window_name, len(_WINDOWS), ', '.join(_WINDOWS.keys())))
    return _WINDOWS[window_name]


def inverse_stft_window_fn(frame_step: int, forward_window_fn: Callable[..., np.ndarray]):
    """``tf.signal.inverse_stft_window_fn`` (used at kapre/time_frequency.py:278-280): the dual
    synthesis window ``w[n] / sum_k w^2[n mod hop + k*hop]``."""

    def inner(frame_length, dtype=np.float32):
        w = np.asarray(forward_window_fn(frame_length, dtype=np.float64), dtype=np.float64)
        overlaps = -(-int(frame_length) // int(frame_step))
        sq = np.zeros(overlaps * int(frame_step))
        sq[:frame_length] = w * w
        den = np.tile(sq.reshape(overlaps, frame_step).sum(axis=0), overlaps)[:frame_length]
        with np.errstate(divide='ignore', invalid='ignore'):
            return (w / den).astype(dtype)

    return inner


def validate_data_format_str(data_format: str) -> None:
    """kapre/backend.py:103-123: ``TypeError`` for non-strings, ``ValueError`` for unknown values."""
    if not isinstance(data_format, str):
        raise TypeError('data_format must be a string, got %s: %s' % (type(data_format).__name__, data_format))
    if data_format not in (_CH_DEFAULT_STR, _CH_FIRST_STR, _CH_LAST_STR):
        raise ValueError('data_format must be one of %s, got: %r'
                         % ([_CH_FIRST_STR, _CH_LAST_STR, _CH_DEFAULT_STR], data_format))


# ------------------------------------------------------------------------------- decibel
def magnitude_to_decibel(x, ref_value: float = 1.0, amin: float = 1e-5, dynamic_range: float = 80.0):
    """Decibel scaling, kapre/backend.py:126-194, on the GPU.

    ``10*log10(max(x, amin)) - 10*log10(max(amin, ref_value))`` clamped from below at (maximum
    over all non-batch axes) - ``dynamic_range``; a 1-D input uses the global maximum.
    Accepts a CUDA ``torch.Tensor`` (returns one) or a NumPy array (returns NumPy).
    """
    if ref_value <= 0:
        raise ValueError('ref_value must be positive, got: %s' % (ref_value,))
    if amin <= 0:
        raise ValueError('amin must be positive, got: %s' % (amin,))
    if dynamic_range <= 0:
        raise ValueError('dynamic_range must be positive, got: %s' % (dynamic_range,))
    from . import ops
    return ops.magnitude_to_decibel(x, ref_value, amin, dynamic_range)


# ------------------------------------------------------------------------------- filterbanks
def _hz_to_mel(freq, htk):
    freq = np.asarray(freq, dtype=np.float64)
    if htk:
        return 2595.0 * np.log10(1.0 + freq / 700.0)
    lin = freq * (3.0 / 200.0)
    knee_hz, knee_mel, step = 1000.0, 15.0, np.log(6.4) / 27.0
    return np.where(freq >= knee_hz, knee_mel + np.log(np.maximum(freq, knee_hz) / knee_hz) / step, lin)


def _mel_to_hz(mel, htk):
    mel = np.asarray(mel, dtype=np.float64)
    if htk:
        return 700.0 * (np.power(10.0, mel / 2595.0) - 1.0)
    knee_hz, knee_mel, step = 1000.0, 15.0, np.log(6.4) / 27.0
    return np.where(mel >= knee_mel, knee_hz * np.exp(step * (mel - knee_mel)), mel * (200.0 / 3.0))


def filterbank_mel(sample_rate: int, n_freq: int, n_mels: int = 128, f_min: float = 0.0,
                   f_max: Optional[float] = None, htk: bool = False,
                   norm: Union[str, int, float, None] = 'slaney') -> np.ndarray:
    """Mel filterbank of shape ``(n_freq, n_mels)``, float32 (kapre/backend.py:197-231).

    Restates ``librosa.filters.mel(sr, n_fft=(n_freq-1)*2, n_mels, fmin, fmax, htk, norm)``
    (librosa >= 0.11): triangles between neighbouring mel-spaced centre frequencies evaluated
    at the FFT-bin frequencies; ``'slaney'`` scales band i by ``2 / (f[i+2] - f[i])``; a numeric
    ``norm`` p-normalises every band; ``None`` leaves the triangles at unit peak.
    """
    n_mels = int(n_mels)
    n_fft = (int(n_freq) - 1) * 2
    top = float(sample_rate) / 2 if f_max is None else f_max
    bin_hz = np.fft.rfftfreq(n_fft, 1.0 / sample_rate)                       # (n_freq,)
    edges = _mel_to_hz(np.linspace(_hz_to_mel(f_min, htk), _hz_to_mel(top, htk), n_mels + 2), htk)
    width = np.diff(edges)                                                   # (n_mels + 1,)
    dist = edges[:, None] - bin_hz[None, :]                                  # (n_mels + 2, n_freq)
    rising = -dist[:-2] / width[:-1, None]
    falling = dist[2:] / width[1:, None]
    tri = np.maximum(0, np.minimum(rising, falling)).astype(np.float32)      # stored as float32
    if isinstance(norm, str):
        if norm != 'slaney':
            raise ValueError('Unsupported norm=%r' % (norm,))
        scale = 2.0 / (edges[2:] - edges[:-2])
        tri = (tri.astype(np.float64) * scale[:, None]).astype(np.float32)
    elif norm is not None:
        p = float(norm)
        mag = np.abs(tri)
        length = np.max(mag, axis=-1, keepdims=True) if np.isinf(p) else \
            np.sum(mag ** np.float32(p), axis=-1, keepdims=True) ** np.float32(1.0 / p)
        length = np.where(length < np.finfo(np.float32).tiny, np.float32(1.0), length)
        tri = (tri / length).astype(np.float32)
    return np.ascontiguousarray(tri.astype(_get_floatx()).T)


def filterbank_log(sample_rate: int, n_freq: int, n_bins: int = 84, bins_per_octave: int = 12,
                   f_min: Optional[float] = None, spread: float = 0.125) -> np.ndarray:
    """Log-frequency (constant-Q-like) filterbank of shape ``(n_freq, n_bins)``
    (kapre/backend.py:234-299): log-normal bumps around geometrically spaced centre
    frequencies, L1-normalised per band."""
    if f_min is None:
        f_min = 32.70319566
    f_max = f_min * 2 ** (n_bins / bins_per_octave)
    if f_max > sample_rate // 2:
        raise RuntimeError(
            'Maximum frequency of log filterbank should be lower or equal to the maximum'
            'frequency of the input (defined by its sample rate), '
            'but f_max=%f and maximum frequency is %f. \n'
            'Fix it by reducing n_bins, increasing bins_per_octave and/or reducing f_min.\n'
            'You can also do it by increasing sample_rate but it means you need to upsample'
            'the input audio data, too.' % (f_max, sample_rate))
    sigma = float(spread) / bins_per_octave
    log_bin = np.log2(np.fft.rfftfreq((int(n_freq) - 1) * 2, 1.0 / sample_rate)[1:])
    centres = np.log2(f_min) + np.arange(n_bins, dtype=np.float64) / bins_per_octave
    z = (log_bin[None, :] - centres[:, None]) / sigma
    basis = np.zeros((n_bins, int(n_freq)))
    basis[:, 1:] = np.exp(-0.5 * z * z - np.log2(sigma) - log_bin[None, :])
    l1 = np.abs(basis).sum(axis=1, keepdims=True)
    l1 = np.where(l1 < np.finfo(np.float64).tiny, 1.0, l1)
    return np.ascontiguousarray((basis / l1).astype(_get_floatx()).T)


BIQUAD_KINDS = ('lowpass', 'highpass', 'bandpass', 'bandreject', 'allpass', 'equalizer')


def biquad_coefficients(kind: str, sample_rate, freq, Q=0.707, gain=0.0):
    """(b, a): float64 arrays of shape (..., 3), not normalised, of torchaudio's biquad designs
    (``lowpass_biquad``, ``highpass_biquad``, ``bandpass_biquad`` with ``const_skirt_gain=False``,
    ``bandreject_biquad``, ``allpass_biquad``, ``equalizer_biquad``; the RBJ audio-EQ cookbook).  ``freq``, ``Q`` and
    ``gain`` (dB, equalizer only) may be arrays of one shape, which gives one filter per element."""
    if kind not in BIQUAD_KINDS:
        raise ValueError('kind must be one of %s, got: %r' % (BIQUAD_KINDS, kind))
    freq, Q, gain = np.broadcast_arrays(np.asarray(freq, np.float64), np.asarray(Q, np.float64),
                                        np.asarray(gain, np.float64))
    if not (np.isfinite(sample_rate) and sample_rate > 0):
        raise ValueError('sample_rate must be positive, got: %r' % (sample_rate,))
    if not (np.all(freq > 0) and np.all(freq < sample_rate / 2)):
        raise ValueError('freq must lie in (0, sample_rate / 2), got: %r' % (freq,))
    if not (np.all(Q > 0) and np.all(np.isfinite(Q))):
        raise ValueError('Q must be positive and finite, got: %r' % (Q,))
    if not np.all(np.isfinite(gain)):
        raise ValueError('gain must be finite, got: %r' % (gain,))
    w0 = 2 * np.pi * freq / sample_rate
    alpha = np.sin(w0) / 2 / Q
    c = np.cos(w0)
    one = np.ones_like(w0)
    a = [1 + alpha, -2 * c, 1 - alpha]
    if kind == 'lowpass':
        b = [(1 - c) / 2, 1 - c, (1 - c) / 2]
    elif kind == 'highpass':
        b = [(1 + c) / 2, -1 - c, (1 + c) / 2]
    elif kind == 'bandpass':
        b = [alpha, 0 * one, -alpha]
    elif kind == 'bandreject':
        b = [one, -2 * c, one]
    elif kind == 'allpass':
        b = [1 - alpha, -2 * c, 1 + alpha]
    else:
        A = np.exp(gain / 40.0 * np.log(10))
        b = [1 + alpha * A, -2 * c, 1 - alpha * A]
        a = [1 + alpha / A, -2 * c, 1 - alpha / A]
    return np.stack(b, -1), np.stack(a, -1)
