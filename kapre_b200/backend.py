"""Host-side mirror of ``kapre/backend.py`` for the hot path.

Same public names, argument meaning and error behaviour as the reference
(``kapre/backend.py``), but the constants are built with NumPy on the host
(the reference calls ``tf.signal.*_window`` / ``librosa.filters.mel``) and the tensor op
``magnitude_to_decibel`` runs as CUDA kernels through the C ABI.
"""
from __future__ import annotations

import math
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


def sos_steady_state(sos):
    """(zi, gain) of a second-order-section cascade ``sos`` (..., S, 6): zi (..., S, 2) is ``scipy.signal.sosfilt_zi``
    (each section's ``lfilter_zi``, the steady state of a unit step, scaled by the DC gain of the sections before it)
    and gain (...) the cascade's DC gain.  Float64 NumPy for host coefficients (normalised by a0, as scipy does);
    float64 torch on the tensor's device for a tensor, with a0 taken to be 1 and no synchronisation.  Closed form per
    biquad: with B1 = b1 - a1 b0, B2 = b2 - a2 b0, z1 = (B1 + B2) / (1 + a1 + a2) and z2 = B2 - a2 z1."""
    import torch
    if isinstance(sos, torch.Tensor):
        s = sos.detach().to(torch.float64)
        lib, stack, cat = torch, torch.stack, torch.cat
    else:
        s = np.asarray(sos, np.float64)
        s = s / s[..., 3:4]
        lib, stack, cat = np, np.stack, np.concatenate
    b0, b1, b2, a1, a2 = (s[..., k] for k in (0, 1, 2, 4, 5))
    den = 1.0 + a1 + a2
    z1 = (b1 - a1 * b0 + b2 - a2 * b0) / den
    z2 = b2 - a2 * b0 - a2 * z1
    g = (b0 + b1 + b2) / den
    before = lib.cumprod(cat([lib.ones_like(g[..., :1]), g[..., :-1]], -1), -1)     # DC gain ahead of each section
    return stack([z1 * before, z2 * before], -1), lib.prod(g, -1)


def sosfilt_zi(sos):
    """``scipy.signal.sosfilt_zi`` restated: the (..., S, 2) initial state of ``sosfilt`` that is the steady state of a
    unit step (``backend.sos_steady_state``).  Float64 NumPy for host coefficients, float64 torch on the device for a
    tensor (a0 is not read; nothing synchronises)."""
    return sos_steady_state(sos)[0]


def inverse_sabine(rt60, room, sound_speed=343.0):
    """The energy absorption ``alpha = 24 ln(10) V / (c S rt60)`` that gives a shoebox room (``room``: its three
    sides, metres) the reverberation time ``rt60`` (seconds) by Sabine's formula, with ``V`` its volume and ``S`` its
    wall area.  Raises ValueError when ``alpha > 1``: no absorption gives so short a reverberation in that room."""
    Lx, Ly, Lz = (float(v) for v in room)
    rt60, sound_speed = float(rt60), float(sound_speed)
    if not (min(Lx, Ly, Lz) > 0 and rt60 > 0 and sound_speed > 0 and np.isfinite([Lx, Ly, Lz, rt60, sound_speed]).all()):
        raise ValueError('room sides, rt60 and sound_speed must be finite and positive, got %r, %r, %r'
                         % (room, rt60, sound_speed))
    V, S = Lx * Ly * Lz, 2.0 * (Lx * Ly + Ly * Lz + Lx * Lz)
    alpha = 24.0 * np.log(10.0) * V / (sound_speed * S * rt60)
    if alpha > 1.0:
        raise ValueError('rt60 %g s is too short for a %g x %g x %g m room: absorption %g > 1' % (rt60, Lx, Ly, Lz, alpha))
    return alpha


def k_weighting_coefficients(sample_rate):
    """The two filters of ITU-R BS.1770's K-weighting as ``torchaudio.functional.loudness`` designs them: ((b, a) of
    ``treble_biquad(sample_rate, 4.0, 1500.0, 1 / sqrt(2))``, (b, a) of ``highpass_biquad(sample_rate, 38.0, 0.5)``),
    float64 arrays of length 3, not normalised.  ``sample_rate`` must be above 3000 Hz, so that the shelf's 1500 Hz lies
    below the Nyquist frequency."""
    if not (isinstance(sample_rate, (int, float, np.integer, np.floating)) and np.isfinite(sample_rate)
            and sample_rate > 3000):
        raise ValueError('sample_rate must be a number above 3000 Hz, got: %r' % (sample_rate,))
    w0 = 2 * np.pi * 1500.0 / sample_rate
    alpha = np.sin(w0) / 2 / (1 / np.sqrt(2))
    A = np.exp(4.0 / 40 * np.log(10))
    t1, t2, t3 = 2 * np.sqrt(A) * alpha, (A - 1) * np.cos(w0), (A + 1) * np.cos(w0)
    shelf = (np.array([A * ((A + 1) + t2 + t1), -2 * A * ((A - 1) + t3), A * ((A + 1) + t2 - t1)]),
             np.array([(A + 1) - t2 + t1, 2 * ((A - 1) - t3), (A + 1) - t2 - t1]))
    return shelf, biquad_coefficients('highpass', sample_rate, 38.0, 0.5)


# ------------------------------------------------------------------------------- Kaldi features
# Host constants of torchaudio.compliance.kaldi (2.11), restated in float64 NumPy: window properties and frame counts,
# the feature windows, the mel banks with VTLN warping, and the DCT with the cepstral lifter.
KALDI_WINDOWS = ('hamming', 'hanning', 'povey', 'rectangular', 'blackman')
KALDI_PADDED_SIZES = (256, 512, 1024, 2048)


def kaldi_window_properties(sample_frequency=16000.0, frame_shift=10.0, frame_length=25.0,
                            round_to_power_of_two=True):
    """(window_size, window_shift, padded_window_size) in samples, as torchaudio derives them from milliseconds."""
    shift = int(sample_frequency * frame_shift * 0.001)
    size = int(sample_frequency * frame_length * 0.001)
    padded = (1 if size == 0 else 2 ** (size - 1).bit_length()) if round_to_power_of_two else size
    return size, shift, padded


def kaldi_num_frames(length, window_size, window_shift, snip_edges=True, min_length=0):
    """Frames of an item of ``length`` samples (an int or an integer array): ``1 + (L - W) // shift`` with
    snip_edges, else ``(L + shift // 2) // shift``; 0 when ``L < W`` (torchaudio refuses such items) or
    ``L < min_length``."""
    L = np.asarray(length, dtype=np.int64)
    n = (1 + (L - window_size) // window_shift) if snip_edges else (L + window_shift // 2) // window_shift
    n = np.where((L < window_size) | (L < min_length) | (L <= 0), 0, n)
    return int(n) if n.ndim == 0 else n


def kaldi_window(window_type, window_size, blackman_coeff=0.42):
    """torchaudio's feature window of ``window_size`` samples (symmetric), float64."""
    n = np.arange(window_size, dtype=np.float64)
    if window_type in ('hanning', 'povey'):
        w = 0.5 - 0.5 * np.cos(2.0 * np.pi * n / (window_size - 1)) if window_size > 1 else np.ones(1)
        return w ** 0.85 if window_type == 'povey' else w
    if window_type == 'hamming':
        return 0.54 - 0.46 * np.cos(2.0 * np.pi * n / (window_size - 1)) if window_size > 1 else np.ones(1)
    if window_type == 'rectangular':
        return np.ones(window_size)
    if window_type == 'blackman':
        a = 2.0 * np.pi / (window_size - 1)
        return blackman_coeff - 0.5 * np.cos(a * n) + (0.5 - blackman_coeff) * np.cos(2.0 * a * n)
    raise ValueError('window_type must be one of %s, got %r' % (KALDI_WINDOWS, window_type))


def _kaldi_mel(f):
    return 1127.0 * np.log(1.0 + np.asarray(f, np.float64) / 700.0)


def _kaldi_inv_mel(m):
    return 700.0 * (np.exp(np.asarray(m, np.float64) / 1127.0) - 1.0)


def _kaldi_vtln_warp_freq(vtln_low, vtln_high, low_freq, high_freq, warp, freq):
    if not (vtln_low > low_freq and vtln_high < high_freq):
        raise ValueError('vtln_low must be above low_freq and vtln_high below high_freq')
    l = vtln_low * max(1.0, warp)
    h = vtln_high * min(1.0, warp)
    scale = 1.0 / warp
    fl, fh = scale * l, scale * h
    scale_left = (fl - low_freq) / (l - low_freq)
    scale_right = (high_freq - fh) / (high_freq - h)
    res = np.empty_like(freq)
    after_h, before_h, before_l = freq >= h, freq < h, freq < l
    outside = (freq < low_freq) | (freq > high_freq)
    res[after_h] = high_freq + scale_right * (freq[after_h] - high_freq)
    res[before_h] = scale * freq[before_h]
    res[before_l] = low_freq + scale_left * (freq[before_l] - low_freq)
    res[outside] = freq[outside]
    return res


def kaldi_mel_banks(num_bins, padded_window_size, sample_frequency, low_freq=20.0, high_freq=0.0, vtln_low=100.0,
                    vtln_high=-500.0, vtln_warp=1.0):
    """torchaudio's ``get_mel_banks`` in float64, with the zero Nyquist column: (num_bins, padded_window_size // 2 + 1).
    ``high_freq <= 0`` and ``vtln_high < 0`` are offsets from the Nyquist frequency."""
    if num_bins < 4:
        raise ValueError('num_mel_bins must be at least 4, got %r' % (num_bins,))
    nyquist = 0.5 * sample_frequency
    if high_freq <= 0.0:
        high_freq += nyquist
    if not (0.0 <= low_freq < nyquist and 0.0 < high_freq <= nyquist and low_freq < high_freq):
        raise ValueError('bad low_freq %r / high_freq %r for Nyquist %r' % (low_freq, high_freq, nyquist))
    if vtln_high < 0.0:
        vtln_high += nyquist
    if vtln_warp != 1.0 and not (low_freq < vtln_low < high_freq and 0.0 < vtln_high < high_freq
                                 and vtln_low < vtln_high):
        raise ValueError('bad vtln_low %r / vtln_high %r for low_freq %r / high_freq %r'
                         % (vtln_low, vtln_high, low_freq, high_freq))
    n_fft_bins = padded_window_size // 2
    mel_low, mel_high = _kaldi_mel(low_freq), _kaldi_mel(high_freq)
    delta = (mel_high - mel_low) / (num_bins + 1)
    b = np.arange(num_bins, dtype=np.float64)[:, None]
    left, center, right = mel_low + b * delta, mel_low + (b + 1.0) * delta, mel_low + (b + 2.0) * delta
    if vtln_warp != 1.0:
        def warp(m):
            return _kaldi_mel(_kaldi_vtln_warp_freq(vtln_low, vtln_high, low_freq, high_freq, vtln_warp,
                                                    _kaldi_inv_mel(m)))
        left, center, right = warp(left), warp(center), warp(right)
    mel = _kaldi_mel(sample_frequency / padded_window_size * np.arange(n_fft_bins, dtype=np.float64))[None, :]
    up = (mel - left) / (center - left)
    down = (right - mel) / (right - center)
    if vtln_warp == 1.0:
        banks = np.maximum(0.0, np.minimum(up, down))
    else:
        banks = np.zeros_like(up)
        ui = (mel > left) & (mel <= center)
        di = (mel > center) & (mel < right)
        banks[ui] = up[ui]
        banks[di] = down[di]
    return np.concatenate([banks, np.zeros((num_bins, 1))], axis=1)


def kaldi_dct(num_ceps, num_mel_bins, cepstral_lifter=22.0):
    """torchaudio's MFCC matrix (num_mel_bins, num_ceps), float64: the orthonormal DCT-II with the first column
    sqrt(1 / num_mel_bins), times the lifter ``1 + 0.5 L sin(pi i / L)`` (none when ``cepstral_lifter == 0``)."""
    n = np.arange(num_mel_bins, dtype=np.float64)[:, None]
    k = np.arange(num_ceps, dtype=np.float64)[None, :]
    d = np.cos(np.pi / num_mel_bins * (n + 0.5) * k) * np.sqrt(2.0 / num_mel_bins)
    d[:, 0] = np.sqrt(1.0 / num_mel_bins)
    if cepstral_lifter != 0.0:
        d = d * (1.0 + 0.5 * cepstral_lifter * np.sin(np.pi * np.arange(num_ceps) / cepstral_lifter))[None, :]
    return d


# ---- constant-Q transform ---------------------------------------------------------------------------------------
CQT_C1 = 32.70319566257483      # C1 in Hz, the default lowest bin
CQT_MAX_OCTAVES = 12            # octaves one launch covers (KAPRE_CQT_MAX_OCTAVES)
CQT_MAX_TAPS = 2048             # longest filter of an octave at its own rate (KAPRE_CQT_MAX_TAPS)
CQT_MAX_SEGMENTS = 256          # (octave, bin group) segments of one plan (KB_CQT_MAX_SEGS)
CQT_GROUP_BYTES = 32 * 1024     # a bin group's complex64 taps (KB_CQT_TAB_BYTES)


def cqt_segments(taps, octave_bins):
    """Forward (octave, bin group) segments of a plan whose octave i has ``octave_bins[i]`` bins and ``taps[i]`` taps
    per bin: groups of an even number of bins whose taps fit CQT_GROUP_BYTES, at most 256 bins (kb_cqt_fwd_group)."""
    n = 0
    for N, nk in zip(taps, octave_bins):
        gk = min((CQT_GROUP_BYTES // (8 * N)) & ~1, (nk + 1) & ~1, 256)
        n += -(-nk // gk)
    return n


def cqt_frequencies(n_bins: int, f_min: Optional[float] = None, bins_per_octave: int = 12) -> np.ndarray:
    """Centre frequencies ``f_k = f_min 2^(k / bins_per_octave)`` of the CQT bins, float64 (``f_min`` default C1)."""
    f_min = CQT_C1 if f_min is None else float(f_min)
    return f_min * 2.0 ** (np.arange(int(n_bins), dtype=np.float64) / int(bins_per_octave))


def cqt_geometry(sample_rate, hop_length, f_min=None, n_bins=84, bins_per_octave=12, filter_scale=1.0, gamma=0.0):
    """Validated geometry of a multirate CQT / VQT: dict with ``freqs``, ``lengths`` (the real full-rate filter
    lengths l_k = Q sr / (f_k + gamma / alpha)), ``alpha``, ``Q``, ``n_octaves`` and ``octaves``, a list of
    (first bin, end bin) per octave, top octave first.  Raises ValueError on a configuration the transform rejects."""
    for name, v in (('sample_rate', sample_rate), ('hop_length', hop_length), ('n_bins', n_bins),
                    ('bins_per_octave', bins_per_octave), ('filter_scale', filter_scale)):
        if isinstance(v, bool) or not np.isfinite(float(v)) or float(v) <= 0:
            raise ValueError('%s must be positive, got %r' % (name, v))
    for name, v in (('hop_length', hop_length), ('n_bins', n_bins), ('bins_per_octave', bins_per_octave)):
        if int(v) != v:
            raise ValueError('%s must be an integer, got %r' % (name, v))
    if f_min is not None and not (np.isfinite(float(f_min)) and float(f_min) > 0):
        raise ValueError('f_min must be positive, got %r' % (f_min,))
    if not (np.isfinite(float(gamma)) and float(gamma) >= 0):
        raise ValueError('gamma must be >= 0, got %r' % (gamma,))
    sr, h, n, B = float(sample_rate), int(hop_length), int(n_bins), int(bins_per_octave)
    freqs = cqt_frequencies(n, f_min, B)
    r = 2.0 ** (1.0 / B)
    alpha = (r * r - 1.0) / (r * r + 1.0)
    Q = float(filter_scale) / alpha
    n_oct = -(-n // B)
    f_max = freqs[-1]
    edge = f_max + (alpha * f_max + float(gamma)) / 2.0
    if edge >= sr / 2.0:
        raise ValueError('the top band edge %.1f Hz (f_max + (alpha f_max + gamma) / 2) is at or above the Nyquist '
                         'frequency %.1f Hz: reduce n_bins or f_min' % (edge, sr / 2.0))
    if n_oct > CQT_MAX_OCTAVES:
        raise ValueError('%d octaves exceed the kernel limit of %d octaves per transform' % (n_oct, CQT_MAX_OCTAVES))
    if h % (1 << (n_oct - 1)):
        raise ValueError('hop_length %d must be a multiple of 2^(n_octaves - 1) = %d for %d octaves'
                         % (h, 1 << (n_oct - 1), n_oct))
    lengths = Q * sr / (freqs + float(gamma) / alpha)
    octaves = [(max(0, n - (i + 1) * B), n - i * B) for i in range(n_oct)]
    for i, (k0, _) in enumerate(octaves):
        N = int(np.ceil(lengths[k0] / 2.0 ** i))
        if N > CQT_MAX_TAPS:
            raise ValueError('the filter of bin %d is %d taps long at octave %d\'s rate, over the kernel limit of %d '
                             'taps: raise f_min, n_bins or sample_rate, or lower filter_scale' % (k0, N, i, CQT_MAX_TAPS))
    taps = [int(np.ceil(lengths[k0] / 2.0 ** i)) for i, (k0, _) in enumerate(octaves)]
    segs = cqt_segments(taps, [k1 - k0 for k0, k1 in octaves])
    if segs > CQT_MAX_SEGMENTS:
        raise ValueError('%d (octave, bin group) segments exceed the kernel limit of %d (a group holds the bins whose '
                         'taps fit %d bytes): lower bins_per_octave or filter_scale' % (segs, CQT_MAX_SEGMENTS,
                                                                                       CQT_GROUP_BYTES))
    return dict(freqs=freqs, lengths=lengths, alpha=alpha, Q=Q, n_octaves=n_oct, octaves=octaves)


def cqt_filters(sample_rate, f_min=None, n_bins=84, bins_per_octave=12, filter_scale=1.0, gamma=0.0, scale=True):
    """Per-octave complex128 tap tables of the multirate CQT, top octave first.  Octave i's table T has shape
    (bins in the octave, N_i) with N_i = ceil(l_k0 / 2^i) the length of its longest (lowest) filter, and
        T[k, j] = s_k conj(psi_k[j - N_i // 2]),   psi_k[n] = w[n + N // 2] exp(2 pi i f_k n / sr_i) / sum(w)
    for n in [-(N // 2), N - N // 2), N = ceil(l_k / 2^i), w the periodic Hann window of N points, 0 elsewhere;
    s_k = sqrt(l_k) with ``scale``, else l_k.  Then C[k, m] = sum_j y_i[m h_i + j - N_i // 2] T[k, j]."""
    g = cqt_geometry(sample_rate, 1 << (-(-int(n_bins) // int(bins_per_octave)) - 1), f_min, n_bins,
                     bins_per_octave, filter_scale, gamma)
    sr = float(sample_rate)
    out = []
    for i, (k0, k1) in enumerate(g['octaves']):
        sr_i = sr / 2.0 ** i
        Ni = int(np.ceil(g['lengths'][k0] / 2.0 ** i))
        half = Ni // 2
        T = np.zeros((k1 - k0, Ni), dtype=np.complex128)
        for kk, k in enumerate(range(k0, k1)):
            lk = g['lengths'][k]
            N = int(np.ceil(lk / 2.0 ** i))
            j = np.arange(N, dtype=np.float64)
            w = 0.5 - 0.5 * np.cos(2.0 * np.pi * j / N)
            nn = j - N // 2
            psi = w * np.exp(2j * np.pi * g['freqs'][k] * nn / sr_i) / w.sum()
            s = np.sqrt(lk) if scale else lk
            T[kk, half - N // 2:half - N // 2 + N] = s * np.conj(psi)
        out.append(T)
    return out


# ---- pitch tracking (YIN / pYIN) --------------------------------------------------------------------------------
PITCH_MAX_FRAME = 8192          # KAPRE_PITCH_MAX_FRAME: the staged frame and its CMNDF fit one CTA
PITCH_MAX_THRESHOLDS = 1024     # KAPRE_PITCH_MAX_THRESHOLDS
PITCH_MAX_BINS = 8192           # KAPRE_PITCH_MAX_BINS: the Viterbi scores of 2 n_pitch states fit shared memory
PITCH_MAX_BAND = 8192           # KAPRE_PITCH_MAX_BAND
PITCH_TINY = 2.0 ** -126


def _positive(name, v, integer=False):
    if isinstance(v, bool) or not np.isfinite(float(v)) or float(v) <= 0:
        raise ValueError('%s must be positive, got %r' % (name, v))
    if integer and int(v) != v:
        raise ValueError('%s must be an integer, got %r' % (name, v))


def pitch_geometry(sample_rate, fmin, fmax, frame_length=2048, win_length=None, hop_length=None, center=True):
    """Validated framing of YIN / pYIN: dict with ``frame_length``, ``win_length``, ``hop_length``, ``pad`` (leading
    zeros), ``min_period = floor(sr / fmax)``, ``max_period = min(ceil(sr / fmin), frame_length - win_length - 1)``
    and ``n_lags``.  Raises ValueError on a configuration the kernels reject."""
    _positive('sample_rate', sample_rate)
    _positive('frame_length', frame_length, True)
    F = int(frame_length)
    W = F // 2 if win_length is None else win_length
    h = F // 4 if hop_length is None else hop_length
    _positive('win_length', W, True)
    _positive('hop_length', h, True)
    W, h = int(W), int(h)
    for name, v in (('fmin', fmin), ('fmax', fmax)):
        if isinstance(v, bool) or not np.isfinite(float(v)):
            raise ValueError('%s must be finite, got %r' % (name, v))
    sr, fmin, fmax = float(sample_rate), float(fmin), float(fmax)
    if fmin <= 0:
        raise ValueError('fmin must be positive, got %r' % fmin)
    if fmin >= fmax:
        raise ValueError('fmin %r must be below fmax %r' % (fmin, fmax))
    if fmax > sr / 2:
        raise ValueError('fmax %r is above the Nyquist frequency %r' % (fmax, sr / 2))
    if not isinstance(center, (bool, np.bool_)):
        raise ValueError('center must be a bool, got %r' % (center,))
    if W >= F:
        raise ValueError('win_length %d must be below frame_length %d' % (W, F))
    if F > PITCH_MAX_FRAME:
        raise ValueError('frame_length %d exceeds the kernel limit of %d samples' % (F, PITCH_MAX_FRAME))
    min_p = int(np.floor(sr / fmax))
    max_p = min(int(np.ceil(sr / fmin)), F - W - 1)
    if min_p < 1:
        raise ValueError('min_period floor(sr / fmax) = %d is below 1' % min_p)
    if max_p - min_p + 1 < 3:
        raise ValueError('the lag range [%d, %d] holds fewer than 3 lags: lower fmin or win_length, raise fmax or '
                         'frame_length' % (min_p, max_p))
    return dict(frame_length=F, win_length=W, hop_length=h, pad=F // 2 if center else 0, center=bool(center),
                min_period=min_p, max_period=max_p, n_lags=max_p - min_p + 1, sample_rate=sr, fmin=fmin, fmax=fmax)


def beta_cdf(x, a, b):
    """Regularised incomplete beta function I_x(a, b) in float64 (the Beta(a, b) CDF), by the continued fraction of
    the incomplete beta function (modified Lentz), on the side where it converges fast."""
    x = np.asarray(x, dtype=np.float64)
    a, b = float(a), float(b)
    lbeta = math.lgamma(a) + math.lgamma(b) - math.lgamma(a + b)

    def cf(x, a, b):
        tiny = 1e-300
        c, d = 1.0, 1.0 - (a + b) * x / (a + 1.0)
        d = 1.0 / (d if abs(d) > tiny else tiny)
        f = d
        for m in range(1, 10000):
            m2 = 2 * m
            num = m * (b - m) * x / ((a + m2 - 1.0) * (a + m2))
            for k in (0, 1):
                d = 1.0 + num * d
                d = 1.0 / (d if abs(d) > tiny else tiny)
                c = 1.0 + num / c
                c = c if abs(c) > tiny else tiny
                f *= c * d
                if k == 0:
                    num = -(a + m) * (a + b + m) * x / ((a + m2) * (a + m2 + 1.0))
            if abs(c * d - 1.0) < 1e-16:
                break
        return f

    out = np.empty(x.shape, dtype=np.float64)
    for idx, v in np.ndenumerate(x):
        v = float(v)
        if v <= 0.0:
            out[idx] = 0.0
        elif v >= 1.0:
            out[idx] = 1.0
        else:
            front = math.exp(a * math.log(v) + b * math.log1p(-v) - lbeta)
            if v < (a + 1.0) / (a + b + 2.0):
                out[idx] = front * cf(v, a, b) / a
            else:
                out[idx] = 1.0 - front * cf(1.0 - v, b, a) / b
    return out


def triangle_window(w):
    """``scipy.signal.windows.triang(w)`` (symmetric) in numpy."""
    w = int(w)
    n = np.arange(1, (w + 1) // 2 + 1, dtype=np.float64)
    half = 2.0 * n / (w + 1.0) if w % 2 else (2.0 * n - 1.0) / w
    return np.concatenate([half, half[-2::-1]]) if w % 2 else np.concatenate([half, half[::-1]])


def pyin_geometry(geometry, n_thresholds=100, beta_parameters=(2, 18), boltzmann_parameter=2, resolution=0.1,
                  max_transition_rate=35.92, switch_prob=0.01, no_trough_prob=0.01):
    """pYIN's sizes on top of ``pitch_geometry``: ``bins_per_semitone = ceil(1 / resolution)``, ``n_pitch``, the
    transition band width ``band_width = round(max_transition_rate 12 h / sr) bins_per_semitone + 1`` and ``n_states
    = 2 n_pitch``.  Raises ValueError on parameters the kernels reject."""
    _positive('n_thresholds', n_thresholds, True)
    _positive('resolution', resolution)
    _positive('max_transition_rate', max_transition_rate)
    _positive('boltzmann_parameter', boltzmann_parameter)
    if len(beta_parameters) != 2:
        raise ValueError('beta_parameters must be a pair, got %r' % (beta_parameters,))
    for v in beta_parameters:
        _positive('beta_parameters', v)
    for name, v in (('switch_prob', switch_prob), ('no_trough_prob', no_trough_prob)):
        if isinstance(v, bool) or not (0.0 <= float(v) <= 1.0):
            raise ValueError('%s must lie in [0, 1], got %r' % (name, v))
    if resolution >= 1:
        raise ValueError('resolution must be below 1 semitone, got %r' % (resolution,))
    if int(n_thresholds) > PITCH_MAX_THRESHOLDS:
        raise ValueError('%d thresholds exceed the kernel limit of %d' % (n_thresholds, PITCH_MAX_THRESHOLDS))
    g = geometry
    bps = int(np.ceil(1.0 / float(resolution)))
    n_pitch = int(np.floor(12 * bps * np.log2(g['fmax'] / g['fmin']))) + 1
    band = int(np.round(float(max_transition_rate) * 12 * g['hop_length'] / g['sample_rate'])) * bps + 1
    if 2 * n_pitch > 65535:
        raise ValueError('%d HMM states exceed the 65535 that uint16 backpointers address' % (2 * n_pitch))
    if n_pitch > PITCH_MAX_BINS:
        raise ValueError('%d pitch bins exceed the kernel limit of %d: raise resolution or narrow [fmin, fmax]'
                         % (n_pitch, PITCH_MAX_BINS))
    if band > PITCH_MAX_BAND:
        raise ValueError('a transition band of %d bins exceeds the kernel limit of %d' % (band, PITCH_MAX_BAND))
    return dict(n_thresholds=int(n_thresholds), beta_parameters=tuple(float(v) for v in beta_parameters),
                boltzmann_parameter=float(boltzmann_parameter), bins_per_semitone=bps, n_pitch=n_pitch,
                band_width=band, n_states=2 * n_pitch, switch_prob=float(switch_prob),
                no_trough_prob=float(no_trough_prob))


def pyin_tables(geometry, pyin):
    """float64 tables of pYIN (see kapre_pitch_tables in include/kapre_b200.h) as a dict of arrays."""
    g, q = geometry, pyin
    nt = q['n_thresholds']
    cdf = beta_cdf(np.arange(nt + 1, dtype=np.float64) / nt, *q['beta_parameters'])
    beta = np.diff(cdf)
    cmax = (g['n_lags'] + 1) // 2
    lam = q['boltzmann_parameter']
    r = np.arange(cmax + 1, dtype=np.float64)
    bpow = np.exp(-lam * r)
    bnorm = np.zeros(cmax + 1)
    bnorm[1:] = -np.expm1(-lam) / -np.expm1(-lam * r[1:])
    bonus = q['no_trough_prob'] * np.concatenate([[0.0], np.cumsum(beta)])
    B = 12 * q['bins_per_semitone']
    m = np.arange(q['n_pitch'], dtype=np.float64)
    freqs = g['fmin'] * 2.0 ** (m / B)
    edges = g['sample_rate'] / (g['fmin'] * 2.0 ** ((m[:-1] + 0.5) / B))
    w = q['band_width']
    tri = triangle_window(w)
    n = q['n_pitch']
    rows = np.zeros(n)
    for i in range(n):
        j0, j1 = max(0, i - w // 2), min(n, i - w // 2 + w)
        rows[i] = tri[j0 - i + w // 2:j1 - i + w // 2].sum()
    return dict(beta_probs=beta, boltzmann_pow=bpow, boltzmann_norm=bnorm, no_trough_bonus=bonus,
                period_edges=edges, freqs=freqs, log_triangle=np.log(tri), log_row_norm=-np.log(rows))


# ---- chroma -----------------------------------------------------------------------------------------------------------
CHROMA_MAX_CHROMA = 64          # KAPRE_CHROMA_MAX_CHROMA
CHROMA_MAX_NFFT = 8192          # n_fft / 2 + 1 <= KAPRE_CHROMA_MAX_BINS
CHROMA_MAX_TUNING_BINS = 1000   # KAPRE_CHROMA_MAX_TUNING_BINS
CHROMA_MAX_SMOOTH = 512         # win_len_smooth + 2 <= KAPRE_CHROMA_MAX_SMOOTH
CHROMA_NORMS = {None: 0, np.inf: 1, 1: 2, 2: 3}   # KAPRE_CHROMA_NORM_*


def chroma_norm_code(norm):
    """``norm`` (``inf``, 1, 2 or None) as the library's normalisation code; ValueError otherwise."""
    if norm is None:
        return 0
    if isinstance(norm, bool) or not isinstance(norm, (int, float, np.integer, np.floating)):
        raise ValueError('norm must be inf, 1, 2 or None, got %r' % (norm,))
    if float(norm) == np.inf:
        return 1
    if float(norm) in (1.0, 2.0):
        return 2 if float(norm) == 1.0 else 3
    raise ValueError('norm must be inf, 1, 2 or None, got %r' % (norm,))


def _check_n_chroma(n_chroma):
    if isinstance(n_chroma, bool) or int(n_chroma) != n_chroma or not 1 <= int(n_chroma) <= CHROMA_MAX_CHROMA:
        raise ValueError('n_chroma must be an integer in [1, %d], got %r' % (CHROMA_MAX_CHROMA, n_chroma))
    return int(n_chroma)


def _check_n_fft(n_fft):
    if isinstance(n_fft, bool) or int(n_fft) != n_fft or not 2 <= int(n_fft) <= CHROMA_MAX_NFFT:
        raise ValueError('n_fft must be an integer in [2, %d], got %r' % (CHROMA_MAX_NFFT, n_fft))
    return int(n_fft)


def chroma_filterbank(sample_rate, n_fft, n_chroma=12, tuning=0.0, ctroct=5.0, octwidth=2.0, base_c=True):
    """librosa's ``filters.chroma``: the float64 (n_chroma, n_fft // 2 + 1) weights of the STFT bins per pitch class.
    Gaussian bumps around each pitch class (2 D / binwidth), each column of unit L2 norm, then weighted by a Gaussian
    over octaves centred on ``ctroct`` of width ``octwidth`` (none when None), rows rolled so that C comes first with
    ``base_c``.  ``tuning`` is in fractions of a chroma bin: A440 becomes 440 2^(tuning / n_chroma)."""
    n_chroma = _check_n_chroma(n_chroma)
    n_fft = _check_n_fft(n_fft)
    sr = float(sample_rate)
    if not (np.isfinite(sr) and sr > 0):
        raise ValueError('sample_rate must be positive, got %r' % (sample_rate,))
    if not np.isfinite(float(tuning)):
        raise ValueError('tuning must be finite, got %r' % (tuning,))
    f = np.linspace(0, sr, n_fft, endpoint=False)[1:]
    a440 = 440.0 * 2.0 ** (float(tuning) / n_chroma)
    frqbins = n_chroma * np.log2(f / (a440 / 16.0))
    frqbins = np.concatenate(([frqbins[0] - 1.5 * n_chroma], frqbins))
    binwidth = np.concatenate((np.maximum(frqbins[1:] - frqbins[:-1], 1.0), [1.0]))
    D = np.subtract.outer(frqbins, np.arange(0, n_chroma, dtype='d')).T
    half = np.round(float(n_chroma) / 2)
    D = np.remainder(D + half + 10 * n_chroma, n_chroma) - half
    wts = np.exp(-0.5 * (2 * D / np.tile(binwidth, (n_chroma, 1))) ** 2)
    wts = wts / np.sqrt(np.sum(wts ** 2, axis=0, keepdims=True))
    if octwidth is not None:
        wts = wts * np.tile(np.exp(-0.5 * (((frqbins / n_chroma - float(ctroct)) / float(octwidth)) ** 2)),
                            (n_chroma, 1))
    if base_c:
        wts = np.roll(wts, -3 * (n_chroma // 12), axis=0)
    return np.ascontiguousarray(wts[:, :n_fft // 2 + 1], dtype=np.float64)


def hz_to_midi(f):
    return 12.0 * (np.log2(np.asarray(f, dtype=np.float64)) - np.log2(440.0)) + 69.0


def cq_to_chroma(n_input, bins_per_octave=12, n_chroma=12, f_min=None, base_c=True):
    """librosa's ``filters.cq_to_chroma`` (without ``window``): the float64 (n_chroma, n_input) 0/1 matrix that merges
    ``bins_per_octave / n_chroma`` adjacent CQT bins into each chroma, rolled so that the bin of ``f_min`` (default C1)
    lands on its pitch class (C first with ``base_c``, else A).  ValueError unless ``bins_per_octave`` is a multiple
    of ``n_chroma``."""
    n_chroma = _check_n_chroma(n_chroma)
    n_input, bpo = int(n_input), int(bins_per_octave)
    if bpo < 1 or n_input < 1:
        raise ValueError('n_input and bins_per_octave must be positive')
    if bpo % n_chroma:
        raise ValueError('bins_per_octave=%d must be an integer multiple of n_chroma=%d' % (bpo, n_chroma))
    n_merge = bpo // n_chroma
    f_min = CQT_C1 if f_min is None else float(f_min)
    m = np.repeat(np.eye(n_chroma), n_merge, axis=1)
    m = np.roll(m, -int(n_merge // 2), axis=1)
    m = np.tile(m, int(np.ceil(float(n_input) / bpo)))[:, :n_input]
    midi0 = np.mod(hz_to_midi(f_min), 12)
    roll = int(np.round((midi0 - (0 if base_c else 9)) * (n_chroma / 12.0)))
    return np.ascontiguousarray(np.roll(m, roll, axis=0), dtype=np.float64)


def tuning_edges(resolution=0.01):
    """The residual histogram edges of ``estimate_tuning``: ``linspace(-0.5, 0.5, ceil(1 / resolution) + 1)``;
    ValueError unless 0 < resolution <= 1 with at most CHROMA_MAX_TUNING_BINS bins."""
    r = float(resolution)
    if isinstance(resolution, bool) or not (np.isfinite(r) and 0.0 < r <= 1.0):
        raise ValueError('resolution must be in (0, 1], got %r' % (resolution,))
    n = int(np.ceil(1.0 / r))
    if n > CHROMA_MAX_TUNING_BINS:
        raise ValueError('resolution %r gives %d histogram bins, over the limit of %d' % (resolution, n,
                                                                                        CHROMA_MAX_TUNING_BINS))
    return np.linspace(-0.5, 0.5, n + 1)


def piptrack_bins(sample_rate, n_fft, fmin=150.0, fmax=4000.0):
    """[lo, hi): the STFT bins piptrack searches, ``fmin <= f_k < min(fmax, sr / 2)`` with librosa's
    ``fft_frequencies`` (``numpy.fft.rfftfreq``)."""
    sr = float(sample_rate)
    f = np.fft.rfftfreq(int(n_fft), 1.0 / sr)
    k = np.nonzero((fmin <= f) & (f < min(float(fmax), sr / 2.0)))[0]
    if k.size == 0:
        return 1, 1
    return max(int(k[0]), 1), min(int(k[-1]) + 1, int(n_fft) // 2)


def cens_window(win_len_smooth=41):
    """The CENS smoothing taps ``hann(win_len_smooth + 2, symmetric) / sum`` (float64); None or 0: the single tap 1."""
    if win_len_smooth is None or win_len_smooth == 0:
        return np.ones(1)
    if isinstance(win_len_smooth, bool) or int(win_len_smooth) != win_len_smooth or not \
            1 <= int(win_len_smooth) <= CHROMA_MAX_SMOOTH:
        raise ValueError('win_len_smooth must be None or an integer in [0, %d], got %r'
                         % (CHROMA_MAX_SMOOTH, win_len_smooth))
    n = int(win_len_smooth) + 2
    w = 0.5 - 0.5 * np.cos(2.0 * np.pi * np.arange(n) / (n - 1))
    return w / w.sum()
