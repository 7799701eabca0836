"""Augmentation layers (reference: kapre/augmentation.py).  ``SpecAugment``: the masks are drawn on the host, the
masking is one CUDA pass (``kapre_spec_augment``).  ``TimeStretch``: a phase vocoder, one CUDA scan over time
(``kapre_time_stretch``).  ``PitchShift``: STFT, that phase vocoder, the inverse STFT and one band-limited
interpolation (``kapre_sinc_resample``) back to the input length.  ``Reverb``: convolution with a room impulse response
drawn from a bank (``kapre_convolve``).  ``RandomBiquad``: a biquad drawn per item (``kapre_lfilter``).
``BackgroundNoise``: a noise excerpt from a bank added at a drawn SNR (``kapre_add_noise``).  ``LoudnessNormalization``:
a gain to a drawn loudness target (``kapre_lfilter`` and ``kapre_loudness``).  ``RoomReverb``: convolution with a room
impulse response simulated per item (``kapre_rir_ism`` and ``kapre_convolve``)."""
from __future__ import annotations

import math

import numpy as np
import torch

from . import _native as N
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


def prepare_rirs(rirs) -> np.ndarray:
    """The room impulse responses of a ``Reverb`` bank, prepared in float64 as the torchaudio augmentation tutorial
    does by hand: each one trimmed to start at its largest-magnitude sample (the direct path), scaled to unit L2
    norm, and zero-padded to the longest.  ``rirs``: a 2-D array or a sequence of 1-D arrays of any lengths.
    Returns an (n_rirs, K) float32 array; an empty bank, or an all-zero or non-finite response, raises."""
    if isinstance(rirs, np.ndarray) and rirs.ndim == 2:
        rows = list(rirs)
    elif isinstance(rirs, np.ndarray) and rirs.ndim != 2:
        raise ValueError('rirs must be a 2-D array or a list of 1-D arrays, got an array of shape %s' % (rirs.shape,))
    else:
        try:
            rows = list(rirs)
        except TypeError:
            raise ValueError('rirs must be a 2-D array or a list of 1-D arrays, got: %r' % (type(rirs),)) from None
    if not rows:
        raise ValueError('rirs is empty')
    out = []
    for i, r in enumerate(rows):
        r = np.asarray(r.detach().cpu() if hasattr(r, 'detach') else r, dtype=np.float64)
        if r.ndim != 1 or r.size == 0:
            raise ValueError('rir %d must be a non-empty 1-D array, got shape %s' % (i, r.shape))
        if not np.all(np.isfinite(r)):
            raise ValueError('rir %d has non-finite samples' % i)
        r = r[int(np.argmax(np.abs(r))):]
        norm = np.sqrt(np.sum(r * r))
        if not norm > 0:
            raise ValueError('rir %d is all zeros' % i)
        out.append(r / norm)
    bank = np.zeros((len(out), max(r.size for r in out)), np.float64)
    for i, r in enumerate(out):
        bank[i, :r.size] = r
    return bank.astype(np.float32)


@register_keras_serializable(package='Kapre')
class Reverb(Layer):
    """Reverberation by a bank of room impulse responses (the RIR step of speed perturbation -> reverberation ->
    noise recipes): ``(batch, time, ch)`` / ``(batch, ch, time)`` in, the same shape out,
    ``y[t] = sum_k h'[k] x[t - k]`` for ``t < time`` with ``h'`` the drawn response after ``prepare_rirs`` (trimmed
    to its direct path, unit L2 norm), so the output is time-aligned with the direct path.  Every channel of an item
    gets the same response.

    ``call(x, rir_index=None)`` draws one response per item, uniformly with ``np.random.default_rng(seed)``, and
    records the draw in ``last_choice``; an int or an array of ``batch`` indices overrides the draw.  The layer
    applies on every call, like ``Speed`` and ``PitchShift`` (``Sequential`` passes no ``training`` flag); a
    captured graph (``Sequential.capture``) replays the draw made when it was captured.

    The bank's block spectra are computed on first use on a device and kept; a call gathers the drawn items' spectra
    and runs ``kapre_convolve`` (three launches).  The gradient reaches ``x`` only: the bank is a constant, like a
    window or a filterbank."""

    def __init__(self, rirs, seed=None, data_format='default', **kwargs):
        super().__init__(**kwargs)
        backend.validate_data_format_str(data_format)
        data_format = _unwrap_format(data_format)
        self.bank = prepare_rirs(rirs)
        self.seed = seed
        self.rng = np.random.default_rng(seed)
        self.last_choice = None
        self.data_format_original = data_format
        self.data_format = _resolve(data_format)
        self.plan = ops.convolve_plan(ops.convolve_block_size(self.bank.shape[1]))
        self._spectra = {}

    def spectra(self, device):
        """(n_rirs, 1, P, B + 1) complex64 block spectra of the bank on ``device``, made on first use."""
        key = device.index if device.index is not None else torch.cuda.current_device()
        H = self._spectra.get(key)
        if H is None:
            with torch.cuda.device(device):
                h = torch.from_numpy(self.bank).to(device).unsqueeze(1)
                H = self._spectra[key] = ops.convolve_ir_spectrum(h, self.plan, _CH_FIRST_STR)
        return H

    def _choice(self, batch, rir_index):
        n = self.bank.shape[0]
        if rir_index is None:
            return self.rng.integers(0, n, size=batch)
        idx = np.asarray(rir_index)
        if idx.dtype.kind not in 'iu' or idx.ndim > 1 or (idx.ndim == 1 and idx.shape[0] != batch):
            raise ValueError('rir_index must be an int or %d ints, got: %r' % (batch, rir_index))
        if np.any(idx < 0) or np.any(idx >= n):
            raise ValueError('rir_index must lie in [0, %d), got: %r' % (n, rir_index))
        return np.broadcast_to(idx, (batch,)).astype(np.int64)

    def call(self, x, rir_index=None):
        if x.dim() != 3:
            raise ValueError('Reverb expects a 3-D batch, got shape %s' % (tuple(x.shape),))
        if not x.is_cuda:
            raise N.KapreNativeError('Reverb needs a CUDA tensor')
        choice = self._choice(x.shape[0], rir_index)
        self.last_choice = choice
        length = x.shape[2] if self.data_format == _CH_FIRST_STR else x.shape[1]
        if x.shape[0] == 0 or length == 0:
            return x.float().clone()
        H = self.spectra(x.device)
        if np.all(choice == choice[0]):
            H = H[int(choice[0]):int(choice[0]) + 1]          # one response: broadcast it, no gather
        elif torch.cuda.is_current_stream_capturing():
            H = torch.stack([H[int(i)] for i in choice])       # device-to-device only, so it can be captured
        else:
            H = H.index_select(0, torch.from_numpy(choice).to(x.device))
        return ops.convolve_spectrum(x, H, self.plan, 0, length, self.data_format)

    def get_config(self):
        config = super().get_config()
        config.update({'rirs': self.bank.tolist(), 'seed': self.seed, 'data_format': self.data_format_original})
        return config


@register_keras_serializable(package='Kapre')
class RandomBiquad(Layer):
    """A random biquad per item (filter augmentation): ``kind`` one of ``backend.BIQUAD_KINDS``; per item the
    frequency is drawn log-uniformly from ``freq_range`` (Hz, inside (0, sample_rate / 2)), ``Q`` uniformly from
    ``Q_range`` and, for the equalizer, ``gain`` (dB) uniformly from ``gain_range``, with
    ``np.random.default_rng(seed)``.  ``(batch, time, ch)`` / ``(batch, ch, time)`` in, the same shape out; every
    channel of an item gets the item's filter, and the output is clamped to [-1, 1] as torchaudio's biquads do.

    The coefficients are designed and normalised in float64 on the host and passed as one ``(batch, 1, 3)`` pair, so
    a call is one ``kapre_lfilter`` (four launches).  ``last_choice`` records the draw as ``(freq, Q, gain)`` arrays.
    The layer applies on every call (``Sequential`` passes no ``training`` flag); a captured graph
    (``Sequential.capture``) replays the draw made when it was captured.  The gradient reaches the input."""

    def __init__(self, kind, sample_rate, freq_range, Q_range=(0.707, 0.707), gain_range=(0.0, 0.0), seed=None,
                 data_format='default', **kwargs):
        super().__init__(**kwargs)
        backend.validate_data_format_str(data_format)
        data_format = _unwrap_format(data_format)
        if kind not in backend.BIQUAD_KINDS:
            raise ValueError('kind must be one of %s, got: %r' % (backend.BIQUAD_KINDS, kind))
        ranges = []
        for name, r in (('freq_range', freq_range), ('Q_range', Q_range), ('gain_range', gain_range)):
            r = tuple(float(v) for v in r)
            if len(r) != 2 or not (np.isfinite(r[0]) and np.isfinite(r[1])) or r[0] > r[1]:
                raise ValueError('%s must be a (low, high) pair of finite numbers, got: %r' % (name, r))
            ranges.append(r)
        # the ends of each range must make valid filters (biquad_coefficients checks them)
        backend.biquad_coefficients(kind, sample_rate, [ranges[0][0], ranges[0][1]], [ranges[1][0], ranges[1][1]],
                                    [ranges[2][0], ranges[2][1]])
        self.kind, self.sample_rate = kind, sample_rate
        self.freq_range, self.Q_range, self.gain_range = ranges
        self.seed = seed
        self.rng = np.random.default_rng(seed)
        self.last_choice = None
        self.data_format_original = data_format
        self.data_format = _resolve(data_format)
        self._captured = []

    def draw(self, batch):
        """(freq, Q, gain) arrays of ``batch`` draws, in that order from the layer's generator."""
        lo, hi = np.log(self.freq_range[0]), np.log(self.freq_range[1])
        freq = np.exp(self.rng.uniform(lo, hi, size=batch))
        Q = self.rng.uniform(self.Q_range[0], self.Q_range[1], size=batch)
        gain = self.rng.uniform(self.gain_range[0], self.gain_range[1], size=batch)
        return freq, Q, gain

    def call(self, x):
        if x.dim() != 3:
            raise ValueError('RandomBiquad expects a 3-D batch, got shape %s' % (tuple(x.shape),))
        if not x.is_cuda:
            raise N.KapreNativeError('RandomBiquad needs a CUDA tensor')
        freq, Q, gain = self.draw(x.shape[0])
        self.last_choice = (freq, Q, gain)
        b, a = backend.biquad_coefficients(self.kind, self.sample_rate, freq, Q, gain)
        host = torch.from_numpy(np.stack([b / a[:, :1], a / a[:, :1]]).astype(np.float32)).reshape(2, -1, 1, 3)
        if torch.cuda.is_current_stream_capturing():
            # the graph's copy node reads this pinned buffer on every replay: it is kept and never written again
            host = host.pin_memory()
            self._captured.append(host)
        coef = host.to(x.device, non_blocking=True)
        from .signal import lfilter
        return lfilter(x, coef[1], coef[0], clamp=True, data_format=self.data_format)

    def get_config(self):
        config = super().get_config()
        config.update({'kind': self.kind, 'sample_rate': self.sample_rate, 'freq_range': list(self.freq_range),
                       'Q_range': list(self.Q_range), 'gain_range': list(self.gain_range), 'seed': self.seed,
                       'data_format': self.data_format_original})
        return config


def _range_pair(name, r, positive=True):
    r = tuple(float(v) for v in r)
    if len(r) != 2 or not (np.isfinite(r[0]) and np.isfinite(r[1])) or r[0] > r[1] or (positive and not r[0] > 0):
        raise ValueError('%s must be a (low, high) pair of finite%s numbers, got: %r'
                         % (name, ' positive' if positive else '', r))
    return r


@register_keras_serializable(package='Kapre')
class RoomReverb(Layer):
    """Reverberation by a room simulated per item with the image-source method: ``(batch, time, ch)`` /
    ``(batch, ch, time)`` in, the same shape out, ``y[t] = sum_k h[k] x[t - k]`` for ``t < time``, every channel of an
    item convolved with the item's response (``Reverb``'s contract, with the response simulated instead of drawn).

    Each call draws, per item in turn, with ``np.random.default_rng(seed)``: the three room sides, each uniform in
    its ``room_range``; the RT60, uniform in ``rt60_range``; the source and then the mic, uniform in the room shrunk by
    ``wall_margin`` on every side, the mic drawn again from the same generator while it is closer than
    ``min_distance`` to the source.  ``last_choice = (room, rt60, source, mic)`` records the draw.  All six walls
    absorb ``backend.inverse_sabine(rt60, room)``.

    The response is ``rir_length`` samples (default ``ceil(rt60_range[1] * sample_rate)``) of
    ``signal.simulate_rir_ism`` (``max_order``, ``delay_filter_length``) starting at ``round(tau) + half``, the sample
    nearest the direct path's peak (``tau = |source - mic| sample_rate / 343``, ``half = (delay_filter_length - 1) /
    2``), scaled to unit L2 norm by a float64 sum in a fixed order.  A call is ``kapre_rir_ism`` with that scaling (two
    launches), the response's block spectra and ``kapre_convolve`` (four).  The gradient reaches ``x`` through the
    convolution's; a captured graph (``Sequential.capture``) replays the draw made when it was captured.

    Construction raises ValueError when a corner of the ranges needs an absorption above 1, when ``min_distance`` is
    more than half the diagonal of the smallest room inside the margins, or when the longest response in the smallest
    room could exceed ``simulate_rir_ism``'s image cap."""

    def __init__(self, sample_rate, room_range=((3, 10), (3, 10), (2.5, 4)), rt60_range=(0.2, 0.8), wall_margin=0.5,
                 min_distance=0.5, max_order=None, rir_length=None, delay_filter_length=81, seed=None,
                 data_format='default', **kwargs):
        super().__init__(**kwargs)
        backend.validate_data_format_str(data_format)
        data_format = _unwrap_format(data_format)
        if not (np.isfinite(float(sample_rate)) and float(sample_rate) > 0):
            raise ValueError('sample_rate must be finite and positive, got: %r' % (sample_rate,))
        if len(room_range) != 3:
            raise ValueError('room_range must hold three (low, high) pairs, got: %r' % (room_range,))
        self.room_range = tuple(_range_pair('room_range', r) for r in room_range)
        self.rt60_range = _range_pair('rt60_range', rt60_range)
        self.wall_margin, self.min_distance = float(wall_margin), float(min_distance)
        if not (self.wall_margin > 0 and self.min_distance > 0):
            raise ValueError('wall_margin and min_distance must be positive, got %r and %r' % (wall_margin, min_distance))
        inner = np.array([r[0] for r in self.room_range]) - 2 * self.wall_margin
        # two uniform points of a box lie at least half its diagonal apart with a probability of about 0.2 or more
        # (1/4 on a segment), so the mic's redraw ends quickly
        if not (np.all(inner > 0) and self.min_distance <= 0.5 * np.sqrt(np.sum(inner ** 2))):
            raise ValueError('the smallest room %s cannot hold a wall margin of %g m and a source-mic distance of %g m '
                             '(at most half the diagonal inside the margins)'
                             % ([r[0] for r in self.room_range], self.wall_margin, self.min_distance))
        for corner in np.ndindex(2, 2, 2):
            backend.inverse_sabine(self.rt60_range[0], [self.room_range[d][corner[d]] for d in range(3)])
        if max_order is not None and (isinstance(max_order, bool) or not isinstance(max_order, (int, np.integer))
                                      or max_order < 0):
            raise ValueError('max_order must be None or a non-negative int, got: %r' % (max_order,))
        self.sample_rate = float(sample_rate)
        self.max_order = max_order
        self.delay_filter_length = int(delay_filter_length)
        if not (1 <= self.delay_filter_length <= 255 and self.delay_filter_length % 2 == 1):
            raise ValueError('delay_filter_length must be an odd int from 1 to 255, got: %r' % (delay_filter_length,))
        self.rir_length = int(math.ceil(self.rt60_range[1] * self.sample_rate)) if rir_length is None else int(rir_length)
        if self.rir_length < 1:
            raise ValueError('rir_length must be >= 1, got: %r' % (rir_length,))
        self._rir_length_arg = rir_length
        # the image cap of kapre_rir_ism, for the longest arrival time in the smallest room: the response ends at most
        # (largest room's inner diagonal + c rir_length / fs) plus the filter's half away from the direct path, and
        # per axis at most R / L + 2 lattice boxes meet a ball of radius R
        far = np.sqrt(np.sum((np.array([r[1] for r in self.room_range]) - 2 * self.wall_margin) ** 2))
        t_end = math.floor(far * self.sample_rate / 343.0 + 0.5) + (self.delay_filter_length - 1) // 2 + self.rir_length
        R = t_end * 343.0 / self.sample_rate
        bound = 8.0 * np.prod([R / r[0] + 2.0 for r in self.room_range])
        if bound > ops.RIR_MAX_IMAGES:
            raise ValueError('rir_length %d in the smallest room %s may need up to %.3g images, above the cap of %d'
                             % (self.rir_length, [r[0] for r in self.room_range], bound, ops.RIR_MAX_IMAGES))
        self.seed = seed
        self.rng = np.random.default_rng(seed)
        self.last_choice = None
        self.data_format_original = data_format
        self.data_format = _resolve(data_format)
        self.plan = ops.convolve_plan(ops.convolve_block_size(self.rir_length))
        self._captured = []

    MAX_REDRAWS = 1000

    def draw(self, batch):
        """(room, rt60, source, mic) arrays of ``batch`` draws, in the documented order.  A mic that is still too
        close after ``MAX_REDRAWS`` redraws raises ValueError (construction keeps that far less likely than 1e-90)."""
        lo = np.array([r[0] for r in self.room_range])
        hi = np.array([r[1] for r in self.room_range])
        room, rt60 = np.zeros((batch, 3)), np.zeros(batch)
        source, mic = np.zeros((batch, 3)), np.zeros((batch, 3))
        m = self.wall_margin
        for b in range(batch):
            room[b] = self.rng.uniform(lo, hi)
            rt60[b] = self.rng.uniform(self.rt60_range[0], self.rt60_range[1])
            source[b] = self.rng.uniform(m, room[b] - m)
            mic[b] = self.rng.uniform(m, room[b] - m)
            redraws = 0
            while np.sqrt(np.sum((mic[b] - source[b]) ** 2)) < self.min_distance:
                if redraws == self.MAX_REDRAWS:
                    raise ValueError('no mic at least %g m from the source after %d redraws in room %s'
                                     % (self.min_distance, redraws, room[b]))
                mic[b] = self.rng.uniform(m, room[b] - m)
                redraws += 1
        return room, rt60, source, mic

    def records(self, room, rt60, source, mic, sound_speed=343.0):
        """The ``kapre_rir_ism`` records of a draw: (B, 14) items, each starting at its direct path's peak."""
        B = room.shape[0]
        rec = np.zeros((B, ops.RIR_RECORD), np.float64)
        rec[:, 0:3], rec[:, 3:6] = room, source
        for b in range(B):
            rec[b, 6:12] = np.sqrt(1.0 - backend.inverse_sabine(rt60[b], room[b], sound_speed))
        rec[:, 12] = -1.0 if self.max_order is None else float(self.max_order)
        tau = np.sqrt(np.sum((source - mic) ** 2, axis=1)) * self.sample_rate / sound_speed
        rec[:, 13] = np.floor(tau + 0.5) + (self.delay_filter_length - 1) // 2
        return rec

    def call(self, x):
        if x.dim() != 3:
            raise ValueError('RoomReverb expects a 3-D batch, got shape %s' % (tuple(x.shape),))
        if not x.is_cuda:
            raise N.KapreNativeError('RoomReverb needs a CUDA tensor')
        room, rt60, source, mic = self.draw(x.shape[0])
        self.last_choice = (room, rt60, source, mic)
        length = x.shape[2] if self.data_format == _CH_FIRST_STR else x.shape[1]
        if x.shape[0] == 0 or length == 0:
            return x.float().clone()
        with torch.cuda.device(x.device):
            h = ops.rir_ism(self.records(room, rt60, source, mic), mic[:, None, :], self.rir_length,
                            self.delay_filter_length, self.sample_rate, 343.0, _CH_FIRST_STR, unit_norm=True,
                            keep=self._captured)
            H = ops.convolve_ir_spectrum(h, self.plan, _CH_FIRST_STR)
        return ops.convolve_spectrum(x, H, self.plan, 0, length, self.data_format)

    def get_config(self):
        config = super().get_config()
        config.update({'sample_rate': self.sample_rate, 'room_range': [list(r) for r in self.room_range],
                       'rt60_range': list(self.rt60_range), 'wall_margin': self.wall_margin,
                       'min_distance': self.min_distance, 'max_order': self.max_order,
                       'rir_length': self._rir_length_arg, 'delay_filter_length': self.delay_filter_length,
                       'seed': self.seed, 'data_format': self.data_format_original})
        return config


def prepare_noises(noises):
    """The clips of a ``BackgroundNoise`` bank: ``noises`` is a 2-D array or a sequence of 1-D arrays of any lengths,
    each non-empty, finite and not all zero (they are not rescaled: the SNR sets the level).  Returns the clips
    concatenated as float32 and their lengths (int64)."""
    if isinstance(noises, np.ndarray) and noises.ndim == 2:
        rows = list(noises)
    elif isinstance(noises, (np.ndarray, str, bytes)):
        raise ValueError('noises must be a 2-D array or a list of 1-D arrays, got: %r' % (type(noises),))
    else:
        try:
            rows = list(noises)
        except TypeError:
            raise ValueError('noises must be a 2-D array or a list of 1-D arrays, got: %r' % (type(noises),)) from None
    if not rows:
        raise ValueError('noises is empty')
    out = []
    for i, r in enumerate(rows):
        r = np.asarray(r.detach().cpu() if hasattr(r, 'detach') else r)
        if r.dtype.kind not in 'iuf' or r.ndim != 1 or r.size == 0:
            raise ValueError('noise %d must be a non-empty 1-D array of numbers, got shape %s' % (i, r.shape))
        r = r.astype(np.float32)
        if not np.all(np.isfinite(r)):
            raise ValueError('noise %d has non-finite samples' % i)
        if not np.any(r != 0):
            raise ValueError('noise %d is all zeros' % i)
        out.append(r)
    return np.concatenate(out), np.array([r.size for r in out], np.int64)


@register_keras_serializable(package='Kapre')
class BackgroundNoise(Layer):
    """Background noise from a bank of clips at a random SNR (the noise step of speed perturbation -> reverberation ->
    noise recipes, as with MUSAN): ``(batch, time, ch)`` / ``(batch, ch, time)`` in, the same shape out.  Item b gets
    ``add_noise(x_b, n_b, snr_b)`` with ``n_b[t] = clip[(offset + t) mod len(clip)]`` for every channel, so a clip
    shorter than the signal loops; the SNR is measured per channel, as ``signal.add_noise`` does, and a silent
    excerpt leaves the item as it is.

    ``call(x, noise_index=None, offset=None, snr=None, lengths=None)`` draws per item, in this order and with
    ``np.random.default_rng(seed)``: the clips (uniformly), the offsets (uniformly in ``[0, len(clip))``) and the
    SNRs (uniformly in ``snr_range``, dB).  Each argument (a number or ``batch`` values) replaces its draw, which is
    then not made; ``lengths`` is passed to ``add_noise``.  ``last_choice = (index, offset, snr)`` records what was
    applied.  The layer applies on every call, like ``Reverb``; a captured graph (``Sequential.capture``) replays
    the draw made when it was captured.

    The bank is uploaded on first use on a device and kept.  A call sends the per-item clip starts, lengths, offsets
    and SNRs in one host-to-device copy and runs ``kapre_add_noise`` in bank mode (two launches): nothing is gathered.
    The gradient reaches ``x`` only: the bank is a constant."""

    def __init__(self, noises, snr_range=(0.0, 20.0), seed=None, data_format='default', **kwargs):
        super().__init__(**kwargs)
        backend.validate_data_format_str(data_format)
        data_format = _unwrap_format(data_format)
        self.bank, self.clip_len = prepare_noises(noises)
        self.clip_start = np.concatenate([[0], np.cumsum(self.clip_len)[:-1]]).astype(np.int64)
        r = tuple(float(v) for v in snr_range)
        if len(r) != 2 or not (np.isfinite(r[0]) and np.isfinite(r[1])) or r[0] > r[1]:
            raise ValueError('snr_range must be a (low, high) pair of finite numbers, got: %r' % (snr_range,))
        self.snr_range = r
        self.seed = seed
        self.rng = np.random.default_rng(seed)
        self.last_choice = None
        self.data_format_original = data_format
        self.data_format = _resolve(data_format)
        self._banks = {}
        self._captured = []

    def clips(self):
        """The clips as a list of float32 arrays."""
        return [self.bank[s:s + n] for s, n in zip(self.clip_start, self.clip_len)]

    def bank_on(self, device):
        """The flat bank on ``device``, uploaded on first use."""
        key = device.index if device.index is not None else torch.cuda.current_device()
        t = self._banks.get(key)
        if t is None:
            t = self._banks[key] = torch.from_numpy(self.bank).to(device)
        return t

    @staticmethod
    def _override(name, v, batch, kind):
        a = np.asarray(v)
        if a.dtype.kind not in kind or a.ndim > 1 or (a.ndim == 1 and a.shape[0] != batch):
            raise ValueError('%s must be a number or %d numbers, got: %r' % (name, batch, v))
        return np.broadcast_to(a, (batch,)).copy()

    def draw(self, batch, noise_index=None, offset=None, snr=None):
        """(index, offset, snr) arrays of ``batch`` items: drawn in that order, or the validated overrides."""
        n = len(self.clip_len)
        if noise_index is None:
            idx = self.rng.integers(0, n, size=batch)
        else:
            idx = self._override('noise_index', noise_index, batch, 'iu').astype(np.int64)
            if np.any(idx < 0) or np.any(idx >= n):
                raise ValueError('noise_index must lie in [0, %d), got: %r' % (n, noise_index))
        if offset is None:
            off = self.rng.integers(0, self.clip_len[idx])
        else:
            off = self._override('offset', offset, batch, 'iu').astype(np.int64)
            if np.any(off < 0) or np.any(off >= self.clip_len[idx]):
                raise ValueError('offset must lie in [0, clip length), got: %r' % (offset,))
        if snr is None:
            s = self.rng.uniform(self.snr_range[0], self.snr_range[1], size=batch)
        else:
            s = self._override('snr', snr, batch, 'iuf').astype(np.float64)
            if not np.all(np.isfinite(s)):
                raise ValueError('snr must be finite, got: %r' % (snr,))
        return idx, np.asarray(off, np.int64), s

    def call(self, x, noise_index=None, offset=None, snr=None, lengths=None):
        if x.dim() != 3:
            raise ValueError('BackgroundNoise expects a 3-D batch, got shape %s' % (tuple(x.shape),))
        if not x.is_cuda:
            raise N.KapreNativeError('BackgroundNoise needs a CUDA tensor')
        B = x.shape[0]
        idx, off, s = self.draw(B, noise_index, offset, snr)
        self.last_choice = (idx, off, s)
        # one host buffer, one copy: rows start, clip length, offset, and the SNRs as float32 in the last row
        host = torch.empty((4, B), dtype=torch.int64)
        host[0] = torch.from_numpy(self.clip_start[idx])
        host[1] = torch.from_numpy(self.clip_len[idx])
        host[2] = torch.from_numpy(off)
        host[3].view(torch.float32)[:B] = torch.from_numpy(s.astype(np.float32))
        if torch.cuda.is_current_stream_capturing():
            # the graph's copy node reads this pinned buffer on every replay: it is kept and never written again
            host = host.pin_memory()
            self._captured.append(host)
        dev = host.to(x.device, non_blocking=True)
        snr_d = dev[3].view(torch.float32)[:B].view(B, 1)
        bank = (self.bank_on(x.device), dev[0], dev[1], dev[2])
        return ops.add_noise(x, None, snr_d, lengths, self.data_format, bank=bank)

    def get_config(self):
        config = super().get_config()
        config.update({'noises': [c.tolist() for c in self.clips()], 'snr_range': list(self.snr_range),
                       'seed': self.seed, 'data_format': self.data_format_original})
        return config


@register_keras_serializable(package='Kapre')
class LoudnessNormalization(Layer):
    """Loudness normalisation to a target per item (EBU R128's -23 LUFS, streaming's -14, or a random target per
    example): ``(batch, time, ch)`` / ``(batch, ch, time)`` in (ch <= 5), the same shape out, each item scaled by
    ``10^((target - L) / 20)`` with L its BS.1770 loudness (``signal.loudness``).  Items whose L is not finite
    (silent, shorter than one 400 ms block, or with a non-finite sample) come back unchanged.

    ``true_peak_limit`` (dBTP, default None) caps the gain so that the output's true peak stays at or below it, as EBU
    R128 pairs a loudness target with a true-peak ceiling (for example -1 dBTP): the gain is then
    ``min(10^((target - L) / 20), 10^((limit - TP) / 20))`` with TP the item's largest ``signal.true_peak`` over its
    channels.  The true peak is linear in the waveform, so the output's is at most the limit up to float32 rounding;
    an item the limit binds lands below its loudness target.  Only the gain scales: the waveform's shape is kept.  The
    gradient follows whichever term is smaller, as ``torch.minimum``'s does.  With None the layer runs as if the
    argument did not exist.

    ``call(x, lufs=None, lengths=None)`` draws the targets uniformly from ``lufs_range`` with
    ``np.random.default_rng(seed)``; ``lufs`` (a number or ``batch`` values) replaces the draw, which is then not made.
    ``lengths`` is passed to ``loudness``.  ``last_choice`` records the targets.  The gain is formed on the device with
    no sync; a captured graph (``Sequential.capture``) replays the draw made when it was captured.  The gradient
    reaches ``x``, through the gain as well."""

    def __init__(self, sample_rate, lufs_range=(-23.0, -23.0), seed=None, data_format='default', true_peak_limit=None,
                 **kwargs):
        super().__init__(**kwargs)
        backend.validate_data_format_str(data_format)
        data_format = _unwrap_format(data_format)
        backend.k_weighting_coefficients(sample_rate)           # validates the rate
        r = tuple(float(v) for v in lufs_range)
        if len(r) != 2 or not (np.isfinite(r[0]) and np.isfinite(r[1])) or r[0] > r[1]:
            raise ValueError('lufs_range must be a (low, high) pair of finite numbers, got: %r' % (lufs_range,))
        if true_peak_limit is not None:
            if isinstance(true_peak_limit, bool) or not isinstance(true_peak_limit, (int, float, np.integer, np.floating)) \
                    or not np.isfinite(true_peak_limit):
                raise ValueError('true_peak_limit must be a finite number of dBTP or None, got: %r' % (true_peak_limit,))
            true_peak_limit = float(true_peak_limit)
        self.true_peak_limit = true_peak_limit
        self.sample_rate = sample_rate
        self.lufs_range = r
        self.seed = seed
        self.rng = np.random.default_rng(seed)
        self.last_choice = None
        self.data_format_original = data_format
        self.data_format = _resolve(data_format)
        self._captured = []

    def draw(self, batch, lufs=None):
        """``batch`` targets in LUFS: drawn, or the validated override."""
        if lufs is None:
            return self.rng.uniform(self.lufs_range[0], self.lufs_range[1], size=batch)
        t = BackgroundNoise._override('lufs', lufs, batch, 'iuf').astype(np.float64)
        if not np.all(np.isfinite(t)):
            raise ValueError('lufs must be finite, got: %r' % (lufs,))
        return t

    def call(self, x, lufs=None, lengths=None):
        if x.dim() != 3:
            raise ValueError('LoudnessNormalization expects a 3-D batch, got shape %s' % (tuple(x.shape),))
        if not x.is_cuda:
            raise N.KapreNativeError('LoudnessNormalization needs a CUDA tensor')
        B = x.shape[0]
        target = self.draw(B, lufs)
        self.last_choice = target
        host = torch.from_numpy(target.astype(np.float32))
        if torch.cuda.is_current_stream_capturing():
            # the graph's copy node reads this pinned buffer on every replay: it is kept and never written again
            host = host.pin_memory()
            self._captured.append(host)
        t = host.to(x.device, non_blocking=True)
        L = ops.loudness(x, self.sample_rate, lengths, self.data_format)
        # a non-finite L gives the exponent 0 (gain 1), and no gradient flows into it
        finite = torch.isfinite(L)
        L = torch.where(finite, L, t)
        if self.true_peak_limit is None:
            gain = torch.pow(10.0, (t - L) / 20.0)
        else:
            # the item's largest channel true peak; items left unchanged get the limit itself (exponent 0, no gradient)
            tp = ops.true_peak(x, lengths, self.data_format).amax(dim=1)
            tp = torch.where(finite, tp, torch.full_like(tp, self.true_peak_limit))
            gain = torch.pow(10.0, torch.minimum(t - L, self.true_peak_limit - tp) / 20.0)
        return x * gain.view(B, 1, 1)

    def get_config(self):
        config = super().get_config()
        config.update({'sample_rate': self.sample_rate, 'lufs_range': list(self.lufs_range), 'seed': self.seed,
                       'data_format': self.data_format_original, 'true_peak_limit': self.true_peak_limit})
        return config
