"""Drop-in mirrors of the hot-path layers of ``kapre/time_frequency.py``.

``STFT``, ``InverseSTFT``, ``Magnitude``, ``Phase``, ``MagnitudeToDecibel`` and
``ApplyFilterbank`` keep the reference's constructor signatures, defaults, validation order
and ``get_config()`` keys (kapre/time_frequency.py:61-559), but ``call`` runs
hand-written sm_90a CUDA through the C ABI instead of ``tf.signal``.

Keras is not a dependency: ``Layer`` below is the minimal part of the Keras layer protocol the
reference relies on (``__call__`` -> ``call``, ``name``, ``get_config`` / ``from_config``).
Inputs may be NumPy arrays or CPU tensors (copied to the current CUDA device, result returned
as NumPy, like ``model.predict``) or CUDA tensors (result stays on the device).
"""
from __future__ import annotations

import itertools
import math

import numpy as np
import torch

from . import _native as N
from . import backend, ops
from .backend import _CH_DEFAULT_STR, _CH_FIRST_STR, _CH_LAST_STR

__all__ = ['Layer', 'STFT', 'InverseSTFT', 'Magnitude', 'Phase', 'MagnitudeToDecibel', 'ApplyFilterbank', 'Delta',
           'PCEN', 'GriffinLim', 'InverseFilterbank', 'KaldiFbank', 'KaldiMFCC', 'KaldiSpectrogram', 'CQT',
           'ChromaSTFT', 'ChromaCQT', 'ChromaCENS', 'HPSS', 'OnsetStrength', 'Tempogram']

_name_counters = {}
_REGISTRY = {}


def register_keras_serializable(package='Kapre'):
    """Same registration key as the reference ('Kapre>ClassName', time_frequency.py:60)."""

    def deco(cls):
        _REGISTRY['%s>%s' % (package, cls.__name__)] = cls
        cls._registered_name = '%s>%s' % (package, cls.__name__)
        return cls

    return deco


def get_registered_object(name):
    return _REGISTRY.get(name)


def _auto_name(cls_name):
    # keras-style snake_case auto names: stft, stft_1, ...
    snake = ''.join(('_' + c.lower()) if c.isupper() and i and not cls_name[i - 1].isupper() else c.lower()
                    for i, c in enumerate(cls_name))
    c = _name_counters.setdefault(snake, itertools.count())
    i = next(c)
    return snake if i == 0 else '%s_%d' % (snake, i)


class Layer:
    """The slice of ``keras.layers.Layer`` the kapre layers use."""

    def __init__(self, name=None, trainable=True, dtype=None, input_shape=None, **kwargs):
        kwargs.pop('batch_input_shape', None)
        kwargs.pop('batch_size', None)
        if kwargs:
            raise TypeError('Unrecognized keyword arguments passed to %s: %s' % (type(self).__name__, kwargs))
        self.name = name if name is not None else _auto_name(type(self).__name__)
        self.trainable = trainable
        self.dtype = dtype or backend._get_floatx()
        self.input_shape_arg = input_shape
        self.built = True

    # -- tensor plumbing ----------------------------------------------------------------
    def __call__(self, x, *args, **kwargs):
        kwargs.pop('training', None)
        t, was_host = ops.to_device(x)
        if was_host:        # host in, NumPy out (like predict): nothing to record for autograd
            with torch.no_grad():
                y = self.call(t, *args, **kwargs)
        else:
            y = self.call(t, *args, **kwargs)
        if was_host and isinstance(y, torch.Tensor):
            return ops.to_host(y)
        return y

    def call(self, x):  # pragma: no cover - abstract
        raise NotImplementedError

    @property
    def weights(self):
        return []

    def count_params(self):
        return 0

    # -- serialisation ------------------------------------------------------------------
    # constructor keywords a subclass reports in get_config(): (config key, attribute holding the value)
    _config_fields = ()

    def get_config(self):
        config = {'name': self.name, 'trainable': self.trainable, 'dtype': self.dtype}
        for key, attr in self._config_fields:
            config[key] = getattr(self, attr)
        return config

    @classmethod
    def from_config(cls, config):
        return cls(**config)


def _unwrap_format(fmt):
    # kapre/time_frequency.py:118-124: workaround for dict-wrapped strings from Keras deserialisation
    return fmt['config'] if isinstance(fmt, dict) else fmt


def _resolve(fmt):
    return backend.image_data_format() if fmt == _CH_DEFAULT_STR else fmt


@register_keras_serializable(package='Kapre')
class STFT(Layer):
    """Short-time Fourier transform layer (reference: kapre/time_frequency.py:61-203).

    ``(batch, time, ch)`` / ``(batch, ch, time)`` float32 waveforms ->
    complex64 ``(batch, time, freq, ch)`` / ``(batch, ch, time, freq)``.
    Semantics of ``tf.signal.stft`` as kapre calls it: frames of ``win_length`` every
    ``hop_length`` samples, window from ``window_name``, right zero-pad to ``n_fft``, one-sided
    FFT; ``pad_begin`` prepends ``n_fft - hop_length`` zeros (sic, :169-172), ``pad_end`` pads
    the tail so that ``ceil(len / hop)`` frames come out.
    """

    def __init__(self, n_fft=2048, win_length=None, hop_length=None, window_name=None, pad_begin=False,
                 pad_end=False, input_data_format='default', output_data_format='default', **kwargs):
        super().__init__(**kwargs)
        for data_format in (input_data_format, output_data_format):
            backend.validate_data_format_str(data_format)  # raises before the dict unwrap, like :115-116
        input_data_format = _unwrap_format(input_data_format)
        output_data_format = _unwrap_format(output_data_format)
        if win_length is None:
            win_length = n_fft
        if hop_length is None:
            hop_length = win_length // 4  # :128-129
        self.n_fft = n_fft
        self.win_length = win_length
        self.hop_length = hop_length
        self.window_name = window_name
        self.window_fn = backend.get_window_fn(window_name)
        self.pad_begin = pad_begin
        self.pad_end = pad_end
        self.input_data_format_original = input_data_format
        self.output_data_format_original = output_data_format
        self.output_data_format = _resolve(output_data_format)
        self.input_data_format = _resolve(input_data_format)
        self._plan = None

    @property
    def plan(self) -> ops.StftPlan:
        if self._plan is None:
            self._plan = ops.StftPlan(self.n_fft, self.win_length, self.hop_length,
                                      self.window_fn(self.win_length))
        return self._plan

    def call(self, x):
        return ops.stft_forward(x, self.plan, self.input_data_format, self.output_data_format,
                                self.pad_begin, self.pad_end, N.OUT_COMPLEX)

    _config_fields = (
        ('n_fft', 'n_fft'),
        ('win_length', 'win_length'),
        ('hop_length', 'hop_length'),
        ('window_name', 'window_name'),
        ('pad_begin', 'pad_begin'),
        ('pad_end', 'pad_end'),
        ('input_data_format', 'input_data_format_original'),
        ('output_data_format', 'output_data_format_original'),
    )


@register_keras_serializable(package='Kapre')
class InverseSTFT(Layer):
    """Inverse STFT layer (reference: kapre/time_frequency.py:207-333).

    complex64 ``(batch, time, freq, ch)`` / ``(batch, ch, time, freq)`` -> float32 waveform of
    length ``(frames - 1) * hop_length + win_length`` (not trimmed, :213-214): irfft(n_fft),
    first ``win_length`` samples, times the dual of ``forward_window_name``
    (``tf.signal.inverse_stft_window_fn``, :278-280), overlap-add.
    """

    def __init__(self, n_fft=2048, win_length=None, hop_length=None, forward_window_name=None,
                 input_data_format='default', output_data_format='default', **kwargs):
        super().__init__(**kwargs)
        for data_format in (input_data_format, output_data_format):
            backend.validate_data_format_str(data_format)
        input_data_format = _unwrap_format(input_data_format)
        output_data_format = _unwrap_format(output_data_format)
        if win_length is None:
            win_length = n_fft
        if hop_length is None:
            hop_length = win_length // 4
        self.n_fft = n_fft
        self.win_length = win_length
        self.hop_length = hop_length
        self.forward_window_name = forward_window_name
        self.window_fn = backend.inverse_stft_window_fn(
            frame_step=hop_length, forward_window_fn=backend.get_window_fn(forward_window_name))
        self.input_data_format_original = input_data_format
        self.output_data_format_original = output_data_format
        self.output_data_format = _resolve(output_data_format)
        self.input_data_format = _resolve(input_data_format)
        self._plan = None

    @property
    def plan(self) -> ops.IstftPlan:
        if self._plan is None:
            self._plan = ops.IstftPlan(self.n_fft, self.win_length, self.hop_length,
                                       self.window_fn(self.win_length))
        return self._plan

    def call(self, x):
        return ops.istft(x, self.plan, self.input_data_format, self.output_data_format)

    _config_fields = (
        ('n_fft', 'n_fft'),
        ('win_length', 'win_length'),
        ('hop_length', 'hop_length'),
        ('forward_window_name', 'forward_window_name'),
        ('input_data_format', 'input_data_format_original'),
        ('output_data_format', 'output_data_format_original'),
    )


@register_keras_serializable(package='Kapre')
class Magnitude(Layer):
    """``tf.abs`` of the complex input (reference: kapre/time_frequency.py:337-359)."""

    def call(self, x):
        return ops.magnitude(x)


@register_keras_serializable(package='Kapre')
class Phase(Layer):
    """``tf.math.angle`` of the complex input (reference: kapre/time_frequency.py:363-411).
    ``approx_atan_accuracy`` (the TFLite-compatible approximation) is accepted and stored for
    config round trips; the exact angle is returned either way."""

    def __init__(self, approx_atan_accuracy=None, **kwargs):
        super().__init__(**kwargs)
        self.approx_atan_accuracy = approx_atan_accuracy

    def call(self, x):
        return ops.phase(x)

    _config_fields = (('approx_atan_accuracy', 'approx_atan_accuracy'),)


@register_keras_serializable(package='Kapre')
class MagnitudeToDecibel(Layer):
    """Decibel scaling (reference: kapre/time_frequency.py:415-465 -> backend.py:126-194).
    Parameters are validated when the layer is called, like the reference."""

    def __init__(self, ref_value=1.0, amin=1e-5, dynamic_range=80.0, **kwargs):
        super().__init__(**kwargs)
        self.ref_value = ref_value
        self.amin = amin
        self.dynamic_range = dynamic_range

    def call(self, x):
        return backend.magnitude_to_decibel(x, ref_value=self.ref_value, amin=self.amin,
                                            dynamic_range=self.dynamic_range)

    _config_fields = (('amin', 'amin'), ('dynamic_range', 'dynamic_range'), ('ref_value', 'ref_value'))


@register_keras_serializable(package='Kapre')
class ApplyFilterbank(Layer):
    """Apply a (n_freq, n_filterbanks) filterbank along the frequency axis
    (reference: kapre/time_frequency.py:469-559).  ``type`` is ``'mel'`` or ``'log'``; any other
    value leaves ``self.filterbank`` undefined, as in the reference (:519-522)."""

    def __init__(self, type, filterbank_kwargs, data_format='default', **kwargs):
        super().__init__(**kwargs)
        backend.validate_data_format_str(data_format)
        data_format = _unwrap_format(data_format)
        self.type = type
        self.filterbank_kwargs = filterbank_kwargs
        if type == 'log':
            self.filterbank = backend.filterbank_log(**filterbank_kwargs)
        elif type == 'mel':
            self.filterbank = backend.filterbank_mel(**filterbank_kwargs)
        self.data_format_original = data_format
        self.data_format = _resolve(data_format)
        self.freq_axis = 3 if self.data_format == _CH_FIRST_STR else 2
        self._fb = None

    @property
    def fb(self) -> ops.Filterbank:
        if self._fb is None:
            self._fb = ops.Filterbank(np.asarray(self.filterbank))
        return self._fb

    def call(self, x):
        return ops.apply_filterbank(x, self.fb, self.data_format)

    _config_fields = (
        ('type', 'type'),
        ('filterbank_kwargs', 'filterbank_kwargs'),
        ('data_format', 'data_format_original'),
    )


@register_keras_serializable(package='Kapre')
class Delta(Layer):
    """Local estimate of the time derivative (reference: kapre/time_frequency.py:563-644):
    ``sum_{m=-n..n} m * x[t+m] / (2 * sum_{m=1..n} m^2)`` with ``n = (win_length - 1) // 2`` on the time
    axis, the input extended by ``mode`` ('symmetric', 'reflect' or 'constant', as ``tf.pad``)."""

    def __init__(self, win_length=5, mode='symmetric', data_format='default', **kwargs):
        super().__init__(**kwargs)
        backend.validate_data_format_str(data_format)
        data_format = _unwrap_format(data_format)
        if not win_length >= 3:
            raise ValueError('win_length should be equal or bigger than 3, but it is %d' % win_length)
        if win_length % 2 != 1:
            raise ValueError('win_length should be an odd number, but it is %d' % win_length)
        if mode.lower() not in ('symmetric', 'reflect', 'constant'):
            raise ValueError('mode.lower() should be one of %sbut it is %s'
                             % (str(('symmetric', 'reflect', 'constant')), mode))
        self.data_format_original = data_format
        self.data_format = _resolve(data_format)
        self.win_length = win_length
        self.mode = mode
        self.n = (self.win_length - 1) // 2
        self.denom = 2 * sum([_n ** 2 for _n in range(1, self.n + 1, 1)])

    def call(self, x):
        return ops.delta(x, self.win_length, self.mode, self.data_format)

    _config_fields = (('win_length', 'win_length'), ('mode', 'mode'), ('data_format', 'data_format_original'))


@register_keras_serializable(package='Kapre')
class ConcatenateFrequencyMap(Layer):
    """Adds a frequency-information channel: ``linspace(0, 1, n_freq)`` along the frequency axis, broadcast over batch
    and time, concatenated on the channel axis (reference: kapre/time_frequency.py:648-744)."""

    def __init__(self, data_format='default', **kwargs):
        super().__init__(**kwargs)
        backend.validate_data_format_str(data_format)
        data_format = _unwrap_format(data_format)
        self.data_format_original = data_format
        self.data_format = _resolve(data_format)

    def call(self, x):
        return ops.concat_frequency_map(x, self.data_format)

    _config_fields = (('data_format', 'data_format_original'),)



def _pcen_value(name, v, low, low_inclusive, high=None):
    """A PCEN parameter as a float, or a list of floats (one per band); finite and in range, else ValueError."""
    def one(e):
        if isinstance(e, (bool, np.bool_)) or not isinstance(e, (int, float, np.integer, np.floating)):
            raise ValueError('%s must be a number or a sequence of numbers, got: %r' % (name, v))
        e = float(e)
        if not math.isfinite(e) or e < low or (e == low and not low_inclusive) or (high is not None and e > high):
            raise ValueError('%s must be finite and %s %s%s, got: %r' % (
                name, '>=' if low_inclusive else '>', low, '' if high is None else ' and <= %s' % high, v))
        return e
    if isinstance(v, (list, tuple, np.ndarray, torch.Tensor)):
        seq = np.asarray(v.detach().cpu() if isinstance(v, torch.Tensor) else v, dtype=object)
        if seq.ndim != 1 or seq.size == 0:
            raise ValueError('%s must be a number or a non-empty 1-D sequence (one value per band), got: %r' % (name, v))
        return [one(e) for e in seq]
    return one(v)


@register_keras_serializable(package='Kapre')
class PCEN(Layer):
    """Per-channel energy normalisation of a non-negative spectrogram (normally mel magnitudes), along time:

    ``M[t] = (1 - s) M[t-1] + s E[t]`` from ``M[-1] = E[0]``, then ``y = (E / (eps + M)^gain + bias)^power -
    bias^power``, computed as ``bias^power expm1(power log1p(E (eps + M)^-gain / bias))`` so that small inputs do not
    cancel.  ``s`` is ``smooth_coef``, or when that is None the coefficient librosa derives from
    ``time_constant`` seconds at ``sample_rate / hop_length`` frames per second.  ``(batch, time, band, ch)`` or
    ``(batch, ch, time, band)`` in, the same shape out.

    ``gain`` (>= 0), ``bias`` (> 0), ``power`` (> 0) and ``smooth_coef`` (in [0, 1]) are each one number shared by
    all bands or a sequence with one value per band.  They are the layer's weights: float32 tensors made on the
    first call, on the input's device, shape ``()`` or ``(bands,)``, with ``requires_grad = trainable``.  Trained
    values are used as they are: nothing clamps them back into the ranges above.  ``eps`` (> 0) is a constant.

    When a batch has too few (item, channel, band) columns to fill the GPU, the time axis is processed in chunks.  The
    result then agrees with the unchunked one to float32 rounding, not bit for bit, so outputs can differ in the last
    bits between batch sizes (for example between a call and ``predict`` with a smaller ``batch_size``)."""

    def __init__(self, sample_rate=22050, hop_length=512, time_constant=0.4, smooth_coef=None, gain=0.98, bias=2.0,
                 power=0.5, eps=1e-6, data_format='default', **kwargs):
        super().__init__(**kwargs)
        backend.validate_data_format_str(data_format)
        data_format = _unwrap_format(data_format)
        self.sample_rate = _pcen_value('sample_rate', sample_rate, 0.0, False)
        self.hop_length = _pcen_value('hop_length', hop_length, 0.0, False)
        self.time_constant = _pcen_value('time_constant', time_constant, 0.0, False)
        for name in ('sample_rate', 'hop_length', 'time_constant'):
            if isinstance(getattr(self, name), list):
                raise ValueError('%s must be a number' % name)
        self.smooth_coef = None if smooth_coef is None else _pcen_value('smooth_coef', smooth_coef, 0.0, True, 1.0)
        self.gain = _pcen_value('gain', gain, 0.0, True)
        self.bias = _pcen_value('bias', bias, 0.0, False)
        self.power = _pcen_value('power', power, 0.0, False)
        self.eps = _pcen_value('eps', eps, 0.0, False)
        if isinstance(self.eps, list):
            raise ValueError('eps must be a number')
        if self.smooth_coef is None:
            t = self.time_constant * self.sample_rate / self.hop_length
            self.smooth_coef_value = (math.sqrt(1.0 + 4.0 * t * t) - 1.0) / (2.0 * t * t)
        else:
            self.smooth_coef_value = self.smooth_coef
        self.data_format_original = data_format
        self.data_format = _resolve(data_format)
        self.built = False
        self._weights = []

    def build(self, bands, device):
        """Make the four weights for ``bands`` bands on ``device``; a per-band value must have ``bands`` entries."""
        ws = []
        for name, v in (('gain', self.gain), ('bias', self.bias), ('power', self.power),
                        ('smooth_coef', self.smooth_coef_value)):
            if isinstance(v, list) and len(v) != bands:
                raise ValueError('%s has %d values but the input has %d bands' % (name, len(v), bands))
            ws.append(torch.tensor(v, dtype=torch.float32, device=device).requires_grad_(bool(self.trainable)))
        self._weights = ws
        self.built = True

    @property
    def weights(self):
        """[gain, bias, power, smooth_coef] once built (the first call), else []."""
        return list(self._weights)

    def count_params(self):
        if not self.built:
            raise ValueError('You tried to call `count_params` on layer %s, but the layer isn\'t built.' % self.name)
        return sum(int(w.numel()) for w in self._weights)

    def call(self, x):
        if x.dim() != 4:
            raise ValueError('PCEN expects a 4-D batch, got shape %s' % (tuple(x.shape),))
        bands = x.shape[3] if self.data_format == _CH_FIRST_STR else x.shape[2]
        if not self.built:
            self.build(bands, x.device)
        elif self._weights[0].device != x.device:
            raise ValueError('PCEN %s was built on %s and cannot run on %s' % (self.name, self._weights[0].device, x.device))
        elif any(w.dim() == 1 and w.shape[0] != bands for w in self._weights):
            raise ValueError('PCEN %s was built for %d bands, the input has %d'
                             % (self.name, max(w.numel() for w in self._weights), bands))
        return ops.pcen(x, self._weights, self.eps, self.data_format)

    _config_fields = (
        ('sample_rate', 'sample_rate'),
        ('hop_length', 'hop_length'),
        ('time_constant', 'time_constant'),
        ('smooth_coef', 'smooth_coef'),
        ('gain', 'gain'),
        ('bias', 'bias'),
        ('power', 'power'),
        ('eps', 'eps'),
        ('data_format', 'data_format_original'),
    )


def _gl_int(name, v, low, high=None):
    """An int in [low, high) (bool and non-integral values rejected), else ValueError."""
    if isinstance(v, (bool, np.bool_)) or not isinstance(v, (int, np.integer)) or v < low or \
            (high is not None and v >= high):
        raise ValueError('%s must be an int >= %d%s, got: %r' % (name, low, '' if high is None else ' and < %d' % high, v))
    return int(v)


@register_keras_serializable(package='Kapre')
class GriffinLim(Layer):
    """Waveform from a magnitude spectrogram by fast Griffin-Lim (the momentum form of librosa and torchaudio), run
    over this library's own transform pair: ``STFT`` without padding and ``InverseSTFT`` with the dual window, so it
    inverts ``get_stft_magnitude_layer`` / ``STFT -> Magnitude`` as they are computed here.

    ``(batch, time, freq, ch)`` / ``(batch, ch, time, freq)`` float32 magnitudes with ``n_fft // 2 + 1`` bins ->
    ``(batch, L, ch)`` / ``(batch, ch, L)`` waveform, ``L = (time - 1) * hop_length + win_length``, untrimmed exactly
    as ``InverseSTFT`` returns it (for a spectrogram from ``get_perfectly_reconstructing_stft_istft``, drop the first
    ``n_fft - hop_length`` samples).  ``win_length``, ``hop_length`` and ``window_name`` default as in ``STFT``.

    Starting from ``X = S A_0``, each of ``n_iter`` iterations runs ``y = ISTFT(X)``, ``Y = STFT(y)``,
    ``A = Y - beta Yprev`` (``beta = momentum / (1 + momentum)``; ``A = Y`` the first time) and
    ``X = S A / (|A| + 1e-16)``; the result is ``ISTFT(X)``.  ``momentum`` is in [0, 1) (torchaudio's rule; 0 is
    the original Griffin-Lim).  ``init='ones'`` starts from zero phase; ``init='random'`` from uniform random phases
    drawn by a counter-based hash of ``seed`` and each element's (item, channel, frame, bin) index, so the result does
    not depend on the data format or strides.  The index counts items within one call: ``predict`` with a
    ``batch_size`` smaller than the batch draws other phases than one call on the whole batch.  ``seed=None`` draws a
    fresh seed from torch's CPU generator on every call; a captured graph (``Sequential.capture``) keeps the seed of
    the call it recorded.

    The whole loop is one library call.  It has no gradient: calling the layer under grad mode on an input that
    requires grad raises ``RuntimeError``; run it under ``torch.no_grad()`` or on a detached tensor."""

    def __init__(self, n_fft=2048, win_length=None, hop_length=None, window_name=None, n_iter=32, momentum=0.99,
                 init='random', seed=0, input_data_format='default', output_data_format='default', **kwargs):
        super().__init__(**kwargs)
        for data_format in (input_data_format, output_data_format):
            backend.validate_data_format_str(data_format)
        input_data_format = _unwrap_format(input_data_format)
        output_data_format = _unwrap_format(output_data_format)
        if win_length is None:
            win_length = n_fft
        if hop_length is None:
            hop_length = win_length // 4
        self.n_iter = _gl_int('n_iter', n_iter, 0)
        if isinstance(momentum, (bool, np.bool_)) or not isinstance(momentum, (int, float, np.integer, np.floating)) \
                or not 0.0 <= float(momentum) < 1.0:
            raise ValueError('momentum must be a number in [0, 1), got: %r' % (momentum,))
        if init not in ('random', 'ones'):
            raise ValueError("init must be 'random' or 'ones', got: %r" % (init,))
        self.seed = None if seed is None else _gl_int('seed', seed, 0, 2 ** 64)
        self.n_fft = n_fft
        self.win_length = win_length
        self.hop_length = hop_length
        self.window_name = window_name
        self.momentum = momentum
        self.init = init
        self.input_data_format_original = input_data_format
        self.output_data_format_original = output_data_format
        self.input_data_format = _resolve(input_data_format)
        self.output_data_format = _resolve(output_data_format)
        self._plans = None

    @property
    def plans(self):
        """(StftPlan, IstftPlan): the forward window and its dual (``tf.signal.inverse_stft_window_fn``)."""
        if self._plans is None:
            window_fn = backend.get_window_fn(self.window_name)
            dual_fn = backend.inverse_stft_window_fn(frame_step=self.hop_length, forward_window_fn=window_fn)
            self._plans = (ops.StftPlan(self.n_fft, self.win_length, self.hop_length, window_fn(self.win_length)),
                           ops.IstftPlan(self.n_fft, self.win_length, self.hop_length, dual_fn(self.win_length)))
        return self._plans

    def call(self, x):
        seed = self.seed
        if seed is None:
            seed = int(torch.randint(-2 ** 63, 2 ** 63 - 1, (1,), dtype=torch.int64)) % 2 ** 64
        stft_plan, istft_plan = self.plans
        return ops.griffin_lim(x, stft_plan, istft_plan, self.n_iter, self.momentum,
                               N.GL_INIT_RANDOM if self.init == 'random' else N.GL_INIT_ONES, seed,
                               self.input_data_format, self.output_data_format)

    _config_fields = (
        ('n_fft', 'n_fft'),
        ('win_length', 'win_length'),
        ('hop_length', 'hop_length'),
        ('window_name', 'window_name'),
        ('n_iter', 'n_iter'),
        ('momentum', 'momentum'),
        ('init', 'init'),
        ('seed', 'seed'),
        ('input_data_format', 'input_data_format_original'),
        ('output_data_format', 'output_data_format_original'),
    )


def _positive(name, v):
    if isinstance(v, (bool, np.bool_)) or not isinstance(v, (int, float, np.integer, np.floating)) or \
            not 0.0 < float(v) < math.inf:
        raise ValueError('%s must be a positive finite number, got: %r' % (name, v))
    return v


@register_keras_serializable(package='Kapre')
class InverseFilterbank(Layer):
    """Linear magnitudes from a filterbank output: the inverse of ``ApplyFilterbank(type, filterbank_kwargs)``, by
    non-negative least squares.  Use it with ``GriffinLim`` to hear a mel spectrogram
    (``composed.get_inverse_melspectrogram_layer``).

    ``(batch, time, n_bands, ch)`` / ``(batch, ch, time, n_bands)`` -> float32 ``(batch, time, n_freq, ch)`` /
    ``(batch, ch, time, n_freq)`` in the same data format.  With ``A`` the ``(n_bands, n_freq)`` transpose of the
    filterbank and ``m`` one frame, the layer runs ``n_iter`` steps of projected accelerated gradient (FISTA) on
    ``min ||A s - m||^2`` subject to ``s >= 0``: ``s_0 = max(A^T (m / d), 0)`` with ``d = A A^T 1``, step
    ``1 / ||A||_2^2``, and returns ``s_n``.  There are more bins than bands, so the minimiser is not unique: the result
    is this iteration's, not the spectrum the mel came from.  Bins that no band touches (for a mel bank, DC, Nyquist
    and bins above ``f_max``) come out exactly 0.  On consistent mel input the residual ``||A s - m||`` falls below
    1e-3 of ``||m||`` within the default 100 iterations; torchaudio's ``InverseMelScale`` (least squares, then
    ``relu``) leaves 1e-2 to 1e-1.

    ``from_decibel=True`` takes the output of ``MagnitudeToDecibel(ref_value=db_ref_value, amin=db_amin)`` (e.g.
    ``get_melspectrogram_layer(return_decibel=True)``) and converts each element on load with
    ``m = 10^(v / 10) * max(db_amin, db_ref_value)``: the exact inverse where the input was at least ``db_amin`` and
    the dynamic-range clamp did not bind; clamped elements come back as the clamp floor.

    One kernel launch.  A frame's output does not depend on its place in the batch or on the data format.  No
    gradient: calling the layer under grad mode on an input that requires grad raises ``RuntimeError``."""

    def __init__(self, type, filterbank_kwargs, n_iter=100, from_decibel=False, db_ref_value=1.0, db_amin=1e-5,
                 data_format='default', **kwargs):
        super().__init__(**kwargs)
        backend.validate_data_format_str(data_format)
        data_format = _unwrap_format(data_format)
        if type == 'log':
            self.filterbank = backend.filterbank_log(**filterbank_kwargs)
        elif type == 'mel':
            self.filterbank = backend.filterbank_mel(**filterbank_kwargs)
        else:
            raise ValueError("type must be 'mel' or 'log', got: %r" % (type,))
        self.type = type
        self.filterbank_kwargs = filterbank_kwargs
        self.n_iter = _gl_int('n_iter', n_iter, 0)
        if not isinstance(from_decibel, (bool, np.bool_)):
            raise ValueError('from_decibel must be a bool, got: %r' % (from_decibel,))
        self.from_decibel = bool(from_decibel)
        self.db_ref_value = _positive('db_ref_value', db_ref_value)
        self.db_amin = _positive('db_amin', db_amin)
        self.data_format_original = data_format
        self.data_format = _resolve(data_format)
        self._plan = None

    @property
    def plan(self) -> ops.FilterbankInversePlan:
        if self._plan is None:
            self._plan = ops.FilterbankInversePlan(np.asarray(self.filterbank))
        return self._plan

    def call(self, x):
        return ops.invert_filterbank(x, self.plan, self.n_iter, self.from_decibel, self.db_ref_value, self.db_amin,
                                     self.data_format)

    _config_fields = (
        ('type', 'type'),
        ('filterbank_kwargs', 'filterbank_kwargs'),
        ('n_iter', 'n_iter'),
        ('from_decibel', 'from_decibel'),
        ('db_ref_value', 'db_ref_value'),
        ('db_amin', 'db_amin'),
        ('data_format', 'data_format_original'),
    )


class _KaldiLayer(Layer):
    """torchaudio.compliance.kaldi features of a batch as a layer: torchaudio's keywords (without ``channel``) and
    ``data_format``.  ``call(x, lengths=None, training=False)``: dither (``dither`` > 0) is applied only with
    ``training=True``, from a seed drawn per call from ``np.random.default_rng(seed)`` and recorded in
    ``last_choice``; ``Sequential`` passes no ``training`` flag, so a captured graph never dithers."""

    _kind = None

    def __init__(self, data_format='default', seed=None, **kwargs):
        keys = ops.KALDI_DEFAULTS[self._kind]
        kaldi = {k: kwargs.pop(k) for k in list(kwargs) if k in keys}
        super().__init__(**kwargs)
        backend.validate_data_format_str(data_format)
        data_format = _unwrap_format(data_format)
        self.options = ops.kaldi_options(self._kind, **kaldi)
        for k, v in self.options.items():
            setattr(self, k, v)
        self.plan = ops.kaldi_plan(self._kind, self.options)
        self.data_format_original = data_format
        self.data_format = _resolve(data_format)
        self.seed = seed
        self.rng = np.random.default_rng(seed)
        self.last_choice = None

    def __call__(self, x, lengths=None, training=None, **kwargs):
        t, was_host = ops.to_device(x)
        if was_host:
            with torch.no_grad():
                return ops.to_host(self.call(t, lengths=lengths, training=training))
        return self.call(t, lengths=lengths, training=training)

    def call(self, x, lengths=None, training=False):
        dither, seed = 0.0, 0
        if training and self.options['dither'] > 0.0:
            dither = self.options['dither']
            seed = int(self.rng.integers(0, 2 ** 63))
            self.last_choice = seed
        return ops.kaldi_features(x, self.plan, lengths, self.data_format, dither, seed)

    @property
    def _config_fields(self):
        return tuple((k, k) for k in ops.KALDI_DEFAULTS[self._kind]) + (
            ('data_format', 'data_format_original'), ('seed', 'seed'))


@register_keras_serializable(package='Kapre')
class KaldiFbank(_KaldiLayer):
    """``torchaudio.compliance.kaldi.fbank`` per (item, channel): ``(batch, time, ch)`` / ``(batch, ch, time)`` ->
    ``(batch, frames, num_mel_bins + use_energy, ch)`` / ``(batch, ch, frames, num_mel_bins + use_energy)``."""
    _kind = 'fbank'


@register_keras_serializable(package='Kapre')
class KaldiMFCC(_KaldiLayer):
    """``torchaudio.compliance.kaldi.mfcc`` per (item, channel): ``num_ceps`` bins per frame."""
    _kind = 'mfcc'


@register_keras_serializable(package='Kapre')
class KaldiSpectrogram(_KaldiLayer):
    """``torchaudio.compliance.kaldi.spectrogram`` per (item, channel): ``padded_window_size // 2 + 1`` bins per
    frame."""
    _kind = 'spectrogram'


@register_keras_serializable(package='Kapre')
class CQT(Layer):
    """Constant-Q transform, modelled on librosa's multirate ``cqt`` (``gamma > 0``: ``vqt``).

    ``(batch, time, ch)`` / ``(batch, ch, time)`` float32 waveforms -> complex64 ``(batch, frames, n_bins, ch)`` /
    ``(batch, ch, frames, n_bins)``, bins in ascending frequency, ``frames = 1 + time // hop_length``, frame m centred on
    sample ``m hop_length``.  Bin k has centre ``f_k = f_min 2^(k / bins_per_octave)`` (``f_min`` default C1) and a
    periodic-Hann complex filter of ``l_k = Q sample_rate / (f_k + gamma / alpha)`` samples, ``Q = filter_scale /
    alpha``, ``alpha = (r^2 - 1) / (r^2 + 1)``, ``r = 2^(1 / bins_per_octave)``, with unit L1 norm; outputs are scaled
    by ``sqrt(l_k)`` (``scale=True``) or ``l_k``.  Each octave is computed at its own rate on a 2:1 polyphase pyramid
    (``scipy.signal.resample_poly(y, 1, 2)``), as an exact time-domain inner product per output.  The decimator's
    response is within 0.25 % of 1 up to 0.2 cycles per sample and below -56 dB from 0.3 on, and every octave's
    bins sit in the same digital band, so with the top band below 0.4 ``sample_rate`` the lower octaves see its flat
    passband.  ``hop_length`` must be a multiple of ``2^(n_octaves - 1)``.  Followed by ``Magnitude()`` in a
    ``Sequential`` it runs as one fused launch writing ``|C|``."""

    def __init__(self, sample_rate=22050, hop_length=512, f_min=None, n_bins=84, bins_per_octave=12, filter_scale=1.0,
                 gamma=0.0, scale=True, input_data_format='default', output_data_format='default', **kwargs):
        super().__init__(**kwargs)
        for data_format in (input_data_format, output_data_format):
            backend.validate_data_format_str(data_format)
        input_data_format = _unwrap_format(input_data_format)
        output_data_format = _unwrap_format(output_data_format)
        backend.cqt_geometry(sample_rate, hop_length, f_min, n_bins, bins_per_octave, filter_scale, gamma)
        self.sample_rate, self.hop_length, self.f_min = sample_rate, hop_length, f_min
        self.n_bins, self.bins_per_octave = n_bins, bins_per_octave
        self.filter_scale, self.gamma, self.scale = filter_scale, gamma, scale
        self.input_data_format_original = input_data_format
        self.output_data_format_original = output_data_format
        self.input_data_format = _resolve(input_data_format)
        self.output_data_format = _resolve(output_data_format)
        self._plan = None

    @property
    def plan(self) -> ops.CqtPlan:
        if self._plan is None:
            self._plan = ops.CqtPlan(self.sample_rate, self.hop_length, self.f_min, self.n_bins, self.bins_per_octave,
                                     self.filter_scale, self.gamma, self.scale)
        return self._plan

    def call(self, x, magnitude=False):
        return ops.cqt(x, self.plan, self.input_data_format, self.output_data_format, magnitude)

    _config_fields = (
        ('sample_rate', 'sample_rate'),
        ('hop_length', 'hop_length'),
        ('f_min', 'f_min'),
        ('n_bins', 'n_bins'),
        ('bins_per_octave', 'bins_per_octave'),
        ('filter_scale', 'filter_scale'),
        ('gamma', 'gamma'),
        ('scale', 'scale'),
        ('input_data_format', 'input_data_format_original'),
        ('output_data_format', 'output_data_format_original'),
    )


class _ChromaLayer(Layer):
    """A chroma function of ``signal`` as a layer: the waveform in, the chroma out.  The constructor takes the
    function's keyword arguments (without the waveform and the precomputed spectrogram), checks them and builds the
    plans on the host."""
    _fn = None

    def __init__(self, data_format, args, **kwargs):
        super().__init__(**kwargs)
        backend.validate_data_format_str(data_format)
        self.data_format_str = _unwrap_format(data_format)
        self._kw = args
        for k, v in args.items():
            setattr(self, k, v)
        self._check()

    def call(self, x):
        from . import signal
        return getattr(signal, self._fn)(x, data_format=self.data_format_str, **self._kw)


@register_keras_serializable(package='Kapre')
class ChromaSTFT(_ChromaLayer):
    """``signal.chroma_stft`` as a layer: ``(batch, time, ch)`` / ``(batch, ch, time)`` waveforms in, ``(batch,
    frames, n_chroma, ch)`` / ``(batch, ch, frames, n_chroma)`` chroma out.  Same arguments."""
    _fn = 'chroma_stft'

    def __init__(self, sample_rate=22050, norm=np.inf, n_fft=2048, hop_length=512, win_length=None, window_name=None,
                 center=True, tuning=None, n_chroma=12, ctroct=5.0, octwidth=2.0, base_c=True, data_format='default',
                 **kwargs):
        super().__init__(data_format, dict(sample_rate=sample_rate, norm=norm, n_fft=n_fft, hop_length=hop_length,
                                           win_length=win_length, window_name=window_name, center=center,
                                           tuning=tuning, n_chroma=n_chroma, ctroct=ctroct, octwidth=octwidth,
                                           base_c=base_c), **kwargs)

    def _check(self):
        from . import signal
        backend.chroma_norm_code(self.norm)
        if self.win_length is not None and self.win_length != self.n_fft:
            raise ValueError('win_length must be None or n_fft=%r, got %r' % (self.n_fft, self.win_length))
        signal._stft_chroma_plans(self.sample_rate, self.n_fft, self.hop_length, self.window_name, self.n_chroma,
                                  self.tuning, self.ctroct, self.octwidth, self.base_c)

    _config_fields = (
        ('sample_rate', 'sample_rate'), ('norm', 'norm'), ('n_fft', 'n_fft'), ('hop_length', 'hop_length'),
        ('win_length', 'win_length'), ('window_name', 'window_name'), ('center', 'center'), ('tuning', 'tuning'),
        ('n_chroma', 'n_chroma'), ('ctroct', 'ctroct'), ('octwidth', 'octwidth'), ('base_c', 'base_c'),
        ('data_format', 'data_format_str'),
    )


@register_keras_serializable(package='Kapre')
class ChromaCQT(_ChromaLayer):
    """``signal.chroma_cqt`` as a layer (waveforms in, chroma out).  Same arguments."""
    _fn = 'chroma_cqt'

    def __init__(self, sample_rate=22050, hop_length=512, f_min=None, norm=np.inf, threshold=0.0, tuning=0.0,
                 n_chroma=12, n_octaves=7, bins_per_octave=36, base_c=True, data_format='default', **kwargs):
        super().__init__(data_format, dict(sample_rate=sample_rate, hop_length=hop_length, f_min=f_min, norm=norm,
                                           threshold=threshold, tuning=tuning, n_chroma=n_chroma, n_octaves=n_octaves,
                                           bins_per_octave=bins_per_octave, base_c=base_c), **kwargs)

    def _check(self):
        from . import signal
        backend.chroma_norm_code(self.norm)
        signal._cqt_chroma_plans(self.sample_rate, self.hop_length, self.f_min, self.tuning, self.n_chroma,
                                 self.n_octaves, self.bins_per_octave, self.base_c, False)

    _config_fields = (
        ('sample_rate', 'sample_rate'), ('hop_length', 'hop_length'), ('f_min', 'f_min'), ('norm', 'norm'),
        ('threshold', 'threshold'), ('tuning', 'tuning'), ('n_chroma', 'n_chroma'), ('n_octaves', 'n_octaves'),
        ('bins_per_octave', 'bins_per_octave'), ('base_c', 'base_c'), ('data_format', 'data_format_str'),
    )


@register_keras_serializable(package='Kapre')
class ChromaCENS(_ChromaLayer):
    """``signal.chroma_cens`` as a layer (waveforms in, CENS out).  Same arguments."""
    _fn = 'chroma_cens'

    def __init__(self, sample_rate=22050, hop_length=512, f_min=None, tuning=0.0, n_chroma=12, n_octaves=7,
                 bins_per_octave=36, base_c=True, norm=2, win_len_smooth=41, data_format='default', **kwargs):
        super().__init__(data_format, dict(sample_rate=sample_rate, hop_length=hop_length, f_min=f_min, tuning=tuning,
                                           n_chroma=n_chroma, n_octaves=n_octaves, bins_per_octave=bins_per_octave,
                                           base_c=base_c, norm=norm, win_len_smooth=win_len_smooth), **kwargs)

    def _check(self):
        from . import signal
        if backend.chroma_norm_code(self.norm) != 3:
            raise ValueError('chroma_cens supports norm=2 only, got %r' % (self.norm,))
        signal._cqt_chroma_plans(self.sample_rate, self.hop_length, self.f_min, self.tuning, self.n_chroma,
                                 self.n_octaves, self.bins_per_octave, self.base_c, self.win_len_smooth)

    _config_fields = (
        ('sample_rate', 'sample_rate'), ('hop_length', 'hop_length'), ('f_min', 'f_min'), ('tuning', 'tuning'),
        ('n_chroma', 'n_chroma'), ('n_octaves', 'n_octaves'), ('bins_per_octave', 'bins_per_octave'),
        ('base_c', 'base_c'), ('norm', 'norm'), ('win_len_smooth', 'win_len_smooth'),
        ('data_format', 'data_format_str'),
    )


@register_keras_serializable(package='Kapre')
class HPSS(Layer):
    """One component of ``signal.hpss`` as a layer: a ``(batch, frames, bins, ch)`` / ``(batch, ch, frames, bins)``
    magnitude (float32) or complex64 spectrogram in, the ``component`` (``'harmonic'`` or ``'percussive'``), or its
    mask with ``mask=True``, out in the same shape.  Other arguments as ``signal.hpss``.  One launch; differentiable
    with respect to the input."""

    def __init__(self, component='harmonic', kernel_size=31, power=2.0, mask=False, margin=1.0, data_format='default',
                 **kwargs):
        super().__init__(**kwargs)
        backend.validate_data_format_str(data_format)
        data_format = _unwrap_format(data_format)
        if component not in ('harmonic', 'percussive'):
            raise ValueError("component must be 'harmonic' or 'percussive', got %r" % (component,))
        self.cfg = ops.hpss_config(kernel_size, power, mask, margin)
        self.component = component
        self.kernel_size = list(kernel_size) if isinstance(kernel_size, (tuple, list)) else kernel_size
        self.power, self.mask = power, mask
        self.margin = list(margin) if isinstance(margin, (tuple, list)) else margin
        self.data_format_str = data_format
        self.data_format = _resolve(data_format)

    def call(self, x):
        h, p = ops.hpss(x, self.cfg, self.data_format, want_h=self.component == 'harmonic',
                        want_p=self.component == 'percussive')
        return h if self.component == 'harmonic' else p

    _config_fields = (
        ('component', 'component'), ('kernel_size', 'kernel_size'), ('power', 'power'), ('mask', 'mask'),
        ('margin', 'margin'), ('data_format', 'data_format_str'),
    )


@register_keras_serializable(package='Kapre')
class OnsetStrength(_ChromaLayer):
    """``signal.onset_strength`` as a layer: ``(batch, time, ch)`` / ``(batch, ch, time)`` waveforms in, the ``(batch,
    frames, ch)`` / ``(batch, ch, frames)`` envelope out.  Same arguments; differentiable with respect to the
    input."""
    _fn = 'onset_strength'

    def __init__(self, sample_rate=22050, lag=1, max_size=1, detrend=False, center=True, aggregate='mean', n_fft=2048,
                 hop_length=512, n_mels=128, fmin=0.0, fmax=None, data_format='default', **kwargs):
        super().__init__(data_format, dict(sample_rate=sample_rate, lag=lag, max_size=max_size, detrend=detrend,
                                           center=center, aggregate=aggregate, n_fft=n_fft, hop_length=hop_length,
                                           n_mels=n_mels, fmin=fmin, fmax=fmax), **kwargs)

    def _check(self):
        from . import signal
        ops.onset_limits(ops.onset_config(self.lag, self.max_size, self.aggregate), self.n_mels, 0)
        signal._rhythm_frontend(self.sample_rate, self.n_fft, self.hop_length, self.n_mels, self.fmin, self.fmax)

    _config_fields = (
        ('sample_rate', 'sample_rate'), ('lag', 'lag'), ('max_size', 'max_size'), ('detrend', 'detrend'),
        ('center', 'center'), ('aggregate', 'aggregate'), ('n_fft', 'n_fft'), ('hop_length', 'hop_length'),
        ('n_mels', 'n_mels'), ('fmin', 'fmin'), ('fmax', 'fmax'), ('data_format', 'data_format_str'),
    )


@register_keras_serializable(package='Kapre')
class Tempogram(_ChromaLayer):
    """``signal.tempogram`` as a layer: waveforms in, ``(batch, frames, win_length, ch)`` / ``(batch, ch, frames,
    win_length)`` out.  Same arguments; no gradient."""
    _fn = 'tempogram'

    def __init__(self, sample_rate=22050, hop_length=512, win_length=384, center=True, norm=np.inf,
                 data_format='default', **kwargs):
        super().__init__(data_format, dict(sample_rate=sample_rate, hop_length=hop_length, win_length=win_length,
                                           center=center, norm=norm), **kwargs)

    def _check(self):
        from . import signal
        ops.tempogram_check(self.win_length)
        if self.norm is not None and self.norm != np.inf:
            raise ValueError('norm must be np.inf or None, got %r' % (self.norm,))
        signal._rhythm_frontend(self.sample_rate, 2048, self.hop_length, 128, 0.0, None)

    _config_fields = (
        ('sample_rate', 'sample_rate'), ('hop_length', 'hop_length'), ('win_length', 'win_length'),
        ('center', 'center'), ('norm', 'norm'), ('data_format', 'data_format_str'),
    )
