"""Time stretch on the GPU: parity with the float64 restatement (time_stretch_ref.py) at the cfg2 complex shape and on
a 10-minute recording (the chunked path), the gradient from a waveform through STFT -> TimeStretch against float64
autograd, the waveform factory on a sinusoid, and bit-identical outputs through Sequential, predict, a captured graph
and requires_grad.  Phase bound as derived in test_time_stretch_emu.py."""
import math

import numpy as np
import pytest
import torch

import grad_ref as R
import time_stretch_ref as TR

pytestmark = pytest.mark.gpu
CL, CF = 'channels_last', 'channels_first'
CFG2 = (256, 427, 513, 1)           # cfg2's complex STFT: 256 x 5 s at 22.05 kHz, n_fft 1024, hop 256
LONG = (1, 25840, 513, 1)           # 10 min at 22.05 kHz, n_fft 1024, hop 512
ANGLE_ERR = 2.8e-7 + 7.3e-10
READ_ERR = 3e-7


def _spectrogram(shape, fmt, seed=0):
    """Complex (B, T, F, C) for channels_last, (B, C, T, F) otherwise, from a (B, T, F, C) description."""
    B, T, F, C = shape
    g = torch.Generator().manual_seed(seed)
    s = (B, T, F, C) if fmt == CL else (B, C, T, F)
    return torch.complex(torch.randn(s, generator=g), torch.randn(s, generator=g)).cuda()


def _canon(t, fmt):
    t = t.detach().cpu()
    return t.permute(0, 3, 1, 2) if fmt == CL else t


def _check(Y, X, rate, fmt):
    """Y against the restatement of X: phase within (2u + 1) angle errors + the read-back error, magnitude within
    4 eps32 of the two moduli it blends."""
    Xc = _canon(X, fmt).to(torch.complex128)
    m, phi = TR.phases(Xc, rate)
    Yc = _canon(Y, fmt).to(torch.complex128)
    assert Yc.shape == m.shape
    k, _ = TR.steps(Xc.shape[2], rate)
    Xa = torch.cat([Xc, torch.zeros_like(Xc[:, :, :2])], dim=2).abs()
    assert bool(((Yc.abs() - m).abs() <= 4 * 2.0 ** -24 * (Xa[:, :, k] + Xa[:, :, k + 1]) + 1e-30).all())
    u = torch.arange(m.shape[2], dtype=torch.float64).view(1, 1, -1, 1)
    d = torch.remainder(Yc.angle() - phi + math.pi, 2 * math.pi) - math.pi
    bound = (2 * u + 1) * ANGLE_ERR + READ_ERR
    assert bool(((m == 0) | (d.abs() <= bound)).all()), float((d.abs() / bound)[m > 0].max())


def _layer(rate, fmt):
    from kapre_b200.augmentation import TimeStretch
    return TimeStretch(rate, data_format=fmt)


@pytest.mark.parametrize('rate', [0.8, 1.25])
@pytest.mark.parametrize('fmt', [CL, CF])
def test_parity_cfg2(rate, fmt):
    X = _spectrogram(CFG2, fmt, seed=1)
    _check(_layer(rate, fmt)(X), X, rate, fmt)


@pytest.mark.parametrize('fmt', [CL, CF])
def test_parity_on_views(fmt):
    full = _spectrogram((8, 120, 520, 2), fmt, seed=2)
    X = full[:, ::2, 3:516, 1:] if fmt == CL else full[:, 1:, ::2, 3:516]
    _check(_layer(0.8, fmt)(X), X, 0.8, fmt)


def test_long_recording_takes_the_chunked_path():
    from kapre_b200 import ops
    X = _spectrogram(LONG, CL, seed=3)
    assert ops._time_stretch_workspace(1, 1, LONG[1], LONG[2], 0.8, X.device)[0] > 1
    Y = _layer(0.8, CL)(X)
    _check(Y, X, 0.8, CL)


def test_edge_shapes():
    layer = _layer(1.3, CF)
    for shape in ((0, 10, 513, 1), (2, 1, 513, 1), (2, 10, 1, 1), (1, 0, 5, 1)):
        X = _spectrogram(shape, CF, seed=4)
        Y = layer(X)
        assert Y.shape == (shape[0], 1, math.ceil(shape[1] / 1.3), shape[2])
        if Y.numel():
            _check(Y, X, 1.3, CF)
    X = _spectrogram((2, 10, 5, 1), CF)
    assert layer(X, rate=1.0) is X
    with pytest.raises(TypeError):
        layer(X.real.contiguous())
    Y64 = layer(X.to(torch.complex128))
    assert Y64.dtype == torch.complex64 and torch.equal(Y64, layer(X))


def test_gradient_from_waveform():
    """STFT -> TimeStretch from a waveform against float64 autograd through grad_ref's STFT and the restatement."""
    from kapre_b200.composed import Sequential
    from kapre_b200.time_frequency import STFT
    stack = Sequential([STFT(n_fft=512, hop_length=128, input_data_format=CL, output_data_format=CL),
                        _layer(0.8, CL)])
    g = torch.Generator().manual_seed(5)
    x = (torch.rand((2, 8000, 1), generator=g) * 2 - 1).cuda().requires_grad_()
    y = stack(x)
    gy = torch.complex(torch.randn(y.shape, generator=g), torch.randn(y.shape, generator=g)).cuda()
    got, = torch.autograd.grad(y, x, gy)
    xr = x.detach().cpu().double().requires_grad_()
    S = R.stft(xr, 512, 512, 128, None, False, False, CL, CL).permute(0, 3, 1, 2)
    want, = torch.autograd.grad(TR.time_stretch(S, 0.8), xr, _canon(gy, CL).to(torch.complex128))
    err = float((got.cpu().double() - want).abs().max())
    assert err <= 1e-3 * float(want.abs().max()), err


def test_waveform_factory_on_a_sinusoid():
    """get_time_stretch_layer keeps the frequency within one bin and scales the duration by 1 / rate."""
    from kapre_b200.composed import get_time_stretch_layer
    sr, f0, n_fft, hop = 16000, 1000.0, 1024, 256
    t = torch.arange(2 * sr, dtype=torch.float64) / sr
    x = torch.sin(2 * math.pi * f0 * t).float().view(1, -1, 1).cuda()
    for rate in (0.5, 1.25):
        model = get_time_stretch_layer(rate, n_fft=n_fft, hop_length=hop, window_name='hann_window',
                                       waveform_data_format=CL)
        y = model(x)
        T = 1 + (x.shape[1] - n_fft) // hop
        L = (math.ceil(T / rate) - 1) * hop + n_fft
        assert y.shape == (1, L, 1)
        assert abs(L / x.shape[1] - 1 / rate) < 0.05
        mid = y[0, n_fft:L - n_fft, 0].double().cpu()
        spec = torch.fft.rfft(mid * torch.hann_window(mid.numel(), dtype=torch.float64)).abs()
        f_peak = float(spec.argmax()) * sr / mid.numel()
        assert abs(f_peak - f0) <= sr / n_fft, f_peak


def test_same_bits_through_sequential_predict_graph_and_grad():
    from kapre_b200 import _native as N
    from kapre_b200.composed import Sequential
    layer = _layer(0.8, CL)
    stack = Sequential([layer])
    X = _spectrogram((64, 427, 513, 1), CL, seed=6)
    want = layer(X)
    torch.cuda.synchronize()
    n0 = N.launch_count()
    got = stack(X)
    assert N.launch_count() - n0 == 1 and torch.equal(got, want)
    host = stack.predict(X.cpu().numpy(), batch_size=16)           # other column counts: the same bits
    assert np.array_equal(host, want.cpu().numpy())
    one = layer(X[:1])                                              # 513 columns: the chunked path
    assert torch.equal(one, want[:1])
    cap = stack.capture(X)
    out = cap(X)
    torch.cuda.synchronize()
    assert torch.equal(out, want)
    tracked = stack(X.clone().requires_grad_())
    assert tracked.requires_grad and torch.equal(tracked.detach(), want)
