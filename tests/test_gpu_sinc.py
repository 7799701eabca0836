"""The band-limited interpolator on the GPU: parity with the float64 restatement (sinc_ref.py) at a bench-sized batch
and on views, its vector-Jacobian product, ``Speed`` in front of the fused log-mel launch, no per-ratio state, graph
capture, and ``PitchShift`` against the restated float64 chain (a sinusoid, a tone burst, an impulse, a gradient).
Bounds as derived in sinc_ref.py.  No scipy needed."""
import math

import numpy as np
import pytest
import torch

import sinc_ref as SR

pytestmark = pytest.mark.gpu
CL, CF = 'channels_last', 'channels_first'


def _signal(fmt, B, C, L, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.rand((B, L, C) if fmt == CL else (B, C, L), generator=g) * 2 - 1
    return x.cuda()


def _ref(x, fmt, ratio, length=None, offset=0.0):
    t = x.detach().cpu().double()
    if fmt == CL:
        return SR.resample(t.transpose(1, 2), ratio, length, offset).transpose(1, 2)
    return SR.resample(t, ratio, length, offset)


def _close(got, want, ratio, xmax, adjoint=False):
    assert tuple(got.shape) == tuple(want.shape), (tuple(got.shape), tuple(want.shape))
    if got.numel():
        err = float((got.detach().cpu().double() - want).abs().max())
        assert err <= SR.error_bound(ratio, adjoint) * xmax, (err, SR.error_bound(ratio, adjoint) * xmax)


@pytest.mark.parametrize('factor', [2.0 ** (4 / 12), 0.9])
@pytest.mark.parametrize('fmt', [CF, CL])
def test_parity_at_bench_size(factor, fmt):
    """256 x 5 s at 22.05 kHz; the restatement is taken on 6 items spread over the batch, every item is checked to be
    the bits of its copy in a batch of one."""
    from kapre_b200.signal import Speed
    layer = Speed(factor, data_format=fmt)
    x = _signal(fmt, 256, 1, 110250, seed=int(factor * 100))
    y = layer(x)
    assert y.shape[0] == 256 and y.numel() == 256 * math.ceil(110250 / factor)
    pick = [0, 1, 100, 131, 254, 255]
    _close(y[pick], _ref(x[pick], fmt, 1.0 / factor, length=math.ceil(110250 / factor)), 1.0 / factor, 1.0)
    assert torch.equal(layer(x[131:132]), y[131:132])


@pytest.mark.parametrize('ratio', [0.25, 2.0 ** (5 / 12), 4.0])
def test_stereo_interleaved_and_planar_agree(ratio):
    from kapre_b200 import ops
    x = _signal(CL, 8, 2, 30000, seed=2)
    Lo = SR.output_length(30000, ratio)
    y = ops.sinc_resample(x, ratio, Lo, 0.25, CL)
    _close(y, _ref(x, CL, ratio, Lo, 0.25), ratio, 1.0)
    planar = ops.sinc_resample(x.transpose(1, 2).contiguous(), ratio, Lo, 0.25, CF)
    assert torch.equal(planar.transpose(1, 2), y)


@pytest.mark.parametrize('fmt', [CF, CL])
def test_parity_views_short_signals_and_lengths(fmt):
    from kapre_b200 import ops
    ratio = 2.0 ** (-4 / 12)
    full = _signal(fmt, 4, 3, 20000, seed=3)
    t_ax = 1 if fmt == CL else 2
    views = [full.narrow(t_ax, 5, 9000), full[::2], full.narrow(3 - t_ax, 1, 1), full.narrow(t_ax, 0, 1),
             full.narrow(t_ax, 0, 0), full.narrow(t_ax, 0, 50),
             full.transpose(1, 2).contiguous().transpose(1, 2)]
    for x in views:
        L = x.shape[t_ax]
        for length in (SR.output_length(L, ratio), 40, SR.output_length(L, ratio) + 300):
            y = ops.sinc_resample(x, ratio, length, -1.75, fmt)
            _close(y, _ref(x, fmt, ratio, length, -1.75), ratio, 1.0)
    x = full.narrow(t_ax, 0, 1000)
    y = ops.sinc_resample(x, ratio, 2000, 0.0, fmt).narrow(t_ax, 900, 1100)
    assert not bool(y.any())                                                    # past the signal: exact zeros


def test_invalid_arguments_raise_before_any_launch():
    from kapre_b200 import _native as N, ops
    from kapre_b200.signal import Speed
    x = _signal(CL, 1, 1, 100)
    n0 = N.launch_count()
    for ratio in (0.2, 4.5, float('nan'), float('inf'), -1.0):
        with pytest.raises(ValueError):
            ops.sinc_resample(x, ratio, 10, 0.0, CL)
    for offset in (float('nan'), float('inf')):
        with pytest.raises(ValueError):
            ops.sinc_resample(x, 1.5, 10, offset, CL)
    with pytest.raises(ValueError):
        Speed(1.1)(x, factor=5.0)
    # the C entry point holds the same line
    y = torch.empty((1, 10, 1), device='cuda')
    xd, _ = ops._wave_desc(x, CL)
    yd, _ = ops._wave_desc(y, CL)
    import ctypes
    for ratio, offset in ((0.2, 0.0), (float('nan'), 0.0), (1.5, float('inf')), (1.5, 2.0 ** 41)):
        rc = N.lib().kapre_sinc_resample(ops._sinc_plan.handle(), ops._ptr(x), ctypes.byref(xd), ops._ptr(y),
                                         ctypes.byref(yd), ratio, offset, ops._stream_ptr())
        assert rc == -1
    assert N.launch_count() == n0
    assert Speed(1.1)(x, factor=1.0) is x and N.launch_count() == n0


@pytest.mark.parametrize('ratio', [0.5, 2.0 ** (-4 / 12), 2.0 ** (5 / 12)])
@pytest.mark.parametrize('fmt', [CF, CL])
def test_vjp_matches_restatement(ratio, fmt):
    from kapre_b200 import ops
    x = _signal(fmt, 2, 2, 12000, seed=7).requires_grad_()
    Lo = SR.output_length(12000, ratio) + 17
    y = ops.sinc_resample(x, ratio, Lo, 1.25, fmt)
    g = (torch.rand(y.shape, generator=torch.Generator().manual_seed(1)) * 2 - 1).cuda()
    (gx,) = torch.autograd.grad(y, x, g)
    xr = x.detach().cpu().double().requires_grad_()
    yr = SR.resample(xr.transpose(1, 2) if fmt == CL else xr, ratio, Lo, 1.25)
    gr = g.cpu().double()
    (want,) = torch.autograd.grad(yr, xr, gr.transpose(1, 2) if fmt == CL else gr)
    _close(gx, want, ratio, 1.0, adjoint=True)


def test_adjoint_identity_at_bench_shape():
    """<A x, g> = <x, A^T g> for 256 x 5 s at 22.05 kHz, ratio 2^(-4/12)."""
    from kapre_b200 import ops
    ratio = 2.0 ** (-4 / 12)
    x = _signal(CF, 256, 1, 110250, seed=9)
    Lo = SR.output_length(110250, ratio)
    y = ops.sinc_resample(x, ratio, Lo, 0.0, CF)
    g = torch.rand(y.shape, device='cuda') * 2 - 1
    gx = ops.sinc_resample_backward(g, ratio, 0.0, CF, x.shape[2])
    lhs = float((y.double() * g.double()).sum())
    rhs = float((x.double() * gx.double()).sum())
    assert abs(lhs - rhs) <= 1e-5 * float(y.double().norm() * g.double().norm())


def _cfg2_mel():
    import kapre_b200
    return kapre_b200.get_melspectrogram_layer(n_fft=1024, hop_length=256, sample_rate=22050, n_mels=128,
                                               return_decibel=True, input_data_format=CL, output_data_format=CL)


def test_speed_keeps_the_fused_launch():
    from kapre_b200 import _native as N
    from kapre_b200.composed import Sequential
    from kapre_b200.signal import Speed
    mel = _cfg2_mel()
    sp = Speed(1.1, data_format=CL)
    stack = Sequential([sp, *mel.layers])
    x = _signal(CL, 8, 1, 44100, seed=4)
    torch.cuda.synchronize()
    n0 = N.launch_count()
    want = mel(sp(x))
    n1 = N.launch_count()
    got = stack(x)
    n2 = N.launch_count()
    assert torch.equal(got, want)
    assert n1 - n0 == 3 and n2 - n1 == 3         # interpolation + fused log-mel + decibel clamp
    host = stack.predict(x.cpu().numpy(), batch_size=4)
    assert np.array_equal(host, want.cpu().numpy())
    cap = stack.capture(x)
    out = cap(x)
    torch.cuda.synchronize()
    assert torch.equal(out, want)


def test_requires_grad_keeps_bits_and_launches():
    from kapre_b200 import _native as N
    from kapre_b200.composed import Sequential
    from kapre_b200.signal import Speed
    stack = Sequential([Speed(0.9, data_format=CL), *_cfg2_mel().layers])
    x = _signal(CL, 4, 1, 48000, seed=6)
    n0 = N.launch_count()
    plain = stack(x)
    n1 = N.launch_count()
    xg = x.clone().requires_grad_()
    tracked = stack(xg)
    n2 = N.launch_count()
    assert torch.equal(plain, tracked) and n1 - n0 == n2 - n1 == 3
    assert tracked.requires_grad
    (gx,) = torch.autograd.grad(tracked.sum(), xg)
    assert gx.shape == x.shape and torch.isfinite(gx).all() and float(gx.abs().max()) > 0


def test_a_new_factor_per_call_creates_no_state():
    from kapre_b200 import _native as N, ops
    from kapre_b200.signal import Speed
    layer = Speed(1.1, data_format=CF)
    x = _signal(CF, 2, 1, 16000, seed=8)
    layer(x)
    n0 = N.launch_count()
    factors = np.random.default_rng(0).uniform(0.8, 1.25, size=20)
    for f in factors:
        y = layer(x, factor=float(f))
        assert y.shape == (2, 1, math.ceil(16000 / float(f)))
    assert N.launch_count() - n0 == 20
    assert len(ops._sinc_plan._per_device) == 1
    _close(y, _ref(x, CF, 1.0 / float(factors[-1]), y.shape[2]), 1.0 / float(factors[-1]), 1.0)


# ------------------------------------------------------------------------------------------ PitchShift
def _pitch_shift(n_steps, fmt=CL, n_fft=1024, hop=256):
    from kapre_b200.augmentation import PitchShift
    return PitchShift(n_steps, n_fft=n_fft, hop_length=hop, window_name='hann_window', data_format=fmt)


@pytest.mark.parametrize('n_steps', [-5, 4, 0.5])
def test_pitch_shift_on_a_sinusoid(n_steps):
    sr, f0, n_fft = 16000, 440.0, 1024
    t = torch.arange(sr, dtype=torch.float64) / sr
    x64 = torch.sin(2 * math.pi * f0 * t).view(1, -1, 1)
    layer = _pitch_shift(n_steps)
    x = x64.float().cuda()
    y = layer(x)
    assert y.shape == x.shape
    mid = y[0, n_fft:sr - n_fft, 0].double().cpu()
    spec = torch.fft.rfft(mid * torch.hann_window(mid.numel(), dtype=torch.float64)).abs()
    f_peak = float(spec.argmax()) * sr / mid.numel()
    assert abs(f_peak - f0 * 2.0 ** (n_steps / 12)) <= sr / n_fft, f_peak
    # and the float64 chain, where the phase vocoder is well conditioned (away from the zero-padded ends)
    want = SR.pitch_shift(x64, n_steps, n_fft=n_fft, hop=256, window_name='hann_window')
    err = (y.double().cpu() - want)[0, 2 * n_fft:sr - 2 * n_fft, 0].abs().max()
    assert float(err) <= 5e-3, float(err)
    assert layer(x, n_steps=0) is x
    both = _pitch_shift(n_steps, CF)(x.transpose(1, 2).contiguous())
    assert torch.equal(both.transpose(1, 2), y)


@pytest.mark.parametrize('n_steps', [-5, 4])
def test_pitch_shift_is_time_aligned(n_steps):
    """A tone burst comes out within hop_length of where it was, a click within half a window (see PitchShift)."""
    n_fft, hop, L = 1024, 256, 12000
    t = torch.arange(L, dtype=torch.float64)
    layer = _pitch_shift(n_steps)
    for i in (4000, 6555):
        burst = (torch.exp(-0.5 * ((t - i) / 600) ** 2) * torch.sin(0.1 * math.pi * t)).view(1, -1, 1)
        y = layer(burst.float().cuda())[0, :, 0].double().cpu()
        assert abs(float((y * y * t).sum() / (y * y).sum()) - i) <= hop
        click = torch.zeros((1, L, 1))
        click[0, i, 0] = 1.0
        y = layer(click.cuda())[0, :, 0].double().cpu()
        env = torch.nn.functional.avg_pool1d((y * y).view(1, 1, -1), hop + 1, 1, hop // 2).view(-1)
        assert abs(int(env.argmax()) - i) <= n_fft // 2


def test_pitch_shift_gradient_from_waveform():
    """Waveform -> PitchShift against float64 autograd of the restated chain."""
    layer = _pitch_shift(4, n_fft=512, hop=128)
    g = torch.Generator().manual_seed(5)
    x = (torch.rand((2, 8000, 1), generator=g) * 2 - 1).cuda().requires_grad_()
    y = layer(x)
    assert y.shape == x.shape and y.requires_grad
    gy = torch.randn(y.shape, generator=g).cuda()
    got, = torch.autograd.grad(y, x, gy)
    xr = x.detach().cpu().double().requires_grad_()
    want, = torch.autograd.grad(SR.pitch_shift(xr, 4, n_fft=512, hop=128, window_name='hann_window'), xr, gy.cpu().double())
    err = float((got.cpu().double() - want).abs().max())
    assert err <= 2e-3 * float(want.abs().max()), (err, float(want.abs().max()))


def test_pitch_shift_through_sequential_and_capture():
    from kapre_b200 import _native as N
    from kapre_b200.composed import Sequential
    layer = _pitch_shift(-3)
    x = _signal(CL, 32, 2, 22050, seed=12)          # 32 x 2 x 513 columns: the time stretch is one launch
    want = layer(x)
    stack = Sequential([layer])
    torch.cuda.synchronize()
    n0 = N.launch_count()
    assert torch.equal(stack(x), want)
    assert N.launch_count() - n0 == 4            # STFT, time stretch, inverse STFT, interpolation
    cap = stack.capture(x)
    out = cap(x)
    torch.cuda.synchronize()
    assert torch.equal(out, want)
