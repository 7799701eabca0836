"""The polyphase resampler on the GPU: parity with the float64 restatement (resample_ref.py) at 10 s signals, its
vector-Jacobian product, and a ``Resample`` layer in front of the fused log-mel launch.  No scipy needed."""
import numpy as np
import pytest
import torch

import resample_ref as RR

pytestmark = pytest.mark.gpu
CL, CF = 'channels_last', 'channels_first'


def _signal(fmt, B, C, L, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.rand((B, L, C) if fmt == CL else (B, C, L), generator=g) * 2 - 1
    return x.cuda()


def _ref(x, fmt, up, down, length=None):
    t = x.detach().cpu().double()
    if fmt == CL:
        return RR.resample(t.transpose(1, 2), up, down, length=length).transpose(1, 2)
    return RR.resample(t, up, down, length=length)


def _close(got, want, scale, tol=1e-5):
    assert tuple(got.shape) == tuple(want.shape), (tuple(got.shape), tuple(want.shape))
    if got.numel():
        err = float((got.detach().cpu().double() - want).abs().max())
        assert err <= tol * scale, (err, scale)


@pytest.mark.parametrize('orig,target', RR.COMMON_PAIRS)
@pytest.mark.parametrize('fmt', [CF, CL])
def test_parity_10s(orig, target, fmt):
    from kapre_b200.signal import Resample
    x = _signal(fmt, 2, 2, 10 * orig, seed=orig + target)
    y = Resample(orig, target, data_format=fmt)(x)
    up, down = RR.up_down(orig, target)
    _close(y, _ref(x, fmt, up, down), float(x.abs().max()))


@pytest.mark.parametrize('fmt', [CF, CL])
def test_parity_views_and_short_signals(fmt):
    from kapre_b200.signal import Resample
    layer = Resample(44100, 16000, data_format=fmt)
    full = _signal(fmt, 4, 3, 20000, seed=3)
    t_ax = 1 if fmt == CL else 2
    views = [full.narrow(t_ax, 5, 9000), full[::2], full.narrow(3 - t_ax, 1, 1), full.narrow(t_ax, 0, 1),
             full.narrow(t_ax, 0, 0), full.narrow(t_ax, 0, 50), full.transpose(1, 2).contiguous().transpose(1, 2)]
    for x in views:
        y = layer(x)
        _close(y, _ref(x, fmt, 160, 441), max(float(x.abs().max()) if x.numel() else 1.0, 1e-30))


def test_equal_rates_return_the_input():
    from kapre_b200 import _native as N
    from kapre_b200.signal import Resample
    x = _signal(CL, 2, 1, 100)
    n0 = N.launch_count()
    assert Resample(16000, 16000, data_format=CL)(x) is x
    assert N.launch_count() == n0


def test_unsupported_ratio_is_an_error():
    from kapre_b200 import _native as N
    from kapre_b200.signal import Resample
    with pytest.raises(N.KapreNativeError, match='max\\(up, down\\)'):
        Resample(44100, 44099)(_signal(CL, 1, 1, 100))


@pytest.mark.parametrize('orig,target', [(48000, 16000), (44100, 16000), (16000, 22050)])
@pytest.mark.parametrize('fmt', [CF, CL])
def test_vjp_matches_restatement(orig, target, fmt):
    from kapre_b200.signal import Resample
    up, down = RR.up_down(orig, target)
    x = _signal(fmt, 2, 2, orig // 2, seed=7).requires_grad_()
    y = Resample(orig, target, data_format=fmt)(x)
    g = torch.randn(y.shape, generator=torch.Generator().manual_seed(1)).cuda()
    (gx,) = torch.autograd.grad(y, x, g)
    xr = x.detach().cpu().double().requires_grad_()
    yr = RR.resample(xr.transpose(1, 2) if fmt == CL else xr, up, down)
    gr = g.cpu().double()
    (want,) = torch.autograd.grad(yr, xr, gr.transpose(1, 2) if fmt == CL else gr)
    _close(gx, want, float(want.abs().max()))


def test_adjoint_identity_at_bench_shape():
    """<A x, g> = <x, A^T g> for 256 x 10 s at 48 kHz -> 16 kHz (tools/resample_bench.py's first case)."""
    from kapre_b200 import ops
    from kapre_b200.signal import Resample
    layer = Resample(48000, 16000, data_format=CF)
    x = _signal(CF, 256, 1, 480000, seed=9)
    y = ops.resample(x, layer.plan, CF)
    g = torch.rand(y.shape, device='cuda') * 2 - 1
    gx = ops.resample_backward(g, layer.plan, CF, x.shape[2])
    lhs = float((y.double() * g.double()).sum())
    rhs = float((x.double() * gx.double()).sum())
    assert abs(lhs - rhs) <= 1e-5 * float(y.double().norm() * g.double().norm())


def _cfg2_mel():
    import kapre_b200
    return kapre_b200.get_melspectrogram_layer(n_fft=1024, hop_length=256, sample_rate=22050, n_mels=128,
                                               return_decibel=True, input_data_format=CL, output_data_format=CL)


def test_resample_keeps_the_fused_launch():
    from kapre_b200 import _native as N
    from kapre_b200.composed import Sequential
    from kapre_b200.signal import Resample
    mel = _cfg2_mel()
    rs = Resample(44100, 22050, data_format=CL)
    stack = Sequential([rs, *mel.layers])
    x = _signal(CL, 8, 1, 44100 * 2, seed=4)
    torch.cuda.synchronize()
    n0 = N.launch_count()
    want = mel(rs(x))
    n1 = N.launch_count()
    got = stack(x)
    n2 = N.launch_count()
    assert torch.equal(got, want)
    assert n1 - n0 == 3 and n2 - n1 == 3         # resample + fused log-mel + decibel clamp
    # predict (pipelined host path) and a captured graph run the same launches
    host = stack.predict(x.cpu().numpy(), batch_size=4)
    assert np.array_equal(host, want.cpu().numpy())
    cap = stack.capture(x)
    out = cap(x)
    torch.cuda.synchronize()
    assert torch.equal(out, want)


def test_requires_grad_keeps_bits_and_launches():
    from kapre_b200 import _native as N
    from kapre_b200.composed import Sequential
    from kapre_b200.signal import Resample
    mel = _cfg2_mel()
    stack = Sequential([Resample(48000, 22050, data_format=CL), *mel.layers])
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
