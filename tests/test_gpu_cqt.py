"""The constant-Q transform on the H100: forward (complex and magnitude) and backward against the float64
restatement (cqt_ref.py) within its derived bound at benchmark size in both formats, B = 36, stereo 44.1 kHz
channels_last and a 10-minute recording; the gradient through get_cqt_layer(return_decibel=True); bit equality across
batch positions, batch sizes and strides; launch counts with and without requires_grad; capture replays; the
waveform layers ahead of the fused CQT -> Magnitude launch."""
import numpy as np
import pytest
import torch

import cqt_ref as R

pytestmark = pytest.mark.gpu

CL, CF = 'channels_last', 'channels_first'


def _x(B, C, L, seed, sr):
    rng = np.random.default_rng(seed)
    t = np.arange(L) / sr
    x = 0.1 * rng.standard_normal((B, C, L))
    x += 0.4 * np.sin(2 * np.pi * rng.uniform(40, sr / 3, size=(B, C, 1)) * t + rng.uniform(0, 6, (B, C, 1)))
    return torch.from_numpy(x.astype(np.float32)).cuda()


def _layer(**kw):
    from kapre_b200.time_frequency import CQT
    return CQT(**kw)


def _cf(y, fmt):
    """(B, M, K, C) -> (B, C, M, K)."""
    return y.permute(0, 3, 1, 2) if fmt == CL else y


def _check(x_cf, plan, y_cf, items, magnitude=False):
    for b in items:
        xb = x_cf[b:b + 1].double().cpu()
        ref = R.cqt(xb, plan, magnitude).numpy()
        bound = R.forward_bound(xb, plan, magnitude).numpy()
        got = y_cf[b:b + 1].cpu().numpy()
        err = np.abs(got.astype(np.complex128 if not magnitude else np.float64) - ref)
        bad = err > bound
        assert not bad.any(), (b, float(err[bad].max()), float(bound[bad].min()), int(bad.sum()))


@pytest.mark.parametrize('fmt', [CL, CF])
def test_benchmark_size_both_formats(fmt):
    x = _x(256, 1, 5 * 22050, 0, 22050)
    q = _layer(input_data_format=fmt, output_data_format=fmt)
    xin = x.transpose(1, 2).contiguous() if fmt == CL else x
    y = q(xin)
    assert y.dtype == torch.complex64 and y.shape == ((256, 216, 84, 1) if fmt == CL else (256, 1, 216, 84))
    _check(x, q.plan, _cf(y, fmt), [0, 131, 255])
    ym = q.call(xin, magnitude=True)
    _check(x, q.plan, _cf(ym, fmt), [0, 255], magnitude=True)
    # an item's bits do not depend on its position, the batch size or the strides
    yc = _cf(y, fmt)
    np.testing.assert_array_equal(_cf(q(xin[131:132]), fmt).cpu().numpy(), yc[131:132].cpu().numpy())
    rev = q(torch.flip(xin, [0]).contiguous())
    np.testing.assert_array_equal(_cf(rev, fmt)[255 - 7].cpu().numpy(), yc[7].cpu().numpy())
    big = torch.zeros((256, 1, 2 * x.shape[2]), device='cuda')
    big[:, :, ::2] = x
    view = big[:, :, ::2].transpose(1, 2) if fmt == CL else big[:, :, ::2]
    np.testing.assert_array_equal(_cf(q(view), fmt).cpu().numpy(), yc.cpu().numpy())


def test_b36_252_bins():
    x = _x(8, 1, 3 * 22050, 1, 22050)
    q = _layer(n_bins=252, bins_per_octave=36, input_data_format=CF, output_data_format=CF)
    _check(x, q.plan, q(x), [0, 7])


def test_stereo_44k_channels_last():
    x = _x(4, 2, 4 * 44100, 2, 44100)
    q = _layer(sample_rate=44100, hop_length=1024, n_bins=96, input_data_format=CL, output_data_format=CL)
    y = q(x.transpose(1, 2).contiguous())
    _check(x, q.plan, _cf(y, CL), [0, 3])


def test_ten_minute_recording():
    x = _x(1, 1, 600 * 22050, 3, 22050)
    q = _layer(input_data_format=CF, output_data_format=CF)
    _check(x, q.plan, q.call(x, magnitude=True), [0], magnitude=True)


@pytest.mark.parametrize('magnitude', [False, True])
def test_backward_within_bound(magnitude):
    from kapre_b200 import ops
    x = _x(3, 1, 2 * 22050, 4, 22050)
    q = _layer(input_data_format=CF, output_data_format=CF)
    xg = x.clone().requires_grad_(True)
    y = ops.cqt(xg, q.plan, CF, CF, magnitude)
    rng = np.random.default_rng(5)
    g = rng.standard_normal(tuple(y.shape)) + (1j * rng.standard_normal(tuple(y.shape)) if not magnitude else 0)
    gt = torch.from_numpy(g.astype(np.float32 if magnitude else np.complex64)).cuda()
    y.backward(gt)
    for b in (0, 2):
        xb = x[b:b + 1].double().cpu()
        gb = gt[b:b + 1].cpu().to(torch.float64 if magnitude else torch.complex128)
        ref = R.vjp(xb, q.plan, gb, magnitude).numpy()
        bound = R.backward_bound(xb, q.plan, gb, magnitude).numpy()
        err = np.abs(xg.grad[b:b + 1].cpu().numpy() - ref)
        bad = err > bound
        assert not bad.any(), (b, float(err[bad].max()), float(bound[bad].min()), int(bad.sum()))
    # the gradient's bits do not depend on the item's batch position
    x1 = x[2:3].clone().requires_grad_(True)
    ops.cqt(x1, q.plan, CF, CF, magnitude).backward(gt[2:3])
    assert torch.equal(x1.grad, xg.grad[2:3])


def test_backward_through_decibel_layer():
    from kapre_b200 import ops
    from kapre_b200.composed import get_cqt_layer
    x = _x(2, 1, 22050, 6, 22050)
    model = get_cqt_layer(return_decibel=True, input_data_format=CF, output_data_format=CF)
    xg = x.clone().requires_grad_(True)
    y = model(xg)
    g = torch.randn(y.shape, device='cuda', generator=torch.Generator('cuda').manual_seed(0))
    y.backward(g)
    plan = model.layers[0].plan
    C, ws = ops.cqt_forward(x, plan, CF, CF, True)
    gm = ops.magnitude_to_decibel_backward(C, g)
    want = ops.cqt_backward(gm, x, ws, plan, CF, CF, True)
    assert torch.equal(xg.grad, want)
    assert torch.isfinite(xg.grad).all() and xg.grad.abs().max() > 0


def test_launch_counts_and_capture():
    from kapre_b200 import _native as N
    from kapre_b200 import ops
    from kapre_b200.composed import Sequential
    from kapre_b200.time_frequency import Magnitude
    x = _x(4, 1, 22050, 7, 22050)
    q = _layer(input_data_format=CF, output_data_format=CF)
    y0 = q(x)
    torch.cuda.synchronize()
    n0 = N.launch_count()
    q(x)
    assert N.launch_count() - n0 == 7
    xg = x.clone().requires_grad_(True)
    n0 = N.launch_count()
    y1 = q(xg)
    assert N.launch_count() - n0 == 7 and torch.equal(y0, y1.detach())
    n0 = N.launch_count()
    y1.abs().sum().backward()
    assert N.launch_count() - n0 >= 13     # 13 of the CQT backward, plus torch's own abs backward
    n0 = N.launch_count()
    ops.cqt_backward(torch.ones_like(y0), x, None, q.plan, CF, CF, False)
    assert N.launch_count() - n0 == 13
    s = Sequential([q, Magnitude()])
    m0 = s(x)
    n0 = N.launch_count()
    m1 = s(xg)
    assert N.launch_count() - n0 == 7 and torch.equal(m0, m1.detach())
    np.testing.assert_allclose(m0.cpu().numpy(), y0.abs().cpu().numpy(), rtol=2e-6, atol=1e-6)
    cap = Sequential([q, Magnitude()]).capture(x)
    r1 = cap(x).clone()
    assert torch.equal(r1, m0)
    assert torch.equal(cap(x), r1)


def test_waveform_layers_run_before_fused_cqt():
    from kapre_b200 import _native as N
    from kapre_b200.augmentation import Reverb
    from kapre_b200.composed import Sequential
    from kapre_b200.signal import Speed
    from kapre_b200.time_frequency import Magnitude
    rng = np.random.default_rng(0)
    rirs = np.exp(-np.arange(4000) / 400.0) * rng.standard_normal(4000)
    q = _layer(input_data_format=CL, output_data_format=CL)
    chain = Sequential([Speed(1.1, data_format=CL), Reverb([rirs], seed=0, data_format=CL), q, Magnitude()])
    x = _x(4, 1, 22050, 8, 22050).transpose(1, 2).contiguous()
    z = chain.call(x)
    assert z.dtype == torch.float32 and z.shape[2] == 84 and torch.isfinite(z).all()
    wave = Sequential(chain.layers[:2])
    wave.call(x)
    torch.cuda.synchronize()
    n0 = N.launch_count()
    w = wave.call(x)
    n_wave = N.launch_count() - n0
    n0 = N.launch_count()
    z = chain.call(x)
    assert N.launch_count() - n0 == n_wave + 7
    assert torch.equal(z, q.call(w, magnitude=True))


def test_invalid_arguments_raise_before_any_launch():
    from kapre_b200 import _native as N
    torch.cuda.synchronize()
    n0 = N.launch_count()
    for kw in [dict(hop_length=500), dict(sample_rate=8000), dict(gamma=-1.0), dict(n_bins=12, sample_rate=48000),
               dict(filter_scale=0.0)]:
        with pytest.raises(ValueError):
            _layer(**kw)
    assert N.launch_count() == n0
