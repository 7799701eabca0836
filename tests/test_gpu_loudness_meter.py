"""The loudness meter on the GPU: loudness_stats and true_peak end to end within the CPU tier's bounds, integrated
loudness bit for bit equal to loudness, true peak against the Resample(4, 1) + amax composition, independence of batch
position, strides, format and lengths, gradients, the peak-limited LoudnessNormalization, CUDA graph capture, launch
counts, and invalid arguments raising before any launch."""
import math

import numpy as np
import pytest
import torch

import loudness_meter_ref as MR

pytestmark = pytest.mark.gpu

CF, CL = 'channels_first', 'channels_last'


def _x(shape, seed, scale=0.1):
    g = torch.Generator(device='cuda').manual_seed(seed)
    return torch.randn(shape, device='cuda', generator=g) * scale


def _bcl(t, fmt):
    a = t.detach().double().cpu().numpy()
    return a.transpose(0, 2, 1) if fmt == CL else a


def _levels(B, fmt, C, L, sr, seed):
    """Noise whose level differs per item and changes every second, so both gates of the range act; below full scale,
    so the K-weighting's clamps stay inactive and its error bound tight."""
    shape = (B, C, L) if fmt == CF else (B, L, C)
    x = _x(shape, seed, 0.02)
    t = torch.arange(L, device='cuda')
    env = torch.where((t // sr) % 3 == 1, 0.05, 1.0) * (1 + (t // sr) % 5) * torch.linspace(0.1, 1.0, B, device='cuda')[:, None]
    return x * (env[:, None, :] if fmt == CF else env[:, :, None])


def _composition(x, fmt, lengths=None):
    """true peak by Resample(4, 1) and amax over each item's valid outputs."""
    from kapre_b200 import ops
    from kapre_b200.signal import resample_filter
    plan = ops.ResamplePlan(4, 1, resample_filter(4, 1))
    B = x.shape[0]
    out = []
    for b in range(B):
        xb = x[b:b + 1]
        if lengths is not None:
            n = int(lengths[b])
            xb = xb[:, :n] if fmt == CL else xb[:, :, :n]
        z = ops.resample(xb.contiguous(), plan, fmt)
        out.append((20 * torch.log10(z.abs().amax(dim=1 if fmt == CL else 2).double())).float())
    return torch.cat(out)


@pytest.mark.parametrize('sr, fmt, C', [(8000, CF, 1), (11025, CL, 2), (16000, CF, 5), (44100, CL, 2), (48000, CF, 2)])
def test_end_to_end_within_bound(sr, fmt, C):
    from kapre_b200.signal import loudness, loudness_stats
    B, L = 3, int(6.3 * sr)
    x = _levels(B, fmt, C, L, sr, 1)
    lengths = torch.tensor([L, int(4.1 * sr), int(2.5 * sr)], device='cuda')
    got = loudness_stats(x, sr, lengths, data_format=fmt)
    G, S, G3 = MR.geometry(sr)
    ln = lengths.cpu().numpy()
    xa = _bcl(x, fmt)
    # the meter's own input: the K-weighting by the same two lfilter launches, so the bounds cover the meter kernels
    from kapre_b200 import ops
    (b1, a1), (b2, a2) = ops.k_weighting(sr, x.device)
    y = ops.lfilter(ops.lfilter(x, b1, a1, clamp=True, data_format=fmt), b2, a2, clamp=True, data_format=fmt)
    y, delta = _bcl(y, fmt), 0.0
    assert torch.equal(got.integrated, loudness(x, sr, lengths, data_format=fmt))
    for W, s in ((G, got.momentary), (G3, got.short_term)):
        s = s.cpu().numpy()
        want = MR.series(y, W, S, ln)
        assert s.shape == want.shape
        fin = np.isfinite(want)
        assert np.array_equal(np.isneginf(s), ~fin)
        assert np.all(np.abs(s[fin] - want[fin]) <= MR.series_bound(y, W, S, delta, ln)[fin])
    want = MR.loudness_range(y, G3, S, ln)
    bound = MR.lra_bound(y, G3, S, delta, ln)
    assert np.all(MR.lra_margin(y, G3, S, ln) > 10 * bound)
    assert np.all(np.abs(got.loudness_range.cpu().numpy() - want) <= bound), (got.loudness_range, want, bound)
    tp = got.true_peak.cpu().numpy()
    assert np.all(np.abs(tp - MR.true_peak(xa, ln)) <= MR.true_peak_bound(xa, ln))
    # the composition: the same float32 z, so the same maximum; the two float64 log10s may differ in the last bit
    comp = _composition(x, fmt, ln)
    assert ((got.true_peak - comp).abs() <= comp.abs() * 2.0 ** -23).all()


def test_short_silent_nan_items_and_independence():
    from kapre_b200.signal import loudness_stats, true_peak
    sr = 16000
    B, C, L = 5, 2, int(4.5 * sr)
    x = _levels(B, CF, C, L, sr, 3)
    x[3] = 0
    x[4, 1, 3 * sr] = float('nan')
    lengths = torch.tensor([L, 6000, 40000, L, L], device='cuda')      # full, < G, < G3, silent, NaN
    got = loudness_stats(x, sr, lengths, data_format=CF)
    assert torch.isneginf(got.momentary[1]).all() and torch.isneginf(got.short_term[1:4]).all()
    assert (got.loudness_range[1:4] == 0).all() and torch.isneginf(got.true_peak[3]).all()
    assert torch.isnan(got.integrated[4]) and torch.isnan(got.loudness_range[4]) and torch.isnan(got.true_peak[4, 1])
    assert torch.isfinite(got.integrated[[0, 2]]).all() and torch.isfinite(got.true_peak[4, 0])
    # an item alone, at another position, channels_last, strided, and cut to its length
    cl = x.transpose(1, 2).contiguous()
    other = loudness_stats(cl, sr, lengths, data_format=CL)
    big = torch.zeros((B, C + 2, L + 9), device='cuda')
    big[:, 1:C + 1, 4:4 + L] = x
    strided = loudness_stats(big[:, 1:C + 1, 4:4 + L], sr, lengths, data_format=CF)
    rev = loudness_stats(x.flip(0), sr, lengths.flip(0), data_format=CF)
    for a, b, c, d in zip(got, other, strided, rev):
        assert torch.equal(a.nan_to_num(), b.nan_to_num()) and torch.equal(a.nan_to_num(), c.nan_to_num())
        assert torch.equal(a.nan_to_num(), d.flip(0).nan_to_num())
    for b in (0, 2):
        n = int(lengths[b])
        alone = loudness_stats(x[b:b + 1, :, :n].contiguous(), sr, data_format=CF)
        assert torch.equal(alone.integrated, got.integrated[b:b + 1])
        assert torch.equal(alone.loudness_range, got.loudness_range[b:b + 1])
        assert torch.equal(alone.true_peak, got.true_peak[b:b + 1])
        assert torch.equal(alone.short_term[0], got.short_term[b, :alone.short_term.shape[1]])
    mixed = lengths.clone()
    mixed[1] = L
    assert torch.equal(loudness_stats(x, sr, mixed, data_format=CF).loudness_range[0], got.loudness_range[0])
    assert torch.equal(true_peak(x, lengths, data_format=CF).nan_to_num(), got.true_peak.nan_to_num())


@pytest.mark.parametrize('fmt', [CF, CL])
def test_true_peak_gradient_is_the_float64_vjp(fmt):
    from kapre_b200.signal import true_peak
    B, C, L = 2, 3, 7000
    x = _x((B, C, L) if fmt == CF else (B, L, C), 4, 0.3)
    if fmt == CF:
        x[1, 2] = 0
    else:
        x[1, :, 2] = 0
    lengths = torch.tensor([L, 5000], device='cuda')
    xr = x.clone().requires_grad_(True)
    tp = true_peak(xr, lengths, data_format=fmt)
    assert torch.equal(tp.detach(), true_peak(x, lengths, data_format=fmt))
    g = torch.tensor([[0.7, -1.3, 2.0], [0.5, 1.5, -0.2]], device='cuda')
    tp.backward(g)
    got = _bcl(xr.grad, fmt)
    want = MR.true_peak_vjp(_bcl(x, fmt).astype(np.float32), g.cpu().numpy(), lengths.cpu().numpy())
    assert np.all(got[1, 2] == 0)
    assert np.all(np.abs(got - want) <= 1e-4 * np.abs(want).max())


def _peaky(B, L, sr, seed):
    """Stereo items: steady noise with a few sharp clicks, so the true-peak limit binds at loud targets."""
    x = _x((B, L, 2), seed, 0.05)
    x[:, ::4000] += 0.4
    return x


def test_peak_limited_normalisation():
    from kapre_b200 import _native as N
    from kapre_b200.augmentation import LoudnessNormalization
    from kapre_b200.signal import true_peak
    sr, B, L = 16000, 4, 3 * 16000
    x = _peaky(B, L, sr, 5)
    x[3] = 0                                                            # -inf loudness: unchanged
    lufs = [-14.0, -40.0, -9.0, -14.0]
    plain = LoudnessNormalization(sr, data_format=CL)
    limited = LoudnessNormalization(sr, data_format=CL, true_peak_limit=-1.0)
    a = plain.call(x, lufs=lufs)
    torch.cuda.synchronize()
    n0 = N.launch_count()
    b = limited.call(x, lufs=lufs)
    assert N.launch_count() - n0 == 10 + 2                               # loudness and true peak
    tp_out = true_peak(b, data_format=CL).amax(dim=1)
    binds = true_peak(a, data_format=CL).amax(dim=1) > -1.0
    assert binds[0] and binds[2] and not binds[1]
    assert (tp_out[:3] <= -1.0 + 1e-4).all()
    for i in range(3):
        if not binds[i]:
            assert torch.equal(a[i], b[i])
        else:
            assert abs(float(tp_out[i]) + 1.0) < 1e-3
    assert torch.equal(b[3], x[3])


def test_peak_limited_gradients():
    from kapre_b200.augmentation import LoudnessNormalization
    from kapre_b200.signal import true_peak
    sr, B, L = 16000, 2, 2 * 16000
    x = _peaky(B, L, sr, 6)
    lufs = [-40.0, -9.0]                                                 # item 0: loudness binds; item 1: the limit
    w = _x((B, L, 2), 7)
    plain = LoudnessNormalization(sr, data_format=CL)
    limited = LoudnessNormalization(sr, data_format=CL, true_peak_limit=-1.0)
    xa = x.clone().requires_grad_(True)
    (plain.call(xa, lufs=lufs) * w).sum().backward()
    xb = x.clone().requires_grad_(True)
    out = limited.call(xb, lufs=lufs)
    (out * w).sum().backward()
    torch.testing.assert_close(xb.grad[0], xa.grad[0], rtol=1e-6, atol=0)
    # where the limit binds: out = x 10^((limit - TP) / 20), TP = tp_c* (the larger channel)
    tp = true_peak(x, data_format=CL)[1]
    c = int(torch.argmax(tp))
    gain = 10 ** ((-1.0 - float(tp[c])) / 20)
    xs = x[1].double().cpu().numpy().T[None]
    ws = w[1].double().cpu().numpy().T
    s = float((ws * xs[0]).sum())
    gtp = np.zeros((1, 2))
    gtp[0, c] = 1.0
    dtp = MR.true_peak_vjp(xs.astype(np.float32), gtp)[0]
    want = ws * gain - s * gain * math.log(10) / 20 * dtp
    got = xb.grad[1].double().cpu().numpy().T
    assert np.all(np.abs(got - want) <= 1e-4 * np.abs(want).max())


def test_graph_capture_and_launch_counts():
    from kapre_b200 import _native as N
    from kapre_b200.augmentation import LoudnessNormalization
    from kapre_b200.signal import loudness_stats, true_peak
    sr, B, L = 16000, 3, 5 * 16000
    x = _levels(B, CF, 2, L, sr, 8)
    lengths = torch.tensor([L, 50000, 30000], device='cuda')
    eager = loudness_stats(x, sr, lengths, data_format=CF)
    torch.cuda.synchronize()
    n0 = N.launch_count()
    loudness_stats(x, sr, lengths, data_format=CF)
    assert N.launch_count() - n0 == 16                                   # 8 K-weighting + 6 meter + 2 true peak
    n0 = N.launch_count()
    true_peak(x, data_format=CF)
    assert N.launch_count() - n0 == 2
    xr = x.clone().requires_grad_(True)
    tp = true_peak(xr, data_format=CF)
    n0 = N.launch_count()
    tp.sum().backward()
    assert N.launch_count() - n0 == 1
    layer = LoudnessNormalization(sr, data_format=CF, true_peak_limit=-1.0)
    xs = x.clone()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        loudness_stats(xs, sr, lengths, data_format=CF)
        layer.call(xs, lufs=-12.0)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        st = loudness_stats(xs, sr, lengths, data_format=CF)
        y = layer.call(xs, lufs=-12.0)
    xs.copy_(x * 0.5)
    g.replay()
    torch.cuda.synchronize()
    want = loudness_stats(x * 0.5, sr, lengths, data_format=CF)
    for a, b in zip(st, want):
        assert torch.equal(a, b)
    assert torch.equal(y, layer.call(x * 0.5, lufs=-12.0))
    assert not torch.equal(st.integrated, eager.integrated)


def test_no_gradient_and_invalid_arguments_raise_before_any_launch():
    from kapre_b200 import _native as N
    from kapre_b200.signal import loudness_stats, true_peak
    x = _x((2, 8000, 2), 9)
    torch.cuda.synchronize()
    n0 = N.launch_count()
    with pytest.raises(ValueError, match='loudness and true_peak'):
        loudness_stats(x.clone().requires_grad_(True), 16000, data_format=CL)
    for args, kw in (((_x((2, 8000, 6), 1), 16000), {}), ((x, 3000), {}), ((x[0], 16000), {}),
                     ((x, 16000), dict(lengths=torch.ones(3, dtype=torch.int64, device='cuda'))),
                     ((x, 16000), dict(lengths=1.5))):
        with pytest.raises(ValueError):
            loudness_stats(*args, data_format=CL, **kw)
    for args, kw in (((x[0],), {}), ((_x((2, 8000, 0), 1),), {}), ((x,), dict(lengths=[1, 2, 3]))):
        with pytest.raises(ValueError):
            true_peak(*args, data_format=CL, **kw)
    with pytest.raises(N.KapreNativeError):
        true_peak(x.cpu(), data_format=CL)
    assert N.launch_count() == n0
    with torch.no_grad():
        loudness_stats(x.clone().requires_grad_(True), 16000, data_format=CL)
