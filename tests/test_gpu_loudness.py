"""Gated loudness on the GPU: the end-to-end result within the derived bound of the float64 restatement, parity with
torchaudio on the same card at benchmark size (mono channels_first, stereo channels_last), bit-independence of batch
position, strides, format and lengths, gradients against the float64 VJP and torchaudio's float64 autograd,
requires_grad leaving the forward unchanged, launch counts, LoudnessNormalization (targets, -inf items, Sequential before
the fused log-mel, graph capture), and invalid arguments raising before any launch."""
import numpy as np
import pytest
import torch

import loudness_ref as LR

pytestmark = pytest.mark.gpu

CF, CL = 'channels_first', 'channels_last'


def _x(shape, seed, scale=0.1):
    g = torch.Generator(device='cuda').manual_seed(seed)
    return torch.randn(shape, device='cuda', generator=g) * scale


def _bcl(t, fmt):
    a = t.detach().double().cpu().numpy()
    return a.transpose(0, 2, 1) if fmt == CL else a


def _levels(B, fmt, C, L, seed):
    """Noise whose level differs per item and changes every second (so that both gates act)."""
    shape = (B, C, L) if fmt == CF else (B, L, C)
    x = _x(shape, seed)
    t = torch.arange(L, device='cuda')
    env = torch.where((t // 8000) % 3 == 1, 0.02, 1.0) * torch.linspace(0.3, 3.0, B, device='cuda')[:, None]
    return x * (env[:, None, :] if fmt == CF else env[:, :, None])


@pytest.mark.parametrize('sr, fmt, C', [(11025, CF, 2), (16000, CL, 1), (48000, CL, 5), (8000, CF, 3)])
def test_end_to_end_within_bound(sr, fmt, C):
    from kapre_b200.signal import loudness
    B, L = 4, int(3.3 * sr)
    x = _levels(B, fmt, C, L, 1)
    lengths = torch.tensor([L, L - 1000, int(0.4 * sr) + 7, 2 * sr], device='cuda')
    got = loudness(x, sr, lengths, data_format=fmt).cpu().numpy()
    coeffs = LR.normalised(LR.k_weighting(sr))
    xa = _bcl(x, fmt)
    y = LR.weight(xa, coeffs)
    G, S = LR.geometry(sr)
    ln = lengths.cpu().numpy()
    want = LR.gated(y, G, S, ln)[0]
    assert (LR.gate_margin(y, G, S, ln) > 1e-3).all()
    bound = LR.lkfs_bound(y, G, S, LR.weighting_error(xa, coeffs), ln)
    assert (np.abs(got - want) <= bound).all(), (got, want, bound)


@pytest.mark.parametrize('B, secs, sr, C, fmt', [(256, 5, 16000, 1, CF), (32, 10, 48000, 2, CL)])
def test_against_torchaudio_on_the_same_card(B, secs, sr, C, fmt):
    F = pytest.importorskip('torchaudio.functional')
    from kapre_b200.signal import loudness
    L = secs * sr
    shape = (B, C, L) if fmt == CF else (B, L, C)
    x = _x(shape, 2) * torch.linspace(0.05, 1.0, B, device='cuda').view(B, 1, 1)
    got = loudness(x, sr, data_format=fmt)
    ta = F.loudness(x if fmt == CF else x.transpose(1, 2), sr)
    G, S = LR.geometry(sr)
    assert (LR.gate_margin(LR.weight(_bcl(x, fmt), LR.k_weighting(sr)), G, S) >= 0.1).all()
    assert torch.isfinite(got).all()
    assert (got - ta).abs().max().item() <= 2e-4


def test_bits_do_not_depend_on_position_strides_format_or_lengths():
    from kapre_b200.signal import loudness
    sr, C, L = 16000, 2, 40000
    x = _levels(6, CF, C, L, 3)
    base = loudness(x, sr, data_format=CF)
    assert torch.equal(loudness(x.flip(0), sr, data_format=CF), base.flip(0))
    assert torch.equal(loudness(x[2:3], sr, data_format=CF), base[2:3])
    big = torch.zeros(6, C + 1, L + 9, device='cuda')
    big[:, 1:, 4:4 + L] = x
    assert torch.equal(loudness(big[:, 1:, 4:4 + L], sr, data_format=CF), base)
    assert torch.equal(loudness(x.transpose(1, 2).contiguous(), sr, data_format=CL), base)
    cut = [L, 30000, 6405, 6400, 6399, 0]
    out = loudness(x, sr, torch.tensor(cut, device='cuda'), data_format=CF)
    for b, n in enumerate(cut):
        if n >= 6400:
            assert torch.equal(loudness(x[b:b + 1, :, :n].contiguous(), sr, data_format=CF), out[b:b + 1])
        else:
            assert torch.isneginf(out[b])
    # a NaN in one item makes that item NaN and leaves the others' bits
    xn = x.clone()
    xn[3, 1, 20000] = float('nan')
    o = loudness(xn, sr, data_format=CF)
    assert torch.isnan(o[3]) and torch.equal(o[:3], base[:3]) and torch.equal(o[4:], base[4:])
    assert torch.isneginf(loudness(torch.zeros(2, 1, L, device='cuda'), sr, data_format=CF)).all()


def test_gradients_match_the_float64_vjp_and_torchaudio():
    F = pytest.importorskip('torchaudio.functional')
    from kapre_b200.signal import loudness
    sr, C, L = 8000, 2, 20000
    x = _levels(3, CF, C, L, 4).requires_grad_(True)
    lengths = torch.tensor([L, 15000, 3000], device='cuda')
    gl = torch.tensor([0.7, -1.2, 2.0], device='cuda')
    out = loudness(x, sr, lengths, data_format=CF)
    out.backward(gl)
    g = x.grad.double().cpu().numpy()
    xa = x.detach().double().cpu().numpy()
    ref = LR.vjp(xa, gl.double().cpu().numpy(), sr, lengths.cpu().numpy(), LR.normalised(LR.k_weighting(sr)))
    scale = np.abs(ref).max()
    np.testing.assert_allclose(g, ref, rtol=0, atol=1e-3 * scale)
    assert np.all(g[2] == 0)                                   # a -inf item
    for b, n in enumerate(lengths.tolist()[:2]):               # torchaudio's autograd on the cut item
        xt = torch.from_numpy(xa[b, :, :n]).requires_grad_(True)
        F.loudness(xt, sr).backward(torch.tensor(float(gl[b]), dtype=torch.float64))
        np.testing.assert_allclose(g[b, :, :n], xt.grad.numpy(), rtol=0, atol=3e-3 * scale)
        assert np.all(g[b, :, n:] == 0)


def test_requires_grad_and_launch_counts():
    from kapre_b200 import _native as N
    from kapre_b200.signal import loudness
    x = _levels(4, CL, 2, 32000, 5)
    loudness(x, 16000, data_format=CL)
    torch.cuda.synchronize()
    n0 = N.launch_count()
    a = loudness(x, 16000, data_format=CL)
    n1 = N.launch_count()
    xg = x.clone().requires_grad_(True)
    b = loudness(xg, 16000, data_format=CL)
    n2 = N.launch_count()
    b.sum().backward()
    n3 = N.launch_count()
    assert torch.equal(a, b.detach())
    assert n1 - n0 == 10 and n2 - n1 == 10 and n3 - n2 == 1 + 4 + 4


def test_loudness_normalization_targets_inf_items_sequential_and_capture():
    import kapre_b200
    from kapre_b200 import _native as N
    from kapre_b200.augmentation import BackgroundNoise, LoudnessNormalization, Reverb
    from kapre_b200.composed import Sequential
    from kapre_b200.signal import Speed, loudness
    sr = 16000
    layer = LoudnessNormalization(sr, lufs_range=(-30.0, -16.0), seed=2, data_format=CL)
    x = _levels(6, CL, 1, 2 * sr, 6) * 0.2                        # no sample reaches the clamp
    x[4] = 0.0                                                   # silent: -inf, returned unchanged
    y = layer.call(x)
    target = layer.last_choice
    got = loudness(y, sr, data_format=CL).cpu().numpy()
    fin = np.arange(6) != 4
    assert np.all(np.abs(got[fin] - target[fin]) < 1e-3), (got, target)
    assert torch.equal(y[4], x[4])
    assert torch.equal(layer.call(x, lufs=-20.0, lengths=8000)[4], x[4])
    # the gradient reaches x, through the gain as well
    xg = x.clone().requires_grad_(True)
    layer.call(xg, lufs=-20.0).square().sum().backward()
    assert torch.isfinite(xg.grad).all() and (xg.grad[4] == 2 * x[4]).all()
    # Sequential: the waveform layers, then one fused log-mel launch
    mel = kapre_b200.get_melspectrogram_layer(n_fft=1024, hop_length=256, sample_rate=sr, n_mels=64,
                                              return_decibel=True, input_data_format=CL, output_data_format=CL)
    model = Sequential([layer, *mel.layers])
    model.call(x)
    torch.cuda.synchronize()
    n0 = N.launch_count()
    out = model.call(x)
    n_model = N.launch_count() - n0
    t = layer.last_choice.copy()
    yy = layer.call(x, lufs=t)
    n0 = N.launch_count()
    assert torch.equal(mel.call(yy), out)
    n_mel = N.launch_count() - n0
    assert n_mel <= 2 and n_model == 10 + n_mel                # the log-mel is the fused launch (and its dB pass)
    rirs = np.exp(-np.arange(4000) / 400.0) * np.random.default_rng(0).standard_normal(4000)
    noise = BackgroundNoise([np.random.default_rng(1).standard_normal(5000)], snr_range=(5.0, 15.0), seed=1,
                            data_format=CL)
    speed, reverb = Speed(1.1, data_format=CL), Reverb([rirs], seed=0, data_format=CL)
    chain = Sequential([speed, reverb, layer, noise, *mel.layers])
    chain.call(x)
    torch.cuda.synchronize()
    n0 = N.launch_count()
    z = chain.call(x)
    n_chain = N.launch_count() - n0
    n0 = N.launch_count()
    w = noise.call(layer.call(reverb.call(speed.call(x))))
    n_wave = N.launch_count() - n0
    assert torch.isfinite(z).all() and n_chain == n_wave + n_mel
    # capture replays the draw made at capture time
    cap = model.capture(x)
    t = layer.last_choice.copy()
    r1 = cap(x).clone()
    layer.call(x)                                                # a new eager draw does not change the graph
    r2 = cap(x).clone()
    assert torch.equal(r1, r2)
    assert torch.equal(r1, mel.call(layer.call(x, lufs=t)))


def test_invalid_arguments_raise_before_any_launch():
    from kapre_b200 import _native as N
    from kapre_b200.augmentation import LoudnessNormalization
    from kapre_b200.signal import Loudness, loudness
    x = _x((2, 8000, 2), 7)
    layer = LoudnessNormalization(16000, data_format=CL)
    torch.cuda.synchronize()
    n0 = N.launch_count()
    for args, kw in (((_x((2, 8000, 6), 1), 16000), {}), ((x, 3000), {}), ((x, -1), {}), ((x[0], 16000), {}),
                     ((x, 16000), dict(lengths=torch.ones(3, dtype=torch.int64, device='cuda'))),
                     ((x, 16000), dict(lengths=1.5)), ((x, 16000), dict(lengths=[[1, 2]]))):
        with pytest.raises(ValueError):
            loudness(*args, data_format=CL, **kw)
    with pytest.raises(N.KapreNativeError):
        loudness(x.cpu(), 16000, data_format=CL)
    with pytest.raises(ValueError):
        Loudness(16000, data_format=CL).call(_x((1, 8000, 6), 2))
    for kw in (dict(lufs=np.nan), dict(lufs=[1.0, 2.0, 3.0])):
        with pytest.raises(ValueError):
            layer.call(x, **kw)
    with pytest.raises(ValueError):
        layer.call(x[0])
    assert N.launch_count() == n0
