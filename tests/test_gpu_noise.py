"""Additive noise at a target SNR on the GPU: parity with the float64 restatement within the derived bound and with
torchaudio at benchmark size (mono channels_first, stereo channels_last), bit-independence of batch position, strides,
format, broadcasting and noise source, gradients against the float64 VJP with broadcast snr and lengths, requires_grad
leaving the forward unchanged, launch counts, BackgroundNoise against add_noise on the looped excerpt, in Sequential
before the fused log-mel and under graph capture, and invalid arguments raising before any launch."""
import numpy as np
import pytest
import torch

import noise_ref as NR

pytestmark = pytest.mark.gpu

SR = 16000
CF, CL = 'channels_first', 'channels_last'


def _x(shape, seed, scale=1.0):
    g = torch.Generator(device='cuda').manual_seed(seed)
    return torch.randn(shape, device='cuda', generator=g) * scale


def _bcl(t, fmt):
    a = t.detach().double().cpu().numpy()
    return a.transpose(0, 2, 1) if fmt == CL else a


def _check(y, x, n, snr, lengths, fmt):
    xa, na = _bcl(x, fmt), _bcl(n, fmt)
    sa = np.broadcast_to(snr.float().cpu().double().numpy() if torch.is_tensor(snr) else np.float32(snr), xa.shape[:2])
    la = None if lengths is None else np.broadcast_to(lengths.cpu().numpy() if torch.is_tensor(lengths) else lengths,
                                                      xa.shape[:2])
    ref, _ = NR.add_noise(xa, na, sa, la)
    bound = NR.forward_bound(xa, na, sa, la)
    err = np.abs(_bcl(y, fmt) - ref)
    assert (err <= bound).all(), (err.max(), (err / np.maximum(bound, 1e-300)).max())
    return err.max()


@pytest.mark.parametrize('fmt,C', [(CF, 1), (CL, 2)])
def test_parity_at_bench_size(fmt, C):
    F = pytest.importorskip('torchaudio.functional')
    from kapre_b200.signal import add_noise
    B, L = 256, 5 * SR
    shape = (B, C, L) if fmt == CF else (B, L, C)
    x, n = _x(shape, 1), _x(shape, 2, 0.3)
    snr = torch.linspace(-5, 30, B * C, device='cuda').view(B, C)
    lengths = torch.randint(L // 2, L + 100, (B, 1), device='cuda')
    for ln in (None, lengths):
        y = add_noise(x, n, snr, ln, data_format=fmt)
        _check(y, x, n, snr, ln, fmt)
        # torchaudio on the same card (float32, its own reduction order): agreement to float32 rounding
        xt, nt = (t if fmt == CF else t.transpose(1, 2) for t in (x, n))
        ta = F.add_noise(xt, nt, snr, None if ln is None else torch.clamp(ln, 0, L).expand(B, C))
        yt = y if fmt == CF else y.transpose(1, 2)
        assert torch.allclose(yt, ta, rtol=1e-5, atol=1e-5)


def test_ten_minute_recording():
    from kapre_b200.signal import add_noise
    x, n = _x((1, 1, 600 * SR), 3), _x((1, 1, 600 * SR), 4, 2.0)
    y = add_noise(x, n, 12.0, data_format=CF)
    print('10 min: max|err| %.3g' % _check(y, x, n, 12.0, None, CF))


def test_bits_do_not_depend_on_position_strides_format_broadcast_or_source():
    from kapre_b200.signal import add_noise
    B, C, L = 5, 3, 3 * 4096 + 123
    x, n = _x((B, C, L), 5), _x((B, C, L), 6)
    snr = torch.rand(B, C, device='cuda') * 20
    lengths = torch.randint(1000, L + 10, (B, C), device='cuda')
    ref = add_noise(x, n, snr, lengths, data_format=CF)
    for i in (0, 4):
        assert torch.equal(add_noise(x[i:i + 1].clone(), n[i:i + 1].clone(), snr[i:i + 1], lengths[i:i + 1],
                                     data_format=CF), ref[i:i + 1])
    big, bign = _x((B + 2, 2 * C, L + 9), 7), _x((B + 2, 2 * C, L + 9), 8)
    big[1:B + 1, ::2, 4:L + 4] = x
    bign[1:B + 1, ::2, 4:L + 4] = n
    assert torch.equal(add_noise(big[1:B + 1, ::2, 4:L + 4], bign[1:B + 1, ::2, 4:L + 4], snr, lengths,
                                 data_format=CF), ref)
    yl = add_noise(x.transpose(1, 2).contiguous(), n.transpose(1, 2).contiguous(), snr, lengths, data_format=CL)
    assert torch.equal(yl.transpose(1, 2), ref)
    for nb in (n[:1], n[:, :1], n[:1, :1]):
        r = add_noise(x, nb, snr, lengths, data_format=CF)
        assert torch.equal(r, add_noise(x, nb.expand(B, C, L).contiguous(), snr, lengths, data_format=CF))
    # bank mode against tensor mode on the materialised excerpt
    from kapre_b200 import ops
    clip = _x((1000,), 9)
    start = torch.zeros(B, dtype=torch.int64, device='cuda')
    clen = torch.full((B,), 1000, dtype=torch.int64, device='cuda')
    off = torch.arange(B, device='cuda') * 199
    yb = ops.add_noise(x, None, snr, lengths, CF, bank=(clip, start, clen, off))
    idx = (off[:, None] + torch.arange(L, device='cuda')[None]) % 1000
    assert torch.equal(yb, add_noise(x, clip[idx][:, None, :], snr, lengths, data_format=CF))


def test_gradients_against_float64_with_broadcast_snr_and_lengths():
    from kapre_b200.signal import add_noise
    B, C, L = 3, 2, 9000
    x = _x((B, L, C), 10).requires_grad_(True)
    n = _x((1, L, C), 11, 0.5).requires_grad_(True)              # broadcast over the batch
    snr = torch.tensor([[3.0], [10.0], [-2.0]], device='cuda', requires_grad=True)    # one per item
    lengths = torch.tensor([L, 5000, 0], device='cuda').view(B, 1)
    g = _x((B, L, C), 12)
    y = add_noise(x, n, snr, lengths, data_format=CL)
    (y * g).sum().backward()
    xa, na, ga = _bcl(x, CL), np.broadcast_to(_bcl(n, CL), (B, C, L)), _bcl(g, CL)
    sa = np.broadcast_to(snr.detach().cpu().double().numpy(), (B, C))
    la = np.broadcast_to(lengths.cpu().numpy(), (B, C))
    (rx, rn, rs), (bx, bn, bs) = NR.backward_bounds(xa, na, sa.astype(np.float32), ga, la)
    assert (np.abs(_bcl(x.grad, CL) - rx) <= bx).all()
    gn = _bcl(n.grad, CL)[0]
    assert np.abs(gn - rn.sum(0)).max() <= bn.sum(0).max() + 1e-6 * np.abs(rn).sum(0).max()
    gs = snr.grad.cpu().double().numpy()[:, 0]
    assert np.abs(gs - rs.sum(1)).max() <= bs.sum(1).max() + 1e-6 * np.abs(rs).sum(1).max()
    assert gs[2] == 0.0                                          # lengths 0: every term through s is 0


def test_requires_grad_leaves_the_forward_unchanged_and_launch_counts():
    from kapre_b200 import _native as N
    from kapre_b200.signal import add_noise
    x, n = _x((4, 1, 50000), 13), _x((4, 1, 50000), 14)
    torch.cuda.synchronize()
    n0 = N.launch_count()
    y0 = add_noise(x, n, 5.0, data_format=CF)
    assert N.launch_count() - n0 == 2                            # energies, mix
    xg = x.clone().requires_grad_(True)
    n0 = N.launch_count()
    y1 = add_noise(xg, n, 5.0, data_format=CF)
    assert N.launch_count() - n0 == 2 and torch.equal(y0, y1.detach())
    n0 = N.launch_count()
    y1.sum().backward()
    assert N.launch_count() - n0 == 2                            # D, gradients


def _layer_and_clips(seed=3, fmt=CL):
    from kapre_b200.augmentation import BackgroundNoise
    rng = np.random.default_rng(seed)
    clips = [rng.standard_normal(n).astype(np.float32) for n in (1, 700, 40000)]
    return BackgroundNoise(clips, snr_range=(0.0, 15.0), seed=seed, data_format=fmt), clips


def test_background_noise_is_add_noise_on_the_looped_excerpt():
    from kapre_b200.signal import add_noise
    layer, clips = _layer_and_clips()
    B, L, C = 8, SR, 2
    x = _x((B, L, C), 15)
    y = layer.call(x)
    idx, off, snr = layer.last_choice
    ex = torch.from_numpy(NR.bank_excerpt(clips, idx, off, L).astype(np.float32)).cuda()
    want = add_noise(x, ex[:, :, None], torch.from_numpy(snr.astype(np.float32)).cuda().view(B, 1), data_format=CL)
    assert torch.equal(y, want)
    # the gradient reaches x
    xg = x.clone().requires_grad_(True)
    layer.call(xg).square().sum().backward()
    assert xg.grad is not None and torch.isfinite(xg.grad).all()


def test_background_noise_in_sequential_chain_and_capture():
    import kapre_b200
    from kapre_b200 import _native as N
    from kapre_b200.augmentation import Reverb
    from kapre_b200.composed import Sequential
    from kapre_b200.signal import Speed
    layer, _ = _layer_and_clips(5)
    mel = kapre_b200.get_melspectrogram_layer(n_fft=1024, hop_length=256, sample_rate=SR, n_mels=64,
                                              return_decibel=True, input_data_format=CL, output_data_format=CL)
    model = Sequential([layer, *mel.layers])
    x = _x((8, SR, 1), 16)
    model.call(x)
    torch.cuda.synchronize()
    n0 = N.launch_count()
    out = model.call(x)
    n_model = N.launch_count() - n0
    idx, off, snr = layer.last_choice
    y = layer.call(x, noise_index=idx, offset=off, snr=snr)
    n0 = N.launch_count()
    assert torch.equal(mel.call(y), out)
    n_mel = N.launch_count() - n0
    assert n_model == 2 + n_mel and n_mel <= 2
    # the whole chain: speed perturbation -> reverberation -> noise -> log-mel
    rirs = np.exp(-np.arange(4000) / 400.0) * np.random.default_rng(0).standard_normal(4000)
    chain = Sequential([Speed(1.1, data_format=CL), Reverb([rirs], seed=0, data_format=CL), layer, *mel.layers])
    z = chain.call(x)
    assert torch.isfinite(z).all()
    # capture replays the draw made at capture time
    cap = model.capture(x)
    idx, off, snr = (v.copy() for v in layer.last_choice)
    r1 = cap(x).clone()
    layer.call(x)                                                # a new eager draw does not change the graph
    r2 = cap(x).clone()
    assert torch.equal(r1, r2)
    assert torch.equal(r1, mel.call(layer.call(x, noise_index=idx, offset=off, snr=snr)))


def test_invalid_arguments_raise_before_any_launch():
    from kapre_b200 import _native as N
    from kapre_b200.signal import add_noise
    layer, _ = _layer_and_clips()
    x = _x((2, 1000, 2), 17)
    n = _x((2, 1000, 2), 18)
    torch.cuda.synchronize()
    n0 = N.launch_count()
    for kw in (dict(noise=n[:, :999]), dict(noise=_x((3, 1000, 2), 1)), dict(noise=_x((2, 1000, 3), 1)),
               dict(noise=n[0]), dict(snr=torch.zeros(3)), dict(snr=torch.zeros(2, 2, 1)), dict(snr='a'),
               dict(lengths=torch.ones(3, dtype=torch.int64)), dict(lengths=1.5)):
        args = dict(noise=n, snr=10.0)
        args.update(kw)
        with pytest.raises(ValueError):
            add_noise(x, args['noise'], args['snr'], kw.get('lengths'), data_format=CL)
    with pytest.raises(ValueError):
        add_noise(x[0], n[0], 10.0, data_format=CL)
    with pytest.raises(N.KapreNativeError):
        add_noise(x.cpu(), n, 10.0, data_format=CL)
    for kw in (dict(noise_index=5), dict(offset=-1), dict(snr=np.inf), dict(noise_index=[0, 1, 2])):
        with pytest.raises(ValueError):
            layer.call(x, **kw)
    with pytest.raises(ValueError):
        layer.call(x[0])
    assert N.launch_count() == n0
