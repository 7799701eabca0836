"""Kaldi features on the H100: parity with float64 torchaudio looped per (item, channel) on the device, at benchmark
size in both formats and at 8 / 22.05 / 48 kHz, for mfcc and spectrogram, with ragged lengths; the VJP against float64
torchaudio autograd; bit equality across batch positions, views, formats and repeated calls (gradient included);
launch counts; the augmentation chain into KaldiFbank and SpecAugment; capture replays; validation before launch."""
import numpy as np
import pytest
import torch

import kaldi_ref as R

pytestmark = pytest.mark.gpu

CL, CF = 'channels_last', 'channels_first'


def _ta(kind, x1, o):
    import torchaudio.compliance.kaldi as TK
    fn = getattr(TK, kind)
    return fn(x1, **{k: v for k, v in o.items() if k in fn.__code__.co_varnames})


def _x(B, C, L, seed, sr=16000.0):
    rng = np.random.default_rng(seed)
    t = np.arange(L) / sr
    x = 0.05 * rng.standard_normal((B, C, L)) * (1.0 + np.sin(2 * np.pi * 3.0 * t))
    x += 0.3 * np.sin(2 * np.pi * rng.uniform(100, sr / 3, size=(B, C, 1)) * t) + rng.uniform(-0.1, 0.1, (B, C, 1))
    return torch.from_numpy(np.clip(x, -1, 1).astype(np.float32)).cuda()


def _ref(kind, x, o, lengths=None):
    """float64 torchaudio per (item, channel) on the device, zero-padded to the batch's frame count: (B, C, T, K)."""
    B, C, L = x.shape
    outs = []
    for b in range(B):
        Lb = L if lengths is None else int(lengths[b])
        outs.append([_ta(kind, x[b, c:c + 1, :Lb].double(), o) if Lb > 0 else None for c in range(C)])
    T = max((r[0].shape[0] for r in outs if r[0] is not None and r[0].dim() == 2), default=0)
    K = next(r[0].shape[1] for r in outs if r[0] is not None and r[0].dim() == 2)
    y = torch.zeros((B, C, T, K), dtype=torch.float64, device=x.device)
    for b in range(B):
        for c in range(C):
            r = outs[b][c]
            if r is not None and r.dim() == 2:
                y[b, c, :r.shape[0]] = r
    return y


def _run(kind, x, fmt, lengths=None, **kw):
    from kapre_b200 import signal
    fn = getattr(signal, 'kaldi_' + kind)
    xin = x.transpose(1, 2).contiguous() if fmt == CL else x
    y = fn(xin, lengths=lengths, data_format=fmt, **kw)
    return y.permute(0, 3, 1, 2) if fmt == CL else y


def _within(kind, x, o, y, ref, lengths=None):
    # torchaudio's mel banks are float32: 2e-4 relative on top of the kernel's bound
    bound = R.log_bound(kind, x.cpu().numpy(), o, lengths, ref.cpu().numpy()) + 2e-4 * np.abs(ref.cpu().numpy())
    err = (y.double() - ref).abs().cpu().numpy()
    assert y.shape == ref.shape
    bad = err > bound
    assert not bad.any(), (float(err[bad].max()), float(bound[bad].min()))


@pytest.mark.parametrize('fmt', [CL, CF])
def test_parity_bench_size(fmt):
    from kapre_b200 import ops
    x = _x(256, 1, 5 * 16000, 1)
    o = ops.kaldi_options('fbank', num_mel_bins=80)
    y = _run('fbank', x, fmt, num_mel_bins=80)
    _within('fbank', x, o, y, _ref('fbank', x, o))


@pytest.mark.parametrize('kind,sr,kw', [('fbank', 8000, dict(num_mel_bins=23)),
                                        ('fbank', 22050, dict(num_mel_bins=64, snip_edges=False, use_energy=True)),
                                        ('fbank', 48000, dict(num_mel_bins=80, window_type='hamming')),
                                        ('mfcc', 16000, dict(use_energy=True, htk_compat=True)),
                                        ('spectrogram', 16000, dict(snip_edges=False))])
def test_parity_rates_and_kinds(kind, sr, kw):
    from kapre_b200 import ops
    x = _x(8, 2, 2 * sr, sr, float(sr))
    o = ops.kaldi_options(kind, sample_frequency=float(sr), **kw)
    for fmt in (CL, CF):
        y = _run(kind, x, fmt, sample_frequency=float(sr), **kw)
        _within(kind, x, o, y, _ref(kind, x, o))


def test_ragged_lengths():
    from kapre_b200 import ops
    x = _x(6, 2, 32000, 3)
    lengths = [32000, 0, 399, 400, 12345, 20001]
    o = ops.kaldi_options('fbank', num_mel_bins=40, snip_edges=False)
    y = _run('fbank', x, CF, lengths=torch.tensor(lengths), num_mel_bins=40, snip_edges=False)
    ref = _ref('fbank', x, o, [l if l >= 400 else 0 for l in lengths])
    _within('fbank', x, o, y, ref, lengths)
    cut = _run('fbank', x[4:5, :, :12345].contiguous(), CF, num_mel_bins=40, snip_edges=False)
    assert torch.equal(y[4:5, :, :cut.shape[2]], cut) and (y[4, :, cut.shape[2]:] == 0).all()


@pytest.mark.parametrize('kind,kw', [('fbank', dict(num_mel_bins=80)),
                                     ('fbank', dict(num_mel_bins=40, subtract_mean=True, snip_edges=False,
                                                    use_energy=True)),
                                     ('mfcc', dict(snip_edges=False)),
                                     ('spectrogram', dict(subtract_mean=True))])
def test_vjp_against_torchaudio(kind, kw):
    x = _x(3, 2, 16000, 7) + 0.01 * torch.randn(3, 2, 16000, device='cuda', generator=torch.Generator('cuda').manual_seed(0))
    xg = x.clone().requires_grad_(True)
    y = _run(kind, xg, CF, **kw)
    g = torch.randn(y.shape, device='cuda', generator=torch.Generator('cuda').manual_seed(1))
    (y * g).sum().backward()
    xd = x.double().requires_grad_(True)
    total = 0
    for b in range(3):
        for c in range(2):
            total = total + (_ta(kind, xd[b, c:c + 1], dict(kw)) * g[b, c].double()).sum()
    total.backward()
    scale = xd.grad.abs().max().item()
    assert (xg.grad.double() - xd.grad).abs().max().item() <= 2e-3 * scale


def test_bits_across_positions_views_formats_and_repeats():
    from kapre_b200 import signal
    x = _x(8, 2, 24000, 9)
    y = _run('mfcc', x, CF)
    assert torch.equal(_run('mfcc', x, CF), y)
    assert torch.equal(_run('mfcc', x, CL), y)
    assert torch.equal(_run('mfcc', x.flip(0), CF).flip(0), y)
    assert torch.equal(_run('mfcc', x[2:5], CF), y[2:5])
    big = torch.zeros(8, 2, 48000, device='cuda')
    big[:, :, ::2] = x
    assert torch.equal(signal.kaldi_mfcc(big[:, :, ::2], data_format=CF), y)
    # dither: repeated calls with the same seed give the same bits, and so does the gradient
    d1 = signal.kaldi_fbank(x, data_format=CF, dither=1.0, seed=5)
    assert torch.equal(signal.kaldi_fbank(x, data_format=CF, dither=1.0, seed=5), d1)
    assert not torch.equal(signal.kaldi_fbank(x, data_format=CF, dither=1.0, seed=6), d1)
    grads = []
    for _ in range(2):
        xg = x.clone().requires_grad_(True)
        yg = signal.kaldi_fbank(xg, data_format=CF, dither=1.0, seed=5)
        assert torch.equal(yg.detach(), d1)
        yg.square().sum().backward()
        grads.append(xg.grad)
    assert torch.equal(grads[0], grads[1])
    xg = x[3:4].clone().requires_grad_(True)
    signal.kaldi_fbank(xg, data_format=CF).square().sum().backward()
    xa = x.clone().requires_grad_(True)
    signal.kaldi_fbank(xa, data_format=CF).square().sum().backward()
    assert torch.equal(xa.grad[3:4], xg.grad)


def test_launch_counts():
    from kapre_b200 import _native as N
    from kapre_b200 import signal
    x = _x(4, 1, 16000, 2)
    signal.kaldi_fbank(x, data_format=CF)
    for kw, fwd, bwd in [(dict(), 1, 2), (dict(subtract_mean=True), 2, 3)]:
        torch.cuda.synchronize()
        n0 = N.launch_count()
        y0 = signal.kaldi_fbank(x, data_format=CF, **kw)
        assert N.launch_count() - n0 == fwd
        xg = x.clone().requires_grad_(True)
        n0 = N.launch_count()
        y1 = signal.kaldi_fbank(xg, data_format=CF, **kw)
        assert N.launch_count() - n0 == fwd and torch.equal(y0, y1.detach())
        n0 = N.launch_count()
        y1.sum().backward()
        assert N.launch_count() - n0 == bwd


def test_chain_into_kaldi_fbank_and_capture():
    from kapre_b200 import _native as N
    from kapre_b200.time_frequency import KaldiFbank
    from kapre_b200.augmentation import BackgroundNoise, Reverb, SpecAugment
    from kapre_b200.composed import Sequential
    from kapre_b200.signal import Speed
    rng = np.random.default_rng(0)
    rirs = np.exp(-np.arange(4000) / 400.0) * rng.standard_normal(4000)
    noise = BackgroundNoise([rng.standard_normal(20000).astype(np.float32)], snr_range=(5.0, 15.0), seed=1,
                            data_format=CL)
    fb = KaldiFbank(num_mel_bins=80, data_format=CL)
    chain = Sequential([Speed(1.1, data_format=CL), Reverb([rirs], seed=0, data_format=CL), noise, fb,
                        SpecAugment(freq_mask_param=5, time_mask_param=10)])
    x = _x(4, 1, 16000, 4).transpose(1, 2).contiguous()
    z = chain.call(x)
    assert z.shape[2] == 80 and torch.isfinite(z).all()
    # the waveform layers first, then one Kaldi launch
    wave = Sequential([chain.layers[0], chain.layers[1], noise])
    wave.call(x)
    torch.cuda.synchronize()
    n0 = N.launch_count()
    w = wave.call(x)
    n_wave = N.launch_count() - n0
    n0 = N.launch_count()
    chain.call(x)
    assert N.launch_count() - n0 == n_wave + 1
    # capture replays give the eager result for the draw made at capture time (KaldiFbank itself draws nothing)
    model = Sequential([fb])
    cap = model.capture(w)
    r1 = cap(w).clone()
    assert torch.equal(r1, fb.call(w))
    assert torch.equal(cap(w), r1)


def test_layer_training_dither_draws_and_records_seed():
    from kapre_b200 import signal
    from kapre_b200.time_frequency import KaldiFbank
    x = _x(2, 1, 16000, 5).transpose(1, 2).contiguous()
    layer = KaldiFbank(num_mel_bins=40, dither=1.0, seed=11, data_format=CL)
    assert torch.equal(layer(x), signal.kaldi_fbank(x, data_format=CL, num_mel_bins=40))
    y = layer(x, training=True)
    s = layer.last_choice
    assert s == int(np.random.default_rng(11).integers(0, 2 ** 63))
    assert torch.equal(y, signal.kaldi_fbank(x, data_format=CL, num_mel_bins=40, dither=1.0, seed=s))


def test_invalid_arguments_raise_before_any_launch():
    from kapre_b200 import _native as N
    from kapre_b200 import signal
    x = _x(2, 1, 8000, 6)
    torch.cuda.synchronize()
    n0 = N.launch_count()
    bad = [dict(round_to_power_of_two=False), dict(sample_frequency=96000.0), dict(num_mel_bins=300),
           dict(preemphasis_coefficient=1.5), dict(dither=float('inf')), dict(lengths=[8001, 1]),
           dict(lengths=[-1, 1]), dict(lengths=[5]), dict(lengths=torch.tensor([1.0, 2.0])), dict(channel=0),
           dict(data_format='nchw')]
    for kw in bad:
        with pytest.raises(Exception):
            signal.kaldi_fbank(x, **dict(dict(data_format=CF), **kw))
    with pytest.raises(Exception):
        signal.kaldi_fbank(x.double(), data_format=CF)
    with pytest.raises(Exception):
        signal.kaldi_mfcc(x, data_format=CF, num_ceps=30)
    assert N.launch_count() == n0
