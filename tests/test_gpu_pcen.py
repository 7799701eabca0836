"""PCEN on the GPU: parity with the float64 restatement (pcen_ref.py) at the cfg2 mel shape and at a 10-minute
recording (the chunked path), input and parameter gradients against float64 autograd, and ``PCEN`` behind the
fused log-mel launch in a ``Sequential``.  Tolerances as derived in test_pcen_emu.py."""
import numpy as np
import pytest
import torch

import grad_ref as R
import pcen_ref as PR

pytestmark = pytest.mark.gpu
CL, CF = 'channels_last', 'channels_first'
CFG2 = (256, 427, 128, 1)           # cfg2's mel magnitudes: 256 x 5 s at 22.05 kHz, hop 256, 128 bands
LONG = (1, 51680, 128, 1)           # 10 min at 22.05 kHz, hop 256


def _spectrogram(shape, fmt, seed=0):
    """(B, T, F, C) for channels_last, (B, C, T, F) otherwise, from a (B, T, F, C) description; four decades."""
    B, T, F, C = shape
    g = torch.Generator().manual_seed(seed)
    x = 10.0 ** (torch.rand((B, T, F, C) if fmt == CL else (B, C, T, F), generator=g) * 4 - 2)
    return x.cuda()


def _canon(t, fmt):
    t = t.detach().cpu().double()
    return t.permute(0, 3, 1, 2) if fmt == CL else t


def _per_band(F, seed=1):
    rng = np.random.default_rng(seed)
    return dict(gain=list(rng.uniform(0.5, 1.0, F)), bias=list(rng.uniform(0.5, 3.0, F)),
                power=list(rng.uniform(0.2, 0.8, F)), smooth_coef=list(rng.uniform(0.01, 0.5, F)))


_SCALAR = dict(gain=0.98, bias=2.0, power=0.5)


def _layer(fmt, per_band, F, hop=256):
    from kapre_b200.time_frequency import PCEN
    kw = _per_band(F) if per_band else _SCALAR
    return PCEN(sample_rate=22050, hop_length=hop, data_format=fmt, **kw)


def _ref_params(layer):
    return [w.detach().cpu().double() for w in layer.weights]


def _close(got, want, rel, scale):
    got = got.detach().cpu().double()
    assert tuple(got.shape) == tuple(want.shape), (tuple(got.shape), tuple(want.shape))
    err = (got - want).abs()
    bound = rel * (want.abs() + scale)
    assert bool((err <= bound).all()), (float((err / bound.clamp_min(1e-300)).max()), float(err.max()))


def _chunks(E, fmt):
    from kapre_b200 import ops
    from kapre_b200.ops import _spec_desc
    _, (B, C, T, F) = _spec_desc(E, fmt)
    return ops._pcen_workspace(B, C, T, F, E.device)[0]


@pytest.mark.parametrize('shape,fmt', [(CFG2, CL), (CFG2, CF), ((64, 427, 128, 2), CL), (LONG, CL)])
@pytest.mark.parametrize('per_band', [False, True])
def test_parity(shape, fmt, per_band):
    E = _spectrogram(shape, fmt, seed=shape[1] + per_band)
    layer = _layer(fmt, per_band, shape[2])
    y = layer(E)
    if shape in (CFG2, LONG):           # 32 768 columns fill the GPU; 128 do not (the stereo case may go either way)
        assert (_chunks(E, fmt) > 1) == (shape == LONG)
    want = PR.pcen(_canon(E, fmt), *_ref_params(layer), eps=layer.eps)
    _close(_canon(y, fmt), want, 1e-4, 1e-4 * float(want.abs().max()))


@pytest.mark.parametrize('shape', [CFG2, LONG])
@pytest.mark.parametrize('per_band', [False, True])
def test_gradients(shape, per_band):
    fmt = CL
    E = _spectrogram(shape, fmt, seed=3).requires_grad_()
    layer = _layer(fmt, per_band, shape[2])
    y = layer(E)
    assert y.requires_grad
    gy = (torch.rand(y.shape, generator=torch.Generator().manual_seed(4)) * 2 - 1).cuda()
    got = torch.autograd.grad(y, [E] + layer.weights, gy)
    gEr, gr, scale = PR.grads(_canon(E, fmt), _ref_params(layer), _canon(gy, fmt), eps=layer.eps)
    _close(_canon(got[0], fmt), gEr, 1e-4, float(gEr.abs().max()))
    for g, w, want, sc in zip(got[1:], layer.weights, gr, scale):
        assert g.shape == w.shape
        assert bool(((g.cpu().double() - want).abs() <= 1e-4 * sc).all()), (g, want, sc)


def test_backward_is_deterministic():
    E = _spectrogram(CFG2, CL, seed=5).requires_grad_()
    layer = _layer(CL, True, 128)
    gy = torch.rand(E.shape, device='cuda')
    a = torch.autograd.grad(layer(E), [E] + layer.weights, gy)
    b = torch.autograd.grad(layer(E), [E] + layer.weights, gy)
    assert all(torch.equal(u, v) for u, v in zip(a, b))


def test_weights_and_device():
    layer = _layer(CF, True, 128)
    assert layer.weights == []
    layer(_spectrogram((2, 10, 128, 1), CF))
    w = layer.weights
    assert [tuple(t.shape) for t in w] == [(128,)] * 4 and all(t.is_cuda and t.requires_grad for t in w)
    assert layer.count_params() == 4 * 128
    with pytest.raises(ValueError):
        layer(_spectrogram((2, 10, 64, 1), CF))
    if torch.cuda.device_count() > 1:
        with pytest.raises(ValueError):
            layer(_spectrogram((2, 10, 128, 1), CF).to('cuda:1'))


def test_host_input_returns_numpy_without_grad():
    layer = _layer(CL, False, 16)
    x = _spectrogram((2, 30, 16, 1), CL).cpu().numpy()
    y = layer(x)
    assert isinstance(y, np.ndarray)
    want = PR.pcen(torch.from_numpy(x).double().permute(0, 3, 1, 2), *_ref_params(layer), eps=layer.eps)
    _close(torch.from_numpy(y).permute(0, 3, 1, 2), want, 1e-4, 1e-4 * float(want.abs().max()))


def _mel(fmt=CL):
    import kapre_b200
    return kapre_b200.get_melspectrogram_layer(n_fft=1024, hop_length=256, sample_rate=22050, n_mels=128,
                                               return_decibel=False, input_data_format=fmt, output_data_format=fmt)


def _wave(B, L, seed=6):
    g = torch.Generator().manual_seed(seed)
    return (torch.rand((B, L, 1), generator=g) * 2 - 1).cuda()


def test_sequential_two_launches_same_bits():
    from kapre_b200 import _native as N
    from kapre_b200.composed import Sequential
    mel = _mel()
    pcen = _layer(CL, True, 128)
    stack = Sequential([*mel.layers, pcen])
    x = _wave(256, 5 * 22050)               # cfg2: 32 768 columns, one time chunk
    want = pcen(mel(x))
    torch.cuda.synchronize()
    n0 = N.launch_count()
    got = stack(x)
    n1 = N.launch_count()
    assert n1 - n0 == 2                      # fused STFT -> magnitude -> mel, then PCEN
    assert torch.equal(got, want)
    # one predict chunk of the whole batch: the time chunking follows the column count, so a smaller predict batch
    # may chunk differently and agree only to float32 rounding
    host = stack.predict(x.cpu().numpy(), batch_size=x.shape[0])
    assert isinstance(host, np.ndarray) and np.array_equal(host, want.detach().cpu().numpy())
    cap = stack.capture(x)
    out = cap(x)
    torch.cuda.synchronize()
    assert torch.equal(out, want) and not out.requires_grad
    xg = x.clone().requires_grad_()
    n2 = N.launch_count()
    tracked = stack(xg)
    n3 = N.launch_count()
    assert n3 - n2 == 2 and tracked.requires_grad and torch.equal(tracked, want)
    with torch.no_grad():
        n4 = N.launch_count()
        plain = stack(x)
        assert N.launch_count() - n4 == 2 and not plain.requires_grad and torch.equal(plain, want)


@pytest.mark.parametrize('per_band', [False, True])
def test_backward_from_waveform(per_band):
    """One backward pass through Sequential([STFT, Magnitude, ApplyFilterbank, PCEN]) from a waveform: the waveform
    and all four weights against grad_ref's stft, magnitude and apply_filterbank chained into pcen_ref, in float64.
    The waveform gradient passes through the float32 STFT backward as well, so it is held to 1e-3 of its maximum."""
    from kapre_b200.composed import Sequential
    mel = _mel()
    pcen = _layer(CL, per_band, 128)
    stack = Sequential([*mel.layers, pcen])
    x = _wave(2, 22050, seed=7).requires_grad_()
    y = stack(x)
    gy = (torch.rand(y.shape, generator=torch.Generator().manual_seed(8)) * 2 - 1).cuda()
    got = torch.autograd.grad(y, [x] + pcen.weights, gy)

    fb = R.filterbank_mel(1024, 22050, 128)
    xr = x.detach().cpu().double().requires_grad_()
    params = [p.requires_grad_() for p in _ref_params(pcen)]
    melr = R.apply_filterbank(R.magnitude(R.stft(xr, 1024, 1024, 256, None, False, False, CL, CL)), fb, CL)
    melr = melr.permute(0, 3, 1, 2)
    yr = PR.pcen(melr, *params, eps=pcen.eps)
    want = torch.autograd.grad(yr, [xr] + params, _canon(gy, CL))
    _close(got[0], want[0], 1e-3, float(want[0].abs().max()))
    _, _, scale = PR.grads(melr.detach(), [p.detach() for p in params], _canon(gy, CL), eps=pcen.eps)
    for g, w, sc in zip(got[1:], want[1:], scale):
        assert g.shape == w.shape
        assert bool(((g.cpu().double() - w).abs() <= 1e-3 * sc).all()), (g, w, sc)
