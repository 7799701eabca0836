"""The IIR filter on the GPU: parity with the float64 restatement within the derived bound at benchmark size (mono
channels_first, stereo channels_last; a biquad, pre-emphasis, an 8th-order filter), per-item and per-channel
coefficients, a 10-minute recording, filtfilt against torchaudio, bit-independence of batch position, strides and
prefix length, gradients against float64 (through a0 and at the clamp boundary, and into a trainable IIRFilter),
requires_grad leaving the forward's bits unchanged, launch counts, Biquad in front of the fused log-mel launch,
RandomBiquad under graph capture, and invalid arguments raising before any launch."""
import numpy as np
import pytest
import scipy.signal
import torch

import iir_ref as IR

pytestmark = pytest.mark.gpu

SR = 16000
CF, CL = 'channels_first', 'channels_last'


def _designs():
    return {'biquad': IR.biquad('lowpass', SR, 1000.0, 0.707),
            'bandpass-q30': IR.biquad('bandpass', SR, 100.0, 30.0),
            'preemph': (np.array([1.0, -0.97]), np.array([1.0, 0.0])),
            'butter8': scipy.signal.butter(8, 0.2)}


def _x(shape, seed, scale=1.0):
    return torch.from_numpy(np.random.default_rng(seed).uniform(-scale, scale, shape).astype(np.float32)).cuda()


def _bcl(t, fmt):
    """(B, C, L) float64 NumPy of a waveform in fmt."""
    a = t.detach().double().cpu().numpy()
    return a.transpose(0, 2, 1) if fmt == CL else a


def _check(y, x, b32, a32, fmt, what=''):
    xa = _bcl(x, fmt)
    ref = IR.lfilter_fast(xa, b32, a32)
    bound = IR.error_bound(b32, a32, np.abs(xa).max(), np.abs(ref).max(), IR.local_max(xa, b32, a32))
    err = np.abs(_bcl(y, fmt) - ref).max()
    assert err <= bound, (what, err, bound)
    return err, bound


@pytest.mark.parametrize('name', ['biquad', 'bandpass-q30', 'preemph', 'butter8'])
@pytest.mark.parametrize('fmt,C', [(CF, 1), (CL, 2)])
def test_parity_at_bench_size(name, fmt, C):
    from kapre_b200.signal import lfilter
    b, a = _designs()[name]
    b32, a32 = IR.normalised32(b, a)
    shape = (256, C, 5 * SR) if fmt == CF else (256, 5 * SR, C)
    x = _x(shape, seed=C)
    y = lfilter(x, a, b, clamp=False, data_format=fmt)
    err, bound = _check(y, x, b32, a32, fmt, name)
    print('%s %s C=%d: max|err| %.3g, bound %.3g' % (name, fmt, C, err, bound))


def test_per_item_and_per_channel_coefficients():
    from kapre_b200.backend import biquad_coefficients
    from kapre_b200.signal import lfilter
    B, C, L = 6, 2, 20000
    x = _x((B, L, C), seed=3)
    freq = np.geomspace(100, 6000, B * C).reshape(B, C)
    b, a = biquad_coefficients('highpass', SR, freq, 0.9)
    y = lfilter(x, torch.from_numpy(a), torch.from_numpy(b), clamp=False, data_format=CL)
    for i in range(B):
        for c in range(C):
            b32, a32 = IR.normalised32(b[i, c], a[i, c])
            _check(y[i:i + 1, :, c:c + 1], x[i:i + 1, :, c:c + 1], b32, a32, CL, (i, c))
    # one filter per channel (2-D coefficients)
    y2 = lfilter(x, torch.from_numpy(a[0]), torch.from_numpy(b[0]), clamp=False, data_format=CL)
    for c in range(C):
        b32, a32 = IR.normalised32(b[0, c], a[0, c])
        _check(y2[:, :, c:c + 1], x[:, :, c:c + 1], b32, a32, CL, c)
    # a shared filter passed per item gives the shared filter's bits
    bs, as_ = biquad_coefficients('highpass', SR, 700.0, 0.9)
    y3 = lfilter(x, torch.from_numpy(np.broadcast_to(as_, (B, C, 3)).copy()),
                 torch.from_numpy(np.broadcast_to(bs, (B, C, 3)).copy()), data_format=CL)
    assert torch.equal(y3, lfilter(x, as_, bs, data_format=CL))


def test_ten_minute_recording():
    from kapre_b200.signal import lfilter
    b, a = IR.biquad('bandpass', SR, 100.0, 30.0)
    b32, a32 = IR.normalised32(b, a)
    x = _x((1, 1, 600 * SR), seed=4)
    y = lfilter(x, a, b, clamp=False, data_format=CF)
    err, bound = _check(y, x, b32, a32, CF)
    print('10 min: max|err| %.3g, bound %.3g' % (err, bound))


def test_filtfilt_against_torchaudio():
    F = pytest.importorskip('torchaudio.functional')
    from kapre_b200.signal import filtfilt
    b, a = IR.biquad('lowpass', SR, 2000.0, 0.707)
    x = _x((4, 2, 30000), seed=5, scale=1.5)
    y = filtfilt(x, a, b, data_format=CF)
    b32, a32 = IR.normalised32(b, a)
    ref = F.filtfilt(x.cpu().double(), torch.from_numpy(a32.astype(np.float64)),
                     torch.from_numpy(b32.astype(np.float64))).numpy()
    assert np.abs(y.cpu().double().numpy() - ref).max() <= 1e-4


def test_bits_do_not_depend_on_batch_position_strides_or_prefix():
    from kapre_b200.signal import lfilter
    b, a = scipy.signal.butter(8, 0.4)
    x = _x((5, 3, 70001), seed=6)
    ref = lfilter(x, a, b, data_format=CF)
    for i in (0, 4):
        assert torch.equal(lfilter(x[i:i + 1].clone(), a, b, data_format=CF), ref[i:i + 1])
    big = _x((7, 4, 70020), seed=7)
    big[1:6, 1:4, 13:70014] = x
    assert torch.equal(lfilter(big[1:6, 1:4, 13:70014], a, b, data_format=CF), ref)
    for n in (1, 65, 2081, 33333):
        assert torch.equal(lfilter(x[..., :n].contiguous(), a, b, data_format=CF), ref[..., :n])
    # interleaved channels_last gives the channels_first bits, and mono either format
    assert torch.equal(lfilter(x.transpose(1, 2).contiguous(), a, b, data_format=CL).transpose(1, 2), ref)


def test_gradients_against_float64_through_a0_and_the_clamp():
    F = pytest.importorskip('torchaudio.functional')
    from kapre_b200.signal import lfilter
    b = np.array([0.4, 0.3, 0.2])
    a = np.array([1.6, -0.8, 0.3])                 # a0 != 1
    x = _x((3, 2, 5000), seed=8, scale=2.0)
    x.requires_grad_(True)
    tb = torch.tensor(b, dtype=torch.float32, device='cuda', requires_grad=True)
    ta = torch.tensor(a, dtype=torch.float32, device='cuda', requires_grad=True)
    gy = _x((3, 2, 5000), seed=9)
    y = lfilter(x, ta, tb, clamp=True, data_format=CF)
    assert float(y.detach().abs().max()) == 1.0                    # the clamp binds
    (y * gy).sum().backward()
    xd = x.detach().cpu().double().requires_grad_(True)
    rb = torch.tensor(b, dtype=torch.float64, requires_grad=True)
    ra = torch.tensor(a, dtype=torch.float64, requires_grad=True)
    yr = F.lfilter(xd, ra, rb, clamp=False)
    # the clamp mask of the float32 forward (outputs within float32 rounding of 1 may fall either way)
    with torch.no_grad():
        y_un = lfilter(x.detach(), ta.detach(), tb.detach(), clamp=False, data_format=CF).cpu().double()
    mask = (y_un.abs() <= 1).double()
    (yr * gy.cpu().double() * mask).sum().backward()
    for got, want in ((x.grad, xd.grad), (tb.grad, rb.grad), (ta.grad, ra.grad)):
        got, want = got.cpu().double().numpy(), want.numpy()
        assert np.abs(got - want).max() <= 2e-4 * max(1.0, np.abs(want).max()), (np.abs(got - want).max(), np.abs(want).max())


def test_trainable_iir_filter_receives_gradients():
    from kapre_b200.signal import IIRFilter
    f = IIRFilter([0.5, 0.2], [1.0, -0.3], trainable=True, data_format=CF)
    x = _x((2, 1, 4000), seed=10, scale=0.5)
    y = f(x)
    y.square().sum().backward()
    b, a = f.weights
    assert b.grad is not None and a.grad is not None
    assert torch.isfinite(b.grad).all() and torch.isfinite(a.grad).all() and float(b.grad.abs().sum()) > 0
    assert f.count_params() == 4


def test_requires_grad_leaves_the_forward_unchanged_and_launch_counts():
    from kapre_b200 import _native as N
    from kapre_b200.signal import filtfilt, lfilter
    b, a = IR.biquad('equalizer', SR, 1000.0, 1.0, 6.0)
    x = _x((4, 1, 50000), seed=11, scale=1.5)
    torch.cuda.synchronize()
    n0 = N.launch_count()
    y0 = lfilter(x, a, b, data_format=CF)
    assert N.launch_count() - n0 == 4                                # powers, state, carry, output
    xg = x.clone().requires_grad_(True)
    n0 = N.launch_count()
    y1 = lfilter(xg, a, b, data_format=CF)
    assert N.launch_count() - n0 == 4
    assert torch.equal(y0, y1.detach())
    n0 = N.launch_count()
    y1.sum().backward()
    assert N.launch_count() - n0 == 4                                # the backward's four
    n0 = N.launch_count()
    filtfilt(x, a, b, data_format=CF)
    assert N.launch_count() - n0 == 8


def test_biquad_before_the_fused_log_mel():
    import kapre_b200
    from kapre_b200 import _native as N
    from kapre_b200.composed import Sequential
    from kapre_b200.signal import Biquad
    bq = Biquad('highpass', SR, 300.0, data_format=CL)
    mel = kapre_b200.get_melspectrogram_layer(n_fft=1024, hop_length=256, sample_rate=SR, n_mels=64,
                                              return_decibel=True, input_data_format=CL, output_data_format=CL)
    model = Sequential([bq, *mel.layers])
    x = _x((8, SR, 1), seed=12)
    model.call(x)
    torch.cuda.synchronize()
    n0 = N.launch_count()
    out = model.call(x)
    n_model = N.launch_count() - n0
    y = bq.call(x)
    n0 = N.launch_count()
    assert torch.equal(mel.call(y), out)
    n_mel = N.launch_count() - n0
    assert n_model == 4 + n_mel and n_mel <= 2


def test_random_biquad_draws_and_capture():
    import kapre_b200
    from kapre_b200.augmentation import RandomBiquad
    from kapre_b200.backend import biquad_coefficients
    from kapre_b200.composed import Sequential
    from kapre_b200.signal import lfilter
    rb = RandomBiquad('bandpass', SR, (200.0, 4000.0), (0.5, 3.0), seed=5, data_format=CL)
    x = _x((8, SR, 1), seed=13)
    y = rb.call(x)
    freq, Q, gain = rb.last_choice
    b, a = biquad_coefficients('bandpass', SR, freq, Q, gain)
    b, a = b / a[:, :1], a / a[:, :1]
    for i in range(8):
        b32, a32 = b[i].astype(np.float32), a[i].astype(np.float32)
        ref = np.clip(IR.lfilter_fast(x[i, :, 0].cpu().double().numpy(), b32, a32), -1, 1)
        assert np.abs(y[i, :, 0].cpu().double().numpy() - ref).max() <= 1e-4
    # the gradient reaches the input
    xg = x.clone().requires_grad_(True)
    rb.call(xg).sum().backward()
    assert xg.grad is not None and torch.isfinite(xg.grad).all()
    # capture replays the draw made at capture time
    mel = kapre_b200.get_melspectrogram_layer(n_fft=512, hop_length=256, sample_rate=SR, n_mels=40,
                                              return_decibel=True, input_data_format=CL, output_data_format=CL)
    model = Sequential([rb, *mel.layers])
    cap = model.capture(x)
    freq, Q, gain = (v.copy() for v in rb.last_choice)
    r1 = cap(x).clone()
    rb.call(x)                                                       # a new eager draw does not change the graph
    r2 = cap(x).clone()
    assert torch.equal(r1, r2)
    b, a = biquad_coefficients('bandpass', SR, freq, Q, gain)
    b, a = b / a[:, :1], a / a[:, :1]
    want = mel.call(lfilter(x, torch.from_numpy(a.astype(np.float32)).reshape(8, 1, 3),
                            torch.from_numpy(b.astype(np.float32)).reshape(8, 1, 3), data_format=CL))
    assert torch.equal(r1, want)


def test_invalid_arguments_raise_before_any_launch():
    from kapre_b200 import _native as N
    from kapre_b200 import ops
    from kapre_b200.signal import lfilter
    x = _x((2, 2, 1000), seed=14)
    torch.cuda.synchronize()
    n0 = N.launch_count()
    for a, b in (([1.0] * 10, [1.0] * 10),                      # order 9
                 ([1.0, 0.5], [1.0, 0.5, 0.2]),                 # mismatched
                 (np.ones((3, 3)), np.ones((3, 3))),            # 3 filters for 2 channels
                 (np.ones((3, 2, 3)), np.ones((3, 2, 3))),      # batch 3 for 2 items
                 ([0.0, 0.5], [1.0, 0.5])):                     # a0 = 0 on the host
        with pytest.raises(ValueError):
            lfilter(x, a, b, data_format=CF)
    with pytest.raises(ValueError):
        lfilter(x[0], [1.0, 0.5], [1.0, 0.0], data_format=CF)
    with pytest.raises(N.KapreNativeError):
        lfilter(x.cpu(), [1.0, 0.5], [1.0, 0.0], data_format=CF)
    with pytest.raises(N.KapreNativeError):
        ops.lfilter_workspace(2, 2, 1000, 9, x.device)
    assert N.lib().kapre_lfilter_workspace_bytes(2, 2, 1000, 9) == -2        # KAPRE_E_UNSUPPORTED
    assert N.lib().kapre_lfilter_workspace_bytes(-1, 2, 1000, 2) == -1
    assert N.launch_count() == n0
