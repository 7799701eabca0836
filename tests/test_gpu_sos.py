"""Second-order-section cascades on the GPU: parity with the float64 restatement within the derived bound at benchmark
size (mono channels_first, stereo channels_last), a 10-minute recording, bit-independence of batch position, strides,
prefix length, format and broadcasting, zi / zf and streaming, sosfiltfilt against scipy, gradients against float64
autograd, requires_grad leaving the forward's bits unchanged, launch counts, SOSFilter in front of the fused log-mel
launch and under graph capture, butter(8, 0.05) against lfilter on the same design, and invalid arguments raising
before any launch."""
import numpy as np
import pytest
import scipy.signal
import torch

import sos_ref as SR

pytestmark = pytest.mark.gpu

FS = 16000
CF, CL = 'channels_first', 'channels_last'


def _designs():
    return {'butter8-0.05': scipy.signal.butter(8, 0.05, output='sos'),
            'telephone': scipy.signal.butter(8, [300, 3400], 'bandpass', fs=FS, output='sos'),
            'ellip8': scipy.signal.ellip(8, 0.5, 60, 0.125, output='sos'),
            'single': scipy.signal.butter(2, 0.1, output='sos')}


def _x(shape, seed, scale=1.0):
    return torch.from_numpy(np.random.default_rng(seed).uniform(-scale, scale, shape).astype(np.float32)).cuda()


def _bcl(t, fmt):
    a = t.detach().double().cpu().numpy()
    return a.transpose(0, 2, 1) if fmt == CL else a


def _check(y, x, sos32, fmt, zi=None, zf=None, what=''):
    xa = _bcl(x, fmt)
    z = None if zi is None else np.broadcast_to(np.asarray(zi, np.float64), xa.shape[:-1] + zi.shape[-2:])
    ref, zref = SR.sosfilt_fast(xa, sos32, z)
    by, bz = SR.error_bounds(xa, sos32, z)
    err = np.abs(_bcl(y, fmt) - ref).max()
    assert err <= by, (what, err, by)
    if zf is not None:
        assert np.abs(zf.cpu().double().numpy() - zref).max() <= bz, what
    return err, by


@pytest.mark.parametrize('name', ['butter8-0.05', 'telephone', 'ellip8', 'single'])
@pytest.mark.parametrize('fmt,C', [(CF, 1), (CL, 2)])
def test_parity_at_bench_size(name, fmt, C):
    from kapre_b200.signal import sosfilt
    sos = _designs()[name]
    shape = (256, C, 5 * FS) if fmt == CF else (256, 5 * FS, C)
    x = _x(shape, seed=C)
    y = sosfilt(x, sos, data_format=fmt)
    err, bound = _check(y, x, sos.astype(np.float32), fmt, what=name)
    print('%s %s C=%d: max|err| %.3g, bound %.3g' % (name, fmt, C, err, bound))


def test_ten_minute_recording():
    from kapre_b200.signal import sosfilt
    sos = _designs()['telephone']
    x = _x((1, 1, 600 * FS), seed=4)
    zi = np.random.default_rng(4).uniform(-1, 1, (8, 2)).astype(np.float32)
    y, zf = sosfilt(x, sos, zi=zi, data_format=CF)
    err, bound = _check(y, x, sos.astype(np.float32), CF, zi, zf)
    print('10 min: max|err| %.3g, bound %.3g' % (err, bound))


def test_bits_do_not_depend_on_batch_position_strides_prefix_format_or_broadcast():
    from kapre_b200.signal import sosfilt
    sos = _designs()['ellip8']
    x = _x((5, 3, 70001), seed=6)
    zi = np.random.default_rng(6).uniform(-1, 1, (5, 3, 4, 2)).astype(np.float32)
    ref, zref = sosfilt(x, sos, zi=zi, data_format=CF)
    for i in (0, 4):
        y, zf = sosfilt(x[i:i + 1].clone(), sos, zi=zi[i:i + 1], data_format=CF)
        assert torch.equal(y, ref[i:i + 1]) and torch.equal(zf, zref[i:i + 1])
    big = _x((7, 4, 70020), seed=7)
    big[1:6, 1:4, 13:70014] = x
    assert torch.equal(sosfilt(big[1:6, 1:4, 13:70014], sos, zi=zi, data_format=CF)[0], ref)
    for n in (1, 65, 2081, 33333):
        assert torch.equal(sosfilt(x[..., :n].contiguous(), sos, zi=zi, data_format=CF)[0], ref[..., :n])
    y, zf = sosfilt(x.transpose(1, 2).contiguous(), sos, zi=zi, data_format=CL)
    assert torch.equal(y.transpose(1, 2), ref) and torch.equal(zf, zref)
    # broadcast coefficients against materialised per-item ones
    s32 = torch.tensor(sos, dtype=torch.float32, device='cuda')
    assert torch.equal(sosfilt(x, s32.expand(5, 3, 4, 6).contiguous(), zi=zi, data_format=CF)[0], ref)


def test_per_item_coefficients_and_streaming():
    from kapre_b200.signal import sosfilt
    B, L = 4, 40000
    x = _x((B, L, 1), seed=3)
    sos = np.stack([scipy.signal.butter(4, [f, 2 * f], 'bandpass', fs=FS, output='sos') for f in (100, 400, 1600, 3000)])
    y = sosfilt(x, sos[:, None], data_format=CL)
    for i in range(B):
        _check(y[i:i + 1], x[i:i + 1], sos[i].astype(np.float32), CL, what=i)
    # pieces through zf -> zi stay within the bound of one call
    s = sos[1].astype(np.float32)
    whole = sosfilt(x, s, data_format=CL)
    _, bound = _check(whole, x, s, CL)
    z = np.zeros((4, 2), np.float32)
    parts = []
    for a, b in ((0, 1000), (1000, 1001), (1001, 25000), (25000, L)):
        yp, z = sosfilt(x[:, a:b], s, zi=z, data_format=CL)
        parts.append(yp)
    ref, _ = SR.sosfilt_fast(_bcl(x, CL), s)
    assert np.abs(_bcl(torch.cat(parts, 1), CL) - ref).max() <= bound


def test_sosfiltfilt_against_scipy():
    from kapre_b200.signal import sosfiltfilt
    x = _x((4, 2, 30000), seed=5)
    for name in ('telephone', 'single'):
        sos = _designs()[name]
        s32 = sos.astype(np.float32).astype(np.float64)
        for padtype, padlen in (('odd', None), ('even', 100), ('constant', None), (None, None)):
            y = sosfiltfilt(x, sos, padtype=padtype, padlen=padlen, data_format=CF)
            want = scipy.signal.sosfiltfilt(s32, x.cpu().double().numpy(), axis=-1, padtype=padtype, padlen=padlen)
            # two passes: the bound of the first carried through the second (its gain is at most ||h||_1), plus the
            # second's own bound on the first's output
            ext = SR.extend(x.cpu().double().numpy(), 3 * SR.n_taps(s32) if padlen is None else padlen, padtype)
            b1 = SR.error_bound(ext, s32)
            b2 = SR.error_bound(np.asarray(want), s32)
            h1 = sum(SR.response_l1(np.vstack([[1, 0, 0, 1, 0, 0], s32]), 0)[-1:])
            assert np.abs(y.cpu().double().numpy() - want).max() <= b1 * h1 + b2 + 1e-6, (name, padtype)
    with pytest.raises(ValueError):
        sosfiltfilt(x[..., :50], _designs()['telephone'], data_format=CF)          # length <= padlen


def test_gradients_against_float64():
    from kapre_b200.signal import sosfilt, sosfiltfilt
    sos = _designs()['telephone']
    s64 = sos.astype(np.float32).astype(np.float64)
    x = _x((2, 1, 3000), seed=8).requires_grad_(True)
    gy = _x((2, 1, 3000), seed=9)
    (sosfilt(x, sos, data_format=CF) * gy).sum().backward()
    # float64 adjoint: the same filter in reverse time
    want = SR.sosfilt_fast(gy.cpu().double().numpy()[..., ::-1], s64)[0][..., ::-1]
    assert np.abs(x.grad.cpu().double().numpy() - want).max() <= SR.error_bound(gy.cpu().double().numpy()[..., ::-1], s64)
    # sosfiltfilt: against central differences of scipy's float64 sosfiltfilt along random directions
    x2 = _x((1, 1, 500), seed=10).requires_grad_(True)
    g2 = _x((1, 1, 500), seed=11)
    (sosfiltfilt(x2, sos, data_format=CF) * g2).sum().backward()
    xn, gn = x2.detach().cpu().double().numpy(), g2.cpu().double().numpy()
    rng = np.random.default_rng(12)
    for _ in range(3):
        d = rng.standard_normal(xn.shape)
        f = lambda v: float((scipy.signal.sosfiltfilt(s64, v, axis=-1) * gn).sum())   # noqa: E731
        fd = (f(xn + 1e-4 * d) - f(xn - 1e-4 * d)) / 2e-4                    # linear: exact up to rounding
        got = float((x2.grad.cpu().double().numpy() * d).sum())
        assert abs(got - fd) <= 1e-3 * max(1.0, abs(fd)), (got, fd)


def test_requires_grad_leaves_the_forward_unchanged_and_launch_counts():
    from kapre_b200 import _native as N
    from kapre_b200.signal import sosfilt, sosfiltfilt
    sos = _designs()['ellip8']
    x = _x((4, 1, 50000), seed=11)
    torch.cuda.synchronize()
    n0 = N.launch_count()
    y0 = sosfilt(x, sos, data_format=CF)
    assert N.launch_count() - n0 == 4                                # powers, state, carry, output
    xg = x.clone().requires_grad_(True)
    n0 = N.launch_count()
    y1 = sosfilt(xg, sos, data_format=CF)
    assert N.launch_count() - n0 == 4
    assert torch.equal(y0, y1.detach())
    n0 = N.launch_count()
    y1.sum().backward()
    assert N.launch_count() - n0 == 4                                # the backward's four
    n0 = N.launch_count()
    sosfiltfilt(x, sos, data_format=CF)
    assert N.launch_count() - n0 == 8


def test_sos_filter_before_the_fused_log_mel_and_under_capture():
    import kapre_b200
    from kapre_b200 import _native as N
    from kapre_b200.composed import Sequential
    from kapre_b200.signal import SOSFilter
    f = SOSFilter(scipy.signal.butter(4, 50, 'highpass', fs=FS, output='sos'), data_format=CL)
    mel = kapre_b200.get_melspectrogram_layer(n_fft=1024, hop_length=256, sample_rate=FS, n_mels=64,
                                              return_decibel=True, input_data_format=CL, output_data_format=CL)
    model = Sequential([f, *mel.layers])
    x = _x((8, FS, 1), seed=12)
    model.call(x)
    torch.cuda.synchronize()
    n0 = N.launch_count()
    out = model.call(x)
    n_model = N.launch_count() - n0
    y = f.call(x)
    n0 = N.launch_count()
    assert torch.equal(mel.call(y), out)
    n_mel = N.launch_count() - n0
    assert n_model == 4 + n_mel and n_mel <= 2
    cap = model.capture(x)
    x2 = _x((8, FS, 1), seed=13)
    assert torch.equal(cap(x2).clone(), model.call(x2))


def test_butter8_stays_bounded_where_direct_form_diverges():
    from kapre_b200.signal import lfilter, sosfilt
    x = _x((2, 1, 5 * FS), seed=14)
    sos = scipy.signal.butter(8, 0.05, output='sos')
    y = sosfilt(x, sos, data_format=CF)
    _check(y, x, sos.astype(np.float32), CF)
    assert float(y.abs().max()) < 2
    b, a = scipy.signal.butter(8, 0.05)
    yd = lfilter(x, a, b, clamp=False, data_format=CF)
    assert not bool(torch.isfinite(yd).all()) or float(yd.abs().max()) > 1e6


def test_invalid_arguments_raise_before_any_launch():
    from kapre_b200 import _native as N
    from kapre_b200.signal import sosfilt, sosfiltfilt
    x = _x((2, 2, 1000), seed=15)
    sos = _designs()['single']
    bad = sos.copy()
    bad[0, 3] = 2.0
    torch.cuda.synchronize()
    n0 = N.launch_count()
    for s in (np.zeros((9, 6)), np.zeros((1, 5)), np.ones((3, 1, 6)), np.ones((3, 2, 1, 6)), bad):
        with pytest.raises(ValueError):
            sosfilt(x, s, data_format=CF)
    for z in (np.zeros((2, 2)), np.zeros((3, 1, 2)), np.zeros((3, 2, 1, 2))):
        with pytest.raises(ValueError):
            sosfilt(x, sos, zi=z, data_format=CF)
    with pytest.raises(ValueError):
        sosfilt(x, torch.tensor(sos, device='cuda', requires_grad=True), data_format=CF)
    with pytest.raises(ValueError):
        sosfilt(x, sos, zi=torch.zeros(1, 2, device='cuda', requires_grad=True), data_format=CF)
    with pytest.raises(ValueError):
        sosfiltfilt(x, sos, padtype='reflect', data_format=CF)
    with pytest.raises(ValueError):
        sosfiltfilt(x, sos, padlen=1000, data_format=CF)
    with pytest.raises(N.KapreNativeError):
        sosfilt(x.cpu(), sos, data_format=CF)
    assert N.launch_count() == n0
