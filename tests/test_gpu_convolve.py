"""The partitioned FFT convolution on the GPU: parity with float64 ``scipy.signal.fftconvolve`` at the benchmark's size
for each filter length and in both formats, every broadcast form and mode, views and short signals, bits that do not
depend on the batch or the format, the vector-Jacobian products to x and h against the float64 restatement and the
adjoint identity, launch counts, ``Reverb`` in front of the fused log-mel launch and under graph capture, requires-grad
leaving the forward unchanged, and invalid arguments raising before any launch.  Bounds: conv_ref.error_bound."""
import numpy as np
import pytest
import scipy.signal
import torch

import conv_ref as CR

pytestmark = pytest.mark.gpu
CL, CF = 'channels_last', 'channels_first'


def _x(fmt, B, C, L, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.rand((B, L, C) if fmt == CL else (B, C, L), generator=g) * 2 - 1
    return x.cuda()


def _h(K, seed=1):
    """A (K,) filter: noise under an exponential decay, like a room response."""
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(K, generator=g) * torch.exp(-torch.arange(K) / (K / 4.0))).cuda()


def _cf(t, fmt):
    """(B, C, L) float64 NumPy view of a (B, L, C) / (B, C, L) tensor."""
    a = t.detach().cpu().double().numpy()
    return a.transpose(0, 2, 1) if fmt == CL else a


def _ref_full(x, h, fmt):
    """float64 full convolution, (B, C, L + K - 1); h (K,) or 3-D in fmt."""
    xa = _cf(x, fmt)
    ha = h.detach().cpu().double().numpy()
    ha = ha[None, None, :] if ha.ndim == 1 else (ha.transpose(0, 2, 1) if fmt == CL else ha)
    return scipy.signal.fftconvolve(xa, ha, axes=-1)


def _check(got, want, x, h, fmt):
    got = _cf(got, fmt)
    assert got.shape == want.shape, (got.shape, want.shape)
    K = h.shape[-1] if h.dim() == 1 else h.shape[1 if fmt == CL else 2]
    B = CR.block_size(K)
    xa, ha = _cf(x, fmt), h.detach().cpu().double().numpy()
    hn = np.sqrt((ha.reshape(-1, K) ** 2).sum(-1)).max() if h.dim() == 1 or fmt == CF else \
        np.sqrt((ha ** 2).sum(1)).max()
    scale = np.sqrt(np.mean(xa ** 2)) * hn
    err = np.abs(got - want).max() / scale
    assert err <= CR.error_bound(B, -(-K // B)), err
    return err


@pytest.mark.parametrize('K', [256, 2000, 16000, 48000])
@pytest.mark.parametrize('fmt,C', [(CF, 1), (CL, 2)])
def test_parity_at_bench_size(K, fmt, C):
    from kapre_b200 import ops
    x = _x(fmt, 256, C, 80000)
    h = _h(K)
    y = ops.convolve(x, h, 'full', fmt)
    torch.cuda.synchronize()
    items = [0, 1, 77, 128, 200, 255]
    sel = y[items]
    _check(sel, _ref_full(x[items], h, fmt), x[items], h, fmt)


@pytest.mark.parametrize('mode', ['full', 'same', 'valid'])
@pytest.mark.parametrize('fmt', [CF, CL])
def test_broadcast_forms_and_modes(mode, fmt):
    from kapre_b200 import ops
    B, C, L, K = 3, 2, 3000, 700
    x = _x(fmt, B, C, L, seed=2)
    g = torch.Generator().manual_seed(3)
    shapes = [(K,)] + [((b, K, c) if fmt == CL else (b, c, K)) for b in (1, B) for c in (1, C)]
    for shp in shapes:
        h = (torch.randn(shp, generator=g) * 0.1).cuda()
        y = ops.convolve(x, h, mode, fmt)
        full = _ref_full(x, h, fmt)
        start, n = CR.span(L, K, mode)
        _check(y, full[..., start:start + n], x, h, fmt)


def test_valid_with_a_filter_longer_than_the_signal_and_short_signals():
    from kapre_b200 import ops
    for L, K in ((50, 3000), (1, 1), (1, 5000), (127, 129), (5, 1)):
        x = _x(CF, 2, 1, L, seed=L)
        h = _h(K, seed=K)
        for mode in ('full', 'same', 'valid'):
            y = ops.convolve(x, h, mode, CF)
            start, n = CR.span(L, K, mode)
            _check(y, _ref_full(x, h, CF)[..., start:start + n], x, h, CF)


def test_strided_views_give_the_bits_of_contiguous_copies():
    from kapre_b200 import ops
    big = _x(CF, 6, 4, 5000, seed=9)
    x = big[1:5, 1:3, 100:4100]
    h_big = torch.randn(3, 2500, device='cuda')
    h = h_big[1, ::2]
    y = ops.convolve(x, h, 'full', CF)
    assert torch.equal(y, ops.convolve(x.contiguous(), h.contiguous(), 'full', CF))


@pytest.mark.parametrize('fmt', [CF, CL])
def test_bits_do_not_depend_on_batch_size_or_position(fmt):
    from kapre_b200 import ops
    x = _x(fmt, 16, 2, 20000, seed=4)
    h = _h(3000)
    y = ops.convolve(x, h, 'full', fmt)
    for i in (0, 5, 15):
        assert torch.equal(ops.convolve(x[i:i + 1], h, 'full', fmt), y[i:i + 1])
    assert torch.equal(ops.convolve(x[3:11], h, 'full', fmt), y[3:11])


def test_formats_agree_and_a_mono_item_gives_the_bits_of_either_format():
    """The multiply-accumulate and the inverse give an element the same bits in either layout, but an interleaved
    multi-channel waveform is transformed by the STFT's all-channel kernel, which agrees with the single-channel
    kernel to float32 rounding, not bit for bit; one channel takes the same kernel in both layouts."""
    from kapre_b200 import ops
    x = _x(CF, 16, 2, 20000, seed=4)
    h = _h(3000)
    y = ops.convolve(x, h, 'full', CF)
    y_cl = ops.convolve(x.transpose(1, 2).contiguous(), h, 'full', CL).transpose(1, 2)
    _check(y_cl, _ref_full(x, h, CF), x, h, CF)
    scale = float(x.pow(2).mean().sqrt() * h.norm())
    assert float((y_cl - y).abs().max()) <= CR.error_bound(CR.block_size(3000), 3) * scale
    m = x[:, :1]
    assert torch.equal(ops.convolve(m.transpose(1, 2).contiguous(), h, 'full', CL).transpose(1, 2),
                       ops.convolve(m, h, 'full', CF))


def _vjp_ref(x, h, g, fmt):
    """float64 gradients of <g, full conv> for a shared filter h (K,): gx = corr(g, h), gh = sum over (b, c)."""
    xa, ga, ha = _cf(x, fmt), _cf(g, fmt), h.detach().cpu().double().numpy()
    L, K = xa.shape[-1], ha.shape[0]
    gx = scipy.signal.fftconvolve(ga, ha[::-1][None, None, :], axes=-1)[..., K - 1:K - 1 + L]
    gh = scipy.signal.fftconvolve(ga, xa[..., ::-1], axes=-1)[..., L - 1:L - 1 + K].sum((0, 1))
    return gx, gh


@pytest.mark.parametrize('fmt,C', [(CF, 1), (CL, 2)])
@pytest.mark.parametrize('K', [300, 16000])
def test_vjp_against_float64(fmt, C, K):
    from kapre_b200 import ops
    x = _x(fmt, 8, C, 20000, seed=5).requires_grad_(True)
    h = _h(K).requires_grad_(True)
    y = ops.convolve(x, h, 'full', fmt)
    g = torch.randn(y.shape, generator=torch.Generator().manual_seed(6)).cuda()
    gx, gh = torch.autograd.grad(y, (x, h), g)
    rgx, rgh = _vjp_ref(x, h, g, fmt)
    B = CR.block_size(K)
    bound = CR.error_bound(B, -(-K // B))
    sx = np.sqrt(np.mean(_cf(g, fmt) ** 2)) * float(h.detach().norm())
    assert np.abs(_cf(gx, fmt) - rgx).max() / sx <= bound
    sh = np.abs(rgh).max()
    assert np.abs(gh.detach().cpu().double().numpy() - rgh).max() / sh <= 1e-4


@pytest.mark.parametrize('mode', ['same', 'valid'])
def test_vjp_of_cropped_and_broadcast_filters(mode):
    from kapre_b200 import ops
    B, C, L, K = 4, 2, 3000, 900
    x = _x(CL, B, C, L, seed=8).requires_grad_(True)
    h = (torch.randn(1, K, C, generator=torch.Generator().manual_seed(9)) * 0.1).cuda().requires_grad_(True)
    y = ops.convolve(x, h, mode, CL)
    g = torch.randn(y.shape, generator=torch.Generator().manual_seed(10)).cuda()
    gx, gh = torch.autograd.grad(y, (x, h), g)
    # float64 autograd through the explicit full convolution, cropped the same way
    xd = x.detach().cpu().double().requires_grad_(True)
    hd = h.detach().cpu().double().requires_grad_(True)
    conv = torch.nn.functional.conv1d                        # cross-correlation: flip the filter
    full = torch.stack([torch.stack([conv(xd[b:b + 1, :, c].reshape(1, 1, L), hd[0, :, c].flip(0).reshape(1, 1, K),
                                          padding=K - 1).reshape(-1) for c in range(C)], -1) for b in range(B)])
    start, n = CR.span(L, K, mode)
    full[:, start:start + n].backward(g.cpu().double())
    assert torch.allclose(gx.cpu().double(), xd.grad, rtol=0, atol=1e-4 * float(xd.grad.abs().max()))
    assert torch.allclose(gh.cpu().double(), hd.grad, rtol=0, atol=1e-4 * float(hd.grad.abs().max()))


def test_adjoint_identity_at_bench_shape():
    from kapre_b200 import ops
    x = _x(CF, 256, 1, 80000, seed=11).requires_grad_(True)
    h = _h(16000).requires_grad_(True)
    y = ops.convolve(x, h, 'full', CF)
    g = torch.randn(y.shape, generator=torch.Generator().manual_seed(12)).cuda()
    gx, gh = torch.autograd.grad(y, (x, h), g)
    # the map is bilinear: <g, y> = <gx, x> = <gh, h>
    y = y.detach()
    gy = float((g.double() * y.double()).sum())
    tol = 1e-5 * float(g.double().norm() * y.double().norm())
    assert abs(float((gx.double() * x.detach().double()).sum()) - gy) <= tol
    assert abs(float((gh.double() * h.detach().double()).sum()) - gy) <= tol


def test_launch_counts_and_requires_grad_leaves_the_forward_unchanged():
    from kapre_b200 import _native as N
    from kapre_b200 import ops
    x = _x(CL, 8, 2, 16000, seed=13)
    h = _h(4000)
    ops.convolve(x, h, 'full', CL)
    torch.cuda.synchronize()
    n0 = N.launch_count()
    y = ops.convolve(x, h, 'same', CL)
    assert N.launch_count() - n0 == 4                       # filter spectra, STFT, MAC, inverse
    plan = ops.convolve_plan(ops.convolve_block_size(4000))
    H = ops.convolve_ir_spectrum(h.view(1, -1, 1), plan, CL)
    n0 = N.launch_count()
    ops.convolve_spectrum(x, H, plan, 0, 16000, CL)
    assert N.launch_count() - n0 == 3                       # with cached spectra
    for xr, hr in ((True, False), (False, True), (True, True)):
        xg, hg = x.clone().requires_grad_(xr), h.clone().requires_grad_(hr)
        n0 = N.launch_count()
        yg = ops.convolve(xg, hg, 'same', CL)
        assert N.launch_count() - n0 == 4
        assert torch.equal(yg.detach(), y)


def test_invalid_arguments_raise_before_any_launch():
    from kapre_b200 import _native as N
    from kapre_b200 import ops
    x = _x(CF, 2, 2, 1000)
    ops.convolve(x, _h(100), 'full', CF)
    n0 = N.launch_count()
    bad = [(x, torch.zeros(0, device='cuda'), 'full'), (x, _h(100), 'circular'),
           (x, torch.zeros(3, 2, 10, device='cuda'), 'full'), (x, torch.zeros(1, 3, 10, device='cuda'), 'full'),
           (x[:, :, :0], _h(100), 'full'), (x, torch.zeros(10, 10, device='cuda'), 'full')]
    for xa, ha, mode in bad:
        with pytest.raises((ValueError, N.KapreNativeError)):
            ops.convolve(xa, ha, mode, CF)
    # (T + 1) B beyond int32: checked by the library before the filter's spectra are made
    with pytest.raises(N.KapreNativeError):
        ops.convolve(torch.zeros(1, 1, 1, device='cuda').expand(1, 1, 2 ** 31 - 2000), _h(16000), 'full', CF)
    assert N.launch_count() == n0
    plan = ops.convolve_plan(128)
    lib = N.lib()
    assert lib.kapre_convolve_workspace_bytes(plan.handle(), 1, 1, 0, 1) == -1
    assert lib.kapre_convolve_workspace_bytes(plan.handle(), 1, 1, 10, 0) == -1
    import ctypes
    out = ctypes.c_void_p()
    assert lib.kapre_convolve_plan_create(300, ctypes.byref(out)) == -1
    assert N.launch_count() == n0


def test_reverb_before_the_fused_log_mel_and_under_capture():
    import kapre_b200
    from kapre_b200 import _native as N
    from kapre_b200.augmentation import Reverb
    from kapre_b200.composed import Sequential
    rng = np.random.default_rng(0)
    rirs = [rng.standard_normal(n) * np.exp(-np.arange(n) / 800.0) for n in (3000, 8000, 16000)]
    rev = Reverb(rirs, seed=1, data_format='channels_last')
    mel = kapre_b200.get_melspectrogram_layer(n_fft=1024, hop_length=256, sample_rate=16000, n_mels=64,
                                              return_decibel=True, input_data_format='channels_last',
                                              output_data_format='channels_last')
    model = Sequential([rev, *mel.layers])
    x = _x(CL, 8, 1, 16000, seed=14)
    model.call(x)
    torch.cuda.synchronize()
    n0 = N.launch_count()
    out = model.call(x)
    n_model = N.launch_count() - n0
    choice = rev.last_choice
    y = rev.call(x, rir_index=choice)
    n0 = N.launch_count()
    assert torch.equal(mel.call(y), out)
    n_mel = N.launch_count() - n0
    assert n_model == 3 + n_mel and n_mel <= 2              # the log-mel behind Reverb is still the fused launch
    # the reverberated signal against float64, time-aligned with the direct path
    bank = rev.bank.astype(np.float64)
    xa = x.cpu().double().numpy()[:, :, 0]
    for i in range(8):
        want = np.convolve(xa[i], bank[choice[i]])[:16000]
        err = np.abs(y[i, :, 0].cpu().double().numpy() - want).max() / np.sqrt(np.mean(xa[i] ** 2))
        assert err <= CR.error_bound(rev.plan.block, -(-bank.shape[1] // rev.plan.block))
    # capture replays the draw made at capture time
    cap = model.capture(x)
    drawn = rev.last_choice.copy()
    r1 = cap(x).clone()
    rev.call(x)                                              # a new eager draw does not change the graph
    r2 = cap(x).clone()
    assert torch.equal(r1, r2)
    assert torch.equal(r1, mel.call(rev.call(x, rir_index=drawn)))


def test_reverb_gradient_reaches_the_input():
    from kapre_b200.augmentation import Reverb
    rng = np.random.default_rng(2)
    rev = Reverb([rng.standard_normal(500), rng.standard_normal(900)], seed=0, data_format='channels_first')
    x = _x(CF, 4, 2, 4000, seed=15).requires_grad_(True)
    y = rev.call(x, rir_index=[0, 1, 1, 0])
    g = torch.randn(y.shape, generator=torch.Generator().manual_seed(16)).cuda()
    (gx,) = torch.autograd.grad(y, (x,), g)
    bank = rev.bank.astype(np.float64)
    ga = g.cpu().double().numpy()
    for i, r in enumerate([0, 1, 1, 0]):
        h = bank[r]
        want = scipy.signal.fftconvolve(ga[i], h[::-1][None, :], axes=-1)[:, h.size - 1:h.size - 1 + 4000]
        assert np.abs(gx[i].cpu().double().numpy() - want).max() <= 1e-4 * np.abs(want).max()
