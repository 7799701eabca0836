"""The persistent kernels where every CTA walks several tiles.

kb_resident_grid launches min(tiles, SMs x resident CTAs per SM) CTAs and each CTA loops over tiles cta, cta + grid,
...  Only when tiles > grid does a CTA reuse its shared buffers, reach the second mbarrier phase and mix bulk-copied
tiles with tiles of the cooperative loader (an item's edge tiles never take the bulk path).  Each test reads the
resident grid of every launch it makes from the launch report ("<kernel> grid=G tiles=T"), picks an input size whose
tiles per item do not divide that grid and give each (item, channel group) edge and interior tiles, and sizes the
batch so that tiles >= 3 x grid.  It then asserts that every item has the bits of the same item run in launches where
no CTA has more than one tile, that the bits do not change with the input's storage offset (1-3 floats) or for a
channels-last view, and that the first, middle and last items are within the kernel's bound of the float64
restatement, forward and backward.  Each test stays well under 2 GB of device memory."""
import math
import re

import numpy as np
import pytest
import torch

import resample_ref as RR
import sinc_ref as SR

pytestmark = pytest.mark.gpu
CF = 'channels_first'


def _launch(fn):
    """fn() on the device, synchronised; (its result, kernel name, grid, tiles) of the first persistent launch the
    call reports."""
    from kapre_b200 import _native as N
    out = fn()
    torch.cuda.synchronize()
    info = N.last_launch_info()
    m = re.search(r'(\w+) grid=(\d+) tiles=(\d+)', info)
    assert m, info
    return out, m.group(1), int(m.group(2)), int(m.group(3))


def _placed(x, k):
    """A contiguous copy of x whose storage starts k floats into a fresh (256 B aligned) allocation."""
    buf = torch.empty(x.numel() + 8, device=x.device, dtype=x.dtype)
    out = buf[k:k + x.numel()].view(x.shape)
    out.copy_(x)
    assert out.storage_offset() == k
    return out


def _channels_last_view(x):
    """x (B, C, ...) with its C channels innermost in memory."""
    perm = [0] + list(range(2, x.dim())) + [1]
    inv = [0, x.dim() - 1] + list(range(1, x.dim() - 1))
    return x.permute(*perm).contiguous().permute(*inv)


def _max_resident(threads):
    return torch.cuda.get_device_properties(0).multi_processor_count * (2048 // threads)


def _pick(sizes, passes, groups, threads):
    """The first size at which every pass (run, make, name) has at least 3 tiles per channel group and tiles per item
    that do not divide its resident grid.  run(input, size) -> output; make(B, size) -> input of B items.  Returns
    (size, B) with B the batch that gives every pass tiles >= 3 x grid."""
    caps = {}
    for size in sizes:
        per = []
        for run, make, name in passes:
            _, nm, g, t = _launch(lambda: run(make(1, size), size))
            assert nm == name and t <= g, (nm, g, t)
            if t < 3 * groups:
                break
            if name not in caps:      # the resident grid depends on the kernel's shape, not on the size
                # (Kaldi's tiles are CTAs of 8 frame jobs, so a batch of n items has at least n (t - 1) of them)
                n = 2 * (_max_resident(threads) // t + 1)
                _, _, caps[name], tiles = _launch(lambda: run(make(n, size), size))
                assert tiles > caps[name]
            per.append((t, caps[name]))
        if len(per) == len(passes) and all(cap % t != 0 for t, cap in per):
            return size, max(math.ceil(3 * cap / (t - 1)) + 1 for t, cap in per)
    raise AssertionError('no size gives tiles per item that do not divide the grid')


def _walk(run, x, name, view=True):
    """run(x) walked (tiles >= 3 grid) against the same items in launches of at most one tile per CTA, at storage
    offsets 1-3 and as a channels-last view.  Returns the walked output."""
    _, nm, g1, per_item = _launch(lambda: run(x[:1]))
    assert nm == name and per_item <= g1
    y, nm, grid, tiles = _launch(lambda: run(x))
    assert nm == name and tiles >= 3 * grid and grid % per_item != 0, (nm, grid, tiles, per_item)
    chunk = max(1, grid // per_item)
    for i in range(0, x.shape[0], chunk):
        yi, nm, g, t = _launch(lambda: run(x[i:i + chunk]))
        assert nm == name and t <= g, (nm, g, t)
        assert torch.equal(yi, y[i:i + chunk]), i
    for k in (1, 2, 3):
        assert torch.equal(run(_placed(x, k)), y), k
    if view:
        assert torch.equal(run(_channels_last_view(x)), y)
    return y


def _sample(B):
    return [0, B // 2, B - 1]


def _uniform(shape, seed):
    g = torch.Generator(device='cuda').manual_seed(seed)
    return torch.rand(shape, device='cuda', generator=g) * 2 - 1


def _zeros(B, C, L):
    return torch.zeros((B, C, L), device='cuda')


SIZES = [1000 * n + 37 for n in range(3, 80)]


# ------------------------------------------------------------------------------------------ polyphase resampler
@pytest.mark.parametrize('orig,target', [(48000, 16000), (16000, 22050)])
def test_resample_walks(orig, target):
    from kapre_b200 import ops
    from kapre_b200.signal import resample_filter
    up, down = RR.up_down(orig, target)
    plan = ops.ResamplePlan(up, down, resample_filter(up, down))

    def fwd(x, L):
        return ops.resample(x, plan, CF)

    def bwd(gy, L):
        return ops.resample_backward(gy, plan, CF, L)

    L, B = _pick(SIZES, [(fwd, lambda B, L: _zeros(B, 2, L), 'resample'),
                         (bwd, lambda B, L: _zeros(B, 2, RR.output_length(L, up, down)), 'resample')], 2, 256)
    x = _uniform((B, 2, L), orig + target)
    y = _walk(lambda t: fwd(t, L), x, 'resample')
    gy = _uniform(tuple(y.shape), orig + target + 1)
    gx = _walk(lambda t: bwd(t, L), gy, 'resample')
    pick = _sample(B)
    want = RR.resample(x[pick].double().cpu(), up, down)
    assert float((y[pick].double().cpu() - want).abs().max()) <= 1e-5 * float(x.abs().max())
    # the adjoint in float64: A^T g = (up / down) resample(g; down, up) with the same filter, cropped to L samples
    want = RR.resample(gy[pick].double().cpu(), down, up, h=RR.taps(up, down), length=L) * (up / down)
    assert float((gx[pick].double().cpu() - want).abs().max()) <= 1e-5 * max(1.0, up / down) * float(gy.abs().max())


# ------------------------------------------------------------------------------------------ band-limited interpolator
@pytest.mark.parametrize('ratio', [2.0 ** (-4 / 12), 1.5])
def test_sinc_walks(ratio):
    from kapre_b200 import ops
    offset = 0.75

    def fwd(x, L):
        return ops.sinc_resample(x, ratio, SR.output_length(L, ratio), offset, CF)

    def bwd(gy, L):
        return ops.sinc_resample_backward(gy, ratio, offset, CF, L)

    L, B = _pick(SIZES, [(fwd, lambda B, L: _zeros(B, 2, L), 'sinc'),
                         (bwd, lambda B, L: _zeros(B, 2, SR.output_length(L, ratio)), 'sinc')], 2, 512)
    x = _uniform((B, 2, L), int(ratio * 1000))
    y = _walk(lambda t: fwd(t, L), x, 'sinc')
    gy = _uniform(tuple(y.shape), int(ratio * 1000) + 1)
    gx = _walk(lambda t: bwd(t, L), gy, 'sinc')
    pick = _sample(B)
    want = SR.resample(x[pick].double().cpu(), ratio, y.shape[2], offset)
    assert float((y[pick].double().cpu() - want).abs().max()) <= SR.error_bound(ratio) * float(x.abs().max())
    for b in pick:
        for c in range(2):
            want = SR.resample(gy[b, c].double().cpu(), ratio, L, _numbers=SR.adjoint_numbers(ratio, offset))
            err = float((gx[b, c].double().cpu() - want).abs().max())
            assert err <= SR.error_bound(ratio, True) * float(gy.abs().max()), (b, c, err)


# ------------------------------------------------------------------------------------------ spectral convolution
def test_spec_conv_walks():
    """The multiply-accumulate of the partitioned convolution, forward and for the signal gradient (tiles of 32 bins
    x 64 output blocks of one (item, channel)), against scipy's float64 convolution within conv_ref.error_bound."""
    import conv_ref as CR
    import scipy.signal
    from kapre_b200 import ops
    from test_gpu_convolve import _h, _vjp_ref
    K = 300
    plan = ops.convolve_plan(ops.convolve_block_size(K))
    h = _h(K)
    H = ops.convolve_ir_spectrum(h.view(1, 1, K), plan, CF)

    def fwd(x, L):
        return ops.convolve_full(x, H, plan, CF)[0]

    def bwd(g_full, L):
        return ops.convolve_backward(g_full, H, None, plan, CF, L, True, False)[0]

    def full_len(L):
        return (-(-L // plan.block) + H.shape[2]) * plan.block

    L, B = _pick(SIZES, [(fwd, lambda B, L: _zeros(B, 2, L), 'spec_conv'),
                         (bwd, lambda B, L: _zeros(B, 2, full_len(L)), 'spec_conv')], 2, 256)
    x = _uniform((B, 2, L), 7)
    y = _walk(lambda t: fwd(t, L), x, 'spec_conv')
    start, n = ops.convolve_span(L, K, 'full')
    g = torch.zeros(y.shape, device='cuda')
    g[..., start:start + n] = torch.randn((B, 2, n), device='cuda', generator=torch.Generator(device='cuda').manual_seed(8))
    gx = _walk(lambda t: bwd(t, L), g, 'spec_conv')
    pick = _sample(B)
    bound = CR.error_bound(plan.block, -(-K // plan.block))
    xa, ha = x[pick].double().cpu().numpy(), h.double().cpu().numpy()
    want = scipy.signal.fftconvolve(xa, ha[None, None, :], axes=-1)
    scale = np.sqrt(np.mean(xa ** 2)) * np.sqrt((ha ** 2).sum())
    assert np.abs(y[pick][..., start:start + n].double().cpu().numpy() - want).max() / scale <= bound
    gs = g[pick][..., start:start + n]
    rgx, _ = _vjp_ref(x[pick], h, gs, CF)
    sx = np.sqrt(np.mean(gs.double().cpu().numpy() ** 2)) * float(h.norm())
    assert np.abs(gx[pick].double().cpu().numpy() - rgx).max() / sx <= bound


# ------------------------------------------------------------------------------------------ filterbank inversion
def test_fbinv_walks():
    """InverseFilterbank (it has no backward): tiles of R frames of one (item, channel), against the float64
    restatement within the bound of test_gpu_filterbank_inverse."""
    import fbinv_ref as FR
    from test_gpu_filterbank_inverse import BANKS, _bound, _frame_err, _layer, _reference
    bank = BANKS[2]
    fb = FR.bank(*bank)
    layer = _layer(bank, 30, CF)
    K = fb.shape[1]

    def fwd(m, T=None):
        with torch.no_grad():
            return layer(m)

    T, B = _pick(list(range(20, 600, 7)), [(fwd, lambda B, T: torch.zeros((B, 2, T, K), device='cuda'), 'fbinv')], 2, 256)
    m = torch.from_numpy(FR.consistent_input(fb, bank[1], bank[2], B, 2, T).astype(np.float32)).cuda()
    y = _walk(fwd, m, 'fbinv')
    pick = _sample(B)
    want, drift = _reference(fb, m[pick].cpu().numpy(), 30)
    assert float(_frame_err(y[pick].double().cpu().numpy(), want).max()) <= _bound(drift)


# ------------------------------------------------------------------------------------------ Kaldi features
def test_kaldi_walks():
    """Forward and backward (fbank, 40 bins).  Their CTAs take jobs of frames with no bulk copy, so the size only has
    to give tiles that do not divide the grid.  The backward is called through its entry point: autograd would run it
    on another thread, whose launch report this one cannot see.  References: torchaudio in float64 on three items,
    within the bounds of test_gpu_kaldi."""
    from kapre_b200 import ops
    import kaldi_ref as R
    from test_gpu_kaldi import _ref, _ta, _x

    kw = dict(num_mel_bins=40)
    o = ops.kaldi_options('fbank', **kw)
    plan = ops.kaldi_plan('fbank', o)

    def fwd(x, L=None):
        return ops.kaldi_features(x, plan, data_format=CF)

    def bwd(x, gy):
        return ops.kaldi_backward(gy, x, plan, None, None, CF, 0.0, 0)

    def make_g(B, L):
        return torch.zeros((B,) + tuple(fwd(_zeros(1, 2, L)).shape[1:]), device='cuda')

    L, B = _pick([16000 + 160 * n + 123 for n in range(60)],
                 [(fwd, lambda B, L: _zeros(B, 2, L), 'kaldi_fwd'),
                  (lambda g, L: bwd(_zeros(g.shape[0], 2, L), g), make_g, 'kaldi_bwd')], 1, 256)
    x = _x(B, 2, L, 5)
    y = _walk(fwd, x, 'kaldi_fwd')
    gy = torch.randn(y.shape, device='cuda', generator=torch.Generator(device='cuda').manual_seed(1))
    # the backward takes two inputs, so its walk is spelled out
    per_item = _launch(lambda: bwd(x[:1], gy[:1]))[3]
    gx, nm, grid, tiles = _launch(lambda: bwd(x, gy))
    assert nm == 'kaldi_bwd' and tiles >= 3 * grid and grid % per_item != 0, (grid, tiles, per_item)
    chunk = max(1, grid // per_item)
    for i in range(0, B, chunk):
        gi, nm, g, t = _launch(lambda: bwd(x[i:i + chunk], gy[i:i + chunk]))
        assert nm == 'kaldi_bwd' and t <= g and torch.equal(gi, gx[i:i + chunk]), i
    for k in (1, 2, 3):
        assert torch.equal(bwd(_placed(x, k), _placed(gy, k)), gx), k
    assert torch.equal(bwd(_channels_last_view(x), _channels_last_view(gy)), gx)

    pick = _sample(B)
    xs = x[pick].contiguous()
    ref = _ref('fbank', xs, o)
    bound = R.log_bound('fbank', xs.cpu().numpy(), o, None, ref.cpu().numpy()) + 2e-4 * np.abs(ref.cpu().numpy())
    assert ((y[pick].double() - ref).abs().cpu().numpy() <= bound).all()
    xd = xs.double().requires_grad_(True)
    total = sum((_ta('fbank', xd[j, c:c + 1], dict(kw)) * gy[b, c].double()).sum()
                for j, b in enumerate(pick) for c in range(2))
    total.backward()
    assert (gx[pick].double() - xd.grad).abs().max().item() <= 2e-3 * xd.grad.abs().max().item()
