"""The persistent kernels where every CTA walks several tiles.

kb_resident_grid launches min(tiles, SMs x resident CTAs per SM) CTAs and each CTA loops over tiles cta, cta + grid,
...  Only when tiles > grid does a CTA reuse its shared buffers, reach the second mbarrier phase and mix bulk-copied
tiles with tiles of the cooperative loader (an item's edge tiles never take the bulk path), or start a tile of another
item, channel or row with what the previous tile left in shared memory.  Each test reads the resident grid of every
launch it makes from the launch report ("<kernel> grid=G tiles=T", joined with "; " when a call makes several), picks
an input size whose tiles per item do not divide that grid and give each (item, channel group) edge and interior
tiles (a partial last tile in every tiled dimension), and sizes the batch so that tiles >= 3 x grid; kernels that take
one row per job only need that many rows.  It then asserts that every item has the bits of the same item run in
launches where no CTA has more than one tile, that the bits do not change with the input's storage offset (1-3
elements) or for a channels-last view, and that the first, middle and last items are within the bound of the op's own
GPU test against the float64 restatement, forward and backward (discrete decisions: the float64 rule applied to the
kernel's own continuous intermediate).  Backward passes are called through their entry points: autograd would run
them on another thread, whose launch report this one cannot see.

Kernels covered: resample, sinc, spec_conv, fbinv, kaldi_fwd and kaldi_bwd; cqt_fwd and every octave's cqt_bwd;
pitch and viterbi; chroma, chroma_bwd, cens, tune_peak, tune_select and tune_argmax; hpss, hpss_bwd and hpss_gather;
onset, onset_bwd, onset_gather, tempogram, tempo_part, tempo, onset_detect and beat_track.  Each test stays under 2 GB
of device memory, which the module asserts."""
import math
import re

import numpy as np
import pytest
import torch

import resample_ref as RR
import sinc_ref as SR

pytestmark = pytest.mark.gpu
CF = 'channels_first'


def _launch(fn, *names):
    """fn() on the device, synchronised; (its result, [(name, grid, tiles)]) of every persistent launch of `names` the
    call reports ("<kernel> grid=G tiles=T", joined with "; " when a call makes several), by name, then launch order."""
    from kapre_b200 import _native as N
    out = fn()
    torch.cuda.synchronize()
    info = N.last_launch_info()
    reps = []
    for name in names:
        found = re.findall(r'(?:^|; )%s grid=(\d+) tiles=(\d+)' % name, info)
        assert found, (name, info)
        reps += [(name, int(g), int(t)) for g, t in found]
    return out, reps


def _placed(x, k):
    """A contiguous copy of x whose storage starts k elements (floats, or complex64 values) into a fresh (256 B
    aligned) allocation."""
    buf = torch.empty(x.numel() + 8, device=x.device, dtype=x.dtype)
    out = buf[k:k + x.numel()].view(x.shape)
    out.copy_(x)
    assert out.storage_offset() == k
    return out


def _channels_last_view(x):
    """x (B, C, ...) with its C channels innermost in memory (x itself when it has no channel dimension)."""
    if x.dim() < 3:
        return x
    perm = [0] + list(range(2, x.dim())) + [1]
    inv = [0, x.dim() - 1] + list(range(1, x.dim() - 1))
    return x.permute(*perm).contiguous().permute(*inv)


def _max_resident(threads):
    return torch.cuda.get_device_properties(0).multi_processor_count * min(32, 2048 // threads)


def _pick(sizes, passes, groups, threads, rows=(), more=None, depth=3):
    """The first size at which every tiled launch of every pass has at least 3 tiles per channel group and tiles per
    item that do not divide its resident grid.  passes: [(call, names)], call(B, size) runs a batch of B items and
    makes the persistent launches `names`; `rows` names those among them that take one job per row (or per element
    block), which only need enough jobs.  more(size): the size with one more frame; when given, the size must leave
    every tiled launch a partial last tile (one more frame adds no tile).  threads: the smallest CTA of the launches.
    Returns (size, B) with B the batch that gives every launch tiles >= depth x grid."""
    caps = {}
    for size in sizes:
        per = []
        for k, (call, names) in enumerate(passes):
            _, reps = _launch(lambda: call(1, size), *names)
            assert all(t <= g for _, g, t in reps), reps
            if any(t < 3 * groups for nm, _, t in reps if nm not in rows):
                break
            if more is not None:
                _, grown = _launch(lambda: call(1, more(size)), *names)
                if any(a[2] != b[2] for a, b in zip(reps, grown) if a[0] not in rows):
                    break
            if any((k, nm) not in caps for nm, _, _ in reps):   # the resident grid depends on the kernel, not the size
                # (Kaldi's tiles are CTAs of 8 frame jobs, so a batch of n items has at least n (t - 1) of them)
                n = 2 * (_max_resident(threads) // min(t for _, _, t in reps) + 1)
                _, big = _launch(lambda: call(n, size), *names)
                for nm, g, t in big:
                    assert t > g, (nm, g, t)
                    caps.setdefault((k, nm), g)
            per += [(nm, t, caps[k, nm]) for nm, _, t in reps]
        else:
            if all(cap % t != 0 for nm, t, cap in per if nm not in rows):
                return size, max(math.ceil(depth * cap / t) if nm in rows else math.ceil(depth * cap / (t - 1)) + 1
                                 for nm, t, cap in per)
    raise AssertionError('no size gives tiles per item that do not divide the grid')


def _same(u, v):
    """Bit equality of tensors or tuples of them (None matches None), NaN equal to NaN."""
    if isinstance(u, (tuple, list)):
        return len(u) == len(v) and all(_same(a, b) for a, b in zip(u, v))
    if u is None or v is None:
        return u is v
    return u.shape == v.shape and (torch.equal(u, v) or bool(((u == v) | ((u != u) & (v != v))).all()))


def _items(y, i, n):
    return tuple(_items(t, i, n) for t in y) if isinstance(y, (tuple, list)) else None if y is None else y[i:i + n]


def _walk(run, xs, names, rows=(), view=True):
    """run(*xs) walked (every launch of `names` has tiles >= 3 grid; a tiled one, tiles per item that do not divide
    its grid) against the same items in launches of at most one tile per CTA, at storage offsets 1-3 and as a
    channels-last view.  xs: a tensor or a tuple of tensors whose first dimension is the batch.  Prints each launch's
    grid, tiles and tiles per item.  Returns the walked output."""
    xs = xs if isinstance(xs, tuple) else (xs,)
    _, one = _launch(lambda: run(*[x[:1] for x in xs]), *names)
    y, full = _launch(lambda: run(*xs), *names)
    assert [r[0] for r in one] == [r[0] for r in full], (one, full)
    chunk = None
    for (nm, g1, per_item), (_, grid, tiles) in zip(one, full):
        print('%s grid=%d tiles=%d per_item=%d' % (nm, grid, tiles, per_item))
        assert per_item <= g1 and tiles >= 3 * grid, (nm, grid, tiles, per_item)
        assert nm in rows or grid % per_item != 0, (nm, grid, per_item)
        chunk = min(chunk or grid, max(1, grid // per_item))
    for i in range(0, xs[0].shape[0], chunk):
        yi, reps = _launch(lambda: run(*[x[i:i + chunk] for x in xs]), *names)
        assert all(t <= g for _, g, t in reps), (i, reps)
        assert _same(yi, _items(y, i, chunk)), i
    for k in (1, 2, 3):
        assert _same(run(*[_placed(x, k) for x in xs]), y), k
    if view:
        assert _same(run(*[_channels_last_view(x) for x in xs]), y)
    return y


def _sample(B):
    return [0, B // 2, B - 1]


def _uniform(shape, seed):
    g = torch.Generator(device='cuda').manual_seed(seed)
    return torch.rand(shape, device='cuda', generator=g) * 2 - 1


def _zeros(B, C, L):
    return torch.zeros((B, C, L), device='cuda')


SIZES = [1000 * n + 37 for n in range(3, 80)]


@pytest.fixture(autouse=True)
def _under_2gb():
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    yield
    peak = torch.cuda.max_memory_allocated()
    print('peak device memory %.0f MiB' % (peak / 2 ** 20))
    assert peak < 2 * 2 ** 30, peak


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

    L, B = _pick(SIZES, [(lambda B, L: fwd(_zeros(B, 2, L), L), ['resample']),
                         (lambda B, L: bwd(_zeros(B, 2, RR.output_length(L, up, down)), L), ['resample'])], 2, 256)
    x = _uniform((B, 2, L), orig + target)
    y = _walk(lambda t: fwd(t, L), x, ['resample'])
    gy = _uniform(tuple(y.shape), orig + target + 1)
    gx = _walk(lambda t: bwd(t, L), gy, ['resample'])
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

    L, B = _pick(SIZES, [(lambda B, L: fwd(_zeros(B, 2, L), L), ['sinc']),
                         (lambda B, L: bwd(_zeros(B, 2, SR.output_length(L, ratio)), L), ['sinc'])], 2, 512)
    x = _uniform((B, 2, L), int(ratio * 1000))
    y = _walk(lambda t: fwd(t, L), x, ['sinc'])
    gy = _uniform(tuple(y.shape), int(ratio * 1000) + 1)
    gx = _walk(lambda t: bwd(t, L), gy, ['sinc'])
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

    L, B = _pick(SIZES, [(lambda B, L: fwd(_zeros(B, 2, L), L), ['spec_conv']),
                         (lambda B, L: bwd(_zeros(B, 2, full_len(L)), L), ['spec_conv'])], 2, 256)
    x = _uniform((B, 2, L), 7)
    y = _walk(lambda t: fwd(t, L), x, ['spec_conv'])
    start, n = ops.convolve_span(L, K, 'full')
    g = torch.zeros(y.shape, device='cuda')
    g[..., start:start + n] = torch.randn((B, 2, n), device='cuda', generator=torch.Generator(device='cuda').manual_seed(8))
    gx = _walk(lambda t: bwd(t, L), g, ['spec_conv'])
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

    T, B = _pick(list(range(20, 600, 7)), [(lambda B, T: fwd(torch.zeros((B, 2, T, K), device='cuda')), ['fbinv'])],
                 2, 256)
    m = torch.from_numpy(FR.consistent_input(fb, bank[1], bank[2], B, 2, T).astype(np.float32)).cuda()
    y = _walk(fwd, m, ['fbinv'])
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
                 [(lambda B, L: fwd(_zeros(B, 2, L)), ['kaldi_fwd']),
                  (lambda B, L: bwd(_zeros(B, 2, L), make_g(B, L)), ['kaldi_bwd'])], 1, 256)
    x = _x(B, 2, L, 5)
    y = _walk(fwd, x, ['kaldi_fwd'])
    gy = torch.randn(y.shape, device='cuda', generator=torch.Generator(device='cuda').manual_seed(1))
    gx = _walk(bwd, (x, gy), ['kaldi_bwd'])

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


# ------------------------------------------------------------------------------------------ constant-Q transform
@pytest.mark.parametrize('magnitude', [False, True])
def test_cqt_walks(magnitude):
    """The transform (one launch over the tiles of every octave) and its gradient (one launch per octave, lowest
    first, each with its own tiles of one (item, channel)'s level), against the float64 restatement within
    cqt_ref's bounds.  Every octave's backward launch walks, so the decimated top octave, which has the fewest tiles,
    sets the batch."""
    import cqt_ref as CQ
    from kapre_b200 import ops
    from test_gpu_cqt import _x
    plan = ops.CqtPlan(22050, 512, f_min=220.0, n_bins=36, bins_per_octave=12)

    def fwd(x):
        return ops.cqt_forward(x, plan, CF, CF, magnitude)[0]

    def bwd(g, x):
        ws = ops.cqt_forward(x, plan, CF, CF, True)[1] if magnitude else None
        return ops.cqt_backward(g, x, ws, plan, CF, CF, magnitude)

    def grad_of(B, L):
        return torch.zeros((B, 2, plan.num_frames(L), 36), device='cuda',
                           dtype=torch.float32 if magnitude else torch.complex64)

    L, B = _pick([2048 * n + 333 for n in range(2, 60)],
                 [(lambda B, L: fwd(_zeros(B, 2, L)), ['cqt_fwd']),
                  (lambda B, L: bwd(grad_of(B, L), _zeros(B, 2, L)), ['cqt_bwd'])], 2, 128)
    x = _x(B, 2, L, 11, 22050)
    y = _walk(fwd, x, ['cqt_fwd'])
    rng = np.random.default_rng(12)
    g = rng.standard_normal(tuple(y.shape)) + (0 if magnitude else 1j * rng.standard_normal(tuple(y.shape)))
    g = torch.from_numpy(g.astype(np.float32 if magnitude else np.complex64)).cuda()
    gx = _walk(bwd, (g, x), ['cqt_bwd'])
    for b in _sample(B):
        xb = x[b:b + 1].double().cpu()
        err = np.abs(y[b:b + 1].cpu().numpy().astype(np.float64 if magnitude else np.complex128)
                     - CQ.cqt(xb, plan, magnitude).numpy())
        assert (err <= CQ.forward_bound(xb, plan, magnitude).numpy()).all(), b
        gb = g[b:b + 1].cpu().to(torch.float64 if magnitude else torch.complex128)
        err = np.abs(gx[b:b + 1].cpu().numpy() - CQ.vjp(xb, plan, gb, magnitude).numpy())
        assert (err <= CQ.backward_bound(xb, plan, gb, magnitude).numpy()).all(), b


# ------------------------------------------------------------------------------------------ YIN / pYIN
def test_pitch_walks():
    """YIN's difference-function launch (tiles of frames of one (item, channel)) and pYIN's, followed by its Viterbi
    decoder (one CTA per row).  The CMNDF against the float64 restatement within pitch_ref's bound; the decisions,
    observation probabilities and Viterbi path against the float64 rules applied to the kernel's own CMNDF, as in
    test_gpu_pitch."""
    import pitch_ref as PR
    from kapre_b200 import ops
    from test_gpu_pitch import _plan, _x
    from test_pitch_emu import _decode_reference, _state_path
    sr = 16000
    kw = dict(sample_rate=sr, fmin=50.0, fmax=600.0, frame_length=1024)
    yplan, plan = _plan(**kw), _plan(pyin={}, **kw)
    hop = plan.geometry['hop_length']

    def yin(x):
        cm = torch.empty((x.shape[0], 2, plan.num_frames(x.shape[2]), plan.n_lags), device='cuda')
        return ops.yin(x, yplan, CF, cmndf=cm), cm

    def pyin(x):
        return ops.pyin(x, plan, CF)

    L, B = _pick([hop * n + 77 for n in range(4, 200)],
                 [(lambda B, L: yin(_zeros(B, 2, L)), ['pitch']), (lambda B, L: pyin(_zeros(B, 2, L)), ['pitch', 'viterbi'])],
                 2, 256, rows=('viterbi',), more=lambda L: L + hop)
    x = torch.from_numpy(_x(B, 2, L, sr, 13)).cuda()
    f0, cm = _walk(yin, x, ['pitch'])
    pf0, flag, vp = _walk(pyin, x, ['pitch', 'viterbi'], rows=('viterbi',))
    g, q, t = plan.geometry, plan.pyin, plan._tables
    n = q['n_pitch']
    A, band = PR.transition(q, t)
    init = np.log(np.concatenate([np.zeros(n), np.full(n, 1.0 / n)]) + PR.TINY)
    xs = x.cpu().numpy()
    for b in _sample(B):
        for c in range(2):
            cmh = cm[b, c].cpu().numpy().astype(np.float64)
            ref, bound = PR.cmndf_bound(xs[b, c], g)
            assert (np.abs(cmh - ref) <= bound).all(), (b, c)
            obs, vps = [], []
            for m in range(cmh.shape[0]):
                _, want = PR.yin_decide(cmh[m], g, 0.1, sr)
                np.testing.assert_allclose(float(f0[b, c, m]), want, rtol=1e-6)
                o, v, _ = PR.pyin_observe(cmh[m], g, q, t)
                obs.append(o)
                vps.append(v)
            np.testing.assert_allclose(vp[b, c].cpu().numpy(), vps, rtol=1e-4, atol=1e-6)
            lobs, la, _, best = _decode_reference(plan, obs, vp[b, c].cpu().numpy().astype(np.float64))
            sp = _state_path(plan, pf0[b, c].cpu().numpy(), flag[b, c].cpu().numpy())
            mask = np.full(lobs.shape, -np.inf)
            for m in range(lobs.shape[0]):
                if sp[m] >= 0:
                    mask[m, sp[m]] = 0.0
                else:
                    mask[m, n:] = 0.0
            kpath, _ = PR.viterbi(lobs + mask, A, band)
            assert PR.path_score(kpath, lobs, la, init) >= best - PR.path_bound(lobs.shape[0], lobs, la), (b, c)


# ------------------------------------------------------------------------------------------ chroma
def test_chroma_walks():
    """The projection of complex STFT frames (tiles of frames of one (item, channel)), its gradient, CENS (the
    projection, then a smoothing launch over tiles of 64 frames) and the tuning estimate (a peak launch over tiles of
    8 frames, five selection passes over tiles of 32 and one decision per item).  36 chroma give tiles of 85 frames.
    References as in test_gpu_chroma: chroma_ref's projection and CENS bounds, torch float64 autograd with the S
    path's tolerance, and the exact tuning estimate."""
    import chroma_ref as CR
    from kapre_b200 import _native as N
    from kapre_b200 import backend, ops
    from test_gpu_chroma import _torch_chroma
    sr, n_fft, NC = 22050, 256, 36
    K = n_fft // 2 + 1
    W = backend.chroma_filterbank(sr, n_fft, NC)
    plan = ops.ChromaPlan(W[None], smooth=backend.cens_window(41))
    cfg = N.ChromaCfg(N.CHROMA_IN_COMPLEX, N.CHROMA_NORM_L2, 0, 0.0)

    def fwd(x):
        return ops.chroma_forward(x, plan, cfg, CF)

    def bwd(g, x):
        return ops.chroma_backward(g, x, plan, cfg, CF)

    def cens(x):
        return ops.chroma_cens(x, plan, N.CHROMA_IN_COMPLEX, CF)

    def spec(B, M, seed=None):
        if seed is None:
            return torch.zeros((B, 2, M, K), dtype=torch.complex64, device='cuda')
        return torch.complex(_uniform((B, 2, M, K), seed), _uniform((B, 2, M, K), seed + 1))

    M, B = _pick([85 * n + 31 for n in range(3, 40)],
                 [(lambda B, M: fwd(spec(B, M)), ['chroma']),
                  (lambda B, M: bwd(torch.zeros((B, 2, M, NC), device='cuda'), spec(B, M)), ['chroma_bwd']),
                  (lambda B, M: cens(spec(B, M)), ['chroma', 'cens'])], 2, 256, more=lambda M: M + 1)
    x = spec(B, M, 14)
    y = _walk(fwd, x, ['chroma'])
    g = _uniform(tuple(y.shape), 16)
    gx = _walk(bwd, (g, x), ['chroma_bwd'])
    q = _walk(cens, x, ['chroma', 'cens'])
    Wt = torch.from_numpy(W).double()
    for b in _sample(B):
        s = x[b].abs().double().cpu().numpy()
        want, bound = CR.project(s, W, 2)
        bound = bound + CR.gamma(2) * want                      # the modulus, rounded once to float32
        assert (np.abs(y[b].double().cpu().numpy() - want) <= bound).all(), b
        # CENS quantises the device's own L1 chroma (threshold 0), as test_gpu_chroma does
        l1 = ops.chroma_forward(x[b:b + 1], plan, N.ChromaCfg(N.CHROMA_IN_COMPLEX, N.CHROMA_NORM_L1, 1, 0.0), CF)
        cw, cb = CR.cens_from_q(CR.quantize(l1[0].cpu().numpy()), backend.cens_window(41))
        assert (np.abs(q[b].double().cpu().numpy() - cw) <= cb).all(), b
        xd = x[b].cpu().to(torch.complex128).requires_grad_(True)
        (ref,) = torch.autograd.grad(_torch_chroma(xd.abs(), Wt, 2), xd, g[b].cpu().double())
        assert torch.allclose(gx[b].cpu().to(torch.complex128), ref, rtol=1e-4, atol=1e-4 * float(ref.abs().max()))

    # the tuning estimate, from a power spectrogram
    from kapre_b200 import signal
    _, tplan = signal._stft_chroma_plans(sr, n_fft, 64, None, 12, None, 5.0, 2.0, True)
    lo, hi = backend.piptrack_bins(sr, n_fft)

    def tuning(S):
        return ops.chroma_tuning(S, tplan, N.CHROMA_IN_LINEAR, CF)

    names = ['tune_peak', 'tune_select', 'tune_argmax']
    M, B = _pick([32 * n + 7 for n in range(1, 40)],
                 [(lambda B, M: tuning(torch.zeros((B, 2, M, K), device='cuda')), names)], 2, 256,
                 rows=('tune_argmax',), more=lambda M: M + 1)
    S = _uniform((B, 2, M, K), 17) ** 4
    tune, tab = _walk(tuning, S, names, rows=('tune_argmax',))
    for b in _sample(B):
        want, idx, _, _ = CR.estimate_tuning(S[b].cpu().numpy(), sr, n_fft, lo, hi, 0.01, 12)
        assert float(tune[b]) == want and int(tab[b]) == idx, (b, float(tune[b]), want)


# ------------------------------------------------------------------------------------------ harmonic/percussive
@pytest.mark.parametrize('cplx,mask', [(True, False), (False, True)])
def test_hpss_walks(cplx, mask):
    """The median-filter launch over tiles of 64 frames x 64 bins of one (item, channel), forward and backward (then
    an element-wise gather), complex input and mask mode.  Frames and bins both end in a partial tile, and each CTA
    walks about 16 tiles: with 3, a tile loop whose closing barrier is missing still gave the right bits.  The forward
    bit for bit against hpss_ref's float32 restatement over the device's own |S|; the gradient against torch
    float64 autograd through hpss_ref at the elements the device's tie rule selects, within test_gpu_hpss's bound."""
    import hpss_ref as HR
    from kapre_b200 import ops
    from test_gpu_hpss import _mag
    kh, kp, K = 17, 31, 100
    cfg = ops.hpss_config((kh, kp), 2.0, mask, (1.0, 1.5))
    dt = torch.complex64 if cplx else torch.float32

    def fwd(S):
        return ops.hpss_forward(S, cfg, CF)

    def bwd(gh, gp, S):
        return ops.hpss_backward(gh, gp, S, cfg, CF)

    def spec(B, T, seed=None):
        if seed is None:
            return torch.zeros((B, 2, T, K), dtype=dt, device='cuda')
        u = _uniform((B, 2, T, K), seed)
        return torch.complex(u, _uniform((B, 2, T, K), seed + 1)) if cplx else u.abs()

    gdt = torch.float32 if mask else dt
    T, B = _pick([64 * n + 23 for n in range(1, 40)],
                 [(lambda B, T: fwd(spec(B, T)), ['hpss']),
                  (lambda B, T: bwd(*[torch.zeros((B, 2, T, K), dtype=gdt, device='cuda')] * 2, spec(B, T)),
                   ['hpss_bwd', 'hpss_gather'])], 2, 128, rows=('hpss_gather',), depth=16)
    S = spec(B, T, 18)
    h, p = _walk(fwd, S, ['hpss'])
    pick = _sample(B)
    m = _mag(S[pick]).cpu().numpy()
    rh, rp = HR.hpss32(m, S[pick].cpu().numpy() if cplx else None, kh, kp, 2.0, (1.0, 1.5), mask)
    np.testing.assert_array_equal(h[pick].cpu().numpy(), rh)
    np.testing.assert_array_equal(p[pick].cpu().numpy(), rp)
    del h, p
    g = [_uniform((B, 2, T, K), 20 + i).to(gdt) for i in range(2)]
    gS = _walk(bwd, (g[0], g[1], S), ['hpss_bwd', 'hpss_gather'], rows=('hpss_gather',))
    sh, sp = HR.select(m, kh, kp)
    if cplx:
        leaf = S[pick].cpu().to(torch.complex128).requires_grad_(True)
        rh, rp = HR.hpss64(None, sh, sp, kh, kp, 2.0, (1.0, 1.5), mask, X=leaf)
    else:
        leaf = S[pick].cpu().double().requires_grad_(True)
        rh, rp = HR.hpss64(leaf, sh, sp, kh, kp, 2.0, (1.0, 1.5), mask)
    rdt = torch.complex128 if (cplx and not mask) else torch.float64
    (ref,) = torch.autograd.grad((rh, rp), leaf, (g[0][pick].cpu().to(rdt), g[1][pick].cpu().to(rdt)))
    ok = torch.isfinite(ref.abs())
    err = ((gS[pick].cpu().to(ref.dtype) - ref).abs() / (1 + ref.abs()))[ok]
    assert float(err.max()) < 2e-4 * 2 * (kh + kp)


# ------------------------------------------------------------------------------------------ onsets, tempo, beats
def test_rhythm_walks():
    """Onset strength (tiles of frames of one (item, channel)) and its gradient (then an element-wise gather), the
    tempogram (tiles of frames), tempo (partial sums over 64-frame chunks, then one decision per row), peak picking
    and the beat tracker (one CTA per row).  References as in test_gpu_rhythm: rhythm_ref's envelope within 1 ulp
    (the median exact), its gradient through torch float64 autograd, the tempogram within (W + 4) 2^-24, and the
    float64 tempo, peak and beat rules applied to the kernel's own tempogram or envelope where rounding cannot decide
    them."""
    import rhythm_ref as RH
    from kapre_b200 import ops
    from test_rhythm_emu import MARGIN
    sr, hop, K, W = 22050, 512, 40, 96

    # onset strength, mean and median, forward and backward
    for agg in ('mean', 'median'):
        cfg = ops.onset_config(2, 3, agg, 2)

        def fwd(S):
            return ops.onset_strength_forward(S, cfg, CF)

        def bwd(g, S):
            return ops.onset_strength_backward(g, S, cfg, CF)

        T, B = _pick([16 * n + 5 for n in range(4, 80)],
                     [(lambda B, T: fwd(torch.zeros((B, 2, T, K), device='cuda')), ['onset']),
                      (lambda B, T: bwd(torch.zeros((B, 2, T), device='cuda'), torch.zeros((B, 2, T, K), device='cuda')),
                       ['onset_bwd', 'onset_gather'])], 2, 128, rows=('onset_gather',), more=lambda T: T + 1)
        S = torch.randn((B, 2, T, K), device='cuda', generator=torch.Generator(device='cuda').manual_seed(21))
        e = _walk(fwd, S, ['onset'])
        g = _uniform((B, 2, T), 22)
        gS = _walk(bwd, (g, S), ['onset_bwd', 'onset_gather'], rows=('onset_gather',))
        for b in _sample(B):
            for c in range(2):
                ref = RH.onset_strength_row(S[b, c].cpu().numpy(), 2, 3, agg, 2)
                d = np.abs(e[b, c].cpu().numpy().view(np.int32).astype(np.int64) - ref.view(np.int32).astype(np.int64))
                assert d.max() <= (0 if agg == 'median' else 1), (agg, b, c)
                St = S[b, c].cpu().double().requires_grad_()
                RH.onset_strength_torch(St, 2, 3, agg, 2).backward(g[b, c].cpu().double())
                np.testing.assert_allclose(gS[b, c].cpu().numpy(), St.grad.numpy(), rtol=1e-5, atol=1e-6)

    # the tempogram of an envelope
    def tempogram(e):
        return ops.tempogram(e, W, True, True, CF)

    T, B = _pick([16 * n + 3 for n in range(2, 80)], [(lambda B, T: tempogram(_zeros(B, 2, T)), ['tempogram'])], 2,
                 128, more=lambda T: T + 1)
    env = _uniform((B, 2, T), 23).abs()
    tg = _walk(tempogram, env, ['tempogram'])
    for b in _sample(B):
        for c in range(2):
            ref = RH.tempogram_row(env[b, c].cpu().numpy(), W)
            assert np.abs(tg[b, c].cpu().numpy() - ref).max() <= (W + 4) * 2.0 ** -24 + 1e-12, (b, c)

    # tempo from a tempogram
    plan = ops.TempoPlan(W, sr, hop)
    bpm, lp = RH.tempo_prior(W, sr, hop)

    def tempo(t):
        return ops.tempo(t, plan, False, CF)

    names = ['tempo_part', 'tempo']
    T, B = _pick([64 * n + 9 for n in range(2, 40)],
                 [(lambda B, T: tempo(torch.zeros((B, 2, T, W), device='cuda')), names)], 2, 128, rows=('tempo',),
                 more=lambda T: T + 1)
    tgs = ops.tempogram(_uniform((B, 2, T), 24).abs(), W, True, True, CF)
    bpms = _walk(tempo, tgs, names, rows=('tempo',))
    checked = 0
    for b in _sample(B):
        for c in range(2):
            t = tgs[b, c].cpu().numpy()
            sc = np.sort(RH.tempo_scores(t.astype(np.float64).mean(axis=0), lp))
            if sc[-1] - sc[-2] > 1e-6 * abs(sc[-1]):                # decided beyond rounding
                assert float(bpms[b, c]) == np.float32(RH.tempo_row(t, lp, bpm)), (b, c)
                checked += 1
    assert checked >= 3

    # peak picking and beat tracking of an envelope with a beat every 22 frames
    dcfg = ops.onset_detect_config(3, 2, 5, 6, 2, 0.07, True)
    bcfg = ops.beat_config(sr, hop, 100.0, True)

    def detect(e):
        return ops.onset_detect(e, dcfg, CF)

    def beats(e):
        return ops.beat_track(e, bcfg, 120.0, CF)

    T = 431
    _, B = _pick([T], [(lambda B, T: detect(_zeros(B, 2, T)), ['onset_detect']),
                       (lambda B, T: beats(_zeros(B, 2, T)), ['beat_track'])], 2, 128,
                 rows=('onset_detect', 'beat_track'))
    env = _uniform((B, 2, T), 25).abs()
    env[:, :, ::22] += 3.0
    mask = _walk(detect, env, ['onset_detect'], rows=('onset_detect',))
    tempo_b, beat = _walk(beats, env, ['beat_track'], rows=('beat_track',))
    checked = 0
    for b in _sample(B):
        for c in range(2):
            e = env[b, c].cpu().numpy()
            ref, margin = RH.peak_pick_row(e, 3, 2, 5, 6, 2, 0.07, True, return_scores=True)
            if np.abs(margin).min() > MARGIN:                      # no candidate decided by rounding
                np.testing.assert_array_equal(mask[b, c].cpu().numpy(), ref)
                checked += 1
            if RH.beat_margin(e, float(tempo_b[b, c]), sr, hop) > 1e-9:
                _, ref = RH.beat_track_row(e, float(tempo_b[b, c]), sr, hop)
                np.testing.assert_array_equal(np.nonzero(beat[b, c].cpu().numpy())[0], ref)
                checked += 1
    assert checked >= 6
