"""GPU tier: the backward passes at every launch shape and input placement, and the fused stack's clamp decisions
against its forward.

The backward passes run the transform launchers with other constant tables (kapre_b200.cu, "backward passes"), so the
launch shape follows the batch exactly as in the forward, and a small test batch only reaches the shapes it picks.
These tests force every feasible shape through the launcher's switches and read back the launch it made
(``last_launch_info``: the adjoints' elementwise passes do not overwrite it).

* ISTFT^T is the forward launch with the window dual 2/N: every single-channel tile, all-channel tile and
  mixed-radix warp budget must give the bits of the default launch, as the forward does
  (test_gpu_launch_invariance.py), including gradients whose items start at odd sample offsets, where a cosine-sum
  adjoint window is read from its table instead of being formed in registers.  Views must give the bits of a
  contiguous copy, and an item the bits it has alone.  The all-channel kernel's pair step differs from the
  single-channel kernel's by design, so switching between the two is held to the oracle only.  There is no 16-warp
  shape here: that CTA is instantiated for the filterbank modes only.
* STFT^T is the inverse launch with the dual window w N/2 and the edge/crop pass.  The inverse kernels sum
  overlapping frames in an order that follows their tile length (the ``predict`` docstring names ``InverseSTFT`` as
  the exception to bit-identity under chunking), so every shape is held to the float64 product, and samples that no
  frame covers must be exactly 0.  A strided gradient (the half-channel views ``_MagPhase`` passes) must give the bits
  of a contiguous copy.
* The fused stack's backward recomputes the pre-decibel values with a second launch and re-derives the clamp mask and
  the item maximum from them.  With a binding dynamic range, the elements whose gradient vanishes must be exactly the
  ones the forward clamped, and the threshold's gradient must land on the forward's maxima.

Tolerances, relative to the largest reference value:
* 1e-4 for the linear adjoints against the float64 vector-Jacobian product (grad_ref.py), as in test_gpu_grad.py: the
  kernels transform in float32 (about 6e-8 relative rounding per operation, O(log N) operations per output) and an
  output sums at most ceil(win / hop) frames;
* 1e-5 per element for the decibel backward away from the threshold (one division and one product per element), and
  1e-4 at the maxima, which add the clamped elements' gradients with float32 atomics (at most 64 x 8 warp partial sums
  of positive terms per item, each rounded once, in an order that varies from run to run);
* none elsewhere: bit-identity, exact zeros and exact masks.
"""
import ctypes
import re

import numpy as np
import pytest

torch = pytest.importorskip('torch')

import grad_ref as R  # noqa: E402
from oracle import reference as ref  # noqa: E402

pytestmark = pytest.mark.gpu

CF, CL = 'channels_first', 'channels_last'
SWITCHES = ['KAPRE_B200_TF', 'KAPRE_B200_NW', 'KAPRE_B200_MC_TF', 'KAPRE_B200_MC_NW', 'KAPRE_B200_NOBULK',
            'KAPRE_B200_NOMC', 'KAPRE_B200_PDL_FWD', 'KAPRE_B200_MR_WARPS', 'KAPRE_B200_ISTFT2_M', 'KAPRE_B200_ISTFT2',
            'KAPRE_B200_INW']
DSCALE = np.float32(10.0 / np.log(10.0))


@pytest.fixture(scope='module')
def K():
    assert torch.cuda.is_available(), 'GPU tier needs a CUDA device'
    import kapre_b200
    from kapre_b200 import _native
    _native.lib()
    return kapre_b200


@pytest.fixture
def env(monkeypatch):
    """Sets launcher switches for one call at a time; none leaks into the next test."""
    for k in SWITCHES:
        monkeypatch.delenv(k, raising=False)

    def set_env(**kw):
        for k in SWITCHES:
            monkeypatch.delenv(k, raising=False)
        for k, v in kw.items():
            monkeypatch.setenv('KAPRE_B200_' + k, str(v))
    return set_env


def bits(t):
    t = t.contiguous()
    if t.is_complex():
        t = torch.view_as_real(t)
    return t.view(torch.int32)


def eq(a, b):
    return a.shape == b.shape and a.dtype == b.dtype and bool(torch.equal(bits(a), bits(b)))


def rel(got, want, tol):
    got = got.detach().cpu().to(want.dtype)
    err = float((got - want).abs().max())
    scale = float(want.abs().max())
    assert err <= tol * scale, (err, scale)


def info():
    from kapre_b200 import _native
    return _native.last_launch_info()


def launched(pattern):
    m = re.search(pattern, info())
    assert m, (pattern, info())
    return m


def try_launch(fn, *a):
    from kapre_b200 import _native
    try:
        return fn(*a)
    except _native.KapreNativeError as e:
        if 'no launch configuration fits' in str(e):
            return None
        raise


def log_shapes(capsys, what, seen):
    with capsys.disabled():
        print('\n%s: %d shapes: %s' % (what, len(seen), ' | '.join(sorted(seen))))


# ------------------------------------------------------------------------------------------------ ISTFT^T
def istft_setup(K, n_fft, win, hop, wname):
    from kapre_b200 import ops
    dual = ref.inverse_stft_window(win, hop, ref.get_window(wname, win)).astype(np.float32)
    plan = ops.IstftPlan(n_fft, win, hop, dual)

    def bwd(gy, frames, spec_fmt=CF, wave_fmt=CF):
        return ops.istft_backward(gy, plan, spec_fmt, wave_fmt, frames)

    def want(gy, frames, spec_fmt=CF, wave_fmt=CF):
        B = gy.shape[0]
        C = gy.shape[2] if wave_fmt == CL else gy.shape[1]
        F = n_fft // 2 + 1
        X = torch.zeros((B, frames, F, C) if spec_fmt == CL else (B, C, frames, F), dtype=torch.complex128)
        return R.vjp(lambda t: R.istft(t, n_fft, win, hop, wname, spec_fmt, wave_fmt), X, gy.cpu().double())[1]
    return bwd, want


def k1_candidates(n_fft):
    """(NW, TF) of the single-channel kernel in the complex mode: FR = NW * 32 / Q frames per round <= 32, TF a
    power of two and a multiple of FR (kb_pick_fwd_cfg)."""
    fpw = 32 // (n_fft // 64)
    return [(nw, tf) for nw in (1, 2, 4, 8) if nw * fpw <= 32 for tf in (32, 16, 8, 4, 2, 1) if tf % (nw * fpw) == 0]


@pytest.mark.parametrize('wname', ['hann_window', 'hamming_window'])
@pytest.mark.parametrize('n_fft,hop', [(256, 64), (512, 128), (1024, 256), (2048, 512)])
def test_istft_adjoint_every_single_channel_shape(K, env, capsys, n_fft, hop, wname):
    bwd, want = istft_setup(K, n_fft, n_fft, hop, wname)
    T = 41
    out_len = (T - 1) * hop + n_fft
    g = torch.Generator(device='cuda').manual_seed(n_fft + len(wname))
    big = torch.randn((4, 1, out_len + 1), generator=g, device='cuda')
    seen = set()
    env()
    ref_even = bwd(big[:, :, :out_len].contiguous(), T)
    rel(ref_even, want(big[:, :, :out_len], T), 1e-4)
    # odd item stride: items 1 and 3 start at odd sample offsets
    for name, gy in (('even', big[:, :, :out_len].contiguous()), ('odd', big[:, :, :out_len])):
        env()
        y = bwd(gy, T)
        seen.add(launched(r'Q\d+ TF\d+ NW\d+ bulk1 ').group(0))
        assert eq(y, ref_even), name
        env(NOBULK=1)
        assert eq(bwd(gy, T), ref_even), name
        launched(r' bulk0 ')
        env(PDL_FWD=0)
        assert eq(bwd(gy, T), ref_even), name
        env()
        for b in range(4):
            assert eq(bwd(gy[b:b + 1].clone(), T), ref_even[b:b + 1]), (name, b)
        ran = 0
        for nw, tf in k1_candidates(n_fft):
            env(NW=nw, TF=tf)
            y = try_launch(bwd, gy, T)
            if y is None:
                continue
            seen.add(launched(r'Q\d+ TF%d NW%d bulk\d ' % (tf, nw)).group(0))
            assert eq(y, ref_even), (name, nw, tf, info())
            ran += 1
        assert ran >= 6, (name, ran)
    log_shapes(capsys, 'ISTFT^T n_fft %d %s' % (n_fft, wname), seen)


@pytest.mark.parametrize('n_fft,hop', [(256, 64), (512, 128), (1024, 256), (2048, 512)])
def test_istft_adjoint_shapes_that_walk_several_tiles(K, env, capsys, n_fft, hop):
    bwd, want = istft_setup(K, n_fft, n_fft, hop, 'hann_window')
    T = 600
    g = torch.Generator(device='cuda').manual_seed(n_fft)
    gy = torch.randn((64, 1, (T - 1) * hop + n_fft), generator=g, device='cuda')
    env()
    ref0 = bwd(gy, T)
    for b in (0, 63):
        rel(ref0[b:b + 1], want(gy[b:b + 1], T), 1e-4)
    walked, seen = 0, set()
    for nw, tf in k1_candidates(n_fft):
        env(NW=nw, TF=tf)
        y = try_launch(bwd, gy, T)
        if y is None:
            continue
        m = launched(r'TF%d NW%d bulk1 grid(\d+) .* tiles(\d+)' % (tf, nw))
        seen.add(m.group(0))
        walked += int(m.group(2)) >= 2 * int(m.group(1))
        assert eq(y, ref0), (nw, tf, info())
    assert walked >= 1
    log_shapes(capsys, 'ISTFT^T multi-tile n_fft %d' % n_fft, seen)


@pytest.mark.parametrize('C', [2, 3, 7, 16, 31, 32, 33])
def test_istft_adjoint_all_channel_shapes(K, env, capsys, C):
    n_fft, hop = (512, 128) if C % 2 else (1024, 256)
    bwd, want = istft_setup(K, n_fft, n_fft, hop, 'hann_window')
    T = 23
    spec_fmt = CF if C % 2 else CL
    g = torch.Generator(device='cuda').manual_seed(C)
    gy = torch.randn((3, (T - 1) * hop + n_fft, C), generator=g, device='cuda')   # interleaved channels
    env()
    ref0 = bwd(gy, T, spec_fmt, CL)
    launched(r'^MC Q' if C <= 32 else r'^Q\d+ TF')
    seen = {info()}
    rel(ref0, want(gy, T, spec_fmt, CL), 1e-4)
    for b in range(3):
        assert eq(bwd(gy[b:b + 1].clone(), T, spec_fmt, CL), ref0[b:b + 1]), b
    if C > 32:
        return
    ran = 0
    for nw in (1, 2, 4, 8):
        for tf in (1, 2, 3, 5, 8, 16):
            env(MC_NW=nw, MC_TF=tf)
            y = bwd(gy, T, spec_fmt, CL)
            if not info().startswith('MC ') or ' TF%d NW%d ' % (tf, nw) not in info():
                continue          # the shape does not fit: single-channel tiles ran instead
            seen.add(info())
            assert eq(y, ref0), (nw, tf, info())
            ran += 1
    assert ran >= 3
    env(NOMC=1)
    y = bwd(gy, T, spec_fmt, CL)
    assert not info().startswith('MC ')
    rel(y, want(gy, T, spec_fmt, CL), 1e-4)     # the two kernels' pair steps differ: the oracle only
    log_shapes(capsys, 'ISTFT^T C=%d' % C, seen)


@pytest.mark.parametrize('n_fft', [400, 98])
def test_istft_adjoint_mixed_radix_and_direct_dft(K, env, capsys, n_fft):
    hop = n_fft // 4
    bwd, want = istft_setup(K, n_fft, n_fft, hop, 'hamming_window')
    T = 30
    out_len = (T - 1) * hop + n_fft
    g = torch.Generator(device='cuda').manual_seed(n_fft)
    big = torch.randn((4, 1, out_len + 1), generator=g, device='cuda')
    env()
    ref0 = bwd(big[:, :, :out_len].contiguous(), T)
    launched(r'^DFT' if n_fft == 98 else r'^MR ')
    seen = {info()}
    rel(ref0, want(big[:, :, :out_len], T), 1e-4)
    assert eq(bwd(big[:, :, :out_len], T), ref0)                       # odd item stride
    for b in range(4):
        assert eq(bwd(big[b:b + 1, :, :out_len].clone(), T), ref0[b:b + 1]), b
    if n_fft != 98:
        # more tiles than resident CTAs: the warp budget changes the grid and the tiles each CTA walks
        xb = torch.randn((256, 1, 199 * hop + n_fft), generator=g, device='cuda')
        env()
        refb = bwd(xb, 200)
        grids = set()
        for w in (8, 16, 24, 32, 48, 64):
            env(MR_WARPS=w)
            y = bwd(xb, 200)
            grids.add(re.search(r'NW\d+ G\d+ grid\d+', info()).group(0))
            seen.add(info())
            assert eq(y, refb), (w, info())
        assert len(grids) >= 2, grids
    log_shapes(capsys, 'ISTFT^T n_fft %d' % n_fft, seen)


def test_istft_adjoint_views_give_the_bits_of_a_contiguous_copy(K, env):
    n_fft, hop, T = 1024, 256, 21
    out_len = (T - 1) * hop + n_fft
    bwd, _ = istft_setup(K, n_fft, n_fft, hop, 'hann_window')
    env()
    g = torch.Generator(device='cuda').manual_seed(7)
    base = torch.randn((5, 3, out_len + 3), generator=g, device='cuda')
    base_cl = torch.randn((4, out_len, 3), generator=g, device='cuda')
    mono_odd = base[:, :1, :out_len + 1].contiguous()[:, :, :out_len]
    views = [('offset_item', mono_odd[1:], CF), ('narrow1', base[:, :, 1:1 + out_len], CF),
             ('narrow2', base[:, :, 2:2 + out_len], CF), ('narrow3', base[:, :, 3:3 + out_len], CF),
             ('channel', base[:, 1:2, :out_len], CF), ('channel_cl', base_cl[:, :, 1:2], CL),
             ('expand', base[:1, :, :out_len].expand(4, -1, -1), CF)]
    for name, v, fmt in views:
        assert eq(bwd(v, T, CF, fmt), bwd(v.contiguous(), T, CF, fmt)), name
    # an item's gradient does not depend on its place in the batch
    whole = bwd(mono_odd, T)
    for b in range(5):
        assert eq(bwd(mono_odd[b:b + 1].contiguous(), T), whole[b:b + 1]), b


# ------------------------------------------------------------------------------------------------- STFT^T
STFT_BWD_CASES = [(512, 512, 128), (1024, 1024, 256), (2048, 2048, 512), (512, 384, 128), (256, 200, 240)]
PADS = [(False, False), (True, False), (False, True), (True, True)]


@pytest.mark.parametrize('pads', PADS, ids=lambda p: 'pb%d_pe%d' % p)
@pytest.mark.parametrize('case', STFT_BWD_CASES, ids=lambda c: 'n%d_w%d_h%d' % c)
def test_stft_adjoint_every_inverse_shape(K, env, capsys, case, pads):
    from kapre_b200 import _native, ops
    n_fft, win, hop = case
    pb, pe = pads
    win_eff = min(win, n_fft)
    plan = ops.StftPlan(n_fft, win, hop, ref.get_window(None, win).astype(np.float32))
    B, C = 3, 2
    L = 40 * hop + 13
    T = plan.num_frames(L, pb, pe)
    pad_left = n_fft - hop if pb else 0
    g = torch.Generator(device='cuda').manual_seed(n_fft + hop + 2 * pb + pe)
    G = torch.complex(torch.randn((B, C, T, n_fft // 2 + 1), generator=g, device='cuda'),
                      torch.randn((B, C, T, n_fft // 2 + 1), generator=g, device='cuda'))
    _, want = R.vjp(lambda t: R.stft(t, n_fft, win, hop, None, pb, pe, CF, CF),
                    torch.zeros((B, C, L), dtype=torch.float64), G.cpu().to(torch.complex128))
    # the overlap-add is written straight into gx without a pad in front and with no sample past the signal's end
    nbytes = int(_native.lib().kapre_stft_backward_workspace_bytes(plan.handle(), B, C, L, int(pb), int(pe)))
    direct = not pb and (T - 1) * hop + win <= L
    assert (nbytes == 0) == direct and direct == (pads == (False, False)), (nbytes, direct)
    u = np.arange(L) + pad_left
    covered = np.zeros(L, bool)
    for t in range(T):
        covered |= (u >= t * hop) & (u < t * hop + win_eff)
    uncovered = torch.from_numpy(~covered).cuda()
    if hop > win_eff or not pe:
        assert uncovered.any()

    def bwd(gg, fmt=CF):
        return ops.stft_backward(gg, plan, CF, fmt, pb, pe, L)

    def check(gx):
        rel(gx, want, 1e-4)
        assert not bool(gx[:, :, uncovered].any())

    ran, seen = 0, set()
    for m in range(1, 9):
        env(ISTFT2_M=m)
        gx = bwd(G)
        if ' rounds%d ' % m not in info():
            continue
        seen.add(info())
        check(gx)
        ran += 1
    assert ran >= 4, ran
    for nw in (4, 2, 1):
        env()
        ops.stft_forward(torch.zeros((1, 1, 4 * n_fft), device='cuda'), plan, CF, CF, False, False)
        env(ISTFT2=0, INW=nw)
        check(bwd(G))
        assert not info().startswith('ISTFT2')         # the class-ordered body ran (it leaves the info as it was)
    # strided gradients: the channel halves of a 2C-channel tensor, as _MagPhase passes them
    env()
    G2 = torch.cat([G, G.flip(1)], dim=1)
    for v, fmt in ((G2[:, :C], CF), (G2[:, C:], CF), (G2.permute(0, 2, 3, 1)[..., C:], CL)):
        assert eq(bwd(v, fmt), bwd(v.contiguous(), fmt))
    log_shapes(capsys, 'STFT^T n_fft %d win %d hop %d pads %s ws %d' % (n_fft, win, hop, pads, nbytes), seen)


# -------------------------------------------------------------------------------- decibel backward chunks
@pytest.mark.parametrize('item', [3000, 9000, 131072, 200000])     # 2, 5, 64 and (capped) 64 CTAs per item
def test_decibel_backward_across_chunks(K, item):
    from kapre_b200 import _native
    dyn, amin = 20.0, 1e-5
    rng = np.random.default_rng(item)
    n = 3
    x = (rng.random((n, item)) ** 4).astype(np.float32)
    x[0, [5, 256 * 3 + 7, item - 1]] = 2.0      # tied maxima; element i is walked by CTA (i // 256) % chunks
    x[2, :100] = 0.0                            # below amin
    for it in range(n):                         # nothing within rounding of the threshold
        d = 10.0 * np.log10(np.maximum(x[it].astype(np.float64), amin))
        near = np.abs(d - (d.max() - dyn)) < 1e-3
        x[it, near] *= np.float32(1.01)
    g = (rng.random((n, item)) + 0.5).astype(np.float32)

    def run(xh, gh):
        xt, gt = torch.from_numpy(xh).cuda(), torch.from_numpy(gh).cuda()
        gx = torch.empty_like(xt)
        ws = torch.zeros(3 * xh.shape[0], dtype=torch.int32, device='cuda')
        dbc = _native.DbCfg(1.0, amin, dyn)
        _native.check(_native.lib().kapre_magnitude_to_decibel_backward(
            ctypes.c_void_p(xt.data_ptr()), ctypes.c_void_p(gt.data_ptr()), ctypes.c_void_p(gx.data_ptr()),
            xh.shape[0], item, ctypes.byref(dbc), ctypes.c_void_p(ws.data_ptr()),
            ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))
        torch.cuda.synchronize()
        assert int(ws.abs().sum()) == 0
        return gx.cpu()

    gx = run(x, g)
    for it in range(n):
        want = R.vjp(lambda t: R.magnitude_to_decibel(t, 1.0, amin, dyn), torch.from_numpy(x[it:it + 1]).double(),
                     torch.from_numpy(g[it:it + 1]).double())[1][0]
        is_max = torch.from_numpy(x[it] == x[it].max())
        err = (gx[it].double() - want).abs()
        assert int(is_max.sum()) == (3 if it == 0 else 1)
        assert bool((err[~is_max] <= 1e-5 * want.abs()[~is_max]).all()), it
        assert bool((err[is_max] <= 1e-4 * want.abs()[is_max]).all()), it
        assert bool(((gx[it] == 0) == (want == 0)).all()), it
    # a NaN item beside finite ones: the finite items keep their gradients.  The maxima's share of the threshold's
    # gradient is summed with float32 atomics, whose order varies from run to run, so there only the tolerance holds.
    xn = np.concatenate([x[:1], x[1:2].copy(), x[2:]])
    xn[1, 1234] = np.nan
    gxn = run(xn, g)
    for it in (0, 2):
        is_max = torch.from_numpy(x[it] == x[it].max())
        assert torch.equal(gxn[it][~is_max].view(torch.int32), gx[it][~is_max].view(torch.int32)), it
        assert bool(((gxn[it] - gx[it]).abs()[is_max] <= 1e-4 * gx[it].abs()[is_max]).all()), it
    assert bool(torch.isfinite(gxn[1][torch.from_numpy(np.isfinite(xn[1]))]).all())


# ----------------------------------------------------------------------- fused stack: clamp against forward
STACK_SHAPES = {'single': (1024, 256, CF, 1), 'all_channel': (512, 128, CL, 2), 'mixed_radix': (400, 160, CF, 1)}


def _stack(K, kind, shape, dyn):
    n_fft, hop, fmt, _ = STACK_SHAPES[shape]
    kw = dict(n_fft=n_fft, hop_length=hop, input_data_format=fmt, output_data_format=fmt, return_decibel=True,
              db_dynamic_range=dyn)
    if kind == 'stftmag':
        return K.get_stft_magnitude_layer(**kw)
    if kind == 'mel':
        return K.get_melspectrogram_layer(sample_rate=16000, n_mels=64, **kw)
    if kind == 'log':
        return K.get_log_frequency_spectrogram_layer(sample_rate=16000, **kw)
    return K.get_stft_mag_phase(None, **kw)


@pytest.mark.parametrize('dyn', [15.0, 40.0])
@pytest.mark.parametrize('kind', ['stftmag', 'mel', 'log', 'mag_phase'])
@pytest.mark.parametrize('shape', list(STACK_SHAPES))
def test_fused_stack_clamps_what_the_forward_clamped(K, env, monkeypatch, capsys, shape, kind, dyn):
    """g = ones: the backward's dL/d(pre) vanishes exactly where the forward clamped (or where pre < amin), and the
    threshold's gradient lands on the elements whose forward dB is the item maximum."""
    from kapre_b200 import ops
    if kind == 'mag_phase' and shape == 'mixed_radix':
        pytest.skip('no fused magnitude + phase launch at a mixed-radix size')
    env()
    n_fft, hop, fmt, C = STACK_SHAPES[shape]
    g = torch.Generator(device='cuda').manual_seed(int(dyn) + len(kind))
    L = 8000
    x = torch.randn((3, L, C) if fmt == CL else (3, C, L), generator=g, device='cuda')
    sl = (slice(None), slice(2000, 3500)) if fmt == CL else (slice(None), slice(None), slice(2000, 3500))
    x *= 100.0                                    # the item maximum well above amin: the threshold can bind
    x[sl] *= 1e-6                                 # a quiet stretch: 60 dB (10 log10 of magnitudes) below the rest
    model, unclamped = _stack(K, kind, shape, dyn), _stack(K, kind, shape, 1e9)
    D = unclamped(x)
    seen = info()
    y = model(x)
    calls = []
    orig = ops.magnitude_to_decibel_backward

    def spy(pre, gg, *db):
        out = orig(pre, gg, *db)
        calls.append((pre.detach(), out))
        return out
    monkeypatch.setattr(ops, 'magnitude_to_decibel_backward', spy)
    xg = x.clone().requires_grad_(True)
    yg = model(xg)
    assert torch.equal(yg.detach(), y)
    torch.autograd.grad(yg, xg, grad_outputs=torch.ones_like(yg))
    assert len(calls) == 1
    pre, gpre = calls[0]
    if kind == 'mag_phase':                       # the magnitude half of the 2C-channel outputs
        y, D = (y[..., :C], D[..., :C]) if fmt == CL else (y[:, :C], D[:, :C])
    # the recomputed pre-decibel values give the forward's decibel bits
    assert eq(ops.magnitude_to_decibel(pre, 1.0, 1e-5, 1e9), D)
    for b in range(3):
        yb, Db, pb, gb = y[b].flatten(), D[b].flatten(), pre[b].flatten(), gpre[b].flatten()
        thr = yb.min()
        clamped = Db < thr
        assert bool(clamped.any()), 'the dynamic range must bind'
        assert eq(yb, torch.maximum(Db, thr))
        is_max = Db == Db.max()
        zero = clamped | (pb < 1e-5)
        assert bool(((gb == 0) == zero)[~is_max].all()), (b, int(((gb == 0) != zero).sum()))
        receivers = gb > 1.5 * (torch.tensor(DSCALE, device='cuda') / pb)
        assert bool(receivers.any()) and not bool((receivers & ~is_max).any()), b
    log_shapes(capsys, 'fused %s %s %g dB' % (shape, kind, dyn), {seen})
