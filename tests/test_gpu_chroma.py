"""Chroma on the H100: chroma_stft, chroma_cqt and chroma_cens at benchmark size in both layouts within the float64
bound (chroma_ref.py) over the device's own magnitudes, the tuning estimate against the reference on the device's
own S with tonal anchors, chroma_stft(tuning=None) against the per-item fixed-tuning result bit for bit, bit equality
across batch positions, layouts and strides, launch counts, CUDA graph replay, gradients against torch.autograd,
no-grad behaviour, non-finite isolation and the ptxas budgets of the new kernels."""
import os
import re
import subprocess

import numpy as np
import pytest
import torch

import chroma_ref as R

pytestmark = pytest.mark.gpu

CL, CF = 'channels_last', 'channels_first'
SR = 22050


def _x(B, C, L, seed):
    """Chords of three random notes with random detuning, plus a little noise: (B, C, L) float32."""
    rng = np.random.default_rng(seed)
    t = np.arange(L) / SR
    x = 0.01 * rng.standard_normal((B, C, L))
    for b in range(B):
        for midi in rng.choice(np.arange(45, 85), 3, replace=False):
            f = 440.0 * 2.0 ** ((midi - 69 + rng.uniform(-0.4, 0.4)) / 12.0)
            x[b] += rng.uniform(0.2, 0.6) * np.sin(2 * np.pi * f * t + rng.uniform(0, 6))[None]
    return x.astype(np.float32)


def _tone(f, L, amp=0.5):
    return (amp * np.sin(2 * np.pi * f * np.arange(L) / SR)).astype(np.float32)


def _cf(t, fmt):
    """A (B, M, K, C) / (B, C, M, K) tensor as (B, C, M, K)."""
    return t.permute(0, 3, 1, 2) if fmt == CL else t


def _same(u, v):
    return torch.equal(u, v) or bool(((u == v) | ((u != u) & (v != v))).all())


def _mag(x, fmt):
    """The library's centred |STFT| at chroma_stft's defaults, in ``fmt``."""
    from kapre_b200 import signal
    stft, _ = signal._stft_chroma_plans(SR, 2048, 512, None, 12, 0.0, 5.0, 2.0, True)
    return signal._centred_magnitude(x, stft, fmt, True)


def _wave(x, fmt):
    t = torch.from_numpy(x).cuda()
    return t.transpose(1, 2).contiguous() if fmt == CL else t


@pytest.mark.parametrize('fmt', [CL, CF])
def test_chroma_stft_benchmark_size_within_bound(fmt):
    from kapre_b200 import backend, signal
    x = _x(256, 1, 5 * SR, 0)
    xin = _wave(x, fmt)
    out = signal.chroma_stft(xin, tuning=0.0, data_format=fmt)
    assert out.shape == ((256, 216, 12, 1) if fmt == CL else (256, 1, 216, 12))
    mag = _cf(_mag(xin, fmt), fmt).cpu().numpy()
    got = _cf(out, fmt).cpu().numpy().astype(np.float64)
    W = backend.chroma_filterbank(SR, 2048)
    for b in (0, 77, 255):
        s = (mag[b].astype(np.float32) ** 2).astype(np.float64)
        want, bound = R.project(s, W, np.inf)
        bound = bound + R.gamma(2) * want
        assert (np.abs(got[b] - want) <= bound).all(), (b, float((np.abs(got[b] - want) - bound).max()))
    # an item's bits do not depend on its position, the batch size, the layout or the strides
    other = signal.chroma_stft(_wave(x, CF if fmt == CL else CL), tuning=0.0, data_format=CF if fmt == CL else CL)
    assert torch.equal(_cf(other, CF if fmt == CL else CL), _cf(out, fmt))
    assert torch.equal(signal.chroma_stft(xin[100:101], tuning=0.0, data_format=fmt), out[100:101])
    S = _mag(xin, fmt) ** 2
    big = torch.zeros(S.shape[:-1] + (2 * S.shape[-1],), device='cuda')
    big[..., ::2] = S
    assert torch.equal(signal.chroma_stft(S=big[..., ::2], tuning=0.0, data_format=fmt),
                       signal.chroma_stft(S=S.contiguous(), tuning=0.0, data_format=fmt))


@pytest.mark.parametrize('fmt', [CL, CF])
def test_chroma_cqt_and_cens_benchmark_size_within_bound(fmt):
    from kapre_b200 import backend, ops, signal
    x = _x(256, 1, 5 * SR, 1)
    xin = _wave(x, fmt)
    cqt, plan = signal._cqt_chroma_plans(SR, 512, None, 0.0, 12, 7, 36, True, 41)
    C = _cf(ops.cqt(xin, cqt, fmt, fmt, True), fmt).cpu().numpy().astype(np.float64)
    Mq = backend.cq_to_chroma(252, 36, 12)
    got = _cf(signal.chroma_cqt(xin, data_format=fmt), fmt).cpu().numpy().astype(np.float64)
    cens = _cf(signal.chroma_cens(xin, data_format=fmt), fmt).cpu().numpy().astype(np.float64)
    l1 = _cf(signal.chroma_cqt(xin, norm=1, data_format=fmt), fmt).cpu().numpy()
    for b in (0, 130, 255):
        want, bound = R.project(C[b], Mq, np.inf, 0.0)
        assert (np.abs(got[b] - want) <= bound).all(), (b, float((np.abs(got[b] - want) - bound).max()))
        q = R.quantize(l1[b])
        cw, cb = R.cens_from_q(q, backend.cens_window(41))
        assert (np.abs(cens[b] - cw) <= cb).all(), (b, float((np.abs(cens[b] - cw) - cb).max()))
    # C= inputs: complex and |C| give the waveform path's bits
    Cc = ops.cqt(xin, cqt, fmt, fmt, False)
    assert torch.equal(signal.chroma_cqt(C=Cc, data_format=fmt), signal.chroma_cqt(xin, data_format=fmt))
    Cm = ops.cqt(xin, cqt, fmt, fmt, True)
    assert torch.equal(signal.chroma_cens(C=Cm, data_format=fmt), signal.chroma_cens(xin, data_format=fmt))


def test_tuning_estimate_equals_reference_on_device_s():
    from kapre_b200 import backend, ops, signal
    x = _x(8, 2, 3 * SR, 2)
    S = _mag(_wave(x, CF), CF) ** 2
    stft, plan = signal._stft_chroma_plans(SR, 2048, 512, None, 12, None, 5.0, 2.0, True)
    tuning, tab = ops.chroma_tuning(S, plan, ops.N.CHROMA_IN_LINEAR, CF)
    lo, hi = backend.piptrack_bins(SR, 2048)
    Sh = S.cpu().numpy()
    for b in range(8):
        want, idx, _, _ = R.estimate_tuning(Sh[b], SR, 2048, lo, hi, 0.01, 12)
        assert float(tuning[b]) == want and int(tab[b]) == idx, (b, float(tuning[b]), want)
    # the magnitude squared in the kernel gives the same estimate
    t2, _ = ops.chroma_tuning(_mag(_wave(x, CF), CF), plan, ops.N.CHROMA_IN_SQUARE, CF)
    assert torch.equal(t2, tuning)


def test_tuning_anchors():
    from kapre_b200 import signal
    L = 3 * SR
    a4 = _tone(440.0, L)
    up = _tone(440.0 * 2 ** (0.235 / 12), L)
    down = _tone(440.0 * 2 ** (-0.315 / 12), L)
    x = torch.from_numpy(np.stack([a4, up, down, np.zeros(L, np.float32)])[:, None]).cuda()
    t = signal.estimate_tuning(x, data_format=CF).cpu().numpy()
    assert abs(t[0]) <= 0.03 and abs(t[1] - 0.235) <= 0.03 and abs(t[2] + 0.315) <= 0.03, t
    assert t[3] == 0.0
    c = signal.chroma_stft(x[:1], data_format=CF)
    assert int(c[0, 0].mean(dim=0).argmax()) == 9                  # A


def test_tuning_none_equals_fixed_tuning_bit_for_bit():
    from kapre_b200 import signal
    x = _x(6, 2, 2 * SR, 3)
    x[5] = 0.0
    xin = _wave(x, CL)
    est = signal.estimate_tuning(S=_mag(xin, CL) ** 2, bins_per_octave=12, data_format=CL)
    out = signal.chroma_stft(xin, data_format=CL)
    for b in range(6):
        one = signal.chroma_stft(xin[b:b + 1], tuning=float(est[b]), data_format=CL)
        assert torch.equal(one, out[b:b + 1]), b


def test_launch_counts_capture_and_no_grad():
    from kapre_b200 import _native as N
    from kapre_b200 import signal
    x = torch.from_numpy(_x(4, 1, SR, 4)).cuda()

    def count(fn):
        fn()
        torch.cuda.synchronize()
        n0 = N.launch_count()
        r = fn()
        torch.cuda.synchronize()
        return N.launch_count() - n0, r
    assert count(lambda: signal.chroma_stft(x, tuning=0.0, data_format=CF))[0] == 2
    assert count(lambda: signal.chroma_stft(x, data_format=CF))[0] == 9
    assert count(lambda: signal.chroma_cqt(x, data_format=CF))[0] == 8
    assert count(lambda: signal.chroma_cens(x, data_format=CF))[0] == 9
    assert count(lambda: signal.estimate_tuning(x, data_format=CF))[0] == 8
    S = _mag(x, CF) ** 2
    assert count(lambda: signal.chroma_stft(S=S, tuning=0.0, data_format=CF))[0] == 1
    assert count(lambda: signal.chroma_stft(S=S, data_format=CF))[0] == 8
    from kapre_b200 import ops
    cqt, _ = signal._cqt_chroma_plans(SR, 512, None, 0.0, 12, 7, 36, True, False)
    Cc = ops.cqt(x, cqt, CF, CF, False)
    assert count(lambda: signal.chroma_cqt(C=Cc, data_format=CF))[0] == 1
    assert count(lambda: signal.chroma_cens(C=Cc, data_format=CF))[0] == 2
    # no gradient for CENS and the tuning estimate
    xg = x.clone().requires_grad_(True)
    for out in (signal.chroma_cens(xg, data_format=CF), signal.estimate_tuning(xg, data_format=CF)):
        assert not out.requires_grad and out.grad_fn is None
    # capture and replay with tuning=None
    ref = signal.chroma_stft(x, data_format=CF)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        signal.chroma_stft(x, data_format=CF)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        cap = signal.chroma_stft(x, data_format=CF)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(cap, ref)
    from kapre_b200.composed import Sequential
    from kapre_b200.time_frequency import ChromaSTFT
    seq = Sequential([ChromaSTFT(data_format=CF)])
    captured = seq.capture(x)
    assert torch.equal(captured(x), ref)


def _torch_chroma(s, W, norm, thr=None):
    y = s @ W.T
    if thr is not None:
        y = torch.where(y < thr, torch.zeros_like(y), y)
    if norm is None:
        return y
    a = y.abs()
    n = a.max(dim=-1, keepdim=True).values if norm == np.inf else a.pow(norm).sum(dim=-1, keepdim=True).pow(1 / norm)
    return y / torch.where(n < R.TINY32, torch.ones_like(n), n)


@pytest.mark.parametrize('norm', [np.inf, 1, 2, None])
def test_gradients_against_torch_autograd(norm):
    from kapre_b200 import backend, signal
    rng = np.random.default_rng(6)
    x = torch.from_numpy(_x(2, 1, 8192, 7)).cuda().requires_grad_(True)
    g = torch.from_numpy(rng.standard_normal((2, 1, 17, 12)).astype(np.float32)).cuda()
    # waveform path: against autograd through the library's own |STFT| (whose gradient has its own tests)
    out = signal.chroma_stft(x, norm=norm, tuning=0.1, data_format=CF)
    (gx,) = torch.autograd.grad(out, x, g)
    W = torch.from_numpy(backend.chroma_filterbank(SR, 2048, tuning=0.1)).cuda().double()
    xr = x.detach().clone().requires_grad_(True)
    m = _mag(xr, CF)
    ref = _torch_chroma(m.double() ** 2, W, norm)
    (gr,) = torch.autograd.grad(ref, xr, g.double())
    assert torch.allclose(gx.double(), gr.double(), rtol=2e-3, atol=2e-3 * float(gr.abs().max()))
    # S path
    S = (m.detach() ** 2).requires_grad_(True)
    (gS,) = torch.autograd.grad(signal.chroma_stft(S=S, norm=norm, tuning=0.1, data_format=CF), S, g)
    Sd = S.detach().double().requires_grad_(True)
    (gSr,) = torch.autograd.grad(_torch_chroma(Sd, W, norm), Sd, g.double())
    assert torch.allclose(gS.double(), gSr, rtol=1e-4, atol=1e-4 * float(gSr.abs().max()))
    # C path (complex and magnitude)
    from kapre_b200 import ops
    cqt, _ = signal._cqt_chroma_plans(SR, 512, 220.0, 0.0, 12, 3, 12, True, False)
    Cc = ops.cqt(x.detach(), cqt, CF, CF, False).requires_grad_(True)
    Mq = torch.from_numpy(backend.cq_to_chroma(36, 12, 12, 220.0)).cuda().double()
    outc = signal.chroma_cqt(C=Cc, f_min=220.0, norm=norm, threshold=0.001, n_octaves=3, bins_per_octave=12,
                             data_format=CF)
    gc = torch.randn_like(outc)
    (gC,) = torch.autograd.grad(outc, Cc, gc)
    Cd = Cc.detach().to(torch.complex128).requires_grad_(True)
    (gCr,) = torch.autograd.grad(_torch_chroma(Cd.abs(), Mq, norm, 0.001), Cd, gc.double())
    assert torch.allclose(gC.to(torch.complex128), gCr, rtol=1e-4, atol=1e-4 * float(gCr.abs().max()))


def test_non_finite_isolation():
    from kapre_b200 import signal
    x = _x(3, 2, 2 * SR, 8)
    y = x.copy()
    y[1, 0, 20000] = np.nan
    a = signal.chroma_stft(torch.from_numpy(x).cuda(), data_format=CF).cpu().numpy()
    b = signal.chroma_stft(torch.from_numpy(y).cuda(), data_format=CF).cpu().numpy()
    m = np.arange(a.shape[2]) * 512 - 1024
    hit = (m <= 20000) & (20000 < m + 2048)
    assert np.isnan(b[1, 0, hit]).all() and not np.isnan(b[1, 0, ~hit]).any()
    # the item's tuning estimate ignores the NaN frames: its other frames' chroma are unchanged
    np.testing.assert_array_equal(b[1, 0, ~hit], a[1, 0, ~hit])
    for bi, ci in [(0, 0), (0, 1), (1, 1), (2, 0), (2, 1)]:
        np.testing.assert_array_equal(a[bi, ci], b[bi, ci])
    ta = signal.estimate_tuning(torch.from_numpy(x).cuda(), data_format=CF)
    tb = signal.estimate_tuning(torch.from_numpy(y).cuda(), data_format=CF)
    assert torch.equal(ta[[0, 2]], tb[[0, 2]])
    ca = signal.chroma_cqt(torch.from_numpy(x).cuda(), data_format=CF).cpu().numpy()
    cb = signal.chroma_cqt(torch.from_numpy(y).cuda(), data_format=CF).cpu().numpy()
    assert np.isnan(cb[1, 0]).any() and not np.isnan(cb[1, 1]).any()
    np.testing.assert_array_equal(ca[[0, 2]], cb[[0, 2]])


def test_invalid_arguments_raise_before_any_launch():
    from kapre_b200 import _native as N
    from kapre_b200 import signal
    torch.cuda.synchronize()
    n0 = N.launch_count()
    x = torch.zeros((1, 1, 4096), device='cuda')
    for fn, kw in [(signal.chroma_stft, dict(norm=3)), (signal.chroma_stft, dict(n_chroma=65)),
                   (signal.chroma_stft, dict(n_fft=16384)), (signal.chroma_stft, dict(win_length=1024)),
                   (signal.estimate_tuning, dict(resolution=0.0)), (signal.chroma_cqt, dict(bins_per_octave=30)),
                   (signal.chroma_cqt, dict(tuning=None)), (signal.chroma_cens, dict(win_len_smooth=1000))]:
        with pytest.raises(ValueError):
            fn(x, data_format=CF, **kw)
    assert N.launch_count() == n0


def test_ptxas_budgets():
    """The new kernels use no stack and no local memory (no spills); as built the projection kernels use 64
    registers and the tuning and CENS kernels at most 48, so each 256-thread CTA fits several per SM."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    lib = os.path.join(root, 'kapre_b200', '_lib', 'libkapre_b200.so')
    out = subprocess.run(['cuobjdump', '-res-usage', lib], capture_output=True, text=True, check=True).stdout
    for name, max_regs in (('kb_chroma_kernel', 64), ('kb_chroma_bwd_kernel', 64), ('kb_tune_peak_kernel', 64),
                           ('kb_tune_sel_kernel', 64), ('kb_tune_argmax_kernel', 64), ('kb_cens_kernel', 64)):
        m = re.search(r'Function _Z\d+%s\w*:\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)' % name, out)
        assert m, name
        regs, stack, local = (int(v) for v in m.groups())
        assert stack == 0 and local == 0, (name, stack, local)
        assert regs <= max_regs, (name, regs)
