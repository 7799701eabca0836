"""YIN / pYIN on the H100: the CMNDF within the float64 bound (pitch_ref.py) at benchmark size in both layouts, the
decisions against the float64 rule applied to the device's own CMNDF, pYIN's observations and Viterbi path score,
tonal anchors, bit equality across batch positions, layouts and strides, launch counts, capture replay, no-grad
behaviour, non-finite isolation and the ptxas budgets of the new kernels."""
import os
import re
import subprocess

import numpy as np
import pytest
import torch

import pitch_ref as R
from test_pitch_emu import _batch, _decode_reference, _state_path, _tone

pytestmark = pytest.mark.gpu

CL, CF = 'channels_last', 'channels_first'


def _plan(pyin=None, **kw):
    from kapre_b200 import ops
    a = dict(sample_rate=22050, fmin=65.40639, fmax=2093.0047)
    a.update(kw)
    return ops.PitchPlan(a.pop('sample_rate'), a.pop('fmin'), a.pop('fmax'), pyin=pyin, **a)


def _same(u, v):
    """Bit equality that counts NaN as equal to NaN."""
    return torch.equal(u, v) or bool(((u == v) | ((u != u) & (v != v))).all())


def _x(B, C, L, sr, seed):
    return _batch(np.random.default_rng(seed), B, C, L, sr)


@pytest.mark.parametrize('fmt', [CL, CF])
def test_benchmark_size_cmndf_and_decisions(fmt):
    from kapre_b200 import ops
    x = _x(256, 1, 5 * 22050, 22050, 0)
    plan = _plan()
    xt = torch.from_numpy(x).cuda()
    xin = xt.transpose(1, 2).contiguous() if fmt == CL else xt
    M = plan.num_frames(x.shape[2])
    cm = torch.empty((256, 1, M, plan.n_lags), device='cuda')
    f0 = ops.yin(xin, plan, fmt, cmndf=cm)
    f0c = (f0.transpose(1, 2) if fmt == CL else f0).cpu().numpy()
    cmh = cm.cpu().numpy()
    g = plan.geometry
    for b in (0, 131, 255):
        ref, bound = R.cmndf_bound(x[b, 0], g)
        err = np.abs(cmh[b, 0].astype(np.float64) - ref)
        assert (err <= bound).all(), (b, float((err - bound).max()))
        for m in range(0, M, 7):
            _, want = R.yin_decide(cmh[b, 0, m].astype(np.float64), g, 0.1, 22050)
            np.testing.assert_allclose(f0c[b, 0, m], want, rtol=1e-6)
    # an item's bits do not depend on its position, the batch size, the layout or the strides
    other = ops.yin(xt, plan, CF) if fmt == CL else ops.yin(xt.transpose(1, 2).contiguous(), plan, CL).transpose(1, 2)
    assert torch.equal(other.cpu(), torch.from_numpy(f0c))
    one = ops.yin(xin[131:132], plan, fmt)
    assert torch.equal(one, f0[131:132])
    big = torch.zeros((256, 1, 2 * x.shape[2]), device='cuda')
    big[:, :, ::2] = xt
    view = big[:, :, ::2].transpose(1, 2) if fmt == CL else big[:, :, ::2]
    assert torch.equal(ops.yin(view, plan, fmt), f0)


def test_pyin_observations_and_path_on_device():
    from kapre_b200 import ops
    plan = _plan(pyin={})
    sr = 22050
    L = 3 * sr
    rng = np.random.default_rng(1)
    x = np.stack([_tone(np.geomspace(110, 440, L), sr, L, rng=rng, noise=0.05),
                  0.3 * rng.standard_normal(L).astype(np.float32), _tone(196.0, sr, L)])[:, None]
    xt = torch.from_numpy(x).cuda()
    M = plan.num_frames(L)
    cm = torch.empty((3, 1, M, plan.n_lags), device='cuda')
    f0, flag, vp = ops.pyin(xt, plan, CF, cmndf=cm)
    f0, flag, vp, cm = f0.cpu().numpy(), flag.cpu().numpy(), vp.cpu().numpy(), cm.cpu().numpy()
    g, q, t = plan.geometry, plan.pyin, plan._tables
    n = q['n_pitch']
    for b in range(3):
        obs, vps = [], []
        for m in range(M):
            o, v, _ = R.pyin_observe(cm[b, 0, m].astype(np.float64), g, q, t)
            obs.append(o)
            vps.append(v)
        np.testing.assert_allclose(vp[b, 0], vps, rtol=1e-4, atol=1e-6)
        lobs, la, path, best = _decode_reference(plan, obs, vp[b, 0].astype(np.float64))
        sp = _state_path(plan, f0[b, 0], flag[b, 0])
        mask = np.full(lobs.shape, -np.inf)
        for m in range(M):
            if sp[m] >= 0:
                mask[m, sp[m]] = 0.0
            else:
                mask[m, n:] = 0.0
        A, band = R.transition(q, t)
        kpath, _ = R.viterbi(lobs + mask, A, band)
        init = np.log(np.concatenate([np.zeros(n), np.full(n, 1.0 / n)]) + R.TINY)
        assert R.path_score(kpath, lobs, la, init) >= best - R.path_bound(M, lobs, la)
    B12 = 12 * q['bins_per_semitone']
    assert flag[2, 0, 2:-2].all() and np.all(np.abs(B12 * np.log2(f0[2, 0, 2:-2] / 196.0)) <= 1.0 + 1e-6)
    assert flag[1, 0].mean() < 0.3


@pytest.mark.parametrize('case', ['speech16k', 'stereo48k'])
def test_other_configurations(case):
    from kapre_b200 import ops, signal
    if case == 'speech16k':
        x = _x(8, 1, 3 * 16000, 16000, 2)
        kw = dict(sample_rate=16000, fmin=50.0, fmax=600.0, frame_length=1024)
        fmt = CF
        xin = torch.from_numpy(x).cuda()
    else:
        x = _x(4, 2, 2 * 48000, 48000, 3)
        kw = dict(sample_rate=48000, fmin=65.0, fmax=2000.0, frame_length=4096)
        fmt = CL
        xin = torch.from_numpy(x).cuda().transpose(1, 2).contiguous()
    plan = _plan(**kw)
    B, C = x.shape[:2]
    M = plan.num_frames(x.shape[2])
    cm = torch.empty((B, C, M, plan.n_lags), device='cuda')
    f0 = ops.yin(xin, plan, fmt, cmndf=cm)
    assert torch.equal(signal.yin(xin, data_format=fmt, **kw), f0)
    f0c = (f0.transpose(1, 2) if fmt == CL else f0).cpu().numpy()
    cmh = cm.cpu().numpy()
    g = plan.geometry
    for b, c in [(0, 0), (B - 1, C - 1)]:
        ref, bound = R.cmndf_bound(x[b, c], g)
        assert (np.abs(cmh[b, c].astype(np.float64) - ref) <= bound).all()
        for m in range(0, M, 5):
            _, want = R.yin_decide(cmh[b, c, m].astype(np.float64), g, 0.1, kw['sample_rate'])
            np.testing.assert_allclose(f0c[b, c, m], want, rtol=1e-6)
    p = signal.pyin(xin, data_format=fmt, **kw)
    assert p[0].shape == f0.shape and p[1].dtype == torch.bool and p[2].dtype == torch.float32


def test_ten_minute_recording():
    from kapre_b200 import signal
    sr = 22050
    L = 600 * sr
    t = np.arange(L) / sr
    f = 220 * 2 ** (np.sin(2 * np.pi * t / 60.0))
    x = _tone(f, sr, L)[None, None]
    f0, flag, vp = signal.pyin(torch.from_numpy(x).cuda(), sr, 65.40639, 2093.0047, data_format=CF)
    h = 512
    m = np.arange(f0.shape[2])
    truth = 220 * 2 ** (np.sin(2 * np.pi * m * h / sr / 60.0))
    fl = flag[0, 0].cpu().numpy()
    assert fl[5:-5].mean() > 0.99
    got = f0[0, 0].cpu().numpy()
    ok = fl & (m > 5) & (m < len(m) - 5)
    assert np.abs(12 * np.log2(got[ok] / truth[ok])).max() < 0.3


def test_launch_counts_capture_and_no_grad():
    from kapre_b200 import _native as N
    from kapre_b200 import ops
    plan = _plan(pyin={})
    x = torch.from_numpy(_x(4, 1, 22050, 22050, 4)).cuda()
    a = ops.yin(x, plan, CF)
    torch.cuda.synchronize()
    n0 = N.launch_count()
    ops.yin(x, plan, CF)
    assert N.launch_count() - n0 == 1
    r = ops.pyin(x, plan, CF)
    n0 = N.launch_count()
    r2 = ops.pyin(x, plan, CF)
    assert N.launch_count() - n0 == 2
    for u, v in zip(r, r2):
        assert _same(u, v)
    xg = x.clone().requires_grad_(True)
    for out in (ops.yin(xg, plan, CF),) + tuple(ops.pyin(xg, plan, CF)):
        assert not out.requires_grad and out.grad_fn is None
    assert torch.equal(ops.yin(xg, plan, CF), a)
    # capture and replay
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ops.pyin(x, plan, CF)
    torch.cuda.current_stream().wait_stream(s)
    gph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gph):
        cap = ops.pyin(x, plan, CF)
    gph.replay()
    torch.cuda.synchronize()
    for u, v in zip(cap, r):
        assert _same(u, v)


def test_non_finite_isolation():
    from kapre_b200 import ops
    plan = _plan(pyin={})
    x = _x(3, 2, 22050, 22050, 5)
    y = x.copy()
    y[1, 0, 9000] = np.nan
    a = [t.cpu().numpy() for t in ops.pyin(torch.from_numpy(x).cuda(), plan, CF)]
    b = [t.cpu().numpy() for t in ops.pyin(torch.from_numpy(y).cuda(), plan, CF)]
    assert np.isnan(b[0][1, 0]).all() and not b[1][1, 0].any() and np.isnan(b[2][1, 0]).all()
    for bi, ci in [(0, 0), (0, 1), (1, 1), (2, 0), (2, 1)]:
        for u, v in zip(a, b):
            np.testing.assert_array_equal(u[bi, ci], v[bi, ci])
    ya = ops.yin(torch.from_numpy(x).cuda(), plan, CF).cpu().numpy()
    yb = ops.yin(torch.from_numpy(y).cuda(), plan, CF).cpu().numpy()
    g = plan.geometry
    start = np.arange(ya.shape[2]) * g['hop_length'] - g['pad']
    hit = (start <= 9000) & (9000 < start + g['frame_length'])
    assert np.isnan(yb[1, 0, hit]).all()
    np.testing.assert_array_equal(yb[1, 0, ~hit], ya[1, 0, ~hit])


def test_invalid_arguments_raise_before_any_launch():
    from kapre_b200 import _native as N
    from kapre_b200 import signal
    torch.cuda.synchronize()
    n0 = N.launch_count()
    x = torch.zeros((1, 1, 4096), device='cuda')
    for kw in [dict(fmin=0.0), dict(fmax=20000.0), dict(fmin=3000.0, fmax=2000.0), dict(win_length=2048),
               dict(frame_length=16384)]:
        a = dict(sample_rate=22050, fmin=65.0, fmax=2000.0, data_format=CF)
        a.update(kw)
        with pytest.raises(ValueError):
            signal.yin(x, **a)
    assert N.launch_count() == n0


def test_ptxas_budgets():
    """The new kernels use no stack and no local memory (no spills), and their registers allow two 256-thread pitch
    CTAs (and one 1024-thread Viterbi CTA) per SM: 78 and 42 registers as built."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    lib = os.path.join(root, 'kapre_b200', '_lib', 'libkapre_b200.so')
    out = subprocess.run(['cuobjdump', '-res-usage', lib], capture_output=True, text=True, check=True).stdout
    for name, max_regs in (('kb_pitch_kernel', 128), ('kb_viterbi_kernel', 64)):
        m = re.search(r'Function _Z\d+%s\w*:\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)' % name, out)
        assert m, name
        regs, stack, local = (int(v) for v in m.groups())
        assert stack == 0 and local == 0, (name, stack, local)
        assert regs <= max_regs, (name, regs)
