"""YIN / pYIN timings on the GPU with CUDA events after warm-up, against a PyTorch restatement on the same device
(cuFFT autocorrelation for the CMNDF, a per-frame torch loop for the Viterbi) and, on a small case, the float64 numpy
reference (tests/pitch_ref.py), each checked against the kernel in the same run.  Prints the card and its power
limit, then one JSON line per case.

FP32 model of the difference launch, per frame and lag tau <= max_period: with segments shared (h < W, g = gcd(W, h)
>= 32) the new segment samples of one hop cost h (sub + fma) and the frame adds W / g partials, so 2 h + W / g lane
instructions; without sharing, 2 W.  At the defaults (256 x 5 s at 22.05 kHz, fmin C2, fmax C7: 216 frames, 338
lags, W 1024, h 512) that is 256 * 216 * 338 * 2048 = 38 G lane-instructions direct, about 1.1 ms at 67 TFLOP/s
counted as 33.5 T lane-instructions/s, and 256 * 216 * 338 * 1026 = 19 G (0.57 ms) shared.  The decisions add
O(n) per frame.  HBM traffic is the input once (plus overlap re-reads from L2) and the outputs: 113 MB at the
defaults, 34 us at 3.35 TB/s, so the launch is FP32-bound.  The Viterbi does 2 w max-plus candidates for each of
n_pitch destination pairs per frame, sequential over frames: it is latency-bound (one CTA per row), and its time is
reported as measured, with no floor."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
from kapre_b200 import ops  # noqa: E402

FP32_LANES = 67e12 / 2          # FP32 lane-instructions per second (an FMA counts 2 FLOPs)
CF, CL = 'channels_first', 'channels_last'


def lane_instructions(plan, B, C, L):
    g = plan.geometry
    M = plan.num_frames(L)
    W, h, P = g['win_length'], g['hop_length'], g['max_period']
    gg = int(np.gcd(W, h))
    per = 2 * h + W // gg if (h < W and gg >= 32) else 2 * W
    return B * C * M * P * per


def timed(fn, warmup, steps):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def torch_cmndf(x, plan):
    """(R, M, n) CMNDF by cuFFT autocorrelation, d = E0 + E_tau - 2 r(tau) (the form the kernel avoids)."""
    g = plan.geometry
    F, W, h, pad, P = g['frame_length'], g['win_length'], g['hop_length'], g['pad'], g['max_period']
    xp = torch.nn.functional.pad(x.reshape(-1, x.shape[-1]), (pad, pad))
    fr = xp.unfold(1, F, h)                                              # (R, M, F)
    a = fr[..., 1:W + 1]
    nfft = 1 << int(np.ceil(np.log2(F + W)))
    r = torch.fft.irfft(torch.fft.rfft(fr, nfft) * torch.fft.rfft(a, nfft).conj(), nfft)[..., 2:P + 2]
    cs = torch.nn.functional.pad(torch.cumsum(fr * fr, -1), (1, 0))
    taus = torch.arange(1, P + 1, device=x.device)
    e0 = cs[..., W + 1] - cs[..., 1]
    et = cs[..., W + 1 + taus] - cs[..., 1 + taus]
    d = (e0[..., None] + et - 2 * r).clamp_min(0)
    c = d / (torch.cumsum(d, -1) / taus + 2.0 ** -126)
    return c[..., g['min_period'] - 1:]


def torch_yin(c, plan, sr, thresh=0.1):
    n = c.shape[-1]
    left = torch.cat([torch.full_like(c[..., :1], float('inf')), c[..., :-1]], -1)
    right = torch.cat([c[..., 1:], torch.full_like(c[..., :1], float('inf'))], -1)
    tr = (c < left) & (c <= right)
    tr[..., 0] = c[..., 0] < c[..., 1]
    tr[..., -1] = c[..., -1] < c[..., -2]
    ok = tr & (c < thresh)
    first = torch.where(ok.any(-1), ok.float().argmax(-1), c.argmin(-1))
    k = first.clamp(1, n - 2)
    c0, c1, c2 = (c.gather(-1, (k + o)[..., None])[..., 0] for o in (-1, 0, 1))
    a, b = c2 + c0 - 2 * c1, (c2 - c0) / 2
    shift = torch.where((b.abs() < a.abs()) & (first > 0) & (first < n - 1), -b / a, torch.zeros_like(a))
    return sr / (plan.geometry['min_period'] + first + shift)


def torch_viterbi(lov, lou, plan):
    """Per-frame torch loop over the banded transition: lov (R, M, n) voiced and lou (R, M) unvoiced log-observations.
    Returns the (R, M) state path."""
    q, t = plan.pyin, plan._tables
    dev = lov.device
    n, w = q['n_pitch'], q['band_width']
    half = w // 2
    ltri = torch.tensor(t['log_triangle'], dtype=torch.float32, device=dev)
    lnorm = torch.tensor(t['log_row_norm'], dtype=torch.float32, device=dev)
    cfg = plan.cfg
    R_, M, _ = lov.shape
    V = cfg.log_init_voiced + lov[:, 0]
    U = cfg.log_init_unvoiced + lou[:, 0, None].expand(R_, n)
    # source i = j + half - q for destination j and tap q
    j = torch.arange(n, device=dev)[:, None]
    qq = torch.arange(w, device=dev)[None, :]
    src = j + half - qq
    valid = (src >= 0) & (src < n)
    srcc = src.clamp(0, n - 1)
    tw = torch.where(valid, ltri[qq.expand(n, w)], torch.full((n, w), -float('inf'), device=dev))
    bps = []
    for m in range(1, M):
        mx = torch.maximum(V.max(1).values, U.max(1).values)[:, None]
        a = V - mx + lnorm
        b = U - mx + lnorm
        ca = a[:, srcc] + tw                              # (R, n, w)
        cb = b[:, srcc] + tw
        ba, ia = ca.max(-1)
        bb, ib = cb.max(-1)
        ia = torch.gather(srcc.expand(R_, n, w), 2, ia[..., None])[..., 0]
        ib = torch.gather(srcc.expand(R_, n, w), 2, ib[..., None])[..., 0]
        x1, x2 = ba + cfg.log_stay, bb + cfg.log_switch
        y1, y2 = ba + cfg.log_switch, bb + cfg.log_stay
        V = torch.where(x1 >= x2, x1, x2) + lov[:, m]
        U = torch.where(y1 >= y2, y1, y2) + lou[:, m, None]
        bps.append(torch.cat([torch.where(x1 >= x2, ia, n + ib), torch.where(y1 >= y2, ia, n + ib)], 1))
    s = torch.cat([V, U], 1).argmax(1)
    path = [s]
    for bp in reversed(bps):
        s = bp.gather(1, s[:, None])[:, 0]
        path.append(s)
    return torch.stack(path[::-1], 1)


def observations(plan, cands, vp, R_, M):
    """Dense log-observations from the kernel's candidate lists (workspace) for the torch Viterbi."""
    n = plan.pyin['n_pitch']
    cn, cb, cp = cands
    lov = torch.full((R_ * M, n), float(np.log(2.0 ** -126)), device=vp.device)
    idx = torch.arange(cb.shape[1], device=vp.device)[None, :] < cn[:, None]
    rows = torch.arange(R_ * M, device=vp.device)[:, None].expand_as(cb)
    lov[rows[idx], cb[idx].long()] = torch.log(cp[idx] + 2.0 ** -126)
    lou = torch.log((1 - vp.reshape(R_, M)) / n + 2.0 ** -126)
    return lov.reshape(R_, M, n), lou


def case(name, sr, fmin, fmax, F, B, C, seconds, fmt, warmup, steps, check_ref=False):
    plan = ops.PitchPlan(sr, fmin, fmax, F, pyin={})
    L = int(seconds * sr)
    rng = np.random.default_rng(0)
    t = np.arange(L) / sr
    f = rng.uniform(100, 600, (B, C, 1)) * 2 ** (0.5 * np.sin(2 * np.pi * 0.5 * t))
    x = (0.5 * np.sin(2 * np.pi * np.cumsum(f, -1) / sr) + 0.02 * rng.standard_normal((B, C, L))).astype(np.float32)
    xt = torch.from_numpy(x).cuda()
    xin = xt.transpose(1, 2).contiguous() if fmt == CL else xt
    M = plan.num_frames(L)
    f0 = ops.yin(xin, plan, fmt)
    ms_yin = timed(lambda: ops.yin(xin, plan, fmt), warmup, steps)
    ms_pyin = timed(lambda: ops.pyin(xin, plan, fmt), warmup, steps)
    li = lane_instructions(plan, B, C, L)
    # baselines
    f0cf = (f0.transpose(1, 2) if fmt == CL else f0).reshape(B * C, M)
    c_t = torch_cmndf(xt, plan)
    base_f0 = torch_yin(c_t, plan, sr)
    agree = float((torch.abs(base_f0 / f0cf - 1) < 1e-3).float().mean())
    assert agree > 0.95, agree
    ms_base_cmndf = timed(lambda: torch_yin(torch_cmndf(xt, plan), plan, sr), 1, 3)
    # the pYIN decode alone: the kernel's candidates through the torch loop, and the Viterbi launch's share
    pf0, flag, vp = ops.pyin(xin, plan, fmt)
    ws = plan.workspace(B, C, L, xt.device)
    N_ = ops.N
    vpc = torch.empty((B, C, M), device='cuda')
    fo = torch.empty_like(vpc)
    fl = torch.empty((B, C, M), dtype=torch.bool, device='cuda')
    xd, _ = ops._wave_desc(xt, CF)
    od = N_.FramesDesc(*vpc.stride())
    N_.check(N_.lib().kapre_pyin(plan.handle(), ops._ptr(xt), ops.ctypes.byref(xd), ops._ptr(fo), ops._ptr(fl),
                                 ops._ptr(vpc), ops.ctypes.byref(od), None, None, ops._ptr(ws), ops._stream_ptr()))
    torch.cuda.synchronize()
    cmax = (plan.n_lags + 1) // 2
    fr = B * C * M
    raw = ws.view(torch.uint8)
    o1 = (fr * 4 + 255) // 256 * 256
    o2 = o1 + (fr * cmax * 4 + 255) // 256 * 256
    cn = raw[:fr * 4].view(torch.int32)
    cp = raw[o1:o1 + fr * cmax * 4].view(torch.float32).reshape(fr, cmax)
    cb = raw[o2:o2 + fr * cmax * 2].view(torch.int16).reshape(fr, cmax).to(torch.int32) & 0xffff
    lov, lou = observations(plan, (cn, cb, cp), vpc, B * C, M)
    path = torch_viterbi(lov, lou, plan)
    n = plan.pyin['n_pitch']
    vagree = float(((path < n) == fl.reshape(B * C, M)).float().mean())
    assert vagree > 0.99, vagree
    ms_base_vit = timed(lambda: torch_viterbi(lov, lou, plan), 0, 1)
    # the decode alone: the Viterbi kernel's time in a profiled run of its own
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        ops.pyin(xin, plan, fmt)
        torch.cuda.synchronize()
    kt = {}
    for e in prof.key_averages():
        for k in ('kb_pitch_kernel', 'kb_viterbi_kernel'):
            if k in e.key:
                kt[k] = e.device_time_total / 1e3 / e.count
    out = dict(case=name, B=B, C=C, seconds=seconds, frames=M, lags=plan.n_lags, yin_ms=round(ms_yin, 4),
               pyin_ms=round(ms_pyin, 4), difference_kernel_ms=round(kt.get('kb_pitch_kernel', -1), 4),
               viterbi_kernel_ms=round(kt.get('kb_viterbi_kernel', -1), 4),
               fp32_floor_ms=round(li / FP32_LANES * 1e3, 4), yin_fp32_floor_share=round(li / FP32_LANES * 1e3 / ms_yin, 3),
               bound='FP32', torch_cmndf_yin_ms=round(ms_base_cmndf, 3), torch_viterbi_ms=round(ms_base_vit, 2),
               yin_agree=round(agree, 4), voicing_agree=round(vagree, 4))
    if check_ref:
        import pitch_ref as R
        g = plan.geometry
        t0 = time.time()
        cm = R.cmndf(x[0, 0], g)
        ref = np.array([R.yin_decide(c, g, 0.1, sr)[1] for c in cm])
        out['numpy_ref_s_per_row'] = round(time.time() - t0, 3)
        out['numpy_ref_agree'] = float(np.mean(np.abs(ref / f0cf[0].cpu().numpy() - 1) < 1e-3))
        assert out['numpy_ref_agree'] > 0.95
    print(json.dumps(out), flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'pitch_bench needs a GPU'
    info = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                          capture_output=True, text=True).stdout.strip()
    print(json.dumps(dict(gpu=info)), flush=True)
    res = [case('defaults 256 x 5 s 22.05 kHz', 22050, 65.40639, 2093.0047, 2048, 256, 1, 5.0, CF, a.warmup, a.steps,
                check_ref=True),
           case('speech 16 kHz fmin 50 fmax 600', 16000, 50.0, 600.0, 1024, 256, 1, 5.0, CF, a.warmup, a.steps),
           case('48 kHz stereo channels_last 64 x 10 s', 48000, 65.40639, 2093.0047, 4096, 64, 2, 10.0, CL, a.warmup,
                a.steps),
           case('one 10-minute recording', 22050, 65.40639, 2093.0047, 2048, 1, 1, 600.0, CF, 1, 2)]
    if a.out:
        with open(a.out, 'w') as f:
            json.dump(dict(gpu=info, cases=res), f, indent=1)


if __name__ == '__main__':
    main()
