"""Constant-Q transform timings on the GPU: the forward, the fused magnitude mode and forward + backward, with CUDA
events, against a PyTorch restatement of the same transform (one conv1d per octave over the same pyramid and taps,
what a user writes without the kernel), checked against each other in the same run.

Byte model (per call): the input read once by the first decimation and by the transform, each pyramid level written
once and read twice (next decimation and transform), the output written.  FLOP model: the useful work, 2 real
multiply-adds per (bin, tap, frame) over each bin's own filter (ceil(l_k / 2^i) taps), plus the decimations (44
multiply-adds per output).  The kernel executes more: each octave's table pads every bin to the octave's longest
filter, which the `executed_GFLOP` column counts.  The default case is bound by the pyramid's traffic (HBM,
3.35 TB/s), B = 36 by the FP32 pipe (67 TFLOP/s).  The pyramid alone (the n_octaves - 1 decimation launches) is timed
too, so that the forward splits into decimation and transform.  The baseline runs cuDNN in full FP32 (no TF32)."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from kapre_b200 import ops  # noqa: E402

HBM, FP32 = 3.35e12, 67e12
CF, CL = 'channels_first', 'channels_last'


def models(plan, B, C, L, magnitude):
    """(useful FLOPs, executed FLOPs, bytes, useful CQT multiply-adds per frame) of one forward call."""
    Ls = [L]
    for _ in range(1, plan.n_octaves):
        Ls.append((Ls[-1] + 1) // 2)
    M = plan.num_frames(L)
    g = plan.geometry
    per_frame = sum(2 * int(np.ceil(g['lengths'][k] / 2.0 ** i)) for i, (k0, k1) in enumerate(g['octaves'])
                    for k in range(k0, k1))
    decim = 44 * sum(Ls[1:])
    useful = per_frame * M + decim
    executed = sum(2 * t.shape[0] * t.shape[1] * M for t in plan.tables) + decim
    out = B * C * M * plan.n_bins * (4 if magnitude else 8)
    byts = 4 * B * C * (2 * Ls[0] + 3 * sum(Ls[1:])) + out
    return 2.0 * B * C * useful, 2.0 * B * C * executed, float(byts), per_frame


def pyramid(x, plan):
    lv = x.reshape(-1, 1, x.shape[-1])
    for _ in range(1, plan.n_octaves):
        lv = ops.resample(lv, plan._rs, CF)
    return lv


def torch_conv(x, plan):
    """(B, C, L) -> (B, C, M, n_bins) complex64 with one conv1d per octave on the kernel's pyramid."""
    B, C, L = x.shape
    M = plan.num_frames(L)
    lv = [x.reshape(B * C, 1, L)]
    for _ in range(1, plan.n_octaves):
        lv.append(ops.resample(lv[-1], plan._rs, CF))
    outs = []
    for i in reversed(range(plan.n_octaves)):
        T = plan._wt[i]
        N, h = T.shape[-1], plan.hop_length >> i
        y = torch.nn.functional.pad(lv[i], (N // 2, N + M * h))
        r = torch.nn.functional.conv1d(y, T, stride=h)[..., :M]
        nb = T.shape[0] // 2
        outs.append(torch.complex(r[:, :nb], r[:, nb:]).transpose(1, 2))
    return torch.cat(outs, -1).reshape(B, C, M, plan.n_bins)


def timed(fn, steps, warmup):
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=5)
    a = ap.parse_args()
    torch.backends.cudnn.allow_tf32 = False
    from kapre_b200.signal import resample_filter
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                       text=True).stdout.strip()
    print('# card: %s' % q)
    cases = [('default 22.05 kHz, 84 bins, 256 x 5 s', 22050, 512, {}, 256, 1, 5 * 22050, CF),
             ('B = 36, 252 bins, 256 x 5 s', 22050, 512, dict(n_bins=252, bins_per_octave=36), 256, 1, 5 * 22050, CF),
             ('44.1 kHz stereo channels_last, 64 x 10 s', 44100, 1024, dict(n_bins=96), 64, 2, 10 * 44100, CL),
             ('one 10-minute recording', 22050, 512, {}, 1, 1, 600 * 22050, CF)]
    for name, sr, hop, kw, B, C, L, fmt in cases:
        plan = ops.CqtPlan(sr, hop, **kw)
        plan._rs = ops.ResamplePlan(1, 2, resample_filter(1, 2))
        plan._wt = [torch.cat([torch.from_numpy(t.real.copy()), torch.from_numpy(t.imag.copy())]).float().cuda()[:, None]
                    for t in plan.tables]
        x = torch.randn(B, C, L, device='cuda')
        xin = x.transpose(1, 2).contiguous() if fmt == CL else x
        y = ops.cqt(xin, plan, fmt, CF)
        yc = torch_conv(x, plan)
        rel = float((y - yc).abs().max() / yc.abs().max())
        assert rel < 1e-4, (name, rel)
        t_f = timed(lambda: ops.cqt(xin, plan, fmt, CF), a.steps, a.warmup)
        t_m = timed(lambda: ops.cqt(xin, plan, fmt, CF, magnitude=True), a.steps, a.warmup)
        xg = xin.clone().requires_grad_(True)
        g = torch.randn_like(y)
        t_fb = timed(lambda: ops.cqt(xg, plan, fmt, CF).backward(g), a.steps, a.warmup)
        t_c = timed(lambda: torch_conv(x, plan), a.steps, a.warmup)
        xcf = xin.transpose(1, 2).contiguous() if fmt == CL else xin
        t_p = timed(lambda: pyramid(xcf, plan), a.steps, a.warmup)
        flops, executed, byts, per_frame = models(plan, B, C, L, False)
        floor_b, floor_c = byts / HBM, flops / FP32
        bound = 'HBM' if floor_b >= floor_c else 'FP32'
        print(json.dumps(dict(case=name, fwd_ms=round(t_f, 4), pyramid_ms=round(t_p, 4),
                              cqt_launch_ms=round(t_f - t_p, 4), mag_ms=round(t_m, 4), fwd_bwd_ms=round(t_fb, 4),
                              conv1d_ms=round(t_c, 4), max_rel_diff_vs_conv1d=rel, model_MB=round(byts / 1e6, 1),
                              cqt_macs_per_frame=per_frame, model_GFLOP=round(flops / 1e9, 2),
                              executed_GFLOP=round(executed / 1e9, 2), GBps=round(byts / t_f / 1e6, 1),
                              fp32_share=round(flops / (t_f * 1e-3) / FP32, 4), bound=bound,
                              floor_ms=round(max(floor_b, floor_c) * 1e3, 4),
                              share_of_floor=round(max(floor_b, floor_c) * 1e3 / t_f, 3))), flush=True)


if __name__ == '__main__':
    main()
