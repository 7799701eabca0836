"""Times the image-source RIR kernel (simulate_rir_ism) and RoomReverb on the current GPU, with the card's name and
power limit read in the same run, against the useful-tap floor and a vectorised torch baseline (float64 geometry,
float32 taps and index_add_).

    python tools/rir_bench.py [--batch 256] [--reps 5]

Prints one JSON line per case: ms per call, images and taps per second, the share of the floor and, at 16 kHz, the
baseline's time per response (its images enumerated on the GPU inside the timed region) and, for the smaller rooms, the
largest error of each over the kernel's derived bound (rir_ref.py).  The floor is the
larger of the useful taps at the FP32 issue rate (one warp instruction per clock per SM sub-partition, times the
instructions a warp issues per image step, from `cuobjdump -sass`) and at the SFU rate (one reciprocal per tap,
16 per clock per SM)."""
import argparse
import json
import math
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

INSTR_PER_STEP = 23          # warp instructions per (image, warp) step of the tap loop, from cuobjdump -sass


def gpu_info():
    out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                         capture_output=True, text=True).stdout.strip().splitlines()
    return out[torch.cuda.current_device()] if out else 'unknown'


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def torch_baseline(room, src, mic, beta, L, W, fs, c=343.0):
    """The same maths in vectorised torch on the GPU, enumeration included: per row (n_x, p_x) the images of the
    arrival ball in float64 (as the kernel forms its geometry), then taps in float32 in the kernel's factored form
    (one sine per image, then a window, a sign and a quotient per tap; a direct float32 sinc of k - half - frac loses its
    zero crossings at |x| up to half) scattered with a float32 index_add_.  Returns a function that computes one
    response."""
    import rir_ref as RR
    dev = torch.device('cuda')
    R = L * c / fs * (1 + 1e-9)
    axes = []
    for d in range(3):
        lo, hi = RR._nrange(room[d], src[d], mic[d], R)
        n = torch.arange(lo, hi + 1, device=dev, dtype=torch.float64).repeat_interleave(2)
        p = torch.tensor([0.0, 1.0], device=dev, dtype=torch.float64).repeat(n.numel() // 2)
        dd = ((2.0 * n) * room[d] + (1.0 - 2.0 * p) * float(src[d])) - float(mic[d])
        bl, bh = (torch.tensor(float(beta[2 * d + j]), device=dev, dtype=torch.float64) for j in (0, 1))
        gain = bl ** (n - p).abs() * bh ** n.abs()
        axes.append((dd, gain))
    (dx, gx), (dy, gy), (dz, gz) = axes
    half = (W - 1) // 2
    w = torch.from_numpy(RR.hanning(W)).float().to(dev)
    k = torch.arange(W, device=dev, dtype=torch.float32)
    ki = torch.arange(W, device=dev)

    def run():
        h = torch.zeros(L, device=dev)
        qy = dy[:, None] * dy[:, None]
        for i in range(dx.numel()):
            r = torch.sqrt((dx[i] * dx[i] + qy) + (dz * dz)[None, :])
            tau = (r * fs) / c
            keep = torch.floor(tau) < L
            tau, r = tau[keep], r[keep]
            g = gx[i] * (gy[:, None] * gz[None, :])[keep] / (4 * math.pi * r)
            n0 = torch.floor(tau)
            up = (tau - n0 >= 0.5).double()
            e = tau - (n0 + up)                     # exact, in [-1/2, 1/2)
            # sinc(k - half - frac) = (-1)^(jj + 1) sin(pi e) / (pi (jj - e)), jj = k - half - up: one sine per image
            A = torch.where(e == 0, g, g * torch.sin(math.pi * e) / math.pi).float()
            jj = k[None, :] - half - up.float()[:, None]
            e32 = e.float()[:, None]
            sign = 1.0 - 2.0 * torch.remainder(jj + 1, 2)
            tap = torch.where(e32 == 0, (jj == 0).float(), sign / (jj - e32)) * (A[:, None] * w[None, :])
            idx = n0.long()[:, None] + ki[None, :]
            ok = idx < L
            h.index_add_(0, idx[ok], tap[ok])
        return h
    return run


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=256)
    ap.add_argument('--reps', type=int, default=5)
    args = ap.parse_args()
    from kapre_b200 import backend, signal
    from kapre_b200.augmentation import RoomReverb
    import rir_ref as RR
    info = gpu_info()
    props = torch.cuda.get_device_properties(0)
    sms = props.multi_processor_count
    clk_hz = float(info.split(',')[2].strip().split()[0]) * 1e6 if info.count(',') >= 2 else 1.98e9
    src, mic = np.array([1.2, 1.1, 1.3]), np.array([2.3, 2.2, 1.6])
    rr = RoomReverb(16000, seed=0)
    r_room, r_rt, _, _ = rr.draw(1)
    cases = [((5.0, 4.0, 3.0), 0.5), ((3.0, 3.0, 2.5), 0.8), (tuple(r_room[0]), float(r_rt[0]))]
    B, W = args.batch, 81
    for room, rt60 in cases:
        alpha = backend.inverse_sabine(rt60, room)
        beta = RR.betas(np.full(6, alpha))
        for fs in (16000.0, 48000.0):
            L = int(math.ceil(rt60 * fs))
            n_img = RR.images(room, src, mic, beta, fs, 343.0, None, L)[2].size
            rooms = np.tile(room, (B, 1))
            ms = timed(lambda: signal.simulate_rir_ism(rooms, src, mic[None], None, alpha, L, sample_rate=fs), args.reps)
            taps = float(n_img) * W * B
            steps = taps / 32 / 0.72                # warp steps: 32 lanes, ~72% of a touching warp's lanes hit
            t_issue = steps * INSTR_PER_STEP / (4 * sms * clk_hz)
            t_sfu = taps / (16 * sms * clk_hz)
            floor = max(t_issue, t_sfu)
            row = dict(case='simulate_rir_ism', room=room, rt60=rt60, fs=fs, batch=B, length=L, images=n_img,
                       ms=round(ms, 3), images_per_s=B * n_img / (ms * 1e-3), taps_per_s=taps / (ms * 1e-3),
                       floor_ms=round(floor * 1e3, 3), floor_share=round(floor / (ms * 1e-3), 3),
                       bound='issue' if t_issue >= t_sfu else 'sfu', gpu=info)
            if fs == 16000.0:
                run = torch_baseline(room, src, mic, beta, L, W, fs)
                ms_base = timed(run, max(1, args.reps // 2))
                row.update(torch_ms_per_item=round(ms_base, 3), torch_ms_times_batch=round(ms_base * B, 1))
                if n_img < 1000000:                 # the float64 restatement of larger rooms takes minutes
                    ref, bound = RR.rir(room, src, mic, beta, L, W, fs)
                    got = signal.simulate_rir_ism(room, src, mic[None], None, alpha, L, sample_rate=fs)[0, :, 0]
                    row.update(kernel_err_over_bound=float(np.max(np.abs(got.double().cpu().numpy() - ref) / bound)),
                               torch_err_over_bound=float(np.max(np.abs(run().double().cpu().numpy() - ref) / bound)))
            print(json.dumps(row), flush=True)
    x = torch.randn(B, 5 * 16000, 1, device='cuda')
    layer = RoomReverb(16000, seed=1)
    ms = timed(lambda: layer.call(x), args.reps)
    print(json.dumps(dict(case='RoomReverb', batch=B, seconds=5, fs=16000, ms=round(ms, 3), gpu=info)), flush=True)


if __name__ == '__main__':
    main()
