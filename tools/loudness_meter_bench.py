"""Times the loudness meter on one GPU: ``signal.loudness_stats``, ``signal.true_peak`` (the fused 4x-oversampled peak
kernel) against the composition it replaces (``Resample(4, 1)`` then ``amax``), and a 10-minute recording.

Each number is the mean of CUDA-event-timed calls after warm-up, printed beside its byte and FLOP floor at the H100
SXM data-sheet rates (3.35 TB/s HBM3, 67 TFLOP/s FP32) and with the card's name and power limit read in the same run.
The true-peak floor reads each input sample once (4 B) and forms 4 outputs of 21 taps (168 FLOP); the composition
writes and reads back the 4x signal as well (36 B a sample).  The loudness_stats floor is reading the waveform
once; ``loudness`` alone is timed beside it.

    python tools/loudness_meter_bench.py [--iters 50] [--out loudness_meter.json]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), '..'))

HBM, FP32 = 3.35e12, 67e12
CF, CL = 'channels_first', 'channels_last'


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return q[torch.cuda.current_device()] if q else torch.cuda.get_device_name()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name() + ' (power limit not read)'


def timed(fn, iters):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters * 1e3            # microseconds


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=50)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('loudness_meter_bench needs a GPU')
    from kapre_b200 import ops
    from kapre_b200.signal import loudness, loudness_stats, resample_filter, true_peak
    plan = ops.ResamplePlan(4, 1, resample_filter(4, 1))
    rows = []
    g = torch.Generator(device='cuda').manual_seed(0)
    for name, (B, secs, sr, C, fmt) in (('256 x 5 s 16 kHz mono', (256, 5, 16000, 1, CF)),
                                        ('64 x 10 s 48 kHz stereo channels_last', (64, 10, 48000, 2, CL)),
                                        ('1 x 10 min 48 kHz stereo channels_last', (1, 600, 48000, 2, CL))):
        L = secs * sr
        shape = (B, C, L) if fmt == CF else (B, L, C)
        x = torch.randn(shape, device='cuda', generator=g) * 0.1
        n = B * C * L
        iters = max(5, args.iters // (10 if B == 1 else 1))
        with torch.no_grad():
            t_stats = timed(lambda: loudness_stats(x, sr, data_format=fmt), iters)
            t_loud = timed(lambda: loudness(x, sr, data_format=fmt), iters)
            t_tp = timed(lambda: true_peak(x, data_format=fmt), iters)
            t_comp = timed(lambda: ops.resample(x, plan, fmt).abs().amax(dim=1 if fmt == CL else 2), iters)
            comp = (20 * torch.log10(ops.resample(x, plan, fmt).abs().amax(dim=1 if fmt == CL else 2).double())).float()
            same = bool(((true_peak(x, data_format=fmt) - comp).abs() <= comp.abs() * 2.0 ** -23).all())
        tp_floor = max(4 * n / HBM, 168 * n / FP32) * 1e6
        rows.append({'shape': name, 'loudness_us': round(t_loud, 1), 'loudness_stats_us': round(t_stats, 1),
                     'loudness_stats_floor_us':
                     round(4 * n / HBM * 1e6, 1), 'true_peak_us': round(t_tp, 1), 'true_peak_floor_us': round(tp_floor, 1),
                     'resample_amax_us': round(t_comp, 1), 'resample_amax_floor_us': round(36 * n / HBM * 1e6, 1),
                     'true_peak_equals_composition': same})
    result = {'card': card(), 'rows': rows}
    print(json.dumps(result, indent=1))
    if args.out:
        os.makedirs(os.path.dirname(args.out) or '.', exist_ok=True)
        with open(args.out, 'w') as f:
            json.dump(result, f, indent=1)


if __name__ == '__main__':
    main()
