"""Times the polyphase resampler (kapre_b200.signal.Resample) with CUDA events and prints one JSON line per case.

Cases: 256 x 10 s mono at 48 -> 16 kHz, 44.1 -> 22.05 kHz and 44.1 -> 16 kHz; 48 -> 16 kHz stereo channels_last; a
Resample in front of the cfg2 log-mel dB stack against the log-mel alone; the backward pass at the first shape.
Each reports ms per call, the algorithmic bytes 4 B C (L_in + L_out), GB/s and the fraction of the H100 SXM's
3.35 TB/s, with the card name and power limit read in the same run.  scipy.signal.resample_poly on the host's cores,
over the same batch as the first case, is the CPU baseline.

    python tools/resample_bench.py [--steps 20] [--warmup 5] [--out FILE] [--no-cpu]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

HBM_PEAK = 3.35e12      # H100 SXM data sheet, HBM3


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = 'unknown'
    return name, q


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
    ap.add_argument('--out', default=None)
    ap.add_argument('--no-cpu', action='store_true', help='skip the scipy baseline')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('resample_bench needs a GPU')
    import kapre_b200
    from kapre_b200 import ops
    from kapre_b200.composed import Sequential
    from kapre_b200.signal import Resample

    name, power = card()
    rows = []

    def report(case, ms, bytes_, **extra):
        row = dict(case=case, ms=round(ms, 4), bytes=int(bytes_), gbps=round(bytes_ / ms / 1e6, 1),
                   frac_hbm_peak=round(bytes_ / (ms * 1e-3) / HBM_PEAK, 3), card=name, power_limit_and_max_sm_clock=power,
                   **extra)
        rows.append(row)
        print(json.dumps(row), flush=True)

    B, secs = 256, 10
    gen = torch.Generator(device='cuda').manual_seed(0)
    cases = [('48k->16k mono', 48000, 16000, 1), ('44.1k->22.05k mono', 44100, 22050, 1),
             ('44.1k->16k mono', 44100, 16000, 1), ('48k->16k stereo channels_last', 48000, 16000, 2)]
    for case, orig, target, C in cases:
        layer = Resample(orig, target, data_format='channels_last')
        x = torch.rand((B, secs * orig, C), device='cuda', generator=gen) * 2 - 1
        y = layer(x)
        ms = timed(lambda: layer(x), args.steps, args.warmup)
        report(case, ms, 4 * B * C * (x.shape[1] + y.shape[1]), shape=list(x.shape), up=layer.up, down=layer.down)
        del x, y

    # Resample -> cfg2 log-mel dB against the log-mel alone (cfg2: 256 x 5 s at 22.05 kHz)
    mel = kapre_b200.get_melspectrogram_layer(n_fft=1024, hop_length=256, sample_rate=22050, n_mels=128,
                                              return_decibel=True, input_data_format='channels_last',
                                              output_data_format='channels_last')
    rs = Resample(44100, 22050, data_format='channels_last')
    stack = Sequential([rs, *mel.layers])
    x44 = torch.rand((B, 5 * 44100, 1), device='cuda', generator=gen) * 2 - 1
    x22 = torch.rand((B, 5 * 22050, 1), device='cuda', generator=gen) * 2 - 1
    ms_stack = timed(lambda: stack(x44), args.steps, args.warmup)
    ms_mel = timed(lambda: mel(x22), args.steps, args.warmup)
    report('44.1k Resample -> cfg2 log-mel dB', ms_stack, 4 * B * (x44.shape[1] + x22.shape[1]), logmel_alone_ms=round(ms_mel, 4),
           resample_share_ms=round(ms_stack - ms_mel, 4))
    del x44, x22

    # backward at the first shape: gradient of L_out samples in, L_in samples out
    layer = Resample(48000, 16000, data_format='channels_last')
    x = torch.rand((B, secs * 48000, 1), device='cuda', generator=gen) * 2 - 1
    g = torch.rand((B, layer.plan.output_length(x.shape[1]), 1), device='cuda', generator=gen)
    ms = timed(lambda: ops.resample_backward(g, layer.plan, 'channels_last', x.shape[1]), args.steps, args.warmup)
    report('48k->16k mono backward', ms, 4 * B * (x.shape[1] + g.shape[1]))

    if not args.no_cpu:
        import scipy.signal
        from concurrent.futures import ThreadPoolExecutor
        xh = x[..., 0].cpu().numpy()
        cores = len(os.sched_getaffinity(0))
        t0 = time.perf_counter()
        with ThreadPoolExecutor(cores) as pool:
            list(pool.map(lambda row: scipy.signal.resample_poly(row, 1, 3), xh))
        s = time.perf_counter() - t0
        rows.append(dict(case='48k->16k mono, scipy.signal.resample_poly on the host', s=round(s, 3), threads=cores,
                         gpu_speedup=round(s * 1e3 / rows[0]['ms'], 1)))
        print(json.dumps(rows[-1]), flush=True)

    if args.out:
        with open(args.out, 'w') as f:
            for r in rows:
                f.write(json.dumps(r) + '\n')


if __name__ == '__main__':
    main()
