"""Times the second-order-section cascade (kapre_b200.signal.sosfilt and friends) with CUDA events and prints one JSON
line per case, each with the card's name and power limit.

Cases, on 16 kHz audio: S = 1, 4 and 8 sections on 256 x 5 s mono (channels_first), S = 8 on stereo channels_last,
one 10-minute recording, the backward, sosfiltfilt, the same sections as chained lfilter biquads (the baseline: four
launches per section and a round trip through HBM), and scipy.signal.sosfilt on the CPU (reference only, one run on a
few items).  GB/s use the byte model of DESIGN.md: 12 B per sample (x read by the state and output passes, y written).

    python tools/sos_bench.py [--warmup 10] [--iters 50]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import scipy.signal
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), '..'))

PEAK = 3.35e12      # H100 SXM HBM3 bytes/s


def timed(fn, warmup, iters):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--warmup', type=int, default=10)
    ap.add_argument('--iters', type=int, default=50)
    args = ap.parse_args()
    from kapre_b200.signal import lfilter, sosfilt, sosfiltfilt
    if not torch.cuda.is_available():
        raise SystemExit('sos_bench needs a GPU')
    props = torch.cuda.get_device_properties(0)
    power = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'],
                           capture_output=True, text=True).stdout.strip() or '?'
    W, I = args.warmup, args.iters
    rng = np.random.default_rng(0)
    sr = 16000

    def emit(case, ms, samples=None, **kw):
        rec = {'case': case, 'ms': round(ms, 4), 'gpu': props.name, 'power_limit': power}
        if samples:
            gbs = samples * 12 / (ms * 1e-3) / 1e9
            rec.update({'GB/s': round(gbs, 1), 'peak_share': round(gbs * 1e9 / PEAK, 3)})
        rec.update(kw)
        print(json.dumps(rec), flush=True)

    designs = {1: scipy.signal.butter(2, 0.1, output='sos'),
               4: scipy.signal.butter(8, 0.05, output='sos'),
               8: scipy.signal.butter(8, [300, 3400], 'bandpass', fs=sr, output='sos')}
    x = torch.from_numpy(rng.uniform(-1, 1, (256, 1, 5 * sr)).astype(np.float32)).cuda()
    n = x.numel()
    for S, sos in designs.items():
        st = torch.tensor(sos, dtype=torch.float32, device='cuda')
        emit('sosfilt S=%d 256x5s mono' % S, timed(lambda: sosfilt(x, st, data_format='channels_first'), W, I), n)
        # the baseline: the same sections as chained lfilter biquads
        bs = [torch.tensor(r[:3], dtype=torch.float32, device='cuda') for r in sos]
        as_ = [torch.tensor(r[3:], dtype=torch.float32, device='cuda') for r in sos]

        def chain():
            y = x
            for b, a in zip(bs, as_):
                y = lfilter(y, a, b, clamp=False, data_format='channels_first')
            return y
        emit('chained lfilter biquads S=%d 256x5s mono' % S, timed(chain, W, I), n)
    st = torch.tensor(designs[8], dtype=torch.float32, device='cuda')
    xs = torch.from_numpy(rng.uniform(-1, 1, (256, 5 * sr, 2)).astype(np.float32)).cuda()
    emit('sosfilt S=8 256x5s stereo channels_last', timed(lambda: sosfilt(xs, st, data_format='channels_last'), W, I),
         xs.numel())
    xl = torch.from_numpy(rng.uniform(-1, 1, (1, 1, 600 * sr)).astype(np.float32)).cuda()
    emit('sosfilt S=8 10 min mono', timed(lambda: sosfilt(xl, st, data_format='channels_first'), W, I), xl.numel())
    xg = x.clone().requires_grad_(True)
    y = sosfilt(xg, st, data_format='channels_first')
    gy = torch.ones_like(y)
    emit('backward S=8 256x5s mono', timed(lambda: torch.autograd.grad(y, [xg], gy, retain_graph=True), W, I), n)
    emit('sosfiltfilt S=8 256x5s mono', timed(lambda: sosfiltfilt(x, st, data_format='channels_first'), W, I), n,
         bytes_note='two passes on the padded signal')
    xc = x[:8, 0].cpu().double().numpy()
    t0 = time.perf_counter()
    scipy.signal.sosfilt(designs[8], xc, axis=-1)
    emit('scipy.signal.sosfilt S=8 8x5s mono (CPU, float64)', (time.perf_counter() - t0) * 1e3)


if __name__ == '__main__':
    main()
