"""Times the IIR filter (kapre_b200.signal.lfilter and friends) with CUDA events and prints one JSON line per case.

Cases: a biquad, pre-emphasis and an 8th-order filter on 256 x 5 s of 16 kHz mono (channels_first), the biquad on
stereo channels_last, per-item RandomBiquad, a 10-minute recording (with the carry kernel's share), the backward with
and without coefficient gradients, torchaudio.functional.lfilter on the same inputs, and Sequential([Biquad, *mel])
against the mel alone.  GB/s use the byte model of DESIGN.md: 12 B per sample forward (x read twice, y written once),
20 B per sample backward with coefficient gradients (gy twice, x, y, gx), 12 B without.

    python tools/iir_bench.py [--warmup 10] [--iters 50]
"""
import argparse
import json
import os
import sys

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
    import kapre_b200
    from kapre_b200 import _native as N
    from kapre_b200.augmentation import RandomBiquad
    from kapre_b200.backend import biquad_coefficients
    from kapre_b200.composed import Sequential
    from kapre_b200.signal import Biquad, lfilter
    props = torch.cuda.get_device_properties(0)
    try:
        import subprocess
        power = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader'], capture_output=True,
                               text=True).stdout.strip()
    except Exception:       # noqa: BLE001
        power = '?'
    W, I = args.warmup, args.iters
    rng = np.random.default_rng(0)
    sr = 16000

    def emit(case, ms, samples=None, bpp=None, **kw):
        rec = {'case': case, 'ms': round(ms, 4), 'gpu': props.name, 'power_limit': power}
        if samples:
            gbs = samples * bpp / (ms * 1e-3) / 1e9
            rec.update({'GB/s': round(gbs, 1), 'peak_share': round(gbs * 1e9 / PEAK, 3)})
        rec.update(kw)
        print(json.dumps(rec), flush=True)

    filters = {'biquad': biquad_coefficients('lowpass', sr, 1000.0, 0.707),
               'preemph': (np.array([1.0, -0.97]), np.array([1.0, 0.0])),
               'order8': scipy.signal.butter(8, 0.2)}
    x = torch.from_numpy(rng.uniform(-1, 1, (256, 1, 5 * sr)).astype(np.float32)).cuda()
    n = x.numel()
    for name, (b, a) in filters.items():
        bt = torch.tensor(b, dtype=torch.float32, device='cuda')
        at = torch.tensor(a, dtype=torch.float32, device='cuda')
        emit('%s 256x5s mono' % name, timed(lambda: lfilter(x, at, bt, data_format='channels_first'), W, I), n, 12)
        try:
            import torchaudio.functional as F
            xt = x[:, 0]
            emit('torchaudio %s 256x5s mono' % name, timed(lambda: F.lfilter(xt, at, bt), max(2, W // 5), max(3, I // 10)))
        except Exception as e:      # noqa: BLE001
            print(json.dumps({'case': 'torchaudio %s' % name, 'error': repr(e)}), flush=True)
    b, a = filters['biquad']
    bt = torch.tensor(b, dtype=torch.float32, device='cuda')
    at = torch.tensor(a, dtype=torch.float32, device='cuda')
    xs = torch.from_numpy(rng.uniform(-1, 1, (256, 5 * sr, 2)).astype(np.float32)).cuda()
    emit('biquad 256x5s stereo channels_last', timed(lambda: lfilter(xs, at, bt, data_format='channels_last'), W, I),
         xs.numel(), 12)
    rb = RandomBiquad('bandpass', sr, (100.0, 4000.0), (0.5, 3.0), seed=0, data_format='channels_first')
    emit('RandomBiquad per item 256x5s mono', timed(lambda: rb.call(x), W, I), n, 12)
    # the 10-minute recording and the carry's share (the profile brackets the state and output kernels only)
    xl = torch.from_numpy(rng.uniform(-1, 1, (1, 1, 600 * sr)).astype(np.float32)).cuda()
    ms = timed(lambda: lfilter(xl, at, bt, data_format='channels_first'), W, I)
    N.profile_enable(True)
    N.profile_read()
    for _ in range(I):
        lfilter(xl, at, bt, data_format='channels_first')
    torch.cuda.synchronize()
    kms, nk = N.profile_read()
    N.profile_enable(False)
    emit('biquad 10 min mono', ms, xl.numel(), 12, state_plus_output_ms=round(kms / max(I, 1), 4),
         carry_and_powers_share=round(1 - kms / max(I, 1) / ms, 3))
    # backward
    for want_coef in (False, True):
        xg = x.clone().requires_grad_(True)
        btg = bt.clone().requires_grad_(want_coef)
        atg = at.clone().requires_grad_(want_coef)
        y = lfilter(xg, atg, btg, clamp=False, data_format='channels_first')
        gy = torch.ones_like(y)
        ms = timed(lambda: torch.autograd.grad(y, [xg] + ([btg, atg] if want_coef else []), gy, retain_graph=True),
                   W, I)
        emit('backward biquad 256x5s%s' % (' with coefficient grads' if want_coef else ''), ms, n,
             20 if want_coef else 12)
    # Sequential([Biquad, *mel]) against the mel alone
    mel = kapre_b200.get_melspectrogram_layer(n_fft=1024, hop_length=256, sample_rate=sr, n_mels=64,
                                              return_decibel=True, input_data_format='channels_first',
                                              output_data_format='channels_last')
    model = Sequential([Biquad('highpass', sr, 300.0, data_format='channels_first'), *mel.layers])
    emit('mel alone 256x5s', timed(lambda: mel.call(x), W, I))
    emit('Sequential([Biquad, *mel]) 256x5s', timed(lambda: model.call(x), W, I))


if __name__ == '__main__':
    main()
