"""Times PCEN (kapre_b200.time_frequency.PCEN) with CUDA events and prints one JSON line per case.

Cases:
  (a) the cfg2 mel shape (256 items, 427 frames, 128 bands, 1 channel) in both formats: the forward, the forward
      that also writes the smoother state M (the autograd path), and the backward pass;
  (b) a 10-minute recording at 22.05 kHz, hop 256 (1 item, 51 680 frames, 128 bands): forward and backward, the
      workload that takes the chunked path (128 columns cannot fill the GPU);
  (c) Sequential([STFT, Magnitude, ApplyFilterbank, PCEN]) against the cfg2 log-mel dB stack, per step.
Each kernel case reports ms per call, the algorithmic bytes (forward 8 B per element, 12 B with M, backward 16 B:
E, M and gy read, gE written), GB/s and the fraction of the H100 SXM's 3.35 TB/s, with the card name and power
limit read in the same run.  The backward time includes the torch reduction of the parameter partial sums.

    python tools/pcen_bench.py [--steps 50] [--warmup 10] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

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
    ap.add_argument('--steps', type=int, default=50)
    ap.add_argument('--warmup', type=int, default=10)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('pcen_bench needs a GPU')
    import kapre_b200
    from kapre_b200 import ops
    from kapre_b200.composed import Sequential
    from kapre_b200.time_frequency import PCEN

    name, power = card()
    rows = []

    def report(case, ms, bytes_, **extra):
        row = dict(case=case, ms=round(ms, 4), bytes=int(bytes_), gbps=round(bytes_ / ms / 1e6, 1),
                   frac_hbm_peak=round(bytes_ / (ms * 1e-3) / HBM_PEAK, 3), card=name, power_limit_and_max_sm_clock=power,
                   **extra)
        rows.append(row)
        print(json.dumps(row), flush=True)

    gen = torch.Generator(device='cuda').manual_seed(0)
    torch.set_grad_enabled(False)

    def kernels(label, shape, fmt, hop):
        B, T, F, C = shape
        E = 10.0 ** (torch.rand((B, T, F, C) if fmt == 'channels_last' else (B, C, T, F), device='cuda', generator=gen) * 4 - 2)
        layer = PCEN(sample_rate=22050, hop_length=hop, data_format=fmt)
        layer(E)
        w = layer.weights
        n = E.numel()
        _, (b, c, t, f) = ops._spec_desc(E, fmt)
        chunks = ops._pcen_workspace(b, c, t, f, E.device)[0]
        ms = timed(lambda: ops.pcen(E, w, layer.eps, fmt), args.steps, args.warmup)
        report('%s forward' % label, ms, 8 * n, shape=list(E.shape), chunks=chunks)
        ms = timed(lambda: ops.pcen_forward(E, w, layer.eps, fmt, save_M=True), args.steps, args.warmup)
        report('%s forward, M saved' % label, ms, 12 * n, shape=list(E.shape), chunks=chunks)
        _, M = ops.pcen_forward(E, w, layer.eps, fmt, save_M=True)
        gy = torch.rand(E.shape, device='cuda', generator=gen)
        ms = timed(lambda: ops.pcen_backward(E, M, gy, w, layer.eps, fmt), args.steps, args.warmup)
        report('%s backward' % label, ms, 16 * n, shape=list(E.shape), chunks=chunks)

    for fmt in ('channels_last', 'channels_first'):
        kernels('cfg2 mel %s' % fmt, (256, 427, 128, 1), fmt, 256)
    kernels('10 min recording channels_last', (1, 51680, 128, 1), 'channels_last', 256)

    # (c) log-mel magnitudes + PCEN against the cfg2 log-mel dB stack, 256 x 5 s at 22.05 kHz
    fmt = 'channels_last'
    kw = dict(n_fft=1024, hop_length=256, sample_rate=22050, n_mels=128, input_data_format=fmt, output_data_format=fmt)
    mel = kapre_b200.get_melspectrogram_layer(return_decibel=False, **kw)
    logmel = kapre_b200.get_melspectrogram_layer(return_decibel=True, **kw)
    stack = Sequential([*mel.layers, PCEN(sample_rate=22050, hop_length=256, data_format=fmt)])
    x = torch.rand((256, 5 * 22050, 1), device='cuda', generator=gen) * 2 - 1
    ms_stack = timed(lambda: stack(x), args.steps, args.warmup)
    ms_db = timed(lambda: logmel(x), args.steps, args.warmup)
    ms_mel = timed(lambda: mel(x), args.steps, args.warmup)
    row = dict(case='cfg2 log-mel + PCEN per step', ms=round(ms_stack, 4), logmel_db_ms=round(ms_db, 4),
               mel_alone_ms=round(ms_mel, 4), pcen_share_ms=round(ms_stack - ms_mel, 4), card=name,
               power_limit_and_max_sm_clock=power)
    rows.append(row)
    print(json.dumps(row), flush=True)

    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            for r in rows:
                f.write(json.dumps(r) + '\n')


if __name__ == '__main__':
    main()
