"""Times the phase-vocoder time stretch (kapre_b200.augmentation.TimeStretch) with CUDA events and prints one JSON
line per case.

Cases:
  (a) the cfg2 complex STFT shape (256 items, 427 frames, 513 bins, 1 channel), rates 0.8 and 1.25, both formats:
      forward and backward;
  (b) a 10-minute recording at 22.05 kHz, n_fft 1024, hop 512 (1 item, 25 840 frames, 513 bins): forward and
      backward, the workload that takes the chunked path (513 columns cannot fill the GPU);
  (c) torchaudio.functional.phase_vocoder on the cfg2 shape, same GPU, for comparison;
  (d) get_time_stretch_layer end to end on the cfg2 waveforms (256 x 5 s at 22.05 kHz, n_fft 1024, hop 256).
Kernel cases report ms per call and the algorithmic bytes: forward 8 B per distinct input frame read plus 8 B per
output frame, backward 16 B per output frame (Y and G read) plus 16 B per input frame (X read, gX written), per
column; with GB/s and the fraction of the H100 SXM's 3.35 TB/s, and the card name and power limit read in the same
run.

    python tools/time_stretch_bench.py [--steps 50] [--warmup 10] [--out FILE]
"""
import argparse
import json
import math
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


def distinct_frames(T, rate):
    """Input frames (of T) that some output reads: k_u and k_u + 1 over the ceil(T / rate) outputs."""
    k = torch.floor(torch.arange(math.ceil(T / rate), dtype=torch.float64) * rate).long()
    return int(torch.unique(torch.cat([k, k + 1])).lt(T).sum())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=50)
    ap.add_argument('--warmup', type=int, default=10)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('time_stretch_bench needs a GPU')
    import kapre_b200  # noqa: F401
    from kapre_b200 import ops
    from kapre_b200.composed import get_time_stretch_layer

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

    def spectrogram(shape, fmt):
        B, T, F, C = shape
        s = (B, T, F, C) if fmt == 'channels_last' else (B, C, T, F)
        return torch.complex(torch.randn(s, device='cuda', generator=gen), torch.randn(s, device='cuda', generator=gen))

    def kernels(label, shape, fmt, rate):
        B, T, F, C = shape
        X = spectrogram(shape, fmt)
        cols = B * C * F
        To = math.ceil(T / rate)
        chunks = ops._time_stretch_workspace(B, C, T, F, rate, X.device)[0]
        ms = timed(lambda: ops.time_stretch_forward(X, rate, fmt), args.steps, args.warmup)
        report('%s rate %g forward' % (label, rate), ms, cols * 8 * (distinct_frames(T, rate) + To), shape=list(X.shape),
               chunks=chunks)
        Y = ops.time_stretch_forward(X, rate, fmt)
        G = torch.complex(torch.randn(Y.shape, device='cuda', generator=gen), torch.randn(Y.shape, device='cuda', generator=gen))
        ms = timed(lambda: ops.time_stretch_backward(X, Y, G, rate, fmt), args.steps, args.warmup)
        report('%s rate %g backward' % (label, rate), ms, cols * 16 * (To + T), shape=list(X.shape), chunks=chunks)
        return X

    for fmt in ('channels_last', 'channels_first'):
        for rate in (0.8, 1.25):
            X = kernels('cfg2 complex %s' % fmt, (256, 427, 513, 1), fmt, rate)
    kernels('10 min recording', (1, 25840, 513, 1), 'channels_last', 0.8)

    # (c) torchaudio on the same GPU and shape, its (..., freq, time) layout
    try:
        import torchaudio
        Xt = X.view(256, 427, 513).transpose(1, 2).contiguous()
        adv = torch.linspace(0, math.pi * 256, 513, device='cuda')[..., None]
        for rate in (0.8, 1.25):
            ms = timed(lambda: torchaudio.functional.phase_vocoder(Xt, rate, adv), args.steps, args.warmup)
            report('torchaudio phase_vocoder cfg2 rate %g' % rate, ms, 513 * 256 * 8 * (distinct_frames(427, rate) +
                                                                                        math.ceil(427 / rate)))
    except ImportError:
        print(json.dumps(dict(case='torchaudio phase_vocoder', skipped='torchaudio not installed')), flush=True)

    # (d) the waveform factory end to end on the cfg2 waveforms
    x = torch.rand((256, 5 * 22050, 1), device='cuda', generator=gen) * 2 - 1
    for rate in (0.8, 1.25):
        model = get_time_stretch_layer(rate, n_fft=1024, hop_length=256, waveform_data_format='channels_last')
        ms = timed(lambda: model(x), args.steps, args.warmup)
        row = dict(case='get_time_stretch_layer cfg2 waveforms rate %g' % rate, ms=round(ms, 4), card=name,
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
