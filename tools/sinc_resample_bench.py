"""Times the band-limited interpolator (ops.sinc_resample, the kernel behind Speed and PitchShift) with CUDA events and
prints one JSON line per case.

Cases: 256 x 10 s mono at 16 kHz at the ratios 1/3, 2^(-4/12), 2^(5/12) and 2; 2^(-4/12) stereo channels_last; the
backward pass of 2^(-4/12); ``Resample(48000, 16000)`` on 256 x 10 s at 48 kHz next to the interpolator at 1/3 on the
same input (the price of a ratio-independent table); ``PitchShift(+4)`` on 256 x 5 s at 22.05 kHz as a whole and split
into its four steps; ``torchaudio.functional.speed`` and ``pitch_shift`` on the same card and input where torchaudio
is installed.  Each kernel case reports ms per call, the algorithmic bytes 4 B C (L_in + L_out), GB/s and the share
of the H100 SXM's 3.35 TB/s, with the card name and power limit read in the same run.

    python tools/sinc_resample_bench.py [--steps 30] [--warmup 5] [--out FILE]
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
CL = 'channels_last'


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
    ap.add_argument('--steps', type=int, default=30)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('sinc_resample_bench needs a GPU')
    from kapre_b200 import ops
    from kapre_b200.augmentation import PitchShift
    from kapre_b200.signal import Resample

    name, power = card()
    rows = []

    def report(case, ms, bytes_=None, **extra):
        row = dict(case=case, ms=round(ms, 4), card=name, power_limit_and_max_sm_clock=power, **extra)
        if bytes_ is not None:
            row.update(bytes=int(bytes_), gbps=round(bytes_ / ms / 1e6, 1),
                       frac_hbm_peak=round(bytes_ / (ms * 1e-3) / HBM_PEAK, 3))
        rows.append(row)
        print(json.dumps(row), flush=True)

    B = 256
    gen = torch.Generator(device='cuda').manual_seed(0)
    L = 10 * 16000
    x = torch.rand((B, L, 1), device='cuda', generator=gen) * 2 - 1
    for label, ratio in (('1/3', 1 / 3), ('2^(-4/12)', 2.0 ** (-4 / 12)), ('2^(5/12)', 2.0 ** (5 / 12)), ('2', 2.0)):
        Lo = math.ceil(L * ratio)
        ms = timed(lambda: ops.sinc_resample(x, ratio, Lo, 0.0, CL), args.steps, args.warmup)
        report('ratio %s mono' % label, ms, 4 * B * (L + Lo), shape=list(x.shape), taps=2 * math.ceil(10 / min(1.0, ratio)))
    ratio = 2.0 ** (-4 / 12)
    Lo = math.ceil(L * ratio)
    g = torch.rand((B, Lo, 1), device='cuda', generator=gen)
    ms = timed(lambda: ops.sinc_resample_backward(g, ratio, 0.0, CL, L), args.steps, args.warmup)
    report('ratio 2^(-4/12) mono backward', ms, 4 * B * (L + Lo))
    del g
    x2 = torch.rand((B, L, 2), device='cuda', generator=gen) * 2 - 1
    ms = timed(lambda: ops.sinc_resample(x2, ratio, Lo, 0.0, CL), args.steps, args.warmup)
    report('ratio 2^(-4/12) stereo channels_last', ms, 4 * B * 2 * (L + Lo), shape=list(x2.shape))
    del x2, x

    # the polyphase kernel and the interpolator on the same 48 kHz input at 1/3
    x48 = torch.rand((B, 10 * 48000, 1), device='cuda', generator=gen) * 2 - 1
    poly = Resample(48000, 16000, data_format=CL)
    ms = timed(lambda: poly(x48), args.steps, args.warmup)
    report('Resample(48000, 16000), polyphase', ms, 4 * B * (x48.shape[1] + 160000), shape=list(x48.shape))
    ms = timed(lambda: ops.sinc_resample(x48, 1 / 3, 160000, 0.0, CL), args.steps, args.warmup)
    report('ratio 1/3 on the same input', ms, 4 * B * (x48.shape[1] + 160000), shape=list(x48.shape))
    del x48

    # PitchShift(+4) on the cfg2 waveform batch, whole and step by step
    xs = torch.rand((B, 5 * 22050, 1), device='cuda', generator=gen) * 2 - 1
    ps = PitchShift(4, n_fft=1024, hop_length=256, window_name='hann_window', data_format=CL)
    rate = ps.rate(4)
    report('PitchShift(+4) 256 x 5 s at 22.05 kHz, n_fft 1024, hop 256', timed(lambda: ps(xs), args.steps, args.warmup))
    S = ps.stft.call(xs)
    Y = ps.stretch.call(S, rate=rate)
    w = ps.istft.call(Y)
    report('  step 1: STFT', timed(lambda: ps.stft.call(xs), args.steps, args.warmup), 4 * xs.numel() + 8 * S.numel())
    report('  step 2: TimeStretch', timed(lambda: ps.stretch.call(S, rate=rate), args.steps, args.warmup),
           8 * (S.numel() + Y.numel()))
    report('  step 3: InverseSTFT', timed(lambda: ps.istft.call(Y), args.steps, args.warmup), 8 * Y.numel() + 4 * w.numel())
    report('  step 4: interpolation', timed(lambda: ops.sinc_resample(w, rate, xs.shape[1], ps.offset(rate), CL),
                                            args.steps, args.warmup), 4 * (w.numel() + xs.numel()))
    del S, Y, w

    ms = timed(lambda: ops.sinc_resample(xs, 1 / 1.1, math.ceil(xs.shape[1] / 1.1), 0.0, CL), args.steps, args.warmup)
    report('Speed(1.1), same input', ms, 4 * (xs.numel() + B * math.ceil(xs.shape[1] / 1.1)))
    xt = xs[..., 0]
    few = max(3, args.steps // 10)
    for case, call in (('torchaudio.functional.pitch_shift(+4), same input',
                        lambda AF: AF.pitch_shift(xt, 22050, 4, n_fft=1024, hop_length=256)),
                       ('torchaudio.functional.speed(1.1), same input', lambda AF: AF.speed(xt, 22050, 1.1))):
        try:
            import torchaudio.functional as AF
            report(case, timed(lambda: call(AF), few, 2))
        except Exception as e:          # not installed, or this torchaudio no longer has the function: not measured
            rows.append(dict(case=case, note='not measured: %s: %s' % (type(e).__name__, e)))
            print(json.dumps(rows[-1]), flush=True)

    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            for r in rows:
                f.write(json.dumps(r) + '\n')


if __name__ == '__main__':
    main()
