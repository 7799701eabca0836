"""Times Griffin-Lim (kapre_b200.time_frequency.GriffinLim) with CUDA events and prints one JSON line per case.

Cases (mono 22.05 kHz noise, |STFT| of it as the magnitude spectrogram, momentum 0.99, init 'ones', 32 iterations):
  (a) 16 x 10 s, n_fft 1024, hop 256: ms per call and per iteration, and the split between the STFT, the inverse STFT
      and the projection: the two transforms timed alone through their own layers at that shape, and every kernel of
      one call summed by torch.profiler (run after the event timings, so it does not disturb them);
  (b) the cfg2-sized batch, 256 x 5 s, n_fft 1024, hop 256;
  (c) 16 x 10 s, n_fft 2048, hop 512;
  (d) torchaudio.functional.griffinlim (rand_init=False) on shape (a): its centred, reflect-padded torch.stft /
      torch.istft loop, the baseline a user has today.  Its conventions differ; its cost per iteration at the same
      n_fft, hop and shape is comparable.
The per-iteration time is (t(32 iterations) - t(0 iterations)) / 32.  Algorithmic bytes per frame per iteration are
44 F + 8 hop (inverse: 8F in, 4 hop out; STFT: 4 hop in, 8F out; projection: 20F in, 8F out); GB/s and the fraction
of the H100 SXM's 3.35 TB/s follow from them, with the card name and power limit read in the same run.

    python tools/griffin_lim_bench.py [--steps 10] [--warmup 3] [--out FILE]
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
N_ITER = 32


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


def kernel_split(fn):
    """{kernel family: device ms} of one call of ``fn``, from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    split = {}
    for ev in prof.key_averages():
        name = ev.key
        fam = ('projection' if 'kb_gl_project' in name else 'init' if 'kb_gl_init' in name else
               'istft' if 'istft' in name or 'idft' in name else 'stft' if ('stft' in name or 'kb_mr' in name or
                                                                          'kb_dft' in name) else None)
        if fam is None:
            continue
        t = getattr(ev, 'device_time_total', None)
        if t is None:
            t = ev.cuda_time_total
        split[fam] = round(split.get(fam, 0.0) + t / 1000.0, 4)
    return split


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('griffin_lim_bench needs a GPU')
    from kapre_b200 import ops
    from kapre_b200 import _native as N
    from kapre_b200.time_frequency import GriffinLim

    name, power = card()
    rows = []
    torch.set_grad_enabled(False)
    gen = torch.Generator(device='cuda').manual_seed(0)
    fmt = 'channels_first'

    def emit(row):
        row.update(card=name, power_limit_and_max_sm_clock=power)
        rows.append(row)
        print(json.dumps(row), flush=True)

    def case(label, B, seconds, n_fft, hop, split=False):
        x = torch.rand((B, 1, int(seconds * 22050)), device='cuda', generator=gen) * 2 - 1
        gl = GriffinLim(n_fft=n_fft, hop_length=hop, n_iter=N_ITER, init='ones', input_data_format=fmt,
                        output_data_format=fmt)
        gl0 = GriffinLim(n_fft=n_fft, hop_length=hop, n_iter=0, init='ones', input_data_format=fmt,
                         output_data_format=fmt)
        stft_plan, istft_plan = gl.plans
        X = ops.stft_forward(x, stft_plan, fmt, fmt, False, False, N.OUT_COMPLEX)
        S = X.abs().contiguous()
        T, F = S.shape[2], S.shape[3]
        ms = timed(lambda: gl(S), args.steps, args.warmup)
        ms0 = timed(lambda: gl0(S), args.steps, args.warmup)
        per_iter = (ms - ms0) / N_ITER
        bytes_iter = (44 * F + 8 * hop) * T * B
        row = dict(case=label, shape=[B, 1, T, F], n_fft=n_fft, hop=hop, n_iter=N_ITER, ms_per_call=round(ms, 3),
                   ms_zero_iterations=round(ms0, 3), ms_per_iteration=round(per_iter, 4), bytes_per_iteration=bytes_iter,
                   gbps=round(bytes_iter / per_iter / 1e6, 1),
                   frac_hbm_peak=round(bytes_iter / (per_iter * 1e-3) / HBM_PEAK, 3))
        if split:
            y = ops.istft(X, istft_plan, fmt, fmt)
            row['stft_alone_ms'] = round(timed(lambda: ops.stft_forward(y, stft_plan, fmt, fmt, False, False,
                                                                        N.OUT_COMPLEX), args.steps, args.warmup), 4)
            row['istft_alone_ms'] = round(timed(lambda: ops.istft(X, istft_plan, fmt, fmt), args.steps, args.warmup), 4)
            row['profiler_ms_per_call_by_kernel'] = kernel_split(lambda: gl(S))
        emit(row)

    case('(a) 16 x 10 s, n_fft 1024 / hop 256', 16, 10, 1024, 256, split=True)
    case('(b) 256 x 5 s (cfg2 size), n_fft 1024 / hop 256', 256, 5, 1024, 256)
    case('(c) 16 x 10 s, n_fft 2048 / hop 512', 16, 10, 2048, 512)

    try:
        import torchaudio
    except ImportError:
        emit(dict(case='(d) torchaudio.functional.griffinlim', skipped='torchaudio is not installed'))
    else:
        n_fft, hop = 1024, 256
        x = torch.rand((16, int(10 * 22050)), device='cuda', generator=gen) * 2 - 1
        win = torch.hann_window(n_fft, device='cuda')
        spec = torch.stft(x, n_fft, hop, window=win, return_complex=True).abs()

        def ta(n):
            return torchaudio.functional.griffinlim(spec, win, n_fft, hop, n_fft, 1.0, n, 0.99, None, False)
        ms = timed(lambda: ta(N_ITER), args.steps, args.warmup)
        ms0 = timed(lambda: ta(0), args.steps, args.warmup)
        per_iter = (ms - ms0) / N_ITER
        emit(dict(case='(d) torchaudio.functional.griffinlim, 16 x 10 s, n_fft 1024 / hop 256, rand_init=False',
                  shape=list(spec.shape), n_iter=N_ITER, ms_per_call=round(ms, 3), ms_zero_iterations=round(ms0, 3),
                  ms_per_iteration=round(per_iter, 4), torchaudio=torchaudio.__version__))
        ours = next(r for r in rows if r['case'].startswith('(a)'))
        emit(dict(case='(a) / (d) speed-up per iteration', ratio=round(per_iter / ours['ms_per_iteration'], 2)))

    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            for r in rows:
                f.write(json.dumps(r) + '\n')


if __name__ == '__main__':
    main()
