"""Cost of the backward passes: CUDA-event time of forward alone and of forward + backward for
  * BASELINE cfg2 log-mel dB (batch 256 mono 22.05 kHz 5 s, n_fft 1024, hop 256, 128 mel, channels_last), and
  * the STFT -> InverseSTFT pair of get_perfectly_reconstructing_stft_istft at the same shape,
with the algorithmic bytes each step moves (computed from shapes below), the card's name and power limit, and
then bench.py's own result line, all in one process tree so the numbers share a card.

usage: python tools/grad_bench.py [--steps 50] [--warmup 5] [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import kapre_b200 as K  # noqa: E402

B, L, SR, N_FFT, HOP, N_MELS = 256, 110250, 22050, 1024, 256, 128


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i',
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ''
    return q or torch.cuda.get_device_name()


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


def logmel_bytes(T, F):
    """Bytes each pass reads and writes (float32 = 4, complex64 = 8)."""
    x, mel, spec = B * L * 4, B * T * N_MELS * 4, B * T * F * 4
    fwd = x + mel
    bwd = (x + 2 * spec                 # recompute the complex spectrum
           + x + mel                    # recompute the pre-dB filterbank output
           + 3 * mel + mel + mel        # dB backward: x three passes, g, gx
           + mel + spec                 # transposed filterbank
           + 2 * spec + spec + 2 * spec  # magnitude backward: S, g, gS
           + 2 * spec + x               # STFT adjoint: inverse kernel reads gS, writes the overlap-add ...
           + x + x)                     # ... the edge/crop pass reads it and writes gx
    return fwd, bwd


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=50)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    res = {'card': card(), 'workload': 'cfg2: batch=256 mono 22.05kHz 5s, n_fft=1024 hop=256 n_mels=128'}
    torch.manual_seed(0)
    x = torch.randn(B, L, 1, device='cuda')

    mel = K.get_melspectrogram_layer(n_fft=N_FFT, hop_length=HOP, sample_rate=SR, n_mels=N_MELS, return_decibel=True,
                                     input_data_format='channels_last', output_data_format='channels_last')
    xg = x.clone().requires_grad_(True)
    y = mel(xg)
    gy = torch.randn_like(y)
    T, F = y.shape[1], N_FFT // 2 + 1

    def mel_fwd():
        with torch.no_grad():
            mel(x)

    def mel_fwd_bwd():
        torch.autograd.grad(mel(xg), xg, grad_outputs=gy)

    fb, bb = logmel_bytes(T, F)
    res['logmel_db'] = {'forward_ms': timed(mel_fwd, args.steps, args.warmup),
                        'forward_backward_ms': timed(mel_fwd_bwd, args.steps, args.warmup),
                        'forward_bytes': fb, 'backward_bytes': bb}

    stft, istft = K.get_perfectly_reconstructing_stft_istft(N_FFT, HOP, 'channels_last', 'channels_last')
    S = stft(x)
    gw = torch.randn_like(istft(S))
    Ts = S.shape[1]
    spec, wav, ola = B * Ts * F * 8, B * L * 4, B * ((Ts - 1) * HOP + N_FFT) * 4

    def pair_fwd():
        with torch.no_grad():
            istft(stft(x))

    def pair_fwd_bwd():
        torch.autograd.grad(istft(stft(xg)), xg, grad_outputs=gw)

    res['stft_istft'] = {'forward_ms': timed(pair_fwd, args.steps, args.warmup),
                         'forward_backward_ms': timed(pair_fwd_bwd, args.steps, args.warmup),
                         'forward_bytes': wav + 2 * spec + ola,
                         # ISTFT adjoint: reads gy, writes gX, fixes 2 bins per frame; STFT adjoint: reads gX, writes
                         # the overlap-add scratch, the edge/crop pass reads it and writes gx
                         'backward_bytes': ola + spec + spec + ola + ola + wav}
    for k in ('logmel_db', 'stft_istft'):
        r = res[k]
        r['backward_ms'] = r['forward_backward_ms'] - r['forward_ms']
        r['backward_GBps'] = r['backward_bytes'] / r['backward_ms'] * 1e-6
    print(json.dumps(res), flush=True)

    del xg, y, gy, S, gw
    torch.cuda.empty_cache()
    bench = subprocess.run([sys.executable, os.path.join(ROOT, 'bench.py'), '--gpus', '1', '--steps', '200',
                            '--warmup', '10', '--no-cpu-baseline'], capture_output=True, text=True, cwd=ROOT)
    line = [ln for ln in bench.stdout.splitlines() if ln.startswith('{')]
    res['bench'] = json.loads(line[-1]) if line else {'rc': bench.returncode, 'stderr': bench.stderr[-2000:]}
    print(json.dumps(res['bench']), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'grad_bench.json'), 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
