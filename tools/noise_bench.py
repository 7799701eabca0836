"""Additive noise at a target SNR (``kapre_add_noise``) on 256 x 5 s at 16 kHz: tensor noise mono channels_first and
stereo channels_last, with ``lengths``, bank mode (clips shorter and longer than the signal), the backward with and
without the noise and SNR gradients, and one 10-minute recording; against ``torchaudio.functional.add_noise`` on the
same card (for the bank, the torch composition: modulo index, gather, ``add_noise``), and log-mel alone against
``Sequential([BackgroundNoise, *mel])``.

    python tools/noise_bench.py [--out DIR] [--iters N]

Byte model (float32 samples, per sample and channel): the forward reads x and n twice (energy pass, mix pass) and
writes y, 20 B; the floor (each read once) is 12 B.  In bank mode the bank (a few MB) stays in L2, so only x (twice) and
y count, 12 B.  The backward reads g and n (D pass), then g and x and writes gx, 20 B; with gn it also reads n and writes
gn, 28 B.  The backward is timed on its own (``ops.add_noise_backward`` with the forward's saved energies).  GB/s is that model over the measured time, and its share of the
data-sheet 3.35 TB/s says how far from the HBM bound a case is.  Prints one JSON line per case and a Markdown table,
written to DIR/noise_bench.md when --out is given.  Times are CUDA events over --iters calls after warm-up; the
card's name and power limit are read in the same run."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

HBM = 3.35e12
BATCH, SR, SECONDS = 256, 16000, 5
CF, CL = 'channels_first', 'channels_last'


def _time(fn, iters, warmup=3):
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


def _card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:    # noqa: BLE001
        pl = 'unknown (%s)' % e
    return name, pl


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    ap.add_argument('--iters', type=int, default=50)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('noise_bench needs a GPU')
    import torchaudio.functional as AF
    import kapre_b200
    from kapre_b200.augmentation import BackgroundNoise
    from kapre_b200.composed import Sequential
    from kapre_b200.signal import add_noise
    card, power = _card()
    g = torch.Generator(device='cuda').manual_seed(0)
    L = SR * SECONDS
    rows = []

    def row(case, ms, bytes_per_sample, samples, ref_name=None, ref_ms=None):
        r = {'case': case, 'ms': ms, 'GB/s': bytes_per_sample * samples / (ms * 1e-3) / 1e9,
             'hbm_share': bytes_per_sample * samples / (ms * 1e-3) / HBM,
             'floor_ms': 12 * samples / HBM * 1e3, 'reference': ref_name, 'reference_ms': ref_ms,
             'card': card, 'power_limit': power}
        print(json.dumps(r), flush=True)
        rows.append(r)

    snr = torch.rand(BATCH, 1, device='cuda', generator=g) * 20
    for fmt, C in ((CF, 1), (CL, 2)):
        shape = (BATCH, C, L) if fmt == CF else (BATCH, L, C)
        x = torch.randn(shape, device='cuda', generator=g)
        n = torch.randn(shape, device='cuda', generator=g)
        ms = _time(lambda: add_noise(x, n, snr, data_format=fmt), args.iters)
        xt, nt = (x, n) if fmt == CF else (x.transpose(1, 2).contiguous(), n.transpose(1, 2).contiguous())
        snr_c = snr.expand(BATCH, C)
        ref = _time(lambda: AF.add_noise(xt, nt, snr_c), args.iters)
        row('tensor %s x%d' % (fmt, C), ms, 20, BATCH * C * L, 'torchaudio.functional.add_noise', ref)
    x = torch.randn(BATCH, 1, L, device='cuda', generator=g)
    n = torch.randn(BATCH, 1, L, device='cuda', generator=g)
    lengths = torch.randint(L // 2, L + 1, (BATCH, 1), device='cuda', generator=g)
    ms = _time(lambda: add_noise(x, n, snr, lengths, data_format=CF), args.iters)
    ref = _time(lambda: AF.add_noise(x, n, snr, lengths), args.iters)
    row('lengths, channels_first x1', ms, 20, BATCH * L, 'torchaudio.functional.add_noise', ref)
    # bank: clips of 1 s (looped five times) and 30 s
    rng = np.random.default_rng(0)
    clips = [rng.standard_normal(n_).astype(np.float32) for n_ in (SR, 30 * SR, SR // 2, 7 * SR)]
    layer = BackgroundNoise(clips, snr_range=(0.0, 20.0), seed=0, data_format=CF)
    ms = _time(lambda: layer.call(x), args.iters)
    bank = layer.bank_on(x.device)
    starts = torch.from_numpy(layer.clip_start).cuda()
    lens = torch.from_numpy(layer.clip_len).cuda()

    def torch_bank():
        idx = torch.randint(0, len(clips), (BATCH,), device='cuda')
        off = (torch.rand(BATCH, device='cuda') * lens[idx]).long()
        pos = starts[idx, None] + (off[:, None] + torch.arange(L, device='cuda')[None]) % lens[idx, None]
        s = torch.rand(BATCH, 1, device='cuda') * 20
        return AF.add_noise(x, bank[pos][:, None, :], s)
    ref = _time(torch_bank, args.iters)
    row('bank (0.5-30 s clips, L2-resident), channels_first x1', ms, 12, BATCH * L,
        'modulo index + gather + torchaudio add_noise', ref)
    # backward, timed on its own from the forward's saved energies
    from kapre_b200 import ops
    snr_b = snr.expand(BATCH, 1)
    _, stats = ops.add_noise_forward(x, n, None, snr_b, None, CF, True)
    gy = torch.randn(BATCH, 1, L, device='cuda', generator=g)
    bx = _time(lambda: ops.add_noise_backward(gy, x, n, None, snr_b, None, stats, CF, False, False), 4 * args.iters)
    row('backward gx', bx, 20, BATCH * L)
    bxn = _time(lambda: ops.add_noise_backward(gy, x, n, None, snr_b, None, stats, CF, True, True), 4 * args.iters)
    xg = x.clone().requires_grad_(True)
    ng = n.clone().requires_grad_(True)
    sg = snr.clone().requires_grad_(True)
    ya = AF.add_noise(xg, ng, sg.expand(BATCH, 1))
    ta_b = _time(lambda: torch.autograd.grad(ya, (xg, ng, sg), gy, retain_graph=True), 4 * args.iters)
    row('backward gx, gn, gsnr', bxn, 28, BATCH * L, 'torchaudio add_noise autograd (backward only)', ta_b)
    del xg, ng, gy, ya
    # one 10-minute recording
    xl = torch.randn(1, 1, 600 * SR, device='cuda', generator=g)
    nl = torch.randn(1, 1, 600 * SR, device='cuda', generator=g)
    s1 = torch.tensor([[10.0]], device='cuda')
    ms = _time(lambda: add_noise(xl, nl, s1, data_format=CF), args.iters)
    ref = _time(lambda: AF.add_noise(xl, nl, s1), args.iters)
    row('10-minute recording', ms, 20, 600 * SR, 'torchaudio.functional.add_noise', ref)
    # log-mel alone against BackgroundNoise ahead of it
    mel = kapre_b200.get_melspectrogram_layer(n_fft=1024, hop_length=256, sample_rate=SR, n_mels=128,
                                              return_decibel=True, input_data_format=CL, output_data_format=CL)
    xm = torch.randn(BATCH, L, 1, device='cuda', generator=g)
    layer_cl = BackgroundNoise(clips, snr_range=(0.0, 20.0), seed=0, data_format=CL)
    chain = Sequential([layer_cl, *mel.layers])
    mel_ms = _time(lambda: mel.call(xm), args.iters)
    chain_ms = _time(lambda: chain.call(xm), args.iters)
    r = {'case': 'log-mel vs Sequential([BackgroundNoise, *mel])', 'log_mel_ms': mel_ms, 'with_noise_ms': chain_ms,
         'card': card, 'power_limit': power}
    print(json.dumps(r), flush=True)
    lines = ['%s, power limit %s; %d x %d s at %d Hz unless stated' % (card, power, BATCH, SECONDS, SR), '',
             '| case | ms | GB/s (model) | HBM share | floor ms | reference | reference ms |', '|' + '---|' * 7]
    for q in rows:
        lines.append('| %s | %.3f | %.0f | %.0f%% | %.3f | %s | %s |' % (
            q['case'], q['ms'], q['GB/s'], 100 * q['hbm_share'], q['floor_ms'], q['reference'] or '-',
            '%.3f' % q['reference_ms'] if q['reference_ms'] is not None else '-'))
    lines += ['', 'log-mel alone %.3f ms; BackgroundNoise + log-mel %.3f ms' % (mel_ms, chain_ms)]
    table = '\n'.join(lines) + '\n'
    print(table)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'noise_bench.md'), 'w') as f:
            f.write(table)


if __name__ == '__main__':
    main()
