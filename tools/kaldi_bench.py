"""Kaldi features (``kapre_kaldi_features``) on 256 x 5 s of mono audio: fbank at 16 kHz / 80 mel, 8 kHz / 23 mel and
48 kHz / 80 mel, and mfcc at 16 kHz, forward and forward + backward; beside (a) ``torchaudio.compliance.kaldi.fbank``
(or ``mfcc``) looped over the items on the same card and (b) this library's fused kapre log-mel launch at the same
n_fft, hop and band count.

    python tools/kaldi_bench.py [--out DIR] [--iters N]

Byte model (float32): the forward reads every sample once (B L 4 bytes) and writes the features once (B T K 4 bytes);
at 16 kHz / 80 mel that is 81.9 MB + 40.8 MB, a 37 us floor at the data-sheet 3.35 TB/s.  GB/s is that model over the
measured time.  The outputs are held to float64 torchaudio at the timed sizes (the first 16 items) within the bound of
tests/kaldi_ref.py.  Prints one JSON line per case and a Markdown table (written to DIR/kaldi_bench.md with --out).
Times are CUDA events over --iters calls after warm-up; the card's name and power limit are read in the same run."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

HBM = 3.35e12
BATCH, SECONDS = 256, 5
CASES = [('fbank', 16000, 80), ('fbank', 8000, 23), ('fbank', 48000, 80), ('mfcc', 16000, 23)]


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
        raise SystemExit('kaldi_bench needs a GPU')
    import torchaudio.compliance.kaldi as TK
    import kaldi_ref as R
    import kapre_b200
    from kapre_b200 import ops, signal
    card, power = _card()
    rng = np.random.default_rng(0)
    rows = []
    for kind, sr, mel in CASES:
        L = SECONDS * sr
        x = torch.from_numpy((0.1 * rng.standard_normal((BATCH, 1, L))).astype(np.float32)).cuda()
        kw = dict(sample_frequency=float(sr), num_mel_bins=mel)
        fn = getattr(signal, 'kaldi_' + kind)
        o = ops.kaldi_options(kind, **kw)
        y = fn(x, data_format='channels_first', **kw)
        # accuracy at the timed size: the first 16 items against float64 torchaudio
        ta_fn = getattr(TK, kind)
        ref = torch.stack([ta_fn(x[b].double(), **kw) for b in range(16)])[:, None]
        bound = R.log_bound(kind, x[:16].cpu().numpy(), o, None, ref.cpu().numpy()) + 2e-4 * ref.abs().cpu().numpy()
        err = (y[:16].double() - ref).abs().cpu().numpy()
        ok = bool((err <= bound).all())
        t_fwd = _time(lambda: fn(x, data_format='channels_first', **kw), args.iters)
        xg = x.clone().requires_grad_(True)

        def fwd_bwd():
            xg.grad = None
            fn(xg, data_format='channels_first', **kw).sum().backward()
        t_fb = _time(fwd_bwd, max(args.iters // 5, 3))
        t_ta = _time(lambda: [ta_fn(x[b], **kw) for b in range(BATCH)], 2, warmup=1)
        W, H, Np = kapre_b200.backend.kaldi_window_properties(float(sr))
        melspec = kapre_b200.get_melspectrogram_layer(n_fft=Np, win_length=W, hop_length=H, sample_rate=sr, n_mels=mel,
                                                      return_decibel=True, input_data_format='channels_first',
                                                      output_data_format='channels_first')
        t_mel = _time(lambda: melspec(x), args.iters)
        T, K = y.shape[2], y.shape[3]
        nbytes = BATCH * L * 4 + BATCH * T * K * 4
        row = dict(case='%s %d Hz %d mel' % (kind, sr, mel), frames=T, bins=K, fwd_ms=round(t_fwd, 4),
                   fwd_bwd_ms=round(t_fb, 4), torchaudio_loop_ms=round(t_ta, 2), kapre_logmel_ms=round(t_mel, 4),
                   bytes=nbytes, gbps=round(nbytes / t_fwd / 1e6, 1), floor_us=round(nbytes / HBM * 1e6, 1),
                   within_bound=ok, max_err=float(err.max()), card=card, power_limit=power)
        print(json.dumps(row), flush=True)
        rows.append(row)
    lines = ['card: %s, power limit %s' % (card, power), '',
             '| case | frames x bins | forward ms | fwd+bwd ms | GB/s (model) | floor us | torchaudio loop ms | '
             'kapre log-mel ms | within bound |', '|---|---|---|---|---|---|---|---|---|']
    for r in rows:
        lines.append('| %s | %d x %d | %.3f | %.3f | %.0f | %.1f | %.1f | %.3f | %s |'
                     % (r['case'], r['frames'], r['bins'], r['fwd_ms'], r['fwd_bwd_ms'], r['gbps'], r['floor_us'],
                        r['torchaudio_loop_ms'], r['kapre_logmel_ms'], r['within_bound']))
    table = '\n'.join(lines)
    print(table)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'kaldi_bench.md'), 'w') as f:
            f.write(table + '\n')


if __name__ == '__main__':
    main()
