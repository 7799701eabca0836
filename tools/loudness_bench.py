"""Gated loudness (``signal.loudness``: two ``kapre_lfilter`` calls and ``kapre_loudness``) against
``torchaudio.functional.loudness`` on the same card: 256 x 5 s 16 kHz mono channels_first, 64 x 10 s 48 kHz stereo
channels_last, 256 x 5 s with ``lengths`` (torchaudio looped over the cut items, as it has no lengths), one 10-minute
recording, forward + backward (against torchaudio's autograd), and log-mel alone against
``Sequential([LoudnessNormalization, *mel])``.  Every case's output is checked in the same run: against torchaudio
(|difference| in LU) and, on its first items, against the float64 restatement of tests/loudness_ref.py.

    python tools/loudness_bench.py [--out DIR] [--iters N] [--ref-iters N]

Byte model (float32 samples, per sample and channel): each ``kapre_lfilter`` reads x twice and writes y once (12 B),
and the energy pass reads the K-weighted signal once (4 B): 28 B.  The floor is 28 B over the data-sheet 3.35 TB/s.
Times are CUDA events over --iters calls after warm-up (--ref-iters for torchaudio); the card's name and power limit
are read in the same run.  Prints one JSON line per case and a Markdown table, written to DIR/loudness_bench.md when
--out is given."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, _ROOT)
sys.path.insert(0, os.path.join(_ROOT, 'tests'))

HBM = 3.35e12
BYTES = 28
CF, CL = 'channels_first', 'channels_last'


def _time(fn, iters, warmup=2):
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


def _ref_err(got, x, sr, fmt, lengths=None, items=4):
    """max |got - float64 restatement| over the first items (the restatement with the kernels' float32 coefficients)."""
    import loudness_ref as LR
    xa = x[:items].double().cpu().numpy()
    if fmt == CL:
        xa = xa.transpose(0, 2, 1)
    G, S = LR.geometry(sr)
    want = LR.gated(LR.weight(xa, LR.normalised(LR.k_weighting(sr))), G, S,
                    None if lengths is None else lengths[:items].cpu().numpy())[0]
    return float(np.abs(got[:items].double().cpu().numpy() - want).max())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    ap.add_argument('--iters', type=int, default=50)
    ap.add_argument('--ref-iters', type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('loudness_bench needs a GPU')
    import torchaudio.functional as AF
    import kapre_b200
    from kapre_b200.augmentation import LoudnessNormalization
    from kapre_b200.composed import Sequential
    from kapre_b200.signal import loudness
    card, power = _card()
    g = torch.Generator(device='cuda').manual_seed(0)
    rows = []

    def row(case, ms, samples, ref_name, ref_ms, ta_diff, ref_err):
        r = {'case': case, 'ms': ms, 'GB/s': BYTES * samples / (ms * 1e-3) / 1e9,
             'hbm_share': BYTES * samples / (ms * 1e-3) / HBM, 'floor_ms': BYTES * samples / HBM * 1e3,
             'reference': ref_name, 'reference_ms': ref_ms, 'max_abs_diff_vs_torchaudio_LU': ta_diff,
             'max_abs_err_vs_float64_LU': ref_err, 'card': card, 'power_limit': power}
        print(json.dumps(r), flush=True)
        rows.append(r)

    def noise(shape):
        x = torch.randn(shape, device='cuda', generator=g) * 0.1
        return x * torch.linspace(0.1, 1.0, shape[0], device='cuda').view(-1, 1, 1)

    for B, secs, sr, C, fmt in ((256, 5, 16000, 1, CF), (64, 10, 48000, 2, CL)):
        L = secs * sr
        x = noise((B, C, L) if fmt == CF else (B, L, C))
        xt = x if fmt == CF else x.transpose(1, 2).contiguous()
        got = loudness(x, sr, data_format=fmt)
        ta = AF.loudness(xt, sr)
        ms = _time(lambda: loudness(x, sr, data_format=fmt), args.iters)
        ref = _time(lambda: AF.loudness(xt, sr), args.ref_iters)
        row('%d x %d s %d Hz %s x%d' % (B, secs, sr, fmt, C), ms, B * C * L, 'torchaudio.functional.loudness', ref,
            float((got - ta).abs().max()), _ref_err(got, x, sr, fmt))
    # lengths: torchaudio looped over the cut items
    B, sr, L = 256, 16000, 80000
    x = noise((B, 1, L))
    lengths = torch.randint(L // 2, L + 1, (B,), device='cuda', generator=g)
    got = loudness(x, sr, lengths, data_format=CF)
    lh = lengths.tolist()
    ta = torch.stack([AF.loudness(x[b, :, :lh[b]], sr) for b in range(B)])
    ms = _time(lambda: loudness(x, sr, lengths, data_format=CF), args.iters)
    ref = _time(lambda: [AF.loudness(x[b, :, :lh[b]], sr) for b in range(B)], 1, warmup=0)
    row('256 x 5 s 16 kHz with lengths', ms, B * L, 'torchaudio loop over cut items', ref,
        float((got - ta).abs().max()), _ref_err(got, x, sr, CF, lengths))
    # one 10-minute recording
    xl = noise((1, 1, 600 * sr))
    got = loudness(xl, sr, data_format=CF)
    ta = AF.loudness(xl, sr)
    ms = _time(lambda: loudness(xl, sr, data_format=CF), args.iters)
    ref = _time(lambda: AF.loudness(xl, sr), 1, warmup=1)
    row('10-minute recording 16 kHz', ms, 600 * sr, 'torchaudio.functional.loudness', ref,
        float((got - ta).abs().max()), _ref_err(got, xl, sr, CF, items=1))
    del xl
    # forward + backward
    xg = x.clone().requires_grad_(True)
    gl = torch.ones(B, device='cuda')

    def fb():
        out = loudness(xg, sr, data_format=CF)
        return torch.autograd.grad(out, xg, gl)
    xt = x.clone().requires_grad_(True)

    def fb_ta():
        return torch.autograd.grad(AF.loudness(xt, sr), xt, gl)
    ms = _time(fb, args.iters)
    ref = _time(fb_ta, args.ref_iters)
    ga, gb = fb()[0], fb_ta()[0]
    row('forward + backward 256 x 5 s 16 kHz', ms, B * L, 'torchaudio autograd', ref,
        float((ga - gb).abs().max() / gb.abs().max()), None)
    rows[-1]['note'] = 'max_abs_diff_vs_torchaudio_LU holds the gradients\' max |difference| over torchaudio\'s max |g|'
    # log-mel alone against LoudnessNormalization ahead of it
    mel = kapre_b200.get_melspectrogram_layer(n_fft=1024, hop_length=256, sample_rate=sr, n_mels=128,
                                              return_decibel=True, input_data_format=CL, output_data_format=CL)
    xm = noise((B, L, 1))
    chain = Sequential([LoudnessNormalization(sr, (-30.0, -16.0), seed=0, data_format=CL), *mel.layers])
    mel_ms = _time(lambda: mel.call(xm), args.iters)
    chain_ms = _time(lambda: chain.call(xm), args.iters)
    r = {'case': 'log-mel vs Sequential([LoudnessNormalization, *mel])', 'log_mel_ms': mel_ms,
         'with_normalisation_ms': chain_ms, 'card': card, 'power_limit': power}
    print(json.dumps(r), flush=True)
    lines = ['%s, power limit %s' % (card, power), '',
             '| case | ms | GB/s (28 B model) | HBM share | floor ms | reference | reference ms | max diff | err vs f64 |',
             '|' + '---|' * 9]
    for q in rows:
        lines.append('| %s | %.3f | %.0f | %.0f%% | %.3f | %s | %.2f | %.2g | %s |' % (
            q['case'], q['ms'], q['GB/s'], 100 * q['hbm_share'], q['floor_ms'], q['reference'], q['reference_ms'],
            q['max_abs_diff_vs_torchaudio_LU'],
            '%.2g' % q['max_abs_err_vs_float64_LU'] if q['max_abs_err_vs_float64_LU'] is not None else '-'))
    lines += ['', 'log-mel alone %.3f ms; LoudnessNormalization + log-mel %.3f ms' % (mel_ms, chain_ms)]
    table = '\n'.join(lines) + '\n'
    print(table)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'loudness_bench.md'), 'w') as f:
            f.write(table)


if __name__ == '__main__':
    main()
