"""Cost of the backward passes of the layers next to the hot path, at shapes derived from BASELINE cfg2 (batch 256
mono 22.05 kHz 5 s; n_fft 1024, hop 256, 128 mel):
  * Delta (win 9), SpecAugment and ConcatenateFrequencyMap on the (256, 427, 128, 1) channels_last log-mel;
  * Frame (1024 samples every 256) and Energy (kapre's defaults, 2205 every 1102) on the 256 x 110250 waveform;
  * get_stft_mag_phase at n_fft 1024 / hop 256: the kapre_mag_phase_backward pass alone, and the whole backward
    (spectrum recompute, the pass, STFT adjoint; with dB also the magnitude recompute and the decibel backward)
    as forward + backward minus forward.
Each pass is timed alone with CUDA events and reported with the algorithmic bytes it moves (every input element read
once, every output element written once; computed from the shapes below) and the GB/s that implies, against the
H100 SXM's 3.35 TB/s.  The card's name and power limit are printed with the numbers.

usage: python tools/grad_adjacent_bench.py [--steps 50] [--warmup 5] [--out DIR]
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import kapre_b200 as K  # noqa: E402
from kapre_b200 import ops  # noqa: E402
from grad_bench import card, timed  # noqa: E402

B, L, SR, N_FFT, HOP, N_MELS = 256, 110250, 22050, 1024, 256, 128
HBM_GBPS = 3350.0
CL = 'channels_last'


def row(ms, nbytes):
    gbps = nbytes / ms * 1e-6
    return {'ms': ms, 'bytes': nbytes, 'GBps': gbps, 'of_hbm_peak': gbps / HBM_GBPS}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=50)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    run = lambda fn: timed(fn, args.steps, args.warmup)   # noqa: E731
    res = {'card': card(), 'workload': 'cfg2-derived shapes: log-mel (256, 427, 128, 1), waveform 256 x 110250'}
    torch.manual_seed(0)

    T = 1 + (L - N_FFT) // HOP
    n_mel = B * T * N_MELS
    g = torch.randn(B, T, N_MELS, 1, device='cuda')
    res['delta_win9'] = row(run(lambda: ops.delta_backward(g, 9, 'symmetric', CL)), 2 * 4 * n_mel)
    aug = K.SpecAugment(freq_mask_param=27, time_mask_param=100, n_freq_masks=2, n_time_masks=2, data_format=CL, seed=0)
    aug.call(g, training=True)
    tm, fm = (torch.as_tensor(m).cuda() for m in aug.last_masks)
    res['spec_augment'] = row(run(lambda: ops.spec_augment_masked(g, tm, fm, 0.0, CL)), 2 * 4 * n_mel)
    g2 = torch.randn(B, T, N_MELS, 2, device='cuda')
    # algorithmic: the C = 1 channel read once, gx written once (the interleaved map channel is not needed)
    res['concat_frequency_map'] = row(run(lambda: ops.concat_frequency_map_backward(g2, CL)), 2 * 4 * n_mel)
    del g, g2

    x = torch.randn(B, L, 1, device='cuda')
    fr = K.Frame(frame_length=1024, hop_length=256, data_format=CL)
    gf = torch.randn_like(fr(x))
    res['frame_1024_256'] = row(run(lambda: ops.frame_backward(gf, 1024, 256, CL, L)), 4 * (gf.numel() + B * L))
    del gf
    en = K.Energy(sample_rate=SR, data_format=CL)
    ge = torch.randn_like(en(x))
    scale = en.ref_duration / (en.frame_length / en.sample_rate)
    res['energy_2205_1102'] = row(run(lambda: ops.energy_backward(x, ge, en.frame_length, en.hop_length, scale, CL)),
                                  4 * (2 * B * L + ge.numel()))

    xr = x.clone().requires_grad_(True)
    for db in (False, True):
        mp = K.get_stft_mag_phase(None, n_fft=N_FFT, hop_length=HOP, return_decibel=db, input_data_format=CL,
                                  output_data_format=CL)
        y = mp(xr)
        gy = torch.randn_like(y)
        S = mp.stft(x)
        gm, gp = gy[..., :1], gy[..., 1:]
        n_bins = S.numel()
        key = 'mag_phase_db' if db else 'mag_phase'

        def fwd():
            with torch.no_grad():
                mp(x)

        def fwd_bwd():
            torch.autograd.grad(mp(xr), xr, grad_outputs=gy)
        f_ms, fb_ms = run(fwd), run(fwd_bwd)
        res[key] = {'pass': row(run(lambda: ops.mag_phase_backward(S, gm, gp, CL)), n_bins * (8 + 4 + 4 + 8)),
                    'forward_ms': f_ms, 'forward_backward_ms': fb_ms, 'backward_ms': fb_ms - f_ms}
        del y, gy, S, gm, gp
    print(json.dumps(res), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'grad_adjacent_bench.json'), 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
