"""Onset, tempogram, tempo, peak-picking and beat-tracking timings on the GPU with CUDA events after warm-up.  Prints
the card and its power limit (read in the same run), then one JSON line per case with the time and, where one is
defined, its floor, and the baselines: a torch restatement on the same GPU (onset: diff, relu and mean / median;
tempogram: ``unfold`` plus an FFT autocorrelation) checked against the kernels, and the numpy/scipy restatement of
``tests/rhythm_ref.py`` on one CPU core for one item (onset, tempogram and the beat DP's per-frame loop), scaled to
the batch.

Floors (arithmetic from shapes, not measurements).  Onset strength from S reads S once and writes the envelope:
at 256 x 216 x 128 float32 that is 28 MB, under 10 us at 3.35 TB/s.  The tempogram is W (W + 1) / 2 FMAs per frame:
at 256 x 216 frames and W = 384 that is 8.2 GFLOP, 0.12 ms at 67 TFLOP/s FP32."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
from kapre_b200 import signal  # noqa: E402
import rhythm_ref as R  # noqa: E402

HBM = 3.35e12
FP32 = 67e12
CF, CL = 'channels_first', 'channels_last'


def timed(fn, warmup, steps):
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


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                       text=True)
    return q.stdout.strip()


def wave(B, C, L, sr, fmt, seed=0):
    rng = np.random.default_rng(seed)
    x = 0.05 * rng.standard_normal((B, C, L))
    per = int(0.5 * sr)
    for k in range(0, L, per):
        x[:, :, k:k + 200] += np.hanning(400)[200:]
    x = x.astype(np.float32)
    return torch.from_numpy(x if fmt == CF else np.ascontiguousarray(x.transpose(0, 2, 1))).cuda()


def torch_onset(S, agg):
    """diff, relu and mean / median over bins of a (B, C, T, K) spectrogram (lag 1, max_size 1, centred at 2048/512)."""
    D = torch.relu(S[:, :, 1:] - S[:, :, :-1])
    if agg == 'mean':
        A = D.double().mean(-1).float()
    else:
        s = D.sort(-1).values
        K = S.shape[-1]
        A = s[..., (K - 1) // 2] if K % 2 else 0.5 * (s[..., K // 2 - 1] + s[..., K // 2])
    out = torch.zeros(S.shape[:3], device=S.device)
    out[:, :, 3:] = A[:, :, :S.shape[2] - 3]
    return out


def torch_tempogram(e, W):
    """unfold of the linear-ramp padded (B, C, T) envelope and an FFT autocorrelation, norm = inf."""
    c = W // 2
    T = e.shape[-1]
    k = torch.arange(c, device=e.device, dtype=torch.float64)
    left = e[..., :1].double() * k / c
    right = e[..., -1:].double() * (c - torch.arange(1, c + 1, device=e.device, dtype=torch.float64)) / c
    ep = torch.cat([left.float(), e, right.float()], -1)
    fr = ep.unfold(-1, W, 1)[..., :T, :] * torch.hann_window(W, periodic=True, device=e.device)
    F = torch.fft.rfft(fr, n=2 * W)
    ac = torch.fft.irfft(F.abs() ** 2, n=2 * W)[..., :W]
    mx = ac.abs().amax(-1, keepdim=True)
    return torch.where(mx >= 1.1754944e-38, ac / mx, ac)


def cpu_time(fn, reps=1):
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    return (time.perf_counter() - t0) / reps * 1e3


def case(name, B, C, seconds, sr, fmt, warmup, steps, cpu):
    hop = 512
    w = wave(B, C, int(seconds * sr), sr, fmt)
    S = signal._onset_feature(w, sr, 2048, hop, 128, 0.0, None, fmt)
    Sc = S.permute(0, 3, 1, 2).contiguous() if fmt == CL else S
    T, K = Sc.shape[2], Sc.shape[3]
    rows = B * C
    res = dict(case=name, batch=B, channels=C, seconds=seconds, sr=sr, layout=fmt, frames=T)
    with torch.no_grad():
        for agg in ('mean', 'median'):
            ms = timed(lambda: signal.onset_strength(S=S, sample_rate=sr, aggregate=agg, data_format=fmt), warmup,
                       steps)
            floor = (S.numel() * 4 + rows * T * 4) / HBM * 1e3
            res['onset_%s_from_S_ms' % agg] = round(ms, 4)
            res['onset_%s_floor_ms' % agg] = round(floor, 4)
            e = signal.onset_strength(S=S, sample_rate=sr, aggregate=agg, data_format=fmt)
            ec = e.permute(0, 2, 1) if fmt == CL else e
            ref = torch_onset(Sc, agg)
            res['onset_%s_torch_ms' % agg] = round(timed(lambda: torch_onset(Sc, agg), warmup, steps), 4)
            res['onset_%s_torch_max_abs_diff' % agg] = float((ref - ec).abs().max())
        res['onset_from_waveform_ms'] = round(timed(lambda: signal.onset_strength(w, sample_rate=sr, data_format=fmt),
                                                    warmup, steps), 4)
        e = signal.onset_strength(S=S, sample_rate=sr, data_format=fmt)
        ec = e.permute(0, 2, 1).contiguous() if fmt == CL else e
        W = 384
        res['tempogram_ms'] = round(timed(lambda: signal.tempogram(onset_envelope=e, sample_rate=sr,
                                                                   data_format=fmt), warmup, steps), 4)
        flop = rows * T * W * (W + 1)
        res['tempogram_gflop'] = round(flop / 1e9, 3)
        res['tempogram_floor_ms'] = round(flop / FP32 * 1e3, 4)
        tg = signal.tempogram(onset_envelope=e, sample_rate=sr, data_format=fmt)
        tgc = tg.permute(0, 3, 1, 2) if fmt == CL else tg
        res['tempogram_torch_ms'] = round(timed(lambda: torch_tempogram(ec, W), warmup, steps), 4)
        res['tempogram_torch_max_abs_diff'] = float((torch_tempogram(ec, W) - tgc).abs().max())
        res['tempo_ms'] = round(timed(lambda: signal.tempo(onset_envelope=e, sample_rate=sr, data_format=fmt),
                                      warmup, steps), 4)
        res['onset_detect_ms'] = round(timed(lambda: signal.onset_detect(onset_envelope=e, sample_rate=sr,
                                                                         data_format=fmt), warmup, steps), 4)
        res['beat_track_ms'] = round(timed(lambda: signal.beat_track(onset_envelope=e, sample_rate=sr,
                                                                     data_format=fmt), warmup, steps), 4)
        res['beat_track_fixed_bpm_ms'] = round(timed(lambda: signal.beat_track(onset_envelope=e, sample_rate=sr,
                                                                               bpm=120.0, data_format=fmt),
                                                     warmup, steps), 4)
        res['beat_track_from_waveform_ms'] = round(timed(lambda: signal.beat_track(w, sample_rate=sr,
                                                                                   data_format=fmt), warmup, steps), 4)
        if cpu:
            S0 = Sc[0, 0].cpu().numpy()
            e0 = ec[0, 0].cpu().numpy()
            res['cpu_onset_ms_per_item'] = round(cpu_time(lambda: R.onset_strength_row(S0, 1, 1, 'mean', 2)), 3)
            res['cpu_tempogram_ms_per_item'] = round(cpu_time(lambda: R.tempogram_row(e0, W)), 3)
            tempo, beats = signal.beat_track(onset_envelope=e, sample_rate=sr, bpm=120.0, data_format=fmt)
            p = R.period(120.0, sr, hop)
            ls = R.local_score(e0, p)
            res['cpu_beat_dp_ms_per_item'] = round(cpu_time(lambda: R.beat_dp(ls, p)), 3)
            cs, back = R.beat_dp(ls, p)
            bm = (beats.permute(0, 2, 1) if fmt == CL else beats)[0, 0].cpu().numpy()
            res['beat_dp_agrees'] = bool(np.array_equal(np.nonzero(bm)[0], R.beats_from(ls, cs, back)))
            res['cpu_scaled_to_batch_ms'] = round((res['cpu_onset_ms_per_item'] + res['cpu_tempogram_ms_per_item']
                                                   + res['cpu_beat_dp_ms_per_item']) * rows, 1)
    print(json.dumps(res), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--no-cpu', action='store_true')
    a = ap.parse_args()
    print(json.dumps({'card': card()}), flush=True)
    case('256x5s_22k', 256, 1, 5.0, 22050, CF, a.warmup, a.steps, not a.no_cpu)
    case('64x10s_48k_stereo', 64, 2, 10.0, 48000, CL, a.warmup, a.steps, not a.no_cpu)
    case('1x600s_22k', 1, 1, 600.0, 22050, CF, a.warmup, max(3, a.steps // 4), not a.no_cpu)


if __name__ == '__main__':
    main()
