"""Chroma timings on the GPU with CUDA events after warm-up, against a PyTorch restatement on the same device
(torch.stft, an einsum with the same filterbank and the normalisation; torch.median and torch.histc for the tuning
estimate), each checked against the kernels in the same run.  Prints the card and its power limit, then one JSON line
per case, and with --profile the kernel time of each launch from torch.profiler (a separate run).

Byte model of the new launches (arithmetic from shapes, not a measurement).  The projection reads its input once
and writes n_chroma floats per frame: at the chroma_stft default (256 x 5 s at 22.05 kHz, n_fft 2048, hop 512) |X|
is 256 x 216 x 1025 float32 = 227 MB, a 68 us floor at 3.35 TB/s.  The tuning estimate's peak pass reads S once more
(68 us) and writes two floats per peak slot (179 slots per frame: 79 MB), and each of its five selection passes reads
the mags (40 MB, the fifth also the pitches).  chroma_cqt's projection reads |C| (256 x 216 x 252 floats, 56 MB,
17 us) after the CQT's own launches, which this work does not change."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from kapre_b200 import backend, ops, signal  # noqa: E402

HBM = 3.35e12
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


def waveform(B, C, L, sr, seed, fmt):
    g = torch.Generator().manual_seed(seed)
    t = torch.arange(L, dtype=torch.float64) / sr
    x = 0.01 * torch.randn((B, C, L), generator=g, dtype=torch.float64)
    f = 110.0 * 2.0 ** (torch.randint(0, 36, (B, 3), generator=g) / 12.0 + torch.rand((B, 3), generator=g) * 0.05)
    for i in range(3):
        x += 0.3 * torch.sin(2 * np.pi * f[:, i, None, None] * t)
    x = x.float().cuda()
    return x.transpose(1, 2).contiguous() if fmt == CL else x


def torch_stft_power(x, n_fft, hop, fmt):
    """(B, C, M, K) power spectrogram by torch.stft (centred, zero padding, periodic Hann)."""
    xc = x.transpose(1, 2) if fmt == CL else x
    B, C, L = xc.shape
    X = torch.stft(xc.reshape(B * C, L), n_fft, hop, window=torch.hann_window(n_fft, device=x.device), center=True,
                   pad_mode='constant', return_complex=True)
    return (X.abs() ** 2).reshape(B, C, X.shape[-2], X.shape[-1]).transpose(2, 3)


def torch_normalize(y, norm):
    a = y.abs()
    n = a.max(-1, keepdim=True).values if norm == np.inf else a.pow(norm).sum(-1, keepdim=True).pow(1.0 / norm)
    return y / torch.where(n < 1.1754944e-38, torch.ones_like(n), n)


def torch_tuning(S, sr, n_fft, resolution=0.01, bpo=12):
    """Per-item tuning by piptrack, torch.median and torch.histc (one item at a time: the peak sets differ)."""
    lo, hi = backend.piptrack_bins(sr, n_fft)
    out = []
    for b in range(S.shape[0]):
        s = S[b]
        ok = torch.isfinite(s).all(-1, keepdim=True)
        ref = 0.1 * s.max(-1, keepdim=True).values
        sp = s * (s > ref)
        k = torch.arange(lo, hi, device=S.device)
        c, l, r = s[..., k], s[..., k - 1], s[..., k + 1]
        pk = (c > ref) & (sp[..., k] > sp[..., k - 1]) & (sp[..., k] >= sp[..., k + 1]) & ok
        a = 0.5 * (r - l)
        d = 2 * c - r - l
        sh = torch.where(d.abs() < 1.1754944e-38, torch.zeros_like(d), a / d)
        pitch = ((k + sh) * sr / n_fft)[pk]
        mag = (c + 0.5 * a * sh)[pk]
        if mag.numel() == 0:
            out.append(0.0)
            continue
        srt = torch.sort(mag).values
        n = srt.numel()
        med = srt[n // 2] if n % 2 else 0.5 * (srt[n // 2 - 1] + srt[n // 2])
        p = pitch[mag >= med].double()
        res = torch.remainder(bpo * torch.log2(p / 27.5), 1.0)
        res = torch.where(res >= 0.5, res - 1.0, res)
        nb = int(np.ceil(1.0 / resolution))
        h = torch.histc(res, nb, -0.5, 0.5)
        out.append(float(np.linspace(-0.5, 0.5, nb + 1)[int(h.argmax())]))
    return torch.tensor(out, dtype=torch.float64)


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                       text=True)
    return q.stdout.strip()


def case_stft(name, B, C, secs, sr, fmt, tuning, warmup, steps):
    L = int(secs * sr)
    x = waveform(B, C, L, sr, 0, fmt)
    n_fft, hop = 2048, 512
    W = torch.from_numpy(backend.chroma_filterbank(sr, n_fft, tuning=0.0 if tuning is None else tuning)).float().cuda()

    def ours():
        return signal.chroma_stft(x, sample_rate=sr, tuning=tuning, data_format=fmt)

    def base():
        S = torch_stft_power(x, n_fft, hop, fmt)
        return torch_normalize(torch.einsum('bcmk,jk->bcmj', S, W), np.inf)
    got = ours()
    got_cf = got.permute(0, 3, 1, 2) if fmt == CL else got
    if tuning is not None:
        err = float((got_cf - base()).abs().max())
        assert err < 2e-3, err
    else:
        S = torch_stft_power(x, n_fft, hop, fmt)
        t_ref = torch_tuning(S[:8], sr, n_fft)
        t_got = signal.estimate_tuning(S=(S.permute(0, 2, 3, 1) if fmt == CL else S).contiguous()[:8], sample_rate=sr,
                                       data_format=fmt).cpu()
        assert float((t_ref - t_got).abs().max()) <= 0.011, (t_ref, t_got)
    xg = x.clone().requires_grad_(True)

    def fwd_bwd():
        out = signal.chroma_stft(xg, sample_rate=sr, tuning=tuning, data_format=fmt)
        out.backward(torch.ones_like(out))
    M = 1 + L // hop
    K = n_fft // 2 + 1
    mag_bytes = B * C * M * K * 4
    r = dict(case=name, forward_ms=timed(ours, warmup, steps), fwd_bwd_ms=timed(fwd_bwd, warmup, steps),
             baseline_ms=timed(base, warmup, steps), mag_MB=mag_bytes / 1e6, mag_read_floor_us=mag_bytes / HBM * 1e6)
    return r


def case_cqt(name, B, C, secs, sr, fmt, cens, warmup, steps):
    L = int(secs * sr)
    x = waveform(B, C, L, sr, 1, fmt)
    cqt, _ = signal._cqt_chroma_plans(sr, 512, None, 0.0, 12, 7, 36, True, False)
    Mq = torch.from_numpy(backend.cq_to_chroma(252, 36, 12)).float().cuda()
    fn = signal.chroma_cens if cens else signal.chroma_cqt

    def ours():
        return fn(x, sample_rate=sr, data_format=fmt)

    def cqt_only():
        return ops.cqt(x, cqt, fmt, fmt, True)

    def base():
        Cm = cqt_only()
        Cm = Cm.permute(0, 3, 1, 2) if fmt == CL else Cm
        return torch_normalize(torch.einsum('bcmk,jk->bcmj', Cm, Mq), np.inf)
    if not cens:
        got = ours()
        got = got.permute(0, 3, 1, 2) if fmt == CL else got
        assert float((got - base()).abs().max()) < 2e-3
    r = dict(case=name, forward_ms=timed(ours, warmup, steps), cqt_ms=timed(cqt_only, warmup, steps),
             baseline_ms=timed(base, warmup, steps))
    if not cens:
        xg = x.clone().requires_grad_(True)

        def fwd_bwd():
            out = fn(xg, sample_rate=sr, data_format=fmt)
            out.backward(torch.ones_like(out))
        r['fwd_bwd_ms'] = timed(fwd_bwd, warmup, steps)
    M = 1 + L // 512
    r['cqt_mag_MB'] = B * C * M * 252 * 4 / 1e6
    return r


def profile(out_dir):
    """Kernel time per launch name from torch.profiler at the chroma_stft default with tuning=None and chroma_cens."""
    from torch.profiler import ProfilerActivity, profile as tprof
    x = waveform(256, 1, 5 * 22050, 22050, 0, CF)
    for _ in range(3):
        signal.chroma_stft(x, data_format=CF)
        signal.chroma_cens(x, data_format=CF)
    torch.cuda.synchronize()
    with tprof(activities=[ProfilerActivity.CUDA]) as p:
        for _ in range(10):
            signal.chroma_stft(x, data_format=CF)
            signal.chroma_cens(x, data_format=CF)
        torch.cuda.synchronize()
    rows = {}
    for e in p.key_averages():
        if e.device_type.name == 'CUDA' and e.count:
            rows[e.key] = (e.count, getattr(e, 'device_time_total', getattr(e, 'cuda_time_total', 0.0)) / e.count)
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, 'chroma_profile.json'), 'w') as f:
        json.dump(rows, f, indent=1)
    for k, (n, us) in sorted(rows.items(), key=lambda kv: -kv[1][1]):
        print(json.dumps(dict(kernel=k[:80], launches=n, us_per_launch=round(us, 2))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--profile', default=None, help='directory for the torch.profiler table (a separate run)')
    a = ap.parse_args()
    print('card:', card())
    if a.profile:
        profile(a.profile)
        return
    w, s = a.warmup, a.steps
    for r in (case_stft('chroma_stft defaults, tuning 0.0, 256 x 5 s', 256, 1, 5, 22050, CF, 0.0, w, s),
              case_stft('chroma_stft defaults, tuning None, 256 x 5 s', 256, 1, 5, 22050, CF, None, w, s),
              case_cqt('chroma_cqt defaults, 256 x 5 s', 256, 1, 5, 22050, CF, False, w, s),
              case_cqt('chroma_cens defaults, 256 x 5 s', 256, 1, 5, 22050, CF, True, w, s),
              case_stft('chroma_stft 44.1 kHz stereo channels_last, 64 x 10 s', 64, 2, 10, 44100, CL, 0.0, w, s),
              case_stft('chroma_stft one 10-minute recording, tuning None', 1, 1, 600, 22050, CF, None, w, s)):
        print(json.dumps({k: (round(v, 3) if isinstance(v, float) else v) for k, v in r.items()}), flush=True)


if __name__ == '__main__':
    main()
