"""HPSS timings on the GPU with CUDA events after warm-up.  Prints the card and its power limit, then one JSON line per
case with the time, the byte floor and the time's share of it, and the baselines: a chunked torch restatement on the
same GPU (``unfold`` + ``median`` for both medians and the harmonic mask; ``torch.median`` returns the lower median,
the same element as rank k // 2 for odd k) checked against the kernel's mask, and scipy's ``median_filter`` on this host's CPU (one
item, one core, scaled to the batch).

Byte model (arithmetic from shapes, not a measurement).  The forward reads S once and writes each requested output
once: at the default size (256 x 216 x 1025) complex64 in and both complex64 outputs is 24 B per element, 1.36 GB or
0.41 ms at 3.35 TB/s; magnitude in and both float32 outputs is 12 B, 0.68 GB or 0.20 ms.  A 64 x 64 tile also reads a
halo of (k_h - 1) frames x 64 bins and 64 frames x (k_p - 1) bins: at k = 31 that is 94 % of the tile again, read by
neighbouring tiles in flight at the same time, so mostly from L2 rather than HBM; the floor counts S once.  Complex
input is read a second time for M X (the tile's own elements, just loaded, so from L2).  The backward reads S, the two
output gradients and writes gS plus a 16 B per element workspace, which the gather pass reads once per element in
(2 k_h - 1) + (2 k_p - 1) neighbours (from L1/L2)."""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from kapre_b200 import signal  # noqa: E402

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


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                       text=True)
    return q.stdout.strip()


def spec(B, T, K, C, fmt, cplx, seed=0):
    g = torch.Generator(device='cuda').manual_seed(seed)
    shape = (B, T, K, C) if fmt == CL else (B, C, T, K)
    if cplx:
        return torch.complex(torch.randn(shape, generator=g, device='cuda'), torch.randn(shape, generator=g, device='cuda'))
    return torch.rand(shape, generator=g, device='cuda')


def _sym_pad(x, h):
    """Pad the last axis by h on each side with the edge repeated (scipy's 'reflect'; torch's 'reflect' omits it)."""
    return torch.cat([x[..., :h].flip(-1), x, x[..., -h:].flip(-1)], dim=-1)


def torch_hpss(S, k=31, chunk=8):
    """(B, C, T, K) float32 magnitudes -> the harmonic mask at power 2, margins 1, chunked over the batch."""
    outs = []
    h = k // 2
    for i in range(0, S.shape[0], chunk):
        s = S[i:i + chunk]
        st = _sym_pad(s.flatten(0, 1).transpose(1, 2), h)
        H = st.unfold(-1, k, 1).median(dim=-1).values.transpose(1, 2).reshape(s.shape)
        sp = _sym_pad(s.flatten(0, 1), h)
        P = sp.unfold(-1, k, 1).median(dim=-1).values.reshape(s.shape)
        z = torch.maximum(H, P).clamp_min(torch.finfo(torch.float32).tiny)
        a, b = (H / z) ** 2, (P / z) ** 2
        outs.append(a / (a + b))
    return torch.cat(outs)


def report(name, ms, floor_bytes, extra=None):
    floor_ms = floor_bytes / HBM * 1e3
    r = dict(case=name, ms=round(ms, 4), floor_ms=round(floor_ms, 4), share_of_floor=round(floor_ms / ms, 3))
    r.update(extra or {})
    print(json.dumps(r), flush=True)
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    print('card:', card(), flush=True)
    rows = []
    B, T, K = 256, 216, 1025
    n = B * T * K

    X = spec(B, T, K, 1, CF, True)
    ms = timed(lambda: signal.hpss(X, data_format=CF), a.warmup, a.steps)
    from kapre_b200 import ops
    from kapre_b200.time_frequency import HPSS
    mag = ops.magnitude(X)
    tms = timed(lambda: torch_hpss(mag), 1, 2)
    ref = torch_hpss(mag[:8])
    got = signal.hpss(mag[:8], mask=True, data_format=CF)[0]
    agree = float((ref - got).abs().max())
    try:
        import scipy.ndimage
        m0 = mag[0, 0].cpu().numpy()
        t0 = time.perf_counter()
        scipy.ndimage.median_filter(m0, size=(31, 1), mode='reflect')
        scipy.ndimage.median_filter(m0, size=(1, 31), mode='reflect')
        scipy_ms = (time.perf_counter() - t0) * 1e3 * B
    except ImportError:
        scipy_ms = None
    rows.append(report('defaults 256 x 5 s 22.05 kHz, complex in, both outputs', ms, 24 * n,
                       dict(torch_unfold_median_ms=round(tms, 2), torch_max_abs_diff=agree,
                            scipy_cpu_one_core_ms_scaled_to_batch=scipy_ms)))
    ms = timed(lambda: signal.hpss(mag, data_format=CF), a.warmup, a.steps)
    rows.append(report('defaults, magnitude in, both outputs', ms, 12 * n))
    ms = timed(lambda: signal.hpss(X, kernel_size=(17, 63), data_format=CF), a.warmup, a.steps)
    rows.append(report('kernel_size=(17, 63), complex in, both outputs', ms, 24 * n))
    del mag

    T2 = 10 * 44100 // 512 + 1
    M2 = spec(64, T2, K, 2, CL, False)
    ms = timed(lambda: signal.hpss(M2, data_format=CL)[0], a.warmup, a.steps)
    layer = HPSS('harmonic', data_format=CL)
    ms1 = timed(lambda: layer(M2), a.warmup, a.steps)
    rows.append(report('64 x 10 s 44.1 kHz stereo channels_last, magnitude in, both outputs', ms, 12 * M2.numel()))
    rows.append(report('the same, harmonic only (HPSS layer)', ms1, 8 * M2.numel()))
    del M2

    T3 = 600 * 22050 // 512 + 1
    X3 = spec(1, T3, K, 1, CF, True)
    ms = timed(lambda: signal.hpss(X3, data_format=CF), a.warmup, a.steps)
    rows.append(report('one 10-minute recording, complex in, both outputs', ms, 24 * X3.numel()))
    del X3

    y = torch.randn((B, 5 * 22050, 1), device='cuda') * 0.1
    ms = timed(lambda: signal.harmonic(y, data_format=CL), a.warmup, a.steps)
    rows.append(report('harmonic() end to end, 256 x 5 s (STFT + HPSS + inverse)', ms, 4 * y.numel() * 2 + 16 * n,
                       dict(note='floor: waveform in and out plus the complex spectrum written, read and written')))
    del y

    Xg = X.clone().requires_grad_(True)

    def fwd_bwd():
        h, p = signal.hpss(Xg, data_format=CF)
        torch.autograd.backward((h, p), (X, X))
    ms = timed(fwd_bwd, a.warmup, a.steps)
    rows.append(report('forward + backward at the defaults, complex', ms, 24 * n + (8 * 3 + 32) * n))
    if a.out:
        os.makedirs(os.path.dirname(a.out), exist_ok=True)
        with open(a.out, 'w') as f:
            json.dump(dict(card=card(), rows=rows), f, indent=1)


if __name__ == '__main__':
    main()
