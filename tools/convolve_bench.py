"""Partitioned FFT convolution (``kapre_convolve``) on 256 x 5 s at 16 kHz: forward, backward to x, backward to x and
h, the time of each forward phase (STFT, per-bin multiply-accumulate, inverse STFT) from torch.profiler kernel
records, each phase's algorithmic bytes and its share of 3.35 TB/s, and the torch route on the same card
(``torchaudio.functional.fftconvolve`` when importable, else ``torch.fft.rfft`` / ``irfft`` at n = L + K - 1).

    python tools/convolve_bench.py [--out DIR] [--iters N]

Prints one JSON line per configuration and then a Markdown table, which is also written to DIR/convolve_bench.md when
--out is given.  The card's name and power limit are read in the same run."""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from kapre_b200 import ops  # noqa: E402

HBM = 3.35e12
BATCH, SR, SECONDS = 256, 16000, 5
KS = (256, 2000, 16000, 48000)


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


def _phases(fn, iters):
    """Mean kernel time per call (ms) of the STFT, the MAC and the inverse, from torch.profiler's CUDA records."""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fn()
        torch.cuda.synchronize()
    t = {'stft': 0.0, 'mac': 0.0, 'inverse': 0.0, 'filter': 0.0}
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        name = ev.name
        us = ev.device_time if hasattr(ev, 'device_time') else ev.cuda_time
        if 'kb_spec_conv_kernel' in name:
            t['mac'] += us
        elif 'istft' in name or 'idft' in name:
            t['inverse'] += us
        elif 'kb_stft' in name or 'kb_mr' in name or 'kb_dft' in name:
            t['stft'] += us
    return {k: v / iters / 1000.0 for k, v in t.items() if k != 'filter'}


def _torch_route():
    try:
        import torchaudio.functional as AF
        return 'torchaudio.functional.fftconvolve', lambda x, h: AF.fftconvolve(x, h)
    except Exception:
        def fft(x, h):
            n = x.shape[-1] + h.shape[-1] - 1
            return torch.fft.irfft(torch.fft.rfft(x, n=n) * torch.fft.rfft(h, n=n), n=n)
        return 'torch.fft.rfft/irfft at n = L + K - 1', fft


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
    ap.add_argument('--iters', type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('convolve_bench needs a GPU')
    card, power = _card()
    route_name, route = _torch_route()
    L = SR * SECONDS
    rows = []
    for fmt, C in (('channels_first', 1), ('channels_last', 2)):
        g = torch.Generator(device='cuda').manual_seed(0)
        shape = (BATCH, C, L) if fmt == 'channels_first' else (BATCH, L, C)
        x = torch.rand(shape, device='cuda', generator=g) * 2 - 1
        for K in KS:
            h = torch.randn(K, device='cuda', generator=g) * torch.exp(-torch.arange(K, device='cuda') / (K / 4.0))
            blk = ops.convolve_block_size(K)
            plan = ops.convolve_plan(blk)
            h3 = h.view(1, 1, K) if fmt == 'channels_first' else h.view(1, K, 1)
            H = ops.convolve_ir_spectrum(h3, plan, fmt)
            P = H.shape[2]
            J = -(-L // blk)
            T = J + P - 1
            F = blk + 1

            def fwd():
                return ops.convolve_spectrum(x, H, plan, 0, L + K - 1, fmt)

            fwd_ms = _time(fwd, args.iters)
            by_block = {}
            if fmt == 'channels_first':          # what the block-size rule weighs: the forward at every B
                for b in (128, 256, 512, 1024):
                    pb = ops.convolve_plan(b)
                    Hb = ops.convolve_ir_spectrum(h3, pb, fmt)
                    by_block[b] = _time(lambda: ops.convolve_spectrum(x, Hb, pb, 0, L + K - 1, fmt), args.iters)
            full_ms = _time(lambda: ops.convolve(x, h, 'full', fmt), args.iters)
            xg = x.clone().requires_grad_(True)
            hg = h.clone().requires_grad_(True)
            y = ops.convolve(xg, h, 'full', fmt)
            gy = torch.randn(y.shape, device='cuda', generator=g)
            bwd_x_ms = _time(lambda: torch.autograd.grad(ops.convolve(xg, h, 'full', fmt), (xg,), gy), args.iters) \
                - full_ms
            bwd_xh_ms = _time(lambda: torch.autograd.grad(ops.convolve(xg, hg, 'full', fmt), (xg, hg), gy),
                              args.iters) - full_ms
            ph = _phases(fwd, args.iters)
            sig = BATCH * C
            nbytes = {'stft': sig * L * 4 + sig * J * F * 8,
                      'mac': sig * J * F * 8 + P * F * 8 + sig * T * F * 8,
                      'inverse': sig * T * F * 8 + sig * (T + 1) * blk * 4}
            xt = x if fmt == 'channels_first' else x.transpose(1, 2).contiguous()
            ref_ms = _time(lambda: route(xt, h.expand(1, 1, K)), args.iters)
            row = {'format': fmt, 'channels': C, 'K': K, 'B': blk, 'P': P, 'forward_ms': fwd_ms,
                   'forward_with_filter_ms': full_ms, 'forward_ms_by_block': by_block, 'backward_x_ms': bwd_x_ms, 'backward_x_h_ms': bwd_xh_ms,
                   'phase_ms': ph, 'phase_bytes': nbytes,
                   'phase_hbm_share': {k: nbytes[k] / (ph[k] * 1e-3) / HBM if ph[k] > 0 else None for k in nbytes},
                   'torch_route': route_name, 'torch_route_ms': ref_ms, 'card': card, 'power_limit': power}
            print(json.dumps(row), flush=True)
            rows.append(row)
            del xg, hg, y, gy
    lines = ['%s, power limit %s; %d x %d s at %d Hz; torch route: %s' % (card, power, BATCH, SECONDS, SR, route_name), '',
             '| format | K | B | P | forward ms | +filter ms | bwd x ms | bwd x,h ms | STFT ms (HBM %) | '
             'MAC ms (HBM %) | inverse ms (HBM %) | torch ms |', '|' + '---|' * 12]
    for r in rows:
        ph, sh = r['phase_ms'], r['phase_hbm_share']
        lines.append('| %s x%d | %d | %d | %d | %.3f | %.3f | %.3f | %.3f | %.3f (%.0f%%) | %.3f (%.0f%%) | '
                     '%.3f (%.0f%%) | %.3f |' % (r['format'], r['channels'], r['K'], r['B'], r['P'], r['forward_ms'],
                                                 r['forward_with_filter_ms'], r['backward_x_ms'], r['backward_x_h_ms'],
                                                 ph['stft'], 100 * (sh['stft'] or 0), ph['mac'], 100 * (sh['mac'] or 0),
                                                 ph['inverse'], 100 * (sh['inverse'] or 0), r['torch_route_ms']))
    table = '\n'.join(lines) + '\n'
    print(table)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'convolve_bench.md'), 'w') as f:
            f.write(table)

if __name__ == '__main__':
    main()
