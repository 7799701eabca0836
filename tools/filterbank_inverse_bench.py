"""Times the filterbank inversion (kapre_b200.time_frequency.InverseFilterbank) with CUDA events and prints one JSON
line per case, with the card name and power limit read in the same run.

Cases (consistent mel input: the library's own mel of a harmonic tone plus noise, tiled over the batch):
  (a) the cfg2 mel shape (256, 427, 128, 1), 22.05 kHz, n_fft 1024, 128 mel: n_iter 32 and 100, both data formats;
  (b) 16 kHz speech, n_fft 400, 80 mel, (256, 601, 80, 1), n_iter 100;
  (c) n_fft 2048, 128 mel, (64, 431, 128, 1), n_iter 100.
For each: ms per call, frames/s, and per the counted work of one frame (init: nnz FMAs; per iteration: 2 nnz FMAs for
A y and A^T r plus 2 F for the gradient step and the momentum update, where nnz is the bank's nonzero count and F the
bins; HBM bytes: 4 (n_bands + F) read and written once), the achieved rates and the share of the larger of the two
bounds (H100 SXM data sheet: FP32 67 TFLOP/s, HBM3 3.35 TB/s).  A shared-memory model is printed beside them: per 32
frames and iteration, one 128-byte wavefront per warp access (padded band-dot reads, the m and r rows, the column-list
reads of r, and the reads and writes of s and y), against 128 B per clock per SM at the card's maximum SM clock.
Comparisons on the same GPU:
  (d) the same FISTA loop written as torch ops (dense float32 matmuls, allow_tf32 off) at the same n_iter;
  (e) torchaudio.transforms.InverseMelScale at the cfg2 shape (its error is recorded if it does not run on CUDA);
  (f) the whole get_inverse_melspectrogram_layer call at the cfg2 shape (32 Griffin-Lim iterations), split into its
      InverseFilterbank and GriffinLim parts timed alone.

    python tools/filterbank_inverse_bench.py [--steps 20] [--warmup 3] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

HBM_PEAK = 3.35e12      # H100 SXM data sheet, HBM3
FP32_PEAK = 67e12       # H100 SXM data sheet, dense FP32
CL, CF = 'channels_last', 'channels_first'


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = 'unknown'
    return name, q


def max_sm_clock_hz(q):
    try:
        return float(q.split(',')[1].strip().split()[0]) * 1e6
    except (IndexError, ValueError):
        return None


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


def mel_input(sr, n_fft, n_mels, B, T, fmt):
    """(B, T, M, 1) / (B, 1, T, M) mel of a tone, from the library's fused launch, tiled over the batch."""
    import kapre_b200
    hop = n_fft // 4
    L = (T - 1) * hop + n_fft
    t = np.arange(L) / sr
    x = sum(0.3 / k * np.sin(2 * np.pi * (k * 180.0 + 20 * np.sin(2 * np.pi * 0.7 * t)) * t) for k in range(1, 8))
    x = x + 0.01 * np.random.default_rng(0).standard_normal(L)
    xt = torch.from_numpy(x.astype(np.float32)).cuda().view(1, 1, L)
    mel = kapre_b200.get_melspectrogram_layer(n_fft=n_fft, hop_length=hop, sample_rate=sr, n_mels=n_mels,
                                              input_data_format=CF, output_data_format=fmt)(xt)
    assert mel.shape[1 if fmt == CL else 2] == T
    return mel.expand(B, *mel.shape[1:]).contiguous()


def counts(fb, n_iter):
    """(FMAs, HBM bytes, shared-memory wavefronts per 32 frames) of one frame, from the bank."""
    F, M = fb.shape
    nz = fb != 0
    nnz = int(nz.sum())
    padded = 0
    for m in range(M):
        idx = np.nonzero(nz[:, m])[0]
        if idx.size:
            padded += -(-(idx[-1] + 1 - idx[0]) // 4) * 4
    fmas = nnz + n_iter * (2 * nnz + 2 * F)
    hbm = 4 * (M + F)
    # per warp (32 frames): init: M m-writes + M r-writes + nnz r-reads + 2F writes; per iteration: padded y reads,
    # M m reads, M r writes, nnz r reads, 2F reads and 2F writes
    wavefronts = 2 * M + nnz + 2 * F + n_iter * (padded + 2 * M + nnz + 4 * F)
    return int(fmas), int(hbm), int(wavefronts)


def fista_torch(fb, n_iter):
    """The same loop as torch ops on (..., M) input, dense float32 matmuls."""
    A = torch.from_numpy(np.asarray(fb, np.float64).T.copy())
    step = float(1.0 / torch.linalg.matrix_norm(A, 2) ** 2)
    d = A @ (A.T @ torch.ones(A.shape[0], dtype=torch.float64))
    inv_d = torch.where(d > 0, 1.0 / d, torch.zeros_like(d)).float().cuda()
    A = A.float().cuda()
    coefs = []
    t = 1.0
    for _ in range(n_iter):
        tn = 0.5 * (1.0 + (1.0 + 4.0 * t * t) ** 0.5)
        coefs.append((t - 1.0) / tn)
        t = tn

    def run(m):
        s = torch.relu((m * inv_d) @ A)
        y = s
        for c in coefs:
            sn = torch.relu(y - step * ((y @ A.T - m) @ A))
            y = sn + c * (sn - s)
            s = sn
        return s
    return run


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    torch.backends.cuda.matmul.allow_tf32 = False
    from kapre_b200 import composed
    from kapre_b200.time_frequency import InverseFilterbank
    name, q = card()
    clk = max_sm_clock_hz(q)
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    smem_bw = 128.0 * n_sm * clk if clk else None
    lines = []

    def emit(d):
        d.update(gpu=name, power_limit_and_max_sm_clock=q)
        print(json.dumps(d), flush=True)
        lines.append(d)

    cases = [('cfg2', 22050, 1024, 128, 256, 427, fmt, n) for n in (32, 100) for fmt in (CL, CF)]
    cases += [('speech16k', 16000, 400, 80, 256, 601, CL, 100), ('nfft2048', 22050, 2048, 128, 64, 431, CL, 100)]
    for tag, sr, n_fft, M, B, T, fmt, n_iter in cases:
        kw = dict(sample_rate=sr, n_freq=n_fft // 2 + 1, n_mels=M)
        layer = InverseFilterbank('mel', kw, n_iter=n_iter, data_format=fmt)
        x = mel_input(sr, n_fft, M, B, T, fmt)
        with torch.no_grad():
            ms = timed(lambda: layer(x), a.steps, a.warmup)
            fmas, hbm, wf = counts(layer.filterbank, n_iter)
            frames = B * T
            flops = 2.0 * fmas * frames
            bytes_ = float(hbm) * frames
            s = ms * 1e-3
            bound = max(flops / FP32_PEAK, bytes_ / HBM_PEAK)
            d = dict(case=tag, shape=list(x.shape), data_format=fmt, n_iter=n_iter, ms=round(ms, 4),
                     frames_per_s=frames / s, fma_per_frame=fmas, hbm_bytes_per_frame=hbm,
                     tflops=flops / s / 1e12, hbm_gbps=bytes_ / s / 1e9,
                     bound='fp32' if flops / FP32_PEAK >= bytes_ / HBM_PEAK else 'hbm', share_of_bound=bound / s,
                     smem_wavefronts_per_32_frames=wf)
            if smem_bw:
                smem_s = wf * 128.0 * frames / 32 / smem_bw
                d.update(smem_model_ms=round(smem_s * 1e3, 4), share_of_smem_model=smem_s / s)
            if fmt == CL:
                ref = fista_torch(layer.filterbank, n_iter)
                xm = x[..., 0]
                d['torch_ops_ms'] = round(timed(lambda: ref(xm), max(2, a.steps // 4), 1), 4)
                got = layer(x)[..., 0]
                d['torch_ops_max_rel_diff'] = float((ref(xm) - got).abs().max() / got.abs().max())
            emit(d)
    # torchaudio's InverseMelScale at the cfg2 shape
    try:
        import torchaudio
        from kapre_b200 import backend
        fb = backend.filterbank_mel(sample_rate=22050, n_freq=513, n_mels=128)
        ims = torchaudio.transforms.InverseMelScale(n_stft=513, n_mels=128, sample_rate=22050).cuda()
        ims.fb.copy_(torch.from_numpy(fb).cuda())
        x = mel_input(22050, 1024, 128, 256, 427, CF)[:, 0].transpose(-1, -2).contiguous()     # (256, 128, 427)
        with torch.no_grad():
            ms = timed(lambda: ims(x), 2, 1)
        emit(dict(case='torchaudio_InverseMelScale_cfg2', shape=list(x.shape), ms=round(ms, 4)))
    except Exception as e:  # noqa: BLE001 - recorded, not hidden
        emit(dict(case='torchaudio_InverseMelScale_cfg2', error='%s: %s' % (type(e).__name__, str(e)[:300])))
    # the whole mel -> waveform factory at the cfg2 shape, and its two parts alone
    inv = composed.get_inverse_melspectrogram_layer(n_fft=1024, hop_length=256, sample_rate=22050, n_mels=128,
                                                    input_data_format=CL, output_data_format=CL)
    x = mel_input(22050, 1024, 128, 256, 427, CL)
    with torch.no_grad():
        ms_all = timed(lambda: inv(x), max(2, a.steps // 4), 1)
        lin = inv.layers[0](x)
        ms_nnls = timed(lambda: inv.layers[0](x), a.steps, a.warmup)
        ms_gl = timed(lambda: inv.layers[1](lin), max(2, a.steps // 4), 1)
    emit(dict(case='get_inverse_melspectrogram_layer_cfg2', shape=list(x.shape), nnls_iter=100, griffin_lim_iter=32,
              ms=round(ms_all, 4), inverse_filterbank_ms=round(ms_nnls, 4), griffin_lim_ms=round(ms_gl, 4)))
    if a.out:
        with open(a.out, 'w') as f:
            for d in lines:
                f.write(json.dumps(d) + '\n')


if __name__ == '__main__':
    main()
