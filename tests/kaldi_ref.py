"""Float64 restatement of torchaudio.compliance.kaldi's fbank / mfcc / spectrogram for a batch: every channel, an
item's own length (reflection at its own end, its own mean for subtract_mean, zero frames past its count), and an
injected dither noise instead of torch.randn.  Differentiable through torch autograd, so it also gives the reference
VJPs; it is held against torchaudio itself in test_kaldi_emu.py.

Error bound of the float32 kernel (log domain), with u = 2^-24, n = log2(N) and E_f the frame's energy of the raw
(dithered) samples, sum x_i^2:
  the preprocessing (mean, pre-emphasis, window, each a few roundings per sample, the mean's float64 sum exact to
  u) perturbs the frame by at most 8 u |x_i| per sample; the radix-2 register FFT with float32 twiddles adds
  ||dX|| <= (n + 2) * 6.7 u ||X|| (Higham, Thm 24.2, eta = u + gamma_4 (sqrt 2 + u)); ||X||^2 <= N ||x||^2, so the
  power error sum_k |dS_k| <= 2 ||X|| ||dX|| + ||dX||^2 <= 2 N E_f (6.7 (n + 2) + 8) u (1 + 1e-3) and every band
  (weights <= 1) and bin of S moves by at most that much;
  the band sum adds len_m u m; log adds 2 u |log m| + u.  So
      |d log m| <= C_K N E_f u (n + 3) / max(m, eps) + (len + 2) u (1 + |log m|),   C_K = 2 * 15 = 30,
  and the same with m = S_k for the spectrogram, and with the energy's own sum for the energy column
  (|d log E| <= 16 W u).  For magnitudes (use_power=False) the power bound is taken through sqrt:
  |dS| <= sqrt(|dS^2|).  MFCC sums the band errors through the DCT: |dc| <= sum_m |D_mc| |d log m|.
"""
import math

import numpy as np
import torch

from kapre_b200 import backend

EPS = float(np.finfo(np.float32).eps)
LOG_EPS32 = float(np.float32(math.log(EPS)))


def src_index(j, length, pad):
    s = j - pad
    return np.where(s < 0, -1 - s, np.where(s < length, s, 2 * length - 1 - s))


def _mix(z):
    z = (z + np.uint64(0x9E3779B97F4A7C15)) & np.uint64(0xFFFFFFFFFFFFFFFF)
    z = ((z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)) & np.uint64(0xFFFFFFFFFFFFFFFF)
    z = ((z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)) & np.uint64(0xFFFFFFFFFFFFFFFF)
    return z ^ (z >> np.uint64(31))


def gauss(seed, b, c, f, n):
    """The kernel's dither values for samples 0..n-1 of frame f of (item b, channel c), unit variance, float32."""
    with np.errstate(over='ignore'):
        h = _mix(np.uint64(seed))
        h = _mix(h ^ np.uint64(b))
        h = _mix(h ^ np.uint64(c))
        h = _mix(h ^ np.uint64(f))
        i = np.arange(n, dtype=np.uint64)
        s = np.zeros(n, np.int64)
        for r in range(6):
            u = _mix(h ^ (np.uint64(6) * i + np.uint64(r)))
            s += (u >> np.uint64(40)).astype(np.int64) + ((u >> np.uint64(16)) & np.uint64(0xFFFFFF)).astype(np.int64)
    n_int = 2 * s - 12 * 0xFFFFFF
    return n_int.astype(np.float32) * np.float32(2.0 ** -25)


def plan_of(kind, o):
    W, H, Np = backend.kaldi_window_properties(o['sample_frequency'], o['frame_shift'], o['frame_length'],
                                               o['round_to_power_of_two'])
    min_len = int(math.ceil(o['min_duration'] * o['sample_frequency'])) if o['min_duration'] > 0 else 0
    return W, H, Np, min_len


def features(kind, x, o, lengths=None, noise=None):
    """x: (B, C, L) float64 torch tensor; o: options as kapre_b200.ops.kaldi_options gives them; noise: callable
    (b, c, f, W) -> W float32 values scaled by dither, or None.  Returns (B, C, T, K) float64."""
    W, H, Np, min_len = plan_of(kind, o)
    B, C, L = x.shape
    lens = [L] * B if lengths is None else [int(v) for v in lengths]
    Tb = [backend.kaldi_num_frames(l, W, H, o['snip_edges'], min_len) for l in lens]
    T = max(Tb) if B else 0
    win = torch.from_numpy(backend.kaldi_window(o['window_type'], W, o['blackman_coeff']))
    outs = []
    for b in range(B):
        rows = []
        for c in range(C):
            rows.append(_one(kind, x[b, c], lens[b], Tb[b], T, W, H, Np, win, o,
                             (lambda f, b=b, c=c: noise(b, c, f, W)) if noise is not None else None))
        outs.append(torch.stack(rows))
    return torch.stack(outs)


def _one(kind, x, length, Tb, T, W, H, Np, win, o, noise):
    K = (o['num_mel_bins'] + int(o['use_energy'])) if kind == 'fbank' else (
        o['num_ceps'] if kind == 'mfcc' else Np // 2 + 1)
    if Tb == 0:
        return torch.zeros((T, K), dtype=torch.float64) + 0.0 * x.sum()
    pad = 0 if o['snip_edges'] else W // 2 - H // 2
    j = np.arange(Tb)[:, None] * H + np.arange(W)[None, :]
    idx = torch.from_numpy(src_index(j, length, pad) if not o['snip_edges'] else j)
    fr = x[idx]
    if noise is not None:
        fr = fr + torch.from_numpy(np.stack([noise(f) for f in range(Tb)]).astype(np.float64))
    if o['remove_dc_offset']:
        fr = fr - fr.mean(dim=1, keepdim=True)

    def log_energy(v):
        e = torch.clamp((v * v).sum(1), min=EPS).log()
        return e if o['energy_floor'] == 0.0 else torch.clamp(e, min=math.log(o['energy_floor']))
    if o['raw_energy']:
        le = log_energy(fr)
    p = o['preemphasis_coefficient']
    if p != 0.0:
        prev = torch.cat([fr[:, :1], fr[:, :-1]], dim=1)
        fr = fr - p * prev
    fr = fr * win[None, :]
    if not o['raw_energy']:
        le = log_energy(fr)
    fr = torch.nn.functional.pad(fr, (0, Np - W))
    spec = torch.fft.rfft(fr).abs()
    if kind == 'spectrogram':
        out = torch.clamp(spec ** 2, min=EPS).log()
        out = torch.cat([le[:, None], out[:, 1:]], dim=1)
    else:
        if o.get('use_power', True):
            spec = spec ** 2
        banks = torch.from_numpy(backend.kaldi_mel_banks(o['num_mel_bins'], Np, o['sample_frequency'], o['low_freq'],
                                                         o['high_freq'], o['vtln_low'], o['vtln_high'],
                                                         o['vtln_warp']))
        mel = spec @ banks.T
        if kind == 'mfcc' or o.get('use_log_fbank', True):
            mel = torch.clamp(mel, min=EPS).log()
        if kind == 'fbank':
            out = mel
            if o['use_energy']:
                out = torch.cat([out, le[:, None]], 1) if o['htk_compat'] else torch.cat([le[:, None], out], 1)
        else:
            d = torch.from_numpy(backend.kaldi_dct(o['num_ceps'], o['num_mel_bins'], o['cepstral_lifter']))
            out = mel @ d
            if o['use_energy']:
                out = torch.cat([le[:, None], out[:, 1:]], 1)
            if o['htk_compat']:
                e = out[:, :1] * (1.0 if o['use_energy'] else math.sqrt(2.0))
                out = torch.cat([out[:, 1:], e], 1)
    if o['subtract_mean']:
        out = out - out.mean(dim=0, keepdim=True)
    if T > Tb:
        out = torch.cat([out, torch.zeros((T - Tb, K), dtype=torch.float64)], 0)
    return out


def log_bound(kind, x, o, lengths, ref):
    """Elementwise bound on |kernel - ref| for the float32 kernel (module docstring), (B, C, T, K) float64."""
    W, H, Np, min_len = plan_of(kind, o)
    B, C, L = x.shape
    u = 2.0 ** -24
    n = math.log2(Np)
    lens = [L] * B if lengths is None else [int(v) for v in lengths]
    T = ref.shape[2]
    pad = 0 if o['snip_edges'] else W // 2 - H // 2
    Ef = np.zeros((B, C, T))
    for b in range(B):
        Tb = backend.kaldi_num_frames(lens[b], W, H, o['snip_edges'], min_len)
        if Tb == 0:
            continue
        j = np.arange(Tb)[:, None] * H + np.arange(W)[None, :]
        idx = src_index(j, lens[b], pad) if not o['snip_edges'] else j
        Ef[b, :, :Tb] = (np.asarray(x[b][:, idx], np.float64) ** 2).sum(-1) + 1.0 * o['dither'] ** 2 * W * 30
    absr = np.abs(np.asarray(ref))
    num = 30.0 * Np * Ef * u * (n + 3)
    if kind == 'spectrogram' or o.get('use_log_fbank', True) or kind == 'mfcc':
        # ref is a log value: max(m, eps) = exp(ref) (>= eps by construction)
        mval = np.exp(np.asarray(ref, np.float64))
        if not o.get('use_power', True) and kind == 'fbank':
            num = np.sqrt(num)
        b_el = num[..., None] / np.maximum(mval, EPS) + 64 * u * (1.0 + absr)
    else:
        b_el = (num if o.get('use_power', True) else np.sqrt(num))[..., None] + 64 * u * absr
    if kind == 'mfcc':
        d = np.abs(backend.kaldi_dct(o['num_ceps'], o['num_mel_bins'], o['cepstral_lifter'])).sum(0)
        b_el = np.max(b_el, axis=-1, keepdims=True) * d.max() + 64 * u * (1.0 + absr)
    if o['subtract_mean']:
        b_el = 2.0 * np.broadcast_to(np.max(b_el, axis=2, keepdims=True), b_el.shape)
    return b_el + 2e-6 * (1.0 + absr)
