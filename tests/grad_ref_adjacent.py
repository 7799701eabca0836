"""Float64 torch restatement of the layers next to the hot path, differentiable by torch autograd: Phase,
get_stft_mag_phase, Delta, Frame, Energy, ConcatenateFrequencyMap and SpecAugment with given masks.

Test infrastructure for the gradient tests, like ``grad_ref.py`` (whose STFT and decibel restatements it reuses);
``test_grad_aux_emu.py`` pins its forward to ``oracle.reference``.  ``delta`` extends the time axis with
``pad_index``, the kernels' single-reflection rule: for axes longer than the half window it is ``tf.pad``'s, for
shorter ones a position more than one reflection away reads zero.
"""
import numpy as np
import torch

import grad_ref as R

CL, CF = 'channels_last', 'channels_first'


def phase(X):
    return torch.angle(X)


def mag_phase(x, n_fft, win_length, hop, window_name=None, pad_begin=False, pad_end=False, in_fmt=CF, out_fmt=CF,
              db=None):
    """get_stft_mag_phase: [|S| (dB-scaled with db = (ref_value, amin, dynamic_range)); angle(S)] on the channel axis."""
    s = R.stft(x, n_fft, win_length, hop, window_name, pad_begin, pad_end, in_fmt, out_fmt)
    mag = s.abs()
    if db is not None:
        mag = R.magnitude_to_decibel(mag, *db)
    return torch.cat([mag, torch.angle(s)], dim=3 if out_fmt == CL else 1)


def pad_index(t, T, mode):
    """Index in [0, T) that position t of the extended axis reads, or -1 for zero (0 symmetric, 1 reflect, 2 constant)."""
    if 0 <= t < T:
        return t
    if mode == 2:
        return -1
    if t < 0:
        t = -t - 1 if mode == 0 else -t
    else:
        t = 2 * T - 1 - t if mode == 0 else 2 * T - 2 - t
    return t if 0 <= t < T else -1


_MODES = {'symmetric': 0, 'reflect': 1, 'constant': 2}


def delta(x, win_length=5, mode='symmetric', data_format=CF):
    """Delta along the time axis (1 for channels_last, 2 for channels_first) as an index gather."""
    ax = 1 if data_format == CL else 2
    xt = x.movedim(ax, -1)
    T = xt.shape[-1]
    xp = torch.cat([xt, xt.new_zeros(xt.shape[:-1] + (1,))], dim=-1)    # index T reads zero
    n = (win_length - 1) // 2
    md = _MODES[mode.lower()]

    def idx(shift):
        return torch.tensor([pad_index(t + shift, T, md) % (T + 1) for t in range(T)], dtype=torch.long, device=x.device)
    out = sum(m * (xp[..., idx(m)] - xp[..., idx(-m)]) for m in range(1, n + 1))
    out = out / (2 * sum(m * m for m in range(1, n + 1)))
    return out.movedim(-1, ax)


def frame(x, frame_length, hop, pad_end=False, pad_value=0.0, data_format=CF):
    """(B, L, C) -> (B, T, frame_length, C) or (B, C, L) -> (B, C, T, frame_length); positions past the signal hold
    pad_value."""
    if data_format == CL:
        x = x.transpose(1, 2)
    L = x.shape[-1]
    T = -(-L // hop) if pad_end else max(0, 1 + (L - frame_length) // hop)
    need = (T - 1) * hop + frame_length if T > 0 else 0
    if need > L:
        x = torch.nn.functional.pad(x, (0, need - L), value=float(pad_value))
    idx = torch.arange(T, device=x.device)[:, None] * hop + torch.arange(frame_length, device=x.device)[None, :]
    fr = x[..., idx]
    return fr.permute(0, 2, 3, 1) if data_format == CL else fr


def energy(x, frame_length, hop, pad_end=False, pad_value=0.0, scale=1.0, data_format=CF):
    fr = frame(x, frame_length, hop, pad_end, pad_value, data_format)
    return scale * (fr ** 2).sum(dim=2 if data_format == CL else 3)


def frequency_map(F):
    """linspace(0, 1, F) as the forward kernel and tf.linspace form it in float32."""
    step = np.float32(1.0) / np.float32(F - 1) if F > 1 else np.float32(0.0)
    m = (np.arange(F, dtype=np.float32) * step).astype(np.float32)
    if F > 1:
        m[-1] = 1.0
    return torch.from_numpy(m.astype(np.float64))


def concat_frequency_map(x, data_format=CF):
    if data_format == CL:
        B, T, F, _ = x.shape
        return torch.cat([x, frequency_map(F).to(x).reshape(1, 1, F, 1).expand(B, T, F, 1)], dim=3)
    B, _, T, F = x.shape
    return torch.cat([x, frequency_map(F).to(x).reshape(1, 1, 1, F).expand(B, 1, T, F)], dim=1)


def spec_augment_mask(time_masks, freq_masks, T, F):
    """(B, T, F) bool: True where an item's time or frequency index lies in [start, start + width] of one of its masks."""
    tm, fm = np.asarray(time_masks).reshape(len(time_masks), -1, 2), np.asarray(freq_masks).reshape(len(freq_masks), -1, 2)
    t, f = np.arange(T), np.arange(F)
    mt = np.zeros((tm.shape[0], T), bool)
    for j in range(tm.shape[1]):
        mt |= (t[None] >= tm[:, j, :1]) & (t[None] <= tm[:, j, :1] + tm[:, j, 1:])
    mf = np.zeros((fm.shape[0], F), bool)
    for j in range(fm.shape[1]):
        mf |= (f[None] >= fm[:, j, :1]) & (f[None] <= fm[:, j, :1] + fm[:, j, 1:])
    return torch.from_numpy(mt[:, :, None] | mf[:, None, :])


def spec_augment(x, time_masks, freq_masks, mask_value=0.0, data_format=CF):
    """Depth-1 (B, T, F, 1) / (B, 1, T, F) batch with the given (B, n, 2) (start, width) masks."""
    T, F = (x.shape[1], x.shape[2]) if data_format == CL else (x.shape[2], x.shape[3])
    m = spec_augment_mask(time_masks, freq_masks, T, F).to(x.device)
    m = m[..., None] if data_format == CL else m[:, None]
    return torch.where(m, torch.full_like(x, float(mask_value)), x)
