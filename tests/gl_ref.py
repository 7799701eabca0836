"""Float64 restatement of fast Griffin-Lim, independent of the CUDA code.

``griffin_lim`` takes the transform pair as arguments, so the same loop is pinned to
``torchaudio.functional.griffinlim`` (with torch's centred transforms) and, over the oracle's ``tf.signal``
restatements (``kapre_pair``), is the reference for the GPU layer.  ``phase_u`` restates the counter-based hash
of the random initial phases documented in include/kapre_b200.h bit for bit.
"""
import numpy as np
import torch

import oracle

_M64 = (1 << 64) - 1


def griffin_lim(S, stft_fn, istft_fn, n_iter, momentum, A0, return_X=False):
    """S: (..., T, F) float64 magnitudes; stft_fn: waveform -> (..., T, F) complex; istft_fn: the inverse;
    A0: the initial phase factor (a scalar or a complex tensor of S's shape).  Returns ISTFT of the last X."""
    beta = momentum / (1 + momentum)
    X = (S * A0).to(torch.complex64 if S.dtype == torch.float32 else torch.complex128)
    Yprev = None
    for _ in range(n_iter):
        Y = stft_fn(istft_fn(X))
        A = Y if Yprev is None else Y - beta * Yprev
        X = S * (A / (A.abs() + 1e-16))
        Yprev = Y
    y = istft_fn(X)
    return (y, X) if return_X else y


def kapre_pair(n_fft, win_length, hop, window_name=None):
    """(stft_fn, istft_fn) over (..., L) / (..., T, F) float64 / complex128 torch tensors: ``tf.signal.stft`` without
    padding and ``tf.signal.inverse_stft`` with the dual window, as the oracle restates them."""
    w = oracle.get_window(window_name, win_length)
    dual = oracle.inverse_stft_window(win_length, hop, w)

    def stft_fn(y):
        return torch.from_numpy(oracle.stft_frames(y.numpy(), n_fft, win_length, hop, w, pad_end=False))

    def istft_fn(X):
        return torch.from_numpy(oracle.inverse_stft_frames(X.numpy(), n_fft, win_length, hop, dual))

    return stft_fn, istft_fn


def kapre_pair32(n_fft, win_length, hop, window_name=None):
    """The same pair computed in float32 / complex64 by torch's CPU FFT: a float32 twin of the loop, whose drift from
    the float64 run measures how much a given input amplifies float32 rounding."""
    w = torch.from_numpy(oracle.get_window(None if window_name is None else window_name, win_length)).float()
    dual = torch.from_numpy(oracle.inverse_stft_window(win_length, hop, w.double().numpy())).float()

    def stft_fn(y):
        T = 1 + (y.shape[-1] - win_length) // hop
        return torch.fft.rfft(y.unfold(-1, win_length, hop)[..., :T, :] * w, n=n_fft, dim=-1)

    def istft_fn(X):
        T = X.shape[-2]
        fr = torch.fft.irfft(X, n=n_fft, dim=-1)[..., :win_length] * dual
        out = torch.zeros(X.shape[:-2] + ((T - 1) * hop + win_length,), dtype=torch.float32)
        for t in range(T):
            out[..., t * hop:t * hop + win_length] += fr[..., t, :]
        return out

    return stft_fn, istft_fn


def _mix(z):
    z = (z + 0x9E3779B97F4A7C15) & _M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & _M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & _M64
    return z ^ (z >> 31)


def phase_u(seed, i):
    """u(seed, i) in [0, 1): the top 24 bits of mix(seed ^ mix(i)), as a Python float (exact)."""
    return (_mix(seed ^ _mix(int(i))) >> 40) / float(1 << 24)


def _mix_np(z):
    """``_mix`` on a uint64 array (NumPy's uint64 arithmetic wraps modulo 2^64)."""
    with np.errstate(over='ignore'):
        z = z + np.uint64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def phase_u_table(seed, n):
    """phase_u(seed, i) for i = 0 .. n-1 as a float64 array."""
    z = _mix_np(np.uint64(seed) ^ _mix_np(np.arange(n, dtype=np.uint64)))
    return (z >> np.uint64(40)).astype(np.float64) / float(1 << 24)


def random_phase(seed, B, C, T, F):
    """exp(2 pi i u(seed, ((b C + c) T + t) F + f)) as a (B, C, T, F) complex128 tensor."""
    u = phase_u_table(seed, B * C * T * F).reshape(B, C, T, F)
    return torch.from_numpy(np.exp(2j * np.pi * u))


def spectral_convergence(y, S, stft_fn):
    """||(|STFT(y)| - S)|| / ||S||."""
    return float(torch.linalg.vector_norm(stft_fn(y).abs() - S) / torch.linalg.vector_norm(S))
