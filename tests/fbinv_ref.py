"""Float64 restatement of the filterbank inversion (NNLS by projected accelerated gradient), independent of the CUDA
code.

``fista`` runs the loop documented in include/kapre_b200.h on a (frames, n_bands) array with the matrix, the
initial back-projection weights and the step as inputs, in float64 or, as a twin whose drift measures how much an
input amplifies rounding, in float32.  ``step_of`` and ``inv_d_of`` give the plan's values in float64.  ``bank`` and
``consistent_input`` make the test banks and the filterbank outputs of a real spectrogram that the tests invert.
"""
import numpy as np

import oracle


def matrix(fb):
    """A: the (n_bands, n_freq) transpose of a (n_freq, n_bands) filterbank, as float64."""
    return np.asarray(fb, np.float64).T.copy()


def step_of(A):
    return 1.0 / np.linalg.norm(A, 2) ** 2


def inv_d_of(A):
    """1 / (A A^T 1), 0 where that is 0."""
    d = A @ (A.T @ np.ones(A.shape[0]))
    out = np.zeros_like(d)
    out[d > 0] = 1.0 / d[d > 0]
    return out


def fista(A, m, n_iter, step=None, inv_d=None, dtype=np.float64):
    """m: (frames, n_bands) -> (frames, n_freq).  s_0 = max(A^T (m / d), 0); n_iter projected accelerated gradient
    steps; returns s_n.  ``step`` / ``inv_d`` default to the float64 values; the momentum coefficient is computed in
    float64 and rounded to ``dtype``."""
    A = np.asarray(A, dtype)
    m = np.asarray(m, dtype)
    step = dtype(step_of(np.asarray(A, np.float64)) if step is None else step)
    inv_d = np.asarray(inv_d_of(np.asarray(A, np.float64)) if inv_d is None else inv_d, dtype)
    s = np.maximum((m * inv_d) @ A, 0)
    y = s.copy()
    t = 1.0
    for _ in range(n_iter):
        tn = 0.5 * (1.0 + np.sqrt(1.0 + 4.0 * t * t))
        coef = dtype((t - 1.0) / tn)
        t = tn
        g = (y @ A.T - m) @ A
        sn = np.maximum(y - step * g, 0)
        y = sn + coef * (sn - s)
        s = sn
    return s


def residual(A, s, m):
    """Per frame ||A s - m|| / ||m||."""
    A = np.asarray(A, np.float64)
    r = np.asarray(s, np.float64) @ A.T - np.asarray(m, np.float64)
    return np.linalg.norm(r, axis=-1) / np.linalg.norm(np.asarray(m, np.float64), axis=-1)


def lstsq_relu(A, m):
    """What ``torchaudio.transforms.InverseMelScale`` computes, with this matrix: the minimum-norm least-squares
    solution, then ``relu``."""
    import torch
    At = torch.from_numpy(np.asarray(A, np.float64))
    sol = torch.linalg.lstsq(At, torch.from_numpy(np.asarray(m, np.float64)).T, driver='gelsd').solution
    return torch.relu(sol).T.numpy()


def bank(kind, sample_rate, n_fft, n_bands):
    """The library's (n_freq, n_bands) 'mel' or 'log' filterbank."""
    from kapre_b200 import backend
    if kind == 'mel':
        return backend.filterbank_mel(sample_rate=sample_rate, n_freq=n_fft // 2 + 1, n_mels=n_bands)
    return backend.filterbank_log(sample_rate=sample_rate, n_freq=n_fft // 2 + 1, n_bins=n_bands)


def signal(C, L, sample_rate, seed=0):
    """(C, L) float64: a vibrato harmonic tone per channel (a different pitch per channel) plus a little noise."""
    t = np.arange(L) / sample_rate
    rng = np.random.default_rng(seed)
    x = np.empty((C, L))
    for c in range(C):
        f0 = 180.0 * (1 + 0.4 * c)
        x[c] = sum(0.3 / k * np.sin(2 * np.pi * (k * f0 + 20 * np.sin(2 * np.pi * 0.7 * t)) * t) for k in range(1, 8))
        x[c] += 0.01 * rng.standard_normal(L)
    return x


def consistent_input(fb, sample_rate, n_fft, B, C, T, seed=0):
    """(B, C, T, n_bands) float32: the filterbank applied to |STFT| (Hann, hop n_fft / 4) of ``signal``, so every frame
    is reachable by a non-negative spectrum."""
    hop = n_fft // 4
    L = (T - 1) * hop + n_fft
    x = np.stack([signal(C, L, sample_rate, seed + b) for b in range(B)])
    S = np.abs(oracle.stft_frames(x, n_fft, n_fft, hop, oracle.get_window(None, n_fft), False))
    assert S.shape[2] == T
    return (S @ np.asarray(fb, np.float64)).astype(np.float32)
