"""Float64 restatement of the partitioned FFT convolution (``kapre_convolve``) and its adjoints, for the tests.

With block size B, the signal's blocks x[jB, jB + B) and the filter's blocks h[pB, pB + B), each zero-padded to 2B, are
transformed by a real FFT of 2B points (X: J blocks, H: P blocks, B + 1 bins).  Per bin,
    Y_i = sum_{p < P} H_p X_{i - p}                              (convolve along the blocks, i < T = J + P - 1)
and y is the overlap-add, hop B, of the inverse FFTs of Y: (T + 1) B samples whose first L + K - 1 are x * h.
The adjoints are correlations along the blocks:
    gX_j = sum_p conj(H_p) G_{j + p},   gH_p = sum_j conj(X_j) G_{j + p}.
"""
import math

import numpy as np

EPS32 = 2.0 ** -24
BLOCKS = (128, 256, 512, 1024)


def block_size(K):
    """The library's rule (kb_conv_block_size): the smallest B with ceil(K / B) <= 8, else 1024."""
    for b in (128, 256, 512):
        if -(-K // b) <= 8:
            return b
    return 1024


def span(L, K, mode):
    """torchaudio.functional.fftconvolve's crop of the full convolution: (start, length)."""
    full = L + K - 1
    if mode == 'full':
        return 0, full
    target = L if mode == 'same' else max(L, K) - min(L, K) + 1
    return (full - target) // 2, target


def blocks(x, B):
    """(..., L) -> (..., ceil(L / B), B + 1) complex128 block spectra."""
    L = x.shape[-1]
    n = -(-L // B)
    pad = np.zeros(x.shape[:-1] + (n * B,), np.float64)
    pad[..., :L] = x
    fr = np.zeros(x.shape[:-1] + (n, 2 * B), np.float64)
    fr[..., :B] = pad.reshape(x.shape[:-1] + (n, B))
    return np.fft.rfft(fr, axis=-1)


def mac(a, b, To, correlate):
    """The kernel's sum along axis -2 (frames) in float64 / complex128: convolve or correlate, To outputs."""
    S, Tb = a.shape[-2], b.shape[-2]
    out = np.zeros(np.broadcast_shapes(a.shape[:-2], b.shape[:-2]) + (To, a.shape[-1]), np.complex128)
    for i in range(To):
        for s in range(S):
            k = i + s if correlate else i - s
            if 0 <= k < Tb:
                out[..., i, :] += (np.conj(a[..., s, :]) if correlate else a[..., s, :]) * b[..., k, :]
    return out


def overlap_add(Y, B):
    """(..., T, B + 1) -> (..., (T + 1) B): inverse FFTs of 2B points, overlap-added at hop B."""
    fr = np.fft.irfft(Y, n=2 * B, axis=-1)
    T = Y.shape[-2]
    y = np.zeros(Y.shape[:-2] + ((T + 1) * B,), np.float64)
    for t in range(T):
        y[..., t * B:t * B + 2 * B] += fr[..., t, :]
    return y


def convolve_full(x, h, B=None):
    """Untrimmed output of the scheme: x (..., L), h broadcastable (..., K) -> (..., (T + 1) B)."""
    B = B or block_size(h.shape[-1])
    X, H = blocks(np.asarray(x, np.float64), B), blocks(np.asarray(h, np.float64), B)
    return overlap_add(mac(H, X, X.shape[-2] + H.shape[-2] - 1, False), B)


def mac_matrix(a, Tb, To, correlate):
    """The explicit (To, Tb) matrix of one bin's sum: out = M b."""
    S = a.shape[0]
    M = np.zeros((To, Tb), np.complex128)
    for i in range(To):
        for s in range(S):
            k = i + s if correlate else i - s
            if 0 <= k < Tb:
                M[i, k] += np.conj(a[s]) if correlate else a[s]
    return M


def error_bound(B, P):
    """Bound on max |y - x * h| per unit of rms(x) ||h||_2 for the float32 chain.

    Rounding model (u = 2^-24 per operation): the register FFT of 2B points has log2(2B) butterfly passes plus the
    twiddle multiply, each adding at most about 2u of relative error in the l2 sense, and the chain runs three of them
    (x's blocks, h's blocks, the inverse): 6 (log2(2B) + 1) u.  The block product adds 2u, the P-term sum along the
    blocks up to P u (each term is rounded once into the accumulator) and the overlap-add of two frames u, i.e.
    (P + 4) u.  That bounds the rms error of y relative to rms(x) ||h||_2; a sample's error exceeds the rms by the
    crest factor of the error signal, taken as 4 (a Gaussian error reaches 4 sigma once in 1.6e4 samples, 5.3 in 1e7),
    and the bound doubles that for margin: 8 (6 (log2(2B) + 1) + P + 4) u.  At B = 1024, P = 16 this is 4.4e-5, where
    emulation and float32 pocketfft measure 1.0 - 1.2e-6, and at B = 128, P = 1 it is 2.1e-5."""
    return 8.0 * (6.0 * (math.log2(2 * B) + 1.0) + P + 4.0) * EPS32
