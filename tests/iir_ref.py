"""Float64 restatement of the IIR filter (kapre_lfilter, torchaudio.functional.lfilter), its adjoint and the error bound
of the chunked float32 kernel (kapre_b200/csrc/iir_core.cuh).

    u[t] = sum_{k=0..N} b[k] x[t-k],   y[t] = u[t] - sum_{k=1..N} a[k] y[t-k],   x, y = 0 before t = 0

with b, a already divided by a[0].  Everything here takes the float32 coefficients the kernel received, upcast to
float64: float32 rounding of the coefficients makes a different filter, not a kernel error.
"""
import numpy as np
import scipy.signal

EPS32 = 2.0 ** -24          # unit roundoff of float32
TC = 65                     # samples per chunk
W = 32                      # chunks per block
MAX_ORDER = 8


def lfilter(x, b, a, clamp=False):
    """The recurrence above along the last axis, by a plain loop in float64 (the definition the tests pin)."""
    x = np.asarray(x, np.float64)
    b = np.asarray(b, np.float64)
    a = np.asarray(a, np.float64)
    N = len(b) - 1
    y = np.zeros_like(x)
    for t in range(x.shape[-1]):
        acc = np.zeros(x.shape[:-1])
        for k in range(N + 1):
            if t - k >= 0:
                acc = acc + b[k] * x[..., t - k]
        for k in range(1, N + 1):
            if t - k >= 0:
                acc = acc - a[k] * y[..., t - k]
        y[..., t] = acc
    return np.clip(y, -1.0, 1.0) if clamp else y


def lfilter_fast(x, b, a, clamp=False):
    """The same by scipy.signal.lfilter (equal to ``lfilter`` to rounding; used for long signals)."""
    y = scipy.signal.lfilter(np.asarray(b, np.float64), np.asarray(a, np.float64), np.asarray(x, np.float64), axis=-1)
    return np.clip(y, -1.0, 1.0) if clamp else y


def filtfilt(x, b, a, clamp=True):
    """torchaudio's filtfilt: lfilter without clamping, then lfilter in reverse time, then the clamp."""
    y = lfilter_fast(x, b, a)
    y = lfilter_fast(y[..., ::-1], b, a)[..., ::-1]
    return np.clip(y, -1.0, 1.0) if clamp else y


def matrix(b, a, L):
    """The L x L matrix of lfilter (lower-triangular Toeplitz of the impulse response)."""
    h = lfilter_fast(np.eye(L)[0], b, a)
    M = np.zeros((L, L))
    for j in range(L):
        M[j:, j] = h[:L - j]
    return M


def allpole_adjoint(gy, a):
    """v[t] = gy[t] - sum_k a[k] v[t+k] (the all-pole recursion in reverse time)."""
    return scipy.signal.lfilter([1.0], np.asarray(a, np.float64), np.asarray(gy, np.float64)[..., ::-1], axis=-1)[..., ::-1]


def vjp(x, gy, b, a):
    """(gx, gb, ga) of y = lfilter(x) (unclamped) at output gradient gy, from the adjoint v:
    gx[t] = sum_k b[k] v[t+k], gb[k] = sum_t v[t] x[t-k], ga[k] = -sum_t v[t] y[t-k] (ga[0] = 0).  x, gy: (..., L);
    the coefficient gradients are summed over the leading axes."""
    x = np.asarray(x, np.float64)
    b = np.asarray(b, np.float64)
    a = np.asarray(a, np.float64)
    N, L = len(b) - 1, x.shape[-1]
    y = lfilter_fast(x, b, a)
    v = allpole_adjoint(gy, a)
    gx = np.zeros_like(v)
    gb, ga = np.zeros(N + 1), np.zeros(N + 1)
    for k in range(N + 1):
        gx[..., :L - k] += b[k] * v[..., k:]
        gb[k] = np.sum(v[..., k:] * x[..., :L - k])
        if k:
            ga[k] = -np.sum(v[..., k:] * y[..., :L - k])
    return gx, gb, ga


def impulse_l1(a, tol=1e-13, max_len=1 << 22):
    """||g||_1 of the all-pole impulse response 1 / A(z), summed until the tail is below tol of the sum."""
    a = np.asarray(a, np.float64)
    n = 4096
    while True:
        imp = np.zeros(n)
        imp[0] = 1.0
        g = np.abs(scipy.signal.lfilter([1.0], a, imp))
        s = g.sum()
        if g[-n // 8:].max() * n < tol * s or n >= max_len:
            return float(s)
        n *= 4


def local_max(x, b, a):
    """max |y| of the zero-start runs over every chunk of TC samples (the state pass's intermediate values): the FIR
    part from the true input, the all-pole part from a zero state in each chunk."""
    x = np.asarray(x, np.float64)
    u = scipy.signal.lfilter(np.asarray(b, np.float64), [1.0], x, axis=-1)
    L = u.shape[-1]
    K = -(-L // TC)
    U = np.zeros(u.shape[:-1] + (K * TC,))
    U[..., :L] = u
    U = U.reshape(u.shape[:-1] + (K, TC))
    return float(np.abs(scipy.signal.lfilter([1.0], np.asarray(a, np.float64), U, axis=-1)).max())


def error_bound(b, a, x_max, y_max, y_local_max):
    """Bound on |y_kernel - y| for float32 data, float32 coefficients b, a (already normalised), |x| <= x_max,
    |y| <= y_max and zero-start chunk runs bounded by y_local_max (``local_max``).

    Each float32 step of the recursion (2N + 2 rounded operations: N + 1 FIR terms, N feedback terms) commits an
    error of at most (2N + 2) eps (||b||_1 x_max + ||a'||_1 Y) with Y the magnitude of the values it runs on (the
    true output in the output pass, the zero-start runs in the state pass), a' = a[1:].  An error committed at step
    s reaches y[t] through the all-pole impulse response: g[t - s] times it, so every step's errors together stay
    below ||g||_1 times the largest.  The state pass's errors reach later chunks only through the float64 carry,
    which adds float64 rounding alone.  The start state of the output pass is rounded to float32 once (N values of
    at most y_max): the same as a perturbation of at most ||a'||_1 eps y_max in each of the chunk's first N steps,
    again through g.  The final store rounds once more.  The sum, with a factor 2 for the float64 parts and the
    terms the first-order analysis drops."""
    b = np.asarray(b, np.float64)
    a = np.asarray(a, np.float64)
    N = len(b) - 1
    g1 = impulse_l1(a)
    nb, na = np.abs(b).sum(), np.abs(a[1:]).sum()
    step_out = (2 * N + 2) * EPS32 * (nb * x_max + na * y_max)
    step_loc = (2 * N + 2) * EPS32 * (nb * x_max + na * max(y_local_max, y_max))
    state = na * EPS32 * y_max
    return 2.0 * (g1 * (step_out + step_loc + state) + EPS32 * y_max) + 1e-30


def biquad(kind, sample_rate, freq, Q=0.707, gain=0.0):
    """torchaudio's biquad designs (lowpass_biquad ... equalizer_biquad; bandpass with const_skirt_gain=False),
    restated: (b, a) float64, each of length 3, not normalised."""
    w0 = 2 * np.pi * freq / sample_rate
    alpha = np.sin(w0) / 2 / Q
    c = np.cos(w0)
    if kind == 'lowpass':
        b = [(1 - c) / 2, 1 - c, (1 - c) / 2]
        a = [1 + alpha, -2 * c, 1 - alpha]
    elif kind == 'highpass':
        b = [(1 + c) / 2, -1 - c, (1 + c) / 2]
        a = [1 + alpha, -2 * c, 1 - alpha]
    elif kind == 'bandpass':
        b = [alpha, 0.0, -alpha]
        a = [1 + alpha, -2 * c, 1 - alpha]
    elif kind == 'bandreject':
        b = [1.0, -2 * c, 1.0]
        a = [1 + alpha, -2 * c, 1 - alpha]
    elif kind == 'allpass':
        b = [1 - alpha, -2 * c, 1 + alpha]
        a = [1 + alpha, -2 * c, 1 - alpha]
    elif kind == 'equalizer':
        A = np.exp(gain / 40.0 * np.log(10))
        b = [1 + alpha * A, -2 * c, 1 - alpha * A]
        a = [1 + alpha / A, -2 * c, 1 - alpha / A]
    else:
        raise ValueError(kind)
    return np.array(b, np.float64), np.array(a, np.float64)


def normalised32(b, a):
    """The float32 coefficients the kernel receives from ``lfilter(x, a, b)``: b and a rounded to float32, then
    divided by a[0] in float32, as the library (and torchaudio) does on the device."""
    b = np.asarray(b, np.float64).astype(np.float32)
    a = np.asarray(a, np.float64).astype(np.float32)
    return b / a[..., :1], a / a[..., :1]
