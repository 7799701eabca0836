"""Float64 restatement of the second-order-section cascade (kapre_sosfilt, scipy.signal.sosfilt / sosfilt_zi /
sosfiltfilt) and the error bound of the chunked float32 kernel (kapre_b200/csrc/sos_core.cuh).

Each row [b0, b1, b2, 1, a1, a2] is one section in direct form II transposed with state (z1, z2):

    y = b0 x + z1,   z1 <- b1 x - a1 y + z2,   z2 <- b2 x - a2 y

and the sections run in row order.  Everything here takes the float32 coefficients the kernel received, upcast to
float64: rounding the coefficients to float32 makes a different filter, not a kernel error.
"""
import numpy as np
import scipy.signal

EPS32 = 2.0 ** -24          # unit roundoff of float32
TC = 65                     # samples per chunk
W = 32                      # chunks per block
MAX_SECTIONS = 8


def sosfilt(x, sos, zi=None):
    """The recurrence above along the last axis of x by a plain loop in float64 (the definition the tests pin).
    sos (S, 6); zi (..., S, 2) or None.  Returns (y, zf)."""
    x = np.asarray(x, np.float64)
    sos = np.asarray(sos, np.float64)
    S = sos.shape[0]
    z = np.zeros(x.shape[:-1] + (S, 2))
    if zi is not None:
        z = z + np.asarray(zi, np.float64)
    y = np.zeros_like(x)
    for t in range(x.shape[-1]):
        v = x[..., t]
        for s in range(S):
            b0, b1, b2, _, a1, a2 = sos[s]
            out = b0 * v + z[..., s, 0]
            z[..., s, 0] = b1 * v - a1 * out + z[..., s, 1]
            z[..., s, 1] = b2 * v - a2 * out
            v = out
        y[..., t] = v
    return y, z


def sosfilt_fast(x, sos, zi=None):
    """The same by scipy.signal.sosfilt (equal to ``sosfilt`` to rounding; used for long signals).  Returns (y, zf)."""
    x = np.asarray(x, np.float64)
    sos = np.asarray(sos, np.float64)
    if zi is None:
        zi = np.zeros(x.shape[:-1] + (sos.shape[0], 2))
    zi = np.broadcast_to(np.asarray(zi, np.float64), x.shape[:-1] + (sos.shape[0], 2))
    y, zf = scipy.signal.sosfilt(sos, x, axis=-1, zi=np.moveaxis(zi, -2, 0))
    return y, np.moveaxis(zf, 0, -2)


def sosfilt_zi(sos):
    """scipy.signal.sosfilt_zi: per-section lfilter_zi (the steady state of a unit step), scaled by the DC gain of the
    sections before it, by the closed form of a biquad."""
    sos = np.asarray(sos, np.float64)
    zi = np.zeros((sos.shape[0], 2))
    scale = 1.0
    for s, (b0, b1, b2, _, a1, a2) in enumerate(sos):
        B1, B2 = b1 - a1 * b0, b2 - a2 * b0
        z1 = (B1 + B2) / (1.0 + a1 + a2)
        zi[s] = scale * z1, scale * (B2 - a2 * z1)
        scale *= (b0 + b1 + b2) / (1.0 + a1 + a2)
    return zi


def n_taps(sos):
    sos = np.asarray(sos)
    return 2 * sos.shape[0] + 1 - min(int((sos[:, 2] == 0).sum()), int((sos[:, 5] == 0).sum()))


def extend(x, n, padtype):
    """scipy's odd / even / constant extension of the last axis by n samples on either side (None: no extension)."""
    if padtype is None or n == 0:
        return x
    left, right = x[..., n:0:-1], x[..., -2:-(n + 2):-1]
    if padtype == 'odd':
        return np.concatenate([2 * x[..., :1] - left, x, 2 * x[..., -1:] - right], -1)
    if padtype == 'even':
        return np.concatenate([left, x, right], -1)
    if padtype == 'constant':
        return np.concatenate([np.repeat(x[..., :1], n, -1), x, np.repeat(x[..., -1:], n, -1)], -1)
    raise ValueError(padtype)


def sosfiltfilt(x, sos, padtype='odd', padlen=None):
    """scipy.signal.sosfiltfilt restated: extend, run forward from sosfilt_zi * x_ext[0], backward from
    sosfilt_zi * y[-1], trim."""
    x = np.asarray(x, np.float64)
    edge = 0 if padtype is None else (3 * n_taps(sos) if padlen is None else padlen)
    ext = extend(x, edge, padtype)
    z = sosfilt_zi(sos)
    y, _ = sosfilt_fast(ext, sos, z * ext[..., :1, None])
    y, _ = sosfilt_fast(y[..., ::-1], sos, z * y[..., -1:, None])
    y = y[..., ::-1]
    return y[..., edge:y.shape[-1] - edge] if edge else y


def _trajectory(x, sos, zi):
    """Per section: (max |x_s|, max |y_s|, max |z1|, max |z2|) over the run (the states before every step and after
    the last), in float64."""
    out = []
    v = np.asarray(x, np.float64)
    for s in range(sos.shape[0]):
        b0, b1, b2, _, a1, a2 = sos[s]
        z0 = np.zeros(v.shape[:-1] + (2,)) if zi is None else np.broadcast_to(zi[..., s, :], v.shape[:-1] + (2,))
        y, zf = scipy.signal.lfilter(sos[s, :3], sos[s, 3:], v, axis=-1, zi=np.ascontiguousarray(z0))
        z1 = max(np.abs(y - b0 * v).max(initial=0.0), np.abs(zf[..., 0]).max(initial=0.0))
        z2 = max(np.abs(b2 * v - a2 * y).max(initial=0.0), np.abs(z0[..., 1]).max(initial=0.0))
        out.append((np.abs(v).max(initial=0.0), np.abs(y).max(initial=0.0), z1, z2))
        v = y
    return out


def _chunked(x):
    """x cut into zero-padded chunks of TC samples along a new last axis (the state pass's zero-start runs)."""
    x = np.asarray(x, np.float64)
    L = x.shape[-1]
    K = -(-L // TC)
    U = np.zeros(x.shape[:-1] + (K * TC,))
    U[..., :L] = x
    return U.reshape(x.shape[:-1] + (K, TC))


def response_l1(sos, s, tol=1e-13, max_len=1 << 22):
    """||g_(s -> s')||_1 for s' = s .. S-1: the response of section s' 's output to a unit error in section s 's z1,
    i.e. 1 / A_s followed by sections s + 1 .. s', summed until the tail is below tol of the sum."""
    n = 4096
    while True:
        h = np.zeros(n)
        h[0] = 1.0
        h = scipy.signal.lfilter([1.0], sos[s, 3:], h)
        out, done = [], True
        for k in range(s, sos.shape[0]):
            if k > s:
                h = scipy.signal.lfilter(sos[k, :3], sos[k, 3:], h)
            g = np.abs(h)
            tot = g.sum()
            out.append(float(tot))
            done &= bool(g[-n // 8:].max() * n < tol * max(tot, 1e-300))
        if done or n >= max_len:
            return out
        n *= 4


def error_bounds(x, sos, zi=None):
    """(bound on |y_kernel - y|, bound on |zf_kernel - zf|) for float32 data x (..., L), float32 coefficients sos and an
    optional float32 initial state zi (..., S, 2), all upcast to float64.

    In section s a float32 step commits at most eps (|y| (1 + |a1| + |a2|) + 2 |x_s| (|b1| + |b2|) + 2 |z2|): one
    rounding in y = fmaf(b0, x, z1), two in z1' and two in z2' (the product b2 x).  Each of them equals an error in z1
    of that section at that step or a later one, and an error in z1 reaches the output of section s' through g_(s->s')
    (``response_l1``), so all steps together stay below ||g_(s->s')||_1 times the largest.  The state pass runs the
    same steps on zero-start chunks (bounded by their own maxima) and reaches later chunks through float64 carries
    only; its end states are rounded to float32 once per chunk, and so are the output pass's start states (and the
    caller's zi): at most eps |z| in each state component, again through g.  The output store does not round (the
    kernel stores its float32 y).  A factor 2 covers the float64 parts and the terms the first-order analysis drops.

    zf is made of the last section-level values: z1 = y_s - b0 x_s one step on, z2 = b2 x_s - a2 y_s, so its error is
    bounded from the bounds on y_(s-1) and y_s, plus the rounding of the last step's state updates."""
    sos = np.asarray(sos, np.float64)
    S = sos.shape[0]
    zi = None if zi is None else np.asarray(zi, np.float64)
    tr = _trajectory(x, sos, zi)
    loc = _trajectory(_chunked(x), sos, None)
    E = []
    for s in range(S):
        b0, b1, b2, _, a1, a2 = sos[s]

        def step(X, Y, Z2):
            return EPS32 * (Y * (1 + abs(a1) + abs(a2)) + 2 * X * (abs(b1) + abs(b2)) + 2 * Z2)
        X, Y, Z1, Z2 = tr[s]
        Xl, Yl, Z1l, Z2l = loc[s]
        E.append(step(X, Y, Z2) + step(max(X, Xl), max(Y, Yl), max(Z2, Z2l)) + EPS32 * (Z1 + Z2 + Z1l + Z2l))
    G = [response_l1(sos, s) for s in range(S)]                  # G[s][s' - s]
    By = [2.0 * sum(G[s][k - s] * E[s] for s in range(k + 1)) + 1e-30 for k in range(S)]
    bz = 0.0
    for k in range(S):
        b0, _, b2, _, _, a2 = sos[k]
        prev = By[k - 1] if k else 0.0
        _, _, Z1, Z2 = tr[k]
        bz = max(bz, By[k] + abs(b0) * prev + 4 * EPS32 * Z1, abs(b2) * prev + abs(a2) * By[k] + 4 * EPS32 * Z2)
    return By[-1], bz


def error_bound(x, sos, zi=None):
    return error_bounds(x, sos, zi)[0]
