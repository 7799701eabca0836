"""Float64 restatement of the image-source room impulse response (kapre_rir_ism, DESIGN.md §RIR) and the elementwise
error bound of the kernel's float32 taps and sums.

The maths is the project's own definition, modelled on pyroomacoustics' shoebox ISM and shaped after torchaudio's old
prototype ``simulate_rir_ism``; it has not been checked against either.  Room ``[0, Lx] x [0, Ly] x [0, Lz]``, walls
``(x=0, x=Lx, y=0, y=Ly, z=0, z=Lz)``, ``beta_w = sqrt(1 - alpha_w)``.  An image ``(n, p)`` (n in Z^3, p in {0, 1}^3) sits
at ``i_d = 2 n_d L_d + (1 - 2 p_d) s_d``, reflects ``|n_d - p_d|`` times off the low wall of axis d and ``|n_d|`` times
off the high one, and adds ``g w[k] sinc(k - half - frac(tau))`` at ``floor(tau) + k`` (k < W), with
``g = prod beta^count / (4 pi r)``, ``r = |i - m|``, ``tau = r fs / c`` and ``w = np.hanning(W)``.

tau is formed here with exactly the kernel's operation order, each step rounded once, so ``floor(tau)`` and
``frac(tau)`` agree bit for bit; everything else is plain float64.

Error bound.  The kernel forms a tap as ``A ws[k] rcp(jj - e)`` in float32, with A = g sin(pi e) / pi and ws = w with
a sign, each rounded once from float64 (u = 2^-24 each), their product (u), the denominator (the rounded e and the
subtraction: at most 2u relative, since |jj - e| >= |e| and |jj - e| >= 1/2), the approximate reciprocal (at most 2
ulp, 4u) and the last product (u): ``|tap' - tap| <= 10u |tap|`` to first order, taken as ``EPS_TAP = 11 u``.  A
sample's n taps are summed in float32 in a fixed order, which adds at most ``gamma_(n-1) sum |tap'|`` with
``gamma_j = j u / (1 - j u)``.  So ``|h' - h| <= (EPS_TAP + gamma_(n-1) (1 + EPS_TAP)) sum |tap|`` per sample.
"""
import math

import numpy as np

U = 2.0 ** -24
EPS_TAP = 11 * U
REC = 14


def hanning(W):
    return np.hanning(W) if W > 1 else np.ones(1)


def betas(absorption):
    """Pressure reflection coefficients of energy absorptions in [0, 1]."""
    return np.sqrt(1.0 - np.asarray(absorption, np.float64))


def inverse_sabine(rt60, room, sound_speed=343.0):
    """alpha = 24 ln(10) V / (c S rt60)."""
    Lx, Ly, Lz = (float(v) for v in room)
    V, S = Lx * Ly * Lz, 2.0 * (Lx * Ly + Ly * Lz + Lx * Lz)
    return 24.0 * math.log(10.0) * V / (sound_speed * S * rt60)


def sabine_rt60(alpha, room, sound_speed=343.0):
    Lx, Ly, Lz = (float(v) for v in room)
    V, S = Lx * Ly * Lz, 2.0 * (Lx * Ly + Ly * Lz + Lx * Lz)
    return 24.0 * math.log(10.0) * V / (sound_speed * S * alpha)


def record(room, source, beta, max_order=None, start=0):
    """One item's float64 record as the kernel reads it."""
    r = np.zeros(REC, np.float64)
    r[0:3], r[3:6], r[6:12] = room, source, beta
    r[12] = -1.0 if max_order is None else float(max_order)
    r[13] = float(start)
    return r


def _nrange(L, s, m, R):
    return int(math.floor((-R + m - s) / (2 * L))) - 1, int(math.ceil((R + m + s) / (2 * L))) + 1


def images(room, source, mic, beta, fs, c=343.0, max_order=None, t_end=None):
    """Every image of order <= max_order (None: any) with floor(tau) < t_end, as arrays
    (n (N, 3), p (N, 3), tau, g, order).  t_end = None needs max_order."""
    room, source, mic = (np.asarray(v, np.float64) for v in (room, source, mic))
    beta = np.asarray(beta, np.float64)
    if t_end is None:
        R = None
        rng = [(-max_order - 1, max_order + 1)] * 3
    else:
        R = t_end * c / fs * (1 + 1e-9)
        rng = [_nrange(room[d], source[d], mic[d], R) for d in range(3)]
    ax = []
    for d in range(3):
        n = np.arange(rng[d][0], rng[d][1] + 1)
        n, p = np.repeat(n, 2), np.tile([0, 1], n.size)
        dd = ((2.0 * n) * room[d] + np.where(p == 1, -source[d], source[d])) - mic[d]
        lo, hi = np.abs(n - p), np.abs(n)
        ax.append((n, p, dd, lo, hi))
    out = []
    nx, px, dx, lox, hix = ax[0]
    ny, py, dy, loy, hiy = ax[1]
    nz, pz, dz, loz, hiz = ax[2]
    for i in range(nx.size):
        q = dx[i] * dx[i] + dy[:, None] * dy[:, None]
        r = np.sqrt(q + dz[None, :] * dz[None, :])
        tau = (r * fs) / c
        order = (lox[i] + hix[i]) + (loy + hiy)[:, None] + (loz + hiz)[None, :]
        keep = np.ones(tau.shape, bool)
        if t_end is not None:
            keep &= np.floor(tau) < t_end
        if max_order is not None:
            keep &= order <= max_order
        jy, jz = np.nonzero(keep)
        if jy.size == 0:
            continue
        g = (beta[0] ** lox[i] * beta[1] ** hix[i]) * beta[2] ** loy[jy] * beta[3] ** hiy[jy] \
            * beta[4] ** loz[jz] * beta[5] ** hiz[jz] / (4 * np.pi * r[jy, jz])
        n = np.stack([np.full(jy.size, nx[i]), ny[jy], nz[jz]], 1)
        p = np.stack([np.full(jy.size, px[i]), py[jy], pz[jz]], 1)
        out.append((n, p, tau[jy, jz], g, order[jy, jz]))
    if not out:
        z = np.zeros((0, 3), np.int64)
        return z, z, np.zeros(0), np.zeros(0), np.zeros(0, np.int64)
    return tuple(np.concatenate([o[k] for o in out]) for k in range(5))


def rir(room, source, mic, beta, length, W=81, fs=16000.0, c=343.0, max_order=None, start=0, with_bound=True):
    """Samples [start, start + length) of one response: (h, bound) float64, bound the elementwise error bound of the
    kernel's float32 output (None without with_bound)."""
    _, _, tau, g, _ = images(room, source, mic, beta, fs, c, max_order, start + length)
    half = (W - 1) // 2
    w = hanning(W)
    h = np.zeros(length)
    sa = np.zeros(length)
    cnt = np.zeros(length, np.int64)
    n0 = np.floor(tau)
    f = tau - n0
    k = np.arange(W)
    for s in range(0, tau.size, 1 << 14):
        sl = slice(s, s + (1 << 14))
        idx = (n0[sl, None] + k[None, :]).astype(np.int64) - start
        tap = g[sl, None] * w[None, :] * np.sinc(k[None, :] - half - f[sl, None])
        ok = (idx >= 0) & (idx < length)
        np.add.at(h, idx[ok], tap[ok])
        if with_bound:
            np.add.at(sa, idx[ok], np.abs(tap[ok]))
            np.add.at(cnt, idx[ok], 1)
    if not with_bound:
        return h, None
    n = np.maximum(cnt - 1, 0).astype(np.float64)
    gamma = n * U / (1 - n * U)
    return h, (EPS_TAP + gamma * (1 + EPS_TAP)) * sa + 1e-37


def image_count(N):
    """Images of order <= N: sum over c_x + c_y + c_z <= N of prod_d (1 if c_d = 0 else 2)."""
    tot = 0
    for cx in range(N + 1):
        for cy in range(N + 1 - cx):
            for cz in range(N + 1 - cx - cy):
                tot += (1 if cx == 0 else 2) * (1 if cy == 0 else 2) * (1 if cz == 0 else 2)
    return tot


# ---- self-checks of the restatement ------------------------------------------------------------------------------
def _close(a, b, tol=1e-12):
    return np.max(np.abs(a - b)) <= tol * max(np.max(np.abs(a)), 1e-300)


def check_reciprocity():
    room, s, m = (4.0, 3.5, 2.7), (1.1, 2.3, 1.4), (2.9, 0.8, 1.9)
    beta = betas([0.1, 0.3, 0.2, 0.5, 0.05, 0.4])
    a, _ = rir(room, s, m, beta, 600, fs=8000.0, with_bound=False)
    b, _ = rir(room, m, s, beta, 600, fs=8000.0, with_bound=False)
    assert _close(a, b)


def check_mirror_symmetry():
    room, s, m = (4.0, 3.5, 2.7), (1.1, 2.3, 1.4), (2.9, 0.8, 1.9)
    al = np.array([0.1, 0.3, 0.2, 0.5, 0.05, 0.4])
    a, _ = rir(room, s, m, betas(al), 600, fs=8000.0, with_bound=False)
    s2, m2 = (room[0] - s[0],) + s[1:], (room[0] - m[0],) + m[1:]
    b, _ = rir(room, s2, m2, betas(al[[1, 0, 2, 3, 4, 5]]), 600, fs=8000.0, with_bound=False)
    assert _close(a, b)


def check_full_absorption_is_the_direct_path():
    room, s, m = (5.0, 4.0, 3.0), (1.0, 1.5, 1.2), (3.5, 2.0, 1.7)
    h, _ = rir(room, s, m, np.zeros(6), 400, W=81, fs=16000.0, with_bound=False)
    r = math.dist(s, m)
    tau = r * 16000.0 / 343.0
    n0, f = math.floor(tau), tau - math.floor(tau)
    want = np.zeros(400)
    k = np.arange(81)
    want[n0 + k] = hanning(81) * np.sinc(k - 40 - f) / (4 * np.pi * r)
    assert _close(h, want, 1e-15)


def check_image_count():
    for N in (0, 1, 2, 5, 9):
        n, p, tau, g, order = images((3.0, 4.0, 5.0), (1.0, 1.0, 1.0), (2.0, 2.0, 2.0), np.ones(6), 16000.0,
                                     max_order=N)
        assert tau.size == image_count(N)
    assert [image_count(N) for N in range(4)] == [1, 7, 25, 63]


def check_beta_zero_with_zero_count_is_one():
    beta = np.array([0.0, 1.0, 0.0, 1.0, 0.0, 1.0])
    n, p, tau, g, order = images((3.0, 4.0, 5.0), (1.0, 1.0, 1.0), (2.0, 2.0, 2.0), beta, 16000.0, max_order=2)
    assert np.all(np.isfinite(g))
    assert np.count_nonzero(g) >= 1


def check_inverse_sabine_round_trip():
    for room, rt in (((5.0, 4.0, 3.0), 0.5), ((3.0, 3.0, 2.5), 0.8), ((10.0, 10.0, 4.0), 0.2)):
        a = inverse_sabine(rt, room)
        assert 0 < a <= 1
        assert abs(sabine_rt60(a, room) - rt) <= 1e-12 * rt
