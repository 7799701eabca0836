"""Float64 restatement of the multirate constant-Q transform (kapre_b200's CQT), in torch so that autograd gives its
exact vector-Jacobian products, and the error bounds of the float32 kernels.

    y_0 = x,  y_{i+1} = resample_poly(y_i, 1, 2) with the float32 taps of resample_filter(1, 2)
    C[k, m] = sum_{j < N_i} y_i[m h_i + j - N_i // 2] T_k[j]    (T: the complex64 tables the plan uploads)

Error bound.  Write u = 2^-24 and g(n) = n u / (1 - n u).  Level 0 is exact.  A resampled level is a float32 sum of at
most K = 44 products (4 partial sums), so with E_i the bound on |y_i(float32) - y_i|, elementwise,
    E_{i+1} <= |h| * E_i + g(K) |h| * |y_i|                     (* the resampling operator)
and since every filter has unit L1 norm (times s_k), each component of an output, a float32 dot product of N_i terms,
    |dC| <= sum_j (|T_k[j].re| + |T_k[j].im|) (E_i + g(N_i + 1) |y_i|)[m h_i + j - N_i // 2].
|C| adds 3 u |C|.  The adjoint runs the same way backwards: at octave i each sample sums at most
n_i = 2 (bins) ceil(N_i / h_i) products plus the addend R^T g_{i+1}, so with F_i the bound on the level gradient,
    F_i <= g(n_i + 2) (|A_i|^T |G| + |R|^T |g_{i+1}|) + |R|^T F_{i+1} + g(K) |R|^T |g_{i+1}|
where |A_i| and |R| are the operators with absolute taps.  The magnitude mode's G = g C / |C| from the kernel's C
moves by at most 2 |g| |dC| / (|C| - |dC|) (capped at 2 |g|), which enters |A_i|^T |G| as an extra term.
"""
import numpy as np
import torch

import resample_ref
from kapre_b200.signal import resample_filter

U = 2.0 ** -24
K_DECIM = 44


def gam(n):
    return n * U / (1 - n * U)


def decimator():
    return torch.from_numpy(resample_filter(1, 2).astype(np.float64))


def pyramid(x, n_oct, h=None):
    """x: (B, C, L) float64 -> [y_0, ..., y_{n_oct - 1}]."""
    h = decimator() if h is None else h
    levels = [x]
    for _ in range(1, n_oct):
        levels.append(resample_ref.resample(levels[-1], 1, 2, h=h))
    return levels


def _frames(y, M, hop, N):
    """(B, C, M, N) frames y[m hop + j - N // 2], zeros outside the signal."""
    half = N // 2
    L = y.shape[-1]
    right = max(0, (M - 1) * hop + N - half - L)
    yp = torch.nn.functional.pad(y, (half, right))
    return yp.unfold(-1, N, hop)[..., :M, :]


def tables(plan):
    """The complex64 tables the plan uploads, as complex128 tensors, top octave first."""
    return [torch.from_numpy(t.astype(np.complex128)) for t in plan.tables]


def apply(levels, tabs, hop, M):
    """C: (B, C, M, n_bins) complex128 from the levels and tables."""
    outs = []
    for i in reversed(range(len(tabs))):
        T = tabs[i]
        fr = _frames(levels[i], M, hop >> i, T.shape[1])
        outs.append(torch.complex(fr @ T.real.T, fr @ T.imag.T))
    return torch.cat(outs, dim=-1)


def cqt(x, plan, magnitude=False):
    """x: (B, C, L) float64 tensor -> (B, C, M, n_bins) complex128 (or |C| float64)."""
    M = plan.num_frames(x.shape[-1])
    C = apply(pyramid(x, plan.n_octaves), tables(plan), plan.hop_length, M)
    return C.abs() if magnitude else C


def forward_bound(x, plan, magnitude=False):
    """Elementwise bound on |kernel - restatement| for the forward, (B, C, M, n_bins) float64."""
    with torch.no_grad():
        n_oct, hop = plan.n_octaves, plan.hop_length
        M = plan.num_frames(x.shape[-1])
        habs = decimator().abs()
        levels = pyramid(x, n_oct)
        E = [torch.zeros_like(x)]
        for i in range(1, n_oct):
            E.append(resample_ref.resample(E[-1], 1, 2, h=habs) + gam(K_DECIM) * resample_ref.resample(
                levels[i - 1].abs(), 1, 2, h=habs))
        outs = []
        for i in reversed(range(n_oct)):
            T = tables(plan)[i]
            N = T.shape[1]
            w = (T.real.abs() + T.imag.abs())
            fr = _frames(E[i] + gam(N + 1) * levels[i].abs(), M, hop >> i, N)
            outs.append(fr @ w.T)
        b = torch.cat(outs, dim=-1)
        if magnitude:
            b = b + 3 * U * apply(levels, tables(plan), hop, M).abs()
        return b


def vjp(x, plan, g, magnitude=False):
    """Exact gradient of sum(Re(conj(g) C)) (complex g, torch's convention) or sum(g |C|) to x."""
    xt = x.detach().clone().requires_grad_(True)
    y = cqt(xt, plan, magnitude)
    (torch.real(torch.conj(g) * y) if not magnitude else g * y).sum().backward()
    return xt.grad


def backward_bound(x, plan, g, magnitude=False):
    """Elementwise bound on |kernel gradient - exact gradient|, (B, C, L) float64."""
    n_oct, hop = plan.n_octaves, plan.hop_length
    L = x.shape[-1]
    M = plan.num_frames(L)
    habs = decimator().abs()
    levels = [lv.detach() for lv in pyramid(x.detach(), n_oct)]
    tabs = tables(plan)
    with torch.no_grad():
        if magnitude:
            C = apply(levels, tabs, hop, M)
            dC = forward_bound(x.detach(), plan)
            mag = C.abs()
            G = (g * C / torch.where(mag > 0, mag, torch.ones_like(mag))).abs()
            dG = torch.minimum(2 * g.abs() * dC / torch.clamp(mag - dC, min=1e-300), 2 * g.abs())
            Gabs = G
        else:
            Gabs, dG = g.abs(), torch.zeros_like(g.abs())
    lv_abs = [torch.zeros_like(lv).requires_grad_(True) for lv in levels]
    # |A_i|^T |G| per level: the VJP of the forward with absolute taps
    Cabs = apply(lv_abs, [torch.complex(t.abs(), torch.zeros_like(t.real)) for t in tabs], hop, M)
    grads = torch.autograd.grad(torch.real(Cabs * Gabs).sum(), lv_abs, retain_graph=True)
    dgrads = torch.autograd.grad(torch.real(Cabs * dG).sum(), lv_abs)
    # the exact level gradients g_i (g_0 = the input gradient) by the same chain without rounding
    lv_ex = [lv.clone().requires_grad_(True) for lv in levels]
    Cex = apply(lv_ex, tabs, hop, M)
    obj = (torch.real(torch.conj(g) * Cex) if not magnitude else g * Cex.abs()).sum()
    direct = torch.autograd.grad(obj, lv_ex)
    with torch.no_grad():

        def rt(v, length):          # |R|^T v
            z = torch.zeros(v.shape[:-1] + (length,), dtype=v.dtype, requires_grad=True)
            with torch.enable_grad():
                out = resample_ref.resample(z, 1, 2, h=habs)
                return torch.autograd.grad((out * v).sum(), z)[0]

        def rt_exact(v, length):    # R^T v
            z = torch.zeros(v.shape[:-1] + (length,), dtype=v.dtype, requires_grad=True)
            with torch.enable_grad():
                out = resample_ref.resample(z, 1, 2, h=decimator())
                return torch.autograd.grad((out * v).sum(), z)[0]

        F = None
        gnext = None
        for i in reversed(range(n_oct)):
            N = tabs[i].shape[1]
            n_i = 2 * tabs[i].shape[0] * (-(-N // (hop >> i))) + 2
            Li = levels[i].shape[-1]
            gi = direct[i].clone()
            base = grads[i].clone()
            if gnext is not None:
                gi = gi + rt_exact(gnext, Li)
                addabs = rt(gnext.abs(), Li)
                Fi = gam(n_i) * (base + addabs) + dgrads[i] + rt(F, Li) + gam(K_DECIM) * addabs
            else:
                Fi = gam(n_i) * base + dgrads[i]
            F, gnext = Fi, gi
        return F
