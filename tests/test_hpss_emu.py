"""HPSS on the CPU: the kernel bodies of hpss_core.cuh (run by a CPU emulation) against the restatements of
hpss_ref.py: the medians (through the elements the gradient pass selects) equal to scipy's median_filter, masks and
outputs bit for bit at power 1, 2 and inf and within a bound at 0.5 and 3, tile orders and CTA counts, NaN isolation,
the gradient against torch.autograd of the float64 restatement, and validation."""
import ctypes
import hashlib
import os
import subprocess
import tempfile

import numpy as np
import pytest
import scipy.ndimage
import torch

import hpss_ref as R
from emu_harness import Checked, emu_cabs
from kapre_b200 import ops, signal, time_frequency

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, 'emu', 'kb_emu_hpss.cpp')
_CSRC = os.path.join(_HERE, '..', 'kapre_b200', 'csrc')
_lib_handle = None
CL, CF = 'channels_last', 'channels_first'
POW_CODE = {1.0: 1, 2.0: 2}
KMAX = 64


def _lib():
    """tests/emu/kb_emu_hpss.cpp built with g++ into the temporary directory (keyed by the sources' contents)."""
    global _lib_handle
    if _lib_handle is None:
        hs = hashlib.sha256()
        for f in [_SRC] + sorted(os.path.join(_CSRC, n) for n in os.listdir(_CSRC) if n.endswith(('.h', '.cuh'))):
            with open(f, 'rb') as fh:
                hs.update(fh.read())
        out = os.path.join(tempfile.gettempdir(), 'kapre_b200_emu_hpss_%s.so' % hs.hexdigest()[:16])
        if not os.path.exists(out):
            tmp = '%s.%d.tmp' % (out, os.getpid())
            subprocess.check_call(['g++', '-O2', '-std=c++17', '-shared', '-fPIC', '-DKB_HOST_EMU', '-Wno-unknown-pragmas',
                                   '-o', tmp, _SRC])
            os.replace(tmp, out)
        lib = ctypes.CDLL(out)
        lib.kb_emu_hpss.argtypes = [ctypes.c_void_p] * 8 + [ctypes.c_int] * 2
        lib.kb_emu_hpss_bwd.argtypes = [ctypes.c_void_p] * 11 + [ctypes.c_int] * 2
        _lib_handle = Checked(lib)
    return _lib_handle


def _p(a):
    return None if a is None else ctypes.c_void_p(a.__array_interface__['data'][0])


def _layout(a, fmt):
    """Canonical (B, C, T, K) -> the array in ``fmt`` and its element strides (b, c, t, k)."""
    x = np.ascontiguousarray(np.transpose(a, (0, 2, 3, 1))) if fmt == CL else np.ascontiguousarray(a)
    st = [s // x.itemsize for s in x.strides]
    return x, np.array([st[0], st[3], st[1], st[2]] if fmt == CL else st, np.int64)


def _canon(x, fmt):
    return np.transpose(x, (0, 3, 1, 2)) if fmt == CL else x


def _cfg(x, kh, kp, power, margin, mask):
    B, C, T, K = x.shape
    pm = 3 if np.isinf(power) else POW_CODE.get(float(power), 0)
    ic = np.array([B, C, T, K, kh, kp, pm, int(margin[0] == 1 and margin[1] == 1), int(np.iscomplexobj(x)),
                   int(mask)], np.int32)
    fc = np.array([margin[0], margin[1], power], np.float32)
    return ic, fc


def emu_hpss(x, kh, kp, power=2.0, margin=(1.0, 1.0), mask=False, fmt=CF, order=0, n_cta=0, want=(True, True),
             xin=None):
    """(harmonic, percussive) of canonical x (B, C, T, K), float32 or complex64, in canonical layout."""
    ic, fc = _cfg(x, kh, kp, power, margin, mask)
    if xin is None:
        xin, xs = _layout(x, fmt)
    else:
        xin, xs = xin
    dt = np.float32 if mask else x.dtype
    outs = []
    for w in want:
        outs.append(_layout(np.full(x.shape, np.nan, dt), fmt) if w else (None, None))
    rc = _lib().kb_emu_hpss(_p(ic), _p(fc), _p(xin), _p(xs), _p(outs[0][0]), _p(outs[0][1]), _p(outs[1][0]),
                            _p(outs[1][1]), order, n_cta)
    assert rc == 0
    return tuple(None if o[0] is None else _canon(o[0], fmt) for o in outs)


def emu_hpss_bwd(x, gh, gp, kh, kp, power=2.0, margin=(1.0, 1.0), mask=False, fmt=CF, order=0, n_cta=0):
    """(gS canonical, srcH, srcP) with the selected indices (B, C, T, K) read from the workspace."""
    ic, fc = _cfg(x, kh, kp, power, margin, mask)
    xin, xs = _layout(x, fmt)
    g = [(None, None) if v is None else _layout(v, fmt) for v in (gh, gp)]
    gx, gxs = _layout(np.full(x.shape, np.nan, x.dtype), fmt)
    n = x.size
    ws = np.zeros(4 * n, np.int32)
    rc = _lib().kb_emu_hpss_bwd(_p(ic), _p(fc), _p(xin), _p(xs), _p(g[0][0]), _p(g[0][1]), _p(g[1][0]), _p(g[1][1]),
                                _p(gx), _p(gxs), _p(ws), order, n_cta)
    assert rc == 0
    src = ws.reshape(2, n, 2)[:, :, 1].reshape((2,) + x.shape)
    return _canon(gx, fmt), src[0], src[1]


def _mag(x):
    if np.iscomplexobj(x):
        return emu_cabs(x.real.astype(np.float32), x.imag.astype(np.float32), 0)
    return x


def _data(rng, shape, cplx=False, ties=False):
    if ties:
        v = rng.integers(0, 4, size=shape).astype(np.float32) * np.float32(0.25)
    else:
        v = rng.random(shape, dtype=np.float32)
    if cplx:
        ph = rng.uniform(-np.pi, np.pi, size=shape)
        return (v * np.cos(ph) + 1j * v * np.sin(ph)).astype(np.complex64)
    return v


# ---- medians --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('kh,kp', [(1, 1), (2, 2), (31, 31), (4, 7), (KMAX, KMAX), (17, 63), (33, 32)])
@pytest.mark.parametrize('T,K', [(70, 130), (1, 5), (2, 3), (3, 2), (65, 1)])
def test_medians_equal_scipy(kh, kp, T, K):
    """The element each median selected holds scipy's median.  Where a window reaches past one reflection (a row
    shorter than half a window) scipy 1.x's line extension reads outside its buffer, so those rows are checked
    against the period-2n restatement alone; a single frame gives that frame itself."""
    rng = np.random.default_rng(kh * 1000 + kp + T)
    x = _data(rng, (2, 1, T, K))
    _, sh, sp = emu_hpss_bwd(x, None, None, kh, kp)
    H = np.take_along_axis(x, sh, axis=2)
    P = np.take_along_axis(x, sp, axis=3)
    rh, rp = R.medians(x, kh, kp)
    np.testing.assert_array_equal(H, rh)
    np.testing.assert_array_equal(P, rp)
    if T == 1:
        np.testing.assert_array_equal(H, x)
    for b in range(2):
        if (kh - 1) - kh // 2 <= T and kh // 2 <= T:
            np.testing.assert_array_equal(H[b, 0], scipy.ndimage.median_filter(x[b, 0], size=(kh, 1), mode='reflect'))
        if (kp - 1) - kp // 2 <= K and kp // 2 <= K:
            np.testing.assert_array_equal(P[b, 0], scipy.ndimage.median_filter(x[b, 0], size=(1, kp), mode='reflect'))


@pytest.mark.parametrize('kh,kp', [(31, 31), (4, 6), (KMAX, 3)])
def test_selected_element_follows_tie_rule(kh, kp):
    rng = np.random.default_rng(5)
    x = _data(rng, (1, 2, 40, 70), ties=True)
    x[0, 0, 10:30, :] = 0.0                                      # a zero region
    x[0, 1, :, 20:50] = 0.5                                      # a constant region
    _, sh, sp = emu_hpss_bwd(x, None, None, kh, kp)
    rh, rp = R.select(x, kh, kp)
    np.testing.assert_array_equal(sh, rh)
    np.testing.assert_array_equal(sp, rp)


# ---- masks and outputs ------------------------------------------------------------------------------------------
@pytest.mark.parametrize('power', [1.0, 2.0, np.inf])
@pytest.mark.parametrize('margin', [(1.0, 1.0), (2.0, 1.0), (1.0, 3.5)])
@pytest.mark.parametrize('cplx', [False, True])
@pytest.mark.parametrize('mask', [False, True])
def test_outputs_bit_exact(power, margin, cplx, mask):
    rng = np.random.default_rng(11)
    x = _data(rng, (2, 2, 67, 70), cplx=cplx)
    x[0, 0, :, :20] = 0                                          # an all-zero tile corner (split_zeros)
    x[1, 1, 5:30, 10:40] *= np.float32(2.0 ** -130)              # subnormal magnitudes
    ref = R.hpss32(_mag(x), x if cplx else None, 31, 31, power, margin, mask)
    for fmt in (CF, CL):
        got = emu_hpss(x, 31, 31, power, margin, mask, fmt=fmt)
        for g, r in zip(got, ref):
            np.testing.assert_array_equal(g, r)


@pytest.mark.parametrize('power', [0.5, 3.0])
def test_outputs_generic_power_within_bound(power):
    """powf of the emulation (and of the device) against numpy's: each power is within 2 ulp, which moves the mask
    pa / (pa + pb) by at most 4 ulp of 1 plus its own rounding."""
    rng = np.random.default_rng(3)
    x = _data(rng, (1, 1, 50, 90))
    Mh, Mp = emu_hpss(x, 13, 9, power, (1.0, 2.0), True)
    rh, rp = R.hpss32(x, None, 13, 9, power, (1.0, 2.0), True)
    bound = 6 * np.finfo(np.float32).eps
    assert np.abs(Mh - rh).max() <= bound and np.abs(Mp - rp).max() <= bound


def test_strided_input_and_single_component():
    rng = np.random.default_rng(2)
    x = _data(rng, (2, 1, 40, 80))
    big = np.zeros((2, 3, 45, 90), np.float32)
    big[:, 1, 2:42, 5:85] = x[:, 0]
    st = np.array([s // 4 for s in big.strides], np.int64)
    view = big[:, 1:2, 2:42, 5:85]
    base = np.ascontiguousarray(big)
    xin = (base[:, 1:, 2:, 5:], st)                               # pointer at (0, 1, 2, 5), parent strides
    h, p = emu_hpss(view.copy(), 31, 31, xin=xin)
    rh, rp = R.hpss32(x, None, 31, 31, 2.0)
    np.testing.assert_array_equal(h, rh)
    np.testing.assert_array_equal(p, rp)
    h1, p1 = emu_hpss(x, 31, 31, want=(False, True))
    assert h1 is None
    np.testing.assert_array_equal(p1, rp)


@pytest.mark.parametrize('order,n_cta', [(0, 0), (1, 0), (2, 0), (0, 3), (1, 5)])
def test_tile_order_and_cta_count_invariance(order, n_cta):
    rng = np.random.default_rng(4)
    x = _data(rng, (2, 2, 150, 140), cplx=True)
    ref = emu_hpss(x, 31, 31)
    got = emu_hpss(x, 31, 31, fmt=CL, order=order, n_cta=n_cta)
    for g, r in zip(got, ref):
        np.testing.assert_array_equal(g, r)
    # an item's output does not depend on its batch position
    solo = emu_hpss(x[1:], 31, 31)
    np.testing.assert_array_equal(solo[0], ref[0][1:])
    gref = emu_hpss_bwd(x, x, x, 31, 31)[0]
    ggot = emu_hpss_bwd(x, x, x, 31, 31, fmt=CL, order=order, n_cta=n_cta)[0]
    np.testing.assert_array_equal(ggot, gref)


def test_nan_isolation_on_short_row():
    """A NaN makes NaN exactly the outputs whose harmonic or percussive window holds it, reflected copies
    included, and changes nothing else."""
    rng = np.random.default_rng(6)
    x = _data(rng, (1, 1, 9, 70))
    x[0, 0, 1, 3] = np.nan
    h, p = emu_hpss(x, 31, 7)
    wh = R.windows(9, 31)
    wp = R.windows(70, 7)
    hit = np.zeros((9, 70), bool)
    hit[:, 3] |= (wh == 1).any(axis=1)
    hit[1, :] |= (wp == 3).any(axis=1)
    assert hit[:, 3].all()                                       # the short row reflects the NaN into every window
    np.testing.assert_array_equal(np.isnan(h[0, 0]), hit)
    np.testing.assert_array_equal(np.isnan(p[0, 0]), hit)
    clean = x.copy()
    clean[0, 0, 1, 3] = 0.5
    rh, rp = emu_hpss(clean, 31, 7)
    np.testing.assert_array_equal(h[0, 0][~hit], rh[0, 0][~hit])


# ---- gradient ---------------------------------------------------------------------------------------------------
def _grad_ref(x, gh, gp, kh, kp, power, margin, mask):
    S = _mag(x)
    sh, sp = R.select(S, kh, kp)
    if np.iscomplexobj(x):
        X = torch.tensor(x.astype(np.complex128), requires_grad=True)
        h, p = R.hpss64(None, sh, sp, kh, kp, power, margin, mask, X=X)
        leaf = X
    else:
        leaf = torch.tensor(S.astype(np.float64), requires_grad=True)
        h, p = R.hpss64(leaf, sh, sp, kh, kp, power, margin, mask)
    dt = torch.float64 if mask or not np.iscomplexobj(x) else torch.complex128
    loss = 0
    for o, g in ((h, gh), (p, gp)):
        if g is not None:
            gt = torch.tensor(g.astype(np.complex128 if dt == torch.complex128 else np.float64))
            loss = loss + (o * gt.conj()).real.sum() if dt == torch.complex128 else loss + (o * gt).sum()
    loss.backward()
    return leaf.grad.numpy()


@pytest.mark.parametrize('power', [1.0, 2.0, 0.5, 3.0])
@pytest.mark.parametrize('cplx,mask', [(False, False), (True, False), (False, True), (True, True)])
@pytest.mark.parametrize('margin', [(1.0, 1.0), (2.0, 1.5)])
def test_gradient_against_autograd(power, cplx, mask, margin):
    rng = np.random.default_rng(8)
    shape = (1, 2, 40, 75)
    x = _data(rng, shape, cplx=cplx, ties=True)
    x[0, 0, :12, :30] = 0                                        # zero medians and Z < FLT_MIN
    gdt = np.float32 if mask or not cplx else np.complex64
    gh = _data(rng, shape, cplx=gdt is np.complex64).astype(gdt) - 0.5
    gp = _data(rng, shape, cplx=gdt is np.complex64).astype(gdt) - 0.5
    got = emu_hpss_bwd(x, gh, gp, 9, 13, power, margin, mask)[0]
    ref = _grad_ref(x, gh, gp, 9, 13, power, margin, mask)
    # each term is a handful of float32 products and quotients of O(1) values with derivatives bounded by p / Z
    # (Z >= the smallest non-zero magnitude, 0.25 here), gathered over at most 2 (2k - 1) terms
    # where autograd's derivative is infinite or undefined (a zero median with p < 1, |X| at X = 0) the kernels take 0
    assert np.isfinite(got).all()
    ok = np.isfinite(ref)
    assert (ok | (x == 0) | (power < 1)).all()
    assert np.max(np.abs(got - ref)[ok] / (1.0 + np.abs(ref[ok]))) < 2e-4 * (2 * (9 + 13))
    # with one gradient absent
    got1 = emu_hpss_bwd(x, gh, None, 9, 13, power, margin, mask)[0]
    ref1 = _grad_ref(x, gh, None, 9, 13, power, margin, mask)
    ok = np.isfinite(ref1)
    assert np.max(np.abs(got1 - ref1)[ok] / (1.0 + np.abs(ref1[ok]))) < 2e-4 * (2 * (9 + 13))


def test_gradient_lands_on_selected_element():
    """The gradients of H and P at one output go to the elements the tie rule selects, on constant columns."""
    x = np.full((1, 1, 20, 10), 0.5, np.float32)
    x[0, 0, :, 3] = 0.25
    x[0, 0, :, 4] = 0.75                          # H at (7, 4): ten tied 0.75; P: (0.25, 0.75, 0.5) selects bin 5
    gh = np.zeros_like(x)
    gh[0, 0, 7, 4] = 1.0
    sh, sp = R.select(x, 5, 3)
    src = {(int(sh[0, 0, 7, 4]), 4), (7, int(sp[0, 0, 7, 4]))}
    assert src == {(7, 4), (7, 5)}
    g = emu_hpss_bwd(x, gh, None, 5, 3, 1.0, (1.0, 1.0), True)[0]
    assert {tuple(int(i) for i in v) for v in np.argwhere(g[0, 0] != 0)} == src
    g = emu_hpss_bwd(x, gh, None, 5, 3, 1.0, (1.0, 1.0), False)[0]
    assert {tuple(int(i) for i in v) for v in np.argwhere(g[0, 0] != 0)} <= src   # the direct term lands on (7, 4)


def test_restatement_gradcheck():
    rng = np.random.default_rng(9)
    S = rng.random((1, 1, 12, 14)) + 0.1                            # tie-free
    sh, sp = R.select(S.astype(np.float32), 5, 3)
    for power, mask in ((2.0, False), (0.7, True), (1.0, False)):
        def f(s):
            h, p = R.hpss64(s, sh, sp, 5, 3, power, (1.0, 1.5), mask)
            return h.sum() + 2 * p.sum()
        assert torch.autograd.gradcheck(f, (torch.tensor(S, requires_grad=True),))


# ---- validation -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('kw', [dict(kernel_size=0), dict(kernel_size=KMAX + 1), dict(kernel_size=(31, KMAX + 1)),
                                dict(kernel_size=2.5), dict(kernel_size=(1, 2, 3)), dict(margin=0.5),
                                dict(margin=(1.0, np.inf)), dict(margin=np.nan), dict(power=0.0),
                                dict(power=-1.0), dict(power=np.nan)])
def test_validation_raises_before_launch(kw):
    S = torch.zeros((1, 4, 5, 1))                                 # a CPU tensor: a launch would fail differently
    with pytest.raises(ValueError):
        signal.hpss(S, **kw)
    with pytest.raises(ValueError):
        ops.hpss_config(**kw)


def test_validation_of_input_and_layer():
    with pytest.raises(ValueError):
        signal.hpss(torch.zeros((4, 5, 1)))                      # not 4-D
    with pytest.raises(ValueError):
        signal.hpss(torch.zeros((1, 4, 5, 1), dtype=torch.float64))
    with pytest.raises(ValueError):
        signal.hpss(torch.zeros((1, 4, 5, 1)))                   # not on CUDA
    with pytest.raises(ValueError):
        time_frequency.HPSS('residual')
    with pytest.raises(ValueError):
        time_frequency.HPSS(kernel_size=KMAX + 1)
    assert ops.hpss_config(kernel_size=KMAX).kernel_h == KMAX
    with pytest.raises(ValueError):
        signal.harmonic(torch.zeros((1, 4000, 1)), n_fft=512, win_length=256, hop_length=300)


def test_layer_config_round_trip():
    layer = time_frequency.HPSS('percussive', kernel_size=(17, 63), power=np.inf, mask=True, margin=(1.0, 2.0),
                                data_format='channels_first')
    cfg = layer.get_config()
    again = time_frequency.HPSS.from_config(cfg)
    assert again.get_config() == cfg
    assert (again.cfg.kernel_h, again.cfg.kernel_p, again.cfg.mask) == (17, 63, 1)
    import kapre
    assert kapre.time_frequency.HPSS is time_frequency.HPSS
