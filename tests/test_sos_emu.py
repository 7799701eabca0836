"""Second-order-section cascades on the CPU: the float64 restatement (sos_ref.py) against scipy's sosfilt, sosfilt_zi
and sosfiltfilt, the kernel bodies of sos_core.cuh (run by a CPU emulation) against the restatement within the derived
error bound (output, zf and the reverse flag), their bit-independence of grid, loader, batch position, strides,
broadcasting, format and length, per-item and per-channel coefficients, streaming through zf, the gradient identities,
validation before any launch and the register budget."""
import ctypes
import hashlib
import os
import re
import shutil
import subprocess
import tempfile

import numpy as np
import pytest
import scipy.signal
import torch

import sos_ref as SR
from emu_harness import Checked

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, 'emu', 'kb_emu_sos.cpp')
_CSRC = os.path.join(_HERE, '..', 'kapre_b200', 'csrc')
_LIB = os.path.join(_HERE, '..', 'kapre_b200', '_lib', 'libkapre_b200.so')
_lib_handle = None


def _lib():
    """tests/emu/kb_emu_sos.cpp built with g++ into the temporary directory (keyed by the sources' contents)."""
    global _lib_handle
    if _lib_handle is None:
        hs = hashlib.sha256()
        for f in [_SRC] + sorted(os.path.join(_CSRC, n) for n in os.listdir(_CSRC) if n.endswith(('.h', '.cuh'))):
            with open(f, 'rb') as fh:
                hs.update(fh.read())
        out = os.path.join(tempfile.gettempdir(), 'kapre_b200_emu_sos_%s.so' % hs.hexdigest()[:16])
        if not os.path.exists(out):
            tmp = '%s.%d.tmp' % (out, os.getpid())
            subprocess.check_call(['g++', '-O2', '-std=c++17', '-shared', '-fPIC', '-DKB_HOST_EMU', '-Wno-unknown-pragmas',
                                   '-o', tmp, _SRC])
            os.replace(tmp, out)
        lib = ctypes.CDLL(out)
        I, P, LL = ctypes.c_int, ctypes.c_void_p, ctypes.c_longlong
        lib.kb_emu_sosfilt.argtypes = [P, P, P, P, P, P, I, I, I, I, I, P, P, P, P, I, I, LL]
        lib.kb_emu_sos_powers.argtypes = [P, I, P]
        _lib_handle = Checked(lib)
    return _lib_handle


def _p(a):
    return ctypes.c_void_p(a.__array_interface__['data'][0]) if a is not None else None


def _es(a):
    return np.array([s // 4 for s in a.strides], np.int64)


def emu(x, sos, zi=None, reverse=False, tile_order=0, bulk=1, fmt='bcl', want_zf=False):
    """Run the bodies on float32 x (B, C, L) ('bcl') or (B, L, C) ('blc'; views allowed) with float32 sos
    (Bc, Cc, S, 6) and zi (Bz, Cz, S, 2) or None (axes of 1 broadcast through stride 0).  Returns (y (B, C, L), zf)."""
    if fmt == 'blc':
        B, L, C = x.shape
        xs = _es(x)[[0, 2, 1]]
    else:
        B, C, L = x.shape
        xs = _es(x)
    S = sos.shape[-2]
    y = np.full((B, C, L), np.nan, np.float32)
    cs = np.array([0 if sos.shape[0] == 1 else sos.strides[0] // 4, 0 if sos.shape[1] == 1 else sos.strides[1] // 4],
                  np.int64)
    zis = None
    if zi is not None:
        zis = np.array([0 if zi.shape[0] == 1 else zi.strides[0] // 4, 0 if zi.shape[1] == 1 else zi.strides[1] // 4,
                        zi.strides[2] // 4], np.int64)
    zf = np.full((B, C, S, 2), np.nan, np.float32) if want_zf else None
    zfs = _es(zf)[:3] if want_zf else None
    base = x if x.base is None else x.base
    numel = int(base.size) - (x.__array_interface__['data'][0] - base.__array_interface__['data'][0]) // 4
    rc = _lib().kb_emu_sosfilt(_p(x), _p(xs), _p(y), _p(_es(y)), _p(sos), _p(cs), S, B, C, L, 2 if reverse else 0,
                               _p(zi), _p(zis), _p(zf), _p(zfs), tile_order, bulk, numel)
    assert rc == 0
    return y, zf


def _filters():
    """(name, sos) float64 designs the tests run (rounded to float32 by the callers)."""
    return [('butter8-0.05', scipy.signal.butter(8, 0.05, output='sos')),
            ('butter8-telephone', scipy.signal.butter(8, [300, 3400], 'bandpass', fs=16000, output='sos')),
            ('ellip8', scipy.signal.ellip(8, 0.5, 60, 0.125, output='sos')),
            ('cheby2-narrow', scipy.signal.cheby2(4, 40, [0.02, 0.04], 'bandpass', output='sos')),
            ('highpass-20Hz-48k', scipy.signal.butter(4, 20, 'highpass', fs=48000, output='sos')),
            ('single', scipy.signal.butter(2, 0.1, output='sos'))]


FILTERS = _filters()
NAMES = [f[0] for f in FILTERS]


def _sos32(name):
    return next(s for n, s in FILTERS if n == name).astype(np.float32)


def _check(x, sos32, y, zi=None, zf=None, what=''):
    """y (and zf) against the float64 restatement on the float32 values, per column, within the derived bound."""
    xa = np.asarray(x, np.float64)
    z = None if zi is None else np.broadcast_to(np.asarray(zi, np.float64), xa.shape[:-1] + zi.shape[-2:])
    ref, zref = SR.sosfilt_fast(xa, sos32, z)
    by, bz = SR.error_bounds(xa, sos32, z)
    err = np.abs(y - ref).max(initial=0.0)
    assert err <= by, (what, err, by)
    if zf is not None:
        ez = np.abs(zf - zref).max(initial=0.0)
        assert ez <= bz, (what, 'zf', ez, bz)
    return err, by


# ------------------------------------------------------------------------------------------ the restatement
def test_restatement_matches_scipy():
    rng = np.random.default_rng(0)
    x = rng.uniform(-1, 1, (2, 3, 300))
    for name, sos in FILTERS:
        zi = rng.uniform(-1, 1, (2, 3, sos.shape[0], 2))
        y, zf = SR.sosfilt(x, sos, zi)
        ry, rzf = scipy.signal.sosfilt(sos, x, axis=-1, zi=np.moveaxis(zi, -2, 0))
        assert np.abs(y - ry).max() <= 1e-9 * max(1, np.abs(ry).max()), name
        assert np.abs(zf - np.moveaxis(rzf, 0, -2)).max() <= 1e-9 * max(1, np.abs(rzf).max()), name
        fy, fzf = SR.sosfilt_fast(x, sos, zi)
        assert np.abs(fy - ry).max() == 0 and np.abs(fzf - np.moveaxis(rzf, 0, -2)).max() == 0
        assert np.abs(SR.sosfilt_zi(sos) - scipy.signal.sosfilt_zi(sos)).max() <= 1e-9, name
        for padtype, padlen in (('odd', None), ('even', None), ('constant', 40), (None, None), ('odd', 0)):
            want = scipy.signal.sosfiltfilt(sos, x, axis=-1, padtype=padtype, padlen=padlen)
            got = SR.sosfiltfilt(x, sos, padtype, padlen)
            assert np.abs(got - want).max() <= 1e-8 * max(1, np.abs(want).max()), (name, padtype, padlen)
    # the padlen rule counts first-order sections
    sos = scipy.signal.butter(3, 0.2, output='sos')
    assert SR.n_taps(sos) == 2 * 2 + 1 - 1


def test_library_sosfilt_zi_is_scipy_s():
    from kapre_b200 import backend
    for name, sos in FILTERS:
        want = scipy.signal.sosfilt_zi(sos)
        assert np.abs(backend.sosfilt_zi(sos) - want).max() <= 1e-9 * max(1, np.abs(want).max()), name
        got = backend.sosfilt_zi(torch.from_numpy(sos)).numpy()
        assert np.abs(got - want).max() <= 1e-9 * max(1, np.abs(want).max()), name
        zi, gain = backend.sos_steady_state(np.stack([sos, sos]))
        assert zi.shape == (2,) + sos.shape[:1] + (2,) and gain.shape == (2,)
        want = np.prod(sos[:, :3].sum(1) / sos[:, 3:].sum(1))          # H(1), section by section
        assert abs(gain[0] - want) <= 1e-9 * max(1, abs(want))


def test_the_stated_test_filters():
    # butter(8, 0.05): stable as sections in float32, unstable in float32 direct form
    sos = _sos32('butter8-0.05').astype(np.float64)
    for s in sos:
        assert np.abs(np.roots(s[3:])).max() < 1
    b, a = scipy.signal.butter(8, 0.05)
    assert np.abs(np.roots(a.astype(np.float32).astype(np.float64))).max() > 1
    assert _sos32('butter8-telephone').shape[0] == 8
    assert _sos32('single').shape[0] == 1


# ------------------------------------------------------------------------------------------ the kernel bodies
def test_powers_are_the_state_matrix_powers():
    for name, sos in FILTERS:
        s32 = sos.astype(np.float32)
        S = s32.shape[0]
        D = 2 * S
        out = np.zeros((6, D, D))
        _lib().kb_emu_sos_powers(_p(np.ascontiguousarray(s32)), S, _p(out))
        # Phi column k: one zero-input step from e_k, by the restatement
        Phi = np.zeros((D, D))
        for k in range(D):
            z = np.zeros((S, 2))
            z.flat[k] = 1.0
            _, zf = SR.sosfilt(np.zeros(1), s32.astype(np.float64), z)
            Phi[:, k] = zf.ravel()
        P = np.linalg.matrix_power(Phi, SR.TC)
        for j in range(6):
            assert np.abs(out[j] - P).max() <= 1e-7 * max(1.0, np.abs(P).max()), (name, j)   # float64, far below float32
            P = P @ P


LENGTHS = [1, 8, SR.TC - 1, SR.TC, SR.TC + 1, SR.TC * SR.W - 1, SR.TC * SR.W, SR.TC * SR.W + 1, 3 * SR.TC * SR.W + 77]


@pytest.mark.parametrize('name', NAMES)
def test_forward_zf_and_reverse_within_bound(name):
    rng = np.random.default_rng(NAMES.index(name))
    s32 = _sos32(name)
    S = s32.shape[0]
    for L in LENGTHS:
        x = rng.uniform(-1, 1, (2, 1, L)).astype(np.float32)
        zi = (rng.uniform(-1, 1, (2, 1, S, 2)) * SR.sosfilt_zi(s32.astype(np.float64))).astype(np.float32)
        y, _ = emu(x, s32[None, None])
        _check(x, s32, y, what=(name, L))
        y, zf = emu(x, s32[None, None], zi, want_zf=True)
        _check(x, s32, y, zi, zf, (name, L, 'zi'))
        yr, zfr = emu(x, s32[None, None], zi, reverse=True, want_zf=True)
        _check(x[..., ::-1], s32, yr[..., ::-1], zi, zfr, (name, L, 'reverse'))


@pytest.mark.parametrize('name', ['butter8-0.05', 'ellip8', 'cheby2-narrow', 'highpass-20Hz-48k'])
def test_forward_long_signal_within_bound(name):
    s32 = _sos32(name)
    x = np.random.default_rng(3).uniform(-1, 1, (1, 1, 1_000_003)).astype(np.float32)
    y, zf = emu(x, s32[None, None], want_zf=True)
    err, bound = _check(x, s32, y, None, zf, name)
    print('%s: max|err| %.3g, bound %.3g' % (name, err, bound))


def test_zero_zi_and_no_zi_give_the_same_bits():
    s32 = _sos32('ellip8')
    x = np.random.default_rng(4).uniform(-1, 1, (2, 2, 5000)).astype(np.float32)
    y0, _ = emu(x, s32[None, None])
    y1, zf = emu(x, s32[None, None], np.zeros((1, 1, 4, 2), np.float32), want_zf=True)
    assert np.array_equal(y0, y1)
    yr, _ = emu(np.ascontiguousarray(x[..., ::-1]), s32[None, None])
    assert np.array_equal(emu(x, s32[None, None], reverse=True)[0], yr[..., ::-1])


def test_bits_do_not_depend_on_grid_loader_position_strides_broadcast_format_or_length():
    rng = np.random.default_rng(5)
    s32 = _sos32('butter8-telephone')
    B, C, L = 3, 2, 2 * SR.TC * SR.W + 300
    x = rng.uniform(-1, 1, (B, C, L)).astype(np.float32)
    sb = s32[None, None]
    zi = (rng.uniform(-1, 1, (B, C, 8, 2))).astype(np.float32)
    ref, zref = emu(x, sb, zi, want_zf=True)
    for kw in (dict(tile_order=1), dict(bulk=0)):
        y, zf = emu(x, sb, zi, want_zf=True, **kw)
        assert np.array_equal(y, ref) and np.array_equal(zf, zref), kw
    r0, _ = emu(x, sb, reverse=True)
    assert np.array_equal(emu(x, sb, reverse=True, bulk=0)[0], r0)
    assert np.array_equal(emu(x, sb, reverse=True, tile_order=1)[0], r0)
    # materialised coefficients per item and channel
    sm = np.ascontiguousarray(np.broadcast_to(sb, (B, C, 8, 6)))
    assert np.array_equal(emu(x, sm, zi)[0], ref)
    # a broadcast zi against the materialised one
    z1 = zi[:1, :1].copy()
    assert np.array_equal(emu(x, sb, z1)[0], emu(x, sb, np.ascontiguousarray(np.broadcast_to(z1, zi.shape)))[0])
    # each item alone and a batch that starts elsewhere
    for i in range(B):
        assert np.array_equal(emu(x[i:i + 1], sb, zi[i:i + 1])[0], ref[i:i + 1])
    assert np.array_equal(emu(x[1:], sb, zi[1:])[0], ref[1:])
    # a strided view (offset items, narrowed time, every other channel)
    big = rng.uniform(-1, 1, (B + 1, 2 * C, L + 11)).astype(np.float32)
    big[1:, ::2, 5:L + 5] = x
    assert np.array_equal(emu(big[1:, ::2, 5:L + 5], sb, zi)[0], ref)
    # channels-last (interleaved) input gives the channels-first bits
    xl = np.ascontiguousarray(x.transpose(0, 2, 1))
    assert np.array_equal(emu(xl, sb, zi, fmt='blc')[0], ref)
    # a prefix of a longer signal
    for n in (1, SR.TC, SR.TC * SR.W + 3, L - 1):
        assert np.array_equal(emu(np.ascontiguousarray(x[..., :n]), sb, zi)[0], ref[..., :n]), n


def test_per_item_and_per_channel_coefficients():
    rng = np.random.default_rng(6)
    B, C, L = 3, 2, 4000
    x = rng.uniform(-1, 1, (B, C, L)).astype(np.float32)
    edges = [[(100, 300), (500, 900)], [(1000, 2000), (200, 4000)], [(3000, 5000), (50, 150)]]
    sos = np.zeros((B, C, 4, 6), np.float32)
    for i in range(B):
        for c in range(C):
            sos[i, c] = scipy.signal.butter(4, edges[i][c], 'bandpass', fs=16000, output='sos').astype(np.float32)
    y, _ = emu(x, sos)
    for i in range(B):
        for c in range(C):
            _check(x[i, c], sos[i, c], y[i, c])
            yi, _ = emu(x[i:i + 1, c:c + 1].copy(), sos[i:i + 1, c:c + 1].copy())
            assert np.array_equal(yi[0, 0], y[i, c])
    # one filter per channel, shared over the batch
    y2, _ = emu(x, sos[:1].copy())
    for c in range(C):
        _check(x[:, c], sos[0, c], y2[:, c])


@pytest.mark.parametrize('name', ['butter8-telephone', 'cheby2-narrow', 'single'])
def test_streaming_in_pieces_through_zf(name):
    rng = np.random.default_rng(7)
    s32 = _sos32(name)
    x = rng.uniform(-1, 1, (2, 1, 30000)).astype(np.float32)
    whole, _ = emu(x, s32[None, None])
    _, bound = _check(x, s32, whole)
    ref, _ = SR.sosfilt_fast(x.astype(np.float64), s32)
    parts, z = [], None
    for a, b in ((0, 1), (1, 700), (700, 2081), (2081, 19999), (19999, 30000)):
        y, z = emu(np.ascontiguousarray(x[..., a:b]), s32[None, None], z, want_zf=True)
        parts.append(y)
    got = np.concatenate(parts, -1)
    assert np.abs(got - ref).max() <= bound, (np.abs(got - ref).max(), bound)


def _sosfilt_torch(x, sos, zi=None):
    """The restatement in float64 torch, for autograd."""
    S = sos.shape[0]
    z = [[zi[..., s, 0], zi[..., s, 1]] if zi is not None else [0.0, 0.0] for s in range(S)]
    out = []
    for t in range(x.shape[-1]):
        v = x[..., t]
        for s in range(S):
            b0, b1, b2, _, a1, a2 = (float(c) for c in sos[s])
            y = b0 * v + z[s][0]
            z[s] = [b1 * v - a1 * y + z[s][1], b2 * v - a2 * y]
            v = y
        out.append(v)
    return torch.stack(out, -1)


def test_gradient_is_the_reverse_run():
    rng = np.random.default_rng(8)
    for name in ('butter8-telephone', 'single', 'ellip8'):
        s32 = _sos32(name)
        s64 = s32.astype(np.float64)
        x = torch.tensor(rng.uniform(-1, 1, (2, 1, 200)), requires_grad=True)
        gy = rng.uniform(-1, 1, (2, 1, 200))
        (_sosfilt_torch(x, s64) * torch.from_numpy(gy)).sum().backward()
        gx, _ = emu(gy.astype(np.float32), s32[None, None], reverse=True)
        bound = SR.error_bound(gy[..., ::-1], s32)
        assert np.abs(gx - x.grad.numpy()).max() <= bound, name
        # and for the reverse pass, the forward run
        x.grad = None
        (_sosfilt_torch(x.flip(-1), s64).flip(-1) * torch.from_numpy(gy)).sum().backward()
        gx, _ = emu(gy.astype(np.float32), s32[None, None])
        assert np.abs(gx - x.grad.numpy()).max() <= SR.error_bound(gy, s32), name


def test_sosfiltfilt_gradient_identity_matches_autograd():
    """sosfiltfilt's data-dependent initial states c z: d/dc <g, y> = H(1) sum(g) - sum(F^T g), checked against
    float64 autograd of the restatement through the whole padded, two-pass sosfiltfilt."""
    from kapre_b200 import backend
    rng = np.random.default_rng(9)
    for name in ('butter8-telephone', 'highpass-20Hz-48k', 'single'):
        s64 = _sos32(name).astype(np.float64)
        z, gain = backend.sos_steady_state(s64)
        x = torch.tensor(rng.uniform(-1, 1, 120), requires_grad=True)
        c = torch.tensor(0.7, dtype=torch.float64, requires_grad=True)
        g = torch.from_numpy(rng.uniform(-1, 1, 120))
        y = _sosfilt_torch(x, s64, torch.from_numpy(z) * c)
        (y * g).sum().backward()
        gx = _sosfilt_torch(g.flip(-1), s64).flip(-1)                  # F^T g
        assert torch.allclose(x.grad, gx, atol=1e-12, rtol=0)
        want = gain * g.sum() - gx.sum()
        assert abs(float(c.grad) - float(want)) <= 1e-9 * max(1.0, abs(float(want))), name
        # the whole sosfiltfilt through torch's autograd equals the composition the library uses
        edge = 3 * SR.n_taps(s64)
        xs = torch.tensor(rng.uniform(-1, 1, 150), requires_grad=True)

        def ff(v, zt):
            left, right = 2 * v[:1] - v[1:edge + 1].flip(0), 2 * v[-1:] - v[-edge - 1:-1].flip(0)
            e = torch.cat([left, v, right])
            y1 = _sosfilt_torch(e, s64, zt * e[0])
            y2 = _sosfilt_torch(y1.flip(0), s64, zt * y1[-1]).flip(0)
            return y2[edge:-edge]
        out = ff(xs, torch.from_numpy(z))
        want = scipy.signal.sosfiltfilt(s64, xs.detach().numpy())
        assert np.abs(out.detach().numpy() - want).max() <= 1e-9 * max(1, np.abs(want).max())


# ------------------------------------------------------------------------------------------ layers
def _kb():
    if not os.path.exists(_LIB):
        pytest.skip('needs the built library')


def test_validation_before_any_launch():
    _kb()
    from kapre_b200 import _native as N
    from kapre_b200 import ops
    x = torch.zeros(4, 100, 2)
    ops.sos_check(x, torch.zeros(3, 6), 'channels_last')
    ops.sos_check(x, torch.zeros(2, 8, 6), 'channels_last')
    ops.sos_check(x, torch.zeros(4, 1, 1, 6), 'channels_last')
    for sos in (torch.zeros(9, 6), torch.zeros(0, 6), torch.zeros(3, 5), torch.zeros(3, 3, 6), torch.zeros(2, 2, 3, 6),
                torch.zeros(6), torch.zeros(1, 1, 1, 1, 6)):
        with pytest.raises(ValueError):
            ops.sos_check(x, sos, 'channels_last')
    ops.sos_state_check(torch.zeros(3, 2), 4, 2, 3, 'zi')
    ops.sos_state_check(torch.zeros(4, 1, 3, 2), 4, 2, 3, 'zi')
    for z in (torch.zeros(2, 2), torch.zeros(3, 3), torch.zeros(3, 3, 2), torch.zeros(3, 2, 3, 2)):
        with pytest.raises(ValueError):
            ops.sos_state_check(z, 4, 2, 3, 'zi')
    assert N.lib().kapre_sosfilt_workspace_bytes(2, 2, 1000, 9) == -2          # KAPRE_E_UNSUPPORTED
    assert N.lib().kapre_sosfilt_workspace_bytes(2, 2, 1000, 0) == -2
    assert N.lib().kapre_sosfilt_workspace_bytes(-1, 2, 1000, 2) == -1
    assert N.lib().kapre_sosfilt_workspace_bytes(65536, 65536, 1 << 30, 8) < 0
    assert N.lib().kapre_sosfilt_workspace_bytes(2, 2, 1000, 3) > 0


def test_layer_validation_and_config():
    _kb()
    import kapre
    from kapre_b200.signal import SOSFilter, sosfilt, sosfiltfilt
    assert kapre.signal.SOSFilter is SOSFilter and kapre.signal.sosfilt is sosfilt
    assert kapre.signal.sosfiltfilt is sosfiltfilt
    sos = scipy.signal.butter(4, 0.1, output='sos')
    bad = sos.copy()
    bad[1, 3] = 2.0                                                  # a0 != 1
    nan = sos.copy()
    nan[0, 0] = np.nan
    for s in (bad, nan, np.zeros((9, 6)), np.zeros((2, 5)), np.zeros(6)):
        with pytest.raises(ValueError):
            SOSFilter(s)
    f = SOSFilter(sos, data_format='channels_first')
    cfg = f.get_config()
    g = SOSFilter.from_config(cfg)
    assert g.get_config() == cfg and np.array_equal(g.sos, sos)


# ------------------------------------------------------------------------------------------ register budget
@pytest.mark.skipif(shutil.which('cuobjdump') is None or not os.path.exists(_LIB),
                    reason='needs cuobjdump and the built library')
def test_sos_kernels_register_and_spill_budget():
    out = subprocess.run(['cuobjdump', '-res-usage', _LIB], capture_output=True, text=True, check=True).stdout
    for S in range(1, 9):
        for name, cap in (('kb_sos_powers_kernel', 64), ('kb_sos_state_kernel', 128), ('kb_sos_carry_kernel', 128),
                          ('kb_sos_out_kernel', 128)):
            m = re.search(r'Function \S*%sILi%dE\S*:\s*\n\s*REG:(\d+) STACK:(\d+)' % (name, S), out)
            assert m, '%s<%d> not in the library' % (name, S)
            assert int(m.group(1)) <= cap, (name, S, m.group(1))
            assert int(m.group(2)) == 0, (name, S, m.group(2))      # no spills, no stack
