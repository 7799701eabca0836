"""Additive noise at a target SNR on the CPU: the float64 restatement (noise_ref.py) against torchaudio, the kernel bodies
of noise_core.cuh (run by a CPU emulation) against the restatement within the derived bounds, their bit-independence of
tile order, batch position, strides, format, broadcasting and noise source, the En == 0 deviation and NaN isolation,
BackgroundNoise's validation, draws and configuration, the workspace rule and the register budget."""
import ctypes
import hashlib
import os
import re
import shutil
import subprocess
import tempfile

import numpy as np
import pytest
import torch

import noise_ref as NR

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, 'emu', 'kb_emu_noise.cpp')
_CSRC = os.path.join(_HERE, '..', 'kapre_b200', 'csrc')
_LIB = os.path.join(_HERE, '..', 'kapre_b200', '_lib', 'libkapre_b200.so')
_lib_handle = None


def _lib():
    """tests/emu/kb_emu_noise.cpp built with g++ into the temporary directory (keyed by the sources' contents)."""
    global _lib_handle
    if _lib_handle is None:
        hs = hashlib.sha256()
        for f in [_SRC] + sorted(os.path.join(_CSRC, n) for n in os.listdir(_CSRC) if n.endswith(('.h', '.cuh'))):
            with open(f, 'rb') as fh:
                hs.update(fh.read())
        out = os.path.join(tempfile.gettempdir(), 'kapre_b200_emu_noise_%s.so' % hs.hexdigest()[:16])
        if not os.path.exists(out):
            tmp = '%s.%d.tmp' % (out, os.getpid())
            subprocess.check_call(['g++', '-O2', '-std=c++17', '-shared', '-fPIC', '-DKB_HOST_EMU', '-Wno-unknown-pragmas',
                                   '-o', tmp, _SRC])
            os.replace(tmp, out)
        lib = ctypes.CDLL(out)
        P, I, LL = ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong
        lib.kb_emu_add_noise.argtypes = [P, P, P, LL, P, P, P, P, P, P, P, P, P, I, I, I, I, P, P, P, I]
        lib.kb_emu_noise_consts.argtypes = [P]
        _lib_handle = lib
    return _lib_handle


def _p(a):
    return ctypes.c_void_p(a.__array_interface__['data'][0]) if a is not None else None


def _bcl_strides(a, fmt):
    """Element strides (b, c, l) of a (B, C, L) ('bcl') or (B, L, C) ('blc') array or view, 0 on axes of size 1."""
    s = [v // 4 for v in a.strides]
    if fmt == 'blc':
        s = [s[0], s[2], s[1]]
    shape = a.shape if fmt == 'bcl' else (a.shape[0], a.shape[2], a.shape[1])
    return [0 if n == 1 else v for n, v in zip(shape, s)], shape


def emu(x, noise=None, snr=0.0, lengths=None, fmt='bcl', nfmt=None, bank=None, order=0, bwd=False, g=None,
        stats=None, want_gn=False, want_gsnr=False):
    """Run the bodies.  x (and g) in fmt, noise in nfmt (default fmt; batch / channels of 1 broadcast) or
    bank = (flat float32 bank, start, clip, offset).  Returns y (B, C, L) and stats, or (gx, gn, gsnr) with bwd."""
    _, (B, C, L) = _bcl_strides(x, fmt)
    st = np.zeros(15, np.int64)
    st[0:3] = _bcl_strides(x, fmt)[0]
    if noise is not None:
        st[3:6] = _bcl_strides(noise, nfmt or fmt)[0]
    y = np.full((B, C, L), np.nan, np.float32)
    st[6:9] = [C * L, L, 1]
    snr = np.ascontiguousarray(np.broadcast_to(np.asarray(snr, np.float32), (B, C)))
    ss = np.array([C, 1, C, 1], np.int64)
    ln = None if lengths is None else np.ascontiguousarray(np.broadcast_to(np.asarray(lengths, np.int32), (B, C)))
    bk = [None, 0, None, None, None]
    if bank is not None:
        flat, start, clip, offset = bank
        bk = [np.ascontiguousarray(flat, np.float32), flat.size, np.ascontiguousarray(start, np.int64),
              np.ascontiguousarray(clip, np.int64), np.ascontiguousarray(offset, np.int64)]
    xin = x
    xr = gn = gsnr = None
    if bwd:
        xin = g
        st[0:3] = _bcl_strides(g, fmt)[0]
        xr = x
        st[9:12] = _bcl_strides(x, fmt)[0]
        if want_gn:
            gn = np.full((B, C, L), np.nan, np.float32)
            st[12:15] = [C * L, L, 1]
        if want_gsnr:
            gsnr = np.full((B, C), np.nan, np.float32)
    else:
        stats = np.full((B, C, 2), np.nan) if stats is None else stats
    rc = _lib().kb_emu_add_noise(_p(xin), _p(noise), _p(bk[0]), bk[1], _p(bk[2]), _p(bk[3]), _p(bk[4]), _p(snr),
                                 _p(ln), _p(st), _p(ss), _p(y), _p(stats), B, C, L, int(bwd), _p(xr), _p(gn),
                                 _p(gsnr), order)
    assert rc == 0
    return (y, gn, gsnr) if bwd else (y, stats)


def _bcl(a, fmt):
    return a if fmt == 'bcl' else a.transpose(0, 2, 1)


def _rand(shape, seed, scale=1.0):
    return (np.random.default_rng(seed).standard_normal(shape) * scale).astype(np.float32)


# ------------------------------------------------------------------------------------------ the restatement
def test_restatement_is_torchaudio_add_noise():
    F = pytest.importorskip('torchaudio.functional')
    rng = np.random.default_rng(0)
    B, C, L = 3, 2, 500
    x = rng.standard_normal((B, C, L))
    n = rng.standard_normal((B, C, L))
    snr = rng.uniform(-5, 30, (B, C))
    for lengths in (None, np.array([[0, 10], [L, L + 7], [250, 1]])):
        y, _ = NR.add_noise(x, n, snr, lengths)
        ta = F.add_noise(torch.from_numpy(x), torch.from_numpy(n), torch.from_numpy(snr),
                         None if lengths is None else torch.from_numpy(lengths)).numpy()
        fin = np.isfinite(ta)
        assert fin.sum() > 0.5 * fin.size
        np.testing.assert_allclose(y[fin], ta[fin], rtol=1e-12, atol=1e-12)
        if lengths is not None:
            assert not np.isfinite(ta[0, 0]).any() and np.array_equal(y[0, 0], x[0, 0])      # len 0: NaN there, x here
    # broadcast noise: one clip for every item and channel
    y, _ = NR.add_noise(x, n[:1, :1], snr)
    ta = F.add_noise(torch.from_numpy(x), torch.from_numpy(np.broadcast_to(n[:1, :1], x.shape).copy()),
                     torch.from_numpy(snr)).numpy()
    np.testing.assert_allclose(y, ta, rtol=1e-12, atol=1e-12)
    # zero noise: torchaudio's NaN is the one deviation
    ta = F.add_noise(torch.from_numpy(x), torch.zeros(B, C, L, dtype=torch.float64), torch.from_numpy(snr)).numpy()
    assert np.isnan(ta).all() and np.array_equal(NR.add_noise(x, 0 * n, snr)[0], x)


def test_restatement_vjp_is_torch_autograd_through_torchaudio():
    F = pytest.importorskip('torchaudio.functional')
    rng = np.random.default_rng(1)
    B, C, L = 2, 3, 200
    x, n, g = (rng.standard_normal((B, C, L)) for _ in range(3))
    snr = rng.uniform(0, 20, (B, C))
    for lengths in (None, np.array([[5, 200, 120], [1, 199, 300]])):
        tx, tn, ts = (torch.tensor(v, requires_grad=True) for v in (x, n, snr))
        y = F.add_noise(tx, tn, ts, None if lengths is None else torch.from_numpy(lengths))
        (y * torch.from_numpy(g)).sum().backward()
        gx, gn, gs = NR.vjp(x, n, snr, g, lengths)
        for got, want in ((gx, tx.grad), (gn, tn.grad), (gs, ts.grad)):
            np.testing.assert_allclose(got, want.numpy(), rtol=1e-10, atol=1e-10)


# ------------------------------------------------------------------------------------------ the kernel bodies
def _check_forward(y, x, n, snr, lengths, what=''):
    ref, _ = NR.add_noise(x, n, snr, lengths)
    bound = NR.forward_bound(x, n, snr, lengths)
    err = np.abs(y - ref)
    assert (err <= bound).all(), (what, err.max(), bound[err > bound][:3])


@pytest.mark.parametrize('C', [1, 2, 3, 7])
@pytest.mark.parametrize('fmt', ['bcl', 'blc'])
def test_forward_within_bound(C, fmt):
    rng = np.random.default_rng(C)
    for L in (1, 31, 129, 4095, 4096, 4097, 3 * 4096 + 777):
        B = 2
        x = _rand((B, C, L), L)
        n = _rand((B, C, L), L + 1, 0.3)
        snr = rng.uniform(-10, 40, (B, C)).astype(np.float32)
        lengths = rng.integers(-3, L + 5, (B, C))
        for ln in (None, lengths):
            y, stats = emu(np.ascontiguousarray(_bcl(x, fmt)), np.ascontiguousarray(_bcl(n, fmt)), snr, ln, fmt)
            _check_forward(y, x, n, snr, ln, (C, fmt, L))
            ex, en = NR.energies(x, n, ln)
            np.testing.assert_allclose(stats[..., 0], ex, rtol=1e-13)
            np.testing.assert_allclose(stats[..., 1], en, rtol=1e-13)


def test_forward_long_signal_within_bound():
    x = _rand((1, 1, 1_000_000), 3)
    n = _rand((1, 1, 1_000_000), 4, 2.0)
    y, _ = emu(x, n, 5.0)
    _check_forward(y, x, n, np.float32(5.0), None)


def _bank(lengths, seed):
    clips = [_rand(n, seed + i, 0.5) for i, n in enumerate(lengths)]
    start = np.cumsum([0] + [c.size for c in clips[:-1]])
    return clips, np.concatenate(clips), start


@pytest.mark.parametrize('fmt', ['bcl', 'blc'])
def test_bank_within_bound_and_equal_to_the_materialised_excerpt(fmt):
    L, C = 9000, 2
    clips, flat, start = _bank([1, 7, 333, 20000], 10)
    idx = np.array([0, 1, 2, 3, 3, 2])
    clen = np.array([clips[i].size for i in idx])
    off = np.array([0, 6, 332, 0, 19999, 5])                 # 0 and len - 1 among them
    B = len(idx)
    x = _rand((B, C, L), 11)
    snr = np.linspace(-5, 25, B * C).reshape(B, C).astype(np.float32)
    y, _ = emu(np.ascontiguousarray(_bcl(x, fmt)), None, snr, fmt=fmt, bank=(flat, start[idx], clen, off))
    ex = NR.bank_excerpt(clips, idx, off, L).astype(np.float32)[:, None, :]
    _check_forward(y, x, ex, snr, None, fmt)
    # the same bits as the excerpt passed as a (channel-broadcast) tensor, and as a materialised one
    nb = np.ascontiguousarray(_bcl(np.broadcast_to(ex, (B, 1, L)), fmt))
    assert np.array_equal(emu(np.ascontiguousarray(_bcl(x, fmt)), nb, snr, fmt=fmt)[0], y)
    nm = np.ascontiguousarray(_bcl(np.broadcast_to(ex, (B, C, L)), fmt))
    assert np.array_equal(emu(np.ascontiguousarray(_bcl(x, fmt)), nm, snr, fmt=fmt)[0], y)


def test_bank_clip_outside_the_bank_reads_zeros():
    clips, flat, start = _bank([100], 12)
    x = _rand((2, 1, 300), 13)
    y, stats = emu(x, None, 10.0, bank=(flat, np.array([0, 50]), np.array([100, 100]), np.array([0, 0])))
    assert np.array_equal(y[1], x[1]) and stats[1, 0, 1] == 0
    y2, _ = emu(x, None, 10.0, bank=(flat, np.array([0, 0]), np.array([0, -4]), np.array([0, 3])))
    assert np.array_equal(y2, x)


def test_bits_do_not_depend_on_order_position_strides_format_or_broadcast():
    rng = np.random.default_rng(20)
    B, C, L = 4, 3, 2 * 4096 + 1000
    x = _rand((B, C, L), 21)
    n = _rand((B, C, L), 22)
    snr = rng.uniform(0, 20, (B, C)).astype(np.float32)
    lengths = rng.integers(100, L + 100, (B, C))
    ref, st = emu(x, n, snr, lengths)
    for order in (1, 2):
        assert np.array_equal(emu(x, n, snr, lengths, order=order)[0], ref)
    for i in range(B):
        assert np.array_equal(emu(x[i:i + 1].copy(), n[i:i + 1].copy(), snr[i:i + 1], lengths[i:i + 1])[0], ref[i:i + 1])
    big = _rand((B + 2, 2 * C, L + 9), 23)
    bign = _rand((B + 2, 2 * C, L + 9), 24)
    big[1:B + 1, ::2, 4:L + 4] = x
    bign[1:B + 1, ::2, 4:L + 4] = n
    assert np.array_equal(emu(big[1:B + 1, ::2, 4:L + 4], bign[1:B + 1, ::2, 4:L + 4], snr, lengths)[0], ref)
    xl = np.ascontiguousarray(x.transpose(0, 2, 1))
    nl = np.ascontiguousarray(n.transpose(0, 2, 1))
    assert np.array_equal(emu(xl, nl, snr, lengths, fmt='blc')[0], ref)
    assert np.array_equal(emu(xl, n, snr, lengths, fmt='blc', nfmt='bcl')[0], ref)
    # broadcast noise (batch and / or channels of 1) against the materialised copy
    for nb in (n[:1], n[:, :1], n[:1, :1]):
        nm = np.ascontiguousarray(np.broadcast_to(nb, x.shape))
        r1 = emu(x, np.ascontiguousarray(nb), snr, lengths)[0]
        assert np.array_equal(r1, emu(x, nm, snr, lengths)[0])
        assert np.array_equal(r1, emu(xl, np.ascontiguousarray(nb), snr, lengths, fmt='blc', nfmt='bcl')[0])


def test_zero_energy_gives_x_and_a_nan_column_stays_alone():
    x = _rand((2, 3, 5000), 30)
    n = _rand((2, 3, 5000), 31)
    n[0, 1] = 0                                  # En == 0
    x[1, 0] = 0                                  # Ex == 0
    lengths = np.array([[5000, 5000, 5000], [5000, 5000, 0]])     # len 0: both energies 0
    y, _ = emu(x, n, 3.0, lengths)
    for b, c in ((0, 1), (1, 0), (1, 2)):
        assert np.array_equal(y[b, c], x[b, c]), (b, c)
    xn = x.copy()
    xn[0, 2, 77] = np.nan
    y2, _ = emu(xn, n, 3.0, lengths)
    assert np.isnan(y2[0, 2]).all()
    keep = np.ones((2, 3), bool)
    keep[0, 2] = False
    assert np.array_equal(y2[keep], y[keep])


@pytest.mark.parametrize('C,fmt', [(1, 'bcl'), (2, 'blc'), (3, 'bcl'), (7, 'blc')])
def test_backward_within_bound(C, fmt):
    rng = np.random.default_rng(40 + C)
    for L in (1, 300, 4097, 2 * 4096 + 5):
        B = 2
        x, n, g = _rand((B, C, L), L), _rand((B, C, L), L + 1, 0.5), _rand((B, C, L), L + 2)
        snr = rng.uniform(-5, 30, (B, C)).astype(np.float32)
        lengths = rng.integers(0, L + 3, (B, C))
        for ln in (None, lengths):
            xf, nf, gf = (np.ascontiguousarray(_bcl(a, fmt)) for a in (x, n, g))
            _, stats = emu(xf, nf, snr, ln, fmt)
            gx, gn, gs = emu(xf, nf, snr, ln, fmt, bwd=True, g=gf, stats=stats, want_gn=True, want_gsnr=True)
            (rx, rn, rs), (bx, bn, bs) = NR.backward_bounds(x, n, snr, g, ln)
            assert (np.abs(gx - rx) <= bx).all(), (C, fmt, L)
            assert (np.abs(gn - rn) <= bn).all(), (C, fmt, L)
            assert (np.abs(gs - rs) <= bs).all(), (C, fmt, L)
            # without gn and gsnr, gx has the same bits
            gx2, gn2, gs2 = emu(xf, nf, snr, ln, fmt, bwd=True, g=gf, stats=stats)
            assert np.array_equal(gx2, gx) and gn2 is None and gs2 is None


def test_backward_bank_long_signal():
    clips, flat, start = _bank([1000, 3], 50)
    L = 1_000_000
    x, g = _rand((2, 1, L), 51), _rand((2, 1, L), 52)
    bank = (flat, start, np.array([1000, 3]), np.array([999, 2]))
    _, stats = emu(x, None, 7.0, bank=bank)
    gx, _, gs = emu(x, None, 7.0, bank=bank, bwd=True, g=g, stats=stats, want_gsnr=True)
    ex = NR.bank_excerpt(clips, [0, 1], [999, 2], L).astype(np.float32)[:, None, :]
    (rx, _, rs), (bx, _, bs) = NR.backward_bounds(x, ex, np.float32(7.0), g)
    assert (np.abs(gx - rx) <= bx).all() and (np.abs(gs - rs) <= bs).all()


# ------------------------------------------------------------------------------------------ the layer and the ABI
def _kb():
    if not os.path.exists(_LIB):
        pytest.skip('needs the built library')


def test_background_noise_validation_draws_and_config():
    _kb()
    import kapre
    import kapre_b200
    from kapre_b200.augmentation import BackgroundNoise, prepare_noises
    from kapre_b200.signal import add_noise
    assert kapre.augmentation.BackgroundNoise is BackgroundNoise and kapre.signal.add_noise is add_noise
    assert 'add_noise' in kapre_b200.signal.__all__
    assert 'BackgroundNoise' not in kapre_b200.__all__ and 'add_noise' not in kapre_b200.__all__
    for bad in ([], [[]], [[0.0, 0.0]], [[1.0, np.nan]], np.zeros((2, 3, 4)), [np.ones((2, 2))], 'noise'):
        with pytest.raises(ValueError):
            prepare_noises(bad)
    for bad in (dict(snr_range=(5.0, 1.0)), dict(snr_range=(0.0, np.inf)), dict(snr_range=(1.0,))):
        with pytest.raises(ValueError):
            BackgroundNoise([[1.0, 2.0]], **bad)
    clips = [np.arange(1, 8, dtype=np.float32), np.ones(3, np.float32), -np.ones(50, np.float32)]
    layer = BackgroundNoise(clips, snr_range=(3.0, 9.0), seed=7, data_format='channels_first')
    assert np.array_equal(layer.bank, np.concatenate(clips)) and list(layer.clip_len) == [7, 3, 50]
    idx, off, snr = layer.draw(6)
    rng = np.random.default_rng(7)
    ri = rng.integers(0, 3, size=6)
    ro = rng.integers(0, np.array([7, 3, 50])[ri])
    rs = rng.uniform(3.0, 9.0, size=6)
    assert np.array_equal(idx, ri) and np.array_equal(off, ro) and np.array_equal(snr, rs)
    # overrides replace their draws and are validated
    idx, off, snr = layer.draw(4, noise_index=1, offset=[0, 1, 2, 0], snr=[1.0, 2.0, 3.0, 4.0])
    assert list(idx) == [1] * 4 and list(off) == [0, 1, 2, 0] and list(snr) == [1.0, 2.0, 3.0, 4.0]
    for kw in (dict(noise_index=3), dict(noise_index=[0, 1]), dict(noise_index=1, offset=3), dict(offset=-1),
               dict(snr=np.nan), dict(snr=[1.0, 2.0]), dict(noise_index=0.5)):
        with pytest.raises(ValueError):
            layer.draw(4, **kw)
    cfg = layer.get_config()
    other = BackgroundNoise.from_config(cfg)
    assert other.get_config() == cfg
    assert all(np.array_equal(a, b) for a, b in zip(other.draw(5), BackgroundNoise.from_config(cfg).draw(5)))


def test_segment_size_is_the_kernels():
    out = np.zeros(3, np.int32)
    _lib().kb_emu_noise_consts(_p(out))
    assert out[0] == NR.SEG                       # the restatement's bound uses the kernel's segment length
    assert NR.SEG % out[1] == 0 and out[1] % 32 == 0 and out[2] == 8


def test_workspace_rule_and_overflow():
    _kb()
    from kapre_b200 import _native as N
    lib = N.lib()
    assert lib.kapre_add_noise_workspace_bytes(256, 1, 80000) == 256 * 20 * 16
    assert lib.kapre_add_noise_workspace_bytes(3, 7, 4097) == (3 * 7 * 2 * 16 + 255) // 256 * 256
    assert lib.kapre_add_noise_workspace_bytes(0, 2, 100) == 0
    assert lib.kapre_add_noise_workspace_bytes(2, 2, 0) == 0
    assert lib.kapre_add_noise_workspace_bytes(-1, 2, 100) == -1
    assert lib.kapre_add_noise_workspace_bytes(2, 2, -5) == -1
    assert lib.kapre_add_noise_workspace_bytes(2 ** 31 - 1, 2 ** 31 - 1, 2 ** 31 - 1) == -1


@pytest.mark.skipif(shutil.which('cuobjdump') is None or not os.path.exists(_LIB),
                    reason='needs cuobjdump and the built library')
def test_noise_kernels_register_and_spill_budget():
    out = subprocess.run(['cuobjdump', '-res-usage', _LIB], capture_output=True, text=True, check=True).stdout
    # __launch_bounds__(128, 4) allows 128: both passes use all of it to keep every operand's batch of loads in flight
    for name, cap in (('kb_noise_sum_kernel', 128), ('kb_noise_out_kernel', 128)):
        m = re.search(r'Function \S*%s\S*:\s*\n\s*REG:(\d+) STACK:(\d+)' % name, out)
        assert m, name + ' not in the library'
        assert int(m.group(1)) <= cap, (name, m.group(1))
        assert int(m.group(2)) == 0, (name, m.group(2))      # no spills, no stack
