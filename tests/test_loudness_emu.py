"""Gated loudness on the CPU: the float64 restatement (loudness_ref.py) against torchaudio, the K-weighting coefficients,
the kernel bodies of loudness_core.cuh (run by a CPU emulation) against the restatement within the derived bound, each
gate, -inf and NaN items, bit-independence of tile order, batch position, strides, format and lengths, the gradient,
validation, layer configs, the workspace rule and the register budget."""
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

import loudness_ref as LR

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, 'emu', 'kb_emu_loudness.cpp')
_CSRC = os.path.join(_HERE, '..', 'kapre_b200', 'csrc')
_LIB = os.path.join(_HERE, '..', 'kapre_b200', '_lib', 'libkapre_b200.so')
_lib_handle = None
RATES = (8000, 11025, 16000, 44100, 48000)


def _lib():
    """tests/emu/kb_emu_loudness.cpp built with g++ into the temporary directory (keyed by the sources' contents)."""
    global _lib_handle
    if _lib_handle is None:
        hs = hashlib.sha256()
        for f in [_SRC] + sorted(os.path.join(_CSRC, n) for n in os.listdir(_CSRC) if n.endswith(('.h', '.cuh'))):
            with open(f, 'rb') as fh:
                hs.update(fh.read())
        out = os.path.join(tempfile.gettempdir(), 'kapre_b200_emu_loudness_%s.so' % hs.hexdigest()[:16])
        if not os.path.exists(out):
            tmp = '%s.%d.tmp' % (out, os.getpid())
            subprocess.check_call(['g++', '-O2', '-std=c++17', '-shared', '-fPIC', '-DKB_HOST_EMU', '-Wno-unknown-pragmas',
                                   '-o', tmp, _SRC])
            os.replace(tmp, out)
        lib = ctypes.CDLL(out)
        P, I = ctypes.c_void_p, ctypes.c_int
        lib.kb_emu_loudness.argtypes = [P, P, P, I, I, I, I, I, P, P, P, P, I]
        lib.kb_emu_loudness_backward.argtypes = [P, P, P, P, I, I, I, I, I, P, P, P, P, I]
        lib.kb_emu_loudness_geometry.argtypes = [I, I, I, P]
        _lib_handle = lib
    return _lib_handle


def _p(a):
    return ctypes.c_void_p(a.__array_interface__['data'][0]) if a is not None else None


def geometry(L, G, S):
    out = np.zeros(5, np.int32)
    _lib().kb_emu_loudness_geometry(L, G, S, _p(out))
    return dict(zip(('rho', 'm', 'Jmax', 'K', 'Kb'), out.tolist()))


def _strides(a, fmt):
    """Element strides (b, c, l) and (B, C, L) of a (B, C, L) ('bcl') or (B, L, C) ('blc') float32 array or view."""
    s = [v // 4 for v in a.strides]
    if fmt == 'blc':
        return np.array([s[0], s[2], s[1]], np.int64), (a.shape[0], a.shape[2], a.shape[1])
    return np.array(s, np.int64), a.shape


def emu(y, G, S, lengths=None, fmt='bcl', order=0):
    """The energy and gate passes on y: (LKFS (B,) float32, stats (B, 2), mask (B, Jmax))."""
    st, (B, C, L) = _strides(y, fmt)
    ln = None if lengths is None else np.ascontiguousarray(np.broadcast_to(np.asarray(lengths, np.int32), (B,)))
    out = np.full(B, 7.0, np.float32)
    stats = np.full((B, 2), np.nan)
    mask = np.full((B, max(geometry(L, G, S)['Jmax'], 1)), 9, np.uint8)
    assert _lib().kb_emu_loudness(_p(y), _p(st), _p(ln), B, C, L, G, S, _p(out), _p(stats), _p(mask), None, order) == 0
    return out, stats, mask


def emu_backward(gl, y, G, S, stats, mask, lengths=None, fmt='bcl', order=0):
    """gy (B, C, L) of the backward pass."""
    st, (B, C, L) = _strides(y, fmt)
    ln = None if lengths is None else np.ascontiguousarray(np.broadcast_to(np.asarray(lengths, np.int32), (B,)))
    gy = np.full((B, C, L), np.nan, np.float32)
    gst = np.array([C * L, L, 1], np.int64)
    gl = np.ascontiguousarray(gl, np.float32)
    assert _lib().kb_emu_loudness_backward(_p(gl), _p(y), _p(st), _p(ln), B, C, L, G, S, _p(stats), _p(mask), _p(gy),
                                           _p(gst), order) == 0
    return gy


def _noise(shape, seed, scale=0.1):
    return np.random.default_rng(seed).standard_normal(shape) * scale


def _sections(C, sr, levels, seed):
    """(1, C, L) noise in consecutive 1 s sections at the given amplitudes."""
    return np.concatenate([_noise((1, C, sr), seed + i, a) for i, a in enumerate(levels)], axis=2)


def _weighted32(x, sr):
    """(y64, y32): the K-weighting of x in float64 with the kernels' float32 coefficients, and y rounded to float32."""
    y = LR.weight(x, LR.normalised(LR.k_weighting(sr)))
    return y, y.astype(np.float32)


# ------------------------------------------------------------------------------------------ the restatement
@pytest.mark.parametrize('sr', RATES)
def test_restatement_is_torchaudio_loudness(sr):
    F = pytest.importorskip('torchaudio.functional')
    for C in range(1, 6):
        x = _sections(C, sr, (0.3, 0.01, 0.2), 10 * C)
        x[:, :, sr:sr + sr // 2] *= 1e-4                          # a stretch under the absolute gate
        got = LR.loudness(x, sr)[0]
        want = float(F.loudness(torch.from_numpy(x[0]), sr))
        assert abs(got - want) < 1e-9, (sr, C, got, want)
    # lengths: the item cut to its length
    x = _sections(2, sr, (0.3, 0.05, 0.2), 99)
    for n in (int(0.4 * sr) + 5, int(1.7 * sr), x.shape[2]):
        got = LR.loudness(np.concatenate([x, x]), sr, lengths=[n, x.shape[2]])[0]
        want = float(F.loudness(torch.from_numpy(x[0, :, :n]), sr))
        assert abs(got - want) < 1e-9, (sr, n, got, want)


def test_restatement_vjp_is_torch_autograd_through_torchaudio():
    F = pytest.importorskip('torchaudio.functional')
    sr = 8000
    x = _sections(2, sr, (0.3, 0.02, 0.2), 5)
    xt = torch.from_numpy(x[0]).requires_grad_(True)
    F.loudness(xt, sr).backward(torch.tensor(0.7, dtype=torch.float64))
    g = LR.vjp(x, np.array([0.7]), sr)[0]
    np.testing.assert_allclose(g, xt.grad.numpy(), rtol=1e-7, atol=1e-12)


def test_k_weighting_coefficients_are_torchaudio_s():
    F = pytest.importorskip('torchaudio.functional')
    import torchaudio.functional.filtering as TF
    from kapre_b200.backend import BIQUAD_KINDS, k_weighting_coefficients
    seen = []
    orig = TF.biquad

    def spy(waveform, b0, b1, b2, a0, a1, a2):
        seen.append(np.array([float(v) for v in (b0, b1, b2, a0, a1, a2)]))
        return orig(waveform, b0, b1, b2, a0, a1, a2)

    TF.biquad = spy
    try:
        for sr in RATES + (3001, 96000):
            seen.clear()
            F.loudness(torch.zeros(1, int(0.4 * sr) + 1, dtype=torch.float64), sr)
            (b1, a1), (b2, a2) = k_weighting_coefficients(sr)
            assert len(seen) == 2
            np.testing.assert_allclose(np.r_[b1, a1], seen[0], rtol=1e-14, atol=1e-14)
            np.testing.assert_allclose(np.r_[b2, a2], seen[1], rtol=1e-14, atol=1e-14)
            (rb1, ra1), (rb2, ra2) = LR.k_weighting(sr)
            np.testing.assert_allclose(np.r_[rb1, ra1, rb2, ra2], np.r_[b1, a1, b2, a2], rtol=1e-14, atol=1e-14)
    finally:
        TF.biquad = orig
    assert 'treble' not in BIQUAD_KINDS
    for bad in (3000, 2000.0, 0, -16000, np.inf, np.nan, '16000', None):
        with pytest.raises(ValueError):
            k_weighting_coefficients(bad)


def test_geometry_is_torchaudio_s():
    for sr, (G, S) in ((8000, (3200, 800)), (11025, (4410, 1102)), (16000, (6400, 1600)), (44100, (17640, 4410)),
                       (48000, (19200, 4800))):
        assert LR.geometry(sr) == (G, S)
        g = geometry(3 * sr, G, S)
        assert (g['rho'], g['m']) == (G % S, G // S)
        assert g['Jmax'] == (3 * sr - G) // S + 1
        assert g['K'] == g['Jmax'] - 1 + g['m'] + (G % S > 0) and g['Kb'] == -(-3 * sr // S)
    assert geometry(100, 200, 50)['Jmax'] == 0 and geometry(100, 200, 50)['K'] == 0


# ------------------------------------------------------------------------------------------ the kernels
@pytest.mark.parametrize('sr', RATES)
@pytest.mark.parametrize('C', [1, 2, 5])
def test_forward_within_bound(sr, C):
    G, S = LR.geometry(sr)
    x = np.concatenate([_sections(C, sr, (0.3, 0.005, 0.2), 7 + C), _sections(C, sr, (0.1, 0.4, 0.02), 70 + C)])
    y, y32 = _weighted32(x, sr)
    got, stats, _ = emu(y32, G, S)
    want = LR.gated(y, G, S)[0]
    bound = LR.lkfs_bound(y, G, S, float(np.abs(y - y32).max()))
    assert np.all(np.abs(got - want) <= bound), (got, want, bound)
    assert np.all(stats[:, 1] > 0)


def test_each_gate_and_the_inf_and_nan_items():
    sr = 11025
    G, S = LR.geometry(sr)
    C = 2
    loud = _sections(C, sr, (0.3, 0.3), 1)
    below_abs = np.concatenate([loud, _sections(C, sr, (1e-6, 1e-6), 2)], axis=2)           # l_j < -70
    below_rel = np.concatenate([loud, _sections(C, sr, (0.01, 0.01), 3)], axis=2)           # -70 < l_j < Gamma
    silent = np.zeros_like(below_abs)
    faint = _sections(C, sr, (1e-6,) * 4, 4)                                                # every block < -70
    x = np.concatenate([below_abs, below_rel, silent, faint, below_abs, below_abs]).astype(np.float32)
    x[5, 1, 3 * sr] = np.nan
    lengths = [4 * sr, 4 * sr, 4 * sr, 4 * sr, G - 1, 0]
    y, y32 = _weighted32(x, sr)
    got, stats, mask = emu(y32, G, S, lengths=lengths)
    ref, E2, masks, es = LR.gated(y, G, S, lengths)
    # the constructions exercise what they claim
    E = [(LR.WEIGHTS[:C, None] * e).sum(0) for e in es]
    l0, l1 = (-0.691 + 10 * np.log10(E[i]) for i in (0, 1))
    assert (l0 < -70).any() and (l0 > -70).any() and not masks[0][l0 < -70].any()
    assert (l1 > -70).all() and not masks[1].all() and masks[1].any()
    assert np.all(np.abs(got[:2] - ref[:2]) <= LR.lkfs_bound(y[:2], G, S, float(np.abs(y - y32)[:2].max()),
                                                             lengths[:2]))
    # silence, every block under -70, len < G and len = 0
    assert np.isneginf(got[2:6]).all() and np.isneginf(ref[2:6]).all() and (stats[2:6, 1] == 0).all()
    # the NaN sits past item 5's length 0: not measured.  Give the whole item and it is NaN, the others unchanged.
    got2, _, _ = emu(y32, G, S, lengths=lengths[:5] + [4 * sr])
    assert np.isnan(got2[5]) and np.array_equal(got2[:5], got[:5])


def test_bits_do_not_depend_on_order_position_strides_format_or_lengths():
    sr = 16000
    G, S = LR.geometry(sr)
    C, L = 3, int(2.3 * sr)
    x = np.concatenate([_sections(C, sr, (0.2, 0.01, 0.3), 20 + i)[:, :, :L] for i in range(4)])
    _, y32 = _weighted32(x, sr)
    base, bstats, bmask = emu(y32, G, S)
    for order in (1, 2):
        o, s, m = emu(y32, G, S, order=order)
        assert np.array_equal(o, base) and np.array_equal(s, bstats) and np.array_equal(m, bmask)
    for b in range(4):                                                  # alone and at another position
        assert np.array_equal(emu(np.ascontiguousarray(y32[b:b + 1]), G, S)[0], base[b:b + 1])
    assert np.array_equal(emu(np.ascontiguousarray(y32[::-1]), G, S)[0], base[::-1])
    big = np.zeros((4, C + 2, L + 11), np.float32)                      # a strided view
    big[:, 1:C + 1, 5:5 + L] = y32
    assert np.array_equal(emu(big[:, 1:C + 1, 5:5 + L], G, S)[0], base)
    blc = np.ascontiguousarray(y32.transpose(0, 2, 1))                  # channels interleaved
    assert np.array_equal(emu(blc, G, S, fmt='blc')[0], base)
    # lengths against the cut item
    cut = [L, int(1.5 * sr), G + S + 3, G]
    o, _, _ = emu(y32, G, S, lengths=cut)
    for b, n in enumerate(cut):
        assert np.array_equal(emu(np.ascontiguousarray(y32[b:b + 1, :, :n]), G, S)[0], o[b:b + 1]), b
        assert np.array_equal(emu(np.ascontiguousarray(blc[b:b + 1, :n]), G, S, fmt='blc')[0], o[b:b + 1]), b


@pytest.mark.parametrize('sr, C, fmt', [(11025, 2, 'bcl'), (16000, 1, 'bcl'), (48000, 5, 'blc')])
def test_backward_within_bound(sr, C, fmt):
    G, S = LR.geometry(sr)
    x = np.concatenate([_sections(C, sr, (0.2, 0.003, 0.3), 40 + C), _sections(C, sr, (0.0, 0.0, 0.0), 1)])
    lengths = [int(2.6 * sr), 3 * sr]
    _, y32 = _weighted32(x, sr)
    yin = y32 if fmt == 'bcl' else np.ascontiguousarray(y32.transpose(0, 2, 1))
    out, stats, mask = emu(yin, G, S, lengths=lengths, fmt=fmt)
    gl = np.array([0.7, -1.3])
    gy = emu_backward(gl, yin, G, S, stats, mask, lengths=lengths, fmt=fmt)
    want = LR.grad_y(y32.astype(np.float64), gl, G, S, lengths)
    assert np.all(np.abs(gy - want) <= np.abs(want) * 4 * LR.EPS32 + 1e-30)
    J = (lengths[0] - G) // S + 1
    assert np.all(gy[0, :, (J - 1) * S + G:] == 0) and np.all(gy[1] == 0)     # past the last block; a -inf item
    assert np.any(gy[0] != 0)


# ------------------------------------------------------------------------------------------ validation and the ABI
def _kb():
    if not os.path.exists(_LIB):
        pytest.skip('needs the built library')


def test_layers_validation_draws_and_config():
    _kb()
    import kapre
    import kapre_b200
    from kapre_b200._native import KapreNativeError
    from kapre_b200.augmentation import LoudnessNormalization
    from kapre_b200.signal import Loudness, loudness
    assert kapre.signal.loudness is loudness and kapre.signal.Loudness is Loudness
    assert kapre.augmentation.LoudnessNormalization is LoudnessNormalization
    assert 'loudness' in kapre_b200.signal.__all__ and 'Loudness' not in kapre_b200.__all__
    with pytest.raises(KapreNativeError):
        loudness(torch.zeros(1, 16000, 1), 16000)
    from kapre_b200.ops import _item_lengths
    cpu = torch.device('cpu')
    assert _item_lengths(8000, 3, 5000, cpu).tolist() == [5000] * 3
    assert _item_lengths(np.int64(-4), 2, 50, cpu).tolist() == [0, 0]
    assert _item_lengths([1, 70, 3], 3, 50, cpu).tolist() == [1, 50, 3]
    assert _item_lengths(torch.tensor([[2]]).view(()), 2, 50, cpu).dtype == torch.int32
    for bad in (1.5, [1, 2], [[1, 2, 3]], torch.ones(3), 'a'):
        with pytest.raises(ValueError):
            _item_lengths(bad, 3, 50, cpu)
    for bad in (2000, 3000, np.nan):
        with pytest.raises(ValueError):
            Loudness(bad)
        with pytest.raises(ValueError):
            LoudnessNormalization(bad)
    for bad in ((5.0, 1.0), (0.0, np.inf), (1.0,)):
        with pytest.raises(ValueError):
            LoudnessNormalization(16000, lufs_range=bad)
    layer = Loudness(44100, data_format='channels_first')
    cfg = layer.get_config()
    assert cfg['sample_rate'] == 44100 and Loudness.from_config(cfg).get_config() == cfg
    norm = LoudnessNormalization(16000, lufs_range=(-30.0, -14.0), seed=3, data_format='channels_last')
    assert np.array_equal(norm.draw(5), np.random.default_rng(3).uniform(-30.0, -14.0, size=5))
    assert list(norm.draw(3, lufs=-20)) == [-20.0] * 3 and list(norm.draw(2, lufs=[-1, -2.5])) == [-1.0, -2.5]
    for bad in (np.nan, [1.0, 2.0, 3.0], 'loud', [[1.0, 2.0]]):
        with pytest.raises(ValueError):
            norm.draw(2, lufs=bad)
    cfg = norm.get_config()
    other = LoudnessNormalization.from_config(cfg)
    assert other.get_config() == cfg
    assert np.array_equal(other.draw(4), LoudnessNormalization.from_config(cfg).draw(4))


def test_workspace_rule_and_overflow():
    _kb()
    from kapre_b200 import _native as N
    lib = N.lib()
    st = ctypes.c_int64(-7)
    # 256 x 5 s at 16 kHz: 47 blocks touch 50 intervals of one piece each (rho = 0) -> 2 sums per interval
    assert lib.kapre_loudness_workspace_bytes(256, 1, 80000, 6400, 1600, ctypes.byref(st)) == 256 * 50 * 2 * 8
    assert st.value == 256 * 16 + 256 * 47
    assert lib.kapre_loudness_workspace_bytes(3, 2, 4409, 4410, 1102, ctypes.byref(st)) == 0 and st.value == 256
    assert lib.kapre_loudness_workspace_bytes(0, 2, 100, 40, 10, None) == 0
    for bad in ((1, 0, 100, 40, 10), (1, 6, 100, 40, 10), (-1, 1, 100, 40, 10), (1, 1, -1, 40, 10), (1, 1, 100, 0, 10),
                (1, 1, 100, 40, 0), (1, 1, 100, 40, 41), (2 ** 31 - 1, 5, 2 ** 31 - 1, 2, 1)):
        assert lib.kapre_loudness_workspace_bytes(*bad, None) < 0, bad


@pytest.mark.skipif(shutil.which('cuobjdump') is None or not os.path.exists(_LIB),
                    reason='needs cuobjdump and the built library')
def test_loudness_kernels_have_no_stack_or_spills():
    out = subprocess.run(['cuobjdump', '-res-usage', _LIB], capture_output=True, text=True, check=True).stdout
    for name in ('kb_loud_energy_kernel', 'kb_loud_gate_kernel', 'kb_loud_bwd_kernel'):
        m = re.search(r'Function \S*%s\S*:\s*\n\s*REG:(\d+) STACK:(\d+)' % name, out)
        assert m, name + ' not in the library'
        assert int(m.group(1)) <= 128, (name, m.group(1))
        assert int(m.group(2)) == 0, (name, m.group(2))
