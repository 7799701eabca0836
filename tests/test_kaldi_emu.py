"""Kaldi features on the CPU: the float64 restatement (kaldi_ref.py) against torchaudio.compliance.kaldi (values and
VJPs), the kernel bodies of kaldi_core.cuh (run by a CPU emulation) against the restatement within its derived bound,
their bit-independence of job order, batch position, strides, format and lengths, the dither generator against its
NumPy restatement, the gradient, validation, layer configuration and the register budget."""
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
import torchaudio.compliance.kaldi as TK

import kaldi_ref as R
from kapre_b200 import backend, ops
from emu_harness import Checked

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, 'emu', 'kb_emu_kaldi.cpp')
_CSRC = os.path.join(_HERE, '..', 'kapre_b200', 'csrc')
_LIB = os.path.join(_HERE, '..', 'kapre_b200', '_lib', 'libkapre_b200.so')
_lib_handle = None


def _lib():
    """tests/emu/kb_emu_kaldi.cpp built with g++ into the temporary directory (keyed by the sources' contents)."""
    global _lib_handle
    if _lib_handle is None:
        hs = hashlib.sha256()
        for f in [_SRC] + sorted(os.path.join(_CSRC, n) for n in os.listdir(_CSRC) if n.endswith(('.h', '.cuh'))):
            with open(f, 'rb') as fh:
                hs.update(fh.read())
        out = os.path.join(tempfile.gettempdir(), 'kapre_b200_emu_kaldi_%s.so' % hs.hexdigest()[:16])
        if not os.path.exists(out):
            tmp = '%s.%d.tmp' % (out, os.getpid())
            subprocess.check_call(['g++', '-O2', '-std=c++17', '-shared', '-fPIC', '-DKB_HOST_EMU', '-Wno-unknown-pragmas',
                                   '-o', tmp, _SRC])
            os.replace(tmp, out)
        _lib_handle = Checked(ctypes.CDLL(out))
    return _lib_handle


def _p(a):
    return None if a is None else ctypes.c_void_p(a.__array_interface__['data'][0])


def emu(kind, x, o, lengths=None, dither=0.0, seed=0, g=None, order=0, fmt='bcl'):
    """Run the bodies on x ((B, C, L) 'bcl' or (B, L, C) 'blc', any strides).  Returns (B, C, T, K) features, or the
    (B, C, L) gradient at g ((B, C, T, K))."""
    plan = ops.KaldiPlan(kind, dict(o, dither=dither))
    s = [v // 4 for v in x.strides]
    if fmt == 'blc':
        B, L, C = x.shape
        xs = np.array([s[0], s[2], s[1]], np.int64)
    else:
        B, C, L = x.shape
        xs = np.array(s, np.int64)
    lens = None if lengths is None else np.ascontiguousarray(lengths, np.int32)
    T = (int(plan.num_frames(lens).max()) if B else 0) if lens is not None else plan.num_frames(L)
    c = plan.cfg
    ic = np.array([c.kind, c.window_size, c.window_shift, c.padded_window_size, c.snip_edges, c.min_length,
                   c.num_mel_bins, c.num_ceps, c.use_energy, c.htk_compat, c.raw_energy, c.use_power, c.use_log_fbank,
                   c.remove_dc_offset, c.subtract_mean, B, C, L, T], np.int32)
    fc = np.array([c.preemphasis_coefficient, c.energy_floor, dither], np.float32)
    K = plan.K
    ys = np.array([C * T * K, T * K, K, 1], np.int64)
    args = [_p(ic), _p(fc), ctypes.c_ulonglong(seed), _p(plan.window), _p(plan.banks), _p(plan.dct), _p(x), _p(xs),
            _p(lens)]
    if g is None:
        y = np.full((B, C, T, K), np.nan, np.float32)
        assert _lib().kb_emu_kaldi(*args, _p(y), _p(ys), 0, None, None, order) == 0
        return y
    g = np.ascontiguousarray(g, np.float32)
    gx = np.full((B, C, L), np.nan, np.float32)
    gxs = np.array([C * L, L, 1], np.int64)
    assert _lib().kb_emu_kaldi(*args, _p(g), _p(ys), 1, _p(gx), _p(gxs), order) == 0
    return gx


def _noise(seed, dither):
    return lambda b, c, f, W: (np.float32(dither) * R.gauss(seed, b, c, f, W)).astype(np.float32)


def _signal(rng, B, C, L, sr, kind='mix'):
    t = np.arange(L) / sr
    x = np.zeros((B, C, L))
    for b in range(B):
        for c in range(C):
            x[b, c] = 0.05 * rng.standard_normal(L) * (1.0 + np.sin(2 * np.pi * 3.0 * t + b + c))   # speech-like bursts
            x[b, c] += 0.3 * np.sin(2 * np.pi * rng.uniform(100, sr / 3) * t) + rng.uniform(-0.2, 0.2)   # tone, DC
    return np.clip(x, -1.0, 1.0).astype(np.float32)


def _ta(kind, x1, o):
    fn = getattr(TK, kind)
    kw = {k: v for k, v in o.items() if k in fn.__code__.co_varnames}
    return fn(x1, **kw)


CASES = [
    ('fbank', dict(num_mel_bins=80)),
    ('fbank', dict(num_mel_bins=23, window_type='hamming', use_energy=True, htk_compat=True)),
    ('fbank', dict(num_mel_bins=40, window_type='hanning', use_power=False, raw_energy=False, snip_edges=False)),
    ('fbank', dict(num_mel_bins=30, window_type='rectangular', use_log_fbank=False, use_energy=True)),
    ('fbank', dict(num_mel_bins=64, window_type='blackman', blackman_coeff=0.4, subtract_mean=True, snip_edges=False)),
    ('fbank', dict(num_mel_bins=40, vtln_warp=0.9, high_freq=-400.0)),
    ('fbank', dict(num_mel_bins=40, vtln_warp=1.1, energy_floor=0.0, min_duration=0.2)),
    ('mfcc', dict()),
    ('mfcc', dict(use_energy=True, htk_compat=True, snip_edges=False, subtract_mean=True, num_ceps=20, num_mel_bins=40)),
    ('mfcc', dict(htk_compat=True, cepstral_lifter=0.0, raw_energy=False)),
    ('spectrogram', dict()),
    ('spectrogram', dict(snip_edges=False, raw_energy=False, window_type='hamming', subtract_mean=True)),
]


@pytest.mark.parametrize('kind,kw', CASES)
def test_reference_matches_torchaudio(kind, kw):
    """The float64 restatement against torchaudio in float64: values and VJPs, per (item, channel)."""
    rng = np.random.default_rng(1)
    o = ops.kaldi_options(kind, **kw)
    x = _signal(rng, 2, 2, 16000, 16000.0).astype(np.float64)
    xt = torch.from_numpy(x).requires_grad_(True)
    ref = R.features(kind, xt, o)
    g = torch.from_numpy(rng.standard_normal(ref.shape))
    (ref * g).sum().backward()
    for b in range(2):
        for c in range(2):
            x1 = torch.from_numpy(x[b, c][None].copy()).requires_grad_(True)
            if 16000 < o['min_duration'] * o['sample_frequency']:
                continue
            ta = _ta(kind, x1, o)
            assert ta.shape == ref[b, c].shape
            # torchaudio computes its mel banks in float32 (relative 1e-4 at most), whatever the waveform dtype
            np.testing.assert_allclose(ref[b, c].detach().numpy(), ta.detach().numpy(), atol=5e-4, rtol=2e-4)
            (ta * g[b, c]).sum().backward()
            gr = xt.grad[b, c].numpy()
            np.testing.assert_allclose(gr, x1.grad[0].numpy(), atol=1e-4 * np.abs(gr).max(), rtol=0)


def _check(kind, x, o, y, lengths=None, dither=0.0, seed=0):
    ref = R.features(kind, torch.from_numpy(x.astype(np.float64)), o, lengths,
                     _noise(seed, dither) if dither else None).numpy()
    bound = R.log_bound(kind, x, o, lengths, ref)
    err = np.abs(y.astype(np.float64) - ref)
    assert y.shape == ref.shape
    assert np.isfinite(y).all()
    bad = err > bound
    assert not bad.any(), (kind, float(err[bad].max()), float(bound[bad].min()))


@pytest.mark.parametrize('kind,kw', CASES)
@pytest.mark.parametrize('sr', [8000, 16000, 22050, 44100, 48000])
def test_emu_within_bound(kind, kw, sr):
    rng = np.random.default_rng(sr)
    o = ops.kaldi_options(kind, sample_frequency=float(sr), **kw)
    if kind != 'spectrogram' and o['num_mel_bins'] > 40 and sr == 8000 and o['vtln_warp'] == 1.0:
        o['num_mel_bins'] = 40
    x = _signal(rng, 2, 1, sr // 2, float(sr))
    _check(kind, x, o, emu(kind, x, o))


@pytest.mark.parametrize('C', [1, 2, 3, 7])
@pytest.mark.parametrize('fmt', ['bcl', 'blc'])
def test_channels_formats_lengths(C, fmt):
    rng = np.random.default_rng(C)
    o = ops.kaldi_options('fbank', num_mel_bins=40, snip_edges=(C % 2 == 0))
    x = _signal(rng, 3, C, 6000, 16000.0)
    lengths = [6000, 0, 1234]
    xin = np.ascontiguousarray(x.transpose(0, 2, 1)) if fmt == 'blc' else x
    y = emu('fbank', xin, o, lengths=lengths, fmt=fmt)
    _check('fbank', x, o, y, lengths)
    # an item computed as if cut to its length, and in any format, gives the same bits
    cut = emu('fbank', np.ascontiguousarray(x[2:3, :, :1234]), o)
    np.testing.assert_array_equal(y[2, :, :cut.shape[2]], cut[0])
    assert (y[2, :, cut.shape[2]:] == 0).all() and (y[1] == 0).all()
    other = emu('fbank', x if fmt == 'blc' else np.ascontiguousarray(x.transpose(0, 2, 1)), o, lengths=lengths,
                fmt='bcl' if fmt == 'blc' else 'blc')
    np.testing.assert_array_equal(y, other)


def test_bits_independent_of_order_position_and_views():
    rng = np.random.default_rng(5)
    o = ops.kaldi_options('mfcc', snip_edges=False)
    x = _signal(rng, 4, 2, 8000, 16000.0)
    y0 = emu('mfcc', x, o, dither=0.5, seed=7)
    for order in (1, 2):
        np.testing.assert_array_equal(emu('mfcc', x, o, dither=0.5, seed=7, order=order), y0)
    np.testing.assert_array_equal(emu('mfcc', x[:, :, ::1], o, dither=0.5, seed=7), y0)
    big = np.zeros((4, 2, 8000 * 2), np.float32)
    big[:, :, ::2] = x
    np.testing.assert_array_equal(emu('mfcc', big[:, :, ::2], o, dither=0.5, seed=7), y0)
    # without dither an item's bits do not depend on its batch position
    z = emu('mfcc', x, o)
    np.testing.assert_array_equal(emu('mfcc', np.ascontiguousarray(x[::-1]), o)[::-1], z)


@pytest.mark.parametrize('L', [0, 1, 399, 400, 401, 560, 10 * 60 * 8000])
def test_lengths_edge(L):
    o = ops.kaldi_options('fbank', sample_frequency=8000.0, num_mel_bins=23, snip_edges=False,
                          frame_length=50.0)
    rng = np.random.default_rng(L)
    x = (0.1 * rng.standard_normal((1, 1, max(L, 1)))).astype(np.float32)[:, :, :L]
    y = emu('fbank', np.ascontiguousarray(x), o)
    W, H, _ = backend.kaldi_window_properties(8000.0, 10.0, 50.0)
    assert y.shape[2] == backend.kaldi_num_frames(L, W, H, False)
    if L in (400, 401, 560):
        _check('fbank', x, o, y)


def test_silence_gives_log_eps():
    o = ops.kaldi_options('fbank', num_mel_bins=23, energy_floor=0.0, use_energy=True)
    y = emu('fbank', np.zeros((1, 1, 4000), np.float32), o)
    assert (y == np.float32(R.LOG_EPS32)).all()
    ta = TK.fbank(torch.zeros(1, 4000), num_mel_bins=23, energy_floor=0.0, use_energy=True).numpy()
    np.testing.assert_array_equal(y[0, 0], ta)
    assert np.float32(R.LOG_EPS32) == np.float32(-15.942385)


def test_dither_bits_and_moments():
    lib = _lib()
    out = np.zeros(4096, np.float32)
    lib.kb_emu_kaldi_gauss(ctypes.c_ulonglong(123), ctypes.c_longlong(5), 2, 17, 4096, _p(out))
    np.testing.assert_array_equal(out, R.gauss(123, 5, 2, 17, 4096))
    v = np.concatenate([R.gauss(9, b, 0, f, 4096) for b in range(4) for f in range(16)]).astype(np.float64)
    n = v.size
    assert abs(v.mean()) < 5.0 / np.sqrt(n)
    assert abs(v.std() - 1.0) < 5.0 * np.sqrt(2.0 / n)
    # the features with dither match the restatement with the same injected noise
    o = ops.kaldi_options('fbank', num_mel_bins=40)
    x = _signal(np.random.default_rng(2), 2, 2, 4000, 16000.0)
    _check('fbank', x, o, emu('fbank', x, o, dither=1.0, seed=3), dither=1.0, seed=3)


def _vjp_ref(kind, x, o, g, lengths=None, dither=0.0, seed=0):
    xt = torch.from_numpy(x.astype(np.float64)).requires_grad_(True)
    r = R.features(kind, xt, o, lengths, _noise(seed, dither) if dither else None)
    (r * torch.from_numpy(g.astype(np.float64))).sum().backward()
    return xt.grad.numpy()


@pytest.mark.parametrize('kind,kw', CASES)
@pytest.mark.parametrize('dither', [0.0, 0.5])
def test_vjp(kind, kw, dither):
    rng = np.random.default_rng(11)
    o = ops.kaldi_options(kind, **kw)
    # a noise floor keeps every bin away from |X| = 0, where the magnitude's gradient X / |X| is ill-conditioned
    # (use_power=False): there a float32 |X| has no correct digits and its direction none either
    x = (_signal(rng, 2, 2, 5000, 16000.0) + 0.01 * rng.standard_normal((2, 2, 5000))).astype(np.float32)
    lengths = [5000, 3333]
    y = emu(kind, x, o, lengths=lengths, dither=dither, seed=4)
    g = rng.standard_normal(y.shape).astype(np.float32)
    gx = emu(kind, x, o, lengths=lengths, dither=dither, seed=4, g=g)
    gr = _vjp_ref(kind, x, o, g, lengths, dither, 4)
    # bound: the float32 forward's relative error (log bound / value scale) times the gradient's l1 reach: each sample
    # gathers at most ceil(W / H) frames, each through float32 chains of O(log2 N + W / 32) roundings
    W, H, Np, _ = R.plan_of(kind, o)
    scale = np.abs(gr).max()
    tol = 2e-3 * scale
    assert np.abs(gx - gr).max() <= tol, (np.abs(gx - gr).max(), tol)
    assert (gx[1, :, 3333:] == 0).all()


def test_validation_before_launch():
    with pytest.raises(Exception, match='256, 512, 1024, 2048'):
        ops.KaldiPlan('fbank', ops.kaldi_options('fbank', round_to_power_of_two=False))
    with pytest.raises(Exception, match='256, 512, 1024, 2048'):
        ops.KaldiPlan('fbank', ops.kaldi_options('fbank', sample_frequency=96000.0))
    with pytest.raises(TypeError):
        ops.kaldi_options('fbank', channel=0)
    with pytest.raises(ValueError):
        ops.kaldi_options('mfcc', preemphasis_coefficient=float('nan'))
    with pytest.raises(ValueError):
        ops.KaldiPlan('mfcc', ops.kaldi_options('mfcc', num_ceps=30))
    with pytest.raises(ValueError):
        ops._kaldi_lengths([5, 11], 2, 10, 'cpu')
    with pytest.raises(ValueError):
        ops._kaldi_lengths([5], 2, 10, 'cpu')


def test_layer_config_and_seeded_draws():
    from kapre_b200.time_frequency import KaldiFbank, KaldiMFCC, KaldiSpectrogram
    a = KaldiFbank(num_mel_bins=80, dither=1.0, seed=3, data_format='channels_first', name='fb')
    cfg = a.get_config()
    assert cfg['num_mel_bins'] == 80 and cfg['dither'] == 1.0 and cfg['seed'] == 3
    assert cfg['data_format'] == 'channels_first' and 'channel' not in cfg
    b = KaldiFbank.from_config(cfg)
    assert b.get_config() == cfg
    assert KaldiMFCC(num_ceps=20, num_mel_bins=40).get_config()['num_ceps'] == 20
    assert KaldiSpectrogram().get_config()['window_type'] == 'povey'
    draws = [int(a.rng.integers(0, 2 ** 63)) for _ in range(3)]
    assert draws == [int(np.random.default_rng(3).integers(0, 2 ** 63, size=3)[i]) for i in range(3)]


def test_register_budget():
    """The built library's Kaldi kernels use no stack and no spills, and fit two forward CTAs per SM."""
    if not os.path.exists(_LIB) or shutil.which('cuobjdump') is None:
        pytest.skip('library or cuobjdump not available')
    out = subprocess.run(['cuobjdump', '-res-usage', _LIB], capture_output=True, text=True).stdout
    seen = 0
    for fn, regs, stack in re.findall(r'Function (\S*kb_kaldi\S*):\s*REG:(\d+) STACK:(\d+)', out):
        seen += 1
        assert int(stack) == 0, fn
        assert int(regs) <= 255, fn
    assert seen >= 10
