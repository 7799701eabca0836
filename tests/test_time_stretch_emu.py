"""Time stretch on the CPU: the float64 restatement (time_stretch_ref.py) pinned to torchaudio's phase vocoder in
complex128, its gradient against autograd through torchaudio and ``gradcheck``; the kernel bodies of ts_core.cuh (run
by a CPU emulation) against the restatement, forward and backward, unchunked and chunked; the ``TimeStretch`` layer's
validation and config.

Tolerances.  Each output phase is q(X[0]) plus 2u fixed-point angle differences, every angle within 2.8e-7 rad
(kb_atan2) + 7.3e-10 rad (the rounding to 2^-32 turn) of the true one, and the sum is exact; so the accumulated phase
is within (2u + 1)(2.8e-7 + 7.3e-10) rad.  Reading the phase back from the float32 output adds at most 3e-7 rad: the
int32 -> float32 conversion of the phase (pi 2^-25), sincospi (an ulp each) and the products by the magnitude
(2^-24 each).  The magnitude is a blend of two float32 moduli, within 4 eps32 of (|X[k]| + |X[k + 1]|).
"""
import ctypes
import hashlib
import math
import os
import subprocess
import tempfile

import numpy as np
import pytest
import torch

import time_stretch_ref as TR
from emu_harness import Checked

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, 'emu', 'kb_emu_ts.cpp')
_CSRC = os.path.join(_HERE, '..', 'kapre_b200', 'csrc')
_lib_handle = None
CL, CF = 'channels_last', 'channels_first'
ANGLE_ERR = 2.8e-7 + 7.3e-10
READ_ERR = 3e-7
EPS32 = 2.0 ** -24


def _lib():
    """tests/emu/kb_emu_ts.cpp built with g++ into the temporary directory (keyed by the sources' contents, so the
    checkout itself may be read-only)."""
    global _lib_handle
    if _lib_handle is None:
        h = hashlib.sha256()
        for f in [_SRC] + sorted(os.path.join(_CSRC, n) for n in os.listdir(_CSRC) if n.endswith(('.h', '.cuh'))):
            with open(f, 'rb') as fh:
                h.update(fh.read())
        out = os.path.join(tempfile.gettempdir(), 'kapre_b200_emu_ts_%s.so' % h.hexdigest()[:16])
        if not os.path.exists(out):
            tmp = '%s.%d.tmp' % (out, os.getpid())
            subprocess.check_call(['g++', '-O2', '-std=c++17', '-shared', '-fPIC', '-DKB_HOST_EMU', '-Wno-unknown-pragmas',
                                   '-o', tmp, _SRC])
            os.replace(tmp, out)
        lib = ctypes.CDLL(out)
        P, I, D = ctypes.c_void_p, ctypes.c_int, ctypes.c_double
        lib.kb_emu_ts.argtypes = [P, P, I, I, I, I, D, I, P, P]
        lib.kb_emu_ts_backward.argtypes = [P, P, P, P, P, P, I, I, I, I, D, I, P, P]
        lib.kb_emu_ts_chunks.argtypes = [ctypes.c_longlong, I, ctypes.c_longlong]
        _lib_handle = Checked(lib)
    return _lib_handle


def _fp(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _dims_strides(x, fmt):
    """(B, C, T, F) and the (b, c, t, f) complex-element strides of a (B, T, F, C) / (B, C, T, F) complex64 array."""
    s = [v // 8 for v in x.strides]
    if fmt == CL:
        B, T, F, C = x.shape
        return (B, C, T, F), np.array([s[0], s[3], s[1], s[2]], np.int64)
    B, C, T, F = x.shape
    return (B, C, T, F), np.array(s, np.int64)


def _alloc(fmt, B, C, T, F):
    a = np.full((B, T, F, C) if fmt == CL else (B, C, T, F), np.nan + 1j * np.nan, np.complex64)
    return a, _dims_strides(a, fmt)[1]


def emu_ts(x, fmt, rate, Tc=0):
    (B, C, T, F), xs = _dims_strides(x, fmt)
    y, ys = _alloc(fmt, B, C, math.ceil(T / rate), F)
    K = _lib().kb_emu_ts(x.ctypes.data, _fp(xs), B, C, T, F, rate, Tc, _fp(y), _fp(ys))
    return y, K


def emu_ts_backward(x, y, g, fmt, rate, Tc=0):
    (B, C, T, F), xs = _dims_strides(x, fmt)
    ys, gs = _dims_strides(y, fmt)[1], _dims_strides(g, fmt)[1]
    gx, os_ = _alloc(fmt, B, C, T, F)
    _lib().kb_emu_ts_backward(x.ctypes.data, _fp(xs), y.ctypes.data, _fp(ys), g.ctypes.data, _fp(gs), B, C, T, F, rate,
                              Tc, _fp(gx), _fp(os_))
    return gx


def _canon(x, fmt):
    """(B, C, T, F) torch tensor of an array in `fmt`."""
    t = torch.from_numpy(np.ascontiguousarray(x))
    return t.permute(0, 3, 1, 2) if fmt == CL else t


def _spectrogram(rng, shape):
    return (rng.standard_normal(shape) + 1j * rng.standard_normal(shape)).astype(np.complex64)


def _check_forward(x, fmt, rate, Tc=0):
    """Emulated forward against the restatement: the phase within the derived bound, the magnitude within 4 eps32."""
    y, K = emu_ts(x, fmt, rate, Tc)
    X = _canon(x, fmt).to(torch.complex128)
    m, phi = TR.phases(X, rate)
    Yc = _canon(y, fmt).to(torch.complex128)
    assert Yc.shape == m.shape
    if Yc.numel():
        k, _ = TR.steps(X.shape[2], rate)
        Xp = torch.cat([X, torch.zeros_like(X[:, :, :2])], dim=2).abs()
        mag_bound = 4 * EPS32 * (Xp[:, :, k] + Xp[:, :, k + 1]) + 1e-30
        assert bool(((Yc.abs() - m).abs() <= mag_bound).all())
        u = torch.arange(m.shape[2], dtype=torch.float64).view(1, 1, -1, 1)
        dphi = torch.remainder(Yc.angle() - phi + math.pi, 2 * math.pi) - math.pi
        bound = (2 * u + 1) * ANGLE_ERR + READ_ERR
        ok = (m == 0) | (dphi.abs() <= bound)
        assert bool(ok.all()), float((dphi.abs() / bound)[m > 0].max())
    return y, K


def _check_backward(x, y, fmt, rate, rng, Tc=0):
    """Emulated backward against autograd through the restatement: within 1e-4 of max|gX|, or within 10x the error of
    the same restatement run in float32 where that is larger (long inputs sum many float32 phase gradients)."""
    g = _spectrogram(rng, y.shape)
    gx = emu_ts_backward(x, y, g, fmt, rate, Tc)
    X = _canon(x, fmt).to(torch.complex128).requires_grad_()
    G = _canon(g, fmt).to(torch.complex128)
    want, = torch.autograd.grad(TR.time_stretch(X, rate), X, G)
    X32 = _canon(x, fmt).clone().requires_grad_()
    twin, = torch.autograd.grad(TR.time_stretch(X32, rate, torch.complex64), X32, G.to(torch.complex64))
    got = _canon(gx, fmt).to(torch.complex128)
    assert got.shape == want.shape
    if got.numel():
        err = float((got - want).abs().max())
        bound = max(1e-4 * float(want.abs().max()), 10 * float((twin.to(torch.complex128) - want).abs().max()))
        assert err <= bound, (err, bound)
    return gx


# ------------------------------------------------------------------------------ the restatement
RATES = [0.5, 0.8, 1.25, 1.3, 2.0, 3.7]


def _torchaudio():
    return pytest.importorskip('torchaudio')


def _phase_advance(F, hop, kind):
    if kind == 'zero':
        return torch.zeros(F, 1, dtype=torch.float64)
    if kind == 'random':
        return torch.from_numpy(np.random.default_rng(F).uniform(-10, 10, (F, 1)))
    return torch.linspace(0, math.pi * hop, F, dtype=torch.float64).view(F, 1)


@pytest.mark.parametrize('rate', RATES + [1.0, 0.25, 0.75, 4.0])
@pytest.mark.parametrize('T,F', [(0, 65), (1, 2), (2, 1), (17, 65), (5000, 2), (427, 513)])
def test_restatement_matches_torchaudio(rate, T, F):
    """complex128 torchaudio with three phase_advance vectors (hop 256, zero and random) against the restatement,
    modulo 2 pi; 0.25, 0.75, 2.0, 4.0 and 0.5 put u * rate exactly on integers."""
    ta = _torchaudio()
    X = torch.from_numpy(_spectrogram(np.random.default_rng(T + F), (2, 1, T, F))).to(torch.complex128)
    k_ta = torch.arange(0, T, rate, dtype=torch.float64)
    k, _ = TR.steps(T, rate)
    assert k_ta.numel() == k.numel() and torch.equal(torch.floor(k_ta).long(), k)
    want = TR.time_stretch(X, rate)
    if T == 0:                          # torchaudio cannot reshape an empty time axis; T' = 0
        assert want.shape == X.shape
        return
    for kind in ('hop', 'zero', 'random'):
        got = TR.torchaudio_layout(ta.functional.phase_vocoder(TR.torchaudio_layout(X), rate,
                                                                _phase_advance(F, 256, kind)))
        assert got.shape == want.shape
        # torchaudio's float64 cumsum runs up to pi hop T' rad: a few ulps of that per sqrt(T') steps
        n = want.shape[2]
        torch.testing.assert_close(got, want, rtol=0, atol=1e-12 + 4 * 2.0 ** -52 * math.pi * 256 * n * math.sqrt(n))


def test_restatement_rate_one_is_identity():
    X = torch.zeros((1, 1, 3, 2), dtype=torch.complex128)
    assert TR.time_stretch(X, 1.0) is X


@pytest.mark.parametrize('rate', [0.8, 1.3, 3.7])
def test_restatement_gradient_matches_torchaudio(rate):
    ta = _torchaudio()
    X = torch.from_numpy(_spectrogram(np.random.default_rng(1), (1, 2, 23, 5))).to(torch.complex128).requires_grad_()
    G = torch.from_numpy(_spectrogram(np.random.default_rng(2), (1, 2, math.ceil(23 / rate), 5))).to(torch.complex128)
    want, = torch.autograd.grad(TR.time_stretch(X, rate), X, G)
    y = TR.torchaudio_layout(ta.functional.phase_vocoder(TR.torchaudio_layout(X), rate, _phase_advance(5, 64, 'hop')))
    got, = torch.autograd.grad(y, X, G)
    torch.testing.assert_close(got, want, rtol=1e-9, atol=1e-9)


@pytest.mark.parametrize('rate', [0.7, 1.5, 2.6])
def test_restatement_gradcheck(rate):
    X = torch.from_numpy(_spectrogram(np.random.default_rng(3), (1, 1, 9, 3))).to(torch.complex128).requires_grad_()
    assert torch.autograd.gradcheck(lambda x: TR.time_stretch(x, rate), (X,))


# ------------------------------------------------------------------------------ the emulated bodies
@pytest.mark.parametrize('rate', RATES)
@pytest.mark.parametrize('T', [0, 1, 2, 17, 40])
@pytest.mark.parametrize('fmt', [CF, CL])
def test_emulated_forward_and_backward(rate, T, fmt):
    """Bins not a multiple of 32 (37), two channels, T not a multiple of the 8-frame register tile."""
    rng = np.random.default_rng(T)
    B, C, F = 2, 2, 37
    x = _spectrogram(rng, (B, T, F, C) if fmt == CL else (B, C, T, F))
    y, K = _check_forward(x, fmt, rate)
    assert K == (1 if T else 0)
    _check_backward(x, y, fmt, rate, rng)


@pytest.mark.parametrize('F', [1, 2, 65, 513])
def test_emulated_bins(F):
    rng = np.random.default_rng(F)
    x = _spectrogram(rng, (1, 1, 30, F))
    y, _ = _check_forward(x, CF, 0.8)
    _check_backward(x, y, CF, 0.8, rng)


@pytest.mark.parametrize('view', ['time_stride', 'bin_slice', 'channel_slice', 'batch_stride', 'transposed'])
@pytest.mark.parametrize('fmt', [CF, CL])
def test_emulated_body_on_views(view, fmt):
    rng = np.random.default_rng(6)
    full = _spectrogram(rng, (3, 30, 40, 3) if fmt == CL else (3, 3, 30, 40))
    t_ax, f_ax, c_ax = (1, 2, 3) if fmt == CL else (2, 3, 1)
    sl = [slice(None)] * 4
    if view == 'time_stride':
        sl[t_ax] = slice(None, None, 2)
    elif view == 'bin_slice':
        sl[f_ax] = slice(3, 36)
    elif view == 'channel_slice':
        sl[c_ax] = slice(1, 3)
    elif view == 'batch_stride':
        sl[0] = slice(None, None, 2)
    x = full[tuple(sl)]
    if view == 'transposed':            # the other format's memory order under this format's shape
        x = np.ascontiguousarray(np.moveaxis(full, c_ax, 1 if fmt == CL else 3))
        x = np.moveaxis(x, 1 if fmt == CL else 3, c_ax)
    y, _ = _check_forward(x, fmt, 1.25)
    _check_backward(x, y, fmt, 1.25, rng)


def test_emulated_zero_elements():
    """Exact zeros in the input: their angle is 0, their gradient 0, and an all-zero pair gives Y = 0."""
    rng = np.random.default_rng(7)
    x = _spectrogram(rng, (1, 1, 20, 6))
    x[:, :, 3:6] = 0
    x[:, :, :, 2] = 0
    y, _ = _check_forward(x, CF, 0.8)
    assert np.all(y[:, :, :, 2] == 0)
    gx = _check_backward(x, y, CF, 0.8, rng)
    assert np.all(gx[:, :, 3:6] == 0) and np.all(gx[:, :, :, 2] == 0)


@pytest.mark.parametrize('rate', [0.5, 0.8, 1.3, 3.7])
@pytest.mark.parametrize('fmt', [CF, CL])
def test_emulated_chunks_at_every_offset(rate, fmt):
    """Chunk lengths 1..T-1 of a 13-frame input: a chunk boundary at every offset.  The forward is bit-identical to
    the unchunked one; the backward writes every gX element (no NaN left) and agrees with the restatement."""
    rng = np.random.default_rng(8)
    T = 13
    x = _spectrogram(rng, (2, T, 33, 2) if fmt == CL else (2, 2, T, 33))
    y1, _ = emu_ts(x, fmt, rate)
    for Tc in range(1, T):
        y, K = _check_forward(x, fmt, rate, Tc)
        assert K == -(-T // Tc)
        assert y.tobytes() == y1.tobytes()
        gx = _check_backward(x, y, fmt, rate, np.random.default_rng(Tc), Tc)
        assert not np.isnan(gx).any()


@pytest.mark.parametrize('rate', [0.8, 1.25])
def test_long_input_phase_does_not_drift(rate):
    """At 5000 frames the RMS phase error of the last output frame is at least 10x below torchaudio's complex64 one
    (against complex128), measured on the same input; and every output keeps the pointwise bound."""
    ta = _torchaudio()
    rng = np.random.default_rng(9)
    T, F = 5000, 513
    x = _spectrogram(rng, (1, 1, T, F))
    y, _ = _check_forward(x, CF, rate)
    X = torch.from_numpy(x)
    adv = _phase_advance(F, 256, 'hop')
    ref = TR.torchaudio_layout(ta.functional.phase_vocoder(TR.torchaudio_layout(X.to(torch.complex128)), rate, adv))
    ta32 = TR.torchaudio_layout(ta.functional.phase_vocoder(TR.torchaudio_layout(X), rate, adv.float()))

    def rms_last(Y):
        d = torch.remainder(Y[..., -1, :].to(torch.complex128).angle() - ref[..., -1, :].angle() + math.pi,
                            2 * math.pi) - math.pi
        return float(d.pow(2).mean().sqrt())
    ours, theirs = rms_last(torch.from_numpy(y)), rms_last(ta32)
    assert ours * 10 <= theirs, (ours, theirs)


def test_chunk_choice():
    """PCEN's rule on input frames: one chunk while the columns fill a sixteenth of the resident threads."""
    lib = _lib()
    resident = 132 * 2048
    assert lib.kb_emu_ts_chunks(256 * 513, 427, resident) == 1           # cfg2 complex shape
    assert lib.kb_emu_ts_chunks(513, 25840, resident) == 32              # 10 min at 22.05 kHz, hop 512
    assert lib.kb_emu_ts_chunks(513, 200, resident) == 3
    assert lib.kb_emu_ts_chunks(513, 100, resident) == 1


def test_kernel_register_and_spill_budget():
    """The four time-stretch kernels do not spill (the register tiles must stay in registers)."""
    import re
    import shutil
    lib = os.path.join(_HERE, '..', 'kapre_b200', '_lib', 'libkapre_b200.so')
    if shutil.which('cuobjdump') is None or not os.path.exists(lib):
        pytest.skip('needs cuobjdump and the built library')
    out = subprocess.run(['cuobjdump', '-res-usage', lib], capture_output=True, text=True, check=True).stdout
    lines = out.splitlines()
    found = [(lines[i], lines[i + 1]) for i in range(len(lines) - 1) if 'kb_ts_' in lines[i]]
    assert len(found) == 4, found
    for name, res in found:
        m = re.search(r'REG:(\d+) STACK:(\d+)', res)
        assert m and int(m.group(1)) <= 128 and int(m.group(2)) == 0, (name, res)


# ------------------------------------------------------------------------------ the layer
def test_layer_validation():
    from kapre_b200.augmentation import TimeStretch
    for kw in ({'rate': 0.0}, {'rate': -1.0}, {'rate': float('nan')}, {'rate': float('inf')}, {'rate': True},
               {'rate': '2'}, {'rate': 1.0, 'data_format': 'channels_middle'}):
        with pytest.raises(ValueError):
            TimeStretch(**kw)
    TimeStretch(1e-3)
    TimeStretch(7)


def test_layer_config_round_trip():
    import kapre
    import kapre_b200
    from kapre_b200.augmentation import TimeStretch
    from kapre_b200.composed import Sequential, get_time_stretch_layer
    assert kapre.augmentation.TimeStretch is TimeStretch
    assert 'TimeStretch' not in kapre_b200.__all__
    layer = TimeStretch(1.3, data_format='channels_first', name='ts_x')
    cfg = layer.get_config()
    assert cfg['rate'] == 1.3 and cfg['data_format'] == 'channels_first' and cfg['name'] == 'ts_x'
    assert TimeStretch.from_config(cfg).get_config() == cfg
    model = get_time_stretch_layer(0.8, n_fft=512, hop_length=128, waveform_data_format='channels_first')
    assert [type(l).__name__ for l in model.layers] == ['STFT', 'TimeStretch', 'InverseSTFT']
    again = Sequential.from_config(model.get_config())
    assert again.get_config() == model.get_config()
