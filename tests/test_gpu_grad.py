"""Gradients on the H100: vector-Jacobian products of the layers and fused stacks against the float64 restatement
(grad_ref.py), adjoint identities at the BASELINE cfg2 shape, and a source-separation mask gradient.

Tolerances are relative to the largest reference value (``_rel``) or the reference's norm (``_rel_l2``):
* linear layers (STFT, InverseSTFT, ApplyFilterbank): 1e-4.  The kernels transform in float32 (about 6e-8 relative
  rounding per operation, O(log N) operations per output for the FFT kernels, O(N) for the direct DFT of n_fft 98)
  and an output sums at most ceil(win / hop) frames;
* Magnitude: 1e-5 (one product and one division per element);
* decibel stacks: 2e-3 in L2.  d dB / dx = 10 / (ln 10 x) magnifies the float32 error of small x, and an element
  within rounding of the dynamic-range threshold may be clamped on one side and not on the other, which moves its
  gradient to the item's maximum.
"""
import numpy as np
import pytest
import torch

import grad_ref as R

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    import kapre_b200 as K

CL, CF = 'channels_last', 'channels_first'
CASES = [(256, 256, 64), (512, 384, 128), (1024, 1024, 256), (2048, 2048, 512), (400, 400, 160), (1000, 1000, 250),
         (96, 128, 32), (75, 75, 25), (98, 98, 49), (256, 200, 240), (512, 512, 600)]
PADS = [(False, False), (True, False), (False, True), (True, True)]


def _rel(got, want, tol):
    got = got.detach().cpu().to(want.dtype)
    err = float((got - want).abs().max())
    scale = float(want.abs().max())
    assert err <= tol * scale, (err, scale)


def _rel_l2(got, want, tol):
    got = got.detach().cpu().to(want.dtype)
    err = float(torch.linalg.vector_norm(got - want))
    assert err <= tol * float(torch.linalg.vector_norm(want)), (err, float(torch.linalg.vector_norm(want)))


def _wave(rng, B, C, L, fmt):
    return torch.from_numpy(rng.standard_normal((B, L, C) if fmt == CL else (B, C, L)).astype(np.float32))


def _cplx(rng, shape):
    return torch.from_numpy((rng.standard_normal(shape) + 1j * rng.standard_normal(shape)).astype(np.complex64))


def _grad(layer, x, g):
    """(output, d<layer(x), g>/dx) through kapre_b200 on the GPU; also checks that recording for autograd leaves the
    forward output bit-identical."""
    xd = x.cuda().requires_grad_(True)
    y = layer(xd)
    with torch.no_grad():
        y0 = layer(x.cuda())
    assert torch.equal(y.detach(), y0)
    (gx,) = torch.autograd.grad(y, xd, grad_outputs=g.cuda().to(y.dtype))
    return y, gx


@pytest.mark.parametrize('case', CASES, ids=lambda c: 'n%d_w%d_h%d' % c)
@pytest.mark.parametrize('pads', PADS, ids=lambda p: 'pb%d_pe%d' % p)
@pytest.mark.parametrize('C', [1, 2])
def test_stft_vjp(case, pads, C):
    n_fft, win, hop = case
    pb, pe = pads
    if pb and hop > n_fft:
        pytest.skip('pad_begin needs hop <= n_fft')
    rng = np.random.default_rng(n_fft * 3 + hop + C)
    for fi, fo in ((CF, CL), (CL, CF)):
        x = _wave(rng, 2, C, 3 * max(n_fft, win) + 2 * hop + 13, fi)
        layer = K.STFT(n_fft=n_fft, win_length=win, hop_length=hop, pad_begin=pb, pad_end=pe, input_data_format=fi,
                       output_data_format=fo)
        y0 = layer(x.cuda())
        g = _cplx(rng, tuple(y0.shape))
        _, gx = _grad(layer, x, g)
        _, want = R.vjp(lambda t: R.stft(t, n_fft, win, hop, None, pb, pe, fi, fo), x.double(), g.to(torch.complex128))
        _rel(gx, want, 1e-4)


@pytest.mark.parametrize('case', CASES, ids=lambda c: 'n%d_w%d_h%d' % c)
@pytest.mark.parametrize('C', [1, 2])
def test_istft_vjp(case, C):
    n_fft, win, hop = case
    rng = np.random.default_rng(n_fft + hop + C)
    for fs, fw in ((CF, CL), (CL, CF)):
        T = 7
        shape = (2, T, n_fft // 2 + 1, C) if fs == CL else (2, C, T, n_fft // 2 + 1)
        X = _cplx(rng, shape)
        # hamming: no zero samples, so the dual window stays finite when hop > win_length
        layer = K.InverseSTFT(n_fft=n_fft, win_length=win, hop_length=hop, forward_window_name='hamming_window',
                              input_data_format=fs, output_data_format=fw)
        y0 = layer(X.cuda())
        g = torch.from_numpy(rng.standard_normal(tuple(y0.shape)).astype(np.float32))
        _, gX = _grad(layer, X, g)
        _, want = R.vjp(lambda t: R.istft(t, n_fft, win, hop, 'hamming_window', fs, fw), X.to(torch.complex128),
                        g.double())
        _rel(gX, want, 1e-4)


@pytest.mark.parametrize('C', [1, 2])
def test_magnitude_filterbank_decibel_vjp(C):
    rng = np.random.default_rng(C)
    X = _cplx(rng, (2, C, 9, 257))
    X[0, 0, 0, :3] = 0
    g = torch.from_numpy(rng.standard_normal(tuple(X.shape)).astype(np.float32))
    _, gX = _grad(K.Magnitude(), X, g)
    _rel(gX, R.vjp(R.magnitude, X.to(torch.complex128), g.double())[1], 1e-5)
    for fmt in (CF, CL):
        layer = K.ApplyFilterbank('mel', dict(sample_rate=16000, n_freq=257, n_mels=40), data_format=fmt)
        x = torch.from_numpy(rng.random((2, C, 9, 257) if fmt == CF else (2, 9, 257, C)).astype(np.float32))
        g = torch.from_numpy(rng.standard_normal((2, C, 9, 40) if fmt == CF else (2, 9, 40, C)).astype(np.float32))
        _, gx = _grad(layer, x, g)
        _rel(gx, R.vjp(lambda t: R.apply_filterbank(t, layer.filterbank, fmt), x.double(), g.double())[1], 1e-4)
    for dyn in (80.0, 20.0):                    # 20 dB: the clamp binds
        x = torch.from_numpy((rng.random((3, C, 11, 40)) ** 4).astype(np.float32))
        x[1, 0, 2, 3] = x[1, 0, 5, 7] = 2.0     # tied maxima
        g = torch.from_numpy(rng.standard_normal(tuple(x.shape)).astype(np.float32))
        _, gx = _grad(K.MagnitudeToDecibel(dynamic_range=dyn), x, g)
        _rel_l2(gx, R.vjp(lambda t: R.magnitude_to_decibel(t, 1.0, 1e-5, dyn), x.double(), g.double())[1], 2e-3)


def test_decibel_backward_workspace_is_left_zero():
    x = torch.rand(4, 5000, device='cuda') ** 4
    g = torch.randn_like(x)
    ws = torch.zeros(12, dtype=torch.int32, device='cuda')
    gx = torch.empty_like(x)
    import ctypes
    dbc = K._native.DbCfg(1.0, 1e-5, 20.0)
    K._native.check(K._native.lib().kapre_magnitude_to_decibel_backward(
        ctypes.c_void_p(x.data_ptr()), ctypes.c_void_p(g.data_ptr()), ctypes.c_void_p(gx.data_ptr()), 4, 5000,
        ctypes.byref(dbc), ctypes.c_void_p(ws.data_ptr()), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))
    torch.cuda.synchronize()
    assert int(ws.abs().sum()) == 0
    _rel_l2(gx, R.vjp(lambda t: R.magnitude_to_decibel(t, 1.0, 1e-5, 20.0), x.cpu().double(), g.cpu().double())[1], 2e-3)


def _stack_ref(kind, n_fft, hop, fmt, db, dyn, fb):
    def f(t):
        s = R.magnitude(R.stft(t, n_fft, n_fft, hop, None, False, False, fmt, fmt))
        if fb is not None:
            s = R.apply_filterbank(s, fb, fmt)
        if kind == 'mfcc':
            s = R.magnitude_to_decibel(s, 1.0, 1e-5, dyn)
            s = R.apply_filterbank(s, K.signal.dct2_htk_matrix(fb.shape[1], 20), fmt)
        elif db:
            s = R.magnitude_to_decibel(s, 1.0, 1e-5, dyn)
        return s
    return f


@pytest.mark.parametrize('kind,db,dyn', [('mel', False, 80.0), ('mel', True, 80.0), ('mel', True, 15.0),
                                         ('stftmag', True, 80.0), ('stftmag', True, 15.0), ('log', True, 80.0),
                                         ('mfcc', True, 80.0)])
@pytest.mark.parametrize('fmt', [CF, CL])
@pytest.mark.parametrize('n_fft,hop', [(512, 128), (1024, 256), (400, 160)])
def test_fused_stack_vjp(kind, db, dyn, fmt, n_fft, hop):
    rng = np.random.default_rng(n_fft + int(dyn) + db)
    common = dict(n_fft=n_fft, hop_length=hop, input_data_format=fmt, output_data_format=fmt)
    if kind == 'stftmag':
        model, fb = K.get_stft_magnitude_layer(return_decibel=db, db_dynamic_range=dyn, **common), None
    elif kind == 'log':
        model = K.get_log_frequency_spectrogram_layer(sample_rate=16000, return_decibel=db, db_dynamic_range=dyn,
                                                      **common)
        fb = model.layers[2].filterbank
    else:
        model = K.get_melspectrogram_layer(sample_rate=16000, n_mels=64, return_decibel=db, db_dynamic_range=dyn,
                                           **common)
        fb = model.layers[2].filterbank
        if kind == 'mfcc':
            model.add(K.LogmelToMFCC(n_mfccs=20, data_format=fmt))
    x = _wave(rng, 2, 2 if fmt == CL else 1, 8000, fmt)
    y0 = model(x.cuda())
    g = torch.from_numpy(rng.standard_normal(tuple(y0.shape)).astype(np.float32))
    _, gx = _grad(model, x, g)
    _, want = R.vjp(_stack_ref(kind, n_fft, hop, fmt, db, dyn, fb), x.double(), g.double())
    _rel_l2(gx, want, 2e-3 if db else 1e-4)


def _dot(a, b):
    if a.is_complex():
        return float((a.real.double() * b.real.double()).sum() + (a.imag.double() * b.imag.double()).sum())
    return float((a.double() * b.double()).sum())


def _norm(a):
    return float(a.detach().abs().double().square().sum()) ** 0.5


def test_adjoint_identities_cfg2():
    """<A x, y> = <x, A^T y> for STFT and InverseSTFT at BASELINE cfg2 (batch 256, 5 s at 22.05 kHz, n_fft 1024,
    hop 256), accumulated in float64."""
    torch.manual_seed(0)
    x = torch.randn(256, 1, 110250, device='cuda')
    stft, istft = K.get_perfectly_reconstructing_stft_istft(1024, 256, CF, CF)
    for layer in (stft, K.STFT(n_fft=1024, hop_length=256, input_data_format=CF, output_data_format=CF)):
        xg = x.clone().requires_grad_(True)
        S = layer(xg)
        Y = torch.randn_like(S)
        (gx,) = torch.autograd.grad(S, xg, grad_outputs=Y)
        # both sides are float32 transforms (relative error ~1e-6 in norm): |<A x, y> - <x, A^T y>| <= 1e-5 |Ax| |y|
        lhs, rhs = _dot(S.detach(), Y), _dot(x, gx)
        assert abs(lhs - rhs) <= 1e-5 * _norm(S) * _norm(Y), (lhs, rhs)
        Xs = S.detach().clone().requires_grad_(True)
        y = istft(Xs)
        gy = torch.randn_like(y)
        (gX,) = torch.autograd.grad(y, Xs, grad_outputs=gy)
        lhs, rhs = _dot(y.detach(), gy), _dot(Xs.detach(), gX)
        assert abs(lhs - rhs) <= 1e-5 * _norm(y) * _norm(gy), (lhs, rhs)
        del S, Y, gx, Xs, y, gy, gX
        torch.cuda.empty_cache()


@pytest.mark.parametrize('fmt', [CF, CL])
def test_source_separation_mask_gradient(fmt):
    """d ||istft(M * stft(x)) - s||^2 / dM through get_perfectly_reconstructing_stft_istft."""
    rng = np.random.default_rng(5)
    n_fft, hop = 512, 128
    stft, istft = K.get_perfectly_reconstructing_stft_istft(n_fft, hop, fmt, fmt)
    x = _wave(rng, 2, 1, 6000, fmt)
    s = _wave(rng, 2, 1, 6000, fmt)
    S = stft(x.cuda())
    M = torch.from_numpy(rng.random(tuple(S.shape)).astype(np.float32)).cuda().requires_grad_(True)
    y = istft(M * S)
    sl = (slice(None), slice(n_fft - hop, n_fft - hop + 6000)) if fmt == CL else \
        (slice(None), slice(None), slice(n_fft - hop, n_fft - hop + 6000))
    loss = ((y[sl] - s.cuda()) ** 2).sum()
    (gM,) = torch.autograd.grad(loss, M)

    Sr = R.stft(x.double(), n_fft, n_fft, hop, 'hann_window', True, True, fmt, fmt)
    Mr = M.detach().cpu().double().requires_grad_(True)
    yr = R.istft(Mr * Sr, n_fft, n_fft, hop, 'hann_window', fmt, fmt)
    ((yr[sl] - s.double()) ** 2).sum().backward()
    _rel(gM, Mr.grad, 1e-4)


def test_double_backward_raises():
    x = torch.randn(1, 1, 4096, device='cuda', requires_grad=True)
    y = K.STFT(n_fft=512, hop_length=128, input_data_format=CF, output_data_format=CF)(x)
    (gx,) = torch.autograd.grad(y.abs().sum(), x, create_graph=True)
    with pytest.raises(RuntimeError, match='twice'):
        gx.sum().backward()


def test_no_grad_path_is_untouched():
    """Without requires_grad the layers return plain tensors (no autograd node), as before."""
    x = torch.randn(2, 1, 4096, device='cuda')
    y = K.get_melspectrogram_layer(n_fft=512, hop_length=128, return_decibel=True, input_data_format=CF,
                                   output_data_format=CF)(x)
    assert y.grad_fn is None and not y.requires_grad
    with torch.no_grad():
        y = K.STFT(n_fft=512, input_data_format=CF, output_data_format=CF)(x.requires_grad_(True))
    assert y.grad_fn is None
