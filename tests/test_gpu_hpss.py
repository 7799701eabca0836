"""HPSS on the H100: hpss at benchmark size in both layouts, complex and magnitude input, bit for bit against the
float32 restatement (hpss_ref.py) over the device's own |X|; bit equality across batch positions, layouts and
strides; the waveform forms against the composition of the library's transforms with the restatement and their sum
against the input; gradients against torch.autograd (also through harmonic() to the waveform); launch counts, CUDA
graph replay, no-grad behaviour, non-finite isolation, power-of-two homogeneity and the ptxas budgets."""
import os
import re
import subprocess

import numpy as np
import pytest
import torch

import hpss_ref as R

pytestmark = pytest.mark.gpu

CL, CF = 'channels_last', 'channels_first'


def _cf(t, fmt):
    """A (B, T, K, C) / (B, C, T, K) tensor as (B, C, T, K)."""
    return t.permute(0, 3, 1, 2) if fmt == CL else t


def _spec(B, T, K, C, fmt, cplx, seed):
    g = torch.Generator(device='cuda').manual_seed(seed)
    shape = (B, T, K, C) if fmt == CL else (B, C, T, K)
    if cplx:
        return torch.complex(torch.randn(shape, generator=g, device='cuda'),
                             torch.randn(shape, generator=g, device='cuda'))
    return torch.rand(shape, generator=g, device='cuda')


def _mag(S):
    from kapre_b200 import ops
    return ops.magnitude(S) if S.is_complex() else S


@pytest.mark.parametrize('fmt', [CF, CL])
@pytest.mark.parametrize('cplx', [True, False])
def test_benchmark_size_bit_exact(fmt, cplx):
    from kapre_b200 import signal
    S = _spec(256, 216, 1025, 1, fmt, cplx, 1)
    h, p = signal.hpss(S, data_format=fmt)
    torch.cuda.synchronize()
    mag = _cf(_mag(S), fmt)
    for b in (0, 137, 255):
        m = mag[b:b + 1].cpu().numpy()
        X = _cf(S, fmt)[b:b + 1].cpu().numpy() if cplx else None
        rh, rp = R.hpss32(m, X, 31, 31, 2.0)
        np.testing.assert_array_equal(_cf(h, fmt)[b:b + 1].cpu().numpy(), rh)
        np.testing.assert_array_equal(_cf(p, fmt)[b:b + 1].cpu().numpy(), rp)


def test_bit_equality_across_positions_layouts_strides():
    from kapre_b200 import signal
    S = _spec(6, 150, 300, 2, CF, True, 2)
    ref = signal.hpss(S, kernel_size=(17, 63), margin=(1.0, 2.0), data_format=CF)
    cl = signal.hpss(S.permute(0, 2, 3, 1).contiguous(), kernel_size=(17, 63), margin=(1.0, 2.0), data_format=CL)
    part = signal.hpss(S[3:5], kernel_size=(17, 63), margin=(1.0, 2.0), data_format=CF)
    big = torch.zeros((6, 3, 160, 320), dtype=torch.complex64, device='cuda')
    big[:, ::2, 5:155, 7:307] = S
    strided = signal.hpss(big[:, ::2, 5:155, 7:307], kernel_size=(17, 63), margin=(1.0, 2.0), data_format=CF)
    for i in range(2):
        assert torch.equal(_cf(cl[i], CL), ref[i])
        assert torch.equal(part[i], ref[i][3:5])
        assert torch.equal(strided[i], ref[i])


def _wave(B, C, L, seed, fmt):
    rng = np.random.default_rng(seed)
    t = np.arange(L) / 22050.0
    x = 0.3 * np.sin(2 * np.pi * 440.0 * t)[None, None] + 0.05 * rng.standard_normal((B, C, L))
    x[:, :, ::2205] += 0.8                                          # clicks every 0.1 s
    x = x.astype(np.float32)
    return torch.from_numpy(x if fmt == CF else np.ascontiguousarray(x.transpose(0, 2, 1))).cuda()


@pytest.mark.parametrize('fmt', [CL, CF])
def test_waveform_round_trip_and_composition(fmt):
    from kapre_b200 import signal
    from kapre_b200.time_frequency import STFT, InverseSTFT
    y = _wave(3, 2, 22050 * 2, 3, fmt)
    h = signal.harmonic(y, n_fft=1024, data_format=fmt)
    p = signal.percussive(y, n_fft=1024, data_format=fmt)
    assert h.shape == y.shape and p.shape == y.shape
    # masks sum to 1 within a few ulp and the inverse reconstructs to ~1e-6 of the signal's peak
    assert float((h + p - y).abs().max()) < 2e-5 * float(y.abs().max())
    stft = STFT(n_fft=1024, pad_begin=True, pad_end=True, input_data_format=fmt, output_data_format=CL)
    istft = InverseSTFT(n_fft=1024, input_data_format=CL, output_data_format=fmt)
    X = stft.call(y)
    mag = _mag(X).permute(0, 3, 1, 2).cpu().numpy()
    rh, rp = R.hpss32(mag, X.permute(0, 3, 1, 2).cpu().numpy(), 31, 31, 2.0)
    for got, r in ((h, rh), (p, rp)):
        yr = istft.call(torch.from_numpy(np.ascontiguousarray(r.transpose(0, 2, 3, 1))).cuda())
        start = 1024 - 256
        yr = yr[:, :, start:start + y.shape[2]] if fmt == CF else yr[:, start:start + y.shape[1], :]
        assert torch.equal(got, yr)


def test_gradients_against_autograd():
    from kapre_b200 import signal
    for cplx, mask, power in ((True, False, 2.0), (False, False, 1.0), (False, True, 3.0), (True, True, 2.0)):
        S = _spec(2, 70, 90, 1, CF, cplx, 4)
        if not cplx:
            S = (S * 4).floor() / 4                                     # exact ties
        Sg = S.clone().requires_grad_(True)
        h, p = signal.hpss(Sg, kernel_size=(9, 13), power=power, mask=mask, margin=(1.0, 1.5), data_format=CF)
        gh, gp = torch.randn_like(h), torch.randn_like(p)
        (gS,) = torch.autograd.grad((h, p), Sg, (gh, gp))
        m = _mag(S).cpu().numpy()
        sh, sp = R.select(m, 9, 13)
        if cplx:
            leaf = S.cpu().to(torch.complex128).requires_grad_(True)
            rh, rp = R.hpss64(None, sh, sp, 9, 13, power, (1.0, 1.5), mask, X=leaf)
        else:
            leaf = S.cpu().double().requires_grad_(True)
            rh, rp = R.hpss64(leaf, sh, sp, 9, 13, power, (1.0, 1.5), mask)
        dt = torch.complex128 if (cplx and not mask) else torch.float64
        (ref,) = torch.autograd.grad((rh, rp), leaf, (gh.cpu().to(dt), gp.cpu().to(dt)))
        ok = torch.isfinite(ref.abs())
        err = ((gS.cpu().to(ref.dtype) - ref).abs() / (1 + ref.abs()))[ok]
        assert float(err.max()) < 2e-4 * 2 * (9 + 13), (cplx, mask, power)


def test_gradient_through_harmonic_to_waveform():
    """harmonic()'s gradient equals the same composition with the HPSS step replaced by the torch restatement at
    the indices the tie rule selects: the STFT and inverse STFT gradients are shared, so this checks the HPSS
    backward inside the pipeline."""
    from kapre_b200 import signal
    from kapre_b200.time_frequency import STFT, InverseSTFT
    y = _wave(2, 1, 8192, 5, CL).requires_grad_(True)
    out = signal.harmonic(y, n_fft=512, data_format=CL)
    g = torch.randn_like(out)
    (gy,) = torch.autograd.grad(out, y, g)
    stft = STFT(n_fft=512, pad_begin=True, pad_end=True, input_data_format=CL, output_data_format=CL)
    istft = InverseSTFT(n_fft=512, input_data_format=CL, output_data_format=CL)
    y2 = y.detach().clone().requires_grad_(True)
    X = stft.call(y2)
    Xc = X.permute(0, 3, 1, 2)
    sh, sp = R.select(_mag(X.detach()).permute(0, 3, 1, 2).cpu().numpy(), 31, 31)
    h, _ = R.hpss64(None, torch.from_numpy(sh).cuda(), torch.from_numpy(sp).cuda(), 31, 31, 2.0, X=Xc)
    yr = istft.call(h.permute(0, 2, 3, 1).contiguous())[:, 384:384 + 8192, :]
    (gr,) = torch.autograd.grad(yr, y2, g)
    assert float((gy - gr).abs().max()) < 1e-3 * float(gr.abs().max())


def test_launch_counts_capture_and_no_grad():
    from kapre_b200 import _native as N
    from kapre_b200 import signal
    from kapre_b200.composed import Sequential, get_stft_magnitude_layer
    from kapre_b200.time_frequency import HPSS
    y = _wave(2, 1, 22050, 6, CL)
    S = _spec(2, 100, 513, 1, CL, False, 6)

    def count(fn):
        fn()
        torch.cuda.synchronize()
        n0 = N.launch_count()
        r = fn()
        torch.cuda.synchronize()
        return N.launch_count() - n0, r
    assert count(lambda: signal.hpss(S, data_format=CL))[0] == 1
    assert count(lambda: signal.hpss(S, mask=True, data_format=CL))[0] == 1
    assert count(lambda: signal.harmonic(y, data_format=CL))[0] == 3
    seq = Sequential([*get_stft_magnitude_layer(n_fft=1024, input_data_format=CL, output_data_format=CL).layers,
                      HPSS('harmonic', data_format=CL)])
    n, out = count(lambda: seq(y))
    assert n == 2 and out.dtype == torch.float32
    # the backward is two launches
    Sg = S.clone().requires_grad_(True)
    h, p = signal.hpss(Sg, data_format=CL)
    torch.cuda.synchronize()
    n0 = N.launch_count()
    (h.sum() + p.sum()).backward()
    torch.cuda.synchronize()
    assert N.launch_count() - n0 == 2
    # no grad
    with torch.no_grad():
        h2, _ = signal.hpss(Sg, data_format=CL)
    assert h2.grad_fn is None and not h2.requires_grad and torch.equal(h2, h)
    # capture and replay
    ref = signal.hpss(S, data_format=CL)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        signal.hpss(S, data_format=CL)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        cap = signal.hpss(S, data_format=CL)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(cap[0], ref[0]) and torch.equal(cap[1], ref[1])


def test_non_finite_isolation():
    from kapre_b200 import signal
    S = _spec(3, 80, 120, 1, CF, False, 7)
    clean = signal.hpss(S, data_format=CF)
    Sb = S.clone()
    Sb[1, 0, 40, 60] = float('nan')
    Sb[2, 0, 10, 5] = float('inf')
    h, p = signal.hpss(Sb, data_format=CF)
    assert torch.equal(h[0], clean[0][0]) and torch.equal(p[0], clean[1][0])
    hit = np.zeros((80, 120), bool)
    hit[R.windows(80, 31).__eq__(40).any(axis=1), 60] = True
    hit[40, R.windows(120, 31).__eq__(60).any(axis=1)] = True
    np.testing.assert_array_equal(torch.isnan(h[1, 0]).cpu().numpy(), hit)
    np.testing.assert_array_equal(torch.isnan(p[1, 0]).cpu().numpy(), hit)
    ref = R.hpss32(Sb[2:3].cpu().numpy(), None, 31, 31, 2.0)
    np.testing.assert_array_equal(h[2:3].cpu().numpy(), ref[0])
    np.testing.assert_array_equal(p[2:3].cpu().numpy(), ref[1])


def test_power_of_two_homogeneity():
    """hpss(2^e S) = 2^e hpss(S) bit for bit with the masks unchanged, over the rungs of the scale-range ladder where
    the values stay normal: S in [2^-2, 1] and the outputs (masks >= 2^-7 here) down to 2^-100, and the complex
    parts, which can be far below |X|, down to 2^-60."""
    from kapre_b200 import signal
    S = (_spec(2, 60, 200, 1, CL, False, 8) * 0.75 + 0.25)
    X = torch.polar(S, S * 7.0)
    base = signal.hpss(S, margin=(2.0, 1.0), data_format=CL)
    base_m = signal.hpss(S, margin=(2.0, 1.0), mask=True, data_format=CL)
    base_x = signal.hpss(X, data_format=CL)
    for e in range(-100, 121, 20):
        s = 2.0 ** e
        got = signal.hpss(S * s, margin=(2.0, 1.0), data_format=CL)
        got_m = signal.hpss(S * s, margin=(2.0, 1.0), mask=True, data_format=CL)
        for i in range(2):
            assert torch.equal(got[i], base[i] * s), e
            assert torch.equal(got_m[i], base_m[i]), e
        if e >= -60:
            got_x = signal.hpss(X * s, data_format=CL)
            for i in range(2):
                assert torch.equal(got_x[i], base_x[i] * s), e


def test_ptxas_budgets():
    """The HPSS kernels use no stack and no local memory (no spills).  As built: the forward 64 registers at the
    default kernel sizes (window slots 32 / 32) and at most 96 with a 64-slot window, the first gradient pass at
    most 128, the gather pass at most 40."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    lib = os.path.join(root, 'kapre_b200', '_lib', 'libkapre_b200.so')
    out = subprocess.run(['cuobjdump', '-res-usage', lib], capture_output=True, text=True, check=True).stdout
    found = re.findall(r'Function _Z\d+(kb_hpss_\w+):\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)', out)
    assert len(found) == 9, found
    for name, regs, stack, local in found:
        regs, stack, local = int(regs), int(stack), int(local)
        assert stack == 0 and local == 0, (name, stack, local)
        if name.startswith('kb_hpss_gather'):
            assert regs <= 40, (name, regs)
        elif name.endswith('ILi32ELi32ELi0EEv12KbHpssParams'):
            assert regs <= 64, (name, regs)
        elif 'ELi0EE' in name:
            assert regs <= 96, (name, regs)
        else:
            assert regs <= 128, (name, regs)
