"""Onsets, tempo and beats on the H100: the benchmark size in both layouts against the float64 restatement
(rhythm_ref.py), the waveform forms bit for bit against the library's own launches run one by one, click-train and
silence anchors, gradients (through the waveform path and detrend), launch counts, CUDA graph replay of beat_track,
no-grad behaviour, power-of-two homogeneity and the ptxas budgets."""
import os
import re
import subprocess

import numpy as np
import pytest
import torch

import rhythm_ref as R

pytestmark = pytest.mark.gpu

CL, CF = 'channels_last', 'channels_first'
SR, HOP = 22050, 512


def _rows(t, fmt):
    """(B, T, C) / (B, C, T) -> (B, C, T) numpy."""
    t = t.detach().cpu().numpy()
    return t.transpose(0, 2, 1) if fmt == CL else t


def _wave(B, C, L, fmt, seed=0, bpm=120.0):
    rng = np.random.default_rng(seed)
    x = 0.02 * rng.standard_normal((B, C, L))
    per = int(round(60.0 / bpm * SR))
    for k in range(0, L, per):
        x[:, :, k:k + 200] += np.hanning(400)[200:] * np.sign(rng.standard_normal((B, C, 1)))
    x = x.astype(np.float32)
    return torch.from_numpy(x if fmt == CF else np.ascontiguousarray(x.transpose(0, 2, 1))).cuda()


def _feature(w, fmt):
    """The library's launches one by one: centred |STFT|, squaring, ApplyFilterbank, MagnitudeToDecibel."""
    from kapre_b200 import backend, ops, signal
    stft, fb = signal._rhythm_frontend(SR, 2048, HOP, 128, 0.0, None)
    X = signal._centred_magnitude(w, stft, fmt, True)
    return backend.magnitude_to_decibel(ops.apply_filterbank(X * X, fb, fmt), ref_value=1.0, amin=1e-10,
                                        dynamic_range=80.0)


@pytest.mark.parametrize('fmt', [CF, CL])
def test_benchmark_size_against_reference(fmt):
    from kapre_b200 import signal
    w = _wave(256, 1, 5 * SR, fmt, 1)
    S = _feature(w, fmt)
    for agg in ('mean', 'median'):
        e = signal.onset_strength(w, aggregate=agg, data_format=fmt)
        e2 = signal.onset_strength(S=S, aggregate=agg, data_format=fmt)
        assert torch.equal(e, e2)
        Sc = (S.permute(0, 3, 1, 2) if fmt == CL else S).cpu().numpy()
        got = _rows(e, fmt)
        for b in (0, 101, 255):
            ref = R.onset_strength_row(Sc[b, 0], 1, 1, agg, 2)
            d = np.abs(got[b, 0].view(np.int32).astype(np.int64) - ref.view(np.int32).astype(np.int64))
            assert d.max() <= (0 if agg == 'median' else 1)
    e = signal.onset_strength(w, data_format=fmt)
    tg = signal.tempogram(onset_envelope=e, data_format=fmt)
    tgc = (tg.permute(0, 3, 1, 2) if fmt == CL else tg).cpu().numpy()
    ec = _rows(e, fmt)
    for b in (0, 255):
        ref = R.tempogram_row(ec[b, 0], 384)
        assert np.abs(tgc[b, 0] - ref).max() <= 388 * 2.0 ** -24 + 1e-12
    t = signal.tempo(onset_envelope=e, data_format=fmt).cpu().numpy()
    bpm, lp = R.tempo_prior(344, SR, HOP)
    tg344 = signal.tempogram(onset_envelope=e, win_length=344, data_format=fmt)
    tg344 = (tg344.permute(0, 3, 1, 2) if fmt == CL else tg344).cpu().numpy()
    for b in (0, 17, 255):
        sc = np.sort(R.tempo_scores(tg344[b, 0].astype(np.float64).mean(axis=0), lp))
        if sc[-1] - sc[-2] > 1e-6 * abs(sc[-1]):         # decided beyond rounding
            assert t[b, 0] == np.float32(R.tempo_row(tg344[b, 0], lp, bpm))
    tempo, beats = signal.beat_track(w, data_format=fmt)
    em = _rows(signal.onset_strength(w, aggregate='median', data_format=fmt), fmt)
    bm = _rows(beats, fmt)
    checked = 0
    for b in (0, 101, 255):
        if R.beat_margin(em[b, 0], float(tempo[b, 0]), SR, HOP) <= 1e-9:
            continue                                   # a decision within rounding of the device's exp, log and fma
        _, ref = R.beat_track_row(em[b, 0], float(tempo[b, 0]), SR, HOP)
        np.testing.assert_array_equal(np.nonzero(bm[b, 0])[0], ref)
        checked += 1
    assert checked >= 2
    # a given tempogram is used with its own lag count (the default 384 here, not ac_size's 344)
    t384 = signal.tempo(tg=tg, data_format=fmt).cpu().numpy()
    bpm384, lp384 = R.tempo_prior(384, SR, HOP)
    checked = 0
    for b in (0, 17, 255):
        sc = np.sort(R.tempo_scores(tgc[b, 0].astype(np.float64).mean(axis=0), lp384))
        if sc[-1] - sc[-2] > 1e-6 * abs(sc[-1]):
            assert t384[b, 0] == np.float32(R.tempo_row(tgc[b, 0], lp384, bpm384))
            checked += 1
    assert checked >= 1


def test_bit_equality_across_positions_layouts_strides():
    from kapre_b200 import signal
    w = _wave(5, 2, 3 * SR, CF, 2)
    S = _feature(w, CF)
    ref = signal.onset_strength(S=S, max_size=3, aggregate='median', data_format=CF)
    cl = signal.onset_strength(S=S.permute(0, 2, 3, 1).contiguous(), max_size=3, aggregate='median', data_format=CL)
    assert torch.equal(cl.permute(0, 2, 1), ref)
    assert torch.equal(signal.onset_strength(S=S[2:4], max_size=3, aggregate='median', data_format=CF), ref[2:4])
    big = torch.zeros((5, 3, S.shape[2] + 4, 140), device='cuda')
    big[:, ::2, 2:-2, 6:134] = S
    assert torch.equal(signal.onset_strength(S=big[:, ::2, 2:-2, 6:134], max_size=3, aggregate='median',
                                             data_format=CF), ref)
    t_ref, b_ref = signal.beat_track(onset_envelope=ref, data_format=CF)
    t2, b2 = signal.beat_track(onset_envelope=ref[3:], data_format=CF)
    assert torch.equal(t2, t_ref[3:]) and torch.equal(b2, b_ref[3:])


@pytest.mark.parametrize('bpm', [90.0, 120.0, 150.0])
def test_click_train_anchors(bpm):
    from kapre_b200 import signal
    w = _wave(2, 1, 20 * SR, CF, 3, bpm)
    tempo, beats = signal.beat_track(w, data_format=CF)
    lag = 60.0 * SR / HOP / bpm
    for b in range(2):
        t = float(tempo[b, 0])
        assert abs(60.0 * SR / HOP / t - lag) <= 1.0, (t, bpm)
        frames = np.nonzero(beats[b, 0].cpu().numpy())[0]
        p = int(np.rint(60.0 * SR / HOP / t))
        assert frames.size > 10
        assert np.all(np.abs(np.diff(frames) - p) <= 1)


def test_onset_detect_clicks():
    from kapre_b200 import signal
    L = 6 * SR
    x = np.zeros((1, 1, L), np.float32)
    times = [0.5, 1.3, 2.2, 3.0, 4.1, 5.2]
    for s in times:
        k = int(s * SR)
        x[0, 0, k:k + 300] = np.sin(np.arange(300) * 0.3) * np.linspace(1, 0, 300)
    mask = signal.onset_detect(torch.from_numpy(x).cuda(), data_format=CF)[0, 0].cpu().numpy()
    found = np.nonzero(mask)[0]
    want = np.rint(np.array([int(s * SR) for s in times]) / HOP).astype(int)
    assert found.size == want.size
    assert np.all(np.abs(found - want) <= 1), (found, want)


def test_silence():
    from kapre_b200 import signal
    w = torch.zeros((2, 3 * SR, 1), device='cuda')
    e = signal.onset_strength(w, data_format=CL)
    assert torch.count_nonzero(e) == 0
    assert not signal.onset_detect(w, data_format=CL).any()
    tempo, beats = signal.beat_track(w, data_format=CL)
    assert torch.count_nonzero(tempo) == 0 and not beats.any()


def test_gradients():
    from kapre_b200 import signal
    g = torch.Generator(device='cuda').manual_seed(4)
    for agg in ('mean', 'median'):
        S = torch.randn((2, 1, 30, 17), generator=g, device='cuda').to(torch.float64)
        S = (S + torch.arange(17, device='cuda') * 1e-3).float().requires_grad_()
        e = signal.onset_strength(S=S, max_size=3, lag=2, aggregate=agg, data_format=CF)
        ge = torch.randn(e.shape, generator=g, device='cuda')
        e.backward(ge)
        for b in range(2):
            St = S[b, 0].detach().cpu().double().requires_grad_()
            R.onset_strength_torch(St, 2, 3, agg, 2).backward(ge[b, 0].cpu().double())
            np.testing.assert_allclose(S.grad[b, 0].cpu().numpy(), St.grad.numpy(), rtol=1e-5, atol=1e-6)
    # detrend: the gradient through lfilter(b=[1, -1], a=[1, -0.99]) is the adjoint of its impulse response
    e0 = torch.rand((1, 1, 200), generator=g, device='cuda').requires_grad_()
    bb = torch.tensor([[[1.0, -1.0]]], device='cuda')
    aa = torch.tensor([[[1.0, -0.99]]], device='cuda')
    from kapre_b200 import ops
    y = ops.lfilter(e0, bb, aa, clamp=False, data_format=CF)
    v = torch.randn(y.shape, generator=g, device='cuda')
    y.backward(v)
    h = np.r_[1.0, -0.01 * 0.99 ** np.arange(199)]
    vv = v[0, 0].cpu().double().numpy()
    ref = np.array([np.dot(h[:200 - t], vv[t:]) for t in range(200)])
    np.testing.assert_allclose(e0.grad[0, 0].cpu().numpy(), ref, rtol=1e-4, atol=1e-4)
    # through the waveform path: the gradient reaching the waveform is the existing backward passes applied to the
    # onset gradient of S
    w = _wave(1, 1, SR, CF, 5).requires_grad_()
    S = _feature(w, CF)
    e = signal.onset_strength(S=S, detrend=True, data_format=CF)
    v = torch.randn(e.shape, generator=g, device='cuda')
    gS, gw = torch.autograd.grad((e * v).sum(), [S, w], retain_graph=True)
    gw2, = torch.autograd.grad(S, w, gS)
    assert torch.equal(gw, gw2) and torch.isfinite(gw).all() and gw.abs().sum() > 0
    w2 = w.detach().clone().requires_grad_()
    (signal.onset_strength(w2, detrend=True, data_format=CF) * v).sum().backward()
    assert torch.equal(w2.grad, gw)


def test_launch_counts():
    from kapre_b200 import _native, signal
    w = _wave(2, 1, 2 * SR, CL, 6)
    e = signal.onset_strength(w, data_format=CL)
    torch.cuda.synchronize()

    def count(fn):
        n0 = _native.launch_count()
        fn()
        torch.cuda.synchronize()
        return _native.launch_count() - n0
    S = _feature(w, CL)
    n_feature = count(lambda: _feature(w, CL))
    assert count(lambda: signal.onset_strength(S=S, data_format=CL)) == 1
    assert count(lambda: signal.onset_strength(w, data_format=CL)) == 1 + n_feature
    assert count(lambda: signal.tempogram(onset_envelope=e, data_format=CL)) == 1
    assert count(lambda: signal.tempo(onset_envelope=e, data_format=CL)) == 3
    tg = signal.tempogram(onset_envelope=e, data_format=CL)
    assert count(lambda: signal.tempo(tg=tg, data_format=CL)) == 2
    assert count(lambda: signal.tempo(tg=tg, aggregate=None, data_format=CL)) == 1
    assert count(lambda: signal.onset_detect(onset_envelope=e, data_format=CL)) == 1
    assert count(lambda: signal.beat_track(onset_envelope=e, data_format=CL)) == 4
    assert count(lambda: signal.beat_track(onset_envelope=e, bpm=120.0, data_format=CL)) == 1
    Sg = S.clone().requires_grad_()
    out = signal.onset_strength(S=Sg, data_format=CL)
    assert count(lambda: out.sum().backward()) == 2


def test_cuda_graph_beat_track():
    from kapre_b200 import signal
    w = _wave(3, 1, 4 * SR, CF, 7)
    t0, b0 = signal.beat_track(w, data_format=CF)
    static = w.clone()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        signal.beat_track(static, data_format=CF)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        tg, bg = signal.beat_track(static, data_format=CF)
    w2 = _wave(3, 1, 4 * SR, CF, 8, 100.0)
    static.copy_(w2)
    graph.replay()
    t2, b2 = signal.beat_track(w2, data_format=CF)
    torch.cuda.synchronize()
    assert torch.equal(tg, t2) and torch.equal(bg, b2)
    static.copy_(w)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(tg, t0) and torch.equal(bg, b0)


def test_no_grad_behaviour():
    from kapre_b200 import signal
    w = _wave(1, 1, 2 * SR, CF, 9).requires_grad_()
    e = signal.onset_strength(w, data_format=CF)
    assert e.grad_fn is not None
    for out in (signal.tempo(w, data_format=CF), signal.onset_detect(w, data_format=CF),
                *signal.beat_track(w, data_format=CF)):
        assert out.grad_fn is None
    with pytest.raises(ValueError):
        signal.tempogram(onset_envelope=e, data_format=CF)
    with pytest.raises(ValueError):
        signal.tempogram(w, data_format=CF)
    with torch.no_grad():
        assert signal.tempogram(onset_envelope=e, data_format=CF).grad_fn is None


@pytest.mark.parametrize('agg', ['mean', 'median'])
def test_power_of_two_homogeneity(agg):
    from kapre_b200 import signal
    g = torch.Generator(device='cuda').manual_seed(10)
    S = torch.rand((3, 1, 40, 65), generator=g, device='cuda') + 0.5
    base = signal.onset_strength(S=S, max_size=3, aggregate=agg, data_format=CF)
    for k in (-100, -60, -20, -1, 1, 20, 60, 100):
        got = signal.onset_strength(S=S * 2.0 ** k, max_size=3, aggregate=agg, data_format=CF)
        assert torch.equal(got, base * 2.0 ** k), k


def test_ptxas_budgets():
    """The rhythm kernels use no stack and no local memory (no spills).  As built: onset forward 72 registers,
    its first gradient pass 80, the gather 26, the tempogram 48, the tempo partial sums 40 and decision 40, peak
    picking 32, the beat tracker 70."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    lib = os.path.join(root, 'kapre_b200', '_lib', 'libkapre_b200.so')
    out = subprocess.run(['cuobjdump', '-res-usage', lib], capture_output=True, text=True, check=True).stdout
    found = re.findall(r'Function _Z\d+(kb_(?:onset|tempogram|tempo|peak|beat)\w*_kernel\w*):\s*REG:(\d+) '
                       r'STACK:(\d+) SHARED:\d+ LOCAL:(\d+)', out)
    assert len(found) == 8, found
    for name, regs, stack, local in found:
        assert int(stack) == 0 and int(local) == 0, (name, stack, local)
        assert int(regs) <= 96, (name, regs)
