"""Image-source room impulse responses on an H100: simulate_rir_ism against the float64 restatement (rir_ref.py) within
its bound at bench-like sizes, bit-independence of batch, neighbours, strides and start, launch counts, RoomReverb
against the composition rebuilt from its draw, its gradient against the convolution's adjoint, Sequential with the
fused log-mel and CUDA graph capture, argument checks before any launch, and the kernel's register budget."""
import os
import re
import subprocess

import numpy as np
import pytest
import torch

import rir_ref as RR

pytestmark = pytest.mark.gpu

CF, CL = 'channels_first', 'channels_last'
_LIB = os.path.join(os.path.dirname(os.path.abspath(__file__)), '..', 'kapre_b200', '_lib', 'libkapre_b200.so')


def _sim(*a, **k):
    from kapre_b200 import signal
    return signal.simulate_rir_ism(*a, **k)


@pytest.mark.parametrize('room,rt60,fs', [((5.0, 4.0, 3.0), 0.5, 16000.0), ((3.0, 3.0, 2.5), 0.3, 48000.0)])
def test_parity_at_bench_size(room, rt60, fs):
    from kapre_b200 import backend
    alpha = backend.inverse_sabine(rt60, room)
    src, mics = np.array([1.2, 1.1, 1.3]), np.array([[2.7, 2.2, 1.6], [0.6, 2.5, 2.1]])
    L = int(rt60 * fs) // 2
    h = _sim(room, src, mics, None, alpha, L, sample_rate=fs, data_format=CF)
    got = h.cpu().double().numpy()
    for m in range(2):
        want, bound = RR.rir(room, src, mics[m], RR.betas(np.full(6, alpha)), L, 81, fs)
        err = np.abs(got[0, m] - want)
        assert np.all(err <= bound), (m, float(np.max(err - bound)))
        assert np.max(np.abs(want)) > 0


def test_bits_independent_of_batch_neighbours_strides_and_start():
    from kapre_b200 import ops
    rng = np.random.default_rng(0)
    B, M, L = 6, 3, 4000
    rooms = rng.uniform([3, 3, 2.5], [8, 8, 4], size=(B, 3))
    src = rng.uniform(0.5, rooms - 0.5)
    mics = rng.uniform(0.5, rooms[:, None, :] - 0.5, size=(B, M, 3))
    recs = np.zeros((B, 14))
    recs[:, :3], recs[:, 3:6], recs[:, 6:12], recs[:, 12] = rooms, src, 0.8, -1
    full_cf = ops.rir_ism(recs, mics, L, 81, 16000.0, 343.0, CF).cpu()
    full_cl = ops.rir_ism(recs, mics, L, 81, 16000.0, 343.0, CL).cpu()
    assert torch.equal(full_cl.transpose(1, 2), full_cf)
    for b in (0, 3, 5):
        alone = ops.rir_ism(recs[b:b + 1], mics[b:b + 1], L, 81, 16000.0, 343.0, CF).cpu()
        assert torch.equal(alone[0], full_cf[b])
        r = recs[b:b + 1].copy()
        for start in (1, 333, 2500):
            r[0, 13] = start
            part = ops.rir_ism(r, mics[b:b + 1], L - start, 81, 16000.0, 343.0, CL).cpu()
            assert torch.equal(part[0].T, full_cf[b][:, start:])
    assert torch.count_nonzero(full_cf) > 0


def test_one_launch_per_call():
    from kapre_b200 import _native as N
    _sim((5.0, 4.0, 3.0), (1.0, 1.0, 1.0), [[2.0, 2.0, 2.0]], None, 0.3, 1000)
    torch.cuda.synchronize()
    n0 = N.launch_count()
    _sim(np.tile([5.0, 4.0, 3.0], (8, 1)), (1.0, 1.0, 1.0), np.full((8, 4, 3), 2.0), 3, np.full(6, 0.3), 8000,
         sample_rate=48000.0)
    assert N.launch_count() - n0 == 1


def _unit(h):
    """Each row scaled to unit L2 norm in the kernel's fixed order: lane l adds squares l, l + 32, ... in float64, then
    the 32 lane sums are added in lane order."""
    h64 = h.astype(np.float64)
    B, K = h64.shape
    pad = np.zeros((B, -(-K // 32) * 32))
    pad[:, :K] = h64 * h64
    part = np.zeros((B, 32))
    for row in range(pad.shape[1] // 32):
        part = part + pad[:, 32 * row:32 * row + 32]
    s = np.zeros(B)
    for lane in range(32):
        s = s + part[:, lane]
    return (h64 * (1.0 / np.sqrt(s))[:, None]).astype(np.float32)


def _composition(layer, choice, x):
    """RoomReverb rebuilt from a draw: simulate_rir_ism from sample 0, trimmed at the direct path, unit norm, Convolve,
    cropped to the input length."""
    from kapre_b200 import backend
    from kapre_b200.signal import Convolve
    room, rt60, source, mic = choice
    start = layer.records(room, rt60, source, mic)[:, 13].astype(np.int64)
    K = layer.rir_length
    alpha = np.array([[backend.inverse_sabine(t, r)] * 6 for t, r in zip(rt60, room)])
    full = _sim(room, source, mic[:, None, :], layer.max_order, alpha, int(start.max()) + K,
                delay_filter_length=layer.delay_filter_length, sample_rate=layer.sample_rate, data_format=CF)
    full = full.cpu().numpy()[:, 0]
    h = _unit(np.stack([full[b, start[b]:start[b] + K] for b in range(len(start))]))
    T = x.shape[1]
    y = Convolve(mode='full', data_format=CL).call(x, torch.from_numpy(h).cuda()[:, :, None])
    return y[:, :T], h


def test_room_reverb_equals_its_composition_and_gradient():
    from kapre_b200.augmentation import RoomReverb
    layer = RoomReverb(16000, seed=7, data_format=CL)
    x = torch.from_numpy(np.random.default_rng(1).standard_normal((4, 16000, 2)).astype(np.float32)).cuda()
    x.requires_grad_(True)
    y = layer.call(x)
    with torch.no_grad():
        want, h = _composition(layer, layer.last_choice, x.detach())
    assert torch.equal(y.detach(), want)
    g = torch.from_numpy(np.random.default_rng(2).standard_normal(y.shape).astype(np.float32)).cuda()
    (gx,) = torch.autograd.grad(y, x, g)
    ga, T = g.double().cpu().numpy(), x.shape[1]
    gxa = gx.double().cpu().numpy()
    for b in range(4):
        for c in range(2):
            ref = np.convolve(ga[b, ::-1, c], h[b].astype(np.float64))[:T][::-1]
            assert np.max(np.abs(gxa[b, :, c] - ref)) <= 1e-4 * np.max(np.abs(ref)), (b, c)


def test_sequential_keeps_the_log_mel_fused_and_replays_under_capture():
    import kapre_b200
    from kapre_b200 import _native as N
    from kapre_b200.augmentation import BackgroundNoise, RoomReverb
    from kapre_b200.composed import Sequential
    from kapre_b200.signal import Speed
    rng = np.random.default_rng(3)
    noises = rng.standard_normal((4, 20000)).astype(np.float32)
    rr = RoomReverb(16000, seed=11, data_format=CL)
    speed, noise = Speed(1.1, data_format=CL), BackgroundNoise(noises, seed=2, data_format=CL)
    mel = kapre_b200.get_melspectrogram_layer(n_fft=1024, hop_length=256, sample_rate=16000, n_mels=64,
                                              return_decibel=True, input_data_format=CL, output_data_format=CL)
    model = Sequential([speed, rr, noise, *mel.layers])
    x = torch.from_numpy(rng.uniform(-1, 1, (8, 16000, 1)).astype(np.float32)).cuda()
    model.call(x)
    torch.cuda.synchronize()
    n0 = N.launch_count()
    model.call(x)
    n_model = N.launch_count() - n0
    counts = []
    y = x
    for layer in (speed, rr, noise, mel):
        n0 = N.launch_count()
        y = layer.call(y)
        counts.append(N.launch_count() - n0)
    assert counts[1] == 6                                   # RIR, unit norm, block spectra, kapre_convolve's three
    assert counts[3] <= 2 and n_model == sum(counts)
    cap = model.capture(x)
    choice, (idx, off, snr) = rr.last_choice, noise.last_choice       # the draws the graph holds
    x2 = torch.from_numpy(rng.uniform(-1, 1, (8, 16000, 1)).astype(np.float32)).cuda()
    out = cap(x2).clone()
    assert torch.equal(cap(x2).clone(), out)
    with torch.no_grad():
        y, _ = _composition(rr, choice, speed.call(x2))
        want = mel.call(noise.call(y, noise_index=idx, offset=off, snr=snr))
    assert torch.equal(out, want)


def test_invalid_arguments_raise_before_any_launch():
    from kapre_b200 import _native as N
    ok = dict(room=(5.0, 4.0, 3.0), source=(1.0, 1.0, 1.0), mic_array=[[2.0, 2.0, 2.0]], max_order=None,
              absorption=0.3, output_length=100)
    torch.cuda.synchronize()
    n0 = N.launch_count()
    for k, v in (('source', (0.0, 1.0, 1.0)), ('mic_array', [[1.0, 1.0, 1.0005]]), ('mic_array', [[6.0, 1.0, 1.0]]),
                 ('room', (5.0, -4.0, 3.0)), ('absorption', -0.1), ('delay_filter_length', 82),
                 ('delay_filter_length', 0), ('max_order', -1), ('output_length', 0),
                 ('room', (1.0, 1.0, 1.0))):
        args = dict(ok, **{k: v})
        if k == 'room' and v[0] == 1.0:
            args.update(source=(0.3, 0.3, 0.3), mic_array=[[0.6, 0.6, 0.6]], absorption=0.0, output_length=40000)
        with pytest.raises(ValueError):
            _sim(**args)
    assert N.launch_count() == n0


def test_register_budget():
    out = subprocess.run(['cuobjdump', '-res-usage', _LIB], capture_output=True, text=True, check=True).stdout
    m = re.search(r'Function _Z13kb_rir_kernel11KbRirParams:\s*\n\s*REG:(\d+) STACK:(\d+)[^\n]*LOCAL:(\d+)', out)
    assert m, 'kb_rir_kernel not found'
    reg, stack, local = (int(v) for v in m.groups())
    assert reg <= 128 and stack == 0 and local == 0, (reg, stack, local)
    m = re.search(r'Function _Z18kb_rir_norm_kernelPfxxxiii:\s*\n\s*REG:(\d+) STACK:(\d+)[^\n]*LOCAL:(\d+)', out)
    assert m and int(m.group(2)) == 0 and int(m.group(3)) == 0
