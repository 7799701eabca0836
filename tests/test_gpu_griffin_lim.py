"""Griffin-Lim on the GPU against the float64 restatement (gl_ref.py) over the oracle's transform pair, plus layout
invariance, seeds, launch counts, composition behind the fused magnitude launch and the no-gradient rule.

Tolerances (a float32 and a float64 run of the same loop on the CPU, n_fft 1024 / hop 256): on a 2 s two-channel signal
the waveform drifts by at most 2.1e-5 of max|y| through 8 iterations on a consistent spectrogram and 1.0e-5 on a random
one, and the spectral convergence of the two runs agrees to 1e-4 at 32 and 100 iterations, where the waveforms themselves
drift apart (Griffin-Lim is not contractive).  The GPU rounds differently from the CPU, so the bounds below carry a 10x
margin: 2e-4 of max|y| per element through 8 iterations, 1e-3 in spectral convergence beyond.

Some inputs amplify rounding far more.  Zero phase (init='ones') puts each frame's energy at the frame's first sample, where
the analysis window is zero, so the first STFT sees mostly rounding; a single frame has no overlap to average it out.  For
the signals here the float32 CPU run drifts by up to 3.4e-4 of max|y| at 8 iterations, and by 8e-3 for a single frame at 4.
So every ladder case also runs that float32 twin (gl_ref.kapre_pair32), and its bound is the larger of 2e-4 and 10x the
twin's drift."""
import functools

import numpy as np
import pytest
import torch

import gl_ref as GR
import oracle

pytestmark = pytest.mark.gpu
CL, CF = 'channels_last', 'channels_first'
MOMENTUM = 0.99


def _signal(B, C, L, seed=0):
    """A chirp per channel plus a little noise, (B, C, L) float32."""
    t = np.arange(L) / 22050.0
    rng = np.random.default_rng(seed)
    x = np.empty((B, C, L), np.float64)
    for b in range(B):
        for c in range(C):
            f0 = 150 + 400 * b + 1100 * c
            x[b, c] = 0.5 * np.sin(2 * np.pi * (f0 + 1200 * t) * t) + 0.05 * rng.standard_normal(L)
    return x.astype(np.float32)


def _spectrogram(kind, n_fft, hop, win, B, C, L, seed=0):
    """(B, C, T, F) float32: |STFT(x)| of a chirp-plus-noise signal ('consistent'), or positive values over three
    decades that no signal has ('random')."""
    T = oracle.num_frames(L, win, hop, False)
    if kind == 'consistent':
        w = oracle.get_window(None, win)
        return np.abs(oracle.stft_frames(_signal(B, C, L, seed), n_fft, win, hop, w, False)).astype(np.float32)
    rng = np.random.default_rng(seed + 100)
    return (10.0 ** rng.uniform(-1.5, 1.5, size=(B, C, T, n_fft // 2 + 1))).astype(np.float32)


def _to_fmt(S, fmt):
    """(B, C, T, F) host array -> CUDA tensor in `fmt`."""
    t = torch.from_numpy(S)
    return (t.permute(0, 2, 3, 1).contiguous() if fmt == CL else t.contiguous()).cuda()


def _wave_canon(y, fmt):
    y = y.detach().cpu().double()
    return y.permute(0, 2, 1) if fmt == CL else y


@functools.lru_cache(maxsize=None)
def _reference(kind, n_fft, hop, B, C, L, init, n_iter, seed=0):
    """(S, float64 waveform, its spectral convergence, the float32 twin's drift from it relative to max|y|)."""
    S = _spectrogram(kind, n_fft, hop, n_fft, B, C, L)
    stft_fn, istft_fn = GR.kapre_pair(n_fft, n_fft, hop)
    A0 = GR.random_phase(seed, *S.shape) if init == 'random' else 1.0
    Sd = torch.from_numpy(S).double()
    y = GR.griffin_lim(Sd, stft_fn, istft_fn, n_iter, MOMENTUM, A0)
    y32 = GR.griffin_lim(torch.from_numpy(S), *GR.kapre_pair32(n_fft, n_fft, hop), n_iter, MOMENTUM, A0)
    drift = float((y32.double() - y).abs().max() / y.abs().max())
    return S, y, GR.spectral_convergence(y, Sd, stft_fn), drift


def _bound(drift):
    return max(2e-4, 10 * drift)


def _layer(n_fft, hop, n_iter, init, fmt_in=CL, fmt_out=CL, seed=0, momentum=MOMENTUM):
    from kapre_b200.time_frequency import GriffinLim
    return GriffinLim(n_fft=n_fft, hop_length=hop, n_iter=n_iter, momentum=momentum, init=init, seed=seed,
                      input_data_format=fmt_in, output_data_format=fmt_out)


def _assert_wave_close(got, want, rel):
    assert tuple(got.shape) == tuple(want.shape), (tuple(got.shape), tuple(want.shape))
    scale = float(want.abs().max())
    err = float((got - want).abs().max())
    assert err <= rel * scale, (err, scale, err / scale)


# (n_fft, hop, B, C, L): odd lengths; the last is the K1d STFT / direct inverse size on a short signal
_SIZES = [(1024, 256, 2, 2, 22050 + 77), (512, 128, 1, 1, 8191), (400, 160, 1, 2, 4001)]


@pytest.mark.parametrize('size', _SIZES, ids=['n1024', 'n512', 'n400'])
@pytest.mark.parametrize('kind', ['consistent', 'random'])
@pytest.mark.parametrize('init', ['ones', 'random'])
@pytest.mark.parametrize('n_iter', [0, 1, 2, 4, 8])
def test_iteration_ladder(size, kind, init, n_iter):
    n_fft, hop, B, C, L = size
    if n_fft == 400 and n_iter > 2:
        pytest.skip('the direct inverse is O(N^2): the short ladder covers it')
    S, want, _, drift = _reference(kind, n_fft, hop, B, C, L, init, n_iter)
    for fmt in (CL, CF):
        y = _layer(n_fft, hop, n_iter, init, fmt, fmt)(_to_fmt(S, fmt))
        _assert_wave_close(_wave_canon(y, fmt), want, _bound(drift))


@pytest.mark.parametrize('init', ['ones', 'random'])
def test_single_frame_and_empty_batch(init):
    n_fft, hop = 1024, 256
    S, want, _, drift = _reference('consistent', n_fft, hop, 1, 2, n_fft, init, 4)
    assert S.shape[2] == 1
    y = _layer(n_fft, hop, 4, init, CF, CF)(_to_fmt(S, CF))
    _assert_wave_close(_wave_canon(y, CF), want, _bound(drift))
    for fmt in (CL, CF):
        empty = torch.zeros((0, 5, 513, 1) if fmt == CL else (0, 1, 5, 513), device='cuda')
        out = _layer(n_fft, hop, 4, init, fmt, fmt)(empty)
        assert tuple(out.shape) == ((0, 4 * 256 + 1024, 1) if fmt == CL else (0, 1, 4 * 256 + 1024))


@pytest.mark.parametrize('kind', ['consistent', 'random'])
def test_long_runs_spectral_convergence(kind):
    n_fft, hop, B, C, L = 1024, 256, 1, 2, 2 * 22050
    init = 'ones' if kind == 'consistent' else 'random'
    stft_fn, _ = GR.kapre_pair(n_fft, n_fft, hop)
    sc = {}
    for n_iter in (8, 32, 100):
        S, _, sc_ref, _ = _reference(kind, n_fft, hop, B, C, L, init, n_iter)
        y = _layer(n_fft, hop, n_iter, init, CF, CF)(_to_fmt(S, CF))
        sc[n_iter] = GR.spectral_convergence(_wave_canon(y, CF), torch.from_numpy(S).double(), stft_fn)
        if n_iter > 8:
            assert abs(sc[n_iter] - sc_ref) <= 1e-3, (n_iter, sc[n_iter], sc_ref)
    if kind == 'consistent':
        assert sc[100] < sc[32] < sc[8], sc


def test_layout_invariance():
    """channels_last / channels_first in and out, and a strided view of S: the same bits."""
    n_fft, hop = 1024, 256
    S = _spectrogram('consistent', n_fft, hop, n_fft, 2, 2, 22050)
    outs = []
    for fi in (CL, CF):
        for fo in (CL, CF):
            y = _layer(n_fft, hop, 6, 'random', fi, fo, seed=3)(_to_fmt(S, fi))
            outs.append(_wave_canon(y, fo))
    big = torch.zeros((2, 2, S.shape[2] * 2, 520), device='cuda')
    big[:, :, ::2, 3:516] = torch.from_numpy(S).cuda()
    view = big[:, :, ::2, 3:516]
    assert not view.is_contiguous()
    outs.append(_wave_canon(_layer(n_fft, hop, 6, 'random', CF, CF, seed=3)(view), CF))
    for o in outs[1:]:
        assert torch.equal(o, outs[0])


def test_seeds():
    n_fft, hop = 512, 128
    S = _to_fmt(_spectrogram('random', n_fft, hop, n_fft, 1, 1, 8192), CF)
    a = _layer(n_fft, hop, 3, 'random', CF, CF, seed=11)(S)
    b = _layer(n_fft, hop, 3, 'random', CF, CF, seed=11)(S)
    c = _layer(n_fft, hop, 3, 'random', CF, CF, seed=12)(S)
    assert torch.equal(a, b) and not torch.equal(a, c)
    top = _layer(n_fft, hop, 3, 'random', CF, CF, seed=2 ** 64 - 1)(S)
    assert torch.isfinite(top).all() and not torch.equal(top, a)
    free = _layer(n_fft, hop, 3, 'random', CF, CF, seed=None)
    assert not torch.equal(free(S), free(S))


@pytest.mark.parametrize('n_iter', [0, 1, 5])
def test_launch_count(n_iter):
    from kapre_b200 import _native as N
    layer = _layer(1024, 256, n_iter, 'random', CL, CL)
    S = _to_fmt(_spectrogram('random', 1024, 256, 1024, 2, 1, 22050), CL)
    layer(S)
    torch.cuda.synchronize()
    n0 = N.launch_count()
    layer(S)
    assert N.launch_count() - n0 == 3 * n_iter + 2


def _mag(fmt=CL):
    import kapre_b200
    return kapre_b200.composed.get_stft_magnitude_layer(n_fft=1024, hop_length=256, input_data_format=fmt,
                                                        output_data_format=fmt)


def test_sequential_composition():
    from kapre_b200 import _native as N
    from kapre_b200.composed import Sequential
    mag = _mag()
    gl = _layer(1024, 256, 4, 'ones', CL, CL)
    stack = Sequential([*mag.layers, gl])
    x = torch.from_numpy(_signal(3, 1, 22050 + 5).transpose(0, 2, 1).copy()).cuda()
    want = gl(mag(x))
    torch.cuda.synchronize()
    n0 = N.launch_count()
    got = stack(x)
    assert N.launch_count() - n0 == 1 + 3 * 4 + 2        # the fused magnitude launch, then the loop
    assert torch.equal(got, want)
    host = stack.predict(x.cpu().numpy(), batch_size=x.shape[0])
    assert isinstance(host, np.ndarray) and np.array_equal(host, want.cpu().numpy())
    cap = stack.capture(x)
    out = cap(x)
    torch.cuda.synchronize()
    assert torch.equal(out, want)
    x2 = torch.from_numpy(_signal(3, 1, 22050 + 5, seed=9).transpose(0, 2, 1).copy()).cuda()
    out2 = cap(x2)
    torch.cuda.synchronize()
    assert torch.equal(out2, stack(x2))


def test_gradients_are_refused():
    layer = _layer(512, 128, 2, 'ones', CF, CF)
    S = _to_fmt(_spectrogram('random', 512, 128, 512, 1, 1, 4096), CF).requires_grad_()
    with pytest.raises(RuntimeError, match='not differentiable'):
        layer(S)
    with torch.no_grad():
        y = layer(S)
    assert not y.requires_grad
    assert torch.equal(layer(S.detach()), y)


def test_call_time_validation():
    from kapre_b200 import _native as N
    from kapre_b200 import ops
    from kapre_b200.time_frequency import GriffinLim
    with pytest.raises(ValueError):
        _layer(1024, 256, 2, 'ones', CF, CF)(torch.ones((1, 1, 4, 257), device='cuda'))
    S = torch.ones((1, 1, 4, 513), device='cuda')
    a = GriffinLim(n_fft=1024, hop_length=256).plans
    b = GriffinLim(n_fft=1024, hop_length=128).plans
    with pytest.raises(N.KapreNativeError, match='disagree'):
        ops.griffin_lim(S, a[0], b[1], 2, 0.5, N.GL_INIT_ONES, 0, CF, CF)
    with pytest.raises(N.KapreNativeError, match='momentum'):
        ops.griffin_lim(S, a[0], a[1], 2, 1.0, N.GL_INIT_ONES, 0, CF, CF)
    with pytest.raises(N.KapreNativeError, match='init'):
        ops.griffin_lim(S, a[0], a[1], 2, 0.5, 7, 0, CF, CF)
    with pytest.raises(N.KapreNativeError, match='n_iter'):
        ops.griffin_lim(S, a[0], a[1], -1, 0.5, N.GL_INIT_ONES, 0, CF, CF)
    assert N.lib().kapre_griffin_lim_workspace_bytes(a[0].handle(), 2, 3, 5) == \
        2 * ((2 * 3 * 5 * 513 * 8 + 255) // 256 * 256) + 2 * 3 * (4 * 256 + 1024) * 4
