"""Filterbank inversion on the GPU: ``InverseFilterbank`` against the float64 restatement (fbinv_ref.py), bitwise frame
independence, one launch per call, graph capture, the no-gradient rule, argument checks, and the whole
waveform -> mel -> waveform chain of ``get_inverse_melspectrogram_layer`` against the same chain with torchaudio's
method (``relu(lstsq)``) in place of the NNLS step.

Tolerances: as in test_filterbank_inverse_emu.py, 10x the drift of a float32 twin of the loop from the float64 run,
with a floor of 1e-6 of each frame's largest bin.  The kernel rounds every operation explicitly, so the GPU runs the
same arithmetic as the emulated body; the margin covers the decibel conversion (``exp10`` on the device).
"""
import numpy as np
import pytest
import torch

import fbinv_ref as FR

pytestmark = pytest.mark.gpu
CL, CF = 'channels_last', 'channels_first'

BANKS = [('mel', 22050, 256, 32), ('mel', 16000, 400, 80), ('mel', 22050, 1024, 128), ('mel', 22050, 2048, 128),
         ('mel', 22050, 4096, 64), ('log', 22050, 1024, 84)]
BANK_IDS = ['%s%d_%d' % (k, n, m) for k, _, n, m in BANKS]


def _kwargs(kind, sr, n_fft, n):
    if kind == 'mel':
        return dict(sample_rate=sr, n_freq=n_fft // 2 + 1, n_mels=n)
    return dict(sample_rate=sr, n_freq=n_fft // 2 + 1, n_bins=n)


def _layer(bank, n_iter=100, fmt=CF, **kw):
    from kapre_b200.time_frequency import InverseFilterbank
    return InverseFilterbank(bank[0], _kwargs(*bank), n_iter=n_iter, data_format=fmt, **kw)


def _to_fmt(a, fmt):
    """(B, C, T, K) host array -> CUDA tensor in `fmt`."""
    t = torch.from_numpy(np.ascontiguousarray(a))
    return (t.permute(0, 2, 3, 1).contiguous() if fmt == CL else t.contiguous()).cuda()


def _canon(y, fmt):
    y = y.detach().cpu().double()
    return (y.permute(0, 3, 1, 2) if fmt == CL else y).numpy()


def _frame_err(got, want):
    return np.abs(got - want).max(-1) / np.maximum(np.abs(want).max(-1), 1e-300)


def _reference(fb, m, n_iter):
    """(float64 restatement, float32 twin's worst per-frame drift).  The plan's step and 1 / d are float32 roundings
    of the float64 values."""
    A = FR.matrix(fb)
    step = np.float32(FR.step_of(A))
    inv_d = FR.inv_d_of(A).astype(np.float32)
    mf = m.reshape(-1, m.shape[-1]).astype(np.float64)
    want = FR.fista(A, mf, n_iter, step=float(step), inv_d=inv_d.astype(np.float64))
    twin = FR.fista(A, mf, n_iter, step=step, inv_d=inv_d, dtype=np.float32)
    drift = float(_frame_err(twin.astype(np.float64), want).max())
    return want.reshape(m.shape[:-1] + (A.shape[1],)), drift


def _bound(drift):
    return max(1e-6, 10 * drift)


@pytest.mark.parametrize('bank', BANKS, ids=BANK_IDS)
@pytest.mark.parametrize('n_iter', [0, 1, 10, 100])
def test_parity_with_restatement(bank, n_iter):
    kind, sr, n_fft, _ = bank
    fb = FR.bank(*bank)
    m = FR.consistent_input(fb, sr, n_fft, 2, 2, 9 if n_fft >= 4096 else 45)
    want, drift = _reference(fb, m, n_iter)
    for fmt in (CF, CL):
        with torch.no_grad():
            got = _canon(_layer(bank, n_iter, fmt)(_to_fmt(m, fmt)), fmt)
        err = float(_frame_err(got, want).max())
        assert err <= _bound(drift), (fmt, err, drift)


def test_views_batch_positions_and_formats_give_identical_bits():
    """Each frame's output does not depend on its batch position, the batch size, the data format or the strides."""
    bank = BANKS[2]
    fb = FR.bank(*bank)
    m = FR.consistent_input(fb, 22050, 1024, 3, 2, 70)
    layer_cf, layer_cl = _layer(bank, 30, CF), _layer(bank, 30, CL)
    base = _canon(layer_cf(_to_fmt(m, CF)), CF)
    np.testing.assert_array_equal(_canon(layer_cl(_to_fmt(m, CL)), CL), base)
    # item 2 alone; item 1 placed first in a batch of 5 beside other items
    np.testing.assert_array_equal(_canon(layer_cf(_to_fmt(m[2:3], CF)), CF)[0], base[2])
    other = FR.consistent_input(fb, 22050, 1024, 4, 2, 70, seed=11)
    mixed = np.concatenate([m[1:2], other], axis=0)
    np.testing.assert_array_equal(_canon(layer_cl(_to_fmt(mixed, CL)), CL)[0], base[1])
    # a few frames cut out of the middle, and one frame
    np.testing.assert_array_equal(_canon(layer_cf(_to_fmt(m[:, :, 33:40], CF)), CF), base[:, :, 33:40])
    np.testing.assert_array_equal(_canon(layer_cf(_to_fmt(m[:, 1:, 64:65], CF)), CF), base[:, 1:, 64:65])
    # strided views: every other frame of a padded buffer and a channel slice, in both formats
    big = torch.full((3, 3, 140, 133), float('nan'), device='cuda')
    big[:, 1:, ::2, 2:130] = torch.from_numpy(m).cuda()
    view_cf = big[:, 1:, ::2, 2:130]
    np.testing.assert_array_equal(_canon(layer_cf(view_cf), CF), base)
    big_cl = big.permute(0, 2, 3, 1).contiguous()
    view_cl = big_cl[:, ::2, 2:130, 1:]
    assert not view_cl.is_contiguous()
    np.testing.assert_array_equal(_canon(layer_cl(view_cl), CL), base)


def test_one_launch_per_call_and_capture():
    from kapre_b200 import _native as N
    from kapre_b200.composed import Sequential
    bank = BANKS[3]
    fb = FR.bank(*bank)
    x = _to_fmt(FR.consistent_input(fb, 22050, 2048, 2, 1, 50), CL)
    layer = _layer(bank, 100, CL)
    want = layer(x)
    torch.cuda.synchronize()
    n0 = N.launch_count()
    got = layer(x)
    assert N.launch_count() - n0 == 1
    assert torch.equal(got, want)
    cap = Sequential([layer]).capture(x)
    out = cap(x)
    torch.cuda.synchronize()
    assert torch.equal(out, want)
    x2 = _to_fmt(FR.consistent_input(fb, 22050, 2048, 2, 1, 50, seed=5), CL)
    out2 = cap(x2)
    torch.cuda.synchronize()
    assert torch.equal(out2, layer(x2))


def test_gradients_are_refused():
    layer = _layer(BANKS[0], 5, CF)
    x = _to_fmt(FR.consistent_input(FR.bank(*BANKS[0]), 22050, 256, 1, 1, 8), CF).requires_grad_()
    with pytest.raises(RuntimeError, match='not differentiable'):
        layer(x)
    with torch.no_grad():
        y = layer(x)
    assert not y.requires_grad
    assert torch.equal(layer(x.detach()), y)


def test_empty_sizes():
    layer_cf, layer_cl = _layer(BANKS[0], 5, CF), _layer(BANKS[0], 5, CL)
    for shape in ((0, 1, 4, 32), (2, 0, 4, 32), (2, 1, 0, 32)):
        assert tuple(layer_cf(torch.zeros(shape, device='cuda')).shape) == shape[:3] + (129,)
    assert tuple(layer_cl(torch.zeros((2, 0, 32, 3), device='cuda')).shape) == (2, 0, 129, 3)


def test_argument_checks_and_unsupported_size():
    from kapre_b200 import _native as N
    from kapre_b200 import ops
    plan = ops.FilterbankInversePlan(FR.bank(*BANKS[0]))
    x = torch.ones((1, 1, 4, 32), device='cuda')
    with pytest.raises(ValueError, match='bands'):
        ops.invert_filterbank(torch.ones((1, 1, 4, 31), device='cuda'), plan, 5, False, 1.0, 1e-5, CF)
    with pytest.raises(N.KapreNativeError, match='n_iter'):
        ops.invert_filterbank(x, plan, -1, False, 1.0, 1e-5, CF)
    with pytest.raises(N.KapreNativeError, match='amin'):
        ops.invert_filterbank(x, plan, 5, True, 1.0, 0.0, CF)
    with pytest.raises(N.KapreNativeError, match='ref_value'):
        ops.invert_filterbank(x, plan, 5, True, float('nan'), 1e-5, CF)
    ops.invert_filterbank(x, plan, 5, False, 0.0, 0.0, CF)      # the dB settings are not read without from_decibel
    big = np.zeros((16385, 128), np.float32)
    big[np.arange(16385), np.arange(16385) % 128] = 1.0
    big_plan = ops.FilterbankInversePlan(big)
    with pytest.raises(N.KapreNativeError, match='does not fit'):
        ops.invert_filterbank(torch.ones((1, 1, 2, 128), device='cuda'), big_plan, 1, False, 1.0, 1e-5, CF)
    fb16k = FR.bank('mel', 44100, 16384, 64)
    m = FR.consistent_input(fb16k, 44100, 16384, 1, 1, 3)
    want, drift = _reference(fb16k, m, 4)
    got = _canon(ops.invert_filterbank(_to_fmt(m, CF), ops.FilterbankInversePlan(fb16k), 4, False, 1.0, 1e-5, CF), CF)
    assert float(_frame_err(got, want).max()) <= _bound(drift)


@pytest.mark.parametrize('ref,amin', [(1.0, 1e-5), (0.5, 1e-4)])
def test_decibel_input_round_trips_the_library_db(ref, amin):
    """The library's own dB (the fused get_melspectrogram_layer(return_decibel=True) launch) inverted with
    from_decibel gives the inversion of its magnitude mel, to float32 tolerance (no clamp binds on this signal)."""
    import kapre_b200
    kw = dict(n_fft=1024, hop_length=256, sample_rate=22050, n_mels=128, db_amin=amin, db_ref_value=ref,
              input_data_format=CF, output_data_format=CF)
    x = torch.from_numpy(np.stack([FR.signal(1, 22050, 22050, seed=b) for b in range(2)]).astype(np.float32)).cuda()
    mel = kapre_b200.get_melspectrogram_layer(**kw)(x)
    mel_db = kapre_b200.get_melspectrogram_layer(return_decibel=True, **kw)(x)
    floor = mel_db.flatten(1).max(1).values - 80.0
    assert bool((mel_db.flatten(1).min(1).values > floor).all())        # unclamped
    bank = ('mel', 22050, 1024, 128)
    want = _layer(bank, 20, CF)(torch.clamp(mel, min=amin))
    got = _layer(bank, 20, CF, from_decibel=True, db_ref_value=ref, db_amin=amin)(mel_db)
    err = float(_frame_err(got.cpu().double().numpy(), want.cpu().double().numpy()).max())
    assert err <= 2e-5, err


# ------------------------------------------------------------------------------ waveform -> mel -> waveform
def _relu_lstsq(fb):
    """torchaudio.transforms.InverseMelScale's method with this library's matrix: min-norm least squares, then relu,
    on a (B, C, T, n_bands) tensor."""
    pinv_t = torch.linalg.pinv(torch.from_numpy(FR.matrix(fb))).T.float().cuda()      # (n_bands, n_freq)
    return lambda m: torch.relu(torch.matmul(m, pinv_t))


@pytest.mark.parametrize('n_fft', [1024, 2048])
@pytest.mark.parametrize('db', [False, True])
def test_mel_round_trip_beats_relu_lstsq(n_fft, db):
    """waveform -> get_melspectrogram_layer -> get_inverse_melspectrogram_layer -> waveform -> mel again: closer to
    the original mel (relative Frobenius error) than the same chain with relu(lstsq) in place of InverseFilterbank,
    with the same GriffinLim settings and seed.  (At 16 kHz / n_fft 400 / 80 bands the two chains come out within
    0.2% of each other in a float64 run, so that shape is not held to the ordering.)"""
    import kapre_b200
    from kapre_b200 import composed
    sr, hop = 22050, n_fft // 4
    kw = dict(n_fft=n_fft, hop_length=hop, sample_rate=sr, n_mels=128, return_decibel=db)
    x = torch.from_numpy(np.stack([FR.signal(1, 2 * sr, sr, seed=b) for b in range(2)]).astype(np.float32)).cuda()
    fwd = kapre_b200.get_melspectrogram_layer(input_data_format=CF, output_data_format=CF, **kw)
    inv = composed.get_inverse_melspectrogram_layer(input_data_format=CF, output_data_format=CF, **kw)
    mel_fwd = kapre_b200.get_melspectrogram_layer(input_data_format=CF, output_data_format=CF, n_fft=n_fft,
                                                  hop_length=hop, sample_rate=sr, n_mels=128)
    m = mel_fwd(x)
    y = inv(fwd(x))
    ifb, gl = inv.layers
    lin = fwd(x)
    if db:
        lin = 10.0 ** (lin / 10.0) * max(1e-5, 1.0)
    y_ls = gl(_relu_lstsq(ifb.filterbank)(lin))
    assert y.shape == y_ls.shape == (2, 1, (m.shape[2] - 1) * hop + n_fft)
    err = float(torch.linalg.vector_norm(mel_fwd(y) - m) / torch.linalg.vector_norm(m))
    err_ls = float(torch.linalg.vector_norm(mel_fwd(y_ls) - m) / torch.linalg.vector_norm(m))
    assert err < err_ls, (err, err_ls)
