"""Launches and timed launches per call, pinned op by op.

``kapre_launch_count()`` counts every kernel launch of the library; the profiler (``profile_enable`` /
``profile_read``, the kernel time ``bench.py`` reports) brackets only the launches marked as timed.  Both are policies
of the one launch helper in ``csrc/kapre_b200.cu``, so this table keeps them from drifting: each row is one call and
the (launches, timed launches) it must make.  Timed are the transform kernels (fused STFT, mixed-radix, inverse STFT,
resample, PCEN, time stretch); the decibel clamp, the direct DFT, the stand-alone filterbank, the element-wise and
gradient kernels, Griffin-Lim's own passes and the filterbank inversion are not."""
import pytest
import torch

pytestmark = pytest.mark.gpu
CL = 'channels_last'


def _wave(B, L, seed=0):
    g = torch.Generator().manual_seed(seed)
    return (torch.rand((B, L, 1), generator=g) * 2 - 1).cuda()


def _positive(shape, seed=0):
    g = torch.Generator().manual_seed(seed)
    return (10.0 ** (torch.rand(shape, generator=g) * 4 - 2)).cuda()


def _complex(shape, seed=0):
    g = torch.Generator().manual_seed(seed)
    return torch.complex(torch.randn(shape, generator=g), torch.randn(shape, generator=g)).cuda()


def _logmel_db():
    import kapre_b200 as K
    layer = K.get_melspectrogram_layer(n_fft=512, hop_length=256, sample_rate=16000, n_mels=64, return_decibel=True,
                                       input_data_format=CL, output_data_format=CL)
    x = _wave(4, 16000)
    return lambda: layer(x), None


def _stft(n_fft, info):
    def make():
        from kapre_b200.time_frequency import STFT
        layer = STFT(n_fft=n_fft, hop_length=160, input_data_format=CL, output_data_format=CL)
        x = _wave(2, 16000)
        return lambda: layer(x), info
    return make


def _istft():
    from kapre_b200.time_frequency import InverseSTFT
    layer = InverseSTFT(n_fft=512, hop_length=128, input_data_format=CL, output_data_format=CL)
    X = _complex((2, 60, 257, 1))
    return lambda: layer(X), 'ISTFT'


def _apply_filterbank():
    from kapre_b200.time_frequency import ApplyFilterbank
    layer = ApplyFilterbank('mel', dict(sample_rate=16000, n_freq=257, n_mels=64), data_format=CL)
    S = _positive((2, 60, 257, 1))
    return lambda: layer(S), None


def _db():
    from kapre_b200 import ops
    S = _positive((3, 60, 64, 1))
    return lambda: ops.magnitude_to_decibel(S), None


def _db_backward():
    from kapre_b200 import ops
    S = _positive((3, 60, 64, 1))
    G = _positive((3, 60, 64, 1), seed=1)
    return lambda: ops.magnitude_to_decibel_backward(S, G), None


def _resample(backward):
    def make():
        from kapre_b200 import ops
        from kapre_b200.signal import Resample
        layer = Resample(16000, 22050, data_format=CL)
        x = _wave(2, 16000)
        if backward:
            g = _wave(2, layer.plan.output_length(16000), seed=1)
            return lambda: ops.resample_backward(g, layer.plan, CL, 16000), None
        return lambda: layer(x), None
    return make


def _pcen(shape, chunked):
    def make():
        from kapre_b200 import ops
        from kapre_b200.time_frequency import PCEN
        layer = PCEN(sample_rate=22050, hop_length=256, data_format=CL)
        E = _positive(shape)
        B, T, F, C = shape
        assert (ops._pcen_workspace(B, C, T, F, E.device)[0] > 1) == chunked
        return lambda: layer(E), None
    return make


def _time_stretch(backward):
    def make():
        from kapre_b200 import ops
        from kapre_b200.augmentation import TimeStretch
        shape = (1, 427, 513, 1)            # 513 columns: the chunked path, a state pass and an output pass
        X = _complex(shape)
        assert ops._time_stretch_workspace(1, 1, 427, 513, 0.8, X.device)[0] > 1
        layer = TimeStretch(0.8, data_format=CL)
        if backward:
            Y = layer(X)
            G = _complex(tuple(Y.shape), seed=1)
            return lambda: ops.time_stretch_backward(X, Y, G, 0.8, CL), None
        return lambda: layer(X), None
    return make


def _griffin_lim(n_iter):
    def make():
        from kapre_b200.time_frequency import GriffinLim
        layer = GriffinLim(n_fft=512, hop_length=128, n_iter=n_iter, input_data_format=CL, output_data_format=CL)
        S = _positive((2, 40, 257, 1))
        return lambda: layer(S), None
    return make


def _invert_filterbank():
    from kapre_b200.time_frequency import InverseFilterbank
    layer = InverseFilterbank('mel', dict(sample_rate=16000, n_freq=257, n_mels=64), n_iter=10, data_format=CL)
    M = _positive((2, 40, 64, 1))
    return lambda: layer(M), None


# (id, make, launches, timed launches); make() -> (call, prefix the launch info must start with, or None)
CASES = [
    ('logmel_db', _logmel_db, 2, 1),                                  # fused kernel (timed) + clamp
    ('stft_n_fft400', _stft(400, 'MR '), 1, 1),                       # mixed-radix kernel
    ('stft_prime_n_fft', _stft(401, 'DFT '), 1, 0),                   # direct DFT
    ('istft', _istft, 1, 1),
    ('apply_filterbank', _apply_filterbank, 1, 0),
    ('magnitude_to_decibel', _db, 2, 0),                              # dB pass + clamp
    ('magnitude_to_decibel_backward', _db_backward, 3, 0),
    ('resample', _resample(False), 1, 1),
    ('resample_backward', _resample(True), 1, 1),
    ('pcen_unchunked', _pcen((256, 427, 128, 1), False), 1, 1),
    ('pcen_chunked', _pcen((1, 4000, 128, 1), True), 2, 2),          # state pass + output pass
    ('time_stretch', _time_stretch(False), 2, 2),
    ('time_stretch_backward', _time_stretch(True), 2, 2),
    ('griffin_lim_0', _griffin_lim(0), 2, 1),                         # 3n + 2 launches, 2n + 1 timed
    ('griffin_lim_3', _griffin_lim(3), 11, 7),
    ('invert_filterbank', _invert_filterbank, 1, 0),
]


@pytest.mark.parametrize('make,launches,timed', [c[1:] for c in CASES], ids=[c[0] for c in CASES])
def test_launches_and_timed_launches_per_call(make, launches, timed):
    from kapre_b200 import _native as N
    with torch.no_grad():
        call, info = make()
        call()                                  # plans, workspaces and adjoints are made on first use
        torch.cuda.synchronize()
        N.profile_read()                        # drop anything recorded before
        N.profile_enable(True, every=1)
        try:
            n0 = N.launch_count()
            call()
            torch.cuda.synchronize()
            n1 = N.launch_count()
            _, n_timed = N.profile_read()
        finally:
            N.profile_enable(False)
    assert (n1 - n0, n_timed) == (launches, timed)
    if info is not None:
        assert N.last_launch_info().startswith(info), N.last_launch_info()
