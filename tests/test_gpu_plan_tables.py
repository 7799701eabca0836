"""GPU tier: plan tables are freed with their plan, and a plan is refused on any device but its own.

Each plan's constant tables live in one device block owned by the plan (``KbTables`` in ``csrc/kapre_b200.cu``).
Destroying every kind of plan must give back all the device memory its tables took, and a creation that fails on a
bad table must leave nothing behind.  Every entry point that takes a plan compares the plan's device with the current
one and returns ``KAPRE_E_INVALID`` when they differ, rather than launching kernels that read another device's
tables; that needs two GPUs to observe."""
import ctypes

import numpy as np
import pytest
import torch

from kapre_b200 import _native as N
from kapre_b200 import backend, ops, signal

pytestmark = pytest.mark.gpu

GRANULE = 2 << 20      # the device memory allocator's page
MAX_HELD = 1 << 16
ATTEMPTS = 4800
FMT = 'channels_last'


def _mel(n_freq=513, n_mels=128):
    return backend.filterbank_mel(22050, n_freq, n_mels)


def _window(n, name=None):
    return backend.get_window_fn(name)(n)


def _chroma_stft_plan():
    """One table per tuning-grid edge and the tuning estimate's edges (a fresh plan, not the shared cached one)."""
    p = signal._stft_chroma_plans(22050, 2048, 512, None, 12, None, 5.0, 2.0, True)[1]
    return ops.ChromaPlan(p.tables, tuning=p.tuning)


def _chroma_cqt_plan():
    """One table and the CENS smoothing taps."""
    p = signal._cqt_chroma_plans(22050, 512, None, 0.0, 12, 7, 36, True, 41)[1]
    return ops.ChromaPlan(p.tables, smooth=p.smooth)


# Fresh plan objects of every kind, between them building every table a plan can hold.
PLANS = {
    'stft(1024, hann)': lambda: ops.StftPlan(1024, 1024, 256, _window(1024)),    # with the tensor-core tables
    'stft(1024, hamming)': lambda: ops.StftPlan(1024, 1024, 256, _window(1024, 'hamming_window')),
    'stft(400)': lambda: ops.StftPlan(400, 400, 160, _window(400)),               # generic tables only
    'istft(1024)': lambda: ops.IstftPlan(1024, 1024, 256, _window(1024)),
    'istft(400)': lambda: ops.IstftPlan(400, 400, 160, _window(400)),
    'filterbank(513, 128)': lambda: ops.Filterbank(_mel()),
    'filterbank(201, 40)': lambda: ops.Filterbank(_mel(201, 40)),
    'fb_inverse': lambda: ops.FilterbankInversePlan(_mel()),
    'resample(3, 2)': lambda: ops.ResamplePlan(3, 2, signal.resample_filter(3, 2)),
    'sinc': ops.SincPlan,
    'convolve(256)': lambda: ops.ConvolvePlan(256),
    'kaldi(fbank)': lambda: ops.KaldiPlan('fbank', ops.kaldi_options('fbank')),
    'kaldi(mfcc)': lambda: ops.KaldiPlan('mfcc', ops.kaldi_options('mfcc')),
    'kaldi(spectrogram)': lambda: ops.KaldiPlan('spectrogram', ops.kaldi_options('spectrogram')),
    'cqt(84)': lambda: ops.CqtPlan(22050, 512, None, 84),
    'yin': lambda: ops.PitchPlan(22050, 65.0, 2093.0),
    'pyin': lambda: ops.PitchPlan(22050, 65.0, 2093.0, pyin={}),
    'chroma(stft)': _chroma_stft_plan,
    'chroma(cqt)': _chroma_cqt_plan,
}


def _free_bytes():
    torch.cuda.synchronize()
    return torch.cuda.mem_get_info()[0]


@pytest.mark.parametrize('kind', sorted(PLANS))
def test_tables_are_freed_with_the_plan(kind):
    torch.cuda.set_device(0)
    lib = N.lib()
    plan = PLANS[kind]()
    destroy = getattr(lib, plan._destroy)

    def make():
        h = ctypes.c_void_p()
        N.check(plan._create(lib, ctypes.byref(h)))
        if isinstance(plan, ops.ResamplePlan):
            # an empty backward call makes the adjoint plan, which the plan owns and destroys
            empty = N.WaveDesc(0, 1, 0, 0, 0, 1)
            N.check(lib.kapre_resample_backward(h, None, ctypes.byref(empty), None, ctypes.byref(empty), None))
        return h

    def hold_and_release(n):
        """Device bytes that n plans held at once took, counted from `start`."""
        held = [make() for _ in range(n)]
        used = start - _free_bytes()
        for h in held:
            destroy(h)
        return used

    destroy(make())     # first use: module and allocator set-up that stays
    start = _free_bytes()
    # Hold enough plans at once that their tables fill several allocator pages, however small one plan's tables are:
    # a destroy that missed them would then leave pages behind that the next plans cannot reuse.
    n = 8
    used = hold_and_release(n)
    while kind != 'yin' and used < 4 * GRANULE and n < MAX_HELD:    # a YIN plan has no device tables
        n *= 4
        used = hold_and_release(n)
    assert kind == 'yin' or used >= 4 * GRANULE, '%d plans take only %d bytes of device memory' % (n, used)
    first = start - _free_bytes()
    hold_and_release(n)
    lost = start - _free_bytes()
    assert lost - first <= GRANULE, '%d plans made after %d were destroyed lost %d more bytes' % (n, n, lost - first)
    assert lost <= GRANULE, '%d bytes of device memory not given back after destroying %d plans' % (lost, n)


def test_non_finite_pitch_table_is_refused_without_a_leak():
    torch.cuda.set_device(0)
    lib = N.lib()
    plan = ops.PitchPlan(22050, 65.0, 2093.0, pyin={})
    tables = dict(plan._tables)
    last = N.PitchTables._fields_[-1][0]      # the last table the plan converts and checks
    tables[last] = tables[last].copy()
    tables[last][-1] = np.nan
    tab = N.PitchTables(*[tables[name].ctypes.data_as(ctypes.c_void_p) for name, _ in N.PitchTables._fields_])

    def attempt():
        h = ctypes.c_void_p()
        rc = lib.kapre_pitch_plan_create(ctypes.byref(plan.cfg), ctypes.byref(tab), ctypes.byref(h))
        assert rc == -1 and h.value is None
        assert lib.kapre_last_error().decode() == 'pitch: non-finite table entry'

    attempt()
    start = _free_bytes()
    # the valid tables before the bad one take a few KB: enough attempts that leaking them would fill several pages
    for _ in range(ATTEMPTS):
        attempt()
    lost = start - _free_bytes()
    assert lost <= GRANULE, '%d bytes of device memory not given back after %d failed creations' % (lost, ATTEMPTS)


# ---- plans of one device used on another --------------------------------------------------------------------------
def _spec(d, T, K, dtype=torch.float32):
    return torch.rand((1, T, K, 1), device=d).to(dtype)


def _wave(d, L):
    return torch.rand((1, L, 1), device=d) - 0.5


def _blocks(d):
    """The spectrum of a filter of one 256-sample block."""
    return torch.rand((1, 1, 1, 257), device=d).to(torch.complex64)


# name: call(P, d), where P(plan) makes the plan answer on the current device and d is the data's device.  Every
# entry point of the C ABI that takes a plan is reached by one of them.
ENTRIES = {
    'stft_forward': lambda P, d: ops.stft_forward(_wave(d, 4096), P(PLANS['stft(1024, hann)']()), FMT, FMT, 0, 0),
    'istft': lambda P, d: ops.istft(_spec(d, 8, 513, torch.complex64), P(PLANS['istft(1024)']()), FMT, FMT),
    'apply_filterbank': lambda P, d: ops.apply_filterbank(_spec(d, 8, 513), P(PLANS['filterbank(513, 128)']()), FMT),
    'stft_backward': lambda P, d: ops.stft_backward(_spec(d, 13, 513, torch.complex64),
                                                    P(PLANS['stft(1024, hann)']()), FMT, FMT, 0, 0, 4096),
    'istft_backward': lambda P, d: ops.istft_backward(_wave(d, 7 * 256 + 1024), P(PLANS['istft(1024)']()), FMT, FMT,
                                                      8),
    'resample': lambda P, d: ops.resample(_wave(d, 3000), P(PLANS['resample(3, 2)']()), FMT),
    'resample_backward': lambda P, d: ops.resample_backward(_wave(d, 4500), P(PLANS['resample(3, 2)']()), FMT, 3000),
    'sinc_resample': lambda P, d: ops.sinc_resample(_wave(d, 3000), 1.3, 3900),
    'sinc_resample_backward': lambda P, d: ops.sinc_resample_backward(_wave(d, 3900), 1.3, 0.0, FMT, 3000),
    'convolve_ir_spectrum': lambda P, d: ops.convolve_ir_spectrum(_wave(d, 200), P(PLANS['convolve(256)']()), FMT),
    'convolve_ir_spectrum_backward': lambda P, d: ops.convolve_ir_spectrum_backward(
        _blocks(d), P(PLANS['convolve(256)']()), 200),
    'convolve': lambda P, d: ops.convolve_full(_wave(d, 3000), _blocks(d), P(PLANS['convolve(256)']()), FMT),
    'convolve_backward': lambda P, d: ops.convolve_backward(_wave(d, 13 * 256), _blocks(d), None,
                                                            P(PLANS['convolve(256)']()), FMT, 3000, True, False),
    'griffin_lim': lambda P, d: ops.griffin_lim(_spec(d, 8, 513), P(PLANS['stft(1024, hann)']()),
                                                P(PLANS['istft(1024)']()), 2, 0.99, N.GL_INIT_ONES, 0, FMT, FMT),
    'invert_filterbank': lambda P, d: ops.invert_filterbank(_spec(d, 8, 128), P(PLANS['fb_inverse']()), 2, False, 1.0,
                                                            1e-5, FMT),
    'kaldi_features': lambda P, d: ops.kaldi_forward(_wave(d, 16000), P(PLANS['kaldi(mfcc)']()), None, None, FMT, 0.0,
                                                     0),
    'kaldi_features_backward': lambda P, d: ops.kaldi_backward(_spec(d, 98, 13), _wave(d, 16000),
                                                               P(PLANS['kaldi(mfcc)']()), None, None, FMT, 0.0, 0),
    'cqt': lambda P, d: ops.cqt_forward(_wave(d, 22050), P(PLANS['cqt(84)']()), FMT, FMT, False),
    'cqt_backward': lambda P, d: ops.cqt_backward(_spec(d, 44, 84, torch.complex64), _wave(d, 22050), None,
                                                  P(PLANS['cqt(84)']()), FMT, FMT, False),
    'yin': lambda P, d: ops.yin(_wave(d, 22050), P(PLANS['yin']())),
    'pyin': lambda P, d: ops.pyin(_wave(d, 22050), P(PLANS['pyin']())),
    'chroma': lambda P, d: ops.chroma_forward(_spec(d, 8, 1025), P(_chroma_stft_plan()),
                                              N.ChromaCfg(N.CHROMA_IN_LINEAR, N.CHROMA_NORM_INF, 0, 0.0), FMT),
    'chroma_backward': lambda P, d: ops.chroma_backward(_spec(d, 8, 12), _spec(d, 8, 1025), P(_chroma_stft_plan()),
                                                        N.ChromaCfg(N.CHROMA_IN_LINEAR, N.CHROMA_NORM_INF, 0, 0.0),
                                                        FMT),
    'chroma_cens': lambda P, d: ops.chroma_cens(_spec(d, 8, 252), P(_chroma_cqt_plan()), N.CHROMA_IN_LINEAR),
    'chroma_tuning': lambda P, d: ops.chroma_tuning(_spec(d, 8, 1025), P(_chroma_stft_plan()), N.CHROMA_IN_SQUARE),
}


def _made_on_device_0(plan):
    """The plan, answering on every device with its handle from cuda:0."""
    with torch.cuda.device(0):
        plan.handle()
    plan._per_device[1] = plan._per_device[0]
    return plan


@pytest.mark.parametrize('entry', sorted(ENTRIES))
def test_plan_of_another_device_is_refused(entry, monkeypatch):
    if torch.cuda.device_count() < 2:
        pytest.skip('needs two GPUs')
    # sinc_resample takes the module's one interpolation plan
    monkeypatch.setattr(ops, '_sinc_plan', _made_on_device_0(ops.SincPlan()))
    d = torch.device('cuda', 1)
    with torch.cuda.device(d):
        with pytest.raises(N.KapreNativeError, match=r'error -1: plan was created on device 0 but device 1 is current'):
            ENTRIES[entry](_made_on_device_0, d)
        torch.cuda.synchronize()
