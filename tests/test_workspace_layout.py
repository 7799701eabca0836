"""The scratch workspaces of libkapre_b200.

Each operation that takes a workspace describes its regions once, in a layout function built on ``KbLayout`` in
``csrc/kapre_b200.cu``; its ``*_workspace_bytes`` function and the operation both call it.  These tests hold the sizes
to the values the library returned before that layout builder existed (callers allocate exactly these), check that a
size beyond int64 is an error rather than a wrapped value, and check that no hand-written 256-byte rounding is left
outside the builder for a new workspace to copy."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, 'kapre_b200', 'csrc', 'kapre_b200.cu')
LIB = os.path.join(ROOT, 'kapre_b200', '_lib', 'libkapre_b200.so')


def _lib():
    if not os.path.exists(LIB):
        pytest.skip('needs the built library')
    from kapre_b200 import _native as N
    return N.lib()


def _code():
    """The source with comments and string literals blanked out."""
    text = open(SRC).read()
    pat = re.compile(r'//[^\n]*|/\*.*?\*/|"(?:\\.|[^"\\\n])*"', re.S)
    return pat.sub(lambda m: ' ' * len(m.group(0)), text)


def test_no_rounding_outside_the_layout_builder():
    code = outside = _code()
    m = re.search(r'\bstruct\s+KbLayout\s*\{', code)
    if m:   # blank the builder's body out, keeping offsets
        depth = 0
        for end in range(code.index('{', m.start()), len(code)):
            depth += {'{': 1, '}': -1}.get(code[end], 0)
            if depth == 0:
                break
        outside = code[:m.start()] + re.sub(r'[^\n]', ' ', code[m.start():end + 1]) + code[end + 1:]
    for idiom in (r'255\s*\)\s*/\s*256\s*\*\s*256', r'&\s*~\s*\(\s*int64_t\s*\)\s*255', r'&\s*~\s*\(\s*size_t\s*\)\s*255',
                  r'/\s*256\s*\*\s*64\b'):
        hits = [outside.count('\n', 0, h.start()) + 1 for h in re.finditer(idiom, outside)]
        assert not hits, 'workspace rounding %r written out by hand (lines %s); use KbLayout' % (idiom, hits)


# Sizes of the workspaces that need no plan, as the library returned them before KbLayout: zero sizes, and odd
# sizes whose regions are not multiples of 256 bytes.
PLAN_FREE = {
    'lfilter': {(0, 1, 100, 2): 0, (1, 1, 0, 2): 3072, (1, 1, 1, 1): 3584, (2, 3, 1000, 2): 22016,
                (3, 5, 4097, 8): 78848, (7, 1, 123457, 3): 474112, (1, 2, 65536, 4): 75008},
    'add_noise': {(0, 2, 100): 0, (2, 2, 0): 0, (1, 1, 1): 256, (3, 7, 4097): 768, (5, 3, 100001): 6144,
                  (256, 1, 80000): 81920},
    'hpss': {(0, 1, 1, 1): 0, (1, 1, 0, 513): 0, (1, 1, 1, 1): 16, (2, 3, 17, 513): 837216,
             (5, 1, 431, 1025): 35342000},
    'onset_strength': {(0, 1, 1, 1): 0, (1, 1, 0, 513): 0, (1, 1, 1, 1): 8, (2, 3, 17, 513): 418608,
                       (5, 1, 431, 1025): 17671000},
    'tempo': {(0, 1, 10, 384): 0, (1, 1, 0, 384): 0, (1, 1, 1, 2): 16, (2, 3, 431, 384): 129024,
              (3, 1, 1001, 7): 2688},
    'beat_track': {(0, 1, 10): 0, (1, 1, 0): 0, (1, 1, 1): 24, (2, 3, 431): 62064, (5, 2, 10007): 2401680},
}
# (workspace bytes, stats bytes) of kapre_loudness_workspace_bytes(batch, channels, length, gate, step)
LOUDNESS = {(0, 2, 100, 40, 10): (0, 0), (1, 1, 0, 40, 10): (0, 256), (1, 1, 1, 1, 1): (256, 256),
            (3, 2, 4409, 4410, 1102): (0, 256), (2, 5, 48001, 19200, 4800): (1792, 256),
            (256, 1, 80000, 6400, 1600): (204800, 16128), (7, 3, 100003, 1999, 3): (11200768, 228864)}


@pytest.mark.parametrize('op', sorted(PLAN_FREE))
def test_plan_free_sizes(op):
    fn = getattr(_lib(), 'kapre_%s_workspace_bytes' % op)
    got = {shape: fn(*shape) for shape in PLAN_FREE[op]}
    assert got == PLAN_FREE[op]


def test_loudness_sizes():
    lib = _lib()
    got = {}
    for shape in LOUDNESS:
        stats = ctypes.c_int64(-7)
        got[shape] = (lib.kapre_loudness_workspace_bytes(*shape, ctypes.byref(stats)), stats.value)
    assert got == LOUDNESS


@pytest.mark.parametrize('op', ['hpss', 'onset_strength'])
def test_size_beyond_int64_is_an_error(op):
    # 2^64 elements: the byte count does not fit in int64, so the size is KAPRE_E_INVALID, not a wrapped value
    assert getattr(_lib(), 'kapre_%s_workspace_bytes' % op)(65536, 65536, 65536, 65536) == -1


# ---- sizes that need a plan (created on the GPU); each plan object is held while its handle is in use ----
def _stft_plan(n_fft, hop):
    from kapre_b200 import backend, ops
    return ops.StftPlan(n_fft, n_fft, hop, backend.get_window_fn(None)(n_fft))


def _stft_backward(n_fft, hop, B, C, L, pad_begin, pad_end):
    from kapre_b200 import _native as N
    plan = _stft_plan(n_fft, hop)
    return N.lib().kapre_stft_backward_workspace_bytes(plan.handle(), B, C, L, pad_begin, pad_end)


def _convolve(block, B, C, L, P, backward):
    from kapre_b200 import _native as N
    from kapre_b200 import ops
    fn = N.lib().kapre_convolve_backward_workspace_bytes if backward else N.lib().kapre_convolve_workspace_bytes
    plan = ops.convolve_plan(block)
    return fn(plan.handle(), B, C, L, P)


def _griffin_lim(n_fft, hop, B, C, T):
    from kapre_b200 import _native as N
    plan = _stft_plan(n_fft, hop)
    return N.lib().kapre_griffin_lim_workspace_bytes(plan.handle(), B, C, T)


def _kaldi(subtract_mean, B, C, T):
    from kapre_b200 import _native as N
    from kapre_b200 import ops
    plan = ops.kaldi_plan('fbank', ops.kaldi_options('fbank', subtract_mean=subtract_mean))
    return N.lib().kapre_kaldi_workspace_bytes(plan.handle(), B, C, T, 1)


def _cqt(f_min, n_bins, B, C, L, backward):
    from kapre_b200 import _native as N
    from kapre_b200 import ops
    plan = ops.CqtPlan(22050, 512, f_min, n_bins)
    return N.lib().kapre_cqt_workspace_bytes(plan.handle(), B, C, L, backward)


def _pyin(B, C, L):
    from kapre_b200 import _native as N
    from kapre_b200 import ops
    plan = ops.PitchPlan(22050, 65.0, 2093.0, pyin={})
    return N.lib().kapre_pitch_workspace_bytes(plan.handle(), B, C, L)


def _chroma_cens(B, C, T):
    from kapre_b200 import _native as N
    from kapre_b200 import signal
    plan = signal._cqt_chroma_plans(22050, 512, None, 0.0, 12, 7, 36, True, 41)[1]
    return N.lib().kapre_chroma_cens_workspace_bytes(plan.handle(), B, C, T)


def _chroma_tuning(B, C, T):
    from kapre_b200 import _native as N
    from kapre_b200 import signal
    plan = signal._stft_chroma_plans(22050, 2048, 512, None, 1, None, 5.0, 2.0, True, tables=False)[1]
    return N.lib().kapre_chroma_tuning_workspace_bytes(plan.handle(), B, C, T)


def _chunked(fn, *args):
    k, n = ctypes.c_int(-1), ctypes.c_int64(-7)
    rc = fn(*args, ctypes.byref(k), ctypes.byref(n))
    return rc, k.value, n.value


def _pcen(B, C, T, F):
    from kapre_b200 import _native as N
    return _chunked(N.lib().kapre_pcen_workspace, B, C, T, F)


def _time_stretch(B, C, T, F, rate):
    from kapre_b200 import _native as N
    return _chunked(N.lib().kapre_time_stretch_workspace, B, C, T, F, rate)


# name: (size function, its value before KbLayout); PCEN and time stretch give (status, chunks, bytes)
PLAN_CASES = {
    'stft_backward(512, 128, 2, 3, 16001, 0, 0)': (lambda: _stft_backward(512, 128, 2, 3, 16001, 0, 0), 0),
    'stft_backward(512, 128, 2, 3, 16001, 1, 0)': (lambda: _stft_backward(512, 128, 2, 3, 16001, 1, 0), 393216),
    'stft_backward(512, 128, 2, 3, 16001, 0, 1)': (lambda: _stft_backward(512, 128, 2, 3, 16001, 0, 1), 396288),
    'stft_backward(512, 128, 2, 3, 16001, 1, 1)': (lambda: _stft_backward(512, 128, 2, 3, 16001, 1, 1), 405504),
    'stft_backward(400, 160, 3, 1, 12345, 1, 1)': (lambda: _stft_backward(400, 160, 3, 1, 12345, 1, 1), 154560),
    'convolve(256, 2, 3, 1024, 3)': (lambda: _convolve(256, 2, 3, 1024, 3, False), 123648),
    'convolve(256, 2, 3, 1000, 3)': (lambda: _convolve(256, 2, 3, 1000, 3, False), 123648),
    'convolve(128, 1, 1, 1, 1)': (lambda: _convolve(128, 1, 1, 1, 1, False), 2560),
    'convolve_backward(256, 2, 3, 1024, 3)': (lambda: _convolve(256, 2, 3, 1024, 3, True), 123648),
    'convolve_backward(256, 2, 3, 1000, 3)': (lambda: _convolve(256, 2, 3, 1000, 3, True), 148224),
    'convolve_backward(128, 1, 1, 1, 1)': (lambda: _convolve(128, 1, 1, 1, 1, True), 3072),
    'griffin_lim(1024, 256, 2, 3, 5)': (lambda: _griffin_lim(1024, 256, 2, 3, 5), 295424),
    'griffin_lim(1024, 256, 0, 3, 5)': (lambda: _griffin_lim(1024, 256, 0, 3, 5), 0),
    'griffin_lim(400, 160, 3, 1, 77)': (lambda: _griffin_lim(400, 160, 3, 1, 77), 893632),
    'kaldi_backward(mean off, 2, 3, 98)': (lambda: _kaldi(False, 2, 3, 98), 940800),
    'kaldi_backward(mean on, 2, 3, 98)': (lambda: _kaldi(True, 2, 3, 98), 994896),
    'kaldi_backward(mean on, 3, 1, 1001)': (lambda: _kaldi(True, 3, 1, 1001), 5081140),
    'cqt(1 octave, 2, 3, 22050)': (lambda: _cqt(500.0, 12, 2, 3, 22050, 0), 0),
    'cqt(7 octaves, 2, 3, 22050)': (lambda: _cqt(None, 84, 2, 3, 22050, 0), 521728),
    'cqt(7 octaves, 3, 1, 12345)': (lambda: _cqt(None, 84, 3, 1, 12345, 0), 146944),
    'cqt_backward(1 octave, 2, 3, 22050)': (lambda: _cqt(500.0, 12, 2, 3, 22050, 1), 0),
    'cqt_backward(7 octaves, 2, 3, 22050)': (lambda: _cqt(None, 84, 2, 3, 22050, 1), 1564416),
    'cqt_backward(7 octaves, 3, 1, 12345)': (lambda: _cqt(None, 84, 3, 1, 12345, 1), 439552),
    'pyin(2, 3, 22050)': (lambda: _pyin(2, 3, 22050), 900160),
    'pyin(3, 1, 12345)': (lambda: _pyin(3, 1, 12345), 256120),
    'pyin(1, 1, 1)': (lambda: _pyin(1, 1, 1), 3944),
    'chroma_cens(2, 3, 44)': (lambda: _chroma_cens(2, 3, 44), 12672),
    'chroma_cens(3, 1, 1001)': (lambda: _chroma_cens(3, 1, 1001), 144144),
    'chroma_tuning(2, 3, 44)': (lambda: _chroma_tuning(2, 3, 44), 387840),
    'chroma_tuning(3, 1, 1001)': (lambda: _chroma_tuning(3, 1, 1001), 4314624),
    'chroma_tuning(1, 1, 0)': (lambda: _chroma_tuning(1, 1, 0), 4864),
    'pcen(1, 1, 4000, 128)': (lambda: _pcen(1, 1, 4000, 128), [0, 32, 16384]),
    'pcen(256, 1, 427, 128)': (lambda: _pcen(256, 1, 427, 128), [0, 1, 0]),
    'time_stretch(1, 1, 427, 513, 0.8)': (lambda: _time_stretch(1, 1, 427, 513, 0.8), [0, 6, 12312]),
    'time_stretch(1, 1, 25840, 513, 0.8)': (lambda: _time_stretch(1, 1, 25840, 513, 0.8), [0, 32, 65664]),
}


@pytest.mark.gpu
@pytest.mark.parametrize('case', sorted(PLAN_CASES))
def test_plan_sizes(case):
    fn, want = PLAN_CASES[case]
    got = fn()
    assert (list(got) if isinstance(got, tuple) else got) == want, case
