"""Image-source room impulse responses on the CPU: the float64 restatement's self-checks (rir_ref.py), the kernel body
of rir_core.cuh (run by a CPU emulation) against the restatement within the derived bound, its bit-independence of
tile size, tile order, batch position and start offset, and the host-side draws and construction checks of
RoomReverb."""
import ctypes
import hashlib
import math
import os
import subprocess
import tempfile

import numpy as np
import pytest

import rir_ref as RR

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, 'emu', 'kb_emu_rir.cpp')
_CSRC = os.path.join(_HERE, '..', 'kapre_b200', 'csrc')
_lib_handle = None


def _lib():
    """tests/emu/kb_emu_rir.cpp built with g++ into the temporary directory (keyed by the sources' contents)."""
    global _lib_handle
    if _lib_handle is None:
        hs = hashlib.sha256()
        for f in [_SRC] + sorted(os.path.join(_CSRC, n) for n in os.listdir(_CSRC) if n.endswith(('.h', '.cuh'))):
            with open(f, 'rb') as fh:
                hs.update(fh.read())
        out = os.path.join(tempfile.gettempdir(), 'kapre_b200_emu_rir_%s.so' % hs.hexdigest()[:16])
        if not os.path.exists(out):
            tmp = '%s.%d.tmp' % (out, os.getpid())
            subprocess.check_call(['g++', '-O2', '-std=c++17', '-shared', '-fPIC', '-DKB_HOST_EMU', '-Wno-unknown-pragmas',
                                   '-o', tmp, _SRC])
            os.replace(tmp, out)
        lib = ctypes.CDLL(out)
        I, P, D = ctypes.c_int, ctypes.c_void_p, ctypes.c_double
        lib.kb_emu_rir_ism.argtypes = [P, P, I, I, I, I, D, D, P, P, P, I, I]
        _lib_handle = lib
    return _lib_handle


def _p(a):
    return ctypes.c_void_p(a.__array_interface__['data'][0])


def signed_window(W):
    """The kernel's table: w[k] (-1)^(k + 1 - half), rounded to float32."""
    half = (W - 1) // 2
    k = np.arange(W)
    w = 0.5 - 0.5 * np.cos(2 * np.pi * k / (W - 1)) if W > 1 else np.ones(1)
    return (w * np.where((k + 1 - half) % 2 == 0, 1.0, -1.0)).astype(np.float32)


def emu(recs, mics, L, W=81, fs=16000.0, c=343.0, nw=8, tile_order=0, layout='bml'):
    """recs (B, 14), mics (B, M, 3) float64 -> (B, M, L) float32 ('bml') or (B, L, M) ('blm', returned as (B, M, L))."""
    recs = np.ascontiguousarray(recs, np.float64)
    mics = np.ascontiguousarray(mics, np.float64)
    B, M = mics.shape[:2]
    if layout == 'bml':
        out = np.full((B, M, L), np.nan, np.float32)
        os_ = np.array([M * L, L, 1], np.int64)
        view = out
    else:
        out = np.full((B, L, M), np.nan, np.float32)
        os_ = np.array([L * M, 1, M], np.int64)
        view = out.transpose(0, 2, 1)
    ws = signed_window(W)
    rc = _lib().kb_emu_rir_ism(_p(recs), _p(mics), B, M, L, W, fs, c, _p(ws), _p(out), _p(os_), nw, tile_order)
    assert rc == 0
    return np.ascontiguousarray(view)


ROOMS = {
    'cube': ((4.0, 4.0, 4.0), (1.3, 2.1, 1.7)),
    'flat': ((8.0, 6.0, 2.5), (2.2, 3.1, 1.2)),
    'corridor': ((12.0, 2.0, 3.0), (1.5, 0.7, 1.6)),
}
ABSORPTION = {
    'zero': np.zeros(6),
    'mix': np.array([0.1, 0.35, 0.2, 0.6, 0.05, 0.45]),
    'one': np.ones(6),
}


def _mics(room, n, seed):
    rng = np.random.default_rng(seed)
    return rng.uniform(0.2, 1.0, size=(n, 3)) * (np.asarray(room) - 0.4) + 0.2


def _check(recs, mics, L, W, fs, **kw):
    got = emu(recs, mics, L, W, fs, **kw)
    for b in range(recs.shape[0]):
        r = recs[b]
        mo = None if r[12] < 0 else int(r[12])
        for m in range(mics.shape[1]):
            want, bound = RR.rir(r[0:3], r[3:6], mics[b, m], r[6:12], L, W, fs, max_order=mo, start=int(r[13]))
            err = np.abs(got[b, m].astype(np.float64) - want)
            assert np.all(err <= bound), (b, m, float(np.max(err - bound)), int(np.argmax(err - bound)))
    return got


@pytest.mark.parametrize('room', sorted(ROOMS))
@pytest.mark.parametrize('absorption', sorted(ABSORPTION))
def test_rooms_against_restatement(room, absorption):
    dims, src = ROOMS[room]
    rec = RR.record(dims, src, RR.betas(ABSORPTION[absorption]), max_order=None)
    mics = _mics(dims, 3, 1)
    got = _check(rec[None], mics[None], 700, 81, 8000.0)
    assert np.any(got != 0)


@pytest.mark.parametrize('max_order', [0, 1, 5, None])
@pytest.mark.parametrize('n_mics', [1, 8])
def test_max_order_and_mics(max_order, n_mics):
    dims, src = ROOMS['flat']
    rec = RR.record(dims, src, RR.betas(ABSORPTION['mix']), max_order=max_order)
    got = _check(rec[None], _mics(dims, n_mics, 2)[None], 500, 81, 8000.0)
    if max_order == 0:
        nz = np.nonzero(got[0, 0])[0]
        assert nz.size <= 81


@pytest.mark.parametrize('fs', [8000.0, 16000.0, 48000.0])
@pytest.mark.parametrize('W', [1, 3, 81, 255])
def test_rates_and_filter_lengths(fs, W):
    dims, src = ROOMS['cube']
    rec = RR.record(dims, src, RR.betas(ABSORPTION['mix']), max_order=None if fs < 40000 else 4)
    L = int(0.03 * fs) + W
    _check(rec[None], _mics(dims, 2, 3)[None], L, W, fs)


@pytest.mark.parametrize('layout', ['bml', 'blm'])
def test_layouts(layout):
    dims, src = ROOMS['corridor']
    rec = RR.record(dims, src, RR.betas(ABSORPTION['mix']))
    _check(rec[None], _mics(dims, 3, 4)[None], 300, 81, 8000.0, layout=layout)


def test_short_outputs():
    dims, src = ROOMS['flat']
    mic = np.array([[7.0, 5.0, 2.0]])
    rec = RR.record(dims, src, RR.betas(ABSORPTION['mix']))
    tau = math.dist(src, mic[0]) * 16000.0 / 343.0
    # shorter than the direct delay: all zeros
    got = _check(rec[None], mic[None], int(tau) - 1, 81, 16000.0)
    assert np.all(got == 0)
    # ends in the middle of the direct path's filter, and one sample into it
    _check(rec[None], mic[None], int(tau) + 20, 81, 16000.0)
    _check(rec[None], mic[None], int(tau) + 1, 81, 16000.0)


def test_bits_independent_of_tiles_batch_and_start():
    dims, src = ROOMS['flat']
    mics = _mics(dims, 2, 5)
    rec = RR.record(dims, src, RR.betas(ABSORPTION['mix']))
    L = 900
    ref = emu(rec[None], mics[None], L, 81, 8000.0, nw=8)
    for nw in (1, 2, 4):
        for order in (0, 1):
            assert np.array_equal(emu(rec[None], mics[None], L, 81, 8000.0, nw=nw, tile_order=order), ref)
    # batch position and neighbours
    other = RR.record((5.0, 4.0, 3.0), (1.0, 1.0, 1.0), RR.betas(np.full(6, 0.3)))
    recs = np.stack([other, rec, other])
    mics3 = np.stack([_mics((5.0, 4.0, 3.0), 2, 6), mics, _mics((5.0, 4.0, 3.0), 2, 7)])
    assert np.array_equal(emu(recs, mics3, L, 81, 8000.0, nw=4)[1], ref[0])
    # a start offset gives a slice of the full response
    for start in (1, 37, 300):
        r2 = rec.copy()
        r2[13] = start
        got = emu(r2[None], mics[None], L - start, 81, 8000.0, nw=2)
        assert np.array_equal(got[0], ref[0][:, start:])


def test_restatement_properties():
    for name in dir(RR):
        if name.startswith('check_'):
            getattr(RR, name)()


# ---- validation (the C entry's checks run on the host: null device pointers validate only) -----------------------
def _validate(recs, mics, L=100, W=81, fs=16000.0, c=343.0):
    import kapre_b200._native as N
    recs = np.ascontiguousarray(recs, np.float64).reshape(-1, RR.REC)
    mics = np.ascontiguousarray(mics, np.float64).reshape(recs.shape[0], -1, 3)
    host = np.concatenate([recs.ravel(), mics.ravel()])
    return N.lib().kapre_rir_ism(_p(host), None, recs.shape[0], mics.shape[1], L, W, fs, c, 0, None, 0, 0, 0, None)


def test_validation_before_any_launch():
    good = RR.record((5.0, 4.0, 3.0), (1.0, 1.0, 1.0), np.full(6, 0.8))
    mic = np.array([[2.0, 2.0, 2.0]])
    assert _validate(good, mic) == 0
    bad = []
    for i, v in ((0, 0.0), (1, np.inf), (3, 0.0), (4, 4.0), (6, 1.5), (9, -0.1), (12, 1.5), (12, -2.0), (13, -1.0),
                 (13, 0.5), (13, 2.0 ** 31)):
        r = good.copy()
        r[i] = v
        bad.append((r, mic, {}))
    bad += [(good, np.array([[5.0, 2.0, 2.0]]), {}), (good, np.array([[1.0005, 1.0, 1.0]]), {}),
            (good, mic, {'W': 80}), (good, mic, {'W': 257}), (good, mic, {'L': 0}), (good, mic, {'fs': 0.0}),
            (good, mic, {'c': np.nan}),
            # the image bound: a 1 m cube for 2 s at 16 kHz has ~2.5e8 images
            (RR.record((1.0, 1.0, 1.0), (0.3, 0.3, 0.3), np.ones(6)), np.array([[0.6, 0.6, 0.6]]), {'L': 32000})]
    for r, m, kw in bad:
        assert _validate(r, m, **kw) == -1, (r, m, kw)


@pytest.mark.parametrize('side,max_order,L', [(1.0, 10, 32000), (0.3, 0, 2000), (1.0, 3, 160000), (0.01, None, 10 ** 6)])
def test_image_cap_holds_whatever_the_max_order(side, max_order, L):
    """The cap bounds the enumeration, which walks the whole arrival ball: a max_order that leaves few images does not
    lift it."""
    r = RR.record((side,) * 3, (0.3 * side,) * 3, np.ones(6), max_order=max_order)
    assert _validate(r, np.array([[0.6 * side] * 3]), L=L) == -1


def test_image_cap_at_its_edge():
    # 3 x 3 x 2.5 m at 0.8 s (16 kHz) has a bound of 7.7e6 and runs; the same room at 1.2 s is above 2^24
    r = RR.record((3.0, 3.0, 2.5), (1.2, 1.1, 1.3), np.full(6, 0.9))
    mic = np.array([[2.3, 2.2, 1.6]])
    assert _validate(r, mic, L=12800) == 0
    assert _validate(r, mic, L=19200) == -1


def test_simulate_rir_ism_argument_checks():
    from kapre_b200 import signal
    ok = dict(room=(5.0, 4.0, 3.0), source=(1.0, 1.0, 1.0), mic_array=[[2.0, 2.0, 2.0]], max_order=None,
              absorption=0.3, output_length=100)
    for k, v in (('max_order', -1), ('max_order', 1.5), ('output_length', 0), ('absorption', 1.5),
                 ('absorption', [0.1] * 5), ('room', (1.0, 2.0)), ('mic_array', [1.0, 2.0, 3.0]),
                 ('delay_filter_length', 8.0)):
        with pytest.raises(ValueError):
            signal.simulate_rir_ism(**dict(ok, **{k: v}))


def test_inverse_sabine():
    from kapre_b200 import backend
    for room, rt in (((5.0, 4.0, 3.0), 0.5), ((3.0, 3.0, 2.5), 0.8)):
        a = backend.inverse_sabine(rt, room)
        assert a == pytest.approx(RR.inverse_sabine(rt, room), rel=1e-15)
        assert RR.sabine_rt60(a, room) == pytest.approx(rt, rel=1e-12)
    with pytest.raises(ValueError):
        backend.inverse_sabine(0.05, (10.0, 10.0, 4.0))


# ---- RoomReverb on the host: draws and construction -----------------------------------------------------------------
def test_room_reverb_draws():
    from kapre_b200.augmentation import RoomReverb
    a, b = RoomReverb(16000, seed=3), RoomReverb(16000, seed=3)
    da, db = a.draw(64), b.draw(64)
    for u, v in zip(da, db):
        assert np.array_equal(u, v)
    room, rt60, source, mic = da
    for d, (lo, hi) in enumerate(a.room_range):
        assert np.all((room[:, d] >= lo) & (room[:, d] <= hi))
    assert np.all((rt60 >= 0.2) & (rt60 <= 0.8))
    for p in (source, mic):
        assert np.all(p >= 0.5) and np.all(p <= room - 0.5)
    assert np.all(np.linalg.norm(source - mic, axis=1) >= 0.5)
    # the documented order, replayed by hand; the redraw reached by a large min_distance
    c = RoomReverb(16000, room_range=((3, 3.2), (3, 3.2), (2.5, 2.6)), min_distance=1.6, seed=5)
    room, rt60, source, mic = c.draw(16)
    rng = np.random.default_rng(5)
    redraws = 0
    for i in range(16):
        assert np.array_equal(rng.uniform([3, 3, 2.5], [3.2, 3.2, 2.6]), room[i])
        assert rng.uniform(0.2, 0.8) == rt60[i]
        assert np.array_equal(rng.uniform(0.5, room[i] - 0.5), source[i])
        m = rng.uniform(0.5, room[i] - 0.5)
        while np.linalg.norm(m - source[i]) < 1.6:
            m = rng.uniform(0.5, room[i] - 0.5)
            redraws += 1
        assert np.array_equal(m, mic[i])
    assert redraws > 0
    assert np.all(np.linalg.norm(source - mic, axis=1) >= 1.6)


def test_room_reverb_records_start_at_the_direct_path():
    from kapre_b200.augmentation import RoomReverb
    layer = RoomReverb(16000, seed=1)
    room, rt60, source, mic = layer.draw(8)
    rec = layer.records(room, rt60, source, mic)
    tau = np.linalg.norm(source - mic, axis=1) * 16000 / 343.0
    assert np.array_equal(rec[:, 13], np.floor(tau + 0.5) + 40)
    assert np.allclose(1 - rec[:, 6:12] ** 2, [[RR.inverse_sabine(t, r)] * 6 for t, r in zip(rt60, room)], rtol=1e-12)
    assert layer.rir_length == 12800
    assert layer.get_config()['rt60_range'] == [0.2, 0.8]


def test_room_reverb_construction_checks():
    from kapre_b200.augmentation import RoomReverb
    with pytest.raises(ValueError):
        RoomReverb(16000, room_range=((3, 20), (3, 10), (2.5, 4)), rt60_range=(0.1, 0.8))    # alpha > 1
    with pytest.raises(ValueError):
        RoomReverb(16000, room_range=((0.9, 3), (3, 10), (2.5, 4)))                        # no room for the margin
    with pytest.raises(ValueError):
        RoomReverb(16000, room_range=((1.2, 3), (1.2, 3), (1.2, 3)), min_distance=1.0)     # nor for the distance
    with pytest.raises(ValueError):
        RoomReverb(16000, delay_filter_length=80)
    # the mic's distance must be at most half the inner diagonal of the smallest room (2, 2, 1.5): 1.6 m
    RoomReverb(16000, room_range=((3, 4), (3, 4), (2.5, 3)), min_distance=1.6)
    with pytest.raises(ValueError):
        RoomReverb(16000, room_range=((3, 4), (3, 4), (2.5, 3)), min_distance=1.61)
    # the longest response in the smallest room must fit the image cap: 1.2 s in 3 x 3 x 2.5 m does not
    with pytest.raises(ValueError):
        RoomReverb(16000, rir_length=19200)
    RoomReverb(48000)


def test_room_reverb_redraws_are_bounded():
    from kapre_b200.augmentation import RoomReverb
    layer = RoomReverb(16000, room_range=((3, 3), (3, 3), (2.5, 2.5)), min_distance=1.6, seed=0)
    layer.MAX_REDRAWS = 0
    with pytest.raises(ValueError):
        for _ in range(50):                      # a first draw closer than 1.6 m comes within a few items
            layer.draw(1)
