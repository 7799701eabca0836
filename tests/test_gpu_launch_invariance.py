"""GPU tier: the forward transforms give the same bits at every launch shape, staging path and input placement.

The launcher picks a tile shape from the batch size (kb_pick_fwd_cfg, kb_pick_mc_cfg, kb_mr_pick), so the shapes a
small test batch runs are not the ones a large batch runs.  These tests force every feasible shape through the
switches the launcher reads at each call, read back the launch it made, and hold every shape to bit-identity with the
default launch: a missing barrier, a wrong mbarrier parity or a bulk copy into a buffer still being read changes bits
long before it breaks an oracle tolerance.  The default launch is held to the oracle.  Views (misaligned bases, time
strides, a zero batch stride) must give the bits of a contiguous copy, and an item must not depend on the batch it is
in, so that ``predict`` chunking and batch sharding do not change the result."""
import re

import numpy as np
import pytest

torch = pytest.importorskip('torch')

import oracle as O  # noqa: E402

pytestmark = pytest.mark.gpu

DB = (1.0, 1e-5, 1e9)   # (ref, amin, dynamic range): the clamp never binds, so the dB outputs are per element
FB_MODES = (3, 4)
MODE_NAMES = ['complex', 'mag', 'mag_db', 'fb', 'fb_db', 'mag_phase']
SWITCHES = ['KAPRE_B200_TF', 'KAPRE_B200_NW', 'KAPRE_B200_MC_TF', 'KAPRE_B200_MC_NW', 'KAPRE_B200_NOBULK',
            'KAPRE_B200_NOMC', 'KAPRE_B200_PDL_FWD', 'KAPRE_B200_MR_WARPS', 'KAPRE_B200_ISTFT2_M', 'KAPRE_B200_ISTFT2',
            'KAPRE_B200_FBMMA', 'KAPRE_B200_PAIRED']


@pytest.fixture(scope='module')
def K():
    assert torch.cuda.is_available(), 'GPU tier needs a CUDA device'
    import kapre_b200
    from kapre_b200 import _native
    _native.lib()
    return kapre_b200


@pytest.fixture
def env(monkeypatch):
    """Sets launcher switches for one call at a time; none leaks into the next test."""
    for k in SWITCHES:
        monkeypatch.delenv(k, raising=False)

    def set_env(**kw):
        for k in SWITCHES:
            monkeypatch.delenv(k, raising=False)
        for k, v in kw.items():
            monkeypatch.setenv('KAPRE_B200_' + k, str(v))
    return set_env


def nerr(a, b):
    return float(np.abs(np.asarray(a) - np.asarray(b)).max() / max(float(np.abs(b).max()), 1e-30))


def bits(t):
    """The tensor's bytes, for bit-for-bit comparison (complex and NaN included)."""
    t = t.contiguous()
    if t.is_complex():
        t = torch.view_as_real(t)
    return t.view(torch.int32)


def eq(a, b):
    return a.shape == b.shape and a.dtype == b.dtype and bool(torch.equal(bits(a), bits(b)))


def close(y, ref, mode):
    """Tolerance between two launches that sum in different orders: 2e-6 of the maximum, dB outputs as linear."""
    y, ref = y.double().cpu().numpy() if not y.is_complex() else y.cpu().numpy(), ref.cpu().numpy()
    if mode in (2, 4):
        y, ref = 10.0 ** (y / 10.0), 10.0 ** (ref.astype(np.float64) / 10.0)
    return nerr(y, ref) < 2e-6


def info():
    from kapre_b200 import _native
    return _native.last_launch_info()


def launched(pattern):
    m = re.search(pattern, info())
    assert m, (pattern, info())
    return m


def oracle_check(y, x, n_fft, win, hop, wname, pads, mode, fbm, fmt_in, fmt_out, C):
    """y against the float64 oracle: linear outputs (dB converted back) within 2e-6 of the maximum."""
    spec = O.stft_layer(x, n_fft, win, hop, wname, pads[0], pads[1], fmt_in, 'channels_first')
    y = y.cpu().numpy()
    if fmt_out == 'channels_last':
        y = np.moveaxis(y, 3, 1)
    mag = np.abs(spec)
    if mode == 0:
        assert nerr(y, spec) < 2e-6
        return
    if mode == 5:
        m, ph = y[:, :C], y[:, C:]
        assert nerr(m, mag) < 2e-6
        ok = mag > 1e-3 * mag.max()
        assert np.abs(np.angle(np.exp(1j * (ph - np.angle(spec)))))[ok].max() < 1e-3
        return
    lin = np.einsum('bctf,fm->bctm', mag, fbm.astype(np.float64)) if mode in FB_MODES else mag
    got = 10.0 ** (y.astype(np.float64) / 10.0) if mode in (2, 4) else y
    if mode in (2, 4):
        lin = np.maximum(lin, DB[1])
    assert nerr(got, lin) < 2e-6


def make(K, n_fft, win, hop, wname, mode, n_mels=64):
    from kapre_b200 import ops
    plan = ops.StftPlan(n_fft, win, hop, O.get_window(wname, win).astype(np.float32))
    fbm = O.filterbank_mel(22050, n_fft // 2 + 1, n_mels, 0.0, None, False, 'slaney').astype(np.float32) \
        if mode in FB_MODES else None
    fb = ops.Filterbank(fbm) if fbm is not None else None

    def fwd(x, fmt_in='channels_first', fmt_out='channels_first', pads=(True, True)):
        db = DB if mode in (2, 4) else None
        return ops.stft_forward(x, plan, fmt_in, fmt_out, pads[0], pads[1], mode, fb, db)
    return fwd, fbm


def try_launch(fwd, x, **kw):
    from kapre_b200 import _native
    try:
        return fwd(x, **kw)
    except _native.KapreNativeError as e:
        if 'no launch configuration fits' in str(e):
            return None
        raise


# ------------------------------------------------------------------------------------------- K1: single channel
K1_CASES = [(256, 64), (512, 128), (1024, 256), (2048, 512)]


def k1_candidates(n_fft, mode):
    Q = n_fft // 64
    fpw = 32 // Q
    out = []
    for nw in (1, 2, 4, 8, 16):
        fr = nw * fpw
        if fr > 32:
            continue
        for tf in (32, 16, 8, 4, 2, 1):
            if (tf == fr) if mode in FB_MODES else (tf % fr == 0):
                out.append((nw, tf))
    return out


@pytest.mark.parametrize('mode', range(6), ids=MODE_NAMES)
@pytest.mark.parametrize('n_fft,hop', K1_CASES)
def test_k1_every_tile_shape_gives_the_same_bits(K, env, n_fft, hop, mode):
    rng = np.random.default_rng(n_fft + mode)
    variants = [{}]
    if mode in FB_MODES:
        variants.append({'FBMMA': 1})
    if n_fft == 1024:
        variants.append({'PAIRED': 0})
    for wname, win in (('hann_window', n_fft), ('hann_window', 3 * n_fft // 4)):
        L = 41 * hop + hop // 2 + 1                       # odd: items 1 and 3 start at odd sample offsets
        x = rng.uniform(-1, 1, size=(4, 1, L)).astype(np.float32)
        xt = torch.from_numpy(x).cuda()
        fwd, fbm = make(K, n_fft, win, hop, wname, mode)
        for var in variants:
            env(**var)
            ref = fwd(xt)
            torch.cuda.synchronize()
            tag = launched(r'Q\d+ TF(\d+) NW(\d+) bulk1 .*fbmma(\d) v(\d)')
            assert tag.group(3) == ('1' if 'FBMMA' in var else '0') and tag.group(4) == ('2' if 'PAIRED' in var else '0')
            oracle_check(ref, x, n_fft, win, hop, wname, (True, True), mode, fbm, 'channels_first', 'channels_first', 1)
            env(NOBULK=1, **var)
            assert eq(fwd(xt), ref)
            launched(r' bulk0 ')
            env(PDL_FWD=0, **var)
            assert eq(fwd(xt), ref)
            for b in range(4):     # each item alone, at an aligned base
                env(**var)
                assert eq(fwd(xt[b:b + 1].clone()), ref[b:b + 1]), b
            ran = 0
            for nw, tf in k1_candidates(n_fft, mode):
                env(NW=nw, TF=tf, **var)
                y = try_launch(fwd, xt)
                if y is None:
                    continue
                launched(r'TF%d NW%d ' % (tf, nw))
                assert eq(y, ref), (nw, tf, var, info())
                ran += 1
            want = 3 if mode in FB_MODES else 6
            if 'FBMMA' in var:
                want = 2
            assert ran >= want, (ran, var)


@pytest.mark.parametrize('n_fft,hop', K1_CASES)
def test_k1_shapes_that_walk_several_tiles(K, env, n_fft, hop):
    """A batch large enough that CTAs walk two or more tiles (mbarrier parity flips, prefetch of the next tile, the
    parked tile plan of the filterbank modes): every shape against the default, items against the oracle."""
    g = torch.Generator(device='cuda').manual_seed(n_fft)
    L = 600 * hop + 3
    xt = torch.rand((64, 1, L), generator=g, device='cuda') * 2 - 1
    for mode in (1, 4):
        fwd, fbm = make(K, n_fft, n_fft, hop, 'hann_window', mode, n_mels=128)
        env()
        ref = fwd(xt)
        for b in (0, 33, 63):
            oracle_check(ref[b:b + 1], xt[b:b + 1].cpu().numpy(), n_fft, n_fft, hop, 'hann_window', (True, True), mode,
                         fbm, 'channels_first', 'channels_first', 1)
        walked = 0
        for nw, tf in k1_candidates(n_fft, mode):
            env(NW=nw, TF=tf)
            y = try_launch(fwd, xt)
            if y is None:
                continue
            m = launched(r'TF%d NW%d bulk1 grid(\d+) .* tiles(\d+)' % (tf, nw))
            walked += int(m.group(2)) >= 2 * int(m.group(1))
            assert eq(y, ref), (nw, tf, info())
        assert walked >= 1


# ---------------------------------------------------------------------------------------- K1b: all-channel tiles
MC_LAYOUTS = [('channels_last', 'channels_first'), ('channels_first', 'channels_last'),
              ('channels_last', 'channels_last')]


@pytest.mark.parametrize('C', [2, 3, 4, 5, 6, 7, 8, 12, 16, 31, 32])
def test_k1b_all_channel_tiles(K, env, C):
    n_fft, hop = (512, 128) if C % 2 else (1024, 256)
    rng = np.random.default_rng(C)
    for li, (fin, fout) in enumerate(MC_LAYOUTS):
        L = 23 * hop + 1
        x = rng.uniform(-1, 1, size=(3, L, C) if fin == 'channels_last' else (3, C, L)).astype(np.float32)
        xt = torch.from_numpy(x).cuda()
        for mode in range(6):
            if (mode + li) % 3 == 2:      # every mode in two of the three layouts
                continue
            fwd, fbm = make(K, n_fft, n_fft, hop, 'hann_window', mode)
            env()
            ref = fwd(xt, fin, fout)
            # the filterbank modes take all-channel tiles while one round of a CTA holds every channel
            if mode not in FB_MODES or C <= 8 * (32 // (n_fft // 64)):
                launched(r'^MC Q')
            oracle_check(ref, x, n_fft, n_fft, hop, 'hann_window', (True, True), mode, fbm, fin, fout, C)
            for b in range(3):
                assert eq(fwd(xt[b:b + 1].clone(), fin, fout), ref[b:b + 1]), b
            assert eq(fwd(xt[1:], fin, fout), ref[1:])
            if mode not in FB_MODES:
                ran = 0
                for nw in (1, 2, 4, 8):
                    for tf in (1, 2, 3, 5, 8, 16):
                        env(MC_NW=nw, MC_TF=tf)
                        y = fwd(xt, fin, fout)
                        if not info().startswith('MC ') or ' TF%d NW%d ' % (tf, nw) not in info():
                            continue          # the shape does not fit: single-channel tiles ran instead
                        assert eq(y, ref), (nw, tf, info())
                        ran += 1
                assert ran >= 3
            env(NOMC=1)
            y = fwd(xt, fin, fout)
            assert not info().startswith('MC ')
            assert close(y, ref, mode)        # the two kernels' pair steps differ: tolerance only


def test_k1b_falls_back_to_single_channel_tiles_above_32_channels(K, env):
    x = torch.rand((2, 4000, 33), device='cuda')
    fwd, _ = make(K, 512, 512, 128, 'hann_window', 1)
    env()
    y = fwd(x, 'channels_last', 'channels_last')
    assert re.match(r'Q8 TF', info()), info()
    ref = O.stft_layer(x.cpu().numpy(), 512, 512, 128, None, True, True, 'channels_last', 'channels_last')
    assert nerr(y.cpu().numpy(), np.abs(ref)) < 2e-6


# ------------------------------------------------------------------------------- K1d: mixed radix, direct DFT
@pytest.mark.parametrize('n_fft', [400, 480, 1000, 4096, 75, 98])
def test_k1d_mixed_radix_and_direct_dft(K, env, n_fft):
    hop = max(1, n_fft // 4)
    rng = np.random.default_rng(n_fft)
    L = 30 * hop + 1
    x = rng.uniform(-1, 1, size=(4, 1, L)).astype(np.float32)
    xt = torch.from_numpy(x).cuda()
    modes = (0, 1) if n_fft == 98 else (0, 1, 2) if n_fft < 200 else (0, 2, 3, 4)
    for mode in modes:
        fwd, fbm = make(K, n_fft, n_fft, hop, 'hann_window', mode, n_mels=40)
        env()
        ref = fwd(xt)
        launched(r'^DFT' if n_fft == 98 else r'^MR ')
        oracle_check(ref, x, n_fft, n_fft, hop, 'hann_window', (True, True), mode, fbm, 'channels_first',
                     'channels_first', 1)
        for b in range(4):
            assert eq(fwd(xt[b:b + 1].clone()), ref[b:b + 1]), b
        assert eq(fwd(xt[1:]), ref[1:])
    if n_fft != 98:
        # a batch with more tiles than the resident CTAs: the warp budget changes the grid and the tiles each CTA walks
        g = torch.Generator(device='cuda').manual_seed(n_fft)
        xb = torch.rand((256, 1, 200 * hop + 1), generator=g, device='cuda') * 2 - 1
        fwd, _ = make(K, n_fft, n_fft, hop, 'hann_window', 2)
        env()
        ref = fwd(xb)
        seen = set()
        for want in (8, 16, 24, 32, 48, 64):
            env(MR_WARPS=want)
            y = fwd(xb)
            seen.add(re.search(r'NW\d+ G\d+ grid\d+', info()).group(0))
            assert eq(y, ref), (want, info())
        assert len(seen) >= 2, seen


# ------------------------------------------------------------------------------------------------------- views
def view_cases(x):
    """(name, view) pairs of a (B, C, L) channels_first tensor with B >= 3, C >= 2 and odd L.  The strided time axis is
    taken from one channel: with several channels it would run the all-channel kernel, whose pair step differs by
    design from the single-channel kernel's that runs on a contiguous copy."""
    L = x.shape[2]
    mono = x[:, :1].contiguous()
    return [('offset_item', mono[1:]), ('narrow1', x.narrow(2, 1, L - 7)), ('narrow2', x.narrow(2, 2, L - 7)),
            ('narrow3', x.narrow(2, 3, L - 7)), ('stride2', mono[:, :, ::2]), ('channel', x[:, 1:2, :]),
            ('expand', x[:1].expand(4, -1, -1))]


@pytest.mark.parametrize('which', ['stft', 'mel_db', 'mag_phase'])
def test_views_give_the_bits_of_a_contiguous_copy(K, env, which):
    env()
    g = torch.Generator(device='cuda').manual_seed(5)
    x = torch.rand((3, 2, 22051), generator=g, device='cuda') * 2 - 1
    kw = dict(n_fft=1024, hop_length=256, input_data_format='channels_first', output_data_format='channels_first')
    if which == 'stft':
        layer = K.STFT(pad_end=True, **kw)
    elif which == 'mel_db':
        layer = K.get_melspectrogram_layer(sample_rate=22050, n_mels=128, return_decibel=True, **kw)
    else:
        layer = K.get_stft_mag_phase(None, return_decibel=True, **kw)
    for name, v in view_cases(x):
        assert eq(layer(v), layer(v.contiguous())), name


# --------------------------------------------------------------------------------------------------- contracts
@pytest.mark.parametrize('which', ['mel_db', 'magnitude'])
def test_predict_chunking_and_sharding_do_not_change_bits(K, env, which):
    env()
    rng = np.random.default_rng(11)
    x = rng.uniform(-1, 1, size=(7, 22051, 1)).astype(np.float32)
    kw = dict(n_fft=1024, hop_length=256, input_data_format='channels_last', output_data_format='channels_last')
    if which == 'mel_db':
        layer = K.get_melspectrogram_layer(sample_rate=22050, n_mels=128, return_decibel=True, **kw)
    else:
        layer = K.get_stft_magnitude_layer(return_decibel=True, **kw)
    xt = torch.from_numpy(x).cuda()
    whole = layer(xt)
    for k in (1, 3, 5):
        got = layer.predict(x, batch_size=k)
        assert got.shape == tuple(whole.shape) and got.tobytes() == whole.cpu().numpy().tobytes(), k
    parts = torch.cat([layer(xt[:2]), layer(xt[2:5]), layer(xt[5:])], dim=0)
    assert eq(parts, whole)


# ---------------------------------------------------------------------------------------- K3: inverse STFT
@pytest.mark.parametrize('n_fft,hop', [(512, 128), (1024, 256), (2048, 512)])
def test_k3_every_tile_length_against_the_oracle(K, env, n_fft, hop):
    rng = np.random.default_rng(n_fft)
    x = rng.uniform(-1, 1, size=(3, 1, 40 * hop + 1)).astype(np.float32)
    X = O.stft_layer(x, n_fft, n_fft, hop, None, False, False, 'channels_first', 'channels_first').astype(np.complex64)
    ref = O.istft_layer(X, n_fft, n_fft, hop, None, 'channels_first', 'channels_first')
    layer = K.InverseSTFT(n_fft=n_fft, hop_length=hop, input_data_format='channels_first',
                          output_data_format='channels_first')
    Xt = torch.from_numpy(X).cuda()
    ran = 0
    for m in range(1, 9):
        env(ISTFT2_M=m)
        y = layer(Xt)
        if ' rounds%d ' % m not in info():
            continue
        assert nerr(y.cpu().numpy(), ref) < 2e-6, (m, info())
        ran += 1
    assert ran >= 4
    K.STFT(n_fft=n_fft, hop_length=hop)(torch.zeros((1, 4 * n_fft, 1), device='cuda'))
    env(ISTFT2=0)
    y = layer(Xt)
    assert not info().startswith('ISTFT2')           # the class-ordered body ran (it leaves the info as it was)
    assert nerr(y.cpu().numpy(), ref) < 2e-6


def test_k3_predict_chunking_within_float32_rounding(K, env):
    """The streaming inverse picks its tile length from the batch size and sums overlapping frames in an order that
    follows it: ``predict`` chunks agree with the whole batch to float32 rounding, not necessarily bit for bit."""
    env()
    rng = np.random.default_rng(3)
    x = rng.uniform(-1, 1, size=(6, 1, 64 * 256 + 1)).astype(np.float32)
    X = O.stft_layer(x, 1024, 1024, 256, None, False, False, 'channels_first', 'channels_first').astype(np.complex64)
    seq = K.composed.Sequential([K.InverseSTFT(n_fft=1024, hop_length=256, input_data_format='channels_first',
                                               output_data_format='channels_first')])
    whole = seq(torch.from_numpy(X).cuda()).cpu().numpy()
    for k in (1, 4):
        assert nerr(seq.predict(X, batch_size=k), whole) < 1e-6
