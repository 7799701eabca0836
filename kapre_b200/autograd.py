"""Gradients of the hot-path layers: one ``torch.autograd.Function`` per op and one for the fused stack.

``ops`` routes a CUDA input through these only when autograd records it (``requires_grad`` and grad mode on);
everything else runs the forward code as before.  The forward of every Function is the launch ``ops`` issues
anyway, so outputs are bit-identical with or without ``requires_grad``.  The backward passes are CUDA launches
of their own (see ``include/kapre_b200.h``, "backward passes"):

* STFT            -> ``kapre_stft_backward``      (inverse-STFT kernel with the window w N/2 + edge/crop pass)
* InverseSTFT     -> ``kapre_istft_backward``     (forward STFT kernel with the window dual 2/N + DC/Nyquist pass)
* Magnitude       -> ``kapre_magnitude_backward`` (g X / |X|)
* ApplyFilterbank -> ``kapre_apply_filterbank`` with the transposed matrix
* MagnitudeToDecibel -> ``kapre_magnitude_to_decibel_backward`` (TensorFlow's tie rules)
* Phase           -> ``kapre_phase_backward``     (g i X / |X|^2)
* Delta           -> ``kapre_delta_backward``     (gather over the padded taps)
* Frame, Energy   -> ``kapre_frame_backward``, ``kapre_energy_backward`` (sum over the frames covering a sample)
* ConcatenateFrequencyMap -> ``kapre_concat_frequency_map_backward`` (the first C channels)
* SpecAugment     -> ``kapre_spec_augment`` over the gradient, mask value 0, the forward's device masks
* Resample        -> ``kapre_resample_backward`` (the resampling kernel with up and down exchanged)
* Speed, PitchShift's last step -> ``kapre_sinc_resample_backward`` (the interpolation kernel with step, offset and
  cutoff exchanged)
* Convolve, Reverb -> ``kapre_convolve_backward`` (correlations of the output spectra's gradient with the filter's and
  the signal's block spectra between the two transforms' adjoints) and ``kapre_convolve_ir_spectrum_backward``
* PCEN            -> ``kapre_pcen_backward`` (reverse-time scan; input and parameter gradients)
* lfilter, filtfilt, IIRFilter, Biquad, RandomBiquad -> ``kapre_lfilter_backward`` (the all-pole recursion run the
  other way on the output gradient; input and normalised-coefficient gradients, the rest through torch's division
  by a0)
* sosfilt, sosfiltfilt, SOSFilter -> ``kapre_sosfilt`` in the other time direction from a zero state (the input
  gradient; sosfiltfilt's data-dependent initial states through the DC gain, no coefficient or zi gradient)
* add_noise, BackgroundNoise -> ``kapre_add_noise_backward`` (a segment-sum pass over g n, then the input, noise and
  snr gradients from the saved energies)
* true_peak, LoudnessNormalization(true_peak_limit=...) -> ``kapre_true_peak_backward`` ((20 / ln 10) 4 h[t* - 4n + 40]
  / z[t*] at the saved first argmax t*)
* loudness, Loudness, LoudnessNormalization -> ``kapre_loudness_backward`` (gL (20 / ln 10) g_c y n(t) / (E2 |J2| G)
  from the saved gate decisions), then the two lfilter gradients of the K-weighting
* kaldi_fbank, kaldi_mfcc, kaldi_spectrogram, KaldiFbank, KaldiMFCC, KaldiSpectrogram -> ``kapre_kaldi_features_backward``
  (each frame's forward recomputed with the same dither and taken back to its samples, then a gather over the
  frames covering every sample)
* CQT (and its fused ``CQT -> Magnitude``) -> ``kapre_cqt_backward`` (per octave, lowest first, a gather of the
  filters' adjoint over the frames covering each sample plus the decimator's adjoint of the octave below; the
  magnitude mode recomputes C from the saved pyramid)
* chroma_stft, chroma_cqt, ChromaSTFT, ChromaCQT -> ``kapre_chroma_backward`` (y = W s recomputed, the gradient
  taken back through the normalisation and the threshold, then W^T and the input's square or modulus), then the STFT
  magnitude or CQT magnitude backward; the tuning estimate is a constant
* hpss, harmonic, percussive, HPSS -> ``kapre_hpss_backward`` (the medians recomputed with the element each one
  selected, the mask gradients written beside those indices, then a gather per element), then the STFT magnitude's
  or the STFT and inverse STFT's backward
* onset_strength, OnsetStrength -> ``kapre_onset_strength_backward`` (the tile recomputed with the bin each window
  maximum came from and the median's selected bins, then a gather per element), then, from a waveform, the existing
  backward passes of MagnitudeToDecibel, ApplyFilterbank and the STFT magnitude; ``detrend`` through lfilter's
* TimeStretch     -> ``kapre_time_stretch_backward`` (reverse-time scan over the saved output and its gradient)

The fused stack (``Sequential``'s STFT -> Magnitude [-> ApplyFilterbank] [-> MagnitudeToDecibel] launch) saves
only the waveform and recomputes the complex spectrum and the pre-decibel values in its backward; so does
``get_stft_mag_phase``'s fused magnitude + phase launch, whose backward ends in ``kapre_mag_phase_backward``.
Backward passes are once-differentiable: a second derivative raises.
"""
from __future__ import annotations

import torch
from torch.autograd.function import once_differentiable

from . import _native as N
from . import ops


class _Stft(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, plan, input_data_format, output_data_format, pad_begin, pad_end, workspace):
        ctx.cfg = (plan, input_data_format, output_data_format, pad_begin, pad_end)
        ctx.length = x.shape[1] if input_data_format == ops._CH_LAST_STR else x.shape[2]
        return ops.stft_forward(x, plan, input_data_format, output_data_format, pad_begin, pad_end, N.OUT_COMPLEX,
                                workspace=workspace)

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        plan, idf, odf, pb, pe = ctx.cfg
        return ops.stft_backward(g, plan, idf, odf, pb, pe, ctx.length), None, None, None, None, None, None


class _FusedStack(torch.autograd.Function):
    """STFT -> Magnitude [-> ApplyFilterbank] [-> MagnitudeToDecibel] as one launch forward, unfused backward."""

    @staticmethod
    def forward(ctx, x, plan, input_data_format, output_data_format, pad_begin, pad_end, mode, fb, db, workspace):
        ctx.save_for_backward(x)
        ctx.cfg = (plan, input_data_format, output_data_format, pad_begin, pad_end, mode, fb, db)
        return ops.stft_forward(x, plan, input_data_format, output_data_format, pad_begin, pad_end, mode, fb, db,
                                workspace)

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        (x,) = ctx.saved_tensors
        plan, idf, odf, pb, pe, mode, fb, db = ctx.cfg
        fbmode = mode in (N.OUT_FB, N.OUT_FB_DB)
        S = ops.stft_forward(x, plan, idf, odf, pb, pe, N.OUT_COMPLEX)
        if mode in (N.OUT_MAG_DB, N.OUT_FB_DB):
            pre = ops.stft_forward(x, plan, idf, odf, pb, pe, N.OUT_FB if fbmode else N.OUT_MAG, fb)
            g = ops.magnitude_to_decibel_backward(pre, g, *db)
        if fbmode:
            g = ops.apply_filterbank(ops._raw(g), fb.transposed(), odf)
        gS = ops.magnitude_backward(S, g)
        gx = ops.stft_backward(gS, plan, idf, odf, pb, pe, x.shape[1] if idf == ops._CH_LAST_STR else x.shape[2])
        return (gx,) + (None,) * 9


class _MagPhase(torch.autograd.Function):
    """``get_stft_mag_phase``'s fused mode (|STFT| [-> dB] and angle(STFT) side by side) as one launch forward."""

    @staticmethod
    def forward(ctx, x, plan, input_data_format, output_data_format, pad_begin, pad_end, db, workspace):
        ctx.save_for_backward(x)
        ctx.cfg = (plan, input_data_format, output_data_format, pad_begin, pad_end, db)
        return ops.stft_forward(x, plan, input_data_format, output_data_format, pad_begin, pad_end, N.OUT_MAG_PHASE,
                                None, db, workspace)

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        (x,) = ctx.saved_tensors
        plan, idf, odf, pb, pe, db = ctx.cfg
        S = ops.stft_forward(x, plan, idf, odf, pb, pe, N.OUT_COMPLEX)
        cl = odf == ops._CH_LAST_STR
        C = S.shape[3] if cl else S.shape[1]

        def half(t, lo):        # channels [lo, lo + C) of the 2C-channel output, as a view
            return t[..., lo:lo + C] if cl else t[:, lo:lo + C]
        g_mag, g_phase = half(g, 0), half(g, C)
        if db is not None:
            # The same fused launch without its decibel tail gives the very magnitudes the forward clamped (the
            # OUT_MAG launch pairs FFT outputs differently at some sizes, so its last bits may differ), and the
            # clamp decision is recomputed from them.  Each batch item is one clamp item, as in the forward.
            pre = ops.stft_forward(x, plan, idf, odf, pb, pe, N.OUT_MAG_PHASE)
            g_mag = ops.magnitude_to_decibel_backward(half(pre, 0), g_mag, *db)
        gS = ops.mag_phase_backward(S, g_mag, g_phase, odf)
        gx = ops.stft_backward(gS, plan, idf, odf, pb, pe, x.shape[1] if idf == ops._CH_LAST_STR else x.shape[2])
        return (gx,) + (None,) * 7


class _Istft(torch.autograd.Function):
    @staticmethod
    def forward(ctx, X, plan, input_data_format, output_data_format):
        ctx.cfg = (plan, input_data_format, output_data_format)
        ctx.frames = X.shape[1] if input_data_format == ops._CH_LAST_STR else X.shape[2]
        return ops.istft(X, plan, input_data_format, output_data_format)

    @staticmethod
    @once_differentiable
    def backward(ctx, gy):
        plan, idf, odf = ctx.cfg
        return ops.istft_backward(gy, plan, idf, odf, ctx.frames), None, None, None


class _Magnitude(torch.autograd.Function):
    @staticmethod
    def forward(ctx, X):
        ctx.save_for_backward(X)
        return ops.magnitude(X)

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        (X,) = ctx.saved_tensors
        return ops.magnitude_backward(X, g)


class _ApplyFilterbank(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, fb, data_format):
        ctx.cfg = (fb, data_format)
        return ops.apply_filterbank(x, fb, data_format)

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        fb, data_format = ctx.cfg
        return ops.apply_filterbank(ops._raw(g), fb.transposed(), data_format), None, None


class _MagnitudeToDecibel(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, ref_value, amin, dynamic_range):
        ctx.save_for_backward(x)
        ctx.db = (ref_value, amin, dynamic_range)
        return ops.magnitude_to_decibel(x, ref_value, amin, dynamic_range)

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        (x,) = ctx.saved_tensors
        return ops.magnitude_to_decibel_backward(x, g, *ctx.db), None, None, None


class _Phase(torch.autograd.Function):
    @staticmethod
    def forward(ctx, X):
        ctx.save_for_backward(X)
        return ops.phase(X)

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        (X,) = ctx.saved_tensors
        return ops.phase_backward(X, g)


class _Delta(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, win_length, mode, data_format):
        ctx.cfg = (win_length, mode, data_format)
        return ops.delta(x, win_length, mode, data_format)

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        return ops.delta_backward(g, *ctx.cfg), None, None, None


class _Frame(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, frame_length, hop_length, pad_end, pad_value, data_format):
        ctx.cfg = (frame_length, hop_length, data_format, x.shape[1] if data_format == ops._CH_LAST_STR else x.shape[2])
        return ops.frame(x, frame_length, hop_length, pad_end, pad_value, data_format)

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        return (ops.frame_backward(g, *ctx.cfg),) + (None,) * 5


class _Energy(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, frame_length, hop_length, pad_end, pad_value, scale, data_format):
        ctx.save_for_backward(x)
        ctx.cfg = (frame_length, hop_length, scale, data_format)
        return ops.energy(x, frame_length, hop_length, pad_end, pad_value, scale, data_format)

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        (x,) = ctx.saved_tensors
        return (ops.energy_backward(x, g, *ctx.cfg),) + (None,) * 6


class _ConcatFrequencyMap(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, data_format):
        ctx.data_format = data_format
        return ops.concat_frequency_map(x, data_format)

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        return ops.concat_frequency_map_backward(g, ctx.data_format), None


class _Resample(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, plan, data_format):
        ctx.cfg = (plan, data_format, x.shape[1] if data_format == ops._CH_LAST_STR else x.shape[2])
        return ops.resample(x, plan, data_format)

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        return ops.resample_backward(g, *ctx.cfg), None, None


class _SincResample(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, ratio, length, offset, data_format):
        ctx.cfg = (ratio, offset, data_format, x.shape[1] if data_format == ops._CH_LAST_STR else x.shape[2])
        return ops.sinc_resample(x, ratio, length, offset, data_format)

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        return ops.sinc_resample_backward(g, *ctx.cfg), None, None, None, None


class _Convolve(torch.autograd.Function):
    """x * h through ``kapre_convolve``.  The forward keeps H, and the signal spectra X only when h needs its
    gradient (they are the start of the forward's workspace, so keeping them costs no launch)."""

    @staticmethod
    def forward(ctx, x, h, h3, plan, mode, data_format):
        L = x.shape[ops._time_axis(data_format)]
        K = h3.shape[ops._time_axis(data_format)]
        H = ops.convolve_ir_spectrum(h3, plan, data_format)
        y, ws = ops.convolve_full(x, H, plan, data_format)
        start, n = ops.convolve_span(L, K, mode)
        want_h = ctx.needs_input_grad[1]
        if want_h:
            Bn, C, P, F = x.shape[0], y.shape[1] if data_format == ops._CH_FIRST_STR else y.shape[2], H.shape[2], H.shape[3]
            J = -(-L // plan.block)
            ctx.save_for_backward(H, ws[:Bn * C * J * F * 8].view(torch.complex64).view(Bn, C, J, F))
        else:
            ctx.save_for_backward(H)
        ctx.cfg = (plan, data_format, L, K, start, tuple(y.shape), tuple(h.shape), h3.shape)
        return ops._crop(y, start, n, data_format)

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        plan, fmt, L, K, start, full_shape, h_shape, h3_shape = ctx.cfg
        H = ctx.saved_tensors[0]
        X = ctx.saved_tensors[1] if len(ctx.saved_tensors) > 1 else None
        g_full = _zero_padded(g, full_shape, start, fmt)
        gx, gH = ops.convolve_backward(g_full, H, X, plan, fmt, L, ctx.needs_input_grad[0], ctx.needs_input_grad[1])
        gh = None
        if gH is not None:
            # a broadcast filter collects the gradient of every item / channel it served
            if H.shape[0] == 1 and gH.shape[0] > 1:
                gH = gH.sum(0, keepdim=True)
            if H.shape[1] == 1 and gH.shape[1] > 1:
                gH = gH.sum(1, keepdim=True)
            gh = ops.convolve_ir_spectrum_backward(gH, plan, K)              # (Bh, Ch, K)
            gh = gh.reshape(h_shape) if len(h_shape) == 1 else (gh if fmt == ops._CH_FIRST_STR else gh.transpose(1, 2))
        return gx, gh, None, None, None, None


class _ConvolveSpectrum(torch.autograd.Function):
    """x * h with constant filter spectra H: the gradient reaches x only."""

    @staticmethod
    def forward(ctx, x, H, plan, start, length, data_format):
        y, _ = ops.convolve_full(x, H, plan, data_format)
        ctx.save_for_backward(H)
        ctx.cfg = (plan, data_format, x.shape[ops._time_axis(data_format)], start, tuple(y.shape))
        return ops._crop(y, start, length, data_format)

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        plan, fmt, L, start, full_shape = ctx.cfg
        (H,) = ctx.saved_tensors
        gx, _ = ops.convolve_backward(_zero_padded(g, full_shape, start, fmt), H, None, plan, fmt, L, True, False)
        return gx, None, None, None, None, None


def _zero_padded(g, full_shape, start, data_format):
    """The gradient of a cropped output, placed in zeros of the untrimmed output's shape."""
    if tuple(g.shape) == tuple(full_shape):
        return g
    g_full = torch.zeros(full_shape, dtype=torch.float32, device=g.device)
    ops._crop(g_full, start, g.shape[ops._time_axis(data_format)], data_format).copy_(g)
    return g_full


class _Pcen(torch.autograd.Function):
    """The forward is the plain PCEN launch that also writes the smoother state M; the backward reads E and M and
    returns the gradients of the input and of the four parameters (gain, bias, power, smooth_coef)."""

    @staticmethod
    def forward(ctx, E, gain, bias, power, smooth, eps, data_format):
        y, M = ops.pcen_forward(E, (gain, bias, power, smooth), eps, data_format, save_M=True)
        ctx.save_for_backward(E, M, gain, bias, power, smooth)
        ctx.cfg = (eps, data_format)
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, gy):
        E, M, *params = ctx.saved_tensors
        gE, gp = ops.pcen_backward(E, M, gy, params, *ctx.cfg)
        return (gE, *gp, None, None)


class _Lfilter(torch.autograd.Function):
    """The forward is the plain lfilter launch without the clamp (the caller clamps with torch.clamp); the output is
    saved only when a coefficient needs its gradient, which is the only time the backward reads x and y."""

    @staticmethod
    def forward(ctx, x, b, a, flags, data_format):
        y = ops.lfilter_forward(x, b, a, flags, data_format)
        want = ctx.needs_input_grad[1] or ctx.needs_input_grad[2]
        ctx.save_for_backward(x if want else None, y if want else None, b, a)
        ctx.cfg = (flags, data_format, want)
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, gy):
        x, y, b, a = ctx.saved_tensors
        flags, data_format, want = ctx.cfg
        gx, gb, ga = ops.lfilter_backward(gy, x, y, b, a, flags, data_format, want)
        return (gx if ctx.needs_input_grad[0] else None, gb if ctx.needs_input_grad[1] else None,
                ga if ctx.needs_input_grad[2] else None, None, None)


class _Sosfilt(torch.autograd.Function):
    """A causal LTI filter's transpose is the same filter run in reverse time, so the backward is one more forward
    launch with the reverse flag flipped, from a zero state: gx = F^T gy.  With ``scale`` the initial state is
    ``scale * z`` for the unit-step steady state z, whose zero-input response is ``scale (H(1) 1 - F 1)``; its adjoint
    is ``H(1) sum(gy) - sum(F^T gy)``, which needs nothing beyond gx.  zf is not differentiable."""

    @staticmethod
    def forward(ctx, x, scale, sos, zi, dc_gain, reverse, data_format, want_zf):
        zi_eff = zi if scale is None else zi * scale.to(zi.dtype).reshape(scale.shape + (1, 1))
        y, zf = ops.sosfilt_forward(x, sos, zi_eff, reverse, data_format, want_zf)
        ctx.save_for_backward(sos, dc_gain)
        ctx.cfg = (reverse, data_format)
        if zf is None:
            zf = y.new_empty(0)
        ctx.mark_non_differentiable(zf)
        return y, zf

    @staticmethod
    @once_differentiable
    def backward(ctx, gy, _gzf):
        sos, dc_gain = ctx.saved_tensors
        reverse, data_format = ctx.cfg
        gx, _ = ops.sosfilt_forward(gy, sos, None, not reverse, data_format, False)
        gscale = None
        if ctx.needs_input_grad[1]:
            t = 1 if data_format == ops._CH_LAST_STR else 2
            gscale = (dc_gain * gy.double().sum(t) - gx.double().sum(t)).float()
        return (gx if ctx.needs_input_grad[0] else None, gscale, None, None, None, None, None, None)


class _AddNoise(torch.autograd.Function):
    """The forward is the plain two-launch mix, which also writes the per-column energies (Ex, En) for the backward;
    the noise is a tensor (differentiable) or a bank (a constant).  snr and the noise arrive as (B, C) / full-shape
    broadcast views, so torch sums their gradients over the broadcast axes."""

    @staticmethod
    def forward(ctx, x, noise, snr, lengths, bank, data_format):
        y, stats = ops.add_noise_forward(x, noise, bank, snr, lengths, data_format, True)
        ctx.save_for_backward(x, noise, snr, lengths, stats)
        ctx.cfg = (bank, data_format)
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        x, noise, snr, lengths, stats = ctx.saved_tensors
        bank, data_format = ctx.cfg
        want_n = ctx.needs_input_grad[1] and noise is not None
        gx, gn, gsnr = ops.add_noise_backward(g, x, noise, bank, snr, lengths, stats, data_format, want_n,
                                              ctx.needs_input_grad[2])
        return gx if ctx.needs_input_grad[0] else None, gn, gsnr, None, None, None


class _Loudness(torch.autograd.Function):
    """Over the K-weighted signal y (the two lfilter calls before it have their own autograd): the forward is the plain
    two-launch measurement, whose stats (E2, |J2| and the J2 decisions) the one-launch backward reads."""

    @staticmethod
    def forward(ctx, y, lengths, G, S, data_format):
        out, stats = ops.loudness_forward(y, lengths, G, S, data_format)
        ctx.save_for_backward(y, lengths, stats)
        ctx.cfg = (G, S, data_format)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        y, lengths, stats = ctx.saved_tensors
        G, S, data_format = ctx.cfg
        return ops.loudness_backward(g, y, lengths, G, S, stats, data_format), None, None, None, None


class _TruePeak(torch.autograd.Function):
    """The forward is the plain two-launch measurement; its stats (z[t*], t*) are all the one-launch backward reads."""

    @staticmethod
    def forward(ctx, x, lengths, data_format):
        out, stats = ops.true_peak_forward(x, lengths, data_format)
        ctx.save_for_backward(lengths, stats)
        B, C, L = (x.shape[0], x.shape[2], x.shape[1]) if data_format == ops._CH_LAST_STR else tuple(x.shape)
        ctx.cfg = ((B, C, L), data_format, x.device)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        lengths, stats = ctx.saved_tensors
        shape, data_format, device = ctx.cfg
        return ops.true_peak_backward(g, lengths, stats, shape, data_format, device), None, None


class _KaldiFeatures(torch.autograd.Function):
    """The forward is the plain feature launch; only the waveform is saved, and the backward regenerates the dither
    from (seed, item, channel, frame, sample)."""

    @staticmethod
    def forward(ctx, x, plan, lengths_h, lengths_d, data_format, dither, seed):
        y = ops.kaldi_forward(x, plan, lengths_h, lengths_d, data_format, dither, seed)
        ctx.save_for_backward(x)
        ctx.cfg = (plan, lengths_h, lengths_d, data_format, dither, seed)
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        x, = ctx.saved_tensors
        plan, lengths_h, lengths_d, data_format, dither, seed = ctx.cfg
        return ops.kaldi_backward(g, x, plan, lengths_h, lengths_d, data_format, dither, seed), None, None, None, \
            None, None, None


class _Cqt(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, plan, input_data_format, output_data_format, magnitude):
        y, ws = ops.cqt_forward(x, plan, input_data_format, output_data_format, magnitude)
        ctx.save_for_backward(x, ws if magnitude else None)
        ctx.cfg = (plan, input_data_format, output_data_format, magnitude)
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        x, ws = ctx.saved_tensors
        plan, idf, odf, magnitude = ctx.cfg
        return ops.cqt_backward(g, x, ws, plan, idf, odf, magnitude), None, None, None, None


class _Chroma(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, plan, cfg, data_format, table):
        ctx.save_for_backward(x, table)
        ctx.cfg = (plan, cfg, data_format)
        return ops.chroma_forward(x, plan, cfg, data_format, table)

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        x, table = ctx.saved_tensors
        plan, cfg, data_format = ctx.cfg
        return ops.chroma_backward(g, x, plan, cfg, data_format, table), None, None, None, None


class _Hpss(torch.autograd.Function):
    """Outputs the components ``want`` names, (harmonic, percussive) or one of them."""

    @staticmethod
    def forward(ctx, S, cfg, data_format, want_h, want_p):
        ctx.set_materialize_grads(False)
        ctx.save_for_backward(S)
        ctx.cfg = (cfg, data_format, want_h, want_p)
        h, p = ops.hpss_forward(S, cfg, data_format, want_h, want_p)
        return tuple(t for t in (h, p) if t is not None)

    @staticmethod
    @once_differentiable
    def backward(ctx, *gs):
        S, = ctx.saved_tensors
        cfg, data_format, want_h, want_p = ctx.cfg
        gs = list(gs)
        gh = gs.pop(0) if want_h else None
        gp = gs.pop(0) if want_p else None
        return ops.hpss_backward(gh, gp, S, cfg, data_format), None, None, None, None


class _TimeStretch(torch.autograd.Function):
    """The forward is the plain time-stretch launch; autograd saves its output, from which the backward takes the
    magnitude and phase gradients, so the forward writes nothing extra."""

    @staticmethod
    def forward(ctx, X, rate, data_format):
        Y = ops.time_stretch_forward(X, rate, data_format)
        ctx.save_for_backward(X, Y)
        ctx.cfg = (rate, data_format)
        return Y

    @staticmethod
    @once_differentiable
    def backward(ctx, G):
        X, Y = ctx.saved_tensors
        return ops.time_stretch_backward(X, Y, G, *ctx.cfg), None, None


class _SpecAugment(torch.autograd.Function):
    """The backward pass is the forward launch over the gradient, with mask value 0 and the masks the forward drew
    (saved on the device): it never draws new ones."""

    @staticmethod
    def forward(ctx, x, time_masks, freq_masks, mask_value, data_format):
        ctx.save_for_backward(time_masks, freq_masks)
        ctx.data_format = data_format
        return ops.spec_augment_masked(x, time_masks, freq_masks, mask_value, data_format)

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        tm, fm = ctx.saved_tensors
        return ops.spec_augment_masked(g, tm, fm, 0.0, ctx.data_format), None, None, None, None


# Entry points used by ``ops``.  Dtype conversions happen outside the Functions so that autograd casts the
# gradient back to the caller's dtype.
def stft_forward(x, plan, input_data_format, output_data_format, pad_begin, pad_end, mode, fb, db, workspace):
    x = x.float()
    if mode == N.OUT_COMPLEX:
        return _Stft.apply(x, plan, input_data_format, output_data_format, pad_begin, pad_end, workspace)
    if mode == N.OUT_MAG_PHASE:
        return _MagPhase.apply(x, plan, input_data_format, output_data_format, pad_begin, pad_end, db, workspace)
    return _FusedStack.apply(x, plan, input_data_format, output_data_format, pad_begin, pad_end, mode, fb, db,
                             workspace)


def phase(X):
    return _Phase.apply(X.to(torch.complex64))


def delta(x, win_length, mode, data_format):
    return _Delta.apply(x.float(), win_length, mode, data_format)


def frame(x, frame_length, hop_length, pad_end, pad_value, data_format):
    return _Frame.apply(x.float(), frame_length, hop_length, pad_end, pad_value, data_format)


def energy(x, frame_length, hop_length, pad_end, pad_value, scale, data_format):
    return _Energy.apply(x.float(), frame_length, hop_length, pad_end, pad_value, scale, data_format)


def concat_frequency_map(x, data_format):
    return _ConcatFrequencyMap.apply(x.float(), data_format)


def spec_augment(x, time_masks, freq_masks, mask_value, data_format):
    return _SpecAugment.apply(x.float(), time_masks, freq_masks, mask_value, data_format)


def resample(x, plan, data_format):
    return _Resample.apply(x.float(), plan, data_format)


def sinc_resample(x, ratio, length, offset, data_format):
    return _SincResample.apply(x.float(), ratio, length, offset, data_format)


def convolve(x, h, h3, plan, mode, data_format):
    return _Convolve.apply(x.float(), h, h3.float(), plan, mode, data_format)


def convolve_spectrum(x, H, plan, start, length, data_format):
    return _ConvolveSpectrum.apply(x.float(), H, plan, start, length, data_format)


def pcen(E, params, eps, data_format):
    return _Pcen.apply(E.float(), *params, eps, data_format)


def lfilter(x, b, a, flags, data_format):
    return _Lfilter.apply(x.float(), b, a, flags, data_format)


def sosfilt(x, scale, sos, zi, dc_gain, reverse, data_format, want_zf):
    y, zf = _Sosfilt.apply(x.float(), scale, sos, zi, dc_gain, reverse, data_format, want_zf)
    return y, (zf if want_zf else None)


def time_stretch(X, rate, data_format):
    return _TimeStretch.apply(X.to(torch.complex64), rate, data_format)


def istft(X, plan, input_data_format, output_data_format):
    return _Istft.apply(X.to(torch.complex64), plan, input_data_format, output_data_format)


def magnitude(X):
    return _Magnitude.apply(X.to(torch.complex64))


def apply_filterbank(x, fb, data_format):
    return _ApplyFilterbank.apply(x.float(), fb, data_format)


def magnitude_to_decibel(x, ref_value, amin, dynamic_range):
    return _MagnitudeToDecibel.apply(x.float(), ref_value, amin, dynamic_range)


def add_noise(x, noise, snr, lengths, bank, data_format):
    return _AddNoise.apply(x.float(), noise, snr, lengths, bank, data_format)


def loudness(y, lengths, G, S, data_format):
    return _Loudness.apply(y, lengths, G, S, data_format)


def true_peak(x, lengths, data_format):
    return _TruePeak.apply(x, lengths, data_format)


def kaldi_features(x, plan, lengths_h, lengths_d, data_format, dither, seed):
    return _KaldiFeatures.apply(x, plan, lengths_h, lengths_d, data_format, dither, seed)


def cqt(x, plan, input_data_format, output_data_format, magnitude):
    return _Cqt.apply(x, plan, input_data_format, output_data_format, magnitude)


def chroma(x, plan, cfg, data_format, table):
    return _Chroma.apply(x, plan, cfg, data_format, table)


def hpss(S, cfg, data_format, want_h, want_p):
    out = _Hpss.apply(S, cfg, data_format, want_h, want_p)
    out = out if isinstance(out, tuple) else (out,)
    it = iter(out)
    return (next(it) if want_h else None), (next(it) if want_p else None)


class _OnsetStrength(torch.autograd.Function):
    @staticmethod
    def forward(ctx, S, cfg, data_format):
        ctx.save_for_backward(S)
        ctx.cfg = (cfg, data_format)
        return ops.onset_strength_forward(S, cfg, data_format)

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        S, = ctx.saved_tensors
        cfg, data_format = ctx.cfg
        return ops.onset_strength_backward(g, S, cfg, data_format), None, None


def onset_strength(S, cfg, data_format):
    return _OnsetStrength.apply(S, cfg, data_format)
