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

The fused stack (``Sequential``'s STFT -> Magnitude [-> ApplyFilterbank] [-> MagnitudeToDecibel] launch) saves
only the waveform and recomputes the complex spectrum and the pre-decibel values in its backward.  Backward
passes are once-differentiable: a second derivative raises.
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


# Entry points used by ``ops``.  Dtype conversions happen outside the Functions so that autograd casts the
# gradient back to the caller's dtype.
def stft_forward(x, plan, input_data_format, output_data_format, pad_begin, pad_end, mode, fb, db, workspace):
    x = x.float()
    if mode == N.OUT_COMPLEX:
        return _Stft.apply(x, plan, input_data_format, output_data_format, pad_begin, pad_end, workspace)
    return _FusedStack.apply(x, plan, input_data_format, output_data_format, pad_begin, pad_end, mode, fb, db,
                             workspace)


def istft(X, plan, input_data_format, output_data_format):
    return _Istft.apply(X.to(torch.complex64), plan, input_data_format, output_data_format)


def magnitude(X):
    return _Magnitude.apply(X.to(torch.complex64))


def apply_filterbank(x, fb, data_format):
    return _ApplyFilterbank.apply(x.float(), fb, data_format)


def magnitude_to_decibel(x, ref_value, amin, dynamic_range):
    return _MagnitudeToDecibel.apply(x.float(), ref_value, amin, dynamic_range)
