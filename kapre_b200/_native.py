"""ctypes binding of libkapre_b200.so (the C ABI in include/kapre_b200.h).

The CUDA library is the product: there is NO fallback.  If the shared object is missing
the import fails loudly with the build command.
"""
from __future__ import annotations

import ctypes
import os
from ctypes import POINTER, Structure, c_char_p, c_double, c_float, c_int, c_int32, c_int64, c_uint64, c_void_p

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, '_lib', 'libkapre_b200.so')

OUT_COMPLEX, OUT_MAG, OUT_MAG_DB, OUT_FB, OUT_FB_DB, OUT_MAG_PHASE = range(6)


class KapreNativeError(RuntimeError):
    pass


class WaveDesc(Structure):
    _fields_ = [('batch', c_int32), ('channels', c_int32), ('length', c_int32),
                ('stride_b', c_int64), ('stride_c', c_int64), ('stride_l', c_int64)]


class SpecDesc(Structure):
    _fields_ = [('stride_b', c_int64), ('stride_c', c_int64), ('stride_t', c_int64),
                ('stride_f', c_int64)]


class PcenParams(Structure):
    _fields_ = [('gain', c_void_p), ('bias', c_void_p), ('power', c_void_p), ('smooth', c_void_p),
                ('gain_stride', c_int), ('bias_stride', c_int), ('power_stride', c_int), ('smooth_stride', c_int),
                ('eps', c_float)]


class GlCfg(Structure):
    _fields_ = [('n_iter', c_int), ('momentum', c_float), ('init', c_int), ('seed', c_uint64)]


GL_INIT_ONES, GL_INIT_RANDOM = 0, 1


class FbInvCfg(Structure):
    _fields_ = [('n_iter', c_int), ('from_decibel', c_int), ('ref_value', c_float), ('amin', c_float)]


class IirCoeffs(Structure):
    _fields_ = [('b', c_void_p), ('a', c_void_p), ('b_stride_b', c_int64), ('b_stride_c', c_int64),
                ('a_stride_b', c_int64), ('a_stride_c', c_int64), ('order', c_int)]


IIR_CLAMP, IIR_REVERSE = 1, 2
RIR_UNIT_NORM = 1


class SosCoeffs(Structure):
    _fields_ = [('sos', c_void_p), ('stride_b', c_int64), ('stride_c', c_int64), ('n_sections', c_int)]


class SosStateDesc(Structure):
    _fields_ = [('stride_b', c_int64), ('stride_c', c_int64), ('stride_s', c_int64)]


class NoiseSource(Structure):
    _fields_ = [('mode', c_int), ('noise', c_void_p), ('noise_desc', WaveDesc), ('bank', c_void_p),
                ('bank_length', c_int64), ('start', c_void_p), ('clip_len', c_void_p), ('offset', c_void_p)]


class SnrDesc(Structure):
    _fields_ = [('snr', c_void_p), ('snr_stride_b', c_int64), ('snr_stride_c', c_int64), ('lengths', c_void_p),
                ('lengths_stride_b', c_int64), ('lengths_stride_c', c_int64)]


NOISE_TENSOR, NOISE_BANK = 0, 1


class KaldiCfg(Structure):
    _fields_ = [('kind', c_int), ('window_size', c_int), ('window_shift', c_int), ('padded_window_size', c_int),
                ('snip_edges', c_int), ('min_length', c_int), ('num_mel_bins', c_int), ('num_ceps', c_int),
                ('use_energy', c_int), ('htk_compat', c_int), ('raw_energy', c_int), ('use_power', c_int),
                ('use_log_fbank', c_int), ('remove_dc_offset', c_int), ('subtract_mean', c_int),
                ('preemphasis_coefficient', c_float), ('energy_floor', c_float)]


CQT_MAX_OCTAVES = 12


class CqtCfg(Structure):
    _fields_ = [('n_bins', c_int), ('bins_per_octave', c_int), ('hop_length', c_int),
                ('taps', c_int * CQT_MAX_OCTAVES)]


class PitchCfg(Structure):
    _fields_ = [('sample_rate', c_float), ('frame_length', c_int), ('win_length', c_int), ('hop_length', c_int),
                ('center', c_int), ('min_period', c_int), ('max_period', c_int), ('trough_threshold', ctypes.c_double),
                ('n_thresholds', c_int), ('n_pitch', c_int), ('band_width', c_int), ('log_stay', c_float),
                ('log_switch', c_float), ('log_init_voiced', c_float), ('log_init_unvoiced', c_float),
                ('fill_na', c_float)]


class PitchTables(Structure):
    _fields_ = [(name, c_void_p) for name in ('beta_probs', 'boltzmann_pow', 'boltzmann_norm', 'no_trough_bonus',
                                              'period_edges', 'freqs', 'log_triangle', 'log_row_norm')]


class FramesDesc(Structure):
    _fields_ = [('stride_b', c_int64), ('stride_c', c_int64), ('stride_t', c_int64)]


class HpssCfg(Structure):
    _fields_ = [('kernel_h', c_int), ('kernel_p', c_int), ('power', c_float), ('margin_h', c_float),
                ('margin_p', c_float), ('mask', c_int)]


HPSS_MAX_KERNEL = 64


class OnsetCfg(Structure):
    _fields_ = [('lag', c_int), ('max_size', c_int), ('aggregate', c_int), ('pad_frames', c_int)]


class OnsetDetectCfg(Structure):
    _fields_ = [('pre_max', c_int), ('post_max', c_int), ('pre_avg', c_int), ('post_avg', c_int), ('wait', c_int),
                ('normalize', c_int), ('delta', ctypes.c_double)]


class BeatCfg(Structure):
    _fields_ = [('fps', ctypes.c_double), ('tightness', ctypes.c_double), ('trim', c_int)]


ONSET_MEAN, ONSET_MEDIAN = 0, 1
ONSET_MAX_BINS = 4097
TEMPOGRAM_MAX_WIN = 4096
BEAT_MAX_PERIOD = 4096
PEAK_MAX_WINDOW = 1 << 30


class ChromaPlanDesc(Structure):
    _fields_ = [('n_chroma', c_int), ('n_bins', c_int), ('n_tables', c_int), ('tables', c_void_p),
                ('n_smooth', c_int), ('smooth', c_void_p), ('n_tuning_bins', c_int), ('tuning_edges', c_void_p),
                ('peak_lo', c_int), ('peak_hi', c_int), ('sample_rate', c_float), ('n_fft', c_float),
                ('bins_per_octave', ctypes.c_double)]


class ChromaCfg(Structure):
    _fields_ = [('in_mode', c_int), ('norm', c_int), ('has_threshold', c_int), ('threshold', c_float)]


CHROMA_IN_LINEAR, CHROMA_IN_SQUARE, CHROMA_IN_COMPLEX = range(3)
CHROMA_NORM_NONE, CHROMA_NORM_INF, CHROMA_NORM_L1, CHROMA_NORM_L2 = range(4)


class DbCfg(Structure):
    _fields_ = [('ref_value', c_float), ('amin', c_float), ('dynamic_range', c_float)]


# every symbol declared in include/kapre_b200.h: (name, restype, argtypes)
SYMBOLS = [
    ('kapre_stft_plan_create', c_int, [c_int, c_int, c_int, c_void_p, POINTER(c_void_p)]),
    ('kapre_stft_plan_destroy', None, [c_void_p]),
    ('kapre_stft_num_frames', c_int, [c_void_p, c_int, c_int, c_int]),
    ('kapre_stft_supports_mode', c_int, [c_void_p, c_int]),
    ('kapre_stft_forward', c_int, [c_void_p, c_void_p, POINTER(WaveDesc), c_int, c_int, c_int, c_void_p,
                                   POINTER(SpecDesc), c_void_p, POINTER(DbCfg), c_void_p, c_void_p]),
    ('kapre_istft_plan_create', c_int, [c_int, c_int, c_int, c_void_p, POINTER(c_void_p)]),
    ('kapre_istft_plan_destroy', None, [c_void_p]),
    ('kapre_istft_inverse', c_int, [c_void_p, c_void_p, c_int, c_int, c_int, POINTER(SpecDesc), c_void_p,
                                    POINTER(WaveDesc), c_void_p]),
    ('kapre_filterbank_create', c_int, [c_void_p, c_int, c_int, POINTER(c_void_p)]),
    ('kapre_filterbank_destroy', None, [c_void_p]),
    ('kapre_apply_filterbank', c_int, [c_void_p, c_void_p, c_int, c_int, c_int, POINTER(SpecDesc), c_void_p,
                                       POINTER(SpecDesc), c_void_p]),
    ('kapre_magnitude', c_int, [c_void_p, c_void_p, c_int64, c_void_p]),
    ('kapre_phase', c_int, [c_void_p, c_void_p, c_int64, c_void_p]),
    ('kapre_magnitude_to_decibel', c_int, [c_void_p, c_void_p, c_int64, c_int64, POINTER(DbCfg), c_void_p, c_void_p]),
    ('kapre_stft_backward_workspace_bytes', c_int64, [c_void_p, c_int, c_int, c_int, c_int, c_int]),
    ('kapre_stft_backward', c_int, [c_void_p, c_void_p, POINTER(SpecDesc), c_int, c_int, c_int, c_int, c_int, c_void_p,
                                    POINTER(WaveDesc), c_void_p, c_void_p]),
    ('kapre_istft_backward', c_int, [c_void_p, c_void_p, POINTER(WaveDesc), c_int, c_int, c_int, c_void_p,
                                     POINTER(SpecDesc), c_void_p]),
    ('kapre_magnitude_backward', c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_void_p]),
    ('kapre_magnitude_to_decibel_backward', c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int64, POINTER(DbCfg),
                                                    c_void_p, c_void_p]),
    ('kapre_phase_backward', c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_void_p]),
    ('kapre_mag_phase_backward', c_int, [c_void_p, POINTER(SpecDesc), c_void_p, POINTER(SpecDesc), c_void_p,
                                         POINTER(SpecDesc), c_void_p, POINTER(SpecDesc), c_int, c_int, c_int, c_int,
                                         c_void_p]),
    ('kapre_delta_backward', c_int, [c_void_p, c_void_p, c_int64, c_int64, c_int64, c_int, c_int, c_void_p]),
    ('kapre_frame_backward', c_int, [c_void_p, POINTER(SpecDesc), c_int, c_int, c_int, c_void_p, POINTER(WaveDesc),
                                     c_void_p]),
    ('kapre_energy_backward', c_int, [c_void_p, POINTER(WaveDesc), c_void_p, POINTER(WaveDesc), c_int, c_int, c_float,
                                      c_void_p, POINTER(WaveDesc), c_void_p]),
    ('kapre_concat_frequency_map_backward', c_int, [c_void_p, c_void_p, c_int64, c_int64, c_int64, c_int64, c_int,
                                                    c_void_p]),
    ('kapre_delta', c_int, [c_void_p, c_void_p, c_int64, c_int64, c_int64, c_int, c_int, c_void_p]),
    ('kapre_frame', c_int, [c_void_p, POINTER(WaveDesc), c_int, c_int, c_int, c_float, c_void_p, POINTER(SpecDesc), c_void_p]),
    ('kapre_energy', c_int, [c_void_p, POINTER(WaveDesc), c_int, c_int, c_int, c_float, c_float, c_void_p, POINTER(WaveDesc), c_void_p]),
    ('kapre_concat_frequency_map', c_int, [c_void_p, c_void_p, c_int64, c_int64, c_int64, c_int64, c_int, c_void_p]),
    ('kapre_spec_augment', c_int, [c_void_p, c_void_p, c_int64, c_int64, c_int64, c_void_p, c_int, c_void_p, c_int, c_float, c_void_p]),
    ('kapre_resample_plan_create', c_int, [c_int, c_int, c_void_p, c_int, POINTER(c_void_p)]),
    ('kapre_resample_plan_destroy', None, [c_void_p]),
    ('kapre_resample_output_length', c_int64, [c_void_p, c_int64]),
    ('kapre_resample', c_int, [c_void_p, c_void_p, POINTER(WaveDesc), c_void_p, POINTER(WaveDesc), c_void_p]),
    ('kapre_resample_backward', c_int, [c_void_p, c_void_p, POINTER(WaveDesc), c_void_p, POINTER(WaveDesc), c_void_p]),
    ('kapre_sinc_plan_create', c_int, [POINTER(c_void_p)]),
    ('kapre_sinc_plan_destroy', None, [c_void_p]),
    ('kapre_sinc_resample', c_int, [c_void_p, c_void_p, POINTER(WaveDesc), c_void_p, POINTER(WaveDesc), ctypes.c_double,
                                    ctypes.c_double, c_void_p]),
    ('kapre_sinc_resample_backward', c_int, [c_void_p, c_void_p, POINTER(WaveDesc), c_void_p, POINTER(WaveDesc),
                                             ctypes.c_double, ctypes.c_double, c_void_p]),
    ('kapre_convolve_block_size', c_int64, [c_int64]),
    ('kapre_convolve_plan_create', c_int, [c_int, POINTER(c_void_p)]),
    ('kapre_convolve_plan_destroy', None, [c_void_p]),
    ('kapre_convolve_ir_spectrum', c_int, [c_void_p, c_void_p, POINTER(WaveDesc), c_void_p, POINTER(SpecDesc), c_void_p]),
    ('kapre_convolve_workspace_bytes', c_int64, [c_void_p, c_int, c_int, c_int, c_int]),
    ('kapre_convolve', c_int, [c_void_p, c_void_p, POINTER(WaveDesc), c_void_p, POINTER(SpecDesc), c_int, c_void_p,
                               POINTER(WaveDesc), c_void_p, c_void_p]),
    ('kapre_convolve_backward_workspace_bytes', c_int64, [c_void_p, c_int, c_int, c_int, c_int]),
    ('kapre_convolve_backward', c_int, [c_void_p, c_void_p, POINTER(WaveDesc), c_void_p, POINTER(SpecDesc), c_void_p,
                                        POINTER(SpecDesc), c_int, c_void_p, POINTER(WaveDesc), c_void_p,
                                        POINTER(SpecDesc), c_void_p, c_void_p]),
    ('kapre_convolve_ir_spectrum_backward', c_int, [c_void_p, c_void_p, POINTER(SpecDesc), c_int, c_void_p,
                                                    POINTER(WaveDesc), c_void_p, c_void_p]),
    ('kapre_lfilter_workspace_bytes', c_int64, [c_int, c_int, c_int, c_int]),
    ('kapre_lfilter', c_int, [c_void_p, POINTER(WaveDesc), POINTER(IirCoeffs), c_int, c_void_p, POINTER(WaveDesc),
                              c_void_p, c_void_p]),
    ('kapre_lfilter_backward', c_int, [c_void_p, POINTER(WaveDesc), c_void_p, POINTER(WaveDesc), c_void_p,
                                       POINTER(WaveDesc), POINTER(IirCoeffs), c_int, c_void_p, POINTER(WaveDesc),
                                       c_void_p, c_void_p, c_void_p]),
    ('kapre_sosfilt_workspace_bytes', c_int64, [c_int, c_int, c_int, c_int]),
    ('kapre_sosfilt', c_int, [c_void_p, POINTER(WaveDesc), POINTER(SosCoeffs), c_void_p, POINTER(SosStateDesc), c_int,
                              c_void_p, POINTER(WaveDesc), c_void_p, POINTER(SosStateDesc), c_void_p, c_void_p]),
    ('kapre_rir_ism', c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_double, c_double, c_int, c_void_p,
                              c_int64, c_int64, c_int64, c_void_p]),
    ('kapre_add_noise_workspace_bytes', c_int64, [c_int, c_int, c_int]),
    ('kapre_add_noise', c_int, [c_void_p, POINTER(WaveDesc), POINTER(NoiseSource), POINTER(SnrDesc), c_void_p,
                                POINTER(WaveDesc), c_void_p, c_void_p, c_void_p]),
    ('kapre_add_noise_backward', c_int, [c_void_p, POINTER(WaveDesc), c_void_p, POINTER(WaveDesc), POINTER(NoiseSource),
                                         POINTER(SnrDesc), c_void_p, c_void_p, POINTER(WaveDesc), c_void_p,
                                         POINTER(WaveDesc), c_void_p, c_void_p, c_void_p]),
    ('kapre_loudness_workspace_bytes', c_int64, [c_int, c_int, c_int, c_int, c_int, POINTER(c_int64)]),
    ('kapre_loudness', c_int, [c_void_p, POINTER(WaveDesc), c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p,
                               c_void_p]),
    ('kapre_loudness_backward', c_int, [c_void_p, c_void_p, POINTER(WaveDesc), c_void_p, c_int, c_int, c_void_p,
                                        c_void_p, POINTER(WaveDesc), c_void_p]),
    ('kapre_loudness_stats_workspace_bytes', c_int64, [c_int, c_int, c_int, c_int, c_int, c_int]),
    ('kapre_loudness_stats', c_int, [c_void_p, POINTER(WaveDesc), c_void_p, c_int, c_int, c_int, c_void_p, c_void_p,
                                     c_void_p, c_void_p, c_void_p, c_void_p]),
    ('kapre_true_peak_workspace_bytes', c_int64, [c_int, c_int, c_int, POINTER(c_int64)]),
    ('kapre_true_peak', c_int, [c_void_p, POINTER(WaveDesc), c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                c_void_p]),
    ('kapre_true_peak_backward', c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, POINTER(WaveDesc),
                                         c_void_p]),
    ('kapre_kaldi_plan_create', c_int, [POINTER(KaldiCfg), c_void_p, c_void_p, c_void_p, POINTER(c_void_p)]),
    ('kapre_kaldi_plan_destroy', None, [c_void_p]),
    ('kapre_kaldi_num_frames', c_int, [c_void_p, c_int]),
    ('kapre_kaldi_num_bins', c_int, [c_void_p]),
    ('kapre_kaldi_workspace_bytes', c_int64, [c_void_p, c_int, c_int, c_int, c_int]),
    ('kapre_kaldi_features', c_int, [c_void_p, c_void_p, POINTER(WaveDesc), c_void_p, c_void_p, c_int, c_float, c_uint64,
                                     c_void_p, POINTER(SpecDesc), c_void_p, c_void_p]),
    ('kapre_kaldi_features_backward', c_int, [c_void_p, c_void_p, POINTER(SpecDesc), c_void_p, POINTER(WaveDesc),
                                              c_void_p, c_void_p, c_int, c_float, c_uint64, c_void_p,
                                              POINTER(WaveDesc), c_void_p, c_void_p]),
    ('kapre_cqt_plan_create', c_int, [POINTER(CqtCfg), c_void_p, c_void_p, c_int, POINTER(c_void_p)]),
    ('kapre_cqt_plan_destroy', None, [c_void_p]),
    ('kapre_cqt_num_frames', c_int, [c_void_p, c_int]),
    ('kapre_cqt_workspace_bytes', c_int64, [c_void_p, c_int, c_int, c_int, c_int]),
    ('kapre_cqt', c_int, [c_void_p, c_void_p, POINTER(WaveDesc), c_int, c_void_p, POINTER(SpecDesc), c_void_p, c_void_p]),
    ('kapre_cqt_backward', c_int, [c_void_p, c_void_p, POINTER(WaveDesc), c_void_p, c_void_p, POINTER(SpecDesc), c_int,
                                   c_void_p, POINTER(WaveDesc), c_void_p, c_void_p]),
    ('kapre_pitch_plan_create', c_int, [POINTER(PitchCfg), POINTER(PitchTables), POINTER(c_void_p)]),
    ('kapre_pitch_plan_destroy', None, [c_void_p]),
    ('kapre_pitch_num_frames', c_int, [c_void_p, c_int]),
    ('kapre_pitch_workspace_bytes', c_int64, [c_void_p, c_int, c_int, c_int]),
    ('kapre_yin', c_int, [c_void_p, c_void_p, POINTER(WaveDesc), c_void_p, POINTER(FramesDesc), c_void_p,
                          POINTER(SpecDesc), c_void_p]),
    ('kapre_pyin', c_int, [c_void_p, c_void_p, POINTER(WaveDesc), c_void_p, c_void_p, c_void_p, POINTER(FramesDesc),
                           c_void_p, POINTER(SpecDesc), c_void_p, c_void_p]),
    ('kapre_chroma_plan_create', c_int, [POINTER(ChromaPlanDesc), POINTER(c_void_p)]),
    ('kapre_chroma_plan_destroy', None, [c_void_p]),
    ('kapre_chroma', c_int, [c_void_p, POINTER(ChromaCfg), c_void_p, POINTER(SpecDesc), c_int, c_int, c_int, c_void_p,
                             c_void_p, POINTER(SpecDesc), c_void_p]),
    ('kapre_chroma_backward', c_int, [c_void_p, POINTER(ChromaCfg), c_void_p, POINTER(SpecDesc), c_int, c_int, c_int,
                                      c_void_p, c_void_p, POINTER(SpecDesc), c_void_p, POINTER(SpecDesc), c_void_p]),
    ('kapre_chroma_cens_workspace_bytes', c_int64, [c_void_p, c_int, c_int, c_int]),
    ('kapre_chroma_cens', c_int, [c_void_p, c_int, c_void_p, POINTER(SpecDesc), c_int, c_int, c_int, c_void_p,
                                  POINTER(SpecDesc), c_void_p, c_void_p]),
    ('kapre_chroma_tuning_workspace_bytes', c_int64, [c_void_p, c_int, c_int, c_int]),
    ('kapre_chroma_tuning', c_int, [c_void_p, c_int, c_void_p, POINTER(SpecDesc), c_int, c_int, c_int, c_void_p,
                                    c_void_p, c_void_p, c_void_p]),
    ('kapre_hpss', c_int, [POINTER(HpssCfg), c_void_p, c_int, POINTER(SpecDesc), c_int, c_int, c_int, c_int, c_void_p,
                           POINTER(SpecDesc), c_void_p, POINTER(SpecDesc), c_void_p]),
    ('kapre_hpss_workspace_bytes', c_int64, [c_int, c_int, c_int, c_int]),
    ('kapre_hpss_backward', c_int, [POINTER(HpssCfg), c_void_p, c_int, POINTER(SpecDesc), c_int, c_int, c_int, c_int,
                                    c_void_p, POINTER(SpecDesc), c_void_p, POINTER(SpecDesc), c_void_p,
                                    POINTER(SpecDesc), c_void_p, c_void_p]),
    ('kapre_onset_strength', c_int, [POINTER(OnsetCfg), c_void_p, POINTER(SpecDesc), c_int, c_int, c_int, c_int,
                                     c_void_p, POINTER(FramesDesc), c_void_p]),
    ('kapre_onset_strength_workspace_bytes', c_int64, [c_int, c_int, c_int, c_int]),
    ('kapre_onset_strength_backward', c_int, [POINTER(OnsetCfg), c_void_p, POINTER(SpecDesc), c_int, c_int, c_int,
                                              c_int, c_void_p, POINTER(FramesDesc), c_void_p, POINTER(SpecDesc),
                                              c_void_p, c_void_p]),
    ('kapre_tempogram', c_int, [c_void_p, POINTER(FramesDesc), c_int, c_int, c_int, c_int, c_int, c_int, c_void_p,
                                POINTER(SpecDesc), c_void_p]),
    ('kapre_tempo_workspace_bytes', c_int64, [c_int, c_int, c_int, c_int]),
    ('kapre_tempo', c_int, [c_void_p, POINTER(SpecDesc), c_int, c_int, c_int, c_int, c_void_p, ctypes.c_double, c_int,
                            c_void_p, POINTER(FramesDesc), c_void_p, c_void_p]),
    ('kapre_onset_detect', c_int, [c_void_p, POINTER(FramesDesc), c_int, c_int, c_int, POINTER(OnsetDetectCfg),
                                   c_void_p, POINTER(FramesDesc), c_void_p]),
    ('kapre_beat_track_workspace_bytes', c_int64, [c_int, c_int, c_int]),
    ('kapre_beat_track', c_int, [c_void_p, POINTER(FramesDesc), c_int, c_int, c_int, POINTER(BeatCfg), c_void_p,
                                 c_float, c_void_p, c_void_p, POINTER(FramesDesc), c_void_p, c_void_p]),
    ('kapre_pcen_workspace', c_int, [c_int, c_int, c_int, c_int, POINTER(c_int), POINTER(c_int64)]),
    ('kapre_pcen', c_int, [c_void_p, POINTER(SpecDesc), c_int, c_int, c_int, c_int, POINTER(PcenParams), c_void_p,
                           POINTER(SpecDesc), c_void_p, POINTER(SpecDesc), c_void_p, c_void_p]),
    ('kapre_pcen_backward', c_int, [c_void_p, POINTER(SpecDesc), c_void_p, POINTER(SpecDesc), c_void_p, POINTER(SpecDesc),
                                    c_int, c_int, c_int, c_int, POINTER(PcenParams), c_void_p, POINTER(SpecDesc),
                                    c_void_p, c_void_p, c_void_p]),
    ('kapre_griffin_lim_workspace_bytes', c_int64, [c_void_p, c_int, c_int, c_int]),
    ('kapre_griffin_lim', c_int, [c_void_p, c_void_p, c_void_p, POINTER(SpecDesc), c_int, c_int, c_int, POINTER(GlCfg),
                                  c_void_p, POINTER(WaveDesc), c_void_p, c_void_p]),
    ('kapre_time_stretch_workspace', c_int, [c_int, c_int, c_int, c_int, ctypes.c_double, POINTER(c_int),
                                             POINTER(c_int64)]),
    ('kapre_time_stretch', c_int, [c_void_p, POINTER(SpecDesc), c_int, c_int, c_int, c_int, ctypes.c_double, c_void_p,
                                   POINTER(SpecDesc), c_void_p, c_void_p]),
    ('kapre_time_stretch_backward', c_int, [c_void_p, POINTER(SpecDesc), c_void_p, POINTER(SpecDesc), c_void_p,
                                            POINTER(SpecDesc), c_int, c_int, c_int, c_int, ctypes.c_double, c_void_p,
                                            POINTER(SpecDesc), c_void_p, c_void_p]),
    ('kapre_fb_inverse_plan_create', c_int, [c_void_p, c_int, c_int, POINTER(c_void_p)]),
    ('kapre_fb_inverse_plan_destroy', None, [c_void_p]),
    ('kapre_filterbank_invert', c_int, [c_void_p, POINTER(FbInvCfg), c_void_p, c_int, c_int, c_int, POINTER(SpecDesc),
                                        c_void_p, POINTER(SpecDesc), c_void_p]),
    ('kapre_last_error', c_char_p, []),
    ('kapre_version', c_int, []),
    ('kapre_launch_count', c_uint64, []),
    ('kapre_last_launch_info', c_char_p, []),
    ('kapre_profile_enable', c_int, [c_int]),
    ('kapre_profile_read', c_int, [POINTER(ctypes.c_double), POINTER(c_uint64)]),
    ('kapre_tc_set_debug', c_int, [c_void_p]),
    ('kapre_tc_dft_stage1', c_int, [c_void_p, c_int, c_int64, c_int, c_void_p, c_int, POINTER(c_int), c_void_p, c_void_p]),
]

_lib = None


def lib():
    """Load (once) and return the shared library; raise loudly if it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise KapreNativeError(
                'kapre_b200: CUDA library %s not found.  Build it with '
                '`python -c "import __graft_entry__ as g; g.build()"` (nvcc, sm_90a).  '
                'There is no CPU or PyTorch fallback.' % LIB_PATH)
        handle = ctypes.CDLL(LIB_PATH)
        for name, restype, argtypes in SYMBOLS:
            fn = getattr(handle, name)  # AttributeError if the ABI and the header drifted apart
            fn.restype = restype
            fn.argtypes = argtypes
        _lib = handle
    return _lib


def check(rc: int):
    if rc != 0:
        msg = lib().kapre_last_error()
        raise KapreNativeError('kapre_b200 error %d: %s' % (rc, msg.decode() if msg else '?'))


def launch_count() -> int:
    return int(lib().kapre_launch_count())


def last_launch_info() -> str:
    s = lib().kapre_last_launch_info()
    return s.decode() if s else ''


def profile_enable(on, every: int = 1):
    """Bracket every `every`-th launch of the dominant kernels with CUDA events (0 / False: off)."""
    lib().kapre_profile_enable(int(every) if on else 0)


def profile_read():
    """(total kernel milliseconds, launches) recorded since the last read."""
    ms, n = ctypes.c_double(0.0), c_uint64(0)
    lib().kapre_profile_read(ctypes.byref(ms), ctypes.byref(n))
    return float(ms.value), int(n.value)
