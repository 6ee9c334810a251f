"""ctypes binding of ``libb2l.so`` (C ABI declared in ``include/b2l.h``).

No PyTorch, no CuPy: device memory, streams and launches all live behind the C ABI.  There is no
CPU fallback — if the shared library is missing or no sm_90 GPU is present, every entry point raises.
"""
from __future__ import annotations

import ctypes as C
import math
import os
import threading
import weakref
from typing import Optional, Tuple

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
# B2L_LIB_PATH loads another build of the same C ABI (another flavour or revision, to compare outputs and timings);
# there is still no fallback.
LIB_PATH = os.environ.get("B2L_LIB_PATH") or os.path.join(_HERE, "csrc", "libb2l.so")

B2L_OK = 0
B2L_ERR_INVALID = 1
B2L_ERR_CUDA = 2
B2L_ERR_UNSUPPORTED = 3
B2L_ERR_OOM = 4
B2L_ERR_NCCL = 5

PAD_MODES = {"constant": 0, "edge": 1, "reflect": 2, "symmetric": 3, "linear_ramp": 4, "empty": 5}


class NativeLibraryError(RuntimeError):
    """libb2l.so is missing / failed, or a CUDA / NCCL call failed."""


class UnsupportedOnGPU(NotImplementedError):
    """Valid for librosa but not built for the sm_90a path yet (never a silent CPU fallback)."""


class PlanDesc(C.Structure):
    """struct b2l_plan_desc (include/b2l.h)."""
    _fields_ = [
        ("n_fft", C.c_int32),
        ("hop_length", C.c_int32),
        ("center", C.c_int32),
        ("pad_mode", C.c_int32),
        ("h_window", C.POINTER(C.c_double)),
        ("n_mels", C.c_int32),
        ("h_mel_basis", C.POINTER(C.c_float)),
        ("power", C.c_float),
        ("n_mfcc", C.c_int32),
        ("h_dct_basis", C.POINTER(C.c_float)),
        ("amin", C.c_float),
        ("ref_value", C.c_float),
        ("top_db", C.c_float),
    ]


class StatsDesc(C.Structure):
    """struct b2l_stats_desc (include/b2l.h)."""
    _fields_ = [
        ("roll_percent", C.c_float),
        ("flat_amin", C.c_float),
        ("flat_power", C.c_float),
        ("bw_p", C.c_float),
        ("bw_norm", C.c_int32),
        ("frame_length", C.c_int32),
        ("want", C.c_int32),
    ]


class OnsetDesc(C.Structure):
    """struct b2l_onset_desc (include/b2l.h)."""
    _fields_ = [
        ("lag", C.c_int32),
        ("max_size", C.c_int32),
        ("pad_width", C.c_int32),
        ("detrend", C.c_int32),
        ("n_channels", C.c_int32),
        ("bounds", C.c_int32 * 33),
    ]


class PcenDesc(C.Structure):
    """struct b2l_pcen_desc (include/b2l.h)."""
    _fields_ = [("gain", C.c_float), ("bias", C.c_float), ("power", C.c_float), ("eps", C.c_float), ("b", C.c_float),
                ("max_size", C.c_int32)]


class ContrastDesc(C.Structure):
    """struct b2l_contrast_desc (include/b2l.h)."""
    _fields_ = [("n_bands", C.c_int32), ("lo", C.c_int32 * 16), ("count", C.c_int32 * 16), ("k", C.c_int32 * 16)]


class PipDesc(C.Structure):
    """struct b2l_pip_desc (include/b2l.h)."""
    _fields_ = [("k_lo", C.c_int32), ("k_hi", C.c_int32), ("threshold", C.c_double), ("thr_wide", C.c_int32),
                ("ref_abs", C.c_double), ("sr", C.c_double), ("n_fft", C.c_double), ("mode", C.c_int32), ("prefix", C.c_uint32), ("mag_threshold", C.c_float),
                ("bins_per_octave", C.c_float), ("n_res_bins", C.c_int32)]


class HpssDesc(C.Structure):
    """struct b2l_hpss_desc (include/b2l.h)."""
    _fields_ = [("win_harm", C.c_int32), ("win_perc", C.c_int32), ("margin_harm", C.c_float),
                ("margin_perc", C.c_float), ("power", C.c_float), ("mask_only", C.c_int32)]


class ReassignDesc(C.Structure):
    """struct b2l_reassign_desc (include/b2l.h)."""
    _fields_ = [("sr", C.c_float), ("mag_threshold", C.c_float), ("max_time", C.c_float),
                ("reassign_frequencies", C.c_int32), ("reassign_times", C.c_int32), ("apply_threshold", C.c_int32),
                ("fill_nan", C.c_int32), ("clip", C.c_int32)]


class YinDesc(C.Structure):
    """struct b2l_yin_desc (include/b2l.h)."""
    _fields_ = [("frame_length", C.c_int32), ("hop_length", C.c_int32), ("center", C.c_int32), ("pad_mode", C.c_int32),
                ("min_period", C.c_int32), ("max_period", C.c_int32), ("sr", C.c_double), ("trough_threshold", C.c_double)]


class PyinDesc(C.Structure):
    """struct b2l_pyin_desc (include/b2l.h); the d_* fields are device pointers."""
    _fields_ = [("min_period", C.c_int32), ("max_period", C.c_int32), ("n_thresholds", C.c_int32),
                ("n_pitch_bins", C.c_int32), ("n_bins_per_semitone", C.c_int32), ("sr", C.c_double),
                ("fmin", C.c_double), ("no_trough_prob", C.c_double), ("d_thresholds", C.c_void_p),
                ("d_beta", C.c_void_p), ("d_beta_cum", C.c_void_p), ("d_pmf", C.c_void_p), ("log_p_init", C.c_double),
                ("fill_na", C.c_double), ("fill", C.c_int32), ("half_width", C.c_int32), ("full", C.c_int32),
                ("log_thr", C.c_double), ("d_cls", C.c_void_p), ("d_ltab", C.c_void_p), ("d_freqs", C.c_void_p)]


class TempogramDesc(C.Structure):
    """struct b2l_tempogram_desc (include/b2l.h)."""
    _fields_ = [("win_length", C.c_int32), ("center", C.c_int32), ("norm", C.c_int32), ("env_f64", C.c_int32),
                ("norm_p", C.c_double)]


class TempoDesc(C.Structure):
    """struct b2l_tempo_desc (include/b2l.h)."""
    _fields_ = [("n_lags", C.c_int32), ("mean", C.c_int32), ("tg_f64", C.c_int32), ("n_frames", C.c_int64),
                ("row_stride", C.c_int64), ("lag_stride", C.c_int64), ("frame_stride", C.c_int64)]


class BeatDesc(C.Structure):
    """struct b2l_beat_desc (include/b2l.h); the d_* fields are device pointers."""
    _fields_ = [("n_fpb", C.c_int32), ("env_f64", C.c_int32), ("dp_f64", C.c_int32), ("trim", C.c_int32),
                ("units", C.c_int32),
                ("tightness", C.c_float), ("hop_length", C.c_int32), ("sr", C.c_double), ("d_fpb", C.c_void_p),
                ("d_logfpb", C.c_void_p), ("d_woff", C.c_void_p), ("d_wtab", C.c_void_p), ("d_logd", C.c_void_p)]


class PlpDesc(C.Structure):
    """struct b2l_plp_desc (include/b2l.h); the d_* fields are device pointers."""
    _fields_ = [("n_bins", C.c_int32), ("c128", C.c_int32), ("sqrt_tiny", C.c_double), ("d_keep", C.c_void_p),
                ("d_logprior", C.c_void_p)]


class PeakDesc(C.Structure):
    """struct b2l_peak_desc (include/b2l.h)."""
    _fields_ = [("pre_max", C.c_int64), ("post_max", C.c_int64), ("pre_avg", C.c_int64), ("post_avg", C.c_int64),
                ("wait", C.c_int64), ("delta", C.c_double), ("method", C.c_int32), ("f64", C.c_int32),
                ("units", C.c_int32), ("hop_length", C.c_int32), ("sr", C.c_double)]


class SeqLogObsDesc(C.Structure):
    """struct b2l_seq_logobs_desc (include/b2l.h); d_log_marginal is a device pointer."""
    _fields_ = [("mode", C.c_int32), ("f64", C.c_int32), ("n_clips", C.c_int64), ("n_states", C.c_int64),
                ("n_steps", C.c_int64), ("eps", C.c_double), ("d_log_marginal", C.c_void_p)]


class SeqModel(C.Structure):
    """struct b2l_seq_model (include/b2l.h); the d_* fields are device pointers."""
    _fields_ = [("n_states", C.c_int32), ("n_models", C.c_int32), ("deg", C.c_int32), ("dense", C.c_int32),
                ("d_lt", C.c_void_p), ("d_idx", C.c_void_p), ("d_log_p_init", C.c_void_p)]


class DtwCostDesc(C.Structure):
    """struct b2l_dtw_cost_desc (include/b2l.h); the h_* fields are host pointers."""
    _fields_ = [("f64", C.c_int32), ("metric", C.c_int32), ("transpose", C.c_int32), ("K", C.c_int64),
                ("N", C.c_int64), ("M", C.c_int64), ("h_x_off", C.c_void_p), ("h_y_off", C.c_void_p)]


class DtwDesc(C.Structure):
    """struct b2l_dtw_desc (include/b2l.h); the h_* fields are host pointers."""
    _fields_ = [("n", C.c_int64), ("m", C.c_int64), ("c_f64", C.c_int32), ("n_steps", C.c_int32),
                ("subseq", C.c_int32), ("band", C.c_int32), ("band_lo", C.c_int64), ("band_hi", C.c_int64),
                ("h_steps", C.c_void_p), ("h_w_add", C.c_void_p), ("h_w_mul", C.c_void_p)]


class CqtOctave(C.Structure):
    """struct b2l_cqt_octave (include/b2l.h): one octave of b2l_cqt_project / b2l_cqt_project_abs; d_D is a device
    pointer."""
    _fields_ = [("d_D", C.c_void_p), ("n_frames", C.c_int64), ("n_fft_bins", C.c_int32), ("row0", C.c_int32),
                ("n_rows", C.c_int32), ("indptr_off", C.c_int32), ("nnz", C.c_int32), ("kind", C.c_int32)]


CQT_MAX_OCTAVES = 32   # B2L_CQT_MAX_OCTAVES
CQT_FULL, CQT_PSEUDO, CQT_DIVIDE = 0, 1, 0x10   # B2L_CQT_FULL / B2L_CQT_PSEUDO / B2L_CQT_DIVIDE


class IirtRate(C.Structure):
    """struct b2l_iirt_rate (include/b2l.h): the chains of one sampling rate of b2l_iirt_filter / b2l_iirt_stmsp;
    the d_* fields are device pointers."""
    _fields_ = [("d_x", C.c_void_p), ("x_stride", C.c_int64), ("n", C.c_int64), ("d_scratch", C.c_void_p),
                ("scratch_stride", C.c_int64), ("d_bands", C.c_void_p), ("n_bands", C.c_int32),
                ("n_leaves", C.c_int32), ("d_starts", C.c_void_p), ("d_leaves", C.c_void_p), ("factor", C.c_double)]


IIRT_MAX_SECTIONS, IIRT_MAX_RATES, IIRT_MAX_DEPTH = 10, 16, 32   # B2L_IIRT_MAX_SECTIONS / _RATES / _DEPTH


class PiptrackDesc(C.Structure):
    """struct b2l_piptrack_desc (include/b2l.h)."""
    _fields_ = [("f64", C.c_int32), ("layout_c", C.c_int32), ("k_lo", C.c_int32), ("k_hi", C.c_int32),
                ("abs_mode", C.c_int32), ("ref_frame", C.c_int32), ("thr_wide", C.c_int32), ("pad_", C.c_int32),
                ("threshold", C.c_double), ("ref_abs", C.c_double), ("sr", C.c_double), ("n_fft", C.c_double)]


PIPTRACK_MAX_ROW_BYTES = 200 * 1024   # B2L_PIPTRACK_MAX_ROW_BYTES
(ELEM_I8, ELEM_U8, ELEM_I16, ELEM_U16, ELEM_I32, ELEM_U32, ELEM_I64, ELEM_U64, ELEM_F32, ELEM_F64,
 ELEM_BOOL) = range(11)   # enum b2l_elem_type: the element types of b2l_localext
ELEM_TYPES = {np.dtype(t): i for i, t in enumerate((np.int8, np.uint8, np.int16, np.uint16, np.int32, np.uint32,
                                                     np.int64, np.uint64, np.float32, np.float64, np.bool_))}


class DeltaDesc(C.Structure):
    """struct b2l_delta_desc (include/b2l.h); the d_* fields are device pointers."""
    _fields_ = [("width", C.c_int32), ("sym", C.c_int32), ("interp", C.c_int32), ("f64", C.c_int32),
                ("cval", C.c_double), ("d_taps", C.c_void_p), ("d_edge", C.c_void_p), ("d_pad", C.c_void_p)]


class StackDesc(C.Structure):
    """struct b2l_stack_desc (include/b2l.h)."""
    _fields_ = [("elem_size", C.c_int32), ("n_steps", C.c_int32), ("delay", C.c_int64), ("clip_stride", C.c_int64),
                ("row_stride", C.c_int64), ("col_stride", C.c_int64), ("fill", C.c_uint8 * 16)]


DELTA_MAX_WIDTH = 255   # B2L_DELTA_MAX_WIDTH


class ChromaDesc(C.Structure):
    """struct b2l_chroma_desc (include/b2l.h): one b2l_chroma_fold; the d_* fields are device pointers."""
    _fields_ = [("input", C.c_int32), ("out_f64", C.c_int32), ("n_bins", C.c_int32), ("n_chroma", C.c_int32),
                ("nnz", C.c_int32), ("norm", C.c_int32), ("norm_p", C.c_double), ("has_threshold", C.c_int32),
                ("epilogue", C.c_int32), ("threshold", C.c_double), ("post_norm", C.c_int32), ("pad_", C.c_int32),
                ("post_p", C.c_double), ("d_row_ptr", C.c_void_p), ("d_cols", C.c_void_p), ("d_weights", C.c_void_p),
                ("d_phi", C.c_void_p)]


CHROMA_IN_C64_FT, CHROMA_IN_F32_FT, CHROMA_IN_F32_C, CHROMA_IN_F64_FT, CHROMA_IN_F64_C = range(5)   # enum b2l_chroma_input
CHROMA_NORM_NONE, CHROMA_NORM_INF, CHROMA_NORM_NEG_INF, CHROMA_NORM_ZERO, CHROMA_NORM_P = range(5)   # enum b2l_chroma_norm
CHROMA_PLAIN, CHROMA_CENS, CHROMA_TONNETZ = range(3)   # enum b2l_chroma_epilogue


class NnDesc(C.Structure):
    """struct b2l_nn_desc (include/b2l.h)."""
    _fields_ = [("metric", C.c_int32), ("mode", C.c_int32), ("k", C.c_int32), ("width", C.c_int32),
                ("n_cand", C.c_int32), ("sym", C.c_int32), ("self_link", C.c_int32), ("f64", C.c_int32),
                ("bw_mode", C.c_int32), ("src_f64", C.c_int32), ("bandwidth", C.c_double), ("n_lead", C.c_int64),
                ("n_feat", C.c_int64), ("lead_stride", C.c_int64), ("feat_stride", C.c_int64),
                ("frame_stride", C.c_int64)]


class NnFilterDesc(C.Structure):
    """struct b2l_nn_filter_desc (include/b2l.h)."""
    _fields_ = [("agg", C.c_int32), ("s_f64", C.c_int32), ("r_f64", C.c_int32), ("max_count", C.c_int32),
                ("stride", C.c_int64)]


NN_MAX_FRAMES, NN_MAX_CANDIDATES, NN_MAX_STATS = 65536, 4096, 256   # B2L_NN_MAX_FRAMES / _CANDIDATES / _STATS
NN_EUCLIDEAN, NN_COSINE = 0, 1                                         # enum b2l_nn_metric
NN_METRICS = {"euclidean": NN_EUCLIDEAN, "cosine": NN_COSINE}
(NN_BW_SCALAR, NN_BW_MEAN_K, NN_BW_GMEAN_K, NN_BW_MEAN_K_AVG, NN_BW_GMEAN_K_AVG, NN_BW_MEAN_K_AVG_AND_PAIR,
 NN_BW_MED_K_SCALAR) = range(7)                                        # enum b2l_nn_bandwidth
NN_BANDWIDTHS = {"mean_k": NN_BW_MEAN_K, "gmean_k": NN_BW_GMEAN_K, "mean_k_avg": NN_BW_MEAN_K_AVG,
                 "gmean_k_avg": NN_BW_GMEAN_K_AVG, "mean_k_avg_and_pair": NN_BW_MEAN_K_AVG_AND_PAIR,
                 "med_k_scalar": NN_BW_MED_K_SCALAR}
NN_MEAN, NN_MEDIAN, NN_AVERAGE = range(3)                              # enum b2l_nn_aggregate


DTW_METRICS = {"euclidean": 0, "sqeuclidean": 1, "cityblock": 2, "chebyshev": 3, "cosine": 4}   # enum b2l_dtw_metric
BEAT_FRAMES, BEAT_SAMPLES, BEAT_TIME = range(3)   # enum b2l_beat_units
SEQ_PLAIN, SEQ_DISC, SEQ_BINARY = range(3)        # enum b2l_seq_mode
SEQ_SMALL, SEQ_MEDIUM, SEQ_LARGE = range(3)       # enum b2l_seq_class
PEAK_GREEDY, PEAK_DP_COUNT, PEAK_DP_VALUE = range(3)   # enum b2l_peak_method
TG_NORM_NONE, TG_NORM_MAX, TG_NORM_MIN, TG_NORM_COUNT, TG_NORM_P = range(5)   # enum b2l_tempogram_norm
N_STATS = 6
STAT_CENTROID, STAT_BANDWIDTH, STAT_ROLLOFF, STAT_FLATNESS, STAT_RMS, STAT_TOTAL = range(6)
FRAME_RMS, FRAME_ZERO_CROSSINGS = 0, 1
UNARY_SQUARE, UNARY_DB_TO_POWER, UNARY_DB_TO_AMPLITUDE = 0, 1, 2
STATUS_NOT_FINITE_SAMPLE, STATUS_NEGATIVE_ENTRY, STATUS_NOT_FINITE_VALUE, STATUS_NEGATIVE_EVENT = 1, 2, 4, 8   # enum b2l_status_bit

_lib = None
_lib_lock = threading.Lock()

_vp = C.c_void_p
_i64 = C.c_int64


def _declare(lib):
    P = C.POINTER
    sig = {
        "b2l_version": (C.c_int, []),
        "b2l_last_error": (C.c_char_p, []),
        "b2l_device_count": (C.c_int, [P(C.c_int)]),
        "b2l_ctx_create": (C.c_int, [C.c_int, P(_vp)]),
        "b2l_ctx_destroy": (C.c_int, [_vp]),
        "b2l_ctx_sync": (C.c_int, [_vp]),
        "b2l_ctx_device": (C.c_int, [_vp, P(C.c_int)]),
        "b2l_ctx_sm_count": (C.c_int, [_vp, P(C.c_int)]),
        "b2l_ctx_launch_count": (C.c_int, [_vp, P(C.c_uint64)]),
        "b2l_status_reset": (C.c_int, [_vp]),
        "b2l_status_read": (C.c_int, [_vp, P(C.c_int)]),
        "b2l_scan_finite": (C.c_int, [_vp, _vp, _i64, _i64, _i64, _i64]),
        "b2l_scan_finite_f64": (C.c_int, [_vp, _vp, _i64, _i64, _i64, _i64]),
        "b2l_alloc": (C.c_int, [_vp, C.c_size_t, P(_vp)]),
        "b2l_free": (C.c_int, [_vp, _vp]),
        "b2l_memset": (C.c_int, [_vp, _vp, C.c_int, C.c_size_t]),
        "b2l_h2d": (C.c_int, [_vp, _vp, _vp, C.c_size_t]),
        "b2l_d2h": (C.c_int, [_vp, _vp, _vp, C.c_size_t]),
        "b2l_d2d": (C.c_int, [_vp, _vp, _vp, C.c_size_t]),
        "b2l_copy2d": (C.c_int, [_vp, _vp, C.c_size_t, _vp, C.c_size_t, C.c_size_t, C.c_size_t]),
        "b2l_host_alloc": (C.c_int, [C.c_size_t, P(_vp)]),
        "b2l_host_free": (C.c_int, [_vp]),
        "b2l_mem_info": (C.c_int, [_vp, P(C.c_size_t), P(C.c_size_t)]),
        "b2l_event_create": (C.c_int, [_vp, P(_vp)]),
        "b2l_event_record": (C.c_int, [_vp, _vp]),
        "b2l_event_elapsed_ms": (C.c_int, [_vp, _vp, P(C.c_float)]),
        "b2l_event_destroy": (C.c_int, [_vp]),
        "b2l_plan_create": (C.c_int, [_vp, P(PlanDesc), P(_vp)]),
        "b2l_plan_destroy": (C.c_int, [_vp]),
        "b2l_plan_n_frames": (C.c_int, [_vp, _i64, P(_i64)]),
        "b2l_stft": (C.c_int, [_vp, _vp, _vp, _i64, _i64, _i64, _vp]),
        "b2l_spectrogram": (C.c_int, [_vp, _vp, _vp, _i64, _i64, _i64, _vp]),
        "b2l_melspectrogram": (C.c_int, [_vp, _vp, _vp, _i64, _i64, _i64, _vp]),
        "b2l_mfcc": (C.c_int, [_vp, _vp, _vp, _i64, _i64, _i64, _vp, _vp]),
        "b2l_istft": (C.c_int, [_vp, _vp, _vp, _i64, _i64, _i64, _vp, _i64, _vp, _i64]),
        "b2l_mel_project": (C.c_int, [_vp, _vp, _vp, _i64, _i64, _vp]),
        "b2l_power_to_db": (C.c_int, [_vp, _vp, _i64, _i64, C.c_float, C.c_float, C.c_float, _vp]),
        "b2l_onset_from_spec": (C.c_int, [_vp, P(OnsetDesc), _vp, _i64, _i64, _i64, _vp]),
        "b2l_onset_median_from_spec": (C.c_int, [_vp, P(OnsetDesc), _vp, _i64, _i64, _i64, _vp]),
        "b2l_pcen": (C.c_int, [_vp, P(PcenDesc), _vp, _i64, _i64, _i64, _vp, _vp, _vp, _vp]),
        "b2l_resample_poly": (C.c_int, [_vp, _vp, _i64, _i64, _i64, _vp, C.c_int32, C.c_int32, C.c_int32, _i64, _i64, _i64,
                                        C.c_float, _vp]),
        "b2l_spectral_contrast": (C.c_int, [_vp, P(ContrastDesc), _vp, _i64, _i64, C.c_int32, _vp, _vp]),
        "b2l_sub": (C.c_int, [_vp, _vp, _vp, _i64, _vp]),
        "b2l_pip_pass": (C.c_int, [_vp, P(PipDesc), _vp, _i64, C.c_int32, _vp, _vp]),
        "b2l_normalize_rows": (C.c_int, [_vp, _vp, _i64, _i64, _i64, C.c_int32, C.c_double, _vp]),
        "b2l_hpss": (C.c_int, [_vp, P(HpssDesc), _vp, _vp, _i64, _i64, _i64, _vp, _vp]),
        "b2l_cabs": (C.c_int, [_vp, _vp, _i64, _vp]),
        "b2l_reassign": (C.c_int, [_vp, P(ReassignDesc), _vp, _vp, _vp, _i64, _i64, _i64, _vp, _vp, _vp, _vp, _vp]),
        "b2l_phase_vocoder": (C.c_int, [_vp, _vp, _i64, _i64, _i64, _i64, _vp, _vp, _vp, _vp, _vp]),
        "b2l_unary": (C.c_int, [_vp, C.c_int32, _vp, _i64, C.c_float, _vp]),
        "b2l_dct_project": (C.c_int, [_vp, _vp, _vp, _i64, _i64, _vp]),
        "b2l_transpose": (C.c_int, [_vp, _vp, _i64, _i64, _i64, C.c_int32, _vp]),
        "b2l_gl_update": (C.c_int, [_vp, _vp, _vp, _vp, C.c_float, C.c_float, _vp, _i64]),
        "b2l_spectral_stats": (C.c_int, [_vp, _vp, P(StatsDesc), _vp, _i64, _i64, _i64, _vp, _vp]),
        "b2l_spectral_stats_from_spec": (C.c_int, [_vp, P(StatsDesc), _vp, _i64, _i64, C.c_int32, _vp, _vp]),
        "b2l_frame_feature": (C.c_int, [_vp, C.c_int32, _vp, _i64, _i64, _i64, C.c_int32, C.c_int32, C.c_int32,
                                        C.c_int32, C.c_float, C.c_int32, C.c_int32, C.c_float, _vp]),
        "b2l_yin_cmnd": (C.c_int, [_vp, P(YinDesc), _vp, _i64, _i64, _i64, _vp]),
        "b2l_yin_pick": (C.c_int, [_vp, P(YinDesc), _vp, _i64, _vp]),
        "b2l_pyin_obs": (C.c_int, [_vp, P(PyinDesc), _vp, _i64, _vp, _vp, _vp, _vp]),
        "b2l_viterbi": (C.c_int, [_vp, P(PyinDesc), _vp, _vp, _vp, _vp, _i64, _i64, _vp, _vp, _vp]),
        "b2l_piptrack": (C.c_int, [_vp, P(PiptrackDesc), _vp, _i64, C.c_int32, _i64, _vp, _vp]),
        "b2l_pitch_tuning": (C.c_int, [_vp, _vp, _i64, C.c_int32, C.c_double, C.c_int32, _vp, _vp]),
        "b2l_tempogram": (C.c_int, [_vp, P(TempogramDesc), _vp, _i64, _i64, _vp, _vp]),
        "b2l_tempo": (C.c_int, [_vp, P(TempoDesc), _vp, _i64, _vp, _vp, _vp]),
        "b2l_beat_track": (C.c_int, [_vp, P(BeatDesc), _vp, _i64, _i64, _vp, _vp, _vp, _vp, _vp, _vp]),
        "b2l_any_nonzero": (C.c_int, [_vp, _vp, _i64, C.c_int32, _vp]),
        "b2l_plp_select": (C.c_int, [_vp, P(PlpDesc), _vp, _i64]),
        "b2l_plp_finish": (C.c_int, [_vp, _vp, _i64, _i64, C.c_int32]),
        "b2l_onset_normalize": (C.c_int, [_vp, _vp, _i64, _i64, C.c_int32, C.c_double, _vp, _vp]),
        "b2l_peak_pick": (C.c_int, [_vp, P(PeakDesc), _vp, _i64, _i64, _vp, _vp, _vp, _vp]),
        "b2l_onset_backtrack": (C.c_int, [_vp, _vp, _i64, C.c_int32, _vp, _i64, _vp, C.c_int32, C.c_int32, C.c_double,
                                          _vp]),
        "b2l_seq_logobs": (C.c_int, [_vp, P(SeqLogObsDesc), _vp, _vp, _vp]),
        "b2l_seq_decode": (C.c_int, [_vp, P(SeqModel), _vp, _i64, _i64, _vp, _vp]),
        "b2l_seq_route": (C.c_int, [_vp, P(SeqModel), _i64, P(C.c_int32)]),
        "b2l_dtw_cost": (C.c_int, [_vp, P(DtwCostDesc), _vp, _vp, _vp, _vp]),
        "b2l_nan_flag": (C.c_int, [_vp, _vp, _i64, C.c_int32, _vp]),
        "b2l_dtw_accumulate": (C.c_int, [_vp, P(DtwDesc), _vp, _vp, _vp]),
        "b2l_dtw_backtrack": (C.c_int, [_vp, P(DtwDesc), _vp, _vp, _i64, C.c_int32, C.c_int32, _vp, _vp, _vp]),
        "b2l_rqa": (C.c_int, [_vp, _vp, _i64, _i64, C.c_int32, C.c_double, C.c_double, C.c_int32, _vp, _vp]),
        "b2l_rqa_path": (C.c_int, [_vp, _vp, _vp, _i64, _i64, C.c_int32, _vp, _vp]),
        "b2l_cqt_project": (C.c_int, [_vp, P(CqtOctave), C.c_int32, _vp, _vp, _vp, _vp, _i64, _i64, C.c_int32, _vp]),
        "b2l_cqt_project_abs": (C.c_int, [_vp, P(CqtOctave), C.c_int32, _vp, _vp, _vp, _vp, _i64, _i64, C.c_int32,
                                          _vp]),
        "b2l_pad_center": (C.c_int, [_vp, _vp, _i64, _i64, C.c_int32, C.c_int32, _vp]),
        "b2l_iirt_filter": (C.c_int, [_vp, P(IirtRate), C.c_int32, _vp, _vp, C.c_int32, _i64]),
        "b2l_iirt_stmsp": (C.c_int, [_vp, P(IirtRate), C.c_int32, _i64, _i64, C.c_int32, _vp]),
        "b2l_delta": (C.c_int, [_vp, P(DeltaDesc), _vp, _i64, _i64, _i64, _vp]),
        "b2l_stack_memory": (C.c_int, [_vp, P(StackDesc), _vp, _i64, _i64, _i64, _vp, _vp]),
        "b2l_localext": (C.c_int, [_vp, _vp, C.c_int32, C.c_int32, _i64, _i64, _i64, _vp]),
        "b2l_nn_graph": (C.c_int, [_vp, P(NnDesc), _vp, _i64, C.c_int32, _vp, _vp, _vp, P(C.c_int32)]),
        "b2l_nn_filter": (C.c_int, [_vp, P(NnFilterDesc), _vp, _i64, _i64, _i64, _vp, _vp, _vp, _vp, _vp,
                                    P(C.c_int32)]),
        "b2l_nn_dense": (C.c_int, [_vp, _vp, _vp, _vp, _i64, C.c_int32, C.c_int32, _vp]),
        "b2l_nn_compact": (C.c_int, [_vp, _vp, C.c_int32, _i64, C.c_int32, _vp, _vp, _vp, _vp]),
        "b2l_chroma_fold": (C.c_int, [_vp, P(ChromaDesc), _vp, _i64, _i64, _vp]),
        "b2l_chroma_smooth": (C.c_int, [_vp, _vp, _i64, C.c_int32, _i64, C.c_int32, _vp, _vp, C.c_int32, C.c_int32,
                                        C.c_int32, C.c_double, _vp]),
        "b2l_stft_f64": (C.c_int, [_vp, _vp, _i64, _i64, _i64, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                   P(C.c_double), _vp]),
        "b2l_istft_f64": (C.c_int, [_vp, _vp, _i64, _i64, _i64, C.c_int32, C.c_int32, C.c_int32, P(C.c_double),
                                    P(C.c_double), _i64, _vp, _i64]),
        "b2l_f64_abs_pow": (C.c_int, [_vp, _vp, _i64, C.c_double, _vp]),
        "b2l_f64_mel": (C.c_int, [_vp, _vp, _i64, _i64, C.c_int32, P(C.c_float), C.c_int32, _vp]),
        "b2l_f64_db": (C.c_int, [_vp, _vp, _i64, _i64, C.c_double, C.c_double, C.c_double, _vp]),
        "b2l_f64_dct": (C.c_int, [_vp, _vp, _i64, C.c_int32, _i64, P(C.c_double), C.c_int32, _vp]),
        "b2l_nnls_mel": (C.c_int, [_vp, _vp, _i64, _i64, C.c_int32, C.c_int32, P(C.c_float), P(C.c_float), C.c_float,
                                   C.c_int32, C.c_float, _vp]),
        "b2l_comm_unique_id": (C.c_int, [_vp]),
        "b2l_comm_init": (C.c_int, [_vp, _vp, C.c_int, C.c_int]),
        "b2l_comm_destroy": (C.c_int, [_vp]),
        "b2l_comm_broadcast": (C.c_int, [_vp, _vp, C.c_size_t, C.c_int]),
        "b2l_comm_scatter": (C.c_int, [_vp, _vp, _vp, C.c_size_t, C.c_int]),
        "b2l_comm_gather": (C.c_int, [_vp, _vp, _vp, C.c_size_t, C.c_int]),
        "b2l_comm_barrier": (C.c_int, [_vp]),
    }
    for name, (res, args) in sig.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    return sig


EXPORTED_SYMBOLS: Tuple[str, ...] = ()


def lib():
    """Load libb2l.so once (raises NativeLibraryError with build instructions if absent)."""
    global _lib, EXPORTED_SYMBOLS
    if _lib is None:
        with _lib_lock:
            if _lib is None:
                if not os.path.exists(LIB_PATH):
                    raise NativeLibraryError(
                        f"{LIB_PATH} not found: build it with `make -C librosa_b200/csrc` or "
                        "`python -c 'import __graft_entry__ as g; g.build()'`. There is no CPU fallback."
                    )
                try:
                    handle = C.CDLL(LIB_PATH, mode=C.RTLD_GLOBAL)
                except OSError as exc:  # pragma: no cover
                    raise NativeLibraryError(f"cannot load {LIB_PATH}: {exc}") from exc
                EXPORTED_SYMBOLS = tuple(_declare(handle))
                _lib = handle
    return _lib


def check(status: int):
    if status == B2L_OK:
        return
    msg = lib().b2l_last_error().decode("utf-8", "replace")
    if status == B2L_ERR_INVALID:
        from .util.exceptions import ParameterError

        raise ParameterError(msg)
    if status == B2L_ERR_UNSUPPORTED:
        raise UnsupportedOnGPU(msg)
    if status == B2L_ERR_OOM:
        raise MemoryError(msg)
    raise NativeLibraryError(msg)


# --------------------------------------------------------------------------------------------- context
class LRUCache(dict):
    """Insertion-ordered dict used as a least-recently-used cache: ``fetch`` moves a hit to the young end and
    ``evict_oldest`` removes from the old end — so the entries handed out during the current call (always the
    youngest) are never the ones released.  ``dict.popitem()`` would evict the NEWEST entry instead."""

    def fetch(self, key):
        try:
            value = self.pop(key)
        except KeyError:
            return None
        self[key] = value
        return value

    def evict_oldest(self):
        key = next(iter(self))
        return key, self.pop(key)


class Context:
    """One CUDA device + stream.  Not thread-safe; create one per thread / per GPU."""

    def __init__(self, device: int = 0):
        self._h = _vp()
        check(lib().b2l_ctx_create(int(device), C.byref(self._h)))
        self.device = int(device)
        self._plans = LRUCache()
        self._constants = LRUCache()
        self._pool = {}
        self._sizes = {}
        self._pooled_bytes = 0
        # cached (released but not returned to the driver) device memory: blocks are exact-size, so variable-length
        # workloads reuse little — keep the cache well below the 80 GB of the device
        self.pool_limit_bytes = int(os.environ.get("B2L_POOL_LIMIT_MB", "16384")) << 20
        self._finalizer = weakref.finalize(self, Context._destroy, self._h, self._plans, self._constants, self._sizes)

    @staticmethod
    def _destroy(h, plans, constants, sizes):
        try:
            L = lib()
            for p in plans.values():
                L.b2l_plan_destroy(p.handle)
            plans.clear()
            for ptr in list(sizes):
                L.b2l_free(h, _vp(ptr))
            sizes.clear()
            constants.clear()
            L.b2l_ctx_destroy(h)
        except Exception:  # pragma: no cover - interpreter shutdown
            pass

    @property
    def handle(self):
        return self._h

    def synchronize(self):
        check(lib().b2l_ctx_sync(self._h))

    @property
    def sm_count(self) -> int:
        v = C.c_int()
        check(lib().b2l_ctx_sm_count(self._h, C.byref(v)))
        return v.value

    @property
    def launch_count(self) -> int:
        v = C.c_uint64()
        check(lib().b2l_ctx_launch_count(self._h, C.byref(v)))
        return int(v.value)

    def mem_info(self):
        f, t = C.c_size_t(), C.c_size_t()
        check(lib().b2l_mem_info(self._h, C.byref(f), C.byref(t)))
        return int(f.value), int(t.value)

    # ---- memory: a size-keyed free list in front of cudaMalloc / cudaFree.  All work of a context is
    # ordered on one stream, so handing a released block to the next request is safe without a sync;
    # it keeps multi-GB cudaMalloc / cudaFree calls (milliseconds each) out of steady-state loops.
    _POOL_QUANTUM = 512

    def alloc(self, nbytes: int) -> int:
        size = (max(int(nbytes), 1) + self._POOL_QUANTUM - 1) // self._POOL_QUANTUM * self._POOL_QUANTUM
        bucket = self._pool.get(size)
        if bucket:
            self._pooled_bytes -= size
            return bucket.pop()
        p = _vp()
        status = lib().b2l_alloc(self._h, size, C.byref(p))
        if status == B2L_ERR_OOM and self._pooled_bytes:
            self.empty_cache()
            status = lib().b2l_alloc(self._h, size, C.byref(p))
        check(status)
        self._sizes[p.value] = size
        return p.value

    def free(self, ptr: int):
        if not ptr:
            return
        size = self._sizes.get(ptr)
        if size is None:   # not ours (or already trimmed): release for real
            check(lib().b2l_free(self._h, _vp(ptr)))
            return
        self._pool.setdefault(size, []).append(ptr)
        self._pooled_bytes += size
        if self._pooled_bytes > self.pool_limit_bytes:
            self.empty_cache()

    def empty_cache(self):
        """Return every pooled block to the driver."""
        L = lib()
        for size, bucket in self._pool.items():
            for ptr in bucket:
                self._sizes.pop(ptr, None)
                L.b2l_free(self._h, _vp(ptr))
        self._pool.clear()
        self._pooled_bytes = 0

    def empty(self, shape, dtype, layout: str = "c") -> "DeviceArray":
        return DeviceArray.empty(self, shape, dtype, layout=layout)

    def zeros(self, shape, dtype) -> "DeviceArray":
        """A C-ordered buffer cleared on the stream."""
        out = DeviceArray.empty(self, shape, dtype)
        if out.nbytes:
            check(lib().b2l_memset(self._h, _vp(out.ptr), 0, out.nbytes))
        return out

    def to_device(self, arr: np.ndarray) -> "DeviceArray":
        arr = np.ascontiguousarray(arr)
        out = DeviceArray.empty(self, arr.shape, arr.dtype)
        check(lib().b2l_h2d(self._h, _vp(out.ptr), arr.ctypes.data_as(_vp), arr.nbytes))
        self.synchronize()
        return out

    def constant(self, key, build) -> int:
        """Device pointer of a small float32 table (bin frequencies, reciprocal window-sum-square, ...) cached per
        context under ``key``; ``build()`` makes its values on a miss.  At most 32 tables: the least recently used
        goes first, so a table fetched earlier in the same call (the youngest entry) stays."""
        ptr = self._constants.fetch(key)
        if ptr is None:
            arr = np.ascontiguousarray(build(), dtype=np.float32)
            while len(self._constants) >= 32:
                _, old = self._constants.evict_oldest()
                self.free(old)
            ptr = self.alloc(max(arr.nbytes, 16))
            check(lib().b2l_h2d(self._h, _vp(ptr), arr.ctypes.data_as(_vp), arr.nbytes))
            self.synchronize()
            self._constants[key] = ptr
        return ptr

    # ---- events
    def event(self) -> "Event":
        return Event(self)


_default_ctx: dict = {}


def default_context(device: Optional[int] = None) -> Context:
    """Process-wide context of a device (device defaults to $B2L_DEVICE, then $LOCAL_RANK, then 0)."""
    if device is None:
        device = int(os.environ.get("B2L_DEVICE", os.environ.get("LOCAL_RANK", "0")))
    ctx = _default_ctx.get(device)
    if ctx is None:
        ctx = Context(device)
        _default_ctx[device] = ctx
    return ctx


def bind_host_to_device(device: int = 0):
    """Pin the calling thread to the CPUs that are local to GPU ``device`` (NUMA node of its PCIe root), so that
    pinned host buffers allocated afterwards — and the staging copies into them — do not cross sockets.  The
    same thing ``numactl --cpunodebind`` does for one-process-per-GPU launches.  Needs NVML (``nvidia-ml-py``);
    returns the CPU list, or None when the topology cannot be read (nothing is changed then)."""
    try:
        import pynvml

        pynvml.nvmlInit()
        h = pynvml.nvmlDeviceGetHandleByIndex(int(device))
        words = (os.cpu_count() + 63) // 64
        mask = pynvml.nvmlDeviceGetCpuAffinity(h, words)
        cpus = [64 * w + b for w, m in enumerate(mask) for b in range(64) if (int(m) >> b) & 1]
        allowed = os.sched_getaffinity(0)
        cpus = [c for c in cpus if c in allowed]
        if not cpus:
            return None
        os.sched_setaffinity(0, cpus)
        return cpus
    except Exception:
        return None


def device_count() -> int:
    n = C.c_int()
    check(lib().b2l_device_count(C.byref(n)))
    return n.value


class Event:
    def __init__(self, ctx: Context):
        self.ctx = ctx
        self._h = _vp()
        check(lib().b2l_event_create(ctx.handle, C.byref(self._h)))
        self._finalizer = weakref.finalize(self, lambda h: lib().b2l_event_destroy(h), self._h)

    def record(self):
        check(lib().b2l_event_record(self.ctx.handle, self._h))
        return self

    def elapsed_ms(self, stop: "Event") -> float:
        ms = C.c_float()
        check(lib().b2l_event_elapsed_ms(self._h, stop._h, C.byref(ms)))
        return float(ms.value)


# --------------------------------------------------------------------------------------------- arrays
class DeviceArray:
    """A device buffer with a logical NumPy-style shape.

    ``layout``:
      * ``"c"``   — memory is C-ordered in the logical shape;
      * ``"ft"``  — logical shape is ``(..., bins, frames)`` (what librosa returns) while memory is
        ``[...][frames][bins]`` (bins contiguous) — the kernels' native spectrogram layout, and for a
        single clip exactly the Fortran order librosa.stft produces.
    """

    def __init__(self, ctx: Context, ptr: int, shape, dtype, layout: str = "c", owner: bool = True):
        self.ctx = ctx
        self.ptr = ptr
        self.shape = tuple(int(s) for s in shape)
        self.dtype = np.dtype(dtype)
        self.layout = layout
        self.base: Optional[DeviceArray] = None   # the buffer a view reads; kept alive with the view
        self._finalizer = weakref.finalize(self, DeviceArray._release, ctx, ptr) if owner and ptr else None

    @staticmethod
    def _release(ctx, ptr):
        try:
            ctx.free(ptr)
        except Exception:  # pragma: no cover
            pass

    @classmethod
    def empty(cls, ctx: Context, shape, dtype, layout: str = "c") -> "DeviceArray":
        shape = tuple(int(s) for s in shape)
        nbytes = int(np.prod(shape, dtype=np.int64)) * np.dtype(dtype).itemsize
        return cls(ctx, ctx.alloc(max(nbytes, 16)), shape, dtype, layout=layout)

    @property
    def ndim(self):
        return len(self.shape)

    @property
    def size(self):
        return int(np.prod(self.shape, dtype=np.int64))

    @property
    def nbytes(self):
        return self.size * self.dtype.itemsize

    def view(self, shape, offset: int = 0) -> "DeviceArray":
        """A non-owning C-ordered array of ``shape`` over this buffer's memory, starting ``offset`` elements in."""
        shape = tuple(int(s) for s in shape)
        start = int(offset)
        # math.prod, not np.prod: the small device calls that return views would notice the microseconds
        if start < 0 or start + math.prod(shape) > math.prod(self.shape):
            raise ValueError(f"a view of {shape} at offset {offset} reaches past a buffer of {self.shape}")
        out = DeviceArray(self.ctx, self.ptr + start * self.dtype.itemsize, shape, self.dtype, layout="c", owner=False)
        out.base = self
        return out

    def free(self):
        if self._finalizer is not None and self._finalizer.alive:
            self._finalizer()
        self.ptr = 0

    def _mem_shape(self):
        if self.layout == "ft":
            return self.shape[:-2] + (self.shape[-1], self.shape[-2])
        return self.shape

    def get(self, out: Optional[np.ndarray] = None) -> np.ndarray:
        """Copy to the host; returns an array of the logical shape (a transposed view for "ft")."""
        mem_shape = self._mem_shape()
        if out is None:
            host = pinned_empty(mem_shape, self.dtype) if self.nbytes >= (1 << 20) else np.empty(mem_shape, dtype=self.dtype)
        else:
            host = out
            if host.shape != mem_shape or host.dtype != self.dtype or not host.flags.c_contiguous:
                raise ValueError("out must be a C-contiguous array of the memory shape and dtype")
        if self.nbytes:
            check(lib().b2l_d2h(self.ctx.handle, host.ctypes.data_as(_vp), _vp(self.ptr), self.nbytes))
            self.ctx.synchronize()
        if self.layout == "ft":
            return np.swapaxes(host, -1, -2)
        return host

    def set(self, arr: np.ndarray):
        arr = np.ascontiguousarray(arr, dtype=self.dtype)
        if arr.shape != self._mem_shape():
            raise ValueError(f"shape mismatch: {arr.shape} vs memory shape {self._mem_shape()}")
        check(lib().b2l_h2d(self.ctx.handle, _vp(self.ptr), arr.ctypes.data_as(_vp), arr.nbytes))
        self.ctx.synchronize()
        return self

    def __repr__(self):
        return f"DeviceArray(shape={self.shape}, dtype={self.dtype}, layout={self.layout!r}, device={self.ctx.device})"


class _PinnedPool:
    """Size-keyed free list of page-locked host blocks.  cudaHostAlloc costs milliseconds and fresh
    pageable pages fault on first touch, so result arrays are carved from recycled pinned blocks: D2H runs
    at full PCIe speed and a block returns to the pool when the NumPy array that wraps it is collected."""

    QUANTUM = 1 << 16

    def __init__(self):
        self.free = {}
        self.pooled = 0
        self.limit = int(os.environ.get("B2L_PINNED_POOL_MB", "8192")) << 20
        self.lock = threading.Lock()

    def take(self, nbytes: int):
        size = (max(int(nbytes), 1) + self.QUANTUM - 1) // self.QUANTUM * self.QUANTUM
        with self.lock:
            bucket = self.free.get(size)
            if bucket:
                self.pooled -= size
                return bucket.pop(), size
        p = _vp()
        check(lib().b2l_host_alloc(size, C.byref(p)))
        return p.value, size

    def give(self, addr: int, size: int):
        with self.lock:
            if self.pooled + size <= self.limit:
                self.free.setdefault(size, []).append(addr)
                self.pooled += size
                return
        try:
            lib().b2l_host_free(_vp(addr))
        except Exception:  # pragma: no cover
            pass

    def empty(self):
        with self.lock:
            blocks = [(a, s) for s, b in self.free.items() for a in b]
            self.free.clear()
            self.pooled = 0
        for a, _ in blocks:
            lib().b2l_host_free(_vp(a))


_pinned_pool = _PinnedPool()


def pinned_empty(shape, dtype=np.float32) -> np.ndarray:
    """NumPy array backed by page-locked host memory (fast, truly asynchronous H2D / D2H)."""
    if not isinstance(shape, tuple):
        shape = tuple(int(s) for s in np.atleast_1d(shape))
    dtype = np.dtype(dtype)
    count = int(np.prod(shape, dtype=np.int64))
    addr, size = _pinned_pool.take(count * dtype.itemsize)
    buf = (C.c_char * size).from_address(addr)
    weakref.finalize(buf, _pinned_pool.give, addr, size)
    return np.frombuffer(buf, dtype=dtype, count=count).reshape(shape)


def empty_pinned_cache():
    _pinned_pool.empty()


# --------------------------------------------------------------------------------------------- plans
class Plan:
    def __init__(self, ctx: Context, handle, n_fft, hop, center, n_mels, n_mfcc):
        self.ctx = ctx
        self.handle = handle
        self.n_fft = n_fft
        self.hop = hop
        self.center = center
        self.n_mels = n_mels
        self.n_mfcc = n_mfcc

    def n_frames(self, n: int) -> int:
        v = _i64()
        check(lib().b2l_plan_n_frames(self.handle, int(n), C.byref(v)))
        return int(v.value)


def make_plan(ctx: Context, key, *, n_fft: int, hop_length: int, center: bool, pad_mode: str,
              window: np.ndarray, mel_basis: Optional[np.ndarray] = None, power: float = 2.0,
              dct_basis: Optional[np.ndarray] = None, amin: float = 1e-10, ref_value: float = 1.0,
              top_db: Optional[float] = 80.0) -> Plan:
    """Create (or fetch from the context's cache) the device constants of one configuration."""
    plan = ctx._plans.fetch(key)
    if plan is not None:
        return plan
    win = np.ascontiguousarray(window, dtype=np.float64)
    desc = PlanDesc()
    desc.n_fft = int(n_fft)
    desc.hop_length = int(hop_length)
    desc.center = 1 if center else 0
    desc.pad_mode = PAD_MODES[pad_mode]
    desc.h_window = win.ctypes.data_as(C.POINTER(C.c_double))
    keep = [win]
    n_mels = n_mfcc = 0
    if mel_basis is not None:
        mb = np.ascontiguousarray(mel_basis, dtype=np.float32)
        keep.append(mb)
        n_mels = mb.shape[0]
        desc.n_mels = n_mels
        desc.h_mel_basis = mb.ctypes.data_as(C.POINTER(C.c_float))
    desc.power = float(power)
    if dct_basis is not None:
        db = np.ascontiguousarray(dct_basis, dtype=np.float32)
        keep.append(db)
        n_mfcc = db.shape[0]
        desc.n_mfcc = n_mfcc
        desc.h_dct_basis = db.ctypes.data_as(C.POINTER(C.c_float))
    desc.amin = float(amin)
    desc.ref_value = float(ref_value)
    desc.top_db = -1.0 if top_db is None else float(top_db)
    h = _vp()
    check(lib().b2l_plan_create(ctx.handle, C.byref(desc), C.byref(h)))
    plan = Plan(ctx, h, int(n_fft), int(hop_length), bool(center), n_mels, n_mfcc)
    ctx._plans[key] = plan
    while len(ctx._plans) > 64:  # bound the cache: drop the least recently used plan (never the new one)
        _, old = ctx._plans.evict_oldest()
        lib().b2l_plan_destroy(old.handle)
    return plan
