"""Case table of the constant-Q chroma features: tests/golden/chroma_v1.npz holds, for each case, what the unmodified
reference's ``chroma_cqt`` / ``chroma_cens`` / ``chroma_vqt`` / ``tonnetz`` returns (``<name>/out``) or the
exception it raises (``<name>/error``, "Class: message"), and ``filters.cq_to_chroma`` maps (``map/<name>``).
The y= cases ran with the reference's ``cqt`` / ``vqt`` called with ``res_type="polyphase"``.  For the cases in
``WITH_STEPS`` it also holds the reference's |C| (``<name>/absC``), its un-normalised chroma (``<name>/raw``) and,
for CENS, the quantised input of the smoothing (``<name>/quant``).  Written by tools/make_golden.py --chroma;
tests/chroma_oracle.py must reproduce every entry bit for bit.

``C=`` / ``V=`` / ``chroma=`` inputs are made from a seed (``inputs``); ``refuse`` names the calls the GPU declines
with UnsupportedOnGPU."""
from __future__ import annotations

import numpy as np

from cqt_cases import signal

P = {"res_type": "polyphase"}
SIG = ((), 44100, 22050, np.float32)          # 2 s
SIG_MC = ((2,), 22050, 22050, np.float32)     # 2 channels of 1 s


def _c(name, fn, kw, inp=None, sig=SIG, refuse=False):
    """``inp``: None for y=, else (argument name, shape, dtype[, "nan"]) of a seeded non-negative input."""
    return {"name": name, "fn": fn, "kw": dict(kw), "inp": inp, "sig": sig + (len(name) + 11,), "refuse": refuse}


def _C(rows=252, T=173, dtype=np.float32, lead=(), arg="C", special=None):
    return (arg, tuple(lead) + (rows, T), dtype) + ((special,) if special else ())


CASES = [
    # chroma_cqt
    _c("cqt_y_defaults", "chroma_cqt", dict(P, hop_length=256)),
    _c("cqt_y_hop128_tuning0", "chroma_cqt", dict(P, hop_length=128, tuning=0.0, n_octaves=6)),
    _c("cqt_y_multichannel", "chroma_cqt", dict(P, hop_length=256, tuning=0.0), sig=SIG_MC),
    _c("cqt_C_f32", "chroma_cqt", {}, _C()),
    _c("cqt_C_f64", "chroma_cqt", {}, _C(dtype=np.float64)),
    _c("cqt_C_norm_none", "chroma_cqt", dict(norm=None), _C()),
    _c("cqt_C_norm_half", "chroma_cqt", dict(norm=0.5), _C()),
    _c("cqt_C_norm_neg_inf", "chroma_cqt", dict(norm=-np.inf), _C()),
    _c("cqt_C_norm_0", "chroma_cqt", dict(norm=0, threshold=0.5), _C()),
    _c("cqt_C_norm_1", "chroma_cqt", dict(norm=1), _C()),
    _c("cqt_C_norm_2", "chroma_cqt", dict(norm=2), _C()),
    _c("cqt_C_norm_3", "chroma_cqt", dict(norm=3.0), _C(dtype=np.float64)),
    _c("cqt_C_threshold", "chroma_cqt", dict(threshold=1.5), _C()),
    _c("cqt_C_threshold_none", "chroma_cqt", dict(threshold=None), _C()),
    _c("cqt_C_n24_bpo48", "chroma_cqt", dict(n_chroma=24, bins_per_octave=48), _C(rows=336)),
    _c("cqt_C_bpo_none", "chroma_cqt", dict(bins_per_octave=None), _C(rows=84)),
    _c("cqt_C_fmin_a1", "chroma_cqt", dict(fmin=55.0), _C()),
    _c("cqt_C_80_rows", "chroma_cqt", dict(bins_per_octave=12), _C(rows=80)),
    _c("cqt_C_window", "chroma_cqt", dict(window=np.array([0.25, 0.5, 0.25])), _C()),
    _c("cqt_C_multichannel", "chroma_cqt", {}, _C(lead=(2, 3), T=40)),
    _c("cqt_C_zero_frames", "chroma_cqt", dict(norm=2), _C(special="zero")),
    _c("cqt_y_tuning_none", "chroma_cqt", dict(P, hop_length=256, n_octaves=6)),
    # chroma_cens
    _c("cens_y_defaults", "chroma_cens", dict(P, hop_length=256)),
    _c("cens_C_defaults", "chroma_cens", {}, _C()),
    _c("cens_C_win_none", "chroma_cens", dict(win_len_smooth=None), _C()),
    _c("cens_C_win_1", "chroma_cens", dict(win_len_smooth=1), _C()),
    _c("cens_C_win_2", "chroma_cens", dict(win_len_smooth=2), _C()),
    _c("cens_C_win_40", "chroma_cens", dict(win_len_smooth=40), _C()),
    _c("cens_C_win_500", "chroma_cens", dict(win_len_smooth=500), _C()),
    _c("cens_C_hamming", "chroma_cens", dict(smoothing_window="hamming"), _C()),
    _c("cens_C_kaiser", "chroma_cens", dict(smoothing_window=("kaiser", 4.0)), _C()),
    _c("cens_C_norm_inf", "chroma_cens", dict(norm=np.inf), _C()),
    _c("cens_C_norm_none", "chroma_cens", dict(norm=None), _C()),
    _c("cens_C_f64", "chroma_cens", {}, _C(dtype=np.float64)),
    # chroma_vqt
    _c("vqt_y_equal", "chroma_vqt", dict(P, intervals="equal", hop_length=256, n_octaves=6)),
    _c("vqt_y_list", "chroma_vqt", dict(P, intervals=[1.0, 1.25, 1.5], hop_length=256, fmin=55.0, n_octaves=6)),
    _c("vqt_V_ji5", "chroma_vqt", dict(intervals="ji5", bins_per_octave=7), _C(rows=49, arg="V")),
    _c("vqt_y_gamma10", "chroma_vqt", dict(P, intervals="equal", hop_length=256, gamma=10, n_octaves=6)),
    # tonnetz
    _c("tonnetz_y", "tonnetz", dict(P, hop_length=256)),
    _c("tonnetz_chroma_stft", "tonnetz", {}, ("chroma", "chroma_stft")),
    _c("tonnetz_chroma_36", "tonnetz", {}, _C(rows=36, arg="chroma")),
    _c("tonnetz_chroma_multichannel", "tonnetz", {}, _C(rows=12, lead=(3,), T=50, arg="chroma", dtype=np.float64)),
    _c("tonnetz_C_norm2", "tonnetz", dict(norm=2), _C()),
    # errors the reference raises
    _c("err_bpo_n_chroma", "chroma_cqt", dict(n_chroma=12, bins_per_octave=40), _C()),
    _c("err_no_input", "chroma_cqt", {}),
    _c("err_cens_win_0", "chroma_cens", dict(win_len_smooth=0), _C()),
    _c("err_cens_win_float", "chroma_cens", dict(win_len_smooth=2.0), _C()),
    _c("err_nan_norm_none", "chroma_cqt", dict(norm=None), _C(special="nan")),
    _c("err_nan_norm_inf", "chroma_cqt", {}, _C(special="nan")),
    _c("err_nan_cens", "chroma_cens", {}, _C(special="nan")),
    _c("err_bad_norm", "chroma_cqt", dict(norm=-1), _C()),
    _c("err_bad_norm_nan", "chroma_cqt", dict(norm="foo"), _C(special="nan")),
    _c("err_tonnetz_no_input", "tonnetz", {}),
    _c("err_vqt_no_input", "chroma_vqt", dict(intervals="equal")),
    # refusals: the GPU declines what the reference runs
    _c("refuse_hybrid", "chroma_cqt", dict(P, cqt_mode="hybrid"), refuse=True),
    _c("refuse_complex_C", "chroma_cqt", {}, _C(dtype=np.complex64), refuse=True),
    _c("refuse_soxr", "chroma_cqt", dict(hop_length=512), refuse=True),
    _c("refuse_vqt_ji5", "chroma_vqt", dict(P, intervals="ji5"), refuse=True),
]
CASES[CASES.index(next(c for c in CASES if c["name"] == "err_no_input"))]["no_y"] = True
CASES[CASES.index(next(c for c in CASES if c["name"] == "err_tonnetz_no_input"))]["no_y"] = True
CASES[CASES.index(next(c for c in CASES if c["name"] == "err_vqt_no_input"))]["no_y"] = True
BY_NAME = {c["name"]: c for c in CASES}

# cases whose fixture also stores |C| / the raw chroma / the quantised CENS input
WITH_STEPS = ("cqt_y_defaults", "cens_y_defaults", "cens_C_defaults", "cens_C_win_2", "cens_C_kaiser", "cens_C_win_500")

# cq_to_chroma maps pinned on their own: name -> keyword arguments (n_input first)
MAPS = {
    "default_252": dict(n_input=252, bins_per_octave=36),
    "n24_bpo48": dict(n_input=336, bins_per_octave=48, n_chroma=24),
    "bpo12_80": dict(n_input=80, bins_per_octave=12),
    "fmin_a1": dict(n_input=252, bins_per_octave=36, fmin=55.0),
    "fmin_odd": dict(n_input=100, bins_per_octave=36, fmin=47.3),
    "base_a": dict(n_input=84, bins_per_octave=12, base_c=False),
    "window": dict(n_input=252, bins_per_octave=36, window=np.array([0.25, 0.5, 0.25])),
    "float64": dict(n_input=84, bins_per_octave=12, dtype=np.float64),
    "perm_7": dict(n_input=49, bins_per_octave=7, n_chroma=7),
}


def stft_chroma_signal():
    return signal(SIG[:3] + (np.float32, 5))


def inputs(case, golden=None):
    """The call's array arguments: {"y": signal} or {argument: seeded array}; the chroma_stft input of a tonnetz
    case is the reference's, stored in the fixture (``golden``) as ``<name>/input``."""
    if case.get("no_y"):
        return {}
    if case["inp"] is None:
        return {"y": signal(case["sig"])}
    arg, spec = case["inp"][0], case["inp"][1:]
    if spec[0] == "chroma_stft":
        return {arg: golden[f"{case['name']}/input"]}
    shape, dtype = spec[0], spec[1]
    rng = np.random.default_rng(len(case["name"]) * 131 + shape[-1])
    x = rng.gamma(0.6, 1.0, size=shape) * rng.uniform(0.2, 3.0, size=shape[:-1] + (1,))
    if np.dtype(dtype).kind == "c":
        x = x * np.exp(1j * rng.uniform(0, 2 * np.pi, size=shape))
    x = x.astype(dtype)
    if len(spec) > 2 and spec[2] == "nan":
        x.reshape(-1)[x.size // 3] = np.nan
    if len(spec) > 2 and spec[2] == "zero":
        x[..., :, 5:9] = 0
    return {arg: x}


def call(lib, case, golden=None, arrays=None, drop_res_type=False):
    """Run one case through ``lib`` (the reference or librosa_b200); ``drop_res_type`` for the reference."""
    kw = dict(case["kw"])
    if drop_res_type:
        kw.pop("res_type", None)
    kw.update(inputs(case, golden) if arrays is None else arrays)
    if "y" in kw or case["fn"] != "tonnetz":
        kw.setdefault("sr", case["sig"][2])
    return getattr(lib.feature, case["fn"])(**kw)
