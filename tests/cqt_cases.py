"""Case table of the constant-Q transforms: tests/golden/cqt_v1.npz holds, for each case, what the unmodified
reference's ``cqt`` / ``vqt`` returns (``<name>/C``) or the exception it raises (``<name>/error``,
"Class: message"), the warnings it emits (``<name>/warnings``), every octave's call (``<name>/octaves``: signal
length, n_fft, hop, filters) and sparse basis (``<name>/basis<i>/indptr|indices|data`` for the cases in
``BASIS_ARRAYS``, else ``<name>/basis<i>/sha256`` of those three arrays), and for the cases in
``WITH_D`` the centred STFT ``D`` of octave ``WITH_D[name]`` (``<name>/D``).  Written by
tools/make_golden.py --cqt; tests/cqt_oracle.py must reproduce every entry bit for bit.

``refuse`` names the cases the GPU declines with UnsupportedOnGPU although the reference runs them (or would,
with its optional resamplers installed): an octave n_fft above 8192, a non-polyphase resampler where resampling
happens, a named interval set."""
from __future__ import annotations

import hashlib

import numpy as np

P = {"res_type": "polyphase"}


def signal(spec):
    """spec: (lead shape, n, sr, dtype, seed[, special]): a few partials with vibrato plus a little noise."""
    lead, n, sr, dtype, seed = spec[:5]
    rng = np.random.default_rng(seed)
    t = np.arange(n) / sr
    shape = tuple(lead) + (n,)
    y = np.zeros(shape)
    flat = y.reshape(-1, n)
    for row in flat:
        for f in rng.uniform(40.0, 0.4 * sr, size=4):
            row += rng.uniform(0.1, 0.5) * np.sin(2 * np.pi * f * t * (1 + 0.002 * np.sin(2 * np.pi * 3 * t)))
        row += 0.01 * rng.standard_normal(n)
    if len(spec) > 5 and spec[5] == "nan":
        flat[0, n // 3] = np.nan
    return y.astype(dtype)


def _c(name, kw, sig=((), 8000, 22050, np.float32), fn="cqt", refuse=False):
    lead, n, sr, dtype = sig
    kw = dict(kw)
    kw.setdefault("sr", sr)
    return {"name": name, "fn": fn, "kw": kw, "sig": (lead, n, sr, dtype, len(name) + 7 * n), "refuse": refuse}


S16 = ((), 8000, 16000, np.float32)
S44 = ((), 8000, 44100, np.float32)

CASES = [
    _c("cqt_defaults", P),
    _c("cqt_hop256", dict(P, hop_length=256)),
    _c("cqt_hop128_bpo24", dict(P, hop_length=128, bins_per_octave=24, n_bins=96)),
    _c("cqt_sr44100_bpo36", dict(P, hop_length=256, bins_per_octave=36, n_bins=252), S44),
    _c("cqt_sr16000_hop160", dict(P, hop_length=160, n_bins=72), S16),
    _c("cqt_sr16000_hop320", dict(P, hop_length=320, n_bins=60, fmin=55.0), S16),
    _c("cqt_fmin_a1", dict(P, fmin=55.0, n_bins=72)),
    _c("cqt_fmin_high", dict(P, fmin=220.0, n_bins=48, hop_length=128)),
    _c("cqt_partial_octave", dict(P, fmin=40.0, n_bins=80)),
    _c("cqt_partial_octave_30", dict(P, fmin=100.0, n_bins=30, hop_length=128)),
    _c("cqt_one_octave_soxr", dict(fmin=1000.0, n_bins=12, hop_length=441)),
    _c("cqt_n_bins_none", dict(P, n_bins=None, fmin=65.0, hop_length=256)),
    _c("cqt_tuning_none", dict(P, tuning=None)),
    _c("cqt_tuning_value", dict(P, tuning=0.3, n_bins=60)),
    _c("cqt_filter_scale_half", dict(P, filter_scale=0.5)),
    _c("cqt_filter_scale_2", dict(P, filter_scale=2, fmin=65.0, n_bins=60)),
    _c("cqt_norm2", dict(P, norm=2)),
    _c("cqt_norm_none", dict(P, norm=None)),
    _c("cqt_norm_inf", dict(P, norm=np.inf, n_bins=60)),
    _c("cqt_sparsity0", dict(P, sparsity=0)),
    _c("cqt_sparsity0_hop128", dict(P, sparsity=0, hop_length=128, n_bins=48, fmin=110.0)),
    _c("cqt_sparsity_05", dict(P, sparsity=0.05)),
    _c("cqt_window_hamming", dict(P, window="hamming")),
    _c("cqt_window_blackman", dict(P, window="blackman", n_bins=60)),
    _c("cqt_window_ones", dict(P, window="ones", n_bins=72)),
    _c("cqt_scale_false", dict(P, scale=False)),
    _c("cqt_scale_false_early", dict(P, scale=False, fmin=32.7, n_bins=24, hop_length=1024)),
    _c("cqt_early_downsample", dict(P, fmin=32.7, n_bins=24, hop_length=1024)),
    _c("cqt_pad_reflect", dict(P, pad_mode="reflect")),
    _c("cqt_pad_edge", dict(P, pad_mode="edge", n_bins=60)),
    _c("cqt_multichannel", dict(P, n_bins=72), ((2, 3), 4000, 22050, np.float32)),
    _c("cqt_float64", dict(P, n_bins=72), ((), 8000, 22050, np.float64)),
    _c("cqt_short_warns", dict(P, hop_length=256), ((), 2000, 22050, np.float32)),
    _c("cqt_dtype_c128", dict(P, n_bins=60, dtype=np.complex128)),
    _c("vqt_gamma_none", dict(P), fn="vqt"),
    _c("vqt_gamma_10", dict(P, gamma=10.0, n_bins=72), fn="vqt"),
    _c("vqt_gamma_30_hop256", dict(P, gamma=30.0, hop_length=256, bins_per_octave=24, n_bins=120), fn="vqt"),
    _c("vqt_intervals", dict(P, intervals=[1.0, 1.25, 1.5], n_bins=18, fmin=55.0), fn="vqt"),
    _c("vqt_intervals_tuning_none", dict(P, intervals=[1.0, 4 / 3, 1.5, 1.875], n_bins=24, tuning=None), fn="vqt"),
    _c("vqt_sr16000", dict(P, hop_length=160, n_bins=72, gamma=5.0), S16, fn="vqt"),
    # refusals: the GPU declines what the reference runs
    _c("cqt_odd_hop", dict(P, hop_length=441), refuse=True),
    _c("cqt_soxr_resamples", dict(n_bins=36), refuse=True),
    _c("vqt_ji5", dict(P, intervals="ji5", n_bins=24), fn="vqt", refuse=True),
    # errors the reference raises
    _c("cqt_fmin_above_nyquist", dict(P, fmin=12000.0)),
    _c("cqt_exceeds_nyquist", dict(P, fmin=500.0, n_bins=84)),
    _c("cqt_too_short", dict(P, fmin=32.7, n_bins=24, hop_length=1024), ((), 2, 22050, np.float32)),
    _c("cqt_not_finite", P),
]
CASES[-1]["sig"] = CASES[-1]["sig"] + ("nan",)
BY_NAME = {c["name"]: c for c in CASES}

# cases whose stored fixture includes one octave's STFT D (octave index)
WITH_D = {"cqt_defaults": 0, "cqt_sparsity0": 3, "vqt_gamma_none": 4, "cqt_sr16000_hop160": 5}

# cases whose bases are stored as arrays; the others store their digest (basis_digest) to keep the fixture small
BASIS_ARRAYS = {"cqt_defaults", "cqt_sr44100_bpo36", "cqt_partial_octave", "cqt_norm2", "cqt_window_hamming",
                "cqt_early_downsample", "vqt_gamma_none", "vqt_intervals", "cqt_sr16000_hop160", "cqt_float64"}


def call(lib, case):
    """Run one case through ``lib`` (the reference or librosa_b200)."""
    fn = getattr(lib, case["fn"])
    return fn(signal(case["sig"]), **case["kw"])


def basis_digest(indptr, indices, data) -> str:
    h = hashlib.sha256()
    for a in (np.asarray(indptr, np.int32), np.asarray(indices, np.int32), np.asarray(data, np.complex64)):
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()
