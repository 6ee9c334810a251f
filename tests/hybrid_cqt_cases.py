"""Case table of pseudo_cqt and hybrid_cqt: tests/golden/hybrid_cqt_v1.npz holds, for each case, what the unmodified
reference returns (``<name>/C``) or the exception it raises (``<name>/error``, "Class: message"), the stft warnings
it emits (``<name>/warnings``), the pseudo part's call (``<name>/n_fft``, ``<name>/n_pseudo``, ``<name>/n_full``,
``<name>/fmin_pseudo``; for hybrid_cqt those of its pseudo_cqt and cqt calls), the pseudo part's |basis| as a CSR
matrix (``<name>/basis/indptr|indices|data``, or for the dense bases in ``BASIS_DIGEST`` the ``<name>/basis/sha256``
of those three arrays, to keep the fixture small) and, for the cases in ``WITH_D``, the pseudo part's centred Hann STFT
(``<name>/D``).  Written by tools/make_golden.py --hybrid-cqt; tests/hybrid_cqt_oracle.py must reproduce every
entry bit for bit.

``refuse`` names the cases the GPU declines with UnsupportedOnGPU although the reference runs them (or would, with
its optional resamplers installed): a pseudo n_fft above 8192, a non-polyphase resampler where the full part
resamples, an octave n_fft above 8192."""
from __future__ import annotations

import hashlib

import numpy as np

from cqt_cases import S16, signal  # noqa: F401  (the same signals as the cqt fixture)

P = {"res_type": "polyphase"}


def _c(name, kw, sig=((), 8000, 22050, np.float32), refuse=False):
    lead, n, sr, dtype = sig
    kw = dict(kw)
    kw.setdefault("sr", sr)
    fn = "pseudo_cqt" if name.startswith("pcqt") else "hybrid_cqt"
    return {"name": name, "fn": fn, "kw": kw, "sig": (lead, n, sr, dtype, len(name) + 7 * n), "refuse": refuse}


F220 = {"fmin": 220.0, "n_bins": 48}

CASES = [
    _c("pcqt_fmin220", F220),
    _c("pcqt_hop256", dict(F220, hop_length=256)),
    _c("pcqt_hop1024", dict(fmin=110.0, n_bins=60, hop_length=1024)),
    _c("pcqt_bpo24", dict(fmin=220.0, n_bins=96, bins_per_octave=24)),
    _c("pcqt_bpo36", dict(fmin=440.0, n_bins=108, bins_per_octave=36, hop_length=256)),
    _c("pcqt_scale_false", dict(F220, scale=False)),
    _c("pcqt_norm2", dict(F220, norm=2)),
    _c("pcqt_norm_none", dict(F220, norm=None)),
    _c("pcqt_norm_inf", dict(F220, norm=np.inf)),
    _c("pcqt_sparsity0", dict(F220, sparsity=0)),
    _c("pcqt_window_hamming", dict(F220, window="hamming")),
    _c("pcqt_window_ones", dict(F220, window="ones")),
    _c("pcqt_pad_reflect", dict(F220, pad_mode="reflect")),
    _c("pcqt_pad_edge", dict(F220, pad_mode="edge")),
    _c("pcqt_n_bins_none", dict(fmin=220.0, n_bins=None)),
    _c("pcqt_one_bin", dict(fmin=440.0, n_bins=1)),
    _c("pcqt_tuning_none", dict(F220, tuning=None)),
    _c("pcqt_multichannel", F220, ((2, 3), 4000, 22050, np.float32)),
    _c("pcqt_float64", F220, ((), 8000, 22050, np.float64)),
    _c("pcqt_dtype_c128", dict(F220, dtype=np.complex128)),
    _c("pcqt_short_warns", F220, ((), 2000, 22050, np.float32)),
    _c("hcqt_defaults", P),
    _c("hcqt_hop256", dict(P, hop_length=256)),
    _c("hcqt_hop128", dict(P, hop_length=128)),
    _c("hcqt_hop2048", dict(P, hop_length=2048)),
    _c("hcqt_hop4096", dict(P, hop_length=4096)),
    _c("hcqt_hop64", dict(P, hop_length=64)),
    _c("hcqt_high_fmin", dict(P, fmin=1200.0, n_bins=24)),
    _c("hcqt_one_pseudo", dict(P, n_bins=56)),
    _c("hcqt_bpo36", dict(P, bins_per_octave=36, n_bins=252)),
    _c("hcqt_sr16000_hop160", dict(P, hop_length=160, n_bins=72), S16),
    _c("hcqt_scale_false", dict(P, scale=False)),
    _c("hcqt_tuning_none", dict(P, tuning=None)),
    _c("hcqt_multichannel", dict(P, n_bins=72), ((2, 3), 4000, 22050, np.float32)),
    _c("hcqt_float64", dict(P, n_bins=72), ((), 8000, 22050, np.float64)),
    # refusals: the GPU declines what the reference runs
    _c("pcqt_defaults", {}, refuse=True),
    _c("hcqt_soxr_resamples", dict(n_bins=36), refuse=True),
    _c("hcqt_odd_hop", dict(P, hop_length=441), refuse=True),
    # errors the reference raises
    _c("pcqt_fmin_above_nyquist", dict(fmin=12000.0)),
    _c("pcqt_exceeds_nyquist", dict(fmin=500.0, n_bins=84)),
    _c("pcqt_not_finite", F220),
    _c("hcqt_fmin_above_nyquist", dict(P, fmin=12000.0)),
    _c("hcqt_exceeds_nyquist", dict(P, fmin=500.0, n_bins=84)),
    _c("hcqt_not_finite", P),
]
for _case in CASES:
    if _case["name"].endswith("not_finite"):
        _case["sig"] = _case["sig"] + ("nan",)
BY_NAME = {c["name"]: c for c in CASES}

# cases whose fixture stores the pseudo part's STFT D
WITH_D = ("pcqt_scale_false", "hcqt_defaults")

# cases whose |basis| is stored as its digest (basis_digest)
BASIS_DIGEST = {"pcqt_sparsity0", "pcqt_window_ones", "pcqt_window_hamming", "pcqt_defaults"}


def basis_digest(indptr, indices, data) -> str:
    h = hashlib.sha256()
    for a in (np.asarray(indptr, np.int32), np.asarray(indices, np.int32), np.asarray(data, np.float32)):
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


def call(lib, case, y=None):
    """Run one case through ``lib`` (the reference or librosa_b200)."""
    return getattr(lib, case["fn"])(signal(case["sig"]) if y is None else y, **case["kw"])
