"""Case table of segment.recurrence_matrix and decompose.nn_filter: tests/golden/nn_filter_v1.npz holds, for each case,
what the unmodified reference returns or the exception it raises (``<name>/error``, "Class: message").  Written by
tools/make_golden.py --nn-filter.

A recurrence matrix is stored as its csc_array: ``<name>/indptr``, ``<name>/indices``, ``<name>/data``; an nn_filter
case stores the reference's rec the same way and its output ``<name>/out``.  The data is made from the case's spec
(seeded), so nothing but the outputs is stored."""
from __future__ import annotations

import numpy as np


def data(spec):
    """spec = (shape, seed, dtype[, n_silent]): non-negative spectrogram-like frames with repeated sections, so that
    the neighbour structure is not noise alone; n_silent frames (every 10th from frame 5) are set to zero."""
    shape, seed, dtype = spec[:3]
    n_silent = spec[3] if len(spec) > 3 else 0
    rng = np.random.default_rng(seed)
    t = shape[-1]
    base = rng.random(shape[:-1] + (8,)) ** 2
    pattern = rng.integers(0, 8, t)
    x = base[..., pattern] * (1.0 + 0.3 * rng.random(shape)) + 0.05 * rng.random(shape)
    for s in range(n_silent):
        x[..., 5 + 10 * s] = 0.0
    if np.issubdtype(np.dtype(dtype), np.integer):
        x = np.round(100 * x)
    return x.astype(dtype)


def _case(name, fn, spec, kw=None, agg=None, rec_kw=None, nan=False):
    return dict(name=name, fn=fn, spec=spec, kw=kw or {}, agg=agg, rec_kw=rec_kw, nan=nan)


CHROMA = ((12, 300), 1, np.float64)
SPEC32 = ((257, 400), 2, np.float32, 40)
NN32 = ((129, 300), 10, np.float32, 30)
F64 = ((64, 250), 3, np.float64)
MULTI = ((2, 48, 200), 4, np.float32)
SMALL = ((40, 120), 5, np.float64)
SMALL32 = ((40, 120), 6, np.float32)

CASES = [
    _case("chroma_default", "rec", CHROMA),
    _case("chroma_cosine", "rec", CHROMA, dict(metric="cosine")),
    _case("spec32_cosine", "rec", SPEC32, dict(metric="cosine", width=3)),
    _case("spec32_cosine_distance", "rec", SPEC32, dict(metric="cosine", width=3, mode="distance")),
    _case("f64_distance", "rec", F64, dict(mode="distance", k=12)),
    _case("multi", "rec", MULTI, dict(width=2)),
    _case("axis0", "rec", ((200, 30), 7, np.float64), dict(axis=0, k=7)),
    _case("explicit_k", "rec", SMALL, dict(k=5)),
    _case("k_over_t", "rec", ((40, 40), 8, np.float64), dict(k=30, width=5)),
    _case("int_data", "rec", ((20, 80), 9, np.int64), dict(k=6)),
]
for _m in ("connectivity", "distance", "affinity"):
    for _sym in (False, True):
        for _self in (False, True):
            CASES.append(_case(f"mode_{_m}_sym{int(_sym)}_self{int(_self)}", "rec", SMALL,
                               dict(mode=_m, sym=_sym, self=_self, k=8, width=2)))
for _bw in ("med_k_scalar", "mean_k", "gmean_k", "mean_k_avg", "gmean_k_avg", "mean_k_avg_and_pair", 0.5):
    CASES.append(_case(f"bw_{_bw}", "rec", SMALL32, dict(mode="affinity", metric="cosine", k=9, bandwidth=_bw,
                                                            self=True)))
CASES += [
    _case("err_width", "rec", SMALL, dict(width=60)),
    _case("err_mode", "rec", SMALL, dict(mode="bogus")),
    _case("err_bandwidth", "rec", SMALL, dict(mode="affinity", bandwidth="bogus")),
    _case("err_scalar_bandwidth", "rec", SMALL, dict(mode="affinity", bandwidth=-1.0)),
    _case("err_no_neighbors", "rec", SMALL, dict(mode="affinity", bandwidth="mean_k", sym=True, k=1, width=2)),
    # nn_filter: the reference's rec and output
    _case("nn_mean", "nn", NN32, agg="mean", rec_kw=dict(metric="cosine", width=3)),
    _case("nn_median_even", "nn", NN32, agg="median", rec_kw=dict(metric="cosine", width=3, k=10)),
    _case("nn_median_odd", "nn", NN32, agg="median", rec_kw=dict(metric="cosine", width=3, k=9)),
    _case("nn_median_f64", "nn", F64, agg="median", rec_kw=dict(k=11)),
    _case("nn_average_aff", "nn", SMALL32, agg="average", rec_kw=dict(mode="affinity", metric="cosine", self=True)),
    _case("nn_average_aff64", "nn", F64, agg="average", rec_kw=dict(mode="affinity", k=7)),
    _case("nn_average_conn", "nn", SMALL32, agg="average", rec_kw=dict(k=6)),
    _case("nn_multi_mean", "nn", MULTI, agg="mean", rec_kw=dict(width=2)),
    _case("nn_nan_median", "nn", SMALL32, agg="median", rec_kw=dict(k=8), nan=True),
    _case("nn_nan_mean", "nn", SMALL32, agg="mean", rec_kw=dict(k=8), nan=True),
    _case("nn_err_shape", "nn", SMALL, agg="mean", rec_kw=dict(k=5)),
]
BY_NAME = {c["name"]: c for c in CASES}
AGG = {"mean": np.mean, "median": np.median, "average": np.average}


def case_data(case):
    x = data(case["spec"])
    return x


def filter_input(case):
    """(S, rec_source): the spectrogram an nn_filter case filters (NaNs planted when asked) and the data its rec
    is computed from (the clean S)."""
    S = data(case["spec"])
    clean = S.copy()
    if case["nan"]:
        S = S.copy()
        S[3, 7] = np.nan
        S[0, 50] = np.nan
    return S, clean


def call(lib, case):
    """Run a case with a librosa-like module ``lib``: a recurrence matrix (sparse) or (rec, nn_filter output)."""
    if case["fn"] == "rec":
        return lib.segment.recurrence_matrix(case_data(case), sparse=True, **case["kw"])
    S, clean = filter_input(case)
    rec = lib.segment.recurrence_matrix(clean, sparse=True, **case["rec_kw"])
    if case["name"] == "nn_err_shape":
        return rec, lib.decompose.nn_filter(S[:, :-1], rec=rec, aggregate=AGG[case["agg"]])
    return rec, lib.decompose.nn_filter(S, rec=rec, aggregate=AGG[case["agg"]])


def unpack(z, name):
    """The stored csc_array of a case."""
    import scipy.sparse

    indptr = z[f"{name}/indptr"]
    t = len(indptr) - 1
    return scipy.sparse.csc_array((z[f"{name}/data"], z[f"{name}/indices"], indptr), shape=(t, t))
