"""Case table of alignment: tests/golden/alignment_v1.npz holds, for each case, what the unmodified reference's
``sequence.dtw`` / ``dtw_backtracking`` / ``rqa`` / ``path_to_steps`` / ``util.fill_off_diagonal`` returns
(``<name>/<output>``) or the exception it raises (``<name>/error``, "Class: message"); written by
tools/make_golden.py --alignment.  Outputs of more than SHA_CELLS cells are stored as ``<name>/<output>_sha256``
(SHA-256 of the C-ordered bytes; the tests rebuild them from the seeded inputs).  tests/alignment_oracle.py must
reproduce every entry bit for bit.

``refuse`` names the cases the GPU declines with UnsupportedOnGPU although the reference runs them (a callable or
another scipy metric, a bool ``sim``)."""
from __future__ import annotations

import hashlib

import numpy as np

SHA_CELLS = 2000


def digest(a) -> str:
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def features(spec):
    """spec: (lead shape, K, N, dtype, seed[, special])."""
    lead, K, N, dtype, seed = spec[:5]
    x = np.random.default_rng(seed).random(tuple(lead) + (K, N)).astype(dtype)
    if len(spec) > 5 and spec[5] == "nan":
        x.reshape(-1)[x.size // 2] = np.nan
    return x


def cost(spec):
    """spec: (N, M, dtype, seed[, special])."""
    N, M, dtype, seed = spec[:4]
    c = np.random.default_rng(seed).random((N, M)).astype(dtype)
    special = spec[4] if len(spec) > 4 else None
    if special == "nan":
        c[N // 2, M // 2] = np.nan
    elif special == "inf":
        c[N // 2, :] = np.inf
    elif special == "inf_cell":
        c[N // 2, M // 3] = np.inf
    elif special == "negative":
        c[:] = -1.0
    return c


def similarity(spec):
    """spec: (kind, N, M, dtype, seed)."""
    kind, N, M, dtype, seed = spec
    rng = np.random.default_rng(seed)
    if kind == "zero":
        return np.zeros((N, M), dtype)
    if kind == "binary":
        return (rng.random((N, M)) > 0.6).astype(dtype)
    if kind == "bool":
        return rng.random((N, M)) > 0.6
    x = rng.random((N, M)) * (rng.random((N, M)) > 0.4)
    if kind == "nan":
        x[N // 2, M // 3] = np.nan
        x[1, 1] = np.nan
    return x.astype(dtype)


CASES = []


def _add(name, op, **kw):
    CASES.append(dict(name=name, op=op, **kw))


F64, F32 = np.float64, np.float32
# ---- dtw on features
for N, M in ((1, 1), (1, 7), (6, 1), (2, 2), (30, 45), (45, 30), (97, 64)):
    _add(f"dtw/size_{N}x{M}", "dtw", X=((), 12, N, F64, N), Y=((), 12, M, F64, M + 100), kw={})
_add("dtw/k1_1d", "dtw", X=((), 1, 40, F64, 1), Y=((), 1, 55, F64, 2), kw={}, squeeze=True)
for K in (1, 12, 20):
    for dt in (F32, F64):
        _add(f"dtw/k{K}_{np.dtype(dt).name}", "dtw", X=((), K, 50, dt, K), Y=((), K, 61, dt, K + 1), kw={})
_add("dtw/lead_f32", "dtw", X=((2, 3), 2, 40, F32, 3), Y=((2, 3), 2, 33, F32, 4), kw={})
_add("dtw/lead_f64", "dtw", X=((2, 3), 2, 40, F64, 5), Y=((6,), 2, 33, F64, 6), kw={})
_add("dtw/mixed_dtype", "dtw", X=((), 12, 40, F32, 7), Y=((), 12, 33, F64, 8), kw={})
for metric in ("euclidean", "sqeuclidean", "cityblock", "chebyshev", "cosine"):
    _add(f"dtw/metric_{metric}", "dtw", X=((), 12, 40, F64, 9), Y=((), 12, 52, F64, 10),
         kw=dict(metric=metric, return_steps=True))
for K in range(1, 18):
    _add(f"dtw/cosine_k{K}", "dtw", X=((), K, 20, F64, 20 + K), Y=((), K, 23, F64, 40 + K), kw=dict(metric="cosine"))
_add("dtw/metric_alias", "dtw", X=((), 12, 20, F64, 11), Y=((), 12, 21, F64, 12), kw=dict(metric="Euclid"))
_add("dtw/metric_correlation", "dtw", X=((), 12, 20, F64, 11), Y=((), 12, 21, F64, 12),
     kw=dict(metric="correlation"), refuse=True)
_add("dtw/metric_callable", "dtw", X=((), 12, 20, F64, 11), Y=((), 12, 21, F64, 12), kw=dict(metric="callable"),
     refuse=True)
_add("dtw/err_metric_unknown", "dtw", X=((), 12, 20, F64, 11), Y=((), 12, 21, F64, 12), kw=dict(metric="nosuch"))
_add("dtw/err_feature_mismatch", "dtw", X=((), 12, 20, F64, 11), Y=((), 11, 21, F64, 12), kw={})
_add("dtw/big_6000x7000", "dtw", X=((), 12, 6000, F32, 13), Y=((), 12, 7000, F32, 14), kw=dict(return_steps=True))
# ---- dtw on a cost matrix
_add("dtw/C_f32", "dtw", C=(40, 50, F32, 15), kw=dict(return_steps=True))
_add("dtw/C_f64", "dtw", C=(40, 50, F64, 16), kw=dict(return_steps=True))
_add("dtw/C_inf_cell", "dtw", C=(40, 50, F64, 17, "inf_cell"), kw={})
# ---- steps
_add("dtw/steps_custom", "dtw", C=(60, 80, F64, 18), kw=dict(step_sizes_sigma=np.array([[2, 1], [1, 2]]),
                                                             return_steps=True))
_add("dtw/steps_weights", "dtw", C=(60, 80, F64, 19),
     kw=dict(step_sizes_sigma=np.array([[2, 1], [1, 2], [1, 1]]), weights_add=np.array([0.1, 0.2, 0.0]),
             weights_mul=np.array([2.0, 1.5, 1.0]), return_steps=True))
_add("dtw/steps_default_weights", "dtw", C=(60, 80, F64, 20),
     kw=dict(weights_add=np.array([0.0, 0.3, 0.3]), weights_mul=np.array([1.0, 2.0, 2.0]), return_steps=True))
_add("dtw/steps_long", "dtw", C=(200, 300, F64, 21),
     kw=dict(step_sizes_sigma=np.array([[70, 1], [1, 1], [1, 3]]), subseq=True, return_steps=True))
_add("dtw/steps_diagonal", "dtw", C=(30, 50, F64, 22), kw=dict(step_sizes_sigma=np.array([[1, 1]]), subseq=True,
                                                               return_steps=True))
# ---- modes and constraints
_add("dtw/subseq_transposed", "dtw", X=((), 12, 80, F64, 23), Y=((), 12, 30, F64, 24),
     kw=dict(subseq=True, return_steps=True))
_add("dtw/subseq_wide", "dtw", X=((), 12, 30, F64, 25), Y=((), 12, 80, F64, 26), kw=dict(subseq=True))
_add("dtw/subseq_C_tall", "dtw", C=(70, 40, F64, 27), kw=dict(subseq=True))
_add("dtw/no_backtrack", "dtw", C=(40, 50, F64, 28), kw=dict(backtrack=False))
for rad in (0.05, 0.25, 0.5):
    for N, M in ((50, 50), (40, 70), (70, 40)):
        _add(f"dtw/band_{rad}_{N}x{M}", "dtw", C=(N, M, F64, 29), kw=dict(global_constraints=True, band_rad=rad,
                                                                           return_steps=True))
_add("dtw/band_X", "dtw", X=((), 12, 300, F32, 30), Y=((), 12, 260, F32, 31),
     kw=dict(global_constraints=True, band_rad=0.1, return_steps=True))
_add("dtw/band_zero", "dtw", C=(20, 20, F64, 32), kw=dict(global_constraints=True, band_rad=0.0))
# ---- data errors
_add("dtw/err_nan_X", "dtw", X=((), 12, 30, F64, 33, "nan"), Y=((), 12, 31, F64, 34), kw={})
_add("dtw/err_nan_C", "dtw", C=(30, 31, F32, 35, "nan"), kw={})
_add("dtw/err_inf_row", "dtw", C=(30, 31, F64, 36, "inf"), kw={})
_add("dtw/err_inf_row_subseq", "dtw", C=(30, 31, F64, 36, "inf"), kw=dict(subseq=True))
_add("dtw/err_inf_row_nobt", "dtw", C=(30, 31, F64, 36, "inf"), kw=dict(backtrack=False))
_add("dtw/err_negative_step", "dtw", C=(10, 11, F64, 37), kw=dict(step_sizes_sigma=np.array([[1, -1]])))
_add("dtw/err_weights_add", "dtw", C=(10, 11, F64, 37), kw=dict(weights_add=np.zeros(2)))
_add("dtw/err_weights_mul", "dtw", C=(10, 11, F64, 37), kw=dict(weights_mul=np.ones(4)))
_add("dtw/err_no_Y", "dtw", X=((), 12, 10, F64, 38), kw={})
_add("dtw/err_C_and_X", "dtw", X=((), 12, 10, F64, 38), C=(10, 11, F64, 37), kw={})
# ---- dtw_backtracking on the steps of a dtw run
_add("bt/default", "dtw_backtracking", C=(40, 50, F64, 39), kw={})
_add("bt/subseq_start", "dtw_backtracking", C=(40, 50, F64, 40), kw=dict(subseq=True, start=17))
_add("bt/subseq_nostart", "dtw_backtracking", C=(40, 50, F64, 40), kw=dict(subseq=True))
_add("bt/custom", "dtw_backtracking", C=(60, 80, F64, 18), kw=dict(step_sizes_sigma=np.array([[2, 1], [1, 2]])))
_add("bt/err_start", "dtw_backtracking", C=(10, 11, F64, 41), kw=dict(start=3))
# ---- path_to_steps on a dtw path
_add("pts/forward", "path_to_steps", C=(40, 70, F64, 42), kw={})
_add("pts/inverse", "path_to_steps", C=(40, 70, F64, 42), kw=dict(inverse=True))
# ---- fill_off_diagonal
for N, M, rad in ((8, 8, 0.25), (8, 12, 0.25), (12, 8, 0.25), (9, 9, 0.5), (20, 7, 0.1)):
    _add(f"fill/{N}x{M}_{rad}", "fill_off_diagonal", C=(N, M, F64, 43), kw=dict(radius=rad, value=np.inf))
# ---- rqa
for kind in ("binary", "cont"):
    for dt in (F32, F64):
        for knight in (True, False):
            for gaps in ((1, 1), (0.25, 0.5), (np.inf, np.inf)):
                _add(f"rqa/{kind}_{np.dtype(dt).name}_{'knight' if knight else 'diag'}_{gaps[0]}_{gaps[1]}", "rqa",
                     sim=(kind, 60, 70, dt, 44), kw=dict(gap_onset=gaps[0], gap_extend=gaps[1], knight_moves=knight))
for N, M in ((1, 1), (1, 9), (8, 1), (2, 2), (2, 9), (9, 2), (70, 60)):
    _add(f"rqa/size_{N}x{M}", "rqa", sim=("cont", N, M, F64, 45), kw={})
_add("rqa/nan_f32", "rqa", sim=("nan", 40, 50, F32, 46), kw={})
_add("rqa/nan_f64_inf_gaps", "rqa", sim=("nan", 40, 50, F64, 46), kw=dict(gap_onset=np.inf, gap_extend=np.inf))
_add("rqa/no_backtrack", "rqa", sim=("cont", 40, 50, F64, 47), kw=dict(backtrack=False))
_add("rqa/zero", "rqa", sim=("zero", 30, 40, F64, 48), kw={})
_add("rqa/big_f32", "rqa", sim=("cont", 500, 600, F32, 49), kw=dict(gap_onset=2, gap_extend=3))
_add("rqa/bool", "rqa", sim=("bool", 20, 30, None, 50), kw={}, refuse=True)
_add("rqa/err_gap_onset", "rqa", sim=("cont", 5, 5, F64, 51), kw=dict(gap_onset=-1))
_add("rqa/err_gap_extend", "rqa", sim=("cont", 5, 5, F64, 51), kw=dict(gap_extend=-1))

BY_NAME = {c["name"]: c for c in CASES}


def _metric(kw):
    kw = dict(kw)
    if kw.get("metric") == "callable":
        kw["metric"] = lambda u, v: float(np.abs(u - v).sum())
    return kw


def inputs(case):
    """(X, Y, C, sim) host inputs of a case (None where absent)."""
    X = features(case["X"]) if "X" in case else None
    if X is not None and case.get("squeeze"):
        X = X[0]
    Y = features(case["Y"]) if "Y" in case else None
    if Y is not None and case.get("squeeze"):
        Y = Y[0]
    C = cost(case["C"]) if "C" in case else None
    sim = similarity(case["sim"]) if "sim" in case else None
    return X, Y, C, sim


def call(lib, case, X=None, Y=None, C=None, sim=None):
    """Run one case through ``lib`` (the reference, or librosa_b200) on the given inputs (default: the case's host
    inputs): {output name: array} or {"error": "Class: message"}."""
    hx, hy, hc, hs = inputs(case)
    X = hx if X is None else X
    Y = hy if Y is None else Y
    C = hc if C is None else C
    sim = hs if sim is None else sim
    op, kw = case["op"], _metric(case["kw"])
    try:
        if op == "dtw":
            out = lib.sequence.dtw(X, Y, C=C, **kw) if X is not None else lib.sequence.dtw(C=C, **kw)
            if not isinstance(out, tuple):
                out = (out,)
            names = ["D"] + (["wp"] if kw.get("backtrack", True) else []) + (["steps"] if kw.get("return_steps")
                                                                             else [])
            return dict(zip(names, out))
        if op in ("dtw_backtracking", "path_to_steps"):
            bt_kw = {k: v for k, v in kw.items() if k != "start"} if op == "dtw_backtracking" else {}
            D, wp, steps = lib.sequence.dtw(C=C, return_steps=True, **bt_kw)
            if op == "path_to_steps":
                return {"steps": lib.sequence.path_to_steps(wp, **kw)}
            return {"wp": lib.sequence.dtw_backtracking(steps, **kw), "dtw_wp": wp}
        if op == "fill_off_diagonal":
            x = np.array(C)
            lib.util.fill_off_diagonal(x, **kw)
            return {"x": x}
        if op == "rqa":
            out = lib.sequence.rqa(sim, **kw)
            return {"score": out} if not kw.get("backtrack", True) else {"score": out[0], "path": out[1]}
    except Exception as exc:  # noqa: BLE001 - the fixture records the reference's exception
        if type(exc).__name__ == "UnsupportedOnGPU":
            raise
        return {"error": f"{type(exc).__name__}: {exc}"}
    raise ValueError(op)


def pack(name, got):
    """Fixture entries of one outcome: small arrays as they are, large ones as SHA-256."""
    store = {}
    for key, arr in got.items():
        if key == "error":
            store[f"{name}/error"] = np.array(arr)
            continue
        arr = np.asarray(arr)
        if arr.size > SHA_CELLS and arr.ndim == 2 and arr.shape[1] != 2:
            store[f"{name}/{key}_sha256"] = np.array(digest(arr))
            store[f"{name}/{key}_meta"] = np.array(f"{arr.dtype.str} {arr.shape}")
        else:
            store[f"{name}/{key}"] = np.ascontiguousarray(arr)
    return store


def matches(golden, name, got):
    """Compare an outcome with the fixture bit for bit: (ok, what differs)."""
    if "error" in got:
        want = golden.get(name + "/error")
        return (want is not None and str(want) == got["error"]), f"error {got['error']!r} vs {want}"
    for key, arr in got.items():
        arr = np.asarray(arr)
        if name + "/" + key in golden:
            want = golden[name + "/" + key]
            if want.dtype != arr.dtype or want.shape != arr.shape or want.tobytes() != np.ascontiguousarray(arr).tobytes():
                return False, f"{key}: {arr.dtype}{arr.shape} vs {want.dtype}{want.shape}"
        elif name + "/" + key + "_sha256" in golden:
            meta = f"{arr.dtype.str} {arr.shape}"
            if str(golden[name + "/" + key + "_meta"]) != meta or digest(arr) != str(golden[name + "/" + key + "_sha256"]):
                return False, f"{key}: sha256 / {meta}"
        else:
            return False, f"{key} not in the fixture"
    return True, ""
