"""segment.recurrence_matrix and decompose.nn_filter without a GPU: the NumPy oracle (tests/nn_filter_oracle.py)
against tests/golden/nn_filter_v1.npz, and the argument errors and refusals raised before any device work."""
from __future__ import annotations

import os

import numpy as np
import pytest
import scipy.sparse

import nn_filter_cases as NC
import nn_filter_oracle as NO

GOLDEN = np.load(os.path.join(os.path.dirname(__file__), "golden", "nn_filter_v1.npz"))
NN = [c for c in NC.CASES if c["fn"] == "nn" and f"{c['name']}/out" in GOLDEN.files]
REC = [c for c in NC.CASES if c["fn"] == "rec" and f"{c['name']}/error" not in GOLDEN.files]
ERR = [c for c in NC.CASES if f"{c['name']}/error" in GOLDEN.files]
DELTA32 = 1e-5   # DESIGN §4.22
DELTA64 = 1e-9
# Frames that may be excused by a boundary tie against the reference; every other case has none.  The silent frames
# of the 400-frame float32 cosine cases are at distance exactly 1 from every frame, so each of their rows is one tie
# class; the integer case has exact integer ties.
SILENT = set(range(5, 5 + 10 * NC.SPEC32[3], 10))
MAY_EXCUSE = {"spec32_cosine": SILENT, "spec32_cosine_distance": SILENT}
MAX_EXCUSED = {"int_data": 1}


@pytest.mark.parametrize("case", NN, ids=lambda c: c["name"])
def test_oracle_aggregation_reproduces_the_fixture(case):
    S, _ = NC.filter_input(case)
    got = NO.aggregate(S, NC.unpack(GOLDEN, case["name"]), NC.AGG[case["agg"]])
    want = GOLDEN[f"{case['name']}/out"]
    assert got.dtype == want.dtype and np.array_equal(got.view(np.uint8), want.view(np.uint8))


@pytest.mark.parametrize("case", REC, ids=lambda c: c["name"])
def test_oracle_graph_equals_the_fixture_except_boundary_ties(case):
    x = NC.case_data(case)
    kw = {key: case["kw"][key] for key in ("k", "width", "metric", "sym", "mode", "self", "axis") if key in case["kw"]}
    rec, D = NO.graph(x, **kw)
    ref = NC.unpack(GOLDEN, case["name"])
    t = D.shape[0]
    delta = DELTA32 if (kw.get("metric") == "cosine" and x.dtype == np.float32) else DELTA64
    rows = NO.excused_rows(rec, ref, D, k=NO.case_k(t, kw), width=kw.get("width", 1),
                           mode=kw.get("mode", "connectivity"), sym=kw.get("sym", False), delta=delta)
    if case["name"] in MAY_EXCUSE:
        assert set(rows) <= MAY_EXCUSE[case["name"]], rows
    else:
        assert len(rows) <= MAX_EXCUSED.get(case["name"], 0), rows


def test_connectivity_keeps_the_lowest_indexed_links_not_the_nearest():
    case = NC.BY_NAME["spec32_cosine"]
    x = NC.case_data(case)
    ref = NC.unpack(GOLDEN, case["name"])
    D = NO.distances(NO.frames(x), "cosine")
    t, width = D.shape[0], 3
    k = int(2 * np.ceil(np.sqrt(t - 2 * width + 1)))
    lowest = nearest = 0
    for i in range(t):
        order = np.lexsort((np.arange(t), D[i]))[:k + 2 * width]
        surv = [j for j in order if abs(j - i) >= width]
        got = set(ref.indices[ref.indptr[i]:ref.indptr[i + 1]].tolist())
        lowest += got == set(sorted(surv)[:k])
        nearest += got == set(surv[:k])
    assert lowest >= 0.9 * t and nearest < 0.1 * t, (lowest, nearest)


def _no_device(monkeypatch):
    from librosa_b200 import _native as nat
    from librosa_b200 import _pipeline as pl

    def no_device(*a, **k):
        raise AssertionError("device work before the check")

    monkeypatch.setattr(pl, "StagedInput", no_device)
    monkeypatch.setattr(nat, "default_context", no_device)
    monkeypatch.setattr(nat, "lib", no_device)


@pytest.mark.parametrize("case", [c for c in ERR if c["name"] != "err_no_neighbors"], ids=lambda c: c["name"])
def test_errors_match_the_reference_before_any_device_work(case, monkeypatch):
    import librosa_b200 as lb

    _no_device(monkeypatch)
    want = str(GOLDEN[f"{case['name']}/error"])
    with pytest.raises(Exception) as ei:
        if case["fn"] == "rec":
            lb.segment.recurrence_matrix(NC.case_data(case), sparse=True, **case["kw"])
        else:
            S, _ = NC.filter_input(case)
            lb.decompose.nn_filter(S[:, :-1], rec=NC.unpack(GOLDEN, case["name"]), aggregate=np.mean)
    assert f"{type(ei.value).__name__}: {ei.value}" == want


REFUSALS = [
    ("rec", dict(metric="manhattan")),
    ("rec", dict(mode="affinity", full=True)),
    ("rec", dict(mode="distance", full=True)),
    ("rec", dict(mode="connectivity", full=True)),   # the reference skips width and top-k in this mode too
    ("rec", dict(full=True)),
    ("nn", dict(full=True)),
    ("rec", dict(mode="affinity", bandwidth=np.ones((120, 120)))),
    ("rec", dict(k=4200)),
    ("nn", dict(aggregate=np.max)),
    ("nn_complex", {}),
    ("nn_int", {}),
]


@pytest.mark.parametrize("kind,kw", REFUSALS)
def test_refusals_before_any_device_work(kind, kw, monkeypatch):
    import librosa_b200 as lb
    from librosa_b200 import _native as nat

    _no_device(monkeypatch)
    x = NC.data(((40, 120), 5, np.float64)) if kind != "rec" or "k" not in kw else NC.data(((4, 5000), 5, np.float32))
    with pytest.raises(nat.UnsupportedOnGPU):
        if kind == "rec":
            lb.segment.recurrence_matrix(x, **kw)
        elif kind == "nn":
            lb.decompose.nn_filter(x, **kw)
        elif kind == "nn_complex":
            lb.decompose.nn_filter(x.astype(np.complex64))
        else:
            lb.decompose.nn_filter(x.astype(np.int32))


def test_too_many_frames_is_refused_before_any_device_work(monkeypatch):
    import librosa_b200 as lb
    from librosa_b200 import _native as nat

    _no_device(monkeypatch)
    with pytest.raises(nat.UnsupportedOnGPU):
        lb.segment.recurrence_matrix(np.zeros((1, 65537), np.float32), k=2)


def test_non_finite_host_data_raises_value_error_before_any_device_work(monkeypatch):
    import librosa_b200 as lb

    _no_device(monkeypatch)
    x = NC.data(((40, 120), 5, np.float64))
    x[3, 9] = np.nan
    with pytest.raises(ValueError, match="NaN or infinity"):
        lb.segment.recurrence_matrix(x)


def test_sparse_host_rec_is_taken_through_csc_array():
    # explicit stored zeros count as neighbours, as in the reference's loop
    rec = scipy.sparse.csr_array((np.array([0.0, 1.0]), np.array([1, 2]), np.array([0, 2, 2, 2])), shape=(3, 3))
    S = np.arange(6, dtype=np.float32).reshape(2, 3)
    out = NO.aggregate(S, rec, np.mean)
    assert np.array_equal(out[:, 1], S[:, 0]) and np.array_equal(out[:, 0], S[:, 0])
