"""segment.recurrence_matrix and decompose.nn_filter on the GPU: nn_filter given the reference's rec bit-identical to
the reference for every aggregate and dtype; the GPU graph equal to the float64 oracle's and the reference's except on
frames where two candidates straddle a selection boundary within the distances' resolution; d(i, j) == d(j, i) bit for
bit; nn_filter end to end equal to the oracle's aggregation over the GPU's own graph; host, device "c" and device "ft"
inputs bit-identical; a dense device rec of every dtype equal to the host one; non-finite data refused alike;
t = 20 000 against the oracle on sampled rows; launch budgets."""
from __future__ import annotations

import os

import numpy as np
import pytest
import scipy.sparse

import nn_filter_cases as NC
import nn_filter_oracle as NO
import librosa_b200 as lb
from librosa_b200 import _native as nat

pytestmark = pytest.mark.gpu

GOLDEN = np.load(os.path.join(os.path.dirname(__file__), "golden", "nn_filter_v1.npz"))
NN = [c for c in NC.CASES if c["fn"] == "nn" and f"{c['name']}/out" in GOLDEN.files]
REC = [c for c in NC.CASES if c["fn"] == "rec" and f"{c['name']}/error" not in GOLDEN.files]
ERR = [c for c in NC.CASES if f"{c['name']}/error" in GOLDEN.files]
DELTA64 = 1e-9     # relative agreement of two float64 distance computations (DESIGN §4.22)
DELTA32 = 1e-5     # float32 cosine distances of the reference (DESIGN §4.22)


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint8)


@pytest.mark.parametrize("case", NN, ids=lambda c: c["name"])
def test_nn_filter_given_the_reference_rec_is_bit_identical(case):
    S, _ = NC.filter_input(case)
    rec = NC.unpack(GOLDEN, case["name"])
    got = lb.decompose.nn_filter(S, rec=rec, aggregate=NC.AGG[case["agg"]])
    want = GOLDEN[f"{case['name']}/out"]
    assert got.dtype == want.dtype and got.shape == want.shape
    assert np.array_equal(_bits(got), _bits(want))


@pytest.mark.parametrize("case", NN[:4], ids=lambda c: c["name"])
def test_nn_filter_device_layouts_and_dense_device_rec(case):
    S, _ = NC.filter_input(case)
    rec = NC.unpack(GOLDEN, case["name"])
    want = lb.decompose.nn_filter(S, rec=rec, aggregate=NC.AGG[case["agg"]])
    ctx = lb.default_context()
    for layout in ("c", "ft"):
        mem = ctx.to_device(S) if layout == "c" else ctx.to_device(np.swapaxes(S, -1, -2).copy())
        dS = mem if layout == "c" else nat.DeviceArray(ctx, mem.ptr, S.shape, S.dtype, layout="ft", owner=False)
        got = lb.decompose.nn_filter(dS, rec=rec, aggregate=NC.AGG[case["agg"]])
        assert got.layout == "ft"
        assert np.array_equal(_bits(got.get()), _bits(want)), layout
    dense = ctx.to_device(rec.toarray())
    got = lb.decompose.nn_filter(S, rec=dense, aggregate=NC.AGG[case["agg"]])
    assert np.array_equal(_bits(got), _bits(want))


def _excused(case, got, want, D, delta):
    kw = case["kw"]
    return NO.excused_rows(got, want, D, k=NO.case_k(D.shape[0], kw), width=kw.get("width", 1),
                           mode=kw.get("mode", "connectivity"), sym=kw.get("sym", False), delta=delta)


# Frames that may differ from the reference through a boundary tie; every other case has none.  The silent frames of
# the 400-frame float32 cosine cases are at distance exactly 1 from every frame (each of their rows is one tie class);
# the integer case has exact integer ties.
SILENT = set(range(5, 5 + 10 * NC.SPEC32[3], 10))
MAY_EXCUSE = {"spec32_cosine": SILENT, "spec32_cosine_distance": SILENT}
MAX_EXCUSED = {"int_data": 1}


@pytest.mark.parametrize("case", REC, ids=lambda c: c["name"])
def test_graph_equals_the_oracle_and_the_reference_except_boundary_ties(case):
    x = NC.case_data(case)
    kw = dict(case["kw"])
    got = lb.segment.recurrence_matrix(x, sparse=True, **kw)
    ref = NC.unpack(GOLDEN, case["name"])
    assert got.dtype == ref.dtype and got.shape == ref.shape
    okw = {key: kw[key] for key in ("k", "width", "metric", "sym", "mode", "self", "axis") if key in kw}
    orc, D = NO.graph(x, **okw)
    # against the float64 oracle, which orders candidates by (distance, index) as the GPU does: boundary ties at the
    # float64 resolution only
    rows = _excused(case, got, orc, D, DELTA64)
    assert len(rows) <= MAX_EXCUSED.get(case["name"], 0), rows
    # against the reference: boundary ties at the resolution of its distances (float32 GEMM for cosine of float32)
    delta = DELTA32 if (kw.get("metric") == "cosine" and x.dtype == np.float32) else DELTA64
    rows = _excused(case, got, ref, D, delta)
    if case["name"] in MAY_EXCUSE:
        assert set(rows) <= MAY_EXCUSE[case["name"]], rows
    else:
        assert len(rows) <= MAX_EXCUSED.get(case["name"], 0), rows
    if kw.get("mode") == "distance" and not rows:
        assert np.allclose(got.data, ref.data, rtol=2e-6 if got.dtype == np.float32 else 1e-10, atol=1e-6)
    if kw.get("mode") == "affinity" and not rows:
        # the reference's float32 cosine distances come from a float32 GEMM (about 1e-6 absolute error), which the
        # data-driven bandwidths (about 1e-2 here) magnify in exp(-d / bandwidth)
        assert np.allclose(got.data, ref.data, rtol=2e-3 if got.dtype == np.float32 else 1e-9, atol=1e-7)


@pytest.mark.parametrize("case", [c for c in ERR if c["fn"] == "rec"], ids=lambda c: c["name"])
def test_errors_match_the_reference(case):
    want = str(GOLDEN[f"{case['name']}/error"])
    with pytest.raises(Exception) as ei:
        lb.segment.recurrence_matrix(NC.case_data(case), sparse=True, **case["kw"])
    assert f"{type(ei.value).__name__}: {ei.value}" == want


@pytest.mark.parametrize("metric", ["euclidean", "cosine"])
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_distances_are_symmetric_bit_for_bit(metric, dtype):
    x = NC.data(((70, 300), 11, dtype, 10))
    R = lb.segment.recurrence_matrix(x, k=80, width=1, metric=metric, mode="distance")
    both = (R != 0) & (R.T != 0)
    assert both.sum() > 1000
    assert np.array_equal(R[both], R.T[both])


@pytest.mark.parametrize("agg", [np.mean, np.median, np.average])
@pytest.mark.parametrize("mode", ["connectivity", "affinity"])
def test_nn_filter_end_to_end_equals_the_oracle_on_its_own_graph(agg, mode):
    S = NC.data(((129, 300), 12, np.float32, 20))
    kw = dict(metric="cosine", width=3, mode=mode)
    got = lb.decompose.nn_filter(S, aggregate=agg, **kw)
    rec = lb.segment.recurrence_matrix(S, sparse=True, **kw)
    want = NO.aggregate(S, rec, agg)
    assert np.array_equal(_bits(got), _bits(want))


def test_host_c_and_ft_inputs_give_identical_graphs():
    # the device strides read the features in the host's F-order flattening ((lead, feature) = lead * d + feature),
    # so pack and Gram run the same operations: bit-identical graphs
    x = NC.data(((2, 48, 200), 13, np.float32))
    host = lb.segment.recurrence_matrix(x, width=2, mode="distance")
    ctx = lb.default_context()
    dc = ctx.to_device(x)
    got_c = lb.segment.recurrence_matrix(dc, width=2, mode="distance").get()
    ft = ctx.to_device(np.swapaxes(x, -1, -2).copy())
    dft = nat.DeviceArray(ctx, ft.ptr, x.shape, x.dtype, layout="ft", owner=False)
    got_ft = lb.segment.recurrence_matrix(dft, width=2, mode="distance").get()
    assert got_c.dtype == host.dtype and got_ft.dtype == host.dtype
    assert np.array_equal(_bits(got_c), _bits(host)) and np.array_equal(_bits(got_ft), _bits(host))
    assert isinstance(lb.segment.recurrence_matrix(dc, width=2, sparse=True), scipy.sparse.csc_array)


def test_non_finite_device_data_raises_value_error_like_host_data():
    x = NC.data(((40, 120), 5, np.float32))
    x[3, 9] = np.inf
    with pytest.raises(ValueError, match="NaN or infinity"):
        lb.segment.recurrence_matrix(x)
    with pytest.raises(ValueError, match="NaN or infinity"):
        lb.segment.recurrence_matrix(lb.default_context().to_device(x))


def test_dense_device_rec_of_every_dtype_compacts_like_csc_array():
    t = 700
    rng = np.random.default_rng(17)
    S = NC.data(((33, t), 18, np.float32))
    dense = np.where(rng.random((t, t)) < 0.02, rng.random((t, t)), 0.0)
    dense[:, 5] = 0.0   # a frame without neighbours copies S
    ctx = lb.default_context()
    for dt in (np.float32, np.float64, np.bool_):
        rec = dense.astype(dt)
        for agg in (np.mean, np.median, np.average):
            if agg is np.average and dt is np.bool_:
                continue
            want = lb.decompose.nn_filter(S, rec=rec, aggregate=agg)
            got = lb.decompose.nn_filter(S, rec=ctx.to_device(rec), aggregate=agg)
            assert np.array_equal(_bits(got), _bits(want)), (dt, agg)
            assert np.array_equal(_bits(want), _bits(NO.aggregate(S, rec, agg))), (dt, agg)


def test_large_t_agrees_with_the_oracle_on_sampled_rows():
    t, d = 20000, 24
    rng = np.random.default_rng(14)
    x = rng.standard_normal((d, t)).astype(np.float64)
    k = 10
    got = lb.segment.recurrence_matrix(x, k=k, width=2, sparse=True, mode="distance")
    X = NO.frames(x)
    sq = np.einsum("ij,ij->i", X, X)
    for i in rng.choice(t, 200, replace=False):
        Di = np.sqrt(np.maximum(sq[i] + sq - 2.0 * X @ X[i], 0.0))
        Di[i] = np.inf
        order = np.lexsort((np.arange(t), Di))[:k + 4]
        surv = [j for j in order if abs(j - i) >= 2][:k]
        g = got.indices[got.indptr[i]:got.indptr[i + 1]]
        assert np.array_equal(g, np.sort(surv)) or NO.boundary_tie(Di, i, k, 2, "distance", DELTA64), i


def test_launch_budgets():
    ctx = lb.default_context()
    x = ctx.to_device(NC.data(((40, 300), 15, np.float32)))
    n0 = ctx.launch_count
    lb.segment.recurrence_matrix(x, k=10, mode="connectivity")
    # pack, one row block (distances + selection), graph, dense scatter
    assert ctx.launch_count - n0 == 5
    n0 = ctx.launch_count
    lb.segment.recurrence_matrix(x, k=10, mode="affinity", sparse=True)
    # ... + the med_k_scalar median + the affinity values, no scatter
    assert ctx.launch_count - n0 == 6
    S = ctx.to_device(NC.data(((129, 300), 16, np.float32)))
    n0 = ctx.launch_count
    lb.decompose.nn_filter(S, aggregate=np.median, k=10)
    # transpose to "ft", the graph (4), the aggregation
    assert ctx.launch_count - n0 == 6
