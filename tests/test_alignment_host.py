"""Alignment without a GPU: tests/alignment_oracle.py reproduces every entry of tests/golden/alignment_v1.npz (written
by the unmodified reference), ``util.fill_off_diagonal`` and ``sequence.path_to_steps`` match it, the device's
feature-offset table matches NumPy's swapaxes / reshape, and every error decided on the host is the reference's."""
import os
import warnings

import numpy as np
import pytest

import alignment_cases as AC
import alignment_oracle as AO
import librosa_b200 as lb
from librosa_b200 import sequence as seq

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# raised before any device work
HOST_ERRORS = ["dtw/err_metric_unknown", "dtw/err_feature_mismatch", "dtw/err_negative_step", "dtw/err_weights_add",
               "dtw/err_weights_mul", "dtw/err_no_Y", "dtw/err_C_and_X", "dtw/err_nan_C", "rqa/err_gap_onset",
               "rqa/err_gap_extend"]


@pytest.fixture(scope="module")
def golden():
    with np.load(os.path.join(ROOT, "tests", "golden", "alignment_v1.npz")) as z:
        return {k: z[k] for k in z.files}


@pytest.mark.parametrize("name", [c["name"] for c in AC.CASES])
def test_oracle_matches_fixture(golden, name):
    if name + "/error" in golden:
        pytest.skip("an error case of the reference")
    case = AC.BY_NAME[name]
    if case.get("refuse") and case["op"] == "dtw":
        pytest.skip("a metric the oracle does not restate")
    if case["op"] == "rqa" and case["sim"][0] == "bool":
        pytest.skip("a bool similarity matrix")
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        got = AO.run(case)
    ok, why = AC.matches(golden, name, got)
    assert ok, why


@pytest.mark.parametrize("name", [c["name"] for c in AC.CASES if c["op"] in ("fill_off_diagonal", "path_to_steps")])
def test_host_functions_match_fixture(golden, name):
    case = AC.BY_NAME[name]
    _, _, C, _ = AC.inputs(case)
    if case["op"] == "fill_off_diagonal":
        x = np.array(C)
        assert lb.util.fill_off_diagonal(x, **case["kw"]) is None
        got = {"x": x}
    else:
        _, wp, _ = AO.dtw(C=C)
        got = {"steps": lb.sequence.path_to_steps(wp, **case["kw"])}
    ok, why = AC.matches(golden, name, got)
    assert ok, why


@pytest.mark.parametrize("shape", [(7,), (12, 9), (2, 3, 4, 5), (3, 1, 6), (1, 5)])
def test_feature_offsets(shape):
    x = np.atleast_2d(np.arange(int(np.prod(shape))).reshape(shape))
    want = np.swapaxes(x, -1, 0).reshape((x.shape[-1], -1), order="F")
    off = seq._feature_offsets(x.shape)
    flat = x.reshape(-1)
    got = flat[off[None, :] + np.arange(x.shape[-1])[:, None]]
    assert np.array_equal(got, want)


@pytest.mark.parametrize("name", HOST_ERRORS + ["bt/err_start"])
def test_host_errors(golden, name):
    case = AC.BY_NAME[name]
    if case["op"] == "dtw_backtracking":
        with pytest.raises(lb.ParameterError) as exc:
            lb.sequence.dtw_backtracking(np.zeros((10, 11), np.int32), **case["kw"])
    else:
        got = AC.call(lb, case)
        assert "error" in got, name
        exc = None
    want = str(golden[name + "/error"])
    assert (f"{type(exc.value).__name__}: {exc.value}" if exc else got["error"]) == want


@pytest.mark.parametrize("name", [c["name"] for c in AC.CASES if c.get("refuse")])
def test_refusals(name):
    with pytest.raises(lb.UnsupportedOnGPU):
        AC.call(lb, AC.BY_NAME[name])


def test_band_matches_fill_off_diagonal():
    for shape in ((8, 8), (8, 12), (12, 8), (9, 30), (31, 5)):
        for rad in (0.0, 0.1, 0.25, 0.5, 1.0, -0.2):
            x = np.ones(shape)
            lb.util.fill_off_diagonal(x, radius=rad)
            lo, hi = seq._band(shape, rad)
            d = np.arange(shape[1])[None, :] - np.arange(shape[0])[:, None]
            assert np.array_equal(x == 1, (d > lo) & (d < hi)), (shape, rad)


def test_other_refusals():
    with pytest.raises(lb.UnsupportedOnGPU, match="int64"):
        lb.sequence.rqa(np.ones((3, 4), np.int64))
    with pytest.raises(lb.UnsupportedOnGPU):
        lb.sequence.dtw_backtracking(np.zeros((4, 5), np.int32), subseq=True, start=5)
    with pytest.raises(lb.UnsupportedOnGPU):
        lb.util.fill_off_diagonal(lb.DeviceArray(None, 0, (3, 3), np.float64, owner=False), radius=0.25)
