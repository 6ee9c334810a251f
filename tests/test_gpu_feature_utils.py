"""feature.delta / feature.stack_memory on the GPU: every case of tests/golden/feature_utils_v1.npz bit-identical to the
oracle (so to the reference everywhere but the interp edges, which the host test holds to their tolerance), with the
reference's dtype, shape and non-finite positions; the reference's errors; host and device calls and both device
layouts identical; one launch per call; delta of device MFCCs; 70 001 lines in one call; rows longer than the
shared-memory tile."""
from __future__ import annotations

import os
import warnings

import numpy as np
import pytest

import feature_utils_cases as FU
import feature_utils_oracle as FO
import librosa_b200 as lb
from librosa_b200 import _native as nat

pytestmark = pytest.mark.gpu

GOLDEN = np.load(os.path.join(os.path.dirname(__file__), "golden", "feature_utils_v1.npz"))
RUNS = [c for c in FU.CASES if f"{c['name']}/out" in GOLDEN.files]
ERRORS = [c for c in FU.CASES if f"{c['name']}/error" in GOLDEN.files]


def _bytes(a):
    return np.ascontiguousarray(a).tobytes()


def _oracle(case, x=None):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        if x is None:
            return FO.run(case)
        return FO.delta(x, **case["kw"]) if case["fn"] == "delta" else FO.stack_memory(x, **case["kw"])


def _same(case, got, want):
    assert got.dtype == want.dtype and got.shape == want.shape, (got.dtype, want.dtype, got.shape, want.shape)
    if case["fn"] == "stack_memory":
        keep = ~FU.empty_cells(case)
        got, want = np.where(keep, got, 0), np.where(keep, want, 0)
    assert _bytes(got) == _bytes(want), case["name"]


@pytest.mark.parametrize("case", RUNS, ids=lambda c: c["name"])
def test_every_case_matches_the_oracle(case):
    ref = GOLDEN[f"{case['name']}/out"]
    got = FU.call(lb, case)
    assert isinstance(got, np.ndarray) and got.flags.c_contiguous
    _same(case, got, _oracle(case))
    assert got.dtype == ref.dtype and got.shape == ref.shape
    if got.dtype.kind == "f":
        for test in (np.isnan, np.isposinf, np.isneginf):
            keep = ~FU.empty_cells(case) if case["fn"] == "stack_memory" else True
            assert np.array_equal(test(got) & keep, test(ref) & keep)


@pytest.mark.parametrize("case", ERRORS, ids=lambda c: c["name"])
def test_errors_match_the_reference(case):
    want = str(GOLDEN[f"{case['name']}/error"])
    with pytest.raises(Exception) as info:
        FU.call(lb, case)
    assert f"{type(info.value).__name__}: {info.value}" == want


def _device(x, layout):
    ctx = lb.default_context()
    if layout == "c":
        return ctx.to_device(x)
    d = nat.DeviceArray.empty(ctx, x.shape, x.dtype, layout="ft")
    return d.set(np.swapaxes(x, -1, -2))


DEVICE = [c for c in RUNS if np.dtype(c["spec"][1]) in (np.float32, np.float64) or c["fn"] == "stack_memory"]


@pytest.mark.parametrize("case", DEVICE, ids=lambda c: c["name"])
def test_device_calls_equal_host_calls(case):
    x = np.atleast_2d(FU.data(case["spec"])) if case["fn"] == "stack_memory" else FU.data(case["spec"])
    host = FU.call(lb, case, x)
    ctx = lb.default_context()
    for layout in ("c", "ft") if x.ndim >= 2 else ("c",):
        d = _device(x, layout)
        before = ctx.launch_count
        out = FU.call(lb, case, d)
        assert ctx.launch_count - before == 1
        assert isinstance(out, nat.DeviceArray)
        assert out.layout == (layout if case["fn"] == "delta" else "c")
        _same(case, out.get(), host)


def test_one_launch_per_host_call():
    ctx = lb.default_context()
    x = FU.data(((20, 431), np.float32, 3))
    for fn, kw in ((lb.feature.delta, {}), (lb.feature.delta, {"order": 2, "mode": "nearest"}),
                   (lb.feature.stack_memory, {"n_steps": 3})):
        before = ctx.launch_count
        fn(x, **kw)
        assert ctx.launch_count - before == 1


def test_delta_of_device_mfcc():
    rng = np.random.default_rng(7)
    y = (0.1 * rng.standard_normal((4, 22050 * 2))).astype(np.float32)
    d_y = lb.to_device(y)
    M = lb.feature.mfcc(y=d_y, sr=22050)
    assert isinstance(M, nat.DeviceArray)
    host = M.get()
    for order in (1, 2):
        got = lb.feature.delta(M, order=order)
        want = lb.feature.delta(host, order=order)
        assert got.layout == M.layout and got.shape == host.shape
        assert _bytes(got.get()) == _bytes(want)
        ref = FO.delta(host, order=order)
        assert _bytes(want) == _bytes(ref)
    S = lb.feature.stack_memory(M, n_steps=3)
    assert _bytes(S.get()) == _bytes(lb.feature.stack_memory(host, n_steps=3))


@pytest.mark.parametrize("mode", FU.MODES)
def test_many_lines_in_one_call(mode):
    ctx = lb.default_context()
    x = FU.data(((70001, 12), np.float32, 8))
    before = ctx.launch_count
    got = lb.feature.delta(x, width=5, mode=mode)
    assert ctx.launch_count - before == 1
    assert _bytes(got) == _bytes(FO.delta(x, width=5, mode=mode))
    for i in (0, 65534, 65535, 65536, 70000):
        assert _bytes(got[i]) == _bytes(lb.feature.delta(x[i], width=5, mode=mode))
    # the strided path: 70 001 lines along the first axis
    xt = np.ascontiguousarray(x.T)
    got = lb.feature.delta(xt, width=5, mode=mode, axis=0)
    assert _bytes(got) == _bytes(FO.delta(xt, width=5, mode=mode, axis=0))
    assert _bytes(got[:, 65535]) == _bytes(lb.feature.delta(xt[:, 65535], width=5, mode=mode))


def test_stack_memory_many_clips():
    x = FU.data(((70001, 2, 5), np.float32, 9))
    got = lb.feature.stack_memory(x, n_steps=3, delay=-1, mode="edge")
    assert _bytes(got) == _bytes(FO.stack_memory(x, n_steps=3, delay=-1, mode="edge"))
    assert _bytes(got[65535]) == _bytes(lb.feature.stack_memory(x[65535], n_steps=3, delay=-1, mode="edge"))


@pytest.mark.parametrize("mode", FU.MODES)
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_rows_longer_than_the_tile(mode, dtype):
    x = FU.data(((3, 2500), dtype, 10))
    for width, order, polyorder in ((9, 1, 1), (31, 2, 4), (255, 3, 3)):
        got = lb.feature.delta(x, width=width, order=order, polyorder=polyorder, mode=mode)
        assert _bytes(got) == _bytes(FO.delta(x, width=width, order=order, polyorder=polyorder, mode=mode))
    got = lb.feature.stack_memory(x, n_steps=4, delay=-700, mode="reflect")
    assert _bytes(got) == _bytes(FO.stack_memory(x, n_steps=4, delay=-700, mode="reflect"))


def test_refusals():
    for case in (c for c in FU.CASES if c["refuse"]):
        with pytest.raises(nat.UnsupportedOnGPU):
            FU.call(lb, case)
    d = lb.to_device(np.zeros((3, 20), np.int32))
    with pytest.raises(nat.UnsupportedOnGPU, match="float32 or float64"):
        lb.feature.delta(d)
