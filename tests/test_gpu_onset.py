"""Onset detection on the GPU: every case of tests/onset_cases.py bit for bit against the reference's fixture
(tests/golden/onset_v1.npz), dense and sparse, the normalised envelope included; ``y=`` against the reference on
click trains and against the oracle on the GPU's own envelope; DeviceArray in and out; the launch counts and
read-backs of each call; and one launch over more than 65 535 rows.

Tolerances: none — picks, lists and the normalised envelope are compared bit for bit."""
import os
import warnings

import numpy as np
import pytest

import onset_cases as OC
import onset_oracle as OO
import librosa_b200 as lb
from librosa_b200 import _native as nat

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def golden():
    with np.load(os.path.join(ROOT, "tests", "golden", "onset_v1.npz")) as z:
        return {k: z[k] for k in z.files}


def _same(got, want, key):
    got = np.asarray(got)
    assert got.dtype == want.dtype and got.shape == want.shape, (key, got.dtype, want.dtype, got.shape, want.shape)
    if got.tobytes() != want.tobytes():
        bad = np.argwhere(got != want) if got.shape else []
        raise AssertionError(f"{key}: {len(bad)} differ, first at {np.asarray(bad)[:3].tolist()}")


def _dev(x):
    return lb.to_device(np.ascontiguousarray(x))


@pytest.mark.parametrize("name", [c["name"] for c in OC.CASES])
def test_vs_golden(golden, name):
    case = OC.BY_NAME[name]
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        got = OC.outcome(lb, case)
    if name + "/error" in golden:
        assert got.get("error") == str(golden[name + "/error"]), got
    else:
        assert "out" in got, got
        _same(got["out"], golden[name + "/out"], name)


@pytest.mark.parametrize("name", [c["name"] for c in OC.CASES
                                  if c["op"] in ("onset_detect", "peak_pick") and c["env"] is not None
                                  and c["kw"].get("axis", -1) == -1])
def test_device_in_device_out(golden, name):
    """The same case with the envelope on the device: a DeviceArray comes back, with the same bits."""
    case = OC.BY_NAME[name]
    if name + "/error" in golden:
        pytest.skip("error case")
    kw = OC.kwargs(case)
    x = _dev(OC.envelope(case["env"]))
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        if case["op"] == "onset_detect":
            got = lb.onset.onset_detect(onset_envelope=x, **kw)
        else:
            got = lb.util.peak_pick(x, **kw)
    assert isinstance(got, lb.DeviceArray)
    _same(got.get(), golden[name + "/out"], name)


@pytest.mark.parametrize("name", [c["name"] for c in OC.CASES if c["op"] == "onset_detect" and c["env"] is not None
                                  and c["kw"].get("normalize", True) and c["env"][2] > 0])
def test_normalised_envelope_bit_exact(golden, name):
    want = golden[name + "/norm"]
    got = lb.onset.detect_stages(OC.envelope(OC.BY_NAME[name]["env"]))
    assert got["normalized"].dtype == want.dtype and got["normalized"].shape == want.shape
    if np.isnan(want).any():
        assert np.array_equal(got["normalized"], want, equal_nan=True), name
    else:
        _same(got["normalized"], want, name + "/norm")
    passes = bool(want.any()) and bool(np.all(np.isfinite(want)))
    assert (got["flags"] == 1) == passes, (name, got["flags"])


@pytest.mark.parametrize("name", list(OC.Y_CASES))
def test_y_vs_golden_click_trains(golden, name):
    got = lb.onset.onset_detect(y=OC.clicks_audio(OC.Y_CASES[name]))
    _same(got, golden[name + "/out"], name)


def test_y_noise_vs_oracle_on_gpu_envelope():
    rng = np.random.default_rng(0)
    y = (0.1 * rng.standard_normal((3, 22050 * 3))).astype(np.float32)
    got = lb.onset.onset_detect(y=y, sparse=False)
    env = lb.onset.onset_strength(y=y)
    _same(got, OO.onset_detect(onset_envelope=env, sparse=False), "noise y=")
    got1 = lb.onset.onset_detect(y=y[0], units="time", backtrack=True)
    _same(got1, OO.onset_detect(onset_envelope=env[0], units="time", backtrack=True), "noise y= 1-D")
    with pytest.raises(lb.ParameterError, match="finite"):
        bad = y[0].copy()
        bad[100] = np.nan
        lb.onset.onset_detect(y=bad)


class _Reads:
    """Counts device-to-host copies and their bytes."""

    def __init__(self, monkeypatch):
        self.calls, self.bytes = 0, 0
        orig = nat.DeviceArray.get
        reads = self

        def get(arr, out=None):
            reads.calls += 1
            reads.bytes += arr.nbytes
            return orig(arr, out)
        monkeypatch.setattr(nat.DeviceArray, "get", get)


def test_launch_counts_and_read_backs(monkeypatch):
    ctx = lb.default_context()
    x1 = _dev(OC.envelope(("clicks", (), 431, "float32", 3)))
    x3 = _dev(OC.envelope(("clicks", (3,), 431, "float32", 3)))
    kw = dict(OC.DEFAULTS)
    reads = _Reads(monkeypatch)

    def count(fn):
        n0, r0, b0 = ctx.launch_count, reads.calls, reads.bytes
        out = fn()
        return out, ctx.launch_count - n0, reads.calls - r0, reads.bytes - b0

    out, n, r, _ = count(lambda: lb.util.peak_pick(x3, sparse=False, **kw))
    assert (n, r) == (1, 0) and isinstance(out, lb.DeviceArray)
    out, n, r, b = count(lambda: lb.util.peak_pick(x1, **kw))
    assert (n, r, b) == (1, 1, 8) and out.dtype == np.int64
    out, n, r, _ = count(lambda: lb.onset.onset_detect(onset_envelope=x3, sparse=False))
    assert (n, r) == (2, 0)
    out, n, r, b = count(lambda: lb.onset.onset_detect(onset_envelope=x1))
    assert n == 2 and r == 1 and b <= 16
    out, n, r, b = count(lambda: lb.onset.onset_detect(onset_envelope=x1, backtrack=True, units="time"))
    assert n == 3 and r == 1 and b <= 16 and out.dtype == np.float64
    frames = lb.onset.onset_detect(onset_envelope=x1)
    out, n, _, _ = count(lambda: lb.onset.onset_backtrack(frames, x1))
    assert n == 1 and isinstance(out, lb.DeviceArray)
    # host input: the same launches after its upload
    host = OC.envelope(("clicks", (3,), 431, "float32", 3))
    _, n, _, _ = count(lambda: lb.onset.onset_detect(onset_envelope=host, sparse=False))
    assert n == 2
    y = _dev(OC.clicks_audio(120.0))
    n0 = ctx.launch_count
    lb.onset.onset_strength(y=y)
    n_env = ctx.launch_count - n0
    _, n, r, _ = count(lambda: lb.onset.onset_detect(y=y, sparse=False))
    assert (n, r) == (n_env + 2, 0)


def test_device_backtrack_negative_event():
    e = _dev(OC.envelope(("random", (), 100, "float32", 1)))
    with pytest.raises(lb.ParameterError, match="min\\(events_to\\) > min\\(events_from\\)"):
        lb.onset.onset_backtrack(_dev(np.array([3, -1, 7], np.int64)), e)
    got = lb.onset.onset_backtrack(_dev(np.array([3, 50, 99], np.int64)), e)
    _same(got.get(), OO.onset_backtrack([3, 50, 99], e.get()), "device backtrack")


def test_many_rows_one_launch():
    """70 000 rows x 16 frames: one launch (rows on grid.x), every row as the oracle."""
    rng = np.random.default_rng(5)
    x = (rng.random((70000, 16)) ** 3).astype(np.float32)
    ctx = lb.default_context()
    d = _dev(x)
    n0 = ctx.launch_count
    got = lb.util.peak_pick(d, sparse=False, **OC.DEFAULTS)
    assert ctx.launch_count - n0 == 1
    _same(got.get(), OO.peak_pick(x, sparse=False, **OC.DEFAULTS), "70000 rows")
