"""Onset detection on the host: the NumPy oracle (tests/onset_oracle.py) reproduces the reference's fixture
(tests/golden/onset_v1.npz) bit for bit; argument errors come in the reference's order before any device work;
the GPU's refusals fire from shapes and dtypes alone.  No GPU needed: every call here raises before the first
launch or runs the oracle only."""
import os
import warnings

import numpy as np
import pytest

import onset_cases as OC
import onset_oracle as OO
import librosa_b200 as lb
from librosa_b200 import _native as nat

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def golden():
    with np.load(os.path.join(ROOT, "tests", "golden", "onset_v1.npz")) as z:
        return {k: z[k] for k in z.files}


def _bits(got, want, key):
    got = np.asarray(got)
    assert got.dtype == want.dtype and got.shape == want.shape, (key, got.dtype, want.dtype, got.shape, want.shape)
    assert got.tobytes() == want.tobytes(), key


@pytest.mark.parametrize("name", [c["name"] for c in OC.CASES])
def test_oracle_reproduces_fixture(golden, name):
    case = OC.BY_NAME[name]
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        got = OC.outcome(OO, case)
    if name + "/error" in golden:
        assert got.get("error") == str(golden[name + "/error"]), (got, golden[name + "/error"])
    else:
        assert "out" in got, got
        _bits(got["out"], golden[name + "/out"], name)


def test_fixture_normalisation_matches_the_formula(golden):
    for case in OC.CASES:
        key = case["name"] + "/norm"
        if key in golden:
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                want = OC.normalized(OC.envelope(case["env"]))
            np.testing.assert_array_equal(golden[key], want)


def test_fragile_case_needs_the_float32_sum(golden):
    """A float64 mean picks differently on the fragile case: only numba's float32 left-to-right sum gives the
    reference's picks."""
    x = OC.envelope(OC.BY_NAME["peak/greedy_fragile"]["env"])
    seq = OO.peak_pick(x, **OC.FRAGILE_KW)
    f64 = OO.peak_pick(x, seq_mean=False, **OC.FRAGILE_KW)
    _bits(seq, golden["peak/greedy_fragile/out"], "fragile")
    assert (OC.FRAGILE_AT in seq) != (OC.FRAGILE_AT in f64)


def _no_device(monkeypatch):
    """Any attempt to reach the device fails the test."""
    def boom(*a, **k):
        raise AssertionError("device work before the argument checks")
    monkeypatch.setattr(nat, "default_context", boom)
    monkeypatch.setattr(nat, "lib", boom)


@pytest.mark.parametrize("name", [c["name"] for c in OC.CASES if "/err_" in c["name"]])
def test_errors_before_any_device_work(golden, monkeypatch, name):
    _no_device(monkeypatch)
    case = OC.BY_NAME[name]
    if name + "/error" not in golden:
        pytest.skip("not an error in the reference")
    if name in ("detect/err_bad_units", "detect/err_backtrack_empty", "detect/err_bad_units_zeros"):
        pytest.skip("raised after detection (tests/test_gpu_onset.py)")
    got = OC.outcome(lb, case)
    assert got.get("error") == str(golden[name + "/error"]), got


def test_deferred_errors_follow_the_verdict(monkeypatch):
    """onset_detect raises peak_pick's argument errors only when there is something to pick (a host envelope's
    verdict is taken on the host), and an all-zero envelope returns the empty result instead."""
    _no_device(monkeypatch)
    zeros = np.zeros(50, np.float32)
    assert lb.onset.onset_detect(onset_envelope=zeros, wait=-1).dtype == np.int64
    assert lb.onset.onset_detect(onset_envelope=np.zeros((2, 50)), backtrack=True, sparse=False).shape == (2, 50)
    assert lb.onset.onset_detect(onset_envelope=np.zeros((2, 50))).shape == (0,)
    assert lb.onset.onset_detect(onset_envelope=zeros, wait=-1, units="time").dtype == np.float64
    with pytest.raises(lb.ParameterError, match="Invalid unit type"):
        lb.onset.onset_detect(onset_envelope=zeros, wait=-1, units="bad")
    nan = np.ones(50, np.float32)
    nan[3] = np.nan
    assert lb.onset.onset_detect(onset_envelope=nan, method="nope").shape == (0,)
    with pytest.raises(TypeError):
        lb.onset.onset_detect(onset_envelope=np.arange(50.0), bogus=1)


def _dev(shape, dtype=np.float32):
    return nat.DeviceArray(None, 0, shape, dtype, owner=False)


def test_refusals_from_shapes(monkeypatch):
    _no_device(monkeypatch)
    kw = dict(OC.DEFAULTS)
    with pytest.raises(lb.UnsupportedOnGPU, match="int64"):
        lb.util.peak_pick(np.arange(10), **kw)
    with pytest.raises(lb.UnsupportedOnGPU, match="float16"):
        lb.util.peak_pick(np.zeros(10, np.float16), **kw)
    with pytest.raises(lb.UnsupportedOnGPU, match="last axis"):
        lb.util.peak_pick(_dev((4, 10)), axis=0, sparse=False, **kw)
    with pytest.raises(lb.UnsupportedOnGPU, match="2\\^31"):
        lb.util.peak_pick(_dev((1 << 31,)), **kw)
    with pytest.raises(lb.UnsupportedOnGPU, match="int32"):
        lb.onset.onset_detect(onset_envelope=np.arange(10, dtype=np.int32))
    with pytest.raises(lb.UnsupportedOnGPU, match="2\\^31"):
        lb.onset.onset_detect(onset_envelope=_dev((1 << 31,)))
    with pytest.raises(lb.UnsupportedOnGPU, match="one-dimensional"):
        lb.onset.onset_detect(onset_envelope=np.arange(10.0), backtrack=True, energy=np.ones((2, 10)))
    with pytest.raises(lb.UnsupportedOnGPU, match="one-dimensional"):
        lb.onset.onset_backtrack(np.array([1, 2]), np.ones((2, 10)))
    with pytest.raises(lb.UnsupportedOnGPU, match="int64 energy"):
        lb.onset.onset_backtrack(np.array([1, 2]), np.arange(10))
    # argument errors come before the refusals, as the reference raises them for any dtype
    with pytest.raises(lb.ParameterError, match="pre_max"):
        lb.util.peak_pick(np.arange(10), **dict(kw, pre_max=-1))


def test_c_abi_declares_the_onset_entry_points():
    header = open(os.path.join(ROOT, "include", "b2l.h")).read()
    for name in ("b2l_onset_normalize", "b2l_peak_pick", "b2l_onset_backtrack"):
        assert f"int {name}(" in header
