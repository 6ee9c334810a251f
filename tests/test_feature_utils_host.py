"""Host side of feature.delta / feature.stack_memory (CPU only): the oracle against tests/golden/feature_utils_v1.npz,
ndimage's tap classification, the padded-index tables against np.pad, the interp edge maps, and the errors and
refusals decided before any device work."""
from __future__ import annotations

import os
import warnings

import numpy as np
import pytest
from scipy.signal import savgol_coeffs

import feature_utils_cases as FU
import feature_utils_oracle as FO
import librosa_b200 as lb
from librosa_b200 import _native as nat
from librosa_b200.feature import utils as U

GOLDEN = np.load(os.path.join(os.path.dirname(__file__), "golden", "feature_utils_v1.npz"))
RUNS = [c for c in FU.CASES if f"{c['name']}/out" in GOLDEN.files]
# errors raised before the device: all but SciPy's complaint about non-finite edge windows, found by the kernel
HOST_ERRORS = [c for c in FU.CASES if f"{c['name']}/error" in GOLDEN.files
               and "must not contain infs" not in str(GOLDEN[f"{c['name']}/error"])]
REFUSALS = [c for c in FU.CASES if c["refuse"]]


def _bytes(a):
    return np.ascontiguousarray(a).tobytes()


def test_fixture_covers_the_issue():
    assert os.path.getsize(os.path.join(os.path.dirname(__file__), "golden", "feature_utils_v1.npz")) < 1 << 20
    kws = [c["kw"] for c in RUNS if c["fn"] == "delta"]
    assert {k.get("mode", "interp") for k in kws} == set(FU.MODES)
    assert max(k.get("width", 9) for k in kws) >= 31 and {k.get("order", 1) for k in kws} == {1, 2, 3}
    assert any(FU.vandermonde_condition(k.get("width", 9), k.get("polyorder", 1)) > 1e3 for k in kws)
    stacks = [c["kw"] for c in RUNS if c["fn"] == "stack_memory"]
    assert {k.get("delay", 1) for k in stacks} >= {1, -1, 3, -3}
    assert {k.get("mode", "constant") for k in stacks} == {"constant", "edge", "reflect", "symmetric", "wrap", "empty"}


@pytest.mark.parametrize("case", RUNS, ids=lambda c: c["name"])
def test_oracle_reproduces_fixture(case):
    ref = GOLDEN[f"{case['name']}/out"]
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        got = FO.run(case)
    assert got.dtype == ref.dtype and got.shape == ref.shape
    if case["fn"] == "stack_memory":
        keep = ~FU.empty_cells(case)
        assert _bytes(np.where(keep, got, 0)) == _bytes(np.where(keep, ref, 0))
        return
    edges = FO.interp_edges(case)
    if edges is None:
        assert _bytes(got) == _bytes(ref)
        return
    ax, h = edges
    g, r = np.moveaxis(got, ax, -1), np.moveaxis(ref, ax, -1)
    n = g.shape[-1]
    assert _bytes(g[..., h:n - h]) == _bytes(r[..., h:n - h])
    kw = case["kw"]
    width = kw.get("width", 9)
    tol_l, tol_r = FU.edge_tolerance(FU.data(case["spec"]), width, kw.get("polyorder", kw.get("order", 1)), ax,
                                     got.dtype)
    assert np.all(np.abs(g[..., :h].astype(np.float64) - r[..., :h]) <= tol_l[..., None])
    assert np.all(np.abs(g[..., n - h:].astype(np.float64) - r[..., n - h:]) <= tol_r[..., None])


@pytest.mark.parametrize("width", [3, 5, 9, 15, 31, 63, 255])
def test_tap_classification_follows_ndimage(width):
    for order in (1, 2, 3):
        for polyorder in range(order, min(order + 4, width)):
            for spacing in (1.0, 0.5, 3.0):
                fw = np.asarray(savgol_coeffs(width, polyorder, deriv=order, delta=spacing))[::-1]
                assert U.classify_taps(fw) == FO.symmetry(fw)
    assert U.classify_taps(np.arange(width, dtype=np.float64) - width // 2) == -1
    assert U.classify_taps(np.zeros(width)) == 1   # order > polyorder: zero taps count as symmetric
    assert U.classify_taps(np.arange(width, dtype=np.float64) ** 2) == 0
    near = np.ones(width)
    near[0] += np.finfo(np.float64).eps   # a difference of DBL_EPSILON still passes
    assert U.classify_taps(near) == 1


@pytest.mark.parametrize("mode", ["constant", "edge", "reflect", "symmetric", "wrap", "empty"])
@pytest.mark.parametrize("n", [1, 2, 3, 5, 17, 400])
def test_pad_index_table_matches_np_pad(mode, n):
    x = np.arange(1, n + 1, dtype=np.float64) * 10.0
    for before, after in ((0, 0), (4, 4), (0, 13), (13, 0), (2 * n + 3, n + 1)):
        table = U.pad_index_table(n, before, after, mode)
        assert table.dtype == np.int64 and table.shape == (before + after,)
        got = np.concatenate([np.where(table[:before] < 0, 0.0, x[table[:before]]), x,
                              np.where(table[before:] < 0, 0.0, x[table[before:]])])
        if mode == "empty":
            assert np.all(table == -1)
            continue
        assert np.array_equal(got, np.pad(x, (before, after), mode=mode))
    if mode in ("reflect", "symmetric"):
        table = U.pad_index_table(n, 7, 7, mode, reflect_type="even")
        assert np.array_equal(table, U.pad_index_table(n, 7, 7, mode))


@pytest.mark.parametrize("width,polyorder,order", [(3, 1, 1), (9, 1, 1), (9, 2, 2), (9, 3, 1), (9, 7, 2),
                                                   (31, 3, 3), (31, 7, 3), (255, 4, 2), (9, 2, 3)])
def test_edge_map(width, polyorder, order):
    h = width // 2
    for spacing in (1.0, 0.25):
        E = U.edge_map(width, polyorder, order, spacing)
        full = FO.fit_map(width, polyorder, order, spacing)
        assert E.shape == (width - 1, width) and E.dtype == np.float64
        assert _bytes(E) == _bytes(np.concatenate([full[:h], full[width - h:]]))
        # exact on polynomials of the fitted degree: the derivative of p(t) = sum c_q t^q at the edge positions
        rng = np.random.default_rng(width + polyorder)
        c = rng.standard_normal(polyorder + 1)
        t = np.arange(width, dtype=np.float64)
        x = np.polynomial.polynomial.polyval(t, c)
        d = np.polynomial.polynomial.polyval(t, np.polynomial.polynomial.polyder(c, order)) / spacing ** order
        want = np.concatenate([d[:h], d[width - h:]])
        assert np.allclose(E @ x, want, rtol=1e-6, atol=1e-6 * np.abs(x).max())


def _no_device(monkeypatch):
    def refuse(*a, **k):
        raise AssertionError("device work started")

    monkeypatch.setattr(nat, "default_context", refuse)
    monkeypatch.setattr(nat, "lib", refuse)


@pytest.mark.parametrize("case", HOST_ERRORS, ids=lambda c: c["name"])
def test_errors_match_the_reference_before_device_work(case, monkeypatch):
    _no_device(monkeypatch)
    want = str(GOLDEN[f"{case['name']}/error"])
    with pytest.raises(Exception) as info:
        FU.call(lb, case)
    assert f"{type(info.value).__name__}: {info.value}" == want


@pytest.mark.parametrize("case", REFUSALS, ids=lambda c: c["name"])
def test_refusals_before_device_work(case, monkeypatch):
    _no_device(monkeypatch)
    with pytest.raises(nat.UnsupportedOnGPU):
        FU.call(lb, case)


def test_stack_memory_refuses_objects_and_wide_elements(monkeypatch):
    _no_device(monkeypatch)
    with pytest.raises(nat.UnsupportedOnGPU, match="object"):
        lb.feature.stack_memory(np.array([[1, "a"]], dtype=object))
    with pytest.raises(nat.UnsupportedOnGPU, match="bytes"):
        lb.feature.stack_memory(np.zeros((2, 3), dtype="U3"))


def test_signatures_match_the_reference():
    import inspect

    d = inspect.signature(lb.feature.delta)
    assert list(d.parameters) == ["data", "width", "order", "axis", "mode", "kwargs"]
    assert [d.parameters[k].default for k in ("width", "order", "axis", "mode")] == [9, 1, -1, "interp"]
    s = inspect.signature(lb.feature.stack_memory)
    assert list(s.parameters) == ["data", "n_steps", "delay", "kwargs"]
    assert [s.parameters[k].default for k in ("n_steps", "delay")] == [2, 1]
    assert all(p.kind == p.KEYWORD_ONLY for k, p in {**d.parameters, **s.parameters}.items()
               if k not in ("data", "kwargs"))
