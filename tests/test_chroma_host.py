"""CPU: the chroma oracle against tests/golden/chroma_v1.npz, filters.cq_to_chroma bit-identical to the reference,
and the argument checks, messages and refusals of the chroma features, raised before any device work."""
from __future__ import annotations

import os
import warnings

import numpy as np
import pytest

import chroma_cases as HC
import chroma_oracle as HO
import librosa_b200 as lb
from librosa_b200.util.exceptions import ParameterError

GOLDEN = np.load(os.path.join(os.path.dirname(__file__), "golden", "chroma_v1.npz"))


def _oracle(case):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return HO.run(case, HC.inputs(case, GOLDEN))


@pytest.mark.parametrize("case", [c for c in HC.CASES if not c["refuse"]], ids=lambda c: c["name"])
def test_oracle_reproduces_the_fixture(case):
    name = case["name"]
    if f"{name}/error" in GOLDEN.files:
        with pytest.raises(Exception) as e:
            _oracle(case)
        assert f"{type(e.value).__name__}: {e.value}" == str(GOLDEN[f"{name}/error"])
        return
    want, got = GOLDEN[f"{name}/out"], _oracle(case)
    assert got.shape == want.shape and got.dtype == want.dtype
    assert np.ascontiguousarray(got).tobytes() == np.ascontiguousarray(want).tobytes()


@pytest.mark.parametrize("name", sorted(HC.MAPS))
def test_cq_to_chroma_bit_identical(name):
    kw = dict(HC.MAPS[name])
    got = lb.filters.cq_to_chroma(kw.pop("n_input"), **kw)
    want = GOLDEN[f"map/{name}"]
    assert got.dtype == want.dtype and np.array_equal(got.view(np.uint8), want.view(np.uint8))


def test_cq_to_chroma_merge_error():
    with pytest.raises(ParameterError, match="Incompatible CQ merge"):
        lb.filters.cq_to_chroma(84, bins_per_octave=18, n_chroma=12)


def test_quantised_cens_input_is_the_oracles():
    for name in ("cens_y_defaults", "cens_C_defaults", "cens_C_win_2"):
        raw = GOLDEN[f"{name}/raw"]
        assert np.array_equal(HO.quantize(HO.normalize(raw, norm=None, axis=-2)), GOLDEN[f"{name}/quant"])


def _no_device(monkeypatch):
    """Any device work fails the test: the context and the library are out of reach."""
    from librosa_b200 import _native as nat

    def boom(*a, **k):
        raise AssertionError("device work before the argument checks")

    monkeypatch.setattr(nat, "default_context", boom)
    monkeypatch.setattr(nat, "lib", boom)


@pytest.mark.parametrize("case", [c for c in HC.CASES if c["name"].startswith("err_") and
                                  f"{c['name']}/error" in GOLDEN.files and "nan" not in c["name"] and
                                  c["name"] != "err_bad_norm"], ids=lambda c: c["name"])
def test_argument_errors_before_device_work(case, monkeypatch):
    _no_device(monkeypatch)
    with pytest.raises(ParameterError) as e:
        HC.call(lb, case, GOLDEN)
    assert f"ParameterError: {e.value}" == str(GOLDEN[f"{case['name']}/error"])


@pytest.mark.parametrize("case", [c for c in HC.CASES if c["refuse"]], ids=lambda c: c["name"])
def test_refusals_before_device_work(case, monkeypatch):
    _no_device(monkeypatch)
    with pytest.raises(lb.UnsupportedOnGPU) as e:
        HC.call(lb, case, GOLDEN)
    if case["name"] == "refuse_soxr":
        assert "res_type='polyphase'" in str(e.value) and "C=" in str(e.value)
    if case["name"] == "refuse_complex_C":
        assert "np.abs" in str(e.value)


def test_res_type_is_the_one_signature_addition():
    import inspect

    for fn in (lb.feature.chroma_cqt, lb.feature.chroma_cens, lb.feature.chroma_vqt):
        p = inspect.signature(fn).parameters["res_type"]
        assert p.default == "soxr_hq" and p.kind == p.KEYWORD_ONLY
    assert "res_type" not in inspect.signature(lb.feature.tonnetz).parameters


def test_smoothing_taps_drop_what_ndimage_drops():
    """Hann's two end points are zero: ndimage's footprint leaves them out, and so do the kernel's taps."""
    from librosa_b200.feature.spectral import _smoothing_taps

    off, w, L = _smoothing_taps("hann", 41)
    assert L == 43 and len(off) == 41 and off[0] == 1 and off[-1] == 41
    off, w, L = _smoothing_taps("hamming", 2)
    assert L == 4 and list(off) == [0, 1, 2, 3]
