"""piptrack, pitch_tuning and util.localmax / localmin without a GPU: tests/piptrack_oracle.py reproduces every entry of
tests/golden/piptrack_v1.npz bit for bit, where oracle/ref_np.py's float32 stencil does not; the reference's errors
and the GPU refusals come before any device work; n_fft is inferred from S as the reference infers it; the residual
binning of the histogram kernel (float64 edges, then correction steps) equals np.histogram's."""
from __future__ import annotations

import os
import warnings

import numpy as np
import pytest

import piptrack_cases as PC
import piptrack_oracle as PO
import librosa_b200 as lb
from oracle import ref_np

GOLDEN = np.load(os.path.join(os.path.dirname(__file__), "golden", "piptrack_v1.npz"))
STORED = [c for c in PC.CASES if not c["refuse"] and f"{c['name']}/error" not in GOLDEN.files]
ERRORS = [c for c in PC.CASES if f"{c['name']}/error" in GOLDEN.files]


def _oracle(case, stft_S=None):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        if case["fn"] != "piptrack":
            return PC.call(PO, case)
        kw = PC.piptrack_args(case)
        if case["y"] is not None:
            kw.pop("y")
            kw["S"] = GOLDEN[f"{case['name']}/S"] if stft_S is None else stft_S
        return PO.piptrack(**kw)


@pytest.mark.parametrize("case", STORED, ids=lambda c: c["name"])
def test_oracle_reproduces_the_fixture(case):
    got = _oracle(case)
    if case["fn"] == "piptrack":
        for g, w in zip(got, PC.dense(GOLDEN, case["name"])):
            assert g.dtype == w.dtype and g.shape == w.shape
            assert g.tobytes() == w.tobytes()
    else:
        want = GOLDEN[f"{case['name']}/out"]
        assert np.asarray(got).dtype == want.dtype and np.asarray(got).tobytes() == want.tobytes()


def test_float32_stencil_of_ref_np_misses_the_fixture():
    """The float64 stencil is what makes the oracle exact: the float32 formula of ref_np changes peaks of float32
    spectrograms, and agrees on float64 ones."""
    differ = []
    for case in (c for c in STORED if c["fn"] == "piptrack" and c["S"] is not None):
        kw = PC.piptrack_args(case)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            p, m = ref_np.piptrack(**kw)
        wp, wm = PC.dense(GOLDEN, case["name"])
        if p.tobytes() != wp.tobytes() or m.tobytes() != wm.tobytes():
            differ.append(case["name"])
            assert wp.dtype == np.float32
    assert "S_f32_wide" in differ and len(differ) >= 10


def _no_device(monkeypatch):
    from librosa_b200 import _native as nat
    from librosa_b200 import _pipeline as pl

    def no_device(*a, **k):
        raise AssertionError("device work before the check")

    monkeypatch.setattr(pl, "StagedInput", no_device)
    monkeypatch.setattr(nat, "default_context", no_device)
    monkeypatch.setattr(nat, "lib", no_device)


@pytest.mark.parametrize("case", ERRORS, ids=lambda c: c["name"])
def test_errors_match_the_reference_before_any_device_work(case, monkeypatch):
    _no_device(monkeypatch)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        with pytest.raises(Exception) as info:
            PC.call(lb, case)
    assert f"{type(info.value).__name__}: {info.value}" == str(GOLDEN[f"{case['name']}/error"])


@pytest.mark.parametrize("case", [c for c in PC.CASES if c["refuse"]], ids=lambda c: c["name"])
def test_refusals_before_any_device_work(case, monkeypatch):
    _no_device(monkeypatch)
    with pytest.raises(lb.UnsupportedOnGPU):
        PC.call(lb, case)


def test_more_refusals_before_any_device_work(monkeypatch):
    _no_device(monkeypatch)
    S = np.ones((10, 4), np.float32)
    with pytest.raises(lb.UnsupportedOnGPU, match="float32, float64 or complex"):
        lb.piptrack(S=S.astype(np.float16))
    with pytest.raises(lb.UnsupportedOnGPU, match="does not fit in shared memory"):
        lb.piptrack(S=np.ones((40000, 2), np.float64))
    with pytest.raises(lb.UnsupportedOnGPU, match="1/2048"):
        lb.pitch_tuning(np.ones(5, np.float32), resolution=1e-4)
    with pytest.raises(lb.UnsupportedOnGPU):
        lb.pitch_tuning(np.ones(5, np.float16))
    with pytest.raises(lb.UnsupportedOnGPU, match="n_fft=16384"):
        lb.piptrack(y=np.zeros(40000, np.float32), n_fft=16384)
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        assert lb.pitch_tuning(np.zeros(4), resolution=0) == 0.0
    assert [str(w.message) for w in caught] == ["Trying to estimate tuning from empty frequency set."]


@pytest.mark.parametrize("F, n_fft, want", [(1025, 2048, 2048), (1025, 2049, 2049), (1025, None, 2048),
                                            (1025, 1024, 2048), (513, 2048, 1024), (201, 400, 400), (201, 401, 401),
                                            (2, 512, 2)])
def test_n_fft_inference(F, n_fft, want, monkeypatch):
    """n_fft is kept when n_fft // 2 + 1 matches the bins, else 2 * (bins - 1), as the reference's _spectrogram."""
    from librosa_b200.core import pitch as P

    seen = {}

    def capture(F_, n_fft_, dtype, **kw):
        seen["n_fft"] = n_fft_
        raise RuntimeError("stop")

    monkeypatch.setattr(P, "_piptrack_desc", capture)
    with pytest.raises(RuntimeError, match="stop"):
        lb.piptrack(S=np.ones((F, 3), np.float32), n_fft=n_fft)
    assert seen["n_fft"] == want


def _kernel_bins(res, edges):
    """tuning_hist_kernel's binning: floor((r + 0.5) * n), clamped, then moved across the float64 edges."""
    n = len(edges) - 1
    out = []
    for r in np.asarray(res, np.float64):
        b = int(np.floor((r + 0.5) * n))
        b = max(0, min(n - 1, b))
        while b > 0 and r < edges[b]:
            b -= 1
        while b < n - 1 and r >= edges[b + 1]:
            b += 1
        out.append(b)
    return np.bincount(out, minlength=n)


@pytest.mark.parametrize("resolution", [0.01, 1 / 3, 1 / 2048, 0.07, 1 / 1000])
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_residual_binning_equals_np_histogram(resolution, dtype):
    edges = np.linspace(-0.5, 0.5, int(np.ceil(1.0 / resolution)) + 1)
    rng = np.random.default_rng(5)
    e = edges.astype(dtype)
    near = np.concatenate([e, np.nextafter(e, dtype(-1)), np.nextafter(e, dtype(1))])
    res = np.concatenate([rng.uniform(-0.5, 0.5, 3000).astype(dtype), near]).astype(dtype)
    res = res[(res >= -0.5) & (res < 0.5)]
    counts, _ = np.histogram(res, edges)
    assert np.array_equal(_kernel_bins(res, edges), counts)


def test_fixture_residuals_near_an_edge():
    """How many pitch_tuning residuals of the fixture lie within one ulp of a bin edge, where a log2 that differs from
    NumPy's by one ulp could move a value to the next bin.  All 39 are float32 residuals of the 1/2048 case, which sit
    on an edge exactly; none moves its argmax (the GPU tests compare the tuning with the reference's)."""
    near = 0
    for case in (c for c in STORED if c["fn"] == "pitch_tuning"):
        f = PC.values(case["spec"])
        r = PO.residuals(f, case["kw"].get("bins_per_octave", 12))
        r = r[np.isfinite(r)]
        if r.size == 0:
            continue
        edges = np.linspace(-0.5, 0.5, int(np.ceil(1.0 / case["kw"].get("resolution", 0.01))) + 1)
        gap = np.min(np.abs(r.astype(np.float64)[:, None] - edges[None, :]), axis=1)
        near += int(np.sum(gap <= np.spacing(np.abs(r)).astype(np.float64)))
    assert near == 39, near
