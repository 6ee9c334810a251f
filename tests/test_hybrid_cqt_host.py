"""Host side of pseudo_cqt / hybrid_cqt (CPU only): the oracle against tests/golden/hybrid_cqt_v1.npz, the host split
and |basis| tables, the float32 projection restatement against SciPy, the reference's signatures, the C-ABI octave
struct, and the errors and refusals decided before any device work."""
from __future__ import annotations

import ctypes as C
import inspect
import os
import warnings

import numpy as np
import pytest
import scipy.sparse

import hybrid_cqt_cases as HC
import hybrid_cqt_oracle as HO
import librosa_b200 as lb
from librosa_b200 import _native as nat
from librosa_b200.util.exceptions import ParameterError

GOLDEN = np.load(os.path.join(os.path.dirname(__file__), "golden", "hybrid_cqt_v1.npz"))
RUNS = [c for c in HC.CASES if f"{c['name']}/C" in GOLDEN.files and not c["refuse"]]
ERRORS = [c for c in HC.CASES if f"{c['name']}/error" in GOLDEN.files and not c["refuse"]]


def _same(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.dtype == b.dtype and a.shape == b.shape and np.ascontiguousarray(a).tobytes() == \
        np.ascontiguousarray(b).tobytes()


def _quiet(fn, *a, **k):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return fn(*a, **k)


@pytest.mark.parametrize("case", RUNS, ids=lambda c: c["name"])
def test_oracle_reproduces_fixture(case):
    ref = GOLDEN[f"{case['name']}/C"]
    got = _quiet(HO.run, case)
    assert _same(got, ref)
    assert got.flags.c_contiguous == ref.flags.c_contiguous and got.flags.f_contiguous == ref.flags.f_contiguous


@pytest.mark.parametrize("case", RUNS, ids=lambda c: c["name"])
def test_host_split_and_tables_match_fixture(case):
    name = case["name"]
    y = HC.signal(case["sig"])
    kw, fmin, pp, n_full = _quiet(HO.split, case, y)
    if case["fn"] == "hybrid_cqt":
        assert n_full == int(GOLDEN[f"{name}/n_full"])
        assert (pp.n_bins if pp else 0) == int(GOLDEN[f"{name}/n_pseudo"])
        if pp is not None:
            assert pp.freqs[0] == float(GOLDEN[f"{name}/fmin_pseudo"])
    if pp is None:
        assert f"{name}/n_fft" not in GOLDEN.files
        return
    assert pp.n_fft == int(GOLDEN[f"{name}/n_fft"])
    m = HO.basis(kw, pp)
    if name in HC.BASIS_DIGEST:
        assert HC.basis_digest(m.indptr, m.indices, m.data) == str(GOLDEN[f"{name}/basis/sha256"])
        return
    assert np.array_equal(m.indptr, GOLDEN[f"{name}/basis/indptr"])
    assert np.array_equal(m.indices, GOLDEN[f"{name}/basis/indices"])
    want = GOLDEN[f"{name}/basis/data"]
    if want.dtype == np.float32:
        assert _same(m.data, want)
    else:   # complex128 basis: the float32 table is the float64 magnitude within a rounding
        assert np.allclose(m.data, want, rtol=2 ** -22, atol=0)


@pytest.mark.parametrize("name", HC.WITH_D)
def test_projection_restatement_is_scipy_and_fixture(name):
    """The unfused float32 restatement equals SciPy's float32 ``|basis| @ np.abs(D)`` bit for bit, and scaled as
    numpy scales it gives the stored pseudo rows (the GPU kernel follows the restatement)."""
    case = HC.BY_NAME[name]
    b = {k: GOLDEN[f"{name}/basis/{k}"] for k in ("indptr", "indices", "data")}
    D = GOLDEN[f"{name}/D"]
    m = scipy.sparse.csr_array((b["data"], b["indices"], b["indptr"]), shape=(len(b["indptr"]) - 1, D.shape[-2]))
    y = HC.signal(case["sig"])
    kw, _, pp, _ = _quiet(HO.split, case, y)
    ref = GOLDEN[f"{name}/C"][..., -pp.n_bins:, :]   # the pseudo part holds the highest bins
    for d in D.reshape((-1,) + D.shape[-2:]):
        got = HO.project_abs(b["indptr"], b["indices"], b["data"], d)
        assert _same(got, m @ np.abs(d))
        T = ref.shape[-1]
        assert _same(HO.scale_pseudo(got, pp, kw["scale"])[:, :T], np.ascontiguousarray(ref))


def test_split_table():
    """hybrid_cqt's split at 22 050 Hz, 12 bins per octave, 84 bins from C1, and 36 x 252 at hop 512."""
    for hop, n_pseudo, n_fft in ((512, 29, 1024), (128, 5, None), (64, 0, None), (4096, 65, 8192)):
        case = HC._c("hcqt_split", dict(HC.P, hop_length=hop))
        _, _, pp, n_full = HO.split(case, HC.signal(case["sig"]))
        assert (pp.n_bins if pp else 0, n_full) == (n_pseudo, 84 - n_pseudo)
        if n_fft is not None and pp is not None and pp.n_bins > 5:
            assert pp.n_fft == n_fft
    case = HC.BY_NAME["hcqt_bpo36"]
    _, _, pp, n_full = HO.split(case, HC.signal(case["sig"]))
    assert (pp.n_bins, n_full) == (32, 220)


def _no_device(monkeypatch):
    def refuse(*a, **k):
        raise AssertionError("device work started")

    monkeypatch.setattr(nat, "default_context", refuse)
    monkeypatch.setattr(lb.core.constantq.pl, "StagedInput", refuse)


def _host_decisions(case):
    """What the entry point decides on the host before it stages anything (tuning given)."""
    y = HC.signal(case["sig"])
    kw, fmin, pp, n_full = HO.split(case, y)
    Q = lb.core.constantq
    if pp is not None:
        Q._check_pseudo_stft(pp, y.shape[-1], kw["pad_mode"])
    if n_full:
        Q._check_full_stft(Q.plan(y.shape[-1], sr=kw["sr"], hop_length=kw["hop_length"], fmin=fmin, n_bins=n_full,
                                  intervals="equal", gamma=0, bins_per_octave=kw["bins_per_octave"],
                                  filter_scale=kw["filter_scale"], window=kw["window"], scale=kw["scale"],
                                  res_type=kw["res_type"]), kw["pad_mode"])


@pytest.mark.parametrize("case", [c for c in ERRORS if not c["name"].endswith("not_finite")], ids=lambda c: c["name"])
def test_errors_before_device_work(case, monkeypatch):
    want = str(GOLDEN[f"{case['name']}/error"])
    with pytest.raises(ParameterError) as e:
        _quiet(_host_decisions, case)
    assert f"ParameterError: {e.value}" == want
    _no_device(monkeypatch)
    with pytest.raises(ParameterError) as e:
        _quiet(HC.call, lb, case)
    assert f"ParameterError: {e.value}" == want


@pytest.mark.parametrize("name, needle", [("pcqt_defaults", "n_fft=16384"), ("hcqt_soxr_resamples", "polyphase"),
                                          ("hcqt_odd_hop", "n_fft=16384")])
def test_refusals_before_device_work(name, needle, monkeypatch):
    case = HC.BY_NAME[name]
    with pytest.raises(lb.UnsupportedOnGPU, match=needle):
        _quiet(_host_decisions, case)
    _no_device(monkeypatch)
    with pytest.raises(lb.UnsupportedOnGPU, match=needle):
        _quiet(HC.call, lb, case)


@pytest.mark.parametrize("case", RUNS, ids=lambda c: c["name"])
def test_stft_warnings(case):
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        if case["kw"].get("tuning", 0.0) is not None:
            _host_decisions(case)
    if case["kw"].get("tuning", 0.0) is not None:
        assert [str(w.message) for w in caught if "n_fft=" in str(w.message)] == \
            list(GOLDEN[f"{case['name']}/warnings"])


def test_signatures_match_reference():
    common = ("y, *, sr: 'float' = 22050, hop_length: 'int' = 512, fmin: 'Optional[float]' = None, "
              "n_bins: 'Optional[int]' = 84, bins_per_octave: 'int' = 12, tuning: 'Optional[float]' = 0.0, "
              "filter_scale: 'float' = 1, norm: 'Optional[float]' = 1, sparsity: 'float' = 0.01, window='hann', "
              "scale: 'bool' = True, pad_mode='constant', ")
    assert str(inspect.signature(lb.pseudo_cqt)) == "(" + common + "dtype=None)"
    assert str(inspect.signature(lb.hybrid_cqt)) == "(" + common + "res_type: 'str' = 'soxr_hq', dtype=None)"
    assert lb.core.pseudo_cqt is lb.pseudo_cqt and lb.core.hybrid_cqt is lb.hybrid_cqt


def test_octave_struct_is_40_bytes():
    assert C.sizeof(nat.CqtOctave) == 40
    assert nat.CqtOctave.kind.offset == 36


def test_numpy_complex_abs_is_the_ratio_form():
    """np.abs of complex64, which pseudo_cqt applies to D and hybrid_cqt to cqt's result, is the larger part times
    sqrtf(fmaf(r, r, 1)) with r = smaller / larger (NumPy's vectorised x86 loop), which the projection kernel's
    np_abs restates; it is not the correctly rounded |z|."""
    rng = np.random.default_rng(0)
    n = 1 << 16
    z = (rng.standard_normal(n) * rng.uniform(0, 3, n) + 1j * rng.standard_normal(n)).astype(np.complex64)
    z[:4] = [0, 1j, 3, -2]
    re, im = np.abs(z.real), np.abs(z.imag)
    big, small = np.maximum(re, im), np.minimum(re, im)
    r = np.divide(small, big, out=np.zeros_like(big), where=big > 0)
    fma = (r.astype(np.float64) ** 2 + 1.0).astype(np.float32)   # r * r is exact in float64: one rounding
    assert _same(np.sqrt(fma) * big, np.abs(z))
