"""Host side of cqt / vqt (CPU only): the oracle and the host constants against tests/golden/cqt_v1.npz, the
projection restatement against SciPy, the launch plan, and the errors and refusals decided before any GPU work."""
from __future__ import annotations

import os
import warnings

import numpy as np
import pytest

import cqt_cases as QC
import cqt_oracle as QO
from librosa_b200 import UnsupportedOnGPU, filters
from librosa_b200.core import constantq as Q
from librosa_b200.util.exceptions import ParameterError

GOLDEN = np.load(os.path.join(os.path.dirname(__file__), "golden", "cqt_v1.npz"))
RUNS = [c for c in QC.CASES if f"{c['name']}/C" in GOLDEN.files and not c["refuse"]]
ERRORS = [c for c in QC.CASES if f"{c['name']}/error" in GOLDEN.files and not c["refuse"]]


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
    assert _same(_quiet(QO.cqt, case), GOLDEN[f"{case['name']}/C"])


@pytest.mark.parametrize("case", RUNS, ids=lambda c: c["name"])
def test_host_plan_and_bases_match_fixture(case):
    name = case["name"]
    y = QC.signal(case["sig"])
    kw, p = _quiet(QO.plan, case, y)
    got = np.array([(o.n, o.n_fft, o.hop, len(p.freqs[o.rows])) for o in p.octaves], dtype=np.int64)
    assert np.array_equal(got, GOLDEN[f"{name}/octaves"])
    assert p.n_frames == GOLDEN[f"{name}/C"].shape[-1]
    for i, b in enumerate(_quiet(QO.bases, case, y)):
        if f"{name}/basis{i}/sha256" in GOLDEN.files:
            assert QC.basis_digest(b.indptr, b.indices, b.data) == str(GOLDEN[f"{name}/basis{i}/sha256"])
            continue
        assert np.array_equal(b.indptr, GOLDEN[f"{name}/basis{i}/indptr"])
        assert np.array_equal(b.indices, GOLDEN[f"{name}/basis{i}/indices"])
        # float64 audio: the reference's complex128 basis, rounded once, is the complex64 table the GPU uses
        assert _same(b.data, GOLDEN[f"{name}/basis{i}/data"].astype(np.complex64))


@pytest.mark.parametrize("name", sorted(QC.WITH_D))
def test_projection_restatement_is_scipy(name):
    """The unfused float32 restatement equals SciPy's complex64 ``csr @ D`` bit for bit (the GPU kernel follows
    the restatement), and stacking its rows gives the stored C of that octave before the scale."""
    import scipy.sparse

    case = QC.BY_NAME[name]
    i = QC.WITH_D[name]
    y = QC.signal(case["sig"])
    b = _quiet(QO.bases, case, y)[i]
    D = GOLDEN[f"{name}/D"]
    m = scipy.sparse.csr_array((b.data, b.indices, b.indptr), shape=(len(b.indptr) - 1, D.shape[-2]))
    for d in D.reshape((-1,) + D.shape[-2:]):
        assert _same(QO.project(b.indptr, b.indices, b.data, d), m @ d)


def test_scale_is_a_reciprocal_multiply():
    """numpy's complex64 /= float64 rounds x * (1 / s) once: what the kernel's double multiply does."""
    rng = np.random.default_rng(0)
    V = (rng.standard_normal(4096) + 1j * rng.standard_normal(4096)).astype(np.complex64)
    s = np.sqrt(rng.uniform(1.0, 5000.0, 4096))
    want = V.copy()
    want /= s
    r = 1.0 / s
    got = (V.real.astype(np.float64) * r).astype(np.float32) + 1j * (V.imag.astype(np.float64) * r).astype(np.float32)
    assert _same(want, got.astype(np.complex64))


def test_frequencies_and_lengths():
    freqs = Q.cqt_frequencies(84, fmin=Q._default_fmin())
    assert freqs[0] == 440.0 * 2.0 ** ((24 - 69.0) / 12.0)
    lengths, cutoff = filters.wavelet_lengths(freqs=freqs, sr=22050)
    assert lengths.shape == (84,) and cutoff < 11025
    assert filters.window_bandwidth("hann") == 1.50018310546875


def _host_call(case):
    """What vqt decides on the host for a case (tuning given or resolved by the oracle)."""
    y = QC.signal(case["sig"])
    kw, p = QO.plan(case, y)
    for o in p.octaves:
        Q.pl.check_stft_geometry(o.n, o.n_fft, True, kw["pad_mode"])
        Q.pl.require_supported_n_fft(o.n_fft)
    return p


@pytest.mark.parametrize("case", [c for c in ERRORS if c["name"] != "cqt_not_finite"], ids=lambda c: c["name"])
def test_host_errors_match_reference(case):
    want = str(GOLDEN[f"{case['name']}/error"])
    with pytest.raises(ParameterError) as e:
        _quiet(_host_call, case)
    assert f"ParameterError: {e.value}" == want


@pytest.mark.parametrize("name, needle", [("cqt_odd_hop", "n_fft=16384"), ("cqt_soxr_resamples", "polyphase"),
                                          ("vqt_ji5", "ji5")])
def test_refusals_are_host_decisions(name, needle):
    with pytest.raises(UnsupportedOnGPU, match=needle):
        _quiet(_host_call, QC.BY_NAME[name])


def test_single_octave_without_resampling_accepts_soxr():
    p = _quiet(_host_call, QC.BY_NAME["cqt_one_octave_soxr"])
    assert p.early == 1 and len(p.octaves) == 1 and not p.octaves[0].resample_after


@pytest.mark.parametrize("case", RUNS, ids=lambda c: c["name"])
def test_stft_warnings_per_octave(case):
    y = QC.signal(case["sig"])
    kw, p = _quiet(QO.plan, case, y)
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        for o in p.octaves:
            Q.pl.check_stft_geometry(o.n, o.n_fft, True, kw["pad_mode"])
    assert [str(w.message) for w in caught] == list(GOLDEN[f"{case['name']}/warnings"])


def test_launch_plan_default():
    """cqt defaults on 8000 samples: 7 octaves at n_fft 256, hop 512 -> 8, no early downsampling."""
    p = _quiet(QO.plan, QC.BY_NAME["cqt_defaults"], QC.signal(QC.BY_NAME["cqt_defaults"]["sig"]))[1]
    assert p.early == 1
    assert [o.n_fft for o in p.octaves] == [256] * 7
    assert [o.hop for o in p.octaves] == [512, 256, 128, 64, 32, 16, 8]
    assert [o.resample_after for o in p.octaves] == [True] * 6 + [False]
    assert Q.octave_rows(p) == [(84 - 12 * (i + 1), 12, 0) for i in range(7)]
    assert p.n_frames == 16


def test_octave_rows_partial():
    p = _quiet(QO.plan, QC.BY_NAME["cqt_partial_octave"], QC.signal(QC.BY_NAME["cqt_partial_octave"]["sig"]))[1]
    rows = Q.octave_rows(p)
    assert rows[-1] == (0, 8, 0) and sum(r[1] for r in rows) == 80


# names whose tabulated bandwidth the symmetric 8193-point window reproduces exactly (DESIGN §4.16)
_ENBW_EXACT = {"hann", "han", "ones", "box", "boxcar", "rect", "rectangular", "triang", "tri", "triangle", "bartlett",
               "bart", "brt", "cosine", "halfcosine", "parzen", "par", "parz", "bohman", "bman", "bmn", "barthann",
               "brthan", "bth"}


def test_window_bandwidth_against_reference_table():
    """Every window the reference tabulates: equal to its value for the names above, within 1e-12 relative for
    hamming, blackman, blackmanharris and nuttall and their aliases; the flat-top window, whose tabulated value is
    not reproduced, is refused."""
    names = [k.split("/", 1)[1] for k in GOLDEN.files if k.startswith("window_bandwidth/")]
    assert len(names) > 30 and _ENBW_EXACT <= set(names)
    for name in names:
        want = float(GOLDEN[f"window_bandwidth/{name}"])
        if name in ("flattop", "flat", "flt"):
            with pytest.raises(UnsupportedOnGPU):
                filters.window_bandwidth(name)
            continue
        got = filters.window_bandwidth(name)
        if name in _ENBW_EXACT:
            assert got == want, name
        else:
            assert abs(got - want) <= 1e-12 * want, name


def test_basis_cache_follows_octave_geometry():
    """Same sr / fmin / n_bins, different hops: hop 512 halves the signal after every octave, hop 160 stops at
    hop 5 and hop 220 at hop 55, so the low octaves run at other rates and n_fft.  Each call gets its own bases."""
    kw = dict(sr=22050, fmin=Q._default_fmin(), n_bins=84, intervals="equal", gamma=0, bins_per_octave=12,
              filter_scale=1, window="hann", scale=True, res_type="polyphase")
    bkw = dict(filter_scale=1, norm=1, sparsity=0.01, window="hann", gamma=0)
    plans = [_quiet(Q.plan, 22050, hop_length=hop, **kw) for hop in (512, 160, 220)]
    assert len({tuple((o.sr, o.n_fft) for o in p.octaves) for p in plans}) == 3
    keys = set()
    for p in plans:
        key, got = Q._bases_cached(p, **bkw)
        keys.add(key)
        for a, b in zip(got, Q.bases(p, **bkw)):
            assert a.n_fft == b.n_fft and _same(a.indptr, b.indptr) and _same(a.indices, b.indices)
            assert _same(a.data, b.data)
    assert len(keys) == 3
