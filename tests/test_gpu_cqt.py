"""cqt / vqt on the GPU against tests/golden/cqt_v1.npz: every case within rtol 1e-4 and atol 1e-5 of the
largest reference magnitude of each octave's row block per clip, host and DeviceArray calls identical, the
projection kernel bit-identical to SciPy's on the stored STFT, launch counts, a batch above 65 535 clips, and
the reference's errors, warnings and the GPU's refusals."""
from __future__ import annotations

import ctypes as C
import os
import warnings

import numpy as np
import pytest

import cqt_cases as QC
import cqt_oracle as QO
import librosa_b200 as lb
from librosa_b200 import _native as nat
from librosa_b200.core import constantq as Q
from librosa_b200.util.exceptions import ParameterError

pytestmark = pytest.mark.gpu

GOLDEN = np.load(os.path.join(os.path.dirname(__file__), "golden", "cqt_v1.npz"))
RUNS = [c for c in QC.CASES if f"{c['name']}/C" in GOLDEN.files and not c["refuse"]]


def _call(case, y=None):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return QC.call(lb, case) if y is None else getattr(lb, case["fn"])(y, **case["kw"])


def _close_per_octave(case, got, ref):
    """rtol 1e-4, atol 1e-5 * max|ref| of each octave's row block of each clip (the low octaves are quieter)."""
    y = QC.signal(case["sig"])
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        _, p = QO.plan(case, y)
    g = np.asarray(got).reshape((-1,) + ref.shape[-2:])
    r = ref.reshape((-1,) + ref.shape[-2:])
    for row0, keep, _ in Q.octave_rows(p):
        for k in range(r.shape[0]):
            rb, gb = r[k, row0:row0 + keep], g[k, row0:row0 + keep]
            atol = 1e-5 * float(np.abs(rb).max())
            err = np.abs(gb - rb) - (atol + 1e-4 * np.abs(rb))
            assert err.max() <= 0, (case["name"], row0, k, float(np.abs(gb - rb).max()), atol)


@pytest.mark.parametrize("case", RUNS, ids=lambda c: c["name"])
def test_matches_reference(case):
    ref = GOLDEN[f"{case['name']}/C"]
    got = _call(case)
    assert isinstance(got, np.ndarray) and got.shape == ref.shape and got.dtype == ref.dtype
    # memory [..., frame, bin]: the reference's order="F"
    assert np.swapaxes(got, -1, -2).flags.c_contiguous
    _close_per_octave(case, got, ref)


@pytest.mark.parametrize("name", ["cqt_defaults", "cqt_multichannel", "vqt_gamma_none", "cqt_early_downsample",
                                  "cqt_tuning_none", "cqt_sparsity0_hop128"])
def test_device_call_identical_to_host_call(name):
    case = QC.BY_NAME[name]
    y = QC.signal(case["sig"])
    host = _call(case, y)
    dev = _call(case, lb.to_device(y))
    assert isinstance(dev, lb.DeviceArray) and dev.layout == "ft" and dev.dtype == np.complex64
    got = dev.get()
    dev.free()
    assert got.shape == host.shape and np.array_equal(got, host)


@pytest.mark.parametrize("name", sorted(QC.WITH_D))
@pytest.mark.parametrize("scale", [False, True])
def test_projection_kernel_bit_identical(name, scale):
    """b2l_cqt_project fed the stored STFT and the octave's CSR table equals the oracle's projection bit for bit."""
    case = QC.BY_NAME[name]
    i = QC.WITH_D[name]
    y = QC.signal(case["sig"])
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        b = QO.bases(case, y)[i]
    D = GOLDEN[f"{name}/D"]
    Dr = np.ascontiguousarray(np.swapaxes(D.reshape((-1,) + D.shape[-2:]), -1, -2)).astype(np.complex64)  # [clip][T][F]
    m, T, F = Dr.shape
    n_rows = len(b.indptr) - 1
    s = np.sqrt(np.random.default_rng(1).uniform(10.0, 3000.0, n_rows))
    rs = 1.0 / s
    ctx = lb.default_context()
    dD, dp, di, dd = (ctx.to_device(a) for a in (Dr, b.indptr.astype(np.int32), b.indices.astype(np.int32), b.data))
    dr = ctx.to_device(rs)
    out = nat.DeviceArray.empty(ctx, (m, T, n_rows), np.complex64)
    desc = (nat.CqtOctave * 1)(nat.CqtOctave(dD.ptr, T, F, 0, n_rows, 0, len(b.data)))
    nat.check(nat.lib().b2l_cqt_project(ctx.handle, desc, 1, C.c_void_p(dp.ptr), C.c_void_p(di.ptr), C.c_void_p(dd.ptr),
                                        C.c_void_p(dr.ptr) if scale else None, m, T, n_rows, C.c_void_p(out.ptr)))
    got = out.get()
    for a in (dD, dp, di, dd, dr, out):
        a.free()
    for k in range(m):
        want = QO.project(b.indptr, b.indices, b.data, Dr[k].T)
        if scale:
            want /= s[:, None]   # numpy's complex64 /= float64, as vqt scales
        assert np.array_equal(np.ascontiguousarray(got[k].T).view(np.uint32), np.ascontiguousarray(want).view(np.uint32))


@pytest.mark.parametrize("name", ["cqt_defaults", "cqt_early_downsample", "cqt_sr16000_hop160", "cqt_one_octave_soxr"])
def test_launch_budget(name):
    """At most 1 + 2 * n_octaves launches before the projection, and one projection launch."""
    case = QC.BY_NAME[name]
    y = lb.to_device(QC.signal(case["sig"]))
    ctx = y.ctx
    _call(case, y).free()   # plans and tables cached
    before = ctx.launch_count
    _call(case, y).free()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        _, p = QO.plan(case, QC.signal(case["sig"]))
    used = ctx.launch_count - before
    expected = (1 if p.early > 1 else 0) + len(p.octaves) + sum(o.resample_after for o in p.octaves) + 1
    assert used == expected <= 1 + 2 * len(p.octaves) + 1
    y.free()


def test_many_clips():
    """70 001 short clips in one call (the projection slices the clip axis at 65 535)."""
    rng = np.random.default_rng(3)
    y = rng.standard_normal((70001, 1024)).astype(np.float32)
    C_ = lb.cqt(y, sr=22050, hop_length=256, fmin=440.0, n_bins=24, res_type="polyphase")
    assert C_.shape == (70001, 24, 5)
    for k in (0, 65534, 65535, 70000):
        want = lb.cqt(y[k], sr=22050, hop_length=256, fmin=440.0, n_bins=24, res_type="polyphase")
        assert np.array_equal(C_[k], want)


@pytest.mark.parametrize("name", ["cqt_odd_hop", "cqt_soxr_resamples", "vqt_ji5"])
def test_refusals(name):
    with pytest.raises(lb.UnsupportedOnGPU):
        _call(QC.BY_NAME[name])


@pytest.mark.parametrize("case", [c for c in QC.CASES if f"{c['name']}/error" in GOLDEN.files and not c["refuse"]],
                         ids=lambda c: c["name"])
def test_errors_match_reference(case):
    with pytest.raises(ParameterError) as e:
        _call(case)
    assert f"ParameterError: {e.value}" == str(GOLDEN[f"{case['name']}/error"])


def test_stft_warning_per_octave():
    case = QC.BY_NAME["cqt_short_warns"]
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        QC.call(lb, case)
    got = [str(w.message) for w in caught if "n_fft=" in str(w.message)]
    assert got == list(GOLDEN["cqt_short_warns/warnings"]) and len(got) > 1


def test_hops_back_to_back_in_one_process():
    """Calls that differ only in the hop have different octave rates and n_fft below the point where the hop turns
    odd (hop 160 stops halving at 5, hop 220 at 55); each must get its own bases, in either order."""
    cases = [QC._c(f"cqt_hop{h}", dict(QC.P, hop_length=h)) for h in (512, 160, 220, 512)]
    for case in cases:
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            ref = QO.cqt(case)
        got = _call(case)
        assert got.shape == ref.shape
        _close_per_octave(case, got, ref)


def test_not_finite_raises_before_the_stft_warnings():
    """The reference's stft raises on non-finite audio before it warns, so a non-finite call emits no warning."""
    case = QC.BY_NAME["cqt_not_finite"]
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        with pytest.raises(ParameterError, match="not finite"):
            QC.call(lb, case)
    got = [str(w.message) for w in caught if "n_fft=" in str(w.message)]
    assert got == list(GOLDEN["cqt_not_finite/warnings"]) == []
