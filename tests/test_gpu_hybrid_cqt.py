"""pseudo_cqt / hybrid_cqt on the GPU against tests/golden/hybrid_cqt_v1.npz: every case within rtol 1e-4 and atol
1e-5 of the largest reference magnitude of each row block per clip (the pseudo rows are one block, the full part's
octaves the others), shape, dtype and memory order as the reference's; b2l_cqt_project_abs bit-identical to the
fixture on the stored STFT and |basis|; hybrid rows bit-identical to the GPU's own np.abs(cqt) and pseudo_cqt; host
and DeviceArray calls identical; launch counts; a batch above 65 535 clips; errors, warnings and refusals."""
from __future__ import annotations

import ctypes as C
import os
import warnings

import numpy as np
import pytest

import cqt_oracle as QO
import hybrid_cqt_cases as HC
import hybrid_cqt_oracle as HO
import librosa_b200 as lb
from librosa_b200 import _native as nat
from librosa_b200.core import constantq as Q
from librosa_b200.util.exceptions import ParameterError

pytestmark = pytest.mark.gpu

GOLDEN = np.load(os.path.join(os.path.dirname(__file__), "golden", "hybrid_cqt_v1.npz"))
RUNS = [c for c in HC.CASES if f"{c['name']}/C" in GOLDEN.files and not c["refuse"]]


def _quiet(fn, *a, **k):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return fn(*a, **k)


def _blocks(case):
    """(row0, rows) of each row block: the full part's octaves, then the pseudo rows."""
    y = HC.signal(case["sig"])
    kw, fmin, pp, n_full = _quiet(HO.split, case, y)
    out = []
    if n_full:
        sub = HO.full_case(case, kw, fmin, n_full)
        _, p = _quiet(QO.plan, sub, y)
        out += [(row0, keep) for row0, keep, _ in Q.octave_rows(p)]
    if pp is not None:
        out.append((n_full, pp.n_bins))
    return out


def _close_per_block(case, got, ref):
    g = np.asarray(got).reshape((-1,) + ref.shape[-2:])
    r = ref.reshape((-1,) + ref.shape[-2:])
    for row0, keep in _blocks(case):
        for k in range(r.shape[0]):
            rb, gb = r[k, row0:row0 + keep], g[k, row0:row0 + keep]
            atol = 1e-5 * float(np.abs(rb).max())
            err = np.abs(gb - rb) - (atol + 1e-4 * np.abs(rb))
            assert err.max() <= 0, (case["name"], row0, k, float(np.abs(gb - rb).max()), atol)


@pytest.mark.parametrize("case", RUNS, ids=lambda c: c["name"])
def test_matches_reference(case):
    ref = GOLDEN[f"{case['name']}/C"]
    got = _quiet(HC.call, lb, case)
    assert isinstance(got, np.ndarray) and got.shape == ref.shape and got.dtype == ref.dtype
    if case["fn"] == "pseudo_cqt":
        assert got.flags.c_contiguous
    else:   # memory [..., frame, bin], as cqt returns it: the reference's order="F" for one clip
        assert np.swapaxes(got, -1, -2).flags.c_contiguous
    _close_per_block(case, got, ref)


@pytest.mark.parametrize("name", HC.WITH_D)
@pytest.mark.parametrize("scale", [True, False])
def test_project_abs_bit_identical(name, scale):
    """b2l_cqt_project_abs fed the stored STFT and |basis| gives the fixture's pseudo rows bit for bit (scale as
    the case has it), and numpy's other scaling of the same sums."""
    case = HC.BY_NAME[name]
    y = HC.signal(case["sig"])
    kw, _, pp, _ = _quiet(HO.split, case, y)
    b = {k: GOLDEN[f"{name}/basis/{k}"] for k in ("indptr", "indices", "data")}
    D = GOLDEN[f"{name}/D"]
    Dr = np.ascontiguousarray(np.swapaxes(D.reshape((-1,) + D.shape[-2:]), -1, -2)).astype(np.complex64)
    m, T, F = Dr.shape
    n = pp.n_bins
    rs = np.full(n, np.sqrt(pp.n_fft)) if scale else np.sqrt(pp.lengths / pp.n_fft)
    ctx = lb.default_context()
    table = b["data"].astype(np.complex64)   # |basis| in the real parts
    dD, dp, di, dd, dr = (ctx.to_device(a) for a in (Dr, b["indptr"].astype(np.int32), b["indices"].astype(np.int32),
                                                      table, rs))
    out = nat.DeviceArray.empty(ctx, (m, T, n), np.float32)
    kind = nat.CQT_PSEUDO | (nat.CQT_DIVIDE if scale else 0)
    desc = (nat.CqtOctave * 1)(nat.CqtOctave(dD.ptr, T, F, 0, n, 0, len(b["data"]), kind))
    nat.check(nat.lib().b2l_cqt_project_abs(ctx.handle, desc, 1, C.c_void_p(dp.ptr), C.c_void_p(di.ptr),
                                            C.c_void_p(dd.ptr), C.c_void_p(dr.ptr), m, T, n, C.c_void_p(out.ptr)))
    got = out.get()
    for a in (dD, dp, di, dd, dr, out):
        a.free()
    for k in range(m):
        want = HO.scale_pseudo(HO.project_abs(b["indptr"], b["indices"], b["data"], Dr[k].T), pp, scale)
        assert np.array_equal(np.ascontiguousarray(got[k].T).view(np.uint32), want.view(np.uint32))
        if scale == kw["scale"]:
            ref = GOLDEN[f"{name}/C"].reshape((-1,) + GOLDEN[f"{name}/C"].shape[-2:])[k, -n:]
            assert np.array_equal(np.ascontiguousarray(got[k].T[:, :ref.shape[-1]]).view(np.uint32),
                                  np.ascontiguousarray(ref).view(np.uint32))


def test_project_refuses_pseudo_octaves():
    ctx = lb.default_context()
    dummy = ctx.to_device(np.zeros(64, np.float32))
    desc = (nat.CqtOctave * 1)(nat.CqtOctave(dummy.ptr, 1, 2, 0, 1, 0, 1, nat.CQT_PSEUDO))
    p = C.c_void_p(dummy.ptr)
    rc = nat.lib().b2l_cqt_project(ctx.handle, desc, 1, p, p, p, None, 1, 1, 1, p)
    dummy.free()
    assert rc != 0


@pytest.mark.parametrize("name", ["hcqt_defaults", "hcqt_scale_false", "hcqt_hop4096", "hcqt_one_pseudo",
                                  "hcqt_multichannel", "hcqt_sr16000_hop160"])
def test_rows_equal_own_cqt_and_pseudo_cqt(name):
    """hybrid_cqt's rows are this library's np.abs(cqt(n_bins=n_full)) and pseudo_cqt(fmin_pseudo, n_pseudo) bit for
    bit, trimmed to the shorter frame count."""
    case = HC.BY_NAME[name]
    y = HC.signal(case["sig"])
    kw, fmin, pp, n_full = _quiet(HO.split, case, y)
    got = _quiet(HC.call, lb, case)
    T = got.shape[-1]
    common = {k: kw[k] for k in ("sr", "hop_length", "bins_per_octave", "filter_scale", "norm", "sparsity", "window",
                                 "scale", "pad_mode")}
    full = np.abs(_quiet(lb.cqt, y, fmin=fmin, n_bins=n_full, res_type=kw["res_type"], **common))
    ps = _quiet(lb.pseudo_cqt, y, fmin=pp.freqs[0], n_bins=pp.n_bins, **common)
    assert np.array_equal(got[..., :n_full, :], full[..., :T])
    assert np.array_equal(got[..., n_full:, :], ps[..., :T])


@pytest.mark.parametrize("name", ["pcqt_fmin220", "pcqt_multichannel", "pcqt_tuning_none", "hcqt_defaults",
                                  "hcqt_multichannel", "hcqt_hop64", "hcqt_high_fmin", "hcqt_tuning_none"])
def test_device_call_identical_to_host_call(name):
    case = HC.BY_NAME[name]
    y = HC.signal(case["sig"])
    host = _quiet(HC.call, lb, case, y)
    dev = _quiet(HC.call, lb, case, lb.to_device(y))
    assert isinstance(dev, lb.DeviceArray) and dev.layout == "ft" and dev.dtype == np.float32
    got = dev.get()
    dev.free()
    assert got.shape == host.shape and np.array_equal(got, host)


@pytest.mark.parametrize("name", ["hcqt_defaults", "hcqt_hop4096", "hcqt_sr16000_hop160", "hcqt_hop64",
                                  "hcqt_high_fmin", "pcqt_fmin220"])
def test_launch_budget(name):
    """hybrid_cqt: the launches of cqt(n_bins=n_full) plus one STFT, still one projection launch; pseudo_cqt: two
    (its STFT and the projection)."""
    case = HC.BY_NAME[name]
    y = HC.signal(case["sig"])
    kw, fmin, pp, n_full = _quiet(HO.split, case, y)
    d = lb.to_device(y)
    ctx = d.ctx

    def count(fn):
        fn().free()   # plans and tables cached
        before = ctx.launch_count
        fn().free()
        return ctx.launch_count - before

    used = count(lambda: _quiet(HC.call, lb, case, d))
    if case["fn"] == "pseudo_cqt":
        assert used == 2
    else:
        want = 1 if pp is not None else 0
        if n_full:
            sub = {k: v for k, v in case["kw"].items() if k != "n_bins"}
            want += count(lambda: _quiet(lb.cqt, d, **dict(sub, fmin=fmin, n_bins=n_full)))
        else:
            want += 1   # the projection alone
        assert used == want
    d.free()


def test_many_clips():
    """70 001 short clips in one call (the projection slices the clip axis at 65 535)."""
    rng = np.random.default_rng(5)
    y = rng.standard_normal((70001, 1024)).astype(np.float32)
    kw = dict(sr=22050, hop_length=256, fmin=440.0, n_bins=24, res_type="polyphase")
    H = lb.hybrid_cqt(y, **kw)
    P_ = lb.pseudo_cqt(y, sr=22050, hop_length=256, fmin=880.0, n_bins=24)
    assert H.shape == (70001, 24, 5) and P_.shape == (70001, 24, 5)
    for k in (0, 65534, 65535, 70000):
        assert np.array_equal(H[k], lb.hybrid_cqt(y[k], **kw))
        assert np.array_equal(P_[k], lb.pseudo_cqt(y[k], sr=22050, hop_length=256, fmin=880.0, n_bins=24))


@pytest.mark.parametrize("name", ["pcqt_defaults", "hcqt_soxr_resamples", "hcqt_odd_hop"])
def test_refusals(name):
    with pytest.raises(lb.UnsupportedOnGPU):
        _quiet(HC.call, lb, HC.BY_NAME[name])


@pytest.mark.parametrize("case", [c for c in HC.CASES if f"{c['name']}/error" in GOLDEN.files and not c["refuse"]],
                         ids=lambda c: c["name"])
def test_errors_match_reference(case):
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        with pytest.raises(ParameterError) as e:
            HC.call(lb, case)
    assert f"ParameterError: {e.value}" == str(GOLDEN[f"{case['name']}/error"])
    assert [str(w.message) for w in caught if "n_fft=" in str(w.message)] == list(GOLDEN[f"{case['name']}/warnings"])


@pytest.mark.parametrize("name", ["pcqt_short_warns", "hcqt_hop4096", "pcqt_tuning_none"])
def test_stft_warnings(name):
    case = HC.BY_NAME[name]
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        HC.call(lb, case)
    assert [str(w.message) for w in caught if "n_fft=" in str(w.message)] == list(GOLDEN[f"{name}/warnings"])
