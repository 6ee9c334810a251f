"""chroma_cqt / chroma_cens / chroma_vqt / tonnetz on the GPU against tests/golden/chroma_v1.npz.

Tolerances, per clip, against the largest reference value of the clip:
  * C= / V= / chroma= (real input): rtol 1e-5, atol 1e-6 * max: only the summation order differs;
  * y= : the CQT's own rtol 1e-4, atol 1e-5 * max (tests/test_gpu_cqt.py);
  * CENS cannot be compared element by element: a chroma value within the CQT's error of a quantisation step moves
    a level, and the smoothing spreads it over the window.  So (a) the smoothing kernel fed the reference's quantised
    input is compared bit for bit, (b) chroma_cens equals the oracle's CENS steps applied to the GPU's own
    chroma_cqt(norm=None) within 1e-6, and (c) against the reference, every frame out of the smoothing reach of a
    value within 1e-3 relative of a step matches, with under 5 % of the frames excluded."""
from __future__ import annotations

import ctypes as C
import os
import warnings

import numpy as np
import pytest

import chroma_cases as HC
import chroma_oracle as HO
import librosa_b200 as lb
from librosa_b200 import _native as nat
from librosa_b200.feature.spectral import _smoothing_taps
from librosa_b200.util.exceptions import ParameterError

pytestmark = pytest.mark.gpu

GOLDEN = np.load(os.path.join(os.path.dirname(__file__), "golden", "chroma_v1.npz"))
RUNS = [c for c in HC.CASES if f"{c['name']}/out" in GOLDEN.files and not c["refuse"]]
STEPS = (0.4, 0.2, 0.1, 0.05)


def _call(case, arrays=None, **over):
    c = dict(case, kw=dict(case["kw"], **over))
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return HC.call(lb, c, GOLDEN, arrays=arrays)


def _close(got, ref, rtol, atol_rel):
    g = np.asarray(got).reshape((-1,) + ref.shape[-2:])
    r = ref.reshape((-1,) + ref.shape[-2:])
    for k in range(r.shape[0]):
        atol = atol_rel * float(np.abs(r[k]).max())
        err = np.abs(g[k] - r[k]) - (atol + rtol * np.abs(r[k]))
        assert err.max() <= 0, (k, float(np.abs(g[k] - r[k]).max()), atol)


def _tol(case):
    return (1e-4, 1e-5) if case["inp"] is None else (1e-5, 1e-6)


@pytest.mark.parametrize("case", [c for c in RUNS if c["fn"] != "chroma_cens"], ids=lambda c: c["name"])
def test_matches_reference(case):
    ref = GOLDEN[f"{case['name']}/out"]
    got = _call(case)
    assert isinstance(got, np.ndarray) and got.shape == ref.shape and got.dtype == ref.dtype
    _close(got, ref, *_tol(case))


def _cens_kw(case):
    kw = {k: case["kw"][k] for k in ("norm", "win_len_smooth", "smoothing_window") if k in case["kw"]}
    return dict(dict(norm=2, win_len_smooth=41, smoothing_window="hann"), **kw)


@pytest.mark.parametrize("case", [c for c in RUNS if c["fn"] == "chroma_cens"], ids=lambda c: c["name"])
def test_cens_against_its_own_chroma(case):
    """(b): the CENS steps of the oracle applied to the GPU's chroma_cqt(norm=None) of the same call."""
    got = _call(case)
    ref = GOLDEN[f"{case['name']}/out"]
    assert got.shape == ref.shape and got.dtype == ref.dtype
    arrays = HC.inputs(case, GOLDEN)
    kw = {k: v for k, v in case["kw"].items() if k not in ("norm", "win_len_smooth", "smoothing_window")}
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        raw = lb.feature.chroma_cqt(**arrays, **kw, norm=None, sr=case["sig"][2])
    want = HO.cens_tail(raw, **_cens_kw(case))
    assert np.abs(got - want).max() <= 1e-6


@pytest.mark.parametrize("name", ["cens_y_defaults", "cens_C_defaults", "cens_C_kaiser", "cens_C_win_500"])
def test_cens_against_the_reference_away_from_steps(name):
    """(c): a quantisation level differs from the reference's only where the reference's L1 chroma lies within
    1e-3 relative of a step; the frames within the smoothing reach of such a difference are excluded (under 5 %),
    and every other frame matches."""
    case = HC.BY_NAME[name]
    got, ref = _call(case), GOLDEN[f"{name}/out"]
    kw = {k: v for k, v in case["kw"].items() if k not in ("norm", "win_len_smooth", "smoothing_window")}
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        raw = lb.feature.chroma_cqt(**HC.inputs(case, GOLDEN), **kw, norm=None, sr=case["sig"][2])
    ref_l1 = HO.normalize(GOLDEN[f"{name}/raw"], norm=1, axis=-2)
    flips = HO.quantize(raw) != HO.quantize(GOLDEN[f"{name}/raw"])
    near = np.zeros(ref_l1.shape, bool)
    for s in STEPS:
        near |= np.abs(ref_l1 - s) <= 1e-3 * s
    assert not (flips & ~near).any()
    L = _cens_kw(case)["win_len_smooth"] + 2
    t = np.arange(ref.shape[-1])
    excluded = np.zeros(ref.shape[-1], bool)
    for f in np.flatnonzero(flips.reshape((-1,) + flips.shape[-2:]).any(axis=(0, 1))):
        excluded |= (t >= f - (L - 1 - L // 2)) & (t <= f + L // 2)   # the output frames a change at f reaches
    assert excluded.mean() < 0.05, excluded.mean()
    _close(got[..., ~excluded], ref[..., ~excluded], *_tol(case))


@pytest.mark.parametrize("name", ["cens_y_defaults", "cens_C_defaults", "cens_C_win_2", "cens_C_kaiser",
                                  "cens_C_win_500"])
def test_smoothing_kernel_bit_identical(name):
    """(a): b2l_chroma_smooth fed the reference's quantised input equals the reference's CENS bit for bit."""
    case = HC.BY_NAME[name]
    kw = _cens_kw(case)
    q = np.ascontiguousarray(GOLDEN[f"{name}/quant"])
    ref = GOLDEN[f"{name}/out"]
    off, w, L = _smoothing_taps(kw["smoothing_window"], kw["win_len_smooth"])
    ctx = lb.default_context()
    dq, doff, dw = ctx.to_device(q), ctx.to_device(off), ctx.to_device(w)
    out = nat.DeviceArray.empty(ctx, q.shape, q.dtype)
    kind, p = lb.feature.spectral._chroma_norm(kw["norm"])
    nat.check(nat.lib().b2l_chroma_smooth(ctx.handle, C.c_void_p(dq.ptr), 1, q.shape[-2], q.shape[-1],
                                          int(q.dtype == np.float64), C.c_void_p(doff.ptr), C.c_void_p(dw.ptr),
                                          len(off), L, kind, p, C.c_void_p(out.ptr)))
    got = out.get()
    for a in (dq, doff, dw, out):
        a.free()
    assert got.tobytes() == np.ascontiguousarray(ref).tobytes()


@pytest.mark.parametrize("name", ["cqt_y_defaults", "cens_y_defaults", "tonnetz_y", "vqt_y_list"])
def test_device_call_identical_to_host_call(name):
    case = HC.BY_NAME[name]
    y = HC.inputs(case)["y"]
    host = _call(case, {"y": y})
    dy = lb.to_device(y)
    dev = _call(case, {"y": dy})
    assert isinstance(dev, lb.DeviceArray) and dev.layout == "c"
    got = dev.get()
    dev.free()
    dy.free()
    assert got.shape == host.shape and np.array_equal(got, host)


@pytest.mark.parametrize("name", ["cqt_C_f32", "cqt_C_f64", "cens_C_defaults", "cqt_C_multichannel"])
def test_device_C_in_both_layouts(name):
    case = HC.BY_NAME[name]
    Ch = HC.inputs(case)["C"]
    host = _call(case, {"C": Ch})
    ctx = lb.default_context()
    dc = ctx.to_device(Ch)
    dft = ctx.to_device(np.ascontiguousarray(np.swapaxes(Ch, -1, -2)))
    dft.shape, dft.layout = Ch.shape, "ft"
    for d in (dc, dft):
        got = _call(case, {"C": d})
        assert isinstance(got, lb.DeviceArray)
        assert np.array_equal(got.get(), host)
        got.free()
    # a host array in [..., frame, bin] memory (cqt's order) gives the same result
    assert np.array_equal(_call(case, {"C": np.swapaxes(np.ascontiguousarray(np.swapaxes(Ch, -1, -2)), -1, -2)}), host)
    dc.free()
    dft.free()


def _launches(fn):
    ctx = lb.default_context()
    fn()
    before = ctx.launch_count
    r = fn()
    if isinstance(r, lb.DeviceArray):
        r.free()
    return ctx.launch_count - before


@pytest.mark.parametrize("name,extra", [("cqt_y_defaults", 1), ("vqt_y_equal", 1), ("tonnetz_y", 1),
                                        ("cens_y_defaults", 2)])
def test_launch_budget_y(name, extra):
    case = HC.BY_NAME[name]
    dy = lb.to_device(HC.inputs(case)["y"])
    kw = {k: v for k, v in case["kw"].items() if k in ("hop_length", "n_octaves", "res_type", "tuning")}
    if case["fn"] == "chroma_vqt":
        bpo, cq = 12, lb.vqt
        kw["gamma"] = case["kw"].get("gamma", 0)
    else:
        bpo, cq = 36, lb.cqt
        kw.setdefault("tuning", None)   # chroma_cqt's default
    n_oct = kw.pop("n_octaves", 7)
    base = _launches(lambda: cq(dy, sr=22050, n_bins=n_oct * bpo, bins_per_octave=bpo, **kw))
    assert _launches(lambda: _call(case, {"y": dy})) == base + extra
    if case["fn"] == "chroma_cens":
        assert _launches(lambda: _call(case, {"y": dy}, win_len_smooth=None)) == base + 1
    dy.free()


def test_launch_budget_C():
    case = HC.BY_NAME["cens_C_defaults"]
    dC = lb.to_device(HC.inputs(case)["C"])
    assert _launches(lambda: lb.feature.chroma_cqt(C=dC)) == 1
    assert _launches(lambda: lb.feature.chroma_cens(C=dC)) == 2
    assert _launches(lambda: lb.feature.chroma_cens(C=dC, win_len_smooth=None)) == 1
    assert _launches(lambda: lb.feature.tonnetz(chroma=lb.feature.chroma_cqt(C=dC).get())) == 1 + 1
    dC.free()


def test_many_clips():
    """70 001 clips through the C= path (the fold and the smoothing slice the clip axis at 65 535)."""
    rng = np.random.default_rng(4)
    Cb = rng.gamma(0.6, 1.0, size=(70001, 36, 6)).astype(np.float32)
    for fn in (lambda c: lb.feature.chroma_cqt(C=c, bins_per_octave=36),
               lambda c: lb.feature.chroma_cens(C=c, win_len_smooth=3)):
        batch = fn(Cb)
        for k in (0, 65534, 65535, 70000):
            assert np.array_equal(batch[k], fn(Cb[k]))


def test_device_chain_cens_to_dtw():
    """chroma_cens(y=DeviceArray) -> sequence.dtw on the device equals the same chain on host arrays."""
    case = HC.BY_NAME["cens_y_defaults"]
    y = HC.inputs(case)["y"]
    a, b = y[: len(y) // 2], y[len(y) // 4: len(y) // 4 + len(y) // 2]
    kw = dict(case["kw"], sr=22050)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        Xh, Yh = lb.feature.chroma_cens(y=a, **kw), lb.feature.chroma_cens(y=b, **kw)
        Dh, wph = lb.sequence.dtw(X=Xh, Y=Yh)
        da, db = lb.to_device(np.ascontiguousarray(a)), lb.to_device(np.ascontiguousarray(b))
        Xd, Yd = lb.feature.chroma_cens(y=da, **kw), lb.feature.chroma_cens(y=db, **kw)
        Dd, wpd = lb.sequence.dtw(X=Xd, Y=Yd)
    Dd = Dd.get() if isinstance(Dd, lb.DeviceArray) else Dd
    wpd = wpd.get() if isinstance(wpd, lb.DeviceArray) else wpd
    assert np.array_equal(Dd, Dh) and np.array_equal(wpd, wph)


@pytest.mark.parametrize("case", [c for c in HC.CASES if f"{c['name']}/error" in GOLDEN.files], ids=lambda c: c["name"])
def test_errors_match_reference(case):
    with pytest.raises(ParameterError) as e:
        _call(case)
    assert f"ParameterError: {e.value}" == str(GOLDEN[f"{case['name']}/error"])


def test_not_finite_audio_raises_the_cqt_error_first():
    y = HC.inputs(HC.BY_NAME["cqt_y_defaults"])["y"].copy()
    y[1000] = np.nan
    with pytest.raises(ParameterError, match="not finite everywhere"):
        lb.feature.chroma_cqt(y=y, hop_length=256, res_type="polyphase")


def test_float64_audio_keeps_the_reference_dtype():
    case = HC.BY_NAME["cens_y_defaults"]
    y = HC.inputs(case)["y"].astype(np.float64)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        got = lb.feature.chroma_cens(y=y, sr=22050, hop_length=256, res_type="polyphase")
    assert got.dtype == np.float64 and got.shape == GOLDEN["cens_y_defaults/out"].shape
