"""yin / pyin on the GPU against tests/pitch_oracle.py: the CMND kernel, each decision kernel on the very input the
oracle sees, end to end on the tonal cases, the reference's own pitch tests, launch counts and the refused sizes."""
import ctypes as C
import os
import warnings

import numpy as np
import pytest

import librosa_b200 as lb
import pitch_cases as PC
import pitch_oracle as PO
from librosa_b200 import _native as nat
from librosa_b200.core import pitch as P

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_vp = C.c_void_p
_PYIN_KW = ("n_thresholds", "beta_parameters", "boltzmann_parameter", "resolution", "max_transition_rate",
            "switch_prob", "no_trough_prob", "fill_na", "transition_min_prob")
_PYIN_DEFAULTS = dict(n_thresholds=100, beta_parameters=(2, 18), boltzmann_parameter=2, resolution=0.1,
                      max_transition_rate=35.92, switch_prob=0.01, no_trough_prob=0.01, fill_na=np.nan,
                      transition_min_prob=1e-4)


def _geometry(case):
    kw = dict(case["kw"])
    sr = kw.get("sr", 22050)
    L = kw.get("frame_length", 2048)
    hop = kw.get("hop_length") or L // 4
    lo, hi = PO.periods(sr, kw["fmin"], kw["fmax"], L)
    return kw, sr, L, hop, lo, hi


def _frame_kw(kw):
    return {k: kw[k] for k in ("fmin", "fmax", "sr", "frame_length", "hop_length", "center", "pad_mode") if k in kw}


def _oracle_cmnd(case):
    """Oracle CMND of a case, rows-major: (lead, [rows][n_lags] float64)."""
    y = PC.make_input(case)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        cm = PO.yin_cmnd(y, **_frame_kw(case["kw"]))
    lead = cm.shape[:-2]
    return y, lead, np.ascontiguousarray(np.swapaxes(cm, -1, -2)).reshape(-1, cm.shape[-2])


def _gpu_cmnd(case, y):
    """GPU CMND of a case through b2l_yin_cmnd: [rows][n_lags] float32."""
    kw, sr, L, hop, lo, hi = _geometry(case)
    ctx = lb.default_context()
    yd = ctx.to_device(np.ascontiguousarray(y, dtype=np.float32))
    lead, n = yd.shape[:-1], yd.shape[-1]
    center = kw.get("center", True)
    T = 1 + (n + (2 * (L // 2) if center else 0) - L) // hop
    n_clips = int(np.prod(lead)) if lead else 1
    desc = nat.YinDesc(frame_length=L, hop_length=hop, center=int(center),
                       pad_mode=nat.PAD_MODES[kw.get("pad_mode", "constant") if center else "constant"],
                       min_period=lo, max_period=hi, sr=float(sr))
    out = ctx.empty((n_clips * T, hi - lo + 1), np.float32)
    nat.check(nat.lib().b2l_yin_cmnd(ctx.handle, C.byref(desc), _vp(yd.ptr), n_clips, n, n, _vp(out.ptr)))
    return out.get().copy()


def _to_frames(rows, lead, n_lags):
    """[rows][n_lags] -> (..., n_lags, n_frames) as the oracle holds it."""
    return np.swapaxes(rows.reshape(lead + (-1, n_lags)), -1, -2)


@pytest.mark.parametrize("name", [c["name"] for c in PC.PITCH_CASES])
def test_cmnd_vs_oracle(name):
    case = PC.BY_NAME[name]
    y, lead, ref = _oracle_cmnd(case)
    got = _gpu_cmnd(case, y).astype(np.float64)
    assert got.shape == ref.shape
    err = np.abs(got - ref)
    excess = err - (1e-5 + 1e-4 * np.abs(ref))
    print(f"{name}: max |d| {err.max():.3g}, max |d| / (|ref| + 1e-3) {(err / (np.abs(ref) + 1e-3)).max():.3g}")
    assert excess.max() <= 0, (err.max(), np.unravel_index(np.argmax(excess), err.shape))


def _pyin_desc(case, where):
    kw, sr, L, hop, lo, hi = _geometry(case)
    opts = dict(_PYIN_DEFAULTS)
    opts.update({k: kw[k] for k in _PYIN_KW if k in kw})
    return P._pyin_setup(where, min_period=lo, max_period=hi, hop_length=hop, sr=sr, fmin=kw["fmin"], fmax=kw["fmax"],
                         **opts), opts


def _run_obs(ctx, desc, max_cand, d_cmnd, rows):
    L = nat.lib()
    cnt, cb = ctx.empty((rows,), np.int32), ctx.empty((rows, max_cand), np.int32)
    cp, vp = ctx.empty((rows, max_cand), np.float64), ctx.empty((rows,), np.float64)
    nat.check(L.b2l_pyin_obs(ctx.handle, C.byref(desc), _vp(d_cmnd.ptr), rows, _vp(cnt.ptr), _vp(cb.ptr), _vp(cp.ptr),
                             _vp(vp.ptr)))
    return cnt.get().copy(), cb.get().copy(), cp.get().copy(), vp.get().copy()


def _dense(cnt, cb, cp, npb):
    """Compact candidates -> the voiced half of the oracle's observation matrix, [rows][npb]."""
    out = np.zeros((len(cnt), npb))
    for r, c in enumerate(cnt):
        out[r, cb[r, :c]] = cp[r, :c]
    return out


def _compact(obs_rows, npb, max_cand):
    """[rows][2 npb] oracle observations -> compact candidates (bins ascending)."""
    rows = obs_rows.shape[0]
    cnt = np.zeros(rows, np.int32)
    cb = np.zeros((rows, max_cand), np.int32)
    cp = np.zeros((rows, max_cand))
    for r in range(rows):
        nz = np.flatnonzero(obs_rows[r, :npb])
        cnt[r] = len(nz)
        cb[r, : len(nz)] = nz
        cp[r, : len(nz)] = obs_rows[r, nz]
    return cnt, cb, cp


def _run_viterbi(ctx, desc, cnt, cb, cp, vp, n_clips, n_frames, with_f0=False):
    L = nat.lib()
    dev = [ctx.to_device(a) for a in (cnt, cb, cp, vp)]
    st = ctx.empty((n_clips, n_frames), np.uint16)
    f0 = ctx.empty((n_clips, n_frames), np.float64) if with_f0 else None
    vf = ctx.empty((n_clips, n_frames), np.bool_) if with_f0 else None
    nat.check(L.b2l_viterbi(ctx.handle, C.byref(desc), *[_vp(d.ptr) for d in dev], n_clips, n_frames, _vp(st.ptr),
                            _vp(f0.ptr) if f0 else None, _vp(vf.ptr) if vf else None))
    if with_f0:
        return st.get().copy(), f0.get().copy(), vf.get().copy()
    return st.get().copy()


@pytest.mark.parametrize("name", [c["name"] for c in PC.PITCH_CASES])
def test_decisions_on_identical_input(name):
    """The oracle's CMND rounded to float32 goes to the decision kernels; the oracle runs on the same values."""
    case = PC.BY_NAME[name]
    kw, sr, L, hop, lo, hi = _geometry(case)
    y, lead, ref = _oracle_cmnd(case)
    c32 = ref.astype(np.float32)
    n_lags = hi - lo + 1
    x64 = _to_frames(c32.astype(np.float64), lead, n_lags)
    ctx = lb.default_context()
    d_c = ctx.to_device(c32)
    rows = c32.shape[0]
    if PC.op(case) == "yin":
        desc = nat.YinDesc(min_period=lo, max_period=hi, sr=float(sr),
                           trough_threshold=float(kw.get("trough_threshold", 0.1)))
        f0 = ctx.empty((rows,), np.float64)
        nat.check(nat.lib().b2l_yin_pick(ctx.handle, C.byref(desc), _vp(d_c.ptr), rows, _vp(f0.ptr)))
        want = PO.yin_pick(x64, sr=sr, min_period=lo, trough_threshold=kw.get("trough_threshold", 0.1))
        assert np.array_equal(f0.get().reshape(want.shape), want)
        return
    (ctx, desc, max_cand), opts = _pyin_desc(case, d_c)
    npb = desc.n_pitch_bins
    cnt, cb, cp, vp = _run_obs(ctx, desc, max_cand, d_c, rows)
    obs, vp_ref = PO.pyin_observations(x64, sr=sr, fmin=kw["fmin"], fmax=kw["fmax"], min_period=lo,
                                       n_thresholds=opts["n_thresholds"], beta_parameters=opts["beta_parameters"],
                                       boltzmann_parameter=opts["boltzmann_parameter"],
                                       resolution=opts["resolution"], no_trough_prob=opts["no_trough_prob"])
    obs_rows = np.swapaxes(obs, -1, -2).reshape(rows, 2 * npb)
    dense = _dense(cnt, cb, cp, npb)
    assert np.array_equal(dense != 0, obs_rows[:, :npb] != 0)
    np.testing.assert_allclose(dense, obs_rows[:, :npb], rtol=1e-12, atol=0)
    np.testing.assert_allclose(vp, vp_ref.reshape(-1), rtol=1e-12, atol=0)
    # the Viterbi on the oracle's own observations
    n_clips = int(np.prod(lead)) if lead else 1
    T = rows // n_clips
    ocnt, ocb, ocp = _compact(obs_rows, npb, max_cand)
    states = _run_viterbi(ctx, desc, ocnt, ocb, ocp, vp_ref.reshape(-1), n_clips, T)
    _, _, want = PO.pyin_decode(obs, fmin=kw["fmin"], n_pitch_bins=npb, n_bins_per_semitone=desc.n_bins_per_semitone,
                                sr=sr, hop_length=hop, max_transition_rate=opts["max_transition_rate"],
                                switch_prob=opts["switch_prob"], transition_min_prob=opts["transition_min_prob"])
    assert np.array_equal(states, want.reshape(n_clips, T))


def _exempt(x64, thresholds, frames):
    """Frames (indices into the last axis of x64 (n_lags, n_frames)) where the oracle has a trough within 1e-5 of a
    threshold or a localmin comparison within 1e-6."""
    out = []
    for t in frames:
        x = x64[:, t]
        tr = PO.localmin(x)
        tr[0] = x[0] < x[1]
        near_thr = np.any(np.abs(x[tr][:, None] - np.asarray(thresholds)[None, :]) < 1e-5)
        near_cmp = np.any(np.abs(np.diff(x)) < 1e-6)
        if near_thr or near_cmp:
            out.append(t)
    return out


TONAL = [c["name"] for c in PC.PITCH_CASES if c["tonal"]]


@pytest.mark.parametrize("name", TONAL)
def test_end_to_end(name):
    case = PC.BY_NAME[name]
    kw, sr, L, hop, lo, hi = _geometry(case)
    y = PC.make_input(case)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        got = PC.run(lb, case)
        want = PC.run(PO, case)
    _, lead, cm = _oracle_cmnd(case)
    n_lags = hi - lo + 1
    xs = _to_frames(cm, lead, n_lags).reshape((-1, n_lags, cm.shape[0] // max(1, int(np.prod(lead)))))
    if PC.op(case) == "yin":
        assert got.dtype == np.float64 and got.shape == want.shape
        bad = ~np.isclose(got, want, rtol=1e-5, atol=0)
        bad_rows = np.argwhere(bad.reshape(xs.shape[0], -1))
        exempt = [(c, t) for c, t in bad_rows if _exempt(xs[c], [kw.get("trough_threshold", 0.1)], [t])]
        print(f"{name}: {len(bad_rows)} differing frames, {len(exempt)} exempt")
        assert len(exempt) == len(bad_rows)
        return
    f0, vf, vp = got
    f0o, vfo, vpo = want
    assert f0.dtype == np.float64 and vf.dtype == np.bool_ and vp.dtype == np.float64
    assert f0.shape == f0o.shape == vf.shape == vp.shape
    n_thr = kw.get("n_thresholds", 100)
    thresholds = np.linspace(0, 1, n_thr + 1)[1:]
    vp_bad = ~np.isclose(vp, vpo, rtol=0, atol=1e-5)
    path_bad = (vf != vfo) | ~((f0 == f0o) | (np.isnan(f0) & np.isnan(f0o)))
    C_ = xs.shape[0]
    vp_rows = np.argwhere(vp_bad.reshape(C_, -1))
    exempt = [(c, t) for c, t in vp_rows if _exempt(xs[c], thresholds, [t])]
    print(f"{name}: voiced_prob differs on {len(vp_rows)} frames ({len(exempt)} exempt); "
          f"path differs on {int(path_bad.sum())} frames")
    assert len(exempt) == len(vp_rows)
    if path_bad.any():
        # the path may move only with its observations: the oracle's Viterbi on the GPU's observations gives it
        (ctx, desc, max_cand), opts = _pyin_desc(case, lb.default_context().empty((1,), np.float32))
        g = _gpu_cmnd(case, y)
        d_c = ctx.to_device(g)
        cnt, cb, cp, vpg = _run_obs(ctx, desc, max_cand, d_c, g.shape[0])
        npb = desc.n_pitch_bins
        obs = np.zeros((g.shape[0], 2 * npb))
        obs[:, :npb] = _dense(cnt, cb, cp, npb)
        obs[:, npb:] = ((1 - vpg) / npb)[:, None]
        obs = np.swapaxes(obs.reshape(C_, -1, 2 * npb), -1, -2)
        f0x, vfx, _ = PO.pyin_decode(obs, fmin=kw["fmin"], n_pitch_bins=npb,
                                     n_bins_per_semitone=desc.n_bins_per_semitone, sr=sr, hop_length=hop,
                                     fill_na=kw.get("fill_na", np.nan),
                                     transition_min_prob=kw.get("transition_min_prob", 1e-4))
        assert np.array_equal(vfx.reshape(vf.shape), vf)
        assert np.array_equal(f0x.reshape(f0.shape), f0, equal_nan=True)
        assert len(exempt) > 0


# ---- the reference's own pitch tests (tests/test_core.py), restated on the GPU
@pytest.mark.parametrize("freq", [110, 220, 440, 880])
def test_yin_tone(freq):
    f0 = lb.yin(PC.tone(freq), fmin=110, fmax=880, center=False)
    assert np.allclose(np.log2(f0), np.log2(freq), rtol=0, atol=1e-2)


@pytest.mark.parametrize("freq", [110, 220, 440, 880])
def test_pyin_tone(freq):
    f0, _, _ = lb.pyin(PC.tone(freq), fmin=110, fmax=1000, center=False)
    assert np.allclose(np.log2(f0), np.log2(freq), rtol=0, atol=1e-2)


def test_yin_chirp():
    f0 = lb.yin(PC.chirp(220, 640), fmin=110, fmax=880, center=False, frame_length=1024, hop_length=512)
    target = np.load(os.path.join(ROOT, "tests", "golden", "pitch-yin.npy"))
    assert np.allclose(np.log2(f0[:-2]), np.log2(target), rtol=0, atol=1e-2)


def test_yin_chirp_instant():
    sr = 22050
    f = 220 * (640 / 220) ** (np.arange(sr) / sr)
    target = PO.frame(f, 2048, 512).mean(axis=0)
    f0 = lb.yin(PC.chirp(220, 640), fmin=110, fmax=880, sr=sr, frame_length=2048, hop_length=512, center=False)
    assert np.allclose(np.log2(f0), np.log2(target), rtol=0, atol=1e-2)


def test_pyin_chirp():
    y = np.pad(PC.chirp(220, 640), (22050,))
    f0, vf, _ = lb.pyin(y, fmin=60, fmax=900, center=False, frame_length=1024, hop_length=512, resolution=0.2)
    f0, vf = f0[:-2], vf[:-2]
    target = np.load(os.path.join(ROOT, "tests", "golden", "pitch-pyin.npy"))
    assert np.array_equal(vf, target > 0)
    assert np.allclose(np.log2(f0[vf]), np.log2(target[target > 0]), rtol=0, atol=1e-2)


def test_pyin_chirp_instant():
    sr = 22050
    f = np.pad(220 * (640 / 220) ** (np.arange(sr) / sr), (sr,))
    fr = PO.frame(f, 2048, 512)
    with np.errstate(invalid="ignore", divide="ignore"), warnings.catch_warnings():
        warnings.simplefilter("ignore")
        target = fr.mean(axis=0, where=fr > 0)
    y = np.pad(PC.chirp(220, 640), (sr,))
    f0, vf, _ = lb.pyin(y, fmin=110, fmax=880, frame_length=2048, hop_length=512, center=False)
    assert np.array_equal(vf, target > 0)
    cents, tc = np.log2(f0[vf]), np.log2(target[target > 0])
    assert np.allclose(np.log2(cents[1:-1]), np.log2(tc[1:-1]), rtol=0, atol=1e-2)
    assert abs(cents[0] - tc[0]) <= 1e-1 and abs(cents[-1] - tc[-1]) <= 1e-1


def test_pyin_multi():
    y = PC.taper(np.stack([PC.tone(440), PC.tone(560)]))
    fall, vall, vpall = lb.pyin(y, fmin=100, fmax=1000, center=False, fill_na=-1)
    for i in range(2):
        f, v, vp = lb.pyin(y[i], fmin=100, fmax=1000, center=False, fill_na=-1)
        assert np.array_equal(fall[i], f) and np.array_equal(vall[i], v) and np.array_equal(vpall[i], vp)


def test_pyin_multi_center():
    y = PC.taper(np.stack([PC.tone(440), PC.tone(560)]))
    fl, vl, vpl = lb.pyin(y, fmin=100, fmax=1000, center=False)
    fc, vc, vpc = lb.pyin(y, fmin=100, fmax=1000, center=True)
    assert np.allclose(vpl, vpc[..., 2:-2])
    assert np.allclose(vl, vc[..., 2:-2])
    assert np.allclose(fl, fc[..., 2:-2], equal_nan=True)


def test_device_in_device_out_and_float64():
    y = PC.make_input(PC.BY_NAME["yin/stereo"])
    yd = lb.to_device(y)
    f0 = lb.yin(yd, fmin=PC.C2, fmax=PC.C7)
    assert isinstance(f0, lb.DeviceArray) and f0.dtype == np.float64
    assert np.array_equal(f0.get(), lb.yin(y, fmin=PC.C2, fmax=PC.C7))
    outs = lb.pyin(yd, fmin=PC.C2, fmax=PC.C7)
    assert all(isinstance(o, lb.DeviceArray) for o in outs)
    assert [o.dtype for o in outs] == [np.float64, np.bool_, np.float64]
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        f64 = lb.yin(y.astype(np.float64), fmin=PC.C2, fmax=PC.C7)
    assert np.array_equal(f64, lb.yin(y, fmin=PC.C2, fmax=PC.C7))


def test_nonfinite_input():
    y = PC.tone(220)
    y[100] = np.nan
    with pytest.raises(lb.ParameterError, match="not finite"):
        lb.yin(y, fmin=110, fmax=880)
    with pytest.raises(lb.ParameterError, match="not finite"):
        lb.pyin(y, fmin=110, fmax=880)


@pytest.mark.parametrize("fn,per_call", [(lb.yin, 2), (lb.pyin, 3)])
def test_launch_counts(fn, per_call):
    """A fixed number of kernels per call, whatever the batch and the length: no per-frame host work."""
    ctx = lb.default_context()
    counts = []
    for shape in [(1, 8000), (8, 8000), (3, 40000)]:
        yd = lb.to_device(PC.make_input(dict(name="x", sig=("mix", "T", shape))))
        fn(yd, fmin=110, fmax=1000)
        ctx.synchronize()
        before = ctx.launch_count
        fn(yd, fmin=110, fmax=1000)
        ctx.synchronize()
        counts.append(ctx.launch_count - before)
    assert counts == [per_call] * 3


def test_unsupported_sizes():
    y = PC.tone(220, duration=2.0)
    with pytest.raises(lb.UnsupportedOnGPU, match="16384"):
        lb.yin(y, fmin=10, fmax=1000, frame_length=8192)
    with pytest.raises(lb.UnsupportedOnGPU, match="states"):
        lb.pyin(y, fmin=PC.C2, fmax=PC.C7, resolution=0.005)
