"""piptrack, pitch_tuning and util.localmax / localmin on the GPU: every case of tests/golden/piptrack_v1.npz
bit-identical to the reference (a case from y: bit-identical to the oracle run on this library's own spectrogram,
whose STFT is not NumPy's), zero off the peaks; host calls, device calls and both device layouts identical;
pitch_tuning of device pitches; the launch budget of each call; more than 65 535 frames in one call."""
from __future__ import annotations

import os
import warnings

import numpy as np
import pytest

import piptrack_cases as PC
import piptrack_oracle as PO
import librosa_b200 as lb
from librosa_b200 import _native as nat

pytestmark = pytest.mark.gpu

GOLDEN = np.load(os.path.join(os.path.dirname(__file__), "golden", "piptrack_v1.npz"))
STORED = [c for c in PC.CASES if not c["refuse"] and f"{c['name']}/error" not in GOLDEN.files]
PIP = [c for c in STORED if c["fn"] == "piptrack"]


def _bytes(a):
    return np.ascontiguousarray(a).tobytes()


def _same(got, want):
    for g, w in zip(got, want):
        assert isinstance(g, np.ndarray) and g.flags.c_contiguous
        assert g.dtype == w.dtype and g.shape == w.shape, (g.dtype, w.dtype, g.shape, w.shape)
        assert _bytes(g) == _bytes(w)


def _device(x, layout):
    ctx = lb.default_context()
    if layout == "c":
        return ctx.to_device(np.ascontiguousarray(x))
    d = nat.DeviceArray.empty(ctx, x.shape, x.dtype, layout="ft")
    return d.set(np.swapaxes(x, -1, -2))


def _own_spectrogram(case):
    """The magnitude spectrogram of this library, as piptrack computes it from y (float32)."""
    kw = PC.piptrack_args(case)
    y = np.asarray(kw["y"], np.float32)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return PO.spectrogram(lambda y_, **k: lb.core.spectrum._spectrogram(y=y_, power=1, **k)[0], y,
                              **{k: v for k, v in kw.items() if k != "y"})


@pytest.mark.parametrize("case", STORED, ids=lambda c: c["name"])
def test_every_case(case):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        got = PC.call(lb, case)
    if case["fn"] == "piptrack":
        if case["y"] is None:
            _same(got, PC.dense(GOLDEN, case["name"]))
        else:
            kw = PC.piptrack_args(case)
            kw.pop("y")
            kw["S"] = _own_spectrogram(case)
            want = PO.piptrack(**kw)
            dt = GOLDEN[f"{case['name']}/p"].dtype
            _same(got, tuple(w.astype(dt) for w in want))
    elif case["fn"] == "pitch_tuning":
        assert got == GOLDEN[f"{case['name']}/out"]
    else:
        want = GOLDEN[f"{case['name']}/out"]
        assert isinstance(got, np.ndarray) and got.dtype == np.bool_ and np.array_equal(got, want)


DEVICE_PIP = [c for c in PIP if c["S"] is not None and np.dtype(PC.spectrum(c["S"]).dtype).kind == "f"]


@pytest.mark.parametrize("case", DEVICE_PIP, ids=lambda c: c["name"])
def test_device_calls_equal_host_calls(case):
    S = PC.spectrum(case["S"])
    host = PC.call(lb, case)
    ctx = lb.default_context()
    for layout in ("c", "ft"):
        d = _device(S, layout)
        before = ctx.launch_count
        p, m = lb.piptrack(**PC.piptrack_args(case, S=d))
        assert ctx.launch_count - before == 2   # the sign pass and the tracking kernel
        assert isinstance(p, nat.DeviceArray) and p.layout == "ft" and m.layout == "ft"
        _same((np.ascontiguousarray(p.get()), np.ascontiguousarray(m.get())), host)
    # a Fortran-ordered host S (np.abs(stft) of one clip) is uploaded as it is
    _same(lb.piptrack(**PC.piptrack_args(case, S=np.asfortranarray(S))), host)


def test_launch_budget():
    ctx = lb.default_context()
    S = PC.spectrum(((1025, 50), np.float32, 3))
    before = ctx.launch_count
    lb.piptrack(S=S)
    assert ctx.launch_count - before == 1
    before = ctx.launch_count
    lb.piptrack(S=-S)   # negative entries: |S| in the same launch
    assert ctx.launch_count - before == 1
    y = PC.signal(((22050,), 4))
    d_y = lb.to_device(y)
    before = ctx.launch_count
    lb.core.spectrum._spectrogram(y=d_y, n_fft=2048, power=1)
    spec = ctx.launch_count - before
    before = ctx.launch_count
    p, _ = lb.piptrack(y=d_y, sr=22050)
    assert ctx.launch_count - before == spec + 1
    before = ctx.launch_count
    lb.pitch_tuning(p)
    assert ctx.launch_count - before == 1
    for fn in (lb.util.localmax, lb.util.localmin):
        before = ctx.launch_count
        fn(S, axis=0)
        assert ctx.launch_count - before == 1


def test_y_host_and_device_agree():
    y = PC.signal(((2, 22050), 5))
    hp, hm = lb.piptrack(y=y, sr=22050, n_fft=1024)
    dp, dm = lb.piptrack(y=lb.to_device(y), sr=22050, n_fft=1024)
    _same((np.ascontiguousarray(dp.get()), np.ascontiguousarray(dm.get())), (hp, hm))
    S = lb.core.spectrum._spectrogram(y=y, n_fft=1024, hop_length=None, power=1)[0]
    _same((hp, hm), PO.piptrack(S=np.asarray(S), sr=22050, n_fft=1024))


def test_pitch_tuning_of_device_pitches():
    y = PC.signal(((3, 22050), 6))
    dp, _ = lb.piptrack(y=lb.to_device(y), sr=22050)
    hp, _ = lb.piptrack(y=y, sr=22050)
    for kw in ({}, {"resolution": 1 / 3}, {"bins_per_octave": 24}):
        assert lb.pitch_tuning(dp, **kw) == lb.pitch_tuning(hp, **kw) == PO.pitch_tuning(hp, **kw)
    d64 = lb.to_device(hp.astype(np.float64))
    assert lb.pitch_tuning(d64) == PO.pitch_tuning(hp.astype(np.float64))


LOCAL = [c for c in STORED if c["fn"] in ("localmax", "localmin") and PC.values(c["spec"]).ndim >= 2]


@pytest.mark.parametrize("case", LOCAL, ids=lambda c: c["name"])
def test_localext_device_layouts(case):
    x = PC.values(case["spec"])
    want = GOLDEN[f"{case['name']}/out"]
    for layout in ("c", "ft"):
        out = PC.call(lb, case, _device(x, layout))
        assert isinstance(out, nat.DeviceArray) and out.layout == layout and out.dtype == np.bool_
        assert np.array_equal(out.get(), want)


def test_more_than_65535_frames():
    S = PC.spectrum(((70001, 65, 3), np.float32, 7))
    S = np.ascontiguousarray(np.swapaxes(S, 0, 1).reshape(65, -1))   # one clip of 210 003 frames
    p, m = lb.piptrack(S=S, fmin=0.0)
    _same((p, m), PO.piptrack(S=S, fmin=0.0))
    clips = np.ascontiguousarray(S.reshape(65, 70001, 3).transpose(1, 0, 2))   # 70 001 clips of 3 frames
    cp, cm = lb.piptrack(S=clips, fmin=0.0)
    for i in (0, 65534, 65535, 65536, 70000):
        _same((cp[i], cm[i]), lb.piptrack(S=clips[i], fmin=0.0))
    lm = lb.util.localmax(S, axis=0)
    assert np.array_equal(lm, PO.localmax(S, axis=0))
    assert np.array_equal(lb.util.localmin(clips, axis=1), PO.localmin(clips, axis=1))
