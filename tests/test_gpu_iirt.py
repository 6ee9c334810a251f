"""iirt on the GPU against tests/golden/iirt_v1.npz: every case within rtol 1e-4 and atol 1e-6 of each clip's
largest reference value, the filter and STMSP kernels bit-identical to the oracle when fed the reference's
resampled signals, host and DeviceArray calls identical, the launch budget, a 60 s clip, several clip groups under
a small memory pool, a batch above 65 535 clips, and the device's non-finite verdict."""
from __future__ import annotations

import os
import subprocess
import sys
import warnings

import numpy as np
import pytest

import iirt_cases as IC
import iirt_oracle as IO
import librosa_b200 as lb
from librosa_b200 import _native as nat
from librosa_b200.core import semitone as S
from librosa_b200.util.exceptions import ParameterError

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = np.load(os.path.join(os.path.dirname(__file__), "golden", "iirt_v1.npz"))
RUNS = [c for c in IC.CASES if f"{c['name']}/S" in GOLDEN.files and not c["refuse"]]


def _call(case, y=None):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return IC.call(lb, case) if y is None else lb.iirt(y, **case["kw"])


def _close_per_clip(got, ref, what=""):
    """rtol 1e-4, atol 1e-6 * the clip's largest reference value."""
    if ref.size == 0:
        assert np.shape(got) == ref.shape
        return
    g = np.asarray(got, dtype=np.float64).reshape((-1,) + ref.shape[-2:])
    r = np.asarray(ref, dtype=np.float64).reshape((-1,) + ref.shape[-2:])
    for k in range(r.shape[0]):
        if r[k].size == 0:
            continue
        atol = 1e-6 * float(r[k].max())
        err = np.abs(g[k] - r[k]) - (atol + 1e-4 * np.abs(r[k]))
        assert err.max() <= 0, (what, k, float(np.abs(g[k] - r[k]).max()), atol)


def _plan(case):
    kw, extra = IO.resolved(case)
    y = IC.signal(case["sig"])
    return S.plan(y.shape, sr=kw["sr"], win_length=kw["win_length"], hop_length=kw["hop_length"],
                  center=kw["center"], tuning=kw["tuning"], pad_mode=kw["pad_mode"], res_type=kw["res_type"],
                  kwargs=extra)


@pytest.mark.parametrize("case", RUNS, ids=lambda c: c["name"])
def test_matches_reference(case):
    ref = GOLDEN[f"{case['name']}/S"]
    got = _call(case)
    assert isinstance(got, np.ndarray) and got.shape == ref.shape and got.dtype == ref.dtype
    _close_per_clip(got, ref, case["name"])


@pytest.mark.parametrize("name", sorted(IC.WITH_STEPS))
def test_kernels_bit_identical(name):
    """b2l_iirt_filter and b2l_iirt_stmsp fed the reference's resampled signals (and the padded signal at sr):
    the stored band's filtered signal equals sosfiltfilt's and the power equals the reference's, bit for bit."""
    case = IC.BY_NAME[name]
    kw, _ = IO.resolved(case)
    y = IC.signal(case["sig"])
    yp = IO.padded(case, y).astype(np.float32)
    p = _plan(case)
    m = int(np.prod(yp.shape[:-1], dtype=np.int64))
    ctx = lb.default_context()
    held, signals = [], []
    for r in p.rates:
        x = yp if r.rate == kw["sr"] else GOLDEN[f"{name}/y{r.rate:g}"]
        d = ctx.to_device(np.ascontiguousarray(x.reshape(m, -1), dtype=np.float32))
        held.append(d)
        signals.append((d.ptr, r.n))
    scratch = nat.DeviceArray.empty(ctx, (p.scratch_bytes(m) // 8,), np.float64)
    out = nat.DeviceArray.empty(ctx, (m, len(p.bank.sos), p.n_frames), np.float32)
    S.filter_and_power(ctx, p, signals, m, scratch.ptr, out.ptr)
    scr, got = scratch.get(), out.get()
    for d in held + [scratch, out]:
        d.free()
    want, _ = IO.iirt(case, {r: GOLDEN[f"{name}/y{r:g}"] for r in (x.rate for x in p.rates) if r != kw["sr"]})
    assert np.array_equal(got.reshape(want.shape), want)
    assert np.array_equal(got.reshape(want.shape), GOLDEN[f"{name}/S"])
    b = IC.WITH_STEPS[name]
    ri = int(p.bank.rate_of[b])
    j = int(np.flatnonzero(p.bank.bands[p.bank.band_off[ri]:p.bank.band_off[ri + 1]] == b)[0])
    off = sum(r.rows * (-(-m * r.n_bands // 32) * 32) for r in p.rates[:ri])
    rr = p.rates[ri]
    st = -(-m * rr.n_bands // 32) * 32
    rows = scr[off:off + rr.rows * st].reshape(rr.rows, st)
    band = GOLDEN[f"{name}/band{b}"].reshape(m, -1)
    for clip in range(m):
        assert np.array_equal(rows[:rr.n, clip * rr.n_bands + j], band[clip])


@pytest.mark.parametrize("name", ["defaults", "multichannel", "tuning_03", "center_false"])
def test_device_call_identical_to_host_call(name):
    case = IC.BY_NAME[name]
    y = IC.signal(case["sig"])
    host = _call(case, y)
    dev = _call(case, lb.to_device(y))
    assert isinstance(dev, lb.DeviceArray) and dev.dtype == np.float32
    got = dev.get()
    dev.free()
    assert got.shape == host.shape and np.array_equal(got, host)


@pytest.mark.parametrize("name", ["defaults", "center_false", "sr_only_no_resample", "sr16000", "multichannel"])
def test_launch_budget(name):
    """A host call: the finite scan, the pad (center=True), one resample per rate other than sr, then one filter
    and one STMSP launch per clip group (one group here); a device call skips the scan."""
    case = IC.BY_NAME[name]
    y = IC.signal(case["sig"])
    p = _plan(case)
    resamples = sum(1 for r in p.rates if r.up)
    ctx = lb.default_context()
    _call(case, y)
    before = ctx.launch_count
    _call(case, y)
    assert ctx.launch_count - before == 1 + (1 if p.pad else 0) + resamples + 2
    d = lb.to_device(y)
    before = ctx.launch_count
    _call(case, d).free()
    assert ctx.launch_count - before == (1 if p.pad else 0) + resamples + 2
    d.free()


def test_long_clip():
    """60 s in one call: chains of 1.3 M samples at 22 050 Hz."""
    case = IC._c("sixty_seconds", IC.P, ((), 60 * 22050, 22050, np.float32))
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        ref, _ = IO.iirt(case)
    got = _call(case)
    assert got.shape == ref.shape == (85, 1 + 60 * 22050 // 512)
    _close_per_clip(got, ref, "60 s")


_GROUPS = r"""
import sys, numpy as np
sys.path.insert(0, sys.argv[1])
import librosa_b200 as lb
from librosa_b200.core import semitone as S
y = np.load(sys.argv[2])
ctx = lb.default_context()
before = ctx.launch_count
out = lb.iirt(y, sr=22050, res_type="polyphase")
p = S.plan(y.shape, sr=22050, win_length=2048, hop_length=None, center=True, tuning=0.0, pad_mode="constant",
           res_type="polyphase", kwargs={})
np.save(sys.argv[3], out)
print(ctx.launch_count - before, S.group_size(p, y.shape[0], ctx.pool_limit_bytes))
"""


def test_clip_groups_under_a_small_pool(tmp_path):
    """B2L_POOL_LIMIT_MB=10 leaves room for two 1 s clips per group: four groups of a batch of eight equal one."""
    y = np.stack([IC.signal(((), 22050, 22050, np.float32, k)) for k in range(8)])
    np.save(tmp_path / "y.npy", y)
    env = dict(os.environ, B2L_POOL_LIMIT_MB="10")
    res = subprocess.run([sys.executable, "-c", _GROUPS, ROOT, str(tmp_path / "y.npy"), str(tmp_path / "out.npy")],
                         env=env, capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stderr
    launches, g = map(int, res.stdout.split()[-2:])
    assert g == 2 and launches == 1 + 1 + 2 + 2 * 4
    want = lb.iirt(y, sr=22050, res_type="polyphase")
    assert np.array_equal(np.load(tmp_path / "out.npy"), want)


def test_many_clips():
    """70 001 clips of 0.1 s in one call equal the clips computed one at a time."""
    rng = np.random.default_rng(5)
    y = (0.1 * rng.standard_normal((70001, 2205))).astype(np.float32)
    out = lb.iirt(y, sr=22050, res_type="polyphase")
    assert out.shape == (70001, 85, 5)
    for k in (0, 65534, 65535, 70000):
        assert np.array_equal(out[k], lb.iirt(y[k], sr=22050, res_type="polyphase"))


def test_not_finite():
    with pytest.raises(ParameterError) as e:
        _call(IC.BY_NAME["not_finite"])
    assert f"ParameterError: {e.value}" == str(GOLDEN["not_finite/error"])


def test_float64_returns_float64():
    case = IC.BY_NAME["float64"]
    got = _call(case)
    assert got.dtype == np.float64
    _close_per_clip(got, GOLDEN["float64/S"])
