"""Alignment on the GPU against tests/golden/alignment_v1.npz (the unmodified reference) and
tests/alignment_oracle.py:

* the public calls with host arrays and with DeviceArrays are bit-identical to the fixture on every case (cosine
  included: the cost kernel keeps scipy's summation order), and error cases raise the reference's class and message;
* launch counts and read-backs: one launch per anti-diagonal of 32 x 32 tiles, one 8-byte length word per path, one
  4-byte verdict word when there is no path to carry it;
* a (0, 0) step on the path, where the reference's walk never ends, is a clean UnsupportedOnGPU;
* one rqa over more than 2^31 cells, with its maximum and path placed past flat index 2^31."""
import ctypes as C
import os
import warnings

import numpy as np
import pytest

import alignment_cases as AC
import librosa_b200 as lb
from librosa_b200 import _native as nat

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TILE = 32
DEVICE_OPS = ("dtw", "dtw_backtracking", "rqa")


@pytest.fixture(scope="module")
def golden():
    with np.load(os.path.join(ROOT, "tests", "golden", "alignment_v1.npz")) as z:
        return {k: z[k] for k in z.files}


def _host(got):
    return {k: (v.get() if isinstance(v, lb.DeviceArray) else v) for k, v in got.items()}


def _device_call(case):
    X, Y, Cm, sim = AC.inputs(case)
    dev = [lb.to_device(np.ascontiguousarray(a)) if a is not None else None for a in (X, Y, Cm, sim)]
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        got = AC.call(lb, case, *dev)
    for k, v in got.items():
        if k != "error":
            assert isinstance(v, lb.DeviceArray), (case["name"], k)
    return _host(got)


@pytest.mark.parametrize("name", [c["name"] for c in AC.CASES if c["op"] in DEVICE_OPS and not c.get("refuse")])
def test_host_arrays_match_fixture(golden, name):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        got = AC.call(lb, AC.BY_NAME[name])
    ok, why = AC.matches(golden, name, got)
    assert ok, why


@pytest.mark.parametrize("name", [c["name"] for c in AC.CASES if c["op"] in DEVICE_OPS and not c.get("refuse")
                                  and c["name"] not in ("dtw/mixed_dtype", "dtw/err_C_and_X", "dtw/err_no_Y")])
def test_device_arrays_match_fixture(golden, name):
    case = AC.BY_NAME[name]
    if name + "/error" in golden:
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            X, Y, Cm, sim = AC.inputs(case)
            got = AC.call(lb, case, *[lb.to_device(np.ascontiguousarray(a)) if a is not None else None
                                      for a in (X, Y, Cm, sim)])
    else:
        got = _device_call(case)
    ok, why = AC.matches(golden, name, got)
    assert ok, why


@pytest.mark.parametrize("name", [c["name"] for c in AC.CASES if c.get("refuse")])
def test_refusals_on_device(name):
    case = AC.BY_NAME[name]
    X, Y, Cm, sim = AC.inputs(case)
    with pytest.raises(lb.UnsupportedOnGPU):
        AC.call(lb, case, *[lb.to_device(np.ascontiguousarray(a)) if a is not None else None
                            for a in (X, Y, Cm, sim)])


def test_mixed_dtype_device_refused():
    X = lb.to_device(np.ones((12, 5), np.float32))
    with pytest.raises(lb.UnsupportedOnGPU, match="share a dtype"):
        lb.sequence.dtw(X, np.ones((12, 6)))


class _Reads:
    def __init__(self, monkeypatch):
        self.calls, self.bytes = 0, 0
        orig = nat.DeviceArray.get
        reads = self

        def get(arr, out=None):
            reads.calls += 1
            reads.bytes += arr.nbytes
            return orig(arr, out)
        monkeypatch.setattr(nat.DeviceArray, "get", get)


def _waves(n, m):
    return -(-n // TILE) + -(-m // TILE) - 1


def test_launch_counts_and_read_backs(monkeypatch):
    ctx = lb.default_context()
    rng = np.random.default_rng(0)
    X = lb.to_device(rng.random((12, 300)).astype(np.float32))
    Y = lb.to_device(rng.random((12, 260)).astype(np.float32))
    Cd = lb.to_device(rng.random((300, 260)))
    sim = lb.to_device((rng.random((300, 260)) > 0.6).astype(np.float32))
    reads = _Reads(monkeypatch)

    def count(fn):
        n0, r0, b0 = ctx.launch_count, reads.calls, reads.bytes
        out = fn()
        return out, ctx.launch_count - n0, reads.calls - r0, reads.bytes - b0

    w = _waves(300, 260)
    _, n, r, b = count(lambda: lb.sequence.dtw(X, Y))                      # cost, waves, walk; the length word
    assert (n, r, b) == (1 + w + 1, 1, 8)
    _, n, r, b = count(lambda: lb.sequence.dtw(X, Y, backtrack=False))     # the verdict word
    assert (n, r, b) == (1 + w, 1, 4)
    _, n, r, b = count(lambda: lb.sequence.dtw(C=Cd, subseq=True))          # NaN flags, waves, walk
    assert (n, r, b) == (1 + w + 1, 1, 8)
    (_, steps), n, r, b = count(lambda: lb.sequence.dtw(C=Cd, backtrack=False, return_steps=True))
    assert (n, r, b) == (1 + w, 1, 4)
    _, n, r, b = count(lambda: lb.sequence.dtw_backtracking(steps))
    assert (n, r, b) == (1, 1, 8)
    _, n, r, b = count(lambda: lb.sequence.rqa(sim))                        # waves, argmax, walk
    assert (n, r, b) == (w + 2, 1, 8)
    _, n, r, b = count(lambda: lb.sequence.rqa(sim, backtrack=False))
    assert (n, r, b) == (w, 0, 0)


def test_zero_step_walk_is_refused():
    """Every cell prefers the custom (0, 0) step (a negative additive weight lowers a cell's own cost): the
    reference's backtracking never ends here, the device walk stops and reports it."""
    Cm = np.zeros((4, 4))
    kw = dict(step_sizes_sigma=np.array([[1, 1], [0, 0]]), weights_add=np.array([0.0, -1.0]))
    D, steps = lb.sequence.dtw(C=Cm, backtrack=False, return_steps=True, **kw)
    assert steps[-1, -1] == 4 and np.isfinite(D[-1, -1])
    with pytest.raises(lb.UnsupportedOnGPU, match=r"\(0, 0\) step"):
        lb.sequence.dtw(C=Cm, **kw)
    with pytest.raises(lb.UnsupportedOnGPU, match=r"\(0, 0\) step"):
        lb.sequence.dtw_backtracking(steps, step_sizes_sigma=kw["step_sizes_sigma"])


def test_rqa_past_2_to_the_31_cells():
    """float32 46 400 x 46 400 (2.15e9 cells, about 19 GB with score and pointers): sim is zero but for a diagonal
    run of RUN ones starting past flat index 2^31, so the score maximum is RUN at the run's end and the path is the
    run."""
    ctx = lb.default_context()
    n, run, c0 = 46400, 50, 100
    free, _ = ctx.mem_info()
    if free < 24 << 30:
        pytest.skip("needs 24 GB of free device memory")
    r0 = (1 << 31) // n + 1
    sim = nat.DeviceArray.empty(ctx, (n, n), np.float32)
    nat.check(nat.lib().b2l_memset(ctx.handle, C.c_void_p(sim.ptr), 0, sim.nbytes))
    one = np.ones(1, np.float32)
    for k in range(run):
        at = (r0 + k) * n + c0 + k
        assert at >= 1 << 31
        nat.check(nat.lib().b2l_h2d(ctx.handle, C.c_void_p(sim.ptr + 4 * at), one.ctypes.data_as(C.c_void_p), 4))
    score, path = lb.sequence.rqa(sim)
    want = np.stack([np.arange(r0, r0 + run), np.arange(c0, c0 + run)], -1).astype(np.uint64)
    assert path.get().tolist() == want.tolist()
    row = np.empty(n, np.float32)
    nat.check(nat.lib().b2l_d2h(ctx.handle, row.ctypes.data_as(C.c_void_p),
                                C.c_void_p(score.ptr + 4 * (r0 + run - 1) * n), 4 * n))
    ctx.synchronize()
    assert row[c0 + run - 1] == run and row.max() == run
    for a in (sim, score, path):
        a.free()
    ctx.empty_cache()
