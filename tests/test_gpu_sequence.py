"""HMM decoding on the GPU against tests/golden/sequence_v1.npz and tests/sequence_oracle.py:

* the decode kernel, fed the fixture's own log-likelihoods, returns states and logp bit-identical to the reference;
* the log-likelihood kernel is within 1 ulp (in NumPy's dtype) of NumPy — 4 for float32, where NumPy's own log is up
  to 4 ulp from the correctly rounded value the kernel forms — and its verdict flags equal NumPy's checks;
* the public calls, host and DeviceArray: states equal the fixture on every case not listed as fragile; on every
  case the oracle's score of the returned path and the returned logp are within n_steps * 2 ulp(max |lp|) of the
  reference's logp;
* launch counts and read-backs, and one decode launch over more than 65 535 problems."""
import ctypes as C
import os
import warnings

import numpy as np
import pytest

import sequence_cases as SC
import sequence_oracle as SO
import librosa_b200 as lb
from librosa_b200 import _native as nat
from librosa_b200 import sequence as seq

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_vp = C.c_void_p
NUMPY_F32_LOG_ULP = 4
DECODED = [c["name"] for c in SC.CASES if c["obs"][3] > 0 and "err_" not in c["name"]]


@pytest.fixture(scope="module")
def golden():
    with np.load(os.path.join(ROOT, "tests", "golden", "sequence_v1.npz")) as z:
        return {k: z[k] for k in z.files}


def _oracle(name):
    case = SC.BY_NAME[name]
    prob, transition, kw = SC.make(case)
    kw.pop("return_logp", None)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return prob, SO.run(case["op"], prob, transition, **kw)


def _decode_fixture_lp(lp, models, n_models):
    """b2l_seq_decode on the fixture's log-likelihoods with the model tables sequence.py builds."""
    ctx = lb.default_context()
    tabs = [seq._predecessors(lt, thr) for lt, _, thr in models]
    S, deg = lp.shape[1], max(t[0] for t in tabs)
    dense = all(t[1] for t in tabs)
    lt = np.full((n_models, deg, S), -np.inf)
    idx = np.zeros((n_models, deg, S), np.uint16)
    for m, (d, is_dense, lt_m, idx_m) in enumerate(tabs):
        lt[m, :d] = lt_m
        idx[m, :d] = np.arange(S)[:, None] if is_dense else idx_m
    keep = [ctx.to_device(np.ascontiguousarray(a)) for a in
            (lp, lt, idx, np.stack([np.asarray(pi, np.float64) for _, pi, _ in models]))]
    model = nat.SeqModel(n_states=S, n_models=n_models, deg=deg, dense=int(dense), d_lt=keep[1].ptr,
                         d_idx=None if dense else keep[2].ptr, d_log_p_init=keep[3].ptr)
    P, T = lp.shape[0], lp.shape[2]
    st = nat.DeviceArray.empty(ctx, (P, T), np.uint16)
    lg = nat.DeviceArray.empty(ctx, (P,), np.float64)
    nat.check(nat.lib().b2l_seq_decode(ctx.handle, C.byref(model), _vp(keep[0].ptr), P, T, _vp(st.ptr), _vp(lg.ptr)))
    return st.get(), lg.get()


@pytest.mark.parametrize("name", DECODED)
def test_decode_kernel_bit_exact(golden, name):
    if name + "/lp_sha256" not in golden:
        pytest.skip("an error case of the reference")
    _, r = _oracle(name)
    assert SO.digest(r["lp"]) == str(golden[name + "/lp_sha256"]), name   # the fixture's own log-likelihoods
    states, logp = _decode_fixture_lp(r["lp"], r["models"], r["n_models"])
    want_s = golden[name + "/states"].reshape(states.shape)
    assert states.tobytes() == want_s.tobytes(), name
    if name + "/logp" in golden:
        want = golden[name + "/logp"].reshape(-1)
        assert logp.view(np.int64).tolist() == want.view(np.int64).tolist() or \
            np.array_equal(logp, want, equal_nan=True), name


def _logobs(prob, mode, log_marginal, eps, n_flags):
    ctx = lb.default_context()
    d = ctx.to_device(np.ascontiguousarray(prob))
    S, T = prob.shape[-2:]
    n_clips = int(np.prod(prob.shape[:-2], dtype=np.int64))
    lm = ctx.to_device(np.ascontiguousarray(log_marginal, np.float64)) if log_marginal is not None else None
    rows = 2 * S if mode == nat.SEQ_BINARY else S
    out = nat.DeviceArray.empty(ctx, (n_clips, rows, T), np.float64)
    flags = nat.DeviceArray.empty(ctx, (n_flags,), np.int32)
    nat.check(nat.lib().b2l_memset(ctx.handle, _vp(flags.ptr), 0, flags.nbytes))
    desc = nat.SeqLogObsDesc(mode=mode, f64=int(prob.dtype == np.float64), n_clips=n_clips, n_states=S, n_steps=T,
                             eps=float(eps), d_log_marginal=lm.ptr if lm is not None else None)
    nat.check(nat.lib().b2l_seq_logobs(ctx.handle, C.byref(desc), _vp(d.ptr), _vp(out.ptr), _vp(flags.ptr)))
    return out.get(), flags.get()


@pytest.mark.parametrize("name", [c["name"] for c in SC.CASES if c["obs"][3] > 0 and c["obs"][0] != "doc"
                                  and "_lead" not in c["name"] and c["name"] not in
                                  ("viterbi/err_shape", "disc/err_trans", "binary/err_binary_trans_shape")])
def test_logobs_within_one_ulp_and_verdict(golden, name):
    case = SC.BY_NAME[name]
    prob, transition, kw = SC.make(case)
    op = case["op"]
    if op == "binary":
        prob = np.atleast_2d(prob)
    S, T = prob.shape[-2:]
    if op == "binary":
        p_state = np.atleast_1d(kw.get("p_state", np.full(S, 0.5)))
        lm = np.log(np.stack([1 - p_state, p_state], -1) + np.finfo(np.float64).tiny)
        got, flags = _logobs(prob, nat.SEQ_BINARY, lm, np.finfo(np.float64).tiny, 1 + S)
        q = (1 - prob).astype(np.float64) + prob.astype(np.float64)
        want_flags = [int(np.any(prob < 0) or np.any(prob > 1))] + \
            [int(not np.allclose(q[..., s, :], 1)) for s in range(S)]
        dt = np.float64
        lm_rows = lm.reshape(-1)[None, :, None]
    else:
        eps = np.finfo(prob.dtype).tiny
        p_state = kw.get("p_state")
        lm = np.log((p_state if p_state is not None else np.full(S, 1.0 / S)) + eps) if op == "disc" else None
        got, flags = _logobs(prob, nat.SEQ_DISC if op == "disc" else nat.SEQ_PLAIN, lm, eps, 1)
        if op == "disc":
            want_flags = [int(bool(np.any(prob < 0) or not np.allclose(prob.sum(axis=-2), 1)))]
        else:
            want_flags = [int(bool(np.any(prob < 0) or np.any(prob > 1)))]
        dt = prob.dtype
        lm_rows = 0.0 if lm is None else lm[None, :, None]
    assert flags.tolist() == want_flags, (name, flags, want_flags)
    if name + "/lp_sha256" not in golden:
        return
    _, r = _oracle(name)
    assert SO.digest(r["lp"]) == str(golden[name + "/lp_sha256"]), name
    want = r["lp"].reshape(got.shape)
    lm_rows = np.broadcast_to(lm_rows, got.shape)
    both = np.isfinite(want)
    assert np.array_equal(np.isnan(got), np.isnan(want)) and np.array_equal(got[~both & ~np.isnan(want)],
                                                                             want[~both & ~np.isnan(want)]), name
    # 1 ulp of the log term in the dtype NumPy takes it in (of the larger of the two, so that a pair straddling a
    # power of two counts as 1 ulp), plus the rounding of the float64 marginal subtraction.  The kernel's float32 log
    # is the correctly rounded one; NumPy's own float32 log (its SIMD loop) is up to 4 ulp away from that on 10^6
    # uniform samples, so float32 allows NUMPY_F32_LOG_ULP.
    g, w, m = got[both], want[both], lm_rows[both]
    term = np.maximum(np.abs(g + m), np.abs(w + m)).astype(dt)
    ulps = NUMPY_F32_LOG_ULP if dt == np.float32 else 1
    tol = ulps * np.spacing(term).astype(np.float64) + np.spacing(np.maximum(np.abs(g), np.abs(w)))
    assert np.all(np.abs(g - w) <= tol), (name, np.max(np.abs(g - w) / tol))


def _public(name, device):
    case = SC.BY_NAME[name]
    prob, transition, kw = SC.make(case)
    x = lb.to_device(np.ascontiguousarray(prob)) if device else prob
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        got = SC.call(lb, case, prob=x)
    if device and "states" in got:
        got = {k: v.get() if isinstance(v, lb.DeviceArray) else v for k, v in got.items()}
    return got


@pytest.mark.parametrize("device", [False, True])
@pytest.mark.parametrize("name", [c["name"] for c in SC.CASES])
def test_public_vs_golden(golden, name, device):
    got = _public(name, device)
    if name + "/error" in golden:
        assert got.get("error") == str(golden[name + "/error"]), got
        return
    assert "states" in got, got
    want = golden[name + "/states"]
    assert got["states"].dtype == want.dtype and got["states"].shape == want.shape, name
    if name not in SC.FRAGILE:
        assert got["states"].tobytes() == want.tobytes(), name
    if name + "/logp" not in golden or want.shape[-1] == 0:
        return
    wl = golden[name + "/logp"]
    assert got["logp"].shape == wl.shape and got["logp"].dtype == wl.dtype, name
    prob, r = _oracle(name)
    bound = SO.fragile_bound(prob.shape[-1], r["max_abs_lp"], prob.dtype)
    st = got["states"].reshape(-1, want.shape[-1])
    for p in range(st.shape[0]):
        lt, lpi, _ = r["models"][p % r["n_models"]]
        sc = SO.score(r["lp"][p], lt, lpi, st[p])
        ref = wl.reshape(-1)[p]
        if np.isfinite(ref):
            assert abs(sc - ref) <= bound and abs(got["logp"].reshape(-1)[p] - ref) <= bound, (name, p, sc, ref)
        else:
            assert got["logp"].reshape(-1)[p] == ref or (np.isnan(ref) and np.isnan(got["logp"].reshape(-1)[p]))


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


def test_launch_counts_and_read_backs(monkeypatch):
    ctx = lb.default_context()
    rng = np.random.default_rng(0)
    p = rng.random((3, 25, 431)).astype(np.float32)
    pd = p / p.sum(axis=-2, keepdims=True)
    x, xd = lb.to_device(p), lb.to_device(pd)
    T = lb.sequence.transition_loop(25, 0.9)
    reads = _Reads(monkeypatch)

    def count(fn):
        n0, r0, b0 = ctx.launch_count, reads.calls, reads.bytes
        out = fn()
        return out, ctx.launch_count - n0, reads.calls - r0, reads.bytes - b0

    out, n, r, b = count(lambda: lb.sequence.viterbi(x, T, return_logp=True))
    assert (n, r, b) == (2, 1, 4) and isinstance(out[0], lb.DeviceArray) and out[1].shape == (3,)
    out, n, r, b = count(lambda: lb.sequence.viterbi_discriminative(xd, T, return_logp=True))
    assert (n, r, b) == (2, 1, 4)
    out, n, r, b = count(lambda: lb.sequence.viterbi_binary(x, np.array([[0.9, 0.1], [0.2, 0.8]])))
    assert (n, r, b) == (2, 1, 4 * 26)
    _, n, _, _ = count(lambda: lb.sequence.viterbi(p, T))
    assert n == 2
    # a data error with a later host error: one flags-only launch and its read-back decide which is raised
    bad = lb.to_device(np.where(p > 0.999, np.float32(2), p))
    with pytest.raises(lb.ParameterError, match="between 0 and 1"):
        count(lambda: lb.sequence.viterbi(bad, T, p_init=np.full(25, 0.5)))
    with pytest.raises(lb.ParameterError, match="between 0 and 1"):
        lb.sequence.viterbi(bad, T)


def test_many_problems_one_launch():
    """70 000 clips x 2 labels x 16 frames: one log-likelihood and one decode launch, every path as the oracle."""
    rng = np.random.default_rng(5)
    x = rng.random((70000, 2, 16))
    trans = np.array([[0.7, 0.3], [0.4, 0.6]])
    ctx = lb.default_context()
    n0 = ctx.launch_count
    got = lb.sequence.viterbi_binary(x, trans)
    assert ctx.launch_count - n0 == 2
    r = SO.run("binary", x[:300], trans)
    assert got[:300].tobytes() == r["states"].tobytes()
    r = SO.run("binary", x[-300:], trans)
    assert got[-300:].tobytes() == r["states"].tobytes()


def test_size_classes():
    ctx = lb.default_context()
    out = (C.c_int32 * 2)()
    for S, deg, cls in ((2, 2, nat.SEQ_SMALL), (25, 25, nat.SEQ_SMALL), (32, 32, nat.SEQ_SMALL),
                        (33, 33, nat.SEQ_MEDIUM), (160, 160, nat.SEQ_MEDIUM), (200, 200, nat.SEQ_LARGE),
                        (1024, 1024, nat.SEQ_LARGE), (720, 20, nat.SEQ_MEDIUM), (720, 31, nat.SEQ_LARGE),
                        (14464, 14464, nat.SEQ_LARGE)):
        dense = int(deg == S)
        m = nat.SeqModel(n_states=S, n_models=1, deg=deg, dense=dense)
        nat.check(nat.lib().b2l_seq_route(ctx.handle, C.byref(m), 1, out))
        assert out[0] == cls, (S, dense, out[0])
    m = nat.SeqModel(n_states=14465, n_models=1, deg=14465, dense=1)
    with pytest.raises(lb.UnsupportedOnGPU, match="14465 states"):
        nat.check(nat.lib().b2l_seq_route(ctx.handle, C.byref(m), 1, out))
