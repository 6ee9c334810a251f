"""Case table of HMM decoding: tests/golden/sequence_v1.npz holds, for each case, what the unmodified reference's
``sequence.viterbi`` / ``viterbi_discriminative`` / ``viterbi_binary`` returns (``<name>/states``, ``<name>/logp``) or
the exception it raises (``<name>/error``, "Class: message"), the SHA-256 of the log-likelihoods its decoder reads
(``<name>/lp_sha256``, of float64 [problem][state][frame]; the tests rebuild the arrays from the seeded inputs with
tests/sequence_oracle.py and check them against it), and every ``transition_*`` builder output (``builder/<name>``);
written by tools/make_golden.py --sequence.  tests/sequence_oracle.py must reproduce it bit for bit.

Observations are seeded, float32 and float64, with leading shapes (), (3,) and (2, 3); 1 to 2 000 states (every
decoder size class), 1 to 10 000 frames; dense, banded and random sparse transition matrices with
``transition_min_prob`` None, 0 and positive; ties (uniform observations, symmetric matrices), zeros, NaN and +-inf."""
from __future__ import annotations

import numpy as np


def builder(ref, spec):
    kind = spec[0]
    if kind == "uniform":
        return ref.sequence.transition_uniform(spec[1])
    if kind == "loop":
        return ref.sequence.transition_loop(spec[1], spec[2])
    if kind == "cycle":
        return ref.sequence.transition_cycle(spec[1], spec[2])
    if kind == "local":
        _, n, width, window, wrap = spec
        return ref.sequence.transition_local(n, width, window=window, wrap=wrap)
    if kind == "random":
        _, n, seed, keep = spec
        rng = np.random.default_rng(seed)
        t = rng.random((n, n)) ** 4
        if keep < 1:
            t[rng.random((n, n)) > keep] = 0
            t[np.arange(n), np.arange(n)] += 0.5
        return t / t.sum(axis=1, keepdims=True)
    if kind == "binary":
        _, n, seed = spec
        p = np.random.default_rng(seed).uniform(0.05, 0.95, size=(n, 2))
        return np.stack([np.stack([p[:, 0], 1 - p[:, 0]], -1), np.stack([1 - p[:, 1], p[:, 1]], -1)], 1)
    if kind == "binary2":
        return np.array([[0.9, 0.1], [0.2, 0.8]])
    raise ValueError(kind)


def observations(op, spec):
    kind, lead, S, T, dtype, seed = spec
    rng = np.random.default_rng(seed)
    shape = tuple(lead) + (S, T)
    if kind == "uniform":
        x = np.full(shape, 1.0 / S if op == "disc" else 0.5)
    elif kind == "peaky":
        x = rng.random(shape) ** 8
    else:
        x = rng.random(shape)
    if op == "disc":
        x = x / x.sum(axis=-2, keepdims=True)
    x = x.astype(dtype)
    if x.size == 0:
        return x
    flat = x.reshape(-1, S, T)
    if kind == "zeros":
        flat[:, :, T // 2] = 0
        flat[:, S // 2, :] = 0
    elif kind == "nan":
        flat[-1, S // 2, T // 2] = np.nan
    elif kind == "inf":
        flat[-1, S // 2, T // 2] = np.inf
    elif kind == "neginf":
        flat[-1, S // 2, T // 2] = -np.inf
    elif kind == "badsum":
        flat[0, 0, 0] += 0.01
    elif kind == "border":      # a column sum just inside / outside np.allclose's tolerance
        flat[0, :, 0] = 0
        flat[0, 0, 0] = 1 + 0.9e-5
        flat[-1, :, -1] = 0
        flat[-1, 0, -1] = 1 + 1.2e-5
    return x


CASES = []


def _add(name, op, obs, trans, **kw):
    CASES.append(dict(name=f"{op}/{name}", op=op, obs=obs, trans=trans, kw=kw))


for dt in ("float32", "float64"):
    for lead in ((), (3,), (2, 3)):
        ls = "x".join(map(str, lead)) or "1"
        _add(f"rand_{dt}_{ls}_25", "viterbi", ("rand", lead, 25, 431, dt, 1), ("loop", 25, 0.9), return_logp=True)
        _add(f"rand_{dt}_{ls}_25", "disc", ("rand", lead, 25, 431, dt, 2), ("loop", 25, 0.9), return_logp=True)
        _add(f"rand_{dt}_{ls}_8", "binary", ("rand", lead, 8, 300, dt, 3), ("binary", 8, 4), return_logp=True)
    for S in (1, 2, 3, 17, 32, 33, 64, 150, 300, 2000):
        T = 20 if S >= 1000 else 120
        trans = ("uniform", S) if S == 1 else ("random", S, S, 1.0)
        _add(f"size_{dt}_{S}", "viterbi", ("peaky", (2,) if S < 1000 else (), S, T, dt, S), trans, return_logp=True)
        _add(f"size_{dt}_{S}", "disc", ("rand", (), S, T, dt, S + 1), trans, return_logp=True)
        if S > 1:
            _add(f"sparse_{dt}_{S}", "viterbi", ("peaky", (), S, T, dt, S + 2), ("random", S, S + 3, 0.2),
                 transition_min_prob=1e-3, return_logp=True)
    for T in (1, 2, 10000):
        _add(f"steps_{dt}_{T}", "viterbi", ("rand", (), 8, T, dt, T), ("loop", 8, 0.5), return_logp=True)
        _add(f"steps_{dt}_{T}", "disc", ("rand", (3,) if T < 10000 else (), 12, T, dt, T), ("cycle", 12, 0.7), return_logp=True)
        _add(f"steps_{dt}_{T}", "binary", ("rand", (), 4, T, dt, T), ("binary2",), return_logp=True)
    for kind in ("uniform", "zeros", "nan", "inf", "neginf"):
        _add(f"{kind}_{dt}", "viterbi", (kind, (3,), 24, 200, dt, 7), ("loop", 24, 0.8), return_logp=True)
        _add(f"{kind}_{dt}", "disc", (kind, (3,), 24, 200, dt, 8), ("local", 24, 5, "triangle", True),
             return_logp=True)
        _add(f"{kind}_{dt}", "binary", (kind, (3,), 6, 200, dt, 9), ("binary2",), return_logp=True)
    for tmp in (None, 0, 1e-4, 0.05):
        _add(f"local_{dt}_{tmp}", "viterbi", ("peaky", (), 720, 30, dt, 11), ("local", 720, 31, "triangle", False),
             transition_min_prob=tmp, return_logp=True)
        _add(f"local_{dt}_{tmp}", "disc", ("rand", (), 48, 300, dt, 12), ("local", 48, 7, "hann", False),
             transition_min_prob=tmp, return_logp=True)
        _add(f"tmp_{dt}_{tmp}", "binary", ("rand", (2,), 5, 200, dt, 13), ("binary", 5, 14),
             transition_min_prob=tmp, return_logp=True)
    _add(f"border_{dt}", "disc", ("border", (2,), 3, 20, dt, 15), ("uniform", 3))
    _add(f"badsum_{dt}", "disc", ("badsum", (), 5, 20, dt, 16), ("uniform", 5))
# custom p_init / p_state, states-only returns, the docstring examples
_P5 = np.array([0.1, 0.2, 0.3, 0.25, 0.15])
_add("p_init", "viterbi", ("rand", (3,), 5, 100, "float64", 20), ("loop", 5, 0.6), p_init=_P5, return_logp=True)
_add("p_init_2d", "viterbi", ("rand", (), 5, 100, "float64", 20), ("loop", 5, 0.6), p_init=_P5, return_logp=True)
_add("p_state", "disc", ("rand", (3,), 5, 100, "float32", 21), ("loop", 5, 0.6), p_state=_P5, p_init=_P5[::-1].copy(),
     return_logp=True)
_add("p_state_init", "binary", ("rand", (), 5, 100, "float64", 22), ("binary", 5, 23), p_state=_P5, p_init=_P5[::-1].copy(),
     return_logp=True)
_add("scalar_p", "binary", ("rand", (), 1, 50, "float64", 24), ("binary2",), p_state=0.3, p_init=0.6, return_logp=True)
_add("states_only", "viterbi", ("rand", (2,), 6, 50, "float32", 25), ("cycle", 6, 0.5))
_add("states_only", "disc", ("rand", (), 6, 50, "float32", 26), ("cycle", 6, 0.5))
_add("states_only", "binary", ("rand", (), 6, 50, "float32", 27), ("binary2",))
_add("one_d", "binary", ("rand", (), 1, 60, "float64", 28), ("binary2",), one_d=True, return_logp=True)
_add("doc_example", "viterbi", ("doc", (), 3, 6, "float64", 0), ("doc",), p_init=np.array([0.6, 0.2, 0.2]),
     return_logp=True)
# errors
_add("err_shape", "viterbi", ("rand", (), 4, 10, "float64", 30), ("uniform", 5))
_add("err_trans", "disc", ("rand", (), 4, 10, "float64", 31), ("bad", 4))
_add("err_range", "viterbi", ("inf", (), 4, 10, "float64", 32), ("uniform", 4))
_add("err_range_and_p_init", "viterbi", ("neginf", (), 4, 10, "float32", 33), ("uniform", 4),
     p_init=np.array([0.5, 0.5, 0.5, 0.5]))
_add("err_p_init", "viterbi", ("rand", (), 4, 10, "float64", 34), ("uniform", 4), p_init=np.array([0.5, 0.5, 0, 0.1]))
_add("err_p_state_shape", "disc", ("rand", (), 4, 10, "float64", 35), ("uniform", 4), p_state=np.ones(3) / 3)
_add("err_p_state", "disc", ("rand", (), 4, 10, "float64", 36), ("uniform", 4), p_state=np.array([0.5, 0.5, 0.5, 0]))
_add("err_sum_and_p_state", "disc", ("badsum", (), 4, 10, "float64", 37), ("uniform", 4),
     p_state=np.array([0.5, 0.5, 0.5, 0]))
_add("err_tmp", "viterbi", ("rand", (), 4, 10, "float64", 38), ("uniform", 4), transition_min_prob=-1.0)
_add("err_nan_and_tmp", "disc", ("nan", (), 4, 10, "float64", 39), ("uniform", 4), transition_min_prob=-1.0)
_add("err_empty", "viterbi", ("rand", (), 4, 10, "float64", 40), ("cycle", 4, 0.9), transition_min_prob=0.95)
_add("err_empty_binary", "binary", ("rand", (), 3, 10, "float64", 41), ("binary", 3, 42), transition_min_prob=0.97)
_add("err_nan_binary", "binary", ("nan", (), 3, 10, "float64", 43), ("binary2",))
_add("err_nan_binary_and_p_state", "binary", ("nan", (), 3, 10, "float32", 44), ("binary2",),
     p_state=np.array([0.5, 2.0, 0.5]))
_add("err_binary_trans_shape", "binary", ("rand", (), 3, 10, "float64", 45), ("binary", 2, 46))
_add("err_binary_p_init", "binary", ("rand", (), 3, 10, "float64", 47), ("binary2",), p_init=np.array([0.5, 0.5]))
_add("err_zero_lead", "viterbi", ("rand", (0,), 4, 10, "float64", 48), ("uniform", 4))
_add("err_zero_lead", "disc", ("rand", (0, 2), 4, 10, "float64", 49), ("uniform", 4))
_add("err_zero_lead", "binary", ("rand", (0,), 4, 10, "float64", 50), ("binary2",))
_add("err_zero_steps_nd", "viterbi", ("rand", (2,), 4, 0, "float64", 51), ("uniform", 4))
_add("err_zero_steps", "disc", ("rand", (), 4, 0, "float64", 52), ("uniform", 4))
_add("err_zero_steps", "binary", ("rand", (2,), 4, 0, "float64", 53), ("binary2",))
_add("zero_steps", "viterbi", ("rand", (), 4, 0, "float64", 54), ("uniform", 4))

BY_NAME = {c["name"]: c for c in CASES}

BUILDERS = {
    "uniform_1": ("uniform", 1), "uniform_7": ("uniform", 7),
    "loop_2": ("loop", 2, 0.99), "loop_5_vec": ("loop", 5, [0.1, 0.5, 0.9, 0.3, 1.0]), "loop_25": ("loop", 25, 0.9),
    "cycle_3": ("cycle", 3, 0.2), "cycle_6_vec": ("cycle", 6, [0.0, 0.2, 0.4, 0.6, 0.8, 1.0]),
    "local_720_31": ("local", 720, 31, "triangle", False), "local_10_3_wrap": ("local", 10, 3, "triangle", True),
    "local_12_vec": ("local", 12, [1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12], "triangle", False),
    "local_9_hann": ("local", 9, 4, "hann", False), "local_9_boxcar_wrap": ("local", 9, 5, "boxcar", True),
    "local_pyin": ("local", 360, 41, "triangle", False),
}
BUILDER_ERRORS = {
    "uniform_0": ("uniform", 0), "loop_1": ("loop", 1, 0.5), "loop_len": ("loop", 3, [0.5, 0.5]),
    "loop_range": ("loop", 3, 1.5), "cycle_range": ("cycle", 3, -0.1), "local_width": ("local", 5, 0, "triangle", False),
    "local_len": ("local", 5, [1, 2], "triangle", False), "local_1": ("local", 1, 1, "triangle", False),
}

DOC_PROB = np.array([[0.1, 0.3, 0.2, 0.4, 0.0, 0.5], [0.6, 0.2, 0.5, 0.3, 0.7, 0.2], [0.3, 0.5, 0.3, 0.3, 0.3, 0.3]])
DOC_TRANS = np.array([[0.5, 0.4, 0.1], [0.3, 0.6, 0.1], [0.2, 0.3, 0.5]])


def make(case, mod=None):
    """(prob, transition, kwargs) of a case; the named matrices come from ``mod``'s builders (default: the
    project's, which tests/test_sequence_host.py holds bit-identical to the reference's)."""
    obs, trans = case["obs"], case["trans"]
    if obs[0] == "doc":
        prob = DOC_PROB.copy()
    else:
        prob = observations(case["op"], obs)
    if trans[0] == "doc":
        transition = DOC_TRANS
    elif trans[0] == "bad":
        transition = np.full((trans[1], trans[1]), 0.5)
    else:
        if mod is None:
            import librosa_b200 as mod
        transition = builder(mod, trans)
    kw = dict(case["kw"])
    if kw.pop("one_d", False):
        prob = prob[0]
    return prob, transition, kw


def call(mod, case, prob=None):
    """Runs the case through ``mod`` (the reference or librosa_b200): {"states", "logp"} or {"error"}."""
    p, transition, kw = make(case, mod)
    if prob is not None:
        p = prob
    fn = {"viterbi": mod.sequence.viterbi, "disc": mod.sequence.viterbi_discriminative,
          "binary": mod.sequence.viterbi_binary}[case["op"]]
    try:
        out = fn(p, transition, **kw)
    except Exception as exc:  # noqa: BLE001 - the class and message are the result
        return {"error": f"{type(exc).__name__}: {exc}"}
    if kw.get("return_logp"):
        return {"states": out[0], "logp": out[1]}
    return {"states": out}

# Cases whose smallest non-zero decision gap (tests/sequence_oracle.py) is below n_steps * 2 ulp(max |log-likelihood|)
# in the dtype the log is taken in: a 1-ulp difference of a log may change their path.  Exact ties are not fragile.
FRAGILE = [
    "viterbi/rand_float32_1_25",
    "disc/rand_float32_1_25",
    "binary/rand_float32_1_8",
    "viterbi/rand_float32_3_25",
    "disc/rand_float32_3_25",
    "binary/rand_float32_3_8",
    "viterbi/rand_float32_2x3_25",
    "disc/rand_float32_2x3_25",
    "binary/rand_float32_2x3_8",
    "disc/size_float32_3",
    "viterbi/size_float32_17",
    "viterbi/sparse_float32_17",
    "viterbi/size_float32_32",
    "disc/size_float32_32",
    "viterbi/sparse_float32_32",
    "viterbi/size_float32_33",
    "disc/size_float32_33",
    "viterbi/sparse_float32_33",
    "viterbi/size_float32_64",
    "disc/size_float32_64",
    "viterbi/sparse_float32_64",
    "viterbi/size_float32_150",
    "disc/size_float32_150",
    "viterbi/sparse_float32_150",
    "viterbi/size_float32_300",
    "disc/size_float32_300",
    "viterbi/sparse_float32_300",
    "viterbi/size_float32_2000",
    "disc/size_float32_2000",
    "viterbi/sparse_float32_2000",
    "viterbi/steps_float32_10000",
    "disc/steps_float32_10000",
    "binary/steps_float32_10000",
    "viterbi/zeros_float32",
    "binary/zeros_float32",
    "viterbi/nan_float32",
    "viterbi/local_float32_None",
    "disc/local_float32_None",
    "viterbi/local_float32_0",
    "disc/local_float32_0",
    "viterbi/local_float32_0.0001",
    "disc/local_float32_0.0001",
    "viterbi/local_float32_0.05",
    "disc/local_float32_0.05",
    "viterbi/zeros_float64",
]
