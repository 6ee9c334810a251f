"""Case table of onset detection: tests/golden/onset_v1.npz holds, for each case, what the unmodified reference returns
(``util.peak_pick``, ``onset.onset_detect``, ``onset.onset_backtrack``, or the exception it raises), written by
tools/make_golden.py --onset.  tests/onset_oracle.py must reproduce it bit for bit and the GPU must match it.

Envelopes are seeded (tests/rhythm_cases.envelope, plus quantised ones with plateaus, ones holding NaN or +-inf, and
one built so that a float64 mean would pick differently from numba's float32 left-to-right sum), float32 and float64,
with leading shapes (), (3,) and (2, 3) and lengths 0, 1, 2, 3, 431, 5000, 16 385 and 20 000 (rows longer than the
greedy kernel's 8192-frame candidate chunk)."""
from __future__ import annotations

import numpy as np

import rhythm_cases as RC

SR, HOP = RC.SR, RC.HOP
# onset_detect's defaults at 22050 Hz / hop 512, as peak_pick keywords
DEFAULTS = dict(pre_max=1.0, post_max=1.0, pre_avg=4.0, post_avg=5.0, delta=0.07, wait=1.0)
FRAGILE_AT = 32


def _fragile():
    """A float32 row and delta for which frame FRAGILE_AT is a greedy pick under exactly one of numba's float32
    window sum and a float64 sum (window of 20 frames)."""
    for seed in range(1000):
        x = np.random.default_rng(seed).random(64).astype(np.float32)
        x[FRAGILE_AT] = 1.5
        w = x[FRAGILE_AT - 10: FRAGILE_AT + 10]
        s = np.float32(0)
        for v in w:
            s = np.float32(s + v)
        avg32 = np.float64(s) / 20.0
        avg64 = float(np.sum(w.astype(np.float64))) / 20.0
        if avg32 == avg64:
            continue
        delta = 1.5 - 0.5 * (avg32 + avg64)
        if (1.5 >= avg32 + delta) != (1.5 >= avg64 + delta):
            return x, float(delta)
    raise RuntimeError("no fragile row")


FRAGILE_X, FRAGILE_DELTA = _fragile()
FRAGILE_KW = dict(pre_max=10, post_max=10, pre_avg=10, post_avg=10, delta=FRAGILE_DELTA, wait=0)


def envelope(spec):
    kind, shape, n, dtype, seed = spec
    if kind == "fragile":
        return FRAGILE_X.astype(dtype)
    if kind == "quant":
        x = np.round(RC.envelope("random", shape, n, "float64", seed) ** 0.3 * 4) / 4
        return x.astype(dtype)
    if kind in ("nan", "inf", "nan_row"):
        x = RC.envelope("clicks", shape, n, dtype, seed)
        flat = x.reshape(-1, n)
        if kind == "nan":
            flat[:, n // 3] = np.nan
        elif kind == "inf":
            flat[:, n // 4] = np.inf
            flat[:, n // 2] = -np.inf
        else:
            flat[-1, n // 2] = np.nan
        return x
    if kind == "transposed":
        return np.ascontiguousarray(RC.envelope("clicks", shape, n, dtype, seed).T)
    return RC.envelope(kind, shape, n, dtype, seed)


def _pp(name, env, **kw):
    return dict(name="peak/" + name, op="peak_pick", env=env, kw=kw)


def _od(name, env, **kw):
    return dict(name="detect/" + name, op="onset_detect", env=env, kw=kw)


def _bt(name, env, events, **kw):
    return dict(name="backtrack/" + name, op="onset_backtrack", env=env, events=events, kw=kw)


CASES = []
for dt in ("float32", "float64"):
    for method in ("greedy", "dp_count", "dp_value"):
        for n in (1, 2, 3, 431):
            CASES.append(_pp(f"{method}_n{n}_{dt}", ("clicks", (), n, dt, n), method=method, **DEFAULTS))
        CASES.append(_pp(f"{method}_b3_{dt}", ("random", (3,), 431, dt, 1), method=method, sparse=False, **DEFAULTS))
        CASES.append(_pp(f"{method}_b23_{dt}", ("clicks", (2, 3), 5000, dt, 2), method=method, sparse=False,
                         **DEFAULTS))
        CASES.append(_pp(f"{method}_quant_{dt}", ("quant", (3,), 431, dt, 3), method=method, sparse=False,
                         **dict(DEFAULTS, delta=0.0)))
        CASES.append(_pp(f"{method}_quant1d_{dt}", ("quant", (), 431, dt, 4), method=method,
                         **dict(DEFAULTS, pre_max=3, post_max=3)))
        CASES.append(_pp(f"{method}_nan_{dt}", ("nan", (2,), 300, dt, 5), method=method, sparse=False, **DEFAULTS))
        CASES.append(_pp(f"{method}_inf_{dt}", ("inf", (2,), 300, dt, 6), method=method, sparse=False, **DEFAULTS))
        CASES.append(_pp(f"{method}_premax0_{dt}", ("random", (), 431, dt, 7), method=method,
                         **dict(DEFAULTS, pre_max=0)))
        CASES.append(_pp(f"{method}_long_{dt}", ("clicks", (2,), 431, dt, 8), method=method, sparse=False,
                         pre_max=500, post_max=600, pre_avg=700, post_avg=800, delta=0.0, wait=0))
        CASES.append(_pp(f"{method}_wait0_{dt}", ("quant", (), 431, dt, 9), method=method,
                         **dict(DEFAULTS, wait=0, delta=0.0)))
        CASES.append(_pp(f"{method}_waitlong_{dt}", ("clicks", (), 431, dt, 10), method=method,
                         **dict(DEFAULTS, wait=1000)))
        CASES.append(_pp(f"{method}_frac_{dt}", ("random", (3,), 431, dt, 11), method=method, sparse=False,
                         pre_max=1.5, post_max=2.2, pre_avg=3.7, post_avg=4.1, delta=0.01, wait=2.5))
        CASES.append(_pp(f"{method}_axis0_{dt}", ("transposed", (3,), 431, dt, 12), method=method, sparse=False,
                         axis=0, **DEFAULTS))
CASES.append(_pp("greedy_fragile", ("fragile", (), 64, "float32", 0), **FRAGILE_KW))
# rows longer than one candidate chunk of the greedy kernel (8192 frames): the walk carries across chunk ends
for dt in ("float32", "float64"):
    for wait in (0, 1, 37, 9000):
        CASES.append(_pp(f"greedy_n20000_wait{wait}_{dt}", ("random", (), 20000, dt, 20 + wait),
                         **dict(DEFAULTS, wait=wait, delta=0.0)))
        CASES.append(_pp(f"greedy_b2_n20000_wait{wait}_{dt}", ("quant", (2,), 20000, dt, 21 + wait), sparse=False,
                         **dict(DEFAULTS, wait=wait, delta=0.0)))
    CASES.append(_pp(f"greedy_n16385_{dt}", ("clicks", (), 16385, dt, 22), **DEFAULTS))
    CASES.append(_pp(f"dp_value_n20000_{dt}", ("random", (), 20000, dt, 23), method="dp_value", **DEFAULTS))

for dt in ("float32", "float64"):
    for n in (1, 2, 3, 431, 5000, 20000):
        CASES.append(_od(f"n{n}_{dt}", ("clicks", (), n, dt, n)))
    CASES.append(_od(f"b3_{dt}", ("clicks", (3,), 431, dt, 1), sparse=False))
    CASES.append(_od(f"b23_{dt}", ("random", (2, 3), 431, dt, 2), sparse=False))
    CASES.append(_od(f"raw_{dt}", ("clicks", (), 431, dt, 3), normalize=False))
    CASES.append(_od(f"raw_b3_{dt}", ("random", (3,), 431, dt, 4), normalize=False, sparse=False))
    for units in ("samples", "time"):
        CASES.append(_od(f"units_{units}_{dt}", ("clicks", (), 431, dt, 5), units=units))
        CASES.append(_od(f"backtrack_{units}_{dt}", ("clicks", (), 431, dt, 6), backtrack=True, units=units))
    CASES.append(_od(f"backtrack_{dt}", ("random", (), 431, dt, 7), backtrack=True))
    CASES.append(_od(f"backtrack_energy_{dt}", ("random", (), 431, dt, 8), backtrack=True,
                     energy=("quant", (), 431, dt, 9)))
    CASES.append(_od(f"nan_channel_{dt}", ("nan_row", (3,), 300, dt, 10), sparse=False))
    CASES.append(_od(f"nan_1d_{dt}", ("nan", (), 300, dt, 11)))
    CASES.append(_od(f"inf_raw_{dt}", ("inf", (), 300, dt, 12), normalize=False))
    CASES.append(_od(f"zeros_{dt}", ("zeros", (), 300, dt, 0)))
    CASES.append(_od(f"zeros_dense_{dt}", ("zeros", (2,), 300, dt, 0), sparse=False))
    CASES.append(_od(f"zeros_backtrack_dense_{dt}", ("zeros", (2,), 300, dt, 0), backtrack=True, sparse=False))
    CASES.append(_od(f"zeros_bad_param_{dt}", ("zeros", (), 300, dt, 0), pre_max=-1))
    CASES.append(_od(f"zeros_2d_sparse_{dt}", ("zeros", (2,), 300, dt, 0)))
    CASES.append(_od(f"zeros_time_{dt}", ("zeros", (), 300, dt, 0), units="time"))
    for method in ("dp_count", "dp_value"):
        CASES.append(_od(f"{method}_{dt}", ("clicks", (), 431, dt, 13), method=method))
        CASES.append(_od(f"{method}_b3_{dt}", ("random", (3,), 431, dt, 14), method=method, sparse=False))
    CASES.append(_od(f"kw_{dt}", ("random", (), 431, dt, 15), pre_max=3, post_max=3, pre_avg=10, post_avg=10,
                     delta=0.2, wait=5))
# errors (the fixture holds the class and message)
for dt in ("float32",):
    CASES.append(_od("err_bad_units", ("clicks", (), 431, dt, 1), units="bad"))
    CASES.append(_od("err_bad_units_zeros", ("zeros", (), 300, dt, 0), units="bad"))
    CASES.append(_od("err_backtrack_empty", ("clicks", (), 431, dt, 1), backtrack=True, delta=2.0))
    CASES.append(_od("err_backtrack_dense", ("clicks", (2,), 431, dt, 1), backtrack=True, sparse=False))
    CASES.append(_od("err_2d_sparse", ("clicks", (2,), 431, dt, 1)))
    CASES.append(_od("err_bad_param", ("clicks", (), 431, dt, 1), wait=-1))
    CASES.append(_od("err_bad_method", ("clicks", (), 431, dt, 1), method="nope"))
    CASES.append(_od("err_no_input", None))
    CASES.append(_od("err_empty_normalize", ("zeros", (), 0, dt, 0)))
    CASES.append(_od("err_empty_normalize_dense", ("zeros", (2,), 0, dt, 0), sparse=False))
    CASES.append(_od("empty_raw", ("zeros", (), 0, dt, 0), normalize=False))
    for key, val in (("pre_max", -1), ("pre_avg", -1), ("delta", -0.1), ("wait", -1), ("post_max", 0),
                     ("post_avg", 0)):
        CASES.append(_pp(f"err_{key}", ("clicks", (), 100, dt, 1), **dict(DEFAULTS, **{key: val})))
    CASES.append(_pp("err_order", ("clicks", (), 100, dt, 1), **dict(DEFAULTS, post_avg=0, wait=-1)))
    CASES.append(_pp("err_2d_sparse", ("clicks", (2,), 100, dt, 1), **DEFAULTS))
    CASES.append(_pp("err_method", ("clicks", (), 100, dt, 1), method="nope", **DEFAULTS))
    CASES.append(_pp("err_method_after_sparse", ("clicks", (2,), 100, dt, 1), method="nope", **DEFAULTS))
    CASES.append(_bt("err_empty", ("random", (), 100, dt, 1), []))
    CASES.append(_bt("err_negative", ("random", (), 100, dt, 1), [3, -1, 7]))

for dt in ("float32", "float64"):
    for n in (1, 2, 3, 431):
        CASES.append(_bt(f"n{n}_{dt}", ("random", (), n, dt, n), [0, 1, 5, 100, 430, 431, 1000]))
    CASES.append(_bt(f"quant_{dt}", ("quant", (), 431, dt, 2), list(range(0, 431, 7))))
    CASES.append(_bt(f"nan_{dt}", ("nan", (), 300, dt, 3), [10, 99, 100, 101, 150, 299]))
    CASES.append(_bt(f"unsorted_{dt}", ("random", (), 300, dt, 4), [250, 3, 3, 120, 0]))
BY_NAME = {c["name"]: c for c in CASES}
assert len(BY_NAME) == len(CASES)


def kwargs(case):
    kw = dict(case["kw"])
    if isinstance(kw.get("energy"), tuple):
        kw["energy"] = envelope(kw["energy"])
    if case["op"] == "onset_detect":
        kw.setdefault("sr", SR)
        kw.setdefault("hop_length", HOP)
    return kw


def run(lib, case):
    """The case through ``lib`` (the reference, tests/onset_oracle.py or librosa_b200)."""
    kw = kwargs(case)
    if case["op"] == "onset_detect":
        if case["env"] is None:
            return lib.onset.onset_detect(**kw)
        return lib.onset.onset_detect(onset_envelope=envelope(case["env"]), **kw)
    if case["op"] == "peak_pick":
        return lib.util.peak_pick(envelope(case["env"]), **kw)
    return lib.onset.onset_backtrack(np.asarray(case["events"], dtype=np.int64), envelope(case["env"]))


def outcome(lib, case):
    """``{"out": array}`` or ``{"error": "Class: message"}``."""
    try:
        return {"out": np.asarray(run(lib, case))}
    except Exception as e:   # noqa: BLE001 — the class and message are the outcome
        return {"error": f"{type(e).__name__}: {e}"}


def normalized(x):
    """onset_detect's normalisation, as the reference computes it."""
    x = x - np.min(x, keepdims=True, axis=-1)
    x /= np.max(x, keepdims=True, axis=-1) + np.finfo(x.dtype).tiny
    return x


# ---- onset_detect(y=) on click trains at three tempi (the fixture holds the reference's onset frames)
def clicks_audio(bpm, seconds=6.0, sr=SR):
    y = np.zeros(int(seconds * sr), np.float32)
    period = int(round(sr * 60.0 / bpm))
    for s in range(period // 2, y.size - 64, period):
        y[s:s + 64] += np.hanning(64).astype(np.float32)
    return y


Y_CASES = {"detect_y/clicks90": 90.0, "detect_y/clicks120": 120.0, "detect_y/clicks170": 170.0}
