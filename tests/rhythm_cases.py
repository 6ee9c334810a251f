"""Case table of the rhythm features (tempogram, fourier_tempogram, tempo): tests/golden/rhythm_v1.npz holds what the
unmodified reference returns for each case (tools/make_golden.py --rhythm); tests/rhythm_oracle.py must reproduce
it bit for bit and the GPU must match the oracle.

Envelopes are seeded: click trains at several tempi, random non-negative, all zeros, a single impulse and strictly
positive noise, in float32 and float64, with leading shapes (), (3,) and (2, 3).  Arrays above GOLDEN_FULL_BYTES
are stored as SHA-256 digests (enough for the bit-exact oracle check; the GPU is checked against the oracle)."""
from __future__ import annotations

import hashlib

import numpy as np
import scipy.signal
import scipy.stats

SR, HOP = 22050, 512
GOLDEN_FULL_BYTES = 64 * 1024


def envelope(kind, shape=(), n=200, dtype="float32", seed=0):
    """One seeded onset envelope batch of shape ``shape + (n,)``."""
    rng = np.random.default_rng(seed)
    rows = int(np.prod(shape)) if shape else 1
    out = np.zeros((rows, n))
    for r in range(rows):
        if kind == "clicks":               # click trains, a different tempo per row
            bpm = (60, 90, 120, 150, 200, 240)[(r + seed) % 6]
            out[r, :: max(1, int(SR * 60.0 // (HOP * bpm)))] = 1.0
            out[r] += 0.05 * rng.random(n)
        elif kind == "random":
            out[r] = rng.random(n) ** 3
        elif kind == "impulse":
            out[r, rng.integers(n)] = 1.0 + r
        elif kind == "positive":
            out[r] = 0.5 + rng.random(n)
        elif kind != "zeros":
            raise ValueError(kind)
    return out.reshape(tuple(shape) + (n,)).astype(dtype)


def window(spec):
    """Window specs that cannot live in a literal: an ndarray and the np.ones callable."""
    if spec == "ones":
        return np.ones
    if isinstance(spec, tuple) and spec[0] == "array":
        return scipy.signal.get_window("hamming", spec[1], fftbins=True) + 0.25
    return spec


def prior(spec):
    if spec is None:
        return None
    if spec == "uniform":
        return scipy.stats.uniform(60, 240)
    if spec == "lognorm":
        return scipy.stats.lognorm(loc=np.log(120), scale=120, s=1)
    raise ValueError(spec)


WINS = (1, 2, 3, 63, 64, 192, 343, 344, 384, 1000, 4096)
NORMS = {"inf": np.inf, "minf": -np.inf, "0": 0, "1": 1, "2": 2, "0.5": 0.5, "none": None}


def _tg(name, env, **kw):
    return dict(name="tempogram/" + name, op="tempogram", env=env, kw=kw)


_tempogram = []
for W in WINS:
    for center in (True, False):
        n = max(200, W + 40) if not center else (200 if W < 1000 else 300)
        _tempogram.append(_tg(f"win{W}_c{int(center)}", ("clicks", (), n, "float32", W), win_length=W, center=center))
for wname, wspec in (("hann", "hann"), ("ones", "ones"), ("array", ("array", 384)), ("kaiser", ("kaiser", 4.0))):
    for dt in ("float32", "float64"):
        _tempogram.append(_tg(f"window_{wname}_{dt}", ("random", (), 240, dt, 3), window=wspec))
for nname, norm in NORMS.items():
    _tempogram.append(_tg(f"norm_{nname}", ("random", (), 220, "float64", 5), win_length=192, norm=norm))
    _tempogram.append(_tg(f"norm_{nname}_positive_ones", ("positive", (), 300, "float32", 6), win_length=192,
                          norm=norm, window="ones", center=False))
for kind in ("zeros", "impulse", "positive", "random"):
    for dt in ("float32", "float64"):
        _tempogram.append(_tg(f"{kind}_{dt}", (kind, (), 260, dt, 7), win_length=192))
for shape in ((3,), (2, 3)):
    for dt in ("float32", "float64"):
        _tempogram.append(_tg(f"batch{len(shape)}_{dt}", ("clicks", shape, 180, dt, 1), win_length=64))
        _tempogram.append(_tg(f"batch{len(shape)}_{dt}_nc", ("random", shape, 180, dt, 2), win_length=63,
                              center=False, norm=2))


def _tempo(name, env, **kw):
    return dict(name="tempo/" + name, op="tempo", env=env, kw=kw)


_tempo_cases = []
for bpm_seed in range(3):
    for agg in ("mean", None):
        for pname in (None, "uniform", "lognorm"):
            _tempo_cases.append(_tempo(f"clicks{bpm_seed}_{agg}_{pname}", ("clicks", (3,), 431, "float32", bpm_seed),
                                       aggregate=agg, prior=pname))
for mt in (None, 200.0):
    for agg in ("mean", None):
        _tempo_cases.append(_tempo(f"max_tempo{mt}_{agg}", ("clicks", (2,), 431, "float64", 4), max_tempo=mt,
                                   aggregate=agg))
for sb, sd, ac in ((60, 1.0, 8.0), (200, 0.5, 8.0), (120, 2.0, 4.0), (90, 1.0, 5.0)):
    _tempo_cases.append(_tempo(f"start{sb}_std{sd}_ac{ac}", ("random", (2, 3), 300, "float32", sb), start_bpm=sb,
                               std_bpm=sd, ac_size=ac))
    _tempo_cases.append(_tempo(f"start{sb}_std{sd}_ac{ac}_frames", ("random", (), 300, "float64", sb), start_bpm=sb,
                               std_bpm=sd, ac_size=ac, aggregate=None))
for kind in ("zeros", "impulse"):
    _tempo_cases.append(_tempo(f"{kind}_mean", (kind, (), 300, "float32", 9)))
for agg in ("mean", None):
    for dt in ("float64", "float32"):
        _tempo_cases.append(dict(name=f"tempo/tg_{dt}_{agg}", op="tempo_tg", env=("clicks", (2,), 300, "float64", 2),
                                 tg_dtype=dt, kw=dict(aggregate=agg)))

_fourier = [dict(name=f"fourier/win{W}", op="fourier_tempogram", env=("clicks", (), 40, "float32", W),
                 kw=dict(win_length=W)) for W in (256, 343, 384, 512)]

RHYTHM_CASES = _tempogram + _tempo_cases + _fourier
BY_NAME = {c["name"]: c for c in RHYTHM_CASES}


def make_input(case):
    kind, shape, n, dtype, seed = case["env"]
    return envelope(kind, shape, n, dtype, seed)


def kwargs(case):
    """Keyword arguments of the public call, with the window / prior specs made into objects."""
    kw = dict(case["kw"])
    if "window" in kw:
        kw["window"] = window(kw["window"])
    if "prior" in kw:
        kw["prior"] = prior(kw["prior"])
    if case["op"].startswith("tempo_") or case["op"] == "tempo":
        if kw.get("aggregate", "mean") == "mean":
            kw["aggregate"] = np.mean
    kw.setdefault("sr", SR)
    kw.setdefault("hop_length", HOP)
    return kw


def tg_input(lib, case):
    """The tempogram a ``tempo_tg`` case hands in: ``lib``'s own default tempogram of its envelope at ac_size 8."""
    x = make_input(case)
    return lib_feature(lib).tempogram(onset_envelope=x, sr=SR, hop_length=HOP, win_length=344).astype(case["tg_dtype"])


def lib_feature(lib):
    return getattr(lib, "feature", lib)


def run(lib, case):
    """Run one case through ``lib`` (the reference, the oracle or librosa_b200)."""
    f = lib_feature(lib)
    kw = kwargs(case)
    if case["op"] == "tempogram":
        return f.tempogram(onset_envelope=make_input(case), **kw)
    if case["op"] == "fourier_tempogram":
        return f.fourier_tempogram(onset_envelope=make_input(case), **kw)
    if case["op"] == "tempo":
        return f.tempo(onset_envelope=make_input(case), **kw)
    if case["op"] == "tempo_tg":
        return f.tempo(tg=tg_input(lib, case), **kw)
    raise ValueError(case["op"])


def sha256(arr) -> np.ndarray:
    a = np.ascontiguousarray(arr)
    h = hashlib.sha256(str((a.dtype.str, a.shape)).encode() + a.tobytes()).digest()
    return np.frombuffer(h, dtype=np.uint8).copy()


def outputs(case, out):
    """Fixture keys and arrays of one case's result: the array itself when small or when the GPU is compared with
    the fixture (fourier_tempogram), else its SHA-256 digest (with its dtype and shape folded in) under
    key + "/sha256"."""
    out = np.asarray(out)
    if out.nbytes <= GOLDEN_FULL_BYTES or case["op"] == "fourier_tempogram":
        return {case["name"]: out}
    return {case["name"] + "/sha256": sha256(out)}
