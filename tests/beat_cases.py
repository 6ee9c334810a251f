"""Case table of beat tracking: tests/golden/beat_v1.npz holds, for each case, what the unmodified reference returns
(``bpm`` and ``beats`` of ``beat.beat_track``) and the tracker's intermediates for that bpm (``localscore``,
``cumscore``, ``backlink``, ``tail``), written by tools/make_golden.py --beat.  tests/beat_oracle.py must reproduce
them bit for bit and the GPU must match them.

Envelopes are seeded (tests/rhythm_cases.envelope): click trains at several tempi, random, a single impulse, all
zeros, and a batch with one all-zero clip among non-zero ones, in float32 and float64, with leading shapes (), (3,)
and (2, 3).  They are crossed with bpm (estimated, scalar, per clip, per frame, and values giving 1, 21, 23 and more
frames per beat than the envelope has, float32 bpm), tightness, trim, units, sparse and the tempo prior.  The file
also holds beat_track(y=) on click trains (Y_CASES) and plp's pulse (PLP_CASES)."""
from __future__ import annotations

import numpy as np

import rhythm_cases as RC

SR, HOP = RC.SR, RC.HOP
FRAME_RATE = SR / HOP


def _case(name, env, **kw):
    return dict(name="beat/" + name, env=env, kw=kw)


def bpm_for_fpb(fpb):
    """A tempo whose frames per beat round to ``fpb``."""
    return FRAME_RATE * 60.0 / fpb


BEAT_CASES = []
for dt in ("float32", "float64"):
    for kind, seed in (("clicks", 0), ("clicks", 2), ("random", 1), ("impulse", 3)):
        BEAT_CASES.append(_case(f"{kind}{seed}_{dt}", (kind, (), 431, dt, seed)))
    for tight in (1e2, 1e4, 0.1):
        for trim in (True, False):
            BEAT_CASES.append(_case(f"bpm120_t{tight:g}_trim{int(trim)}_{dt}", ("clicks", (), 431, dt, 2), bpm=120.0,
                                    tightness=tight, trim=trim))
    BEAT_CASES.append(_case(f"batch3_{dt}", ("clicks", (3,), 300, dt, 1), sparse=False))
    BEAT_CASES.append(_case(f"batch23_{dt}", ("random", (2, 3), 260, dt, 4), sparse=False))
    BEAT_CASES.append(_case(f"perclip_{dt}", ("clicks", (3,), 300, dt, 5), bpm=("perclip", (90.0, 120.0, 150.0)),
                            sparse=False))
    BEAT_CASES.append(_case(f"tv_{dt}", ("clicks", (2,), 300, dt, 6), bpm=("ramp", 100.0, 160.0), sparse=False))
    BEAT_CASES.append(_case(f"tv1d_{dt}", ("random", (), 300, dt, 7), bpm=("ramp", 60.0, 200.0)))
    for fpb in (1, 2, 21, 23):
        BEAT_CASES.append(_case(f"fpb{fpb}_{dt}", ("random", (), 200, dt, fpb), bpm=bpm_for_fpb(fpb)))
    BEAT_CASES.append(_case(f"fpb_large_{dt}", ("clicks", (), 200, dt, 8), bpm=1.0))
    BEAT_CASES.append(_case(f"zero_clip_{dt}", ("zero_clip", (3,), 300, dt, 9), bpm=120.0, sparse=False))
    BEAT_CASES.append(_case(f"zeros_{dt}", ("zeros", (), 200, dt, 0)))
    BEAT_CASES.append(_case(f"zeros_dense_{dt}", ("zeros", (2,), 200, dt, 0), sparse=False))
for units in ("samples", "time"):
    BEAT_CASES.append(_case(f"units_{units}", ("clicks", (), 431, "float32", 3), units=units))
    BEAT_CASES.append(_case(f"units_{units}_bpm", ("clicks", (), 431, "float32", 3), units=units, bpm=130.0))
for dt in ("float32", "float64"):   # float32 bpm: numba's float32 DP when the envelope is float32 too
    BEAT_CASES.append(_case(f"bpm_f32_{dt}", ("clicks", (), 431, dt, 2), bpm=("f32", 120.0)))
    BEAT_CASES.append(_case(f"tv_f32_{dt}", ("random", (), 300, dt, 7), bpm=("ramp32", 60.0, 200.0)))
BEAT_CASES.append(_case("prior_lognorm", ("clicks", (), 431, "float32", 4), prior="lognorm"))
BEAT_CASES.append(_case("prior_uniform_dense", ("random", (3,), 300, "float64", 5), prior="uniform", sparse=False))
BY_NAME = {c["name"]: c for c in BEAT_CASES}


def make_input(case):
    kind, shape, n, dtype, seed = case["env"]
    if kind == "zero_clip":
        x = RC.envelope("clicks", shape, n, dtype, seed)
        x[..., 1, :] = 0
        return x
    return RC.envelope(kind, shape, n, dtype, seed)


def bpm_arg(case):
    """The bpm a case passes (None: estimated)."""
    spec = case["kw"].get("bpm")
    if spec is None or isinstance(spec, float):
        return spec
    kind = spec[0]
    x = make_input(case)
    if kind == "f32":
        return np.float32(spec[1])
    if kind == "ramp32":
        return np.linspace(spec[1], spec[2], x.shape[-1]).astype(np.float32)
    if kind == "perclip":
        return np.array(spec[1], dtype=np.float64).reshape(x.shape[:-1])
    if kind == "ramp":
        return np.broadcast_to(np.linspace(spec[1], spec[2], x.shape[-1]), x.shape).copy()
    raise ValueError(kind)


def kwargs(case):
    kw = dict(case["kw"])
    kw["bpm"] = bpm_arg(case)
    if "prior" in kw:
        kw["prior"] = RC.prior(kw["prior"])
    kw.setdefault("sr", SR)
    kw.setdefault("hop_length", HOP)
    return kw


def stage_kwargs(case):
    """tightness and trim of the tracker stages."""
    return dict(tightness=case["kw"].get("tightness", 100), trim=case["kw"].get("trim", True))


def has_stages(case):
    """All-zero envelopes return before the tracker runs."""
    return case["env"][0] != "zeros"


def run(lib, case):
    """``lib.beat.beat_track`` on the case (the reference, the oracle or librosa_b200)."""
    return lib.beat.beat_track(onset_envelope=make_input(case), **kwargs(case))


# ---- beat_track(y=) on the reference's kind of 120 BPM pulse train (the fixture holds the reference's beats and bpm)
def clicks_audio(bpm=120.0, seconds=10.0, sr=SR):
    """Hann-shaped clicks of 64 samples every 60 / bpm seconds."""
    y = np.zeros(int(seconds * sr), np.float32)
    period = int(round(sr * 60.0 / bpm))
    for s in range(period // 2, y.size - 64, period):
        y[s:s + 64] += np.hanning(64).astype(np.float32)
    return y


Y_CASES = {"beat_y/clicks120": 120.0, "beat_y/clicks95": 95.0}


# ---- plp: the pulse of each case (tests/golden/beat_v1.npz "<name>/pulse").  Seeds are chosen so that no frame is
# fragile (beat_oracle.plp_fragile): the peak selection does not hang on the last bits of ftmag.
def _plp(name, env, **kw):
    return dict(name="plp/" + name, env=env, kw=kw)


PLP_CASES = []
for W in (192, 384):
    PLP_CASES.append(_plp(f"win{W}", ("clicks", (), 431, "float32", 3), win_length=W))
for (tmin, tmax), seed in (((None, None), 0), ((60, 200), 1), ((None, 300), 0), ((30, None), 7)):
    PLP_CASES.append(_plp(f"range_{tmin}_{tmax}", ("clicks", (), 431, "float32", seed), tempo_min=tmin,
                          tempo_max=tmax))
PLP_CASES.append(_plp("lognorm", ("clicks", (), 431, "float32", 4), prior="lognorm"))
PLP_CASES.append(_plp("float64", ("clicks", (), 431, "float64", 3)))
PLP_CASES.append(_plp("batch3", ("clicks", (3,), 300, "float32", 3), win_length=192))
PLP_BY_NAME = {c["name"]: c for c in PLP_CASES}


def plp_kwargs(case):
    kw = dict(case["kw"])
    if "prior" in kw:
        kw["prior"] = RC.prior(kw["prior"])
    kw.setdefault("sr", SR)
    kw.setdefault("hop_length", HOP)
    return kw


def run_plp(lib, case):
    return lib.beat.plp(onset_envelope=make_input(case), **plp_kwargs(case))
