"""Case table of the pitch trackers (yin / pyin): tests/golden/pitch_v1.npz holds what the unmodified reference
returns for each case (tools/make_golden.py --pitch); tests/pitch_oracle.py must reproduce it bit for bit and
the GPU must match the oracle.

Every input is float32: the reference then runs the FFT of its autocorrelation in float32, like the GPU does.
"tonal" cases are checked end to end frame by frame on the GPU; the noise mixes A / B / C only through the CMND
and the decision kernels (noise has near-ties everywhere)."""
from __future__ import annotations

import numpy as np
import scipy.signal

import signals

C2, C7 = 65.40639132514966, 2093.004522404789   # note_to_hz("C2"), note_to_hz("C7")


def tone(freq, sr=22050, duration=1.0):
    """librosa.tone (core/audio.py:1859-1937), float32."""
    n = int(duration * sr)
    return np.cos(2 * np.pi * freq * np.arange(n) / sr - np.pi * 0.5).astype(np.float32)


def chirp(fmin, fmax, sr=22050, duration=1.0, linear=False):
    """librosa.chirp (core/audio.py:1940-2052), float32."""
    return scipy.signal.chirp(np.arange(int(duration * sr)) / sr, fmin, duration, fmax,
                              method="linear" if linear else "logarithmic", phi=-90.0).astype(np.float32)


def taper(y):
    """The triangle taper of the reference's pyin_multi tests."""
    return (y * scipy.signal.get_window("triangle", y.shape[-1])[np.newaxis, :]).astype(np.float32)


def make_input(case):
    sig = case["sig"]
    kind = sig[0]
    if kind == "mix":
        _, mix, shape = sig
        return signals.make(mix, shape, seed=len(case["name"]))
    if kind == "tone":
        return tone(sig[1])
    if kind == "chirp":
        y = chirp(220, 640, linear=sig[1] == "linear")
        return np.pad(y, (sig[2],)) if len(sig) > 2 else y
    if kind == "multi":
        return taper(np.stack([tone(440), tone(560)]))
    raise ValueError(kind)


_yin = [
    dict(name="yin/mixT", sig=("mix", "T", (22050,)), kw=dict(fmin=C2, fmax=C7), tonal=True),
    *[dict(name=f"yin/tone{f}", sig=("tone", f), kw=dict(fmin=110, fmax=880, center=False), tonal=True)
      for f in (110, 220, 440, 880)],
    dict(name="yin/chirp", sig=("chirp", "log"),
         kw=dict(fmin=110, fmax=880, center=False, frame_length=1024, hop_length=512), tonal=True),
    dict(name="yin/chirp_instant", sig=("chirp", "log"),
         kw=dict(fmin=110, fmax=880, frame_length=2048, hop_length=512, center=False), tonal=True),
    dict(name="yin/stereo", sig=("mix", "T", (2, 11025)), kw=dict(fmin=C2, fmax=C7), tonal=True),
    dict(name="yin/3d", sig=("mix", "T", (2, 2, 6000)), kw=dict(fmin=110, fmax=1000, frame_length=1024),
         tonal=True),
    dict(name="yin/reflect", sig=("mix", "T", (8000,)), kw=dict(fmin=110, fmax=1000, pad_mode="reflect"),
         tonal=True),
    dict(name="yin/edge", sig=("mix", "T", (8000,)), kw=dict(fmin=110, fmax=1000, pad_mode="edge"), tonal=True),
    dict(name="yin/odd", sig=("mix", "T", (9000,)), kw=dict(fmin=100, fmax=1000, frame_length=1501,
                                                            hop_length=333, trough_threshold=0.2), tonal=True),
    *[dict(name=f"yin/mix{m}", sig=("mix", m, (11025,)), kw=dict(fmin=C2, fmax=C7), tonal=False)
      for m in "ABC"],
]

_pyin = [
    dict(name="pyin/mixT", sig=("mix", "T", (22050,)), kw=dict(fmin=C2, fmax=C7), tonal=True),
    *[dict(name=f"pyin/tone{f}", sig=("tone", f), kw=dict(fmin=110, fmax=1000, center=False), tonal=True)
      for f in (110, 220, 440, 880)],
    dict(name="pyin/chirp", sig=("chirp", "log", 22050),
         kw=dict(fmin=60, fmax=900, center=False, frame_length=1024, hop_length=512, resolution=0.2), tonal=True),
    dict(name="pyin/chirp_instant", sig=("chirp", "log", 22050),
         kw=dict(fmin=110, fmax=880, frame_length=2048, hop_length=512, center=False), tonal=True),
    dict(name="pyin/multi", sig=("multi",), kw=dict(fmin=100, fmax=1000, center=False, fill_na=-1), tonal=True),
    dict(name="pyin/multi_center", sig=("multi",), kw=dict(fmin=100, fmax=1000, center=True), tonal=True),
    dict(name="pyin/3d", sig=("mix", "T", (2, 2, 6000)), kw=dict(fmin=110, fmax=1000, frame_length=1024),
         tonal=True),
    dict(name="pyin/reflect", sig=("mix", "T", (8000,)), kw=dict(fmin=110, fmax=1000, pad_mode="reflect"),
         tonal=True),
    dict(name="pyin/edge", sig=("mix", "T", (8000,)), kw=dict(fmin=110, fmax=1000, pad_mode="edge"), tonal=True),
    dict(name="pyin/odd", sig=("mix", "T", (9000,)), kw=dict(fmin=100, fmax=1000, frame_length=1501,
                                                             hop_length=333), tonal=True),
    dict(name="pyin/fill_none", sig=("mix", "T", (8000,)), kw=dict(fmin=110, fmax=1000, fill_na=None),
         tonal=True),
    dict(name="pyin/full_search", sig=("mix", "T", (6000,)), kw=dict(fmin=110, fmax=1000, transition_min_prob=None),
         tonal=True),
    dict(name="pyin/res02", sig=("mix", "T", (8000,)), kw=dict(fmin=C2, fmax=C7, resolution=0.2), tonal=True),
    *[dict(name=f"pyin/mix{m}", sig=("mix", m, (11025,)), kw=dict(fmin=C2, fmax=C7), tonal=False)
      for m in "ABC"],
]

PITCH_CASES = _yin + _pyin
BY_NAME = {c["name"]: c for c in PITCH_CASES}


def op(case):
    return case["name"].split("/")[0]


def outputs(case, out):
    """Fixture keys and arrays of one case's result."""
    if op(case) == "yin":
        return {case["name"] + "/f0": out}
    f0, vf, vp = out
    return {case["name"] + "/f0": f0, case["name"] + "/voiced_flag": vf, case["name"] + "/voiced_prob": vp}


def run(lib, case):
    """Run one case through ``lib`` (the reference, the oracle or librosa_b200)."""
    y = make_input(case)
    fn = lib.yin if op(case) == "yin" else lib.pyin
    kw = dict(case["kw"])
    kw.setdefault("sr", 22050)
    return fn(y, **kw)
