"""Case table of the semitone filter-bank spectrogram: tests/golden/iirt_v1.npz holds, for each case, what the
unmodified reference's ``iirt`` returns (``<name>/S``) or the exception it raises (``<name>/error``, "Class:
message"), and for the cases in ``WITH_STEPS`` the signal it filtered at every rate other than ``sr``
(``<name>/y<rate>``) and the ``sosfiltfilt`` output of one band (``<name>/band<i>``).  Written by
tools/make_golden.py --iirt; tests/iirt_oracle.py must reproduce every entry bit for bit.

``refuse`` names the cases the GPU declines with UnsupportedOnGPU although the reference runs them (or would,
with its optional resamplers installed); the fixture stores nothing for them, since only the refusal is checked.

The fixture is kept under 1 MB: the stored steps are of 0.5-1 s signals at rates below 22 050 Hz or at sr."""
from __future__ import annotations

import numpy as np

from cqt_cases import signal

P = {"res_type": "polyphase"}


def _c(name, kw, sig=((), 22050, 22050, np.float32), refuse=False, special=None):
    lead, n, sr, dtype = sig
    kw = dict(kw)
    kw.setdefault("sr", sr)
    spec = (lead, n, sr, dtype, len(name) + 11 * n) + ((special,) if special else ())
    return {"name": name, "kw": kw, "sig": spec, "refuse": refuse}


def _midi_to_hz(notes):
    return 440.0 * (2.0 ** ((np.asanyarray(notes) - 69.0) / 12.0))


CASES = [
    _c("defaults", P),
    _c("hop256", dict(P, hop_length=256)),
    _c("center_false", dict(P, center=False)),
    _c("pad_reflect", dict(P, pad_mode="reflect")),
    _c("pad_edge", dict(P, pad_mode="edge")),
    _c("tuning_03", dict(P, tuning=0.3)),
    _c("sr44100", P, ((), 44100, 44100, np.float32)),
    _c("sr16000", P, ((), 32000, 16000, np.float32)),
    _c("custom_bank", dict(P, center_freqs=_midi_to_hz(np.arange(60, 72)), sample_rates=np.repeat(4410.0, 12))),
    _c("custom_bank_sr", dict(P, center_freqs=_midi_to_hz(np.array([40.0, 64.0, 90.0])),
                              sample_rates=np.array([882.0, 22050.0, 22050.0]), win_length=1024)),
    _c("butter", dict(P, ftype="butter")),
    _c("cheby1", dict(P, ftype="cheby1")),
    _c("cheby2", dict(P, ftype="cheby2")),
    _c("q15", dict(P, Q=15)),
    _c("multichannel", P, ((2, 3), 11025, 22050, np.float32)),
    _c("float64", P, ((), 22050, 22050, np.float64)),
    _c("fix_length", dict(P, center=False), ((), 7168, 22050, np.float32)),
    _c("zero_frames", dict(P, center=False), ((), 2000, 22050, np.float32)),
    _c("win1000_hop300", dict(P, win_length=1000, hop_length=300), ((), 33075, 22050, np.float32)),
    _c("sr_only_no_resample", dict(center_freqs=_midi_to_hz(np.arange(70, 76)), sample_rates=np.repeat(22050.0, 6))),
    # refusals: the GPU declines what the reference runs
    _c("refuse_default_res_type", {}, refuse=True),
    _c("refuse_ba", dict(P, flayout="ba"), refuse=True),
    _c("refuse_callable_pad", dict(P, pad_mode=lambda v, w, a, k: None), refuse=True),
    _c("refuse_pad_wrap", dict(P, pad_mode="wrap"), refuse=True),
    # errors the reference raises
    _c("bad_flayout", dict(P, flayout="zpk")),
    _c("negative_frames", dict(P, center=False), ((), 1000, 22050, np.float32)),
    _c("short_at_882", dict(P, center=False, win_length=256), ((), 600, 22050, np.float32)),
    _c("not_finite", P, special="nan"),
    _c("not_finite_and_short", dict(P, center=False, win_length=256), ((), 600, 22050, np.float32), special="nan"),
    _c("non_integer_rate", dict(P, sr=22050.5)),
    _c("bad_pad_mode", dict(P, pad_mode="nope")),
    _c("centre_freqs_without_rates", dict(P, center_freqs=_midi_to_hz(np.arange(60, 62)))),
]
BY_NAME = {c["name"]: c for c in CASES}

# cases that store the signals the reference filtered (rates other than sr) and one band's filtered signal
WITH_STEPS = {"defaults": 40, "multichannel": 10, "tuning_03": 0, "butter": 50, "fix_length": 5}

# filter-bank configurations whose designed filters the fixture stores (``bank/<name>/...``)
BANKS = {"defaults": {}, "tuning_03": dict(tuning=0.3), "butter": dict(ftype="butter"), "cheby1": dict(ftype="cheby1"),
         "cheby2": dict(ftype="cheby2"), "q15": dict(Q=15)}


def call(lib, case):
    """Run one case through ``lib`` (the reference or librosa_b200)."""
    return lib.iirt(signal(case["sig"]), **case["kw"])
