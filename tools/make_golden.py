"""Generate tests/golden/hotpath_v1.npz (tests/cases.py), tests/golden/features_v1.npz
(tests/feature_cases.py) and tests/golden/reference_pins_v1.npz (tests/reference_pins.py) by running the
cases through the UNMODIFIED reference; ``--pitch`` writes only tests/golden/pitch_v1.npz (tests/pitch_cases.py)
and leaves the other fixtures as they are; ``--rhythm`` likewise writes only tests/golden/rhythm_v1.npz
(tests/rhythm_cases.py), ``--beat`` only tests/golden/beat_v1.npz (tests/beat_cases.py), and ``--onset`` only
tests/golden/onset_v1.npz (tests/onset_cases.py).

Needs a checkout of the reference (see tools/ref_shim.py); the tests only read the stored fixtures.  Also
stores a handful of constant tables (mel bases, window sum-square, mel-scale known answers) produced by the
reference.

    python tools/make_golden.py
    python tools/make_golden.py --pitch
    python tools/make_golden.py --rhythm
    python tools/make_golden.py --beat
    python tools/make_golden.py --onset
"""
from __future__ import annotations

import os
import sys
import warnings

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import ref_shim  # noqa: E402
from cases import BY_NAME, CASES  # noqa: E402
import signals  # noqa: E402


def run_case(ref, case, store):
    op, kw = case["op"], dict(case["kw"])
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        if op == "istft":
            D = store[case["src"]]
            return ref.istft(D, **kw)
        sr = kw.get("sr", 22050)
        y = signals.make(case["mix"], case["shape"], seed=len(case["name"]), sr=sr)
        if op == "stft":
            return ref.stft(y, **kw)
        if op == "mel":
            return ref.feature.melspectrogram(y=y, **kw)
        if op == "mfcc":
            return ref.feature.mfcc(y=y, **kw)
    raise ValueError(op)


def main():
    ref = ref_shim.load_reference()
    store = {}
    for case in CASES:
        out = run_case(ref, case, store)
        store[case["name"]] = np.ascontiguousarray(out)
        print(f"{case['name']:40s} {out.shape} {out.dtype}")
    # constant tables straight from the reference
    consts = {
        "const/mel_22050_2048": ref.filters.mel(sr=22050, n_fft=2048),
        "const/mel_44100_4096": ref.filters.mel(sr=44100, n_fft=4096),
        "const/mel_16000_1024_htk40": ref.filters.mel(sr=16000, n_fft=1024, n_mels=40, htk=True),
        "const/mel_22050_2048_norm1": ref.filters.mel(sr=22050, n_fft=2048, norm=1, fmin=300.0, fmax=8000.0, n_mels=64),
        "const/wss_hann_2048_512_50": ref.filters.window_sumsquare(window="hann", n_frames=50, hop_length=512, n_fft=2048),
        "const/wss_hamming_600_1024_300_20": ref.filters.window_sumsquare(window="hamming", n_frames=20, hop_length=300, win_length=600, n_fft=1024),
        "const/hz_to_mel": ref.hz_to_mel(np.array([0.0, 60.0, 440.0, 999.0, 1000.0, 5000.0, 11025.0])),
        "const/hz_to_mel_htk": ref.hz_to_mel(np.array([0.0, 60.0, 440.0, 999.0, 1000.0, 5000.0, 11025.0]), htk=True),
        "const/mel_to_hz": ref.mel_to_hz(np.array([0.0, 3.0, 14.9, 15.0, 25.0, 40.0])),
        "const/mel_to_hz_htk": ref.mel_to_hz(np.array([0.0, 300.0, 1000.0, 2000.0, 3000.0]), htk=True),
        "const/mel_frequencies_40": ref.mel_frequencies(n_mels=40),
        "const/window_hann_2048": ref.filters.get_window("hann", 2048),
        "const/power_to_db_in": (np.abs(np.random.default_rng(7).standard_normal((2, 16, 12))) ** 2).astype(np.float32),
    }
    consts["const/power_to_db_out"] = ref.power_to_db(consts["const/power_to_db_in"])
    consts["const/power_to_db_out_refmax"] = ref.power_to_db(consts["const/power_to_db_in"], ref=np.max)
    consts["const/power_to_db_out_top40"] = ref.power_to_db(consts["const/power_to_db_in"], top_db=40.0)
    store.update(consts)
    path = os.path.join(ROOT, "tests", "golden", "hotpath_v1.npz")
    np.savez_compressed(path, **store)
    print("wrote", path, os.path.getsize(path), "bytes; reference", ref.__version__)
    # ---- frame-wise consumers (tests/feature_cases.py)
    from feature_cases import FEATURE_CASES, call, fixture_names, outputs

    feats = {}
    for case in FEATURE_CASES:
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            out = call(ref, case, store)
        outs = outputs(out)
        for key, arr in zip(fixture_names(case, len(outs)), outs):
            feats[key] = np.ascontiguousarray(arr) if arr.ndim else arr
            print(f"{key:40s} {arr.shape} {arr.dtype}")
    path = os.path.join(ROOT, "tests", "golden", "features_v1.npz")
    np.savez_compressed(path, **feats)
    print("wrote", path, os.path.getsize(path), "bytes")
    write_reference_pins(ref)


def write_reference_pins(ref):
    """tests/golden/reference_pins_v1.npz: what tests/test_oracle_vs_reference.py compares against."""
    import reference_pins

    path = os.path.join(ROOT, "tests", "golden", "reference_pins_v1.npz")
    np.savez_compressed(path, **reference_pins.pack(reference_pins.reference_outputs(ref)))
    print("wrote", path, os.path.getsize(path), "bytes")


def write_pitch():
    """tests/golden/pitch_v1.npz: yin / pyin of every case of tests/pitch_cases.py."""
    from pitch_cases import PITCH_CASES, outputs, run

    ref = ref_shim.load_reference()
    store = {}
    for case in PITCH_CASES:
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            for key, arr in outputs(case, run(ref, case)).items():
                store[key] = np.ascontiguousarray(arr)
                print(f"{key:40s} {arr.shape} {arr.dtype}")
    path = os.path.join(ROOT, "tests", "golden", "pitch_v1.npz")
    np.savez_compressed(path, **store)
    print("wrote", path, os.path.getsize(path), "bytes")


def write_rhythm():
    """tests/golden/rhythm_v1.npz: tempogram / fourier_tempogram / tempo of every case of tests/rhythm_cases.py."""
    from rhythm_cases import RHYTHM_CASES, outputs, run

    ref = ref_shim.load_reference()
    store = {}
    for case in RHYTHM_CASES:
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            for key, arr in outputs(case, run(ref, case)).items():
                store[key] = np.ascontiguousarray(arr)
                print(f"{key:48s} {arr.shape} {arr.dtype}")
    path = os.path.join(ROOT, "tests", "golden", "rhythm_v1.npz")
    np.savez_compressed(path, **store)
    print("wrote", path, os.path.getsize(path), "bytes")


def write_beat():
    """tests/golden/beat_v1.npz: per case of tests/beat_cases.py, beat_track's ``bpm`` and ``beats``, plp's ``pulse``,
    beat_track(y=) on click trains, and the tracker stages (the reference module's own private functions) for that bpm: ``localscore``, ``cumscore``, ``backlink``
    and ``tail``.  The batch with an all-zero clip has no ``beats``: the reference's trim loop runs past the end of
    that clip's array."""
    import beat_cases as BC

    ref = ref_shim.load_reference()
    rb = ref.beat
    stage = {name: getattr(rb, "__" + name) for name in ("normalize_onsets", "beat_local_score", "beat_track_dp",
                                                           "last_beat")}
    store = {}
    for case in BC.BEAT_CASES:
        name, kw = case["name"], BC.kwargs(case)
        x = BC.make_input(case)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            bpm = kw["bpm"]
            if bpm is None and BC.has_stages(case):
                bpm = ref.feature.tempo(onset_envelope=x, sr=kw["sr"], hop_length=kw["hop_length"],
                                        prior=kw.get("prior"))
            if case["env"][0] != "zero_clip":
                got_bpm, beats = BC.run(ref, case)
                store[name + "/beats"] = np.asarray(beats)
                store[name + "/bpm"] = np.asarray(got_bpm, dtype=np.float64)
            else:
                store[name + "/bpm"] = np.asarray(bpm, dtype=np.float64)
            if BC.has_stages(case):
                _bpm = np.atleast_1d(bpm)
                bpm_exp = ref.util.expand_to(_bpm, ndim=x.ndim, axes=range(_bpm.ndim))
                fpb = np.round(float(kw["sr"]) / kw["hop_length"] * 60.0 / bpm_exp)
                ls = np.empty_like(x)
                stage["beat_local_score"](stage["normalize_onsets"](x), fpb, ls)
                back, cum = stage["beat_track_dp"](ls, fpb, BC.stage_kwargs(case)["tightness"])
                store[name + "/localscore"] = ls
                store[name + "/cumscore"] = cum
                store[name + "/backlink"] = back
                store[name + "/tail"] = np.asarray(stage["last_beat"](cum), dtype=np.int64)
        for key in [k for k in store if k.startswith(name + "/")]:
            print(f"{key:48s} {store[key].shape} {store[key].dtype}")
    for case in BC.PLP_CASES:
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            store[case["name"] + "/pulse"] = np.ascontiguousarray(BC.run_plp(ref, case))
    for name, bpm in BC.Y_CASES.items():
        got_bpm, beats = ref.beat.beat_track(y=BC.clicks_audio(bpm), sr=BC.SR, hop_length=BC.HOP)
        store[name + "/bpm"] = np.asarray(got_bpm, dtype=np.float64)
        store[name + "/beats"] = np.asarray(beats)
        print(name, got_bpm, beats)
    path = os.path.join(ROOT, "tests", "golden", "beat_v1.npz")
    np.savez_compressed(path, **store)
    print("wrote", path, os.path.getsize(path), "bytes")


def write_onset():
    """tests/golden/onset_v1.npz: per case of tests/onset_cases.py, ``<name>/out`` (the reference's result) or
    ``<name>/error`` ("Class: message"); ``<name>/norm``, onset_detect's normalised envelope, for the detection
    cases that normalise; and ``onset_detect(y=)`` on click trains."""
    import onset_cases as OC

    ref = ref_shim.load_reference()
    store = {}
    for case in OC.CASES:
        name = case["name"]
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            got = OC.outcome(ref, case)
        if "out" in got:
            store[name + "/out"] = np.ascontiguousarray(got["out"])
        else:
            store[name + "/error"] = np.array(got["error"])
        if (case["op"] == "onset_detect" and case["env"] is not None and case["kw"].get("normalize", True)
                and case["env"][2] > 0):   # zero frames: the reference's np.min raises
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                store[name + "/norm"] = OC.normalized(OC.envelope(case["env"]))
        print(f"{name:48s} {got.get('error') or (got['out'].shape, got['out'].dtype)}")
    for name, bpm in OC.Y_CASES.items():
        store[name + "/out"] = np.asarray(ref.onset.onset_detect(y=OC.clicks_audio(bpm), sr=OC.SR, hop_length=OC.HOP))
        print(name, store[name + "/out"])
    path = os.path.join(ROOT, "tests", "golden", "onset_v1.npz")
    np.savez_compressed(path, **store)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    if "--pitch" in sys.argv[1:]:
        write_pitch()
    elif "--rhythm" in sys.argv[1:]:
        write_rhythm()
    elif "--beat" in sys.argv[1:]:
        write_beat()
    elif "--onset" in sys.argv[1:]:
        write_onset()
    else:
        main()
