"""Generate tests/golden/hotpath_v1.npz (tests/cases.py), tests/golden/features_v1.npz
(tests/feature_cases.py) and tests/golden/reference_pins_v1.npz (tests/reference_pins.py) by running the
cases through the UNMODIFIED reference; ``--pitch`` writes only tests/golden/pitch_v1.npz (tests/pitch_cases.py)
and leaves the other fixtures as they are; ``--rhythm`` likewise writes only tests/golden/rhythm_v1.npz
(tests/rhythm_cases.py), ``--beat`` only tests/golden/beat_v1.npz (tests/beat_cases.py), ``--onset`` only
tests/golden/onset_v1.npz (tests/onset_cases.py), ``--sequence`` only tests/golden/sequence_v1.npz
(tests/sequence_cases.py), ``--alignment`` only tests/golden/alignment_v1.npz (tests/alignment_cases.py),
``--cqt`` only tests/golden/cqt_v1.npz (tests/cqt_cases.py), ``--chroma`` only tests/golden/chroma_v1.npz
(tests/chroma_cases.py), ``--iirt`` only tests/golden/iirt_v1.npz (tests/iirt_cases.py), ``--hybrid-cqt`` only
tests/golden/hybrid_cqt_v1.npz (tests/hybrid_cqt_cases.py), and ``--feature-utils`` only
tests/golden/feature_utils_v1.npz (tests/feature_utils_cases.py), and ``--piptrack`` only tests/golden/piptrack_v1.npz
(tests/piptrack_cases.py), ``--nn-filter`` only tests/golden/nn_filter_v1.npz (tests/nn_filter_cases.py).

Needs a checkout of the reference (see tools/ref_shim.py); the tests only read the stored fixtures.  Also
stores a handful of constant tables (mel bases, window sum-square, mel-scale known answers) produced by the
reference.

    python tools/make_golden.py
    python tools/make_golden.py --pitch
    python tools/make_golden.py --rhythm
    python tools/make_golden.py --beat
    python tools/make_golden.py --onset
    python tools/make_golden.py --sequence
    python tools/make_golden.py --alignment
    python tools/make_golden.py --cqt
    python tools/make_golden.py --chroma
    python tools/make_golden.py --iirt
    python tools/make_golden.py --hybrid-cqt
    python tools/make_golden.py --feature-utils
    python tools/make_golden.py --piptrack
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


def _zero_frames_outcome(ref, case):
    """The reference's outcome for a zero-frame case, run in a forked child.  Its numba decoder writes value[0] of a
    zero-row array (no bounds checks), so the process may die there; a dead child is reported, not recorded."""
    import multiprocessing as mp
    import sequence_cases as SC

    def child(conn):
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            conn.send(SC.call(ref, case))

    parent, conn = mp.get_context("fork").Pipe(duplex=False)
    proc = mp.get_context("fork").Process(target=child, args=(conn,))
    proc.start()
    got = parent.recv() if parent.poll(60) else None
    proc.join()
    if got is None:
        raise RuntimeError(f"{case['name']}: the reference's process died (exit code {proc.exitcode})")
    return got


def write_sequence():
    """tests/golden/sequence_v1.npz: per case of tests/sequence_cases.py, the reference's ``<name>/states`` and
    ``<name>/logp`` or ``<name>/error``; ``<name>/lp_sha256``, the SHA-256 of the float64 log-likelihoods its decoder
    reads (formed with the reference's own expressions, tests/sequence_oracle.py; the arrays themselves are megabytes
    of incompressible float64, rebuilt from the seeded inputs by the tests); and ``builder/<name>``, each ``transition_*`` output or
    ``builder/<name>/error``."""
    import sequence_cases as SC
    import sequence_oracle as SO

    ref = ref_shim.load_reference()
    store = {}
    for case in SC.CASES:
        name = case["name"]
        if case["obs"][3] == 0:
            got = _zero_frames_outcome(ref, case)
        else:
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                got = SC.call(ref, case)
        if "error" in got:
            store[name + "/error"] = np.array(got["error"])
        else:
            store[name + "/states"] = np.asarray(got["states"])
            if "logp" in got:
                store[name + "/logp"] = np.asarray(got["logp"])
            prob, transition, kw = SC.make(case, ref)
            kw.pop("return_logp", None)
            if prob.shape[-1] == 0:
                continue
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                store[name + "/lp_sha256"] = np.array(SO.digest(SO.run(case["op"], prob, transition, **kw)["lp"]))
        print(f"{name:44s} {got.get('error') or (got['states'].shape, got['states'].dtype)}")
    for key, spec in SC.BUILDERS.items():
        store["builder/" + key] = SC.builder(ref, spec)
    for key, spec in SC.BUILDER_ERRORS.items():
        try:
            SC.builder(ref, spec)
            raise RuntimeError(key)
        except ref.util.exceptions.ParameterError as exc:
            store["builder/" + key + "/error"] = np.array(f"{type(exc).__name__}: {exc}")
    path = os.path.join(ROOT, "tests", "golden", "sequence_v1.npz")
    np.savez_compressed(path, **store)
    print("wrote", path, os.path.getsize(path), "bytes")


def write_alignment():
    """tests/golden/alignment_v1.npz: per case of tests/alignment_cases.py, the reference's outputs (large ones as
    SHA-256) or ``<name>/error``.  A dtw whose path takes a (0, 0) step is never run: the reference's walk does not
    end there."""
    import alignment_cases as AC

    ref = ref_shim.load_reference()
    store = {}
    for case in AC.CASES:
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            got = AC.call(ref, case)
        store.update(AC.pack(case["name"], got))
        print(f"{case['name']:44s} {got.get('error') or {k: np.shape(v) for k, v in got.items()}}")
    path = os.path.join(ROOT, "tests", "golden", "alignment_v1.npz")
    np.savez_compressed(path, **store)
    print("wrote", path, os.path.getsize(path), "bytes")


def write_cqt():
    """tests/golden/cqt_v1.npz: per case of tests/cqt_cases.py, the reference's C (or ``<name>/error``), its
    warnings, and what each octave's response step received (signal length, n_fft, hop, the sparse basis; one
    octave's STFT for the cases in WITH_D), recorded by wrapping the reference's per-octave response function; and
    the reference's table of window bandwidths (``window_bandwidth/<name>``)."""
    import cqt_cases as QC

    ref = ref_shim.load_reference()
    import importlib

    cq = importlib.import_module("librosa.core.constantq")
    inner = cq.__dict__["__cqt_response"]
    calls = []

    def recorder(y, n_fft, hop_length, fft_basis, mode, window="ones", phase=True, dtype=None):
        calls.append((y, n_fft, hop_length, fft_basis, mode, dtype))
        return inner(y, n_fft, hop_length, fft_basis, mode, window=window, phase=phase, dtype=dtype)

    cq.__dict__["__cqt_response"] = recorder
    store = {}
    for case in QC.CASES:
        name = case["name"]
        calls.clear()
        with warnings.catch_warnings(record=True) as caught:
            warnings.simplefilter("always")
            try:
                C = QC.call(ref, case)
                store[f"{name}/C"] = C
            except Exception as e:   # the reference's own error, stored as "Class: message"
                store[f"{name}/error"] = np.array(f"{type(e).__name__}: {e}")
        store[f"{name}/warnings"] = np.array([str(w.message) for w in caught if "n_fft=" in str(w.message)])
        store[f"{name}/octaves"] = np.array([(y.shape[-1], n_fft, hop, b.shape[0]) for y, n_fft, hop, b, _, _ in calls],
                                            dtype=np.int64).reshape(-1, 4)
        for i, (y, n_fft, hop, b, mode, dtype) in enumerate(calls):
            if name not in QC.BASIS_ARRAYS:
                store[f"{name}/basis{i}/sha256"] = np.array(QC.basis_digest(b.indptr, b.indices, b.data))
            else:
                store[f"{name}/basis{i}/indptr"] = b.indptr
                store[f"{name}/basis{i}/indices"] = b.indices
                store[f"{name}/basis{i}/data"] = b.data
            if QC.WITH_D.get(name) == i:
                store[f"{name}/D"] = ref.stft(y, n_fft=n_fft, hop_length=hop, window="ones", pad_mode=mode, dtype=dtype)
        print(f"{name:32s} {store.get(f'{name}/error', np.shape(store.get(f'{name}/C')))} octaves={len(calls)}")
    for key, value in sorted(importlib.import_module("librosa.filters").WINDOW_BANDWIDTHS.items()):
        if isinstance(key, str):   # the reference's tabulated equivalent noise bandwidths
            store[f"window_bandwidth/{key}"] = np.float64(value)
    path = os.path.join(ROOT, "tests", "golden", "cqt_v1.npz")
    np.savez_compressed(path, **store)
    print("wrote", path, os.path.getsize(path), "bytes")


def write_chroma():
    """tests/golden/chroma_v1.npz: per case of tests/chroma_cases.py, the reference's result (or ``<name>/error``);
    the y= cases run with the reference's feature module calling the reference's own cqt / vqt with
    res_type="polyphase" (rebound only while they run).  For WITH_STEPS, |C| (the argument of the reference's
    cq_to_chroma einsum), the raw chroma (recorded around util.normalize) and CENS's quantised input (recorded
    around scipy.ndimage.convolve); and the cq_to_chroma maps of MAPS."""
    import functools
    import importlib

    import scipy.ndimage

    import chroma_cases as HC

    ref = ref_shim.load_reference()
    spectral = importlib.import_module("librosa.feature.spectral")
    store = {}
    for name, kw in HC.MAPS.items():
        kw = dict(kw)
        store[f"map/{name}"] = ref.filters.cq_to_chroma(kw.pop("n_input"), **kw)
    store["tonnetz_chroma_stft/input"] = ref.feature.chroma_stft(y=HC.stft_chroma_signal(), sr=22050, hop_length=512,
                                                                 tuning=0.0)
    orig = {k: spectral.__dict__[k] for k in ("cqt", "vqt", "np")}
    for case in HC.CASES:
        if case["refuse"]:
            continue
        name = case["name"]
        rec = {}
        polyphase = case["kw"].get("res_type") == "polyphase"

        class _Np:   # np as the feature module sees it, with einsum recorded (its second operand is |C|)
            def __getattr__(self, attr):
                return getattr(np, attr)

            @staticmethod
            def einsum(spec, *ops, **kw):
                out = np.einsum(spec, *ops, **kw)
                if spec == "cf,...ft->...ct":
                    rec.setdefault("absC", ops[1])
                    rec.setdefault("raw", out.copy())
                return out

        conv = scipy.ndimage.convolve

        def convolve(x, w, **kw):
            rec.setdefault("quant", np.array(x))
            return conv(x, w, **kw)

        if polyphase:
            spectral.cqt = functools.partial(orig["cqt"], res_type="polyphase")
            spectral.vqt = functools.partial(orig["vqt"], res_type="polyphase")
        spectral.np = _Np()
        scipy.ndimage.convolve = convolve
        try:
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                out = HC.call(ref, case, golden=store, drop_res_type=True)
            store[f"{name}/out"] = out
        except Exception as e:   # the reference's own error, stored as "Class: message"
            store[f"{name}/error"] = np.array(f"{type(e).__name__}: {e}")
        finally:
            spectral.__dict__.update(orig)
            scipy.ndimage.convolve = conv
        if name in HC.WITH_STEPS:
            for k, v in rec.items():
                if k != "absC" or case["inp"] is None:   # a C= case's |C| is its seeded input
                    store[f"{name}/{k}"] = v
        print(f"{name:32s} {store.get(f'{name}/error', np.shape(store.get(f'{name}/out')))} {sorted(rec)}")
    path = os.path.join(ROOT, "tests", "golden", "chroma_v1.npz")
    np.savez_compressed(path, **store)
    print("wrote", path, os.path.getsize(path), "bytes")


def write_iirt():
    """tests/golden/iirt_v1.npz: per case of tests/iirt_cases.py, the reference's result (or ``<name>/error``); for
    WITH_STEPS, what its resample returned for each rate other than sr and what its sosfiltfilt returned for one
    band, recorded by wrapping the two functions only while the case runs."""
    import importlib

    import scipy.signal

    import iirt_cases as IC

    ref = ref_shim.load_reference()
    spectrum = importlib.import_module("librosa.core.spectrum")
    resample, sosfiltfilt = spectrum.resample, scipy.signal.sosfiltfilt
    store = {}
    for case in IC.CASES:
        name = case["name"]
        if case["refuse"]:   # only the refusal is checked
            continue
        seen = {"y": {}, "bands": []}

        def rec_resample(y, *, orig_sr, target_sr, **kw):
            out = resample(y, orig_sr=orig_sr, target_sr=target_sr, **kw)
            if target_sr != orig_sr:
                seen["y"][float(target_sr)] = out
            return out

        def rec_sosfiltfilt(sos, x, *a, **kw):
            out = sosfiltfilt(sos, x, *a, **kw)
            seen["bands"].append(out)
            return out

        spectrum.resample, scipy.signal.sosfiltfilt = rec_resample, rec_sosfiltfilt
        try:
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                store[f"{name}/S"] = IC.call(ref, case)
        except Exception as e:   # the reference's own error, stored as "Class: message"
            store[f"{name}/error"] = np.array(f"{type(e).__name__}: {e}")
        finally:
            spectrum.resample, scipy.signal.sosfiltfilt = resample, sosfiltfilt
        if name in IC.WITH_STEPS and f"{name}/S" in store:
            for rate, y in seen["y"].items():
                store[f"{name}/y{rate:g}"] = y
            b = IC.WITH_STEPS[name]
            store[f"{name}/band{b}"] = seen["bands"][b]
        print(f"{name:32s} {store.get(f'{name}/error', np.shape(store.get(f'{name}/S')))}")
    for cfg, kw in IC.BANKS.items():   # the designed filter banks: sections stacked, sections per band, rates
        sos, srs = ref.filters.semitone_filterbank(flayout="sos", **kw)
        store[f"bank/{cfg}/sos"] = np.concatenate(sos)
        store[f"bank/{cfg}/sections"] = np.array([len(s) for s in sos])
        store[f"bank/{cfg}/rates"] = srs
    ba, _ = ref.filters.semitone_filterbank(flayout="ba")
    store["bank/defaults/b"] = np.stack([b for b, _ in ba])
    store["bank/defaults/a"] = np.stack([a for _, a in ba])
    store["mr_frequencies/0.3"] = np.stack(ref.filters.mr_frequencies(0.3))
    path = os.path.join(ROOT, "tests", "golden", "iirt_v1.npz")
    np.savez_compressed(path, **store)
    print("wrote", path, os.path.getsize(path), "bytes")


def write_hybrid_cqt():
    """tests/golden/hybrid_cqt_v1.npz: per case of tests/hybrid_cqt_cases.py, the reference's C (or
    ``<name>/error``), its stft warnings, the split of hybrid_cqt (recorded around the reference's pseudo_cqt and cqt,
    which hybrid_cqt calls through the module's globals), and what the pseudo part's response step received
    (n_fft, the |basis| or its digest, and the STFT for WITH_D), recorded around the reference's __cqt_response."""
    import hybrid_cqt_cases as HC

    ref = ref_shim.load_reference()
    import importlib

    cq = importlib.import_module("librosa.core.constantq")
    inner = {k: cq.__dict__[k] for k in ("__cqt_response", "pseudo_cqt", "cqt")}
    calls, parts = [], []

    def recorder(y, n_fft, hop_length, fft_basis, mode, window="ones", phase=True, dtype=None):
        if not phase:
            calls.append((y, n_fft, hop_length, fft_basis, mode, dtype))
        return inner["__cqt_response"](y, n_fft, hop_length, fft_basis, mode, window=window, phase=phase, dtype=dtype)

    def rec_pseudo(y, **kw):
        parts.append(("pseudo", kw["fmin"], kw["n_bins"]))
        return inner["pseudo_cqt"](y, **kw)

    def rec_cqt(y, **kw):
        parts.append(("full", kw["fmin"], kw["n_bins"]))
        return inner["cqt"](y, **kw)

    cq.__dict__["__cqt_response"] = recorder
    store = {}
    for case in HC.CASES:
        name = case["name"]
        calls.clear()
        parts.clear()
        hybrid = case["fn"] == "hybrid_cqt"
        if hybrid:
            cq.__dict__["pseudo_cqt"], cq.__dict__["cqt"] = rec_pseudo, rec_cqt
        with warnings.catch_warnings(record=True) as caught:
            warnings.simplefilter("always")
            try:
                store[f"{name}/C"] = HC.call(ref, case)
            except Exception as e:   # the reference's own error, stored as "Class: message"
                store[f"{name}/error"] = np.array(f"{type(e).__name__}: {e}")
            finally:
                cq.__dict__["pseudo_cqt"], cq.__dict__["cqt"] = inner["pseudo_cqt"], inner["cqt"]
        store[f"{name}/warnings"] = np.array([str(w.message) for w in caught if "n_fft=" in str(w.message)])
        if hybrid:
            got = {kind: (fmin, n) for kind, fmin, n in parts}
            store[f"{name}/n_pseudo"] = np.int64(got.get("pseudo", (0, 0))[1])
            store[f"{name}/n_full"] = np.int64(got.get("full", (0, 0))[1])
            if "pseudo" in got:
                store[f"{name}/fmin_pseudo"] = np.float64(got["pseudo"][0])
        for y, n_fft, hop, b, mode, dtype in calls[:1]:
            store[f"{name}/n_fft"] = np.int64(n_fft)
            if name in HC.BASIS_DIGEST:
                store[f"{name}/basis/sha256"] = np.array(HC.basis_digest(b.indptr, b.indices, b.data))
            else:
                store[f"{name}/basis/indptr"] = b.indptr
                store[f"{name}/basis/indices"] = b.indices
                store[f"{name}/basis/data"] = b.data
            if name in HC.WITH_D:
                store[f"{name}/D"] = ref.stft(y, n_fft=n_fft, hop_length=hop, window="hann", pad_mode=mode, dtype=dtype)
        print(f"{name:32s} {store.get(f'{name}/error', np.shape(store.get(f'{name}/C')))} "
              f"pseudo calls={len(calls)} parts={[(k, n) for k, _, n in parts]}")
    cq.__dict__["__cqt_response"] = inner["__cqt_response"]
    path = os.path.join(ROOT, "tests", "golden", "hybrid_cqt_v1.npz")
    np.savez_compressed(path, **store)
    print("wrote", path, os.path.getsize(path), "bytes")


def write_feature_utils():
    """tests/golden/feature_utils_v1.npz: per case of tests/feature_utils_cases.py that the GPU does not refuse, the
    reference's delta / stack_memory output (``<name>/out``) or its error (``<name>/error``)."""
    import feature_utils_cases as FU

    ref = ref_shim.load_reference()
    store = {}
    for case in FU.CASES:
        if case["refuse"]:
            continue
        name = case["name"]
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            try:
                store[f"{name}/out"] = np.asarray(FU.call(ref, case))
            except Exception as e:   # the reference's own error, stored as "Class: message"
                store[f"{name}/error"] = np.array(f"{type(e).__name__}: {e}")
        print(f"{name:40s} {store.get(f'{name}/error', np.shape(store.get(f'{name}/out')))}")
    path = os.path.join(ROOT, "tests", "golden", "feature_utils_v1.npz")
    np.savez_compressed(path, **store)
    print("wrote", path, os.path.getsize(path), "bytes")


def write_piptrack():
    """tests/golden/piptrack_v1.npz: per case of tests/piptrack_cases.py that the GPU does not refuse, the reference's
    piptrack result in sparse form (and, from y, its magnitude spectrogram), pitch_tuning value or localmax / localmin
    mask, or its error (``<name>/error``)."""
    import piptrack_cases as PC

    ref = ref_shim.load_reference()
    store = {}
    for case in PC.CASES:
        if case["refuse"]:
            continue
        name = case["name"]
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            try:
                out = PC.call(ref, case)
            except Exception as e:   # the reference's own error, stored as "Class: message"
                store[f"{name}/error"] = np.array(f"{type(e).__name__}: {e}")
                print(f"{name:40s} {store[f'{name}/error']}")
                continue
        if case["fn"] == "piptrack":
            p, m = out
            store[f"{name}/shape"] = np.array(p.shape, dtype=np.int64)
            store[f"{name}/dtype"] = np.array(p.dtype.name)
            store[f"{name}/idx"], store[f"{name}/p"], store[f"{name}/m"] = PC.sparse(p, m)
            if case["y"] is not None:
                kw = PC.piptrack_args(case)
                store[f"{name}/S"] = ref.core.spectrum._spectrogram(
                    y=kw["y"], n_fft=kw.get("n_fft", 2048), hop_length=kw.get("hop_length"), power=1,
                    win_length=kw.get("win_length"), window=kw.get("window", "hann"), center=kw.get("center", True),
                    pad_mode=kw.get("pad_mode", "constant"))[0]
            print(f"{name:40s} {p.shape} {p.dtype} peaks={store[f'{name}/idx'].size}")
        else:
            store[f"{name}/out"] = np.asarray(out)
            print(f"{name:40s} {store[f'{name}/out'].shape} {store[f'{name}/out'].dtype}")
    path = os.path.join(ROOT, "tests", "golden", "piptrack_v1.npz")
    np.savez_compressed(path, **store)
    print("wrote", path, os.path.getsize(path), "bytes")


def write_nn_filter():
    """tests/golden/nn_filter_v1.npz: per case of tests/nn_filter_cases.py, the reference's recurrence matrix (csc
    indptr / indices / data) and, for nn_filter cases, its output, or its error (``<name>/error``)."""
    import nn_filter_cases as NC

    ref = ref_shim.load_reference()
    store = {}
    for case in NC.CASES:
        name = case["name"]
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            try:
                out = NC.call(ref, case)
            except Exception as e:   # the reference's own error, stored as "Class: message"
                store[f"{name}/error"] = np.array(f"{type(e).__name__}: {e}")
                print(f"{name:40s} {store[f'{name}/error']}")
                if case["fn"] == "nn":   # the rec of a failing nn_filter case is still stored
                    S, clean = NC.filter_input(case)
                    out = (ref.segment.recurrence_matrix(clean, sparse=True, **case["rec_kw"]), None)
                else:
                    continue
        rec, res = (out, None) if case["fn"] == "rec" else out
        store[f"{name}/indptr"] = rec.indptr.astype(np.int64)
        store[f"{name}/indices"] = rec.indices.astype(np.int32)
        store[f"{name}/data"] = rec.data
        if res is not None:
            store[f"{name}/out"] = res
        print(f"{name:40s} nnz={rec.nnz} {rec.dtype}")
    path = os.path.join(ROOT, "tests", "golden", "nn_filter_v1.npz")
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
    elif "--sequence" in sys.argv[1:]:
        write_sequence()
    elif "--alignment" in sys.argv[1:]:
        write_alignment()
    elif "--cqt" in sys.argv[1:]:
        write_cqt()
    elif "--chroma" in sys.argv[1:]:
        write_chroma()
    elif "--iirt" in sys.argv[1:]:
        write_iirt()
    elif "--hybrid-cqt" in sys.argv[1:]:
        write_hybrid_cqt()
    elif "--feature-utils" in sys.argv[1:]:
        write_feature_utils()
    elif "--piptrack" in sys.argv[1:]:
        write_piptrack()
    elif "--nn-filter" in sys.argv[1:]:
        write_nn_filter()
    else:
        main()
