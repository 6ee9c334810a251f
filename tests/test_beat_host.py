"""beat_track without a GPU: the oracle against the reference's outputs and tracker stages (tests/golden/beat_v1.npz,
bit for bit), the libm tables against the same expressions compiled with numba, the unit converters, and the
argument errors, their order and the refused sizes, all raised before any tracker launch."""
import math
import os
import warnings

import numpy as np
import pytest

import beat_cases as BC
import beat_oracle as BO
import librosa_b200 as lb
from librosa_b200 import beat as B

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def beat_golden():
    with np.load(os.path.join(ROOT, "tests", "golden", "beat_v1.npz")) as z:
        return {k: z[k] for k in z.files}


def _same(got, want, key):
    got = np.asarray(got)
    assert got.dtype == want.dtype and got.shape == want.shape, (key, got.dtype, want.dtype, got.shape, want.shape)
    assert got.tobytes() == want.tobytes(), key


@pytest.mark.parametrize("name", [c["name"] for c in BC.BEAT_CASES])
def test_oracle_bit_exact(beat_golden, name):
    case = BC.BY_NAME[name]
    if name + "/beats" in beat_golden:
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            bpm, beats = BC.run(BO, case)
        _same(beats, beat_golden[name + "/beats"], name + "/beats")
        if case["kw"].get("bpm") is None and BC.has_stages(case):
            _same(np.asarray(bpm, dtype=np.float64), beat_golden[name + "/bpm"], name + "/bpm")
    if BC.has_stages(case):
        x = BC.make_input(case)
        _, fpb = BO.frames_per_beat(beat_golden[name + "/bpm"] if BC.bpm_arg(case) is None else BC.bpm_arg(case),
                                    BC.SR, BC.HOP, x.shape)
        got = BO.track_stages(x, fpb, **BC.stage_kwargs(case))
        for key in ("localscore", "cumscore", "backlink", "tail"):
            _same(got[key], beat_golden[f"{name}/{key}"], f"{name}/{key}")


def test_zero_clip_yields_no_beats():
    case = BC.BY_NAME["beat/zero_clip_float32"]
    x = BC.make_input(case)
    _, fpb = BO.frames_per_beat(120.0, BC.SR, BC.HOP, x.shape)
    beats = BO.track_stages(x, fpb)["beats"]
    assert not beats[1].any() and beats[0].any() and beats[2].any()


def test_libm_tables_match_numba():
    """The host tables against the same expressions compiled with numba, for fpb 1 .. 4096."""
    nb = pytest.importorskip("numba")

    @nb.njit
    def win(fpb):
        return np.exp(-0.5 * (np.arange(-fpb, fpb + 1) * 32.0 / fpb) ** 2)

    @nb.njit
    def logs(top):
        out = np.empty(top + 1)
        out[0] = 0.0
        for d in range(1, top + 1):
            out[d] = np.log(d)
        return out

    @nb.njit
    def logf(f):
        return np.log(f)

    fpbs = np.arange(1, 4097)
    for f in fpbs:
        assert B.window(int(f), int(f)).tobytes() == win(float(f)).tobytes(), f
        assert B.log_fpb(int(f), True) == logf(np.float64(f))
        assert B.log_fpb(int(f), False) == float(logf(np.float32(f)))
    assert B.log_table(8192).tobytes() == logs(8192).tobytes()


def test_window_truncation_is_a_slice():
    """Windows wider than the envelope keep only the |d| <= n - 1 part, the same values."""
    full = B.window(50, 50)
    assert B.window(50, 10).tobytes() == full[40:61].tobytes()


@pytest.mark.parametrize("frames", [np.arange(5), np.array([0, 3, 431]), 7, np.array([], dtype=int)])
@pytest.mark.parametrize("hop,sr,n_fft", [(512, 22050, None), (256, 16000, 1024), (1, 44100, 3)])
def test_unit_converters(frames, hop, sr, n_fft):
    want_s = (np.asanyarray(frames) * hop + (0 if n_fft is None else n_fft // 2)).astype(int)[()]
    got_s = lb.frames_to_samples(frames, hop_length=hop, n_fft=n_fft)
    assert np.asarray(got_s).dtype == np.asarray(want_s).dtype and np.array_equal(got_s, want_s)
    got_t = lb.frames_to_time(frames, sr=sr, hop_length=hop, n_fft=n_fft)
    want_t = np.asanyarray(want_s)[()] / float(sr)
    assert np.asarray(got_t).tobytes() == np.asarray(want_t).tobytes()
    assert np.asarray(lb.samples_to_time(want_s, sr=sr)).tobytes() == np.asarray(want_t).tobytes()
    assert lb.core.frames_to_time is lb.frames_to_time and "frames_to_samples" in lb.core.__all__


_ENV = BC.make_input(BC.BY_NAME["beat/bpm120_t100_trim1_float32"])
_ZERO = np.zeros(200, dtype=np.float32)

# (keyword arguments, exception, message): each raised before the tracker runs
_ERRORS = [
    (dict(), lb.ParameterError, "y or onset_envelope must be provided"),
    (dict(onset_envelope=np.stack([_ENV, _ENV])), lb.ParameterError, "sparse=True .* 2-dimensional"),
    (dict(onset_envelope=_ENV, bpm=0.0), lb.ParameterError, "must be strictly positive"),
    (dict(onset_envelope=_ENV, bpm=-3.0, tightness=-1), lb.ParameterError, "bpm=.* must be strictly positive"),
    (dict(onset_envelope=_ENV, bpm=120.0, tightness=0), lb.ParameterError, "tightness must be strictly positive"),
    (dict(onset_envelope=_ENV, bpm=np.full(7, 120.0)), lb.ParameterError, "Invalid bpm shape"),
    (dict(onset_envelope=_ENV, bpm=120.0, units="beats"), lb.ParameterError, "Invalid unit type: beats"),
    (dict(onset_envelope=_ENV, bpm=120.0 * BC.FRAME_RATE * 1.5), lb.UnsupportedOnGPU, "rounds to 0 frames per beat"),
    (dict(onset_envelope=_ENV, bpm=1e-9), lb.UnsupportedOnGPU, "frames per beat above"),
    (dict(onset_envelope=_ENV.astype(np.int32)), lb.UnsupportedOnGPU, "float32 or float64"),
]


class _NoTracker(Exception):
    pass


@pytest.mark.parametrize("kw,exc,msg", _ERRORS, ids=[str(i) for i in range(len(_ERRORS))])
def test_errors_before_tracker(monkeypatch, kw, exc, msg):
    """Checks run on the host before the tracker: neither the staging nor a launch is reached."""
    from librosa_b200.feature import rhythm as R

    class Env:
        def __init__(self, y, sr, onset_envelope, hop_length, aggregate=None):
            if onset_envelope is None:
                raise _NoTracker()
            self.dev = np.asarray(onset_envelope)
            self.ctx, self.on_device = None, False

        def verdict(self):
            pass

        def release(self):
            pass

    def no_launch(*a, **k):
        raise AssertionError("tracker launched before the argument checks")

    monkeypatch.setattr(R, "_Envelope", Env)
    monkeypatch.setattr(B, "_launch", no_launch)
    with pytest.raises(exc, match=msg):
        lb.beat.beat_track(**kw)


def test_zero_envelope_returns_before_bpm_checks(monkeypatch):
    """An all-zero envelope returns before tightness / bpm are validated, as in the reference."""
    from librosa_b200.feature import rhythm as R

    class Env:
        def __init__(self, y, sr, onset_envelope, hop_length, aggregate=None):
            self.dev = np.asarray(onset_envelope)
            self.ctx, self.on_device = None, False

        def verdict(self):
            pass

        def release(self):
            pass

    monkeypatch.setattr(R, "_Envelope", Env)
    bpm, beats = lb.beat.beat_track(onset_envelope=_ZERO, bpm=-1.0, tightness=-5)
    assert bpm == 0.0 and beats.dtype == np.asarray([], dtype=int).dtype and beats.size == 0
    bpm, beats = lb.beat.beat_track(onset_envelope=np.zeros((2, 50), np.float64), sparse=False, tightness=0)
    assert bpm.shape == (2,) and bpm.dtype == np.float64 and beats.shape == (2, 50) and beats.dtype == bool


def test_median_refusal_before_any_device_work(monkeypatch):
    """Channels wider than the median kernel's 512 rows, and other aggregates, are refused from the shapes alone."""
    from librosa_b200 import _native as nat
    from librosa_b200 import _pipeline as pl

    def no_device(*a, **k):
        raise AssertionError("device work before the refusal")

    monkeypatch.setattr(pl, "StagedInput", no_device)
    monkeypatch.setattr(nat, "default_context", no_device)
    monkeypatch.setattr(nat, "lib", no_device)
    with pytest.raises(lb.UnsupportedOnGPU, match="600 rows"):
        lb.onset.onset_strength(S=np.zeros((600, 20), np.float32), aggregate=np.median)
    with pytest.raises(lb.UnsupportedOnGPU, match="513 rows"):
        lb.onset.onset_strength_multi(S=np.zeros((2, 700, 20), np.float32), aggregate=np.median, channels=[0, 513, 700])
    with pytest.raises(lb.UnsupportedOnGPU, match="640 rows"):
        lb.onset.onset_strength(y=np.zeros(22050, np.float32), aggregate=np.median, n_mels=640)
    with pytest.raises(lb.UnsupportedOnGPU, match="only mean or median"):
        lb.onset.onset_strength(S=np.zeros((10, 20), np.float32), aggregate=np.max)


@pytest.mark.parametrize("name", [c["name"] for c in BC.PLP_CASES])
def test_plp_oracle_vs_golden(beat_golden, name):
    case = BC.PLP_BY_NAME[name]
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        got = BC.run_plp(BO, case)
    want = beat_golden[name + "/pulse"]
    assert got.dtype == want.dtype and got.shape == want.shape
    assert np.max(np.abs(got - want)) <= 1e-6, float(np.max(np.abs(got - want)))


@pytest.mark.parametrize("name", [c["name"] for c in BC.PLP_CASES])
def test_plp_cases_have_no_fragile_frame(name):
    """The GPU's peak selection is compared mask for mask; no case may hang on the last bits of ftmag."""
    import rhythm_oracle as RO

    case = BC.PLP_BY_NAME[name]
    kw = BC.plp_kwargs(case)
    W = kw.get("win_length", 384)
    ft = RO.fourier_tempogram(onset_envelope=BC.make_input(case), sr=kw["sr"], hop_length=kw["hop_length"],
                              win_length=W)
    freqs = RO.fourier_tempo_frequencies(sr=kw["sr"], hop_length=kw["hop_length"], win_length=W)
    keep = BO.plp_keep(freqs, kw.get("tempo_min", 30), kw.get("tempo_max", 300))
    prior = kw.get("prior")
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        fragile = BO.plp_fragile(ft, keep, None if prior is None else prior.logpdf(freqs))
    assert not fragile.any(), np.argwhere(fragile)[:5]


def test_plp_errors():
    with pytest.raises(lb.ParameterError, match="tempo_max=60 must be larger than tempo_min=120"):
        lb.beat.plp(onset_envelope=_ENV, tempo_min=120, tempo_max=60)
    with pytest.raises(lb.ParameterError, match="tempo_max=60 must be larger than tempo_min=60"):
        lb.beat.plp(onset_envelope=_ENV, tempo_min=60, tempo_max=60)
    with pytest.raises(lb.ParameterError):
        lb.beat.plp()


def test_public_names():
    assert lb.beat.beat_track is B.beat_track and lb.beat.plp is B.plp and "beat" in lb.__all__
    for name in ("frames_to_samples", "frames_to_time", "samples_to_time"):
        assert name in lb.__all__ and name in lb.core.__all__
    assert math.isclose(float(lb.frames_to_time(1)), 512 / 22050)
