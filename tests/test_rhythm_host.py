"""tempogram / fourier_tempogram / tempo without a GPU: the oracle against the reference's outputs
(tests/golden/rhythm_v1.npz, bit for bit), the tempo-axis converters, and the argument errors and refusals of the
public functions, which are all raised before any device work."""
import os
import warnings

import numpy as np
import pytest

import librosa_b200 as lb
import rhythm_cases as RC
import rhythm_oracle as RO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def rhythm_golden():
    with np.load(os.path.join(ROOT, "tests", "golden", "rhythm_v1.npz")) as z:
        return {k: z[k] for k in z.files}


@pytest.mark.parametrize("name", [c["name"] for c in RC.RHYTHM_CASES])
def test_oracle_bit_exact(rhythm_golden, name):
    case = RC.BY_NAME[name]
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        got = RC.outputs(case, RC.run(RO, case))
    for key, arr in got.items():
        ref = rhythm_golden[key]
        assert arr.dtype == ref.dtype and arr.shape == ref.shape, key
        assert arr.tobytes() == ref.tobytes(), key


@pytest.mark.parametrize("n_bins,hop,sr", [(1, 512, 22050), (2, 512, 22050), (384, 512, 22050), (4096, 256, 16000),
                                           (344, 1024, 44100)])
def test_tempo_frequencies_exact(n_bins, hop, sr):
    got = lb.tempo_frequencies(n_bins, hop_length=hop, sr=sr)
    want = RO.tempo_frequencies(n_bins, hop_length=hop, sr=sr)
    assert got.dtype == np.float64 and got.tobytes() == want.tobytes()


@pytest.mark.parametrize("win,hop,sr", [(1, 512, 22050), (384, 512, 22050), (343, 256, 16000), (4096, 1024, 44100)])
def test_fourier_tempo_frequencies_exact(win, hop, sr):
    got = lb.fourier_tempo_frequencies(sr=sr, win_length=win, hop_length=hop)
    want = RO.fourier_tempo_frequencies(sr=sr, win_length=win, hop_length=hop)
    assert got.dtype == np.float64 and got.tobytes() == want.tobytes()


def test_time_to_frames():
    from librosa_b200.feature import rhythm as R

    for ac, sr, hop in ((8.0, 22050, 512), (4, 16000, 1024), (5, 22050, 512), (0.01, 22050, 512)):
        assert R._time_to_frames(ac, sr, hop) == RO.time_to_frames(ac, sr=sr, hop_length=hop).item()


_ENV = RC.envelope("clicks", (), 200)

# (call, keyword arguments, exception, message) — each raised before anything reaches the device
_ERRORS = [
    ("tempogram", dict(onset_envelope=_ENV, win_length=0), lb.ParameterError, "win_length must be a positive"),
    ("tempogram", dict(onset_envelope=_ENV, win_length=-384), lb.ParameterError, "win_length must be a positive"),
    ("tempogram", dict(onset_envelope=_ENV, window=np.ones(3)), lb.ParameterError, "Window size mismatch"),
    ("tempogram", dict(), lb.ParameterError, "Either y or onset_envelope"),
    ("tempogram", dict(onset_envelope=_ENV, norm="fro"), lb.ParameterError, "Unsupported norm"),
    ("tempogram", dict(onset_envelope=_ENV, norm=-2), lb.ParameterError, "Unsupported norm"),
    ("tempogram", dict(onset_envelope=_ENV, win_length=4097), lb.UnsupportedOnGPU, "win_length=4097"),
    ("fourier_tempogram", dict(onset_envelope=_ENV, win_length=0), lb.ParameterError, "win_length must be a positive"),
    ("fourier_tempogram", dict(), lb.ParameterError, "Either y or onset_envelope"),
    ("tempo", dict(onset_envelope=_ENV, start_bpm=0), lb.ParameterError, "start_bpm must be strictly positive"),
    ("tempo", dict(onset_envelope=_ENV, start_bpm=-120), lb.ParameterError, "start_bpm must be strictly positive"),
    ("tempo", dict(), lb.ParameterError, "Either y or onset_envelope"),
    ("tempo", dict(onset_envelope=_ENV, aggregate=np.median), lb.UnsupportedOnGPU, "aggregate"),
    ("tempo", dict(onset_envelope=_ENV, ac_size=0.01), lb.ParameterError, "win_length must be a positive"),
    ("tempo", dict(onset_envelope=_ENV, ac_size=100.0), lb.UnsupportedOnGPU, "win_length=4306"),
]


@pytest.mark.parametrize("fn,kw,exc,msg", _ERRORS, ids=[f"{e[0]}-{i}" for i, e in enumerate(_ERRORS)])
def test_errors_before_device_work(monkeypatch, fn, kw, exc, msg):
    """The reference's argument errors (and the GPU's refusals) come before any staging: a device touch fails."""
    from librosa_b200 import _pipeline as pl

    def no_device(*a, **k):
        raise AssertionError("device work before the argument checks")

    monkeypatch.setattr(pl, "StagedInput", no_device)
    monkeypatch.setattr(pl, "to_native", no_device)
    with pytest.raises(exc, match=msg):
        getattr(lb.feature, fn)(**kw)


@pytest.mark.parametrize("fn,kw", [("tempogram", dict(win_length=0)), ("tempogram", dict()),
                                   ("tempogram", dict(window=np.ones(3))), ("tempo", dict(start_bpm=0)),
                                   ("tempogram", dict(norm="fro"))])
def test_error_messages_match_oracle(fn, kw):
    env = None if fn == "tempogram" and not kw else _ENV
    with pytest.raises(lb.ParameterError) as got:
        getattr(lb.feature, fn)(onset_envelope=env, **kw)
    with pytest.raises(RO.ParameterError) as want:
        getattr(RO, fn)(onset_envelope=env, **kw)
    assert str(got.value) == str(want.value)


def test_public_names():
    assert lb.feature.tempogram is lb.feature.rhythm.tempogram
    for name in ("tempogram", "fourier_tempogram", "tempo"):
        assert name in lb.feature.__all__
    for name in ("tempo_frequencies", "fourier_tempo_frequencies"):
        assert name in lb.__all__ and name in lb.core.__all__
