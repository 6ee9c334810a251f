"""GPU: a call that fails after it has staged or allocated device buffers gives them all back to the context's pool
before the exception reaches the caller, even while the caller keeps the exception and its traceback alive (the
frames of the failed call then still reference every buffer they held).  A successful griffinlim keeps nothing
either."""
import gc
import warnings

import numpy as np
import pytest

from librosa_b200._native import UnsupportedOnGPU
from librosa_b200.util.exceptions import ParameterError

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def lb():
    import librosa_b200

    librosa_b200.default_context()
    return librosa_b200


def _outstanding(ctx):
    """Device blocks of the context that are handed out, not back in its size-keyed pool."""
    return len(ctx._sizes) - sum(len(bucket) for bucket in ctx._pool.values())


def _y(n=4096):
    return (0.1 * np.random.default_rng(1).standard_normal(n)).astype(np.float32)


def _mag(shape):
    return np.abs(np.random.default_rng(2).standard_normal(shape)).astype(np.float32)


# (call, exception, message): each fails after its device work has begun
FAILING = {
    "spectral_contrast past Nyquist": (lambda lb: lb.feature.spectral_contrast(y=_y(), sr=22050, fmin=8000.0),
                                       ParameterError, "exceeds Nyquist"),
    "pcen zi shape": (lambda lb: lb.pcen(_mag((2, 16, 40)), zi=np.zeros(3)), ValueError, "zi has shape"),
    "chroma_stft norm": (lambda lb: lb.feature.chroma_stft(y=_y(), sr=22050, norm="bad"), ParameterError,
                         "Unsupported norm"),
    "time_stretch one frame": (lambda lb: lb.effects.time_stretch(_y(256), rate=1.5, n_fft=256, hop_length=64,
                                                                  center=False), UnsupportedOnGPU, "two frames"),
    "griffinlim length": (lambda lb: lb.griffinlim(_mag((129, 10)), n_iter=2, length=100), ParameterError,
                          "length=100"),
    "spectral statistics of a 1-D S": (lambda lb: lb.feature.spectral_centroid(S=_mag(129)), ParameterError,
                                       "at least two dimensions"),
}


def _settled(lb, call):
    """The outstanding blocks once ``call`` has run (so that the plans, constant tables and pool blocks of its shapes
    exist) and every reference it left has gone."""
    call()
    gc.collect()
    return _outstanding(lb.default_context())


@pytest.mark.parametrize("name", sorted(FAILING))
def test_failed_call_releases_its_buffers(lb, name):
    call, exc, match = FAILING[name]

    def failing():
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            with pytest.raises(exc, match=match) as excinfo:
                call(lb)
        return excinfo

    base = _settled(lb, failing)
    gc.disable()   # only reference counting frees: the traceback kept below must not pin anything
    try:
        excinfo = failing()
        assert _outstanding(lb.default_context()) == base, excinfo.traceback[-1]
    finally:
        gc.enable()


def test_griffinlim_keeps_nothing(lb):
    S = _mag((2, 129, 20))

    def run():
        return lb.griffinlim(S, n_iter=3, n_fft=256)

    base = _settled(lb, run)
    gc.disable()
    try:
        y = run()
        assert y.shape == (2, 64 * 19) and _outstanding(lb.default_context()) == base
    finally:
        gc.enable()
