"""NumPy / SciPy statement of the rhythm features the GPU implements: tempogram, fourier_tempogram, tempo and the
pieces they are made of (linear-ramp padding, autocorrelation, util.normalize, the tempo-axis converters).

Written from librosa's documented behaviour (librosa/feature/rhythm.py:38-470, util/utils.py normalize,
core/audio.py autocorrelate, core/convert.py tempo_frequencies / fourier_tempo_frequencies); it must reproduce
tests/golden/rhythm_v1.npz bit for bit.  It lives next to the tests because the existing ``oracle/`` module is left
unchanged."""
from __future__ import annotations

import numpy as np
import scipy.fft
import scipy.signal

from librosa_b200.util.exceptions import ParameterError

from oracle import ref_np as O


# --------------------------------------------------------------------------------------------- converters
def tempo_frequencies(n_bins, *, hop_length=512, sr=22050):
    """BPM of lag k: 60 sr / (hop_length k); the zero lag is +inf."""
    out = np.empty(int(n_bins), dtype=np.float64)
    out[0] = np.inf
    out[1:] = 60.0 * sr / (hop_length * np.arange(1.0, n_bins))
    return out


def fourier_tempo_frequencies(*, sr=22050, win_length=384, hop_length=512):
    """The rfft bin frequencies of a win_length-point transform at the onset rate, in BPM."""
    return np.fft.rfftfreq(n=win_length, d=1.0 / (sr * 60 / float(hop_length)))


def time_to_frames(seconds, *, sr=22050, hop_length=512):
    samples = (np.asanyarray(seconds) * sr).astype(int)
    return np.floor(samples // hop_length).astype(int)


# --------------------------------------------------------------------------------------------- pieces
def linear_ramp_pad(x, p):
    """np.pad of the last axis by p on both sides, ramping linearly to 0."""
    widths = [(0, 0)] * (x.ndim - 1) + [(p, p)]
    return np.pad(x, widths, mode="linear_ramp", end_values=0)


def autocorrelate(y, max_size=None, axis=-1):
    """Linear autocorrelation through a zero-padded real FFT (scipy's next fast length), first max_size lags."""
    n = y.shape[axis]
    if max_size is None:
        max_size = n
    n_pad = scipy.fft.next_fast_len(2 * n - 1, real=True)
    spec = scipy.fft.rfft(y, n=n_pad, axis=axis)
    power = spec.real ** 2 + spec.imag ** 2
    ac = scipy.fft.irfft(power, n=n_pad, axis=axis)
    return np.take(ac, np.arange(min(max_size, n_pad)), axis=axis)


def normalize(S, *, norm=np.inf, axis=0):
    """util.normalize with threshold tiny(S) and fill=None: divide by the norm unless it is below the threshold."""
    if not np.all(np.isfinite(S)):
        raise ParameterError("Input must be finite")
    mag = np.abs(S).astype(float)
    if norm is None:
        return S
    if norm == np.inf:
        length = np.max(mag, axis=axis, keepdims=True)
    elif norm == -np.inf:
        length = np.min(mag, axis=axis, keepdims=True)
    elif norm == 0:
        length = np.sum(mag > 0, axis=axis, keepdims=True, dtype=mag.dtype)
    elif np.issubdtype(type(norm), np.number) and norm > 0:
        length = np.sum(mag ** norm, axis=axis, keepdims=True) ** (1.0 / norm)
    else:
        raise ParameterError(f"Unsupported norm: {norm!r}")
    length[length < np.finfo(S.dtype).tiny] = 1.0
    out = np.empty_like(S)
    out[:] = S / length
    return out


def _window(window, n):
    if callable(window):
        return window(n)
    if isinstance(window, (str, tuple)) or np.isscalar(window):
        return scipy.signal.get_window(window, n, fftbins=True)
    w = np.asarray(window)
    if len(w) != n:
        raise ParameterError(f"Window size mismatch: {len(w):d} != {n:d}")
    return w


def frames(x, win_length):
    """(..., n) -> (..., win_length, n - win_length + 1): hop-1 frames along a new second-to-last axis."""
    if x.shape[-1] < win_length:
        raise ParameterError(f"Input is too short (n={x.shape[-1]:d}) for frame_length={win_length:d}")
    return np.swapaxes(np.lib.stride_tricks.sliding_window_view(x, win_length, axis=-1), -1, -2)


# --------------------------------------------------------------------------------------------- features
def tempogram(*, y=None, sr=22050, onset_envelope=None, hop_length=512, win_length=384, center=True, window="hann",
              norm=np.inf):
    if win_length < 1:
        raise ParameterError("win_length must be a positive integer")
    w = _window(window, win_length)
    if onset_envelope is None:
        if y is None:
            raise ParameterError("Either y or onset_envelope must be provided")
        onset_envelope = O.onset_strength(y=y, sr=sr, hop_length=hop_length)
    n = onset_envelope.shape[-1]
    x = linear_ramp_pad(onset_envelope, win_length // 2) if center else onset_envelope
    fr = frames(x, win_length)
    if center:
        fr = fr[..., :n]
    return normalize(autocorrelate(fr * w[:, np.newaxis], axis=-2), norm=norm, axis=-2)


def fourier_tempogram(*, y=None, sr=22050, onset_envelope=None, hop_length=512, win_length=384, center=True,
                      window="hann"):
    if win_length < 1:
        raise ParameterError("win_length must be a positive integer")
    if onset_envelope is None:
        if y is None:
            raise ParameterError("Either y or onset_envelope must be provided")
        onset_envelope = O.onset_strength(y=y, sr=sr, hop_length=hop_length)
    return O.stft(onset_envelope, n_fft=win_length, hop_length=1, center=center, window=window)


def log_prior(bpms, *, start_bpm=120, std_bpm=1.0, max_tempo=320.0, prior=None):
    """The log prior over the lag BPMs, -inf from the zero lag up to the first BPM below max_tempo."""
    if prior is None:
        lp = -0.5 * ((np.log2(bpms) - np.log2(start_bpm)) / std_bpm) ** 2
    else:
        lp = prior.logpdf(bpms)
    if max_tempo is not None:
        lp[: int(np.argmax(bpms < max_tempo))] = -np.inf
    return lp


def tempo_scores(tg, logprior):
    """log1p(1e6 tg) + logprior along the lag axis (-2), in the tempogram's precision then float64."""
    return np.log1p(1e6 * tg) + logprior[:, np.newaxis]


def tempo(*, y=None, sr=22050, onset_envelope=None, tg=None, hop_length=512, start_bpm=120, std_bpm=1.0, ac_size=8.0,
          max_tempo=320.0, aggregate=np.mean, prior=None):
    if start_bpm <= 0:
        raise ParameterError("start_bpm must be strictly positive")
    if tg is None:
        win_length = time_to_frames(ac_size, sr=sr, hop_length=hop_length).item()
        tg = tempogram(y=y, sr=sr, onset_envelope=onset_envelope, hop_length=hop_length, win_length=win_length)
    else:
        win_length = tg.shape[-2]
    if aggregate is not None:
        tg = aggregate(tg, axis=-1, keepdims=True)
    bpms = tempo_frequencies(win_length, hop_length=hop_length, sr=sr)
    lp = log_prior(bpms, start_bpm=start_bpm, std_bpm=std_bpm, max_tempo=max_tempo, prior=prior)
    return bpms[np.argmax(tempo_scores(tg, lp), axis=-2)]
