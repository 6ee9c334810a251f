"""Frequency-scale conversions feeding ``filters.mel`` (host side, float64).

Mirrors librosa/core/convert.py: hz_to_mel (:1004-1058), mel_to_hz (:1069-1121),
mel_frequencies (:1432-1508), fft_frequencies (:1369), tempo_frequencies (:1514-1548) and
fourier_tempo_frequencies (:1551-1579).
"""
from __future__ import annotations

import numpy as np

# Slaney (Auditory Toolbox) mel scale: linear below 1 kHz, logarithmic above
_F_SP = 200.0 / 3
_BREAK_HZ = 1000.0
_BREAK_MEL = _BREAK_HZ / _F_SP
_LOGSTEP = np.log(6.4) / 27.0


def hz_to_mel(frequencies, *, htk: bool = False):
    f = np.asanyarray(frequencies)[()]
    if htk:
        return 2595.0 * np.log10(1.0 + f / 700.0)
    if np.ndim(f):
        f = np.asarray(f, dtype=float)
        mels = f / _F_SP
        hi = f >= _BREAK_HZ
        mels[hi] = _BREAK_MEL + np.log(f[hi] / _BREAK_HZ) / _LOGSTEP
        return mels
    if f >= _BREAK_HZ:
        return _BREAK_MEL + np.log(f / _BREAK_HZ) / _LOGSTEP
    return f / _F_SP


def mel_to_hz(mels, *, htk: bool = False):
    m = np.asanyarray(mels)[()]
    if htk:
        return 700.0 * (10.0 ** (m / 2595.0) - 1.0)
    if np.ndim(m):
        m = np.asarray(m, dtype=float)
        freqs = _F_SP * m
        hi = m >= _BREAK_MEL
        freqs[hi] = _BREAK_HZ * np.exp(_LOGSTEP * (m[hi] - _BREAK_MEL))
        return freqs
    if m >= _BREAK_MEL:
        return _BREAK_HZ * np.exp(_LOGSTEP * (m - _BREAK_MEL))
    return _F_SP * m


def mel_frequencies(n_mels: int = 128, *, fmin: float = 0.0, fmax: float = 11025.0, htk: bool = False):
    lo = hz_to_mel(fmin, htk=htk)
    hi = hz_to_mel(fmax, htk=htk)
    return mel_to_hz(np.linspace(lo, hi, n_mels), htk=htk)


def fft_frequencies(*, sr: float = 22050, n_fft: int = 2048):
    return np.fft.rfftfreq(n=n_fft, d=1.0 / sr)


def hz_to_octs(frequencies, *, tuning: float = 0.0, bins_per_octave: int = 12):
    """Octave number of each frequency relative to A0 = A440 / 16 (mirror of core/convert.py:hz_to_octs)."""
    a440 = 440.0 * 2.0 ** (tuning / bins_per_octave)
    octs = np.log2(np.asanyarray(frequencies) / (float(a440) / 16))
    return octs[()]


def tempo_frequencies(n_bins: int, *, hop_length: int = 512, sr: float = 22050):
    """BPM of each lag of a tempogram: lag k spans k * hop_length / sr seconds; the zero lag is ``inf``."""
    bpm = np.empty(int(n_bins), dtype=np.float64)
    bpm[0] = np.inf                    # an IndexError for n_bins < 1, like the reference's
    bpm[1:] = 60.0 * sr / (hop_length * np.arange(1.0, n_bins))
    return bpm


def fourier_tempo_frequencies(*, sr: float = 22050, win_length: int = 384, hop_length: int = 512):
    """BPM of each bin of a Fourier tempogram."""
    return fft_frequencies(sr=sr * 60 / float(hop_length), n_fft=win_length)


def frames_to_samples(frames, *, hop_length: int = 512, n_fft=None):
    """Sample index of each frame index (plus ``n_fft // 2`` when ``n_fft`` is given), as integers."""
    offset = 0 if n_fft is None else int(n_fft // 2)
    return (np.asanyarray(frames) * hop_length + offset).astype(int)[()]


def samples_to_time(samples, *, sr: float = 22050):
    """Time in seconds of each sample index."""
    return np.asanyarray(samples)[()] / float(sr)


def frames_to_time(frames, *, sr: float = 22050, hop_length: int = 512, n_fft=None):
    """Time in seconds of each frame index: ``frames_to_samples`` then ``samples_to_time``."""
    return samples_to_time(frames_to_samples(frames, hop_length=hop_length, n_fft=n_fft), sr=sr)
