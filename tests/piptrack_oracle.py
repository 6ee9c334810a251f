"""NumPy restatement of librosa.piptrack, pitch_tuning and util.localmax / localmin in the reference's exact roundings;
reproduces every entry of tests/golden/piptrack_v1.npz bit for bit.

It differs from oracle/ref_np.py in one place, the parabolic-interpolation stencil.  The reference's numba stencil
evaluates ``a = x[1] + x[-1] - 2 * x[0]`` and ``b = (x[1] - x[-1]) / 2`` with the two sums in the data type but the
product ``2 * x[0]``, the subtraction and the division by 2 promoted to float64, and rounds the shift to the data type
once when it is stored.  ref_np computes the whole formula in float32 for float32 data."""
from __future__ import annotations

import warnings

import numpy as np


def fft_frequencies(sr, n_fft):
    return np.fft.rfftfreq(n=n_fft, d=1.0 / sr)


def parabolic_shift(S):
    """The reference's _parabolic_interpolation along axis -2, with its float64 stencil."""
    xi = np.swapaxes(S, -1, -2)
    l, c, r = xi[..., :-2], xi[..., 1:-1], xi[..., 2:]
    a = (r + l).astype(np.float64) - 2.0 * c.astype(np.float64)
    b = (r - l).astype(np.float64) / 2.0
    with np.errstate(divide="ignore", invalid="ignore"):
        inner = np.where(np.abs(b) >= np.abs(a), 0.0, -b / a)
    shifts = np.zeros_like(xi)
    shifts[..., 1:-1] = inner
    return np.swapaxes(shifts, -1, -2)


def localmax(x, axis=0):
    xi = np.swapaxes(np.asarray(x), -1, axis)
    out = np.zeros(xi.shape, dtype=bool)
    out[..., 1:-1] = (xi[..., 1:-1] > xi[..., :-2]) & (xi[..., 1:-1] >= xi[..., 2:])
    out[..., -1] = xi[..., -1] > xi[..., -2]
    return np.swapaxes(out, -1, axis)


def localmin(x, axis=0):
    xi = np.swapaxes(np.asarray(x), -1, axis)
    out = np.zeros(xi.shape, dtype=bool)
    out[..., 1:-1] = (xi[..., 1:-1] < xi[..., :-2]) & (xi[..., 1:-1] <= xi[..., 2:])
    out[..., -1] = xi[..., -1] < xi[..., -2]
    return np.swapaxes(out, -1, axis)


class util:   # the namespace piptrack_cases.call looks the peak test up in
    localmax = staticmethod(localmax)
    localmin = staticmethod(localmin)


def piptrack(*, y=None, sr=22050, S=None, n_fft=2048, hop_length=None, fmin=150.0, fmax=4000.0, threshold=0.1,
             win_length=None, window="hann", center=True, pad_mode="constant", ref=None):
    """From ``S`` only: a ``y`` case is run on the spectrogram of whichever STFT is under test (``spectrogram``)."""
    if S is None:
        raise ValueError("the oracle takes S; compute the spectrogram of y first")
    if n_fft is None or n_fft // 2 + 1 != S.shape[-2]:
        n_fft = 2 * (S.shape[-2] - 1)
    if np.iscomplexobj(S) or S.min() < 0:
        S = np.abs(S)
    fmin = np.maximum(fmin, 0)
    fmax = np.minimum(fmax, float(sr) / 2)
    fft_freqs = fft_frequencies(sr, n_fft)
    avg = np.gradient(S, axis=-2)
    shift = parabolic_shift(S)
    dskew = 0.5 * avg * shift
    pitches = np.zeros_like(S)
    mags = np.zeros_like(S)
    freq_mask = (fmin <= fft_freqs) & (fft_freqs < fmax)
    freq_mask = freq_mask.reshape((1,) * (S.ndim - 2) + (-1, 1))
    if ref is None:
        ref = np.max
    if callable(ref):
        ref_value = np.expand_dims(threshold * ref(S, axis=-2), -2)
    else:
        ref_value = np.abs(ref)
    with np.errstate(invalid="ignore"):
        idx = np.nonzero(freq_mask & localmax(S * (S > ref_value), axis=-2))
    pitches[idx] = (idx[-2] + shift[idx]) * float(sr) / n_fft
    mags[idx] = S[idx] + dskew[idx]
    return pitches, mags


def spectrogram(magnitude, y, *, n_fft=2048, hop_length=None, win_length=None, window="hann", center=True,
                pad_mode="constant", **_):
    """The magnitude spectrogram of y with piptrack's STFT arguments, from a ``magnitude(y, **stft_args)`` under
    test."""
    return np.asarray(magnitude(y, n_fft=n_fft, hop_length=hop_length, win_length=win_length, window=window,
                                center=center, pad_mode=pad_mode))


def residuals(frequencies, bins_per_octave=12):
    """pitch_tuning's folded residuals of the values > 0, in the data's precision."""
    f = np.atleast_1d(frequencies)
    f = f[f > 0]
    with np.errstate(invalid="ignore"):
        r = np.mod(bins_per_octave * np.log2(f / 27.5), 1.0)
        r[r >= 0.5] -= 1.0
    return r


def pitch_tuning(frequencies, *, resolution=0.01, bins_per_octave=12):
    frequencies = np.atleast_1d(frequencies)
    frequencies = frequencies[frequencies > 0]
    if not np.any(frequencies):
        warnings.warn("Trying to estimate tuning from empty frequency set.", stacklevel=2)
        return 0.0
    residual = residuals(frequencies, bins_per_octave)
    bins = np.linspace(-0.5, 0.5, int(np.ceil(1.0 / resolution)) + 1)
    counts, tuning = np.histogram(residual, bins)
    return tuning[np.argmax(counts)]
