"""Window and filter-bank construction (host side, float64) — mirror of the hot-path parts of
librosa/filters.py: ``mel`` (:117-251), ``get_window`` (:915-977), ``window_sumsquare`` (:1268-1339), and the
constant-Q wavelet basis: ``wavelet_lengths`` (:424-552), ``_relative_bandwidth`` (:555-585), ``wavelet``
(:589-733), ``window_bandwidth`` (:865-912), and the multirate semitone filter bank of ``iirt``:
``mr_frequencies`` (:1075-1117) and ``semitone_filterbank`` (:1120-1230).

These constants are tiny and parity-critical, so they are computed on the host with the same float64
expressions as the reference and uploaded once per plan; the GPU only *applies* them.
"""
from __future__ import annotations

import warnings

import numpy as np
import scipy.signal

from .core.convert import fft_frequencies, hz_to_octs, mel_frequencies
from .util.exceptions import ParameterError
from .util.utils import normalize, pad_center


def get_window(window, Nx: int, *, fftbins: bool = True) -> np.ndarray:
    """Resolve a window specification to an array of length ``Nx`` (librosa/filters.py:961-977)."""
    if callable(window):
        return window(Nx)
    if isinstance(window, (str, tuple)) or np.isscalar(window):
        return scipy.signal.get_window(window, Nx, fftbins=fftbins)
    if isinstance(window, (np.ndarray, list)):
        if len(window) == Nx:
            return np.asarray(window)
        raise ParameterError(f"Window size mismatch: {len(window):d} != {Nx:d}")
    raise ParameterError(f"Invalid window specification: {window!r}")


def mel(*, sr: float, n_fft: int, n_mels: int = 128, fmin: float = 0.0, fmax=None, htk: bool = False,
        norm="slaney", dtype=np.float32) -> np.ndarray:
    """Triangular mel filter bank, shape ``(n_mels, 1 + n_fft//2)`` (librosa/filters.py:206-251)."""
    if fmax is None:
        fmax = float(sr) / 2
    n_mels = int(n_mels)
    weights = np.zeros((n_mels, int(1 + n_fft // 2)), dtype=dtype)
    bin_hz = fft_frequencies(sr=sr, n_fft=n_fft)
    edges = mel_frequencies(n_mels + 2, fmin=fmin, fmax=fmax, htk=htk)
    widths = np.diff(edges)
    offsets = np.subtract.outer(edges, bin_hz)
    for i in range(n_mels):
        up = -offsets[i] / widths[i]
        down = offsets[i + 2] / widths[i + 1]
        weights[i] = np.maximum(0, np.minimum(up, down))
    if isinstance(norm, str):
        if norm != "slaney":
            raise ParameterError(f"Unsupported norm={norm}")
        weights *= (2.0 / (edges[2 : n_mels + 2] - edges[:n_mels]))[:, np.newaxis]
    else:
        weights = normalize(weights, norm=norm, axis=-1)
    if not np.all((edges[:-2] == 0) | (weights.max(axis=1) > 0)):
        warnings.warn(
            "Empty filters detected in mel frequency basis. "
            "Some channels will produce empty responses. "
            "Try increasing your sampling rate (and fmax) or "
            "reducing n_mels.",
            stacklevel=2,
        )
    return weights


def window_sumsquare(*, window, n_frames: int, hop_length: int = 512, win_length=None, n_fft: int = 2048,
                     dtype=np.float32, norm=None) -> np.ndarray:
    """Sum of squared, hop-shifted windows, length ``n_fft + hop*(n_frames-1)``
    (librosa/filters.py:1325-1339; the fill loop of :1258-1265 is vectorised per frame)."""
    if win_length is None:
        win_length = n_fft
    n = n_fft + hop_length * (n_frames - 1)
    x = np.zeros(n, dtype=dtype)
    win_sq = get_window(window, win_length)
    win_sq = normalize(win_sq, norm=norm) ** 2
    win_sq = pad_center(win_sq, size=n_fft)
    for i in range(n_frames):
        s = i * hop_length
        x[s : min(n, s + n_fft)] += win_sq[: max(0, min(n_fft, n - s))]
    return x


def chroma(*, sr: float, n_fft: int, n_chroma: int = 12, tuning: float = 0.0, ctroct: float = 5.0, octwidth=2,
           norm=2, base_c: bool = True, dtype=np.float32) -> np.ndarray:
    """Chroma filter bank ``(n_chroma, 1 + n_fft/2)`` projecting FFT bins onto pitch classes; host-side
    constant with the values of ``librosa.filters.chroma`` (filters.py:254-392): Gaussian bumps around each
    bin's pitch class, column-normalised, optionally weighted by a Gaussian over octaves."""
    # position of every FFT bin (DC excluded) on the chroma axis, in bins
    bin_hz = np.linspace(0, sr, n_fft, endpoint=False)[1:]
    pos = n_chroma * hz_to_octs(bin_hz, tuning=tuning, bins_per_octave=n_chroma)
    # the 0 Hz bin gets a made-up position 1.5 octaves below bin 1
    pos = np.concatenate(([pos[0] - 1.5 * n_chroma], pos))
    width = np.concatenate((np.maximum(pos[1:] - pos[:-1], 1.0), [1]))
    half = np.round(float(n_chroma) / 2)
    # signed distance of every bin to every pitch class, wrapped to [-n_chroma/2, n_chroma/2)
    dist = np.subtract.outer(pos, np.arange(0, n_chroma, dtype="d")).T
    dist = np.remainder(dist + half + 10 * n_chroma, n_chroma) - half
    wts = np.exp(-0.5 * (2 * dist / np.tile(width, (n_chroma, 1))) ** 2)
    wts = normalize(wts, norm=norm, axis=0)
    if octwidth is not None:
        wts *= np.exp(-0.5 * (((pos / n_chroma - ctroct) / octwidth) ** 2))[np.newaxis, :]
    if base_c:
        wts = np.roll(wts, -3 * (n_chroma // 12), axis=0)
    return np.ascontiguousarray(wts[:, : int(1 + n_fft / 2)], dtype=dtype)


_ENBW_POINTS = 8193   # window_bandwidth's tabulated values are the ENBW of the symmetric 8193-point window
_ENBW_UNREPRODUCED = ("flattop", "flat", "flt")


def window_bandwidth(window, n: int = 1000) -> float:
    """Equivalent noise bandwidth ``n * sum(w**2) / sum(w)**2`` of a window (librosa/filters.py:865-912).

    Named windows use the symmetric 8193-point window, which reproduces librosa's tabulated value exactly for
    "hann" (the constant-Q default), "ones", "boxcar", "triangle", "bartlett", "cosine", "parzen", "bohman" and
    "barthann", and within 1e-15 relative for "hamming", "blackman", "blackmanharris" and "nuttall".  librosa's
    value for "flattop" is not the ENBW of SciPy's flat-top window (2.78 against 3.77), so it raises
    ``UnsupportedOnGPU`` rather than move the cutoff of the wavelet basis.  Other specifications use
    ``get_window(window, n)`` as librosa does."""
    if isinstance(window, str) and window in _ENBW_UNREPRODUCED:
        from ._native import UnsupportedOnGPU

        raise UnsupportedOnGPU(f"window_bandwidth({window!r}): librosa's tabulated bandwidth of this window is not "
                               "reproduced here; use another window")
    if isinstance(window, str):
        try:
            w = scipy.signal.get_window(window, _ENBW_POINTS, fftbins=False)
        except ValueError:
            w = None
        if w is not None:
            return float(_ENBW_POINTS * np.sum(w ** 2) / (np.sum(w) ** 2))
    w = get_window(window, n)
    return float(n * np.sum(w ** 2) / (np.sum(w) ** 2 + np.finfo(np.asarray(w).dtype).tiny))


def _relative_bandwidth(*, freqs: np.ndarray) -> np.ndarray:
    """Relative bandwidth alpha of each frequency from its neighbours on a log2 axis (librosa/filters.py:555-585)."""
    if len(freqs) <= 1:
        raise ParameterError(f"2 or more frequencies are required to compute bandwidths. Given freqs={freqs}")
    logf = np.log2(freqs)
    bpo = np.empty_like(freqs)
    bpo[0] = 1 / (logf[1] - logf[0])
    bpo[-1] = 1 / (logf[-1] - logf[-2])
    bpo[1:-1] = 2 / (logf[2:] - logf[:-2])
    return (2.0 ** (2 / bpo) - 1) / (2.0 ** (2 / bpo) + 1)


def wavelet_lengths(*, freqs, sr: float = 22050, window="hann", filter_scale: float = 1, gamma=0, alpha=None):
    """Filter lengths of a wavelet basis and the cutoff frequency of its top filter (librosa/filters.py:424-552)."""
    freqs = np.asarray(freqs)
    if filter_scale <= 0:
        raise ParameterError(f"filter_scale={filter_scale} must be positive")
    if gamma is not None and gamma < 0:
        raise ParameterError(f"gamma={gamma} must be non-negative")
    if np.any(freqs <= 0):
        raise ParameterError("frequencies must be strictly positive")
    if len(freqs) > 1 and np.any(freqs[:-1] > freqs[1:]):
        raise ParameterError(f"Frequency array={freqs} must be in strictly ascending order")
    alpha = _relative_bandwidth(freqs=freqs) if alpha is None else np.asarray(alpha)
    offset = alpha * 24.7 / 0.108 if gamma is None else gamma     # ERB-proportional bandwidth offset for None
    Q = float(filter_scale) / alpha
    f_cutoff = max(freqs * (1 + 0.5 * window_bandwidth(window) / Q) + 0.5 * offset)
    return Q * sr / (freqs + offset / alpha), f_cutoff


def _fractional_window(window, n: float) -> np.ndarray:
    """``ceil(n)`` samples: the window of ``floor(n)`` samples, zero from sample ``floor(n)`` on."""
    lo, hi = int(np.floor(n)), int(np.ceil(n))
    w = get_window(window, lo)
    if len(w) < hi:
        w = np.pad(w, [(0, hi - len(w))], mode="constant")
    w[lo:] = 0.0
    return w


def wavelet(*, freqs: np.ndarray, sr: float = 22050, window="hann", filter_scale: float = 1, pad_fft: bool = True,
            norm=1, dtype=np.complex64, gamma=0, alpha=None, **kwargs):
    """Windowed complex sinusoids at ``freqs``, centred in rows of a common length (a power of two when ``pad_fft``),
    and their fractional lengths (librosa/filters.py:589-733)."""
    lengths, _ = wavelet_lengths(freqs=freqs, sr=sr, window=window, filter_scale=filter_scale, gamma=gamma,
                                 alpha=alpha)
    rows = []
    for ilen, freq in zip(lengths, freqs, strict=True):
        phase = np.arange(-ilen // 2, ilen // 2, dtype=float) * 2 * np.pi * freq / sr
        sig = np.cos(phase) + 1j * np.sin(phase)
        sig *= _fractional_window(window, len(sig))
        rows.append(normalize(sig, norm=norm))
    size = max(lengths)
    size = int(2.0 ** (np.ceil(np.log2(size)))) if pad_fft else int(np.ceil(size))
    return np.asarray([pad_center(r, size=size, **kwargs) for r in rows], dtype=dtype), lengths


def _hz_to_midi(frequencies):
    """MIDI note number of a frequency (librosa/core/convert.py:913-940)."""
    return (12 * (np.log2(np.asanyarray(frequencies)) - np.log2(440.0)) + 69)[()]


def cq_to_chroma(n_input: int, *, bins_per_octave: int = 12, n_chroma: int = 12, fmin=None, window=None,
                 base_c: bool = True, dtype=np.float32) -> np.ndarray:
    """Map of constant-Q bins onto chroma bins, shape ``(n_chroma, n_input)`` (librosa/filters.py:737-861): the
    identity tiled ``bins_per_octave / n_chroma`` times, rolled to centre on each target bin, repeated over the
    octaves, rolled so that the first chroma bin is C (A when not ``base_c``), then convolved with ``window`` when
    one is given (float64 then).  ``fmin`` None is C1."""
    n_merge = float(bins_per_octave) / n_chroma
    if fmin is None:
        fmin = 440.0 * (2.0 ** ((np.asanyarray(24) - 69.0) / 12.0))   # note_to_hz("C1")
    if np.mod(n_merge, 1) != 0:
        raise ParameterError("Incompatible CQ merge: input bins must be an integer multiple of output bins.")
    cq_to_ch = np.repeat(np.eye(n_chroma), int(n_merge), axis=1)
    cq_to_ch = np.roll(cq_to_ch, -int(n_merge // 2), axis=1)
    n_octaves = np.ceil(float(n_input) / bins_per_octave)
    cq_to_ch = np.tile(cq_to_ch, int(n_octaves))[:, :n_input]
    midi_0 = np.mod(_hz_to_midi(fmin), 12)
    roll = midi_0 if base_c else midi_0 - 9
    roll = int(np.round(roll * (n_chroma / 12.0)))
    cq_to_ch = np.roll(cq_to_ch, roll, axis=0).astype(dtype)
    if window is not None:
        cq_to_ch = scipy.signal.convolve(cq_to_ch, np.atleast_2d(window), mode="same")
    return cq_to_ch


def _multirate_fb(center_freqs=None, sample_rates=None, Q: float = 25.0, passband_ripple: float = 1,
                  stopband_attenuation: float = 50, ftype: str = "ellip", flayout: str = "sos"):
    """One ``scipy.signal.iirdesign`` band-pass per centre frequency (librosa/filters.py:981-1072): passband centre
    +- bw/2, stopband centre +- bw, bw = centre / Q, edges relative to each band's Nyquist rate."""
    if center_freqs is None:
        raise ParameterError("center_freqs must be provided.")
    if sample_rates is None:
        raise ParameterError("sample_rates must be provided.")
    if center_freqs.shape != sample_rates.shape:
        raise ParameterError("Number of provided center_freqs and sample_rates must be equal.")
    nyquist = 0.5 * sample_rates
    bandwidths = center_freqs / float(Q)
    bank = []
    for f0, nyq, bw in zip(center_freqs, nyquist, bandwidths, strict=True):
        wp = [f0 - 0.5 * bw, f0 + 0.5 * bw] / nyq
        ws = [f0 - bw, f0 + bw] / nyq
        bank.append(scipy.signal.iirdesign(wp, ws, passband_ripple, stopband_attenuation, analog=False, ftype=ftype,
                                           output=flayout))
    return bank, sample_rates


def mr_frequencies(tuning: float):
    """Centre frequencies of MIDI pitches 24 .. 108 (shifted by ``tuning`` semitones) and the rate each band runs at:
    36 at 882 Hz, 34 at 4 410 Hz, 15 at 22 050 Hz (librosa/filters.py:1075-1117)."""
    notes = np.arange(24 + tuning, 109 + tuning)
    center_freqs = 440.0 * (2.0 ** ((np.asanyarray(notes)[()] - 69.0) / 12.0))
    sample_rates = np.asarray(36 * [882.0] + 34 * [4410.0] + 15 * [22050.0])
    return center_freqs, sample_rates


def semitone_filterbank(*, center_freqs=None, tuning: float = 0.0, sample_rates=None, flayout: str = "ba", **kwargs):
    """Multirate IIR band-pass filter bank (librosa/filters.py:1120-1230): ``mr_frequencies(tuning)`` unless
    centre frequencies or rates are given; ``kwargs`` (Q, passband_ripple, stopband_attenuation, ftype) go to the
    design.  Returns (one filter per band in ``flayout``, the rate of each band)."""
    if center_freqs is None and sample_rates is None:
        center_freqs, sample_rates = mr_frequencies(tuning)
    return _multirate_fb(center_freqs=center_freqs, sample_rates=sample_rates, flayout=flayout, **kwargs)
