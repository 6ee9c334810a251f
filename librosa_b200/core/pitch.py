"""``librosa.estimate_tuning`` (reference: librosa/core/pitch.py:28-109, on top of ``piptrack`` :182-366 and
``pitch_tuning`` :112-179), as needed by ``feature.chroma_stft``.

The peak picking and parabolic interpolation of ``piptrack`` run on the GPU over the whole spectrogram; the
peak list is never materialised.  The median magnitude that gates the peaks is found exactly by radix selection
over three histogram passes, the tuning by one residual-histogram pass; the host only reads those histograms."""
from __future__ import annotations

import ctypes as C
import warnings
from typing import Optional

import numpy as np

from .. import _native as nat
from .. import _pipeline as pl
from ..util.exceptions import ParameterError
from .convert import fft_frequencies

_vp = C.c_void_p


def _key_to_float(key: int) -> np.float32:
    """Inverse of the order-preserving uint32 key of a float32 (csrc/common.cuh float_to_key)."""
    u = (key & 0x7FFFFFFF) if key & 0x80000000 else (~key & 0xFFFFFFFF)
    return np.array([u], dtype=np.uint32).view(np.float32)[0]


def _tuning_from_device_spec(ctx, Sd, sr, n_fft, *, resolution, bins_per_octave, fmin, fmax, threshold, ref):
    """Sd: float32 DeviceArray (..., bins, frames), any layout.  Returns the tuning estimate (float)."""
    F, T = Sd.shape[-2], Sd.shape[-1]
    L = nat.lib()
    src, own = pl.to_native(Sd)
    freqs = fft_frequencies(sr=sr, n_fft=n_fft)
    fmin = np.maximum(fmin, 0)
    fmax = np.minimum(fmax, float(sr) / 2)
    mask = np.flatnonzero((fmin <= freqs) & (freqs < fmax))
    desc = nat.PipDesc(k_lo=int(mask[0]) if mask.size else 0, k_hi=int(mask[-1]) + 1 if mask.size else 0,
                       threshold=float(threshold), ref_abs=-1.0, hz_per_bin=float(sr) / n_fft,
                       bins_per_octave=float(bins_per_octave))
    if ref is not None and ref is not np.max:
        if callable(ref):
            raise nat.UnsupportedOnGPU("piptrack(ref=callable) other than np.max is not supported on the GPU")
        desc.ref_abs = float(np.abs(ref))
    rows = pl.clip_count(Sd.shape[:-2]) * T
    hist = (C.c_uint64 * 2048)()

    def run(mode, prefix=0, mag_threshold=0.0, edges=None, n_res=0):
        desc.mode, desc.prefix, desc.mag_threshold, desc.n_res_bins = mode, prefix, float(mag_threshold), n_res
        e = edges.ctypes.data_as(_vp) if edges is not None else None
        nat.check(L.b2l_pip_pass(ctx.handle, C.byref(desc), _vp(src.ptr), rows, F, e, hist))
        n = n_res if mode == 3 else (1024 if mode == 2 else 2048)
        return np.frombuffer(hist, dtype=np.uint64, count=n).astype(np.int64)

    h0 = run(0)
    n_peaks = int(h0.sum())
    try:
        if n_peaks == 0:
            warnings.warn("Trying to estimate tuning from empty frequency set.", stacklevel=3)
            return 0.0

        def select(rank):
            """float32 value of the peak magnitude with this 0-based rank (ascending)."""
            c0 = np.cumsum(h0)
            b0 = int(np.searchsorted(c0, rank, side="right"))
            r = rank - (int(c0[b0 - 1]) if b0 else 0)
            c1 = np.cumsum(run(1, prefix=b0))
            b1 = int(np.searchsorted(c1, r, side="right"))
            r -= int(c1[b1 - 1]) if b1 else 0
            c2 = np.cumsum(run(2, prefix=(b0 << 11) | b1))
            b2 = int(np.searchsorted(c2, r, side="right"))
            return _key_to_float((b0 << 21) | (b1 << 10) | b2)

        if n_peaks % 2:
            med = select((n_peaks - 1) // 2)
        else:
            lo, hi = select(n_peaks // 2 - 1), select(n_peaks // 2)
            med = np.float32(np.float32(lo + hi) / np.float32(2.0))      # np.median -> mean of the two middles
        edges = np.linspace(-0.5, 0.5, int(np.ceil(1.0 / resolution)) + 1)
        if len(edges) - 1 > 2048:
            raise nat.UnsupportedOnGPU("tuning resolution finer than 1/2048 is not supported on the GPU")
        counts = run(3, mag_threshold=med, edges=np.ascontiguousarray(edges, dtype=np.float64), n_res=len(edges) - 1)
        return edges[int(np.argmax(counts))]
    finally:
        if own:
            src.free()


def estimate_tuning(*, y=None, sr: float = 22050, S=None, n_fft: Optional[int] = 2048, resolution: float = 0.01,
                    bins_per_octave: int = 12, **kwargs):
    """Estimate the tuning deviation (fractions of a bin) of a signal or spectrogram; same contract as
    ``librosa.estimate_tuning`` (``kwargs`` go to ``piptrack``: hop_length, fmin, fmax, threshold, win_length,
    window, center, pad_mode, ref — ``ref`` a number or ``np.max``)."""
    from .spectrum import _spectrogram

    allowed = {"hop_length", "fmin", "fmax", "threshold", "win_length", "window", "center", "pad_mode", "ref"}
    extra = set(kwargs) - allowed
    if extra:
        raise TypeError(f"piptrack() got an unexpected keyword argument '{sorted(extra)[0]}'")
    pip = dict(fmin=kwargs.get("fmin", 150.0), fmax=kwargs.get("fmax", 4000.0), threshold=kwargs.get("threshold", 0.1),
               ref=kwargs.get("ref", None))
    staged = None
    if S is None:
        if y is None:
            raise ParameterError("Input signal must be provided to compute a spectrogram")
        pl.precheck_signal(y)
        staged = pl.StagedInput(y)
        Sd, n_fft = _spectrogram(y=staged.dev, n_fft=n_fft, hop_length=kwargs.get("hop_length"), power=1,
                                 win_length=kwargs.get("win_length"), window=kwargs.get("window", "hann"),
                                 center=kwargs.get("center", True), pad_mode=kwargs.get("pad_mode", "constant"))
        own = True
        staged.scan_uncovered(n_fft, kwargs.get("hop_length"), kwargs.get("win_length"), kwargs.get("center", True),
                              Sd.shape[-1])
    else:
        if not isinstance(S, nat.DeviceArray) and np.iscomplexobj(S):
            S = np.abs(S)
        Sd, _, on_device = pl.spectrogram_input(S)
        own = not on_device
        if n_fft is None or n_fft // 2 + 1 != Sd.shape[-2]:
            n_fft = 2 * (Sd.shape[-2] - 1)
    try:
        est = _tuning_from_device_spec(Sd.ctx, Sd, sr, n_fft, resolution=resolution, bins_per_octave=bins_per_octave,
                                       **pip)
    finally:
        if own:
            Sd.free()
    if staged is not None:
        staged.check_finite()
    return est
