"""``librosa.onset.onset_strength`` / ``onset_strength_multi`` with librosa's signatures (reference:
librosa/onset.py:217-367 and :445-640).  ``y=`` inputs run melspectrogram (the fused FFT kernel) and
power_to_db on the device and feed the log-mel block straight to the spectral-flux kernel; only the
``(..., channels, frames)`` envelope ever leaves the GPU."""
from __future__ import annotations

import ctypes as C
import numpy as np

from . import _native as nat
from . import _pipeline as pl
from .core.spectrum import power_to_db
from .util.exceptions import ParameterError
from .util.utils import is_positive_int

_vp = C.c_void_p

__all__ = ["onset_strength", "onset_strength_multi"]

MAX_MEDIAN_ROWS = 512   # csrc/feat_kernels.cuh kOnsetMedMaxRows: rows of one channel under np.median


def _edges(channels, n_rows: int, pad: bool):
    """Row boundaries of the aggregation channels (util.sync -> index_to_slice -> fix_frames)."""
    if all(isinstance(c, slice) for c in channels):
        spans = [c.indices(n_rows) for c in channels]
        if any(st != 1 for _, _, st in spans) or any(spans[i][1] != spans[i + 1][0] for i in range(len(spans) - 1)):
            raise nat.UnsupportedOnGPU("onset channels must be contiguous unit-stride row ranges on the GPU")
        return [spans[0][0]] + [b for _, b, _ in spans]
    if not all(np.issubdtype(type(c), np.integer) for c in channels):
        raise ParameterError(f"Invalid index set: {channels}")
    frames = np.asarray(channels)
    if np.any(frames < 0):
        raise ParameterError("Negative frame index detected")
    if pad:
        frames = np.concatenate((np.asarray([0, n_rows]), np.clip(frames, 0, n_rows)))
    frames = frames[(frames >= 0) & (frames <= n_rows)]
    return [int(v) for v in np.unique(frames)]


def onset_strength_multi(*, y=None, sr: float = 22050, S=None, n_fft: int = 2048, hop_length: int = 512, lag: int = 1,
                         max_size: int = 1, ref=None, detrend: bool = False, center: bool = True, feature=None,
                         aggregate=None, channels=None, **kwargs):
    """Spectral-flux onset strength over sub-bands, shape ``(..., n_channels, frames)``; same contract as
    ``librosa.onset.onset_strength_multi`` for the default ``feature`` (mel) and mean or median aggregation
    (``np.mean`` / ``np.median``; channels of up to 512 rows under the median), or ``aggregate=False`` for the
    per-bin flux."""
    from .feature.spectral import melspectrogram

    if feature is not None and feature is not melspectrogram:
        raise nat.UnsupportedOnGPU("a custom `feature` callable cannot run on the GPU (no CPU fallback)")
    if S is None:
        kwargs.setdefault("fmax", 0.5 * sr)
    if aggregate is None:
        aggregate = np.mean
    if callable(aggregate) and aggregate is not np.mean and aggregate is not np.median:
        raise nat.UnsupportedOnGPU("only mean or median aggregation (or aggregate=False) is computed on the GPU")
    if not is_positive_int(lag):
        raise ParameterError(f"lag={lag} must be a positive integer")
    if not is_positive_int(max_size):
        raise ParameterError(f"max_size={max_size} must be a positive integer")
    if ref is not None:
        raise nat.UnsupportedOnGPU("a caller-supplied reference spectrum is not supported on the GPU")
    if aggregate is np.median:   # the kernel's channel limit, known from the shapes before any device work
        n_rows = kwargs.get("n_mels", 128) if S is None else (S.shape[-2] if np.ndim(S) >= 2 else 1)
        edges = _edges([slice(None)] if channels is None else list(channels), n_rows, channels is None)
        widest = max((b - a for a, b in zip(edges[:-1], edges[1:])), default=0)
        if widest > MAX_MEDIAN_ROWS:
            raise nat.UnsupportedOnGPU(f"median onset aggregation over a channel of {widest} rows: the GPU kernel takes "
                                       f"up to {MAX_MEDIAN_ROWS} (no CPU fallback)")

    staged = None
    if S is None:
        if y is None:
            raise ParameterError("Input signal must be provided to compute a spectrogram")
        _, req = pl.precheck_signal(y)
        # one upload, every intermediate on the device; the mel frames are always centred (``center`` only
        # sets the pad width below)
        staged = pl.StagedInput(y)
        mel = melspectrogram(y=staged.dev, sr=sr, n_fft=n_fft, hop_length=hop_length, **kwargs)
        staged.scan_uncovered(n_fft, hop_length, kwargs.get("win_length"), True, mel.shape[-1])
        Sd = power_to_db(mel)
        mel.free()
        res_dtype = np.dtype(req)
    else:
        if not isinstance(S, nat.DeviceArray):
            S = np.atleast_2d(np.asarray(S))
        Sd, res_dtype, on_device = pl.spectrogram_input(S)
        if Sd.layout != "c":
            raise ParameterError("device spectrogram must be C-ordered (..., rows, frames)")
    if Sd.ndim < 2:
        raise ParameterError("spectrogram input must have at least two dimensions")
    rows, T = Sd.shape[-2], Sd.shape[-1]
    if T <= lag:
        raise ParameterError(f"lag={lag} needs more than {T} frames")
    ctx = Sd.ctx
    lead = Sd.shape[:-2]
    desc = nat.OnsetDesc(lag=int(lag), max_size=int(max_size), detrend=int(bool(detrend)),
                         pad_width=int(lag) + (n_fft // (2 * hop_length) if center else 0))
    if callable(aggregate):
        edges = _edges([slice(None)] if channels is None else list(channels), rows, channels is None)
        if len(edges) - 1 > 32:
            raise nat.UnsupportedOnGPU("at most 32 onset channels are supported on the GPU")
        desc.n_channels = len(edges) - 1
        for i, e in enumerate(edges):
            desc.bounds[i] = e
        n_out = len(edges) - 1
    else:
        desc.n_channels = 0
        n_out = rows
    out = nat.DeviceArray.empty(ctx, tuple(lead) + (n_out, T), np.float32)
    entry = nat.lib().b2l_onset_median_from_spec if aggregate is np.median else nat.lib().b2l_onset_from_spec
    nat.check(entry(ctx.handle, C.byref(desc), _vp(Sd.ptr), pl.clip_count(lead), rows, T, _vp(out.ptr)))
    if staged is not None or not on_device:
        Sd.free()
    if detrend:   # scipy.signal.lfilter with float64 coefficients returns float64
        res_dtype = np.result_type(res_dtype, np.float64)
    if staged is not None:
        return staged.result(out, res_dtype)
    return out if on_device else pl.finish(out, res_dtype)


def onset_strength(*, y=None, sr: float = 22050, S=None, lag: int = 1, max_size: int = 1, ref=None,
                   detrend: bool = False, center: bool = True, feature=None, aggregate=None, **kwargs):
    """Spectral-flux onset strength envelope, shape ``(..., frames)``; same contract as
    ``librosa.onset.onset_strength``."""
    if aggregate is False:
        raise ParameterError("aggregate parameter cannot be False when computing full-spectrum onset strength.")
    odf = onset_strength_multi(y=y, sr=sr, S=S, lag=lag, max_size=max_size, ref=ref, detrend=detrend, center=center,
                               feature=feature, aggregate=aggregate, channels=None, **kwargs)
    if isinstance(odf, nat.DeviceArray):
        # (..., 1, T) -> (..., T): same memory without the unit axis; the view keeps the owner alive
        view = nat.DeviceArray(odf.ctx, odf.ptr, odf.shape[:-2] + odf.shape[-1:], odf.dtype, layout="c", owner=False)
        view._base = odf
        return view
    return odf[..., 0, :]
