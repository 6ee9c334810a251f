"""The I/O edge of the hot path (SURVEY 8f rank 4): ``librosa.stream``'s block semantics for in-memory audio.

``librosa.stream`` (librosa/core/audio.py:223-500) reads a sound file in blocks that line up with STFT frames:
a block holds ``block_length`` frames, i.e. ``(block_length - 1) * hop_length + frame_length`` samples, and
consecutive blocks advance by ``block_length * hop_length`` samples (they overlap by ``frame_length - hop_length``),
so that ``stft(block, center=False)`` over the blocks concatenates to ``stft(y, center=False)`` of the whole signal.
Decoding audio files and resampling (soundfile / soxr) are outside the path and outside this repository; this
module provides the same block walk over an array that is already in memory (or a ``DeviceArray``), which is
what a decoder thread would feed.
"""
from __future__ import annotations

import ctypes as C
import math
from functools import lru_cache
from typing import Iterator, Optional

import numpy as np

from .. import _native as nat
from .. import _pipeline as pl
from ..util.exceptions import ParameterError
from ..util.utils import is_positive_int

__all__ = ["stream", "resample"]


def stream(y, *, block_length: int, frame_length: int, hop_length: int, mono: bool = True, offset: float = 0.0,
           duration: Optional[float] = None, fill_value: Optional[float] = None, sr: Optional[float] = None,
           dtype=np.float32) -> Iterator[np.ndarray]:
    """Yield blocks of ``block_length`` frames of an in-memory signal ``y`` (shape ``(n,)`` or ``(channels, n)``).

    Same arguments and block geometry as ``librosa.stream`` (audio.py:385-500), with the file replaced by an
    array: ``offset`` / ``duration`` are in seconds when ``sr`` is given and in samples otherwise; the last block
    is shorter than the others unless ``fill_value`` is given.  A path (``str`` / ``os.PathLike``) is refused:
    audio decoding is not part of the GPU path and there is no CPU fallback."""
    if not is_positive_int(block_length):
        raise ParameterError(f"block_length={block_length} must be a positive integer")
    if not is_positive_int(frame_length):
        raise ParameterError(f"frame_length={frame_length} must be a positive integer")
    if not is_positive_int(hop_length):
        raise ParameterError(f"hop_length={hop_length} must be a positive integer")
    if sr is not None and not (np.isfinite(sr) and sr > 0):
        raise ParameterError(f"sr={sr} must be a positive number")
    if isinstance(y, (str, bytes)) or hasattr(y, "__fspath__"):
        raise nat.UnsupportedOnGPU("stream: decoding audio files (soundfile / soxr) is outside the GPU path; pass the "
                                   "decoded samples as an array")
    if isinstance(y, nat.DeviceArray):
        raise nat.UnsupportedOnGPU("stream: slice the DeviceArray's host source instead (blocks are host views)")
    y = np.asarray(y)
    if y.ndim not in (1, 2):
        raise ParameterError(f"stream expects a (n,) or (channels, n) array, got shape {y.shape}")
    if mono and y.ndim == 2:
        y = np.mean(y, axis=0)
    scale = float(sr) if sr is not None else 1.0
    n = y.shape[-1]
    start = int(offset * scale) if offset >= 0 else max(0, n - int(abs(offset) * scale))
    stop = n if duration is None else min(n, start + int(duration * scale))
    size = (block_length - 1) * hop_length + frame_length
    advance = block_length * hop_length
    pos = start
    while pos < stop:
        block = y[..., pos: min(pos + size, stop)]
        if block.shape[-1] < size and fill_value is not None:
            pad = [(0, 0)] * (block.ndim - 1) + [(0, size - block.shape[-1])]
            block = np.pad(block, pad, mode="constant", constant_values=fill_value)
        yield np.ascontiguousarray(block, dtype=dtype)
        if pos + size >= stop:
            break
        pos += advance


# --------------------------------------------------------------------------------------------- resampling
@lru_cache(maxsize=32)
def _poly_filter(up: int, down: int):
    """The low-pass scipy.signal.resample_poly designs for float32 data, zero padded as it pads it, and the crop
    positions of its upfirdn output (scipy/signal/_signaltools.py, resample_poly): returns (h float32, n_pre_remove)."""
    import scipy.signal

    max_rate = max(up, down)
    half_len = 10 * max_rate
    h = scipy.signal.firwin(2 * half_len + 1, 1.0 / max_rate, window=("kaiser", 5.0)).astype(np.float32)
    h *= up
    n_pre_pad = down - half_len % down
    n_pre_remove = (half_len + n_pre_pad) // down
    h = np.concatenate((np.zeros(n_pre_pad, dtype=h.dtype), h))
    return h, n_pre_remove


def resample(y, *, orig_sr: float, target_sr: float, res_type: str = "soxr_hq", fix: bool = True, scale: bool = False,
             axis: int = -1, **kwargs):
    """Resample ``y`` from ``orig_sr`` to ``target_sr``; same contract as ``librosa.resample``
    (librosa/core/audio.py:1002-1179) for ``res_type="polyphase"`` — scipy.signal.resample_poly's zero-phase FIR,
    integer rates only — which runs as one kernel (``b2l_resample_poly``).  librosa's default ``soxr_hq`` and the
    resampy / samplerate / FFT resamplers are third-party algorithms with no oracle here: they raise
    ``UnsupportedOnGPU`` (there is no CPU fallback), so pass ``res_type="polyphase"`` explicitly."""
    if isinstance(y, nat.DeviceArray):
        n, req = y.shape[-1], np.dtype(np.float32)
        if y.dtype != np.float32 or y.layout != "c":
            raise ParameterError("device input must be a C-ordered float32 DeviceArray")
    else:
        n, req = pl.precheck_signal(y)            # util.valid_audio's host checks (audio.py:1116)
    if orig_sr == target_sr:
        return y
    if res_type != "polyphase":
        raise nat.UnsupportedOnGPU(f"resample(res_type={res_type!r}): only the 'polyphase' resampler runs on the GPU "
                                   "(soxr / resampy / samplerate / FFT resamplers are not part of this library)")
    if axis not in (-1, getattr(y, "ndim", 1) - 1):
        raise nat.UnsupportedOnGPU("resample: only the last axis can be resampled on the GPU")
    if kwargs:
        raise nat.UnsupportedOnGPU("resample: np.pad keyword arguments for fix_length are not supported on the GPU")
    ratio = float(target_sr) / orig_sr
    n_samples = int(np.ceil(n * ratio))
    if int(orig_sr) != orig_sr or int(target_sr) != target_sr:
        raise ParameterError("polyphase resampling is only supported for integer-valued sampling rates.")
    g = math.gcd(int(orig_sr), int(target_sr))
    up, down = int(target_sr) // g, int(orig_sr) // g
    h, n_pre_remove = _poly_filter(up, down)
    n_out = (n * up + down - 1) // down                       # resample_poly's own output length
    n_total = n_samples if fix else n_out
    with pl.Scope(y) as sc:
        staged = pl.StagedInput(y)
        staged.scan_all()
        d_h = sc.stage(h)
        out = sc.empty(tuple(staged.lead) + (n_total,), np.float32)
        nat.check(nat.lib().b2l_resample_poly(sc.ctx.handle, C.c_void_p(staged.dev.ptr), staged.n_clips, n, n,
                                              C.c_void_p(d_h.ptr), len(h), up, down, n_pre_remove, min(n_out, n_total),
                                              n_total, float(1.0 / np.sqrt(ratio)) if scale else 1.0,
                                              C.c_void_p(out.ptr)))
        staged.release()
        return sc.result(out, req, validate=True)
