"""``librosa.beat.beat_track`` and ``librosa.beat.plp`` (reference: librosa/beat.py:44-317, :320-507, tracker
:510-742).

The dynamic-programming tracker runs in one kernel launch, one CTA per clip (csrc/beat_kernels.cuh).  It is
discrete — one rounding difference moves a beat — so it restates the reference's numba arithmetic step by step, and
every transcendental it needs comes from tables built here with the C library's ``log`` / ``logf`` / ``exp``, which
is what numba calls (NumPy's vectorised ``log`` and ``exp`` differ from them in the last bit on some arguments).
Without ``bpm`` the tempo comes from the GPU ``feature.tempo``; with ``y=`` the envelope is the device's median
``onset_strength``, and it never leaves the GPU.

``plp`` is the Fourier tempogram (``stft`` at hop 1), one select launch per call that keeps each frame's peak bin and
normalises its phase, the ``istft`` at hop 1 and one launch for the clip and ``util.normalize``."""
from __future__ import annotations

import ctypes as C
import ctypes.util
import functools
import math

import numpy as np

from . import _native as nat
from . import _pipeline as pl
from .util.exceptions import ParameterError

_vp = C.c_void_p

__all__ = ["beat_track", "plp"]

MAX_FRAMES_PER_BEAT = 1 << 24   # fpb is cast to float32 for float32 envelopes: exact integers only
_UNITS = {"frames": nat.BEAT_FRAMES, "samples": nat.BEAT_SAMPLES, "time": nat.BEAT_TIME}

_libm = None


def _logf(x: float) -> float:
    """The C library's single-precision log (numba's np.log of a float32)."""
    global _libm
    if _libm is None:
        lib = C.CDLL(ctypes.util.find_library("m") or "libm.so.6")
        lib.logf.restype = C.c_float
        lib.logf.argtypes = [C.c_float]
        _libm = lib
    return float(_libm.logf(x))


@functools.lru_cache(maxsize=512)
def window(fpb: int, half: int) -> np.ndarray:
    """w(d) = exp(-0.5 * x * x), x = d * 32.0 / fpb, for d = -half .. half (the local-score window's centre)."""
    f = float(fpb)
    out = np.empty(2 * half + 1)
    for i, d in enumerate(range(-half, half + 1)):
        x = float(d) * 32.0 / f
        out[i] = math.exp(-0.5 * (x * x))
    return out


@functools.lru_cache(maxsize=64)
def log_table(top: int) -> np.ndarray:
    """log(d) for d = 0 .. top (entry 0 is unused)."""
    return np.array([0.0] + [math.log(d) for d in range(1, top + 1)])


def log_fpb(fpb: int, f64: bool) -> float:
    """np.log(frames_per_beat) as the tracker's DP evaluates it: float64 log, or float32 logf in the float32 DP."""
    return math.log(float(fpb)) if f64 else _logf(float(fpb))


def frames_per_beat(bpm, sr, hop_length, env_shape):
    """``np.atleast_1d(bpm)`` expanded like ``util.expand_to(..., axes=range(bpm.ndim))``, and the frame rate."""
    _bpm = np.atleast_1d(bpm)
    if _bpm.ndim > len(env_shape):
        raise ParameterError(f"bpm of shape {_bpm.shape} has more dimensions than the onset envelope {env_shape}")
    bpm_expanded = _bpm.reshape(_bpm.shape + (1,) * (len(env_shape) - _bpm.ndim))
    return bpm_expanded, float(sr) / hop_length


def _check_tracker_args(bpm_expanded, frame_rate, tightness, env_shape):
    """The reference's bpm / tightness / shape checks in its order, then ``np.round(frame_rate * 60 / bpm)`` and the
    GPU's own limits; returns frames per beat broadcast to ``lead + (1 or n,)`` (as float64) and whether they were
    float64 (the DP's precision: numba runs the float64 loop unless the envelope and fpb are both float32)."""
    if np.any(bpm_expanded <= 0):
        raise ParameterError(f"bpm={bpm_expanded} must be strictly positive")
    if tightness <= 0:
        raise ParameterError("tightness must be strictly positive")
    if bpm_expanded.shape[-1] not in (1, env_shape[-1]):
        raise ParameterError(f"Invalid bpm shape={bpm_expanded.shape} does not match "
                             f"onset envelope shape={env_shape}")
    fpb = np.round(frame_rate * 60.0 / bpm_expanded)
    if not np.all(np.isfinite(fpb)) or np.any(fpb > MAX_FRAMES_PER_BEAT):
        raise nat.UnsupportedOnGPU(f"beat_track: frames per beat above {MAX_FRAMES_PER_BEAT} (bpm too small for the "
                                   "frame rate) are not supported on the GPU")
    if np.any(fpb < 1):
        raise nat.UnsupportedOnGPU(f"beat_track: bpm above 120 x the frame rate ({120 * frame_rate:g}) rounds to 0 "
                                   "frames per beat, which the GPU tracker does not support")
    lead = tuple(env_shape[:-1])
    return np.ascontiguousarray(np.broadcast_to(fpb, lead + (fpb.shape[-1],)), dtype=np.float64), fpb.dtype == np.float64


def host_tables(fpb: np.ndarray, n: int, f64: bool):
    """(per-clip table [3][n_clips * n_fpb] = fpb, log fpb, window centre; window table; log table)."""
    flat = fpb.reshape(-1)
    uniq, inv = np.unique(flat, return_inverse=True)
    pieces, centres, offset = [], [], 0
    for f in uniq:
        half = min(int(f), n - 1)
        pieces.append(window(int(f), half))
        centres.append(offset + half)
        offset += 2 * half + 1
    logs = np.array([log_fpb(int(f), f64) for f in uniq])
    per_clip = np.concatenate([flat, logs[inv.reshape(-1)], np.asarray(centres, dtype=np.float64)[inv.reshape(-1)]])
    return per_clip, np.concatenate(pieces), log_table(max(1, min(2 * int(uniq.max()), n - 1)))


def _launch(ctx, x, fpb, fpb_f64, *, tightness, trim, units=None, hop_length=512, sr=22050.0, stages=None):
    """One launch of the tracker on the device envelope ``x`` (..., n).  Returns the dense beats (DeviceArray of
    bool) and, with ``units``, the compacted list and its count.  ``stages``: a dict that receives the
    localscore / cumscore / backlink DeviceArrays."""
    n, f64 = x.shape[-1], x.dtype == np.float64
    dp64 = f64 or fpb_f64
    per_clip, wtab, logd = host_tables(fpb, n, dp64)
    d_clip = ctx.to_device(per_clip)
    m = per_clip.size // 3
    d_wtab = pl.f64_constant(ctx, ("beat_window", pl.digest(wtab)), wtab)
    d_logd = pl.f64_constant(ctx, ("beat_log", logd.size), logd)
    desc = nat.BeatDesc(n_fpb=int(fpb.shape[-1]), env_f64=int(f64), dp_f64=int(dp64), trim=int(bool(trim)),
                        units=_UNITS.get(units, 0), tightness=float(np.float32(tightness)),
                        hop_length=int(hop_length), sr=float(sr), d_fpb=d_clip.ptr, d_logfpb=d_clip.ptr + 8 * m,
                        d_woff=d_clip.ptr + 16 * m, d_wtab=d_wtab, d_logd=d_logd)
    beats = nat.DeviceArray.empty(ctx, x.shape, np.bool_)
    ptrs = [None, None, None]
    if stages is not None:
        stages["localscore"] = nat.DeviceArray.empty(ctx, x.shape, x.dtype)
        stages["cumscore"] = nat.DeviceArray.empty(ctx, x.shape, np.float64 if dp64 else np.float32)
        stages["backlink"] = nat.DeviceArray.empty(ctx, x.shape, np.int32)
        ptrs = [_vp(stages[k].ptr) for k in ("localscore", "cumscore", "backlink")]
    lst = count = None
    if units is not None:
        lst = nat.DeviceArray.empty(ctx, (n,), np.float64 if units == "time" else np.int64)
        count = nat.DeviceArray.empty(ctx, (1,), np.int64)
    nat.check(nat.lib().b2l_beat_track(ctx.handle, C.byref(desc), _vp(x.ptr), pl.clip_count(x.shape[:-1]), n, *ptrs,
                                       _vp(beats.ptr), _vp(lst.ptr) if lst else None,
                                       _vp(count.ptr) if count else None))
    d_clip.free()
    return beats, lst, count


def _any_nonzero(x: nat.DeviceArray) -> bool:
    flag = nat.DeviceArray.empty(x.ctx, (1,), np.int32)
    nat.check(nat.lib().b2l_any_nonzero(x.ctx.handle, _vp(x.ptr), x.size, int(x.dtype == np.float64), _vp(flag.ptr)))
    return bool(flag.get()[0])


def _zeros(ctx, shape, dtype):
    out = nat.DeviceArray.empty(ctx, shape, dtype)
    if out.nbytes:
        nat.check(nat.lib().b2l_memset(ctx.handle, _vp(out.ptr), 0, out.nbytes))
    return out


def beat_track(*, y=None, sr: float = 22050, onset_envelope=None, hop_length: int = 512, start_bpm: float = 120.0,
               tightness: float = 100, trim: bool = True, bpm=None, prior=None, units: str = "frames",
               sparse: bool = True):
    """Dynamic-programming beat tracker; same contract as ``librosa.beat.beat_track``.

    Returns ``(bpm, beats)``: ``bpm`` as passed, else ``feature.tempo``'s ``(..., 1)`` estimate; ``beats`` the beat
    positions in ``units`` (``sparse=True``, one-dimensional envelopes only) or a dense bool ``(..., n)``.  Host
    inputs give NumPy arrays, DeviceArray inputs give DeviceArrays.  float32 and float64 envelopes use the
    reference's float32 and float64 tracker arithmetic; a ``y=`` envelope is float32."""
    from .feature.rhythm import _Envelope, tempo

    if onset_envelope is None:
        if y is None:
            raise ParameterError("y or onset_envelope must be provided")
        pl.precheck_signal(y)
    elif isinstance(onset_envelope, nat.DeviceArray):
        if onset_envelope.dtype not in (np.float32, np.float64) or onset_envelope.layout != "c":
            raise ParameterError("device onset envelope must be a C-ordered float32 or float64 DeviceArray")
    elif np.asarray(onset_envelope).dtype not in (np.float32, np.float64):
        raise nat.UnsupportedOnGPU("onset_envelope must be float32 or float64 on the GPU")
    env = _Envelope(y, sr, onset_envelope, hop_length, aggregate=np.median)
    try:
        env.verdict()
        x, ctx, on_device = env.dev, env.ctx, env.on_device
        if sparse and x.ndim != 1:
            raise ParameterError(f"sparse=True (default) does not support "
                                 f"{x.ndim}-dimensional inputs. "
                                 f"Either set sparse=False or convert the signal to mono.")
        if onset_envelope is not None and not on_device:
            nonzero = bool(np.asarray(onset_envelope).any())
        else:
            nonzero = _any_nonzero(x)
        if not nonzero:
            if sparse:
                return 0.0, (nat.DeviceArray.empty(ctx, (0,), np.int64) if on_device else np.array([], dtype=int))
            if on_device:
                return _zeros(ctx, x.shape[:-1], np.float64), _zeros(ctx, x.shape, np.bool_)
            return np.zeros(shape=x.shape[:-1], dtype=float), np.zeros(x.shape, dtype=bool)
        if bpm is None:
            bpm = tempo(onset_envelope=x, sr=sr, hop_length=hop_length, start_bpm=start_bpm, prior=prior)
            bpm_host = bpm.get()   # 8 bytes per clip: the host builds the tracker's tables
            if not on_device:
                bpm = bpm_host
        else:
            bpm_host = bpm.get() if isinstance(bpm, nat.DeviceArray) else bpm
        bpm_expanded, frame_rate = frames_per_beat(bpm_host, sr, hop_length, x.shape)
        fpb, fpb_f64 = _check_tracker_args(bpm_expanded, frame_rate, tightness, x.shape)
        if sparse and units not in _UNITS:
            raise ParameterError(f"Invalid unit type: {units}")
        dense, lst, count = _launch(ctx, x, fpb, fpb_f64, tightness=tightness, trim=trim, units=units if sparse else None,
                                    hop_length=hop_length, sr=sr)
    finally:
        env.release()
    if not sparse:
        return bpm, (dense if on_device else dense.get())
    dense.free()
    k = int(count.get()[0])
    if on_device:
        view = nat.DeviceArray(ctx, lst.ptr, (k,), lst.dtype, layout="c", owner=False)
        view._base = lst
        return bpm, view
    return bpm, lst.get()[:k].copy()


def track_stages(onset_envelope, *, bpm, sr: float = 22050, hop_length: int = 512, tightness: float = 100,
                 trim: bool = True):
    """The tracker's intermediates for a host envelope and tempo (testing aid): a dict of NumPy arrays
    ``localscore``, ``cumscore``, ``backlink`` and the dense ``beats``."""
    x_host = np.ascontiguousarray(onset_envelope)
    ctx = nat.default_context()
    x = ctx.to_device(x_host)
    bpm_expanded, frame_rate = frames_per_beat(bpm, sr, hop_length, x.shape)
    fpb, fpb_f64 = _check_tracker_args(bpm_expanded, frame_rate, tightness, x.shape)
    stages = {}
    dense, _, _ = _launch(ctx, x, fpb, fpb_f64, tightness=tightness, trim=trim, stages=stages)
    out = {k: v.get() for k, v in stages.items()}
    out["beats"] = dense.get()
    return out



def select_peaks(ft: nat.DeviceArray, keep: np.ndarray, logprior=None):
    """plp's step 3 in place on a device Fourier tempogram (..., bins, frames) in layout "ft": one launch.
    ``keep``: bool per bin (the tempo range); ``logprior``: float64 per bin or None."""
    ctx = ft.ctx
    if ft.layout != "ft" or ft.dtype not in (np.complex64, np.complex128):
        raise ParameterError("the Fourier tempogram must be a complex DeviceArray in layout 'ft'")
    c128 = ft.dtype == np.complex128
    keep64 = np.ascontiguousarray(keep, dtype=np.float64)
    d_keep = pl.f64_constant(ctx, ("plp_keep", pl.digest(keep64)), keep64)
    d_prior = None if logprior is None else pl.f64_constant(ctx, ("plp_prior", pl.digest(logprior)), logprior)
    tiny = np.finfo(np.float64 if c128 else np.float32).tiny
    desc = nat.PlpDesc(n_bins=int(ft.shape[-2]), c128=int(c128), sqrt_tiny=float(tiny ** 0.5), d_keep=d_keep,
                       d_logprior=d_prior)
    nat.check(nat.lib().b2l_plp_select(ctx.handle, C.byref(desc), _vp(ft.ptr),
                                       pl.clip_count(ft.shape[:-2]) * ft.shape[-1]))


def plp(*, y=None, sr: float = 22050, onset_envelope=None, hop_length: int = 512, win_length: int = 384,
        tempo_min=30, tempo_max=300, prior=None):
    """Predominant local pulse; same contract as ``librosa.beat.plp``.

    Returns the pulse ``(..., n)`` in the envelope's dtype: a NumPy array for host input, a DeviceArray for device
    input.  ``prior`` is any object with ``logpdf`` (a scipy.stats distribution)."""
    from .core.convert import fourier_tempo_frequencies
    from .core.spectrum import istft
    from .feature.rhythm import _Envelope, fourier_tempogram

    if onset_envelope is None:
        if y is None:
            raise ParameterError("Input signal must be provided to compute a spectrogram")
        pl.precheck_signal(y)
    elif isinstance(onset_envelope, nat.DeviceArray):
        if onset_envelope.dtype not in (np.float32, np.float64) or onset_envelope.layout != "c":
            raise ParameterError("device onset envelope must be a C-ordered float32 or float64 DeviceArray")
    elif np.asarray(onset_envelope).dtype not in (np.float32, np.float64):
        raise nat.UnsupportedOnGPU("onset_envelope must be float32 or float64 on the GPU")
    if tempo_min is not None and tempo_max is not None and tempo_max <= tempo_min:
        raise ParameterError(f"tempo_max={tempo_max} must be larger than tempo_min={tempo_min}")
    freqs = fourier_tempo_frequencies(sr=sr, hop_length=hop_length, win_length=win_length)
    keep = np.ones(freqs.shape, dtype=bool)
    if tempo_min is not None:
        keep &= ~(freqs < tempo_min)
    if tempo_max is not None:
        keep &= ~(freqs > tempo_max)
    logprior = None if prior is None else np.ascontiguousarray(prior.logpdf(freqs), dtype=np.float64)
    env = _Envelope(y, sr, onset_envelope, hop_length, aggregate=np.median)
    try:
        env.verdict()
        x, ctx = env.dev, env.ctx
        ft = fourier_tempogram(onset_envelope=x, sr=sr, hop_length=hop_length, win_length=win_length)
    finally:
        env.release()
    select_peaks(ft, keep, logprior)
    n = x.shape[-1]
    pulse = istft(ft, hop_length=1, n_fft=win_length, length=n)
    ft.free()
    nat.check(nat.lib().b2l_plp_finish(ctx.handle, _vp(pulse.ptr), pl.clip_count(pulse.shape[:-1]), n,
                                       int(pulse.dtype == np.float64)))
    if pl.status_word(ctx) & 4:
        pulse.free()
        raise ParameterError("Input must be finite")
    return pulse if env.on_device else pl.finish(pulse)
