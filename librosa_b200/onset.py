"""``librosa.onset.onset_strength`` / ``onset_strength_multi``, ``onset_detect`` and ``onset_backtrack`` with
librosa's signatures (reference: librosa/onset.py:31-214, :217-367, :370-441 and :445-640).  ``y=`` inputs run
melspectrogram (the fused FFT kernel) and power_to_db on the device and feed the log-mel block straight to the
spectral-flux kernel; only the ``(..., channels, frames)`` envelope ever leaves the GPU.

``onset_detect`` is two launches on the envelope (csrc/onset_kernels.cuh): the normaliser, which also sets the call's
verdict flags (some value nonzero, some value not finite: the reference's ``.any()`` / ``isfinite`` test over the
whole array), and the peak picker, which reads those flags on the device; backtracking adds a third."""
from __future__ import annotations

import ctypes as C
import numpy as np

from . import _native as nat
from . import _pipeline as pl
from .core.spectrum import power_to_db
from .util.exceptions import ParameterError
from .util import peak as pk
from .util.utils import is_positive_int

_vp = C.c_void_p

__all__ = ["onset_strength", "onset_strength_multi", "onset_detect", "onset_backtrack"]

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

    with pl.Scope(y if S is None else S) as sc:
        if S is None:
            if y is None:
                raise ParameterError("Input signal must be provided to compute a spectrogram")
            _, req = pl.precheck_signal(y)
            # one upload, every intermediate on the device; the mel frames are always centred (``center`` only
            # sets the pad width below)
            staged = pl.StagedInput(y)
            mel = melspectrogram(y=staged.dev, sr=sr, n_fft=n_fft, hop_length=hop_length, **kwargs)
            staged.scan_uncovered(n_fft, hop_length, kwargs.get("win_length"), True, mel.shape[-1])
            Sd = sc.own(power_to_db(mel))
            mel.free()
            res_dtype = np.dtype(req)
        else:
            if not isinstance(S, nat.DeviceArray):
                S = np.atleast_2d(np.asarray(S))
            Sd, res_dtype = sc.spectrogram(S)
            if Sd.layout != "c":
                raise ParameterError("device spectrogram must be C-ordered (..., rows, frames)")
        if Sd.ndim < 2:
            raise ParameterError("spectrogram input must have at least two dimensions")
        rows, T = Sd.shape[-2], Sd.shape[-1]
        if T <= lag:
            raise ParameterError(f"lag={lag} needs more than {T} frames")
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
        out = sc.empty(tuple(lead) + (n_out, T), np.float32)
        entry = nat.lib().b2l_onset_median_from_spec if aggregate is np.median else nat.lib().b2l_onset_from_spec
        nat.check(entry(sc.ctx.handle, C.byref(desc), _vp(Sd.ptr), pl.clip_count(lead), rows, T, _vp(out.ptr)))
        if detrend:   # scipy.signal.lfilter with float64 coefficients returns float64
            res_dtype = np.result_type(res_dtype, np.float64)
        return sc.result(out, res_dtype, validate=S is None)


def onset_strength(*, y=None, sr: float = 22050, S=None, lag: int = 1, max_size: int = 1, ref=None,
                   detrend: bool = False, center: bool = True, feature=None, aggregate=None, **kwargs):
    """Spectral-flux onset strength envelope, shape ``(..., frames)``; same contract as
    ``librosa.onset.onset_strength``."""
    if aggregate is False:
        raise ParameterError("aggregate parameter cannot be False when computing full-spectrum onset strength.")
    odf = onset_strength_multi(y=y, sr=sr, S=S, lag=lag, max_size=max_size, ref=ref, detrend=detrend, center=center,
                               feature=feature, aggregate=aggregate, channels=None, **kwargs)
    if isinstance(odf, nat.DeviceArray):
        return odf.view(odf.shape[:-2] + odf.shape[-1:])   # (..., 1, T) -> (..., T)
    return odf[..., 0, :]


_EMPTY_MATCH = "Attempting to match empty event list"
_NEGATIVE_MATCH = "Cannot match events with right=False and min(events_to) > min(events_from)"
_PEAK_KEYS = ("pre_max", "post_max", "pre_avg", "post_avg", "delta", "wait", "method")


def _peak_kwargs(kwargs, sr, hop_length):
    """onset_detect's peak_pick arguments: the reference's defaults under the caller's keywords."""
    for k in kwargs:
        if k not in _PEAK_KEYS:
            raise TypeError(f"peak_pick() got an unexpected keyword argument '{k}'")
    kw = dict(kwargs)
    kw.setdefault("pre_max", 0.03 * sr // hop_length)
    kw.setdefault("post_max", 0.00 * sr // hop_length + 1)
    kw.setdefault("pre_avg", 0.10 * sr // hop_length)
    kw.setdefault("post_avg", 0.10 * sr // hop_length + 1)
    kw.setdefault("wait", 0.03 * sr // hop_length)
    kw.setdefault("delta", 0.07)
    return kw


def _host_verdict(x, normalize):
    """The reference's "any onsets to grab?" test on a host envelope."""
    if normalize:
        x = x - np.min(x, keepdims=True, axis=-1)
        x /= np.max(x, keepdims=True, axis=-1) + np.finfo(x.dtype).tiny
    return bool(x.any()) and bool(np.all(np.isfinite(x)))


def _empty(shape, sparse, units, ctx, on_device):
    """What onset_detect returns when there is nothing to pick."""
    if sparse:
        dtype = np.float64 if units == "time" else np.int64
        return nat.DeviceArray.empty(ctx, (0,), dtype) if on_device else np.array([], dtype=dtype)
    return ctx.zeros(shape, np.bool_) if on_device else np.zeros(shape, dtype=bool)


def _check_units(sparse, units):
    if sparse and units not in pk.UNITS:
        raise ParameterError(f"Invalid unit type: {units}")


def _normalize(sc, x, normalize):
    """One launch: the normalised envelope (None when ``normalize`` is off) and the verdict pair
    (int64 [2]: flags, pick count), owned by the scope ``sc``."""
    ctx = sc.ctx
    flags = sc.empty((2,), np.int64)
    norm = sc.empty(x.shape, x.dtype) if normalize else None
    nat.check(nat.lib().b2l_onset_normalize(ctx.handle, _vp(x.ptr), pl.clip_count(x.shape[:-1]), x.shape[-1],
                                            int(x.dtype == np.float64), float(np.finfo(x.dtype).tiny),
                                            _vp(norm.ptr) if norm is not None else None, _vp(flags.ptr)))
    return norm, flags


def _check_normalizable(shape, normalize):
    """The reference normalises with np.min over the frames, which has no identity for zero frames."""
    if normalize and len(shape) and shape[-1] == 0:
        raise ValueError("zero-size array to reduction operation minimum which has no identity")


def _passes(flags_host) -> bool:
    return bool(flags_host[0] & 1) and not flags_host[0] & 2


def _check_energy(energy):
    """The GPU's refusals for a backtracking energy, from its shape and dtype."""
    shape = energy.shape if isinstance(energy, nat.DeviceArray) else np.shape(energy)
    dtype = energy.dtype if isinstance(energy, nat.DeviceArray) else np.asarray(energy).dtype
    if len(shape) != 1:
        raise nat.UnsupportedOnGPU(f"onset_backtrack: energy of shape {tuple(shape)}; the GPU takes one-dimensional "
                                   "energy only")
    if dtype not in (np.float32, np.float64):
        raise nat.UnsupportedOnGPU(f"onset_backtrack: {dtype} energy is not supported on the GPU (float32 and float64 "
                                   "only)")
    if shape[0] > pk.MAX_FRAMES:
        raise nat.UnsupportedOnGPU("onset_backtrack: energy of 2^31 frames or more")
    if isinstance(energy, nat.DeviceArray) and energy.layout != "c":
        raise nat.UnsupportedOnGPU("onset_backtrack needs a C-ordered energy DeviceArray")


def _backtrack_launch(sc, energy, events, n_events, count, units, hop_length, sr):
    """One launch; returns the backtracked list (DeviceArray of n_events entries in ``units``, owned by ``sc``)."""
    ctx = sc.ctx
    out = sc.empty((n_events,), np.float64 if units == "time" else np.int64)
    nat.check(nat.lib().b2l_onset_backtrack(ctx.handle, _vp(energy.ptr), energy.shape[0],
                                            int(energy.dtype == np.float64), _vp(events.ptr), n_events,
                                            _vp(count.ptr) if count is not None else None, pk.UNITS[units],
                                            int(hop_length), float(sr), _vp(out.ptr)))
    return out


def onset_detect(*, y=None, sr: float = 22050, onset_envelope=None, hop_length: int = 512, backtrack: bool = False,
                 energy=None, units: str = "frames", normalize: bool = True, sparse: bool = True, **kwargs):
    """Locate note onset events by picking peaks in an onset strength envelope; same contract as
    ``librosa.onset.onset_detect``.

    Host input gives NumPy output, a DeviceArray envelope (or signal) gives DeviceArray output: the dense bool
    picks, or a view of the compacted list.  The envelope of ``y=`` is the device's float32 ``onset_strength``, also
    for float64 audio (the reference computes a float64 envelope there)."""
    from .feature.rhythm import _Envelope

    if onset_envelope is None:
        if y is None:
            raise ParameterError("y or onset_envelope must be provided")
        _, _ = pl.precheck_signal(y)
        ndim = y.ndim if isinstance(y, nat.DeviceArray) else np.ndim(y)
        shape = None
    else:
        if not isinstance(onset_envelope, nat.DeviceArray):
            onset_envelope = np.asarray(onset_envelope)
        elif onset_envelope.layout != "c":
            raise nat.UnsupportedOnGPU("onset_detect needs a C-ordered DeviceArray envelope")
        ndim, shape = onset_envelope.ndim, tuple(onset_envelope.shape)
        pk.check_data(onset_envelope.dtype, shape)
        _check_normalizable(shape, normalize)
    deferred = None   # the reference raises these only when there are onsets to pick
    try:
        kw = _peak_kwargs(kwargs, sr, hop_length)
        windows, method = pk.check_args(ndim, sparse=sparse, **kw)
    except (ParameterError, TypeError, ValueError, OverflowError) as e:
        deferred = e
    if deferred is None and backtrack and not sparse:
        deferred = ParameterError("onset backtracking is only supported if sparse=True")
    if deferred is None and backtrack and energy is not None:
        _check_energy(energy)
    if deferred is not None and onset_envelope is not None and not isinstance(onset_envelope, nat.DeviceArray):
        if _host_verdict(onset_envelope, normalize):
            raise deferred
        _check_units(sparse, units)
        return _empty(shape, sparse, units, None, False)

    with pl.Scope(y if onset_envelope is None else onset_envelope) as sc:
        env = _Envelope(y, sr, onset_envelope, hop_length)
        try:
            if env.audio is not None:
                env.audio.check_finite()
            x, ctx, on_device = env.dev, env.ctx, env.on_device
            if onset_envelope is None:
                pk.check_data(x.dtype, x.shape)
                _check_normalizable(x.shape, normalize)
            norm, flags = _normalize(sc, x, normalize)
            if deferred is not None:
                if _passes(flags.get()):
                    raise deferred
                _check_units(sparse, units)
                return _empty(x.shape, sparse, units, ctx, on_device)
            picked = norm if norm is not None else x
            out_units = ("frames" if backtrack or units not in pk.UNITS else units) if sparse else None
            dense, lst, count = pk.launch(sc, picked, windows, method, kw["delta"], flags=flags, dense=not sparse,
                                          units=out_units, hop_length=hop_length, sr=sr)
            if sparse and backtrack:
                e_dev = picked if energy is None else sc.stage(energy)
                lst = _backtrack_launch(sc, e_dev, lst, x.shape[-1], count, units if units in pk.UNITS else "frames",
                                        hop_length, sr)
        finally:
            env.release()
        if not sparse:
            return sc.result(dense)
        verdict = flags.get()   # 16 bytes: the verdict and the pick count
        k = int(verdict[1]) if _passes(verdict) else 0
        if _passes(verdict) and backtrack and k == 0:
            raise ParameterError(_EMPTY_MATCH)
        _check_units(sparse, units)
        if on_device:
            return sc.keep(lst).view((k,))
        return lst.get()[:k].copy()


def onset_backtrack(events, energy):
    """Backtrack onset events to the nearest preceding local minimum of an energy function; same contract as
    ``librosa.onset.onset_backtrack``.  ``energy`` is one-dimensional float32 or float64; ``events`` one-dimensional
    (a DeviceArray of int64 frames, or host integers).  Returns int64 frames: a DeviceArray when either input is
    one."""
    _check_energy(energy)
    ev_dev = isinstance(events, nat.DeviceArray)
    on_device = ev_dev or isinstance(energy, nat.DeviceArray)
    if ev_dev:
        if events.ndim != 1 or events.dtype != np.int64 or events.layout != "c":
            raise nat.UnsupportedOnGPU("onset_backtrack takes a C-ordered one-dimensional int64 DeviceArray of events")
        n_events = events.shape[0]
    else:
        ev = np.asarray(events)
        if ev.ndim != 1 or not (np.issubdtype(ev.dtype, np.integer) or np.issubdtype(ev.dtype, np.floating)):
            raise nat.UnsupportedOnGPU("onset_backtrack takes one-dimensional integer or float event lists on the GPU")
        n_events = ev.shape[0]
    if n_events == 0:
        raise ParameterError(_EMPTY_MATCH)
    n = energy.shape[0] if isinstance(energy, nat.DeviceArray) else np.shape(energy)[0]
    if not ev_dev:
        if np.issubdtype(ev.dtype, np.floating) and not np.all(np.isfinite(ev)):
            raise nat.UnsupportedOnGPU("onset_backtrack: non-finite event positions are not supported on the GPU")
        if ev.min() < 0:
            raise ParameterError(_NEGATIVE_MATCH)
        # the last minimum at or before a frame only depends on the frame's integer part, and frames past the end
        # take the last minimum
        ev = np.minimum(np.floor(ev) if ev.dtype.kind == "f" else ev, max(n, 1)).astype(np.int64)
    with pl.Scope(events, energy) as sc:
        e_dev = sc.stage(energy)
        d_ev = sc.stage(events if ev_dev else ev)
        if ev_dev:
            nat.check(nat.lib().b2l_status_reset(sc.ctx.handle))
        out = _backtrack_launch(sc, e_dev, d_ev, n_events, None, "frames", 512, 22050.0)
        if ev_dev and pl.status_word(sc.ctx) & nat.STATUS_NEGATIVE_EVENT:
            raise ParameterError(_NEGATIVE_MATCH)
        return sc.result(out)


def detect_stages(onset_envelope, *, normalize: bool = True):
    """The normaliser's output and verdict for a host envelope (testing aid): ``normalized`` (the envelope the
    picker reads) and ``flags`` (bit 0: some value nonzero, bit 1: some value not finite)."""
    with pl.Scope() as sc:
        norm, flags = _normalize(sc, sc.stage(onset_envelope), normalize)
        return {"normalized": norm.get() if norm is not None else np.asarray(onset_envelope),
                "flags": int(flags.get()[0])}
