"""``librosa.util.peak_pick`` (reference: librosa/util/utils.py:1188-1496) on the device.

One kernel launch, one CTA per row (csrc/onset_kernels.cuh).  The picks are discrete, so the kernel restates the
reference's numba arithmetic: the window mean is a left-to-right sum in the data's dtype divided by the count in
float64, the dynamic-programming pickers use a sequential cumsum in the data's dtype and a float64 DP, and a NaN in
the max window stops a greedy pick.  ``onset.onset_detect`` runs the same launch behind its normaliser."""
from __future__ import annotations

import ctypes as C

import numpy as np

from .. import _native as nat
from .exceptions import ParameterError

_vp = C.c_void_p

__all__ = ["peak_pick"]

METHODS = {"greedy": nat.PEAK_GREEDY, "dp_count": nat.PEAK_DP_COUNT, "dp_value": nat.PEAK_DP_VALUE}
UNITS = {"frames": nat.BEAT_FRAMES, "samples": nat.BEAT_SAMPLES, "time": nat.BEAT_TIME}
MAX_FRAMES = (1 << 31) - 1   # frames per row the kernels index with int


def check_args(ndim, *, pre_max, post_max, pre_avg, post_avg, delta, wait, sparse=True, method="greedy"):
    """peak_pick's argument checks in the reference's order; returns the windows as ints (``valid_int`` with
    ``np.ceil``) and the method's code."""
    if pre_max < 0:
        raise ParameterError("pre_max must be non-negative")
    if pre_avg < 0:
        raise ParameterError("pre_avg must be non-negative")
    if delta < 0:
        raise ParameterError("delta must be non-negative")
    if wait < 0:
        raise ParameterError("wait must be non-negative")
    if post_max <= 0:
        raise ParameterError("post_max must be positive")
    if post_avg <= 0:
        raise ParameterError("post_avg must be positive")
    if sparse and ndim != 1:
        raise ParameterError(
            f"sparse=True (default) does not support "
            f"{ndim}-dimensional inputs. "
            f"Either set sparse=False or process each dimension independently."
        )
    windows = tuple(int(np.ceil(v)) for v in (pre_max, post_max, pre_avg, post_avg, wait))
    if method not in METHODS:
        raise ParameterError(f"Unknown method {method}")
    return windows, METHODS[method]


def check_data(dtype, shape):
    """The GPU's refusals from the dtype and the row length."""
    if np.dtype(dtype) not in (np.float32, np.float64):
        raise nat.UnsupportedOnGPU(f"peak picking of {np.dtype(dtype)} data is not supported on the GPU "
                                   "(float32 and float64 only)")
    if len(shape) and shape[-1] > MAX_FRAMES:
        raise nat.UnsupportedOnGPU(f"peak picking of rows of {shape[-1]} frames: the GPU takes fewer than 2^31")


def launch(sc, x, windows, method, delta, *, flags=None, dense=True, units=None, hop_length=512, sr=22050.0):
    """One launch of the picker on the C-ordered device data ``x`` (..., n), its buffers owned by the scope ``sc``.
    ``flags``: the verdict pair of ``onset_normalize`` (picks only where it passed).  Returns the dense picks
    (DeviceArray of bool, or None) and, with ``units`` (one row only), the list in those units and a count
    DeviceArray (``flags``'s second word when ``flags`` is given)."""
    from .. import _pipeline as pl

    ctx, n = sc.ctx, x.shape[-1]
    pre_max, post_max, pre_avg, post_avg, wait = (min(v, n) for v in windows)
    desc = nat.PeakDesc(pre_max=pre_max, post_max=max(1, post_max), pre_avg=pre_avg, post_avg=max(1, post_avg),
                        wait=wait, delta=float(delta), method=method, f64=int(x.dtype == np.float64),
                        units=UNITS[units] if units is not None else 0, hop_length=int(hop_length), sr=float(sr))
    out = sc.empty(x.shape, np.bool_) if dense else None
    lst = count = None
    if units is not None:
        lst = sc.empty((n,), np.float64 if units == "time" else np.int64)
        count = flags.view((1,), offset=1) if flags is not None else sc.empty((1,), np.int64)
    nat.check(nat.lib().b2l_peak_pick(ctx.handle, C.byref(desc), _vp(x.ptr), pl.clip_count(x.shape[:-1]), n,
                                      _vp(flags.ptr) if flags is not None else None,
                                      _vp(out.ptr) if out is not None else None, _vp(lst.ptr) if lst else None,
                                      _vp(count.ptr) if count else None))
    return out, lst, count


def peak_pick(x, *, pre_max, post_max, pre_avg, post_avg, delta, wait, sparse: bool = True, method: str = "greedy",
              axis: int = -1):
    """Pick peaks in a signal; same contract as ``librosa.util.peak_pick``.

    Host input gives NumPy output and may pick along any ``axis``; a DeviceArray (C-ordered, float32 or float64,
    ``axis`` the last) gives a DeviceArray: the dense bool picks, or a view of the compacted int64 list."""
    from .. import _pipeline as pl

    on_device = isinstance(x, nat.DeviceArray)
    if not on_device:
        x = np.asarray(x)
    windows, code = check_args(x.ndim, pre_max=pre_max, post_max=post_max, pre_avg=pre_avg, post_avg=post_avg,
                               delta=delta, wait=wait, sparse=sparse, method=method)
    if on_device:
        if axis not in (-1, x.ndim - 1):
            raise nat.UnsupportedOnGPU("peak_pick of a DeviceArray runs along its last axis only")
        if x.layout != "c":
            raise nat.UnsupportedOnGPU("peak_pick needs a C-ordered DeviceArray")
        check_data(x.dtype, x.shape)
    else:
        x = np.moveaxis(x, axis, -1)
        check_data(x.dtype, x.shape)
    with pl.Scope(x) as sc:
        dense, lst, count = launch(sc, sc.stage(x), windows, code, delta, dense=not sparse,
                                   units="frames" if sparse else None)
        if sparse:
            k = int(count.get()[0])
            return sc.keep(lst).view((k,)) if on_device else lst.get()[:k].copy()
        return sc.result(dense) if on_device else np.moveaxis(sc.result(dense), -1, axis)
