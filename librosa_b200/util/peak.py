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


def launch(x, windows, method, delta, *, flags=None, dense=True, units=None, hop_length=512, sr=22050.0):
    """One launch of the picker on the C-ordered device data ``x`` (..., n).  ``flags``: the verdict pair of
    ``onset_normalize`` (picks only where it passed).  Returns the dense picks (DeviceArray of bool, or None) and,
    with ``units`` (one row only), the list in those units and a count DeviceArray (``flags``'s second word when
    ``flags`` is given)."""
    from .. import _pipeline as pl

    ctx, n = x.ctx, x.shape[-1]
    pre_max, post_max, pre_avg, post_avg, wait = (min(v, n) for v in windows)
    desc = nat.PeakDesc(pre_max=pre_max, post_max=max(1, post_max), pre_avg=pre_avg, post_avg=max(1, post_avg),
                        wait=wait, delta=float(delta), method=method, f64=int(x.dtype == np.float64),
                        units=UNITS[units] if units is not None else 0, hop_length=int(hop_length), sr=float(sr))
    out = nat.DeviceArray.empty(ctx, x.shape, np.bool_) if dense else None
    lst = count = None
    if units is not None:
        lst = nat.DeviceArray.empty(ctx, (n,), np.float64 if units == "time" else np.int64)
        if flags is not None:
            count = nat.DeviceArray(ctx, flags.ptr + 8, (1,), np.int64, layout="c", owner=False)
            count._base = flags
        else:
            count = nat.DeviceArray.empty(ctx, (1,), np.int64)
    nat.check(nat.lib().b2l_peak_pick(ctx.handle, C.byref(desc), _vp(x.ptr), pl.clip_count(x.shape[:-1]), n,
                                      _vp(flags.ptr) if flags is not None else None,
                                      _vp(out.ptr) if out is not None else None, _vp(lst.ptr) if lst else None,
                                      _vp(count.ptr) if count else None))
    return out, lst, count


def list_view(lst, k):
    """The first ``k`` entries of a device list, as a view that keeps the list alive."""
    view = nat.DeviceArray(lst.ctx, lst.ptr, (k,), lst.dtype, layout="c", owner=False)
    view._base = lst
    return view


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
        dev = x
    else:
        moved = np.moveaxis(x, axis, -1)
        check_data(x.dtype, moved.shape)
        dev = pl.context_for(None).to_device(np.ascontiguousarray(moved))
    dense, lst, count = launch(dev, windows, code, delta, dense=not sparse, units="frames" if sparse else None)
    if not on_device:
        dev.free()
    if sparse:
        k = int(count.get()[0])
        count.free()
        if on_device:
            return list_view(lst, k)
        out = lst.get()[:k].copy()
        lst.free()
        return out
    if on_device:
        return dense
    return np.moveaxis(pl.finish(dense), -1, axis)
