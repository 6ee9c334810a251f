"""``librosa.decompose.hpss`` and ``nn_filter`` with librosa's signatures.

hpss (reference: librosa/decompose.py:241-389): both median filters, the two soft masks and the masked spectrograms
come out of ONE kernel (``hpss_kernel``: the filter window of every element is sorted in registers by a compile-time
bitonic network).

nn_filter (reference: librosa/decompose.py:409-592): the neighbours come from ``segment.recurrence_matrix`` on the
device (or from the caller's ``rec``), and ``nn_agg_kernel`` aggregates them with np.mean, np.median or np.average,
bit for bit as the reference's loop does."""
from __future__ import annotations

import ctypes as C

import numpy as np
import scipy.sparse

from . import _native as nat
from . import _pipeline as pl
from .util.exceptions import ParameterError

_vp = C.c_void_p

__all__ = ["hpss", "nn_filter"]


def _pair(v):
    return (v[0], v[1]) if isinstance(v, (tuple, list)) else (v, v)


def _hpss_device(sc, Sd, *, kernel_size, power, mask, margin):
    """Sd: DeviceArray (..., bins, frames), complex64 or float32, layout "ft" or "c".  Returns two DeviceArrays in
    layout "ft", owned by the scope ``sc``."""
    win_harm, win_perc = _pair(kernel_size)
    margin_harm, margin_perc = _pair(margin)
    if margin_harm < 1 or margin_perc < 1:
        raise ParameterError("Margins must be >= 1.0. A typical range is between 1 and 10.")
    if power <= 0:
        raise ParameterError("power must be strictly positive")
    if int(win_harm) > 64 or int(win_perc) > 64:
        raise nat.UnsupportedOnGPU("hpss: median filters longer than 64 are not supported on the GPU")
    if Sd.ndim < 2:
        raise ParameterError("hpss needs an input of shape (..., bins, frames)")
    is_complex = Sd.dtype == np.complex64
    F, T = Sd.shape[-2], Sd.shape[-1]
    ctx = sc.ctx
    n_clips = pl.clip_count(Sd.shape[:-2])
    L = nat.lib()
    src = sc.native(Sd)
    if is_complex:
        mag = sc.empty(Sd.shape, np.float32, layout="ft")
        nat.check(L.b2l_cabs(ctx.handle, _vp(src.ptr), src.size, _vp(mag.ptr)))
    else:
        mag = src
    out_dtype = np.float32 if (mask or not is_complex) else np.complex64
    harm = sc.empty(Sd.shape, out_dtype, layout="ft")
    perc = sc.empty(Sd.shape, out_dtype, layout="ft")
    desc = nat.HpssDesc(win_harm=int(win_harm), win_perc=int(win_perc), margin_harm=float(margin_harm),
                        margin_perc=float(margin_perc), power=float(power), mask_only=int(bool(mask)))
    nat.check(L.b2l_hpss(ctx.handle, C.byref(desc), _vp(mag.ptr), _vp(src.ptr if is_complex else None), n_clips, T, F,
                         _vp(harm.ptr), _vp(perc.ptr)))
    sc.free(mag, src)
    return harm, perc


def hpss(S, *, kernel_size=31, power: float = 2.0, mask: bool = False, margin=1.0):
    """Median-filtering harmonic / percussive separation of a spectrogram ``S`` (real magnitudes or a complex
    STFT); same contract as ``librosa.decompose.hpss``."""
    with pl.Scope(S) as sc:
        if sc.on_device:
            if S.dtype not in (np.dtype(np.float32), np.dtype(np.complex64)):
                raise ParameterError("device spectrogram must be float32 or complex64")
            dev = S
            res_dtype = mask_dtype = None   # a device call returns its DeviceArrays
        else:
            S = np.asarray(S)
            if np.iscomplexobj(S):
                res_dtype = np.dtype(S.dtype)
                if res_dtype == np.complex128 and not pl.wide_complex_ok("hpss input"):
                    raise ParameterError("complex128 input refused (B2L_FLOAT64=error)")
                dev = sc.stage(S, np.complex64)
                mask_dtype = np.dtype(np.float32 if res_dtype == np.complex64 else np.float64)
            else:
                dev, res_dtype = sc.spectrogram(S, "hpss input", stacklevel=5)
                mask_dtype = res_dtype
        harm, perc = _hpss_device(sc, dev, kernel_size=kernel_size, power=power, mask=mask, margin=margin)
        out_dtype = mask_dtype if mask else res_dtype
        return sc.result(harm, out_dtype), sc.result(perc, out_dtype)


_AGGREGATES = {id(np.mean): nat.NN_MEAN, id(np.median): nat.NN_MEDIAN, id(np.average): nat.NN_AVERAGE}


def _host_table(sc, rec_s, S_dtype, agg):
    """A host csc_array uploaded as the aggregation's table: (start, count, idx, weights, compute dtype, max count)."""
    indptr = np.asarray(rec_s.indptr, dtype=np.int64)
    count = np.diff(indptr).astype(np.int32)
    rt = np.result_type(S_dtype, rec_s.dtype)
    start = sc.stage(indptr[:-1])
    cnt = sc.stage(count)
    idx = sc.stage(np.asarray(rec_s.indices, dtype=np.int32))
    w = sc.stage(np.asarray(rec_s.data).astype(rt).astype(np.float64)) if agg == nat.NN_AVERAGE else None
    return start, cnt, idx, w, rt, int(count.max()) if count.size else 0


def _device_table(sc, rec, agg):
    """A dense t x t DeviceArray as the aggregation's table (csc_array(rec): column i's non-zero rows, ascending)."""
    if rec.ndim != 2 or rec.shape[0] != rec.shape[1] or rec.layout != "c":
        return None
    if rec.dtype not in (np.float32, np.float64, np.bool_):
        raise nat.UnsupportedOnGPU("nn_filter: a device rec must be float32, float64 or bool")
    t = rec.shape[0]
    L = nat.lib()
    elem = nat.ELEM_TYPES[np.dtype(rec.dtype)]
    cnt = sc.empty((t,), np.int32)
    nat.check(L.b2l_nn_compact(sc.ctx.handle, _vp(rec.ptr), elem, t, 0, _vp(cnt.ptr), None, None, None))
    count = cnt.get().astype(np.int64)
    indptr = np.concatenate([[0], np.cumsum(count)])
    start = sc.stage(indptr[:-1])
    idx = sc.empty((max(int(indptr[-1]), 1),), np.int32)
    w = sc.empty((max(int(indptr[-1]), 1),), np.float64)
    nat.check(L.b2l_nn_compact(sc.ctx.handle, _vp(rec.ptr), elem, t, 1, _vp(cnt.ptr), _vp(start.ptr), _vp(idx.ptr),
                               _vp(w.ptr)))
    return start, cnt, idx, w, int(count.max()) if count.size else 0


def nn_filter(S, *, rec=None, aggregate=None, axis: int = -1, **kwargs):
    """Filter by nearest-neighbour aggregation; same contract as ``librosa.decompose.nn_filter``.

    ``S``: a real float32 / float64 NumPy array, or a DeviceArray (..., bins, frames) in either layout filtered along
    its last axis (the result is a DeviceArray in the "ft" layout).  ``rec``: None (``segment.recurrence_matrix(S,
    axis=axis, **kwargs)`` on the device), a NumPy array or any SciPy sparse array or matrix (taken through
    ``scipy.sparse.csc_array`` on the host, as the reference does, then uploaded), or a dense t x t DeviceArray.
    ``aggregate``: np.mean (default), np.median or np.average; others are refused with ``UnsupportedOnGPU``."""
    from . import segment

    if aggregate is None:
        aggregate = np.mean
    agg = _AGGREGATES.get(id(aggregate))
    if agg is None:
        raise nat.UnsupportedOnGPU("nn_filter: aggregate must be np.mean, np.median or np.average on the GPU")
    on_device = isinstance(S, nat.DeviceArray)
    if not on_device:
        S = np.asarray(S)
    if S.dtype not in (np.float32, np.float64):
        raise nat.UnsupportedOnGPU(f"nn_filter: S of dtype {S.dtype} is not supported on the GPU (float32 and float64 "
                                   "are)")
    if on_device and (S.ndim < 2 or axis not in (-1, S.ndim - 1)):
        raise nat.UnsupportedOnGPU("nn_filter: device S (..., bins, frames) is filtered along its last axis only")
    t = S.shape[axis]
    dev_rec = isinstance(rec, nat.DeviceArray)
    rec_s = None
    if rec is not None and not dev_rec:
        rec_s = scipy.sparse.csc_array(rec)
        if rec_s.shape[0] != t or rec_s.shape[0] != rec_s.shape[1]:
            raise ParameterError("Invalid self-similarity matrix shape "
                                 f"rec.shape={rec_s.shape} for S.shape={S.shape}")
        if agg == nat.NN_AVERAGE and np.result_type(S.dtype, rec_s.dtype) not in (np.float32, np.float64):
            raise nat.UnsupportedOnGPU(f"nn_filter: np.average over weights of dtype {rec_s.dtype} is not supported")
    elif dev_rec and (rec.ndim != 2 or rec.shape[0] != t or rec.shape[0] != rec.shape[1]):
        raise ParameterError("Invalid self-similarity matrix shape "
                             f"rec.shape={rec.shape} for S.shape={S.shape}")
    with pl.Scope(S, rec) as sc:
        stride, start = 0, None
        if rec is None:
            kw = dict(kwargs)
            kw.pop("sparse", None)
            g = segment._graph(sc, S, axis=axis, **{**dict(k=None, width=1, metric="euclidean", sym=False,
                                                           mode="connectivity", bandwidth=None, self=False,
                                                           full=False), **kw})
            cnt, idx, w, stride = g.count, g.idx, g.val, g.k_out
            rt = np.result_type(S.dtype, g.dtype)
            max_count = g.k_out
        elif dev_rec:
            tab = _device_table(sc, rec, agg)
            if tab is None:
                raise nat.UnsupportedOnGPU("nn_filter: a device rec must be a C-ordered t x t DeviceArray")
            start, cnt, idx, w, max_count = tab
            rt = np.result_type(S.dtype, rec.dtype)
        else:
            start, cnt, idx, w, rt, max_count = _host_table(sc, rec_s, S.dtype, agg)
        if on_device:
            src = sc.native(S)
            n_lead, F = pl.clip_count(S.shape[:-2]), S.shape[-2]
            out = sc.empty(S.shape, S.dtype, layout="ft")
        else:
            moved = np.moveaxis(S, axis, 0)
            src = sc.stage(np.ascontiguousarray(moved.reshape(t, -1)))
            n_lead, F = 1, src.shape[1]
            out = sc.empty(src.shape, S.dtype)
        desc = nat.NnFilterDesc(agg=agg, s_f64=int(S.dtype == np.float64), r_f64=int(rt == np.float64),
                                max_count=int(max_count), stride=int(stride))
        zero = C.c_int32(0)
        nat.check(nat.lib().b2l_nn_filter(sc.ctx.handle, C.byref(desc), _vp(src.ptr), n_lead, t, F,
                                          _vp(start.ptr if start is not None else None), _vp(cnt.ptr), _vp(idx.ptr),
                                          _vp(w.ptr if w is not None else None), _vp(out.ptr), C.byref(zero)))
        if zero.value:
            raise ZeroDivisionError("Weights sum to zero, can't be normalized")
        if on_device:
            return sc.keep(out)
        res = out.get()
        return np.moveaxis(res.reshape(moved.shape), 0, axis)
