"""``librosa.segment.recurrence_matrix`` on the GPU (reference: librosa/segment.py:391-706, the bandwidths of
1332-1437).  The rest of ``librosa.segment`` is not provided.

The k-nearest-neighbour search runs in ``b2l_nn_graph``: float64 frame distances on the FP64 tensor cores, a
deterministic selection per frame in (distance, frame index) order, then the reference's rules for width, k, ``sym``,
``self`` and the affinity bandwidth.  Where the reference's neighbour search meets two frames at exactly the same
distance, which one it returns is decided by NumPy's partition; the GPU takes the lower frame index."""
from __future__ import annotations

import ctypes as C

import numpy as np
import scipy.sparse

from . import _native as nat
from . import _pipeline as pl
from .util.exceptions import ParameterError

_vp = C.c_void_p

__all__ = ["recurrence_matrix"]

_MODES = ["connectivity", "distance", "affinity"]
_NOT_FINITE = "Input contains NaN or infinity."   # sklearn's check_array refuses such data


class Graph:
    """A recurrence matrix on the device as a neighbour table: row i of ``idx`` / ``val`` [t][k_out] holds the
    ``count[i]`` links of frame i (column i of the reference's csc_array), ascending frame index.  ``dtype`` is the
    reference's output dtype."""

    def __init__(self, sc, t, k_out, dtype):
        self.t, self.k_out, self.dtype = t, k_out, np.dtype(dtype)
        self.idx = sc.empty((t, k_out), np.int32)
        self.val = sc.empty((t, k_out), np.float64)
        self.count = sc.empty((t,), np.int32)

    def to_sparse(self):
        """The host scipy.sparse.csc_array of the table."""
        count = self.count.get().astype(np.int64)
        idx, val = self.idx.get(), self.val.get()
        keep = np.arange(self.k_out)[np.newaxis, :] < count[:, np.newaxis]
        indptr = np.concatenate([[0], np.cumsum(count)])
        data = val[keep].astype(self.dtype)
        return scipy.sparse.csc_array((data, idx[keep], indptr), shape=(self.t, self.t))


def _check(t, *, k, width, metric, mode, bandwidth, full, axis):
    """The reference's argument checks in its order (width, mode), then what the GPU refuses; returns k."""
    if width < 1 or width >= (t - 1) // 2:
        raise ParameterError("width={} must be at least 1 and at most (data.shape[{}] - 1) // 2={}".format(
            width, axis, (t - 1) // 2))
    if mode not in _MODES:
        raise ParameterError(f"Invalid mode='{mode}'. Must be one of ['connectivity', 'distance', 'affinity']")
    if k is None:
        k = 2 * np.ceil(np.sqrt(t - 2 * width + 1))
    k = int(k)
    if full:
        # the reference's full=True skips the width exclusion and the top-k trim in every mode (segment.py:650)
        raise nat.UnsupportedOnGPU("recurrence_matrix: full=True is not supported on the GPU")
    if metric not in nat.NN_METRICS:
        raise nat.UnsupportedOnGPU(f"recurrence_matrix: metric={metric!r} is not supported on the GPU "
                                   "(euclidean and cosine are)")
    if k < 1:
        raise nat.UnsupportedOnGPU(f"recurrence_matrix: k={k} is not supported on the GPU")
    if t > nat.NN_MAX_FRAMES:
        raise nat.UnsupportedOnGPU(f"recurrence_matrix: {t} frames; up to {nat.NN_MAX_FRAMES} are supported on the GPU")
    n_cand = min(t - 1, k + 2 * width)
    if n_cand > nat.NN_MAX_CANDIDATES:
        raise nat.UnsupportedOnGPU(f"recurrence_matrix: k + 2 * width = {k + 2 * width} candidates per frame; up to "
                                   f"{nat.NN_MAX_CANDIDATES} are supported on the GPU")
    bw_mode, bw = 0, 0.0
    if mode == "affinity":
        if isinstance(bandwidth, np.ndarray):
            raise nat.UnsupportedOnGPU("recurrence_matrix: an ndarray bandwidth is not supported on the GPU")
        if isinstance(bandwidth, (int, float)):
            bw = float(bandwidth)
            if bw <= 0:
                raise ParameterError(f"Invalid scalar bandwidth={bw}. Must be strictly positive.")
        else:
            name = "med_k_scalar" if bandwidth is None else bandwidth
            if name not in nat.NN_BANDWIDTHS:
                raise ParameterError(
                    f"Invalid bandwidth='{name}'. Must be either a positive scalar or one of "
                    "['med_k_scalar', 'mean_k', 'gmean_k', 'mean_k_avg', 'gmean_k_avg', 'mean_k_avg_and_pair']")
            bw_mode = nat.NN_BANDWIDTHS[name]
            if min(k, n_cand) + 1 > nat.NN_MAX_STATS:
                raise nat.UnsupportedOnGPU(f"recurrence_matrix: bandwidth={name!r} with k={k}; the GPU estimates "
                                           f"bandwidths over at most {nat.NN_MAX_STATS - 1} neighbours")
    return k, n_cand, bw_mode, bw


def _graph(sc, data, *, k, width, metric, sym, mode, bandwidth, self, axis, full) -> Graph:
    """Checks, then the neighbour table of ``data`` on the device (owned by ``sc``)."""
    if isinstance(data, nat.DeviceArray):
        if data.dtype not in (np.float32, np.float64):
            raise nat.UnsupportedOnGPU("recurrence_matrix: device data must be float32 or float64")
        if data.ndim < 2:
            raise nat.UnsupportedOnGPU("recurrence_matrix: device data must have at least two dimensions")
        if axis not in (-1, data.ndim - 1):
            raise nat.UnsupportedOnGPU("recurrence_matrix: device data is compared along its last axis only")
        t, d = data.shape[-1], data.shape[-2]
        n_lead = pl.clip_count(data.shape[:-2])
        if data.layout == "ft":
            geo = dict(n_lead=n_lead, n_feat=d, lead_stride=t * d, feat_stride=1, frame_stride=d)
        else:
            geo = dict(n_lead=n_lead, n_feat=d, lead_stride=t * d, feat_stride=t, frame_stride=1)
        src, dtype = data, data.dtype
    else:
        x = np.atleast_2d(data)
        if np.iscomplexobj(x):
            raise nat.UnsupportedOnGPU("recurrence_matrix: complex data is not supported on the GPU")
        x = np.swapaxes(x, axis, 0)
        t = x.shape[0]
        x = x.reshape((t, -1), order="F")
        # sklearn's check_array: float32 stays, everything else is computed as float64
        dtype = np.dtype(np.float32) if x.dtype == np.float32 else np.dtype(np.float64)
        geo = None
    k, n_cand, bw_mode, bw = _check(t, k=k, width=width, metric=metric, mode=mode, bandwidth=bandwidth,
                                    full=full, axis=axis)
    if geo is None:
        if not np.isfinite(x).all():
            raise ValueError(_NOT_FINITE)
        src = sc.stage(np.ascontiguousarray(x, dtype=dtype))
        geo = dict(n_lead=1, n_feat=x.shape[1], lead_stride=0, feat_stride=1, frame_stride=x.shape[1])
    # cosine distances of float32 data are float32 (sklearn's float32 GEMM); every other case is float64
    out = np.float32 if (metric == "cosine" and dtype == np.float32) else np.float64
    if mode == "connectivity":
        out_dtype = np.dtype(np.bool_)
    else:
        out_dtype = np.dtype(out)
    k_out = min(k, n_cand) + 1
    g = Graph(sc, t, k_out, out_dtype)
    desc = nat.NnDesc(metric=nat.NN_METRICS[metric], mode=_MODES.index(mode), k=k, width=int(width), n_cand=n_cand,
                      sym=int(bool(sym)), self_link=int(bool(self)), f64=int(out == np.float64), bw_mode=bw_mode,
                      src_f64=int(src.dtype == np.float64), bandwidth=bw, **geo)
    bad = C.c_int32(0)
    nat.check(nat.lib().b2l_nn_graph(sc.ctx.handle, C.byref(desc), _vp(src.ptr), t, k_out, _vp(g.idx.ptr),
                                     _vp(g.val.ptr), _vp(g.count.ptr), C.byref(bad)))
    if bad.value:
        raise ValueError(_NOT_FINITE)
    sc.free(src)
    return g


def recurrence_matrix(data, *, k=None, width: int = 1, metric: str = "euclidean", sym: bool = False,
                      sparse: bool = False, mode: str = "connectivity", bandwidth=None, self: bool = False,
                      axis: int = -1, full: bool = False):
    """Recurrence (k-nearest-neighbour) matrix of the frames of ``data``; same contract as
    ``librosa.segment.recurrence_matrix``.

    ``data`` may be a NumPy array or a float32 / float64 DeviceArray (compared along its last axis).  The dense result
    follows the input: a NumPy array for host data, a C-ordered DeviceArray for device data.  ``sparse=True`` returns
    a host ``scipy.sparse.csc_array`` in both cases, the one host result: SciPy's sparse arrays have no device form.

    Data with a NaN or an infinity raises ``ValueError``, host or device alike, as sklearn's ``check_array`` does.
    Refused with ``UnsupportedOnGPU``: metrics other than euclidean and cosine, ``full=True``, an ndarray bandwidth,
    more than 65 536 frames and more than 4 096 candidates per frame (k + 2 width)."""
    with pl.Scope(data) as sc:
        g = _graph(sc, data, k=k, width=width, metric=metric, sym=sym, mode=mode, bandwidth=bandwidth, self=self,
                   axis=axis, full=full)
        if sparse:
            return g.to_sparse()
        if sc.on_device:
            rec = sc.empty((g.t, g.t), g.dtype)
            nat.check(nat.lib().b2l_nn_dense(sc.ctx.handle, _vp(g.idx.ptr), _vp(g.val.ptr), _vp(g.count.ptr), g.t,
                                             g.k_out, nat.ELEM_TYPES[g.dtype], _vp(rec.ptr)))
            return sc.keep(rec)
        return g.to_sparse().toarray()
