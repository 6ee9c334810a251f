"""Host-side array helpers of the hot path (mirror of the relevant parts of librosa/util/utils.py).

These are tiny shape / dtype utilities: they run on the host exactly as in the reference; all
per-sample and per-frame arithmetic is done by the CUDA library.
"""
from __future__ import annotations

from typing import Any

import numpy as np

from .exceptions import ParameterError

# librosa/util/utils.py:41 — kept for API parity; the GPU kernels tile by frames, not by bytes.
MAX_MEM_BLOCK = 2 ** 8 * 2 ** 10


def frame(x, *, frame_length: int, hop_length: int, axis: int = -1, writeable: bool = False,
          subok: bool = False) -> np.ndarray:
    """Zero-copy overlapping-frame view, ``xf[..., k, j] = x[..., j*hop + k]`` for ``axis=-1``.

    Same contract as librosa.util.frame (librosa/util/utils.py:79-242): the frame axis is inserted
    right before ``axis`` when ``axis < 0`` and right after it otherwise; raises ParameterError when the
    input is shorter than one frame or ``hop_length < 1``.
    """
    x = np.asanyarray(x) if subok else np.asarray(x)
    n = x.shape[axis]
    if n < frame_length:
        raise ParameterError(f"Input is too short (n={n:d}) for frame_length={frame_length:d}")
    if hop_length < 1:
        raise ParameterError(f"Invalid hop_length: {hop_length:d}")
    ax = axis % x.ndim
    step = x.strides[ax]
    n_pos = n - frame_length + 1
    # windows at every position first (new trailing axis), then keep every hop-th position
    shape = x.shape[:ax] + (n_pos,) + x.shape[ax + 1:] + (frame_length,)
    strides = x.strides + (step,)
    view = np.lib.stride_tricks.as_strided(x, shape=shape, strides=strides, subok=subok, writeable=writeable)
    target = axis - 1 if axis < 0 else axis + 1
    view = np.moveaxis(view, -1, target)
    sl = [slice(None)] * view.ndim
    sl[axis] = slice(0, None, hop_length)
    return view[tuple(sl)]


def valid_audio(y) -> bool:
    """librosa/util/utils.py:246-308: ndarray, floating, ndim >= 1, finite everywhere."""
    if not isinstance(y, np.ndarray):
        raise ParameterError("Audio data must be of type numpy.ndarray")
    if not np.issubdtype(y.dtype, np.floating):
        raise ParameterError("Audio data must be floating-point")
    if y.ndim == 0:
        raise ParameterError(f"Audio data must be at least one-dimensional, given y.shape={y.shape}")
    if not np.isfinite(y).all():
        raise ParameterError("Audio buffer is not finite everywhere")
    return True


def is_positive_int(x: Any) -> bool:
    """librosa/util/utils.py:344-358."""
    return isinstance(x, (int, np.integer)) and not isinstance(x, bool) and x > 0


def pad_center(data: np.ndarray, *, size: int, axis: int = -1, **kwargs) -> np.ndarray:
    """Centre ``data`` in an array of length ``size`` along ``axis`` (librosa/util/utils.py:387-458)."""
    kwargs.setdefault("mode", "constant")
    n = data.shape[axis]
    left = int((size - n) // 2)
    if left < 0:
        raise ParameterError(f"Target size ({size:d}) must be at least input size ({n:d})")
    widths = [(0, 0)] * data.ndim
    widths[axis] = (left, int(size - n - left))
    return np.pad(data, widths, **kwargs)


def expand_to(x: np.ndarray, *, ndim: int, axes) -> np.ndarray:
    """Reshape ``x`` to ``ndim`` dimensions, its axes landing on ``axes`` (librosa/util/utils.py:461-529)."""
    try:
        axes_t = tuple(axes)
    except TypeError:
        axes_t = (axes,)
    if len(axes_t) != x.ndim:
        raise ParameterError(f"Shape mismatch between axes={axes_t} and input x.shape={x.shape}")
    if ndim < x.ndim:
        raise ParameterError(f"Cannot expand x.shape={x.shape} to fewer dimensions ndim={ndim}")
    shape = [1] * ndim
    for i, ax in enumerate(axes_t):
        shape[ax] = x.shape[i]
    return x.reshape(shape)


def fix_length(data: np.ndarray, *, size: int, axis: int = -1, **kwargs) -> np.ndarray:
    """Trim or pad on the right to exactly ``size`` (librosa/util/utils.py:532-588)."""
    kwargs.setdefault("mode", "constant")
    n = data.shape[axis]
    if n > size:
        sl = [slice(None)] * data.ndim
        sl[axis] = slice(0, size)
        return data[tuple(sl)]
    if n < size:
        widths = [(0, 0)] * data.ndim
        widths[axis] = (0, size - n)
        return np.pad(data, widths, **kwargs)
    return data


def tiny(x) -> float:
    """Smallest positive normal number of ``x``'s floating type (librosa/util/utils.py:1935-2001)."""
    x = np.asarray(x)
    if np.issubdtype(x.dtype, np.floating) or np.issubdtype(x.dtype, np.complexfloating):
        dtype = x.dtype
    else:
        dtype = np.dtype(np.float32)
    return np.finfo(dtype).tiny


def normalize(S: np.ndarray, *, norm=np.inf, axis=0, threshold=None, fill=None) -> np.ndarray:
    """Norm-scale along ``axis`` (librosa/util/utils.py:797-1026)."""
    if threshold is None:
        threshold = tiny(S)
    elif threshold <= 0:
        raise ParameterError(f"threshold={threshold} must be strictly positive")
    if fill not in (None, False, True):
        raise ParameterError(f"fill={fill} must be None or boolean")
    if not np.isfinite(S).all():
        raise ParameterError("Input must be finite")
    mag = np.abs(S).astype(float)
    fill_norm = 1
    if norm is None:
        return S
    if norm == np.inf:
        length = np.max(mag, axis=axis, keepdims=True)
    elif norm == -np.inf:
        length = np.min(mag, axis=axis, keepdims=True)
    elif norm == 0:
        if fill is True:
            raise ParameterError("Cannot normalize with norm=0 and fill=True")
        length = np.sum(mag > 0, axis=axis, keepdims=True, dtype=mag.dtype)
    elif np.issubdtype(type(norm), np.number) and norm > 0:
        length = np.sum(mag ** norm, axis=axis, keepdims=True) ** (1.0 / norm)
        fill_norm = mag.shape[axis] ** (-1.0 / norm) if axis is not None else mag.size ** (-1.0 / norm)
    else:
        raise ParameterError(f"Unsupported norm: {repr(norm)}")
    small = length < threshold
    out = np.empty_like(S)
    if fill is None:
        length[small] = 1.0
        out[:] = S / length
    elif fill:
        length[small] = np.nan
        out[:] = S / length
        out[np.isnan(out)] = fill_norm
    else:
        length[small] = np.inf
        out[:] = S / length
    return out


def dtype_r2c(d, *, default=np.complex64):
    """Real -> complex dtype of the same precision (librosa/util/utils.py:2362-2417)."""
    table = {np.dtype(np.float32): np.complex64, np.dtype(np.float64): np.complex128}
    if hasattr(np, "longdouble"):
        table.setdefault(np.dtype(np.longdouble), np.clongdouble)
    dt = np.dtype(d)
    if dt.kind == "c":
        return dt
    return np.dtype(table.get(dt, default))


def dtype_c2r(d, *, default=np.float32):
    """Complex -> real dtype of the same precision (librosa/util/utils.py:2420-2476)."""
    table = {np.dtype(np.complex64): np.float32, np.dtype(np.complex128): np.float64}
    if hasattr(np, "clongdouble"):
        table.setdefault(np.dtype(np.clongdouble), np.longdouble)
    dt = np.dtype(d)
    if dt.kind == "f":
        return dt
    return np.dtype(table.get(dt, default))


def abs2(x, dtype=None):
    """Squared magnitude (librosa/util/utils.py:2580-2632)."""
    x = np.asarray(x)
    if np.iscomplexobj(x):
        y = x.real ** 2 + x.imag ** 2
    else:
        y = np.square(x)
    return y if dtype is None else y.astype(dtype)


def cyclic_gradient(data: np.ndarray, *, edge_order: int = 1, axis: int = -1) -> np.ndarray:
    """Gradient of a periodic array: wrap-pad, ``np.gradient``, un-pad (mirror of util/utils.py cyclic_gradient)."""
    pad = [(0, 0)] * data.ndim
    pad[axis] = (edge_order, edge_order)
    grad = np.gradient(np.pad(data, pad, mode="wrap"), edge_order=edge_order, axis=axis)
    keep = [slice(None)] * data.ndim
    keep[axis] = slice(edge_order, -edge_order)
    return grad[tuple(keep)]


def fill_off_diagonal(x: np.ndarray, *, radius: float, value: float = 0) -> None:
    """Set every entry of ``x`` outside the Sakoe-Chiba band to ``value``, in place; same contract as
    ``librosa.util.fill_off_diagonal``.  The band's half-width is ``int(np.round(radius * min(x.shape)))``, widened
    by ``|N - M|`` on the long side so that ``x[-1, -1]`` stays inside.  dtw's ``global_constraints`` applies the
    same band on the device (sequence._band)."""
    from .._native import DeviceArray, UnsupportedOnGPU

    if isinstance(x, DeviceArray):
        raise UnsupportedOnGPU("fill_off_diagonal works in place on a host ndarray")
    nx, ny = x.shape
    radius = int(np.round(radius * np.min(x.shape)))
    offset = np.abs(x.shape[0] - x.shape[1])
    if nx < ny:
        idx_u = np.triu_indices_from(x, k=radius + offset)
        idx_l = np.tril_indices_from(x, k=-radius)
    else:
        idx_u = np.triu_indices_from(x, k=radius)
        idx_l = np.tril_indices_from(x, k=-radius - offset)
    x[idx_u] = value
    x[idx_l] = value


def _localext(x, axis: int, is_max: bool):
    """localmax / localmin on the GPU: one launch over ``x`` viewed as [outer][n][inner] along the logical ``axis``."""
    import ctypes as C

    from numpy.lib.array_utils import normalize_axis_index

    from .. import _native as nat
    from .. import _pipeline as pl

    on_device = isinstance(x, nat.DeviceArray)
    if not on_device:
        x = np.asarray(x)
    shape, dtype = tuple(x.shape), np.dtype(x.dtype)
    ax = normalize_axis_index(axis, len(shape), msg_prefix="axis2")   # the AxisError of x.swapaxes(-1, axis)
    if dtype not in nat.ELEM_TYPES:
        raise nat.UnsupportedOnGPU(f"localmax / localmin: dtype {dtype} is not supported on the GPU (integers, float32, "
                                   "float64, bool)")
    if shape[ax] < 2:   # the reference's x[..., -2] on the rotated axis
        raise IndexError(f"index -2 is out of bounds for axis {len(shape) - 1} with size {shape[ax]}")
    layout = x.layout if on_device else "c"
    mem = shape[:-2] + (shape[-1], shape[-2]) if layout == "ft" else shape
    m = {len(shape) - 1: len(shape) - 2, len(shape) - 2: len(shape) - 1}.get(ax, ax) if layout == "ft" else ax
    outer, n, inner = pl.clip_count(mem[:m]), mem[m], pl.clip_count(mem[m + 1:])
    with pl.Scope(x) as sc:
        out = sc.empty(shape, np.bool_, layout=layout)
        if out.size:
            d_x = sc.stage(x)
            nat.check(nat.lib().b2l_localext(sc.ctx.handle, C.c_void_p(d_x.ptr), nat.ELEM_TYPES[dtype], int(is_max),
                                             outer, n, inner, C.c_void_p(out.ptr)))
        return sc.result(out)


def localmax(x, *, axis: int = 0):
    """Local maxima along ``axis``; same contract as ``librosa.util.localmax``: ``x[i] > x[i-1]`` and ``x[i] >=
    x[i+1]``, never at the first element, ``x[-1] > x[-2]`` at the last.  Computed on the GPU for integer, float32,
    float64 and bool data (other dtypes are refused with UnsupportedOnGPU).  ``x`` may be a host array or a
    DeviceArray (layout "c" or "ft"); returns a bool array of the same shape, a DeviceArray of the same layout for
    device input."""
    return _localext(x, axis, True)


def localmin(x, *, axis: int = 0):
    """Local minima along ``axis``; same contract as ``librosa.util.localmin`` (``localmax`` mirrored)."""
    return _localext(x, axis, False)
