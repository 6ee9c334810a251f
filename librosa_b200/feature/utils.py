"""``librosa.feature.delta`` and ``stack_memory`` (reference: librosa/feature/utils.py), one kernel launch each.

``delta`` is ``scipy.signal.savgol_filter`` along one axis.  Its coefficients come from SciPy's own
``savgol_coeffs`` on the host; the kernel (csrc/featutil_kernels.cuh) applies them in scipy.ndimage's order and
precision, so every output that ndimage computes is bit-identical to the reference.  The exception is
``mode="interp"``: SciPy fits the first and last ``width`` samples of a line in the data's precision, while this
module applies the exact float64 fit map (``edge_map``).  The two agree within a few ``eps(dtype) * cond(V) *
max|x|`` of the edge window, where ``V`` is the column-normalised Vandermonde matrix of the fit; for a float32 fit
of high polynomial order the float64 map is the more accurate one.

``stack_memory`` is one gather.  Both functions decide ``np.pad``'s semantics in one place, ``pad_index_table``:
the source index of every padded position, computed by ``np.pad`` on an index vector."""
from __future__ import annotations

import ctypes as C
import functools
import math

import numpy as np
from numpy.lib.array_utils import normalize_axis_index

from .. import _native as nat
from .. import _pipeline as pl
from ..util.exceptions import ParameterError

_vp = C.c_void_p

__all__ = ["delta", "stack_memory"]

# scipy.ndimage's boundary modes as np.pad modes; interp's interior is the constant convolution with cval = 0
_NDIMAGE_PAD = {"mirror": "reflect", "nearest": "edge", "wrap": "wrap", "constant": "constant", "interp": "constant"}
# np.pad modes that compute new values instead of copying samples
_COMPUTED_PAD = ("linear_ramp", "maximum", "mean", "median", "minimum")


def pad_index_table(n: int, before: int, after: int, mode: str, **kwargs) -> np.ndarray:
    """Where each padded position of an axis of ``n`` samples comes from under ``np.pad(x, (before, after), mode,
    **kwargs)``: int64 ``[before + after]`` for positions ``-before .. -1`` then ``n .. n + after - 1``, holding the
    source sample, or -1 for the constant ("constant"; "empty" is read as the constant too)."""
    idx = np.arange(n, dtype=np.int64)
    if mode in ("constant", "empty"):
        full = np.pad(idx, (before, after), mode="constant", constant_values=-1)
    else:
        full = np.pad(idx, (before, after), mode=mode, **kwargs)
    return np.ascontiguousarray(np.concatenate([full[:before], full[before + n:]]), dtype=np.int64)


def classify_taps(fw: np.ndarray) -> int:
    """scipy.ndimage's test of correlation weights of odd length: 1 symmetric, -1 antisymmetric, 0 neither.  Pairs
    agree when they differ by at most DBL_EPSILON in absolute terms (a NaN difference passes, as in the C test)."""
    h = len(fw) // 2
    eps = np.finfo(np.float64).eps
    right, left = fw[h + 1:], fw[:h][::-1]
    if not np.any(np.abs(right - left) > eps):
        return 1
    if not np.any(np.abs(right + left) > eps):
        return -1
    return 0


def edge_map(width: int, polyorder: int, deriv: int, delta: float) -> np.ndarray:
    """float64 ``[width - 1][width]``: savgol_filter(mode="interp")'s first ``h`` outputs of a line as a linear map of
    its first ``width`` samples (rows 0 .. h-1), and its last ``h`` outputs of its last ``width`` samples (rows h ..):
    the degree-``polyorder`` least-squares fit, differentiated ``deriv`` times, divided by ``delta ** deriv``."""
    h = width // 2
    t = np.arange(width, dtype=np.float64)
    V = t[:, None] ** np.arange(polyorder + 1)
    scale = np.sqrt((V * V).sum(axis=0))   # unit-norm columns, as SciPy's polyfit scales them
    fit = np.linalg.pinv(V / scale) / scale[:, None]   # polynomial coefficients from samples
    der = np.zeros((width, polyorder + 1))
    for q in range(deriv, polyorder + 1):
        der[:, q] = math.perm(q, deriv) * t ** (q - deriv)
    full = (der @ fit) / (delta ** deriv)
    return np.ascontiguousarray(np.concatenate([full[:h], full[width - h:]]))


# The host tables of one configuration, with their digests (the keys of their device copies), cached: building them
# takes longer than the kernel that reads them.
@functools.lru_cache(maxsize=64)
def _taps(width, polyorder, deriv, delta):
    """(fw, symmetry class, digest): savgol_coeffs reversed, as ndimage.convolve1d applies them (SciPy's errors pass)."""
    from scipy.signal import savgol_coeffs

    fw = np.ascontiguousarray(np.asarray(savgol_coeffs(width, polyorder, deriv=deriv, delta=delta), np.float64)[::-1])
    return fw, classify_taps(fw), pl.digest(fw)


@functools.lru_cache(maxsize=64)
def _pad_table(n, before, after, mode):
    table = pad_index_table(n, before, after, mode)
    return table, pl.digest(table)


@functools.lru_cache(maxsize=16)
def _edge_table(width, polyorder, deriv, delta):
    E = edge_map(width, polyorder, deriv, delta)
    return E, pl.digest(E)


def _shape_dtype(x):
    """(logical shape, at least 1-D; dtype) of a host array or DeviceArray."""
    return (tuple(x.shape) or (1,)), np.dtype(x.dtype)


def savgol_filter(x, window_length, polyorder, deriv=0, delta=1.0, axis=-1, mode="interp", cval=0.0):
    """``scipy.signal.savgol_filter`` with its signature, checks and errors, computed on the GPU (the call
    ``delta`` makes).  ``x`` is a host array (float32 and float64 kept, anything else computed as float64) or a
    float32 / float64 DeviceArray in layout "c" or "ft", filtered along the logical ``axis``.  Returns a NumPy
    array for host input, a DeviceArray of the input's layout for device input."""
    if mode not in ["mirror", "constant", "nearest", "interp", "wrap"]:
        raise ValueError("mode must be 'mirror', 'constant', 'nearest' 'wrap' or 'interp'.")
    on_device = isinstance(x, nat.DeviceArray)
    if not on_device:
        x = np.asarray(x)
    shape, dtype = _shape_dtype(x)
    fw, sym, fw_key = _taps(window_length, polyorder, deriv, delta)
    if mode == "interp" and window_length > shape[axis]:
        raise ValueError("If mode is 'interp', window_length must be less than or equal to the size of x.")
    ax = normalize_axis_index(axis, len(shape))
    if dtype.kind == "c":
        raise nat.UnsupportedOnGPU("delta: complex data is not filtered on the GPU (SciPy would discard the imaginary "
                                   "part); pass its real part")
    if on_device and dtype not in (np.float32, np.float64):
        raise nat.UnsupportedOnGPU(f"delta: device data must be float32 or float64, got {dtype}")
    if window_length > nat.DELTA_MAX_WIDTH:
        raise nat.UnsupportedOnGPU(f"delta: width={window_length} exceeds the {nat.DELTA_MAX_WIDTH} taps the GPU "
                                   "kernels hold in shared memory")
    if dtype not in (np.float32, np.float64):
        dtype = np.dtype(np.float64)
    h, interp = window_length // 2, mode == "interp"
    layout = x.layout if on_device else "c"
    mem = shape[:-2] + (shape[-1], shape[-2]) if layout == "ft" else shape
    swap = {len(shape) - 1: len(shape) - 2, len(shape) - 2: len(shape) - 1} if layout == "ft" else {}
    m = swap.get(ax, ax)   # the filtered axis in memory order
    outer, n, inner = pl.clip_count(mem[:m]), mem[m], pl.clip_count(mem[m + 1:])
    with pl.Scope(x) as sc:
        out = sc.empty(shape, dtype, layout=layout)
        if out.size == 0:
            return sc.result(out)
        d_x = sc.stage(x, dtype)
        ctx = sc.ctx
        desc = nat.DeltaDesc(width=window_length, sym=sym, interp=int(interp), f64=int(dtype == np.float64),
                             cval=float(cval))
        desc.d_taps = pl.f64_constant(ctx, ("delta_taps", fw_key), fw)
        pad, pad_key = _pad_table(n, h, h, _NDIMAGE_PAD[mode])
        desc.d_pad = pl.f64_constant(ctx, ("delta_pad", pad_key), pad)
        if interp:
            E, e_key = _edge_table(window_length, polyorder, deriv, delta)
            desc.d_edge = pl.f64_constant(ctx, ("delta_edge", e_key), E)
            nat.check(nat.lib().b2l_status_reset(ctx.handle))
        nat.check(nat.lib().b2l_delta(ctx.handle, C.byref(desc), _vp(d_x.ptr), outer, n, inner, _vp(out.ptr)))
        if interp and pl.status_word(ctx) & nat.STATUS_NOT_FINITE_VALUE:
            raise ValueError("array must not contain infs or NaNs")   # SciPy's fit of the edges (lstsq)
        return sc.result(out)


def delta(data, *, width: int = 9, order: int = 1, axis: int = -1, mode="interp", **kwargs):
    """Local estimate of the derivative of ``data`` along ``axis`` by Savitzky-Golay filtering; same contract as
    ``librosa.feature.delta``.

    ``data`` may be a host array or a float32 / float64 DeviceArray in layout "c" or "ft"; device input gives a
    DeviceArray of the same layout.  ``kwargs`` are ``savgol_filter``'s ``polyorder``, ``delta`` and ``cval``
    (``deriv`` is dropped, as in the reference).  Every output is bit-identical to the reference except, under
    ``mode="interp"``, the first and last ``width // 2`` of each line, which use the float64 fit (module docstring).
    """
    if not isinstance(data, nat.DeviceArray):
        data = np.atleast_1d(data)
    shape, _ = _shape_dtype(data)
    if mode == "interp" and width > shape[axis]:
        raise ParameterError(f"when mode='interp', width={width} cannot exceed data.shape[axis]={shape[axis]}")
    if width < 3 or np.mod(width, 2) != 1:
        raise ParameterError("width must be an odd integer >= 3")
    if order <= 0 or not isinstance(order, (int, np.integer)):
        raise ParameterError("order must be a positive integer")
    kwargs.pop("deriv", None)
    kwargs.setdefault("polyorder", order)
    return savgol_filter(data, width, deriv=order, axis=axis, mode=mode, **kwargs)


def stack_memory(data, *, n_steps: int = 2, delay: int = 1, **kwargs):
    """Short-term history embedding: ``data`` (..., d, t) stacked with ``n_steps - 1`` delayed copies of itself into
    (..., n_steps * d, t); same contract as ``librosa.feature.stack_memory``.

    ``kwargs`` go to ``np.pad`` (default: zeros).  Its modes that copy samples ("constant", "edge", "reflect",
    "symmetric", "wrap", "empty", whose cells are zeros here) run on the GPU; the modes that compute values
    ("linear_ramp", "maximum", "mean", "median", "minimum", ``reflect_type="odd"``, callables) are refused with
    UnsupportedOnGPU.  Any dtype of 1, 2, 4, 8 or 16 bytes is gathered as it is.  Host input gives a C-ordered NumPy
    array; a DeviceArray (layout "c" or "ft") gives a C-ordered DeviceArray."""
    if n_steps < 1:
        raise ParameterError("n_steps must be a positive integer")
    if delay == 0:
        raise ParameterError("delay must be a non-zero integer")
    on_device = isinstance(data, nat.DeviceArray)
    if not on_device:
        data = np.atleast_2d(data)
    shape, dtype = tuple(data.shape), np.dtype(data.dtype)
    shape = (1,) * (2 - len(shape)) + shape
    t = shape[-1]
    if t < 1:
        raise ParameterError(f"Cannot stack memory when input data has no columns. Given data.shape={shape}")
    kwargs.setdefault("mode", "constant")
    if kwargs["mode"] == "constant":
        kwargs.setdefault("constant_values", [0])
    mode = kwargs["mode"]
    n_pad = int((n_steps - 1) * abs(delay))
    padding = [(0, 0)] * (len(shape) - 1) + [(n_pad, 0) if delay > 0 else (0, n_pad)]
    if callable(mode):
        raise nat.UnsupportedOnGPU("stack_memory: a callable pad mode computes values on the host; the GPU gathers "
                                   "samples only")
    if dtype.kind == "O" or dtype.itemsize not in (1, 2, 4, 8, 16):
        raise nat.UnsupportedOnGPU(f"stack_memory: dtype {dtype} is not gathered on the GPU (elements of 1, 2, 4, 8 "
                                   "or 16 bytes, no objects)")
    # np.pad's own checks of mode and kwargs, and the constant cast as np.pad casts it, on a one-element stand-in
    stand_in = np.pad(np.zeros((1,) * len(shape), dtype=dtype), padding, **kwargs)
    if mode in _COMPUTED_PAD or (mode in ("reflect", "symmetric") and kwargs.get("reflect_type") == "odd"):
        raise nat.UnsupportedOnGPU(f"stack_memory: pad mode {mode!r} computes values; the GPU gathers samples only "
                                   "(constant, edge, reflect, symmetric, wrap, empty)")
    extra = {"reflect_type": kwargs["reflect_type"]} if "reflect_type" in kwargs else {}
    table = pad_index_table(t, *padding[-1], mode, **extra)
    desc = nat.StackDesc(elem_size=dtype.itemsize, n_steps=int(n_steps), delay=int(delay))
    if mode == "constant" and n_pad:
        fill = np.ascontiguousarray(stand_in.reshape(-1)[0 if delay > 0 else -1]).tobytes()
        C.memmove(desc.fill, fill, len(fill))
    d, lead = shape[-2], shape[:-2]
    ft = on_device and data.layout == "ft"
    desc.clip_stride, desc.row_stride, desc.col_stride = d * t, (1 if ft else t), (d if ft else 1)
    with pl.Scope(data) as sc:
        out = sc.empty(lead + (n_steps * d, t), dtype)
        if out.size == 0:
            return sc.result(out)
        d_x = sc.stage(data)
        ctx = sc.ctx
        d_pad = pl.f64_constant(ctx, ("stack_pad", pl.digest(table)), table)
        nat.check(nat.lib().b2l_stack_memory(ctx.handle, C.byref(desc), _vp(d_x.ptr), pl.clip_count(lead), d, t,
                                             _vp(d_pad), _vp(out.ptr)))
        return sc.result(out)
