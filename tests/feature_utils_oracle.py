"""NumPy restatement of feature.delta and feature.stack_memory in the order the GPU kernels compute them
(csrc/featutil_kernels.cuh).  It reproduces tests/golden/feature_utils_v1.npz bit for bit, apart from the interp edges
of delta, and the kernels reproduce it bit for bit everywhere.

delta: savgol_coeffs on the host, reversed; ndimage's symmetry test; the line padded by np.pad in the matching mode,
widened to float64; the correlation summed in ndimage's order (NumPy's float64 multiplies and adds are separately
rounded, like the kernel's __dmul_rn / __dadd_rn); one rounding to the output dtype.  The interp edges apply the
float64 least-squares fit map E to the first / last ``width`` samples, in ascending order.

stack_memory: np.pad of the data, then block s of the output is the padded data shifted by s * delay."""
from __future__ import annotations

import math

import numpy as np
from scipy.signal import savgol_coeffs

import feature_utils_cases as FU

_PAD = {"mirror": "reflect", "nearest": "edge", "wrap": "wrap", "constant": "constant", "interp": "constant"}


def symmetry(fw) -> int:
    """1 symmetric, -1 antisymmetric, 0 neither: ndimage's DBL_EPSILON test of each pair around the centre."""
    h = len(fw) // 2
    eps = np.finfo(np.float64).eps
    if all(not abs(fw[h + i] - fw[h - i]) > eps for i in range(1, h + 1)):
        return 1
    if all(not abs(fw[h + i] + fw[h - i]) > eps for i in range(1, h + 1)):
        return -1
    return 0


def fit_map(width, polyorder, deriv, delta):
    """[width][width] float64: the value of the deriv-th derivative of the least-squares polynomial at every sample
    position, as a map of the samples (pinv of the Vandermonde matrix)."""
    t = np.arange(width, dtype=np.float64)
    V = t[:, None] ** np.arange(polyorder + 1)
    scale = np.sqrt((V * V).sum(axis=0))
    fit = np.linalg.pinv(V / scale) / scale[:, None]
    der = np.zeros((width, polyorder + 1))
    for q in range(deriv, polyorder + 1):
        der[:, q] = math.perm(q, deriv) * t ** (q - deriv)
    return (der @ fit) / (delta ** deriv)


def _correlate(xp, fw, h, n):
    """ndimage's correlation of every line of the padded float64 xp [..., n + 2h] in its summation order."""
    c = lambda jj: xp[..., h + jj:h + jj + n]   # noqa: E731  (sample jj away from each output)
    sym = symmetry(fw)
    if sym:
        acc = c(0) * fw[h]
        for jj in range(-h, 0):
            pair = c(jj) + c(-jj) if sym > 0 else c(jj) - c(-jj)
            acc = acc + pair * fw[h + jj]
        return acc
    acc = c(h) * fw[2 * h]
    for jj in range(-h, h):
        acc = acc + c(jj) * fw[h + jj]
    return acc


def _edge(xw, rows):
    """rows [k][width] applied to windows xw [..., width]: [..., k], ascending and unfused."""
    acc = xw[..., None, 0] * rows[:, 0]
    for k in range(1, rows.shape[1]):
        acc = acc + xw[..., None, k] * rows[:, k]
    return acc


def delta(x, width=9, order=1, axis=-1, mode="interp", polyorder=None, delta=1.0, cval=0.0, deriv=None):
    """feature.delta of the host array x (arguments already checked by the reference)."""
    x = np.atleast_1d(x)
    dtype = x.dtype if x.dtype in (np.float32, np.float64) else np.dtype(np.float64)
    polyorder = order if polyorder is None else polyorder
    fw = np.asarray(savgol_coeffs(width, polyorder, deriv=order, delta=delta), dtype=np.float64)[::-1]
    h = width // 2
    line = np.moveaxis(x.astype(np.float64), axis, -1)
    n = line.shape[-1]
    pad = [(0, 0)] * (line.ndim - 1) + [(h, h)]
    if _PAD[mode] == "constant":
        xp = np.pad(line, pad, mode="constant", constant_values=0.0 if mode == "interp" else float(cval))
    else:
        xp = np.pad(line, pad, mode=_PAD[mode])
    y = _correlate(xp, fw, h, n)
    if mode == "interp":
        E = fit_map(width, polyorder, order, delta)
        y[..., :h] = _edge(line[..., :width], E[:h])
        y[..., n - h:] = _edge(line[..., n - width:], E[width - h:])
    return np.ascontiguousarray(np.moveaxis(y.astype(dtype), -1, axis))


def stack_memory(x, n_steps=2, delay=1, **kwargs):
    """feature.stack_memory of the host array x."""
    x = np.atleast_2d(x)
    t, d = x.shape[-1], x.shape[-2]
    kwargs.setdefault("mode", "constant")
    if kwargs["mode"] == "constant":
        kwargs.setdefault("constant_values", [0])
    p = (n_steps - 1) * abs(delay)
    xp = np.pad(x, [(0, 0)] * (x.ndim - 1) + [(p, 0) if delay > 0 else (0, p)], **kwargs)
    out = np.empty(x.shape[:-2] + (n_steps * d, t), dtype=x.dtype)
    for s in range(n_steps):
        start = p - s * delay if delay > 0 else -s * delay
        out[..., s * d:(s + 1) * d, :] = xp[..., start:start + t]
    return out


def run(case):
    """The oracle's output of one fixture case."""
    x = FU.data(case["spec"])
    return delta(x, **case["kw"]) if case["fn"] == "delta" else stack_memory(x, **case["kw"])


def interp_edges(case):
    """(axis, h) of a delta case whose first / last h outputs along axis are interp edges, else None."""
    kw = case["kw"]
    if case["fn"] != "delta" or kw.get("mode", "interp") != "interp":
        return None
    return kw.get("axis", -1), kw.get("width", 9) // 2
