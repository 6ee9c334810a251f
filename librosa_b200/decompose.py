"""``librosa.decompose.hpss`` with librosa's signature (reference: librosa/decompose.py:241-389): both median
filters, the two soft masks and the masked spectrograms come out of ONE kernel (``hpss_kernel``: the filter
window of every element is sorted in registers by a compile-time bitonic network)."""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _native as nat
from . import _pipeline as pl
from .util.exceptions import ParameterError

_vp = C.c_void_p

__all__ = ["hpss"]


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
