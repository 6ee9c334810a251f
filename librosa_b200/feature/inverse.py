"""``librosa.feature.inverse`` on the device (reference: librosa/feature/inverse.py:28-381).

* ``mel_to_stft``  — non-negative least squares per frame on the band-sparse mel basis (``b2l_nnls_mel``): the
  reference's start point ``max(0, pinv(A) M)`` refined by accelerated projected-gradient steps instead of SciPy's
  L-BFGS-B (the problem is under-determined: any minimiser is as good; the reference's test bounds the residual);
* ``mfcc_to_mel``  — inverse DCT as an explicit matrix (lifter folded in) + ``db_to_power``, both existing kernels;
* ``mel_to_audio`` / ``mfcc_to_audio`` — the above followed by the device Griffin-Lim iteration.
"""
from __future__ import annotations

import ctypes as C
import warnings
from functools import lru_cache
from typing import Optional

import numpy as np
import scipy.fft

from .. import _native as nat
from .. import _pipeline as pl
from .. import filters
from ..core.spectrum import db_to_power, griffinlim
from ..util.exceptions import ParameterError
from ..util.utils import tiny

_vp = C.c_void_p
_fp = C.POINTER(C.c_float)

NNLS_ITERATIONS = 100   # FISTA steps after the projected least-squares start (residual <= L-BFGS-B's, see tests)


@lru_cache(maxsize=16)
def _nnls_constants(sr, n_fft, n_mels, items):
    """(basis, pinv, step) of one mel configuration: float64 SVD on the host, float32 tables for the kernel."""
    basis = filters.mel(sr=sr, n_fft=n_fft, n_mels=n_mels, dtype=np.float32, **dict(items))
    b64 = basis.astype(np.float64)
    sigma = np.linalg.svd(b64, compute_uv=False)
    pinv = np.linalg.pinv(b64)
    step = 1.0 / float(sigma[0]) ** 2
    return (np.ascontiguousarray(basis, dtype=np.float32), np.ascontiguousarray(pinv, dtype=np.float32), step)


def mel_to_stft(M, *, sr: float = 22050, n_fft: int = 2048, power: float = 2.0, **kwargs):
    """Approximate STFT magnitude ``(..., 1 + n_fft/2, T)`` from a mel power spectrogram ``(..., n_mels, T)``;
    same contract as ``librosa.feature.inverse.mel_to_stft``."""
    on_device = isinstance(M, nat.DeviceArray)
    if not on_device:
        M = np.asarray(M)
        if not np.issubdtype(M.dtype, np.floating):
            M = M.astype(np.float32)
    if M.ndim < 2:
        raise ParameterError("mel spectrogram must have at least two dimensions (n_mels, frames)")
    if not (power > 0):
        raise ParameterError(f"power={power} must be strictly positive")
    req = np.dtype(np.float32) if on_device else pl.check_real_dtype(M.dtype, "mel_to_stft input")
    n_mels, T = M.shape[-2], M.shape[-1]
    kwargs.pop("dtype", None)
    try:
        basis, pinv, step = _nnls_constants(float(sr), int(n_fft), int(n_mels), tuple(sorted(kwargs.items())))
    except TypeError:   # unhashable kwarg
        basis, pinv, step = _nnls_constants.__wrapped__(float(sr), int(n_fft), int(n_mels), tuple(kwargs.items()))
    F = basis.shape[1]
    ctx = M.ctx if on_device else nat.default_context()
    if on_device:
        if M.dtype != np.float32 or M.layout != "c":
            raise ParameterError("device mel spectrogram must be C-ordered float32")
        Md = M
    else:
        Md = ctx.to_device(np.ascontiguousarray(M, dtype=np.float32))
    lead = tuple(M.shape[:-2])
    out = nat.DeviceArray.empty(ctx, lead + (F, T), np.float32)
    nat.check(nat.lib().b2l_nnls_mel(ctx.handle, _vp(Md.ptr), pl.clip_count(lead), T, n_mels, F,
                                     basis.ctypes.data_as(_fp), pinv.ctypes.data_as(_fp), float(step), NNLS_ITERATIONS,
                                     float(1.0 / power), _vp(out.ptr)))
    if on_device:
        return out
    res = pl.finish(out, req)
    Md.free()
    return res


def mel_to_audio(M, *, sr: float = 22050, n_fft: int = 2048, hop_length: Optional[int] = None,
                 win_length: Optional[int] = None, window="hann", center: bool = True, pad_mode="constant",
                 power: float = 2.0, n_iter: int = 32, length: Optional[int] = None, dtype=np.float32, **kwargs):
    """Invert a mel power spectrogram to audio with Griffin-Lim; same contract as
    ``librosa.feature.inverse.mel_to_audio`` (feature/inverse.py:117-211)."""
    stft = mel_to_stft(M, sr=sr, n_fft=n_fft, power=power, **kwargs)
    return griffinlim(stft, n_iter=n_iter, hop_length=hop_length, win_length=win_length, n_fft=n_fft, window=window,
                      center=center, dtype=dtype, length=length, pad_mode=pad_mode)


def _idct_basis(n_mfcc: int, n_mels: int, dct_type: int, norm, lifter: float, dtype) -> np.ndarray:
    """``scipy.fft.idct(., axis=-2, type, norm, n=n_mels)`` of (de-liftered) MFCCs as an explicit
    ``(n_mels, n_mfcc)`` matrix (feature/inverse.py:268-286)."""
    basis = scipy.fft.idct(np.eye(n_mfcc, dtype=np.float64), axis=0, type=dct_type, norm=norm, n=n_mels)
    if lifter > 0:
        idx = np.arange(1, 1 + n_mfcc, dtype=dtype)
        lifter_sine = 1 + lifter * 0.5 * np.sin(np.pi * idx / lifter)
        if np.any(np.abs(lifter_sine) < np.finfo(lifter_sine.dtype).eps):
            warnings.warn(message="lifter array includes critical values that may invoke underflow.",
                          category=UserWarning, stacklevel=3)
        basis = basis / (lifter_sine.astype(np.float64) + float(tiny(np.zeros(1, dtype=dtype))))[np.newaxis, :]
    elif lifter != 0:
        raise ParameterError("MFCC to mel lifter must be a non-negative number.")
    return np.ascontiguousarray(basis, dtype=np.float32)


def mfcc_to_mel(mfcc, *, n_mels: int = 128, dct_type: int = 2, norm="ortho", ref: float = 1.0, lifter: float = 0):
    """Invert MFCCs to a mel power spectrogram ``(..., n_mels, T)``; same contract as
    ``librosa.feature.inverse.mfcc_to_mel`` (feature/inverse.py:214-287)."""
    on_device = isinstance(mfcc, nat.DeviceArray)
    if not on_device:
        mfcc = np.asarray(mfcc)
        if not np.issubdtype(mfcc.dtype, np.floating):
            mfcc = mfcc.astype(np.float32)
    if mfcc.ndim < 2:
        raise ParameterError("mfcc must have at least two dimensions (n_mfcc, frames)")
    if not (lifter >= 0):
        raise ParameterError("MFCC to mel lifter must be a non-negative number.")
    n_mfcc, T = mfcc.shape[-2], mfcc.shape[-1]
    basis = _idct_basis(n_mfcc, n_mels, dct_type, norm, lifter, np.float32 if on_device else mfcc.dtype)
    req = np.dtype(np.float32) if on_device else pl.check_real_dtype(mfcc.dtype, "mfcc_to_mel input")
    ctx = mfcc.ctx if on_device else nat.default_context()
    if on_device:
        if mfcc.dtype != np.float32 or mfcc.layout != "c":
            raise ParameterError("device mfcc must be C-ordered float32")
        Cd = mfcc
    else:
        Cd = ctx.to_device(np.ascontiguousarray(mfcc, dtype=np.float32))
    # the matrix product runs on the DCT kernel: "mel rows" = n_mfcc inputs, "coefficients" = n_mels outputs
    plan = nat.make_plan(ctx, ("idct", n_mfcc, pl.digest(basis)), n_fft=8, hop_length=1, center=True,
                         pad_mode="constant", window=np.ones(8),
                         mel_basis=np.zeros((n_mfcc, 5), dtype=np.float32), dct_basis=basis)
    lead = tuple(mfcc.shape[:-2])
    logmel = nat.DeviceArray.empty(ctx, lead + (n_mels, T), np.float32)
    nat.check(nat.lib().b2l_dct_project(ctx.handle, plan.handle, _vp(Cd.ptr), pl.clip_count(lead), T,
                                        _vp(logmel.ptr)))
    mel = db_to_power(logmel, ref=ref)
    logmel.free()
    if on_device:
        return mel
    Cd.free()
    return pl.finish(mel, req)


def mfcc_to_audio(mfcc, *, n_mels: int = 128, dct_type: int = 2, norm="ortho", ref: float = 1.0, lifter: float = 0,
                  **kwargs):
    """MFCCs -> mel -> STFT magnitude -> audio; same contract as ``librosa.feature.inverse.mfcc_to_audio``
    (feature/inverse.py:290-381).  ``kwargs`` go to ``mel_to_audio``."""
    mel_spec = mfcc_to_mel(mfcc, n_mels=n_mels, dct_type=dct_type, norm=norm, ref=ref, lifter=lifter)
    return mel_to_audio(mel_spec, **kwargs)
