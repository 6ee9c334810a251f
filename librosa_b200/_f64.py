"""Double-precision path (C ABI: ``b2l_stft_f64`` ... ``b2l_f64_dct``, csrc/f64_kernels.cuh).

librosa computes float64 audio in float64 — complex128 STFT (core/spectrum.py:341), float64 spectrogram, mel
(feature/spectral.py:2160), dB (core/spectrum.py:1866-1881) and MFCC (feature/spectral.py:2005) — and most of
its own tests use float64 signals.  With ``B2L_FLOAT64=native`` (the default) the drop-in does the same on the
GPU in FP64: a correctness path next to the float32 hot path, not a throughput path.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional

import numpy as np

from . import _native as nat
from . import _pipeline as pl
from . import filters
from .util.exceptions import ParameterError
from .util.utils import fix_length, tiny

_vp = C.c_void_p
_dp = C.POINTER(C.c_double)

MAX_FFT = 1 << 20    # power-of-two n_fft: in-place FFT (shared memory up to 16384, global memory above)
MAX_DFT = 1 << 16    # any other n_fft: direct O(n_fft^2) DFT


def supported(n_fft: int) -> bool:
    n_fft = int(n_fft)
    pow2 = n_fft > 0 and (n_fft & (n_fft - 1)) == 0
    return (pow2 and 4 <= n_fft <= MAX_FFT) or (2 <= n_fft <= MAX_DFT)


def require_supported(n_fft: int):
    if not supported(n_fft):
        raise nat.UnsupportedOnGPU(f"float64: n_fft={n_fft} is outside the FP64 kernels' range (powers of two up to "
                                   f"{MAX_FFT}, other sizes up to {MAX_DFT}; no CPU fallback)")


def stft(y, *, n_fft, hop_length, center, mode, win: np.ndarray):
    """complex128 STFT of a float64 signal batch ``(..., n)``, host or device -> (its StagedInput, DeviceArray
    ``(..., F, T)`` in the native ``[frame][bin]`` memory layout).  ``staged.result`` gives the caller's value."""
    require_supported(n_fft)
    staged = pl.StagedInput(y, np.float64)
    ctx, n = staged.ctx, staged.n
    n_frames = pl.frame_count(n, n_fft, hop_length, center)
    D = nat.DeviceArray.empty(ctx, staged.lead + (1 + n_fft // 2, n_frames), np.complex128, layout="ft")
    w = np.ascontiguousarray(win, dtype=np.float64)
    nat.check(nat.lib().b2l_stft_f64(ctx.handle, _vp(staged.dev.ptr), staged.n_clips, n, n, int(n_fft),
                                     int(hop_length), 1 if center else 0, nat.PAD_MODES[mode], w.ctypes.data_as(_dp),
                                     _vp(D.ptr)))
    staged.scan_uncovered(n_fft, hop_length, None, center, n_frames)   # samples no frame reads (host signals only)
    staged.release()
    return staged, D


def inv_wss(window, n_frames, win_length, n_fft, hop_length, start, out_len) -> np.ndarray:
    """Reciprocal trimmed window-sum-square in float64 (core/spectrum.py:606-624)."""
    wss = filters.window_sumsquare(window=window, n_frames=n_frames, win_length=win_length, n_fft=n_fft,
                                   hop_length=hop_length, dtype=np.float64)
    wss = fix_length(wss[start:], size=out_len)
    inv = np.ones(out_len, dtype=np.float64)
    nz = wss > tiny(wss)
    inv[nz] = 1.0 / wss[nz]
    return inv


def istft(ctx, Dd: nat.DeviceArray, *, n_frames_used, n_fft, hop_length, center, win, inv, out_len) -> nat.DeviceArray:
    lead = tuple(Dd.shape[:-2])
    T_stored = Dd.shape[-1]
    y = nat.DeviceArray.empty(ctx, lead + (out_len,), np.float64)
    w = np.ascontiguousarray(win, dtype=np.float64)
    iv = np.ascontiguousarray(inv, dtype=np.float64)
    nat.check(nat.lib().b2l_istft_f64(ctx.handle, _vp(Dd.ptr), pl.clip_count(lead), T_stored, int(n_frames_used),
                                      int(n_fft), int(hop_length), 1 if center else 0, w.ctypes.data_as(_dp),
                                      iv.ctypes.data_as(_dp), int(out_len), _vp(y.ptr), int(out_len)))
    return y


def abs_pow(ctx, Dd: nat.DeviceArray, power: float) -> nat.DeviceArray:
    S = nat.DeviceArray.empty(ctx, Dd.shape, np.float64, layout=Dd.layout)
    nat.check(nat.lib().b2l_f64_abs_pow(ctx.handle, _vp(Dd.ptr), Dd.size, float(power), _vp(S.ptr)))
    return S


def mel(ctx, Sd: nat.DeviceArray, basis: np.ndarray) -> nat.DeviceArray:
    """``Sd`` (..., F, T) in the native [frame][bin] layout -> (..., n_mels, T) C-ordered float64."""
    if Sd.layout != "ft":
        raise ParameterError("float64 mel projection expects the native [frame][bin] layout")
    lead, F, T = tuple(Sd.shape[:-2]), Sd.shape[-2], Sd.shape[-1]
    b = np.ascontiguousarray(basis, dtype=np.float32)
    if b.shape[1] != F:
        raise ParameterError(f"mel basis has {b.shape[1]} bins, the spectrogram {F}")
    out = nat.DeviceArray.empty(ctx, lead + (b.shape[0], T), np.float64)
    nat.check(nat.lib().b2l_f64_mel(ctx.handle, _vp(Sd.ptr), pl.clip_count(lead), T, F,
                                    b.ctypes.data_as(C.POINTER(C.c_float)), b.shape[0], _vp(out.ptr)))
    return out


def power_to_db(ctx, Sd: nat.DeviceArray, *, ref_value: float, amin: float, top_db: Optional[float]) -> nat.DeviceArray:
    """dB of a (..., rows, frames) float64 device array; the ``top_db`` maximum is per leading index."""
    lead = tuple(Sd.shape[:-2])
    per = Sd.shape[-2] * Sd.shape[-1]
    out = nat.DeviceArray.empty(ctx, Sd.shape, np.float64, layout=Sd.layout)
    nat.check(nat.lib().b2l_f64_db(ctx.handle, _vp(Sd.ptr), pl.clip_count(lead), per, float(amin), float(ref_value),
                                   -1.0 if top_db is None else float(top_db), _vp(out.ptr)))
    return out


def dct(ctx, Ld: nat.DeviceArray, basis64: np.ndarray) -> nat.DeviceArray:
    lead, n_mels, T = tuple(Ld.shape[:-2]), Ld.shape[-2], Ld.shape[-1]
    b = np.ascontiguousarray(basis64, dtype=np.float64)
    out = nat.DeviceArray.empty(ctx, lead + (b.shape[0], T), np.float64)
    nat.check(nat.lib().b2l_f64_dct(ctx.handle, _vp(Ld.ptr), pl.clip_count(lead), n_mels, T, b.ctypes.data_as(_dp),
                                    b.shape[0], _vp(out.ptr)))
    return out
