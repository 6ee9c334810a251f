"""``melspectrogram`` and ``mfcc`` with librosa's signatures (reference:
librosa/feature/spectral.py:2022-2161 and :1843-2019), fused on the GPU:

* ``melspectrogram(y=...)`` is ONE kernel — frame, window, real FFT, ``|.|**power`` and the band-sparse
  mel projection; the STFT and power spectrogram never exist in HBM;
* ``mfcc(y=...)`` adds the dB conversion (per-clip ``top_db`` reference maximum) and the DCT.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional

import numpy as np
import scipy.fft

from .. import _f64 as f64
from .. import _native as nat
from .. import _pipeline as pl
from ..core.spectrum import power_to_db
from ..util.exceptions import ParameterError

_vp = C.c_void_p


def melspectrogram(*, y=None, sr: float = 22050, S=None, n_fft: int = 2048, hop_length: int = 512,
                   win_length: Optional[int] = None, window="hann", center: bool = True,
                   pad_mode="constant", power: float = 2.0, **kwargs):
    """Mel-scaled spectrogram, shape ``(..., n_mels, n_frames)``; same contract as
    ``librosa.feature.melspectrogram``.  ``kwargs`` go to ``filters.mel`` (n_mels, fmin, fmax, htk, norm, dtype)."""
    if S is not None:
        # mel_basis . S for a caller-supplied spectrogram (feature/spectral.py:2158-2160)
        Sd, req, on_device = pl.spectrogram_input(S)
        F, T = Sd.shape[-2], Sd.shape[-1]
        if n_fft is None or n_fft // 2 + 1 != F:
            n_fft = 2 * (F - 1)
        basis, bkey = pl.mel_basis(sr, n_fft, kwargs)
        ctx = Sd.ctx
        plan = nat.make_plan(ctx, ("melproj", n_fft, bkey), n_fft=n_fft, hop_length=1, center=True,
                             pad_mode="constant", window=np.ones(n_fft), mel_basis=basis)
        lead = Sd.shape[:-2]
        src, own = pl.to_native(Sd)
        out = nat.DeviceArray.empty(ctx, lead + (basis.shape[0], T), np.float32)
        nat.check(nat.lib().b2l_mel_project(ctx.handle, plan.handle, _vp(src.ptr), pl.clip_count(lead), T,
                                            _vp(out.ptr)))
        if own:
            src.free()
        return out if on_device else pl.finish(out, np.result_type(req, basis.dtype))
    if n_fft is None:
        raise ParameterError(f"Unable to compute spectrogram with n_fft={n_fft}")
    if y is None:
        raise ParameterError("Input signal must be provided to compute a spectrogram")
    fr = pl.forward_front(y, n_fft, hop_length, win_length, window, center, pad_mode)
    basis, bkey = pl.mel_basis(sr, n_fft, kwargs)
    res_dtype = np.result_type(fr.dtype, basis.dtype)
    if pl.wide_route(y, fr.dtype, n_fft):
        staged, mel_d = _mel_f64(y, n_fft, fr, center, power, basis)
        return staged.result(mel_d, res_dtype)
    pl.require_supported_n_fft(n_fft)
    if not pl.fused_front_end(n_fft):
        # chirp-z frames: |STFT|**power on the device, then the band-sparse projection (two kernels)
        return _compose_nonpow2(y, lambda Sd: melspectrogram(S=Sd, sr=sr, n_fft=n_fft, **kwargs), res_dtype,
                                n_fft=n_fft, hop_length=fr.hop, power=power, win_length=win_length,
                                window=window, center=center, pad_mode=pad_mode)

    def launch(ctx, plan, d_in, m, n_, d_out, d_scr):
        nat.check(nat.lib().b2l_melspectrogram(ctx.handle, plan.handle, _vp(d_in), m, n_, n_, _vp(d_out)))

    res = pl.run_forward(y, plan_key=("mel", n_fft, fr.hop, bool(center), fr.mode, fr.wkey, bkey, float(power)),
                         plan_kw=dict(n_fft=n_fft, hop_length=fr.hop, center=center, pad_mode=fr.mode, window=fr.window,
                                      mel_basis=basis, power=float(power)),
                         n_frames=fr.n_frames, out_tail=(basis.shape[0], fr.n_frames), dtype=np.float32,
                         launch=launch)
    return res if isinstance(res, nat.DeviceArray) or res.dtype == res_dtype else res.astype(res_dtype)


def _mel_f64(y, n_fft, fr, center, power, basis):
    """float64 signal -> float64 mel spectrogram on the device in FP64: stft, |.|**power, band projection
    (feature/spectral.py:2145-2160 in the input's precision).  Returns (StagedInput, DeviceArray)."""
    staged, D = f64.stft(y, n_fft=n_fft, hop_length=fr.hop, center=center, mode=fr.mode, win=fr.window)
    Sd = f64.abs_pow(staged.ctx, D, power)
    D.free()
    mel_d = f64.mel(staged.ctx, Sd, basis)
    Sd.free()
    return staged, mel_d


def _compose_nonpow2(y, tail, res_dtype, **spec_kw):
    """melspectrogram / mfcc for n_fft that is not a power of two: the chirp-z spectrogram kernel followed by
    the S= kernels, all on the device; host inputs get the device-side valid_audio verdict at the end."""
    from ..core.spectrum import _spectrogram

    staged = pl.StagedInput(y)
    Sd, _ = _spectrogram(y=staged.dev, **spec_kw)
    staged.scan_uncovered(spec_kw["n_fft"], spec_kw["hop_length"], spec_kw["win_length"], spec_kw["center"],
                          Sd.shape[-1])
    return staged.result(tail(Sd), res_dtype)


def chroma_stft(*, y=None, sr: float = 22050, S=None, norm=np.inf, n_fft: int = 2048, hop_length: int = 512,
                win_length: Optional[int] = None, window="hann", center: bool = True, pad_mode="constant",
                tuning: Optional[float] = None, n_chroma: int = 12, **kwargs):
    """Chromagram from a waveform or power spectrogram, shape ``(..., n_chroma, t)``; same contract as
    ``librosa.feature.chroma_stft`` (feature/spectral.py:1137-1293).  ``kwargs`` go to ``filters.chroma``.
    Power spectrogram, tuning estimation (when ``tuning`` is None), projection and per-frame normalisation all
    run on the device; like the reference, ONE tuning value is estimated for the whole input."""
    from .. import filters
    from ..core.pitch import _tuning_from_device_spec
    from ..core.spectrum import _spectrogram

    staged = None
    if S is None:
        if y is None:
            raise ParameterError("Input signal must be provided to compute a spectrogram")
        _, req = pl.precheck_signal(y)
        staged = pl.StagedInput(y)
        Sd, n_fft = _spectrogram(y=staged.dev, n_fft=n_fft, hop_length=hop_length, power=2, win_length=win_length,
                                 window=window, center=center, pad_mode=pad_mode)
        staged.scan_uncovered(n_fft, hop_length, win_length, center, Sd.shape[-1])
        src, own = Sd, True
    else:
        Sd, req, on_device = pl.spectrogram_input(S)
        if n_fft is None or n_fft // 2 + 1 != Sd.shape[-2]:
            n_fft = 2 * (Sd.shape[-2] - 1)
        src, own = pl.to_native(Sd)
    ctx = src.ctx
    F, T = src.shape[-2], src.shape[-1]
    lead = src.shape[:-2]
    n_clips = pl.clip_count(lead)
    L = nat.lib()
    try:
        if tuning is None:
            tuning = _tuning_from_device_spec(ctx, src, sr, n_fft, resolution=0.01, bins_per_octave=n_chroma,
                                              fmin=150.0, fmax=4000.0, threshold=0.1, ref=None)
        fb = filters.chroma(sr=sr, n_fft=n_fft, tuning=tuning, n_chroma=n_chroma, **kwargs)
        if fb.shape[1] != F:
            raise ParameterError(f"chroma filter bank has {fb.shape[1]} bins, the spectrogram {F}")
        plan = nat.make_plan(ctx, ("chroma", n_fft, pl.digest(fb)), n_fft=n_fft, hop_length=1, center=True,
                             pad_mode="constant", window=np.ones(n_fft), mel_basis=fb)
        raw = nat.DeviceArray.empty(ctx, tuple(lead) + (fb.shape[0], T), np.float32)
        nat.check(L.b2l_mel_project(ctx.handle, plan.handle, _vp(src.ptr), n_clips, T, _vp(raw.ptr)))
    finally:
        if own:
            src.free()
    if norm is None:
        out = raw
    else:
        if norm == np.inf:
            kind, p = 0, 0.0
        elif norm == -np.inf:
            kind, p = 1, 0.0
        elif norm == 0:
            kind, p = 2, 0.0
        elif np.issubdtype(type(norm), np.number) and norm > 0:
            kind, p = 3, float(norm)
        else:
            raise ParameterError(f"Unsupported norm: {repr(norm)}")
        out = nat.DeviceArray.empty(ctx, raw.shape, np.float32)
        nat.check(L.b2l_normalize_rows(ctx.handle, _vp(raw.ptr), n_clips, fb.shape[0], T, kind, p, _vp(out.ptr)))
        raw.free()
    res_dtype = np.result_type(req, fb.dtype)
    if staged is not None:
        return staged.result(out, res_dtype)
    return out if on_device else pl.finish(out, res_dtype)


def _dct_basis(n_mels: int, n_mfcc: int, dct_type: int, norm, lifter: float, dtype=np.float32) -> np.ndarray:
    """Rows 0..n_mfcc-1 of the DCT applied along the mel axis, as an explicit matrix, with the
    sinusoidal lifter ``1 + (lifter/2) sin(pi (k+1) / lifter)`` folded in
    (feature/spectral.py:2005-2015).  Built in float64 from scipy.fft.dct itself, so every
    type / norm combination SciPy accepts is covered."""
    basis = scipy.fft.dct(np.eye(n_mels, dtype=np.float64), axis=0, type=dct_type, norm=norm)[:n_mfcc]
    if lifter > 0:
        lift = 1 + (lifter / 2) * np.sin(np.pi * np.arange(1, 1 + basis.shape[0], dtype=np.float64) / lifter)
        basis = basis * lift[:, np.newaxis]
    return np.ascontiguousarray(basis, dtype=dtype)


def mfcc(*, y=None, sr: float = 22050, S=None, n_mfcc: int = 20, dct_type: int = 2, norm="ortho",
         lifter: float = 0, mel_norm="slaney", **kwargs):
    """Mel-frequency cepstral coefficients, shape ``(..., n_mfcc, n_frames)``; same contract as
    ``librosa.feature.mfcc``."""
    if not (lifter >= 0):   # also catches NaN, like the reference's final else-branch
        raise ParameterError(f"MFCC lifter={lifter} must be a non-negative number")
    if S is not None:
        Sd, req, on_device = pl.spectrogram_input(S)
        if Sd.layout != "c":
            raise ParameterError("device log-mel input must be C-ordered (..., n_mels, frames)")
        ctx = Sd.ctx
        n_mels, T = Sd.shape[-2], Sd.shape[-1]
        dct = _dct_basis(n_mels, n_mfcc, dct_type, norm, lifter)
        plan = nat.make_plan(ctx, ("dct", n_mels, pl.digest(dct)), n_fft=8, hop_length=1, center=True,
                             pad_mode="constant", window=np.ones(8),
                             mel_basis=np.zeros((n_mels, 5), dtype=np.float32), dct_basis=dct)
        lead = Sd.shape[:-2]
        out = nat.DeviceArray.empty(ctx, lead + (dct.shape[0], T), np.float32)
        nat.check(nat.lib().b2l_dct_project(ctx.handle, plan.handle, _vp(Sd.ptr), pl.clip_count(lead), T,
                                            _vp(out.ptr)))
        return out if on_device else pl.finish(out, req)
    # y path: fused stft -> |.|^power -> mel -> dB (+ per-clip max), then clamp + DCT
    n_fft = kwargs.pop("n_fft", 2048)
    hop_length = kwargs.pop("hop_length", 512)
    win_length = kwargs.pop("win_length", None)
    window = kwargs.pop("window", "hann")
    center = kwargs.pop("center", True)
    pad_mode = kwargs.pop("pad_mode", "constant")
    power = kwargs.pop("power", 2.0)
    if n_fft is None:
        raise ParameterError(f"Unable to compute spectrogram with n_fft={n_fft}")
    if y is None:
        raise ParameterError("Input signal must be provided to compute a spectrogram")
    fr = pl.forward_front(y, n_fft, hop_length, win_length, window, center, pad_mode)
    mel_kwargs = dict(kwargs)
    mel_kwargs["norm"] = mel_norm
    basis, bkey = pl.mel_basis(sr, n_fft, mel_kwargs)
    n_mels = basis.shape[0]
    res_dtype = np.result_type(fr.dtype, basis.dtype)
    if pl.wide_route(y, fr.dtype, n_fft):
        # float64 signal (or a frame length only the FP64 kernels cover): mel -> power_to_db (ref 1.0, amin 1e-10,
        # top_db 80) -> DCT, all in FP64
        staged, mel_d = _mel_f64(y, n_fft, fr, center, power, basis)
        db_d = f64.power_to_db(staged.ctx, mel_d, ref_value=1.0, amin=1e-10, top_db=80.0)
        mel_d.free()
        out = f64.dct(staged.ctx, db_d, _dct_basis(n_mels, n_mfcc, dct_type, norm, lifter, dtype=np.float64))
        db_d.free()
        return staged.result(out, res_dtype)
    dct = _dct_basis(n_mels, n_mfcc, dct_type, norm, lifter)
    pl.require_supported_n_fft(n_fft)
    if not pl.fused_front_end(n_fft):
        def tail(Sd):
            mel_d = melspectrogram(S=Sd, sr=sr, n_fft=n_fft, norm=mel_norm, **kwargs)
            return mfcc(S=power_to_db(mel_d), n_mfcc=n_mfcc, dct_type=dct_type, norm=norm, lifter=lifter)

        return _compose_nonpow2(y, tail, res_dtype, n_fft=n_fft, hop_length=fr.hop, power=power,
                                win_length=win_length, window=window, center=center, pad_mode=pad_mode)

    def launch(ctx, plan, d_in, m, n_, d_out, d_scr):
        nat.check(nat.lib().b2l_mfcc(ctx.handle, plan.handle, _vp(d_in), m, n_, n_, _vp(d_out), _vp(d_scr)))

    T = fr.n_frames
    # power_to_db defaults used by mfcc: ref=1.0, amin=1e-10, top_db=80 (feature/spectral.py:2001)
    res = pl.run_forward(y, plan_key=("mfcc", n_fft, fr.hop, bool(center), fr.mode, fr.wkey, bkey, float(power),
                                      pl.digest(dct)),
                         plan_kw=dict(n_fft=n_fft, hop_length=fr.hop, center=center, pad_mode=fr.mode, window=fr.window,
                                      mel_basis=basis, power=float(power), dct_basis=dct, amin=1e-10, ref_value=1.0,
                                      top_db=80.0),
                         n_frames=T, out_tail=(dct.shape[0], T), dtype=np.float32, launch=launch,
                         scratch_per_clip=n_mels * ((T + 63) // 64 * 64))
    return res if isinstance(res, nat.DeviceArray) or res.dtype == res_dtype else res.astype(res_dtype)
