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
        with pl.Scope(S) as sc:
            Sd, req = sc.spectrogram(S)
            F, T = Sd.shape[-2], Sd.shape[-1]
            if n_fft is None or n_fft // 2 + 1 != F:
                n_fft = 2 * (F - 1)
            basis, bkey = pl.mel_basis(sr, n_fft, kwargs)
            ctx = sc.ctx
            plan = nat.make_plan(ctx, ("melproj", n_fft, bkey), n_fft=n_fft, hop_length=1, center=True,
                                 pad_mode="constant", window=np.ones(n_fft), mel_basis=basis)
            lead = Sd.shape[:-2]
            src = sc.native(Sd)
            out = sc.empty(lead + (basis.shape[0], T), np.float32)
            nat.check(nat.lib().b2l_mel_project(ctx.handle, plan.handle, _vp(src.ptr), pl.clip_count(lead), T,
                                                _vp(out.ptr)))
            return sc.result(out, np.result_type(req, basis.dtype))
    if n_fft is None:
        raise ParameterError(f"Unable to compute spectrogram with n_fft={n_fft}")
    if y is None:
        raise ParameterError("Input signal must be provided to compute a spectrogram")
    fr = pl.forward_front(y, n_fft, hop_length, win_length, window, center, pad_mode)
    basis, bkey = pl.mel_basis(sr, n_fft, kwargs)
    res_dtype = np.result_type(fr.dtype, basis.dtype)
    if pl.wide_route(y, fr.dtype, n_fft):
        with pl.Scope(y) as sc:
            return sc.result(_mel_f64(sc, y, n_fft, fr, center, power, basis), res_dtype, validate=True)
    pl.require_supported_n_fft(n_fft)
    if pl.transform_path(n_fft) == "czt":
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


def _mel_f64(sc, y, n_fft, fr, center, power, basis):
    """float64 signal -> float64 mel spectrogram on the device in FP64: stft, |.|**power, band projection
    (feature/spectral.py:2145-2160 in the input's precision), owned by the scope ``sc`` of ``y``."""
    _, D = f64.stft(y, n_fft=n_fft, hop_length=fr.hop, center=center, mode=fr.mode, win=fr.window)
    Sd = sc.own(f64.abs_pow(sc.ctx, sc.own(D), power))
    D.free()
    mel_d = sc.own(f64.mel(sc.ctx, Sd, basis))
    Sd.free()
    return mel_d


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

    with pl.Scope(y if S is None else S) as sc:
        if S is None:
            if y is None:
                raise ParameterError("Input signal must be provided to compute a spectrogram")
            _, req = pl.precheck_signal(y)
            staged = pl.StagedInput(y)
            sc.own(staged.dev)
            Sd, n_fft = _spectrogram(y=staged.dev, n_fft=n_fft, hop_length=hop_length, power=2, win_length=win_length,
                                     window=window, center=center, pad_mode=pad_mode)
            staged.scan_uncovered(n_fft, hop_length, win_length, center, Sd.shape[-1])
            src = sc.own(Sd)
        else:
            Sd, req = sc.spectrogram(S)
            if n_fft is None or n_fft // 2 + 1 != Sd.shape[-2]:
                n_fft = 2 * (Sd.shape[-2] - 1)
            src = sc.native(Sd)
        ctx = sc.ctx
        F, T = src.shape[-2], src.shape[-1]
        lead = src.shape[:-2]
        n_clips = pl.clip_count(lead)
        L = nat.lib()
        if tuning is None:
            tuning = _tuning_from_device_spec(src, sr, n_fft, resolution=0.01, bins_per_octave=n_chroma, fmin=150.0,
                                              fmax=4000.0, threshold=0.1, ref=None)
        fb = filters.chroma(sr=sr, n_fft=n_fft, tuning=tuning, n_chroma=n_chroma, **kwargs)
        if fb.shape[1] != F:
            raise ParameterError(f"chroma filter bank has {fb.shape[1]} bins, the spectrogram {F}")
        plan = nat.make_plan(ctx, ("chroma", n_fft, pl.digest(fb)), n_fft=n_fft, hop_length=1, center=True,
                             pad_mode="constant", window=np.ones(n_fft), mel_basis=fb)
        raw = sc.empty(tuple(lead) + (fb.shape[0], T), np.float32)
        nat.check(L.b2l_mel_project(ctx.handle, plan.handle, _vp(src.ptr), n_clips, T, _vp(raw.ptr)))
        sc.free(src)
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
            out = sc.empty(raw.shape, np.float32)
            nat.check(L.b2l_normalize_rows(ctx.handle, _vp(raw.ptr), n_clips, fb.shape[0], T, kind, p, _vp(out.ptr)))
        return sc.result(out, np.result_type(req, fb.dtype), validate=S is None)


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
        with pl.Scope(S) as sc:
            Sd, req = sc.spectrogram(S)
            if Sd.layout != "c":
                raise ParameterError("device log-mel input must be C-ordered (..., n_mels, frames)")
            n_mels, T = Sd.shape[-2], Sd.shape[-1]
            dct = _dct_basis(n_mels, n_mfcc, dct_type, norm, lifter)
            plan = nat.make_plan(sc.ctx, ("dct", n_mels, pl.digest(dct)), n_fft=8, hop_length=1, center=True,
                                 pad_mode="constant", window=np.ones(8),
                                 mel_basis=np.zeros((n_mels, 5), dtype=np.float32), dct_basis=dct)
            lead = Sd.shape[:-2]
            out = sc.empty(lead + (dct.shape[0], T), np.float32)
            nat.check(nat.lib().b2l_dct_project(sc.ctx.handle, plan.handle, _vp(Sd.ptr), pl.clip_count(lead), T,
                                                _vp(out.ptr)))
            return sc.result(out, req)
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
        with pl.Scope(y) as sc:
            mel_d = _mel_f64(sc, y, n_fft, fr, center, power, basis)
            db_d = sc.own(f64.power_to_db(sc.ctx, mel_d, ref_value=1.0, amin=1e-10, top_db=80.0))
            mel_d.free()
            out = sc.own(f64.dct(sc.ctx, db_d, _dct_basis(n_mels, n_mfcc, dct_type, norm, lifter, dtype=np.float64)))
            db_d.free()
            return sc.result(out, res_dtype, validate=True)
    dct = _dct_basis(n_mels, n_mfcc, dct_type, norm, lifter)
    pl.require_supported_n_fft(n_fft)
    if pl.transform_path(n_fft) == "czt":
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


# --------------------------------------------------------------------------------------------- constant-Q chroma
# chroma_cqt / chroma_cens / chroma_vqt / tonnetz (feature/spectral.py:1296-1839).  Everything after the CQT is one
# launch of b2l_chroma_fold (a second, b2l_chroma_smooth, for CENS smoothing); the y= paths run this library's cqt /
# vqt on the staged signal and fold its complex64 result, so |C| never reaches memory.
def _chroma_norm(norm):
    """(enum b2l_chroma_norm, p) of util.normalize's ``norm``, or None for a norm that normalize refuses."""
    if norm is None:
        return nat.CHROMA_NORM_NONE, 0.0
    if norm == np.inf:
        return nat.CHROMA_NORM_INF, 0.0
    if norm == -np.inf:
        return nat.CHROMA_NORM_NEG_INF, 0.0
    if norm == 0:
        return nat.CHROMA_NORM_ZERO, 0.0
    if np.issubdtype(type(norm), np.number) and norm > 0:
        return nat.CHROMA_NORM_P, float(norm)
    return None


def _map_table(ctx, M):
    """Device CSR of a dense map (row offsets, columns, float64 weights; ascending columns), cached by the context."""
    M = np.asarray(M)
    rows, cols = np.nonzero(M)
    ptr = np.zeros(M.shape[0] + 1, dtype=np.int32)
    np.cumsum(np.bincount(rows, minlength=M.shape[0]), out=ptr[1:])
    key = (pl.digest(M.astype(np.float64)), M.shape)
    return (pl.f64_constant(ctx, ("chroma_ptr",) + key, ptr),
            pl.f64_constant(ctx, ("chroma_cols",) + key, cols.astype(np.int32)),
            pl.f64_constant(ctx, ("chroma_w",) + key, M[rows, cols].astype(np.float64)), len(cols))


def _tonnetz_phi(n_chroma: int) -> np.ndarray:
    """tonnetz's 6 x n_chroma transform (feature/spectral.py:1821-1833)."""
    dim_map = np.linspace(0, 12, num=n_chroma, endpoint=False)
    scale = np.asarray([7.0 / 6, 7.0 / 6, 3.0 / 2, 3.0 / 2, 2.0 / 3, 2.0 / 3])
    V = np.multiply.outer(scale, dim_map)
    V[::2] -= 0.5
    R = np.array([1, 1, 1, 1, 0.5, 0.5])
    return R[:, np.newaxis] * np.cos(np.pi * V)


def _smoothing_taps(smoothing_window, win_len_smooth):
    """chroma_cens's normalised smoothing window of win_len_smooth + 2 points as the taps scipy.ndimage.convolve
    uses: the window reversed, positions whose weight exceeds DBL_EPSILON in magnitude, ascending."""
    from .. import filters

    win = filters.get_window(smoothing_window, win_len_smooth + 2, fftbins=False)
    win = win / np.sum(win)
    flipped = np.asarray(win, dtype=np.float64)[::-1]
    keep = np.flatnonzero(np.abs(flipped) > np.finfo(np.float64).eps)
    return keep.astype(np.int32), np.ascontiguousarray(flipped[keep]), len(win)


def _stage_real(sc, X, what: str):
    """A real ``(..., rows, frames)`` argument on the device, in the layout it has -> (DeviceArray, enum
    b2l_chroma_input, host copy kept alive until the call has synchronised)."""
    if isinstance(X, nat.DeviceArray):
        dt, shape = X.dtype, X.shape
    else:
        X = np.asarray(X)
        dt, shape = X.dtype, X.shape
    if np.issubdtype(dt, np.complexfloating):
        raise nat.UnsupportedOnGPU(f"{what}: complex input would give complex chroma; pass the magnitude np.abs({what})")
    if len(shape) < 2:
        raise ParameterError(f"{what} must have at least two dimensions (..., bins, frames), given shape={shape}")
    host = None
    if isinstance(X, nat.DeviceArray):
        if dt not in (np.float32, np.float64):
            raise ParameterError(f"device {what} must be float32 or float64")
        d = X
    else:
        dt = dt if dt in (np.float32, np.float64) else np.result_type(dt, np.float32)
        mem = np.swapaxes(X, -1, -2)
        if mem.flags.c_contiguous and not X.flags.c_contiguous and mem.dtype == dt:
            host, layout = mem, "ft"   # [..., frame, bin] memory, cqt's order="F": uploaded as it is
        else:
            host, layout = np.ascontiguousarray(X, dtype=dt), "c"
        d = sc.empty(shape, dt, layout)
        if host.nbytes:
            nat.check(nat.lib().b2l_h2d(sc.ctx.handle, _vp(d.ptr), host.ctypes.data_as(_vp), host.nbytes))
    f64 = d.dtype == np.float64
    kind = {(False, "ft"): nat.CHROMA_IN_F32_FT, (False, "c"): nat.CHROMA_IN_F32_C,
            (True, "ft"): nat.CHROMA_IN_F64_FT, (True, "c"): nat.CHROMA_IN_F64_C}[(f64, d.layout)]
    return d, kind, host


def _chroma_pipeline(*, y, X, what, transform, make_map, norm, threshold, epilogue, post_norm=None, taps=None):
    """The body of chroma_cqt / chroma_vqt / chroma_cens / tonnetz after their argument checks.

    ``X`` (C, V or chroma) or, when it is None, ``transform(staged device signal)`` (a complex64 "ft" cqt / vqt)
    is folded with ``make_map(n_rows)``; ``norm`` and ``threshold`` are chroma_cqt's; ``epilogue`` is the
    b2l_chroma_fold epilogue; CENS: ``post_norm`` is its final norm and ``taps`` its smoothing (None: none).
    Non-finite data and unsupported norms raise in the reference's order once the device has finished."""
    staged = None
    with pl.Scope(y if X is None else X) as sc:
        if X is None:
            _, req = pl.precheck_signal(y)
            staged = pl.StagedInput(y)
            if staged.on_device:
                nat.check(nat.lib().b2l_status_reset(staged.ctx.handle))
            src = sc.own(transform(staged.dev))
            staged.scan_all()
            staged.release()
            kind, req = nat.CHROMA_IN_C64_FT, np.dtype(req)
        else:
            src, kind, host = _stage_real(sc, X, what)
            nat.check(nat.lib().b2l_status_reset(sc.ctx.handle))
            req = src.dtype
        ctx, L = sc.ctx, nat.lib()
        M = make_map(src.shape[-2])
        prec = np.result_type(M.dtype, np.float32 if kind == nat.CHROMA_IN_C64_FT else src.dtype)
        lead, T = tuple(src.shape[:-2]), src.shape[-1]
        d_ptr, d_cols, d_w, nnz = _map_table(ctx, M)
        nk = _chroma_norm(norm) or (nat.CHROMA_NORM_NONE, 0.0)
        pk = _chroma_norm(post_norm) or (nat.CHROMA_NORM_NONE, 0.0)
        d_phi = 0
        if epilogue == nat.CHROMA_TONNETZ:
            d_phi = pl.f64_constant(ctx, ("tonnetz_phi", M.shape[0]), _tonnetz_phi(M.shape[0]))
            out = sc.empty(lead + (6, T), np.float64)
        else:
            out = sc.empty(lead + (M.shape[0], T), prec)
        if taps is not None:
            pk = (nat.CHROMA_NORM_NONE, 0.0)
        desc = nat.ChromaDesc(kind, int(prec == np.float64), src.shape[-2], M.shape[0], nnz, nk[0], nk[1],
                              int(threshold is not None), epilogue, float(threshold or 0.0), pk[0], 0, pk[1],
                              d_ptr, d_cols, d_w, d_phi or None)
        n_clips = pl.clip_count(lead)
        nat.check(L.b2l_chroma_fold(ctx.handle, C.byref(desc), _vp(src.ptr), n_clips, T, _vp(out.ptr)))
        if taps is not None:
            off, w, win_len = taps
            fk = _chroma_norm(post_norm) or (nat.CHROMA_NORM_NONE, 0.0)
            d_off = pl.f64_constant(ctx, ("cens_off", off.tobytes()), off)
            d_tw = pl.f64_constant(ctx, ("cens_w", w.tobytes()), w)
            smoothed = sc.empty(out.shape, prec)
            nat.check(L.b2l_chroma_smooth(ctx.handle, _vp(out.ptr), n_clips, M.shape[0], T, int(prec == np.float64),
                                          _vp(d_off), _vp(d_tw), len(off), win_len, fk[0], fk[1], _vp(smoothed.ptr)))
            out = smoothed
        flags = pl.status_word(ctx)
        if staged is not None:
            staged.check_finite()
        if flags & nat.STATUS_NOT_FINITE_VALUE:
            raise ParameterError("Input must be finite")
        for n in (norm, post_norm):
            if _chroma_norm(n) is None:
                raise ParameterError(f"Unsupported norm: {n!r}")
        if epilogue == nat.CHROMA_TONNETZ:
            dtype = np.dtype(np.float64)
        else:
            dtype = np.result_type(M.dtype, req if kind == nat.CHROMA_IN_C64_FT else src.dtype)
        return sc.result(out, dtype)


def _cqt_transform(*, sr, hop_length, fmin, n_bins, bins_per_octave, tuning, res_type, intervals="equal", gamma=0):
    """The y= transform of the chroma features: this library's vqt on the staged signal (a DeviceArray result)."""
    from ..core.constantq import vqt

    return lambda dev: vqt(dev, sr=sr, hop_length=hop_length, fmin=fmin, n_bins=n_bins, intervals=intervals,
                           gamma=gamma, bins_per_octave=bins_per_octave, tuning=tuning, res_type=res_type)


def _refuse_resampling(y, *, sr, hop_length, fmin, n_bins, bins_per_octave, tuning, res_type, intervals="equal",
                       gamma=0):
    """Refuse, before any device work, a y= call whose CQT would resample with a resampler other than polyphase
    (the reference's default res_type is soxr_hq).  Argument errors are left to the CQT, which raises them in the
    reference's order."""
    from ..core import constantq as Q

    if res_type == "polyphase":
        return
    try:
        n = y.shape[-1]
        f0 = Q._default_fmin() if fmin is None else fmin
        Q.plan(n, sr=sr, hop_length=hop_length, fmin=f0 * 2.0 ** ((tuning or 0.0) / bins_per_octave), n_bins=n_bins,
               intervals=intervals, gamma=gamma, bins_per_octave=bins_per_octave, filter_scale=1, window="hann",
               scale=True, res_type=res_type)
    except nat.UnsupportedOnGPU:
        raise nat.UnsupportedOnGPU(
            f"res_type={res_type!r}: this CQT resamples, and only the 'polyphase' resampler runs on the GPU; pass "
            "res_type='polyphase', or compute the CQT yourself and pass its magnitude as C= (V= for chroma_vqt)") from None
    except Exception:
        return


def _cqt_chroma_args(y, C, n_chroma, bins_per_octave, cqt_mode):
    """chroma_cqt's first checks (feature/spectral.py:1378-1393) -> bins_per_octave."""
    if bins_per_octave is None:
        bins_per_octave = n_chroma
    elif np.remainder(bins_per_octave, n_chroma) != 0:
        raise ParameterError(f"bins_per_octave={bins_per_octave} must be an integer multiple of n_chroma={n_chroma}")
    if C is None:
        if y is None:
            raise ParameterError("At least one of C or y must be provided to compute chroma")
        if cqt_mode == "hybrid":
            raise nat.UnsupportedOnGPU("chroma_cqt(cqt_mode='hybrid') does not compute the CQT itself; pass "
                                       "C=hybrid_cqt(y, ...) (its float32 result is taken as it is) or use "
                                       "cqt_mode='full'")
        if cqt_mode != "full":
            raise KeyError(cqt_mode)
    return bins_per_octave


def _chroma_cqt(*, y, sr, C, hop_length, fmin, norm, threshold, tuning, n_chroma, n_octaves, window,
                bins_per_octave, cqt_mode, res_type, epilogue, post_norm=None, taps=None):
    from .. import filters

    bins_per_octave = _cqt_chroma_args(y, C, n_chroma, bins_per_octave, cqt_mode)
    cq = dict(sr=sr, hop_length=hop_length, fmin=fmin, n_bins=n_octaves * bins_per_octave,
              bins_per_octave=bins_per_octave, tuning=tuning, res_type=res_type)
    if C is None:
        pl.precheck_signal(y)
        _refuse_resampling(y, **cq)
    return _chroma_pipeline(
        y=y, X=C, what="C", transform=_cqt_transform(**cq),
        make_map=lambda n: filters.cq_to_chroma(n, bins_per_octave=bins_per_octave, n_chroma=n_chroma, fmin=fmin,
                                                window=window),
        norm=norm, threshold=threshold, epilogue=epilogue, post_norm=post_norm, taps=taps)


def chroma_cqt(*, y=None, sr: float = 22050, C=None, hop_length: int = 512, fmin=None, norm=np.inf,
               threshold: float = 0.0, tuning: Optional[float] = None, n_chroma: int = 12, n_octaves: int = 7,
               window=None, bins_per_octave: Optional[int] = 36, cqt_mode: str = "full", res_type: str = "soxr_hq"):
    """Constant-Q chromagram, shape ``(..., n_chroma, t)``; same contract as ``librosa.feature.chroma_cqt``
    (feature/spectral.py:1296-1423), plus ``res_type``, forwarded to ``cqt``: the reference's own cqt call uses its
    default "soxr_hq", and only "polyphase" resamples on the GPU.  ``C`` is a real CQT magnitude, host or device,
    float32 or float64; the result is float32, float64 for float64 ``C`` or a ``window``."""
    return _chroma_cqt(y=y, sr=sr, C=C, hop_length=hop_length, fmin=fmin, norm=norm, threshold=threshold,
                       tuning=tuning, n_chroma=n_chroma, n_octaves=n_octaves, window=window,
                       bins_per_octave=bins_per_octave, cqt_mode=cqt_mode, res_type=res_type,
                       epilogue=nat.CHROMA_PLAIN)


def chroma_cens(*, y=None, sr: float = 22050, C=None, hop_length: int = 512, fmin=None,
                tuning: Optional[float] = None, n_chroma: int = 12, n_octaves: int = 7, bins_per_octave: int = 36,
                cqt_mode: str = "full", window=None, norm=2, win_len_smooth: Optional[int] = 41,
                smoothing_window="hann", res_type: str = "soxr_hq"):
    """Chroma Energy Normalized, shape ``(..., n_chroma, t)``; same contract as ``librosa.feature.chroma_cens``
    (feature/spectral.py:1426-1573), plus chroma_cqt's ``res_type``.  The chroma, its L1 normalisation and
    quantisation are one launch; the smoothing (scipy.ndimage.convolve along frames) and the final normalisation
    another, unless ``win_len_smooth`` is None."""
    if not ((win_len_smooth is None) or (isinstance(win_len_smooth, (int, np.integer)) and win_len_smooth > 0)):
        raise ParameterError(f"win_len_smooth={win_len_smooth} must be a positive integer or None")
    _cqt_chroma_args(y, C, n_chroma, bins_per_octave, cqt_mode)
    taps = _smoothing_taps(smoothing_window, win_len_smooth) if win_len_smooth else None
    return _chroma_cqt(y=y, sr=sr, C=C, hop_length=hop_length, fmin=fmin, norm=None, threshold=0.0, tuning=tuning,
                       n_chroma=n_chroma, n_octaves=n_octaves, window=window, bins_per_octave=bins_per_octave,
                       cqt_mode=cqt_mode, res_type=res_type, epilogue=nat.CHROMA_CENS, post_norm=norm, taps=taps)


def chroma_vqt(*, y=None, sr: float = 22050, V=None, hop_length: int = 512, fmin=None, intervals, norm=np.inf,
               threshold: float = 0.0, n_octaves: int = 7, bins_per_octave: int = 12, gamma: float = 0,
               res_type: str = "soxr_hq"):
    """Variable-Q chromagram, shape ``(..., bins_per_octave, t)``; same contract as
    ``librosa.feature.chroma_vqt`` (feature/spectral.py:1576-1706), plus chroma_cqt's ``res_type``.  On the y= path
    ``intervals`` is "equal" or explicit ratios (the named interval sets are not part of this library's vqt)."""
    from .. import filters

    if not isinstance(intervals, str):
        bins_per_octave = len(intervals)
    cq = dict(sr=sr, hop_length=hop_length, fmin=fmin, n_bins=n_octaves * bins_per_octave,
              bins_per_octave=bins_per_octave, tuning=0.0, res_type=res_type, intervals=intervals, gamma=gamma)
    if V is None:
        if y is None:
            raise ParameterError("At least one of y or V must be provided to compute chroma")
        if isinstance(intervals, str) and intervals != "equal":
            raise nat.UnsupportedOnGPU(f"chroma_vqt(y=..., intervals={intervals!r}): only 'equal' and explicit "
                                       "interval ratios are supported on the y= path; pass V= for named interval sets")
        pl.precheck_signal(y)
        _refuse_resampling(y, **cq)
    return _chroma_pipeline(
        y=y, X=V, what="V", transform=_cqt_transform(**cq),
        make_map=lambda n: filters.cq_to_chroma(n, bins_per_octave=bins_per_octave, n_chroma=bins_per_octave,
                                                fmin=fmin),
        norm=norm, threshold=threshold, epilogue=nat.CHROMA_PLAIN)


def tonnetz(*, y=None, sr: float = 22050, chroma=None, **kwargs):
    """Tonal centroid features, shape ``(..., 6, t)`` float64; same contract as ``librosa.feature.tonnetz``
    (feature/spectral.py:1709-1839).  ``kwargs`` go to chroma_cqt when ``chroma`` is None; the chroma, its L1
    normalisation and the projection are one launch after the CQT."""
    if y is None and chroma is None:
        raise ParameterError("Either the audio samples or the chromagram must be passed as an argument.")
    if chroma is None:
        kw = dict(sr=sr, C=None, hop_length=512, fmin=None, norm=np.inf, threshold=0.0, tuning=None, n_chroma=12,
                  n_octaves=7, window=None, bins_per_octave=36, cqt_mode="full", res_type="soxr_hq")
        unknown = set(kwargs) - set(kw)
        if unknown:
            raise TypeError(f"chroma_cqt() got an unexpected keyword argument {sorted(unknown)[0]!r}")
        kw.update(kwargs)
        return _chroma_cqt(y=y, epilogue=nat.CHROMA_TONNETZ, **kw)
    return _chroma_pipeline(y=None, X=chroma, what="chroma", transform=None,
                            make_map=lambda n: np.eye(n, dtype=np.float32), norm=None, threshold=None,
                            epilogue=nat.CHROMA_TONNETZ)
