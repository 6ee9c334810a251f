"""``stft`` / ``istft`` / ``_spectrogram`` / ``power_to_db`` with librosa's signatures, executed by
libb2l.so on an H100 (reference: librosa/core/spectrum.py:58-391, 395-626, 2920-3015, 1735-1883).

Inputs may be NumPy arrays (results come back as NumPy arrays with librosa's shapes and dtypes) or
``DeviceArray`` objects (results stay on the device, so ``stft -> istft`` or ``melspectrogram`` chains
never touch the host).
"""
from __future__ import annotations

import ctypes as C
import warnings
from typing import Optional

import numpy as np

from .. import _f64 as f64
from .. import _native as nat
from .. import _pipeline as pl
from .. import filters
from ..util.exceptions import ParameterError
from ..util.utils import dtype_c2r, dtype_r2c, fix_length, is_positive_int, pad_center, tiny

_vp = C.c_void_p


def stft(y, *, n_fft: int = 2048, hop_length: Optional[int] = None, win_length: Optional[int] = None,
         window="hann", center: bool = True, dtype=None, pad_mode="constant", out=None):
    """Short-time Fourier transform; same contract as ``librosa.stft`` (core/spectrum.py:58-391).

    Returns ``(..., 1 + n_fft/2, n_frames)`` complex64.  For a NumPy input the result is a view whose
    memory is ``[..., frame, bin]`` — for a 1-D signal that is the Fortran order librosa returns.
    """
    fr = pl.forward_front(y, n_fft, hop_length, win_length, window, center, pad_mode)
    if dtype is None:
        dtype = dtype_r2c(fr.dtype)
    dtype = np.dtype(dtype)
    if pl.wide_route(y, fr.dtype, n_fft):
        return _stft_f64(y, fr, n_fft, center, dtype, out)
    if dtype != np.complex64 and not (dtype.kind == "c" and pl.wide_complex_ok("stft dtype")):
        raise nat.UnsupportedOnGPU(f"stft dtype={dtype}: only complex64 is computed on the GPU "
                                   "(B2L_FLOAT64=error forbids returning float32 results in a wider dtype)")
    shape = tuple(y.shape[:-1]) + (1 + n_fft // 2, fr.n_frames)
    if out is not None:
        _check_out(out, shape)
    pl.require_supported_n_fft(n_fft)

    def launch(ctx, plan, d_in, m, n_, d_out, d_scr):
        nat.check(nat.lib().b2l_stft(ctx.handle, plan.handle, _vp(d_in), m, n_, n_, _vp(d_out)))

    res = pl.run_forward(y, plan_key=("stft", n_fft, fr.hop, bool(center), fr.mode, fr.wkey),
                         plan_kw=dict(n_fft=n_fft, hop_length=fr.hop, center=center, pad_mode=fr.mode,
                                      window=fr.window),
                         n_frames=fr.n_frames, out_tail=shape[-2:], dtype=np.complex64, layout="ft", launch=launch)
    if isinstance(res, nat.DeviceArray):
        if out is None:
            return res
        res = pl.finish(res, dtype)
    elif res.dtype != dtype:
        res = res.astype(dtype)
    return res if out is None else _write_out(out, res)


def _check_out(out, shape):
    if isinstance(out, nat.DeviceArray):
        raise ParameterError("out= must be a NumPy array")
    if not (tuple(out.shape[:-1]) == tuple(shape[:-1]) and out.shape[-1] >= shape[-1]):
        raise ParameterError(f"Shape mismatch for provided output array out.shape={out.shape} and "
                             f"target shape={list(shape)}")
    if not np.iscomplexobj(out):
        raise ParameterError(f"output with dtype={out.dtype} is not of complex type")


def _write_out(out, res):
    """stft(out=...): the result goes into the first frames of ``out`` (librosa allows a longer buffer)."""
    target = out if out.shape[-1] == res.shape[-1] else out[..., : res.shape[-1]]
    target[...] = res
    return target


def _stft_f64(y, fr, n_fft, center, dtype, out):
    """float64 signal -> complex128 STFT in FP64 on the device (what the reference computes: dtype_r2c,
    core/spectrum.py:341; window product and rfft in double, :388)."""
    if dtype.kind != "c":
        raise ParameterError(f"stft dtype={dtype} is not complex")
    if out is not None:
        _check_out(out, tuple(y.shape[:-1]) + (1 + n_fft // 2, fr.n_frames))
    staged, D = f64.stft(y, n_fft=n_fft, hop_length=fr.hop, center=center, mode=fr.mode, win=fr.window)
    if staged.on_device and out is None:
        return D
    res = pl.finish(D, dtype, validate=not staged.on_device)
    return res if out is None else _write_out(out, res)


def _inv_wss(ctx, window, n_frames, win_length, n_fft, hop_length, start, out_len, wkey):
    """Reciprocal window-sum-square, trimmed as istft does (core/spectrum.py:606-624), cached on device."""
    def build():
        wss = filters.window_sumsquare(window=window, n_frames=n_frames, win_length=win_length, n_fft=n_fft,
                                       hop_length=hop_length, dtype=np.float32)
        wss = fix_length(wss[start:], size=out_len)
        inv = np.ones(out_len, dtype=np.float32)
        nz = wss > tiny(wss)
        inv[nz] = (np.float32(1.0) / wss[nz]).astype(np.float32)
        return inv

    return ctx.constant(("wss", wkey, n_frames, n_fft, hop_length, start, out_len), build)


def _istft_out_len(n_fft, hop_length, n_frames, center, length) -> int:
    if length:
        return int(length)
    return n_fft + hop_length * (n_frames - 1) - (2 * (n_fft // 2) if center else 0)


def _check_istft_out(out, shape):
    if out is not None:
        if isinstance(out, nat.DeviceArray):
            raise ParameterError("out= must be a NumPy array")
        if tuple(out.shape) != shape:
            raise ParameterError(f"Shape mismatch for provided output array out.shape={out.shape} != {list(shape)}")


def _istft_result(sc, y, dtype, out):
    """istft's return value: the device signal for a device call without ``out``, else ``y`` copied to the host as
    ``dtype`` (written into ``out`` when given)."""
    if sc.on_device and out is None:
        return sc.keep(y)
    res = pl.finish(y, dtype)
    if out is None:
        return res
    out[...] = res
    return out


def _istft_f64(stft_matrix, n_frames, T_stored, F, n_fft, hop_length, win_length, window, win, center, dtype, length,
               out):
    """complex128 STFT -> float64 signal in FP64 on the device (core/spectrum.py:506-626 in double)."""
    if dtype is None:
        dtype = np.float64
    dtype = np.dtype(dtype)
    if not np.issubdtype(dtype, np.floating):
        raise ParameterError(f"istft dtype={dtype} must be a floating-point type")
    out_len = _istft_out_len(n_fft, hop_length, n_frames, center, length)
    _check_istft_out(out, tuple(stft_matrix.shape[:-2]) + (out_len,))
    f64.require_supported(n_fft)
    with pl.Scope(stft_matrix) as sc:
        if sc.on_device and stft_matrix.layout != "ft":
            raise ParameterError("device complex128 stft_matrix must be in the native [frame][bin] layout")
        Dd = sc.native(stft_matrix, np.complex128, host_transpose=True)
        start = n_fft // 2 if center else 0
        inv = f64.inv_wss(window, n_frames, win_length, n_fft, hop_length, start, out_len)
        y = sc.own(f64.istft(sc.ctx, Dd, n_frames_used=n_frames, n_fft=n_fft, hop_length=hop_length, center=center,
                             win=win, inv=inv, out_len=out_len))
        return _istft_result(sc, y, dtype, out)


def istft(stft_matrix, *, hop_length: Optional[int] = None, win_length: Optional[int] = None,
          n_fft: Optional[int] = None, window="hann", center: bool = True, dtype=None,
          length: Optional[int] = None, out=None):
    """Inverse STFT; same contract as ``librosa.istft`` (core/spectrum.py:395-626)."""
    on_device = isinstance(stft_matrix, nat.DeviceArray)
    if not on_device:
        stft_matrix = np.asarray(stft_matrix)
    if stft_matrix.ndim < 2:
        raise ParameterError("stft_matrix must have at least two dimensions (bins, frames)")
    F, T_stored = stft_matrix.shape[-2], stft_matrix.shape[-1]
    if n_fft is None:
        n_fft = 2 * (F - 1)
    if win_length is None:
        win_length = n_fft
    if hop_length is None:
        hop_length = int(win_length // 4)
    win, wkey = pl.resolve_window(window, win_length, n_fft)
    if F != n_fft // 2 + 1:
        raise nat.UnsupportedOnGPU(f"istft: n_fft={n_fft} does not match {F} frequency bins")
    if length:
        padded = length + 2 * (n_fft // 2) if center else length
        n_frames = min(T_stored, int(np.ceil(padded / hop_length)))
    else:
        n_frames = T_stored
    in_dtype = np.dtype(stft_matrix.dtype)
    if (in_dtype == np.complex128 and pl.native_float64(in_dtype)) or \
            (in_dtype == np.complex64 and not on_device and pl.transform_path(n_fft) is None and f64.supported(n_fft)):
        wide = stft_matrix if in_dtype == np.complex128 else stft_matrix.astype(np.complex128)
        return _istft_f64(wide, n_frames, T_stored, F, n_fft, hop_length, win_length, window, win, center,
                          dtype if dtype is not None else dtype_c2r(in_dtype), length, out)
    if in_dtype != np.complex64:
        if in_dtype.kind == "c" and pl.wide_complex_ok("istft input"):
            pass
        elif in_dtype.kind == "c":
            raise nat.UnsupportedOnGPU("istft: only complex64 input is computed on the GPU "
                                       "(B2L_FLOAT64=error forbids computing complex128 data in float32)")
        else:
            raise ParameterError(f"stft_matrix must be complex, got {in_dtype}")
    if dtype is None:
        dtype = dtype_c2r(in_dtype)
    dtype = pl.check_real_dtype(dtype, "istft dtype")
    out_len = _istft_out_len(n_fft, hop_length, n_frames, center, length)
    lead = tuple(stft_matrix.shape[:-2])
    _check_istft_out(out, lead + (out_len,))
    pl.require_supported_n_fft(n_fft)
    with pl.Scope(stft_matrix) as sc:
        ctx = sc.ctx
        key = ("stft", n_fft, hop_length, bool(center), "constant", wkey)
        plan = nat.make_plan(ctx, key, n_fft=n_fft, hop_length=hop_length, center=center, pad_mode="constant",
                             window=win)
        if on_device and stft_matrix.dtype != np.complex64:
            raise ParameterError("device stft_matrix must be complex64")
        # a host matrix whose memory already is [.., frame, bin] complex64 (stft's own output) uploads as it is
        zero_copy = not on_device and in_dtype == np.complex64 and np.swapaxes(stft_matrix, -1, -2).flags.c_contiguous
        Dd = sc.native(stft_matrix, np.complex64, host_transpose=zero_copy)
        start = n_fft // 2 if center else 0
        inv_ptr = _inv_wss(ctx, window, n_frames, win_length, n_fft, hop_length, start, out_len, wkey)
        y = sc.empty(lead + (out_len,), np.float32)
        nat.check(nat.lib().b2l_istft(ctx.handle, plan.handle, _vp(Dd.ptr), pl.clip_count(lead), T_stored, n_frames,
                                      _vp(inv_ptr), out_len, _vp(y.ptr), out_len))
        return _istft_result(sc, y, dtype, out)


def _spectrogram(*, y=None, S=None, n_fft: Optional[int] = 2048, hop_length: Optional[int] = 512,
                 power: float = 1, win_length: Optional[int] = None, window="hann", center: bool = True,
                 pad_mode="constant"):
    """``|stft|**power`` (or pass ``S`` through); mirror of core/spectrum.py:2920-3015."""
    if S is not None:
        if n_fft is None or n_fft // 2 + 1 != S.shape[-2]:
            n_fft = 2 * (S.shape[-2] - 1)
        return S, n_fft
    if n_fft is None:
        raise ParameterError(f"Unable to compute spectrogram with n_fft={n_fft}")
    if y is None:
        raise ParameterError("Input signal must be provided to compute a spectrogram")
    fr = pl.forward_front(y, n_fft, hop_length, win_length, window, center, pad_mode)
    if pl.wide_route(y, fr.dtype, n_fft):
        with pl.Scope(y) as sc:
            _, D = f64.stft(y, n_fft=n_fft, hop_length=fr.hop, center=center, mode=fr.mode, win=fr.window)
            Sd = sc.own(f64.abs_pow(sc.ctx, sc.own(D), power))
            return sc.result(Sd, fr.dtype, validate=True), n_fft
    pl.require_supported_n_fft(n_fft)

    def launch(ctx, plan, d_in, m, n_, d_out, d_scr):
        nat.check(nat.lib().b2l_spectrogram(ctx.handle, plan.handle, _vp(d_in), m, n_, n_, _vp(d_out)))

    res = pl.run_forward(y, plan_key=("spec", n_fft, fr.hop, bool(center), fr.mode, fr.wkey, float(power)),
                         plan_kw=dict(n_fft=n_fft, hop_length=fr.hop, center=center, pad_mode=fr.mode, window=fr.window,
                                      power=float(power)),
                         n_frames=fr.n_frames, out_tail=(1 + n_fft // 2, fr.n_frames), dtype=np.float32, layout="ft",
                         launch=launch)
    if isinstance(res, nat.DeviceArray) or res.dtype == fr.dtype:
        return res, n_fft
    return res.astype(fr.dtype), n_fft


def power_to_db(S, *, ref=1.0, amin: float = 1e-10, top_db: Optional[float] = 80.0, axes="auto"):
    """``10*log10(S/ref)`` with the ``top_db`` floor; mirror of core/spectrum.py:1735-1883.

    The reference maximum of ``top_db`` is taken per leading index over the last two axes
    (``axes="auto"``), which is what ``mfcc`` relies on for multichannel input."""
    return _to_db(S, ref, amin, top_db, axes, amplitude=False)


def amplitude_to_db(S, *, ref=1.0, amin: float = 1e-5, top_db: Optional[float] = 80.0, axes="auto"):
    """``20*log10(|S|/ref)``: ``power_to_db(S**2, ref=ref**2, amin=amin**2)``; mirror of
    core/spectrum.py:1946-2038."""
    return _to_db(S, ref, amin, top_db, axes, amplitude=True)


def _to_db(S, ref, amin, top_db, axes, amplitude: bool):
    name = "amplitude_to_db" if amplitude else "power_to_db"
    on_device = isinstance(S, nat.DeviceArray)
    if not on_device:
        S = np.asarray(S)
    if amin <= 0:
        raise ParameterError("amin must be strictly positive")
    if not on_device and np.issubdtype(S.dtype, np.complexfloating):
        hint = "amplitude_to_db(np.abs(S))" if amplitude else "power_to_db(np.abs(D)**2)"
        warnings.warn(f"{name} was called on complex input so phase information will be discarded. "
                      f"To suppress this warning, call {hint} instead.", stacklevel=3)
        S = np.abs(S)
    if top_db is not None and top_db < 0:
        raise ParameterError("top_db must be non-negative")
    if not (isinstance(axes, str) and axes == "auto"):
        # explicit reduction axes for the top_db maximum / callable ref (core/spectrum.py:1855-1881): bring the
        # reduced axes to the end, run the "auto" kernel on (kept, 1, reduced), undo the permutation
        if on_device:
            raise nat.UnsupportedOnGPU(f"{name}: explicit axes need a host array")
        if S.ndim == 0:
            return _to_db(S, ref, amin, top_db, "auto", amplitude)
        ax = tuple(range(S.ndim)) if axes is None else tuple(np.atleast_1d(axes).astype(int).tolist())
        ax = tuple(sorted({a % S.ndim if -S.ndim <= a < S.ndim else a for a in ax}))
        if any(not (0 <= a < S.ndim) for a in ax):
            raise np.exceptions.AxisError(f"axis {axes} is out of bounds for array of dimension {S.ndim}")
        kept = [i for i in range(S.ndim) if i not in ax]
        perm = kept + list(ax)
        Sp = np.transpose(S, perm)
        n_keep = pl.clip_count(tuple(S.shape[i] for i in kept))
        flat = np.ascontiguousarray(Sp).reshape(n_keep, 1, -1)
        res = _to_db(flat, ref, amin, top_db, "auto", amplitude)
        return np.transpose(np.asarray(res).reshape(Sp.shape), np.argsort(perm))[()]
    with pl.Scope(S) as sc:
        if not on_device and S.dtype == np.float64 and pl.native_float64(S.dtype) and S.ndim >= 1:
            return _to_db_f64(sc, S, ref, amin, top_db, amplitude)
        if not on_device and not np.issubdtype(S.dtype, np.floating):
            S = S.astype(np.float32)
        dev, req = sc.spectrogram(S, f"{name} input", stacklevel=5)
        ctx = sc.ctx
        ndim = len(dev.shape)
        if ndim >= 2:
            lead = dev.shape[:-2]
            per = dev.shape[-2] * dev.shape[-1]
        else:
            lead = ()
            per = dev.size
        n_lead = pl.clip_count(lead)
        out = sc.empty(dev.shape, np.float32, layout=dev.layout)
        tdb = -1.0 if top_db is None else float(top_db)
        L = nat.lib()
        src = dev
        if amplitude:
            # power = |S|**2 (written into the output buffer, converted in place), amin**2, ref**2
            nat.check(L.b2l_unary(ctx.handle, nat.UNARY_SQUARE, _vp(dev.ptr), dev.size, 0.0, _vp(out.ptr)))
            src = out
            amin = float(amin) ** 2
        if callable(ref):
            if on_device:
                raise nat.UnsupportedOnGPU("callable ref needs a host array")
            ax = (-2, -1) if ndim >= 2 else ((-1,) if ndim == 1 else None)
            try:
                ref_value = np.asarray(ref(np.abs(S) if amplitude else S, axis=ax, keepdims=True),
                                       dtype=np.float64).reshape(-1)
            except TypeError as exc:
                raise ParameterError("The provided reference function must support 'axis' and 'keepdims' "
                                     "arguments for proper multichannel processing.") from exc
            if amplitude:
                ref_value = ref_value ** 2
            for i in range(n_lead):   # one reference level per leading index
                nat.check(L.b2l_power_to_db(ctx.handle, _vp(src.ptr + 4 * i * per), 1, per, float(amin),
                                            float(ref_value[i if ref_value.size > 1 else 0]), tdb,
                                            _vp(out.ptr + 4 * i * per)))
        else:
            ref_value = float(np.abs(ref)) ** 2 if amplitude else float(np.abs(ref))
            nat.check(L.b2l_power_to_db(ctx.handle, _vp(src.ptr), n_lead, per, float(amin), ref_value, tdb,
                                        _vp(out.ptr)))
        res = sc.result(out, req)
        return res if on_device else res[()]


def _to_db_f64(sc, S, ref, amin, top_db, amplitude):
    """power_to_db / amplitude_to_db of a float64 host array in FP64 (core/spectrum.py:1866-1881, :1990-2038)."""
    shape = S.shape
    work = S if S.ndim >= 2 else S.reshape(1, -1)
    n_lead = pl.clip_count(work.shape[:-2])
    mag = np.abs(work) if amplitude else work
    if callable(ref):
        try:
            ref_value = np.asarray(ref(mag, axis=(-2, -1), keepdims=True), dtype=np.float64).reshape(-1)
        except TypeError as exc:
            raise ParameterError("The provided reference function must support 'axis' and 'keepdims' "
                                 "arguments for proper multichannel processing.") from exc
    else:
        ref_value = np.asarray([np.abs(ref)], dtype=np.float64)
    if amplitude:                                   # 20 log10(|S| / ref) == 10 log10(|S|^2 / ref^2), amin^2
        power, amin, ref_value = mag ** 2, float(amin) ** 2, ref_value ** 2
    else:
        power = mag
    dev = sc.stage(np.reshape(power, (n_lead,) + work.shape[-2:]), np.float64)
    if ref_value.size > 1:
        parts = []
        for i in range(n_lead):                     # one reference level per leading index
            one = dev.view((1,) + work.shape[-2:], offset=i * work.shape[-2] * work.shape[-1])
            parts.append(sc.own(f64.power_to_db(sc.ctx, one, ref_value=float(ref_value[i]), amin=amin, top_db=top_db)))
        res = np.concatenate([pl.finish(p) for p in parts], axis=0)
    else:
        res = pl.finish(sc.own(f64.power_to_db(sc.ctx, dev, ref_value=float(ref_value[0]), amin=amin, top_db=top_db)))
    return res.reshape(shape)[()]


def _db_inverse(S_db, op, param):
    on_device = isinstance(S_db, nat.DeviceArray)
    if not on_device:
        S_db = np.asarray(S_db)
        if np.iscomplexobj(S_db):
            raise nat.UnsupportedOnGPU("complex dB values are not supported on the GPU")
    with pl.Scope(S_db) as sc:
        dev, req = sc.spectrogram(S_db, "dB input", stacklevel=5)
        if not on_device and not np.issubdtype(S_db.dtype, np.floating):
            req = np.dtype(np.float64)
        out = sc.empty(dev.shape, np.float32, layout=dev.layout)
        nat.check(nat.lib().b2l_unary(sc.ctx.handle, op, _vp(dev.ptr), dev.size, float(param), _vp(out.ptr)))
        res = sc.result(out, req)
        return res if on_device else res[()]


def db_to_power(S_db, *, ref: float = 1.0):
    """``ref * 10**(S_db / 10)``; mirror of core/spectrum.py:1899-1925."""
    return _db_inverse(S_db, nat.UNARY_DB_TO_POWER, ref)


def db_to_amplitude(S_db, *, ref: float = 1.0):
    """``db_to_power(S_db, ref=ref**2) ** 0.5``; mirror of core/spectrum.py:2054-2081."""
    return _db_inverse(S_db, nat.UNARY_DB_TO_AMPLITUDE, float(ref) ** 2)


def pcen(S, *, sr: float = 22050, hop_length: int = 512, gain: float = 0.98, bias: float = 2, power: float = 0.5,
         time_constant: float = 0.400, eps: float = 1e-6, b: Optional[float] = None, max_size: int = 1, ref=None,
         axis: int = -1, max_axis: Optional[int] = None, zi=None, return_zf: bool = False):
    """Per-channel energy normalisation; mirror of core/spectrum.py:2396-2666 for spectrograms laid out
    ``(..., bins, frames)`` (``axis=-1``, ``max_axis=-2``).  Like the reference, host results are float64
    (SciPy's ``lfilter`` promotes); the arithmetic on the GPU is float32."""
    if power < 0:
        raise ParameterError(f"power={power} must be nonnegative")
    if gain < 0:
        raise ParameterError(f"gain={gain} must be non-negative")
    if bias < 0:
        raise ParameterError(f"bias={bias} must be non-negative")
    if eps <= 0:
        raise ParameterError(f"eps={eps} must be strictly positive")
    if time_constant <= 0:
        raise ParameterError(f"time_constant={time_constant} must be strictly positive")
    if not is_positive_int(max_size):
        raise ParameterError(f"max_size={max_size} must be a positive integer")
    if b is None:
        t_frames = time_constant * sr / float(hop_length)
        b = (np.sqrt(1 + 4 * t_frames ** 2) - 1) / (2 * t_frames ** 2)
    if not 0 <= b <= 1:
        raise ParameterError(f"b={b} must be between 0 and 1")
    on_device = isinstance(S, nat.DeviceArray)
    if not on_device:
        S = np.asarray(S)
        if np.issubdtype(S.dtype, np.complexfloating):
            warnings.warn("pcen was called on complex input so phase information will be discarded. "
                          "To suppress this warning, call pcen(np.abs(D)) instead.", stacklevel=2)
            S = np.abs(S)
    ndim = S.ndim
    if ref is not None:
        raise nat.UnsupportedOnGPU("pcen(ref=...) is not supported on the GPU (no CPU fallback)")
    if axis not in (-1, ndim - 1):
        raise nat.UnsupportedOnGPU("pcen on the GPU filters along the last axis (axis=-1)")
    if max_size > 1:
        if ndim == 1:
            raise ParameterError("Max-filtering cannot be applied to 1-dimensional input")
        if max_axis is None:
            if ndim != 2:
                raise ParameterError(f"Max-filtering a {ndim:d}-dimensional spectrogram requires you to specify max_axis")
            max_axis = 0
        if max_axis not in (-2, ndim - 2):
            raise nat.UnsupportedOnGPU("pcen on the GPU max-filters along the second-to-last axis (max_axis=-2)")
    with pl.Scope(S) as sc:
        if not on_device and not np.issubdtype(S.dtype, np.floating):
            S = S.astype(np.float32)
        dev, req = sc.spectrogram(S, "pcen input", stacklevel=5)
        if dev.layout != "c":
            raise ParameterError("device pcen input must be C-ordered")
        T = dev.shape[-1]
        rows = dev.shape[-2] if ndim >= 2 else 1
        lead = dev.shape[:-2] if ndim >= 2 else ()
        n_lead = pl.clip_count(lead)
        state_shape = dev.shape[:-1] + (1,)
        d_zi = None
        if zi is not None:
            zi = np.asarray(zi, dtype=np.float64)
            try:
                zi_full = np.broadcast_to(zi, state_shape)
            except ValueError as exc:
                raise ValueError(f"zi has shape {zi.shape}, expected a shape broadcastable to {state_shape}") from exc
            d_zi = sc.stage(zi_full, np.float32)
        d_zf = sc.empty(state_shape, np.float32) if return_zf else None
        out = sc.empty(dev.shape, np.float32)
        scratch = sc.empty(dev.shape, np.float32) if max_size > 1 else None
        desc = nat.PcenDesc(gain=float(gain), bias=float(bias), power=float(power), eps=float(eps), b=float(b),
                            max_size=int(max_size))
        nat.check(nat.lib().b2l_pcen(sc.ctx.handle, C.byref(desc), _vp(dev.ptr), n_lead, rows, T,
                                     _vp(d_zi.ptr if d_zi is not None else None),
                                     _vp(d_zf.ptr if d_zf is not None else None),
                                     _vp(scratch.ptr if scratch is not None else None), _vp(out.ptr)))
        res_dtype = np.result_type(req, np.float64)
        res = sc.result(out, res_dtype)
        return (res, sc.result(d_zf, res_dtype)) if return_zf else res


def reassigned_spectrogram(y, *, sr: float = 22050, S=None, n_fft: int = 2048, hop_length: Optional[int] = None,
                           win_length: Optional[int] = None, window="hann", center: bool = True,
                           reassign_frequencies: bool = True, reassign_times: bool = True, ref_power=1e-6,
                           fill_nan: bool = False, clip: bool = True, dtype=None, pad_mode="constant"):
    """Time-frequency reassigned spectrogram ``(freqs, times, mags)``; same contract as
    ``librosa.reassigned_spectrogram`` (core/spectrum.py:1019-1293) for a numeric ``ref_power``.  The three
    STFTs (window, cyclic window derivative, time-weighted window) and the reassignment arithmetic stay on the
    device.  float32 arithmetic: cells whose magnitude is near float32 round-off of the loudest bin carry a
    visibly larger relative error in the reassigned coordinates than the reference's float64 FFT."""
    from ..util.utils import cyclic_gradient

    if callable(ref_power):
        raise nat.UnsupportedOnGPU("reassigned_spectrogram(ref_power=callable) is not supported on the GPU")
    if ref_power < 0:
        raise ParameterError("ref_power must be non-negative or callable.")
    if not reassign_frequencies and not reassign_times:
        raise ParameterError("reassign_frequencies or reassign_times must be True.")
    if S is not None and isinstance(S, nat.DeviceArray):
        raise nat.UnsupportedOnGPU("reassigned_spectrogram(S=DeviceArray) is not supported; pass y only")
    if win_length is None:
        win_length = n_fft
    if hop_length is None:
        hop_length = int(win_length // 4)
    n, req = pl.precheck_signal(y)
    w = pad_center(filters.get_window(window, win_length, fftbins=True), size=n_fft)
    with pl.Scope(y) as sc:
        staged = pl.StagedInput(y)
        ctx, yd = sc.ctx, sc.own(staged.dev)
        kw = dict(n_fft=n_fft, hop_length=hop_length, center=center, pad_mode=pad_mode)
        if S is None:
            Sh = sc.own(stft(yd, window=w, **kw))
        else:
            Sh = sc.native(np.asarray(S), np.complex64, host_transpose=True)
        F, T = Sh.shape[-2], Sh.shape[-1]
        staged.scan_uncovered(n_fft, hop_length, win_length, center, T)
        Sdh = sc.own(stft(yd, window=cyclic_gradient(w), **kw)) if reassign_frequencies else None
        Sth = None
        if reassign_times:
            half = n_fft // 2
            window_times = np.arange(-half, half + 1) if n_fft % 2 else np.arange(0.5 - half, half)
            Sth = sc.own(stft(yd, window=w * window_times, **kw))
        offset = 0 if center else int(n_fft // 2)
        frame_times = (np.arange(T) * hop_length + offset).astype(int) / float(sr)
        from .convert import fft_frequencies

        d_bf = ctx.constant(("fftfreq", float(sr), int(n_fft)), lambda: fft_frequencies(sr=sr, n_fft=n_fft))
        d_ft = ctx.constant(("frametimes", float(sr), int(hop_length), int(offset), int(T)), lambda: frame_times)
        n_clips = pl.clip_count(Sh.shape[:-2])
        outs = [sc.empty(Sh.shape, np.float32, layout="ft") for _ in range(3)]
        desc = nat.ReassignDesc(sr=float(sr), mag_threshold=float(ref_power) ** 0.5, max_time=float(n) / float(sr),
                                reassign_frequencies=int(bool(reassign_frequencies)),
                                reassign_times=int(bool(reassign_times)), apply_threshold=int(ref_power > 0),
                                fill_nan=int(bool(fill_nan)), clip=int(bool(clip)))
        nat.check(nat.lib().b2l_reassign(ctx.handle, C.byref(desc), _vp(Sh.ptr),
                                         _vp(Sdh.ptr if Sdh is not None else None),
                                         _vp(Sth.ptr if Sth is not None else None), n_clips, T, F, _vp(d_bf),
                                         _vp(d_ft), _vp(outs[0].ptr), _vp(outs[1].ptr), _vp(outs[2].ptr)))
        wide = np.result_type(req, np.float64)
        return sc.result(outs[0], wide, validate=True), sc.result(outs[1], wide), sc.result(outs[2], req)


class _Deprecated:
    """Marker for deprecated keyword arguments (the reference's ``util.decorators.Deprecated``)."""

    def __repr__(self):
        return "<DEPRECATED parameter>"


def phase_vocoder(D, *, rate: Optional[float] = None, t_out=None, kind="linear", hop_length=_Deprecated(),
                  n_fft=_Deprecated()):
    """Phase vocoder: re-time an STFT by ``rate`` (or to the frame positions ``t_out``); same contract as
    ``librosa.phase_vocoder`` (core/spectrum.py:1364-1530) for ``kind="linear"``.  ``D`` may be a complex NumPy
    array ``(..., bins, frames)`` or a complex64 ``DeviceArray`` (result stays on the device)."""
    for name, val in (("hop_length", hop_length), ("n_fft", n_fft)):
        if not isinstance(val, _Deprecated):
            warnings.warn(f"The `{name}` parameter is deprecated as of 1.0 and will be removed in 1.1. "
                          "It is unused in the current implementation.", FutureWarning, stacklevel=2)
    n_frames = D.shape[-1]
    if (rate is None) == (t_out is None):
        raise ParameterError("Must specify exactly one of `rate` or `t_out`")
    if (rate is not None) and (rate <= 0):
        raise ParameterError(f"rate={rate} must be a positive number")
    if t_out is None:
        t_out = np.arange(0.0, n_frames, rate)
    t_out = np.asarray(t_out, dtype=float)
    if np.any(t_out < 0) or np.any(t_out >= n_frames):
        raise ParameterError("t_out values must be in the range [0, D.shape[-1])")
    if np.any(np.diff(t_out) < 0):
        warnings.warn("t_out is not monotonic; phase estimation may be unstable", stacklevel=2)
    if kind != "linear":
        raise nat.UnsupportedOnGPU(f"phase_vocoder(kind={kind!r}): only linear magnitude interpolation runs on the GPU")
    if n_frames < 2:
        raise nat.UnsupportedOnGPU("phase_vocoder needs at least two frames on the GPU")
    on_device = isinstance(D, nat.DeviceArray)
    if on_device:
        if D.dtype != np.complex64:
            raise ParameterError("device STFT must be complex64")
        res_dtype = np.dtype(np.complex64)
    else:
        D = np.asarray(D)
        if not np.iscomplexobj(D):
            raise ParameterError("phase_vocoder expects a complex STFT matrix")
        res_dtype = np.dtype(D.dtype)
        if res_dtype == np.complex128 and not pl.wide_complex_ok("phase_vocoder input"):
            raise ParameterError("complex128 input refused (B2L_FLOAT64=error)")
    with pl.Scope(D) as sc:
        src = sc.native(D, np.complex64, host_transpose=True)
        F = D.shape[-2]
        lead = tuple(D.shape[:-2])
        n_clips = pl.clip_count(lead)
        n_out = int(t_out.shape[0])
        # phase increments: frames floor(t), floor(t) + 1 (:1498-1512); magnitudes: the segment scipy's interp1d
        # picks — searchsorted(x, t) clipped to [1, n - 1], minus one — and the offset inside it (:1517-1527)
        i0 = np.floor(t_out).astype(np.int32)
        i1 = np.minimum(i0 + 1, n_frames - 1).astype(np.int32)
        hi = np.clip(np.searchsorted(np.arange(n_frames, dtype=float), t_out), 1, n_frames - 1)
        lo = (hi - 1).astype(np.int32)
        dx = np.ascontiguousarray(t_out - lo, dtype=np.float64)
        tables = [sc.stage(a) for a in (i0, i1, lo, dx)]
        out = sc.empty(lead + (F, n_out), np.complex64, layout="ft")
        nat.check(nat.lib().b2l_phase_vocoder(sc.ctx.handle, _vp(src.ptr), n_clips, n_frames, F, n_out,
                                              _vp(tables[0].ptr), _vp(tables[1].ptr), _vp(tables[2].ptr),
                                              _vp(tables[3].ptr), _vp(out.ptr)))
        return sc.result(out, res_dtype)


def griffinlim(S, *, n_iter: int = 32, hop_length: Optional[int] = None, win_length: Optional[int] = None,
               n_fft: Optional[int] = None, window="hann", center: bool = True, dtype=None,
               length: Optional[int] = None, pad_mode="constant", momentum: float = 0.99, init="random",
               rng=None):
    """Approximate magnitude-spectrogram inversion with the fast Griffin-Lim algorithm; same contract as
    ``librosa.griffinlim`` (core/spectrum.py:2669-2917).  The whole iteration — istft, stft and the phase
    update — stays on the device; only ``S`` goes up and the final signal comes down."""
    on_device = isinstance(S, nat.DeviceArray)
    if not isinstance(rng, np.random.RandomState):
        rng = np.random.default_rng(rng)
    if momentum > 1:
        warnings.warn(f"Griffin-Lim with momentum={momentum} > 1 can be unstable. Proceed with caution!",
                      stacklevel=2)
    elif momentum < 0:
        raise ParameterError(f"griffinlim() called with momentum={momentum} < 0")
    if not on_device:
        S = np.asarray(S)
    if n_fft is None:
        n_fft = 2 * (S.shape[-2] - 1)
    if init not in ("random", None):
        raise ParameterError(f"init={init} must either None or 'random'")
    s_dtype = pl.check_real_dtype(S.dtype, "griffinlim S")
    cdtype = dtype_r2c(np.float32)
    eps = float(tiny(np.zeros(1, dtype=cdtype)))
    F, T = S.shape[-2], S.shape[-1]
    n_clips = pl.clip_count(S.shape[:-2])
    pl.require_supported_n_fft(n_fft)
    with pl.Scope(S) as sc:
        ctx = sc.ctx
        L = nat.lib()
        S_ft = sc.native(S, np.float32)
        S_host_shape = S.shape
        if init == "random":
            # same generator calls as the reference, so a given seed gives the same starting phases
            ph = 2 * np.pi * rng.random(size=S_host_shape)
            a0 = (np.cos(ph) + 1j * np.sin(ph)).astype(np.complex64)
            a0 = a0 * (np.asarray(S.get()) if on_device else S.astype(np.float32))
            angles = sc.native(a0, np.complex64)
        else:
            angles = sc.empty(S_host_shape, np.complex64, layout="ft")
            ones = sc.native(np.ones(S_host_shape, dtype=np.complex64), np.complex64)
            nat.check(L.b2l_gl_update(ctx.handle, _vp(ones.ptr), None, _vp(S_ft.ptr), 0.0, 0.0, _vp(angles.ptr),
                                      n_clips * F * T))
        kw_i = dict(hop_length=hop_length, win_length=win_length, n_fft=n_fft, window=window, center=center,
                    length=length)
        kw_f = dict(n_fft=n_fft, hop_length=hop_length, win_length=win_length, window=window, center=center,
                    pad_mode=pad_mode)
        scale = float(momentum / (1 + momentum))
        tprev = None
        for _ in range(int(n_iter)):
            inverse = sc.own(istft(angles, **kw_i))
            rebuilt = sc.own(stft(inverse, **kw_f))
            inverse.free()
            if tuple(rebuilt.shape) != tuple(S_host_shape):
                # a `length` that does not correspond to T frames: the reference fails at `angles[:] = rebuilt`
                # (core/spectrum.py:2884) with a broadcast error; the update kernel would run out of bounds
                raise ParameterError(f"length={length} gives an STFT of shape {tuple(rebuilt.shape)}, expected "
                                     f"{tuple(S_host_shape)}")
            nat.check(L.b2l_gl_update(ctx.handle, _vp(rebuilt.ptr), _vp(tprev.ptr) if tprev is not None else None,
                                      _vp(S_ft.ptr), scale, eps, _vp(angles.ptr), n_clips * F * T))
            if tprev is not None:
                tprev.free()
            tprev = rebuilt
        return sc.result(istft(angles, **kw_i), np.dtype(dtype) if dtype is not None else s_dtype)
