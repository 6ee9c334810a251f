"""Frame-wise consumers of ``_spectrogram`` with librosa's signatures: ``spectral_centroid``,
``spectral_bandwidth``, ``spectral_rolloff``, ``spectral_flatness``, ``rms`` and ``zero_crossing_rate``
(reference: librosa/feature/spectral.py:46-191, :194-352, :535-684, :687-803, :806-916, :1062-1133).

On the GPU the ``y=`` forms are ONE kernel each: frame, window, real FFT, ``|.|`` and the per-frame
reductions are fused (``fwd_kernel`` MODE_STATS), so the magnitude spectrogram the reference materialises
(cfg-2 batch: 1.8 GB) never exists in HBM; the kernel produces all statistics of a frame at once and each
public function returns its row.  ``S=`` inputs go through ``stats_kernel`` on the stored spectrogram, the
two time-domain framings (``rms(y=...)``, ``zero_crossing_rate``) through ``frame_td_kernel``.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional

import numpy as np

from .. import _native as nat
from .. import _pipeline as pl
from ..core.convert import fft_frequencies
from ..util.exceptions import ParameterError

_vp = C.c_void_p

_NP_PAD_ONLY = ("maximum", "mean", "median", "minimum", "wrap")


def _freq_table(freq, sr, n_fft, n_bins):
    """``freq`` argument of the spectral statistics -> (float32-able table, cache key, result dtype)."""
    if freq is None:
        return fft_frequencies(sr=sr, n_fft=n_fft), ("fftfreq", float(sr), int(n_fft)), np.dtype(np.float64)
    freq = np.asarray(freq)
    if freq.ndim != 1:
        raise nat.UnsupportedOnGPU("time-varying `freq` (ndim > 1) is not supported on the GPU (no CPU fallback)")
    if freq.shape[0] != n_bins:
        raise ValueError(f"operands could not be broadcast together: freq has {freq.shape[0]} bins, S has {n_bins}")
    return freq, ("freq", pl.digest(np.ascontiguousarray(freq, dtype=np.float64))), freq.dtype


def _desc(row, *, roll_percent=0.85, amin=1e-10, power=2.0, p=2.0, norm=True, frame_length=2):
    """struct b2l_stats_desc asking for statistic ``row`` only (the kernel skips what the others need)."""
    return nat.StatsDesc(roll_percent=float(roll_percent), flat_amin=float(amin), flat_power=float(power),
                         bw_p=float(p), bw_norm=int(bool(norm)), frame_length=int(frame_length), want=1 << row)


def _take_row(ctx, stats, lead, T, row, on_device, res_dtype):
    """Row ``row`` of a [clip][N_STATS][T] block -> array of shape lead + (1, T)."""
    n_clips = pl.clip_count(lead)
    if isinstance(stats, np.ndarray):
        out = stats.reshape(n_clips, nat.N_STATS, T)[:, row:row + 1, :].reshape(tuple(lead) + (1, T))
        return np.ascontiguousarray(out).astype(res_dtype, copy=False)
    dst = nat.DeviceArray.empty(ctx, tuple(lead) + (1, T), np.float32)
    if n_clips and T:
        nat.check(nat.lib().b2l_copy2d(ctx.handle, _vp(dst.ptr), T * 4, _vp(stats.ptr + row * T * 4),
                                       nat.N_STATS * T * 4, T * 4, n_clips))
    stats.free()                      # stream-ordered pool: safe right after the copy has been enqueued
    return dst if on_device else pl.finish(dst, res_dtype)


def _stats_from_S(S, desc, freq, sr, n_fft, what, check_negative=True):
    """S= form: stats_kernel over a stored spectrogram.  Returns (stats block, ctx, lead, T, on_device,
    S dtype, freq dtype).  ``check_negative``: fetch the kernel's "negative entry" verdict and raise like the
    reference (skipped for spectrograms this package has just computed itself)."""
    if not isinstance(S, nat.DeviceArray) and np.iscomplexobj(S):
        raise ParameterError(f"{what} is only defined with real-valued input")
    ctx = pl.context_for(S)
    if check_negative:
        nat.check(nat.lib().b2l_status_reset(ctx.handle))
    Sd, req, on_device = pl.spectrogram_input(S)
    if Sd.ndim < 2:
        raise ParameterError("spectrogram input must have at least two dimensions")
    F, T = Sd.shape[-2], Sd.shape[-1]
    if n_fft is None or n_fft // 2 + 1 != F:
        n_fft = 2 * (F - 1)
    table, fkey, fdtype = _freq_table(freq, sr, n_fft, F)
    d_freq = ctx.constant(fkey, lambda: table)
    lead = Sd.shape[:-2]
    src, own = pl.to_native(Sd)
    stats = nat.DeviceArray.empty(ctx, tuple(lead) + (nat.N_STATS, T), np.float32)
    nat.check(nat.lib().b2l_spectral_stats_from_spec(ctx.handle, C.byref(desc), _vp(src.ptr), pl.clip_count(lead), T,
                                                     F, _vp(d_freq), _vp(stats.ptr)))
    if own:
        src.free()
    if not on_device:
        Sd.free()
    if check_negative and pl.status_word(ctx) & 2:
        stats.free()
        raise ParameterError(f"{what} is only defined with non-negative energies")
    return stats, ctx, lead, T, on_device, req, fdtype


def _stats_from_y(y, desc, freq, sr, *, n_fft, hop_length, win_length, window, center, pad_mode, what):
    """y= form: the fused kernel (power-of-two n_fft) or chirp-z spectrogram + stats_kernel."""
    if n_fft is None:
        raise ParameterError(f"Unable to compute spectrogram with n_fft={n_fft}")
    if y is None:
        raise ParameterError("Input signal must be provided to compute a spectrogram")
    fr = pl.forward_front(y, n_fft, hop_length, win_length, window, center, pad_mode, native_ok=False)
    pl.require_supported_n_fft(n_fft)
    table, fkey, fdtype = _freq_table(freq, sr, n_fft, 1 + n_fft // 2)
    if not pl.is_pow2(n_fft):
        from .spectral import _compose_nonpow2

        box = {}

        def tail(Sd):
            stats, ctx, lead, T_, _, _, _ = _stats_from_S(Sd, desc, freq, sr, n_fft, what, check_negative=False)
            box["v"] = (ctx, lead, T_)
            return stats

        on_device = isinstance(y, nat.DeviceArray)
        stats = _compose_nonpow2(y, tail, np.float32, n_fft=n_fft, hop_length=fr.hop, power=1, win_length=win_length,
                                 window=window, center=center, pad_mode=pad_mode)
        ctx, lead, T_ = box["v"]
        return stats, ctx, lead, T_, on_device, fr.dtype, fdtype

    def launch(ctx, plan, d_in, m, n_, d_out, d_scr):
        nat.check(nat.lib().b2l_spectral_stats(ctx.handle, plan.handle, C.byref(desc), _vp(d_in), m, n_, n_,
                                               _vp(ctx.constant(fkey, lambda: table)), _vp(d_out)))

    T = fr.n_frames
    stats = pl.run_forward(y, plan_key=("stats", n_fft, fr.hop, bool(center), fr.mode, fr.wkey),
                           plan_kw=dict(n_fft=n_fft, hop_length=fr.hop, center=center, pad_mode=fr.mode,
                                        window=fr.window, power=1.0),
                           n_frames=T, out_tail=(nat.N_STATS, T), dtype=np.float32, launch=launch)
    on_device = isinstance(y, nat.DeviceArray)
    return stats, pl.context_for(y), tuple(y.shape[:-1]), T, on_device, fr.dtype, fdtype


def _statistic(row, what, desc, res_of, *, y, S, sr, n_fft, hop_length, freq, win_length, window, center, pad_mode):
    if S is not None:
        stats, ctx, lead, T, on_device, sdt, fdt = _stats_from_S(S, desc, freq, sr, n_fft, what)
    else:
        stats, ctx, lead, T, on_device, sdt, fdt = _stats_from_y(
            y, desc, freq, sr, n_fft=n_fft, hop_length=hop_length, win_length=win_length, window=window,
            center=center, pad_mode=pad_mode, what=what)
    return _take_row(ctx, stats, lead, T, row, on_device, res_of(sdt, fdt))


def spectral_centroid(*, y=None, sr: float = 22050, S=None, n_fft: int = 2048, hop_length: int = 512, freq=None,
                      win_length: Optional[int] = None, window="hann", center: bool = True, pad_mode="constant"):
    """Spectral centroid per frame, shape ``(..., 1, t)``; same contract as ``librosa.feature.spectral_centroid``
    (``freq`` must be 1-D or None on the GPU)."""
    return _statistic(nat.STAT_CENTROID, "Spectral centroid", _desc(nat.STAT_CENTROID), lambda s, f: np.result_type(s, f),
                      y=y, S=S, sr=sr, n_fft=n_fft, hop_length=hop_length, freq=freq, win_length=win_length,
                      window=window, center=center, pad_mode=pad_mode)


def spectral_bandwidth(*, y=None, sr: float = 22050, S=None, n_fft: int = 2048, hop_length: int = 512,
                       win_length: Optional[int] = None, window="hann", center: bool = True, pad_mode="constant",
                       freq=None, centroid=None, norm: bool = True, p: float = 2):
    """p-th order spectral bandwidth per frame; same contract as ``librosa.feature.spectral_bandwidth``.
    A caller-supplied ``centroid`` is not supported on the GPU (the kernel uses the frame's own centroid)."""
    if centroid is not None:
        raise nat.UnsupportedOnGPU("spectral_bandwidth(centroid=...) is not supported on the GPU (no CPU fallback)")
    if not p > 0:
        raise ParameterError(f"p={p} must be strictly positive")
    return _statistic(nat.STAT_BANDWIDTH, "Spectral bandwidth", _desc(nat.STAT_BANDWIDTH, p=p, norm=norm),
                      lambda s, f: np.result_type(s, f),
                      y=y, S=S, sr=sr, n_fft=n_fft, hop_length=hop_length, freq=freq, win_length=win_length,
                      window=window, center=center, pad_mode=pad_mode)


def spectral_rolloff(*, y=None, sr: float = 22050, S=None, n_fft: int = 2048, hop_length: int = 512,
                     win_length: Optional[int] = None, window="hann", center: bool = True, pad_mode="constant",
                     freq=None, roll_percent: float = 0.85):
    """Roll-off frequency per frame; same contract as ``librosa.feature.spectral_rolloff``."""
    if not 0.0 < roll_percent < 1.0:
        raise ParameterError("roll_percent must lie in the range (0, 1)")
    return _statistic(nat.STAT_ROLLOFF, "Spectral rolloff", _desc(nat.STAT_ROLLOFF, roll_percent=roll_percent),
                      lambda s, f: np.result_type(s, f),
                      y=y, S=S, sr=sr, n_fft=n_fft, hop_length=hop_length, freq=freq, win_length=win_length,
                      window=window, center=center, pad_mode=pad_mode)


def spectral_flatness(*, y=None, S=None, n_fft: int = 2048, hop_length: int = 512, win_length: Optional[int] = None,
                      window="hann", center: bool = True, pad_mode="constant", amin: float = 1e-10,
                      power: float = 2.0):
    """Spectral flatness per frame; same contract as ``librosa.feature.spectral_flatness``."""
    if amin <= 0:
        raise ParameterError("amin must be strictly positive")
    return _statistic(nat.STAT_FLATNESS, "Spectral flatness", _desc(nat.STAT_FLATNESS, amin=amin, power=power), lambda s, f: np.dtype(s),
                      y=y, S=S, sr=22050, n_fft=n_fft, hop_length=hop_length, freq=None, win_length=win_length,
                      window=window, center=center, pad_mode=pad_mode)


def spectral_contrast(*, y=None, sr: float = 22050, S=None, n_fft: int = 2048, hop_length: int = 512,
                      win_length: Optional[int] = None, window="hann", center: bool = True, pad_mode="constant",
                      freq=None, fmin: float = 200.0, n_bands: int = 6, quantile: float = 0.02,
                      linear: bool = False):
    """Spectral contrast, shape ``(..., n_bands + 1, t)``; same contract as
    ``librosa.feature.spectral_contrast`` (the bins of every octave band must be contiguous, which holds for
    any increasing ``freq``)."""
    from ..core.spectrum import _spectrogram, power_to_db

    staged = None
    if S is None:
        if y is None:
            raise ParameterError("Input signal must be provided to compute a spectrogram")
        _, req = pl.precheck_signal(y)
        staged = pl.StagedInput(y)
        Sd, n_fft = _spectrogram(y=staged.dev, n_fft=n_fft, hop_length=hop_length, power=1, win_length=win_length,
                                 window=window, center=center, pad_mode=pad_mode)
        staged.scan_uncovered(n_fft, hop_length, win_length, center, Sd.shape[-1])
        own_S = True
    else:
        if not isinstance(S, nat.DeviceArray) and np.iscomplexobj(S):
            raise nat.UnsupportedOnGPU("spectral_contrast of a complex S is not supported on the GPU: pass np.abs(S)")
        Sd, req, on_device = pl.spectrogram_input(S)
        own_S = not on_device
        if n_fft is None or n_fft // 2 + 1 != Sd.shape[-2]:
            n_fft = 2 * (Sd.shape[-2] - 1)
    ctx = Sd.ctx
    F, T = Sd.shape[-2], Sd.shape[-1]
    if freq is None:
        freq = fft_frequencies(sr=sr, n_fft=n_fft)
    freq = np.atleast_1d(freq)
    if freq.ndim != 1 or len(freq) != F:
        raise ParameterError(f"freq.shape mismatch: expected ({F:d},)")
    if n_bands < 1 or not isinstance(n_bands, (int, np.integer)):
        raise ParameterError("n_bands must be a positive integer")
    if not 0.0 < quantile < 1.0:
        raise ParameterError("quantile must lie in the range (0, 1)")
    if fmin <= 0:
        raise ParameterError("fmin must be a positive number")
    octa = np.zeros(n_bands + 2)
    octa[1:] = fmin * (2.0 ** np.arange(0, n_bands + 1))
    if np.any(octa[:-1] >= 0.5 * sr):
        raise ParameterError("Frequency band exceeds Nyquist. Reduce either fmin or n_bands.")
    if n_bands + 1 > 16:
        raise nat.UnsupportedOnGPU("spectral_contrast: at most 15 octave bands on the GPU")
    desc = nat.ContrastDesc(n_bands=n_bands + 1)
    for k in range(n_bands + 1):
        # the reference's band mask (feature/spectral.py:483-499), reduced to (first bin, count, tail length)
        band = np.logical_and(freq >= octa[k], freq <= octa[k + 1])
        idx = np.flatnonzero(band)
        if k > 0:
            band[idx[0] - 1] = True
        if k == n_bands:
            band[idx[-1] + 1:] = True
        sel = np.flatnonzero(band)
        if sel.size and sel[-1] - sel[0] + 1 != sel.size:
            raise nat.UnsupportedOnGPU("spectral_contrast: non-contiguous band (freq must be increasing)")
        count = sel.size - (1 if k < n_bands else 0)
        desc.lo[k] = int(sel[0]) if sel.size else 0
        desc.count[k] = max(int(count), 0)
        desc.k[k] = int(max(np.rint(quantile * np.sum(band)), 1))
    lead = Sd.shape[:-2]
    n_clips = pl.clip_count(lead)
    L = nat.lib()
    src, own = pl.to_native(Sd)
    shape = tuple(lead) + (n_bands + 1, T)
    peak = nat.DeviceArray.empty(ctx, shape, np.float32)
    valley = nat.DeviceArray.empty(ctx, shape, np.float32)
    nat.check(L.b2l_spectral_contrast(ctx.handle, C.byref(desc), _vp(src.ptr), n_clips, T, F, _vp(peak.ptr),
                                      _vp(valley.ptr)))
    if own:
        src.free()
    if own_S:
        Sd.free()
    if not linear:
        p_db, v_db = power_to_db(peak), power_to_db(valley)
        peak.free()
        valley.free()
        peak, valley = p_db, v_db
    out = nat.DeviceArray.empty(ctx, shape, np.float32)
    nat.check(L.b2l_sub(ctx.handle, _vp(peak.ptr), _vp(valley.ptr), peak.size, _vp(out.ptr)))
    peak.free()
    valley.free()
    res_dtype = np.result_type(req, np.float64)
    if staged is not None:
        return staged.result(out, res_dtype)
    return out if on_device else pl.finish(out, res_dtype)


# --------------------------------------------------------------------------------------------- time-domain framings
def _frame_feature(what, y, frame_length, hop_length, center, pad_mode, *, threshold=0.0, zero_pos=1, pad_first=0,
                   out_scale=1.0, validate=False):
    """Run frame_td_kernel over ``y`` (host ndarray or DeviceArray) -> (values, on_device) with values of shape
    lead + (1, T) (NumPy float32 array or DeviceArray)."""
    frame_length, hop_length = int(frame_length), int(hop_length)
    n = y.shape[-1]
    padded = n + (2 * (frame_length // 2) if center else 0)
    if padded < frame_length:
        raise ParameterError(f"Input is too short (n={padded}) for frame_length={frame_length}")
    if hop_length < 1:
        raise ParameterError(f"Invalid hop_length: {hop_length}")
    T = pl.frame_count(n, frame_length, hop_length, center)
    staged = pl.StagedInput(y)
    ctx = staged.ctx
    out = nat.DeviceArray.empty(ctx, staged.lead + (1, T), np.float32)
    nat.check(nat.lib().b2l_frame_feature(ctx.handle, what, _vp(staged.dev.ptr), staged.n_clips, staged.n, staged.n,
                                          frame_length, hop_length, int(bool(center)), nat.PAD_MODES[pad_mode],
                                          float(threshold), int(zero_pos), int(pad_first), float(out_scale),
                                          _vp(out.ptr)))
    if staged.on_device:
        return out, True
    if validate:
        staged.scan_uncovered(frame_length, hop_length, None, center, T)
    res = pl.finish(out, validate=validate)
    staged.release()
    return res, False


def rms(*, y=None, S=None, frame_length: int = 2048, hop_length: int = 512, center: bool = True,
        pad_mode="constant", dtype=np.float32):
    """Root-mean-square value per frame from samples ``y`` or from a magnitude spectrogram ``S``; same contract
    as ``librosa.feature.rms``."""
    if y is not None:
        if not isinstance(y, nat.DeviceArray):
            y = np.asarray(y)
            if np.iscomplexobj(y):
                raise nat.UnsupportedOnGPU("rms of a complex signal is not supported on the GPU")
            if y.ndim == 0:
                raise ParameterError("Audio data must be at least one-dimensional")
            if not np.issubdtype(y.dtype, np.floating):
                y = y.astype(np.float32)
            elif y.dtype == np.float64:
                pl.check_real_dtype(y.dtype, "input signal")
        if center:
            if callable(pad_mode):
                raise nat.UnsupportedOnGPU("callable pad_mode cannot run on the GPU (no CPU fallback)")
            if pad_mode in _NP_PAD_ONLY:
                raise nat.UnsupportedOnGPU(f"pad_mode='{pad_mode}' is not supported on the GPU (no CPU fallback)")
            if pad_mode not in nat.PAD_MODES:
                raise ValueError(f"mode '{pad_mode}' is not supported")
        mode = pad_mode if center else "constant"
        res, on_device = _frame_feature(nat.FRAME_RMS, y, frame_length, hop_length, center, mode)
        return res if on_device else res.astype(dtype, copy=False)
    if S is not None:
        if S.shape[-2] != frame_length // 2 + 1:
            raise ParameterError(
                "Since S.shape[-2] is {}, frame_length is expected to be {} or {}; found {}".format(
                    S.shape[-2], S.shape[-2] * 2 - 2, S.shape[-2] * 2 - 1, frame_length))
        if not isinstance(S, nat.DeviceArray) and np.iscomplexobj(S):
            raise nat.UnsupportedOnGPU("rms(S=...) with a complex S is not supported on the GPU: pass np.abs(S)")
        # rms only squares S, so the sign of an entry is irrelevant (no non-negativity requirement)
        stats, ctx, lead, T, on_device, _, _ = _stats_from_S(S, _desc(nat.STAT_RMS, frame_length=frame_length), None, 22050,
                                                             frame_length, "rms", check_negative=False)
        return _take_row(ctx, stats, lead, T, nat.STAT_RMS, on_device, np.dtype(dtype))
    raise ParameterError("Either `y` or `S` must be input.")


def zero_crossing_rate(y, *, frame_length: int = 2048, hop_length: int = 512, center: bool = True, **kwargs):
    """Fraction of zero crossings per frame, shape ``(..., 1, t)`` (float64 for host input, like the reference's
    ``np.mean`` over booleans); ``kwargs``: ``threshold``, ``ref_magnitude`` (number), ``pad``, ``zero_pos``."""
    pl.precheck_signal(y)                     # util.valid_audio (the finite check runs on the device)
    allowed = {"threshold", "ref_magnitude", "pad", "zero_pos", "axis"}
    extra = set(kwargs) - allowed
    if extra:
        raise TypeError(f"zero_crossings() got an unexpected keyword argument '{sorted(extra)[0]}'")
    threshold = kwargs.get("threshold", 1e-10)
    ref_magnitude = kwargs.get("ref_magnitude", None)
    if callable(ref_magnitude):
        raise nat.UnsupportedOnGPU("callable ref_magnitude is not supported on the GPU (no CPU fallback)")
    if ref_magnitude is not None:
        threshold = threshold * ref_magnitude
    # largest float32 not above the (float64) threshold: |x| <= t32 <=> |x| <= threshold for float32 samples
    t32 = np.float32(threshold)
    if float(t32) > float(threshold):
        t32 = np.nextafter(t32, np.float32(-np.inf))
    on_device = isinstance(y, nat.DeviceArray)
    res, _ = _frame_feature(nat.FRAME_ZERO_CROSSINGS, y, frame_length, hop_length, center, "edge",
                            threshold=float(t32), zero_pos=int(bool(kwargs.get("zero_pos", True))),
                            pad_first=int(bool(kwargs.get("pad", False))),
                            out_scale=(1.0 / frame_length) if on_device else 1.0, validate=True)
    if on_device:
        return res
    return res.astype(np.float64) / float(int(frame_length))
