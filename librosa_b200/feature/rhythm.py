"""``librosa.feature.tempogram``, ``fourier_tempogram`` and ``tempo`` (reference: librosa/feature/rhythm.py:38-470).

``tempogram`` is one kernel launch over every (envelope row, frame): linear-ramp padding, window, autocorrelation
and ``util.normalize`` (csrc/rhythm_kernels.cuh).  The reference computes the tempogram in float64 whatever the
envelope's dtype (its float64 window promotes the frames before the autocorrelation), so the kernel's arithmetic is
FP64 for float32 and float64 envelopes alike and ``B2L_FLOAT64`` does not apply.  ``tempo`` adds one launch for the
prior-weighted argmax over the lags; ``fourier_tempogram`` is ``stft`` at hop 1.  With ``y=``, tempogram and tempo
compute the onset envelope on the device and it never leaves it."""
from __future__ import annotations

import ctypes as C

import numpy as np

from .. import _native as nat
from .. import _pipeline as pl
from .. import filters
from .._pipeline import Envelope as _Envelope
from ..core.convert import tempo_frequencies
from ..util.exceptions import ParameterError

_vp = C.c_void_p

__all__ = ["tempogram", "fourier_tempogram", "tempo"]

MAX_WIN_LENGTH = 4096   # csrc/rhythm_api.cu: the packed FP64 transform of 8192 points fills 64 KB of shared memory


def _norm_mode(norm):
    """util.normalize's choice of norm: (B2L_TG_NORM_*, exponent)."""
    if norm is None:
        return nat.TG_NORM_NONE, 0.0
    if norm == np.inf:
        return nat.TG_NORM_MAX, 0.0
    if norm == -np.inf:
        return nat.TG_NORM_MIN, 0.0
    if norm == 0:
        return nat.TG_NORM_COUNT, 0.0
    if np.issubdtype(type(norm), np.number) and norm > 0:
        return nat.TG_NORM_P, float(norm)
    raise ParameterError(f"Unsupported norm: {norm!r}")


def _time_to_frames(seconds, sr, hop_length) -> int:
    """core/convert.py time_to_frames of a scalar: whole samples, then whole hops."""
    samples = (np.asanyarray(seconds) * sr).astype(int)
    return int(np.floor(samples // hop_length).astype(int))


class _Front:
    """tempogram's argument checks in the reference's order (win_length, window, input), then the GPU's own limits
    and the norm — all before any device work."""

    def __init__(self, y, onset_envelope, win_length, window, norm):
        if win_length < 1:
            raise ParameterError("win_length must be a positive integer")
        self.window = np.ascontiguousarray(filters.get_window(window, win_length, fftbins=True), dtype=np.float64)
        pl.check_envelope(y, onset_envelope)
        self.mode, self.p = _norm_mode(norm)
        if win_length > MAX_WIN_LENGTH:
            raise nat.UnsupportedOnGPU(f"tempogram: win_length={win_length} exceeds the {MAX_WIN_LENGTH} onset frames "
                                       "the GPU kernel supports (no CPU fallback)")
        self.win_length = int(win_length)


def _launch_tempogram(sc: pl.Scope, x: nat.DeviceArray, front: _Front, center: bool) -> nat.DeviceArray:
    """One launch on the envelope ``x``: the float64 tempogram (..., win_length, frames) in layout "ft" (lags
    contiguous)."""
    ctx = sc.ctx
    W, n, lead = front.win_length, x.shape[-1], x.shape[:-1]
    padded = n + (2 * (W // 2) if center else 0)
    if padded < W:
        raise ParameterError(f"Input is too short (n={padded:d}) for frame_length={W:d}")
    T = n if center else n - W + 1
    out = sc.empty(lead + (W, T), np.float64, layout="ft")
    desc = nat.TempogramDesc(win_length=W, center=int(bool(center)), norm=front.mode,
                             env_f64=int(x.dtype == np.float64), norm_p=front.p)
    d_win = pl.f64_constant(ctx, ("tempogram_window", pl.digest(front.window)), front.window)
    nat.check(nat.lib().b2l_tempogram(ctx.handle, C.byref(desc), _vp(x.ptr), pl.clip_count(lead), n, _vp(d_win),
                                      _vp(out.ptr)))
    return out


def tempogram(*, y=None, sr: float = 22050, onset_envelope=None, hop_length: int = 512, win_length: int = 384,
              center: bool = True, window="hann", norm=np.inf):
    """Local autocorrelation of the onset strength envelope; same contract as ``librosa.feature.tempogram``.

    Returns float64 ``(..., win_length, n)``: a NumPy array for host input, a DeviceArray in layout "ft" (memory
    ``[...][frame][lag]``) for device input."""
    front = _Front(y, onset_envelope, win_length, window, norm)
    with pl.Scope(y if onset_envelope is None else onset_envelope) as sc:
        env = _Envelope(y, sr, onset_envelope, hop_length)
        try:
            out = _launch_tempogram(sc, env.dev, front, center)
        finally:
            env.release()
        env.verdict()
        return sc.result(out)


def fourier_tempogram(*, y=None, sr: float = 22050, onset_envelope=None, hop_length: int = 512,
                      win_length: int = 384, center: bool = True, window="hann"):
    """Short-time Fourier transform of the onset strength envelope (``stft`` with ``n_fft=win_length`` at hop 1);
    same contract as ``librosa.feature.fourier_tempogram``.  The envelope of ``y=`` has the dtype onset_strength
    gives it, so a float64 signal takes the FP64 ``stft`` as in the reference."""
    from ..core.spectrum import stft
    from ..onset import onset_strength

    if win_length < 1:
        raise ParameterError("win_length must be a positive integer")
    if onset_envelope is None:
        if y is None:
            raise ParameterError("Either y or onset_envelope must be provided")
        onset_envelope = onset_strength(y=y, sr=sr, hop_length=hop_length)
    return stft(onset_envelope, n_fft=win_length, hop_length=1, center=center, window=window)


def _prior_tables(win_length, *, sr, hop_length, start_bpm, std_bpm, max_tempo, prior):
    """The lag BPMs and the log prior over them, -inf above max_tempo (float64, host)."""
    bpms = tempo_frequencies(win_length, hop_length=hop_length, sr=sr)
    if prior is None:
        logprior = -0.5 * ((np.log2(bpms) - np.log2(start_bpm)) / std_bpm) ** 2
    else:
        logprior = np.array(prior.logpdf(bpms), dtype=np.float64)
    if max_tempo is not None:
        logprior[: int(np.argmax(bpms < max_tempo))] = -np.inf
    return bpms, np.ascontiguousarray(logprior, dtype=np.float64)


def tempo(*, y=None, sr: float = 22050, onset_envelope=None, tg=None, hop_length: int = 512, start_bpm: float = 120,
          std_bpm: float = 1.0, ac_size: float = 8.0, max_tempo=320.0, aggregate=np.mean, prior=None):
    """Estimate the tempo (beats per minute); same contract as ``librosa.feature.tempo``.

    ``aggregate`` is ``np.mean`` or ``None``; ``prior`` any object with ``logpdf`` (a scipy.stats distribution).
    ``tg`` may be a host array or a DeviceArray in layout "c" or "ft", float32 or float64.  Returns float64
    ``(..., 1)`` (mean) or ``(..., n_frames)`` (``aggregate=None``): a NumPy array for host input, a DeviceArray for
    device input."""
    if start_bpm <= 0:
        raise ParameterError("start_bpm must be strictly positive")
    front = None
    if tg is None:
        front = _Front(y, onset_envelope, _time_to_frames(ac_size, sr, hop_length), "hann", np.inf)
        win_length = front.win_length
    else:
        win_length = tg.shape[-2]
    if aggregate is not None and aggregate is not np.mean:
        raise nat.UnsupportedOnGPU("tempo: only aggregate=np.mean or None is computed on the GPU (no CPU fallback)")
    bpms, logprior = _prior_tables(win_length, sr=sr, hop_length=hop_length, start_bpm=start_bpm, std_bpm=std_bpm,
                                   max_tempo=max_tempo, prior=prior)
    source = tg if tg is not None else y if onset_envelope is None else onset_envelope
    with pl.Scope(source) as sc:
        env = None
        if front is not None:
            env = _Envelope(y, sr, onset_envelope, hop_length)
            try:
                d_tg = _launch_tempogram(sc, env.dev, front, center=True)
            finally:
                env.release()
        elif isinstance(tg, nat.DeviceArray):
            if tg.dtype not in (np.float32, np.float64) or tg.layout not in ("c", "ft"):
                raise ParameterError("device tempogram must be float32 or float64 in layout 'c' or 'ft'")
            d_tg = tg
        else:
            tg = np.asarray(tg)
            dtype = tg.dtype if tg.dtype in (np.float32, np.float64) else np.dtype(np.float64)
            d_tg = sc.native(tg, dtype=dtype, host_transpose=True)
        ctx = sc.ctx
        lead, F = d_tg.shape[:-2], d_tg.shape[-1]
        mean = aggregate is not None
        out = sc.empty(lead + ((1,) if mean else (F,)), np.float64)
        ft = d_tg.layout == "ft"
        desc = nat.TempoDesc(n_lags=win_length, mean=int(mean), tg_f64=int(d_tg.dtype == np.float64), n_frames=F,
                             row_stride=win_length * F, lag_stride=1 if ft else F, frame_stride=win_length if ft else 1)
        key = ("tempo", pl.digest(bpms), pl.digest(logprior))
        d_bpms = pl.f64_constant(ctx, key + ("bpms",), bpms)
        d_logprior = pl.f64_constant(ctx, key + ("logprior",), logprior)
        nat.check(nat.lib().b2l_tempo(ctx.handle, C.byref(desc), _vp(d_tg.ptr), pl.clip_count(lead), _vp(d_logprior),
                                      _vp(d_bpms), _vp(out.ptr)))
        if env is not None:
            env.verdict()
        return sc.result(out)
