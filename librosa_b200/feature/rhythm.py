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
from ..core.convert import tempo_frequencies
from ..util.exceptions import ParameterError

_vp = C.c_void_p

__all__ = ["tempogram", "fourier_tempogram", "tempo"]

MAX_WIN_LENGTH = 4096   # csrc/rhythm_api.cu: the packed FP64 transform of 8192 points fills 64 KB of shared memory
_STATUS_NOT_FINITE = 4  # bit 2 of the status word: a tempogram value is not finite (b2l_tempogram)


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
        if onset_envelope is None:
            if y is None:
                raise ParameterError("Either y or onset_envelope must be provided")
            pl.precheck_signal(y)
        elif isinstance(onset_envelope, nat.DeviceArray):
            if onset_envelope.dtype not in (np.float32, np.float64) or onset_envelope.layout != "c":
                raise ParameterError("device onset envelope must be a C-ordered float32 or float64 DeviceArray")
        elif np.asarray(onset_envelope).dtype not in (np.float32, np.float64):
            raise nat.UnsupportedOnGPU("onset_envelope must be float32 or float64 on the GPU")
        self.mode, self.p = _norm_mode(norm)
        if win_length > MAX_WIN_LENGTH:
            raise nat.UnsupportedOnGPU(f"tempogram: win_length={win_length} exceeds the {MAX_WIN_LENGTH} onset frames "
                                       "the GPU kernel supports (no CPU fallback)")
        self.win_length = int(win_length)


class _Envelope:
    """The onset envelope of a call on the device, C-ordered (..., n).

    ``y`` runs onset_strength on the device: a host signal is uploaded once and checked like util.valid_audio,
    the envelope never leaves the GPU.  A host envelope is uploaded as it is.  The status word is cleared for this
    call's verdict (``verdict``); ``on_device``: the caller passed device data and gets a DeviceArray back.
    ``aggregate`` is onset_strength's (beat tracking uses np.median)."""

    def __init__(self, y, sr, onset_envelope, hop_length, aggregate=None):
        from ..onset import onset_strength

        self.audio = None
        if onset_envelope is None:
            self.audio = pl.StagedInput(y)
            self.dev = onset_strength(y=self.audio.dev, sr=sr, hop_length=hop_length, aggregate=aggregate)
            self.audio.scan_all()
            self.staged = self.audio
        else:
            x = onset_envelope if isinstance(onset_envelope, nat.DeviceArray) else np.asarray(onset_envelope)
            self.staged = pl.StagedInput(x, dtype=x.dtype)
            self.dev = self.staged.dev
        self.on_device = self.staged.on_device
        self.ctx = self.staged.ctx
        if self.dev.ndim < 1:
            raise ParameterError("onset envelope must be at least one-dimensional")
        if self.on_device:   # a host input was staged after a reset of the status word
            nat.check(nat.lib().b2l_status_reset(self.ctx.handle))

    def release(self):
        self.staged.release()
        self.dev = None   # the envelope onset_strength made goes with its last reference (stream-ordered free)

    def verdict(self):
        """Raise like the reference when a kernel of this call flagged non-finite data (synchronises)."""
        flags = pl.status_word(self.ctx)
        if self.audio is not None and not self.on_device and flags & 1:
            self.audio.check_finite()
        if flags & _STATUS_NOT_FINITE:
            raise ParameterError("Input must be finite")


def _launch_tempogram(env: _Envelope, front: _Front, center: bool) -> nat.DeviceArray:
    """One launch: the float64 tempogram (..., win_length, frames) in layout "ft" (lags contiguous)."""
    ctx, x = env.ctx, env.dev
    W, n, lead = front.win_length, x.shape[-1], x.shape[:-1]
    padded = n + (2 * (W // 2) if center else 0)
    if padded < W:
        raise ParameterError(f"Input is too short (n={padded:d}) for frame_length={W:d}")
    T = n if center else n - W + 1
    out = nat.DeviceArray.empty(ctx, lead + (W, T), np.float64, layout="ft")
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
    env = _Envelope(y, sr, onset_envelope, hop_length)
    try:
        out = _launch_tempogram(env, front, center)
    finally:
        env.release()
    try:
        env.verdict()
    except ParameterError:
        out.free()
        raise
    return out if env.on_device else pl.finish(out)


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
    env = None
    own_tg = False
    if front is not None:
        env = _Envelope(y, sr, onset_envelope, hop_length)
        try:
            d_tg = _launch_tempogram(env, front, center=True)
        finally:
            env.release()
        own_tg, on_device, ctx = True, env.on_device, env.ctx
    elif isinstance(tg, nat.DeviceArray):
        if tg.dtype not in (np.float32, np.float64) or tg.layout not in ("c", "ft"):
            raise ParameterError("device tempogram must be float32 or float64 in layout 'c' or 'ft'")
        d_tg, on_device, ctx = tg, True, tg.ctx
    else:
        tg = np.asarray(tg)
        dtype = tg.dtype if tg.dtype in (np.float32, np.float64) else np.dtype(np.float64)
        d_tg, own_tg = pl.to_native(tg, dtype=dtype, host_transpose=True)
        on_device, ctx = False, d_tg.ctx
    lead, F = d_tg.shape[:-2], d_tg.shape[-1]
    mean = aggregate is not None
    out = nat.DeviceArray.empty(ctx, lead + ((1,) if mean else (F,)), np.float64)
    ft = d_tg.layout == "ft"
    desc = nat.TempoDesc(n_lags=win_length, mean=int(mean), tg_f64=int(d_tg.dtype == np.float64), n_frames=F,
                         row_stride=win_length * F, lag_stride=1 if ft else F, frame_stride=win_length if ft else 1)
    key = ("tempo", pl.digest(bpms), pl.digest(logprior))
    d_bpms = pl.f64_constant(ctx, key + ("bpms",), bpms)
    d_logprior = pl.f64_constant(ctx, key + ("logprior",), logprior)
    try:
        nat.check(nat.lib().b2l_tempo(ctx.handle, C.byref(desc), _vp(d_tg.ptr), pl.clip_count(lead), _vp(d_logprior),
                                      _vp(d_bpms), _vp(out.ptr)))
    finally:
        if own_tg:
            d_tg.free()
    if env is not None:
        try:
            env.verdict()
        except ParameterError:
            out.free()
            raise
    return out if on_device else pl.finish(out)
