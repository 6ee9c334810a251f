"""``librosa.estimate_tuning`` (reference: librosa/core/pitch.py:28-109, on top of ``piptrack`` :182-366 and
``pitch_tuning`` :112-179), as needed by ``feature.chroma_stft``; the pitch trackers ``yin`` and ``pyin``
(:369-968) further down.

The peak picking and parabolic interpolation of ``piptrack`` run on the GPU over the whole spectrogram; the
peak list is never materialised.  The median magnitude that gates the peaks is found exactly by radix selection
over three histogram passes, the tuning by one residual-histogram pass; the host only reads those histograms."""
from __future__ import annotations

import ctypes as C
import warnings
from functools import lru_cache
from typing import Optional

import numpy as np

from .. import _native as nat
from .. import _pipeline as pl
from ..util.exceptions import ParameterError
from ..util.utils import pad_center
from .convert import fft_frequencies

_vp = C.c_void_p


def _key_to_float(key: int) -> np.float32:
    """Inverse of the order-preserving uint32 key of a float32 (csrc/common.cuh float_to_key)."""
    u = (key & 0x7FFFFFFF) if key & 0x80000000 else (~key & 0xFFFFFFFF)
    return np.array([u], dtype=np.uint32).view(np.float32)[0]


def _tuning_from_device_spec(ctx, Sd, sr, n_fft, *, resolution, bins_per_octave, fmin, fmax, threshold, ref):
    """Sd: float32 DeviceArray (..., bins, frames), any layout.  Returns the tuning estimate (float)."""
    F, T = Sd.shape[-2], Sd.shape[-1]
    L = nat.lib()
    src, own = pl.to_native(Sd)
    freqs = fft_frequencies(sr=sr, n_fft=n_fft)
    fmin = np.maximum(fmin, 0)
    fmax = np.minimum(fmax, float(sr) / 2)
    mask = np.flatnonzero((fmin <= freqs) & (freqs < fmax))
    desc = nat.PipDesc(k_lo=int(mask[0]) if mask.size else 0, k_hi=int(mask[-1]) + 1 if mask.size else 0,
                       threshold=float(threshold), ref_abs=-1.0, hz_per_bin=float(sr) / n_fft,
                       bins_per_octave=float(bins_per_octave))
    if ref is not None and ref is not np.max:
        if callable(ref):
            raise nat.UnsupportedOnGPU("piptrack(ref=callable) other than np.max is not supported on the GPU")
        desc.ref_abs = float(np.abs(ref))
    rows = pl.clip_count(Sd.shape[:-2]) * T
    hist = (C.c_uint64 * 2048)()

    def run(mode, prefix=0, mag_threshold=0.0, edges=None, n_res=0):
        desc.mode, desc.prefix, desc.mag_threshold, desc.n_res_bins = mode, prefix, float(mag_threshold), n_res
        e = edges.ctypes.data_as(_vp) if edges is not None else None
        nat.check(L.b2l_pip_pass(ctx.handle, C.byref(desc), _vp(src.ptr), rows, F, e, hist))
        n = n_res if mode == 3 else (1024 if mode == 2 else 2048)
        return np.frombuffer(hist, dtype=np.uint64, count=n).astype(np.int64)

    h0 = run(0)
    n_peaks = int(h0.sum())
    try:
        if n_peaks == 0:
            warnings.warn("Trying to estimate tuning from empty frequency set.", stacklevel=3)
            return 0.0

        def select(rank):
            """float32 value of the peak magnitude with this 0-based rank (ascending)."""
            c0 = np.cumsum(h0)
            b0 = int(np.searchsorted(c0, rank, side="right"))
            r = rank - (int(c0[b0 - 1]) if b0 else 0)
            c1 = np.cumsum(run(1, prefix=b0))
            b1 = int(np.searchsorted(c1, r, side="right"))
            r -= int(c1[b1 - 1]) if b1 else 0
            c2 = np.cumsum(run(2, prefix=(b0 << 11) | b1))
            b2 = int(np.searchsorted(c2, r, side="right"))
            return _key_to_float((b0 << 21) | (b1 << 10) | b2)

        if n_peaks % 2:
            med = select((n_peaks - 1) // 2)
        else:
            lo, hi = select(n_peaks // 2 - 1), select(n_peaks // 2)
            med = np.float32(np.float32(lo + hi) / np.float32(2.0))      # np.median -> mean of the two middles
        edges = np.linspace(-0.5, 0.5, int(np.ceil(1.0 / resolution)) + 1)
        if len(edges) - 1 > 2048:
            raise nat.UnsupportedOnGPU("tuning resolution finer than 1/2048 is not supported on the GPU")
        counts = run(3, mag_threshold=med, edges=np.ascontiguousarray(edges, dtype=np.float64), n_res=len(edges) - 1)
        return edges[int(np.argmax(counts))]
    finally:
        if own:
            src.free()


def estimate_tuning(*, y=None, sr: float = 22050, S=None, n_fft: Optional[int] = 2048, resolution: float = 0.01,
                    bins_per_octave: int = 12, **kwargs):
    """Estimate the tuning deviation (fractions of a bin) of a signal or spectrogram; same contract as
    ``librosa.estimate_tuning`` (``kwargs`` go to ``piptrack``: hop_length, fmin, fmax, threshold, win_length,
    window, center, pad_mode, ref — ``ref`` a number or ``np.max``)."""
    from .spectrum import _spectrogram

    allowed = {"hop_length", "fmin", "fmax", "threshold", "win_length", "window", "center", "pad_mode", "ref"}
    extra = set(kwargs) - allowed
    if extra:
        raise TypeError(f"piptrack() got an unexpected keyword argument '{sorted(extra)[0]}'")
    pip = dict(fmin=kwargs.get("fmin", 150.0), fmax=kwargs.get("fmax", 4000.0), threshold=kwargs.get("threshold", 0.1),
               ref=kwargs.get("ref", None))
    staged = None
    if S is None:
        if y is None:
            raise ParameterError("Input signal must be provided to compute a spectrogram")
        pl.precheck_signal(y)
        staged = pl.StagedInput(y)
        Sd, n_fft = _spectrogram(y=staged.dev, n_fft=n_fft, hop_length=kwargs.get("hop_length"), power=1,
                                 win_length=kwargs.get("win_length"), window=kwargs.get("window", "hann"),
                                 center=kwargs.get("center", True), pad_mode=kwargs.get("pad_mode", "constant"))
        own = True
        staged.scan_uncovered(n_fft, kwargs.get("hop_length"), kwargs.get("win_length"), kwargs.get("center", True),
                              Sd.shape[-1])
    else:
        if not isinstance(S, nat.DeviceArray) and np.iscomplexobj(S):
            S = np.abs(S)
        Sd, _, on_device = pl.spectrogram_input(S)
        own = not on_device
        if n_fft is None or n_fft // 2 + 1 != Sd.shape[-2]:
            n_fft = 2 * (Sd.shape[-2] - 1)
    try:
        est = _tuning_from_device_spec(Sd.ctx, Sd, sr, n_fft, resolution=resolution, bins_per_octave=bins_per_octave,
                                       **pip)
    finally:
        if own:
            Sd.free()
    if staged is not None:
        staged.check_finite()
    return est


# --------------------------------------------------------------------------------------------- yin / pyin
# librosa.yin / librosa.pyin (reference: librosa/core/pitch.py:369-968, sequence.py:1174-1432).  Four kernels
# (csrc/pitch_kernels.cuh): frames -> CMND (register FFT autocorrelation), then the yin decision, or pyin's
# observation candidates and the Viterbi decoding.  The host only checks arguments and builds constant tables.
_PITCH_PAD = ("wrap", "maximum", "mean", "median", "minimum")   # np.pad modes the GPU index map does not cover


def _check_yin_params(*, sr, fmax, fmin, frame_length):
    """librosa/core/pitch.py:934-967."""
    if fmax > sr / 2:
        raise ParameterError(f"fmax={fmax:.3f} cannot exceed Nyquist frequency {sr/2}")
    if fmin >= fmax:
        raise ParameterError(f"fmin={fmin:.3f} must be less than fmax={fmax:.3f}")
    if fmin <= 0:
        raise ParameterError(f"fmin={fmin:.3f} must be strictly positive")
    if sr / fmin >= frame_length - 1:
        fmin_feasible = sr / (frame_length - 1)
        frame_length_feasible = int(np.ceil(sr / fmin) + 1)
        raise ParameterError(
            f"fmin={fmin:.3f} is too small for frame_length={frame_length} and sr={sr}. "
            f"Either increase to fmin={fmin_feasible:.3f} or frame_length={frame_length_feasible}")
    if sr / fmin >= frame_length // 2:
        fmin_optimal = sr / (frame_length / 2)
        frame_length_optimal = int(np.ceil(sr / fmin) * 2 + 1)
        warnings.warn(
            f"With fmin={fmin:.3f}, sr={sr} and frame_length={frame_length}, less than two periods of fmin "
            f"fit into the frame, which can cause inaccurate pitch detection. "
            f"Consider increasing to fmin={fmin_optimal:.3f} or frame_length={frame_length_optimal}.",
            stacklevel=4)


class _Frames:
    """Argument checks, framing geometry and the staged input shared by yin and pyin, in the reference's order:
    the yin parameters, util.valid_audio, np.pad's mode, util.frame's length check."""

    def __init__(self, y, *, fmin, fmax, sr, frame_length, hop_length, center, pad_mode):
        if fmin is None or fmax is None:
            raise ParameterError('both "fmin" and "fmax" must be provided')
        _check_yin_params(sr=sr, fmax=fmax, fmin=fmin, frame_length=frame_length)
        if hop_length is None:
            hop_length = frame_length // 4
        n, _ = pl.precheck_signal(y, stacklevel=5)
        if center:
            if callable(pad_mode):
                raise nat.UnsupportedOnGPU("callable pad_mode cannot run on the GPU (no CPU fallback)")
            if pad_mode in _PITCH_PAD:
                raise nat.UnsupportedOnGPU(f"pad_mode='{pad_mode}' is not supported on the GPU (no CPU fallback)")
            if pad_mode not in nat.PAD_MODES:
                raise ValueError(f"mode '{pad_mode}' is not supported")   # what np.pad raises
        padded = n + (2 * (frame_length // 2) if center else 0)
        if padded < frame_length:
            raise ParameterError(f"Input is too short (n={padded:d}) for frame_length={frame_length:d}")
        if hop_length < 1:
            raise ParameterError(f"Invalid hop_length: {hop_length:d}")
        self.frame_length, self.hop, self.center = int(frame_length), int(hop_length), bool(center)
        self.n_frames = 1 + (padded - frame_length) // self.hop
        self.min_period = int(np.floor(sr / fmax))
        self.max_period = min(int(np.ceil(sr / fmin)), frame_length - 1)
        self.n_lags = self.max_period - self.min_period + 1
        self.desc = nat.YinDesc(frame_length=self.frame_length, hop_length=self.hop, center=int(self.center),
                                pad_mode=nat.PAD_MODES[pad_mode if center else "constant"],
                                min_period=self.min_period, max_period=self.max_period, sr=float(sr))
        self.y = y

    def cmnd(self):
        """Stage the signal and run the CMND kernel: (staged input, device pointer of [rows][n_lags] float32)."""
        staged = pl.StagedInput(self.y)
        ctx = staged.ctx
        self.rows = staged.n_clips * self.n_frames
        d_cmnd = ctx.alloc(self.rows * self.n_lags * 4)
        try:
            nat.check(nat.lib().b2l_yin_cmnd(ctx.handle, C.byref(self.desc), _vp(staged.dev.ptr), staged.n_clips,
                                             staged.n, staged.n, _vp(d_cmnd)))
            staged.scan_uncovered(self.frame_length, self.hop, self.frame_length, self.center, self.n_frames)
        except Exception:
            ctx.free(d_cmnd)
            raise
        return staged, d_cmnd


def yin(y: np.ndarray, *, fmin: float, fmax: float, sr: float = 22050, frame_length: int = 2048,
        hop_length: Optional[int] = None, trough_threshold: float = 0.1, center: bool = True,
        pad_mode="constant"):
    """Fundamental frequency (F0) estimation with YIN; same contract as ``librosa.yin``.

    ``y`` (..., n) host or device float32 (float64 is computed in float32, see ``B2L_FLOAT64``).  Returns float64
    ``f0`` (..., n_frames): a NumPy array for host input, a DeviceArray for device input."""
    fr = _Frames(y, fmin=fmin, fmax=fmax, sr=sr, frame_length=frame_length, hop_length=hop_length, center=center,
                 pad_mode=pad_mode)
    staged, d_cmnd = fr.cmnd()
    ctx = staged.ctx
    try:
        f0 = nat.DeviceArray.empty(ctx, staged.lead + (fr.n_frames,), np.float64)
        fr.desc.trough_threshold = float(trough_threshold)
        nat.check(nat.lib().b2l_yin_pick(ctx.handle, C.byref(fr.desc), _vp(d_cmnd), fr.rows, _vp(f0.ptr)))
    finally:
        ctx.free(d_cmnd)
    staged.release()
    return staged.result(f0)


def _transition_loop(n_states, prob):
    """librosa/sequence.py:1905-1967 for a scalar probability."""
    prob = np.asarray(prob, dtype=np.float64)
    if np.any(prob < 0) or np.any(prob > 1):
        raise ParameterError(f"prob={np.tile(prob, n_states)} must have values in the range [0, 1]")
    transition = np.empty((n_states, n_states), dtype=np.float64)
    for i in range(n_states):
        transition[i] = (1.0 - prob) / (n_states - 1)
        transition[i, i] = prob
    return transition


def _transition_local(n_states, width):
    """librosa/sequence.py:2034-2146 for a scalar width, triangle window, no wrap: (the window padded to n_states,
    the row sums before normalisation, the normalised matrix)."""
    import scipy.signal

    if not (n_states > 1):
        raise ParameterError(f"n_states={n_states} must be a positive integer > 1")
    if width < 1:
        raise ParameterError(f"width={np.tile(width, n_states)} must be at least 1")
    transition = np.zeros((n_states, n_states), dtype=np.float64)
    row = pad_center(scipy.signal.get_window("triangle", width, fftbins=False), size=n_states)
    for i in range(n_states):
        trans_row = np.roll(row, n_states // 2 + i + 1)
        trans_row[min(n_states, i + width // 2 + 1):] = 0
        trans_row[: max(0, i - width // 2)] = 0
        transition[i] = trans_row
    sums = transition.sum(axis=1, keepdims=True)
    transition /= sums
    return row, sums[:, 0], transition


@lru_cache(maxsize=8)
def _viterbi_tables(n_pitch_bins, width, switch_prob, transition_min_prob):
    """log(T + tiny) of pyin's transition matrix T = kron(transition_loop(2, 1 - switch_prob), transition_local(...))
    in the form the Viterbi kernel reads (include/b2l.h, b2l_pyin_desc), plus the search threshold.

    local[p, q] = window(q - p) / rowsum[p], so a value depends on the class of rowsum[p] (rows whose sums are equal
    to the last bit), on q - p and on whether the transition switches voicing: a table of classes x 2 x (2 hw + 1)
    values.  Each is formed with the reference's own operations and the whole form is compared with the dense
    matrix, so the kernel sees exactly the reference's log_trans and predecessor sets (flatnonzero(log_trans[:, j] >=
    log_thr), librosa/sequence.py:1215-1224)."""
    eps = np.finfo(np.float64).tiny
    row, sums, local = _transition_local(n_pitch_bins, width)
    t_switch = _transition_loop(2, 1 - switch_prob)
    log_trans = np.log(np.kron(t_switch, local) + eps)
    if transition_min_prob is not None and transition_min_prob > 0:
        log_thr = np.log(transition_min_prob + eps)
    elif transition_min_prob is None or transition_min_prob == 0:
        log_thr = -np.inf
    else:
        raise ParameterError(f"Invalid transition_min_prob={transition_min_prob}, must be None or non-negative.")
    S = 2 * n_pitch_bins
    if np.isfinite(log_thr):
        empty = np.flatnonzero(~(log_trans >= log_thr).any(axis=0))
        if empty.size:
            raise ParameterError(f"Empty transition matrix detected for state {empty[0]} in Viterbi. "
                                 f"Try reducing your minimum transition probability threshold.")
    hw = width // 2
    classes, cls = np.unique(sums, return_inverse=True)
    d = np.arange(-hw, hw + 1)
    wd = row[(d - n_pitch_bins // 2 - 1) % n_pitch_bins]              # window value at q - p = d (np.roll above)
    ltab = np.empty((len(classes), 2, len(d)))
    for c, s_c in enumerate(classes):
        for h, sw in enumerate((t_switch[0, 0], t_switch[0, 1])):
            ltab[c, h] = np.log(sw * (wd / s_c) + eps)
    # the same matrix rebuilt from the table: exact by construction, checked once per configuration
    p = np.arange(n_pitch_bins)
    dd = p[np.newaxis, :] - p[:, np.newaxis]                          # q - p for [p, q]
    inside = np.abs(dd) <= hw
    rebuilt = np.full((S, S), np.log(eps))
    for a in range(2):
        for b in range(2):
            blk = np.full((n_pitch_bins, n_pitch_bins), np.log(eps))
            blk[inside] = ltab[cls[:, np.newaxis].repeat(n_pitch_bins, 1)[inside], int(a != b), dd[inside] + hw]
            rebuilt[a * n_pitch_bins:(a + 1) * n_pitch_bins, b * n_pitch_bins:(b + 1) * n_pitch_bins] = blk
    if not np.array_equal(rebuilt.view(np.int64), log_trans.view(np.int64)):
        raise nat.UnsupportedOnGPU("pyin: the transition matrix has no compact form on the GPU for these parameters")
    full = not np.isfinite(log_thr) or np.log(eps) >= log_thr
    return dict(half_width=hw, full=int(full), log_thr=float(log_thr) if np.isfinite(log_thr) else -1e308,
                cls=cls.astype(np.int32), ltab=ltab)


@lru_cache(maxsize=8)
def _obs_tables(n_thresholds, beta_parameters, boltzmann_parameter, max_cand):
    """Threshold grid, beta weights, their prefix sums np.sum(beta[:c]) and the Boltzmann prior
    scipy.stats.boltzmann.pmf(pos, lambda, n) for n = 1 .. max_cand (librosa/core/pitch.py:800-904)."""
    import scipy.stats

    thresholds = np.linspace(0, 1, n_thresholds + 1)
    beta = np.diff(scipy.stats.beta.cdf(thresholds, beta_parameters[0], beta_parameters[1]))
    beta_cum = np.array([np.sum(beta[:c]) for c in range(n_thresholds + 1)])
    n = np.repeat(np.arange(1, max_cand + 1), np.arange(1, max_cand + 1))
    pos = np.arange(len(n)) - (n * (n - 1)) // 2
    pmf = scipy.stats.boltzmann.pmf(pos, boltzmann_parameter, n)
    return thresholds, beta, beta_cum, pmf


# 18 bytes of shared memory per Viterbi state (csrc/pitch_kernels.cuh viterbi_smem) within the 227 KiB an H100 CTA
# may opt into; checked here before the host builds the transition tables of an oversized configuration
_VITERBI_MAX_STATES = min(65535, (227 * 1024) // 18)


def _pyin_setup(where, *, min_period, max_period, hop_length, sr, fmin, fmax, n_thresholds, beta_parameters,
                boltzmann_parameter, resolution, max_transition_rate, switch_prob, no_trough_prob, fill_na,
                transition_min_prob):
    """The b2l_pyin_desc of one configuration, its device tables cached by the context of ``where`` (a signal or a
    DeviceArray; the host tables are built, and their argument errors raised, before any device is touched):
    (context, desc, max_cand)."""
    n_bins_per_semitone = int(np.ceil(1.0 / resolution))
    n_pitch_bins = int(np.floor(12 * n_bins_per_semitone * np.log2(fmax / fmin))) + 1
    if 2 * n_pitch_bins > _VITERBI_MAX_STATES:
        raise nat.UnsupportedOnGPU(f"pyin: {2 * n_pitch_bins} Viterbi states (resolution={resolution}) exceed the "
                                   f"{_VITERBI_MAX_STATES} that fit in shared memory")
    max_semitones_per_frame = round(max_transition_rate * 12 * hop_length / sr)
    width = max_semitones_per_frame * n_bins_per_semitone + 1
    vt = _viterbi_tables(n_pitch_bins, width, float(switch_prob), transition_min_prob)
    max_cand = (max_period - min_period + 2) // 2
    bp = tuple(float(b) for b in beta_parameters)
    thresholds, beta, beta_cum, pmf = _obs_tables(int(n_thresholds), bp, boltzmann_parameter, max_cand)
    ctx = pl.context_for(where)
    okey = ("pyin_obs", int(n_thresholds), bp, boltzmann_parameter, max_cand)
    vkey = ("pyin_viterbi", n_pitch_bins, width, float(switch_prob), transition_min_prob)
    desc = nat.PyinDesc(min_period=min_period, max_period=max_period, n_thresholds=int(n_thresholds),
                        n_pitch_bins=n_pitch_bins, n_bins_per_semitone=n_bins_per_semitone, sr=float(sr),
                        fmin=float(fmin), no_trough_prob=float(no_trough_prob),
                        log_p_init=float(np.log(1.0 / (2 * n_pitch_bins) + np.finfo(np.float64).tiny)),
                        fill_na=float(fill_na) if fill_na is not None else 0.0, fill=int(fill_na is not None),
                        half_width=vt["half_width"], full=vt["full"], log_thr=vt["log_thr"])
    for name, arr in (("thresholds", thresholds), ("beta", beta), ("beta_cum", beta_cum), ("pmf", pmf)):
        setattr(desc, "d_" + name, pl.f64_constant(ctx, okey + (name,), arr))
    for name in ("cls", "ltab"):
        setattr(desc, "d_" + name, pl.f64_constant(ctx, vkey + (name,), vt[name]))
    freqs = fmin * 2 ** (np.arange(n_pitch_bins) / (12 * n_bins_per_semitone))
    desc.d_freqs = pl.f64_constant(ctx, vkey + ("freqs", float(fmin), n_bins_per_semitone), freqs)
    return ctx, desc, max_cand


def pyin(y: np.ndarray, *, fmin: float, fmax: float, sr: float = 22050, frame_length: int = 2048,
         hop_length: Optional[int] = None, n_thresholds: int = 100, beta_parameters=(2, 18),
         boltzmann_parameter: float = 2, resolution: float = 0.1, max_transition_rate: float = 35.92,
         switch_prob: float = 0.01, no_trough_prob: float = 0.01, fill_na: Optional[float] = np.nan,
         center: bool = True, pad_mode="constant", transition_min_prob: Optional[float] = 1e-4):
    """Fundamental frequency (F0) estimation with probabilistic YIN; same contract as ``librosa.pyin``.

    Returns ``(f0, voiced_flag, voiced_prob)`` (..., n_frames): float64, bool, float64 — NumPy arrays for host input,
    DeviceArrays for device input."""
    fr = _Frames(y, fmin=fmin, fmax=fmax, sr=sr, frame_length=frame_length, hop_length=hop_length, center=center,
                 pad_mode=pad_mode)
    ctx, desc, max_cand = _pyin_setup(y, min_period=fr.min_period, max_period=fr.max_period, hop_length=fr.hop,
                                      sr=sr, fmin=fmin, fmax=fmax, n_thresholds=n_thresholds,
                                      beta_parameters=beta_parameters, boltzmann_parameter=boltzmann_parameter,
                                      resolution=resolution, max_transition_rate=max_transition_rate,
                                      switch_prob=switch_prob, no_trough_prob=no_trough_prob, fill_na=fill_na,
                                      transition_min_prob=transition_min_prob)
    staged, d_cmnd = fr.cmnd()
    lead, rows = staged.lead, fr.rows
    L = nat.lib()
    d_count = ctx.alloc(rows * 4)
    d_bin = ctx.alloc(rows * max_cand * 4)
    d_prob = ctx.alloc(rows * max_cand * 8)
    d_states = ctx.alloc(rows * 2)
    try:
        vp = nat.DeviceArray.empty(ctx, lead + (fr.n_frames,), np.float64)
        f0 = nat.DeviceArray.empty(ctx, lead + (fr.n_frames,), np.float64)
        vf = nat.DeviceArray.empty(ctx, lead + (fr.n_frames,), np.bool_)
        nat.check(L.b2l_pyin_obs(ctx.handle, C.byref(desc), _vp(d_cmnd), rows, _vp(d_count), _vp(d_bin), _vp(d_prob),
                                 _vp(vp.ptr)))
        nat.check(L.b2l_viterbi(ctx.handle, C.byref(desc), _vp(d_count), _vp(d_bin), _vp(d_prob), _vp(vp.ptr),
                                staged.n_clips, fr.n_frames, _vp(d_states), _vp(f0.ptr), _vp(vf.ptr)))
    finally:
        for p in (d_cmnd, d_count, d_bin, d_prob, d_states):
            ctx.free(p)
    staged.release()
    if staged.on_device:
        return f0, vf, vp
    out_f0 = pl.finish(f0, validate=True)
    return out_f0, pl.finish(vf), pl.finish(vp)
