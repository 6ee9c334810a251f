"""``cqt`` / ``vqt`` with librosa's signatures, executed by libb2l.so on an H100 (reference:
librosa/core/constantq.py:620-1266).

The octave pyramid runs on the device with one staging of the input and no host round trip: an optional early
downsample by 2^k (polyphase resampler), then per octave, from the top down, a centred STFT with a rectangular
window into frame-major scratch and a halving of the signal for the next octave.  One launch of
``b2l_cqt_project`` then applies every octave's sparse complex filter basis and writes the stacked result.  The
filter bases, frequencies and lengths are host constants built with the reference's float64 expressions.
"""
from __future__ import annotations

import ctypes as C
import warnings
from typing import NamedTuple, Optional, Tuple

import numpy as np
import scipy.fft

from .. import _native as nat
from .. import _pipeline as pl
from .. import filters
from ..util.exceptions import ParameterError
from ..util.utils import dtype_r2c
from .audio import _poly_filter

__all__ = ["cqt", "vqt", "cqt_frequencies"]

_vp = C.c_void_p


def cqt_frequencies(n_bins: int, *, fmin: float, bins_per_octave: int = 12, tuning: float = 0.0) -> np.ndarray:
    """Centre frequencies of the constant-Q bins (librosa/core/convert.py:1395-1429)."""
    correction = 2.0 ** (float(tuning) / bins_per_octave)
    return correction * fmin * 2.0 ** (np.arange(0, n_bins, dtype=float) / bins_per_octave)


def _default_fmin() -> float:
    """note_to_hz("C1"): MIDI note 24 through midi_to_hz's expression."""
    return float(440.0 * (2.0 ** ((np.asanyarray(24) - 69.0) / 12.0)))


def _interval_frequencies(n_bins: int, fmin: float, intervals, bins_per_octave: int) -> np.ndarray:
    """interval_frequencies(sort=True) for "equal" and explicit ratios (librosa/core/intervals.py:23-134)."""
    if isinstance(intervals, str):
        if intervals != "equal":
            raise nat.UnsupportedOnGPU(f"vqt(intervals={intervals!r}): only 'equal' and explicit interval ratios are "
                                       "supported (the named just-intonation sets are not part of this library)")
        ratios = 2.0 ** ((0.0 + np.arange(0, bins_per_octave, dtype=float)) / bins_per_octave)
    else:
        ratios = np.array(intervals)
        bins_per_octave = len(ratios)
    n_octaves = np.ceil(n_bins / bins_per_octave)
    all_ratios = np.sort(np.multiply.outer(2.0 ** np.arange(n_octaves), ratios).flatten()[:n_bins])
    return all_ratios * fmin


def _clip_freqs(freqs, window, filter_scale, gamma, sr) -> np.ndarray:
    """n_bins=None: the frequencies whose filters stay below sr/2 (librosa/core/constantq.py:1599-1659)."""
    logf = np.log2(freqs)
    bpo = 1 / np.diff(logf, prepend=0)
    bpo[0] = 1 / (logf[1] - logf[0])
    alpha = (2.0 ** (2 / bpo) - 1) / (2.0 ** (2 / bpo) + 1)
    offset = alpha * 24.7 / 0.108 if gamma is None else gamma
    Q = float(filter_scale) / alpha
    f_cutoff = np.maximum.accumulate(freqs * (1 + 0.5 * filters.window_bandwidth(window) / Q) + 0.5 * offset)
    idx = np.searchsorted(f_cutoff, sr / 2.0, side="left")
    if idx < 1:
        raise ParameterError(f"Unable to construct wavelet basis for fmin={freqs[0]:.2f} Hz and sr={sr:.2f} Hz.")
    return freqs[:idx]


def _two_factors(x: int) -> int:
    n = 0
    while x > 0 and x % 2 == 0:
        n += 1
        x //= 2
    return n


class Basis(NamedTuple):
    """One octave's sparse filter basis as ``scipy.sparse.csr_array`` stores it (complex64 data)."""
    indptr: np.ndarray
    indices: np.ndarray
    data: np.ndarray
    n_fft: int


def _sparsify(x: np.ndarray, quantile: float, dtype) -> np.ndarray:
    """util.sparsify_rows as a dense array: per row, drop the smallest entries holding ``quantile`` of the row's
    total magnitude (librosa/util/utils.py:1500-1597)."""
    if not 0.0 <= quantile < 1:
        raise ParameterError(f"Invalid quantile {quantile:.2f}")
    mags = np.abs(x)
    norms = np.sum(mags, axis=1, keepdims=True)
    mag_sort = np.sort(mags, axis=1)
    cumulative = np.cumsum(mag_sort / norms, axis=1)
    thresh = mag_sort[np.arange(x.shape[0]), np.argmin(cumulative < quantile, axis=1)]
    return (x * (mags >= thresh[:, np.newaxis])).astype(dtype, copy=False)


def filter_basis(sr, freqs, alpha, filter_scale, norm, sparsity, window, gamma, rescale) -> Basis:
    """The FFT of one octave's wavelets at rate ``sr``, rescaled by ``lengths / n_fft``, non-negative bins only,
    sparsified and multiplied by ``rescale`` (sqrt of the top rate over this octave's rate) (librosa/core/constantq.py:1067-1080, 1123-1166)."""
    basis, lengths = filters.wavelet(freqs=freqs, sr=sr, filter_scale=filter_scale, norm=norm, pad_fft=True,
                                     window=window, gamma=gamma, alpha=alpha)
    n_fft = basis.shape[1]
    basis *= lengths[:, np.newaxis] / float(n_fft)
    fft_basis = scipy.fft.fft(basis, n=n_fft, axis=1)[:, : (n_fft // 2) + 1]
    dense = _sparsify(fft_basis, sparsity, np.complex64)
    rows, cols = np.nonzero(dense)
    data = (dense[rows, cols] * np.float64(rescale)).astype(np.complex64)
    indptr = np.zeros(dense.shape[0] + 1, dtype=np.int32)
    np.cumsum(np.bincount(rows, minlength=dense.shape[0]), out=indptr[1:])
    return Basis(indptr, cols.astype(np.int32), data, int(n_fft))


class Octave(NamedTuple):
    sr: float            # sampling rate of this octave's signal
    n: int               # its length
    hop: int
    n_fft: int
    n_frames: int
    rows: slice          # rows of ``freqs`` this octave's basis covers
    resample_after: bool


class Plan(NamedTuple):
    freqs: np.ndarray
    alpha: np.ndarray
    lengths: np.ndarray    # at the post-downsampling rate, for scale=True
    n_bins: int
    early: int             # early downsampling factor (1: none)
    early_scale: float     # the resampler's output scale of the early step
    sr: float              # rate after early downsampling
    octaves: Tuple[Octave, ...]
    n_frames: int


def plan(n: int, *, sr, hop_length, fmin, n_bins, intervals, gamma, bins_per_octave, filter_scale, window, scale,
         res_type) -> Plan:
    """The host half of vqt (librosa/core/constantq.py:992-1100) for a signal of ``n`` samples and a resolved
    ``fmin`` (tuning applied): the reference's checks in its order, the early downsampling, and every octave's
    geometry (signal length, hop, n_fft, frames, whether the signal is halved after it)."""
    if fmin >= sr / 2:
        raise ParameterError(f"fmin={fmin} must be less than sr/2={sr/2}")
    auto_n_bins = n_bins is None
    if auto_n_bins:
        n_bins = int(np.ceil(bins_per_octave * (np.log2(sr) - np.log2(fmin))))
    freqs = _interval_frequencies(n_bins, fmin, intervals, bins_per_octave)
    if auto_n_bins:
        freqs = _clip_freqs(freqs, window, filter_scale, gamma, sr)
        n_bins = len(freqs)
    if n_bins == 1:
        r = 2 ** (1 / bins_per_octave)
        alpha = np.atleast_1d((r ** 2 - 1) / (r ** 2 + 1))
    else:
        alpha = filters._relative_bandwidth(freqs=freqs)
    lengths, filter_cutoff = filters.wavelet_lengths(freqs=freqs, sr=sr, window=window, filter_scale=filter_scale,
                                                     gamma=gamma, alpha=alpha)
    nyquist = sr / 2.0
    if filter_cutoff > nyquist:
        raise ParameterError(f"Wavelet basis with max frequency={np.max(freqs[-bins_per_octave:])} would exceed the "
                             f"Nyquist frequency={nyquist}. Try reducing the number of frequency bins.")
    n_octaves = int(np.ceil(float(n_bins) / bins_per_octave))
    n_filters = min(bins_per_octave, n_bins)
    # early downsampling (constantq.py:1226-1266)
    count = min(max(0, int(np.ceil(np.log2(nyquist / filter_cutoff)) - 1) - 1),
                max(0, _two_factors(hop_length) - n_octaves + 1))
    early, early_scale = 1, 1.0
    if count > 0:
        early = 2 ** count
        hop_length //= early
        if n < early:
            raise ParameterError(f"Input signal length={n:d} is too short for {n_octaves:d}-octave CQT")
        if res_type != "polyphase":
            _refuse_resampler(res_type)
        early_scale = float(np.sqrt(early)) * (1.0 if scale else float(np.sqrt(early)))
        sr = sr / float(early)
        n = -(-n // early)
        lengths, _ = filters.wavelet_lengths(freqs=freqs, sr=sr, window=window, filter_scale=filter_scale,
                                             gamma=gamma, alpha=alpha)
    octaves = []
    my_sr, my_hop, my_n = sr, hop_length, n
    for i in range(n_octaves):
        sl = slice(-n_filters, None) if i == 0 else slice(-n_filters * (i + 1), -n_filters * i)
        lens, _ = filters.wavelet_lengths(freqs=freqs[sl], sr=my_sr, window=window, filter_scale=filter_scale,
                                          gamma=gamma, alpha=alpha[sl])
        n_fft = int(2.0 ** (np.ceil(np.log2(max(lens)))))
        resample_after = False
        if i < n_octaves - 1:
            resample_after = my_hop % 2 == 0 and freqs[sl.start - 1] <= my_sr / 5
        if resample_after and res_type != "polyphase":
            _refuse_resampler(res_type)
        octaves.append(Octave(my_sr, my_n, my_hop, n_fft, 1 + my_n // my_hop, sl, resample_after))
        if resample_after:
            my_hop //= 2
            my_sr /= 2.0
            my_n = -(-my_n // 2)
    return Plan(freqs, alpha, lengths, n_bins, early, early_scale, sr, tuple(octaves),
                min(o.n_frames for o in octaves))


def _refuse_resampler(res_type):
    raise nat.UnsupportedOnGPU(f"cqt/vqt(res_type={res_type!r}): this call resamples, and only the 'polyphase' "
                               "resampler runs on the GPU; pass res_type='polyphase'")


def octave_rows(p: Plan):
    """Where each octave's rows land (__trim_stack, constantq.py:1169-1194): (output row0, rows kept, first kept
    row of the octave's basis) per octave, in octave order."""
    out, end = [], p.n_bins
    for o in p.octaves:
        n_oct = len(p.freqs[o.rows])
        keep = min(end, n_oct)
        out.append((end - keep, keep, n_oct - keep))
        end -= n_oct
    return out


def bases(p: Plan, *, filter_scale, norm, sparsity, window, gamma):
    """Every octave's Basis, in octave order."""
    return [filter_basis(o.sr, p.freqs[o.rows], p.alpha[o.rows], filter_scale, norm, sparsity, window, gamma,
                         np.sqrt(p.sr / o.sr)) for o in p.octaves]


def _table(ctx, key, arr) -> int:
    """Device copy of a host table, cached by the context under ``key`` (its bytes as 4-byte words)."""
    arr = np.ascontiguousarray(arr)
    return ctx.constant(key, lambda: arr.reshape(-1).view(np.float32))


def _resample_half(ctx, d_x, n_clips: int, n: int, down: int, out_scale: float, d_out):
    """librosa.resample(y, orig_sr=down, target_sr=1, res_type="polyphase") on the device: ceil(n / down) samples."""
    h, n_pre_remove = _poly_filter(1, down)
    d_h = _table(ctx, ("resample_poly", 1, down), h)
    n_out = -(-n // down)
    nat.check(nat.lib().b2l_resample_poly(ctx.handle, _vp(d_x), n_clips, n, n, _vp(d_h), len(h), 1, down, n_pre_remove,
                                          n_out, n_out, out_scale, _vp(d_out)))


def vqt(y, *, sr: float = 22050, hop_length: int = 512, fmin: Optional[float] = None, n_bins: Optional[int] = 84,
        intervals="equal", gamma: Optional[float] = None, bins_per_octave: int = 12, tuning: Optional[float] = 0.0,
        filter_scale: float = 1, norm: Optional[float] = 1, sparsity: float = 0.01, window="hann",
        scale: bool = True, pad_mode="constant", res_type: str = "soxr_hq", dtype=None):
    """Variable-Q transform; same contract as ``librosa.vqt`` (core/constantq.py:820-1120).

    Returns ``(..., n_bins, T)`` complex64 (complex128 for float64 audio, computed in float32); the memory is
    ``[..., frame, bin]``, the reference's ``order="F"``.  A DeviceArray in gives a DeviceArray out.  Resampling
    runs only with ``res_type="polyphase"``; a call that needs no resampling accepts any ``res_type``."""
    if not isinstance(intervals, str):
        bins_per_octave = len(intervals)
    if fmin is None:
        fmin = _default_fmin()
    n, req = pl.precheck_signal(y)
    on_device = isinstance(y, nat.DeviceArray)
    out_dtype = np.dtype(dtype) if dtype is not None else dtype_r2c(req)
    if on_device and out_dtype != np.complex64:
        raise nat.UnsupportedOnGPU(f"cqt/vqt dtype={out_dtype}: device results are complex64")
    staged = pl.StagedInput(y)
    try:
        if tuning is None:
            from .pitch import estimate_tuning

            tuning = estimate_tuning(y=staged.dev, sr=sr, bins_per_octave=bins_per_octave)
        fmin = fmin * 2.0 ** (tuning / bins_per_octave)
        p = plan(n, sr=sr, hop_length=hop_length, fmin=fmin, n_bins=n_bins, intervals=intervals, gamma=gamma,
                 bins_per_octave=bins_per_octave, filter_scale=filter_scale, window=window, scale=scale,
                 res_type=res_type)
        # stft's "n_fft=... is too large" warning, once per octave: held back until the finite verdict, because the
        # reference's stft raises on non-finite audio before it warns
        with warnings.catch_warnings(record=True) as held:
            warnings.simplefilter("always")
            for o in p.octaves:
                pl.check_stft_geometry(o.n, o.n_fft, True, pad_mode)
                pl.require_supported_n_fft(o.n_fft)
        if len(p.octaves) > nat.CQT_MAX_OCTAVES:
            raise nat.UnsupportedOnGPU(f"cqt/vqt: {len(p.octaves)} octaves; the GPU projection takes at most "
                                       f"{nat.CQT_MAX_OCTAVES}")
        out = _run(staged, p, filter_scale=filter_scale, norm=norm, sparsity=sparsity, window=window, gamma=gamma,
                   scale=scale, pad_mode=pad_mode)
    finally:
        staged.release()
    res = staged.result(out, out_dtype)
    for w in held:
        warnings.warn(w.message, w.category, stacklevel=2)
    return res


def _run(staged, p: Plan, *, filter_scale, norm, sparsity, window, gamma, scale, pad_mode):
    """Enqueue the octave pyramid and the projection for a staged signal; returns the (..., n_bins, T) "ft" result."""
    ctx, m = staged.ctx, staged.n_clips
    key, bs = _bases_cached(p, filter_scale=filter_scale, norm=norm, sparsity=sparsity, window=window, gamma=gamma)
    rows = octave_rows(p)
    indptr, nnz_off, ip_off, descs = [], 0, 0, []
    for b, (row0, keep, first) in zip(bs, rows):
        indptr.append(b.indptr + nnz_off)
        descs.append((row0, keep, ip_off + first, int(b.indptr[first + keep] - b.indptr[first])))
        ip_off += len(b.indptr)
        nnz_off += len(b.data)
    d_indptr = _table(ctx, ("cqt_indptr",) + key, np.concatenate(indptr).astype(np.int32))
    d_indices = _table(ctx, ("cqt_indices",) + key, np.concatenate([b.indices for b in bs]).astype(np.int32))
    d_data = _table(ctx, ("cqt_data",) + key, np.concatenate([b.data for b in bs]).astype(np.complex64))
    d_rscale = _table(ctx, ("cqt_rscale", p.lengths.tobytes()), 1.0 / np.sqrt(p.lengths)) if scale else 0
    with pl.Scope(staged.dev) as sc:
        staged.scan_all()
        cur, n_cur = staged.dev.ptr, staged.n
        if p.early > 1:
            d = sc.empty((m, -(-n_cur // p.early)), np.float32)
            _resample_half(ctx, cur, m, n_cur, p.early, p.early_scale, d.ptr)
            cur, n_cur = d.ptr, d.shape[-1]
        octs = (nat.CqtOctave * len(p.octaves))()
        for i, (o, b) in enumerate(zip(p.octaves, bs)):
            assert n_cur == o.n
            F = o.n_fft // 2 + 1
            D = sc.empty((m, o.n_frames, F), np.complex64)
            plan_ = nat.make_plan(ctx, ("stft", o.n_fft, o.hop, True, pad_mode, "ones"), n_fft=o.n_fft,
                                  hop_length=o.hop, center=True, pad_mode=pad_mode, window=np.ones(o.n_fft))
            nat.check(nat.lib().b2l_stft(ctx.handle, plan_.handle, _vp(cur), m, n_cur, n_cur, _vp(D.ptr)))
            row0, keep, ip, nnz = descs[i]
            octs[i] = nat.CqtOctave(D.ptr, o.n_frames, F, row0, keep, ip, nnz)
            if o.resample_after:
                d = sc.empty((m, -(-n_cur // 2)), np.float32)
                _resample_half(ctx, cur, m, n_cur, 2, float(np.sqrt(2.0)), d.ptr)
                cur, n_cur = d.ptr, d.shape[-1]
        out = sc.empty(tuple(staged.lead) + (p.n_bins, p.n_frames), np.complex64, layout="ft")
        nat.check(nat.lib().b2l_cqt_project(ctx.handle, octs, len(p.octaves), _vp(d_indptr), _vp(d_indices),
                                            _vp(d_data), _vp(d_rscale) if scale else None, m, p.n_frames, p.n_bins,
                                            _vp(out.ptr)))
        return sc.keep(out)


_BASES = {}


def _bases_cached(p: Plan, *, filter_scale, norm, sparsity, window, gamma):
    """(key, bases()) memoised per configuration, as the reference caches __vqt_filter_fft.  The key holds everything
    a basis depends on: the frequencies and bandwidths, the rate after early downsampling, and every octave's rows,
    rate and n_fft (which follow from the hop: the signal is halved only while the hop stays even)."""
    key = (p.freqs.tobytes(), p.alpha.tobytes(), p.sr,
           tuple((o.rows.start, o.rows.stop, o.sr, o.n_fft) for o in p.octaves),
           str(filter_scale), str(norm), str(sparsity), repr(window), str(gamma))
    got = _BASES.get(key)
    if got is None:
        if len(_BASES) >= 32:
            _BASES.clear()
        got = _BASES[key] = bases(p, filter_scale=filter_scale, norm=norm, sparsity=sparsity, window=window,
                                  gamma=gamma)
    return key, got


def cqt(y, *, sr: float = 22050, hop_length: int = 512, fmin: Optional[float] = None, n_bins: Optional[int] = 84,
        bins_per_octave: int = 12, tuning: Optional[float] = 0.0, filter_scale: float = 1, norm: Optional[float] = 1,
        sparsity: float = 0.01, window="hann", scale: bool = True, pad_mode="constant", res_type: str = "soxr_hq",
        dtype=None):
    """Constant-Q transform; same contract as ``librosa.cqt`` (core/constantq.py:620-817): ``vqt`` with gamma=0."""
    return vqt(y, sr=sr, hop_length=hop_length, fmin=fmin, n_bins=n_bins, intervals="equal", gamma=0,
               bins_per_octave=bins_per_octave, tuning=tuning, filter_scale=filter_scale, norm=norm,
               sparsity=sparsity, window=window, scale=scale, pad_mode=pad_mode, res_type=res_type, dtype=dtype)
