"""``cqt`` / ``vqt`` / ``pseudo_cqt`` / ``hybrid_cqt`` with librosa's signatures, executed by libb2l.so on an H100
(reference: librosa/core/constantq.py:209-590, 620-1266).

The octave pyramid runs on the device with one staging of the input and no host round trip: an optional early
downsample by 2^k (polyphase resampler), then per octave, from the top down, a centred STFT with a rectangular
window into frame-major scratch and a halving of the signal for the next octave.  One launch of
``b2l_cqt_project`` then applies every octave's sparse complex filter basis and writes the stacked result.  The
filter bases, frequencies and lengths are host constants built with the reference's float64 expressions.

``pseudo_cqt`` is one centred Hann STFT at a single n_fft whose magnitudes meet the magnitudes of one filter basis;
``hybrid_cqt`` stacks such a pseudo part (the high bins, whose filters fit in two hops) on top of ``np.abs`` of a
``cqt`` of the remaining low bins.  Both run as the same staged pass: the pseudo part's STFT, the full part's
pyramid, and one launch of ``b2l_cqt_project_abs`` writing every row as float32 magnitudes (DESIGN §4.19).
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
from ..util.utils import dtype_c2r, dtype_r2c
from .audio import _poly_filter

__all__ = ["cqt", "vqt", "pseudo_cqt", "hybrid_cqt", "cqt_frequencies"]

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


def _et_relative_bw(bins_per_octave: int) -> np.ndarray:
    """The relative bandwidth of one bin of an equal-tempered scale (librosa/core/constantq.py:1577-1598)."""
    r = 2 ** (1 / bins_per_octave)
    return np.atleast_1d((r ** 2 - 1) / (r ** 2 + 1))


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


def _pseudo_n_fft(lengths, hop_length: int) -> int:
    """pseudo_cqt's transform size: the longest filter's power of two, at least two hops (constantq.py:1144-1145)."""
    return max(int(2.0 ** (np.ceil(np.log2(np.max(lengths))))), int(2.0 ** (1 + np.ceil(np.log2(hop_length)))))


def filter_basis(sr, freqs, alpha, filter_scale, norm, sparsity, window, gamma, rescale, hop_length=None) -> Basis:
    """The FFT of one octave's wavelets at rate ``sr``, rescaled by ``lengths / n_fft``, non-negative bins only,
    sparsified and multiplied by ``rescale`` (sqrt of the top rate over this octave's rate) (librosa/core/constantq.py:1067-1080, 1123-1166).

    With ``hop_length`` (pseudo_cqt): n_fft covers at least two hops, and the table holds ``np.abs`` of the sparse
    basis (float32 magnitudes in the real parts)."""
    basis, lengths = filters.wavelet(freqs=freqs, sr=sr, filter_scale=filter_scale, norm=norm, pad_fft=True,
                                     window=window, gamma=gamma, alpha=alpha)
    n_fft = basis.shape[1] if hop_length is None else _pseudo_n_fft(lengths, hop_length)
    basis *= lengths[:, np.newaxis] / float(n_fft)
    fft_basis = scipy.fft.fft(basis, n=n_fft, axis=1)[:, : (n_fft // 2) + 1]
    dense = _sparsify(fft_basis, sparsity, np.complex64)
    rows, cols = np.nonzero(dense)
    data = dense[rows, cols]
    data = (np.abs(data) if hop_length is not None else data * np.float64(rescale)).astype(np.complex64)
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
    alpha = _et_relative_bw(bins_per_octave) if n_bins == 1 else filters._relative_bandwidth(freqs=freqs)
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


class PseudoPlan(NamedTuple):
    sr: float
    freqs: np.ndarray
    alpha: np.ndarray
    lengths: np.ndarray
    n_bins: int
    n_fft: int
    hop: int
    n_frames: int


def _equal_bins(*, sr, fmin, n_bins, bins_per_octave, filter_scale, window):
    """pseudo_cqt's and hybrid_cqt's (freqs, alpha, lengths) for a resolved ``fmin``, with the reference's checks in
    its order (librosa/core/constantq.py:318-358, 519-555)."""
    if fmin >= sr / 2:
        raise ParameterError(f"fmin={fmin} must be less than sr/2={sr/2}")
    auto_n_bins = n_bins is None
    if auto_n_bins:
        n_bins = int(np.ceil(bins_per_octave * (np.log2(sr) - np.log2(fmin))))
    freqs = cqt_frequencies(n_bins, fmin=fmin, bins_per_octave=bins_per_octave)
    if auto_n_bins:
        freqs = _clip_freqs(freqs, window, filter_scale, 0, sr)
        n_bins = len(freqs)
    alpha = _et_relative_bw(bins_per_octave) if n_bins == 1 else filters._relative_bandwidth(freqs=freqs)
    lengths, filter_cutoff = filters.wavelet_lengths(freqs=freqs, sr=sr, window=window, filter_scale=filter_scale,
                                                     alpha=alpha)
    if filter_cutoff > sr / 2:
        raise ParameterError(f"Filter cutoff frequency {filter_cutoff} exceeds Nyquist frequency {sr/2}. "
                             "Try reducing the number of frequency bins.")
    return freqs, alpha, lengths


def pseudo_plan(n: int, *, sr, hop_length, fmin, n_bins, bins_per_octave, filter_scale, window) -> PseudoPlan:
    """The host half of pseudo_cqt (librosa/core/constantq.py:519-590) for a signal of ``n`` samples and a resolved
    ``fmin``: its checks, its bins and its single n_fft."""
    freqs, alpha, lengths = _equal_bins(sr=sr, fmin=fmin, n_bins=n_bins, bins_per_octave=bins_per_octave,
                                        filter_scale=filter_scale, window=window)
    return PseudoPlan(sr, freqs, alpha, lengths, len(freqs), _pseudo_n_fft(lengths, hop_length), hop_length,
                      1 + n // hop_length)


def hybrid_split(lengths, hop_length: int) -> np.ndarray:
    """hybrid_cqt's pseudo bins: those whose filter, padded to a power of two, is shorter than two hops
    (librosa/core/constantq.py:360-366)."""
    return 2.0 ** np.ceil(np.log2(lengths)) < 2 * hop_length


def _check_pseudo_stft(pp: PseudoPlan, n: int, pad_mode):
    """The pseudo part's stft checks (its "n_fft=... is too large" warning) and the GPU's limit on its n_fft."""
    pl.check_stft_geometry(n, pp.n_fft, True, pad_mode)
    if pp.n_fft > pl.MAX_N_FFT:
        raise nat.UnsupportedOnGPU(f"pseudo_cqt: n_fft={pp.n_fft} (the longest filter of fmin={pp.freqs[0]:.2f} Hz, "
                                   f"or two hops); the float32 STFT kernels stop at n_fft={pl.MAX_N_FFT}: raise fmin "
                                   "or lower the hop")
    pl.require_supported_n_fft(pp.n_fft)


def _check_full_stft(p: Plan, pad_mode):
    for o in p.octaves:
        pl.check_stft_geometry(o.n, o.n_fft, True, pad_mode)
        pl.require_supported_n_fft(o.n_fft)


def _staged(y, *, what, real, sr, bins_per_octave, tuning, dtype, prepare, **kw):
    """What every constant-Q entry point does around the device pass: the signal's checks, ``tuning``
    (estimate_tuning on the staged signal when None), ``prepare(n, tuning) -> (full Plan or None, PseudoPlan or
    None)`` with the reference's checks, then ``_run``; with a given tuning nothing touches the device before
    ``prepare`` has passed.  The stft's "n_fft=... is too large" warnings are held back until the finite
    verdict, because the reference's stft raises on non-finite audio before it warns.  ``real``: float32
    magnitudes (the reference's real dtype of ``dtype``), else complex64."""
    n, req = pl.precheck_signal(y, stacklevel=5)
    on_device = isinstance(y, nat.DeviceArray)
    out_dtype = np.dtype(dtype) if dtype is not None else dtype_r2c(req)
    if real:
        out_dtype = np.dtype(dtype_c2r(out_dtype))
    dev_dtype = np.dtype(np.float32 if real else np.complex64)
    if on_device and out_dtype != dev_dtype:
        raise nat.UnsupportedOnGPU(f"{what} dtype={out_dtype}: device results are {dev_dtype}")
    staged = None
    try:
        if tuning is None:
            from .pitch import estimate_tuning

            staged = pl.StagedInput(y)
            tuning = estimate_tuning(y=staged.dev, sr=sr, bins_per_octave=bins_per_octave)
        with warnings.catch_warnings(record=True) as held:
            warnings.simplefilter("always")
            full, pseudo = prepare(n, tuning)
        n_oct = (len(full.octaves) if full else 0) + (1 if pseudo else 0)
        if n_oct > nat.CQT_MAX_OCTAVES:
            raise nat.UnsupportedOnGPU(f"{what}: {n_oct} octaves; the GPU projection takes at most "
                                       f"{nat.CQT_MAX_OCTAVES}")
        if staged is None:
            staged = pl.StagedInput(y)
        out = _run(staged, full, pseudo, mag=real, **kw)
    finally:
        if staged is not None:
            staged.release()
    res = staged.result(out, out_dtype)
    for w in held:
        warnings.warn(w.message, w.category, stacklevel=3)
    return res


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

    def prepare(n, tuning):
        p = plan(n, sr=sr, hop_length=hop_length, fmin=fmin * 2.0 ** (tuning / bins_per_octave), n_bins=n_bins,
                 intervals=intervals, gamma=gamma, bins_per_octave=bins_per_octave, filter_scale=filter_scale,
                 window=window, scale=scale, res_type=res_type)
        _check_full_stft(p, pad_mode)
        return p, None

    return _staged(y, what="cqt/vqt", real=False, sr=sr, bins_per_octave=bins_per_octave, tuning=tuning, dtype=dtype,
                   prepare=prepare, filter_scale=filter_scale, norm=norm, sparsity=sparsity, window=window,
                   gamma=gamma, scale=scale, pad_mode=pad_mode)


def _run(staged, full: Optional[Plan], pseudo: Optional[PseudoPlan], *, mag, filter_scale, norm, sparsity, window,
         gamma, scale, pad_mode):
    """Enqueue one pass for a staged signal: the pseudo part's centred Hann STFT, the full part's octave pyramid,
    then one projection launch writing every row; the pseudo part's rows are the top (highest) bins, after the
    full part's.  Returns the (..., n_bins, T) "ft"
    result: complex64 (b2l_cqt_project), or float32 magnitudes with ``mag`` (b2l_cqt_project_abs)."""
    ctx, m = staged.ctx, staged.n_clips
    n_low = full.n_bins if full is not None else 0
    parts, keys, rscale = [], [], []   # parts: (basis, output row0, rows kept, first kept row, kind)
    if pseudo is not None:
        key, b = _pseudo_basis_cached(pseudo, filter_scale=filter_scale, norm=norm, sparsity=sparsity, window=window)
        keys.append(key)
        parts.append((b, n_low, pseudo.n_bins, 0, nat.CQT_PSEUDO | (nat.CQT_DIVIDE if scale else 0)))
        # pseudo_cqt's C /= np.sqrt(n_fft) or C *= np.sqrt(lengths / n_fft), each in float64 with one rounding
        rscale.append(np.full(pseudo.n_bins, np.sqrt(pseudo.n_fft)) if scale else np.sqrt(pseudo.lengths / pseudo.n_fft))
    if full is not None:
        key, bs = _bases_cached(full, filter_scale=filter_scale, norm=norm, sparsity=sparsity, window=window,
                                gamma=gamma)
        keys.append(key)
        parts += [(b, row0, keep, first, nat.CQT_FULL) for b, (row0, keep, first) in zip(bs, octave_rows(full))]
        rscale.insert(0, 1.0 / np.sqrt(full.lengths) if scale else np.ones(full.n_bins))
    n_bins = n_low + (pseudo.n_bins if pseudo is not None else 0)
    T = min(x.n_frames for x in (full, pseudo) if x is not None)
    indptr, nnz_off, ip_off, descs = [], 0, 0, []
    for b, row0, keep, first, kind in parts:
        indptr.append(b.indptr + nnz_off)
        descs.append((row0, keep, ip_off + first, int(b.indptr[first + keep] - b.indptr[first]), kind))
        ip_off += len(b.indptr)
        nnz_off += len(b.data)
    key = tuple(keys)
    d_indptr = _table(ctx, ("cqt_indptr",) + key, np.concatenate(indptr).astype(np.int32))
    d_indices = _table(ctx, ("cqt_indices",) + key, np.concatenate([p[0].indices for p in parts]).astype(np.int32))
    d_data = _table(ctx, ("cqt_data",) + key, np.concatenate([p[0].data for p in parts]).astype(np.complex64))
    rs = np.concatenate(rscale)
    scaled = scale or pseudo is not None   # unscaled full rows multiply by 1.0: exact
    d_rscale = _table(ctx, ("cqt_rscale", rs.tobytes()), rs) if scaled else 0
    octs = (nat.CqtOctave * len(parts))()
    with pl.Scope(staged.dev) as sc:
        staged.scan_all()
        i = 0
        if pseudo is not None:
            F = pseudo.n_fft // 2 + 1
            D = sc.empty((m, pseudo.n_frames, F), np.complex64)
            win, wkey = pl.resolve_window("hann", pseudo.n_fft, pseudo.n_fft)
            plan_ = nat.make_plan(ctx, ("stft", pseudo.n_fft, pseudo.hop, True, pad_mode, wkey), n_fft=pseudo.n_fft,
                                  hop_length=pseudo.hop, center=True, pad_mode=pad_mode, window=win)
            nat.check(nat.lib().b2l_stft(ctx.handle, plan_.handle, _vp(staged.dev.ptr), m, staged.n, staged.n,
                                         _vp(D.ptr)))
            row0, keep, ip, nnz, kind = descs[0]
            octs[0] = nat.CqtOctave(D.ptr, pseudo.n_frames, F, row0, keep, ip, nnz, kind)
            i = 1
        if full is not None:
            cur, n_cur = staged.dev.ptr, staged.n
            if full.early > 1:
                d = sc.empty((m, -(-n_cur // full.early)), np.float32)
                _resample_half(ctx, cur, m, n_cur, full.early, full.early_scale, d.ptr)
                cur, n_cur = d.ptr, d.shape[-1]
            for o in full.octaves:
                assert n_cur == o.n
                F = o.n_fft // 2 + 1
                D = sc.empty((m, o.n_frames, F), np.complex64)
                plan_ = nat.make_plan(ctx, ("stft", o.n_fft, o.hop, True, pad_mode, "ones"), n_fft=o.n_fft,
                                      hop_length=o.hop, center=True, pad_mode=pad_mode, window=np.ones(o.n_fft))
                nat.check(nat.lib().b2l_stft(ctx.handle, plan_.handle, _vp(cur), m, n_cur, n_cur, _vp(D.ptr)))
                row0, keep, ip, nnz, kind = descs[i]
                octs[i] = nat.CqtOctave(D.ptr, o.n_frames, F, row0, keep, ip, nnz, kind)
                i += 1
                if o.resample_after:
                    d = sc.empty((m, -(-n_cur // 2)), np.float32)
                    _resample_half(ctx, cur, m, n_cur, 2, float(np.sqrt(2.0)), d.ptr)
                    cur, n_cur = d.ptr, d.shape[-1]
        out = sc.empty(tuple(staged.lead) + (n_bins, T), np.float32 if mag else np.complex64, layout="ft")
        project = nat.lib().b2l_cqt_project_abs if mag else nat.lib().b2l_cqt_project
        nat.check(project(ctx.handle, octs, len(parts), _vp(d_indptr), _vp(d_indices), _vp(d_data),
                          _vp(d_rscale) if scaled else None, m, T, n_bins, _vp(out.ptr)))
        return sc.keep(out)


_BASES = {}


def _cached(key, build):
    """(key, build()) memoised per configuration, as the reference caches __vqt_filter_fft."""
    got = _BASES.get(key)
    if got is None:
        if len(_BASES) >= 32:
            _BASES.clear()
        got = _BASES[key] = build()
    return key, got


def pseudo_basis(pp: PseudoPlan, *, filter_scale, norm, sparsity, window) -> Basis:
    """pseudo_cqt's |basis| (librosa/core/constantq.py:557-571)."""
    return filter_basis(pp.sr, pp.freqs, pp.alpha, filter_scale, norm, sparsity, window, 0, 1.0, hop_length=pp.hop)


def _pseudo_basis_cached(pp: PseudoPlan, *, filter_scale, norm, sparsity, window):
    key = ("pseudo", pp.freqs.tobytes(), pp.alpha.tobytes(), pp.sr, pp.n_fft, str(filter_scale), str(norm),
           str(sparsity), repr(window))
    return _cached(key, lambda: pseudo_basis(pp, filter_scale=filter_scale, norm=norm, sparsity=sparsity,
                                             window=window))


def _bases_cached(p: Plan, *, filter_scale, norm, sparsity, window, gamma):
    """(key, bases()) memoised per configuration.  The key holds everything a basis depends on: the frequencies and
    bandwidths, the rate after early downsampling, and every octave's rows, rate and n_fft (which follow from the
    hop: the signal is halved only while the hop stays even)."""
    key = (p.freqs.tobytes(), p.alpha.tobytes(), p.sr,
           tuple((o.rows.start, o.rows.stop, o.sr, o.n_fft) for o in p.octaves),
           str(filter_scale), str(norm), str(sparsity), repr(window), str(gamma))
    return _cached(key, lambda: bases(p, filter_scale=filter_scale, norm=norm, sparsity=sparsity, window=window,
                                      gamma=gamma))


def cqt(y, *, sr: float = 22050, hop_length: int = 512, fmin: Optional[float] = None, n_bins: Optional[int] = 84,
        bins_per_octave: int = 12, tuning: Optional[float] = 0.0, filter_scale: float = 1, norm: Optional[float] = 1,
        sparsity: float = 0.01, window="hann", scale: bool = True, pad_mode="constant", res_type: str = "soxr_hq",
        dtype=None):
    """Constant-Q transform; same contract as ``librosa.cqt`` (core/constantq.py:620-817): ``vqt`` with gamma=0."""
    return vqt(y, sr=sr, hop_length=hop_length, fmin=fmin, n_bins=n_bins, intervals="equal", gamma=0,
               bins_per_octave=bins_per_octave, tuning=tuning, filter_scale=filter_scale, norm=norm,
               sparsity=sparsity, window=window, scale=scale, pad_mode=pad_mode, res_type=res_type, dtype=dtype)


def pseudo_cqt(y, *, sr: float = 22050, hop_length: int = 512, fmin: Optional[float] = None,
               n_bins: Optional[int] = 84, bins_per_octave: int = 12, tuning: Optional[float] = 0.0,
               filter_scale: float = 1, norm: Optional[float] = 1, sparsity: float = 0.01, window="hann",
               scale: bool = True, pad_mode="constant", dtype=None):
    """Pseudo constant-Q transform; same contract as ``librosa.pseudo_cqt`` (core/constantq.py:430-590).

    One centred Hann STFT at n_fft = the longest filter's power of two, at least two hops, and the magnitude of one
    filter basis applied to its magnitude.  Returns ``(..., n_bins, T)`` float32 (float64 for float64 audio or
    ``dtype=complex128``, computed in float32), C-ordered like the reference's.  A DeviceArray in gives a float32
    DeviceArray out whose memory is ``[..., frame, bin]`` (layout "ft").

    n_fft above 8192 is refused (UnsupportedOnGPU): the float32 STFT kernels stop there.  That includes the
    defaults (fmin C1, 84 bins), whose longest filter needs n_fft=16384; from about fmin=65.4 Hz (C2) up, with
    hops up to 4096, the transform runs."""
    if fmin is None:
        fmin = _default_fmin()

    def prepare(n, tuning):
        pp = pseudo_plan(n, sr=sr, hop_length=hop_length, fmin=fmin * 2.0 ** (tuning / bins_per_octave),
                         n_bins=n_bins, bins_per_octave=bins_per_octave, filter_scale=filter_scale, window=window)
        _check_pseudo_stft(pp, n, pad_mode)
        return None, pp

    res = _staged(y, what="pseudo_cqt", real=True, sr=sr, bins_per_octave=bins_per_octave, tuning=tuning,
                  dtype=dtype, prepare=prepare, filter_scale=filter_scale, norm=norm, sparsity=sparsity,
                  window=window, gamma=0, scale=scale, pad_mode=pad_mode)
    return res if isinstance(res, nat.DeviceArray) else np.ascontiguousarray(res)


def hybrid_cqt(y, *, sr: float = 22050, hop_length: int = 512, fmin: Optional[float] = None,
               n_bins: Optional[int] = 84, bins_per_octave: int = 12, tuning: Optional[float] = 0.0,
               filter_scale: float = 1, norm: Optional[float] = 1, sparsity: float = 0.01, window="hann",
               scale: bool = True, pad_mode="constant", res_type: str = "soxr_hq", dtype=None):
    """Hybrid constant-Q transform; same contract as ``librosa.hybrid_cqt`` (core/constantq.py:208-428).

    The bins whose filters, padded to a power of two, are shorter than two hops take ``pseudo_cqt`` (the highest rows),
    the others ``np.abs(cqt(...))``, trimmed to the shorter frame count.  Returns ``(..., n_bins, T)`` float32
    (float64 for float64 audio, computed in float32) with memory ``[..., frame, bin]``, the reference's
    ``order="F"``; a DeviceArray in gives a float32 DeviceArray out (layout "ft").

    Refused (UnsupportedOnGPU): a pseudo part whose n_fft exceeds 8192 (a hop above 4096), and whatever ``cqt``
    refuses for the full part: a resampler other than ``res_type="polyphase"`` where the pyramid resamples, an
    octave n_fft above 8192 (an odd hop stops the halving early)."""
    if fmin is None:
        fmin = _default_fmin()

    def prepare(n, tuning):
        fmin_t = fmin * 2.0 ** (tuning / bins_per_octave)
        freqs, _, lengths = _equal_bins(sr=sr, fmin=fmin_t, n_bins=n_bins, bins_per_octave=bins_per_octave,
                                        filter_scale=filter_scale, window=window)
        is_pseudo = hybrid_split(lengths, hop_length)
        n_pseudo = int(np.sum(is_pseudo))
        n_full = len(freqs) - n_pseudo
        full = pseudo = None
        if n_pseudo > 0:
            pseudo = pseudo_plan(n, sr=sr, hop_length=hop_length, fmin=np.min(freqs[is_pseudo]), n_bins=n_pseudo,
                                 bins_per_octave=bins_per_octave, filter_scale=filter_scale, window=window)
            _check_pseudo_stft(pseudo, n, pad_mode)
        if n_full > 0:
            full = plan(n, sr=sr, hop_length=hop_length, fmin=fmin_t, n_bins=n_full, intervals="equal", gamma=0,
                        bins_per_octave=bins_per_octave, filter_scale=filter_scale, window=window, scale=scale,
                        res_type=res_type)
            _check_full_stft(full, pad_mode)
        return full, pseudo

    return _staged(y, what="hybrid_cqt", real=True, sr=sr, bins_per_octave=bins_per_octave, tuning=tuning,
                   dtype=dtype, prepare=prepare, filter_scale=filter_scale, norm=norm, sparsity=sparsity,
                   window=window, gamma=0, scale=scale, pad_mode=pad_mode)
