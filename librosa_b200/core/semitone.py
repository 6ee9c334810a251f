"""``iirt`` with librosa's signature, executed by libb2l.so on an H100 (reference: librosa/core/spectrum.py:1522-1713).

The semitone filter bank runs on the device with one staging of the input and no host round trip: the centre
padding (``b2l_pad_center``), one polyphase resample per band rate that differs from ``sr``, then per group of
clips one launch of ``b2l_iirt_filter`` (``scipy.signal.sosfiltfilt`` of every (clip, band) chain in float64, bit
for bit) and one of ``b2l_iirt_stmsp`` (the short-time mean-square power, summed in NumPy's pairwise order).  The
filters, their initial states and padding lengths, and each rate's window, factor and frame starts are host
tables built with the reference's own SciPy and NumPy calls.
"""
from __future__ import annotations

import ctypes as C
import math
from typing import NamedTuple, Tuple

import numpy as np
import scipy.signal

from .. import _native as nat
from .. import _pipeline as pl
from .. import filters
from ..util.exceptions import ParameterError
from .audio import _poly_filter

__all__ = ["iirt"]

_vp = C.c_void_p
_NP_PAD_ONLY = ("maximum", "mean", "median", "minimum", "wrap")   # np.pad modes without a device index map
_LEAF = 128                                                        # NumPy's PW_BLOCKSIZE


def padlen(sos: np.ndarray) -> int:
    """sosfiltfilt's default padding: 3 * (2 n_sections + 1 - min(#b2 == 0, #a2 == 0))."""
    ntaps = 2 * len(sos) + 1 - min(int((sos[:, 2] == 0).sum()), int((sos[:, 5] == 0).sum()))
    return 3 * ntaps


class Bank(NamedTuple):
    """The designed filter bank as the kernels read it."""
    sos: Tuple[np.ndarray, ...]   # per band, float64 [sections][6]
    sample_rates: np.ndarray      # per band
    rates: np.ndarray             # np.unique(sample_rates): the order the reference resamples in
    rate_of: np.ndarray           # per band: index into ``rates``
    coef: np.ndarray              # [bands][IIRT_MAX_SECTIONS][8] float64: b0 b1 b2 a1 a2, sosfilt_zi, 0; then 1 0 ... 0
    info: np.ndarray              # [bands][2] int32: sections, padlen
    bands: np.ndarray             # int32: band indices grouped by rate, rates in ``rates`` order
    band_off: Tuple[int, ...]     # where each rate's bands start in ``bands`` (and a final end)
    max_sections: int


def make_bank(sos, sample_rates) -> Bank:
    sos = tuple(np.asarray(s, dtype=np.float64) for s in sos)
    sample_rates = np.asarray(sample_rates)
    rates = np.unique(sample_rates)
    rate_of = np.searchsorted(rates, sample_rates)
    max_sections = max(len(s) for s in sos)
    coef = np.zeros((len(sos), max(max_sections, nat.IIRT_MAX_SECTIONS), 8))
    info = np.zeros((len(sos), 2), dtype=np.int32)
    coef[:, :, 0] = 1.0   # pass-through sections after each band's own: the kernel runs max_sections for all
    for i, s in enumerate(sos):
        coef[i, :len(s), :3] = s[:, :3]
        coef[i, :len(s), 3:5] = s[:, 4:6]
        coef[i, :len(s), 5:7] = scipy.signal.sosfilt_zi(s)
        info[i] = len(s), padlen(s)
    bands = np.concatenate([np.flatnonzero(rate_of == r) for r in range(len(rates))]).astype(np.int32)
    band_off = tuple(int(v) for v in np.concatenate([[0], np.cumsum(np.bincount(rate_of, minlength=len(rates)))]))
    return Bank(sos, sample_rates, rates, rate_of, coef[:, :nat.IIRT_MAX_SECTIONS], info, bands, band_off,
                max_sections)


def _key(v):
    if isinstance(v, np.ndarray):
        return ("ndarray", v.dtype.str, v.shape, v.tobytes())
    return (type(v).__name__, repr(v))


_BANKS = {}


def bank_cached(tuning, kwargs) -> Tuple[tuple, Bank]:
    """(key, Bank) of ``semitone_filterbank(tuning=tuning, flayout="sos", **kwargs)``, memoised per configuration as
    the reference caches ``mr_frequencies``; the key holds the tuning and every keyword argument by value."""
    key = (_key(tuning),) + tuple((k, _key(v)) for k, v in sorted(kwargs.items()))
    got = _BANKS.get(key)
    if got is None:
        sos, srs = filters.semitone_filterbank(tuning=tuning, flayout="sos", **kwargs)
        if len(_BANKS) >= 16:
            _BANKS.clear()
        got = _BANKS[key] = make_bank(sos, srs)
    return key, got


def pairwise_leaves(n: int) -> np.ndarray:
    """NumPy's pairwise summation of ``n`` terms as a leaf program: (offset, length, partial sums combined after
    the leaf, 0) per leaf in order.  Blocks of at most 128 terms are leaves; a longer block splits at
    n/2 - (n/2 mod 8) and its halves' sums are added, left + right."""
    out = []

    def walk(off, m):
        if m <= _LEAF:
            out.append([off, m, 0, 0])
            return
        h = m // 2
        h -= h % 8
        walk(off, h)
        walk(off + h, m - h)
        out[-1][2] += 1

    walk(0, n)
    return np.asarray(out, dtype=np.int32).reshape(-1, 4)


def leaves_depth(leaves: np.ndarray) -> int:
    """Largest number of partial sums a leaf program holds at once."""
    sp = top = 0
    for _, _, comb, _ in leaves:
        sp += 1
        top = max(top, sp)
        sp -= int(comb)
    return top


class Rate(NamedTuple):
    rate: float
    n: int                 # samples of the signal at this rate (= the filtered length)
    up: int                # resampling ratio from sr (up = down = 0: this rate is sr, no resampling)
    down: int
    w: int                 # STMSP window
    factor: float          # sr / rate
    starts: np.ndarray     # [T] int32 frame starts
    leaves: np.ndarray     # pairwise-sum program of w terms
    rows: int              # scratch rows per chain: n + the largest padlen of the rate's bands
    n_bands: int


class Plan(NamedTuple):
    bank_key: tuple
    bank: Bank
    pad: int               # centre padding on each side (0: center=False)
    pad_mode: str
    n_pad: int             # padded signal length
    n_frames: int
    rates: Tuple[Rate, ...]

    def clip_bytes(self) -> int:
        """Float64 scratch of one clip: rows x bands per rate."""
        return sum(8 * r.rows * r.n_bands for r in self.rates)

    def scratch_bytes(self, m: int) -> int:
        """Float64 scratch of ``m`` clips: per rate, rows x (m x bands rounded up to 32) doubles."""
        return sum(8 * r.rows * (-(-m * r.n_bands // 32) * 32) for r in self.rates)


def _refuse_resampler(res_type):
    raise nat.UnsupportedOnGPU(f"iirt(res_type={res_type!r}): this call resamples, and only the 'polyphase' "
                               "resampler runs on the GPU; pass res_type='polyphase'")


def check_pad_mode(pad_mode, n: int, ndim: int, pad: int) -> str:
    """What np.pad accepts and the device index map covers; an empty signal takes only zero padding."""
    if callable(pad_mode):
        raise nat.UnsupportedOnGPU("iirt: a callable pad_mode cannot run on the GPU (no CPU fallback); pass one of "
                                   f"{sorted(m for m in nat.PAD_MODES)}")
    if pad_mode in _NP_PAD_ONLY:
        raise nat.UnsupportedOnGPU(f"iirt(pad_mode={pad_mode!r}): the GPU pads with "
                                   f"{sorted(m for m in nat.PAD_MODES)} only (no CPU fallback)")
    if pad_mode not in nat.PAD_MODES:
        raise ValueError(f"mode '{pad_mode}' is not supported")   # what np.pad raises
    if n == 0 and pad and pad_mode not in ("constant", "empty"):
        raise ValueError(f"can't extend empty axis {ndim - 1} using modes other than 'constant' or 'empty'")
    return pad_mode


def rate_tables(bank: Bank, n_pad: int, *, sr, win_length: int, hop_length: int, n_frames: int) -> Tuple[Rate, ...]:
    """Per rate: the resampled length, the resampling ratio, and the STMSP window, factor and frame starts with the
    reference's float64 expressions and NumPy's own arange / round (librosa/core/spectrum.py:1673-1711)."""
    out = []
    for ri, rate in enumerate(bank.rates):
        if rate == sr:
            n, up, down = n_pad, 0, 0
        else:
            n = int(np.ceil(n_pad * (float(rate) / sr)))
            g = math.gcd(int(sr), int(rate))
            up, down = int(rate) // g, int(sr) // g
        factor = sr / rate
        hop_f = hop_length / factor
        w = round(win_length / factor)
        start = np.arange(0, n - w, hop_f)
        if len(start) < n_frames:   # util.fix_length zero-pads the filtered signal: the kernel reads zeros past n
            min_length = int(np.ceil(n_frames * hop_f)) + w
            start = np.arange(0, min_length - w, hop_f)
        starts = np.round(start).astype(int)[:n_frames]
        assert len(starts) == n_frames
        leaves = pairwise_leaves(w)
        if leaves_depth(leaves) > nat.IIRT_MAX_DEPTH:
            raise nat.UnsupportedOnGPU(f"iirt: a window of {w} samples is too long for the GPU's pairwise sum")
        lo, hi = bank.band_off[ri], bank.band_off[ri + 1]
        p_max = int(bank.info[bank.bands[lo:hi], 1].max())
        out.append(Rate(float(rate), n, up, down, int(w), float(factor), starts.astype(np.int32), leaves, n + p_max,
                        hi - lo))
    return tuple(out)


def plan(shape, *, sr, win_length: int, hop_length, center: bool, tuning, pad_mode, res_type, kwargs) -> Plan:
    """The host half of iirt for a signal of ``shape`` after the flayout and util.valid_audio checks: the
    reference's remaining checks in its order (padding, filter design, resampling, frame count, sosfiltfilt's
    length check per band), the GPU's refusals where the reference would use what is refused, and every table."""
    n = shape[-1]
    if hop_length is None:
        hop_length = win_length // 4
    pad = 0
    if center:
        pad = win_length // 2
        pad_mode = check_pad_mode(pad_mode, n, len(shape), pad)
    n_pad = n + 2 * pad
    key, bank = bank_cached(tuning, kwargs)
    if bank.max_sections > nat.IIRT_MAX_SECTIONS:
        raise nat.UnsupportedOnGPU(f"iirt: a filter of {bank.max_sections} second-order sections; the GPU filter "
                                   f"kernel takes at most {nat.IIRT_MAX_SECTIONS} (ellip / cheby1 / cheby2 / butter "
                                   "at the default Q need 4 / 6 / 6 / 10): raise Q or lower the attenuation")
    for rate in bank.rates:
        if rate == sr:
            continue
        if res_type != "polyphase":
            _refuse_resampler(res_type)
        if int(sr) != sr or int(rate) != rate:
            raise ParameterError("polyphase resampling is only supported for integer-valued sampling rates.")
    if len(bank.rates) > nat.IIRT_MAX_RATES:
        raise nat.UnsupportedOnGPU(f"iirt: {len(bank.rates)} distinct sample_rates; the GPU kernels take at most "
                                   f"{nat.IIRT_MAX_RATES}")
    n_frames = int(1 + (n_pad - win_length) // hop_length)
    if n_frames < 0:
        raise ValueError("negative dimensions are not allowed")   # np.empty_like's error
    lengths = [n_pad if r == sr else int(np.ceil(n_pad * (float(r) / sr))) for r in bank.rates]
    for b in range(len(bank.sos)):
        p = int(bank.info[b, 1])
        if lengths[bank.rate_of[b]] <= p:
            raise ValueError(f"The length of the input vector x must be greater than padlen, which is {p}.")
    rates = rate_tables(bank, n_pad, sr=sr, win_length=win_length, hop_length=hop_length, n_frames=n_frames)
    return Plan(key, bank, pad, pad_mode if center else "constant", n_pad, n_frames, rates)


def _table(ctx, key, arr) -> int:
    return pl.f64_constant(ctx, key, arr)


def group_size(p: Plan, n_clips: int, pool_bytes: int) -> int:
    """Clips per filter launch: as many as keep the float64 scratch within the context's memory pool."""
    per_clip = max(1, p.clip_bytes())
    return int(max(1, min(n_clips, pool_bytes // per_clip)))


def descriptors(ctx, p: Plan, signals, m: int, d_scratch: int):
    """The b2l_iirt_rate array of one group of ``m`` clips: ``signals`` holds per rate (device pointer of the
    group's first clip, row stride in samples); the scratch is carved per rate from ``d_scratch``."""
    bank = p.bank
    d_bands = _table(ctx, ("iirt_bands",) + p.bank_key, bank.bands)
    starts = np.concatenate([r.starts for r in p.rates])
    d_starts = _table(ctx, ("iirt_starts", starts.tobytes(), p.n_frames), starts)
    leaves = np.concatenate([r.leaves for r in p.rates])
    d_leaves = _table(ctx, ("iirt_leaves", leaves.tobytes()), leaves)
    descs = (nat.IirtRate * len(p.rates))()
    off = leaf_off = 0
    for ri, (r, (ptr, stride)) in enumerate(zip(p.rates, signals)):
        st = -(-m * r.n_bands // 32) * 32
        descs[ri] = nat.IirtRate(ptr, stride, r.n, d_scratch + off, st, d_bands + 4 * bank.band_off[ri], r.n_bands,
                                 len(r.leaves), d_starts + 4 * ri * p.n_frames, d_leaves + 16 * leaf_off, r.factor)
        off += 8 * r.rows * st
        leaf_off += len(r.leaves)
    return descs


def filter_and_power(ctx, p: Plan, signals, m: int, d_scratch: int, d_out: int):
    """Launch b2l_iirt_filter and b2l_iirt_stmsp for ``m`` clips whose per-rate signals are ``signals``
    ((device pointer, row stride) per rate), into ``d_out`` [m][bands][T]; the filtered chains stay in
    ``d_scratch`` (``p.scratch_bytes(m)`` bytes)."""
    bank = p.bank
    d_coef = _table(ctx, ("iirt_coef",) + p.bank_key, bank.coef)
    d_info = _table(ctx, ("iirt_info",) + p.bank_key, bank.info)
    descs = descriptors(ctx, p, signals, m, d_scratch)
    L = nat.lib()
    nat.check(L.b2l_iirt_filter(ctx.handle, descs, len(descs), _vp(d_coef), _vp(d_info), bank.max_sections, m))
    nat.check(L.b2l_iirt_stmsp(ctx.handle, descs, len(descs), m, p.n_frames, len(bank.sos), _vp(d_out)))


def _run(staged, p: Plan):
    """Enqueue padding, resampling, filtering and power for a staged signal; returns the (..., bands, T) result."""
    ctx, m = staged.ctx, staged.n_clips
    L = nat.lib()
    n_bands = len(p.bank.sos)
    with pl.Scope(staged.dev) as sc:
        staged.scan_all()
        x = staged.dev.ptr
        if p.pad:
            padded = sc.empty((m, p.n_pad), np.float32)
            if m:
                nat.check(L.b2l_pad_center(ctx.handle, _vp(x), m, staged.n, p.pad, nat.PAD_MODES[p.pad_mode],
                                           _vp(padded.ptr)))
            x = padded.ptr
        signals = []
        for r in p.rates:
            if not r.up:
                signals.append((x, p.n_pad))
                continue
            d = sc.empty((m, r.n), np.float32)
            h, n_pre_remove = _poly_filter(r.up, r.down)
            d_h = _table(ctx, ("resample_poly", r.up, r.down), h)
            n_out = (p.n_pad * r.up + r.down - 1) // r.down
            if m:
                nat.check(L.b2l_resample_poly(ctx.handle, _vp(x), m, p.n_pad, p.n_pad, _vp(d_h), len(h), r.up, r.down,
                                              n_pre_remove, min(n_out, r.n), r.n, 1.0, _vp(d.ptr)))
            signals.append((d.ptr, r.n))
        out = sc.empty(tuple(staged.lead) + (n_bands, p.n_frames), np.float32)
        if m and p.n_frames:
            g = group_size(p, m, ctx.pool_limit_bytes)
            scratch = sc.empty((p.scratch_bytes(g) // 8,), np.float64)
            for c0 in range(0, m, g):
                mm = min(g, m - c0)
                filter_and_power(ctx, p, [(ptr + 4 * c0 * st, st) for ptr, st in signals], mm, scratch.ptr,
                                 out.ptr + 4 * c0 * n_bands * p.n_frames)
        return sc.keep(out)


def iirt(y, *, sr: float = 22050, win_length: int = 2048, hop_length=None, center: bool = True, tuning: float = 0.0,
         pad_mode="constant", flayout: str = "sos", res_type: str = "soxr_hq", **kwargs):
    """Semitone filter-bank spectrogram; same contract as ``librosa.iirt`` (core/spectrum.py:1522-1713).

    Returns ``(..., n_bands, n_frames)`` of the input's dtype (float64 audio is computed in float32).  A DeviceArray
    in gives a float32 DeviceArray out.  The filtering follows ``flayout="sos"`` only: ``"ba"`` is ill-conditioned
    in the reference itself and is refused.  Resampling runs only with ``res_type="polyphase"``; a call whose band
    rates all equal ``sr`` accepts any ``res_type``."""
    if flayout not in ("ba", "sos"):
        raise ParameterError(f"Unsupported flayout={flayout}")
    n, req = pl.precheck_signal(y)
    try:
        if flayout == "ba":
            filters.semitone_filterbank(tuning=tuning, flayout="ba", **kwargs)
            raise nat.UnsupportedOnGPU("iirt(flayout='ba'): the transfer-function form is ill-conditioned for these "
                                       "filters (its float64 result moves by up to 1e-4 relative under a change of "
                                       "evaluation order) and is not run on the GPU; pass flayout='sos'")
        p = plan(tuple(y.shape), sr=sr, win_length=win_length, hop_length=hop_length, center=center, tuning=tuning,
                 pad_mode=pad_mode, res_type=res_type, kwargs=kwargs)
    except Exception:
        # the reference's util.valid_audio raises on non-finite audio before any of these checks
        if not isinstance(y, nat.DeviceArray) and not np.isfinite(y).all():
            raise ParameterError(pl._NOT_FINITE) from None
        raise
    staged = pl.StagedInput(y)
    try:
        out = _run(staged, p)
    finally:
        staged.release()
    return staged.result(out, req)
