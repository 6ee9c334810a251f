"""NumPy restatements of what the reference computes around the onset-strength, dB, row-normalisation, tuning and
polyphase-resampling kernels (csrc/feat_kernels.cuh), in the reference's precision where a test compares bit for bit
and in float64 where it compares within a bound.  tests/test_feature_tail_host.py pins them against the reference's
outputs stored in tests/golden/features_v1.npz; tests/test_gpu_feature_kernels_tail.py compares the kernels with them.
"""
from __future__ import annotations

import warnings

import numpy as np
import scipy.ndimage
import scipy.signal



def max_filter_rows(S, size):
    """scipy.ndimage.maximum_filter1d(S, size, axis=-2) (reflect boundary) for finite and infinite data; a NaN in a
    window makes that window's maximum NaN, as np.maximum does (scipy's running-max filter keeps or drops a NaN
    depending on where it sits in the window)."""
    if size == 1:
        return S
    if not np.isnan(S).any():
        return scipy.ndimage.maximum_filter1d(S, size, axis=-2, mode="reflect")
    n = S.shape[-2]
    out = np.empty_like(S)
    for m in range(n):
        rows = []
        for j in range(size):
            mm = m - size // 2 + j
            while mm < 0 or mm >= n:
                mm = -mm - 1 if mm < 0 else 2 * n - mm - 1
            rows.append(mm)
        out[..., m, :] = np.maximum.reduce([S[..., r, :] for r in rows])
    return out


def onset_flux(S, lag, max_size):
    """onset_strength_multi after the spectrogram (librosa/onset.py:580-612): the float32 lag difference against the
    max-filtered reference, negatives discarded with np.maximum (which keeps NaN).  S [..., rows, T]."""
    S = np.asarray(S, np.float32)
    ref = max_filter_rows(S, max_size)
    with np.errstate(invalid="ignore"):
        return np.maximum(0.0, S[..., lag:] - ref[..., :-lag])


def onset_envelope(S, *, lag, max_size, pad_width, bounds=None, median=False):
    """The C entries' output [..., n_out, T]: util.sync mean / median of the flux over the channel rows
    [bounds[c], bounds[c + 1]) (bounds None: aggregate=False), then the left pad of pad_width zeros and the crop to
    T frames.  With pad_width < lag the frames past the flux are zero."""
    S = np.asarray(S, np.float32)
    T = S.shape[-1]
    flux = onset_flux(S, lag, max_size) if T > lag else S[..., :0]
    if bounds is not None:
        agg = np.median if median else np.mean
        with warnings.catch_warnings():           # the mean / median of an empty channel is NaN
            warnings.simplefilter("ignore")
            flux = np.stack([agg(flux[..., a:b, :], axis=-2).astype(np.float32)
                             for a, b in zip(bounds[:-1], bounds[1:])], axis=-2)
    out = np.zeros(flux.shape[:-1] + (T,), np.float32)
    n = max(0, min(flux.shape[-1], T - pad_width))
    out[..., pad_width:pad_width + n] = flux[..., :n]
    return out


def normalize(S, norm):
    """librosa.util.normalize(S, norm=norm, axis=-2) with the default threshold and fill (util/utils.py:797-1026):
    mag = |S| in float64, NumPy's own power shortcuts, S / length rounded once to S's type."""
    S = np.asarray(S)
    mag = np.abs(S).astype(float)
    if norm == np.inf:
        length = np.max(mag, axis=-2, keepdims=True)
    elif norm == -np.inf:
        length = np.min(mag, axis=-2, keepdims=True)
    elif norm == 0:
        length = np.sum(mag > 0, axis=-2, keepdims=True, dtype=mag.dtype)
    else:
        length = np.sum(mag ** norm, axis=-2, keepdims=True) ** (1.0 / norm)
    length[length < np.finfo(S.dtype).tiny] = 1.0
    return (S / length).astype(S.dtype)


def tuning_histograms(pitch, mag, *, prefix0, prefix1, mag_threshold, bins_per_octave, edges):
    """The four pass histograms of estimate_tuning over a dense piptrack output (pitch, mag): the top 11 / middle
    11 (under prefix0) / low 10 (under prefix1) bits of the order-preserving key of mag at pitch > 0, and the
    residual histogram of the peaks with mag >= mag_threshold."""
    sel = pitch > 0
    keys = float_keys(mag[sel])
    h0 = np.bincount(keys >> 21, minlength=2048)
    h1 = np.bincount((keys[(keys >> 21) == prefix0] >> 10) & 0x7FF, minlength=2048)
    h2 = np.bincount(keys[(keys >> 10) == prefix1] & 0x3FF, minlength=1024)
    res = residuals(pitch[sel & (mag >= mag_threshold)], bins_per_octave)
    h3, _ = np.histogram(res[~np.isnan(res)], edges)
    return h0, h1, h2, h3


def residuals(f, bins_per_octave):
    """pitch_tuning's folded residuals mod(bins_per_octave * log2(f / 27.5), 1) of float32 f > 0, each operation in
    float32 as the reference does it, with log2 correctly rounded: NumPy's float32 log2 rounds differently on CPUs
    with and without its SIMD loops (about one value in 150 differs in the last bit), the kernels round once from
    float64."""
    f = np.asarray(f, np.float32)
    f = f[f > 0]
    with np.errstate(invalid="ignore"):
        x = np.float32(bins_per_octave) * np.log2((f / np.float32(27.5)).astype(np.float64)).astype(np.float32)
        r = np.mod(x, np.float32(1.0))
        r[r >= 0.5] -= np.float32(1.0)
    return r


def float_keys(x):
    """The order-preserving uint32 key of float32 values (csrc/common.cuh float_to_key)."""
    u = np.asarray(x, np.float32).view(np.uint32).astype(np.uint64)
    return np.where(u & 0x80000000, ~u & 0xFFFFFFFF, u | 0x80000000).astype(np.int64)


def resample_poly64(x, h, up, down, n_pre_remove, n_keep, n_total):
    """scipy.signal.resample_poly's upfirdn over the float32 taps h in float64, cropped to [n_pre_remove,
    n_pre_remove + n_keep) and zero filled to n_total; also the same sums over |h| and |x| (the error bound's
    scale).  x [..., n]."""
    def crop(v):
        out = np.zeros(v.shape[:-1] + (n_total,))
        seg = v[..., n_pre_remove:n_pre_remove + n_keep]
        out[..., :seg.shape[-1]] = seg
        return out

    h64 = np.asarray(h, np.float64)
    x64 = np.asarray(x, np.float64)
    return (crop(scipy.signal.upfirdn(h64, x64, up, down, axis=-1)),
            crop(scipy.signal.upfirdn(np.abs(h64), np.abs(x64), up, down, axis=-1)))
