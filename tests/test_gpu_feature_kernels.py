"""GPU (-m gpu): the kernels of csrc/feat_kernels.cuh that sit next to the FFT path — contrast_kernel
(spectral_contrast), frame_td_block_kernel and frame_td_kernel (rms(y=), zero_crossing_rate), hpss_kernel<NS>
(decompose.hpss, effects.hpss / harmonic / percussive), pcen_kernel and maxfilter_rows_kernel (pcen) — at every
path, sort rung, warps-per-block rung and tile boundary, against a float64 reference built here.  The host side
(path and instance choice, sizing, the block decomposition of the framings) is restated in
tests/test_feature_kernels_algorithm.py, which also generates the contrast case list.

The tests call b2l_spectral_contrast / b2l_frame_feature / b2l_hpss / b2l_pcen with the descriptors the public
functions build, into NaN-filled outputs with guard words on both sides: every valid value must come back written
and every guard word must still be NaN.  Before each checked call the same instance runs once on NaN input, so
shared memory holds NaN when the checked call starts.

Tolerances (u = 2^-24; the selected or filtered values are exact float32 inputs, so only the arithmetic after the
selection is bounded).
    contrast        valley / peak: the mean of the kk = min(k, n) extremes of the band.  The extremes themselves are
                    selected exactly; their float32 sum has at most m roundings on the way, m = kk - 1 for the
                    sorted-run and knock-out paths (kk sequential adds) and ceil(kk / 32) - 1 + 5 for the bitonic
                    path (a per-lane chunk, then the 5-level butterfly of warp_sum); the division adds one:
                        |mean - mean64| <= (m + 1) u mean|tail|      (n = 0: NaN, like np.mean of an empty slice)
                    One wrong element moves the mean by (its distance from the right one) / kk, far more.
    contrast public linear=False: power_to_db of both means (10 log10 in float32: 2 u relative in the value, 2 ulp
                    of log10f) and the subtraction; checked at 1e-3 dB.  From y=, the spectrogram's own contract
                    (1e-4 |S| + 1e-5 max S, the order statistics are 1-Lipschitz in the max norm) carried into dB.
    rms             e2 = sum x^2 over the frame: per-lane fma chain of c terms, 5-level butterfly, R block adds (block
                    kernel) -> |e2 - e2_64| <= (c + R + 6) u e2_64, then / L and sqrtf (2 roundings, halved by the
                    root): |rms - rms64| <= ((c + R + 8) / 2 + 2) u rms64, c = max(ceil(hop / 32), 4 ceil(hop / 128))
                    (block) or ceil(L / 32), R = 0 (per frame).  linear_ramp padding adds 1 u per ramp sample (the
                    kernel rounds i * edge / pad once to float32, np.pad keeps float64): 2 u more.
    zero crossings  exact (integer counts), and bit-identical between the float4 and scalar block paths.
    hpss masks      a = x / z, b = x_ref / z (1 rounding each), a^p (p = 2: 1 more, twice the relative error of a),
                    pa + pb, the division: |m - m64| <= C_MASK u m64 with C_MASK = 8 (p = 1 needs 4); the masked
                    output one rounding more.  power = inf: the hard mask, exact (x_ref = perc * margin rounded to
                    float32 in the reference, as the kernel and the reference's float32 arithmetic do).
    pcen            M: each step M = fma(b, r, z) and z = (1 - b) M round once each and are damped by (1 - b) per
                    step: 2 u / b in all; the float32 coefficient 1 - b is off by u, which accumulates over the
                    1 / b-step memory to u / b more; so |M - M64| <= dM M64 with dM = (3 / b + 2) u.  The log of
                    the smoother: inv_eps, M * inv_eps (1 u each), log1pf (1 ulp), logf(eps) (1 ulp), the sum, the
                    product with -gain:  E = gain ((dM + 4 u) + 2 u |ln eps| + 2 u log1p(M / eps)) + 2 u |ls|.
                    g = x exp(ls): E + 4 u relative (expf 2 ulp, the product).  Then per mode, with the ulp bounds of
                    the CUDA C++ Programming Guide (logf, log1pf, expm1f 1 ulp; expf, powf 2 ulp):
                      mode 0  log1pf(g):               (E + 4 u) g / (1 + g) + 2 u |out|
                      mode 1  expf(p (logf x + ls)):   |out| (p (E + 2 u |ln x| + 2 u |ln x + ls|) + 4 u)
                      mode 2  bias^p expm1f(p log1pf(g / bias)):  with h = log1p(g / bias),
                              dh = (E + 5 u) (g / bias) / (1 + g / bias) + 2 u h, dv = p dh + u p h,
                              |out| 6 u + bias^p e^(p h) dv
                    each doubled in count (every ulp counted as 2 u) to absorb second-order terms.

Largest ratio (error / bound) each family saw on an H100 80GB HBM3 at a 700 W power limit:
    contrast 0.62, contrast public (S=, in dB) 0.013, rms 0.35, hpss soft masks and masked outputs 0.55, pcen 0.15;
    zero crossings and the hard masks exact, the streaming split bit for bit.  The whole file runs in about 11 s.
"""
import ctypes

import numpy as np
import pytest

from test_feature_kernels_algorithm import (CONTRAST_LADDER, CONTRAST_REFUSED_F, contrast_cases, contrast_path,
                                            hpss_instance, layout, td_choice)
from test_gpu_mel_front_end import GUARD, device_input, nan_buffer, unguard

pytestmark = [pytest.mark.gpu, pytest.mark.filterwarnings("ignore")]

U = 2.0 ** -24
TINY32 = float(np.finfo(np.float32).tiny)
C_MASK = 8.0
GUARD_C = 38                 # complex outputs: float2 stores need 8-byte alignment
RATIOS = {}
vp = ctypes.c_void_p


def note(name, ratio):
    RATIOS[name] = max(RATIOS.get(name, 0.0), float(ratio))


@pytest.fixture(scope="module")
def lb():
    import librosa_b200

    librosa_b200.default_context()
    yield librosa_b200
    print("\nlargest error / bound ratios:", {k: round(v, 3) for k, v in sorted(RATIOS.items())})


def ctx_lib(lb):
    from librosa_b200 import _native as nat

    return lb.default_context(), nat.lib(), nat


def out_buffer(lb, words, guard=GUARD):
    return nan_buffer(lb, words + 2 * guard)


# ------------------------------------------------------------------ spectral contrast
def contrast_native(lb, S, bands, n_clips=1, offset=0):
    """b2l_spectral_contrast on float32 rows S [n_clips * n_frames, F] -> (peak, valley) [band, row]."""
    ctx, L, nat = ctx_lib(lb)
    rows, F = S.shape
    nb = len(bands)
    desc = nat.ContrastDesc(n_bands=nb)
    for b, (lo, n, k) in enumerate(bands):
        desc.lo[b], desc.count[b], desc.k[b] = lo, n, k
    din = device_input(lb, S, offset)
    peak, valley = out_buffer(lb, nb * rows), out_buffer(lb, nb * rows)
    nat.check(L.b2l_spectral_contrast(ctx.handle, ctypes.byref(desc), vp(din.ptr + 4 * offset), n_clips,
                                      rows // n_clips, F, vp(peak.ptr + 4 * GUARD), vp(valley.ptr + 4 * GUARD)))
    what = f"contrast F={F} bands={bands}"
    res = []
    for buf in (peak, valley):
        v = unguard(buf.get(), what).reshape(n_clips, nb, rows // n_clips)
        res.append(v.transpose(1, 0, 2).reshape(nb, rows))
        buf.free()
    din.free()
    return res[0], res[1]


def contrast_ref(S, bands):
    """float64 valley / peak: np.sort of the band, the means of its kk smallest and kk largest."""
    peak = np.empty((len(bands), S.shape[0]))
    valley = np.empty_like(peak)
    for b, (lo, n, k) in enumerate(bands):
        s = np.sort(S[:, lo:lo + n].astype(np.float64), axis=-1)
        kk = min(k, n)
        valley[b] = s[:, :kk].mean(axis=-1) if kk else np.nan
        peak[b] = s[:, n - kk:].mean(axis=-1) if kk else np.nan
    return peak, valley


def contrast_roundings(n, k):
    kk = min(k, n)
    path = contrast_path(n, kk)[0]
    return (kk - 1 if path != "bitonic" else -(-kk // 32) - 1 + 5) + 1


def contrast_close(peak, valley, S, bands, what):
    rp, rv = contrast_ref(S, bands)
    for b, (lo, n, k) in enumerate(bands):
        for got, ref, side in ((peak[b], rp[b], "peak"), (valley[b], rv[b], "valley")):
            if min(k, n) == 0:
                assert np.isnan(got).all(), f"{what} band {b}: an empty band must give NaN"
                continue
            assert np.isfinite(got).all(), f"{what} band {b} {side}: {int((~np.isfinite(got)).sum())} not written"
            bound = contrast_roundings(n, k) * U * np.abs(ref)
            err = np.abs(got.astype(np.float64) - ref)
            note("contrast", (err / np.maximum(bound, 1e-300)).max())
            bad = ~(err <= bound)
            assert not bad.any(), (f"{what} band {b} (n={n}, k={k}) {side}: {int(bad.sum())} rows, "
                                   f"max err {err.max():.3e} vs bound {bound[bad].min():.3e}")


def contrast_rows(n, k, lo, F, n_rows, seed):
    """n_rows rows of F magnitudes: random rows and the adversarial layouts of the band [lo, lo + n)."""
    rng = np.random.default_rng(seed)
    kinds = ["random", "equal", "zeros", "lane0", "lane31", "lastlane", "dups"]
    S = rng.uniform(0.5, 2.0, (n_rows, F)).astype(np.float32)
    for r in range(n_rows):
        S[r, lo:lo + n] = layout(kinds[r % len(kinds)], n, k, rng)
    return S


@pytest.mark.parametrize("n, k", contrast_cases())
def test_contrast_every_path_and_rung(lb, n, k):
    lo = 5 if n % 2 else 36                        # first bin: not a multiple of 4 / a multiple of 4 but not of 32
    F = lo + n + 3
    bands = [(lo, n, k), (0, min(F, 40), 2)]
    S = contrast_rows(n, k, lo, F, 2 * 21, seed=n * 97 + k)
    contrast_native(lb, np.full_like(S, np.nan), bands, n_clips=2)
    peak, valley = contrast_native(lb, S, bands, n_clips=2, offset=1)
    contrast_close(peak, valley, S, bands, f"n={n} k={k}")


def test_contrast_many_bands_and_empty(lb):
    """16 bands in one call, an empty band (count 0 -> NaN), k above the count, several warps of a block."""
    rng = np.random.default_rng(7)
    F = 1025
    bands = [(0, 0, 1), (0, 3, 1), (3, 3, 5), (6, 29, 1), (35, 64, 2), (99, 65, 3), (164, 129, 9), (293, 257, 17),
             (550, 475, 10), (0, 1025, 20), (1000, 25, 25), (7, 512, 16), (7, 513, 16), (100, 33, 16), (60, 32, 17),
             (1024, 1, 1)]
    S = rng.exponential(1.0, (3 * 37, F)).astype(np.float32)
    S[::5, 100:300] = 0.0
    contrast_native(lb, np.full_like(S, np.nan), bands, n_clips=3)
    peak, valley = contrast_native(lb, S, bands, n_clips=3)
    contrast_close(peak, valley, S, bands, "16 bands")


def ladder_edges():
    ends = [f for _, f in CONTRAST_LADDER[1:]] + [CONTRAST_REFUSED_F]
    return [(nw, f) for (nw, f0), f1 in zip(CONTRAST_LADDER, ends) for f in (f0, f1 - 1) if f >= 64]


@pytest.mark.parametrize("nw, F", ladder_edges())
def test_contrast_warps_per_block_rungs(lb, nw, F):
    """The first and last F of every warps-per-block rung (one band over the whole row sets the sort capacity), with
    more rows than warps of a block."""
    rng = np.random.default_rng(F)
    bands = [(0, F, 3), (F // 3, min(700, F - F // 3), 30), (F - 40, 40, 16)]
    S = rng.uniform(0.0, 1.0, (2 * nw + 3, F)).astype(np.float32)
    contrast_native(lb, np.full_like(S, np.nan), bands)
    peak, valley = contrast_native(lb, S, bands)
    contrast_close(peak, valley, S, bands, f"F={F} nw={nw}")


def test_contrast_refused_row(lb):
    from librosa_b200 import _native as nat

    S = np.ones((2, CONTRAST_REFUSED_F), np.float32)
    with pytest.raises(nat.UnsupportedOnGPU, match="shared memory"):
        contrast_native(lb, S, [(0, CONTRAST_REFUSED_F, 3)])


def ref_power_to_db(x):
    """power_to_db(ref=1.0, amin=1e-10, top_db=80) in float64."""
    d = 10.0 * np.log10(np.maximum(1e-10, x))
    return np.maximum(d, d.max() - 80.0)


def ref_contrast(S64, freq, sr, fmin, n_bands, quantile, linear):
    """librosa's spectral_contrast restated in float64 (feature/spectral.py:483-532)."""
    octa = np.zeros(n_bands + 2)
    octa[1:] = fmin * (2.0 ** np.arange(0, n_bands + 1))
    peak = np.zeros((n_bands + 1, S64.shape[-1]))
    valley = np.zeros_like(peak)
    for k in range(n_bands + 1):
        band = np.logical_and(freq >= octa[k], freq <= octa[k + 1])
        idx = np.flatnonzero(band)
        if k > 0:
            band[idx[0] - 1] = True
        if k == n_bands:
            band[idx[-1] + 1:] = True
        sub = S64[band]
        if k < n_bands:
            sub = sub[:-1]
        q = int(max(np.rint(quantile * np.sum(band)), 1))
        s = np.sort(sub, axis=0)
        valley[k] = np.mean(s[:q], axis=0)
        peak[k] = np.mean(s[-q:], axis=0)
    if linear:
        return peak - valley, peak, valley
    return ref_power_to_db(peak) - ref_power_to_db(valley), peak, valley


@pytest.mark.parametrize("n_fft, sr, fmin, n_bands, quantile, linear", [
    (2048, 22050, 200.0, 6, 0.02, False), (1024, 16000, 100.0, 4, 0.25, True), (4096, 44100, 60.0, 8, 0.1, False),
    (400, 16000, 200.0, 5, 0.02, False)])
def test_contrast_public(lb, n_fft, sr, fmin, n_bands, quantile, linear):
    """spectral_contrast(S=...) against the float64 formula on the same S, and (y=...) against it on the float64
    spectrogram (the STFT contract carried through the order statistics and the dB conversion)."""
    import scipy.fft as sf

    from test_gpu_inverse_pow2 import window

    rng = np.random.default_rng(n_fft)
    F = n_fft // 2 + 1
    S = rng.gamma(0.5, 1.0, (F, 40)).astype(np.float32)
    freq = np.fft.rfftfreq(n_fft, 1.0 / sr)
    kw = dict(sr=sr, fmin=fmin, n_bands=n_bands, quantile=quantile, linear=linear)
    got = lb.feature.spectral_contrast(S=S, n_fft=n_fft, **kw)
    ref = ref_contrast(S.astype(np.float64), freq, sr, fmin, n_bands, quantile, linear)[0]
    err = np.abs(got - ref)
    tol = 1e-3 if not linear else 40 * U * np.abs(S).max()       # at most 17 roundings on each mean, the difference
    note("contrast public", (err / tol).max())
    assert (err <= tol).all(), f"S=: max err {err.max():.3e}"
    # y=: float64 |stft|
    y = (0.1 * rng.standard_normal(n_fft * 12)).astype(np.float32)
    hop = n_fft // 4
    got = lb.feature.spectral_contrast(y=y, n_fft=n_fft, hop_length=hop, **kw)
    yp = np.pad(y.astype(np.float64), n_fft // 2)
    frames = np.lib.stride_tricks.sliding_window_view(yp, n_fft)[::hop] * window("hann", n_fft)
    S64 = np.abs(sf.rfft(frames, axis=-1)).T
    ref, p64, v64 = ref_contrast(S64, freq, sr, fmin, n_bands, quantile, linear)
    ds = 1e-4 * S64.max() + 1e-5 * S64.max()                 # order statistics: 1-Lipschitz in the max norm
    if linear:
        tol = 2 * ds + 1e-6
    else:
        tol = 10 / np.log(10) * ds * (1 / np.maximum(p64 - ds, 1e-10) + 1 / np.maximum(v64 - ds, 1e-10)) + 1e-3
    err = np.abs(got - ref)
    assert (err <= tol).all(), f"y=: {int((err > tol).sum())} values, max err {err.max():.3e}"


# ------------------------------------------------------------------ rms and zero crossings
PAD_MODES = ["constant", "edge", "reflect", "symmetric", "linear_ramp"]


def frame_native(lb, y, what, L, hop, center=True, pad_mode="constant", threshold=0.0, zero_pos=1, pad_first=0,
                 offset=0):
    """b2l_frame_feature (out_scale 1: rms, or the zero-crossing count) on float32 clips y [n_clips, n]."""
    ctx, lib, nat = ctx_lib(lb)
    n_clips, n = y.shape
    pad = L // 2 if center else 0
    T = 1 + (n + 2 * pad - L) // hop
    din = device_input(lb, y, offset)
    out = out_buffer(lb, n_clips * T)
    nat.check(lib.b2l_status_reset(ctx.handle))
    nat.check(lib.b2l_frame_feature(ctx.handle, what, vp(din.ptr + 4 * offset), n_clips, n, n, L, hop, int(center),
                                    nat.PAD_MODES[pad_mode], float(threshold), int(zero_pos), int(pad_first), 1.0,
                                    vp(out.ptr + 4 * GUARD)))
    res = unguard(out.get(), f"frame_feature L={L} hop={hop}").reshape(n_clips, T)
    out.free()
    din.free()
    return res


def padded_frames(y, L, hop, center, pad_mode):
    y64 = y.astype(np.float64)
    if center:
        y64 = np.pad(y64, [(0, 0), (L // 2, L // 2)], mode=pad_mode)
    return np.lib.stride_tricks.sliding_window_view(y64, L, axis=-1)[:, ::hop]


def ref_rms(y, L, hop, center, pad_mode):
    return np.sqrt(np.mean(padded_frames(y, L, hop, center, pad_mode) ** 2, axis=-1))


def ref_crossings(y, L, hop, center, pad_mode, threshold, zero_pos, pad_first):
    x = padded_frames(y, L, hop, center, pad_mode).copy()
    x[np.abs(x) <= threshold] = 0.0
    c = np.signbit(x) if zero_pos else np.sign(x)
    return (c[..., 1:] != c[..., :-1]).sum(axis=-1) + int(bool(pad_first))


def rms_close(got, y, L, hop, center, pad_mode, what):
    ref = ref_rms(y, L, hop, center, pad_mode)
    block = td_choice(L, hop, y.shape[0], ref.shape[-1])
    R = L // hop if block else 0
    c = max(-(-hop // 32), 4 * -(-hop // 128)) if block else -(-L // 32)
    bound = ((c + R + 8) / 2 + 2 + (2 if pad_mode == "linear_ramp" else 0)) * U * ref
    err = np.abs(got.astype(np.float64) - ref)
    note("rms", (err / np.maximum(bound, 1e-300)).max())
    assert (err <= bound).all(), f"{what}: max err {err.max():.3e}"


def td_signal(n_clips, n, seed, zeros=0.2):
    rng = np.random.default_rng(seed)
    y = rng.standard_normal((n_clips, n)).astype(np.float32)
    y[rng.random(y.shape) < zeros] = 0.0
    y[rng.random(y.shape) < 0.05] *= 1e-3
    return y


def check_td(lb, y, L, hop, center, pad_mode, threshold=0.0, zero_pos=1, pad_first=0, offset=0):
    from librosa_b200 import _native as nat

    what = f"L={L} hop={hop} center={center} {pad_mode} thr={threshold} zp={zero_pos} pf={pad_first} off={offset}"
    for w in (nat.FRAME_RMS, nat.FRAME_ZERO_CROSSINGS):
        frame_native(lb, np.full_like(y, np.nan), w, L, hop, center, pad_mode, threshold, zero_pos, pad_first, offset)
        got = frame_native(lb, y, w, L, hop, center, pad_mode, threshold, zero_pos, pad_first, offset)
        if w == nat.FRAME_RMS:
            rms_close(got, y, L, hop, center, pad_mode, what)
        else:
            ref = ref_crossings(y, L, hop, center, pad_mode, threshold, zero_pos, pad_first)
            assert np.array_equal(got, ref.astype(np.float32)), f"{what}: {int((got != ref).sum())} frames differ"
    return got


@pytest.mark.parametrize("L, hop", [(2048, 512), (1024, 256), (12, 4), (600, 150), (1032, 516), (64, 1), (129, 129),
                                    (384, 128), (8192, 128), (8320, 130), (1000, 300), (513, 512)])
@pytest.mark.parametrize("center, pad_mode", [(False, "constant")] + [(True, m) for m in PAD_MODES])
def test_frame_features_geometries(lb, L, hop, center, pad_mode):
    """Both kernels (block: frame_length a multiple of hop, R <= 64; per frame otherwise) at T = 1 (mod 64) and
    T = 0 (mod 64) and every pad mode; rms to its a priori bound, zero crossings exactly."""
    for T in (65, 64):
        n = (T - 1) * hop + (L - 2 * (L // 2) if center else L) + (hop // 2 if T == 65 else 0)
        y = td_signal(2, n, seed=L + hop + T)
        check_td(lb, y, L, hop, center, pad_mode)


@pytest.mark.parametrize("L, hop", [(2048, 512), (12, 4), (600, 150), (36, 12), (2064, 516)])
def test_zero_crossings_vector_and_scalar_paths(lb, L, hop):
    """Aligned input (float4 path where hop % 4 == 0 and pad % 4 == 0) against input one float off (scalar path):
    the counts agree with the reference and with each other, with zero_pos on and off, pad on and off, and
    thresholds equal to sample magnitudes."""
    rng = np.random.default_rng(L)
    y = (rng.integers(-3, 4, (3, 40 * hop + 7)) * 0.25).astype(np.float32)
    y += (rng.random(y.shape) < 0.3) * rng.standard_normal(y.shape).astype(np.float32) * 1e-3
    for threshold in (0.0, float(np.abs(y[0, 5])), 0.25, 0.5):
        for zero_pos in (1, 0):
            for pad_first in (0, 1):
                a = check_td(lb, y, L, hop, True, "edge", threshold, zero_pos, pad_first, offset=0)
                b = check_td(lb, y, L, hop, True, "edge", threshold, zero_pos, pad_first, offset=1)
                assert np.array_equal(a, b)


def test_frame_features_many_clips(lb):
    """65 536 short clips: more than grid.y holds, so the per-frame kernel serves a block geometry."""
    assert not td_choice(16, 4, 65536, 17)
    y = td_signal(65536, 64, seed=3)
    check_td(lb, y, 16, 4, True, "edge", threshold=0.0, zero_pos=1, pad_first=0)


def test_uncovered_nan(lb):
    """A NaN in a sample no frame reads: zero_crossing_rate's host scan still raises, as the reference's
    util.valid_audio does; rms(y=) validates nothing in the reference either and returns the covered frames."""
    from librosa_b200.util.exceptions import ParameterError

    y = td_signal(1, 4096 + 100, seed=9)[0]
    y[-3] = np.nan                                       # center=False, frame 2048 hop 512: the last 100+ unread
    with pytest.raises(ParameterError):
        lb.feature.zero_crossing_rate(y, frame_length=2048, hop_length=512, center=False)
    got = lb.feature.rms(y=y, frame_length=2048, hop_length=512, center=False)
    rms_close(got[0], y[None], 2048, 512, False, "constant", "rms, uncovered NaN")


# ------------------------------------------------------------------ hpss
def hpss_native(lb, M, Sc, wh, wp, margin=(1.0, 1.0), power=2.0, mask=False):
    """b2l_hpss on magnitudes M [clip, T, F] (bins contiguous) and optionally the complex Sc of the same shape."""
    ctx, L, nat = ctx_lib(lb)
    n_clips, T, F = M.shape
    complex_out = Sc is not None and not mask
    words = M.size * (2 if complex_out else 1)
    dm = device_input(lb, M, 0)
    ds = lb.DeviceArray.empty(ctx, (2 * Sc.size,), np.float32).set(Sc.view(np.float32).ravel()) if Sc is not None \
        else None
    g = GUARD_C if complex_out else GUARD
    oh, op = out_buffer(lb, words, g), out_buffer(lb, words, g)
    desc = nat.HpssDesc(win_harm=wh, win_perc=wp, margin_harm=margin[0], margin_perc=margin[1], power=power,
                        mask_only=int(mask))
    nat.check(L.b2l_hpss(ctx.handle, ctypes.byref(desc), vp(dm.ptr), vp(ds.ptr if ds is not None else None), n_clips,
                         T, F, vp(oh.ptr + 4 * g), vp(op.ptr + 4 * g)))
    res = []
    for buf in (oh, op):
        v = unguard(buf.get(), f"hpss T={T} F={F} w=({wh},{wp})", g)
        res.append(v.view(np.complex64).reshape(M.shape) if complex_out else v.reshape(M.shape))
        buf.free()
    dm.free()
    if ds is not None:
        ds.free()
    return res


def ref_median(M, w, axis, rank=None):
    """Median over w neighbours along `axis` of the np.pad symmetric extension, rank w // 2 (scipy's
    median_filter(mode='reflect') where it is defined; it is not where w // 2 exceeds the axis)."""
    pw = [(0, 0)] * M.ndim
    pw[axis] = (w // 2, w - 1 - w // 2)
    xp = np.pad(M, pw, mode="symmetric")
    win = np.lib.stride_tricks.sliding_window_view(xp, w, axis=axis)
    return np.sort(win, axis=-1)[..., w // 2 if rank is None else rank]


def ref_softmask(x, xr, power, split_zeros):
    """util.softmask in float64 on float32 inputs."""
    x, xr = x.astype(np.float64), xr.astype(np.float64)
    if np.isinf(power):
        return (x > xr).astype(np.float64)
    z = np.maximum(x, xr)
    bad = z < TINY32
    z = np.where(bad, 1.0, z)
    a, b = (x / z) ** power, (xr / z) ** power
    return np.where(bad, 0.5 if split_zeros else 0.0, a / np.where(bad, 1.0, a + b))


def hpss_ref(M, wh, wp, margin, power, rank_h=None, rank_p=None):
    harm = ref_median(M, wh, 1, rank_h)
    perc = ref_median(M, wp, 2, rank_p)
    split = margin[0] == 1.0 and margin[1] == 1.0
    mh = ref_softmask(harm, perc * np.float32(margin[0]), power, split)      # float32 products, as the kernel
    mp = ref_softmask(perc, harm * np.float32(margin[1]), power, split)
    return mh, mp


def hpss_close(got, M, Sc, wh, wp, margin, power, mask, what, rank_h=None, rank_p=None):
    mh, mp = hpss_ref(M, wh, wp, margin, power, rank_h, rank_p)
    for g, m, side in ((got[0], mh, "harm"), (got[1], mp, "perc")):
        if mask:
            ref, scale, c = m, m, C_MASK
        elif Sc is not None:
            ref, scale, c = Sc.astype(np.complex128) * m, np.abs(Sc) * m, C_MASK + 1
        else:
            ref, scale, c = M.astype(np.float64) * m, M * m, C_MASK + 1
        err = np.abs(g.astype(ref.dtype) - ref)
        if np.isinf(power):
            assert np.array_equal(g.astype(ref.dtype), ref), f"{what} {side}: hard mask not exact"
            continue
        bound = c * U * scale
        note("hpss", (err / np.maximum(bound, 1e-300)).max())
        bad = ~(err <= bound)
        assert not bad.any(), f"{what} {side}: {int(bad.sum())} elements, max err {err.max():.3e}"


def hpss_input(n_clips, T, F, seed, complex_=True):
    rng = np.random.default_rng(seed)
    Sc = (rng.standard_normal((n_clips, T, F)) + 1j * rng.standard_normal((n_clips, T, F))).astype(np.complex64)
    Sc[:, ::7, :] = 0                                     # all-zero frames
    Sc[:, :, 1::5] = 0                                    # all-zero bins
    if F > 3:
        Sc[:, :, 2] *= 1e3                                # a strong harmonic line
    M = np.abs(Sc).astype(np.float32)
    return M, (Sc if complex_ else None)


def check_hpss(lb, M, Sc, wh, wp, margin=(1.0, 1.0), power=2.0, mask=False):
    what = f"T={M.shape[1]} F={M.shape[2]} w=({wh},{wp}) margin={margin} power={power} mask={mask}"
    hpss_native(lb, np.full_like(M, np.nan), Sc, wh, wp, margin, power, mask)
    got = hpss_native(lb, M, Sc, wh, wp, margin, power, mask)
    hpss_close(got, M, Sc, wh, wp, margin, power, mask, what)


WINDOWS = [1, 7, 8, 9, 16, 17, 32, 33, 63, 64]


@pytest.mark.parametrize("w", WINDOWS)
def test_hpss_windows(lb, w):
    """Every NS instance at both ends, odd and even windows, as harmonic and as percussive window."""
    M, Sc = hpss_input(2, 45, 70, seed=w)
    check_hpss(lb, M, None, w, 5, mask=True)
    check_hpss(lb, M, None, 3, w, mask=True)
    check_hpss(lb, M, Sc, w, w, power=1.0)
    assert hpss_instance(w, 5) == hpss_instance(3, w)


@pytest.mark.parametrize("T", [1, 2, 3, 31, 129])
@pytest.mark.parametrize("F", [1, 2, 3, 31, 129])
def test_hpss_short_axes(lb, T, F):
    """Half-windows longer than the axis: the np.pad symmetric extension, repeated."""
    M, Sc = hpss_input(1, T, F, seed=T * 131 + F)
    check_hpss(lb, M, Sc, 31, 17, power=2.0)
    check_hpss(lb, M, None, 64, 6, power=1.0, mask=True)


@pytest.mark.parametrize("power", [1.0, 2.0, np.inf])
@pytest.mark.parametrize("margin", [(1.0, 1.0), (1.0, 3.0), (2.5, 1.5)])
@pytest.mark.parametrize("kind", ["mask", "complex", "real"])
def test_hpss_masks(lb, power, margin, kind):
    """Masks and masked components with power 1, 2 and inf, margins of 1 (zeros split) and above, all-zero frames
    and bins; the hard mask exactly."""
    M, Sc = hpss_input(2, 40, 33, seed=int(margin[1] * 10))
    check_hpss(lb, M, Sc if kind == "complex" else None, 17, 9, margin, power, mask=kind == "mask")


# ------------------------------------------------------------------ pcen
def pcen_native(lb, S, gain=0.98, bias=2.0, power=0.5, eps=1e-6, b=0.025, max_size=1, zi=None, want_zf=False):
    """b2l_pcen on S [clip, rows, T] -> (out, zf or None)."""
    ctx, L, nat = ctx_lib(lb)
    n_clips, rows, T = S.shape
    din = device_input(lb, S, 0)
    out = out_buffer(lb, S.size)
    zf = out_buffer(lb, n_clips * rows) if want_zf else None
    dzi = lb.DeviceArray.empty(ctx, (n_clips * rows,), np.float32).set(zi.astype(np.float32).ravel()) \
        if zi is not None else None
    scr = nan_buffer(lb, S.size) if max_size > 1 else None
    desc = nat.PcenDesc(gain=gain, bias=bias, power=power, eps=eps, b=b, max_size=max_size)
    nat.check(L.b2l_pcen(ctx.handle, ctypes.byref(desc), vp(din.ptr), n_clips, rows, T,
                         vp(dzi.ptr if dzi is not None else None), vp(zf.ptr + 4 * GUARD if zf is not None else None),
                         vp(scr.ptr if scr is not None else None), vp(out.ptr + 4 * GUARD)))
    what = f"pcen rows={rows} T={T}"
    res = unguard(out.get(), what).reshape(S.shape)
    z = unguard(zf.get(), what).reshape(n_clips, rows) if zf is not None else None
    for buf in (din, out, zf, dzi, scr):
        if buf is not None:
            buf.free()
    return res, z


def pcen_ref(S, gain, bias, power, eps, b, max_size, zi=None):
    """float64 pcen with the kernel's float32 parameters: np.pad symmetric max filter over rows, scipy lfilter with
    zi = 1 - b, the reference's three output forms.  Returns (out, M)."""
    import scipy.signal as ss

    gain, bias, power, eps, b = (float(np.float32(v)) for v in (gain, bias, power, eps, b))
    S64 = S.astype(np.float64)
    if max_size > 1:
        pw = [(0, 0), (max_size // 2, max_size - 1 - max_size // 2), (0, 0)]
        ref = np.lib.stride_tricks.sliding_window_view(np.pad(S64, pw, mode="symmetric"), max_size, axis=1).max(-1)
    else:
        ref = S64
    z0 = np.full(S.shape[:-1] + (1,), 1.0 - b) if zi is None else zi.astype(np.float64)[..., None]
    M, _ = ss.lfilter([b], [1.0, b - 1.0], ref, axis=-1, zi=z0)
    ls = -gain * (np.log(eps) + np.log1p(M / eps))
    smooth = np.exp(ls)
    if power == 0:
        out = np.log1p(S64 * smooth)
    elif bias == 0:
        with np.errstate(divide="ignore"):
            out = np.exp(power * (np.log(S64) + ls))
    else:
        out = bias ** power * np.expm1(power * np.log1p(S64 * smooth / bias))
    return out, M


def pcen_bound(S, M, out, gain, bias, power, eps, b):
    """The a priori bound of the module docstring, elementwise (every ulp counted as 2 u)."""
    gain, bias, power, eps, b = (float(np.float32(v)) for v in (gain, bias, power, eps, b))
    x = S.astype(np.float64)
    dM = (3.0 / max(b, 1e-30) + 2.0) * U
    ls = -gain * (np.log(eps) + np.log1p(M / eps))
    E = gain * ((dM + 4 * U) + 2 * U * abs(np.log(eps)) + 2 * U * np.log1p(M / eps)) + 2 * U * np.abs(ls)
    g = x * np.exp(ls)
    if power == 0:
        bnd = (E + 4 * U) * g / (1 + g) + 2 * U * np.abs(out)
    elif bias == 0:
        with np.errstate(divide="ignore", invalid="ignore"):
            lx = np.where(x > 0, np.abs(np.log(np.where(x > 0, x, 1.0))), 0.0)
            bnd = np.abs(out) * (power * (E + 2 * U * lx + 2 * U * np.abs(lx + ls)) + 4 * U)
    else:
        r = g / bias
        h = np.log1p(r)
        dh = (E + 5 * U) * r / (1 + r) + 2 * U * h
        dv = power * dh + U * power * h
        bnd = np.abs(out) * 6 * U + bias ** power * np.exp(power * h) * dv
    return 2.0 * bnd + 1e-30


def pcen_close(got, S, gain, bias, power, eps, b, max_size, what, zi=None):
    ref, M = pcen_ref(S, gain, bias, power, eps, b, max_size, zi)
    bnd = pcen_bound(S, M, ref, gain, bias, power, eps, b)
    g = got.astype(np.float64)
    err = np.where(g == ref, 0.0, np.abs(g - ref))
    note("pcen", (err / bnd).max())
    bad = ~(err <= bnd)
    assert not bad.any(), f"{what}: {int(bad.sum())} elements, max err {err.max():.3e}"


def pcen_input(n_clips, rows, T, seed):
    rng = np.random.default_rng(seed)
    S = (rng.gamma(0.7, 1.0, (n_clips, rows, T)) * 2.0 ** 31 * 1e-9).astype(np.float32)
    if T > 5:
        S[..., ::5] = 0.0
    return S


def check_pcen(lb, S, **kw):
    what = f"pcen {S.shape} {kw}"
    pcen_native(lb, np.full_like(S, np.nan), **kw)
    got, _ = pcen_native(lb, S, **kw)
    full = dict(gain=0.98, bias=2.0, power=0.5, eps=1e-6, b=0.025, max_size=1)
    full.update(kw)
    pcen_close(got, S, what=what, **full)


@pytest.mark.parametrize("rows", [1, 31, 32, 33, 127, 128, 129])
@pytest.mark.parametrize("T", [1, 31, 32, 33, 65])
def test_pcen_tiles(lb, rows, T):
    """32 x 32 tiles of pcen_kernel at every row and time remainder, over two clips (rows flattened)."""
    check_pcen(lb, pcen_input(2, rows, T, seed=rows * 100 + T))


@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("max_size", [1, 2, 3])
@pytest.mark.parametrize("b", [1e-3, 0.025, 0.999, 1.0])
def test_pcen_modes(lb, mode, max_size, b):
    """power == 0, bias == 0, general; max_size 1, 2 (even size: window [m - 1, m]) and 3; b near 0 and 1."""
    kw = {0: dict(power=0.0), 1: dict(bias=0.0, eps=1e-3), 2: dict(power=0.25, bias=10.0, gain=0.8)}[mode]
    check_pcen(lb, pcen_input(3, 33, 70, seed=mode * 10 + max_size), max_size=max_size, b=b, **kw)


@pytest.mark.parametrize("split", [1, 17, 45])
def test_pcen_streaming(lb, split):
    """zi / zf streaming split at a non-multiple of 32 equals the one-shot call bit for bit, and zi is honoured."""
    S = pcen_input(2, 35, 77, seed=split)
    one, zf_one = pcen_native(lb, S, want_zf=True)
    a, za = pcen_native(lb, np.ascontiguousarray(S[..., :split]), want_zf=True)
    c, zc = pcen_native(lb, np.ascontiguousarray(S[..., split:]), zi=za, want_zf=True)
    assert np.array_equal(np.concatenate([a, c], axis=-1), one)
    assert np.array_equal(zc, zf_one)
    zi = np.random.default_rng(split).uniform(0.0, 3.0, (2, 35)).astype(np.float32)
    got, _ = pcen_native(lb, S, zi=zi)
    pcen_close(got, S, 0.98, 2.0, 0.5, 1e-6, 0.025, 1, "pcen zi", zi=zi)


# ------------------------------------------------------------------ batches beyond 65 535 frames / clips / rows
def test_hpss_many_frames(lb):
    """hpss of F = 3, T = 70 001: frames run in slices of 65 535 (public call, against the float64 reference)."""
    M, Sc = hpss_input(1, 70001, 3, seed=70001)
    harm, perc = lb.decompose.hpss(np.ascontiguousarray(M[0].T))      # magnitudes: the complex form computes its own
    hpss_close((harm.T[None], perc.T[None]), M, None, 31, 31, (1.0, 1.0), 2.0, False, "hpss T=70001")
    hpss_native(lb, np.full_like(M, np.nan), Sc, 31, 31)
    h, p = hpss_native(lb, M, Sc, 31, 31)
    hpss_close((h, p), M, Sc, 31, 31, (1.0, 1.0), 2.0, False, "hpss complex T=70001")
    h, p = hpss_native(lb, M, None, 31, 31, mask=True)
    hpss_close((h, p), M, None, 31, 31, (1.0, 1.0), 2.0, True, "hpss masks T=70001")


def test_hpss_many_clips(lb):
    """70 001 clips of a 3 x 4 spectrogram: clips run in slices of 65 535."""
    M, Sc = hpss_input(70001, 4, 3, seed=4)
    M *= np.random.default_rng(1).uniform(0.5, 1.5, (70001, 1, 1)).astype(np.float32)
    harm, perc = lb.decompose.hpss(np.ascontiguousarray(M.transpose(0, 2, 1)), kernel_size=(3, 5), margin=2.0)
    hpss_close((harm.transpose(0, 2, 1), perc.transpose(0, 2, 1)), M, None, 3, 5, (2.0, 2.0), 2.0, False,
               "hpss 70001 clips")


@pytest.mark.parametrize("max_size", [1, 3])
def test_pcen_many_clips(lb, max_size):
    """pcen of 70 001 clips of 3 x 4: the max filter runs in slices of 65 535 clips."""
    S = pcen_input(70001, 3, 4, seed=max_size)
    S[65530:65540] *= 7.0
    got = lb.pcen(S, max_size=max_size, max_axis=-2 if max_size > 1 else None)
    b = (np.sqrt(1 + 4 * (0.4 * 22050 / 512.0) ** 2) - 1) / (2 * (0.4 * 22050 / 512.0) ** 2)
    pcen_close(got, S, 0.98, 2.0, 0.5, 1e-6, b, max_size, "pcen 70001 clips")


def test_pcen_many_rows(lb):
    """pcen of a 2-D S with 70 001 rows, max_size 1 and 3 (rows run in slices of 65 535)."""
    S = pcen_input(1, 70001, 8, seed=5)
    for max_size in (1, 3):
        got = lb.pcen(S[0], max_size=max_size)
        b = (np.sqrt(1 + 4 * (0.4 * 22050 / 512.0) ** 2) - 1) / (2 * (0.4 * 22050 / 512.0) ** 2)
        pcen_close(got[None], S, 0.98, 2.0, 0.5, 1e-6, b, max_size, f"pcen 70001 rows max_size={max_size}")
