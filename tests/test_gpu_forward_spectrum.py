"""GPU (-m gpu): the STFT, spectrogram and spectral-statistics epilogues of the forward kernels — fwd_kernel in
MODE_STFT, MODE_SPEC and MODE_STATS (csrc/fwd_kernel.cuh) for the powers of two, mr_kernel<0, G> and mr_kernel<1, G>
(csrc/mr_kernel.cuh) for the mixed-radix sizes, and stats_kernel (csrc/feat_kernels.cuh) for the S= statistics — at
every kernel instance, tile geometry and clip boundary, against a float64 reference built here: the float32 samples
widened, np.pad, the float64 window (get_window + pad_center), scipy.fft.rfft, |X|**power, and the statistics with
the reference's formulas (librosa/feature/spectral.py) in float64.  The host side (instance choice, stats_kernel
sizing, the frame_stats partition) is restated in tests/test_forward_spectrum_algorithm.py.

The tests call b2l_stft / b2l_spectrogram / b2l_spectral_stats / b2l_spectral_stats_from_spec the way core/spectrum.py
and feature/stats.py do (same plans), but into NaN-filled outputs with guard words on both sides: every valid value
must come back finite and every guard word must still be NaN.  Before each checked call the same instance runs on NaN
audio through the public function (which raises ParameterError), so shared memory holds NaN when the checked call
starts and a read of a word the tile did not write shows up.

Tolerances (u = 2^-24).
    stft, elementwise (the contract)   |X - X64| <= 1e-4 |X64| + 1e-5 max|X64 of the clip|
    stft, norm-wise per frame          ||X - X64||_2 <= C_STFT u log2(n_fft) ||X64||_2 over the bins; a split twiddle
                                       table rounded to 12 mantissa bits exceeds it and passes the contract in most bins
    spectrogram |X|^p                  the same bounds carried through |.|^p: elementwise rtol p 1e-4, atol
                                       p 1e-5 max(S of the clip); per frame ||S - S64|| <= p max|X64|^(p-1)
                                       C_STFT u log2(n_fft) ||X64|| + 4 u ||S64|| (first order, p >= 1)
    statistics from y (fused)          the feature suite's contract: centroid / bandwidth / total rtol 1e-4, atol
                                       1e-6 max; flatness rtol 1e-4, atol 1e-7; rms rtol 1e-4, atol 1e-7 max; roll-off
                                       as below with the spectrum's error added to the running-sum bound
    stats_kernel on identical S        a priori bounds from the summation order of frame_stats: lane chunks of
                                       c = ((F + 31) / 32) | 1 sequential terms, then a 32-lane tree (5 levels):
                                         total    |t - t64| <= (c + 6) u sum|s|
                                         centroid |m1 - m1_64| <= (c + 6) u sum|f s|, divided by the total (its own
                                                  (c + 6) u relative error) and rounded
                                         bandwidth per term d = |f - centroid| (1 rounding), d^2 or powf(d, p) (8 u
                                                  for powf), the fma, the sum (c + 5) u, the centroid's error carried
                                                  through p sum s (d + dc)^(p-1) dc, then /total and ^(1/p) (1/p
                                                  rounded: u |ln b| / p more)
                                         rms      |e2a - e2a_64| <= (c + 8) u sum s^2, then / L^2 and sqrt
                                         roll-off the float64 bin exactly, except where the float64 running sum lies
                                                  within (2 c + 12) u sum|s| of the threshold (lane walk on top of the
                                                  exclusive scan: 2 c + 5 additions, the threshold product and
                                                  roll_percent rounded to float32)
                                         flatness __log2f: 2^-22 absolute on [0.5, 2], 2 ulp of the result elsewhere;
                                                  exp2f: 2 ulp (CUDA C++ Programming Guide, intrinsic and single
                                                  precision function accuracy tables); each term's th = max(amin,
                                                  s^power) 2 u off (s*s and amin rounded), so the mean of log2 is off
                                                  by (sum e_i + (c + 5) u sum|log2 th|) / F + 2 u |mean|, and the
                                                  result by ln 2 that + 4 u + (c + 11) u (arithmetic mean and division)
    bit for bit                        a clip in a batch against the clip alone; input one float off alignment (per-
                                       sample gather, scalar loads) against aligned input (TMA bulk copy, float2
                                       loads); MODE_STATS against b2l_spectrogram(power=1) followed by
                                       b2l_spectral_stats_from_spec (same FFT, same sqrt.approx, same frame_stats: only
                                       the exchange addressing differs) in every row but rms, and each single-row
                                       `want` against want = 0.  The rms row differs in about one frame in ten by one
                                       ulp: stats_kernel accumulates sum s^2 with FFMA (s * s + e2, one rounding), the
                                       fused kernel with FMUL + FADD (two), because its loop keeps s * s for the
                                       flatness (cuobjdump -sass of both, sm_90a, CUDA 12.9).  That row is held to the
                                       a priori rms bound on both paths instead.

C_STFT is the largest ratio ||X - X64|| / (u log2(n_fft) ||X64||) measured by test_stft_every_size and
test_mixed_radix_sizes on an H100 80GB HBM3 (700 W power limit), with about 3x headroom:
    n_fft       8     16     32     64    128    256    512   1024   2048   4096   8192   mixed radix (96 sizes)
    ratio    0.54   0.54   0.40   0.38   0.34   0.28   0.24   0.25   0.22   0.21   0.19   at most 0.54 (n_fft 12)
The largest ratio over every stft call of this file is 0.62 (n_fft 8, test_pads_windows_hops).       C_STFT = 2
"""
import ctypes

import numpy as np
import pytest

from test_forward_spectrum_algorithm import (H100_SPECTRUM_VARIANTS, H100_STATS_VARIANTS, STATS_LADDER,
                                             chunk_of, mr_spectrum_block)
from test_gpu_chirpz import contract_close, ref_stft
from test_gpu_mel_front_end import GUARD, device_input, n_samples, nan_buffer, signals, unguard
from test_mel_front_end_algorithm import MODE_SPEC, MODE_STATS, MODE_STFT, forward_choice, mr_sizes

pytestmark = [pytest.mark.gpu, pytest.mark.filterwarnings("ignore")]

SIZES = [2 << q for q in range(2, 13)]
U = 2.0 ** -24
C_STFT = 2.0                 # norm-wise bound in units of u log2(n_fft), see the module docstring
GUARD_C = 38                 # complex outputs: 8-byte aligned, off 16-byte alignment
TINY32 = float(np.finfo(np.float32).tiny)
KIND_MODE = {"stft": MODE_STFT, "spec": MODE_SPEC, "stats": MODE_STATS}
# The rms row is the one row of MODE_STATS that may differ from stats_kernel on the same magnitudes, by one rounding
# of sum s^2: ptxas contracts `e2 += s * s` of frame_stats (stats.cuh) into FFMA in stats_kernel, but keeps FMUL + FADD
# in the fused kernel, whose loop reuses the product for the flatness (cuobjdump -sass, sm_90a, CUDA 12.9).
RMS_CONTRACTION = 4


@pytest.fixture(scope="module")
def lb():
    import librosa_b200

    librosa_b200.default_context()
    return librosa_b200


# ------------------------------------------------------------------ the float64 reference
def ref_spectrum(y, n_fft, hop, win_length=None, center=True, pad_mode="constant"):
    """rfft(frame * window) in float64, [clip, frame, bin]."""
    return ref_stft(np.asarray(y, dtype=np.float64), n_fft, hop, win_length, center, pad_mode)


def fft_freq(sr, n_fft):
    """The frequency table the statistics read: fft_frequencies in float32 (widened for the reference)."""
    return np.fft.rfftfreq(n_fft, 1.0 / sr).astype(np.float32)


def ref_stats(S, freq, roll=0.85, amin=1e-10, power=2.0, p=2.0, norm=True, frame_length=2):
    """librosa's centroid, bandwidth, roll-off, flatness, rms(S=) and the total, in float64, from S [..., frame, bin]
    (rows [..., 6, frame])."""
    S = np.asarray(S, dtype=np.float64)
    f = np.asarray(freq, dtype=np.float64)
    tot = S.sum(axis=-1)
    nrm = np.where(tot < TINY32, 1.0, tot)                              # util.normalize(norm=1), threshold tiny
    cen = (S * f).sum(axis=-1) / nrm
    dev = np.abs(f - cen[..., None])
    bwt = (S * dev ** p).sum(axis=-1)
    bw = (bwt / nrm if norm else bwt) ** (1.0 / p)
    cum = np.cumsum(S, axis=-1)
    ok = cum >= roll * tot[..., None]
    roll_f = np.where(ok, f, np.inf).min(axis=-1)
    th = np.maximum(amin, S ** power)
    flat = np.exp(np.log(th).mean(axis=-1)) / th.mean(axis=-1)
    x = S ** 2
    x[..., 0] *= 0.5
    if frame_length % 2 == 0:
        x[..., -1] *= 0.5
    rms = np.sqrt(2.0 * x.sum(axis=-1) / float(frame_length) ** 2)
    return np.stack([cen, bw, roll_f, flat, rms, tot], axis=-2)


# ------------------------------------------------------------------ checks
def norm_ratio(got, ref):
    """max over frames of ||got - ref||_2 / (u ||ref||_2) along the bins, [clip, frame, bin]; silent frames exact."""
    err = np.sqrt((np.abs(got.astype(ref.dtype) - ref) ** 2).sum(axis=-1))
    nrm = np.sqrt((np.abs(ref) ** 2).sum(axis=-1))
    assert not err[nrm == 0].any(), "a silent frame is not exactly zero"
    return float((err[nrm > 0] / nrm[nrm > 0]).max(initial=0.0)) / U


def stft_close(got, ref, n_fft, what):
    """The stft checks: the elementwise contract and the per-frame norm-wise bound; returns the ratio in units of
    u log2(n_fft)."""
    contract_close(got, ref, what, rtol=1e-4, atol_rel=1e-5)
    ratio = norm_ratio(got, ref) / np.log2(n_fft)
    assert ratio <= C_STFT, f"{what}: ||err|| = {ratio:.3f} u log2(n_fft) ||X|| (bound {C_STFT})"
    return ratio


def spec_close(got, X64, n_fft, power, what):
    """|X|^power against the float64 magnitudes: the stft bounds carried through |.|^p (module docstring)."""
    A = np.abs(X64)
    S64 = A ** power
    contract_close(got, S64, what, rtol=power * 1e-4, atol_rel=power * 1e-5)
    err = np.sqrt(((got.astype(np.float64) - S64) ** 2).sum(axis=-1))
    xn = np.sqrt((A ** 2).sum(axis=-1))
    bound = power * A.max(axis=-1) ** (power - 1) * C_STFT * U * np.log2(n_fft) * xn + \
        4 * U * np.sqrt((S64 ** 2).sum(axis=-1))
    bad = err > bound
    assert not bad.any(), f"{what}: {int(bad.sum())} frames over the norm-wise bound, worst " \
                          f"{float((err / np.maximum(bound, 1e-300)).max()):.2f} of it"


def rolloff_check(got, S64, freq, roll, tol, what):
    """Roll-off against float64 sums: every frame's value is the float64 answer, except that bins whose float64
    running sum lies within `tol` of the threshold may go either way (got is then the frequency of such a bin, or
    of a bin that is clearly past the threshold, and never above the clear answer)."""
    f = np.asarray(freq, dtype=np.float32).astype(np.float64)
    cum = np.cumsum(S64, axis=-1)
    thr = roll * S64.sum(axis=-1)[..., None]
    tol = np.broadcast_to(np.asarray(tol, dtype=np.float64), thr.shape[:-1])[..., None]
    strict = cum >= thr + tol
    loose = cum >= thr - tol
    hi = np.where(strict, f, np.inf).min(axis=-1)
    hi = np.where(np.isinf(hi), f[-1], hi)                              # nothing clearly past: the kernel's fallback
    lo = np.where(loose, f, np.inf).min(axis=-1)
    g = got.astype(np.float64)
    member = (np.where(loose, f, np.nan)[..., :] == g[..., None]).any(axis=-1) | (g == f[-1])
    bad = ~((g >= np.minimum(lo, hi)) & (g <= hi) & member)
    assert not bad.any(), f"{what}: roll-off of {int(bad.sum())} frames, first {np.argwhere(bad)[0].tolist()}"
    return int((loose & ~strict).any(axis=-1).sum())                   # frames with a bin inside the bound


def stats_bounds(S, freq, p=2.0, norm=True, power=2.0, frame_length=2):
    """A priori bounds of frame_stats on float32 rows S [..., frame, bin] against float64 on the same values (module
    docstring): dict row -> bound array [..., frame], and the roll-off running-sum tolerance."""
    S = np.asarray(S, dtype=np.float32).astype(np.float64)
    f = np.asarray(freq, dtype=np.float32).astype(np.float64)
    F = S.shape[-1]
    c = chunk_of(F)
    g = (c + 6) * U
    A = np.abs(S).sum(axis=-1)
    tot = S.sum(axis=-1)
    nrm = np.where(tot < TINY32, 1.0, tot)
    out = {"total": g * A}
    m1 = (S * f).sum(axis=-1)
    cen = m1 / nrm
    dc = 1.01 * ((g * np.abs(S * f).sum(axis=-1) + np.abs(cen) * g * A) / nrm + 2 * U * np.abs(cen))
    out["centroid"] = dc
    d = np.abs(f - cen[..., None])
    W = (S * d ** p).sum(axis=-1)
    term = (4 if p == 2 else p + 9) * U
    Eb = (term + (c + 5) * U) * W + p * (S * (d + dc[..., None]) ** (p - 1)).sum(axis=-1) * dc
    bwt = W / nrm if norm else W
    with np.errstate(divide="ignore", invalid="ignore"):
        rel = Eb / W + ((g * A / nrm + U) if norm else 0.0)
        rel = rel / p + (U if p == 2 else 8 * U + U * np.abs(np.log(np.where(bwt > 0, bwt, 1.0))) / p)
        bw = bwt ** (1.0 / p)
        out["bandwidth"] = np.where(W > 0, 1.01 * bw * rel, 0.0)
    out["rolloff_tol"] = (2 * c + 12) * U * A
    th = np.maximum(1e-10, S ** power)
    lg = np.log2(th)
    e = 2 * U / np.log(2) + np.where((th >= 0.5) & (th <= 2), 2.0 ** -22, 4 * U * np.abs(lg))
    mean = lg.mean(axis=-1)
    Em = (e.sum(axis=-1) + (c + 5) * U * np.abs(lg).sum(axis=-1)) / F + 2 * U * np.abs(mean)
    flat = np.exp2(mean) / th.mean(axis=-1)
    out["flatness"] = 1.01 * flat * (np.log(2) * Em + 4 * U + (c + 11) * U)
    L = float(frame_length)
    x = S ** 2
    x[..., 0] *= 0.5
    if frame_length % 2 == 0:
        x[..., -1] *= 0.5
    r2 = 2.0 * x.sum(axis=-1) / L ** 2
    rms = np.sqrt(r2)
    d2 = 2 * (c + 8) * U * (S ** 2).sum(axis=-1) / L ** 2 + 3 * U * r2
    with np.errstate(divide="ignore", invalid="ignore"):
        out["rms"] = np.where(rms > 0, 1.01 * (d2 / (2 * rms) + U * rms), np.sqrt(d2))
    return out


ROWS = ("centroid", "bandwidth", "rolloff", "flatness", "rms", "total")


def stats_exact_check(got, S, freq, what, roll=0.85, p=2.0, norm=True, power=2.0, frame_length=2):
    """stats_kernel / MODE_STATS rows [clip, 6, frame] against float64 on the identical float32 rows S [clip, frame,
    bin] at the a priori bounds; returns the number of frames whose roll-off was decided by rounding."""
    ref = ref_stats(S, freq, roll, 1e-10, power, p, norm, frame_length)
    b = stats_bounds(S, freq, p, norm, power, frame_length)
    for r, name in enumerate(ROWS):
        if name == "rolloff":
            continue
        err = np.abs(got[:, r].astype(np.float64) - ref[:, r])
        bad = ~(err <= b[name])
        assert not bad.any(), f"{what}: {name} of {int(bad.sum())} frames off, worst " \
                              f"{float(np.nanmax(err / np.maximum(b[name], 1e-300))):.2f} of the bound"
    return rolloff_check(got[:, 2], S.astype(np.float64), freq, np.float32(roll), b["rolloff_tol"], what)


def fused_stats_close(got, X64, freq, n_fft, what, frame_length):
    """MODE_STATS rows [clip, 6, frame] from y against float64 statistics of |X64|: the feature suite's contract."""
    S64 = np.abs(X64)
    ref = ref_stats(S64, freq.astype(np.float64), frame_length=frame_length)
    for r, name, rtol, atol in ((0, "centroid", 1e-4, 1e-6), (1, "bandwidth", 1e-4, 1e-6), (3, "flatness", 1e-4, None),
                                (4, "rms", 1e-4, 1e-7), (5, "total", 1e-4, 1e-6)):
        a = 1e-7 if atol is None else atol * float(np.abs(ref[:, r]).max())
        contract = np.abs(got[:, r] - ref[:, r]) <= rtol * np.abs(ref[:, r]) + a
        assert contract.all(), f"{what}: {name} of {int((~contract).sum())} frames"
    # the spectrum's own error, summed over the bins (Cauchy-Schwarz on the norm-wise stft bound), on top of the
    # running-sum bound
    F = S64.shape[-1]
    spec_err = np.sqrt(F) * (C_STFT * U * np.log2(n_fft) + 4 * U) * np.sqrt((S64 ** 2).sum(axis=-1))
    tol = (2 * chunk_of(F) + 12) * U * S64.sum(axis=-1) + spec_err
    rolloff_check(got[:, 2], S64, freq, np.float32(0.85), tol, what)


# ------------------------------------------------------------------ the kernels under NaN-filled outputs
def plan_for(lb, kind, n_fft, hop, win_length=None, center=True, pad_mode="constant", power=2.0):
    """The plan core/spectrum.py (stft, _spectrogram) or feature/stats.py (the y= statistics) makes."""
    from librosa_b200 import _native as nat, _pipeline as pl

    w, wkey = pl.resolve_window("hann", win_length or n_fft, n_fft)
    mode = pad_mode if center else "constant"
    kw = dict(n_fft=n_fft, hop_length=hop, center=center, pad_mode=mode, window=w)
    if kind == "stft":
        key = ("stft", n_fft, hop, bool(center), mode, wkey)
    elif kind == "spec":
        key = ("spec", n_fft, hop, bool(center), mode, wkey, float(power))
        kw["power"] = float(power)
    else:
        key = ("stats", n_fft, hop, bool(center), mode, wkey)
        kw["power"] = 1.0
    return nat.make_plan(lb.default_context(), key, **kw)


def stats_desc(want=0, roll=0.85, amin=1e-10, power=2.0, p=2.0, norm=True, frame_length=2):
    from librosa_b200 import _native as nat

    return nat.StatsDesc(roll_percent=roll, flat_amin=amin, flat_power=power, bw_p=p, bw_norm=int(norm),
                         frame_length=frame_length, want=want)


def device_floats(lb, x):
    x = np.ascontiguousarray(x, dtype=np.float32).ravel()
    return lb.DeviceArray.empty(lb.default_context(), x.shape, np.float32).set(x)


def native(lb, y, n_fft, hop, kind="stft", offset=0, want=0, frame_length=None, **kw):
    """b2l_stft ([clip, frame, bin] complex64), b2l_spectrogram ([clip, frame, bin]) or b2l_spectral_stats ([clip, 6,
    frame], all six rows unless `want` names one) on the float32 batch y [clip, n], the input `offset` floats into its
    allocation, the output between NaN guard words."""
    from librosa_b200 import _native as nat, _pipeline as pl

    ctx = lb.default_context()
    vp = ctypes.c_void_p
    plan = plan_for(lb, kind, n_fft, hop, kw.get("win_length"), kw.get("center", True), kw.get("pad_mode", "constant"),
                    kw.get("power", 2.0))
    n_clips, n = y.shape
    T = plan.n_frames(n)
    M1 = n_fft // 2 + 1
    what = f"{kind} n_fft={n_fft} hop={hop} clips={n_clips} T={T} {kw}"
    din = device_input(lb, y, offset)
    nat.check(nat.lib().b2l_status_reset(ctx.handle))
    src = vp(din.ptr + 4 * offset)
    if kind == "stft":
        out = nan_buffer(lb, 2 * n_clips * T * M1 + 2 * GUARD_C)
        nat.check(nat.lib().b2l_stft(ctx.handle, plan.handle, src, n_clips, n, n, vp(out.ptr + 4 * GUARD_C)))
        res = unguard(out.get(), what, GUARD_C).view(np.complex64).reshape(n_clips, T, M1)
        rows = res
    elif kind == "spec":
        out = nan_buffer(lb, n_clips * T * M1 + 2 * GUARD)
        nat.check(nat.lib().b2l_spectrogram(ctx.handle, plan.handle, src, n_clips, n, n, vp(out.ptr + 4 * GUARD)))
        res = rows = unguard(out.get(), what).reshape(n_clips, T, M1)
    else:
        fq = device_floats(lb, fft_freq(22050, n_fft))
        out = nan_buffer(lb, n_clips * 6 * T + 2 * GUARD)
        desc = stats_desc(want, frame_length=frame_length or n_fft)
        nat.check(nat.lib().b2l_spectral_stats(ctx.handle, plan.handle, ctypes.byref(desc), src, n_clips, n, n,
                                               vp(fq.ptr), vp(out.ptr + 4 * GUARD)))
        res = unguard(out.get(), what).reshape(n_clips, 6, T)
        rows = res if not want else res[:, int(np.log2(want))]
        fq.free()
    out.free()
    din.free()
    assert not pl.status_word(ctx) & nat.STATUS_NOT_FINITE_SAMPLE, f"{what}: finite input flagged"
    assert np.isfinite(rows).all(), f"{what}: {int((~np.isfinite(rows)).sum())} values not written"
    return res


def native_from_spec(lb, S, freq, desc, n_bins=None):
    """b2l_spectral_stats_from_spec on host rows S [clip, frame, bin]: ([clip, 6, frame], status word)."""
    from librosa_b200 import _native as nat, _pipeline as pl

    ctx = lb.default_context()
    vp = ctypes.c_void_p
    n_clips, T, F = S.shape
    dS = device_floats(lb, S)
    fq = device_floats(lb, freq)
    out = nan_buffer(lb, n_clips * 6 * T + 2 * GUARD)
    nat.check(nat.lib().b2l_status_reset(ctx.handle))
    try:
        nat.check(nat.lib().b2l_spectral_stats_from_spec(ctx.handle, ctypes.byref(desc), vp(dS.ptr), n_clips, T,
                                                         n_bins or F, vp(fq.ptr), vp(out.ptr + 4 * GUARD)))
        res = unguard(out.get(), f"stats_kernel F={F}").reshape(n_clips, 6, T)
        status = pl.status_word(ctx)
    finally:
        for a in (dS, fq, out):
            a.free()
    return res, status


def poison(lb, kind, y_shape, n_fft, hop, **kw):
    """The same instance on NaN audio through the public function: raises, and leaves NaN in shared memory."""
    from librosa_b200.core.spectrum import _spectrogram
    from librosa_b200.util.exceptions import ParameterError

    nan = np.full(y_shape, np.nan, np.float32)
    pk = dict(n_fft=n_fft, hop_length=hop, center=kw.get("center", True), pad_mode=kw.get("pad_mode", "constant"),
              win_length=kw.get("win_length"))
    with pytest.raises(ParameterError):
        if kind == "stft":
            lb.stft(nan, **pk)
        elif kind == "spec":
            _spectrogram(y=nan, power=kw.get("power", 2.0), **pk)
        else:
            lb.feature.spectral_centroid(y=nan, sr=22050, **pk)


def check_stft(lb, y, n_fft, hop, **kw):
    """native stft after a poisoning call, against float64; returns (X, X64, ratio)."""
    poison(lb, "stft", y.shape, n_fft, hop, **kw)
    X = native(lb, y, n_fft, hop, "stft", **kw)
    X64 = ref_spectrum(y, n_fft, hop, kw.get("win_length"), kw.get("center", True), kw.get("pad_mode", "constant"))
    ratio = stft_close(X, X64, n_fft, f"stft n_fft={n_fft} hop={hop} {kw}")
    print(f"RATIO all n_fft={n_fft} hop={hop} {ratio:.3f}")
    return X, X64, ratio


def check_spec(lb, y, n_fft, hop, X64=None, **kw):
    poison(lb, "spec", y.shape, n_fft, hop, **kw)
    S = native(lb, y, n_fft, hop, "spec", **kw)
    if X64 is None:
        X64 = ref_spectrum(y, n_fft, hop, kw.get("win_length"), kw.get("center", True), kw.get("pad_mode", "constant"))
    spec_close(S, X64, n_fft, kw.get("power", 2.0), f"spectrogram n_fft={n_fft} hop={hop} {kw}")
    return S


def check_stats(lb, y, n_fft, hop, X64=None, frame_length=None, **kw):
    """fused statistics after a poisoning call, against float64 from y; returns the rows."""
    poison(lb, "stats", y.shape, n_fft, hop, **kw)
    R = native(lb, y, n_fft, hop, "stats", frame_length=frame_length, **kw)
    if X64 is None:
        X64 = ref_spectrum(y, n_fft, hop, kw.get("win_length"), kw.get("center", True), kw.get("pad_mode", "constant"))
    fused_stats_close(R, X64, fft_freq(22050, n_fft), n_fft, f"stats n_fft={n_fft} hop={hop} {kw}",
                      frame_length or n_fft)
    return R


def tile_frames(n_fft, hop, kind):
    return forward_choice(n_fft, hop, None, mode=KIND_MODE[kind])[1]


def tma_staging(n_fft, hop, y_stride, offset, kind):
    """run_forward's tma_ok (spectrum_api.cu) for a clip `offset` floats past a 16-byte aligned allocation, with FT
    taken from the instance `kind` selects: base, row stride and staged span (FT - 1) hop + n_fft all 16-byte aligned.
    Interior tiles then stage by TMA bulk copy (TILE_TMA), edge tiles with constant padding by TILE_TMA_ZERO."""
    return offset % 4 == 0 and y_stride % 4 == 0 and ((tile_frames(n_fft, hop, kind) - 1) * hop + n_fft) % 4 == 0


# ------------------------------------------------------------------ every instance window
def window_cases(table):
    """(n_fft, hop, FT) at the first and last hop of every instance window, and n_fft // 4 where it falls inside."""
    out = []
    for n_fft, (runs, _) in table.items():
        for first, last, v, ft in runs:
            for hop in sorted({first, last, n_fft // 4} & set(range(first, last + 1))):
                out.append((n_fft, hop, ft))
    return out


@pytest.mark.parametrize("n_fft,hop,ft", window_cases(H100_SPECTRUM_VARIANTS))
def test_spectrum_every_instance_window(lb, n_fft, hop, ft):
    """MODE_STFT and MODE_SPEC (power 2): two clips of 2 FT + 1 frames (the last tile holds one frame)."""
    assert tile_frames(n_fft, hop, "stft") == tile_frames(n_fft, hop, "spec") == ft
    y = signals(2, n_samples(2 * ft + 1, n_fft, hop, True), n_fft, seed=n_fft + hop)
    _, X64, _ = check_stft(lb, y, n_fft, hop)
    check_spec(lb, y, n_fft, hop, X64=X64)


def stats_identity(lb, y, n_fft, hop, **kw):
    """MODE_STATS (want = 0) against b2l_spectrogram(power=1) followed by b2l_spectral_stats_from_spec: centroid,
    bandwidth, roll-off, flatness and the total bit for bit; rms (see RMS_CONTRACTION) at the a priori bounds of
    stats_kernel on the same rows.  Each single-row want gives the same bits as want = 0."""
    full = native(lb, y, n_fft, hop, "stats", **kw)
    S = native(lb, y, n_fft, hop, "spec", power=1.0, **{k: v for k, v in kw.items() if k != "power"})
    freq = fft_freq(22050, n_fft)
    two, status = native_from_spec(lb, S, freq, stats_desc(frame_length=n_fft))
    assert not status
    exact = [r for r in range(6) if r != RMS_CONTRACTION]
    np.testing.assert_array_equal(full[:, exact], two[:, exact],
                                  err_msg=f"MODE_STATS vs spectrogram + stats_kernel n_fft={n_fft} hop={hop}")
    stats_exact_check(full, S, freq, f"MODE_STATS on its own magnitudes n_fft={n_fft} hop={hop}", frame_length=n_fft)
    stats_exact_check(two, S, freq, f"stats_kernel n_fft={n_fft} hop={hop}", frame_length=n_fft)
    for r in range(6):
        one = native(lb, y, n_fft, hop, "stats", want=1 << r, **kw)
        np.testing.assert_array_equal(one[:, r], full[:, r], err_msg=f"want row {r} n_fft={n_fft} hop={hop}")
    return full, S


@pytest.mark.parametrize("n_fft,hop,ft", window_cases(H100_STATS_VARIANTS))
def test_stats_every_instance_window(lb, n_fft, hop, ft):
    """MODE_STATS: two clips of 2 FT + 1 frames against float64, and reduced to the spectrogram and stats_kernel."""
    assert tile_frames(n_fft, hop, "stats") == ft
    y = signals(2, n_samples(2 * ft + 1, n_fft, hop, True), n_fft, seed=n_fft + hop + 1)
    check_stats(lb, y, n_fft, hop)
    stats_identity(lb, y, n_fft, hop)


@pytest.mark.parametrize("n_fft", SIZES)
def test_first_refused_hop(lb, n_fft):
    """The refusals stay where they are: the first hop past the last window of each mode raises UnsupportedOnGPU."""
    from librosa_b200 import _native as nat
    from librosa_b200.core.spectrum import _spectrogram

    for table, calls in ((H100_SPECTRUM_VARIANTS, ("stft", "spec")), (H100_STATS_VARIANTS, ("stats",))):
        stop = table[n_fft][1]
        y = lb.to_device(signals(1, n_samples(3, n_fft, stop, True), n_fft, seed=1))
        for kind in calls:
            with pytest.raises(nat.UnsupportedOnGPU):
                if kind == "stft":
                    lb.stft(y, n_fft=n_fft, hop_length=stop)
                elif kind == "spec":
                    _spectrogram(y=y, n_fft=n_fft, hop_length=stop, power=2.0)
                else:
                    lb.feature.spectral_centroid(y=y, sr=22050, n_fft=n_fft, hop_length=stop)


def test_plans_exist_exactly_where_a_transform_path_does(lb):
    """The size rule is written twice, once per side of the C ABI: for every n_fft from 1 to 8200, b2l_plan_create
    (plan_path in csrc/plan.cu) makes a plan exactly when _pipeline.transform_path names a path, and refuses every
    other size with require_supported_n_fft's error type and text."""
    from librosa_b200 import _native as nat
    from librosa_b200 import _pipeline as pl

    L = nat.lib()
    win = np.ones(8200)
    desc = nat.PlanDesc(hop_length=1, h_window=win.ctypes.data_as(ctypes.POINTER(ctypes.c_double)), power=2.0,
                        amin=1e-10, ref_value=1.0, top_db=80.0)
    wrong = []
    for n_fft in range(1, 8201):
        desc.n_fft = n_fft
        h = ctypes.c_void_p()
        rc = L.b2l_plan_create(lb.default_context().handle, ctypes.byref(desc), ctypes.byref(h))
        if rc == nat.B2L_OK:
            L.b2l_plan_destroy(h)
            if pl.transform_path(n_fft) is None:
                wrong.append((n_fft, "plan made"))
            continue
        msg = L.b2l_last_error().decode()
        try:
            pl.require_supported_n_fft(n_fft)
            want = None
        except nat.UnsupportedOnGPU as exc:
            want = str(exc)
        if rc != nat.B2L_ERR_UNSUPPORTED or msg != want:
            wrong.append((n_fft, rc, msg, want))
    assert not wrong, wrong[:10]


# ------------------------------------------------------------------ every size, norm-wise; the spectrogram powers
@pytest.mark.parametrize("n_fft", SIZES)
def test_stft_every_size(lb, n_fft):
    """Power-of-two stft at the default hop with frames of very different level in one tile; records the ratio.
    The spectrogram at powers 1 (sqrt.approx), 1.5 (powf) and 2 (the square), and the fused statistics."""
    hop = n_fft // 4
    ft = tile_frames(n_fft, hop, "stft")
    y = signals(3, n_samples(3 * ft + 1, n_fft, hop, True), n_fft, seed=n_fft + 5)
    _, X64, ratio = check_stft(lb, y, n_fft, hop)
    print(f"RATIO pow2 n_fft={n_fft} {ratio:.3f}")
    for power in (1.0, 1.5, 2.0):
        check_spec(lb, y, n_fft, hop, X64=X64, power=power)
    check_stats(lb, y, n_fft, hop, X64=X64)


# ------------------------------------------------------------------ frame counts, pads, windows, hops
@pytest.mark.parametrize("n_fft", [64, 256, 1024, 2048, 4096, 8192])
def test_frame_counts(lb, n_fft):
    """T = 1 and T == 1 mod FT, for each mode with its own FT."""
    hop = n_fft // 4
    for kind in ("stft", "spec", "stats"):
        ft = tile_frames(n_fft, hop, kind)
        for T in sorted({1, ft + 1, 3 * ft + 1}):
            y = signals(2, n_samples(T, n_fft, hop, True), n_fft, seed=n_fft + T)
            {"stft": check_stft, "spec": check_spec, "stats": check_stats}[kind](lb, y, n_fft, hop)


GEOMETRIES = [dict(pad_mode="reflect"), dict(pad_mode="edge"), dict(pad_mode="symmetric"),
              dict(pad_mode="linear_ramp"), dict(center=False), dict(pad_mode="constant")]


@pytest.mark.parametrize("n_fft", [8, 32, 256, 512, 2048, 8192])
def test_pads_windows_hops(lb, n_fft):
    """Every pad mode and center=False, win_length < n_fft on every other geometry, and a hop above n_fft inside the
    window of each mode."""
    spec_stop, stats_stop = H100_SPECTRUM_VARIANTS[n_fft][1], H100_STATS_VARIANTS[n_fft][1]
    big = min(n_fft + n_fft // 3 + 1, spec_stop - 1, stats_stop - 1)
    assert big > n_fft
    for i, g in enumerate(GEOMETRIES):
        kw = dict(g)
        if i % 2:
            kw["win_length"] = n_fft - n_fft // 4 - 1
        hop = big if i == len(GEOMETRIES) - 1 else n_fft // 4
        center = kw.get("center", True)
        y = signals(2, n_samples(9 + i, n_fft, hop, center), n_fft, seed=n_fft + i)
        _, X64, _ = check_stft(lb, y, n_fft, hop, **kw)
        check_spec(lb, y, n_fft, hop, X64=X64, power=(1.0, 1.5, 2.0)[i % 3], **kw)
        check_stats(lb, y, n_fft, hop, X64=X64, **kw)


# ------------------------------------------------------------------ batches that walk across clips
@pytest.mark.parametrize("n_fft", [64, 512, 1024, 2048, 4096, 8192])
def test_batches_across_clips(lb, n_fft):
    """More tiles than resident CTAs (three tiles a clip, T odd): each clip equals the clip run alone, bit for bit."""
    hop = n_fft // 4
    sm = lb.default_context().sm_count
    for kind in ("stft", "spec", "stats"):
        ft = tile_frames(n_fft, hop, kind)
        T = 2 * ft + 1
        n_clips = min(2 * sm + 7, 300)
        y = signals(n_clips, n_samples(T, n_fft, hop, True), n_fft, seed=n_fft + len(kind))
        y[1::3] *= 100.0
        full = {"stft": check_stft, "spec": check_spec, "stats": check_stats}[kind](lb, y, n_fft, hop)
        full = full[0] if kind == "stft" else full
        for c in sorted({0, 1, 2, n_clips // 2, n_clips - 2, n_clips - 1}):
            np.testing.assert_array_equal(native(lb, y[c:c + 1], n_fft, hop, kind)[0], full[c],
                                          err_msg=f"{kind} clip {c}")


# ------------------------------------------------------------------ bit for bit across input paths
@pytest.mark.parametrize("n_fft", [16, 64, 1024, 2048, 4096, 8192])
def test_input_paths_agree(lb, n_fft):
    """The clip at the start of its allocation, stride a multiple of 4, hop % 4 == 0 (interior tiles by TMA bulk copy,
    the edge tiles of constant padding by TILE_TMA_ZERO) against the same clips one float further on (per-sample
    gather), four floats on (aligned again), and reflect padding (edge tiles by the gather) against itself shifted."""
    hop = n_fft // 4
    for kind in ("stft", "spec", "stats"):
        T = 3 * tile_frames(n_fft, hop, kind) + 2
        n = n_samples(T, n_fft, hop, True)
        assert tma_staging(n_fft, hop, n, 0, kind) and tma_staging(n_fft, hop, n, 4, kind)
        assert not tma_staging(n_fft, hop, n, 1, kind)
        y = signals(3, n, n_fft, seed=n_fft + 17)
        for pad_mode in ("constant", "reflect"):
            base = native(lb, y, n_fft, hop, kind, pad_mode=pad_mode)
            for off in (1, 4):
                np.testing.assert_array_equal(native(lb, y, n_fft, hop, kind, offset=off, pad_mode=pad_mode), base,
                                              err_msg=f"{kind} {pad_mode} offset {off}")


# ------------------------------------------------------------------ stats_kernel on identical float32 input
def stats_rows(n_clips, T, F, seed, silent=()):
    """Magnitude-like rows [clip, frame, bin]: a few strong peaks on a noise floor 60 dB down; frames in `silent`
    are all zero."""
    rng = np.random.default_rng(seed)
    S = 1e-3 * np.abs(rng.standard_normal((n_clips, T, F)))
    for c in range(n_clips):
        for t in range(T):
            k = rng.integers(0, F, size=3)
            S[c, t, k] += rng.uniform(0.5, 2.0, size=3)
    for c, t in silent:
        S[c, t] = 0.0
    return S.astype(np.float32)


def check_from_spec(lb, S, freq, what, **kw):
    frame_length = kw.pop("frame_length", 2 * (S.shape[-1] - 1))
    got, status = native_from_spec(lb, S, freq, stats_desc(frame_length=frame_length, **kw))
    assert not status, f"{what}: status {status}"
    assert np.isfinite(got).all(), f"{what}: values not written"
    stats_exact_check(got, S, freq, what, roll=kw.get("roll", 0.85), p=kw.get("p", 2.0), norm=kw.get("norm", True),
                      power=kw.get("power", 2.0), frame_length=frame_length)
    return got


@pytest.mark.parametrize("F", [2, 3, 31, 32, 33, 64, 65, 66, 513, 1025, 1026, 4097])
def test_stats_kernel_bins(lb, F):
    """F == 0, 1, 2 mod 32 and the odd chunk lengths: every row at the a priori bounds, silent frames (centroid 0,
    roll-off freq[0]), odd and even frame_length, bandwidth p = 2 and p = 3 with norm on and off, flatness at
    powers 2 and 1."""
    freq = fft_freq(22050, 2 * (F - 1))
    S = stats_rows(3, 7, F, seed=F, silent=[(0, 0), (2, 6)])
    got = check_from_spec(lb, S, freq, f"F={F}")
    assert got[0, 0, 0] == 0.0 and got[0, 2, 0] == freq[0] and got[2, 2, 6] == freq[0]
    check_from_spec(lb, S, freq, f"F={F} odd frame_length", frame_length=2 * F - 1)
    check_from_spec(lb, S, freq, f"F={F} p=3 norm off", p=3.0, norm=False)
    check_from_spec(lb, S, freq, f"F={F} p=1.5 flatness power 1", p=1.5, power=1.0, roll=0.3)


def test_stats_kernel_custom_frequencies(lb):
    """A custom increasing table and a decreasing one (the roll-off is then the smallest frequency of the bins past
    the threshold, not the first bin)."""
    F = 257
    rng = np.random.default_rng(5)
    S = stats_rows(2, 9, F, seed=7)
    up = np.sort(rng.uniform(10.0, 9000.0, F)).astype(np.float32)
    check_from_spec(lb, S, up, "custom freq")
    check_from_spec(lb, S, up[::-1].copy(), "decreasing freq")


def test_stats_kernel_negative_entry(lb):
    """A negative entry sets STATUS_NEGATIVE_ENTRY (the reference raises); the public function raises."""
    from librosa_b200 import _native as nat
    from librosa_b200.util.exceptions import ParameterError

    S = stats_rows(2, 5, 129, seed=3)
    S[1, 3, 77] = -0.25
    _, status = native_from_spec(lb, S, fft_freq(22050, 256), stats_desc(frame_length=256))
    assert status & nat.STATUS_NEGATIVE_ENTRY
    with pytest.raises(ParameterError, match="non-negative"):
        lb.feature.spectral_centroid(S=np.swapaxes(S, -1, -2), sr=22050)


@pytest.mark.parametrize("F", [b for _, b in STATS_LADDER] + [b + 1 for _, b in STATS_LADDER[:-1]])
def test_stats_kernel_warp_ladder(lb, F):
    """n_bins at each switch of the warp ladder 8 -> 4 -> 2 -> 1 (last of one rung, first of the next), up to the
    largest accepted 29 056."""
    S = stats_rows(2, 5, F, seed=F)
    check_from_spec(lb, S, fft_freq(22050, 2 * (F - 1)), f"F={F}")


def test_stats_kernel_refused_bins(lb):
    """The first n_bins past the ladder is refused, not truncated."""
    from librosa_b200 import _native as nat

    F = STATS_LADDER[-1][1] + 1
    with pytest.raises(nat.UnsupportedOnGPU, match="do not fit"):
        native_from_spec(lb, np.zeros((1, 2, F), np.float32), np.zeros(F, np.float32), stats_desc(frame_length=2 * F))


# ------------------------------------------------------------------ the mixed-radix sizes
@pytest.mark.parametrize("n_fft", mr_sizes())
def test_mixed_radix_sizes(lb, n_fft):
    """mr_kernel<0, G> (stft) and <1, G> (spectrogram), G = 16 up to n_fft 1024 and 32 above: three clips of 37
    frames (the two lane groups of a warp sit in different clips at some boundaries) over the pad modes and powers,
    T = 1, and the scalar-load path (input one float off) against the float2 path, bit for bit."""
    G, w, _ = mr_spectrum_block(n_fft)
    assert G == (16 if n_fft <= 1024 else 32) and w >= 1
    i = mr_sizes().index(n_fft)
    hop = n_fft // 4 + (n_fft // 4) % 2 + 1
    pad_mode = ("constant", "reflect", "edge", "symmetric", "linear_ramp")[i % 5]
    y = signals(3, n_samples(37, n_fft, hop, True), n_fft, seed=n_fft)
    _, X64, ratio = check_stft(lb, y, n_fft, hop, pad_mode=pad_mode)
    print(f"RATIO mr n_fft={n_fft} {ratio:.3f}")
    check_spec(lb, y, n_fft, hop, X64=X64, pad_mode=pad_mode, power=(1.0, 1.5, 2.0)[i % 3])
    y1 = signals(2, hop // 2, n_fft, seed=n_fft + 1)                    # T = 1
    assert check_stft(lb, y1, n_fft, hop)[0].shape[1] == 1
    # float2 loads need an 8-byte aligned base, an even row stride and even frame starts
    center = (n_fft // 2) % 2 == 0
    ev = hop - hop % 2
    y2 = signals(2, n_samples(9, n_fft, ev, center) // 2 * 2, n_fft, seed=n_fft + 2)
    base = native(lb, y2, n_fft, ev, "stft", center=center)
    np.testing.assert_array_equal(native(lb, y2, n_fft, ev, "stft", offset=1, center=center), base)
    np.testing.assert_array_equal(native(lb, y2, n_fft, ev, "stft", offset=2, center=center), base)
