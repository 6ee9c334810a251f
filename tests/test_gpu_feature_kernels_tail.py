"""GPU (-m gpu): the rest of csrc/feat_kernels.cuh — onset_kernel, onset_median_kernel and detrend_kernel (onset
strength), db_kernel / db_clamp_kernel and the float64 db64 pair (power_to_db), unary_kernel (db_to_power,
db_to_amplitude), normalize_rows_kernel (util.normalize inside chroma_stft), pip_pass_kernel (estimate_tuning) and
resample_poly_kernel (resample, pitch_shift, the constant-Q octave pyramid) — at every path and edge, against the
NumPy restatements of tests/feature_tail_restate.py (pinned to the reference in tests/test_feature_tail_host.py).

The tests call the C entries with the descriptors the public functions build, into NaN-filled outputs with guard
words on both sides: every value must come back written and every guard word must still be NaN.  Before each checked
call the same instance runs once on NaN input.

Comparisons (u = 2^-24 for float32, 2^-53 for float64):
    onset mean / median / aggregate=False   bit for bit.  The flux is one float32 subtraction and np.maximum; the
                    mean adds the channel's rows in order and divides once, as NumPy reduces a non-last axis; the
                    median sorts and takes the middle (the float32 mean of the two middles).  A NaN flux (NaN cells,
                    inf - inf) makes its frame NaN on every path, as np.maximum keeps it.  The max filter follows
                    scipy's maximum_filter1d (reflect) on finite and infinite data; a NaN in a window gives NaN, as
                    np.maximum does (scipy's running maximum keeps or drops a NaN by its place in the window, a rule
                    the restatement does not copy).
    detrend         y_t = x_t + z_{t-1}, z_t = 0.99 y_t - x_t in float32, one rounding per operation, against float64
                    lfilter([1, -1], [1, -0.99]) of the kernel's own undetrended output.  Step t commits
                    c_t = u (|y_t| + |z_t| + 0.99 |y_t|) + d |y_t| (the two roundings of z, the product, and the
                    float32 pole 0.99f, off by d = |0.99f - 0.99| = 9.5e-9), and the recurrence damps an error by
                    0.99 per step:  |y_t - y64_t| <= B_t,  B_t = 0.99 B_{t-1} + c_t + u |y_t|, doubled for the
                    second-order terms.
    power_to_db     v = 10 log10f(max(amin, S)) - db_sub (db_sub = 10 log10f(max(amin, |ref|)) formed on the host):
                    log10f is within 2 ulp (CUDA C++ Programming Guide), the product with 10 and the subtraction
                    round once each:  |v - v64| <= 5 u (|10 log10 S| + |db_sub|) + u |v|.  top_db clamps at the
                    clip maximum minus top_db; np.maximum is 1-Lipschitz, so a clamped cell is within the larger of
                    its own bound and the maximum's plus u |floor|.  A NaN cell is NaN, and makes its whole clip NaN
                    under top_db; +inf stays +inf.  The float64 path: the same with u = 2^-53 and 4 ulp for log10.
    db_to_power     ref * powf(10, 0.1 x): the exponent 0.1 x carries 1.25 u relative (the product and the float32
                    0.1f), which 10^(.) turns into ln(10) |0.1 x| 1.25 u; powf 4 ulp, the product with ref 1 u:
                    |p - p64| <= (ln(10) |0.1 x| 1.25 + 9) u p64; db_to_amplitude halves that through sqrtf, plus u.
    normalize       exact for the inf, -inf and 0 norms and for p in {0.5, 1, 2} (NumPy's square root / copy /
                    square shortcuts and the in-order float64 sum round as the kernel does); other p go through
                    float64 pow on both sides (CUDA pow within 2 ulp), which moves the float32 quotient by at most
                    one ulp.
    tuning          exact: every pass histogram equals the one built from the public piptrack's (pitch, mag), and
                    estimate_tuning(S=S) equals pitch_tuning over the peaks at or above their median.  The residual
                    histogram takes log2 correctly rounded, as the kernels do (NumPy's float32 log2 rounds one value
                    in about 150 differently, by CPU), so a peak on a bin edge may land one bin over from where a
                    given CPU's reference puts it.
    resample_poly   float32 fma chain of k taps against float64 upfirdn over the same float32 taps:
                    |y - y64| <= (k + 1) u sum|h x| (+ 2 u |y| for the float32 1 / sqrt(ratio) scale and its product); the zeros of fix_length
                    past n_keep are exactly 0.  The first and last three outputs of each row are checked on their own.

Largest ratio (error / bound) each family saw on an H100 80GB HBM3 at a 700 W power limit:
    detrend 0.14, power_to_db 0.53 (float64 path 0.26), db_to_power 0.71, db_to_amplitude 0.70, resample 0.25,
    normalize 0 (p = 3 and 10 came out bit-identical too); onset and tuning bit for bit.  The whole file runs in
    about 10 s.
"""
import ctypes
import itertools
import math
import warnings

import numpy as np
import pytest
import scipy.signal

import feature_tail_restate as R
from piptrack_oracle import pitch_tuning as pitch_tuning_ref
from test_gpu_mel_front_end import GUARD, device_input, nan_buffer, unguard

pytestmark = [pytest.mark.gpu, pytest.mark.filterwarnings("ignore")]

U = 2.0 ** -24
U64 = 2.0 ** -53
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


def within(name, got, ref, bound, what):
    got = np.asarray(got, np.float64)
    err = np.abs(got - ref)
    same = (got == ref) | (np.isnan(got) & np.isnan(ref))
    ok = same | (err <= bound)
    finite = np.isfinite(ref) & np.isfinite(got)
    if finite.any():
        note(name, (err[finite] / np.maximum(bound[finite] if np.ndim(bound) else bound, 1e-300)).max())
    assert ok.all(), (f"{what}: {int((~ok).sum())} values off, first at {np.argwhere(~ok)[0]}: "
                      f"got {got[~ok][0]!r} want {ref[~ok][0]!r} bound {np.broadcast_to(bound, ref.shape)[~ok][0]:.3e}")


def run_guarded(lb, words, call, what):
    """call(out_ptr) into a NaN-filled float32 buffer with GUARD words on each side; returns the unguarded words."""
    buf = nan_buffer(lb, words + 2 * GUARD)
    call(buf.ptr + 4 * GUARD)
    host = buf.get()
    buf.free()
    return unguard(host, what)


# ------------------------------------------------------------------ onset strength
def onset_native(lb, S, *, lag, max_size, pad_width, bounds=None, median=False, detrend=False):
    """b2l_onset_from_spec / b2l_onset_median_from_spec on float32 S [n_clips, rows, T] -> [n_clips, n_out, T],
    after the same call on NaN input."""
    ctx, L, nat = ctx_lib(lb)
    n_clips, rows, T = S.shape
    desc = nat.OnsetDesc(lag=lag, max_size=max_size, detrend=int(detrend), pad_width=pad_width)
    if bounds is not None:
        desc.n_channels = len(bounds) - 1
        for i, b in enumerate(bounds):
            desc.bounds[i] = b
    n_out = rows if bounds is None else len(bounds) - 1
    entry = L.b2l_onset_median_from_spec if median else L.b2l_onset_from_spec
    what = f"onset lag={lag} max_size={max_size} pad={pad_width} T={T} bounds={bounds} median={median}"
    res = None
    for data in (np.full_like(S, np.nan), S):
        din = device_input(lb, data, 0)
        host = run_guarded(lb, n_clips * n_out * T, lambda p: nat.check(
            entry(ctx.handle, ctypes.byref(desc), vp(din.ptr), n_clips, rows, T, vp(p))), what)
        din.free()
        res = host.reshape(n_clips, n_out, T)
    return res


def onset_input(rng, n_clips, rows, T, special):
    """dB-like values on a 0.5 grid (ties), with -inf, +inf and NaN cells when `special`."""
    S = (np.round(rng.uniform(-80, 0, (n_clips, rows, T)) * 2) / 2).astype(np.float32)
    if special:
        for v, frac in ((-np.inf, 0.08), (np.inf, 0.03), (np.nan, 0.03)):
            S[rng.random(S.shape) < frac] = v
    return S


def channel_layouts(rows):
    """aggregate=False, one channel over every row, one-row channels with an empty one, and 32 channels."""
    layouts = [None, [0, rows], [0, 1, 1, min(2, rows)]]
    cuts = np.sort(np.random.default_rng(rows).integers(0, rows + 1, 31))
    layouts.append([0] + [int(c) for c in cuts] + [rows])
    return layouts


ONSET_T = [1, 15, 16, 17, 33]


@pytest.mark.parametrize("T", ONSET_T)
@pytest.mark.parametrize("median", [False, True], ids=["mean", "median"])
def test_onset_paths_bit_exact(lb, T, median):
    rng = np.random.default_rng(T + 100 * median)
    rows = 9
    n = 0
    for lag in sorted({1, 2, 7, max(1, T - 1)}):
        for max_size in (1, 2, 3, 4, rows + 3):
            for pad in sorted({0, lag, lag + 2, T + 1}):
                for bounds in channel_layouts(rows):
                    if median and bounds is None:
                        continue
                    n += 1
                    S = onset_input(rng, 3, rows, T, special=n % 2 == 0)
                    got = onset_native(lb, S, lag=lag, max_size=max_size, pad_width=pad, bounds=bounds, median=median)
                    want = R.onset_envelope(S, lag=lag, max_size=max_size, pad_width=pad, bounds=bounds, median=median)
                    np.testing.assert_array_equal(got, want, err_msg=f"lag={lag} max_size={max_size} pad={pad} "
                                                                     f"bounds={bounds} T={T}")


@pytest.mark.parametrize("width", [1, 31, 32, 33, 63, 64, 65, 511, 512])
def test_onset_median_every_rung(lb, width):
    rng = np.random.default_rng(width)
    rows = width + 2
    S = onset_input(rng, 2, rows, 17, special=False)
    S[0, :, 5] = np.nan                       # one NaN cell per frame 5 of clip 0
    for bounds in ([0, width, rows], [0, 1, 1 + width if width < rows - 1 else rows, rows]):
        got = onset_native(lb, S, lag=1, max_size=1, pad_width=3, bounds=bounds, median=True)
        want = R.onset_envelope(S, lag=1, max_size=1, pad_width=3, bounds=bounds, median=True)
        np.testing.assert_array_equal(got, want, err_msg=f"width={width} bounds={bounds}")


def test_onset_refusals(lb):
    ctx, L, nat = ctx_lib(lb)
    S = np.zeros((1, 513, 4), np.float32)
    din = device_input(lb, S, 0)
    out = nan_buffer(lb, 513 * 4)
    desc = nat.OnsetDesc(lag=1, max_size=1, pad_width=1, n_channels=1)
    desc.bounds[0], desc.bounds[1] = 0, 513
    assert L.b2l_onset_median_from_spec(ctx.handle, ctypes.byref(desc), vp(din.ptr), 1, 513, 4, vp(out.ptr)) != 0
    desc.bounds[1] = 512
    assert L.b2l_onset_median_from_spec(ctx.handle, ctypes.byref(desc), vp(din.ptr), 1, 513, 4, vp(out.ptr)) == 0
    desc.n_channels = 33
    for entry in (L.b2l_onset_from_spec, L.b2l_onset_median_from_spec):
        assert entry(ctx.handle, ctypes.byref(desc), vp(din.ptr), 1, 513, 4, vp(out.ptr)) != 0
    din.free()
    out.free()


def test_onset_many_clips(lb):
    """More than 65 535 clips in one call: each clip's envelope stays its own."""
    rng = np.random.default_rng(7)
    S = onset_input(rng, 70000, 3, 4, special=False)
    S[69999, :, 3] = np.nan
    for median in (False, True):
        got = onset_native(lb, S, lag=1, max_size=2, pad_width=1, bounds=[0, 3], median=median)
        want = R.onset_envelope(S, lag=1, max_size=2, pad_width=1, bounds=[0, 3], median=median)
        np.testing.assert_array_equal(got, want)


def detrend_bound(x, y64):
    """B_t of the module docstring over a float64 row y64 (the float64 lfilter output) of input x."""
    d = abs(float(np.float32(0.99)) - 0.99)
    z = 0.99 * y64 - x
    B = np.empty_like(y64)
    b = 0.0
    for t in range(len(y64)):
        b = 0.99 * b + U * (2.99 * abs(y64[t]) + abs(z[t])) + d * abs(y64[t])
        B[t] = b
    return 2.0 * B + 1e-300


@pytest.mark.parametrize("median", [False, True], ids=["mean", "median"])
def test_onset_detrend_bound(lb, median):
    rng = np.random.default_rng(11)
    S = onset_input(rng, 3, 40, 700, special=False)
    kw = dict(lag=2, max_size=3, pad_width=5, bounds=[0, 10, 40], median=median)
    raw = onset_native(lb, S, **kw)
    got = onset_native(lb, S, detrend=True, **kw)
    for c in range(3):
        for ch in range(2):
            y64 = scipy.signal.lfilter([1.0, -1.0], [1.0, -0.99], raw[c, ch].astype(np.float64))
            within("detrend", got[c, ch], y64, detrend_bound(raw[c, ch].astype(np.float64), y64), f"detrend {c} {ch}")


def test_onset_public_nan_propagates(lb):
    """onset_strength(S=log(power)) with silent cells: -inf - -inf is NaN, which np.maximum keeps."""
    rng = np.random.default_rng(3)
    P = rng.uniform(0, 1, (16, 30)).astype(np.float32)
    P[:, 10:13] = 0.0
    with np.errstate(divide="ignore"):
        S = np.log(P)
    for agg in (np.mean, np.median):
        got = lb.onset.onset_strength(S=S, aggregate=agg)
        want = R.onset_envelope(S[None], lag=1, max_size=1, pad_width=1 + 2048 // 1024, bounds=[0, 16],
                                median=agg is np.median)[0, 0]
        np.testing.assert_array_equal(got, want)
        assert np.isnan(got).any()


# ------------------------------------------------------------------ power_to_db and its inverses
def db_native(lb, S, *, amin, ref_value, top_db):
    ctx, L, nat = ctx_lib(lb)
    n_clips, per = S.shape
    res = None
    for data in (np.full_like(S, np.nan), S):
        din = device_input(lb, data, 0)
        res = run_guarded(lb, n_clips * per, lambda p: nat.check(L.b2l_power_to_db(
            ctx.handle, vp(din.ptr), n_clips, per, amin, ref_value, -1.0 if top_db is None else top_db, vp(p))),
            f"power_to_db {S.shape}").reshape(S.shape)
        din.free()
    return res


def db_ref(S, *, amin, ref_value, top_db, u=U, log_ulps=2):
    """float64 dB and its bound per cell (module docstring)."""
    S = np.asarray(S, np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        L10 = 10.0 * np.log10(np.maximum(amin, S))
        sub = 10.0 * np.log10(max(amin, abs(ref_value)))
        v = L10 - sub
        k = 2 * log_ulps + 1
        bound = k * u * (np.abs(L10) + abs(sub)) + u * np.abs(v)
        if top_db is not None:
            mx = v.max(axis=-1, keepdims=True)
            floor = mx - top_db
            ib = np.argmax(np.where(np.isnan(v), -np.inf, v), axis=-1)[:, None]
            fb = np.take_along_axis(bound, ib, axis=-1) + u * np.abs(floor)
            v = np.maximum(v, floor)
            bound = np.maximum(bound, np.nan_to_num(fb, nan=0.0, posinf=0.0))
    return v, bound


DB_CASES = [
    dict(name="plain", top_db=None, ref=1.0),
    dict(name="top80", top_db=80.0, ref=1.0),
    dict(name="top0", top_db=0.0, ref=1.0),
    dict(name="ref_ne_1", top_db=80.0, ref=3.7),
]


@pytest.mark.parametrize("case", DB_CASES, ids=lambda c: c["name"])
@pytest.mark.parametrize("per_clip", [1, 7, 2049, 256 * 8 * 3 + 5])
def test_power_to_db_kernel(lb, case, per_clip):
    rng = np.random.default_rng(per_clip)
    amin = float(np.float32(1e-10))
    S = (10.0 ** rng.uniform(-14, 3, (5, per_clip))).astype(np.float32)
    S[1] = 1e-12                                              # a clip entirely below amin
    S[2, per_clip // 2] = np.nan                              # a NaN cell
    S[3, -1] = np.inf                                         # +inf
    S[4, 0] = 0.0
    got = db_native(lb, S, amin=amin, ref_value=case["ref"], top_db=case["top_db"])
    want, bound = db_ref(S, amin=amin, ref_value=case["ref"], top_db=case["top_db"])
    within("power_to_db", got, want, bound, f"power_to_db {case} per_clip={per_clip}")
    if case["top_db"] is not None:
        assert np.isnan(got[2]).all() and np.isinf(got[3]).all(), "a NaN / +inf maximum must reach the whole clip"
    else:
        assert np.isnan(got[2]).sum() == 1


def test_power_to_db_many_clips(lb):
    rng = np.random.default_rng(5)
    S = rng.uniform(1e-6, 1.0, (70000, 3)).astype(np.float32)
    S[66000, 1] = np.nan
    got = db_native(lb, S, amin=1e-10, ref_value=1.0, top_db=10.0)
    want, bound = db_ref(S, amin=1e-10, ref_value=1.0, top_db=10.0)
    within("power_to_db", got, want, bound, "power_to_db 70000 clips")
    assert np.isnan(got[66000]).all() and not np.isnan(np.delete(got, 66000, axis=0)).any()


@pytest.mark.parametrize("top_db", [None, 80.0])
def test_power_to_db_public_nan(lb, top_db):
    """float32 and float64 host input: a NaN cell is NaN, and under top_db the whole clip is NaN."""
    S = np.abs(np.random.default_rng(1).standard_normal((2, 6, 9)))
    S[1, 2, 3] = np.nan
    for dt, u, ulps in ((np.float32, U, 2), (np.float64, U64, 4)):
        got = np.asarray(lb.power_to_db(S.astype(dt), top_db=top_db))
        want, bound = db_ref(S.astype(dt).reshape(2, -1), amin=1e-10, ref_value=1.0, top_db=top_db, u=u, log_ulps=ulps)
        within("power_to_db64" if dt == np.float64 else "power_to_db", got.reshape(2, -1), want, bound,
               f"power_to_db {dt.__name__} top_db={top_db}")
        assert np.isnan(got[1]).all() == (top_db is not None) and np.isnan(got[1]).any()


@pytest.mark.parametrize("op", ["power", "amplitude"])
def test_db_inverse_unary(lb, op):
    ctx, L, nat = ctx_lib(lb)
    rng = np.random.default_rng(2)
    x = rng.uniform(-120, 40, 5000).astype(np.float32)
    ref = 2.5
    param = ref if op == "power" else ref * ref
    code = nat.UNARY_DB_TO_POWER if op == "power" else nat.UNARY_DB_TO_AMPLITUDE
    din = device_input(lb, x, 0)
    got = run_guarded(lb, x.size, lambda p: nat.check(L.b2l_unary(ctx.handle, code, vp(din.ptr), x.size, param, vp(p))),
                      f"unary {op}")
    din.free()
    x64 = x.astype(np.float64)
    p64 = param * 10.0 ** (0.1 * x64)
    rel = (math.log(10) * np.abs(0.1 * x64) * 1.25 + 9) * U
    if op == "amplitude":
        p64, rel = np.sqrt(p64), rel / 2 + U
    within("db_to_" + op, got, p64, rel * p64, f"db_to_{op}")


# ------------------------------------------------------------------ util.normalize (chroma_stft(norm=...))
NORMS = [(np.inf, 0, 0.0), (-np.inf, 1, 0.0), (0, 2, 0.0), (0.5, 3, 0.5), (1, 3, 1.0), (2, 3, 2.0), (3, 3, 3.0),
         (10, 3, 10.0)]


def normalize_native(lb, S, kind, p):
    ctx, L, nat = ctx_lib(lb)
    n_clips, rows, T = S.shape
    res = None
    for data in (np.full_like(S, np.nan), S):
        din = device_input(lb, data, 0)
        res = run_guarded(lb, S.size, lambda q: nat.check(L.b2l_normalize_rows(
            ctx.handle, vp(din.ptr), n_clips, rows, T, kind, p, vp(q))), f"normalize {S.shape} {kind} {p}")
        din.free()
    return res.reshape(S.shape)


def normalize_input(rng, n_clips, rows, T):
    """Columns at magnitudes from 1e-25 to 1e20, negative values, zero columns and a column around 1e-23."""
    scale = 10.0 ** rng.uniform(-25, 20, (n_clips, 1, T))
    S = (rng.uniform(-1, 1, (n_clips, rows, T)) * scale).astype(np.float32)
    S[:, :, 0] = 0.0
    if T > 2:
        S[:, :, 1] = np.float32(1e-23) * rng.uniform(0.5, 1.5, (n_clips, rows))
        S[:, :, 2] = np.float32(1e5) * rng.uniform(0.5, 1.5, (n_clips, rows))
    S[:, rows // 2, T // 2] = 0.0
    return S


@pytest.mark.parametrize("rows", [1, 12, 24, 84])
@pytest.mark.parametrize("T", [3, 127, 128, 129, 300])
def test_normalize_rows(lb, rows, T):
    rng = np.random.default_rng(rows * 1000 + T)
    S = normalize_input(rng, 2, rows, T)
    for norm, kind, p in NORMS:
        got = normalize_native(lb, S, kind, p)
        want = R.normalize(S, norm)
        if norm in (np.inf, -np.inf, 0, 0.5, 1, 2):
            np.testing.assert_array_equal(got, want, err_msg=f"norm={norm} rows={rows} T={T}")
            continue
        ulp = np.spacing(np.abs(want).astype(np.float32)).astype(np.float64)
        within("normalize", got, want.astype(np.float64), ulp, f"norm={norm} rows={rows} T={T}")


def test_normalize_many_clips(lb):
    S = normalize_input(np.random.default_rng(9), 70000, 2, 3)
    np.testing.assert_array_equal(normalize_native(lb, S, 3, 2.0), R.normalize(S, 2))


@pytest.mark.parametrize("norm", [1, 2, 10, np.inf])
def test_chroma_norm_public(lb, norm):
    """chroma_stft(S=, norm=p) is util.normalize of the unnormalised chroma, at full-scale and tiny levels."""
    rng = np.random.default_rng(4)
    S = rng.uniform(0, 1, (1025, 20)).astype(np.float32)
    S[:, :10] *= np.float32(1e6)
    S[:, 10:14] *= np.float32(1e-22)
    raw = np.asarray(lb.feature.chroma_stft(S=S, sr=22050, tuning=0.0, norm=None))
    got = np.asarray(lb.feature.chroma_stft(S=S, sr=22050, tuning=0.0, norm=norm))
    want = R.normalize(raw, norm)
    ulp = np.spacing(np.abs(want)).astype(np.float64)
    within("normalize", got, want.astype(np.float64), ulp if norm == 10 else 0.0 * ulp, f"chroma norm={norm}")


# ------------------------------------------------------------------ tuning (estimate_tuning's passes)
def tuning_spectrum(kind, F=1025, T=40, seed=0):
    rng = np.random.default_rng(seed)
    S = rng.uniform(0, 1, (F, T)).astype(np.float32)
    if kind == "ties":
        S = np.round(S * 4) / 4
    elif kind == "edges":
        S[-1] = 3.0                                         # peaks at k = F - 1
        S[-2] = 1.0
        S[1] = 2.5                                          # a peak at k = 1
        S[0] = 0.1
        S[200, :] = S[201, :] = 2.0                         # flat tops
        mx = S.max(axis=0)
        S[300] = np.float32(0.1) * mx                       # exactly at threshold * max
        S[299] = S[301] = 0.0
    elif kind == "nan_frame":
        S[:, 7] = np.nan
    elif kind == "silent":
        S[:] = 0.0
    return S.astype(np.float32)


def pip_native(lb, S, *, sr, n_fft, fmin, fmax, threshold, ref, mode, prefix=0, mag_threshold=0.0, edges=None,
               bins_per_octave=12):
    from librosa_b200.core import pitch as P

    ctx, L, nat = ctx_lib(lb)
    F, T = S.shape[-2:]
    freqs = np.fft.rfftfreq(n_fft, 1.0 / sr)
    mask = np.flatnonzero((max(fmin, 0) <= freqs) & (freqs < min(fmax, sr / 2)))
    ref_frame, thr, thr_wide, ref_abs = P._pip_reference(threshold, ref, np.dtype(np.float32))
    desc = nat.PipDesc(k_lo=int(mask[0]) if mask.size else 0, k_hi=int(mask[-1]) + 1 if mask.size else 0,
                       threshold=thr, thr_wide=thr_wide, ref_abs=-1.0 if ref_frame else ref_abs, sr=float(sr),
                       n_fft=float(n_fft), bins_per_octave=float(bins_per_octave), mode=mode, prefix=prefix,
                       mag_threshold=float(mag_threshold), n_res_bins=0 if edges is None else len(edges) - 1)
    rows = np.ascontiguousarray(np.swapaxes(S, -1, -2)).reshape(-1, F)   # one row per frame, bins contiguous
    hist = (ctypes.c_uint64 * 2048)()
    e = None if edges is None else np.ascontiguousarray(edges, np.float64)
    for data in (np.full_like(rows, np.nan), rows):
        din = device_input(lb, data, 0)
        nat.check(L.b2l_pip_pass(ctx.handle, ctypes.byref(desc), vp(din.ptr), rows.shape[0], F,
                                 None if e is None else e.ctypes.data_as(vp), hist))
        din.free()
    n = desc.n_res_bins if mode == 3 else (1024 if mode == 2 else 2048)
    return np.frombuffer(hist, np.uint64, count=n).astype(np.int64)


TUNING_CASES = [
    dict(kind="random", fmin=150.0, fmax=4000.0, threshold=0.1, ref=None),
    dict(kind="ties", fmin=150.0, fmax=4000.0, threshold=0.1, ref=None),
    dict(kind="edges", fmin=0.0, fmax=1e9, threshold=0.1, ref=None),               # k_lo = 0, k = F - 1
    dict(kind="edges", fmin=10.0, fmax=1e9, threshold=np.float64(0.1), ref=None),  # k_lo = 1, float64 threshold
    dict(kind="nan_frame", fmin=150.0, fmax=4000.0, threshold=0.1, ref=None),
    dict(kind="random", fmin=150.0, fmax=4000.0, threshold=0.1, ref=0.55),          # ref as a number
    dict(kind="silent", fmin=150.0, fmax=4000.0, threshold=0.1, ref=None),
    dict(kind="random", fmin=0.0, fmax=1e9, threshold=0.2, ref=None, F=8001),       # under 8 warps per block
]


@pytest.mark.parametrize("case", TUNING_CASES, ids=lambda c: f"{c['kind']}-{c.get('F', 1025)}-{c['fmin']}-{c['ref']}")
def test_tuning_passes_match_piptrack(lb, case):
    F = case.get("F", 1025)
    sr, n_fft = 22050, 2 * (F - 1) + 1          # odd: the last bin lies below sr / 2, inside fmax
    S = tuning_spectrum(case["kind"], F=F)
    kw = dict(sr=sr, n_fft=n_fft, fmin=case["fmin"], fmax=case["fmax"], threshold=case["threshold"], ref=case["ref"])
    pitch, mag = lb.piptrack(S=S, **kw)
    pitch, mag = np.asarray(pitch), np.asarray(mag)
    sel = pitch > 0
    med = np.median(mag[sel]) if sel.any() else np.float32(0)
    k = int(R.float_keys(np.float32(med))[()]) if sel.any() else 0
    edges = np.linspace(-0.5, 0.5, 101)
    want = R.tuning_histograms(pitch, mag, prefix0=k >> 21, prefix1=k >> 10, mag_threshold=med, bins_per_octave=12,
                               edges=edges)
    got = [pip_native(lb, S, mode=0, **kw), pip_native(lb, S, mode=1, prefix=k >> 21, **kw),
           pip_native(lb, S, mode=2, prefix=k >> 10, **kw), pip_native(lb, S, mode=3, mag_threshold=med, edges=edges, **kw)]
    for m, (g, w) in enumerate(zip(got, want)):
        np.testing.assert_array_equal(g, w, err_msg=f"pass {m} {case}")


@pytest.mark.parametrize("case", [c for c in TUNING_CASES if c["kind"] != "nan_frame"],
                         ids=lambda c: f"{c['kind']}-{c.get('F', 1025)}-{c['fmin']}-{c['ref']}")
@pytest.mark.parametrize("resolution", [0.01, 0.001])
def test_estimate_tuning_matches_piptrack(lb, case, resolution):
    """estimate_tuning(S=S) is pitch_tuning over the public piptrack's peaks at or above their median."""
    F = case.get("F", 1025)
    S = tuning_spectrum(case["kind"], F=F, seed=1)
    kw = dict(sr=22050, n_fft=2 * (F - 1) + 1, fmin=case["fmin"], fmax=case["fmax"], threshold=case["threshold"],
              ref=case["ref"])
    pitch, mag = (np.asarray(v) for v in lb.piptrack(S=S, **kw))
    sel = pitch > 0
    med = np.median(mag[sel]) if sel.any() else 0.0
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        est = lb.estimate_tuning(S=S, resolution=resolution, **kw)
        want = pitch_tuning_ref(pitch[(mag >= med) & sel], resolution=resolution)
    assert est == want, (est, want)


# ------------------------------------------------------------------ polyphase resampling
RATES = [(5, 2), (2, 7), (160, 147), (441, 80), (1, 6)]


def resample_native(lb, x, stride, h, up, down, n_pre_remove, n_keep, n_total, scale):
    ctx, L, nat = ctx_lib(lb)
    n_clips, n = x.shape
    X = np.zeros((n_clips, stride), np.float32)
    X[:, :n] = x
    d_h = device_input(lb, h, 0)
    res = None
    for data in (np.full_like(X, np.nan), X):
        din = device_input(lb, data, 0)
        res = run_guarded(lb, n_clips * n_total, lambda p: nat.check(L.b2l_resample_poly(
            ctx.handle, vp(din.ptr), n_clips, n, stride, vp(d_h.ptr), len(h), up, down, n_pre_remove, n_keep, n_total,
            scale, vp(p))), f"resample {up}/{down} n={n}")
        din.free()
    d_h.free()
    return res.reshape(n_clips, n_total)


@pytest.mark.parametrize("up,down", RATES)
def test_resample_poly(lb, up, down):
    from librosa_b200.core.audio import _poly_filter

    h, n_pre_remove = _poly_filter(up, down)
    k = -(-len(h) // up) + 1
    rng = np.random.default_rng(up * 1000 + down)
    half = len(h) // up // 2
    for n, fix, extra, stride_pad in itertools.product((1, max(2, half // 2), 1000), (True, False), (0, 37), (0, 5)):
        n_out = (n * up + down - 1) // down
        n_total = (int(np.ceil(n * up / down)) + extra) if fix else n_out
        n_keep = min(n_out, n_total)
        scale = float(1.0 / np.sqrt(up / down)) if extra else 1.0
        x = rng.uniform(-1, 1, (3, n)).astype(np.float32)
        got = resample_native(lb, x, n + stride_pad, h, up, down, n_pre_remove, n_keep, n_total, np.float32(scale))
        y64, scale64 = R.resample_poly64(x, h, up, down, n_pre_remove, n_keep, n_total)
        bound = (k + 1) * U * scale64 * scale + 2 * U * np.abs(y64 * scale)
        what = f"resample {up}/{down} n={n} fix={fix} n_keep={n_keep} n_total={n_total} stride+{stride_pad}"
        assert (got[:, n_keep:] == 0).all(), f"{what}: the fix_length tail must be exactly zero"
        e = min(3, n_keep)
        within("resample", got[:, :e], y64[:, :e] * scale, bound[:, :e], what + " (first three)")
        within("resample", got[:, n_keep - e:n_keep], y64[:, n_keep - e:n_keep] * scale,
               bound[:, n_keep - e:n_keep], what + " (last three)")
        within("resample", got, y64 * scale, bound, what)
