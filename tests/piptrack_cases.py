"""Case table of piptrack, pitch_tuning and util.localmax / localmin: tests/golden/piptrack_v1.npz holds, for each case,
what the unmodified reference returns or the exception it raises (``<name>/error``, "Class: message").  Written by
tools/make_golden.py --piptrack; tests/piptrack_oracle.py must reproduce every entry bit for bit.

piptrack results are stored sparsely: ``<name>/shape``, ``<name>/dtype``, the flat indices ``<name>/idx`` where
pitches or mags are non-zero (NaN included) and the values ``<name>/p`` and ``<name>/m`` there; a case from ``y`` also
stores the reference's magnitude spectrogram ``<name>/S``, from which the oracle reproduces it.  pitch_tuning stores
``<name>/out`` (the tuning, float64), localmax / localmin ``<name>/out`` (bool).  A case's data is made from its
spec (seeded), so nothing but the outputs is stored.  ``refuse`` names the cases the GPU declines with
UnsupportedOnGPU although the reference runs them; nothing is stored for them."""
from __future__ import annotations

import numpy as np

SR = 22050


def signal(spec):
    """spec = (shape, seed[, dtype]): a few harmonic tones with vibrato plus noise, float32 unless given."""
    shape, seed = spec[:2]
    dtype = np.dtype(spec[2]) if len(spec) > 2 else np.dtype(np.float32)
    rng = np.random.default_rng(seed)
    n = shape[-1]
    t = np.arange(n) / SR
    lead = shape[:-1]
    y = 0.05 * rng.standard_normal(shape)
    for _ in range(3):
        f0 = rng.uniform(110.0, 880.0, size=lead + (1,))
        phase = 2 * np.pi * f0 * t + 0.3 * np.sin(2 * np.pi * 5.0 * t)
        for h in range(1, 5):
            y = y + (0.3 / h) * np.sin(h * phase + rng.uniform(0, 2 * np.pi, size=lead + (1,)))
    return y.astype(dtype)


def spectrum(spec):
    """spec = (shape, dtype, seed[, specials]): |normal| for real dtypes ("signed" in the dtype's place gives float32
    with its signs kept), a complex normal for complex dtypes; specials ((index, value), ...) written after."""
    shape, dtype, seed = spec[:3]
    rng = np.random.default_rng(seed)
    if dtype == "signed":
        x = rng.standard_normal(shape).astype(np.float32)
    elif dtype == "signed64":
        x = rng.standard_normal(shape)
    else:
        dtype = np.dtype(dtype)
        if dtype.kind == "c":
            x = (rng.standard_normal(shape) + 1j * rng.standard_normal(shape)).astype(dtype)
        else:
            x = np.abs(rng.standard_normal(shape)).astype(dtype)
    for idx, v in (spec[3] if len(spec) > 3 else ()):
        x[idx] = v
    return x


def values(spec):
    """spec = (shape, dtype, seed[, specials]) for pitch_tuning and localmax: frequencies in 20 .. 5000 Hz (with a
    share of non-positive values) for floats; small integers (plateaus) for the peak test."""
    shape, dtype, seed = spec[:3]
    rng = np.random.default_rng(seed)
    dtype = np.dtype(dtype)
    if dtype.kind == "b":
        x = rng.integers(0, 2, size=shape).astype(bool)
    elif dtype.kind in "iu":
        x = rng.integers(0 if dtype.kind == "u" else -3, 4, size=shape).astype(dtype)
    else:
        x = np.exp(rng.uniform(np.log(20.0), np.log(5000.0), size=shape)).astype(dtype)
        x[rng.random(shape) < 0.1] = 0
    for idx, v in (spec[3] if len(spec) > 3 else ()):
        x[idx] = v
    return x


def _p(name, refuse=False, y=None, S=None, **kw):
    return {"name": name, "fn": "piptrack", "y": y, "S": S, "kw": kw, "refuse": refuse}


def _t(name, spec, refuse=False, **kw):
    return {"name": name, "fn": "pitch_tuning", "spec": spec, "kw": kw, "refuse": refuse}


def _l(name, fn, spec, refuse=False, **kw):
    return {"name": name, "fn": fn, "spec": spec, "kw": kw, "refuse": refuse}


Y = ((4096,), 1)
S32 = ((257, 24), np.float32, 2)
CASES = [
    # from y: three frame lengths (1024 is a power of two, 400 mixed radix), hops, centring, channels
    _p("y_default", y=Y),
    _p("y_1024_hop256", y=Y, n_fft=1024, hop_length=256),
    _p("y_400_hop100", y=((4000,), 3), n_fft=400, hop_length=100, fmin=50.0),
    _p("y_400_hop160_uncentered", y=((4000,), 4), n_fft=400, hop_length=160, center=False),
    _p("y_2048_hop333_uncentered", y=((6000,), 5), hop_length=333, center=False, fmax=8000.0),
    _p("y_1024_reflect", y=((3000,), 6), n_fft=1024, pad_mode="reflect", threshold=0.05),
    _p("y_multichannel", y=((2, 4096), 7), n_fft=1024, hop_length=512),
    _p("y_multichannel_3d", y=((2, 2, 2000), 8), n_fft=400, hop_length=200),
    _p("y_float64", y=((3000,), 9, np.float64), n_fft=1024),
    # from S: dtypes, complex, negative entries, n_fft inference
    _p("S_f32", S=S32),
    _p("S_f64", S=((257, 24), np.float64, 3)),
    _p("S_complex64", S=((129, 16), np.complex64, 4)),
    _p("S_complex128", S=((129, 16), np.complex128, 5)),
    _p("S_signed", S=((257, 20), "signed", 6)),
    _p("S_signed64", S=((129, 20), "signed64", 7)),
    _p("S_nfft_none", S=S32, n_fft=None),
    _p("S_nfft_kept", S=S32, n_fft=513),
    _p("S_nfft_mismatch", S=S32, n_fft=2048),
    _p("S_multichannel", S=((2, 3, 129, 10), np.float32, 8)),
    _p("S_sr16k", S=S32, sr=16000),
    _p("S_two_bins", S=((2, 30), np.float32, 9), fmin=0.0),
    # the float64 stencil: many interior peaks of a float32 spectrogram
    _p("S_f32_wide", S=((1025, 40), np.float32, 10), fmin=0.0, fmax=11025.0, threshold=0.0),
    # NaN and infinities
    _p("S_nan", S=((129, 12), np.float32, 11, (((20, 3), np.nan), ((40, 5), np.nan)))),
    _p("S_nan_signed", S=((129, 12), "signed", 12, (((20, 3), np.nan),))),
    _p("S_inf", S=((129, 12), np.float32, 13, (((20, 3), np.inf), ((60, 7), np.inf), ((128, 8), np.inf)))),
    _p("S_neg_inf", S=((129, 12), np.float32, 14, (((30, 2), -np.inf), ((31, 9), np.inf)))),
    _p("S_inf_f64_ref", S=((129, 12), np.float64, 15, (((20, 3), np.inf),)), ref=0.5),
    _p("S_nan_ref", S=((129, 12), np.float32, 16, (((50, 4), np.nan),)), ref=1.0),
    # the reference value and the threshold
    _p("S_ref_max", S=S32, ref=np.max),
    _p("S_ref_number", S=S32, ref=0.8),
    _p("S_ref_negative", S=S32, ref=-1.2),
    _p("S_ref_zero", S=S32, ref=0),
    _p("S_ref_f32", S=S32, ref=np.float32(0.7)),
    _p("S_threshold_0", S=S32, threshold=0.0),
    _p("S_threshold_1", S=S32, threshold=1.0),
    _p("S_threshold_f64", S=S32, threshold=np.float64(0.3)),
    _p("S_fmin_0", S=S32, fmin=0.0),
    _p("S_fmax_above_nyquist", S=S32, fmax=30000.0, fmin=0.0),
    _p("S_empty_band", S=S32, fmin=9000.0, fmax=100.0),
    # errors the reference raises
    _p("err_no_input"),
    _p("err_nfft_none_y", y=Y, n_fft=None),
    _p("err_S_1d", S=((30,), np.float32, 1)),
    _p("err_S_no_frames", S=((129, 0), np.float32, 1)),
    _p("err_S_one_bin", S=((1, 10), np.float32, 1)),
    _p("err_S_one_bin_nfft", S=((1, 10), np.float32, 1), n_fft=1),
    _p("err_hop", y=Y, hop_length=0),
    _p("err_y_int", y=((100,), 1, np.int16)),
    _p("err_uncentered_short", y=((1000,), 1), center=False),
    _p("err_pad_mode", y=((4000,), 1), pad_mode="wrap"),
    # refusals
    _p("refuse_ref_mean", S=S32, ref=np.mean, refuse=True),
]

F32 = ((500,), np.float32, 20)
CASES += [
    _t("tuning_empty", ((0,), np.float32, 21)),
    _t("tuning_nonpositive", ((5,), np.float32, 22, ((slice(None), -1.0),))),
    _t("tuning_zeros", ((5,), np.float64, 23, ((slice(None), 0.0),))),
    _t("tuning_f32", F32), _t("tuning_f64", ((500,), np.float64, 24)),
    _t("tuning_2d", ((20, 30), np.float32, 25)), _t("tuning_3d", ((3, 4, 50), np.float64, 26)),
    _t("tuning_res_third", F32, resolution=1 / 3), _t("tuning_res_2048", ((4000,), np.float32, 27), resolution=1 / 2048),
    _t("tuning_res_2048_f64", ((4000,), np.float64, 28), resolution=1 / 2048),
    _t("tuning_bpo24", F32, bins_per_octave=24), _t("tuning_bpo36", ((500,), np.float64, 29), bins_per_octave=36),
    _t("tuning_nonfinite", ((200,), np.float32, 30, ((3, np.inf), (4, np.nan), (5, -np.inf)))),
    _t("tuning_on_pitch", ((1000,), np.float32, 31, ((slice(0, 500), 440.0 * 2 ** (0.23 / 12)),))),
    _t("tuning_scalar_like", ((1,), np.float64, 32, ((0, 445.0),))),
    _t("err_tuning_resolution_zero", F32, resolution=0),
    _t("tuning_resolution_zero_empty", ((3,), np.float32, 33, ((slice(None), 0.0),)), resolution=0),
    _t("refuse_tuning_res_4096", F32, resolution=1 / 4096, refuse=True),
]

DTYPES = (np.int8, np.uint8, np.int16, np.uint16, np.int32, np.uint32, np.int64, np.uint64, np.float32, np.float64,
          bool)
for _fn in ("localmax", "localmin"):
    for _i, _dt in enumerate(DTYPES):
        _name = np.dtype(_dt).name
        CASES.append(_l(f"{_fn}_{_name}_2d_axis0", _fn, ((9, 6), _dt, 40 + _i)))
        CASES.append(_l(f"{_fn}_{_name}_2d_axis1", _fn, ((5, 11), _dt, 60 + _i), axis=1))
    CASES += [
        _l(f"{_fn}_1d", _fn, ((40,), np.float32, 80)),
        _l(f"{_fn}_1d_example", _fn, ((8,), np.int64, 81, ((slice(None), np.array([1, 0, 1, 2, -1, 0, -2, 1])),))),
        _l(f"{_fn}_3d_axis1", _fn, ((3, 7, 5), np.int32, 82), axis=1),
        _l(f"{_fn}_3d_axis_m1", _fn, ((3, 4, 9), np.float64, 83), axis=-1),
        _l(f"{_fn}_4d_axis2", _fn, ((2, 3, 6, 4), np.int16, 84), axis=2),
        _l(f"{_fn}_4d_axis0", _fn, ((5, 2, 3, 4), np.float32, 85), axis=0),
        _l(f"{_fn}_4d_axis_m2", _fn, ((2, 3, 6, 5), np.uint8, 86), axis=-2),
        _l(f"{_fn}_len2", _fn, ((2, 5), np.float32, 87)), _l(f"{_fn}_len3", _fn, ((3, 5), np.int8, 88)),
        _l(f"{_fn}_len2_axis1", _fn, ((4, 2), np.float64, 89), axis=1),
        _l(f"{_fn}_plateau", _fn, ((12,), np.float32, 90, ((slice(2, 5), 3.0), (slice(7, 10), -1.0)))),
        _l(f"{_fn}_nan", _fn, ((12, 3), np.float32, 91, (((3, 0), np.nan), ((4, 1), np.nan), ((11, 2), np.nan)))),
        _l(f"{_fn}_inf", _fn, ((10,), np.float64, 92, ((2, np.inf), (5, -np.inf)))),
        _l(f"err_{_fn}_len1", _fn, ((1, 5), np.float32, 93)),
        _l(f"err_{_fn}_len1_axis1", _fn, ((3, 1), np.int32, 94), axis=1),
        _l(f"err_{_fn}_axis", _fn, ((3, 4), np.float32, 95), axis=2),
        _l(f"refuse_{_fn}_float16", _fn, ((6, 3), np.float16, 96), refuse=True),
        _l(f"refuse_{_fn}_complex", _fn, ((6, 3), np.complex64, 97), refuse=True),
    ]
BY_NAME = {c["name"]: c for c in CASES}
assert len(BY_NAME) == len(CASES)


def piptrack_args(case, y=None, S=None):
    """The keyword arguments of one piptrack case (``y`` / ``S`` override the case's data)."""
    kw = dict(case["kw"])
    if case["y"] is not None:
        kw["y"] = signal(case["y"]) if y is None else y
    if case["S"] is not None:
        kw["S"] = spectrum(case["S"]) if S is None else S
    if kw.get("y") is not None and "sr" not in kw:
        kw["sr"] = SR
    return kw


def call(lib, case, x=None):
    """Run one case through ``lib`` (the reference, librosa_b200 or the oracle): piptrack returns (pitches, mags)."""
    if case["fn"] == "piptrack":
        return lib.piptrack(**piptrack_args(case))
    data = values(case["spec"]) if x is None else x
    if case["fn"] == "pitch_tuning":
        return lib.pitch_tuning(data, **case["kw"])
    return getattr(lib.util, case["fn"])(data, **case["kw"])


def sparse(pitches, mags):
    """The stored form of a piptrack result: (flat indices, pitches there, mags there)."""
    idx = np.flatnonzero((pitches != 0) | (mags != 0)).astype(np.int32)
    return idx, pitches.reshape(-1)[idx], mags.reshape(-1)[idx]


def dense(store, name):
    """The (pitches, mags) pair of a stored case."""
    shape, dtype = tuple(store[f"{name}/shape"]), np.dtype(str(store[f"{name}/dtype"]))
    p, m = np.zeros(shape, dtype), np.zeros(shape, dtype)
    idx = store[f"{name}/idx"]
    p.reshape(-1)[idx] = store[f"{name}/p"]
    m.reshape(-1)[idx] = store[f"{name}/m"]
    return p, m
