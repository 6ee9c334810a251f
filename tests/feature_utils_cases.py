"""Case table of feature.delta and feature.stack_memory: tests/golden/feature_utils_v1.npz holds, for each case, what
the unmodified reference returns (``<name>/out``) or the exception it raises (``<name>/error``, "Class: message").
Written by tools/make_golden.py --feature-utils; tests/feature_utils_oracle.py must reproduce every entry bit for bit,
except the interp edges of delta, which it computes with the float64 fit map (see ``edge_tolerance``).

A case's data is made from its spec by ``data`` (seeded, so nothing but the outputs is stored).  ``refuse`` names the
cases the GPU declines with UnsupportedOnGPU although the reference runs them; nothing is stored for them."""
from __future__ import annotations

import numpy as np


def data(spec):
    """spec = (shape, dtype, seed[, specials]); specials: ((index, value), ...) written after the draw."""
    shape, dtype, seed = spec[:3]
    rng = np.random.default_rng(seed)
    dtype = np.dtype(dtype)
    if dtype.kind in "iu":
        x = rng.integers(-50 if dtype.kind == "i" else 0, 50, size=shape).astype(dtype)
    elif dtype.kind == "b":
        x = rng.integers(0, 2, size=shape).astype(bool)
    elif dtype.kind == "c":
        x = (rng.standard_normal(shape) + 1j * rng.standard_normal(shape)).astype(dtype)
    else:
        x = (3.0 * rng.standard_normal(shape)).astype(dtype)
    for idx, v in (spec[3] if len(spec) > 3 else ()):
        x[idx] = v
    return x


def _d(name, spec, refuse=False, **kw):
    return {"name": name, "fn": "delta", "spec": spec, "kw": kw, "refuse": refuse}


def _s(name, spec, refuse=False, **kw):
    return {"name": name, "fn": "stack_memory", "spec": spec, "kw": kw, "refuse": refuse}


F32 = ((3, 40), np.float32, 1)
MFCC = ((20, 431), np.float32, 2)
MODES = ("interp", "nearest", "mirror", "constant", "wrap")

CASES = [_d("delta_mfcc_default", MFCC), _d("delta_mfcc_order2", MFCC, order=2)]
for _mode in MODES:
    for _w in (3, 9, 31):
        for _o in (1, 2, 3):
            CASES.append(_d(f"delta_{_mode}_w{_w}_o{_o}", F32, width=_w, order=_o, mode=_mode))
CASES += [
    _d("delta_w5_o1", F32, width=5), _d("delta_w7_o2", F32, width=7, order=2), _d("delta_w11_o1", F32, width=11),
    _d("delta_w15_o2_f64", ((3, 40), np.float64, 3), width=15, order=2), _d("delta_w21_o3", F32, width=21, order=3),
    # polyorder above the order, including the ill-conditioned fit of the edges
    _d("delta_poly3_o1", F32, polyorder=3), _d("delta_poly7_w9_o2", F32, order=2, polyorder=7),
    _d("delta_poly7_w9_o1_f64", ((3, 40), np.float64, 4), polyorder=7),
    _d("delta_poly5_w31_o3", F32, width=31, order=3, polyorder=5),
    _d("delta_poly7_w31_o3", F32, width=31, order=3, polyorder=7),
    _d("delta_poly4_nearest", F32, order=2, polyorder=4, mode="nearest"),
    # order above polyorder: zero coefficients
    _d("delta_order_above_poly", F32, order=3, polyorder=2),
    _d("delta_order_above_poly_mirror", F32, order=3, polyorder=1, mode="mirror"),
    _d("delta_deriv_dropped", F32, deriv=5),
    _d("delta_spacing", F32, delta=0.5, order=2), _d("delta_spacing_wrap", F32, delta=2.0, mode="wrap"),
    _d("delta_cval", F32, mode="constant", cval=2.5), _d("delta_cval_o2", F32, order=2, mode="constant", cval=-1.0),
    # axes and ranks
    _d("delta_1d", ((50,), np.float32, 5)), _d("delta_1d_axis0", ((50,), np.float32, 5), axis=0),
    _d("delta_2d_axis0", ((30, 6), np.float32, 6), axis=0),
    _d("delta_2d_axis_m2", ((30, 6), np.float32, 6), axis=-2, mode="mirror"),
    _d("delta_3d_axis0", ((12, 3, 5), np.float32, 7), axis=0, mode="nearest"),
    _d("delta_3d_axis1", ((2, 15, 4), np.float32, 8), axis=1),
    _d("delta_3d_axis_m1", ((2, 3, 25), np.float64, 9), order=2),
    _d("delta_4d_axis_m2", ((2, 3, 13, 4), np.float32, 10), axis=-2, width=5),
    _d("delta_4d_axis0", ((11, 2, 3, 4), np.float32, 11), axis=0, mode="wrap"),
    _d("delta_4d_axis_m1", ((2, 2, 3, 17), np.float32, 12), mode="constant"),
    # lines shorter than h, and width == n under interp
    _d("delta_short_mirror", ((3, 2), np.float32, 13), mode="mirror"),
    _d("delta_short_nearest", ((3, 3), np.float32, 13), mode="nearest"),
    _d("delta_short_wrap", ((3, 2), np.float32, 13), mode="wrap", width=11),
    _d("delta_short_constant", ((3, 1), np.float32, 13), mode="constant"),
    _d("delta_one_mirror", ((4, 1), np.float64, 14), mode="mirror", width=5),
    _d("delta_short_axis0_wrap", ((3, 5), np.float32, 15), axis=0, mode="wrap", width=7),
    _d("delta_width_eq_n", ((4, 9), np.float32, 16)), _d("delta_width_eq_n_o3", ((4, 31), np.float32, 16), width=31, order=3),
    # non-finite data: interior of interp, and every position of the padded modes
    _d("delta_nan_interior", ((3, 40), np.float32, 17, (((0, 20), np.nan), ((1, 25), np.inf), ((2, 9), -np.inf)))),
    _d("delta_nan_nearest", ((3, 40), np.float32, 17, (((0, 0), np.nan), ((1, 39), np.inf), ((2, 5), -np.inf))),
       mode="nearest"),
    _d("delta_inf_wrap", ((3, 40), np.float64, 17, (((0, 1), np.inf), ((0, 2), -np.inf))), mode="wrap"),
    _d("delta_nan_edge_interp", ((3, 40), np.float32, 17, (((1, 2), np.nan),))),
    _d("delta_inf_right_edge_interp", ((3, 40), np.float32, 17, (((2, 38), np.inf),))),
    # dtypes
    _d("delta_int16", ((3, 40), np.int16, 18)), _d("delta_int64_mirror", ((3, 40), np.int64, 19), mode="mirror"),
    _d("delta_float64", ((3, 40), np.float64, 20), order=2),
    _d("delta_bool", ((2, 12), bool, 21), mode="nearest"),
    _d("delta_float16", ((2, 12), np.float16, 22), mode="mirror"),
    # errors the reference raises
    _d("delta_err_width_even", F32, width=4), _d("delta_err_width_one", F32, width=1),
    _d("delta_err_order_zero", F32, order=0), _d("delta_err_order_float", F32, order=1.0),
    _d("delta_err_interp_wide", ((3, 7), np.float32, 1)),
    _d("delta_err_mode", F32, mode="reflect"),
    _d("delta_err_polyorder", F32, width=5, polyorder=5),
    _d("delta_err_kwarg", F32, foo=1),
    _d("delta_err_axis_interp", F32, axis=2), _d("delta_err_axis_nearest", F32, axis=-3, mode="nearest"),
    # refusals
    _d("delta_complex", ((3, 40), np.complex64, 23), refuse=True),
    _d("delta_width_257", ((2, 20), np.float32, 24), width=257, mode="nearest", refuse=True),
]

S32 = ((5, 12), np.float32, 30)
CASES += [_s("stack_default", S32), _s("stack_mfcc_n3", MFCC, n_steps=3)]
for _delay in (1, -1, 3, -3):
    for _mode, _kw in (("constant", {}), ("constant7", {"constant_values": 7}), ("edge", {}), ("reflect", {}),
                       ("symmetric", {}), ("wrap", {}), ("empty", {})):
        CASES.append(_s(f"stack_{_mode}_d{_delay}".replace("-", "m"), S32, n_steps=3, delay=_delay,
                        mode=_mode.rstrip("7"), **_kw))
CASES += [
    _s("stack_long_delay", ((3, 6), np.float32, 31), n_steps=5, delay=4),
    _s("stack_long_delay_neg_reflect", ((3, 6), np.float32, 31), n_steps=5, delay=-4, mode="reflect"),
    _s("stack_long_delay_wrap", ((3, 6), np.float32, 31), n_steps=4, delay=3, mode="wrap"),
    _s("stack_long_delay_symmetric", ((3, 5), np.float64, 31), n_steps=3, delay=-7, mode="symmetric"),
    _s("stack_one_step", S32, n_steps=1),
    _s("stack_one_column_edge", ((4, 1), np.float32, 32), n_steps=3, delay=2, mode="edge"),
    _s("stack_constant_pairs", ((2, 3, 6), np.float32, 33), delay=-2, n_steps=3, mode="constant",
       constant_values=((1, 2), (3, 4), (5, 6))),
    _s("stack_constant_cast", ((3, 8), np.int32, 34), n_steps=3, constant_values=1.7),
    _s("stack_reflect_even", S32, n_steps=3, mode="reflect", reflect_type="even"),
    _s("stack_1d", ((10,), np.int64, 35), n_steps=3),
    _s("stack_3d", ((2, 3, 9), np.float32, 36), n_steps=2, delay=2, mode="edge"),
    _s("stack_4d", ((2, 2, 3, 9), np.float64, 37), n_steps=3, delay=-1, mode="wrap"),
    _s("stack_int8", ((4, 9), np.int8, 38), n_steps=3), _s("stack_uint16", ((4, 9), np.uint16, 39), n_steps=3, delay=-2),
    _s("stack_int32_edge", ((4, 9), np.int32, 40), n_steps=2, mode="edge"),
    _s("stack_uint64", ((4, 9), np.uint64, 41), n_steps=2, constant_values=5),
    _s("stack_bool", ((4, 9), bool, 42), n_steps=3, mode="reflect"),
    _s("stack_complex64", ((4, 9), np.complex64, 43), n_steps=3, constant_values=1 + 2j),
    _s("stack_complex128", ((4, 9), np.complex128, 44), n_steps=2, delay=-3, mode="symmetric"),
    _s("stack_nan", ((3, 9), np.float32, 45, (((0, 0), np.nan), ((1, 8), np.inf))), n_steps=3, mode="edge"),
    # errors the reference raises
    _s("stack_err_steps", S32, n_steps=0), _s("stack_err_delay", S32, delay=0),
    _s("stack_err_no_columns", ((3, 0), np.float32, 46)),
    _s("stack_err_mode", S32, mode="foo"),
    _s("stack_err_kwarg", S32, mode="edge", constant_values=3),
    # refusals
    _s("stack_mean", S32, mode="mean", refuse=True), _s("stack_linear_ramp", S32, mode="linear_ramp", refuse=True),
    _s("stack_reflect_odd", S32, mode="reflect", reflect_type="odd", refuse=True),
    _s("stack_callable", S32, mode=lambda vector, pad_width, iaxis, kwargs: None, refuse=True),
]
BY_NAME = {c["name"]: c for c in CASES}
assert len(BY_NAME) == len(CASES)


def call(lib, case, x=None):
    """Run one case through ``lib`` (the reference or librosa_b200)."""
    fn = getattr(lib.feature, case["fn"])
    return fn(data(case["spec"]) if x is None else x, **case["kw"])


def empty_cells(case):
    """Boolean mask of the output cells that NumPy leaves undefined (stack_memory with mode="empty")."""
    x = data(case["spec"])
    x = np.atleast_2d(x)
    kw = case["kw"]
    n, delay, t = kw.get("n_steps", 2), kw.get("delay", 1), x.shape[-1]
    mask = np.zeros(x.shape[:-2] + (n * x.shape[-2], t), dtype=bool)
    if kw.get("mode") != "empty":
        return mask
    for s in range(n):
        q = np.arange(t) - s * delay
        mask[..., s * x.shape[-2]:(s + 1) * x.shape[-2], :] = ((q < 0) | (q >= t))
    return mask


def vandermonde_condition(width: int, polyorder: int) -> float:
    """cond_2 of the Vandermonde matrix on 0 .. width-1 (powers 0 .. polyorder) with unit-norm columns."""
    V = np.arange(width, dtype=np.float64)[:, None] ** np.arange(polyorder + 1)
    return float(np.linalg.cond(V / np.linalg.norm(V, axis=0)))


def edge_tolerance(x, width: int, polyorder: int, axis: int, dtype) -> np.ndarray:
    """Allowed |difference| of each interp edge output from the reference: 32 eps(dtype) cond_2(V) max|x| over its
    edge window, per line and side; returns (left, right) arrays of the line shape."""
    x = np.moveaxis(np.asarray(x, dtype=np.float64), axis, -1)
    k = 32 * np.finfo(dtype).eps * vandermonde_condition(width, polyorder)
    return k * np.abs(x[..., :width]).max(axis=-1), k * np.abs(x[..., -width:]).max(axis=-1)
