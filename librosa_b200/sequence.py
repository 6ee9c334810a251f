"""``librosa.sequence`` (reference: librosa/sequence.py): alignment — ``dtw``, ``dtw_backtracking``, ``rqa`` and
``path_to_steps`` — and HMM decoding — ``viterbi``, ``viterbi_discriminative``, ``viterbi_binary`` and the
``transition_*`` builders.

The builders run on the host in NumPy.  The decoders build every model constant on the host with NumPy's own
operations — ``log(transition + eps)``, ``log(p_init + eps)``, ``log(p_state + eps)``, the threshold and the
predecessor lists — and upload them exactly as float64; two kernels (csrc/sequence_kernels.cuh) then form the
log-likelihoods from ``prob`` and decode every clip.  A DeviceArray ``prob`` gives DeviceArray results."""
from __future__ import annotations

import ctypes as C
from typing import Optional

import numpy as np

from . import _native as nat
from . import _pipeline as pl
from .filters import get_window
from .util.exceptions import ParameterError
from .util.utils import is_positive_int, pad_center

_vp = C.c_void_p

__all__ = ["dtw", "dtw_backtracking", "rqa", "path_to_steps", "viterbi", "viterbi_discriminative", "viterbi_binary", "transition_uniform", "transition_loop",
           "transition_cycle", "transition_local"]

# Two float64 value rows per state in the 227 KiB of shared memory an H100 CTA may opt into, less 1 KiB of static
# reduction scratch (csrc/sequence_api.cu); 16-bit states cap it at 65 535 anyway.
MAX_STATES = (227 * 1024 - 1024) // 16
# Device scratch per slice of the batch: 8 bytes of log-likelihood and 2 of back-pointer per state and frame.
SCRATCH_BYTES = 1 << 30


# --------------------------------------------------------------------------------------------- builders
def transition_uniform(n_states: int) -> np.ndarray:
    """Uniform transition matrix; same contract as ``librosa.sequence.transition_uniform``."""
    if not is_positive_int(n_states):
        raise ParameterError(f"n_states={n_states} must be a positive integer")
    transition = np.empty((n_states, n_states), dtype=np.float64)
    transition.fill(1.0 / n_states)
    return transition


def _per_state(n_states, prob):
    prob = np.asarray(prob, dtype=np.float64)
    if prob.ndim == 0:
        prob = np.tile(prob, n_states)
    if prob.shape != (n_states,):
        raise ParameterError(f"prob={prob} must have length equal to n_states={n_states}")
    if np.any(prob < 0) or np.any(prob > 1):
        raise ParameterError(f"prob={prob} must have values in the range [0, 1]")
    return prob


def transition_loop(n_states: int, prob) -> np.ndarray:
    """Self-loop transition matrix; same contract as ``librosa.sequence.transition_loop``."""
    if not (is_positive_int(n_states) and n_states > 1):
        raise ParameterError(f"n_states={n_states} must be a positive integer > 1")
    transition = np.empty((n_states, n_states), dtype=np.float64)
    prob = _per_state(n_states, prob)
    for i, prob_i in enumerate(prob):
        transition[i] = (1.0 - prob_i) / (n_states - 1)
        transition[i, i] = prob_i
    return transition


def transition_cycle(n_states: int, prob) -> np.ndarray:
    """Cyclic transition matrix; same contract as ``librosa.sequence.transition_cycle``."""
    if not (is_positive_int(n_states) and n_states > 1):
        raise ParameterError(f"n_states={n_states} must be a positive integer > 1")
    transition = np.zeros((n_states, n_states), dtype=np.float64)
    prob = _per_state(n_states, prob)
    for i, prob_i in enumerate(prob):
        transition[i, np.mod(i + 1, n_states)] = 1.0 - prob_i
        transition[i, i] = prob_i
    return transition


def _transition_local_rows(n_states, width, window="triangle", wrap=False):
    """``transition_local`` before its rows are normalised: (matrix, row sums as a column).  pyin's compact
    transition table (core/pitch.py) reads the row sums."""
    if not (is_positive_int(n_states) and n_states > 1):
        raise ParameterError(f"n_states={n_states} must be a positive integer > 1")
    width = np.asarray(width, dtype=int)
    if width.ndim == 0:
        width = np.tile(width, n_states)
    if width.shape != (n_states,):
        raise ParameterError(f"width={width} must have length equal to n_states={n_states}")
    if np.any(width < 1):
        raise ParameterError(f"width={width} must be at least 1")
    transition = np.zeros((n_states, n_states), dtype=np.float64)
    for i, width_i in enumerate(width):
        trans_row = pad_center(get_window(window, width_i, fftbins=False), size=n_states)
        trans_row = np.roll(trans_row, n_states // 2 + i + 1)
        if not wrap:
            trans_row[min(n_states, i + width_i // 2 + 1):] = 0
            trans_row[: max(0, i - width_i // 2)] = 0
        transition[i] = trans_row
    return transition, transition.sum(axis=1, keepdims=True)


def transition_local(n_states: int, width, *, window="triangle", wrap: bool = False) -> np.ndarray:
    """Banded transition matrix; same contract as ``librosa.sequence.transition_local``."""
    transition, sums = _transition_local_rows(n_states, width, window, wrap)
    transition /= sums
    return transition


# --------------------------------------------------------------------------------------------- argument checks
class _Checks:
    """The reference's checks in its order.  Host checks raise at once.  A check of the data (``prob``) is decided
    on the host for host input; for a DeviceArray it is a verdict flag of the log-likelihood kernel, read once after
    the decode — or earlier, by a flags-only launch, when a later host check fails, so that the data error still
    wins as in the reference."""

    def __init__(self, prob, verdict):
        self.prob, self.on_device = prob, isinstance(prob, nat.DeviceArray)
        self.verdict = verdict       # () -> int32 flags array: one flags-only launch and one read-back
        self.pending = []            # (flag word, exception) of device data checks not yet decided

    def data(self, host_bad, word, exc):
        if not self.on_device:
            if host_bad():
                raise exc
        else:
            self.pending.append((word, exc))

    def fail(self, exc):
        """A host check failed: an earlier data error is raised instead, if there is one."""
        if self.pending:
            self.settle(self.verdict())
        raise exc

    def settle(self, flags):
        for word, exc in self.pending:
            if flags[word]:
                raise exc
        self.pending = []


def _log_threshold(transition_min_prob, epsilon):
    if transition_min_prob is not None and transition_min_prob > 0:
        return np.log(transition_min_prob + epsilon)
    if transition_min_prob is None or transition_min_prob == 0:
        return -np.inf
    raise ParameterError(f"Invalid transition_min_prob={transition_min_prob}, must be None or non-negative.")


def _predecessors(log_trans, threshold):
    """Predecessor table of one model as the decode kernel reads it: (deg, dense, lt [deg][S], idx [deg][S]).
    Entry m of state j is its m-th predecessor in ascending order (flatnonzero(log_trans[:, j] >= threshold)),
    padded with (0, -inf); a full search lists every state.  Raises the reference's empty-column error."""
    S = log_trans.shape[0]
    log_trans = np.asarray(log_trans, dtype=np.float64)
    if not np.isfinite(threshold):
        return S, True, np.ascontiguousarray(log_trans), None
    mask = log_trans >= threshold
    deg = mask.sum(axis=0)
    empty = np.flatnonzero(deg == 0)
    if empty.size:
        raise ParameterError(f"Empty transition matrix detected for state {empty[0]} in Viterbi. "
                             f"Try reducing your minimum transition probability threshold.")
    if np.all(deg == S):
        return S, True, np.ascontiguousarray(log_trans), None
    D = int(deg.max())
    order = np.argsort(~mask, axis=0, kind="stable")[:D]          # the predecessors first, ascending
    valid = np.arange(D)[:, None] < deg[None, :]
    lt = np.where(valid, log_trans[order, np.arange(S)[None, :]], -np.inf)
    idx = np.where(valid, order, 0).astype(np.uint16)
    return D, False, lt, idx


def _float_dtype(dtype, what):
    if np.dtype(dtype) not in (np.float32, np.float64):
        raise nat.UnsupportedOnGPU(f"{what} of {np.dtype(dtype)} probabilities is not supported on the GPU "
                                   "(float32 and float64 only)")


def _check_states(n_states, what):
    if n_states > MAX_STATES:
        raise nat.UnsupportedOnGPU(f"{what}: {n_states} states; the GPU decoder holds at most {MAX_STATES} (two "
                                   f"float64 value rows in shared memory)")


def _zero_lead(lead):
    if lead and 0 in lead:
        raise ValueError("cannot call `vectorize` with a signature including new output dimensions on size 0 inputs")


# --------------------------------------------------------------------------------------------- device runner
class _Run:
    """One call's device side: the verdict flags and the sliced log-likelihood + decode launches over ``prob``
    (C order, [clip][n_states][n_steps])."""

    def __init__(self, prob, mode, n_flags):
        self.on_device = isinstance(prob, nat.DeviceArray)
        if self.on_device and prob.layout != "c":
            raise nat.UnsupportedOnGPU("viterbi needs a C-ordered DeviceArray")
        self.prob, self.mode, self.n_flags = prob, mode, n_flags
        self.shape, self.dtype = prob.shape, np.dtype(prob.dtype)
        self.n_clips = pl.clip_count(self.shape[:-2])
        self.S, self.T = self.shape[-2], self.shape[-1]

    def _desc(self, eps, d_lm, n_clips):
        return nat.SeqLogObsDesc(mode=self.mode, f64=int(self.dtype == np.float64), n_clips=n_clips,
                                 n_states=self.S, n_steps=self.T, eps=float(eps), d_log_marginal=d_lm)

    def verdict(self):
        """Flags-only launch over the whole batch and one read-back."""
        with pl.Scope(self.prob) as sc:
            flags = sc.zeros((self.n_flags,), np.int32)
            nat.check(nat.lib().b2l_seq_logobs(sc.ctx.handle, C.byref(self._desc(0.0, None, self.n_clips)),
                                               _vp(sc.stage(self.prob).ptr), None, _vp(flags.ptr)))
            return flags.get()

    def decode(self, checks, states_shape, logp_shape, *, eps, log_marginal, n_models, lt, idx, deg, dense,
               log_p_init):
        """Log-likelihoods and decode in slices of whole clips (SCRATCH_BYTES of scratch each), then the device data
        checks (one read-back of the flags).  Returns the states ``states_shape`` and logp ``logp_shape`` of
        problem = clip * n_models + model, host or device like ``prob``."""
        with pl.Scope(self.prob) as sc:
            ctx, L = sc.ctx, nat.lib()
            dev = sc.stage(self.prob)
            S_dec = 2 if self.mode == nat.SEQ_BINARY else self.S
            per_clip = n_models * S_dec * self.T * 10
            clips = max(1, min(self.n_clips, SCRATCH_BYTES // max(per_clip, 1)))
            n_problems = self.n_clips * n_models
            states = sc.empty((n_problems, self.T), np.uint16)
            logp = sc.empty((n_problems,), np.float64)
            flags = sc.zeros((self.n_flags,), np.int32)
            d_lm = sc.stage(log_marginal, np.float64).ptr if log_marginal is not None else None
            model = nat.SeqModel(n_states=S_dec, n_models=n_models, deg=deg, dense=int(dense),
                                 d_lt=sc.stage(lt, np.float64).ptr,
                                 d_idx=sc.stage(idx, np.uint16).ptr if idx is not None else None,
                                 d_log_p_init=sc.stage(log_p_init, np.float64).ptr)
            lp = sc.empty((clips * n_models * S_dec * self.T,), np.float64)
            item = self.dtype.itemsize
            for c0 in range(0, self.n_clips, clips):
                m = min(clips, self.n_clips - c0)
                nat.check(L.b2l_seq_logobs(ctx.handle, C.byref(self._desc(eps, d_lm, m)),
                                           _vp(dev.ptr + c0 * self.S * self.T * item), _vp(lp.ptr), _vp(flags.ptr)))
                p0 = c0 * n_models
                nat.check(L.b2l_seq_decode(ctx.handle, C.byref(model), _vp(lp.ptr), m * n_models, self.T,
                                           _vp(states.ptr + p0 * self.T * 2), _vp(logp.ptr + p0 * 8)))
            if checks.pending:
                checks.settle(flags.get())
            if self.on_device:
                return sc.keep(states).view(states_shape), sc.keep(logp).view(logp_shape)
            return sc.result(states).reshape(states_shape), sc.result(logp).reshape(logp_shape)


def _empty_steps(run, states_shape, return_logp, what):
    if return_logp:
        raise nat.UnsupportedOnGPU(f"{what} of zero frames with return_logp=True: the reference's log-probability "
                                   "is read past the end of its array")
    if run.on_device:
        return run.prob.ctx.empty(states_shape, np.uint16)
    return np.zeros(states_shape, dtype=np.uint16)


# --------------------------------------------------------------------------------------------- decoders
def _prob_info(prob):
    if isinstance(prob, nat.DeviceArray):
        return prob
    return np.asarray(prob)


def viterbi(prob, transition, *, p_init: Optional[np.ndarray] = None, return_logp: bool = False,
            transition_min_prob: Optional[float] = None):
    """Viterbi decoding from observation likelihoods; same contract as ``librosa.sequence.viterbi``.

    ``prob`` (..., n_states, n_steps) float32 or float64, host or DeviceArray; ``transition`` and ``p_init`` are
    host arrays.  Returns uint16 states (..., n_steps) and, with ``return_logp``, float64 ``logp``: shape (1,) for
    2-D ``prob``, else (...)."""
    prob = _prob_info(prob)
    _float_dtype(prob.dtype, "viterbi")
    n_states, n_steps = prob.shape[-2:]
    _check_states(n_states, "viterbi")
    run = _Run(prob, nat.SEQ_PLAIN, 1)
    chk = _Checks(prob, run.verdict)
    if transition.shape != (n_states, n_states):
        raise ParameterError(f"transition.shape={transition.shape}, must be (n_states, n_states)={n_states, n_states}")
    if np.any(transition < 0) or not np.allclose(transition.sum(axis=1), 1):
        raise ParameterError("Invalid transition matrix: must be non-negative and sum to 1 on each row.")
    chk.data(lambda: np.any(prob < 0) or np.any(prob > 1), 0,
             ParameterError("Invalid probability values: must be between 0 and 1."))
    epsilon = np.finfo(prob.dtype).tiny
    if p_init is None:
        p_init = np.empty(n_states)
        p_init.fill(1.0 / n_states)
    elif np.any(p_init < 0) or not np.allclose(p_init.sum(), 1) or p_init.shape != (n_states,):
        chk.fail(ParameterError(f"Invalid initial state distribution: p_init={p_init}"))
    log_trans = np.log(transition + epsilon)
    log_p_init = np.log(p_init + epsilon)
    try:
        thr = _log_threshold(transition_min_prob, epsilon)
        if prob.ndim > 2:
            _zero_lead(prob.shape[:-2])
        deg, dense, lt, idx = _predecessors(log_trans, thr)
    except (ParameterError, ValueError) as exc:
        chk.fail(exc)
    lead = prob.shape[:-2]
    logp_shape = (1,) if prob.ndim == 2 else lead
    if n_steps == 0:
        if prob.ndim > 2:
            chk.fail(IndexError(f"index 0 is out of bounds for axis {len(lead)} with size 0"))
        return _empty_steps(run, lead + (0,), return_logp, "viterbi")
    states, logp = run.decode(chk, lead + (n_steps,), logp_shape, eps=epsilon, log_marginal=None, n_models=1, lt=lt,
                              idx=idx, deg=deg, dense=dense, log_p_init=log_p_init)
    if return_logp:
        return states, logp
    return states


def viterbi_discriminative(prob, transition, *, p_state: Optional[np.ndarray] = None,
                           p_init: Optional[np.ndarray] = None, return_logp: bool = False,
                           transition_min_prob: Optional[float] = None):
    """Viterbi decoding from discriminative state predictions; same contract as
    ``librosa.sequence.viterbi_discriminative``.  Returns uint16 states (..., n_steps) and, with ``return_logp``,
    float64 ``logp`` (...) — a 0-d array for 2-D ``prob``."""
    prob = _prob_info(prob)
    _float_dtype(prob.dtype, "viterbi_discriminative")
    n_states, n_steps = prob.shape[-2:]
    _check_states(n_states, "viterbi_discriminative")
    run = _Run(prob, nat.SEQ_DISC, 1)
    chk = _Checks(prob, run.verdict)
    if transition.shape != (n_states, n_states):
        raise ParameterError(f"transition.shape={transition.shape}, must be (n_states, n_states)={n_states, n_states}")
    if np.any(transition < 0) or not np.allclose(transition.sum(axis=1), 1):
        raise ParameterError("Invalid transition matrix: must be non-negative and sum to 1 on each row.")
    chk.data(lambda: np.any(prob < 0) or not np.allclose(prob.sum(axis=-2), 1), 0,
             ParameterError("Invalid probability values: each column must sum to 1 and be non-negative"))
    epsilon = np.finfo(prob.dtype).tiny
    if p_state is None:
        p_state = np.empty(n_states)
        p_state.fill(1.0 / n_states)
    elif p_state.shape != (n_states,):
        chk.fail(ParameterError(f"Marginal distribution p_state must have shape (n_states,). "
                                f"Got p_state.shape={p_state.shape}"))
    elif np.any(p_state < 0) or not np.allclose(p_state.sum(axis=-1), 1):
        chk.fail(ParameterError(f"Invalid marginal state distribution: p_state={p_state}"))
    if p_init is None:
        p_init = np.empty(n_states)
        p_init.fill(1.0 / n_states)
    elif np.any(p_init < 0) or not np.allclose(p_init.sum(), 1) or p_init.shape != (n_states,):
        chk.fail(ParameterError(f"Invalid initial state distribution: p_init={p_init}"))
    log_p_init = np.log(p_init + epsilon)
    log_trans = np.log(transition + epsilon)
    log_marginal = np.log(p_state + epsilon)
    try:
        thr = _log_threshold(transition_min_prob, epsilon)
        if prob.ndim > 2:
            _zero_lead(prob.shape[:-2])
        deg, dense, lt, idx = _predecessors(log_trans, thr)
    except (ParameterError, ValueError) as exc:
        chk.fail(exc)
    lead = prob.shape[:-2]
    if n_steps == 0:
        chk.fail(IndexError(f"index 0 is out of bounds for axis {len(lead)} with size 0"))
    states, logp = run.decode(chk, lead + (n_steps,), lead, eps=epsilon, log_marginal=log_marginal, n_models=1, lt=lt,
                              idx=idx, deg=deg, dense=dense, log_p_init=log_p_init)
    if return_logp:
        return states, logp
    return states


def viterbi_binary(prob, transition, *, p_state=None, p_init=None, return_logp: bool = False,
                   transition_min_prob: Optional[float] = None):
    """Viterbi decoding of independent binary states; same contract as ``librosa.sequence.viterbi_binary``.
    Returns uint16 states (..., n_states, n_steps) and, with ``return_logp``, float64 ``logp`` (..., n_states).
    All labels of all clips are decoded in one launch."""
    prob = _prob_info(prob)
    if prob.ndim < 2:
        prob = prob.view((1,) * (2 - prob.ndim) + prob.shape) if isinstance(prob, nat.DeviceArray) \
            else np.atleast_2d(prob)
    _float_dtype(prob.dtype, "viterbi_binary")
    n_states, n_steps = prob.shape[-2:]
    run = _Run(prob, nat.SEQ_BINARY, 1 + n_states)
    chk = _Checks(prob, run.verdict)
    if transition.shape == (2, 2):
        transition = np.tile(transition, (n_states, 1, 1))
    elif transition.shape != (n_states, 2, 2):
        raise ParameterError(f"transition.shape={transition.shape}, must be (2, 2) or (n_states, 2, 2)={n_states}")
    if np.any(transition < 0) or not np.allclose(transition.sum(axis=-1), 1):
        raise ParameterError("Invalid transition matrix: must be non-negative and sum to 1 on each row.")
    chk.data(lambda: np.any(prob < 0) or np.any(prob > 1), 0,
             ParameterError("Invalid probability values: prob must be between [0, 1]"))
    if p_state is None:
        p_state = np.empty(n_states)
        p_state.fill(0.5)
    else:
        p_state = np.atleast_1d(p_state)
    if p_state.shape != (n_states,) or np.any(p_state < 0) or np.any(p_state > 1):
        chk.fail(ParameterError(f"Invalid marginal state distributions: p_state={p_state}"))
    if p_init is None:
        p_init = np.empty(n_states)
        p_init.fill(0.5)
    else:
        p_init = np.atleast_1d(p_init)
    if p_init.shape != (n_states,) or np.any(p_init < 0) or np.any(p_init > 1):
        chk.fail(ParameterError(f"Invalid initial state distributions: p_init={p_init}"))
    lead = prob.shape[:-2]
    if n_states == 0:
        states = np.empty(lead + (0, n_steps), dtype=np.uint16)
        return (states, np.empty(lead + (0,))) if return_logp else states
    # per label, what viterbi_discriminative(prob_binary, transition[label], ...) forms and checks
    eps = np.finfo(np.float64).tiny
    two = np.empty(2)
    log_marginal = np.empty((n_states, 2))
    log_p_init = np.empty((n_states, 2))
    tables = []
    if not run.on_device:
        q = (1 - prob).astype(np.float64) + prob.astype(np.float64)
        close = np.moveaxis(np.isclose(q, 1), -2, 0).reshape(n_states, -1).all(axis=1)
    msg = ParameterError("Invalid probability values: each column must sum to 1 and be non-negative")
    for label in range(n_states):
        chk.data(lambda: not close[label], 1 + label, msg)
        two[0], two[1] = 1 - p_state[label], p_state[label]
        log_marginal[label] = np.log(two + eps)
        two[0], two[1] = 1 - p_init[label], p_init[label]
        log_p_init[label] = np.log(two + eps)
        try:
            if label == 0:
                thr = _log_threshold(transition_min_prob, eps)
                if lead:
                    _zero_lead(lead)
            tables.append(_predecessors(np.log(transition[label] + eps), thr))
        except (ParameterError, ValueError) as exc:
            chk.fail(exc)
        if label == 0 and n_steps == 0:
            chk.fail(IndexError(f"index 0 is out of bounds for axis {len(lead)} with size 0"))
    deg = max(t[0] for t in tables)
    dense = all(t[1] for t in tables)
    lt = np.full((n_states, deg, 2), -np.inf)
    idx = np.zeros((n_states, deg, 2), dtype=np.uint16)
    for label, (d, is_dense, lt_l, idx_l) in enumerate(tables):
        lt[label, :d] = lt_l
        idx[label, :d] = np.arange(2)[:, None] if is_dense else idx_l
    states, logp = run.decode(chk, lead + (n_states, n_steps), lead + (n_states,), eps=eps, log_marginal=log_marginal,
                              n_models=n_states, lt=lt, idx=None if dense else idx, deg=deg, dense=dense,
                              log_p_init=log_p_init)
    if return_logp:
        return states, logp
    return states


# --------------------------------------------------------------------------------------------- alignment
# librosa.sequence.dtw, dtw_backtracking, rqa and path_to_steps (reference: librosa/sequence.py:185-1172).  Argument
# checks and the step tables are the reference's, on the host; the cost matrix, the accumulation, the argmin / argmax
# and the path walks run on the device (csrc/align_kernels.cuh).  Host arrays in give host arrays out; a DeviceArray
# in gives DeviceArrays out.
_byref = C.byref     # dtw's argument C hides the ctypes module inside it
_DEFAULT_STEPS = np.array([[1, 1], [0, 1], [1, 0]], dtype=np.uint32)
# Status words of b2l_dtw_backtrack (include/b2l.h): the negated length word
_WALK_ALL_INF, _WALK_INF_END, _WALK_NOT_ORIGIN, _WALK_ZERO_STEP, _WALK_BAD_STEP, _WALK_NAN = range(1, 7)
_NO_PATH = "No valid sub-sequence warping path could be constructed with the given step sizes."
_CDIST_ERROR = ("scipy.spatial.distance.cdist returned an error.\nPlease provide your input in the form X.shape=(K, N) "
                "and Y.shape=(K, M).\n 1-dimensional sequences should be reshaped to X.shape=(1, N) and Y.shape=(1, M).")


def _feature_offsets(shape):
    """Element offset, in the C-ordered array of ``shape`` (..., K, N), of each feature of frame 0 in the order of the
    reference's ``swapaxes(X, -1, 0).reshape(N, -1, order="F")``; feature f of frame n is at offset[f] + n."""
    n = shape[-1]
    base = (np.arange(int(np.prod(shape[:-1], dtype=np.int64)), dtype=np.int64) * n).reshape(shape[:-1] + (1,))
    return np.ascontiguousarray(np.swapaxes(base, -1, 0).reshape((1, -1), order="F")[0])


def _band(shape, band_rad):
    """fill_off_diagonal's band as (lo, hi): cell (n, m) keeps its cost iff lo < m - n < hi."""
    radius = int(np.round(band_rad * np.min(shape)))
    offset = abs(shape[0] - shape[1])
    if shape[0] < shape[1]:
        return -radius, radius + offset
    return -radius - offset, radius


def _metric_code(metric):
    """The device metric of a cdist metric name; UnsupportedOnGPU for a callable or another metric scipy knows,
    the reference's ParameterError for a name scipy rejects."""
    from scipy.spatial import distance

    if callable(metric):
        raise nat.UnsupportedOnGPU("dtw: a callable metric is not supported on the GPU (euclidean, sqeuclidean, "
                                   "cityblock, chebyshev and cosine are)")
    if not isinstance(metric, str):
        raise TypeError("2nd argument metric must be a string identifier or a function.")
    name = metric.lower()
    info = distance._METRIC_ALIAS.get(name)
    if info is None and not name.startswith("test_"):
        raise ParameterError(_CDIST_ERROR)
    code = nat.DTW_METRICS.get(info.canonical_name) if info is not None else None
    if code is None:
        raise nat.UnsupportedOnGPU(f"dtw: metric {metric!r} is not supported on the GPU (euclidean, sqeuclidean, "
                                   "cityblock, chebyshev and cosine are)")
    return code


def _features(x, what):
    """(array to upload or DeviceArray, shape, f64) of dtw's X or Y, at least 2-D."""
    if isinstance(x, nat.DeviceArray):
        if x.layout != "c" or x.dtype not in (np.float32, np.float64):
            raise nat.UnsupportedOnGPU(f"dtw: {what} must be a C-ordered float32 or float64 DeviceArray")
        if x.ndim < 2:
            x = x.view((1,) * (2 - x.ndim) + x.shape)
        return x, x.shape, x.dtype == np.float64
    x = np.atleast_2d(np.asarray(x))
    if np.iscomplexobj(x):
        raise nat.UnsupportedOnGPU(f"dtw: complex {what} is not supported on the GPU")
    if x.dtype != np.float32:
        x = x.astype(np.float64)      # what cdist computes in
    return np.ascontiguousarray(x), x.shape, x.dtype == np.float64


def _dtw_desc(shape, steps, w_add, w_mul, *, c_f64=True, subseq=False, band=None):
    lo, hi = band if band is not None else (0, 0)
    desc = nat.DtwDesc(n=shape[0], m=shape[1], c_f64=int(c_f64), n_steps=len(steps), subseq=int(bool(subseq)),
                       band=int(band is not None), band_lo=lo, band_hi=hi, h_steps=steps.ctypes.data,
                       h_w_add=w_add.ctypes.data, h_w_mul=w_mul.ctypes.data)
    return desc


def _walk(run, desc, d_steps, d_D, start, check_end, flip, flags):
    """b2l_dtw_backtrack and one 8-byte read-back of the length word: (wp buffer, length or -status)."""
    n, m = desc.n, desc.m
    wp = run.empty((n + m, 2), np.int64)
    length = run.empty((1,), np.int64)
    nat.check(nat.lib().b2l_dtw_backtrack(run.ctx.handle, C.byref(desc), _vp(d_steps.ptr),
                                          _vp(d_D.ptr) if d_D is not None else None, start, check_end, flip,
                                          _vp(flags.ptr) if flags is not None else None, _vp(wp.ptr),
                                          _vp(length.ptr)))
    return wp, int(length.get()[0])


def _walk_refusal(status):
    if status == -_WALK_ZERO_STEP:
        raise nat.UnsupportedOnGPU("dtw: the warping path takes a (0, 0) step, where the reference's backtracking "
                                   "never ends")
    if status == -_WALK_BAD_STEP:
        raise nat.UnsupportedOnGPU("dtw: steps holds an index outside the step table")


def _path_out(run, buf, length):
    if run.on_device:
        return run.keep(buf).view((length, 2))
    return buf.get()[:length].copy()


def dtw(X=None, Y=None, *, C=None, metric: str = "euclidean", step_sizes_sigma=None, weights_add=None,
        weights_mul=None, subseq: bool = False, backtrack: bool = True, global_constraints: bool = False,
        band_rad: float = 0.25, return_steps: bool = False):
    """Dynamic time warping; same contract as ``librosa.sequence.dtw``.

    ``X`` (..., K, N) / ``Y`` (..., K, M) features, or a cost matrix ``C`` (N, M), float32 or float64, host or
    DeviceArray.  Returns float64 ``D``, with ``backtrack`` the int64 warping path ``wp`` (end to start) and with
    ``return_steps`` the int32 step matrix.  The metrics euclidean, sqeuclidean, cityblock, chebyshev and cosine
    give scipy's cdist bit for bit; another metric, or a callable, raises UnsupportedOnGPU."""
    default_weights_add = np.zeros(3, dtype=np.float64)
    default_weights_mul = np.ones(3, dtype=np.float64)
    if step_sizes_sigma is None:
        step_sizes_sigma = _DEFAULT_STEPS
        if weights_add is None:
            weights_add = default_weights_add
        if weights_mul is None:
            weights_mul = default_weights_mul
    else:
        if weights_add is None:
            weights_add = np.zeros(len(step_sizes_sigma), dtype=np.float64)
        if weights_mul is None:
            weights_mul = np.ones(len(step_sizes_sigma), dtype=np.float64)
        default_weights_add.fill(np.inf)
        default_weights_mul.fill(np.inf)
        step_sizes_sigma = np.concatenate((_DEFAULT_STEPS, step_sizes_sigma))
        weights_add = np.concatenate((default_weights_add, weights_add))
        weights_mul = np.concatenate((default_weights_mul, weights_mul))
    if np.any(step_sizes_sigma < 0):
        raise ParameterError("step_sizes_sigma cannot contain negative values")
    if len(step_sizes_sigma) != len(weights_add):
        raise ParameterError("len(weights_add) must be equal to len(step_sizes_sigma)")
    if len(step_sizes_sigma) != len(weights_mul):
        raise ParameterError("len(weights_mul) must be equal to len(step_sizes_sigma)")
    if C is None and (X is None or Y is None):
        raise ParameterError("If C is not supplied, both X and Y must be supplied")
    if C is not None and (X is not None or Y is not None):
        raise ParameterError("If C is supplied, both X and Y must not be supplied")

    with pl.Scope(X, Y, C) as run:
        transposed = False
        flags = None
        if C is None:
            X, x_shape, x_f64 = _features(X, "X")
            Y, y_shape, y_f64 = _features(Y, "Y")
            N, M = x_shape[-1], y_shape[-1]
            K = int(np.prod(x_shape[:-1], dtype=np.int64))
            if K != int(np.prod(y_shape[:-1], dtype=np.int64)):
                raise ParameterError(_CDIST_ERROR)
            code = _metric_code(metric)
            if x_f64 != y_f64:        # the kernel reads both in one dtype; widening is exact
                if run.on_device:
                    raise nat.UnsupportedOnGPU("dtw: X and Y must share a dtype when one is a DeviceArray")
                X, Y, x_f64 = X.astype(np.float64), Y.astype(np.float64), True
            if N == 0 or M == 0 or K == 0:
                raise nat.UnsupportedOnGPU("dtw: empty features (the reference indexes past its arrays)")
            transposed = bool(subseq and N > M)
            shape = (M, N) if transposed else (N, M)
            dX, dY = run.stage(X), run.stage(Y)
            d_C = run.empty(shape, np.float64)
            flags = run.zeros((1,), np.int32)
            x_off, y_off = _feature_offsets(x_shape), _feature_offsets(y_shape)
            cdesc = nat.DtwCostDesc(f64=int(x_f64), metric=code, transpose=int(transposed), K=K, N=N, M=M,
                                    h_x_off=x_off.ctypes.data, h_y_off=y_off.ctypes.data)
            nat.check(nat.lib().b2l_dtw_cost(run.ctx.handle, _byref(cdesc), _vp(dX.ptr), _vp(dY.ptr), _vp(d_C.ptr),
                                             _vp(flags.ptr)))
            c_f64 = True
        else:
            if isinstance(C, nat.DeviceArray):
                if C.layout != "c" or C.dtype not in (np.float32, np.float64):
                    raise nat.UnsupportedOnGPU("dtw: C must be a C-ordered float32 or float64 DeviceArray")
                d_C = C if C.ndim == 2 else C.view((1,) * (2 - C.ndim) + C.shape)
                if C.ndim > 2:
                    raise nat.UnsupportedOnGPU("dtw: C must be 2-D")
            else:
                C = np.atleast_2d(np.asarray(C))
                if C.ndim != 2 or np.iscomplexobj(C):
                    raise nat.UnsupportedOnGPU("dtw: C must be a real 2-D matrix")
                if C.dtype != np.float32:
                    C = C.astype(np.float64)
                d_C = None
            shape = (C.shape[-2], C.shape[-1]) if not isinstance(C, nat.DeviceArray) else d_C.shape
            c_f64 = C.dtype == np.float64
            if 0 in shape:
                raise nat.UnsupportedOnGPU("dtw: an empty cost matrix (the reference indexes past its arrays)")
        if np.array_equal(step_sizes_sigma, np.array([[1, 1]])) and shape[0] > shape[1]:
            raise ParameterError("For diagonal matching: Y.shape[-1] >= X.shape[-11] (C.shape[1] >= C.shape[0])")
        nan_error = ParameterError("DTW cost matrix C has NaN values. ")
        if C is not None:
            if isinstance(C, nat.DeviceArray):
                flags = run.zeros((1,), np.int32)
                nat.check(nat.lib().b2l_nan_flag(run.ctx.handle, _vp(d_C.ptr), d_C.size, int(c_f64), _vp(flags.ptr)))
            else:
                if np.any(np.isnan(C)):
                    raise nan_error
                d_C = run.stage(np.ascontiguousarray(C))
        steps_tab = np.ascontiguousarray(step_sizes_sigma, dtype=np.int64).reshape(-1, 2)
        w_add = np.ascontiguousarray(weights_add, dtype=np.float64)
        w_mul = np.ascontiguousarray(weights_mul, dtype=np.float64)
        desc = _dtw_desc(shape, steps_tab, w_add, w_mul, c_f64=c_f64, subseq=subseq,
                         band=_band(shape, band_rad) if global_constraints else None)
        D = run.empty(shape, np.float64)
        steps = run.empty(shape, np.int32)
        nat.check(nat.lib().b2l_dtw_accumulate(run.ctx.handle, _byref(desc), _vp(d_C.ptr), _vp(D.ptr), _vp(steps.ptr)))
        out = []
        if backtrack:
            flip = int(bool(subseq) and (transposed or shape[0] > shape[1]))
            wp, length = _walk(run, desc, steps, D, -1, 1, flip, flags)
            if length == -_WALK_NAN:
                raise nan_error
            if length in (-_WALK_ALL_INF, -_WALK_INF_END):
                raise ParameterError(_NO_PATH)
            if length == -_WALK_NOT_ORIGIN:
                raise ParameterError("Unable to compute a full DTW warping path. "
                                     "You may want to try again with subseq=True.")
            _walk_refusal(length)
            out.append(_path_out(run, wp, length))
        elif flags is not None and flags.get()[0]:
            raise nan_error
        D_out = run.result(D)
        steps_out = run.result(steps) if return_steps else None
    ret = [D_out] + out + ([steps_out] if return_steps else [])
    return tuple(ret) if len(ret) > 1 else ret[0]


def dtw_backtracking(steps, *, step_sizes_sigma=None, subseq: bool = False, start=None):
    """Backtrack a warping path from a step matrix; same contract as ``librosa.sequence.dtw_backtracking``.
    ``steps`` (N, M) host integer array or int32 DeviceArray; returns the int64 path (L, 2), end to start."""
    if subseq is False and start is not None:
        raise ParameterError(f"start is only allowed to be set if subseq is True (start={start}, subseq={subseq})")
    if step_sizes_sigma is None:
        step_sizes_sigma = _DEFAULT_STEPS
    else:
        step_sizes_sigma = np.concatenate((_DEFAULT_STEPS, step_sizes_sigma))
    table = np.ascontiguousarray(step_sizes_sigma, dtype=np.int64).reshape(-1, 2)
    if np.any(table < 0):
        raise nat.UnsupportedOnGPU("dtw_backtracking: negative step sizes")
    on_device = isinstance(steps, nat.DeviceArray)
    if on_device:
        if steps.layout != "c" or steps.dtype != np.int32 or steps.ndim != 2:
            raise nat.UnsupportedOnGPU("dtw_backtracking: steps must be a C-ordered 2-D int32 DeviceArray")
    else:
        steps = np.asarray(steps)
        if steps.ndim != 2 or steps.dtype.kind not in "iu" or np.any(steps.astype(np.int32) != steps):
            raise nat.UnsupportedOnGPU("dtw_backtracking: steps must be a 2-D integer array of step indices")
        steps = np.ascontiguousarray(steps, dtype=np.int32)
    n, m = steps.shape
    if 0 in (n, m):
        raise nat.UnsupportedOnGPU("dtw_backtracking: an empty step matrix")
    if start is not None and not 0 <= int(start) < m:
        raise nat.UnsupportedOnGPU(f"dtw_backtracking: start={start} outside the {m} columns (the reference reads "
                                   "outside its array)")
    zeros = np.zeros(len(table))
    with pl.Scope(steps) as run:
        desc = _dtw_desc((n, m), table, zeros, zeros, subseq=subseq)
        wp, length = _walk(run, desc, run.stage(steps), None, -1 if start is None else int(start), 0, 0, None)
        _walk_refusal(length)
        return _path_out(run, wp, length)


def rqa(sim, *, gap_onset: float = 1, gap_extend: float = 1, knight_moves: bool = True, backtrack: bool = True):
    """Recurrence quantification analysis; same contract as ``librosa.sequence.rqa``.

    ``sim`` (N, M) float32 or float64, host or DeviceArray.  Returns ``score`` in sim's dtype and, with ``backtrack``,
    the uint64 ``path`` (k, 2) start to end — (0, 2) when there is none."""
    if gap_onset < 0:
        raise ParameterError("gap_onset={} must be strictly positive")
    if gap_extend < 0:
        raise ParameterError("gap_extend={} must be strictly positive")
    on_device = isinstance(sim, nat.DeviceArray)
    if not on_device:
        sim = np.asarray(sim)
    if np.dtype(sim.dtype) not in (np.float32, np.float64):
        raise nat.UnsupportedOnGPU(f"rqa of a {np.dtype(sim.dtype)} similarity matrix is not supported on the GPU "
                                   "(float32 and float64 only)")
    if sim.ndim != 2 or 0 in sim.shape:
        raise nat.UnsupportedOnGPU("rqa needs a non-empty 2-D similarity matrix")
    if on_device and sim.layout != "c":
        raise nat.UnsupportedOnGPU("rqa needs a C-ordered DeviceArray")
    n, m = sim.shape
    f64 = int(sim.dtype == np.float64)
    with pl.Scope(sim) as run:
        d_sim = run.stage(sim)
        score = run.empty((n, m), sim.dtype)
        ptr = run.empty((n, m), np.int8)
        L = nat.lib()
        nat.check(L.b2l_rqa(run.ctx.handle, _vp(d_sim.ptr), n, m, f64, float(gap_onset), float(gap_extend),
                            int(bool(knight_moves)), _vp(score.ptr), _vp(ptr.ptr)))
        if not backtrack:
            return run.result(score)
        path = run.empty((n, 2), np.uint64)
        length = run.empty((1,), np.int64)
        nat.check(L.b2l_rqa_path(run.ctx.handle, _vp(score.ptr), _vp(ptr.ptr), n, m, f64, _vp(path.ptr),
                                 _vp(length.ptr)))
        k = int(length.get()[0])
        if k < 0:
            raise nat.UnsupportedOnGPU("rqa: the path's column index passes -M (the reference raises IndexError)")
        score_out = run.result(score)
        return score_out, _path_out(run, path, k)


def path_to_steps(path, *, inverse: bool = False):
    """Fractional steps from a warping path by linear interpolation; same contract as
    ``librosa.sequence.path_to_steps``.  Runs on the host (a DeviceArray path is read back first)."""
    import scipy.interpolate

    if isinstance(path, nat.DeviceArray):
        path = path.get()
    if inverse:
        idx_from, idx_to = 1, 0
    else:
        idx_from, idx_to = 0, 1
    step_interp = scipy.interpolate.interp1d(path[:, idx_to], path[:, idx_from], kind="linear")
    frames_in = np.arange(path[:, idx_to].min(), path[:, idx_to].max() + 1)
    return step_interp(frames_in)
