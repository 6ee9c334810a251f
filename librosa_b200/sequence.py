"""``librosa.sequence`` HMM decoding (reference: librosa/sequence.py:1175-2146): ``viterbi``,
``viterbi_discriminative``, ``viterbi_binary`` and the ``transition_*`` builders.

The builders run on the host in NumPy.  The decoders build every model constant on the host with NumPy's own
operations — ``log(transition + eps)``, ``log(p_init + eps)``, ``log(p_state + eps)``, the threshold and the
predecessor lists — and upload them exactly as float64; two kernels (csrc/sequence_kernels.cuh) then form the
log-likelihoods from ``prob`` and decode every clip.  A DeviceArray ``prob`` gives DeviceArray results."""
from __future__ import annotations

import ctypes as C
from typing import Optional

import numpy as np

from . import _native as nat
from .filters import get_window
from .util.exceptions import ParameterError
from .util.utils import is_positive_int, pad_center

_vp = C.c_void_p

__all__ = ["viterbi", "viterbi_discriminative", "viterbi_binary", "transition_uniform", "transition_loop",
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
    """One call's device side: the staged ``prob`` (C order, [clip][n_states][n_steps]), the verdict flags and the
    sliced log-likelihood + decode launches."""

    def __init__(self, prob, mode, n_flags):
        from . import _pipeline as pl

        self.on_device = isinstance(prob, nat.DeviceArray)
        self._ctx = prob.ctx if self.on_device else None
        if self.on_device and prob.layout != "c":
            raise nat.UnsupportedOnGPU("viterbi needs a C-ordered DeviceArray")
        self.shape, self.dtype, self.mode = prob.shape, np.dtype(prob.dtype), mode
        self.lead = self.shape[:-2]
        self.n_clips = pl.clip_count(self.lead)
        self.S, self.T = self.shape[-2], self.shape[-1]
        self.host = None if self.on_device else np.ascontiguousarray(prob)
        self.dev = prob if self.on_device else None
        self.n_flags = n_flags
        self.flags = None
        self._owned = []

    @property
    def ctx(self):
        """The device context; a host call creates it only when it reaches device work."""
        if self._ctx is None:
            self._ctx = nat.default_context()
        return self._ctx

    def _stage(self):
        if self.dev is None:
            self.dev = self.ctx.to_device(self.host)
            self._owned.append(self.dev)

    def _new_flags(self):
        flags = nat.DeviceArray.empty(self.ctx, (self.n_flags,), np.int32)
        nat.check(nat.lib().b2l_memset(self.ctx.handle, _vp(flags.ptr), 0, flags.nbytes))
        return flags

    def _desc(self, eps, d_lm, n_clips):
        return nat.SeqLogObsDesc(mode=self.mode, f64=int(self.dtype == np.float64), n_clips=n_clips,
                                 n_states=self.S, n_steps=self.T, eps=float(eps), d_log_marginal=d_lm)

    def verdict(self):
        """Flags-only launch over the whole batch and one read-back."""
        self._stage()
        flags = self._new_flags()
        nat.check(nat.lib().b2l_seq_logobs(self.ctx.handle, C.byref(self._desc(0.0, None, self.n_clips)),
                                           _vp(self.dev.ptr), None, _vp(flags.ptr)))
        return flags.get()

    def upload(self, arr, dtype):
        d = self.ctx.to_device(np.ascontiguousarray(arr, dtype=dtype))
        self._owned.append(d)
        return d.ptr

    def decode(self, *, eps, log_marginal, n_models, lt, idx, deg, dense, log_p_init):
        """Log-likelihoods and decode in slices of whole clips (SCRATCH_BYTES of scratch each).  Returns the states
        [problem][n_steps] and logp [problem] DeviceArrays, problem = clip * n_models + model."""
        self._stage()
        ctx, L = self.ctx, nat.lib()
        S_dec = 2 if self.mode == nat.SEQ_BINARY else self.S
        per_clip = n_models * S_dec * self.T * 10
        clips = max(1, min(self.n_clips, SCRATCH_BYTES // max(per_clip, 1)))
        n_problems = self.n_clips * n_models
        states = nat.DeviceArray.empty(ctx, (n_problems, self.T), np.uint16)
        logp = nat.DeviceArray.empty(ctx, (n_problems,), np.float64)
        self.flags = self._new_flags()
        d_lm = self.upload(log_marginal, np.float64) if log_marginal is not None else None
        model = nat.SeqModel(n_states=S_dec, n_models=n_models, deg=deg, dense=int(dense),
                             d_lt=self.upload(lt, np.float64), d_idx=self.upload(idx, np.uint16) if idx is not None
                             else None, d_log_p_init=self.upload(log_p_init, np.float64))
        lp = ctx.alloc(clips * n_models * S_dec * self.T * 8)
        try:
            item = self.dtype.itemsize
            for c0 in range(0, self.n_clips, clips):
                m = min(clips, self.n_clips - c0)
                nat.check(L.b2l_seq_logobs(ctx.handle, C.byref(self._desc(eps, d_lm, m)),
                                           _vp(self.dev.ptr + c0 * self.S * self.T * item), _vp(lp),
                                           _vp(self.flags.ptr)))
                p0 = c0 * n_models
                nat.check(L.b2l_seq_decode(ctx.handle, C.byref(model), _vp(lp), m * n_models, self.T,
                                           _vp(states.ptr + p0 * self.T * 2), _vp(logp.ptr + p0 * 8)))
        finally:
            ctx.free(lp)
        return states, logp

    def release(self):
        for d in self._owned:
            d.free()
        self._owned = []


def _view(arr, shape):
    """A reshaped view of a C-ordered DeviceArray that keeps it alive."""
    out = nat.DeviceArray(arr.ctx, arr.ptr, shape, arr.dtype, layout="c", owner=False)
    out._base = arr
    return out


def _finish(run, checks, states, logp, states_shape, logp_shape):
    """Settles the device data checks (one read-back of the flags), then returns host or device results."""
    if run.on_device:
        if checks.pending:
            checks.settle(run.flags.get())
        run.release()
        return _view(states, states_shape), _view(logp, logp_shape)
    run.release()
    s, lg = states.get().reshape(states_shape), logp.get().reshape(logp_shape)
    states.free()
    logp.free()
    return s, lg


def _empty_steps(run, states_shape, return_logp, what):
    if return_logp:
        raise nat.UnsupportedOnGPU(f"{what} of zero frames with return_logp=True: the reference's log-probability "
                                   "is read past the end of its array")
    if run.on_device:
        return nat.DeviceArray.empty(run.ctx, states_shape, np.uint16)
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
    states, logp = run.decode(eps=epsilon, log_marginal=None, n_models=1, lt=lt, idx=idx, deg=deg, dense=dense,
                              log_p_init=log_p_init)
    states, logp = _finish(run, chk, states, logp, lead + (n_steps,), logp_shape)
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
    states, logp = run.decode(eps=epsilon, log_marginal=log_marginal, n_models=1, lt=lt, idx=idx, deg=deg,
                              dense=dense, log_p_init=log_p_init)
    states, logp = _finish(run, chk, states, logp, lead + (n_steps,), lead)
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
        prob = _view(prob, (1,) * (2 - prob.ndim) + prob.shape) if isinstance(prob, nat.DeviceArray) \
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
    states, logp = run.decode(eps=eps, log_marginal=log_marginal, n_models=n_states, lt=lt,
                              idx=None if dense else idx, deg=deg, dense=dense, log_p_init=log_p_init)
    states, logp = _finish(run, chk, states, logp, lead + (n_states, n_steps), lead + (n_states,))
    if return_logp:
        return states, logp
    return states
