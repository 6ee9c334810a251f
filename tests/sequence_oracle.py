"""NumPy restatement of librosa.sequence's decoders (librosa/sequence.py:1175-1876), built on
tests/pitch_oracle.py's predecessor lists and threshold: the log-likelihood stage each decoder forms, a decode that,
like the reference's numba loop, never takes a NaN cost, and the smallest non-zero gap between the winning and the
runner-up cost of every decision (how far a 1-ulp change of a log-likelihood is from flipping the path)."""
from __future__ import annotations

import hashlib

import numpy as np

import pitch_oracle as PO
from oracle.ref_np import tiny


def _models(op, prob, transition, p_init=None, p_state=None, transition_min_prob=None):
    """(lp [problem][state][frame] float64, [(log_trans, log_p_init, threshold)] per model, n_models) as the
    reference forms them."""
    if op == "binary":
        prob = np.atleast_2d(prob)
        L, T = prob.shape[-2:]
        if transition.shape == (2, 2):
            transition = np.tile(transition, (L, 1, 1))
        p_state = np.full(L, 0.5) if p_state is None else np.atleast_1d(p_state)
        p_init = np.full(L, 0.5) if p_init is None else np.atleast_1d(p_init)
        eps = tiny(np.empty(0))
        lp = np.empty(prob.shape[:-2] + (L, 2, T))
        models = []
        for s in range(L):
            pb = np.empty(prob.shape[:-2] + (2, T))
            pb[..., 0, :] = 1 - prob[..., s, :]
            pb[..., 1, :] = prob[..., s, :]
            ps, pi = np.empty(2), np.empty(2)
            ps[0], ps[1] = 1 - p_state[s], p_state[s]
            pi[0], pi[1] = 1 - p_init[s], p_init[s]
            lp[..., s, :, :] = np.log(pb + eps) - np.log(ps + eps)[:, None]
            models.append((np.log(transition[s] + eps), np.log(pi + eps),
                           PO.log_threshold(transition_min_prob, eps)))
        return lp.reshape(-1, 2, T), models, L
    S, T = prob.shape[-2:]
    eps = tiny(prob)
    if p_init is None:
        p_init = np.full(S, 1.0 / S)
    lp = np.log(prob + eps)
    if op == "disc":
        if p_state is None:
            p_state = np.full(S, 1.0 / S)
        lp = lp - np.log(p_state + eps)[:, None]
    return (lp.astype(np.float64).reshape(-1, S, T),
            [(np.log(transition + eps), np.log(p_init + eps), PO.log_threshold(transition_min_prob, eps))], 1)


def decode(lp, log_trans, log_p_init, threshold):
    """One problem: lp (n_states, n_steps) -> (states uint16, logp float64, smallest non-zero decision gap)."""
    S, T = lp.shape
    preds = PO.predecessors(log_trans, threshold)
    D = max(len(p) for p in preds)
    K = np.zeros((S, D), dtype=np.int64)
    W = np.full((S, D), -np.inf)
    for j, p in enumerate(preds):
        K[j, : len(p)] = p
        K[j, len(p):] = p[0]
        W[j, : len(p)] = log_trans[p, j]
    cols = np.arange(S)
    value = lp[:, 0] + log_p_init
    ptr = np.zeros((T, S), dtype=np.uint16)
    gap = np.inf

    def _gap(c, best):
        if c.shape[1] < 2:
            return np.inf
        top = c[np.arange(c.shape[0]), best]
        c2 = c.copy()
        c2[np.arange(c.shape[0]), best] = -np.inf
        g = top - c2.max(axis=1)
        g = g[np.isfinite(g) & (g > 0)]
        return g.min() if g.size else np.inf

    for t in range(1, T):
        cost = value[K] + W
        c = np.where(np.isnan(cost), -np.inf, cost)     # a NaN cost never beats the running best
        best = np.argmax(c, axis=1)
        bc = c[cols, best]
        ptr[t] = np.where(bc > -np.inf, K[cols, best], 0)
        gap = min(gap, _gap(c, best))
        value = lp[:, t] + bc
    last = int(np.argmax(value))
    gap = min(gap, _gap(np.where(np.isnan(value), -np.inf, value)[None, :], np.array([last])))
    states = np.zeros(T, dtype=np.uint16)
    states[-1] = last
    for t in range(T - 2, -1, -1):
        states[t] = ptr[t + 1, states[t + 1]]
    return states, value[last], gap


def score(lp, log_trans, log_p_init, states):
    """The reference's value of the path ``states`` under its own log terms, summed in its order."""
    s = states.astype(np.int64)
    v = lp[s[0], 0] + log_p_init[s[0]]
    for t in range(1, lp.shape[1]):
        v = lp[s[t], t] + (v + log_trans[s[t - 1], s[t]])
    return v


def run(op, prob, transition, *, p_init=None, p_state=None, transition_min_prob=None, return_logp=False,
        one_d=False):
    """A non-error case end to end: {"states", "logp", "lp", "gap", "max_abs_lp"} with the reference's shapes."""
    prob = np.asarray(prob)
    if op == "binary" and prob.ndim == 1:
        prob = prob[None, :]
    lp, models, n_models = _models(op, prob, transition, p_init, p_state, transition_min_prob)
    T = prob.shape[-1]
    states = np.empty((lp.shape[0], T), dtype=np.uint16)
    logp = np.empty(lp.shape[0])
    gap = np.inf
    for p in range(lp.shape[0]):
        lt, lpi, thr = models[p % n_models]
        states[p], logp[p], g = decode(lp[p], lt, lpi, thr)
        gap = min(gap, g)
    lead = prob.shape[:-2]
    if op == "binary":
        states, logp = states.reshape(lead + (n_models, T)), logp.reshape(lead + (n_models,))
    else:
        states = states.reshape(lead + (T,))
        logp = logp.reshape((1,) if (op == "viterbi" and prob.ndim == 2) else lead)
    finite = np.abs(lp[np.isfinite(lp)])
    return dict(states=states, logp=logp, lp=lp, gap=gap, max_abs_lp=float(finite.max()) if finite.size else 0.0,
                models=models, n_models=n_models)


def digest(lp):
    """SHA-256 of a C-ordered float64 log-likelihood array, as the fixture stores it."""
    return hashlib.sha256(np.ascontiguousarray(lp, dtype=np.float64).tobytes()).hexdigest()


def fragile_bound(n_steps, max_abs_lp, dtype):
    """n_steps * 2 ulp(max |log-likelihood|) in the dtype the log is taken in."""
    return n_steps * 2 * float(np.spacing(np.asarray(max_abs_lp, dtype=dtype)))
