"""NumPy restatement of ``util.peak_pick``, ``onset.onset_detect`` and ``onset.onset_backtrack`` (reference:
librosa/util/utils.py:1188-1496, librosa/onset.py:31-214 and :370-441, librosa/util/matching.py:215-390), written
from the arithmetic numba runs: the greedy window mean is a left-to-right sum in the data's dtype divided by the
count in float64; the dynamic-programming pickers use a sequential cumsum in the data's dtype and a float64 DP;
numba's np.max returns NaN as soon as it meets one.  tests/test_onset_host.py checks it bit for bit against the
reference's fixture; the GPU tests use it where the fixture has no entry."""
from __future__ import annotations

import types

import numpy as np

from librosa_b200.util.exceptions import ParameterError

_EMPTY_MATCH = "Attempting to match empty event list"
_NEGATIVE_MATCH = "Cannot match events with right=False and min(events_to) > min(events_from)"


def _max(w):
    """numba's np.max: NaN as soon as one is met."""
    nan = np.isnan(w)
    return w[np.argmax(nan)] if nan.any() else w.max()


def _seq_sum(w, T):
    s = T(0)
    for v in w:
        s = T(s + v)
    return s


def window_mean(x, lo, hi, seq=True):
    """np.mean(x[lo:hi]) as numba computes it (``seq``), or a float64 mean (for comparison)."""
    T = x.dtype.type
    if seq:
        return np.float64(_seq_sum(x[lo:hi], T)) / np.float64(hi - lo)
    return np.float64(np.sum(x[lo:hi].astype(np.float64))) / np.float64(hi - lo)


def _greedy(x, pre_max, post_max, pre_avg, post_avg, delta, wait, seq=True):
    N = x.shape[0]
    peaks = np.zeros(N, dtype=bool)
    delta = np.float64(delta)
    n = 0
    while n < N:
        maxn = _max(x[max(0, n - pre_max): min(n + post_max, N)])
        if x[n] == maxn and np.float64(x[n]) >= window_mean(x, max(0, n - pre_avg), min(n + post_avg, N), seq) + delta:
            peaks[n] = True
            n += wait + 1
        else:
            n += 1
    return peaks


def _dp(x, pre_max, post_max, pre_avg, post_avg, delta, wait, count):
    N = x.shape[0]
    T = x.dtype.type
    peaks = np.zeros(N, dtype=bool)
    values = np.zeros(N + 1)
    pointers = np.zeros(N + 1, dtype=np.int64)
    taken = np.zeros(N + 1, dtype=bool)
    cum = np.empty(N, dtype=x.dtype)
    c = T(0)
    for i in range(N):
        c = T(c + x[i])
        cum[i] = c
    delta = np.float64(delta)
    pointers[N] = -1
    for n in range(N - 1, -1, -1):
        values[n] = values[n + 1]
        pointers[n] = n + 1
        maxn = _max(x[max(0, n - pre_max): min(n + post_max, N)])
        if x[n] < maxn:
            continue
        lo, hi = max(0, n - pre_avg), min(n + post_avg, N)
        if lo == 0:
            avgn = np.float64(cum[hi - 1]) / np.float64(hi)
        else:
            avgn = np.float64(T(cum[hi - 1] - cum[lo - 1])) / np.float64(hi - lo)
        v = 1.0 if count else np.float64(x[n])
        nxt = min(N, n + wait + 1)
        if np.float64(x[n]) >= avgn + delta and values[nxt] + v > values[n + 1]:
            values[n] = values[nxt] + v
            pointers[n] = nxt
            taken[n] = True
    n = 0
    while pointers[n] >= 0:
        peaks[n] = taken[n]
        n = pointers[n]
    return peaks


def peak_pick(x, *, pre_max, post_max, pre_avg, post_avg, delta, wait, sparse=True, method="greedy", axis=-1,
              seq_mean=True):
    """``seq_mean=False``: the greedy picker with a float64 mean (not the reference; for comparison)."""
    from librosa_b200.util.peak import check_args

    x = np.asarray(x)
    (pre_max, post_max, pre_avg, post_avg, wait), _ = check_args(
        x.ndim, pre_max=pre_max, post_max=post_max, pre_avg=pre_avg, post_avg=post_avg, delta=delta, wait=wait,
        sparse=sparse, method=method)
    xs = np.moveaxis(x, axis, -1)
    peaks = np.zeros(xs.shape, dtype=bool)
    rows, out = xs.reshape(-1, xs.shape[-1]), peaks.reshape(-1, xs.shape[-1])
    for r in range(rows.shape[0]):
        if rows.shape[1] == 0:
            continue
        if method == "greedy":
            out[r] = _greedy(rows[r], pre_max, post_max, pre_avg, post_avg, delta, wait, seq_mean)
        else:
            out[r] = _dp(rows[r], pre_max, post_max, pre_avg, post_avg, delta, wait, method == "dp_count")
    peaks = np.moveaxis(peaks, -1, axis)
    return np.flatnonzero(peaks) if sparse else peaks


def onset_backtrack(events, energy):
    energy = np.asarray(energy)
    minima = np.flatnonzero((energy[1:-1] <= energy[:-2]) & (energy[1:-1] < energy[2:])) + 1
    minima = np.unique(np.concatenate(([0], minima))).astype(np.int64)
    events = np.asarray(events)
    if len(events) == 0:
        raise ParameterError(_EMPTY_MATCH)
    if events.min() < 0:
        raise ParameterError(_NEGATIVE_MATCH)
    # the largest minimum at or before each event (minima[0] == 0 <= every event)
    return minima[np.searchsorted(minima, events, side="right") - 1]


def _units(onsets, units, hop_length, sr):
    if units == "frames":
        return onsets
    if units == "samples":
        return (np.asanyarray(onsets) * hop_length).astype(int)
    if units == "time":
        return (np.asanyarray(onsets) * hop_length).astype(int) / float(sr)
    raise ParameterError(f"Invalid unit type: {units}")


def onset_detect(*, y=None, sr=22050, onset_envelope=None, hop_length=512, backtrack=False, energy=None,
                 units="frames", normalize=True, sparse=True, **kwargs):
    """Envelope input only (``y=`` is checked on the GPU against this function run on the GPU's envelope)."""
    if onset_envelope is None:
        if y is None:
            raise ParameterError("y or onset_envelope must be provided")
        raise NotImplementedError("the oracle takes onset_envelope only")
    x = np.asarray(onset_envelope)
    if normalize:
        x = x - np.min(x, keepdims=True, axis=-1)
        x /= np.max(x, keepdims=True, axis=-1) + np.finfo(x.dtype).tiny
    if not x.any() or not np.all(np.isfinite(x)):
        onsets = np.array([], dtype=int) if sparse else np.zeros_like(x, dtype=bool)
    else:
        kwargs.setdefault("pre_max", 0.03 * sr // hop_length)
        kwargs.setdefault("post_max", 0.00 * sr // hop_length + 1)
        kwargs.setdefault("pre_avg", 0.10 * sr // hop_length)
        kwargs.setdefault("post_avg", 0.10 * sr // hop_length + 1)
        kwargs.setdefault("wait", 0.03 * sr // hop_length)
        kwargs.setdefault("delta", 0.07)
        onsets = peak_pick(x, sparse=sparse, axis=-1, **kwargs)
        if backtrack:
            if not sparse:
                raise ParameterError("onset backtracking is only supported if sparse=True")
            onsets = onset_backtrack(onsets, x if energy is None else energy)
    if sparse:
        onsets = _units(onsets, units, hop_length, sr)
    return onsets


# namespaces shaped like the library, for tests/onset_cases.run
onset = types.SimpleNamespace(onset_detect=onset_detect, onset_backtrack=onset_backtrack)
util = types.SimpleNamespace(peak_pick=peak_pick)
