"""NumPy restatement of segment.recurrence_matrix (neighbours only: modes, sym, self; no affinity bandwidth) and of
decompose.nn_filter's aggregation, for tests/test_nn_filter_host.py and tests/test_gpu_nn_filter.py.

Distances are float64 (Gram form for euclidean, normalised rows for cosine, a zero frame at distance 1 from every
frame); the candidates of frame i are the M = min(t - 1, k + 2 width) other frames first in (distance, index) order,
the rules after that are the reference's (librosa/segment.py:648-701)."""
from __future__ import annotations

import numpy as np
import scipy.sparse


def frames(data, axis=-1):
    """The (t, features) float64 matrix the reference compares (swap axis to the front, flatten in F order)."""
    x = np.swapaxes(np.atleast_2d(data), axis, 0)
    return x.reshape((x.shape[0], -1), order="F").astype(np.float64)


def distances(X, metric):
    """Float64 distance matrix; the diagonal is +inf (a frame is not its own candidate)."""
    sq = np.einsum("ij,ij->i", X, X)
    G = X @ X.T
    if metric == "cosine":
        nrm = np.sqrt(sq)
        inv = np.where(nrm > 0, 1.0 / np.where(nrm > 0, nrm, 1.0), 0.0)
        D = np.clip(1.0 - G * inv[:, None] * inv[None, :], 0.0, 2.0)
        zero = nrm == 0
        D[zero, :] = 1.0
        D[:, zero] = 1.0
    else:
        D = np.sqrt(np.maximum(sq[:, None] + sq[None, :] - 2.0 * G, 0.0))
    np.fill_diagonal(D, np.inf)
    return D


def neighbours(D, k, width, mode):
    """Per frame i: the kept links (ascending index) before sym / self, and the candidate distances used."""
    t = D.shape[0]
    M = min(t - 1, k + 2 * width)
    out = []
    for i in range(t):
        order = np.lexsort((np.arange(t), D[i]))[:M]
        surv = [j for j in order if abs(j - i) >= width and (mode == "connectivity" or D[i, j] != 0)]
        kept = sorted(surv)[:k] if mode == "connectivity" else sorted(surv[:k])
        out.append(np.array(kept, dtype=np.int64))
    return out


def graph(data, *, k=None, width=1, metric="euclidean", sym=False, mode="connectivity", self=False, axis=-1,
          dtype=np.float64):
    """The recurrence matrix as a csc_array (distance values in ``dtype``; affinity values are the distances)."""
    X = frames(data, axis)
    t = X.shape[0]
    if k is None:
        k = 2 * np.ceil(np.sqrt(t - 2 * width + 1))
    k = int(k)
    D = distances(X, metric)
    links = neighbours(D, k, width, mode)
    rows, cols, vals = [], [], []
    sets = [set(l.tolist()) for l in links]
    for i in range(t):
        for j in links[i]:
            if sym and i not in sets[j]:
                continue
            rows.append(j), cols.append(i), vals.append(1.0 if mode == "connectivity" else D[i, j])
        if self and mode != "distance":
            rows.append(i), cols.append(i), vals.append(1.0 if mode == "connectivity" else 0.0)
    out = np.bool_ if mode == "connectivity" else dtype
    rec = scipy.sparse.csc_array((np.array(vals).astype(out), (rows, cols)), shape=(t, t))
    rec.sort_indices()
    return rec, D


def aggregate(S, rec, agg, axis=-1):
    """decompose.nn_filter given ``rec``: the reference's loop over csc columns, in stored order."""
    rec_s = scipy.sparse.csc_array(rec)
    Sw = np.swapaxes(S, 0, axis)
    out = np.empty_like(Sw)
    for i in range(len(rec_s.indptr) - 1):
        lo, hi = rec_s.indptr[i], rec_s.indptr[i + 1]
        targets = rec_s.indices[lo:hi]
        if not len(targets):
            out[i] = Sw[i]
            continue
        nb = np.take(Sw, targets, axis=0)
        out[i] = np.average(nb, axis=0, weights=rec_s.data[lo:hi]) if agg is np.average else agg(nb, axis=0)
    return np.swapaxes(out, 0, axis)


def boundary_tie(row, i, k, width, mode, delta):
    """True when frame i's links can legitimately differ between two distance computations that agree to ``delta``
    (relative): two candidates straddle one of its selection boundaries within delta, an exact tie included.  The
    boundaries are the edge of the candidate set (the M-th and (M + 1)-th nearest other frames, M = min(t - 1,
    k + 2 width)) and, in distance and affinity mode, the k-th and (k + 1)-th surviving candidates (|i - j| >= width,
    non-zero distance); a surviving distance within delta of zero may also drop out.  Ties away from a boundary
    change nothing and are not excused.  ``row``: the distances from frame i, +inf at i."""
    t = len(row)
    M = min(t - 1, k + 2 * width)
    order = np.lexsort((np.arange(t), row))   # the frame itself (+inf) last

    def close(a, b):
        return abs(a - b) <= delta * max(1.0, abs(b))

    if M < t - 1 and close(row[order[M - 1]], row[order[M]]):
        return True
    if mode != "connectivity":
        surv = [j for j in order[:M] if abs(j - i) >= width and row[j] != 0]
        if len(surv) > k and close(row[surv[k - 1]], row[surv[k]]):
            return True
        if any(close(row[j], 0.0) for j in order[:M]):
            return True
    return False


def excused_rows(got, want, D, *, k, width, mode, sym, delta):
    """Frames whose link sets differ between the csc arrays ``got`` and ``want``; each must be a boundary tie (with
    ``sym``, of the frame or of a frame in the difference, whose own selection decides the mutual link).  Returns
    them; raises AssertionError naming the first frame that is not excused."""
    out = []
    for i in range(D.shape[0]):
        g = got.indices[got.indptr[i]:got.indptr[i + 1]]
        w = want.indices[want.indptr[i]:want.indptr[i + 1]]
        if np.array_equal(g, w):
            continue
        ok = boundary_tie(D[i], i, k, width, mode, delta)
        if not ok and sym:
            ok = any(boundary_tie(D[j], j, k, width, mode, delta) for j in set(g.tolist()) ^ set(w.tolist()))
        assert ok, (i, g, w)
        out.append(i)
    return out


def case_k(t, kw):
    """The reference's k of a call with keyword arguments ``kw`` over t frames."""
    width = kw.get("width", 1)
    k = kw.get("k")
    return int(2 * np.ceil(np.sqrt(t - 2 * width + 1))) if k is None else int(k)
