"""NumPy restatement of the reference's alignment (librosa/sequence.py:185-1172, util/utils.py:2003-2067), vectorised
per anti-diagonal so that grids of tens of millions of cells run in seconds.  It reproduces every entry of
tests/golden/alignment_v1.npz bit for bit (tests/test_alignment_host.py), and the GPU tests hold the kernels to it.

The arithmetic is the reference's: cdist's metrics as sequential, unfused float64 sums over the features (cosine with
two interleaved partial sums), the dtw step scan in table order taking strictly better costs, and rqa's float64
candidates rounded once to sim's dtype."""
from __future__ import annotations

import numpy as np

DEFAULT_STEPS = np.array([[1, 1], [0, 1], [1, 0]], dtype=np.uint32)
METRICS = ("euclidean", "sqeuclidean", "cityblock", "chebyshev", "cosine")


def feature_matrix(x):
    """(frames, features) in the reference's order: swapaxes(x, -1, 0).reshape(N, -1, order="F"), as float64."""
    x = np.atleast_2d(x)
    return np.swapaxes(x, -1, 0).reshape((x.shape[-1], -1), order="F").astype(np.float64)


def cost(X, Y, metric="euclidean"):
    from scipy.spatial import distance

    metric = distance._METRIC_ALIAS[metric.lower()].canonical_name    # cdist's aliases ("Euclid", "cos", ...)
    a, b = feature_matrix(X), feature_matrix(Y)
    K = a.shape[1]
    if metric == "cosine":
        part = [[np.zeros((a.shape[0], b.shape[0])) for _ in range(2)] for _ in range(3)]
        xx, yy = [np.zeros((a.shape[0], 1)) for _ in range(2)], [np.zeros((1, b.shape[0])) for _ in range(2)]
        pairs = K // 2 * 2
        for f in range(pairs):
            u, v = a[:, f:f + 1], b[:, f][None]
            part[0][f & 1] = part[0][f & 1] + u * v
            xx[f & 1] = xx[f & 1] + u * u
            yy[f & 1] = yy[f & 1] + v * v
        sxy, sxx, syy = part[0][0] + part[0][1], xx[0] + xx[1], yy[0] + yy[1]
        if pairs < K:
            u, v = a[:, pairs:pairs + 1], b[:, pairs][None]
            sxy, sxx, syy = sxy + u * v, sxx + u * u, syy + v * v
        with np.errstate(invalid="ignore", divide="ignore"):
            c = sxy / (np.sqrt(sxx) * np.sqrt(syy))
        c = np.where(np.abs(c) > 1, np.copysign(1.0, c), c)
        return 1.0 - c
    r = np.zeros((a.shape[0], b.shape[0]))
    for f in range(K):
        d = a[:, f:f + 1] - b[:, f][None]
        if metric == "cityblock":
            r = r + np.abs(d)
        elif metric == "chebyshev":
            r = np.where(r < np.abs(d), np.abs(d), r)
        else:
            r = r + d * d
    return np.sqrt(r) if metric == "euclidean" else r


def band(shape, band_rad):
    radius = int(np.round(band_rad * np.min(shape)))
    offset = abs(shape[0] - shape[1])
    return (-radius, radius + offset) if shape[0] < shape[1] else (-radius - offset, radius)


def fill_off_diagonal(x, radius, value=0):
    lo, hi = band(x.shape, radius)
    d = np.arange(x.shape[1])[None, :] - np.arange(x.shape[0])[:, None]
    x[(d <= lo) | (d >= hi)] = value


def step_table(step_sizes_sigma=None, weights_add=None, weights_mul=None):
    if step_sizes_sigma is None:
        return (DEFAULT_STEPS.astype(np.int64), np.zeros(3) if weights_add is None else np.asarray(weights_add, float),
                np.ones(3) if weights_mul is None else np.asarray(weights_mul, float))
    n = len(step_sizes_sigma)
    wa = np.zeros(n) if weights_add is None else weights_add
    wm = np.ones(n) if weights_mul is None else weights_mul
    return (np.concatenate((DEFAULT_STEPS, step_sizes_sigma)).astype(np.int64),
            np.concatenate((np.full(3, np.inf), wa)).astype(np.float64),
            np.concatenate((np.full(3, np.inf), wm)).astype(np.float64))


def accumulate(C, steps_tab, w_add, w_mul, subseq=False):
    """D (float64) and steps (int32), one anti-diagonal at a time."""
    N, M = C.shape
    C = C.astype(np.float64)
    D = np.full((N, M), np.inf)
    S = np.zeros((N, M), dtype=np.int32)
    for d in range(N + M - 1):
        i = np.arange(max(0, d - M + 1), min(d, N - 1) + 1)
        j = d - i
        c = C[i, j]
        best = np.where((i == 0) & ((j == 0) | bool(subseq)), c, np.inf)
        st = np.zeros(i.size, dtype=np.int32)
        for k, (a, b) in enumerate(steps_tab):
            if a == 0 and b == 0:
                pred = best
            else:
                ok = (i >= a) & (j >= b)
                pred = np.full(i.size, np.inf)
                pred[ok] = D[i[ok] - a, j[ok] - b]
            with np.errstate(invalid="ignore"):
                cost_k = pred + (w_mul[k] * c + w_add[k])
            better = cost_k < best
            best = np.where(better, cost_k, best)
            st = np.where(better, k, st)
        D[i, j] = best
        S[i, j] = st
    return D, S


def backtrack(steps, steps_tab, subseq, start=None):
    """The reference's walk (a (0, 0) step would loop forever; it raises here instead)."""
    n, m = steps.shape
    i, j = n - 1, (m - 1 if start is None else start)
    wp = [(i, j)]
    while (subseq and i > 0) or (not subseq and (i, j) != (0, 0)):
        a, b = steps_tab[steps[i, j]]
        if a == 0 and b == 0:
            raise RuntimeError("a (0, 0) step")
        i, j = i - a, j - b
        if min(i, j) < 0:
            break
        wp.append((i, j))
    return np.asarray(wp, dtype=np.int64)


def dtw(X=None, Y=None, *, C=None, metric="euclidean", step_sizes_sigma=None, weights_add=None, weights_mul=None,
        subseq=False, backtrack_path=True, global_constraints=False, band_rad=0.25):
    """(D, wp or None, steps); the reference's errors are not restated here."""
    transposed = False
    if C is None:
        C = cost(X, Y, metric)
        if subseq and C.shape[0] > C.shape[1]:
            C, transposed = C.T, True
    C = np.atleast_2d(C).astype(np.float64)
    if global_constraints:
        C = C.copy()
        fill_off_diagonal(C, band_rad, np.inf)
    tab, wa, wm = step_table(step_sizes_sigma, weights_add, weights_mul)
    D, S = accumulate(C, tab, wa, wm, subseq)
    wp = None
    if backtrack_path:
        start = int(np.argmin(D[-1])) if subseq else None
        wp = backtrack(S, tab, subseq, start)
        if subseq and (transposed or C.shape[0] > C.shape[1]):
            wp = np.fliplr(wp)
    return D, wp, S


def _first_argmax(cands):
    """np.argmax over the candidate axis (the first NaN, else the first maximum) and the chosen values."""
    bv, bi = cands[0].copy(), np.zeros(cands[0].shape, dtype=np.int8)
    for k in range(1, len(cands)):
        take = ~np.isnan(bv) & (np.isnan(cands[k]) | (cands[k] > bv))
        bv = np.where(take, cands[k], bv)
        bi = np.where(take, k, bi)
    return bv, bi


def _rqa_cells(sim, score, ptr, i, j, cand, gap_onset, gap_extend):
    """One vector of cells (i, j) with candidate cells cand [(ci, cj), ...]."""
    s = sim[i, j]
    sv = [score[ci, cj].astype(np.float64) for ci, cj in cand]
    with np.errstate(invalid="ignore"):
        pos = s > 0
        bv, bi = _first_argmax(sv)
        up = (bv + s.astype(np.float64)).astype(sim.dtype)
        vec = []
        for (ci, cj), v in zip(cand, sv):
            t = (sim[ci, cj] > 0).astype(np.float64)
            vec.append(v - t * gap_onset - (1.0 - t) * gap_extend)
        gv, gi = _first_argmax(vec)
        gap = np.where(gv > 0, gv, 0.0).astype(sim.dtype)
    score[i, j] = np.where(pos, up, gap)
    ptr[i, j] = np.where(pos, bi, np.where(gap == 0, -1, gi))


def rqa(sim, gap_onset=1, gap_extend=1, knight_moves=True):
    """(score in sim's dtype, int8 pointers)."""
    sim = np.asarray(sim)
    N, M = sim.shape
    score = np.zeros(sim.shape, dtype=sim.dtype)
    ptr = np.zeros(sim.shape, dtype=np.int8)
    score[0, :] = sim[0, :]
    score[:, 0] = sim[:, 0]
    ptr[:, 0] = np.where(sim[:, 0] != 0, -2, -1)
    ptr[0, :] = np.where(sim[0, :] != 0, -2, -1)
    if N == 1 or M == 1:
        return score, ptr
    go, ge = float(gap_onset), float(gap_extend)
    if sim[1, 1] > 0:
        score[1, 1] = score[0, 0] + sim[1, 1]
        ptr[1, 1] = 0
    else:
        link = 1.0 if sim[0, 0] > 0 else 0.0
        with np.errstate(invalid="ignore"):
            v = float(score[0, 0]) - link * go - (1.0 - link) * ge
        score[1, 1] = v if v > 0 else 0.0
        ptr[1, 1] = 0 if score[1, 1] > 0 else -1
    lim = 2 if knight_moves else 1
    j = np.arange(2, M)
    if j.size:
        i = np.ones_like(j)
        _rqa_cells(sim, score, ptr, i, j, [(i - 1, j - 1), (i - 1, j - 2)][:lim], go, ge)
    i = np.arange(2, N)
    if i.size:
        j = np.ones_like(i)
        _rqa_cells(sim, score, ptr, i, j, [(i - 1, j - 1), (i - 2, j - 1)][:lim], go, ge)
    lim = 3 if knight_moves else 1
    for d in range(4, N + M - 1):
        i = np.arange(max(2, d - M + 1), min(d - 2, N - 1) + 1)
        if not i.size:
            continue
        j = d - i
        _rqa_cells(sim, score, ptr, i, j, [(i - 1, j - 1), (i - 1, j - 2), (i - 2, j - 1)][:lim], go, ge)
    return score, ptr


def rqa_path(score, ptr):
    """The reference's walk, with its Python indexing (a column index of -1 reads the last column)."""
    offsets = [(-1, -1), (-1, -2), (-2, -1)]
    idx = list(np.unravel_index(np.argmax(score), score.shape))
    path = []
    while True:
        bt = ptr[tuple(idx)]
        if bt == -1:
            break
        path.insert(0, idx)
        if bt == -2:
            break
        idx = [idx[k] + offsets[bt][k] for k in range(2)]
    if not path:
        return np.empty((0, 2), dtype=np.uint)
    return np.asarray(path, dtype=np.int64).astype(np.uint64)


def path_to_steps(path, inverse=False):
    import scipy.interpolate

    idx_from, idx_to = (1, 0) if inverse else (0, 1)
    f = scipy.interpolate.interp1d(path[:, idx_to], path[:, idx_from], kind="linear")
    return f(np.arange(path[:, idx_to].min(), path[:, idx_to].max() + 1))


def run(case, C_override=None):
    """The outputs of one non-error case of tests/alignment_cases.py, keyed as the fixture keys them.  C_override
    replaces the cost matrix dtw accumulates (the GPU tests pass the kernel's own)."""
    import alignment_cases as AC

    X, Y, C, sim = AC.inputs(case)
    op, kw = case["op"], dict(case["kw"])
    if op == "dtw":
        bt, steps_out = kw.pop("backtrack", True), kw.pop("return_steps", False)
        if C_override is not None:
            transposed = C is None and kw.get("subseq") and C_override.shape[0] < np.shape(X)[-1]
            D, wp, S = dtw(C=C_override, backtrack_path=bt, **{k: v for k, v in kw.items() if k != "metric"})
            if transposed and wp is not None:
                wp = np.fliplr(wp)
        else:
            D, wp, S = dtw(X, Y, C=C, backtrack_path=bt, **kw)
        out = {"D": D}
        if bt:
            out["wp"] = wp
        if steps_out:
            out["steps"] = S
        return out
    if op in ("dtw_backtracking", "path_to_steps"):
        bt_kw = {k: v for k, v in kw.items() if k in ("subseq", "step_sizes_sigma")}
        D, wp, S = dtw(C=C, **bt_kw)
        if op == "path_to_steps":
            return {"steps": path_to_steps(wp, **kw)}
        tab = step_table(kw.get("step_sizes_sigma"))[0]
        return {"wp": backtrack(S, tab, kw.get("subseq", False), kw.get("start")), "dtw_wp": wp}
    if op == "fill_off_diagonal":
        x = np.array(C)
        fill_off_diagonal(x, kw["radius"], kw["value"])
        return {"x": x}
    if op == "rqa":
        bt = kw.pop("backtrack", True)
        score, ptr = rqa(sim, **kw)
        return {"score": score, "path": rqa_path(score, ptr)} if bt else {"score": score}
    raise ValueError(op)
