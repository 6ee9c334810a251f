"""NumPy / SciPy restatement of the reference's iirt for the cases of tests/iirt_cases.py: np.pad, the oracle's
polyphase resampler, the filter bank of librosa_b200.filters (pinned to the reference by tests/test_iirt_host.py),
``scipy.signal.sosfiltfilt`` and the short-time mean-square power over NumPy windows.  Reproduces every entry of
tests/golden/iirt_v1.npz bit for bit.  ``leaf_program_sum`` evaluates the GPU kernel's pairwise-sum program."""
from __future__ import annotations

import os
import sys

import numpy as np
import scipy.signal

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from librosa_b200 import filters  # noqa: E402
from oracle import ref_np as O  # noqa: E402

DEFAULTS = dict(sr=22050, win_length=2048, hop_length=None, center=True, tuning=0.0, pad_mode="constant",
                flayout="sos", res_type="soxr_hq")


def resolved(case):
    """(iirt's own arguments with the reference's defaults, the filter-bank keyword arguments)."""
    kw = dict(DEFAULTS)
    extra = {}
    for k, v in case["kw"].items():
        (kw if k in DEFAULTS else extra)[k] = v
    if kw["hop_length"] is None:
        kw["hop_length"] = kw["win_length"] // 4
    return kw, extra


def padded(case, y):
    kw, _ = resolved(case)
    if not kw["center"]:
        return y
    w = [(0, 0)] * (y.ndim - 1) + [(kw["win_length"] // 2, kw["win_length"] // 2)]
    return np.pad(y, w, mode=kw["pad_mode"])


def bank(case):
    kw, extra = resolved(case)
    return filters.semitone_filterbank(tuning=kw["tuning"], flayout="sos", **extra)


def resampled(case, y):
    """The signal at every band rate other than sr: np.pad, then the oracle's polyphase resampler."""
    kw, _ = resolved(case)
    yp = padded(case, y)
    _, srs = bank(case)
    return {float(r): O.resample(yp, orig_sr=kw["sr"], target_sr=r, res_type="polyphase")
            for r in np.unique(srs) if r != kw["sr"]}


def frame_starts(n, *, sr, rate, win_length, hop_length, n_frames):
    """(factor, window, frame starts, length after util.fix_length) of a filtered signal of ``n`` samples."""
    factor = sr / rate
    hop = hop_length / factor
    w = round(win_length / factor)
    start = np.arange(0, n - w, hop)
    if len(start) < n_frames:
        n = int(np.ceil(n_frames * hop)) + w
        start = np.arange(0, n - w, hop)
    return factor, w, np.round(start).astype(int)[:n_frames], n


def stmsp(x, *, sr, rate, win_length, hop_length, n_frames):
    """factor * sum of squares over each frame's window of the filtered signal ``x`` (..., n) at ``rate``."""
    factor, w, start, n = frame_starts(x.shape[-1], sr=sr, rate=rate, win_length=win_length, hop_length=hop_length,
                                       n_frames=n_frames)
    x = O.fix_length(x, n)
    windows = x[..., start[:, None] + np.arange(w)[None, :]]
    return factor * np.sum(windows ** 2, axis=-1)


def iirt(case, signals=None):
    """(the reference's result for one case, {band: filtered signal}); ``signals`` replaces the resampled signals
    (rate -> (..., n) float32) that the oracle would compute."""
    import iirt_cases as IC

    y = IC.signal(case["sig"])
    kw, _ = resolved(case)
    yp = padded(case, y)
    sos, srs = bank(case)
    ys = resampled(case, y) if signals is None else signals
    n_frames = int(1 + (yp.shape[-1] - kw["win_length"]) // kw["hop_length"])
    out = np.empty(yp.shape[:-1] + (len(sos), n_frames), dtype=y.dtype)
    bands = {}
    for i, (s, r) in enumerate(zip(sos, srs)):
        x = yp if r == kw["sr"] else ys[float(r)]
        f = scipy.signal.sosfiltfilt(s, x, axis=-1)
        bands[i] = f
        out[..., i, :] = stmsp(f, sr=kw["sr"], rate=r, win_length=kw["win_length"], hop_length=kw["hop_length"],
                               n_frames=n_frames)
    return out, bands


def leaf_program_sum(a: np.ndarray, leaves: np.ndarray) -> np.float64:
    """Sum of ``a`` as the GPU's STMSP kernel evaluates a leaf program: each leaf summed like NumPy's pairwise_sum
    sums a block of at most 128 terms, partial sums combined on a stack in post-order."""
    stack = []
    for off, n, comb, _ in leaves:
        b = a[off:off + n]
        if n < 8:
            s = np.float64(0.0)
            for v in b:
                s = s + v
        else:
            r = b[:8].copy()
            i = 8
            while i < n - n % 8:
                r = r + b[i:i + 8]
                i += 8
            s = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]))
            for v in b[i:]:
                s = s + v
        stack.append(s)
        for _ in range(comb):
            right = stack.pop()
            stack[-1] = stack[-1] + right
    assert len(stack) == 1
    return stack[0]
