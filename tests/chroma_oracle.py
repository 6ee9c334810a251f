"""NumPy / SciPy restatement of the reference's chroma_cqt / chroma_cens / chroma_vqt / tonnetz for the cases of
tests/chroma_cases.py: librosa_b200.filters.cq_to_chroma (pinned to the fixture on its own), the same einsum, and
librosa_b200.util.normalize; the y= cases take |C| from tests/cqt_oracle.py.  Reproduces every result of
tests/golden/chroma_v1.npz bit for bit.  ``cens_tail`` is also the GPU tests' yardstick for the CENS steps."""
from __future__ import annotations

import os
import sys

import numpy as np
import scipy.ndimage

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from librosa_b200 import filters  # noqa: E402
from librosa_b200.util.exceptions import ParameterError  # noqa: E402
from librosa_b200.util.utils import normalize  # noqa: E402

CQT_DEFAULTS = dict(sr=22050, hop_length=512, fmin=None, norm=np.inf, threshold=0.0, tuning=None, n_chroma=12,
                    n_octaves=7, window=None, bins_per_octave=36, cqt_mode="full")


def fold(C, M, threshold, norm):
    chroma = np.einsum("cf,...ft->...ct", M, C, optimize=True)
    if threshold is not None:
        chroma[chroma < threshold] = 0.0
    return normalize(chroma, norm=norm, axis=-2)


def quantize(chroma):
    """chroma_cens's L1 normalisation and quantisation."""
    chroma = normalize(chroma, norm=1, axis=-2)
    q = np.zeros_like(chroma)
    for step in [0.4, 0.2, 0.1, 0.05]:
        q += (chroma > step) * 0.25
    return q


def smooth(q, *, norm=2, win_len_smooth=41, smoothing_window="hann"):
    """chroma_cens's smoothing along frames and final normalisation."""
    if win_len_smooth:
        win = filters.get_window(smoothing_window, win_len_smooth + 2, fftbins=False)
        win = win / np.sum(win)
        win = win.reshape((1,) * (q.ndim - 1) + (-1,))
        q = scipy.ndimage.convolve(q, win, mode="constant")
    return normalize(q, norm=norm, axis=-2)


def cens_tail(chroma, **kw):
    """The CENS steps after chroma_cqt(norm=None)."""
    return smooth(quantize(chroma), **kw)


def tonnetz_from(chroma):
    from librosa_b200.feature.spectral import _tonnetz_phi

    return np.einsum("pc,...ci->...pi", _tonnetz_phi(chroma.shape[-2]), normalize(chroma, norm=1, axis=-2),
                     optimize=True)


def abs_cqt(case, y, kw, vqt=False):
    """|C| of a y= case through tests/cqt_oracle.py."""
    import cqt_oracle as QO

    if vqt:
        bpo = len(kw["intervals"]) if not isinstance(kw["intervals"], str) else kw["bins_per_octave"]
        ckw = dict(sr=kw["sr"], hop_length=kw["hop_length"], fmin=kw["fmin"], intervals=kw["intervals"],
                   n_bins=kw["n_octaves"] * bpo, bins_per_octave=bpo, gamma=kw["gamma"], res_type="polyphase")
    else:
        bpo = kw["n_chroma"] if kw["bins_per_octave"] is None else kw["bins_per_octave"]
        ckw = dict(sr=kw["sr"], hop_length=kw["hop_length"], fmin=kw["fmin"], n_bins=kw["n_octaves"] * bpo,
                   bins_per_octave=bpo, tuning=kw["tuning"], res_type="polyphase")
    return np.abs(QO.cqt({"fn": "vqt" if vqt else "cqt", "kw": ckw, "sig": case["sig"]}))


def chroma_cqt(case, arrays, **over):
    kw = dict(CQT_DEFAULTS)
    kw.update({k: v for k, v in case["kw"].items() if k != "res_type"})
    kw.update(over)
    bpo = kw["bins_per_octave"]
    if bpo is None:
        bpo = kw["n_chroma"]
    elif np.remainder(bpo, kw["n_chroma"]) != 0:
        raise ParameterError(f"bins_per_octave={bpo} must be an integer multiple of n_chroma={kw['n_chroma']}")
    C = arrays.get("C")
    if C is None:
        if "y" not in arrays:
            raise ParameterError("At least one of C or y must be provided to compute chroma")
        C = abs_cqt(case, arrays["y"], kw)
    M = filters.cq_to_chroma(C.shape[-2], bins_per_octave=bpo, n_chroma=kw["n_chroma"], fmin=kw["fmin"],
                             window=kw["window"])
    return fold(C, M, kw["threshold"], kw["norm"])


def run(case, arrays):
    """The reference's result for one case (or its exception)."""
    fn, kw = case["fn"], {k: v for k, v in case["kw"].items() if k != "res_type"}
    if fn == "chroma_cqt":
        return chroma_cqt(case, arrays)
    if fn == "chroma_cens":
        w = kw.pop("win_len_smooth", 41)
        if not ((w is None) or (isinstance(w, (int, np.integer)) and w > 0)):
            raise ParameterError(f"win_len_smooth={w} must be a positive integer or None")
        tail = dict(norm=kw.pop("norm", 2), win_len_smooth=w, smoothing_window=kw.pop("smoothing_window", "hann"))
        chroma = chroma_cqt(dict(case, kw=kw), arrays, norm=None)
        return cens_tail(chroma, **tail)
    if fn == "chroma_vqt":
        kw = dict(dict(sr=22050, hop_length=512, fmin=None, norm=np.inf, threshold=0.0, n_octaves=7,
                       bins_per_octave=12, gamma=0), **kw)
        if not isinstance(kw["intervals"], str):
            kw["bins_per_octave"] = len(kw["intervals"])
        V = arrays.get("V")
        if V is None:
            if "y" not in arrays:
                raise ParameterError("At least one of y or V must be provided to compute chroma")
            V = abs_cqt(case, arrays["y"], kw, vqt=True)
        M = filters.cq_to_chroma(V.shape[-2], bins_per_octave=kw["bins_per_octave"],
                                 n_chroma=kw["bins_per_octave"], fmin=kw["fmin"])
        return fold(V, M, kw["threshold"], kw["norm"])
    if fn == "tonnetz":
        if "y" not in arrays and "chroma" not in arrays:
            raise ParameterError("Either the audio samples or the chromagram must be passed as an argument.")
        chroma = arrays.get("chroma")
        if chroma is None:
            chroma = chroma_cqt(case, arrays)
        return tonnetz_from(chroma)
    raise ValueError(fn)
