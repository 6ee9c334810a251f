"""NumPy / SciPy restatement of the reference's cqt / vqt for the cases of tests/cqt_cases.py: the host plan and
filter bases of librosa_b200.core.constantq (pinned to the fixture on their own by tests/test_cqt_host.py), the
oracle's polyphase resampler and STFT, and the projection written out as separate float32 operations in the
order SciPy's csr_matvecs uses (``project``).  Reproduces every C of tests/golden/cqt_v1.npz bit for bit."""
from __future__ import annotations

import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from librosa_b200.core import constantq as Q  # noqa: E402
from oracle import ref_np as O  # noqa: E402


def resolved(case, y):
    """(vqt keyword arguments with the reference's defaults, fmin with tuning applied)."""
    kw = dict(sr=22050, hop_length=512, fmin=None, n_bins=84, intervals="equal", gamma=0 if case["fn"] == "cqt" else None,
              bins_per_octave=12, tuning=0.0, filter_scale=1, norm=1, sparsity=0.01, window="hann", scale=True,
              pad_mode="constant", res_type="soxr_hq", dtype=None)
    kw.update(case["kw"])
    if not isinstance(kw["intervals"], str):
        kw["bins_per_octave"] = len(kw["intervals"])
    fmin = Q._default_fmin() if kw["fmin"] is None else kw["fmin"]
    tuning = kw["tuning"]
    if tuning is None:
        tuning = O.estimate_tuning(y=y, sr=kw["sr"], bins_per_octave=kw["bins_per_octave"])
    return kw, fmin * 2.0 ** (tuning / kw["bins_per_octave"])


def plan(case, y):
    kw, fmin = resolved(case, y)
    p = Q.plan(y.shape[-1], sr=kw["sr"], hop_length=kw["hop_length"], fmin=fmin, n_bins=kw["n_bins"],
               intervals=kw["intervals"], gamma=kw["gamma"], bins_per_octave=kw["bins_per_octave"],
               filter_scale=kw["filter_scale"], window=kw["window"], scale=kw["scale"], res_type=kw["res_type"])
    return kw, p


def bases(case, y):
    kw, p = plan(case, y)
    return Q.bases(p, filter_scale=kw["filter_scale"], norm=kw["norm"], sparsity=kw["sparsity"],
                   window=kw["window"], gamma=kw["gamma"])


def project(indptr, indices, data, D):
    """``csr @ D`` for complex64, one output row at a time: per nonzero in storage order, the complex product as
    unfused float32 multiplies and adds, added to the running sum."""
    D = np.asarray(D)
    out = np.zeros((len(indptr) - 1, D.shape[-1]), dtype=np.complex64)
    xr, xi = D.real.astype(np.float32), D.imag.astype(np.float32)
    for r in range(len(indptr) - 1):
        re = np.zeros(D.shape[-1], np.float32)
        im = np.zeros(D.shape[-1], np.float32)
        for k in range(indptr[r], indptr[r + 1]):
            vr, vi = np.float32(data[k].real), np.float32(data[k].imag)
            c = indices[k]
            re = re + (vr * xr[c] - vi * xi[c])
            im = im + (vr * xi[c] + vi * xr[c])
        out[r].real, out[r].imag = re, im
    return out


def cqt(case):
    """The reference's C for one case (complex64 for float32 audio, complex128 for float64 audio)."""
    import cqt_cases as QC
    import scipy.sparse

    y = QC.signal(case["sig"])
    kw, p = plan(case, y)
    dtype = np.dtype(kw["dtype"]) if kw["dtype"] is not None else O.dtype_r2c(y.dtype)
    bs = Q.bases(p, filter_scale=kw["filter_scale"], norm=kw["norm"], sparsity=kw["sparsity"], window=kw["window"],
                 gamma=kw["gamma"])
    if p.early > 1:
        y = O.resample(y, orig_sr=p.early, target_sr=1, res_type="polyphase", scale=True)
        if not kw["scale"]:
            y *= np.sqrt(p.early)
    resp = []
    for o, b in zip(p.octaves, bs):
        D = O.stft(y, n_fft=o.n_fft, hop_length=o.hop, window="ones", pad_mode=kw["pad_mode"], dtype=dtype)
        basis = scipy.sparse.csr_array((b.data.astype(dtype), b.indices, b.indptr),
                                       shape=(len(b.indptr) - 1, o.n_fft // 2 + 1))
        if dtype != np.complex64:   # the reference's basis in this dtype, scaled in it
            basis = _wide_basis(case, y, o, p, kw, dtype)
        Dr = D.reshape((-1,) + D.shape[-2:])
        resp.append(np.stack([basis @ d for d in Dr]).reshape(D.shape[:-2] + (basis.shape[0], D.shape[-1])))
        if o.resample_after:
            y = O.resample(y, orig_sr=2, target_sr=1, res_type="polyphase", scale=True)
    T = min(r.shape[-1] for r in resp)
    V = np.empty(resp[0].shape[:-2] + (p.n_bins, T), dtype=dtype, order="F")
    end = p.n_bins
    for r in resp:
        n_oct = r.shape[-2]
        if end < n_oct:
            V[..., :end, :] = r[..., -end:, :T]
        else:
            V[..., end - n_oct:end, :] = r[..., :T]
        end -= n_oct
    if kw["scale"]:
        V /= np.sqrt(p.lengths)[:, np.newaxis]
    return V


def _wide_basis(case, y, o, p, kw, dtype):
    """A complex128 octave basis: sparsified in complex128 and scaled there, as the reference does for dtype=
    complex128 (float64 audio or an explicit dtype)."""
    import scipy.fft
    import scipy.sparse

    from librosa_b200 import filters

    basis, lengths = filters.wavelet(freqs=p.freqs[o.rows], sr=o.sr, filter_scale=kw["filter_scale"], norm=kw["norm"],
                                     pad_fft=True, window=kw["window"], gamma=kw["gamma"], alpha=p.alpha[o.rows])
    n_fft = basis.shape[1]
    basis *= lengths[:, np.newaxis] / float(n_fft)
    fft_basis = scipy.fft.fft(basis, n=n_fft, axis=1)[:, : (n_fft // 2) + 1]
    m = scipy.sparse.csr_array(Q._sparsify(fft_basis, kw["sparsity"], dtype))
    m.data *= np.sqrt(p.sr / o.sr)
    return m
