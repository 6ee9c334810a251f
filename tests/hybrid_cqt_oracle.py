"""NumPy / SciPy restatement of the reference's pseudo_cqt and hybrid_cqt for the cases of tests/hybrid_cqt_cases.py:
the host plan, split and |basis| of librosa_b200.core.constantq (pinned to the fixture on their own by
tests/test_hybrid_cqt_host.py), the oracle's Hann STFT, SciPy's float32 ``csr @ np.abs(D)`` (restated as separate
float32 operations by ``project_abs``), numpy's float64 scaling, and for the full part tests/cqt_oracle.py's cqt.
Reproduces every C of tests/golden/hybrid_cqt_v1.npz bit for bit."""
from __future__ import annotations

import numpy as np
import scipy.sparse

import cqt_oracle as QO
import hybrid_cqt_cases as HC
from librosa_b200.core import constantq as Q
from oracle import ref_np as O

DEFAULTS = dict(sr=22050, hop_length=512, fmin=None, n_bins=84, bins_per_octave=12, tuning=0.0, filter_scale=1, norm=1,
                sparsity=0.01, window="hann", scale=True, pad_mode="constant", res_type="soxr_hq", dtype=None)


def resolved(case, y):
    """(keyword arguments with the reference's defaults, fmin with tuning applied)."""
    kw = dict(DEFAULTS, **case["kw"])
    fmin = Q._default_fmin() if kw["fmin"] is None else kw["fmin"]
    tuning = kw["tuning"]
    if tuning is None:
        tuning = O.estimate_tuning(y=y, sr=kw["sr"], bins_per_octave=kw["bins_per_octave"])
    return kw, fmin * 2.0 ** (tuning / kw["bins_per_octave"])


def _pseudo_plan(kw, n, fmin, n_bins):
    return Q.pseudo_plan(n, sr=kw["sr"], hop_length=kw["hop_length"], fmin=fmin, n_bins=n_bins,
                         bins_per_octave=kw["bins_per_octave"], filter_scale=kw["filter_scale"], window=kw["window"])


def split(case, y):
    """(kw, tuned fmin, pseudo plan or None, n_full): what hybrid_cqt hands to pseudo_cqt and cqt; pseudo_cqt's own
    call for a pseudo_cqt case."""
    kw, fmin = resolved(case, y)
    if case["fn"] == "pseudo_cqt":
        return kw, fmin, _pseudo_plan(kw, y.shape[-1], fmin, kw["n_bins"]), 0
    freqs, _, lengths = Q._equal_bins(sr=kw["sr"], fmin=fmin, n_bins=kw["n_bins"],
                                      bins_per_octave=kw["bins_per_octave"], filter_scale=kw["filter_scale"],
                                      window=kw["window"])
    is_pseudo = Q.hybrid_split(lengths, kw["hop_length"])
    n_pseudo = int(np.sum(is_pseudo))
    pp = _pseudo_plan(kw, y.shape[-1], np.min(freqs[is_pseudo]), n_pseudo) if n_pseudo else None
    return kw, fmin, pp, len(freqs) - n_pseudo


def basis(kw, pp):
    """The GPU's |basis| table (float32 magnitudes in complex64 real parts) as a float32 CSR matrix."""
    b = Q.pseudo_basis(pp, filter_scale=kw["filter_scale"], norm=kw["norm"], sparsity=kw["sparsity"],
                       window=kw["window"])
    return scipy.sparse.csr_array((b.data.real.astype(np.float32), b.indices, b.indptr),
                                  shape=(len(b.indptr) - 1, pp.n_fft // 2 + 1))


def _wide_basis(kw, pp, dtype):
    """The reference's |basis| for dtype=complex128: sparsified in complex128, magnitudes in float64."""
    import scipy.fft

    from librosa_b200 import filters

    w, lengths = filters.wavelet(freqs=pp.freqs, sr=pp.sr, filter_scale=kw["filter_scale"], norm=kw["norm"],
                                 pad_fft=True, window=kw["window"], alpha=pp.alpha)
    w *= lengths[:, np.newaxis] / float(pp.n_fft)
    fft_basis = scipy.fft.fft(w, n=pp.n_fft, axis=1)[:, : (pp.n_fft // 2) + 1]
    return abs(scipy.sparse.csr_array(Q._sparsify(fft_basis, kw["sparsity"], dtype)))


def project_abs(indptr, indices, data, D):
    """``csr @ np.abs(D)`` for float32, one output row at a time: per nonzero in storage order, an unfused float32
    multiply added to the running sum."""
    X = np.abs(np.asarray(D))
    out = np.zeros((len(indptr) - 1, X.shape[-1]), dtype=np.float32)
    for r in range(len(indptr) - 1):
        acc = np.zeros(X.shape[-1], np.float32)
        for k in range(indptr[r], indptr[r + 1]):
            acc = acc + np.float32(data[k]) * X[indices[k]]
        out[r] = acc
    return out


def scale_pseudo(C, pp, scale):
    """pseudo_cqt's scaling, as numpy does it in place (float64 right-hand sides, one rounding)."""
    if scale:
        C /= np.sqrt(pp.n_fft)
    else:
        C *= np.sqrt(pp.lengths / pp.n_fft)[:, np.newaxis]
    return C


def pseudo_part(kw, pp, y, dtype):
    m = _wide_basis(kw, pp, dtype) if dtype != np.complex64 else basis(kw, pp)
    D = np.abs(O.stft(y, n_fft=pp.n_fft, hop_length=kw["hop_length"], window="hann", pad_mode=kw["pad_mode"],
                      dtype=dtype))
    Dr = D.reshape((-1,) + D.shape[-2:])
    C = np.stack([m @ d for d in Dr]).reshape(D.shape[:-2] + (pp.n_bins, D.shape[-1]))
    return scale_pseudo(C, pp, kw["scale"])


def full_case(case, kw, fmin, n_full):
    """hybrid_cqt's cqt call as a tests/cqt_cases.py-style case."""
    sub = {k: kw[k] for k in ("sr", "hop_length", "bins_per_octave", "filter_scale", "norm", "sparsity", "window",
                              "scale", "pad_mode", "res_type", "dtype")}
    return {"name": case["name"] + "/full", "fn": "cqt", "kw": dict(sub, fmin=fmin, n_bins=n_full), "sig": case["sig"]}


def run(case):
    """The reference's C for one case."""
    y = HC.signal(case["sig"])
    kw, fmin, pp, n_full = split(case, y)
    dtype = np.dtype(kw["dtype"]) if kw["dtype"] is not None else O.dtype_r2c(y.dtype)
    resp = [pseudo_part(kw, pp, y, dtype)] if pp is not None else []
    if case["fn"] == "pseudo_cqt":
        return resp[0]
    if n_full:
        resp.append(np.abs(QO.cqt(full_case(case, kw, fmin, n_full))))
    T = min(r.shape[-1] for r in resp)
    n_bins = sum(r.shape[-2] for r in resp)
    out = np.empty(resp[0].shape[:-2] + (n_bins, T), dtype=resp[-1].dtype, order="F")
    end = n_bins
    for r in resp:
        out[..., end - r.shape[-2]:end, :] = r[..., :T]
        end -= r.shape[-2]
    return out
