"""NumPy restatement of ``librosa.beat.beat_track`` and its tracker stages (librosa/beat.py:44-317, :510-742).

The reference's tracker is numba code: every scalar ``log`` / ``exp`` is the C library's (math.log / math.exp here, and
libm's logf for float32 data), ``x ** 2`` is ``x * x``, sums are left to right, and float32 data keep float32
storage with float64 arithmetic in between.  The tempo comes from tests/rhythm_oracle.py."""
from __future__ import annotations

import ctypes
import ctypes.util
import math

import numpy as np

import rhythm_oracle as RO
from oracle import ref_np as O
from rhythm_oracle import ParameterError

_libm = ctypes.CDLL(ctypes.util.find_library("m") or "libm.so.6")
_libm.logf.restype = ctypes.c_float
_libm.logf.argtypes = [ctypes.c_float]


def window(fpb):
    """exp(-0.5 * (arange(-fpb, fpb + 1) * 32.0 / fpb) ** 2), element by element with libm."""
    f = float(fpb)
    out = []
    for d in range(-int(fpb), int(fpb) + 1):
        x = float(d) * 32.0 / f
        out.append(math.exp(-0.5 * (x * x)))
    return np.array(out)


def normalize_onsets(x):
    return x / (x.std(ddof=1, axis=-1, keepdims=True) + np.finfo(x.dtype).tiny)


def local_score(x, fpb):
    """One row: localscore[i] += window[k] * x[i + K//2 - k] for k ascending, each sum rounded to x's type."""
    n = x.shape[-1]
    t = x.dtype.type
    out = np.zeros(n, dtype=x.dtype)
    tv = fpb.shape[-1] == n and n > 1
    wins = {f: window(f) for f in np.unique(fpb)}
    for i in range(n):
        f = int(fpb[i] if tv else fpb[0])
        w = wins[f]
        K = 2 * f + 1
        acc = t(0)
        for k in range(max(0, i + K // 2 - n + 1), min(i + K // 2, K)):
            acc = t(float(acc) + w[k] * float(x[i + K // 2 - k]))
        out[i] = acc
    return out


def _round_half_even(v):
    return int(round(v))


def track_dp(ls, fpb, tightness):
    """One row of the DP: (backlink int32, cumscore).  Numba runs the float64 loop unless localscore and fpb are
    both float32."""
    n = ls.shape[-1]
    f64 = ls.dtype == np.float64 or fpb.dtype == np.float64
    t = np.float64 if f64 else np.float32
    tight = float(np.float32(tightness))
    tv = fpb.shape[-1] > 1
    mx = ls.max() if not np.isnan(ls).any() else np.nan
    score_thresh = 0.01 * float(mx)
    cum = np.zeros(n, dtype=t)
    back = np.zeros(n, dtype=np.int32)
    first = True
    logs = {}
    for i in range(n):
        f = float(fpb[i] if tv else fpb[0])
        if f not in logs:
            logs[f] = math.log(f) if f64 else float(_libm.logf(f))
        lf = logs[f]
        best, loc_best = -np.inf, -1
        hi = i - _round_half_even(f / 2)
        lo_ex = int(i - 2 * f - 1)
        for loc in range(hi, lo_ex, -1):
            if loc < 0:
                break
            if loc == i:          # log(0): the score is -inf or NaN and never wins
                continue
            d = math.log(i - loc) - lf
            s = float(cum[loc]) - tight * (d * d)
            if s > best:
                best, loc_best = s, loc
        si = ls[i]
        cum[i] = t(float(si) + best) if loc_best >= 0 else si
        if first and float(si) < score_thresh:
            back[i] = -1
        else:
            back[i] = loc_best
            first = False
    return back, cum


def localmax(x):
    """util.localmax along the last axis (edge padding)."""
    pad = np.concatenate([x[..., :1], x, x[..., -1:]], axis=-1)
    return (x > pad[..., :-2]) & (x >= pad[..., 2:])


def last_beat(cum):
    mask = ~localmax(cum)
    med = np.ma.median(np.ma.masked_array(data=cum, mask=mask), axis=-1)
    thr = 0.5 * np.ma.getdata(med)
    n = cum.shape[-1] - 1
    while n >= 0:
        if not mask[n] and cum[n] >= thr:
            return n
        n -= 1
    return cum.shape[-1] - 1


def backtrack(back, tail, n):
    beats = np.zeros(n, dtype=bool)
    t = tail
    while t >= 0:
        beats[t] = True
        t = back[t]
    return beats


def trim_beats(ls, beats, trim):
    """__trim_beats, with the frame loops bounded (an all-zero row clears every frame)."""
    out = beats.copy()
    n = ls.shape[-1]
    w = np.hanning(5)
    smooth = np.convolve(ls[beats], w)[len(w) // 2: n + len(w) // 2]
    if trim:
        acc = 0.0
        for v in smooth ** 2:
            acc += float(v)
        thr = 0.5 * ((acc / smooth.size) ** 0.5)
    else:
        thr = 0.0
    i = 0
    while i < n and ls[i] <= thr:
        out[i] = False
        i += 1
    i = n - 1
    while i >= 0 and ls[i] <= thr:
        out[i] = False
        i -= 1
    return out


def frames_per_beat(bpm, sr, hop_length, shape):
    _bpm = np.atleast_1d(bpm)
    bpm_expanded = _bpm.reshape(_bpm.shape + (1,) * (len(shape) - _bpm.ndim))
    return bpm_expanded, np.round(float(sr) / hop_length * 60.0 / bpm_expanded)


def track_stages(x, fpb, tightness=100, trim=True):
    """Every row of ``x`` (..., n): dict of localscore, cumscore, backlink, tail and the dense beats."""
    lead, n = x.shape[:-1], x.shape[-1]
    fpb = np.broadcast_to(fpb, lead + (fpb.shape[-1],))
    xn = normalize_onsets(x)
    out = {k: [] for k in ("localscore", "cumscore", "backlink", "tail", "beats")}
    for idx in np.ndindex(*lead):
        ls = local_score(xn[idx], fpb[idx])
        back, cum = track_dp(ls, fpb[idx], tightness)
        tail = last_beat(cum)
        out["localscore"].append(ls)
        out["cumscore"].append(cum)
        out["backlink"].append(back)
        out["tail"].append(tail)
        out["beats"].append(trim_beats(ls, backtrack(back, tail, n), trim))
    res = {k: np.array(v).reshape(lead + np.shape(v[0])) for k, v in out.items()}
    res["tail"] = res["tail"].astype(np.int64)
    return res


def plp_keep(freqs, tempo_min, tempo_max):
    keep = np.ones(freqs.shape, dtype=bool)
    if tempo_min is not None:
        keep &= ~(freqs < tempo_min)
    if tempo_max is not None:
        keep &= ~(freqs > tempo_max)
    return keep


def plp_select(ftgram, keep, logprior=None):
    """plp's step 3 on (..., bins, frames): returns (selected tempogram, ftmag)."""
    ftgram = ftgram.copy()
    ftgram[..., ~keep, :] = 0
    ftmag = np.log1p(1e6 * np.abs(ftgram))
    if logprior is not None:
        ftmag += logprior[:, None]
    peak = ftmag.max(axis=-2, keepdims=True)
    ftgram[ftmag < peak] = 0
    ftgram /= np.finfo(ftgram.real.dtype).tiny ** 0.5 + np.abs(ftgram.max(axis=-2, keepdims=True))
    return ftgram, ftmag


def plp_fragile(ftgram, keep, logprior=None):
    """Frames whose selection hangs on the last bits: the top two ftmag within 1e-5 relative, or a surviving peak
    whose real part is within 1e-5 |X| of zero (its sign decides the lexicographic complex max)."""
    sel, ftmag = plp_select(ftgram, keep, logprior)
    top2 = -np.sort(-ftmag, axis=-2)[..., :2, :]
    close = np.abs(top2[..., 0, :] - top2[..., 1, :]) <= 1e-5 * np.abs(top2[..., 0, :])
    z = np.where(sel != 0, ftgram, 0)
    tiny_re = np.any((z != 0) & (np.abs(z.real) < 1e-5 * np.abs(z)), axis=-2)
    return close | tiny_re


class _Beat:
    @staticmethod
    def beat_track(*, y=None, sr=22050, onset_envelope=None, hop_length=512, start_bpm=120.0, tightness=100,
                   trim=True, bpm=None, prior=None, units="frames", sparse=True):
        if onset_envelope is None:
            raise ParameterError("y or onset_envelope must be provided")
        if sparse and onset_envelope.ndim != 1:
            raise ParameterError(f"sparse=True (default) does not support "
                                 f"{onset_envelope.ndim}-dimensional inputs. "
                                 f"Either set sparse=False or convert the signal to mono.")
        if not onset_envelope.any():
            if sparse:
                return 0.0, np.array([], dtype=int)
            return np.zeros(onset_envelope.shape[:-1], dtype=float), np.zeros_like(onset_envelope, dtype=bool)
        if bpm is None:
            bpm = RO.tempo(onset_envelope=onset_envelope, sr=sr, hop_length=hop_length, start_bpm=start_bpm,
                           prior=prior)
        bpm_expanded, fpb = frames_per_beat(bpm, sr, hop_length, onset_envelope.shape)
        if np.any(bpm_expanded <= 0):
            raise ParameterError(f"bpm={bpm_expanded} must be strictly positive")
        if tightness <= 0:
            raise ParameterError("tightness must be strictly positive")
        if bpm_expanded.shape[-1] not in (1, onset_envelope.shape[-1]):
            raise ParameterError(f"Invalid bpm shape={bpm_expanded.shape} does not match "
                                 f"onset envelope shape={onset_envelope.shape}")
        beats = track_stages(onset_envelope, fpb, tightness, trim)["beats"]
        if sparse:
            beats = np.flatnonzero(beats)
            if units == "frames":
                pass
            elif units == "samples":
                return bpm, (beats * hop_length).astype(int)
            elif units == "time":
                return bpm, (beats * hop_length).astype(int) / float(sr)
            else:
                raise ParameterError(f"Invalid unit type: {units}")
        return bpm, beats


    @staticmethod
    def plp(*, y=None, sr=22050, onset_envelope=None, hop_length=512, win_length=384, tempo_min=30, tempo_max=300,
            prior=None):
        if tempo_min is not None and tempo_max is not None and tempo_max <= tempo_min:
            raise ParameterError(f"tempo_max={tempo_max} must be larger than tempo_min={tempo_min}")
        ft = RO.fourier_tempogram(onset_envelope=onset_envelope, sr=sr, hop_length=hop_length, win_length=win_length)
        freqs = RO.fourier_tempo_frequencies(sr=sr, hop_length=hop_length, win_length=win_length)
        logprior = None if prior is None else prior.logpdf(freqs)
        sel, _ = plp_select(ft, plp_keep(freqs, tempo_min, tempo_max), logprior)
        pulse = O.istft(sel, hop_length=1, n_fft=win_length, length=onset_envelope.shape[-1])
        pulse = np.clip(pulse, 0, None, pulse)
        return O.normalize(pulse, axis=-1)


beat = _Beat()
