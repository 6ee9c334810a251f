"""NumPy / SciPy restatement of librosa's pitch trackers: ``yin`` and ``pyin`` (librosa/core/pitch.py:369-968)
with the pieces of librosa/sequence.py they use (``viterbi`` :1174-1432, ``transition_loop`` :1905-1967,
``transition_local`` :2034-2146) and ``util.localmin`` (util/utils.py:1035-1180).

Bit-exact against the reference on every case of tests/pitch_cases.py (tests/golden/pitch_v1.npz).  The
decision stages take a CMND array of any float dtype so that the GPU's decision kernels can be checked on the
very input they received.  The Viterbi is vectorised over states: ``argmax`` over a padded predecessor matrix in
ascending order keeps the reference's first-maximum tie rule."""
from __future__ import annotations

import warnings

import numpy as np
import scipy.fft
import scipy.signal
import scipy.stats

from oracle.ref_np import ParameterError, frame, pad_center, tiny, valid_audio


def check_yin_params(sr, fmax, fmin, frame_length):
    """librosa/core/pitch.py:934-967."""
    if fmax > sr / 2:
        raise ParameterError(f"fmax={fmax:.3f} cannot exceed Nyquist frequency {sr/2}")
    if fmin >= fmax:
        raise ParameterError(f"fmin={fmin:.3f} must be less than fmax={fmax:.3f}")
    if fmin <= 0:
        raise ParameterError(f"fmin={fmin:.3f} must be strictly positive")
    if sr / fmin >= frame_length - 1:
        fmin_feasible = sr / (frame_length - 1)
        frame_length_feasible = int(np.ceil(sr / fmin) + 1)
        raise ParameterError(
            f"fmin={fmin:.3f} is too small for frame_length={frame_length} and sr={sr}. "
            f"Either increase to fmin={fmin_feasible:.3f} or frame_length={frame_length_feasible}")
    if sr / fmin >= frame_length // 2:
        fmin_optimal = sr / (frame_length / 2)
        frame_length_optimal = int(np.ceil(sr / fmin) * 2 + 1)
        warnings.warn(
            f"With fmin={fmin:.3f}, sr={sr} and frame_length={frame_length}, less than two periods of fmin "
            f"fit into the frame, which can cause inaccurate pitch detection. "
            f"Consider increasing to fmin={fmin_optimal:.3f} or frame_length={frame_length_optimal}.",
            stacklevel=3)


def autocorrelate(y, max_size, axis=-1):
    """librosa/core/audio.py:1320-1394 for real input."""
    max_size = int(min(max_size, y.shape[axis]))
    n_pad = scipy.fft.next_fast_len(2 * y.shape[axis] - 1, real=True)
    X = scipy.fft.rfft(y, n=n_pad, axis=axis)
    powspec = X.real ** 2 + X.imag ** 2                       # util.abs2
    autocorr = scipy.fft.irfft(powspec, n=n_pad, axis=axis)
    sl = [slice(None)] * autocorr.ndim
    sl[axis] = slice(max_size)
    return autocorr[tuple(sl)]


def cumulative_mean_normalized_difference(y_frames, min_period, max_period):
    """librosa/core/pitch.py:369-418: y_frames (..., frame_length, n_frames) -> (..., n_lags, n_frames).
    float32 frames give a float64 result: the running mean divides by an int64 lag range."""
    acf = autocorrelate(y_frames, max_period + 1, axis=-2)
    yf = np.square(y_frames)
    np.cumsum(yf, out=yf, axis=-2)
    k = slice(1, max_period + 1)
    yf[..., 0, :] = 0
    yf[..., k, :] = 2 * (acf[..., 0:1, :] - acf[..., k, :]) - yf[..., : k.stop - 1, :]
    num = yf[..., min_period: max_period + 1, :]
    k_range = np.r_[k].reshape((-1, 1))
    cum_mean = np.cumsum(yf[..., k, :], axis=-2) / k_range
    den = cum_mean[..., min_period - 1: max_period, :]
    return np.asarray(num / (den + tiny(den)))


def parabolic_interpolation(x, axis=-2):
    """librosa/core/pitch.py:421-477 (the numba stencil evaluates in the array's dtype; both ends are 0)."""
    xi = np.moveaxis(np.asarray(x), axis, -1)
    shifts = np.zeros_like(xi)
    a = xi[..., 2:] + xi[..., :-2] - 2 * xi[..., 1:-1]
    b = (xi[..., 2:] - xi[..., :-2]) / 2
    with np.errstate(divide="ignore", invalid="ignore"):
        shifts[..., 1:-1] = np.where(np.abs(b) >= np.abs(a), 0, -b / a)
    return np.moveaxis(shifts, -1, axis)


def localmin(x, axis=0):
    """librosa/util/utils.py:1121-1180: x[i] < x[i-1] and x[i] <= x[i+1]; first False, last x[-1] < x[-2]."""
    xi = np.moveaxis(np.asarray(x), axis, -1)
    out = np.zeros(xi.shape, dtype=bool)
    out[..., 1:-1] = (xi[..., 1:-1] < xi[..., :-2]) & (xi[..., 1:-1] <= xi[..., 2:])
    out[..., -1] = xi[..., -1] < xi[..., -2]
    return np.moveaxis(out, -1, axis)


def _frames(y, sr, fmin, fmax, frame_length, hop_length, center, pad_mode):
    """Argument checks, padding and framing shared by yin / pyin (:562-590, :763-791)."""
    if fmin is None or fmax is None:
        raise ParameterError('both "fmin" and "fmax" must be provided')
    check_yin_params(sr=sr, fmax=fmax, fmin=fmin, frame_length=frame_length)
    if hop_length is None:
        hop_length = frame_length // 4
    valid_audio(y)
    if center:
        padding = [(0, 0)] * y.ndim
        padding[-1] = (frame_length // 2, frame_length // 2)
        y = np.pad(y, padding, mode=pad_mode)
    y_frames = frame(y, frame_length=frame_length, hop_length=hop_length)
    min_period = int(np.floor(sr / fmax))
    max_period = min(int(np.ceil(sr / fmin)), frame_length - 1)
    return y_frames, min_period, max_period, hop_length


def periods(sr, fmin, fmax, frame_length):
    """(min_period, max_period) of yin / pyin."""
    return int(np.floor(sr / fmax)), min(int(np.ceil(sr / fmin)), frame_length - 1)


def yin_cmnd(y, *, fmin, fmax, sr=22050, frame_length=2048, hop_length=None, center=True, pad_mode="constant"):
    """CMND of every frame, (..., n_lags, n_frames)."""
    y_frames, lo, hi, _ = _frames(y, sr, fmin, fmax, frame_length, hop_length, center, pad_mode)
    return cumulative_mean_normalized_difference(y_frames, lo, hi)


def yin_pick(yin_frames, *, sr, min_period, trough_threshold=0.1):
    """librosa/core/pitch.py:592-628 on a CMND array (..., n_lags, n_frames) -> f0 (..., n_frames)."""
    parabolic_shifts = parabolic_interpolation(yin_frames)
    is_trough = localmin(yin_frames, axis=-2)
    is_trough[..., 0, :] = yin_frames[..., 0, :] < yin_frames[..., 1, :]
    is_threshold_trough = np.logical_and(is_trough, yin_frames < trough_threshold)
    target_shape = list(yin_frames.shape)
    target_shape[-2] = 1
    global_min = np.argmin(yin_frames, axis=-2).reshape(target_shape)
    yin_period = np.argmax(is_threshold_trough, axis=-2).reshape(target_shape)
    no_trough_below_threshold = np.all(~is_threshold_trough, axis=-2, keepdims=True)
    yin_period[no_trough_below_threshold] = global_min[no_trough_below_threshold]
    yin_period = (min_period + yin_period + np.take_along_axis(parabolic_shifts, yin_period, axis=-2))[..., 0, :]
    return sr / yin_period


def yin(y, *, fmin, fmax, sr=22050, frame_length=2048, hop_length=None, trough_threshold=0.1, center=True,
        pad_mode="constant"):
    """librosa/core/pitch.py:480-628."""
    y_frames, lo, hi, _ = _frames(y, sr, fmin, fmax, frame_length, hop_length, center, pad_mode)
    return yin_pick(cumulative_mean_normalized_difference(y_frames, lo, hi), sr=sr, min_period=lo,
                    trough_threshold=trough_threshold)


def pitch_bins(fmin, fmax, resolution):
    """(n_bins_per_semitone, n_pitch_bins) of pyin (:806-807)."""
    n_bins_per_semitone = int(np.ceil(1.0 / resolution))
    return n_bins_per_semitone, int(np.floor(12 * n_bins_per_semitone * np.log2(fmax / fmin))) + 1


def beta_probs(n_thresholds, beta_parameters):
    """Threshold grid and beta weights of pyin (:802-804)."""
    thresholds = np.linspace(0, 1, n_thresholds + 1)
    beta_cdf = scipy.stats.beta.cdf(thresholds, beta_parameters[0], beta_parameters[1])
    return thresholds, np.diff(beta_cdf)


def pyin_helper(yin_frames, parabolic_shifts, sr, thresholds, boltzmann_parameter, beta_probs_, no_trough_prob,
                min_period, fmin, n_pitch_bins, n_bins_per_semitone):
    """librosa/core/pitch.py:855-931 for one channel: (n_lags, n_frames) -> observation_probs (1, 2*bins, n_frames),
    voiced_prob (1, n_frames)."""
    yin_probs = np.zeros_like(yin_frames)
    for i, yin_frame in enumerate(yin_frames.T):
        is_trough = localmin(yin_frame)
        is_trough[0] = yin_frame[0] < yin_frame[1]
        (trough_index,) = np.nonzero(is_trough)
        if len(trough_index) == 0:
            continue
        trough_heights = yin_frame[trough_index]
        trough_thresholds = np.less.outer(trough_heights, thresholds[1:])
        trough_positions = np.cumsum(trough_thresholds, axis=0) - 1
        n_troughs = np.count_nonzero(trough_thresholds, axis=0)
        trough_prior = scipy.stats.boltzmann.pmf(trough_positions, boltzmann_parameter, n_troughs)
        trough_prior[~trough_thresholds] = 0
        probs = trough_prior.dot(beta_probs_)
        global_min = np.argmin(trough_heights)
        n_thresholds_below_min = np.count_nonzero(~trough_thresholds[global_min, :])
        probs[global_min] += no_trough_prob * np.sum(beta_probs_[:n_thresholds_below_min])
        yin_probs[trough_index, i] = probs
    yin_period, frame_index = np.nonzero(yin_probs)
    period_candidates = min_period + yin_period
    period_candidates = period_candidates + parabolic_shifts[yin_period, frame_index]
    f0_candidates = sr / period_candidates
    bin_index = 12 * n_bins_per_semitone * np.log2(f0_candidates / fmin)
    bin_index = np.clip(np.round(bin_index), 0, n_pitch_bins).astype(int)
    observation_probs = np.zeros((2 * n_pitch_bins, yin_frames.shape[1]))
    observation_probs[bin_index, frame_index] = yin_probs[yin_period, frame_index]
    voiced_prob = np.clip(np.sum(observation_probs[:n_pitch_bins, :], axis=0, keepdims=True), 0, 1)
    observation_probs[n_pitch_bins:, :] = (1 - voiced_prob) / n_pitch_bins
    return observation_probs[np.newaxis], voiced_prob


def pyin_observations(yin_frames, *, sr, fmin, fmax, min_period, n_thresholds=100, beta_parameters=(2, 18),
                      boltzmann_parameter=2, resolution=0.1, no_trough_prob=0.01):
    """Stage 3 of pyin (:793-825) on a CMND array (..., n_lags, n_frames) -> observation_probs
    (..., 2*bins, n_frames), voiced_prob (..., n_frames)."""
    parabolic_shifts = parabolic_interpolation(yin_frames)
    thresholds, bprobs = beta_probs(n_thresholds, beta_parameters)
    nbps, n_pitch_bins = pitch_bins(fmin, fmax, resolution)

    def _helper(a, b):
        return pyin_helper(a, b, sr, thresholds, boltzmann_parameter, bprobs, no_trough_prob, min_period, fmin,
                           n_pitch_bins, nbps)

    helper = np.vectorize(_helper, signature="(f,t),(k,t)->(1,d,t),(j,t)")
    observation_probs, voiced_prob = helper(yin_frames, parabolic_shifts)
    return observation_probs[..., 0, :, :], voiced_prob[..., 0, :]


def transition_loop(n_states, prob):
    """librosa/sequence.py:1905-1967 for a scalar probability."""
    transition = np.empty((n_states, n_states), dtype=np.float64)
    prob = np.tile(np.asarray(prob, dtype=np.float64), n_states)
    for i, prob_i in enumerate(prob):
        transition[i] = (1.0 - prob_i) / (n_states - 1)
        transition[i, i] = prob_i
    return transition


def transition_local(n_states, width, window="triangle", wrap=False):
    """librosa/sequence.py:2034-2146 for a scalar width."""
    width = np.tile(np.asarray(width, dtype=int), n_states)
    if np.any(width < 1):
        raise ParameterError(f"width={width} must be at least 1")
    transition = np.zeros((n_states, n_states), dtype=np.float64)
    for i, width_i in enumerate(width):
        trans_row = pad_center(scipy.signal.get_window(window, width_i, fftbins=False), size=n_states)
        trans_row = np.roll(trans_row, n_states // 2 + i + 1)
        if not wrap:
            trans_row[min(n_states, i + width_i // 2 + 1):] = 0
            trans_row[: max(0, i - width_i // 2)] = 0
        transition[i] = trans_row
    transition /= transition.sum(axis=1, keepdims=True)
    return transition


def pyin_transition(n_pitch_bins, n_bins_per_semitone, *, sr, hop_length, max_transition_rate=35.92,
                    switch_prob=0.01):
    """The transition matrix of pyin (:827-837)."""
    max_semitones_per_frame = round(max_transition_rate * 12 * hop_length / sr)
    transition_width = max_semitones_per_frame * n_bins_per_semitone + 1
    transition = transition_local(n_pitch_bins, transition_width, window="triangle", wrap=False)
    t_switch = transition_loop(2, 1 - switch_prob)
    return np.kron(t_switch, transition)


def log_threshold(transition_min_prob, eps):
    """librosa/sequence.py:1398-1405."""
    if transition_min_prob is not None and transition_min_prob > 0:
        return np.log(transition_min_prob + eps)
    if transition_min_prob is None or transition_min_prob == 0:
        return -np.inf
    raise ParameterError(f"Invalid transition_min_prob={transition_min_prob}, must be None or non-negative.")


def predecessors(log_trans, log_trans_threshold):
    """Predecessor lists of every state, ascending (librosa/sequence.py:1215-1224; all states for a full search)."""
    n_states = log_trans.shape[0]
    out = []
    for j in range(n_states):
        if np.isfinite(log_trans_threshold):
            possible = np.flatnonzero(log_trans[:, j] >= log_trans_threshold)
            if len(possible) == 0:
                raise ParameterError(f"Empty transition matrix detected for state {j} in Viterbi. "
                                     f"Try reducing your minimum transition probability threshold.")
        else:
            possible = np.arange(n_states)
        out.append(possible)
    return out


def viterbi(prob, transition, *, p_init=None, transition_min_prob=None):
    """librosa/sequence.py:1174-1432 (states only) for prob (..., n_states, n_steps)."""
    n_states, n_steps = prob.shape[-2:]
    eps = tiny(prob)
    if p_init is None:
        p_init = np.empty(n_states)
        p_init.fill(1.0 / n_states)
    log_trans = np.log(transition + eps)
    log_prob = np.log(prob + eps)
    log_p_init = np.log(p_init + eps)
    thr = log_threshold(transition_min_prob, eps)
    preds = predecessors(log_trans, thr)
    width = max(len(p) for p in preds)
    K = np.zeros((n_states, width), dtype=np.int64)     # padded with the first predecessor and -inf costs
    W = np.full((n_states, width), -np.inf)
    for j, p in enumerate(preds):
        K[j, : len(p)] = p
        K[j, len(p):] = p[0]
        W[j, : len(p)] = log_trans[p, j]
    cols = np.arange(n_states)

    def _one(lp):   # lp: (n_states, n_steps)
        lp = lp.T
        value = np.zeros((n_steps, n_states))
        ptr = np.zeros((n_steps, n_states), dtype=np.uint16)
        value[0] = lp[0] + log_p_init
        for t in range(1, n_steps):
            cost = value[t - 1][K] + W
            best = np.argmax(cost, axis=1)
            bc = cost[cols, best]
            # the reference keeps ptr = 0 when no cost beats -inf
            ptr[t] = np.where(bc > -np.inf, K[cols, best], 0)
            value[t] = lp[t] + bc
        state = np.zeros(n_steps, dtype=np.uint16)
        state[-1] = np.argmax(value[-1])
        for t in range(n_steps - 2, -1, -1):
            state[t] = ptr[t + 1, state[t + 1]]
        return state

    lead = log_prob.shape[:-2]
    flat = log_prob.reshape((-1, n_states, n_steps))
    return np.stack([_one(flat[i]) for i in range(flat.shape[0])]).reshape(lead + (n_steps,))


def pyin_decode(observation_probs, *, fmin, n_pitch_bins, n_bins_per_semitone, sr, hop_length,
                max_transition_rate=35.92, switch_prob=0.01, fill_na=np.nan, transition_min_prob=1e-4):
    """Stage 4 of pyin (:827-852): observation_probs (..., 2*bins, n_frames) -> (f0, voiced_flag, states)."""
    transition = pyin_transition(n_pitch_bins, n_bins_per_semitone, sr=sr, hop_length=hop_length,
                                 max_transition_rate=max_transition_rate, switch_prob=switch_prob)
    p_init = np.ones(2 * n_pitch_bins) / (2 * n_pitch_bins)
    states = viterbi(observation_probs, transition, p_init=p_init, transition_min_prob=transition_min_prob)
    freqs = fmin * 2 ** (np.arange(n_pitch_bins) / (12 * n_bins_per_semitone))
    f0 = freqs[states % n_pitch_bins]
    voiced_flag = states < n_pitch_bins
    if fill_na is not None:
        f0[~voiced_flag] = fill_na
    return f0, voiced_flag, states


def pyin(y, *, fmin, fmax, sr=22050, frame_length=2048, hop_length=None, n_thresholds=100, beta_parameters=(2, 18),
         boltzmann_parameter=2, resolution=0.1, max_transition_rate=35.92, switch_prob=0.01, no_trough_prob=0.01,
         fill_na=np.nan, center=True, pad_mode="constant", transition_min_prob=1e-4):
    """librosa/core/pitch.py:631-852 -> (f0, voiced_flag, voiced_prob)."""
    y_frames, lo, hi, hop_length = _frames(y, sr, fmin, fmax, frame_length, hop_length, center, pad_mode)
    cmnd = cumulative_mean_normalized_difference(y_frames, lo, hi)
    obs, voiced_prob = pyin_observations(cmnd, sr=sr, fmin=fmin, fmax=fmax, min_period=lo,
                                         n_thresholds=n_thresholds, beta_parameters=beta_parameters,
                                         boltzmann_parameter=boltzmann_parameter, resolution=resolution,
                                         no_trough_prob=no_trough_prob)
    nbps, n_pitch_bins = pitch_bins(fmin, fmax, resolution)
    f0, voiced_flag, _ = pyin_decode(obs, fmin=fmin, n_pitch_bins=n_pitch_bins, n_bins_per_semitone=nbps, sr=sr,
                                     hop_length=hop_length, max_transition_rate=max_transition_rate,
                                     switch_prob=switch_prob, fill_na=fill_na,
                                     transition_min_prob=transition_min_prob)
    return f0, voiced_flag, voiced_prob
