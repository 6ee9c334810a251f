"""beat_track and median onset strength on the GPU: the tracker stages bit for bit against the reference's fixture
(tests/golden/beat_v1.npz), the public call against the fixture, median onset aggregation bit for bit against NumPy,
``y=`` end to end against the oracle run on the GPU's own envelope, DeviceArray in and out, and the launch counts.

Tolerances: none on the tracker — localscore, cumscore, backlink and the beats are compared bit for bit.  The bpm
that ``beat_track`` estimates is compared exactly with the reference's (none of the cases is a tempo near-tie)."""
import os
import warnings

import numpy as np
import pytest

import beat_cases as BC
import beat_oracle as BO
import librosa_b200 as lb
from librosa_b200 import beat as B

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def beat_golden():
    with np.load(os.path.join(ROOT, "tests", "golden", "beat_v1.npz")) as z:
        return {k: z[k] for k in z.files}


def _quiet(fn, *a, **k):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return fn(*a, **k)


def _same(got, want, key):
    got = np.asarray(got)
    assert got.dtype == want.dtype and got.shape == want.shape, (key, got.dtype, want.dtype, got.shape, want.shape)
    if got.tobytes() != want.tobytes():
        bad = np.argwhere(got != want)
        raise AssertionError(f"{key}: {len(bad)} differ, first at {bad[:3].tolist()}")


_STAGE_CASES = [c["name"] for c in BC.BEAT_CASES if BC.has_stages(c)]


@pytest.mark.parametrize("name", _STAGE_CASES)
def test_tracker_stages_bit_exact(beat_golden, name):
    """Host envelope and bpm: localscore / cumscore / backlink bit-identical to the reference's, beats identical."""
    case = BC.BY_NAME[name]
    x = BC.make_input(case)
    bpm = BC.bpm_arg(case)
    if bpm is None:
        bpm = beat_golden[name + "/bpm"]
    got = B.track_stages(x, bpm=bpm, sr=BC.SR, hop_length=BC.HOP, **BC.stage_kwargs(case))
    for key in ("localscore", "cumscore", "backlink"):
        _same(got[key], beat_golden[f"{name}/{key}"], f"{name}/{key}")
    _, fpb = BO.frames_per_beat(bpm, BC.SR, BC.HOP, x.shape)
    _same(got["beats"], BO.track_stages(x, fpb, **BC.stage_kwargs(case))["beats"], name + "/beats")


@pytest.mark.parametrize("name", [c["name"] for c in BC.BEAT_CASES])
def test_beat_track_vs_golden(beat_golden, name):
    case = BC.BY_NAME[name]
    bpm, beats = _quiet(BC.run, lb, case)
    if name + "/beats" in beat_golden:
        _same(beats, beat_golden[name + "/beats"], name + "/beats")
    else:   # the all-zero clip of a batch: no beats there, the other clips as the oracle
        x = BC.make_input(case)
        _, fpb = BO.frames_per_beat(BC.bpm_arg(case), BC.SR, BC.HOP, x.shape)
        want = BO.track_stages(x, fpb)["beats"]
        _same(beats, want, name + "/beats")
        assert not beats[1].any()
    if case["kw"].get("bpm") is None:
        _same(np.asarray(bpm, dtype=np.float64), beat_golden[name + "/bpm"], name + "/bpm")


def _device(x):
    return lb.to_device(np.ascontiguousarray(x))


def test_device_in_device_out_and_launch_counts(beat_golden):
    ctx = lb.default_context()
    case = BC.BY_NAME["beat/clicks0_float32"]
    d = _device(BC.make_input(case))
    n0 = ctx.launch_count
    bpm, beats = lb.beat.beat_track(onset_envelope=d)
    n1 = ctx.launch_count
    assert isinstance(bpm, lb.DeviceArray) and isinstance(beats, lb.DeviceArray)
    # np.any, tempogram, tempo, tracker
    assert n1 - n0 == 4, n1 - n0
    _same(beats.get(), beat_golden["beat/clicks0_float32/beats"], "device beats")
    _same(bpm.get(), beat_golden["beat/clicks0_float32/bpm"], "device bpm")
    n0 = ctx.launch_count
    bpm2, dense = lb.beat.beat_track(onset_envelope=d, bpm=120.0, sparse=False)
    assert ctx.launch_count - n0 == 2 and bpm2 == 120.0 and dense.dtype == np.bool_
    # host envelope with bpm: the tracker alone
    n0 = ctx.launch_count
    lb.beat.beat_track(onset_envelope=BC.make_input(case), bpm=120.0)
    assert ctx.launch_count - n0 == 1
    for units in ("samples", "time"):
        c = BC.BY_NAME[f"beat/units_{units}_bpm"]
        _, got = lb.beat.beat_track(onset_envelope=_device(BC.make_input(c)), bpm=130.0, units=units)
        assert isinstance(got, lb.DeviceArray)
        _same(got.get(), beat_golden[f"beat/units_{units}_bpm/beats"], units)


def test_zero_device_envelope():
    d = _device(np.zeros((2, 100), np.float32))
    bpm, beats = lb.beat.beat_track(onset_envelope=d, sparse=False)
    assert isinstance(beats, lb.DeviceArray) and not beats.get().any() and bpm.get().shape == (2,)
    bpm, beats = lb.beat.beat_track(onset_envelope=_device(np.zeros(100, np.float64)))
    assert bpm == 0.0 and beats.shape == (0,)


def _median_flux(S, lag=1, pad=0, bounds=None):
    flux = np.maximum(0.0, S[..., lag:] - S[..., :-lag])
    bounds = bounds or [0, S.shape[-2]]
    rows = [np.median(flux[..., a:b, :], axis=-2) for a, b in zip(bounds[:-1], bounds[1:])]
    env = np.stack(rows, axis=-2).astype(np.float32)
    env = np.pad(env, [(0, 0)] * (env.ndim - 1) + [(lag + pad, 0)])
    return env[..., : S.shape[-1]]


@pytest.mark.parametrize("rows", [1, 2, 7, 128, 129, 512])
def test_median_onset_kernel_bit_exact(rows):
    rng = np.random.default_rng(rows)
    S = (rng.standard_normal((3, rows, 97)) * 20).astype(np.float32)
    S[0, :, 5] = S[0, :, 4]      # ties
    got = lb.onset.onset_strength(S=S, aggregate=np.median, center=False)
    _same(got, _median_flux(S)[..., 0, :], f"median {rows}")


def test_median_onset_channels_and_nan():
    rng = np.random.default_rng(3)
    S = (rng.standard_normal((2, 96, 50)) * 10).astype(np.float32)
    got = lb.onset.onset_strength_multi(S=S, aggregate=np.median, channels=[0, 10, 41, 96], center=False)
    _same(got, _median_flux(S, bounds=[0, 10, 41, 96]), "channels")
    S[1, 20, 30] = np.nan
    got = lb.onset.onset_strength(S=S, aggregate=np.median, center=False)
    assert np.isnan(got[1, 30]) and np.isnan(got[1, 31]) and not np.isnan(np.delete(got[1], [30, 31])).any()


def test_median_refusal():
    with pytest.raises(lb.UnsupportedOnGPU, match="600 rows"):
        lb.onset.onset_strength(S=np.zeros((600, 20), np.float32), aggregate=np.median)
    with pytest.raises(lb.UnsupportedOnGPU, match="only mean or median"):
        lb.onset.onset_strength(S=np.zeros((10, 20), np.float32), aggregate=np.max)


def _clicks_audio(bpm, seconds=10.0, sr=22050):
    y = np.zeros(int(seconds * sr), np.float32)
    period = int(round(sr * 60.0 / bpm))
    for s in range(period // 2, y.size - 64, period):
        y[s:s + 64] += np.hanning(64).astype(np.float32)
    return y


def test_y_end_to_end_vs_oracle_on_gpu_envelope():
    y = np.stack([_clicks_audio(120.0), _clicks_audio(95.0)])
    bpm, beats = lb.beat.beat_track(y=y, sparse=False)
    env = lb.onset.onset_strength(y=y, aggregate=np.median)
    bpm_e = lb.feature.tempo(onset_envelope=env)
    _same(bpm, bpm_e, "bpm")
    _, fpb = BO.frames_per_beat(bpm, BC.SR, BC.HOP, env.shape)
    want = BO.track_stages(env, fpb)["beats"]
    _same(beats, want, "y= beats")
    assert np.all(beats.sum(axis=-1) > 5)


def test_restated_reference_beat_tests():
    """The reference's test_beat_no_input / test_beat_no_onsets / test_beat_units / test_beat_bad_bpm, restated."""
    with pytest.raises(lb.ParameterError):
        lb.beat.beat_track()
    bpm, beats = lb.beat.beat_track(onset_envelope=np.zeros(1000, np.float32))
    assert bpm == 0.0 and len(beats) == 0
    env = lb.onset.onset_strength(y=_clicks_audio(120.0), aggregate=np.median)
    _, frames = lb.beat.beat_track(onset_envelope=env)
    _, samples = lb.beat.beat_track(onset_envelope=env, units="samples")
    _, times = lb.beat.beat_track(onset_envelope=env, units="time")
    assert np.array_equal(samples, lb.frames_to_samples(frames)) and np.array_equal(times, lb.frames_to_time(frames))
    with pytest.raises(lb.ParameterError):
        lb.beat.beat_track(onset_envelope=env, units="bad")
    for bad in (-1.0, 0.0, np.array([120.0, -1.0])):
        with pytest.raises(lb.ParameterError):
            lb.beat.beat_track(onset_envelope=np.stack([env, env]), bpm=bad, sparse=False)


@pytest.mark.parametrize("name", list(BC.Y_CASES))
def test_y_vs_golden_pulse_trains(beat_golden, name):
    """beat_track(y=) on click trains against the reference's own beats and bpm."""
    bpm, beats = lb.beat.beat_track(y=BC.clicks_audio(BC.Y_CASES[name]))
    _same(np.asarray(bpm, dtype=np.float64), beat_golden[name + "/bpm"], name + "/bpm")
    _same(beats, beat_golden[name + "/beats"], name + "/beats")


@pytest.mark.parametrize("name", [c["name"] for c in BC.PLP_CASES])
def test_plp_vs_golden(beat_golden, name):
    """The end-to-end pulse within 1e-4 of the reference's (its maximum is 1)."""
    case = BC.PLP_BY_NAME[name]
    got = _quiet(BC.run_plp, lb, case)
    want = beat_golden[name + "/pulse"]
    assert got.dtype == want.dtype and got.shape == want.shape, (got.dtype, got.shape)
    err = float(np.max(np.abs(got - want)))
    assert err <= 1e-4, (name, err)


@pytest.mark.parametrize("name", [c["name"] for c in BC.PLP_CASES])
def test_plp_select_kernel_alone(name):
    """The select kernel on the GPU's own Fourier tempogram against the oracle's selection of the same data: the
    same surviving bins in every frame, the values to float rounding."""
    import rhythm_oracle as RO

    case = BC.PLP_BY_NAME[name]
    kw = BC.plp_kwargs(case)
    W = kw.get("win_length", 384)
    ft = lb.feature.fourier_tempogram(onset_envelope=_device(BC.make_input(case)), win_length=W)
    host = ft.get().copy()
    freqs = RO.fourier_tempo_frequencies(sr=kw["sr"], hop_length=kw["hop_length"], win_length=W)
    keep = BO.plp_keep(freqs, kw.get("tempo_min", 30), kw.get("tempo_max", 300))
    prior = kw.get("prior")
    lp = None if prior is None else np.asarray(prior.logpdf(freqs), dtype=np.float64)
    B.select_peaks(ft, keep, lp)
    got = ft.get()
    want, _ = _quiet(BO.plp_select, host, keep, lp)
    assert np.array_equal(got != 0, want != 0), name
    scale = np.max(np.abs(want), axis=-2, keepdims=True)
    assert np.all(np.abs(got - want) <= 1e-5 * scale), name


def test_plp_device_in_device_out():
    case = BC.PLP_BY_NAME["plp/batch3"]
    x = BC.make_input(case)
    ctx = lb.default_context()
    d = _device(x)
    ft = lb.feature.fourier_tempogram(onset_envelope=d, win_length=192)
    n0 = ctx.launch_count
    pulse_ft = lb.istft(ft, hop_length=1, n_fft=192, length=x.shape[-1])
    n_istft = ctx.launch_count - n0
    n0 = ctx.launch_count
    lb.feature.fourier_tempogram(onset_envelope=d, win_length=192)
    n_stft = ctx.launch_count - n0
    n0 = ctx.launch_count
    pulse = lb.beat.plp(onset_envelope=d, win_length=192)
    # stft, select, istft, clip + normalize
    assert ctx.launch_count - n0 == n_stft + n_istft + 2
    assert isinstance(pulse, lb.DeviceArray) and pulse.shape == x.shape and pulse_ft.shape == x.shape
    host = _quiet(lb.beat.plp, onset_envelope=x, win_length=192)
    assert np.array_equal(pulse.get(), host)


def test_restated_reference_plp():
    """The reference's test_plp: the pulse keeps the envelope's shape and dtype, lies in [0, 1] and peaks at 1;
    the y= form runs the median envelope."""
    y = BC.clicks_audio(120.0)
    env = lb.onset.onset_strength(y=y, aggregate=np.median)
    for kw in (dict(), dict(prior=scipy_lognorm()), dict(tempo_min=None, tempo_max=None)):
        pulse = lb.beat.plp(onset_envelope=env, **kw)
        assert pulse.shape == env.shape and pulse.dtype == env.dtype
        assert np.all(pulse >= 0) and np.isclose(pulse.max(), 1.0)
    assert np.array_equal(lb.beat.plp(y=y), lb.beat.plp(onset_envelope=env))


def scipy_lognorm():
    import scipy.stats

    return scipy.stats.lognorm(loc=np.log(120), scale=120, s=1)
