"""tempogram / fourier_tempogram / tempo on the GPU: every case of tests/rhythm_cases.py against tests/rhythm_oracle.py
(tempogram) or the reference's fixture (tempo, fourier_tempogram), the tempo kernel alone on the oracle's own
tempogram, the reference's own rhythm tests restated, the interface, the errors, the refused sizes and the launch
counts.

Tolerances:
    tempogram          |gpu - oracle| <= 1e-12 max|oracle| per frame.  norm=-inf, norm=0 and norms p < 1 are
                       checked only on strictly positive envelopes with np.ones and center=False: elsewhere they
                       depend on rounding noise where the exact autocorrelation is 0 (the last lag under a Hann
                       window; |r|^p with p < 1 lifts noise of 1e-17 to 3e-9 for p = 0.5), and the reference's own
                       result is noise there.
    tempo              the BPM is identical except on frames whose oracle margin (best minus runner-up score) is
                       below 1e-9 (1e-6 for a float32 tempogram, whose mean and log1p are float32), where either
                       tied lag is accepted.
    fourier_tempogram  the stft tolerance of test_gpu_parity: rtol 1e-4, atol 1e-5 max|ref|."""
import os
import warnings

import numpy as np
import pytest
import scipy.stats

import librosa_b200 as lb
import rhythm_cases as RC
import rhythm_oracle as RO

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def rhythm_golden():
    with np.load(os.path.join(ROOT, "tests", "golden", "rhythm_v1.npz")) as z:
        return {k: z[k] for k in z.files}


def _quiet(fn, *a, **k):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return fn(*a, **k)


def _ill_conditioned(case):
    norm = case["kw"].get("norm", np.inf)
    return norm is not None and (norm == -np.inf or norm < 1) and "positive_ones" not in case["name"]


def _assert_tempogram_close(got, ref, what=""):
    assert got.shape == ref.shape and got.dtype == np.float64, (got.shape, ref.shape, got.dtype)
    scale = np.max(np.abs(ref), axis=-2, keepdims=True)
    err = np.abs(got - ref)
    assert np.all(err <= 1e-12 * scale), (what, float((err / np.where(scale > 0, scale, 1)).max()))


_TG_CASES = [c["name"] for c in RC.RHYTHM_CASES if c["op"] == "tempogram" and not _ill_conditioned(c)]


@pytest.mark.parametrize("name", _TG_CASES)
def test_tempogram_vs_oracle(name):
    case = RC.BY_NAME[name]
    ref = _quiet(RC.run, RO, case)
    got = _quiet(RC.run, lb, case)
    _assert_tempogram_close(got, ref, name)


def _margins(scores):
    """Best minus runner-up score along the lag axis (-2); +inf with a single finite candidate."""
    s = np.where(np.isnan(scores), np.inf, scores)
    if s.shape[-2] == 1:
        return np.full(s.shape[:-2] + s.shape[-1:], np.inf)
    top2 = -np.sort(-s, axis=-2)[..., :2, :]
    with np.errstate(invalid="ignore"):
        return top2[..., 0, :] - top2[..., 1, :]


def _check_bpm(got, want, margins, tol, what):
    assert got.shape == want.shape and got.dtype == np.float64, (got.shape, want.shape, got.dtype)
    differ = got != want
    tied = margins < tol
    assert not np.any(differ & ~tied), (what, np.argwhere(differ & ~tied)[:5])
    print(f"{what}: {int(np.count_nonzero(tied))} near-tied frames, {int(np.count_nonzero(differ))} differ")


def _oracle_scores(case, tg):
    kw = RC.kwargs(case)
    W = tg.shape[-2]
    bpms = RO.tempo_frequencies(W, hop_length=kw["hop_length"], sr=kw["sr"])
    lp = RO.log_prior(bpms, start_bpm=kw.get("start_bpm", 120), std_bpm=kw.get("std_bpm", 1.0),
                      max_tempo=kw.get("max_tempo", 320.0), prior=kw.get("prior"))
    if kw.get("aggregate") is not None:
        tg = np.mean(tg, axis=-1, keepdims=True)
    return RO.tempo_scores(tg, lp)


def _oracle_tg(case):
    if case["op"] == "tempo_tg":
        return RC.tg_input(RO, case)
    kw = RC.kwargs(case)
    W = RO.time_to_frames(kw.get("ac_size", 8.0), sr=kw["sr"], hop_length=kw["hop_length"]).item()
    return RO.tempogram(onset_envelope=RC.make_input(case), sr=kw["sr"], hop_length=kw["hop_length"], win_length=W)


_TEMPO_CASES = [c["name"] for c in RC.RHYTHM_CASES if c["op"] in ("tempo", "tempo_tg")]


@pytest.mark.parametrize("name", _TEMPO_CASES)
def test_tempo_vs_golden(rhythm_golden, name):
    case = RC.BY_NAME[name]
    tg = _oracle_tg(case)
    tol = 1e-6 if tg.dtype == np.float32 else 1e-9
    got = _quiet(RC.run, lb, case)
    _check_bpm(got, rhythm_golden[name], _margins(_oracle_scores(case, tg)), tol, name)


@pytest.mark.parametrize("name", _TEMPO_CASES)
def test_tempo_kernel_on_oracle_tg(name):
    """The tempo kernel alone, fed the oracle's own tempogram (host, float32 or float64)."""
    case = RC.BY_NAME[name]
    tg = _oracle_tg(case)
    kw = RC.kwargs(case)
    kw.pop("ac_size", None)
    want = _quiet(RO.tempo, tg=tg, **kw)
    got = _quiet(lb.feature.tempo, tg=tg, **kw)
    tol = 1e-6 if tg.dtype == np.float32 else 1e-9
    _check_bpm(got, want, _margins(_oracle_scores(case, tg)), tol, name)


@pytest.mark.parametrize("W,mr", [(256, "1"), (512, "1"), (384, "1"), (384, "0"), (343, "1")])
def test_fourier_tempogram_vs_golden(rhythm_golden, monkeypatch, W, mr):
    """stft at hop 1 on each forward path: fwd_kernel (256, 512), mr_kernel (384) and chirp-z (384 with B2L_MR=0,
    343)."""
    monkeypatch.setenv("B2L_MR", mr)
    case = RC.BY_NAME[f"fourier/win{W}"]
    ref = rhythm_golden[case["name"]]
    got = _quiet(RC.run, lb, case)
    assert got.shape == ref.shape and got.dtype == ref.dtype == np.complex64
    assert np.allclose(got, ref, rtol=1e-4, atol=1e-5 * float(np.abs(ref).max())), float(np.abs(got - ref).max())


# ------------------------------------------------------------------------- the reference's own tests, restated
def _clicks(tempo, n, sr=22050, hop=512, rows=None):
    odf = np.zeros(n if rows is None else (rows, n))
    if rows is None:
        odf[:: int(sr * 60.0 // (hop * tempo))] = 1
    return odf


@pytest.mark.parametrize("tempo", [60, 120, 200])
@pytest.mark.parametrize("center", [False, True])
def test_tempogram_odf_equiv(tempo, center):
    odf = _clicks(tempo, 8 * 22050 // 512)
    odf_ac = RO.autocorrelate(odf)
    tg = lb.feature.tempogram(onset_envelope=odf, sr=22050, hop_length=512, win_length=len(odf), window=np.ones,
                              center=center, norm=None)
    idx = len(odf) // 2 if center else 0
    assert np.allclose(odf_ac, tg[:, idx])


def _localmax(x):
    """util.localmax along the only axis: x[i] > x[i-1] and x[i] >= x[i+1] (edges padded by repetition)."""
    xp = np.pad(x, 1, mode="edge")
    return (x > xp[:-2]) & (x >= xp[2:])


@pytest.mark.parametrize("tempo", [60, 90, 200])
@pytest.mark.parametrize("win_length", [192, 384])
@pytest.mark.parametrize("window", ["hann", np.ones])
@pytest.mark.parametrize("norm", [None, 1, 2, np.inf])
def test_tempogram_odf_peak(tempo, win_length, window, norm):
    odf = _clicks(tempo, 8 * 22050 // 512)
    spacing = 22050 * 60.0 // (512 * tempo)
    tg = lb.feature.tempogram(onset_envelope=odf, sr=22050, hop_length=512, win_length=win_length, window=window,
                              norm=norm)
    assert tg.shape == (win_length, len(odf))
    idx = np.where(_localmax(tg.max(axis=1)))[0]
    assert np.allclose(idx, spacing * np.arange(1, 1 + len(idx)))


@pytest.mark.parametrize("center", [False, True])
@pytest.mark.parametrize("win_length", [192, 384])
@pytest.mark.parametrize("window", ["hann", np.ones])
@pytest.mark.parametrize("norm", [None, 1, 2, np.inf])
def test_tempogram_odf_multi(center, win_length, window, norm):
    odf = np.zeros((10, 8 * 22050 // 512))
    for i in range(10):
        odf[i, :: int(22050 * 60.0 // (512 * (60 + 12 * i)))] = 1
    kw = dict(sr=22050, hop_length=512, win_length=win_length, window=window, norm=norm, center=center)
    if not center and win_length > odf.shape[-1]:
        # 344 frames cannot hold an uncentred 384-frame window: the reference raises util.frame's error here too
        with pytest.raises(lb.ParameterError, match="Input is too short"):
            lb.feature.tempogram(onset_envelope=odf, **kw)
        return
    tg = lb.feature.tempogram(onset_envelope=odf, **kw)
    for i in range(10):
        one = lb.feature.tempogram(onset_envelope=odf[i], **kw)
        assert np.array_equal(tg[i], one)


def _chirp():
    import scipy.signal

    t = np.arange(5 * 22050) / 22050
    return scipy.signal.chirp(t, 110, 5.0, 880, method="logarithmic", phi=-90.0)


@pytest.mark.parametrize("hop_length", [512, 1024])
@pytest.mark.parametrize("fn", ["tempogram", "fourier_tempogram"])
def test_tempogram_audio(hop_length, fn):
    y, sr = _chirp(), 22050
    f = getattr(lb.feature, fn)
    oenv = _quiet(lb.onset.onset_strength, y=y, sr=sr, hop_length=hop_length)
    t1 = _quiet(f, y=y, sr=sr, onset_envelope=None, hop_length=hop_length)
    t2 = _quiet(f, y=None, sr=sr, onset_envelope=oenv, hop_length=hop_length)
    t3 = _quiet(f, y=y, sr=sr, onset_envelope=oenv, hop_length=hop_length)
    t4 = _quiet(f, y=0 * y, sr=sr, onset_envelope=oenv, hop_length=hop_length)
    if fn == "fourier_tempogram":
        assert np.iscomplexobj(t1) and t1.dtype == np.complex128   # float64 audio, as the reference
    assert np.allclose(t1, t2) and np.allclose(t1, t3) and np.allclose(t1, t4)


@pytest.mark.parametrize("fn", ["tempogram", "fourier_tempogram"])
@pytest.mark.parametrize("win_length,window", [(-384, "hann"), (0, "hann"), (384, np.ones(3))])
def test_tempogram_fail_badwin(fn, win_length, window):
    with pytest.raises(lb.ParameterError):
        getattr(lb.feature, fn)(y=np.zeros(10 * 1000), sr=1000, win_length=win_length, window=window)


@pytest.mark.parametrize("fn", ["tempogram", "fourier_tempogram"])
def test_tempogram_fail_noinput(fn):
    with pytest.raises(lb.ParameterError):
        getattr(lb.feature, fn)(y=None, onset_envelope=None)


@pytest.mark.parametrize("sr", [22050])
@pytest.mark.parametrize("hop_length", [512])
@pytest.mark.parametrize("win_length", [192, 384])
@pytest.mark.parametrize("center", [False, True])
@pytest.mark.parametrize("window", ["hann", np.ones])
def test_fourier_tempogram_invert(sr, hop_length, win_length, center, window):
    odf = np.zeros(16 * sr // hop_length, dtype=np.float32)
    odf[:: int(sr * 60.0 // (hop_length * 100))] = 1
    tg = lb.feature.fourier_tempogram(onset_envelope=odf, sr=sr, hop_length=hop_length, win_length=win_length,
                                      window=window, center=center)
    sl = slice(None) if center else slice(win_length // 2, -win_length // 2)
    odf_inv = lb.istft(tg, hop_length=1, center=center, window=window, length=len(odf))
    assert np.allclose(odf_inv[sl], odf[sl], atol=1e-6)


@pytest.mark.parametrize("tempo", [60, 160])
@pytest.mark.parametrize("sr", [22050, 16000])
@pytest.mark.parametrize("hop_length", [512, 1024])
@pytest.mark.parametrize("ac_size", [4, 8])
@pytest.mark.parametrize("aggregate", [None, np.mean])
@pytest.mark.parametrize("prior", [None, scipy.stats.uniform(60, 240)])
def test_tempo(tempo, sr, hop_length, ac_size, aggregate, prior):
    y = np.zeros(20 * sr)
    y[:: int(60.0 / tempo * sr)] = 1
    est = _quiet(lb.feature.tempo, y=y, sr=sr, hop_length=hop_length, ac_size=ac_size, aggregate=aggregate,
                 prior=prior)
    if aggregate is None:
        w = int(ac_size * sr // hop_length)
        assert np.all(np.abs(est[w:-w] - tempo) <= 0.05 * tempo)
    else:
        assert np.abs(est - tempo) <= 0.05 * tempo, (tempo, est)


@pytest.mark.parametrize("start_bpm", [40, 60, 117, 235])
@pytest.mark.parametrize("aggregate", [None, np.mean])
def test_tempo_no_onsets(start_bpm, aggregate):
    est = lb.feature.tempo(onset_envelope=np.zeros(30 * 22050 // 512), sr=22050, hop_length=512,
                           start_bpm=start_bpm, aggregate=aggregate)
    assert np.allclose(est, start_bpm, atol=1e0)


def test_tempo_tgin():
    y = _chirp() + _clicks_audio()
    t1 = _quiet(lb.feature.tempo, y=y, sr=22050, ac_size=5, aggregate=None)
    W = RO.time_to_frames(5, sr=22050).item()
    tg = _quiet(lb.feature.tempogram, y=y, sr=22050, win_length=W)
    t2 = lb.feature.tempo(tg=tg, sr=22050, aggregate=None)
    assert np.allclose(t1, t2)


def _clicks_audio(sr=22050, n=5 * 22050):
    y = np.zeros(n)
    y[:: int(0.5 * sr)] = 1.0
    return y


# ------------------------------------------------------------------------- interface
def test_interface_host_and_device():
    ctx = lb.default_context()
    x = RC.envelope("clicks", (2, 3), 300, "float32", 1)
    host = lb.feature.tempogram(onset_envelope=x)
    dev = lb.feature.tempogram(onset_envelope=ctx.to_device(x))
    assert isinstance(host, np.ndarray) and host.dtype == np.float64 and host.shape == (2, 3, 384, 300)
    assert isinstance(dev, lb.DeviceArray) and dev.layout == "ft" and dev.shape == (2, 3, 384, 300)
    assert np.array_equal(dev.get(), host)
    x64 = x.astype(np.float64)
    assert lb.feature.tempogram(onset_envelope=x64).dtype == np.float64
    # tempo from an envelope, and from the tempogram in both layouts and both precisions
    t_host = lb.feature.tempo(onset_envelope=x)
    t_dev = lb.feature.tempo(onset_envelope=ctx.to_device(x))
    assert t_host.shape == (2, 3, 1) and t_host.dtype == np.float64
    assert isinstance(t_dev, lb.DeviceArray) and np.array_equal(t_dev.get(), t_host)
    tg = lb.feature.tempogram(onset_envelope=x, win_length=344)
    ref_frames = lb.feature.tempo(tg=tg, aggregate=None)
    assert ref_frames.shape == (2, 3, 300)
    d_ft = lb.feature.tempogram(onset_envelope=ctx.to_device(x), win_length=344)
    d_c = ctx.to_device(np.ascontiguousarray(tg))
    for d in (d_ft, d_c):
        got = lb.feature.tempo(tg=d, aggregate=None)
        assert isinstance(got, lb.DeviceArray) and np.array_equal(got.get(), ref_frames)
        assert np.array_equal(lb.feature.tempo(tg=d).get(), lb.feature.tempo(tg=tg))
    f32 = lb.feature.tempo(tg=tg.astype(np.float32), aggregate=None)
    assert f32.dtype == np.float64 and f32.shape == (2, 3, 300)
    # fourier_tempogram: complex64 for float32 envelopes, complex128 for float64
    F = lb.feature.fourier_tempogram(onset_envelope=x)
    assert F.dtype == np.complex64 and F.shape == (2, 3, 193, 301)
    assert lb.feature.fourier_tempogram(onset_envelope=x64).dtype == np.complex128


def test_center_false_too_short():
    with pytest.raises(lb.ParameterError, match="Input is too short"):
        lb.feature.tempogram(onset_envelope=np.ones(100, np.float32), win_length=384, center=False)


@pytest.mark.parametrize("norm", [np.inf, None])
@pytest.mark.parametrize("where", ["host", "device"])
def test_non_finite_envelope(norm, where):
    x = RC.envelope("random", (), 300, "float64", 1)
    x[150] = np.nan
    if where == "device":
        x = lb.default_context().to_device(x)
    with pytest.raises(lb.ParameterError, match="Input must be finite"):
        lb.feature.tempogram(onset_envelope=x, norm=norm)
    with pytest.raises(lb.ParameterError, match="Input must be finite"):
        lb.feature.tempo(onset_envelope=x)
    # the status word is clean again for the next call
    assert np.all(np.isfinite(lb.feature.tempogram(onset_envelope=np.ones(300))))


def test_refused_window():
    with pytest.raises(lb.UnsupportedOnGPU, match="4097"):
        lb.feature.tempogram(onset_envelope=np.ones(5000, np.float32), win_length=4097)


def test_launch_counts():
    ctx = lb.default_context()
    x = ctx.to_device(RC.envelope("clicks", (4,), 431, "float32", 1))
    tg = lb.feature.tempogram(onset_envelope=x, win_length=344)
    y = ctx.to_device(np.zeros((2, 22050 * 3), np.float32))

    def count(fn):
        ctx.synchronize()
        l0 = ctx.launch_count
        out = fn()
        ctx.synchronize()
        del out
        return ctx.launch_count - l0

    onset = count(lambda: lb.onset.onset_strength(y=y))
    stft = count(lambda: lb.stft(x, n_fft=384, hop_length=1))
    table = {
        "tempogram(onset_envelope=dev)": (count(lambda: lb.feature.tempogram(onset_envelope=x)), 1),
        "tempo(onset_envelope=dev)": (count(lambda: lb.feature.tempo(onset_envelope=x)), 2),
        "tempo(onset_envelope=dev, aggregate=None)": (count(lambda: lb.feature.tempo(onset_envelope=x,
                                                                                     aggregate=None)), 2),
        "tempo(tg=dev)": (count(lambda: lb.feature.tempo(tg=tg)), 1),
        "tempogram(y=dev)": (count(lambda: lb.feature.tempogram(y=y)), onset + 1),
        "tempo(y=dev)": (count(lambda: lb.feature.tempo(y=y)), onset + 2),
        "fourier_tempogram(onset_envelope=dev)": (count(lambda: lb.feature.fourier_tempogram(onset_envelope=x)),
                                                  stft),
    }
    bad = {k: v for k, v in table.items() if v[0] != v[1]}
    assert not bad, bad
