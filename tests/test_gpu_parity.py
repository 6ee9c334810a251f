"""GPU (-m gpu): the CUDA path, called through the public drop-in API (ctypes -> C ABI -> sm_90a
kernels), against the oracle on identical inputs and against the fixtures produced by the unmodified
reference.  Nothing here reads /root/reference.

Stated tolerances (north_star: float32, rtol 1e-4; SURVEY §8d for the atol terms — the reference runs its
forward FFT in float64, the GPU in float32, so near-zero bins need an absolute term relative to max|ref|):
    stft            rtol 1e-4, atol 1e-5 * max|ref|
    melspectrogram  rtol 1e-4, atol 1e-6 * max|ref|
    mfcc            rtol 1e-4, atol 1e-3 (dB-domain values up to ~1e2)
    istft           atol 1e-5 * max|ref| on the un-normalised overlap-add (see _istft_close), SNR >= 60 dB
"""
import os
import sys
import warnings

import numpy as np
import pytest

from cases import BY_NAME, CASES
from conftest import case_input

pytestmark = pytest.mark.gpu

TOL = {
    "stft": dict(rtol=1e-4, atol_rel=1e-5),
    "mel": dict(rtol=1e-4, atol_rel=1e-6),
    "mfcc": dict(rtol=1e-4, atol_abs=1e-3),
    "istft": dict(rtol=1e-4, atol_rel=1e-5),
}


@pytest.fixture(scope="module")
def lb():
    import librosa_b200

    librosa_b200.default_context()   # fails loudly if the library or the GPU is missing
    return librosa_b200


def close(got, ref, rtol, atol_rel=None, atol_abs=None):
    got, ref = np.asarray(got), np.asarray(ref)
    assert got.shape == ref.shape, (got.shape, ref.shape)
    assert got.dtype == ref.dtype, (got.dtype, ref.dtype)
    atol = atol_abs if atol_abs is not None else atol_rel * float(np.abs(ref).max() if ref.size else 0.0)
    np.testing.assert_allclose(got, ref, rtol=rtol, atol=atol)


def _istft_close(O, got, ref, case_kw, n_fft, T):
    """istft divides by the window-sum-square, which tends to 0 at the ends when center=False; there the
    quotient of two roundings is ill-conditioned in the reference itself.  Compare the un-normalised
    overlap-add (y * wss) — identical to comparing y wherever wss is O(1)."""
    kw = dict(case_kw)
    center = kw.get("center", True)
    hop = kw.get("hop_length") or int((kw.get("win_length") or n_fft) // 4)
    wss = O.window_sumsquare(kw.get("window", "hann"), T, hop_length=hop, win_length=kw.get("win_length"), n_fft=n_fft)
    start = n_fft // 2 if center else 0
    wss = O.fix_length(wss[start:], ref.shape[-1])
    w = np.where(wss > O.tiny(wss), wss, 1.0)
    close(got * w, ref * w, **TOL["istft"])
    assert got.shape == ref.shape and got.dtype == ref.dtype


def run_gpu(lb, case, golden):
    kw = dict(case["kw"])
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        if case["op"] == "istft":
            return lb.istft(golden[case["src"]], **kw)
        y = case_input(case)
        if case["op"] == "stft":
            return lb.stft(y, **kw)
        if case["op"] == "mel":
            return lb.feature.melspectrogram(y=y, **kw)
        if case["op"] == "mfcc":
            return lb.feature.mfcc(y=y, **kw)
    raise ValueError(case["op"])


def run_oracle(O, case, golden):
    kw = dict(case["kw"])
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        if case["op"] == "istft":
            return O.istft(golden[case["src"]], **kw)
        y = case_input(case)
        return {"stft": lambda: O.stft(y, **kw), "mel": lambda: O.melspectrogram(y=y, **kw),
                "mfcc": lambda: O.mfcc(y=y, **kw)}[case["op"]]()


@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_case_against_oracle_and_reference_fixture(case, lb, oracle, golden):
    if case.get("gpu") == "unsupported":
        with pytest.raises(lb.UnsupportedOnGPU):
            run_gpu(lb, case, golden)
        return
    got = run_gpu(lb, case, golden)
    want = run_oracle(oracle, case, golden)
    fixture = golden[case["name"]]
    if case["op"] == "istft":
        D = golden[case["src"]]
        n_fft = case["kw"].get("n_fft") or 2 * (D.shape[-2] - 1)
        T = D.shape[-1]
        length = case["kw"].get("length")
        if length:
            center = case["kw"].get("center", True)
            hop = case["kw"].get("hop_length") or n_fft // 4
            T = min(T, int(np.ceil((length + (2 * (n_fft // 2) if center else 0)) / hop)))
        _istft_close(oracle, got, want, case["kw"], n_fft, T)
        _istft_close(oracle, got, fixture, case["kw"], n_fft, T)
    else:
        close(got, want, **TOL[case["op"]])
        close(got, fixture, **TOL[case["op"]])


@pytest.mark.parametrize("name", ["stft_400_160_stereo_A", "stft_2000_500_nocenter_A", "stft_12_5_edge_A",
                                  "stft_600_winlen400_hamming_A", "stft_486_oddhop_A", "mel_16000_400_80_B",
                                  "mfcc_16000_400_C", "mfcc_16000_400_lifter_A", "istft_400_160_stereo",
                                  "istft_2000_nocenter", "istft_486_oddhop"])
def test_even_smooth_sizes_still_pass_on_the_chirpz_kernels(name, lb, oracle, golden, monkeypatch):
    """Even frame lengths with a 5-smooth half take the mixed-radix kernel by default (mr_kernel.cuh); with
    B2L_MR=0 they run on the chirp-z kernels (and the composed S= kernels) as before — both stay pinned."""
    monkeypatch.setenv("B2L_MR", "0")
    case = BY_NAME[name]
    got = run_gpu(lb, case, golden)
    if case["op"] == "istft":
        D = golden[case["src"]]
        n_fft = case["kw"].get("n_fft") or 2 * (D.shape[-2] - 1)
        T, length = D.shape[-1], case["kw"].get("length")
        if length:
            hop = case["kw"].get("hop_length") or n_fft // 4
            T = min(T, int(np.ceil((length + (2 * (n_fft // 2) if case["kw"].get("center", True) else 0)) / hop)))
        _istft_close(oracle, got, run_oracle(oracle, case, golden), case["kw"], n_fft, T)
        return
    close(got, run_oracle(oracle, case, golden), **TOL[case["op"]])
    close(got, golden[name], **TOL[case["op"]])


def test_mixed_radix_device_resident_and_batch_identity(lb, oracle):
    """mr_kernel on a DeviceArray batch: every clip equals the single-clip result bit for bit (a warp owns a frame,
    nothing depends on the batch), non-finite samples are reported like util.valid_audio, and frames at both clip
    edges (reflect padding, odd hop, clip length that is not a multiple of anything) match the oracle."""
    import signals

    Y = signals.make("B", (5, 7003), seed=11, sr=16000)
    kw = dict(n_fft=400, hop_length=161, pad_mode="reflect")
    Dd = lb.stft(lb.to_device(Y), **kw).get()
    for c in range(Y.shape[0]):
        np.testing.assert_array_equal(Dd[c], lb.stft(Y[c], **kw))
    close(Dd, oracle.stft(Y, **kw), **TOL["stft"])
    M = lb.feature.melspectrogram(y=lb.to_device(Y), sr=16000, n_fft=400, hop_length=160, n_mels=80).get()
    close(M, oracle.melspectrogram(y=Y, sr=16000, n_fft=400, hop_length=160, n_mels=80), **TOL["mel"])
    C_ = lb.feature.mfcc(y=lb.to_device(Y), sr=16000, n_mfcc=13, n_fft=400, hop_length=160, n_mels=80).get()
    close(C_, oracle.mfcc(y=Y, sr=16000, n_mfcc=13, n_fft=400, hop_length=160, n_mels=80), **TOL["mfcc"])
    bad = Y.copy()
    bad[2, 3000] = np.inf
    for fn in (lambda a: lb.stft(a, n_fft=400, hop_length=160),
               lambda a: lb.feature.melspectrogram(y=a, sr=16000, n_fft=400, hop_length=160, n_mels=80),
               lambda a: lb.feature.mfcc(y=a, sr=16000, n_mfcc=13, n_fft=400, hop_length=160, n_mels=80)):
        with pytest.raises(lb.ParameterError):
            fn(bad)


def _smooth_even_sizes(limit=4096):
    out = []
    for n in range(12, limit + 1, 2):
        m = n // 2
        for q in (2, 3, 5):
            while m % q == 0:
                m //= q
        if m == 1 and n & (n - 1):
            out.append(n)
    return out


def test_mixed_radix_every_size(lb, oracle):
    """All 96 frame lengths mr_inv_kernel serves (even, 12 .. 4096, half = 2^a 3^b 5^c, not a power of two) — every
    radix schedule the host can produce: istft of the oracle's spectrum (length given) against the signal at the
    float32 bound the power-of-two path is held to (SNR >= 60 dB).  The forward direction (mr_kernel modes 0 and 1)
    is held to a float64 reference at every size by test_gpu_forward_spectrum.test_mixed_radix_sizes."""
    import signals

    sizes = _smooth_even_sizes()
    assert len(sizes) == 96
    for idx, n_fft in enumerate(sizes):
        hop = max(1, n_fft // 4 - (idx % 3))                 # also hops that do not divide n_fft
        y = signals.make("AB"[idx % 2], (2, 3 * n_fft + 17 * (idx % 5)), seed=100 + idx)
        kw = dict(n_fft=n_fft, hop_length=hop, pad_mode=("constant", "reflect", "edge")[idx % 3])
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            Do = oracle.stft(y, **kw)
        yr = lb.istft(Do, hop_length=hop, n_fft=n_fft, length=y.shape[-1])
        err = yr - y
        snr = 10 * np.log10(float((y ** 2).sum()) / max(float((err ** 2).sum()), 1e-30))
        assert snr >= 60.0, (n_fft, hop, snr)


# ------------------------------------------------------------------ API behaviour on the device path
def test_stft_layout_and_out(lb, oracle):
    import signals

    y = signals.make("A", (9000,), seed=1)
    D = lb.stft(y)
    assert D.shape == (1025, 18) and D.dtype == np.complex64
    assert D.flags.f_contiguous                      # same memory order as the reference (spectrum.py:356)
    out = np.zeros((1025, 30), dtype=np.complex64)   # oversize out -> prefix slice, returned by identity of base
    res = lb.stft(y, out=out)
    assert res.base is out or res is out
    np.testing.assert_array_equal(res, D)
    np.testing.assert_array_equal(out[:, 18:], 0)
    exact = np.zeros((1025, 18), dtype=np.complex64, order="F")
    assert lb.stft(y, out=exact) is exact
    yo = np.zeros(512 * (D.shape[1] - 1), dtype=np.float32)   # default istft length: hop * (T - 1)
    assert lb.istft(D, out=yo) is yo
    close(yo, oracle.istft(D), **TOL["istft"])


def test_multichannel_equals_per_channel(lb):
    import signals

    y = signals.make("C", (2, 3, 9000), seed=21)
    for fn, kw in [(lb.stft, {}), (lambda y, **k: lb.feature.melspectrogram(y=y, **k), dict(sr=22050)),
                   (lambda y, **k: lb.feature.mfcc(y=y, **k), dict(sr=22050, n_mfcc=13))]:
        full = fn(y, **kw)
        for i in range(2):
            for j in range(3):
                np.testing.assert_array_equal(full[i, j], fn(y[i, j], **kw))   # bit-identical: same kernel, same data


def test_device_resident_chain(lb, oracle):
    import signals

    y = signals.make("A", (4, 30000), seed=5)
    d = lb.to_device(y)
    D = lb.stft(d, n_fft=1024, hop_length=256)
    assert isinstance(D, lb.DeviceArray) and D.shape == (4, 513, 118) and D.layout == "ft"
    yr = lb.istft(D, hop_length=256, length=30000)
    assert isinstance(yr, lb.DeviceArray)
    back = yr.get()
    snr = 10 * np.log10((y.astype(np.float64) ** 2).sum() / ((y - back).astype(np.float64) ** 2).sum())
    assert snr >= 60.0, snr
    close(D.get(), oracle.stft(y, n_fft=1024, hop_length=256), **TOL["stft"])
    M = lb.feature.melspectrogram(y=d, sr=22050, n_fft=1024, hop_length=256)
    close(M.get(), oracle.melspectrogram(y=y, sr=22050, n_fft=1024, hop_length=256), **TOL["mel"])


def test_s_inputs_and_power_to_db(lb, oracle, golden):
    rng = np.random.default_rng(3)
    S = (np.abs(rng.standard_normal((2, 1025, 40))) ** 2).astype(np.float32)
    close(lb.feature.melspectrogram(S=S, sr=22050), oracle.melspectrogram(S=S, sr=22050), **TOL["mel"])
    Sp = golden["const/power_to_db_in"]
    close(lb.power_to_db(Sp), golden["const/power_to_db_out"], rtol=1e-5, atol_abs=1e-4)
    close(lb.power_to_db(Sp, ref=np.max), golden["const/power_to_db_out_refmax"], rtol=1e-5, atol_abs=1e-4)
    close(lb.power_to_db(Sp, top_db=40.0), golden["const/power_to_db_out_top40"], rtol=1e-5, atol_abs=1e-4)
    assert abs(float(lb.power_to_db(np.float32(2.0))) - 3.0103) < 1e-3
    L = oracle.power_to_db((np.abs(rng.standard_normal((2, 128, 50))) ** 2).astype(np.float32))
    close(lb.feature.mfcc(S=L, n_mfcc=20), oracle.mfcc(S=L, n_mfcc=20), **TOL["mfcc"])
    Sg, n_fft = lb._spectrogram(y=(0.1 * rng.standard_normal(8000)).astype(np.float32), n_fft=1024, hop_length=256, power=2.0)
    assert n_fft == 1024 and Sg.shape == (513, 32)


def test_ragged_and_edge_shapes(lb, oracle):
    import signals

    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        for n, n_fft, hop in [(1, 8, 2), (7, 16, 1), (2048, 2048, 2048), (2049, 2048, 4096), (100, 2048, 512), (33333, 2048, 511)]:
            y = signals.make("A", (n,), seed=n)
            close(lb.stft(y, n_fft=n_fft, hop_length=hop), oracle.stft(y, n_fft=n_fft, hop_length=hop), **TOL["stft"])
    y0 = np.zeros((0, 4096), dtype=np.float32)                       # empty batch
    assert lb.stft(y0).shape == (0, 1025, 9)
    assert lb.feature.melspectrogram(y=y0).shape == (0, 128, 9)
    z = np.zeros(4096, dtype=np.float32)                             # all-zero clip: amin floor and top_db clamp
    close(lb.feature.mfcc(y=z), oracle.mfcc(y=z), **TOL["mfcc"])


def test_float64_inputs_follow_librosa_dtypes(lb, oracle):
    """float64 / complex128 data is computed in float32 (default policy, one warning) and comes back in the
    dtype librosa returns; values agree with the float64 reference to float32 accuracy."""
    import signals

    y = signals.make("A", (9000,), seed=8).astype(np.float64)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        D = lb.stft(y)
        Do = oracle.stft(y)
        assert D.dtype == np.complex128 and D.shape == Do.shape
        np.testing.assert_allclose(D, Do, rtol=1e-4, atol=1e-5 * float(np.abs(Do).max()))
        M = lb.feature.melspectrogram(y=y, sr=22050)
        Mo = oracle.melspectrogram(y=y, sr=22050)
        assert M.dtype == Mo.dtype == np.float64
        np.testing.assert_allclose(M, Mo, rtol=1e-4, atol=1e-6 * float(Mo.max()))
        yr = lb.istft(Do, length=9000)
        assert yr.dtype == np.float64
        np.testing.assert_allclose(yr, y, atol=1e-5)


def test_griffinlim(lb, oracle):
    """SURVEY 8f rank 1: istft -> stft -> phase update iterated on the device.  With identical starting
    phases the first iterations track the oracle; after many iterations the phase of near-zero bins is
    ill-conditioned in the reference itself, so the long run is judged by spectral convergence."""
    import signals

    y = signals.make("B", (12000,), seed=4)
    S = np.abs(oracle.stft(y, n_fft=1024, hop_length=256))
    for kw in (dict(n_iter=1, rng=0), dict(n_iter=2, init=None), dict(n_iter=3, rng=3, length=12000, momentum=0.5)):
        got = lb.griffinlim(S, hop_length=256, **kw)
        want = oracle.griffinlim(S, hop_length=256, **kw)
        assert got.shape == want.shape and got.dtype == want.dtype
        np.testing.assert_allclose(got, want, rtol=0, atol=2e-3 * float(np.abs(want).max()))

    def inconsistency(x):
        R = np.abs(oracle.stft(np.asarray(x), n_fft=1024, hop_length=256))
        n = min(R.shape[-1], S.shape[-1])
        return float(np.linalg.norm(R[:, :n] - S[:, :n]) / np.linalg.norm(S[:, :n]))

    e0 = inconsistency(lb.griffinlim(S, hop_length=256, n_iter=0, rng=0))
    e32 = inconsistency(lb.griffinlim(S, hop_length=256, n_iter=32, rng=0))
    o32 = inconsistency(oracle.griffinlim(S, hop_length=256, n_iter=32, rng=0))
    assert e32 < 0.5 * e0 and e32 < 1.5 * o32 + 0.02, (e0, e32, o32)
    # batch: two channels give the per-channel results, and device inputs stay on the device
    S2 = np.stack([S, 0.5 * S])
    g2 = lb.griffinlim(S2, hop_length=256, n_iter=2, init=None)
    np.testing.assert_allclose(g2[0], lb.griffinlim(S, hop_length=256, n_iter=2, init=None), rtol=1e-5, atol=1e-6)
    assert isinstance(lb.griffinlim(lb.to_device(S), hop_length=256, n_iter=1, init=None), lb.DeviceArray)
    with pytest.raises(lb.ParameterError):
        lb.griffinlim(S, init="garbage")
    with pytest.raises(lb.ParameterError):
        lb.griffinlim(S, momentum=-1)


def test_nonfinite_input_raises_like_valid_audio(lb):
    """util.valid_audio's finite check (librosa/util/utils.py:303-306) runs on the device: same exception,
    same message, for a bad sample anywhere — inside a frame, in the uncovered tail, or in a hop gap."""
    y = np.zeros((3, 20000), dtype=np.float32)
    for bad_pos, kw in [(12345, {}), (19999, dict(center=False, hop_length=1500)), (3000, dict(n_fft=256, hop_length=1024)),
                        (0, {}), (19999, {})]:
        for bad in (np.nan, np.inf, -np.inf):
            z = y.copy()
            z[1, bad_pos] = bad
            for fn in (lambda a: lb.stft(a, **kw), lambda a: lb.feature.melspectrogram(y=a, **kw),
                       lambda a: lb.feature.mfcc(y=a, **kw)):
                with pytest.raises(lb.ParameterError, match="not finite everywhere"):
                    fn(z)
    assert np.isfinite(lb.stft(y)).all()          # and the flag does not stick


# ------------------------------------------------------------------ BASELINE.json sizes: size-independent properties
def _block(n_clips, n, seed=0):
    import signals

    base = signals.make("A", (64, n), seed=seed)
    reps = -(-n_clips // 64)
    scale = (1.0 + 0.01 * np.arange(reps, dtype=np.float32))[:, None, None]
    return (base[None] * scale).reshape(-1, n)[:n_clips]


def test_cfg1_single_60s_clip(lb, oracle):
    """cfg 1: one 60 s mono clip @ 22050, stft 2048/512 center=True, and its inverse — a single clip is split
    into many frame segments per CTA half (halo frames recomputed at every segment start)."""
    import signals

    y = signals.make("B", (1323000,), seed=0)
    D = lb.stft(y, n_fft=2048, hop_length=512)
    Do = oracle.stft(y, n_fft=2048, hop_length=512)
    assert D.shape == (1025, 2584)
    close(D, Do, **TOL["stft"])
    yr = lb.istft(Do, hop_length=512, length=len(y))
    yo = oracle.istft(Do, hop_length=512, length=len(y))
    close(yr, yo, **TOL["istft"])
    snr = 10 * np.log10((y.astype(np.float64) ** 2).sum() / ((y - yr).astype(np.float64) ** 2).sum())
    assert snr >= 60.0, snr


@pytest.mark.parametrize("n_fft,hop,window", [(256, 300, "hann"), (256, 256, "hann"), (512, 128, "blackmanharris"),
                                              (1024, 512, "hann"), (64, 100, "hamming"), (2048, 2048, "hann")])
def test_istft_hop_geometries(lb, oracle, n_fft, hop, window):
    """hop > n_fft leaves gaps (window-sum-square is 0 there and the output stays 0), hop == n_fft has no
    overlap, small hops have deep overlap; several clips so that segment boundaries are exercised."""
    import signals

    y = signals.make("A", (3, 20000), seed=n_fft + hop)
    D = oracle.stft(y, n_fft=n_fft, hop_length=hop, window=window)
    for length in (None, 20000):
        got = lb.istft(D, hop_length=hop, window=window, length=length)
        want = oracle.istft(D, hop_length=hop, window=window, length=length)
        assert got.shape == want.shape
        T = D.shape[-1] if not length else min(D.shape[-1], int(np.ceil((length + 2 * (n_fft // 2)) / hop)))
        _istft_close(oracle, got, want, dict(hop_length=hop, window=window), n_fft, T)


def test_cfg2_full_size_mel_properties(lb, oracle):
    """cfg 2: 1024 clips x 10 s @ 22050 -> melspectrogram 2048/512/128."""
    Y = _block(1024, 220500)
    d = lb.to_device(Y)
    M = lb.feature.melspectrogram(y=d, sr=22050, n_fft=2048, hop_length=512)
    assert M.shape == (1024, 128, 431)
    Mh = M.get()
    assert np.isfinite(Mh).all() and (Mh >= 0).all()
    # power-2 homogeneity: clip 64*r + i is clip i scaled by (1 + 0.01 r) -> mel scales by its square
    for r in (1, 7, 15):
        s = np.float64(1.0 + 0.01 * r) ** 2
        np.testing.assert_allclose(Mh[64 * r : 64 * r + 64], Mh[:64] * s, rtol=2e-5)
    # sampled clips against the oracle
    for i in (0, 63, 517, 1023):
        close(Mh[i], oracle.melspectrogram(y=Y[i], sr=22050, n_fft=2048, hop_length=512), **TOL["mel"])
    # checksum of checksums: the batch result equals per-clip results
    for i in (5, 1000):
        np.testing.assert_array_equal(Mh[i], lb.feature.melspectrogram(y=Y[i], sr=22050, n_fft=2048, hop_length=512))


def test_cfg5_round_trip_snr(lb):
    """cfg 5: stft -> istft on 2048 clips x 10 s, 2048/512, reconstruction SNR >= 60 dB (per clip)."""
    Y = _block(2048, 220500, seed=9)
    d = lb.to_device(Y)
    D = lb.stft(d, n_fft=2048, hop_length=512)
    assert D.shape == (2048, 1025, 431)
    yr = lb.istft(D, hop_length=512, length=220500).get()
    D.free()
    err = ((Y - yr).astype(np.float64) ** 2).sum(axis=1)
    sig = (Y.astype(np.float64) ** 2).sum(axis=1)
    snr = 10 * np.log10(sig / np.maximum(err, 1e-300))
    assert snr.min() >= 60.0, snr.min()


def _fetch_clip(lb, dev, index, per_clip_shape, dtype):
    """One clip's block of a device-resident result (memory layout [clip][...]) without downloading the rest."""
    import ctypes as C

    from librosa_b200 import _native as nat

    host = np.empty(per_clip_shape, dtype=dtype)
    nat.check(nat.lib().b2l_d2h(dev.ctx.handle, host.ctypes.data_as(C.c_void_p), C.c_void_p(dev.ptr + index * host.nbytes),
                                host.nbytes))
    dev.ctx.synchronize()
    return host


def test_cfg3_cfg4_full_shards_sampled(lb, oracle):
    """cfg 3 and cfg 4 at the per-GPU shard sizes of BASELINE.json — ONE launch over 2 048 channel-clips (1 024 stereo
    clips x 10 s @ 44.1 kHz, stft 4096/1024: 3.6 GB in, 14.5 GB out, device resident) and ONE over 512 clips x 30 s
    @ 16 kHz (mfcc 40 / 128 mels, 1024/256) — with clips sampled from the start, the middle and the end of the launch
    compared against the oracle, and stft linearity as the size-independent property."""
    Y = _block(2048, 441000, seed=3).reshape(1024, 2, 441000)
    d = lb.to_device(Y)
    D = lb.stft(d, n_fft=4096, hop_length=1024)
    assert D.shape == (1024, 2, 2049, 431)
    picks = {}
    for flat in (0, 67, 1023, 1500, 2047):                      # channel-clip index in launch order
        blk = _fetch_clip(lb, D, flat, (431, 2049), np.complex64)   # native layout [frame][bin]
        picks[flat] = blk.T
        close(picks[flat], oracle.stft(Y.reshape(2048, -1)[flat], n_fft=4096, hop_length=1024), **TOL["stft"])
    D.free()
    d.free()
    flatY = Y.reshape(2048, -1)
    both = lb.stft(flatY[0] + flatY[1500], n_fft=4096, hop_length=1024)
    scale = float(np.abs(both).max())
    np.testing.assert_allclose(both, picks[0] + picks[1500], rtol=1e-4, atol=2e-6 * scale)
    del Y, flatY
    Z = _block(512, 480000, seed=4)
    C_ = lb.feature.mfcc(y=lb.to_device(Z), sr=16000, n_mfcc=40, n_fft=1024, hop_length=256).get()
    assert C_.shape == (512, 40, 1876)
    for i in (0, 129, 300, 511):
        close(C_[i], oracle.mfcc(y=Z[i], sr=16000, n_mfcc=40, n_fft=1024, hop_length=256), **TOL["mfcc"])


def test_more_than_65535_clips_through_the_helpers(lb, oracle):
    """Batches of more than 65 535 (short) clips: the main kernels walk (clip, tile) pairs in grid.x and always took
    them; the helpers around them (finite scan, layout transpose of a C-ordered STFT, power_to_db with its per-clip
    maximum) carry the clip index in grid.y / grid.z and now run in slices."""
    rng = np.random.default_rng(3)
    y = (0.1 * rng.standard_normal((70001, 96))).astype(np.float32)
    kw = dict(n_fft=32, hop_length=8)
    D = lb.stft(y, **kw)
    Do = oracle.stft(y, **kw)
    close(D, Do, **TOL["stft"])
    yr = lb.istft(np.ascontiguousarray(Do), hop_length=8, length=96)      # C-ordered host matrix
    assert yr.shape == y.shape
    np.testing.assert_allclose(yr, y, atol=2e-6)
    S = (np.abs(Do[:, :, :6]) ** 2).astype(np.float32)                   # (70001, 17, 6): 70 001 leading indices
    close(lb.power_to_db(S, top_db=30.0), oracle.power_to_db(S, top_db=30.0), rtol=1e-5, atol_abs=1e-4)


def test_pinned_host_end_to_end(lb, oracle):
    import signals

    y = lb.pinned_empty((8, 50000), np.float32)
    y[...] = signals.make("B", (8, 50000), seed=2)
    M = lb.feature.melspectrogram(y=y, sr=22050)
    close(M, oracle.melspectrogram(y=np.array(y), sr=22050), **TOL["mel"])


def _y(lb):
    y = 0.1 * np.random.default_rng(5).standard_normal((2, 12000))
    return lb.default_context().to_device(y.astype(np.float32))


def _dev_c(lb, a):
    """A C-ordered device copy of a logical (..., bins, frames) array."""
    return lb.default_context().to_device(np.ascontiguousarray(a))


# (input builder, call, kernel launches of the call): every spectrogram input in the native [frame][bin] layout goes
# straight to its kernel, a C-ordered one costs exactly one transpose; host batches take no extra kernel
LAUNCHES = {
    "stft host": (lambda lb: np.zeros(4096, dtype=np.float32), lambda lb, x: lb.stft(x), 1),
    "mfcc host": (lambda lb: np.zeros(4096, dtype=np.float32), lambda lb, x: lb.feature.mfcc(y=x), 2),
    "stft": (_y, lambda lb, x: lb.stft(x), 1),
    "istft ft": (lambda lb: lb.stft(_y(lb)), lambda lb, x: lb.istft(x), 1),
    "istft c": (lambda lb: _dev_c(lb, lb.stft(_y(lb)).get()), lambda lb, x: lb.istft(x), 2),
    "_spectrogram": (_y, lambda lb, x: lb._spectrogram(y=x), 1),
    "melspectrogram": (_y, lambda lb, x: lb.feature.melspectrogram(y=x), 1),
    "melspectrogram S ft": (lambda lb: lb._spectrogram(y=_y(lb), power=2)[0],
                            lambda lb, x: lb.feature.melspectrogram(S=x), 1),
    "melspectrogram S c": (lambda lb: _dev_c(lb, lb._spectrogram(y=_y(lb), power=2)[0].get()),
                           lambda lb, x: lb.feature.melspectrogram(S=x), 2),
    "mfcc": (_y, lambda lb, x: lb.feature.mfcc(y=x), 2),   # fused mel kernel + clamp/DCT kernel
    "spectral_centroid": (_y, lambda lb, x: lb.feature.spectral_centroid(y=x), 1),
    "spectral_centroid S ft": (lambda lb: lb._spectrogram(y=_y(lb))[0],
                               lambda lb, x: lb.feature.spectral_centroid(S=x), 1),
    "spectral_centroid S c": (lambda lb: _dev_c(lb, lb._spectrogram(y=_y(lb))[0].get()),
                              lambda lb, x: lb.feature.spectral_centroid(S=x), 2),
    "spectral_contrast": (_y, lambda lb, x: lb.feature.spectral_contrast(y=x), 7),
    "spectral_contrast S ft": (lambda lb: lb._spectrogram(y=_y(lb))[0],
                               lambda lb, x: lb.feature.spectral_contrast(S=x), 6),
    "spectral_contrast S c": (lambda lb: _dev_c(lb, lb._spectrogram(y=_y(lb))[0].get()),
                              lambda lb, x: lb.feature.spectral_contrast(S=x), 7),
    "chroma_stft": (_y, lambda lb, x: lb.feature.chroma_stft(y=x, tuning=0.0), 3),
    "chroma_stft S ft": (lambda lb: lb._spectrogram(y=_y(lb), power=2)[0],
                         lambda lb, x: lb.feature.chroma_stft(S=x, tuning=0.0), 2),
    "chroma_stft S c": (lambda lb: _dev_c(lb, lb._spectrogram(y=_y(lb), power=2)[0].get()),
                        lambda lb, x: lb.feature.chroma_stft(S=x, tuning=0.0), 3),
    "onset_strength": (_y, lambda lb, x: lb.onset.onset_strength(y=x), 4),
    "decompose.hpss ft": (lambda lb: lb.stft(_y(lb)), lambda lb, x: lb.decompose.hpss(x), 2),
    "decompose.hpss c": (lambda lb: _dev_c(lb, lb.stft(_y(lb)).get()), lambda lb, x: lb.decompose.hpss(x), 3),
    "effects.harmonic": (_y, lambda lb, x: lb.effects.harmonic(x), 4),
    "phase_vocoder ft": (lambda lb: lb.stft(_y(lb)), lambda lb, x: lb.phase_vocoder(x, rate=1.25), 1),
    "phase_vocoder c": (lambda lb: _dev_c(lb, lb.stft(_y(lb)).get()), lambda lb, x: lb.phase_vocoder(x, rate=1.25), 2),
}


def test_launch_counter_and_no_fallback(lb):
    ctx = lb.default_context()
    counted = {}
    for name, (build, call, _) in LAUNCHES.items():
        x = build(lb)
        before = ctx.launch_count
        call(lb, x)
        counted[name] = ctx.launch_count - before
    assert counted == {name: expected for name, (_, _, expected) in LAUNCHES.items()}


def test_single_rank_communicator_roundtrip(lb, oracle):
    """b2l_comm_* through NCCL on ONE GPU (world = 1): unique id, init, broadcast, scatter, compute, gather,
    barrier, destroy — the product's split / join path exercised on a box that has a single GPU."""
    import signals
    from librosa_b200 import distributed as D

    ctx = lb.Context(0)
    comm = D.Communicator(ctx, 0, 1, lambda payload: payload)
    Y = signals.make("A", (6, 30000), seed=78)
    full = ctx.to_device(Y)
    shard = ctx.empty(Y.shape, np.float32)
    comm.scatter(full, shard)
    comm.broadcast(shard)
    M = lb.feature.melspectrogram(y=shard, sr=22050)
    out = ctx.empty(M.shape, np.float32)
    comm.gather(M, out)
    comm.barrier()
    ctx.synchronize()
    close(out.get(), oracle.melspectrogram(y=Y, sr=22050), **TOL["mel"])
    comm.close()


@pytest.mark.skipif("__import__('librosa_b200').device_count() < 2")
def test_two_rank_split_join_on_gpu(lb, oracle):
    """Two GPUs of one box: scatter a device-resident batch from rank 0 over NCCL, compute per rank,
    gather back (run under pytest on a >= 2 GPU box; each rank is a thread with its own context)."""
    import threading

    import signals
    from librosa_b200 import distributed as D

    Y = signals.make("A", (8, 40000), seed=77)
    box, results, errors = {}, {}, []
    ready = threading.Barrier(2)

    def bcast(payload):
        if payload is not None:
            box["uid"] = payload
        ready.wait()
        return box["uid"]

    def rank_fn(rank):
        try:
            ctx = lb.Context(rank)
            comm = D.Communicator(ctx, rank, 2, bcast)
            full = ctx.to_device(Y) if rank == 0 else None
            shard = ctx.empty((4, 40000), np.float32)
            comm.scatter(full, shard)
            M = lb.feature.melspectrogram(y=shard, sr=22050)
            out = ctx.empty((8,) + M.shape[1:], np.float32) if rank == 0 else None
            comm.gather(M, out)
            ctx.synchronize()
            comm.barrier()
            if rank == 0:
                results["mel"] = out.get()
            comm.close()
        except Exception as exc:  # pragma: no cover
            errors.append(exc)

    threads = [threading.Thread(target=rank_fn, args=(r,)) for r in range(2)]
    [t.start() for t in threads]
    [t.join(timeout=120) for t in threads]
    assert not errors, errors
    close(results["mel"], oracle.melspectrogram(y=Y, sr=22050), **TOL["mel"])


@pytest.mark.parametrize("mr", ["0", "1"], ids=["chirpz", "mixed_radix"])
def test_chirpz_frames_are_paired_inside_a_clip(lb, oracle, monkeypatch, mr):
    """Two frames share one complex chirp-z transform; the pairs must not straddle clips: a clip 80 dB louder
    (or a non-finite one) next to a quiet clip may not touch the quiet clip's spectrum.  Per-clip tolerance.
    n_fft = 400 runs on the mixed-radix kernel by default (one warp per frame: nothing is shared between frames);
    B2L_MR=0 sends it to the chirp-z kernels this test was written for.  The inverse is chirp-z either way."""
    import signals

    monkeypatch.setenv("B2L_MR", mr)

    quiet = signals.make("A", (1, 4000), seed=3)[0] * 1e-4
    loud = signals.make("A", (1, 4000), seed=4)[0]
    Y = np.stack([loud, quiet, loud]).astype(np.float32)
    kw = dict(n_fft=400, hop_length=160)                     # 26 frames per clip would pair evenly; 4001 -> odd count
    Yo = np.concatenate([Y, Y[:, :1]], axis=1)               # 4001 samples: 26 frames -> use hop 150 for an odd count
    kw = dict(n_fft=400, hop_length=150)
    D, Do = lb.stft(Yo, **kw), oracle.stft(Yo, **kw)
    assert D.shape[-1] % 2 == 1                              # odd frame count: the last frame of a clip rides alone
    for c in range(3):
        close(D[c], Do[c], rtol=1e-4, atol_rel=1e-5)      # relative to THIS clip's peak
    yr, yo = lb.istft(Do, hop_length=150, n_fft=400, length=Yo.shape[-1]), oracle.istft(Do, hop_length=150, n_fft=400,
                                                                                      length=Yo.shape[-1])
    for c in range(3):
        close(yr[c], yo[c], rtol=1e-4, atol_rel=2e-5)
    # a clip with a NaN poisons only itself (device-resident input: no valid_audio check in front)
    Yn = Yo.copy()
    Yn[0, 100] = np.nan
    Dn = lb.stft(lb.to_device(Yn), **kw).get()
    assert np.isnan(Dn[0]).any() and np.isfinite(Dn[1]).all() and np.isfinite(Dn[2]).all()
