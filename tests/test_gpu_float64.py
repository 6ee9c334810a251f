"""GPU (-m gpu): the FP64 path (csrc/f64_kernels.cuh, csrc/f64_api.cu, librosa_b200/_f64.py) at every size class it
serves, against the oracle (oracle/ref_np.py: the window product and scipy.fft.rfft / irfft in float64, pinned to the
reference's own fixtures by test_oracle_golden.py).  Nothing here reads the reference tree.

The FP64 kernels serve float64 / complex128 data, and float32 host data at frame lengths the float32 kernels are not
built for (``_pipeline.wide_route``).  The size classes are written as the switch points themselves:

    tiny          2, 3, 5, 6, 7 (direct DFT) and 4, 8 (radix-2 with log2m 1 and 2)
    FFT, shared   16 ... 16 384 (n_fft/2 complex doubles: exactly 128 KiB at 16 384)
    FFT, global   32 768 ... 2^20 (work area in global memory, one slice per frame)
    DFT, shared   1000 ... 16 383 (forward: n_fft doubles; inverse: n_fft/2 + 1 complex doubles = 128 KiB at 16 383)
    DFT, global   16 385 ... 65 535
    refused       65 537 and 2^21 (UnsupportedOnGPU, for float64 and float32 host data)

Tolerances.  Per clip, relative to that clip's max|ref|; each is at least 1000x tighter than float32 rounding
(6e-8), so a single-precision twiddle table, window or accumulator fails them:
    radix-2 path (powers of two >= 4)            1e-13 * log2(n_fft)
    direct DFT (any other n_fft; it accumulates  1e-15 * n_fft
      sequentially over n_fft terms)
    istft                                        the same bound for its n_fft, on the un-normalised overlap-add
                                                 (y * window-sum-square, as _istft_close in test_gpu_parity.py)
    istft(stft(y)) == y where wss >= 1e-3        |y_rt - y| * wss <= 2 * bound * max|y * wss|
    melspectrogram                               rtol 1e-9, plus 1e-12 * max|ref|
    power_to_db / amplitude_to_db                rtol 1e-10, atol 1e-9 dB
    mfcc                                         rtol 1e-8, atol 1e-8
float32 data routed to FP64 is compared with the oracle evaluated in float64 on the same float32 samples; a result
computed in FP64 and rounded once to float32 / complex64 is within half an ulp of it, so element by element
    |got - ref| <= 1e-7 * |ref| + (the FP64 bound above).
"""
import warnings

import numpy as np
import pytest

from oracle import ref_np as O

pytestmark = [pytest.mark.gpu, pytest.mark.filterwarnings("ignore")]

PAD_MODES = ("constant", "reflect", "edge", "symmetric", "linear_ramp")


@pytest.fixture(scope="module")
def lb():
    import librosa_b200

    librosa_b200.default_context()
    return librosa_b200


def is_fft(n_fft: int) -> bool:
    """The FP64 kernels take the radix-2 path for powers of two >= 4, the direct DFT for everything else."""
    return n_fft >= 4 and (n_fft & (n_fft - 1)) == 0


def bound(n_fft: int) -> float:
    return 1e-13 * np.log2(n_fft) if is_fft(n_fft) else 1e-15 * n_fft


def signal(n: int, seed: int, dtype=np.float64, scales=(1.0, 1e-3, 1e3)) -> np.ndarray:
    """Noise + DC offset + tone, one independent clip per scale (never silence: a clip leaking into its neighbour,
    or a wrong per-frame work-area offset, shows in the quiet clip)."""
    rng = np.random.default_rng(seed)
    t = np.arange(n, dtype=np.float64)
    clips = [s * (0.3 * rng.standard_normal(n) + 0.2 + 0.5 * np.sin(2 * np.pi * (0.0371 + 0.01 * i) * t + i))
             for i, s in enumerate(scales)]
    return np.stack(clips).astype(dtype)


def per_clip_close(got, ref, atol_rel, rtol=0.0, what=""):
    """|got - ref| <= rtol |ref| + atol_rel * max|ref of that clip|, for every leading index; returns the largest
    error relative to the clip maximum."""
    got, ref = np.asarray(got), np.asarray(ref)
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    lead = ref.shape[:-2] if ref.ndim > 2 else ()
    g = got.reshape((-1,) + ref.shape[len(lead):]).astype(np.complex128 if np.iscomplexobj(got) else np.float64)
    r = ref.reshape(g.shape)
    worst = 0.0
    for c in range(g.shape[0]):
        scale = float(np.abs(r[c]).max())
        err = np.abs(g[c] - r[c])
        rel = float(err.max()) / scale if scale > 0 else float(err.max())
        worst = max(worst, rel)
        ok = err <= rtol * np.abs(r[c]) + atol_rel * scale
        assert ok.all(), f"{what} clip {c}: max |err| / max|ref| = {rel:.3e} (bound {atol_rel:.1e})"
    return worst


def natural_length(n_fft, hop, n_frames, center):
    return n_fft + hop * (n_frames - 1) - (2 * (n_fft // 2) if center else 0)


def trimmed_wss(n_fft, hop, win_length, n_frames, center, out_len):
    """The window-sum-square istft divides by, trimmed like istft does (core/spectrum.py:606-624)."""
    wss = O.window_sumsquare("hann", n_frames, hop_length=hop, win_length=win_length, n_fft=n_fft, dtype=np.float64)
    return O.fix_length(wss[(n_fft // 2 if center else 0):], out_len)


# ------------------------------------------------------------------ size classes
# (class, n_fft, hop, win_length, center, pad_mode): centre on / off, all five pad modes, hops that do not divide
# n_fft, one hop > n_fft per class, some win_length < n_fft.  Signals are ~3 * n_fft samples.
CASES = [
    ("tiny", 2, 1, None, True, "constant"),
    ("tiny", 3, 2, None, False, "constant"),
    ("tiny", 4, 3, 3, True, "reflect"),
    ("tiny", 5, 7, None, True, "edge"),
    ("tiny", 6, 4, None, True, "symmetric"),
    ("tiny", 7, 3, 5, False, "constant"),
    ("tiny", 8, 5, None, True, "linear_ramp"),
    ("fft_shared", 16, 5, None, True, "reflect"),
    ("fft_shared", 1024, 1500, None, False, "constant"),
    ("fft_shared", 4096, 1000, 3000, True, "edge"),
    ("fft_shared", 16384, 6000, None, True, "symmetric"),
    ("fft_global", 32768, 10000, None, True, "linear_ramp"),
    ("fft_global", 65536, 70000, None, True, "constant"),
    ("fft_global", 1 << 17, 50000, 100000, False, "constant"),
    ("fft_global", 1 << 20, 1 << 19, None, True, "reflect"),
    ("dft_shared", 1000, 333, None, True, "edge"),
    ("dft_shared", 3001, 4000, None, False, "constant"),
    ("dft_shared", 4097, 1000, 4000, True, "symmetric"),
    ("dft_shared", 12345, 5000, None, True, "linear_ramp"),
    ("dft_shared", 16383, 7000, None, True, "constant"),
    ("dft_global", 16385, 7001, None, True, "reflect"),
    ("dft_global", 30001, 12000, 25000, False, "constant"),
    ("dft_global", 65534, 70000, None, True, "edge"),
    ("dft_global", 65535, 30000, None, True, "symmetric"),
]
# the first case of every class also runs with a float64 DeviceArray input
DEVICE_CASES = {c[1] for i, c in enumerate(CASES) if i == 0 or CASES[i - 1][0] != c[0]}


def case_id(c):
    return f"{c[0]}-{c[1]}"


def case_signal(n_fft, seed):
    return signal(max(3 * n_fft, 40), seed)


@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_forward_float64_size_classes(lb, case):
    cls, n_fft, hop, win_length, center, pad_mode = case
    y = case_signal(n_fft, n_fft)
    kw = dict(n_fft=n_fft, hop_length=hop, win_length=win_length, center=center, pad_mode=pad_mode)
    ref = O.stft(y, **kw)
    assert ref.dtype == np.complex128
    D = lb.stft(y, **kw)
    assert D.dtype == np.complex128
    per_clip_close(D, ref, bound(n_fft), what=f"stft {cls} n_fft={n_fft}")
    if n_fft in DEVICE_CASES:
        dev = lb.default_context().to_device(y)
        Dd = lb.stft(dev, **kw)
        assert isinstance(Dd, lb.DeviceArray) and Dd.dtype == np.complex128 and Dd.layout == "ft"
        per_clip_close(Dd.get(), ref, bound(n_fft), what=f"device stft {cls} n_fft={n_fft}")


@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_inverse_float64_size_classes(lb, case):
    cls, n_fft, hop, win_length, center, pad_mode = case
    i = CASES.index(case)
    y = case_signal(n_fft, n_fft + 1)
    n = y.shape[-1]
    Do = O.stft(y, n_fft=n_fft, hop_length=hop, win_length=win_length, center=center, pad_mode=pad_mode)
    T = Do.shape[-1]
    nat_len = natural_length(n_fft, hop, T, center)
    length = [nat_len, max(1, nat_len - hop // 2 - 1), nat_len + n_fft // 3 + 5][i % 3]   # equal, shorter, longer
    kw = dict(n_fft=n_fft, hop_length=hop, win_length=win_length, center=center, length=length)
    ref = O.istft(Do, **kw)
    got = lb.istft(Do, **kw)
    assert got.dtype == ref.dtype == np.float64 and got.shape == ref.shape == (3, length)
    padded = length + 2 * (n_fft // 2) if center else length
    used = min(T, int(np.ceil(padded / hop)))
    wss = trimmed_wss(n_fft, hop, win_length, used, center, length)
    w = np.where(wss > O.tiny(wss), wss, 1.0)
    per_clip_close(got * w, ref * w, bound(n_fft), what=f"istft {cls} n_fft={n_fft} length={length}")
    # the round trip, wherever the window-sum-square is not tiny
    m = min(n, length)
    mask = wss[:m] >= 1e-3
    assert mask.any()
    for c in range(3):
        lim = 2 * bound(n_fft) * float(np.abs(y[c, :m] * wss[:m]).max())
        err = np.abs(got[c, :m] - y[c, :m]) * wss[:m]
        assert (err[mask] <= lim).all(), (cls, n_fft, c, float(err[mask].max()), lim)
    if hop > n_fft:   # the gaps between frames come back as exact zeros
        gaps = wss == 0
        assert gaps.any() and not got[:, gaps].any()


# ------------------------------------------------------------------ refusals
@pytest.mark.parametrize("n_fft", [65537, 1 << 21])
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_sizes_beyond_the_fp64_kernels_are_refused(lb, n_fft, dtype):
    y = signal(70000, 5, dtype=dtype, scales=(1.0,))[0]
    with pytest.raises(lb.UnsupportedOnGPU):
        lb.stft(y, n_fft=n_fft, hop_length=n_fft // 2)


def test_float32_device_input_is_not_routed_to_fp64(lb):
    """wide_route only takes float32 host data: a float32 DeviceArray at a size the float32 kernels lack is refused."""
    dev = lb.default_context().to_device(signal(50000, 6, dtype=np.float32, scales=(1.0,)))
    with pytest.raises(lb.UnsupportedOnGPU):
        lb.stft(dev, n_fft=16384)


# ------------------------------------------------------------------ float32 host data routed to FP64
ROUTED = [2, 4, 16384, 32768, 4097, 20001]


def _routed_kw(n_fft):
    return dict(n_fft=n_fft, hop_length=max(1, n_fft // 3 + 1))


def _mel_kw(n_fft):
    n_mels = 4 if n_fft < 16 else 64
    return dict(sr=22050, n_mels=n_mels)


def routed_close(got, ref, n_fft, dtype, rtol=0.0, atol_rel=None):
    got = np.asarray(got)
    assert got.dtype == dtype, (got.dtype, dtype)
    return per_clip_close(got, ref, bound(n_fft) if atol_rel is None else atol_rel, rtol=1e-7 + rtol,
                          what=f"float32 -> FP64 n_fft={n_fft}")


@pytest.mark.parametrize("n_fft", ROUTED)
def test_float32_host_data_routed_to_fp64(lb, n_fft):
    y32 = signal(max(3 * n_fft, 64), 7 + n_fft, dtype=np.float32)
    y = y32.astype(np.float64)            # the same samples: what the oracle computes before rounding its output
    kw = _routed_kw(n_fft)
    routed_close(lb.stft(y32, **kw), O.stft(y, **kw), n_fft, np.complex64)
    S, n_out = lb._spectrogram(y=y32, power=1, **kw)
    assert n_out == n_fft
    routed_close(S, O.spectrogram(y, power=1, **kw), n_fft, np.float32)
    mk = _mel_kw(n_fft)
    routed_close(lb.feature.melspectrogram(y=y32, **kw, **mk), O.melspectrogram(y=y, **kw, **mk), n_fft, np.float32,
                 rtol=1e-9, atol_rel=1e-12)
    n_mfcc = min(13, mk["n_mels"])
    got = lb.feature.mfcc(y=y32, n_mfcc=n_mfcc, **kw, **mk)
    ref = O.mfcc(y=y, n_mfcc=n_mfcc, **kw, **mk)
    assert got.dtype == np.float32 and got.shape == ref.shape
    assert (np.abs(got - ref) <= (1e-7 + 1e-8) * np.abs(ref) + 1e-8).all(), float(np.abs(got - ref).max())
    # istft of complex64 host data
    D32 = O.stft(y32, **kw)
    assert D32.dtype == np.complex64
    length = y32.shape[-1]
    got = lb.istft(D32, length=length, **kw)
    ref = O.istft(D32.astype(np.complex128), length=length, **kw)
    assert got.dtype == np.float32
    used = min(D32.shape[-1], int(np.ceil((length + 2 * (n_fft // 2)) / kw["hop_length"])))
    wss = trimmed_wss(n_fft, kw["hop_length"], None, used, True, length)
    w = np.where(wss > O.tiny(wss), wss, 1.0)
    routed_close(got.astype(np.float64) * w, ref * w, n_fft, np.float64)


# ------------------------------------------------------------------ mel, dB and DCT in float64
@pytest.mark.parametrize("n_mels", [1, 16, 128, 256])
@pytest.mark.parametrize("n_fft", [4096, 16384, 32768, 5000])
def test_melspectrogram_float64(lb, n_fft, n_mels):
    y = signal(3 * n_fft, n_fft + n_mels)
    kw = dict(sr=22050, n_fft=n_fft, hop_length=n_fft // 3 + 1, n_mels=n_mels)
    got, ref = lb.feature.melspectrogram(y=y, **kw), O.melspectrogram(y=y, **kw)
    assert got.dtype == ref.dtype == np.float64
    per_clip_close(got, ref, 1e-12, rtol=1e-9, what=f"mel n_fft={n_fft} n_mels={n_mels}")


def test_melspectrogram_float64_empty_rows_are_zero(lb):
    """256 mel bands over 257 bins: many filters are empty, and those rows are exactly 0, as in the reference."""
    y = signal(4000, 11)
    kw = dict(sr=22050, n_fft=512, hop_length=200, n_mels=256)
    basis = O.mel(sr=22050, n_fft=512, n_mels=256)
    empty = basis.max(axis=1) == 0
    assert empty.sum() > 10
    got, ref = lb.feature.melspectrogram(y=y, **kw), O.melspectrogram(y=y, **kw)
    assert not ref[:, empty].any() and not got[:, empty].any()
    per_clip_close(got, ref, 1e-12, rtol=1e-9, what="mel with empty rows")


@pytest.mark.parametrize("n_fft,n_mels,extra", [
    (4096, 128, dict(n_mfcc=128)),
    (16384, 64, dict(n_mfcc=40, lifter=22)),
    (5000, 128, dict(n_mfcc=20, dct_type=3)),
    (32768, 128, dict(n_mfcc=128, norm=None)),
])
def test_mfcc_float64(lb, n_fft, n_mels, extra):
    y = signal(3 * n_fft, n_fft + 3)
    kw = dict(sr=22050, n_fft=n_fft, hop_length=n_fft // 3 + 1, n_mels=n_mels, **extra)
    got, ref = lb.feature.mfcc(y=y, **kw), O.mfcc(y=y, **kw)
    assert got.dtype == ref.dtype == np.float64 and got.shape == ref.shape
    np.testing.assert_allclose(got, ref, rtol=1e-8, atol=1e-8)


def test_mfcc_float64_dct_too_large_for_shared_memory_is_refused(lb):
    """256 mel bands x 128 coefficients: a 256 KiB DCT matrix, more than one CTA's shared memory."""
    y = signal(8192, 12)
    with pytest.raises(lb.UnsupportedOnGPU):
        lb.feature.mfcc(y=y, sr=22050, n_fft=2048, n_mels=256, n_mfcc=128)


@pytest.mark.parametrize("kw", [dict(), dict(top_db=None), dict(ref=np.max), dict(ref=np.median),
                                dict(ref=np.max, top_db=40.0), dict(amin=1e-4, top_db=None)],
                         ids=["default", "top_db_none", "ref_max", "ref_median", "ref_max_top_db_40", "amin"])
def test_power_and_amplitude_to_db_float64(lb, kw):
    rng = np.random.default_rng(13)
    S = np.abs(O.stft(signal(6000, 13)[:, None, :].repeat(2, axis=1) * rng.uniform(0.5, 2.0, (1, 2, 1)),
                      n_fft=256, hop_length=100)) ** 2                       # (3, 2, 129, 61): six leading indices
    for fn, ofn, X in ((lb.power_to_db, O.power_to_db, S), (lb.amplitude_to_db, O.amplitude_to_db, np.sqrt(S))):
        for arr in (X, X[0, 0], X[1, 1, 5]):                                # several leading indices, 2-D, 1-D
            got, ref = fn(arr, **kw), ofn(arr, **kw)
            assert got.dtype == np.float64 and got.shape == ref.shape
            np.testing.assert_allclose(got, ref, rtol=1e-10, atol=1e-9, err_msg=f"{fn.__name__} {kw} {arr.shape}")


# ------------------------------------------------------------------ util.valid_audio on the FP64 path
def _nonfinite_positions(n_fft):
    """(position, kwargs): inside a frame, in the tail after the last frame (center=False), in a hop gap, first and
    last sample, and under a zero tap of the periodic Hann window (hop == n_fft, center=False: one frame reads it)."""
    if n_fft == 2048:                     # float64 data at the default frame length, 20 000 samples
        return [(12345, {}), (19999, dict(center=False, hop_length=1500)), (2500, dict(n_fft=256, hop_length=1024)),
                (1200, dict(n_fft=1024, hop_length=1500, center=False)), (0, {}), (19999, {}),
                (4096, dict(n_fft=1024, hop_length=1024, center=False))]
    # float32 data at n_fft 16 384 (FP64 kernels), 60 000 samples
    return [(30000, {}), (59999, dict(center=False, hop_length=15000)), (10000, dict(hop_length=20000)), (0, {}),
            (59999, {}), (16384, dict(hop_length=16384, center=False))]


@pytest.mark.parametrize("dtype,n_fft,n", [(np.float64, 2048, 20000), (np.float32, 16384, 60000)],
                         ids=["float64", "float32_16384"])
def test_nonfinite_input_raises_like_valid_audio(lb, dtype, n_fft, n):
    y = signal(n, 17, dtype=dtype)
    fns = (lambda a, kw: lb.stft(a, **kw), lambda a, kw: lb._spectrogram(y=a, **kw),
           lambda a, kw: lb.feature.melspectrogram(y=a, **kw), lambda a, kw: lb.feature.mfcc(y=a, **kw))
    for pos, extra in _nonfinite_positions(n_fft):
        kw = dict(n_fft=n_fft, hop_length=n_fft // 4)
        kw.update(extra)
        for bad in (np.nan, np.inf, -np.inf):
            z = y.copy()
            z[1, pos] = bad
            for fn in fns:
                with pytest.raises(lb.ParameterError, match="not finite everywhere"):
                    fn(z, kw)
            D = lb.stft(y, **kw)                    # a clean call right after a failing one sees no stale flag
            assert np.isfinite(D).all()


def test_nan_in_a_hop_gap_of_float64_audio(lb):
    """No frame reads sample 1200 (frames [0, 1024) and [1500, 2524)); util.valid_audio still rejects it."""
    y = signal(5000, 19)[0]
    y[1200] = np.nan
    with pytest.raises(lb.ParameterError, match="not finite everywhere"):
        lb.stft(y, n_fft=1024, hop_length=1500, center=False)


def test_large_finite_float64_samples_are_accepted(lb):
    """np.isfinite accepts 1e301 and +-1.7e308, and so does the FP64 path (the spectrum may overflow to inf, as in
    the reference)."""
    y = signal(20000, 23)
    z = y.copy()
    z[0, 777] = 1e301
    z[2, 12345] = -1e301
    kw = dict(n_fft=1024, hop_length=256)
    D = lb.stft(z, **kw)
    per_clip_close(D, O.stft(z, **kw), bound(1024), what="stft with 1e301")
    for fn in (lambda a: lb._spectrogram(y=a, **kw), lambda a: lb.feature.melspectrogram(y=a, **kw),
               lambda a: lb.feature.mfcc(y=a, **kw)):
        fn(z)
    w = y.copy()
    w[1, 5000] = 1.7e308
    w[1, 9000] = -1.7e308
    w[2, 0] = np.finfo(np.float64).max
    D = lb.stft(w, **kw)
    assert D.dtype == np.complex128
    assert np.isfinite(D[0]).all()               # the clean clip is untouched
    lb._spectrogram(y=w, **kw)
    lb.feature.melspectrogram(y=w, **kw)


# ------------------------------------------------------------------ more than 65 535 leading indices
def test_more_than_65535_clips_float64(lb):
    rng = np.random.default_rng(29)
    y = 0.1 * rng.standard_normal((70001, 96)) + 0.05
    kw = dict(n_fft=32, hop_length=8)
    Do = O.stft(y, **kw)                                                  # (70001, 17, 13) complex128
    S = np.abs(Do[:, :, :6]) ** 2                                         # (70001, 17, 6)
    got = lb.power_to_db(S)
    assert got.dtype == np.float64
    np.testing.assert_allclose(got, O.power_to_db(S), rtol=1e-10, atol=1e-9)
    mk = dict(n_mels=8, n_mfcc=4, sr=22050)
    C_ = lb.feature.mfcc(y=y, **kw, **mk)
    assert C_.dtype == np.float64
    np.testing.assert_allclose(C_, O.mfcc(y=y, **kw, **mk), rtol=1e-8, atol=1e-8)
    yr = lb.istft(Do, hop_length=8)
    ref = O.istft(Do, hop_length=8)
    assert yr.dtype == np.float64 and yr.shape == ref.shape == (70001, 96)
    np.testing.assert_allclose(yr, ref, rtol=0, atol=bound(32) * float(np.abs(ref).max()))


# ------------------------------------------------------------------ launch counts
def _y64(n_clips=2, n=12000):
    return 0.1 * np.random.default_rng(31).standard_normal((n_clips, n)) + 0.05


def _S64(n_clips):
    return np.abs(np.random.default_rng(37).standard_normal((n_clips, 17, 6))) + 1e-3


# (input builder, call, kernel launches of the call), float64 data.  A host signal adds one finite-scan launch when
# some of its samples are read by no frame (the tail after the last frame with center=False, or every sample when
# hop > n_fft leaves gaps), as on the float32 path; a device signal is not validated and adds none.  Helpers that
# carry the clip index in grid.y run in slices of 65 535 clips: no extra launch up to 65 535 clips.
LAUNCHES = {
    "stft": (lambda lb: _y64(), lambda lb, x: lb.stft(x), 1),
    "stft device": (lambda lb: lb.to_device(_y64()), lambda lb, x: lb.stft(x), 1),
    "stft, uncovered tail (+1 scan)": (lambda lb: _y64(n=12001), lambda lb, x: lb.stft(x, center=False, hop_length=1000), 2),
    "stft, hop > n_fft (+1 scan)": (lambda lb: _y64(), lambda lb, x: lb.stft(x, n_fft=256, hop_length=300), 2),
    "istft": (lambda lb: O.stft(_y64()), lambda lb, x: lb.istft(x), 2),
    "melspectrogram": (lambda lb: _y64(), lambda lb, x: lb.feature.melspectrogram(y=x), 3),
    "mfcc (top_db 80)": (lambda lb: _y64(), lambda lb, x: lb.feature.mfcc(y=x), 6),
    "power_to_db top_db": (lambda lb: _S64(2), lambda lb, x: lb.power_to_db(x), 2),
    "power_to_db top_db=None": (lambda lb: _S64(2), lambda lb, x: lb.power_to_db(x, top_db=None), 1),
    "power_to_db 65535 clips": (lambda lb: _S64(65535), lambda lb, x: lb.power_to_db(x), 2),
    "power_to_db 65536 clips (two slices)": (lambda lb: _S64(65536), lambda lb, x: lb.power_to_db(x), 4),
    "mfcc 65535 clips": (lambda lb: _y64(65535, 96), lambda lb, x: lb.feature.mfcc(y=x, n_fft=32, hop_length=8,
                                                                                     n_mels=8, n_mfcc=4), 6),
    "istft 65535 clips": (lambda lb: O.stft(_y64(65535, 96), n_fft=32, hop_length=8),
                          lambda lb, x: lb.istft(x, hop_length=8), 2),
}


def test_float64_launch_counts(lb):
    ctx = lb.default_context()
    counted = {}
    for name, (build, call, _) in LAUNCHES.items():
        x = build(lb)
        before = ctx.launch_count
        call(lb, x)
        counted[name] = ctx.launch_count - before
    assert counted == {name: expected for name, (_, _, expected) in LAUNCHES.items()}
