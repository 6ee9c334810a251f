"""CPU: host-side logic of the drop-in layer — array helpers, constant builders and the argument
validation that must raise exactly like the reference *before* any GPU work
(reference tests: tests/test_util.py:23-170, tests/test_filters.py:120-210, 486-514,
tests/test_core.py:295-314, tests/test_failures.py:76-127, tests/test_features.py:890-894)."""
import warnings

import os

import numpy as np
import pytest
import scipy.signal

import librosa_b200 as lb
from librosa_b200 import ParameterError, UnsupportedOnGPU


# ------------------------------------------------------------------ util.frame
@pytest.mark.parametrize("frame_length,hop_length", [(4, 1), (4, 3), (16, 7), (50, 50)])
def test_frame_1d(frame_length, hop_length):
    y = np.arange(103.0)
    f = lb.util.frame(y, frame_length=frame_length, hop_length=hop_length)
    assert f.shape == (frame_length, 1 + (len(y) - frame_length) // hop_length)
    for j in range(f.shape[1]):
        np.testing.assert_array_equal(f[:, j], y[j * hop_length : j * hop_length + frame_length])
    assert not f.flags.writeable
    assert np.shares_memory(f, y)


def test_frame_axes():
    x = np.arange(2 * 3 * 40.0).reshape(2, 3, 40)
    f = lb.util.frame(x, frame_length=8, hop_length=4)            # axis=-1 -> (..., frame_length, n_frames)
    assert f.shape == (2, 3, 8, 9)
    np.testing.assert_array_equal(f[1, 2, :, 3], x[1, 2, 12:20])
    g = lb.util.frame(x, frame_length=2, hop_length=1, axis=0)    # axis=0 -> (n_frames, frame_length, ...)
    assert g.shape == (1, 2, 3, 40)
    np.testing.assert_array_equal(g[0], x)


def test_frame_errors():
    with pytest.raises(ParameterError):
        lb.util.frame(np.zeros(10), frame_length=11, hop_length=1)
    with pytest.raises(ParameterError):
        lb.util.frame(np.zeros(10), frame_length=4, hop_length=0)


# ------------------------------------------------------------------ small helpers
def test_pad_center_fix_length_tiny_dtypes():
    w = lb.util.pad_center(np.ones(5), size=12)
    np.testing.assert_array_equal(w, [0, 0, 0, 1, 1, 1, 1, 1, 0, 0, 0, 0])
    with pytest.raises(ParameterError):
        lb.util.pad_center(np.ones(5), size=4)
    np.testing.assert_array_equal(lb.util.fix_length(np.arange(5), size=3), [0, 1, 2])
    np.testing.assert_array_equal(lb.util.fix_length(np.arange(3), size=5), [0, 1, 2, 0, 0])
    assert lb.util.tiny(np.float32(1.0)) == np.finfo(np.float32).tiny
    assert lb.util.tiny(3) == np.finfo(np.float32).tiny
    assert lb.util.dtype_r2c(np.float32) == np.complex64 and lb.util.dtype_r2c(np.float64) == np.complex128
    assert lb.util.dtype_c2r(np.complex64) == np.float32 and lb.util.dtype_c2r(np.complex128) == np.float64
    assert lb.util.dtype_r2c(np.int16) == np.complex64 and lb.util.dtype_c2r(np.float32) == np.float32
    assert lb.util.expand_to(np.arange(3), ndim=3, axes=-2).shape == (1, 3, 1)
    assert lb.util.is_positive_int(3) and not lb.util.is_positive_int(0) and not lb.util.is_positive_int(2.0)
    x = np.array([3 + 4j, 1 - 1j])
    np.testing.assert_allclose(lb.util.abs2(x), np.abs(x) ** 2)


def test_valid_audio():
    assert lb.util.valid_audio(np.zeros(4, dtype=np.float32))
    for bad in ([0.0, 1.0], np.zeros(4, dtype=np.int16), np.float32(1.0) * np.ones(()), np.array([0.0, np.nan])):
        with pytest.raises(ParameterError):
            lb.util.valid_audio(bad)


# ------------------------------------------------------------------ filters
def test_get_window():
    for w in ["hann", "hamming", ("kaiser", 4.0), 4.0]:
        np.testing.assert_array_equal(lb.filters.get_window(w, 32), scipy.signal.get_window(w, 32, fftbins=True))
    np.testing.assert_array_equal(lb.filters.get_window(np.ones(8), 8), np.ones(8))
    assert np.allclose(lb.filters.get_window(lambda n: np.arange(n), 4), [0, 1, 2, 3])
    with pytest.raises(ParameterError):
        lb.filters.get_window(np.ones(7), 8)
    with pytest.raises(ParameterError):
        lb.filters.get_window(None, 8)


@pytest.mark.parametrize("n_fft,n_mels,htk", [(2048, 128, False), (2048, 40, True), (1024, 128, False)])
def test_mel_properties(n_fft, n_mels, htk):
    sr = 22050
    W = lb.filters.mel(sr=sr, n_fft=n_fft, n_mels=n_mels, htk=htk)
    assert W.shape == (n_mels, 1 + n_fft // 2) and W.dtype == np.float32
    assert (W >= 0).all()
    # every filter peaks within one bin of its mel centre (reference tests/test_filters.py:120-165)
    centres = lb.mel_frequencies(n_mels + 2, fmin=0, fmax=sr / 2, htk=htk)[1:-1]
    bins = lb.fft_frequencies(sr=sr, n_fft=n_fft)
    peak = bins[W.argmax(axis=1)]
    assert np.all(np.abs(peak - centres) <= sr / n_fft)
    # band structure the CUDA kernel relies on: contiguous support, <= 2 filters per bin
    assert ((W > 0).sum(axis=0) <= 2).all()
    for row in W:
        nz = np.flatnonzero(row)
        assert nz.size == 0 or nz[-1] - nz[0] + 1 == nz.size


def test_mel_golden_and_norms(golden):
    np.testing.assert_array_equal(lb.filters.mel(sr=22050, n_fft=2048), golden["const/mel_22050_2048"])
    np.testing.assert_array_equal(lb.filters.mel(sr=44100, n_fft=4096), golden["const/mel_44100_4096"])
    np.testing.assert_array_equal(lb.filters.mel(sr=16000, n_fft=1024, n_mels=40, htk=True), golden["const/mel_16000_1024_htk40"])
    np.testing.assert_allclose(lb.filters.mel(sr=22050, n_fft=2048, norm=1, fmin=300.0, fmax=8000.0, n_mels=64),
                               golden["const/mel_22050_2048_norm1"], rtol=1e-6)
    W1 = lb.filters.mel(sr=22050, n_fft=2048, norm=1)
    np.testing.assert_allclose(W1.sum(axis=1), 1.0, rtol=1e-5)
    with pytest.raises(ParameterError):
        lb.filters.mel(sr=22050, n_fft=2048, norm="bogus")
    with pytest.warns(UserWarning, match="Empty filters"):
        lb.filters.mel(sr=22050, n_fft=64, n_mels=128)


def test_window_sumsquare_and_scales(golden):
    np.testing.assert_allclose(lb.filters.window_sumsquare(window="hann", n_frames=50, hop_length=512, n_fft=2048),
                               golden["const/wss_hann_2048_512_50"], rtol=1e-6)
    np.testing.assert_allclose(
        lb.filters.window_sumsquare(window="hamming", n_frames=20, hop_length=300, win_length=600, n_fft=1024),
        golden["const/wss_hamming_600_1024_300_20"], rtol=1e-6)
    f = np.array([0.0, 60.0, 440.0, 999.0, 1000.0, 5000.0, 11025.0])
    np.testing.assert_allclose(lb.hz_to_mel(f), golden["const/hz_to_mel"], rtol=1e-12)
    np.testing.assert_allclose(lb.hz_to_mel(f, htk=True), golden["const/hz_to_mel_htk"], rtol=1e-12)
    np.testing.assert_allclose(lb.mel_to_hz(np.array([0.0, 3.0, 14.9, 15.0, 25.0, 40.0])), golden["const/mel_to_hz"], rtol=1e-12)
    np.testing.assert_allclose(lb.mel_to_hz(np.array([0.0, 300.0, 1000.0, 2000.0, 3000.0]), htk=True),
                               golden["const/mel_to_hz_htk"], rtol=1e-12)
    np.testing.assert_allclose(lb.mel_frequencies(40), golden["const/mel_frequencies_40"], rtol=1e-12)
    assert np.allclose(lb.hz_to_mel(60), 0.9) and np.allclose(lb.mel_to_hz(3), 200.0)


# ------------------------------------------------------------------ argument errors raised before any GPU work
Y = np.zeros(4096, dtype=np.float32)


@pytest.mark.parametrize("call", [
    lambda: lb.stft(Y, hop_length=0),
    lambda: lb.stft(Y, hop_length=2.5),
    lambda: lb.stft(Y, pad_mode="wrap"),
    lambda: lb.stft(Y, pad_mode="mean"),
    lambda: lb.stft(Y, window=np.ones(7)),
    lambda: lb.stft(Y, win_length=4096),                       # window longer than n_fft
    lambda: lb.stft(np.zeros(100, dtype=np.float32), center=False),
    lambda: lb.stft(np.zeros(4096, dtype=np.int32)),
    lambda: lb.stft([0.0] * 4096),
    lambda: lb.stft(Y, out=np.zeros((1025, 3), dtype=np.complex64)),      # too few frames
    lambda: lb.stft(Y, out=np.zeros((1025, 9), dtype=np.float32)),        # not complex
    lambda: lb.istft(np.zeros((1025, 9), dtype=np.complex64), out=np.zeros(5, dtype=np.float32)),
    lambda: lb.feature.melspectrogram(y=None),
    lambda: lb.feature.melspectrogram(y=Y, n_fft=None),
    lambda: lb.feature.mfcc(y=Y, lifter=-1),
    lambda: lb.feature.mfcc(y=Y, lifter=np.nan),
    lambda: lb.power_to_db(np.ones((4, 4), dtype=np.float32), amin=0),
    lambda: lb.power_to_db(np.ones((4, 4), dtype=np.float32), top_db=-1),
    lambda: lb.feature.melspectrogram(y=Y, norm="bogus"),
])
def test_parameter_errors(call):
    with pytest.raises(ParameterError):
        call()


@pytest.fixture
def strict_float64(monkeypatch):
    monkeypatch.setenv("B2L_FLOAT64", "error")


@pytest.mark.parametrize("call", [
    lambda: lb.stft(np.zeros(3_000_000, dtype=np.float32), n_fft=70001),   # beyond the FP64 direct-DFT range too
    lambda: lb.stft(lb.DeviceArray(None, 0, (40000,), np.float32, owner=False), n_fft=16384),  # device f32, FP64-only size
    lambda: lb.stft(Y.astype(np.float64)),  # float64 needs an explicit opt-in to be computed in float32
    lambda: lb.stft(Y, dtype=np.complex128),
    lambda: lb.stft(Y, pad_mode=lambda *a, **k: None),
    lambda: lb.istft(np.zeros((1025, 9), dtype=np.complex128)),
])
def test_unsupported_is_loud(call, strict_float64):
    with pytest.raises(UnsupportedOnGPU):
        call()


def test_float64_policy_native_by_default(monkeypatch):
    """float64 audio takes the FP64 kernels by default (no downcast, no warning); a function that has float32
    kernels only warns once that it computes in float32; B2L_FLOAT64=downcast restores the old behaviour."""
    import warnings

    import librosa_b200._pipeline as pl

    monkeypatch.delenv("B2L_FLOAT64", raising=False)
    monkeypatch.setattr(pl, "_warned_float64", False)
    assert pl.float64_policy() == "native" and pl.native_float64(np.float64) and pl.native_float64(np.complex128)
    assert not pl.native_float64(np.float32)
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        try:
            lb.stft(Y.astype(np.float64))          # FP64 path: no warning before the device is touched
        except lb.NativeLibraryError:
            pass
    with pytest.warns(UserWarning, match="computed in float32"):
        try:
            lb.feature.spectral_centroid(y=Y.astype(np.float64))   # float32 kernels only
        except lb.NativeLibraryError:
            pass
    monkeypatch.setenv("B2L_FLOAT64", "downcast")
    monkeypatch.setattr(pl, "_warned_float64", False)
    assert not pl.native_float64(np.float64)
    with pytest.warns(UserWarning, match="computed in float32"):
        try:
            lb.stft(Y.astype(np.float64))
        except lb.NativeLibraryError:
            pass


def test_warnings_match_reference():
    with pytest.warns(UserWarning, match="is too large for input signal"):
        try:
            lb.stft(np.zeros(100, dtype=np.float32), n_fft=2048)
        except lb.NativeLibraryError:
            pass   # no GPU here: the warning is issued before the device is touched


def test_shard_ranges():
    from librosa_b200.distributed import join_batches, shard_range, split_batch

    for n in (0, 1, 7, 8, 1024, 1031):
        for world in (1, 2, 3, 8):
            cover = []
            for r in range(world):
                lo, hi = shard_range(n, r, world)
                assert 0 <= lo <= hi <= n
                cover.extend(range(lo, hi))
            assert cover == list(range(n))
    y = np.arange(7 * 3).reshape(7, 3)
    np.testing.assert_array_equal(join_batches([split_batch(y, r, 4) for r in range(4)]), y)


def test_frame_statistics_argument_errors_before_any_gpu_work():
    """Argument errors of the frame-wise features are raised on the host exactly as in the reference
    (feature/spectral.py:641, :772, :893-902; core/spectrum.py:237) — no GPU needed to see them."""
    import librosa_b200 as lb

    y = np.zeros(4000, dtype=np.float32)
    with pytest.raises(lb.ParameterError, match="roll_percent"):
        lb.feature.spectral_rolloff(y=y, roll_percent=1.0)
    with pytest.raises(lb.ParameterError, match="amin"):
        lb.feature.spectral_flatness(y=y, amin=0)
    with pytest.raises(lb.ParameterError, match="frame_length is expected"):
        lb.feature.rms(S=np.ones((100, 5), dtype=np.float32), frame_length=2048)
    with pytest.raises(lb.ParameterError, match="Either"):
        lb.feature.rms()
    with pytest.raises(lb.ParameterError, match="hop_length"):
        lb.feature.spectral_centroid(y=y, hop_length=0)
    with pytest.raises(lb.ParameterError, match="Input signal must be provided"):
        lb.feature.spectral_centroid()
    with pytest.raises(lb.ParameterError, match="too short"):
        lb.feature.rms(y=np.zeros(100, dtype=np.float32), frame_length=2048, center=False)
    with pytest.raises(TypeError):
        lb.feature.zero_crossing_rate(y, bogus=1)
    with pytest.raises(lb.ParameterError, match="floating-point"):
        lb.feature.zero_crossing_rate(np.zeros(4000, dtype=np.int16))
    with pytest.raises(lb.UnsupportedOnGPU):
        lb.feature.zero_crossing_rate(y, ref_magnitude=np.max)
    with pytest.raises(lb.UnsupportedOnGPU):
        lb.feature.rms(y=y, pad_mode="wrap")
    with pytest.raises(ValueError):
        lb.feature.rms(y=y, pad_mode="nonsense")


def test_stream_blocks_line_up_with_frames():
    """librosa.stream's block geometry (core/audio.py:407-408) over an in-memory signal: stft(center=False) of the
    blocks, concatenated, is stft(center=False) of the whole signal (checked with the oracle: no GPU here)."""
    from oracle import ref_np as O

    rng = np.random.default_rng(5)
    y = rng.standard_normal(50000).astype(np.float32)
    for block_length, frame_length, hop in ((16, 1024, 256), (7, 512, 512), (5, 400, 100)):
        blocks = list(lb.stream(y, block_length=block_length, frame_length=frame_length, hop_length=hop))
        size = (block_length - 1) * hop + frame_length
        assert all(b.shape[-1] == size for b in blocks[:-1]) and blocks[-1].shape[-1] <= size
        parts = [O.stft(b, n_fft=frame_length, hop_length=hop, center=False) for b in blocks if b.shape[-1] >= frame_length]
        whole = O.stft(y, n_fft=frame_length, hop_length=hop, center=False)
        got = np.concatenate(parts, axis=-1)
        assert got.shape == whole.shape
        np.testing.assert_array_equal(got, whole)
    st = np.stack([y, -y])
    b0 = next(lb.stream(st, block_length=4, frame_length=64, hop_length=16, mono=False))
    assert b0.shape == (2, 3 * 16 + 64)
    assert next(lb.stream(st, block_length=4, frame_length=64, hop_length=16)).shape == (3 * 16 + 64,)
    last = list(lb.stream(y[:1000], block_length=4, frame_length=256, hop_length=64, fill_value=0.0))[-1]
    assert last.shape == (3 * 64 + 256,)
    with pytest.raises(UnsupportedOnGPU):
        next(lb.stream("song.wav", block_length=4, frame_length=64, hop_length=16))
    with pytest.raises(lb.ParameterError):
        next(lb.stream(y, block_length=0, frame_length=64, hop_length=16))


def test_resample_argument_handling_without_a_gpu():
    """librosa.resample's host-side contract (core/audio.py:1115-1133): equal rates return the input itself, polyphase
    needs integer rates, and the resamplers this library does not implement are refused loudly."""
    import librosa_b200 as lb

    y = np.zeros(100, dtype=np.float32)
    assert lb.resample(y, orig_sr=22050, target_sr=22050) is y
    with pytest.raises(lb.ParameterError):
        lb.resample(y, orig_sr=22050.5, target_sr=16000, res_type="polyphase")
    for res_type in ("soxr_hq", "kaiser_best", "fft", "scipy", "linear"):
        with pytest.raises(lb.UnsupportedOnGPU):
            lb.resample(y, orig_sr=22050, target_sr=16000, res_type=res_type)
    with pytest.raises(lb.ParameterError):
        lb.resample([0.0, 1.0], orig_sr=22050, target_sr=16000, res_type="polyphase")
    with pytest.raises(lb.ParameterError):
        lb.effects.pitch_shift(y, sr=22050, n_steps=1, bins_per_octave=0, res_type="polyphase")


def test_transform_path_table():
    """Which kernels a frame length goes to (``transform_path``, host mirror of ``plan_path`` in csrc/plan.cu): powers
    of two 8 .. 8192 -> fwd_kernel, the 96 even sizes 12 .. 4050 with a 5-smooth half -> the mixed-radix kernels, any
    other size from 3 to 2047 -> chirp-z; the rest is refused by the float32 path.  The C side is held to the same
    table at every size by tests/test_gpu_forward_spectrum.py."""
    from librosa_b200 import _pipeline as pl

    smooth = [n for n in range(2, 5000) if pl.transform_path(n) == "mr"]
    assert len(smooth) == 96 and smooth[0] == 12 and smooth[-1] == 4050
    assert smooth == [n for n in range(2, 5000) if pl.mr_covers(n)]
    assert all(n % 2 == 0 and not pl.is_pow2(n) for n in smooth)
    for n in (400, 320, 480, 800, 960, 1200, 3000, 4000):
        assert pl.transform_path(n) == "mr"
    for n in (401, 1025, 14, 2 * 7 * 25):
        assert pl.transform_path(n) == "czt"
    for n in (8, 2048, 8192):
        assert pl.transform_path(n) == "pow2"
        pl.require_supported_n_fft(n)
    for n in (501, 1023, 2047):
        assert pl.transform_path(n) == "czt"
    for n in (501, 1023, 2047, 3000):
        pl.require_supported_n_fft(n)
    for n in (3001, 2049, 16384, 4102, 4098, 4, 1):
        assert pl.transform_path(n) is None
        with pytest.raises(UnsupportedOnGPU):
            pl.require_supported_n_fft(n)
    with pytest.raises(UnsupportedOnGPU, match=r"^n_fft=16384: the sm_90a kernels are built for powers of two from "
                                               r"8 to 8192 \(no CPU fallback\)$"):
        pl.require_supported_n_fft(16384)
    with pytest.raises(UnsupportedOnGPU, match=r"^n_fft=3001: non-power-of-two sizes are supported from 3 to 2047, "
                                               r"and even sizes up to 4096 whose half has no prime factor above 5 "
                                               r"\(no CPU fallback\)$"):
        pl.require_supported_n_fft(3001)


def test_kernels_launch_only_through_launch():
    """Every kernel of the C ABI is enqueued by b2l::launch (csrc/internal.h), the only code that counts launches:
    a `<<<...>>>` or a `launches++` anywhere else would make Context.launch_count miss or double-count a kernel."""
    import glob
    import re

    csrc = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "librosa_b200", "csrc")
    with open(os.path.join(csrc, "internal.h")) as f:
        header = f.read()
    body = re.search(r"\nint launch\(.*?\n\}\n", header, re.S)
    assert body and "<<<" in body.group(0) and "launches++" in body.group(0)
    sources = {"internal.h": header.replace(body.group(0), "\n")}
    for path in sorted(glob.glob(os.path.join(csrc, "*.cu"))):
        with open(path) as f:
            sources[os.path.basename(path)] = f.read()
    assert len(sources) > 5
    stray = [(name, i + 1, line.strip()) for name, text in sources.items() for i, line in enumerate(text.splitlines())
             if "<<<" in line or "launches++" in line]
    assert not stray, stray


def test_device_array_view_stays_inside_its_base():
    base = lb.DeviceArray(None, 4096, (2, 3), np.float64, owner=False)
    v = base.view((1, 3), offset=3)
    assert (v.ptr, v.shape, v.dtype, v.layout, v.base) == (4096 + 24, (1, 3), np.float64, "c", base)
    for shape, offset in (((4,), 3), ((7,), 0), ((1,), -1)):
        with pytest.raises(ValueError, match="reaches past"):
            base.view(shape, offset=offset)


def test_views_zeroed_buffers_and_status_bits_have_one_home():
    """Non-owning views and cleared buffers are made only by DeviceArray.view and Context.zeros (_native.py), and the
    status word's bits are written and read by name (enum b2l_status_bit, nat.STATUS_*), never as digits."""
    import glob
    import re

    pkg = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "librosa_b200")
    stray = []
    for path in sorted(glob.glob(os.path.join(pkg, "**", "*.py"), recursive=True)):
        with open(path) as f:
            text = f.read()
        name = os.path.relpath(path, pkg)
        if name != "_native.py":
            stray += [(name, w) for w in ("owner=False", "b2l_memset") if w in text]
        stray += [(name, m.group(0)) for m in re.finditer(r"\b_base\b|status_word\([^)]*\)\s*&\s*\d", text)]
    for path in sorted(glob.glob(os.path.join(pkg, "csrc", "*.cu*")) + glob.glob(os.path.join(pkg, "csrc", "*.h"))):
        with open(path) as f:
            text = f.read()
        pat = r"atomicOr\([^,;]*status[^,;]*,\s*\d|\*\s*[\w.>-]*status\s*=\s*\d"
        stray += [(os.path.basename(path), m.group(0)) for m in re.finditer(pat, text)]
    assert not stray, stray


def test_device_buffers_of_a_call_belong_to_its_scope():
    """The spectrum, spectral-feature, statistics, inverse, HPSS, effects, tuning and resampling calls stage, allocate
    and free through _pipeline.Scope, which frees what a call still owns on its normal and its exception path alike:
    no module stages a spectrogram or a host array, or allocates a device buffer, by hand."""
    import glob
    import re

    # the two free functions Scope.native / Scope.spectrogram replaced, spelled with a character class so that a
    # search of the repository for their names finds nothing, this test included
    retired = re.compile(r"to_[n]ative|spectrogram_[i]nput")
    pkg = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "librosa_b200")
    stray = []
    for path in sorted(glob.glob(os.path.join(pkg, "**", "*.py"), recursive=True)):
        with open(path) as f:
            text = f.read()
        stray += [(os.path.relpath(path, pkg), m.group(0)) for m in retired.finditer(text)]
    for name in ("core/spectrum.py", "core/pitch.py", "core/audio.py", "feature/spectral.py", "feature/stats.py",
                 "feature/inverse.py", "decompose.py", "effects.py"):
        with open(os.path.join(pkg, name)) as f:
            text = f.read()
        stray += [(name, w) for w in ("default_context(", ".to_device(", "DeviceArray.empty(", "in locals()")
                  if w in text]
    assert not stray, stray


def test_polyphase_filter_bookkeeping_matches_scipy():
    """The host half of resample(res_type="polyphase"): the zero-padded low-pass and the crop offset handed to
    b2l_resample_poly, checked by evaluating the kernel's formula  y[j] = sum_m x[m] h[(n_pre_remove + j) down - m up]
    in NumPy against scipy.signal.resample_poly itself (float64 accumulation here: only the bookkeeping is under test)."""
    import scipy.signal

    from librosa_b200.core.audio import _poly_filter

    rng = np.random.default_rng(2)
    for up, down, n in ((320, 441, 700), (160, 441, 1000), (441, 160, 300), (1, 2, 501), (3, 1, 50), (147, 160, 999)):
        x = rng.standard_normal(n).astype(np.float32)
        h, n_pre_remove = _poly_filter(up, down)
        n_out = (n * up + down - 1) // down
        got = np.zeros(n_out)
        for j in range(n_out):
            t = (n_pre_remove + j) * down
            m_hi = min(t // up, n - 1)
            m_lo = max(0, -(-(t - (len(h) - 1)) // up))
            m = np.arange(m_lo, m_hi + 1)
            got[j] = np.dot(x[m].astype(np.float64), h[t - m * up].astype(np.float64))
        want = scipy.signal.resample_poly(x, up, down)
        assert want.shape == (n_out,)
        np.testing.assert_allclose(got, want, rtol=1e-4, atol=2e-6 * float(np.abs(want).max()))
