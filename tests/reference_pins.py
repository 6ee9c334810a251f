"""Inputs and reference-side calls pinned by tests/test_oracle_vs_reference.py.

tools/make_golden.py stores ``pack(reference_outputs(ref))`` as tests/golden/reference_pins_v1.npz.  The
comparisons are exact, so larger outputs are stored as SHA-256 digests of dtype, shape and bytes.
"""
import hashlib
import warnings

import numpy as np

STFT_GRID = [
    (22050, 2048, 512, True, "constant"), (5000, 1024, 256, True, "reflect"), (4000, 512, None, False, "constant"),
    (1000, 2048, 512, True, "constant"), (3000, 501, 128, True, "edge"), (7000, 1025, 300, True, "symmetric"),
    (6000, 256, 64, True, "linear_ramp"), (900, 64, 7, True, "reflect"),
]
CHROMA_KW = [dict(sr=22050, n_fft=2048), dict(sr=16000, n_fft=1024, tuning=0.27), dict(sr=22050, n_fft=400, n_chroma=24, octwidth=None),
             dict(sr=44100, n_fft=4096, norm=None, base_c=False, ctroct=4.0, octwidth=1.5), dict(sr=22050, n_fft=1025, tuning=-0.3)]
OCTS_F = np.array([27.5, 55.0, 440.0, 1234.5])
MEL_KW = [dict(sr=22050, n_fft=2048), dict(sr=44100, n_fft=4096), dict(sr=16000, n_fft=1024, n_mels=40, htk=True),
          dict(sr=22050, n_fft=2048, norm=1), dict(sr=22050, n_fft=2048, norm=None, fmin=300, fmax=8000),
          dict(sr=22050, n_fft=2048, norm=np.inf), dict(sr=8000, n_fft=512, n_mels=20, dtype=np.float64)]
WINDOWS = ["hann", "hamming", ("kaiser", 4.0), np.ones(64)]
HZ = np.array([0.0, 60.0, 999.0, 1000.0, 5000.0])
GL_KW = [dict(n_iter=4, rng=0), dict(n_iter=3, init=None, momentum=0.5), dict(n_iter=2, rng=7, length=6000)]
DB_KW = [dict(), dict(axes=(-1,)), dict(axes=(-2,)), dict(axes=None, ref=np.max), dict(axes=(0, -1), top_db=30.0),
         dict(axes=(-1,), ref=np.max)]
F64_STFT_KW = [dict(n_fft=1024, hop_length=256), dict(n_fft=1000, hop_length=250, pad_mode="reflect")]
MFCC_TO_MEL_KW = [dict(), dict(lifter=3, dct_type=3), dict(n_mels=64, norm=None), dict(ref=2.5, lifter=22)]


INPUT_KEYS = ("inverse/M_float32", "inverse/M_float64")
WHOLE_UP_TO = 64   # elements; larger outputs are stored as digests


def digest(a):
    a = np.ascontiguousarray(a)
    h = hashlib.sha256(f"{a.dtype.str}{a.shape}".encode())
    h.update(a.tobytes())
    return h.hexdigest()


def pack(outputs):
    return {k: (np.asarray(v) if k in INPUT_KEYS or np.size(v) <= WHOLE_UP_TO else np.array(digest(v)))
            for k, v in outputs.items()}


def assert_pinned(pins, key, got):
    want = pins[key]
    if want.dtype.kind == "U":
        got = np.asarray(got)
        assert digest(got) == str(want), f"{key}: {got.dtype}{got.shape} differs from the reference output"
    else:
        np.testing.assert_array_equal(want, got, err_msg=key)


def stft_key(n, n_fft, hop, center, pad_mode):
    return f"stft/{n}_{n_fft}_{hop}_{center}_{pad_mode}"


def stft_input(n):
    return (0.1 * np.random.default_rng(n).standard_normal(n)).astype(np.float32)


def features_input():
    return (0.1 * np.random.default_rng(5).standard_normal((2, 3, 8000))).astype(np.float32)


def frame_input():
    return np.arange(40.0).reshape(2, 20)


def griffinlim_input():
    return (0.1 * np.random.default_rng(2).standard_normal(6000)).astype(np.float32)


def db_inputs():
    """(P, y): the power spectrogram of the power_to_db checks and the float64 audio, from one generator."""
    rng = np.random.default_rng(9)
    P = np.abs(rng.standard_normal((2, 3, 40, 30))) ** 2
    y = 0.1 * rng.standard_normal((2, 9000))
    return P, y


def inverse_inputs():
    """(S32, S64, mf): the magnitude spectra of mel_to_stft (float32, float64) and the MFCCs of mfcc_to_mel."""
    rng = np.random.default_rng(21)
    S = [np.abs(rng.standard_normal((513, 6))).astype(dtype) ** 2 for dtype in (np.float32, np.float64)]
    mf = rng.standard_normal((2, 13, 20)).astype(np.float32) * 10
    return S[0], S[1], mf


def reference_outputs(ref):
    out = {}
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        for n, n_fft, hop, center, pad_mode in STFT_GRID:
            key = stft_key(n, n_fft, hop, center, pad_mode)
            D = ref.stft(stft_input(n), n_fft=n_fft, hop_length=hop, center=center, pad_mode=pad_mode)
            out[key] = D
            for length in (None, n):
                out[f"{key}/istft_{length}"] = ref.istft(D, hop_length=hop, n_fft=n_fft, center=center, length=length)
    y = features_input()
    out["features/mel"] = ref.feature.melspectrogram(y=y, sr=16000, n_fft=1024, hop_length=256)
    out["features/mfcc40"] = ref.feature.mfcc(y=y, sr=16000, n_mfcc=40, n_fft=1024, hop_length=256)
    out["features/mfcc13_lifter_dct3"] = ref.feature.mfcc(y=y, sr=16000, n_mfcc=13, lifter=22, dct_type=3)
    for i, kw in enumerate(CHROMA_KW):
        out[f"chroma/{i}"] = ref.filters.chroma(**kw)
    out["hz_to_octs"] = ref.hz_to_octs(OCTS_F, tuning=0.2, bins_per_octave=24)
    S = np.abs(ref.stft(griffinlim_input(), n_fft=512, hop_length=128))
    out["griffinlim/S"] = S
    for i, kw in enumerate(GL_KW):
        out[f"griffinlim/{i}"] = ref.griffinlim(S, hop_length=128, **kw)
    for i, kw in enumerate(MEL_KW):
        out[f"mel/{i}"] = ref.filters.mel(**kw)
    out["window_sumsquare_hann_50"] = ref.filters.window_sumsquare(window="hann", n_frames=50)
    for i, w in enumerate(WINDOWS):
        out[f"get_window/{i}"] = ref.filters.get_window(w, 64)
    for htk in (False, True):
        out[f"hz_to_mel/{htk}"] = ref.hz_to_mel(HZ, htk=htk)
        out[f"mel_to_hz/{htk}"] = ref.mel_to_hz(HZ / 50, htk=htk)
    out["hz_to_mel_60"] = np.float64(ref.hz_to_mel(60.0))
    out["mel_to_hz_20"] = np.float64(ref.mel_to_hz(20.0))
    x = frame_input()
    for axis in (-1, 0, 1):
        if x.shape[axis] >= 5:
            out[f"frame/{axis}"] = ref.util.frame(x, frame_length=5, hop_length=2, axis=axis)
    out["pad_center"] = ref.util.pad_center(np.ones(5), size=12)
    out["fix_length"] = ref.util.fix_length(np.ones(5), size=3)
    out["tiny_float32"] = np.asarray(ref.util.tiny(np.float32(1)))
    P, y64 = db_inputs()
    for i, kw in enumerate(DB_KW):
        out[f"power_to_db/{i}"] = ref.power_to_db(P, **kw)
    for i, kw in enumerate(F64_STFT_KW):
        D = ref.stft(y64, **kw)
        out[f"f64/stft/{i}"] = D
        out[f"f64/istft/{i}"] = ref.istft(D, hop_length=kw["hop_length"], n_fft=kw["n_fft"])
    out["f64/mel"] = ref.feature.melspectrogram(y=y64, sr=16000, n_fft=1024)
    out["f64/mfcc"] = ref.feature.mfcc(y=y64, sr=16000, n_fft=1024)
    S32, S64, mf = inverse_inputs()
    for name, S_, dtype in (("float32", S32, np.float32), ("float64", S64, np.float64)):
        M = ref.filters.mel(sr=22050, n_fft=1024, n_mels=64, dtype=dtype).dot(S_)
        out[f"inverse/M_{name}"] = M
        out[f"inverse/mel_to_stft_{name}"] = ref.feature.inverse.mel_to_stft(M, n_fft=1024, power=2.0)
    for i, kw in enumerate(MFCC_TO_MEL_KW):
        out[f"inverse/mfcc_to_mel/{i}"] = ref.feature.inverse.mfcc_to_mel(mf, **kw)
    return out
