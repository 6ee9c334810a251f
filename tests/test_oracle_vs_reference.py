"""CPU: the oracle and the product's host-side constants against the unmodified reference's outputs, stored
by tools/make_golden.py (tests/reference_pins.py).  Every comparison is exact."""
import os
import warnings

import numpy as np
import pytest

import reference_pins as RP

PINS_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_pins_v1.npz")


@pytest.fixture(scope="module")
def ref():
    with np.load(PINS_PATH) as z:
        return {k: z[k] for k in z.files}


@pytest.mark.parametrize("n,n_fft,hop,center,pad_mode", RP.STFT_GRID)
def test_stft_istft_bit_exact(ref, oracle, n, n_fft, hop, center, pad_mode):
    y = RP.stft_input(n)
    key = RP.stft_key(n, n_fft, hop, center, pad_mode)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        D = oracle.stft(y, n_fft=n_fft, hop_length=hop, center=center, pad_mode=pad_mode)
        RP.assert_pinned(ref, key, D)
        for length in (None, n):
            b = oracle.istft(D, hop_length=hop, n_fft=n_fft, center=center, length=length)
            RP.assert_pinned(ref, f"{key}/istft_{length}", b)


def test_features_bit_exact(ref, oracle):
    y = RP.features_input()
    RP.assert_pinned(ref, "features/mel", oracle.melspectrogram(y=y, sr=16000, n_fft=1024, hop_length=256))
    RP.assert_pinned(ref, "features/mfcc40", oracle.mfcc(y=y, sr=16000, n_mfcc=40, n_fft=1024, hop_length=256))
    RP.assert_pinned(ref, "features/mfcc13_lifter_dct3", oracle.mfcc(y=y, sr=16000, n_mfcc=13, lifter=22, dct_type=3))


def test_frame_statistics_bit_exact(oracle, golden):
    # tests/golden/features_v1.npz holds the reference's outputs of the same cases on the same inputs
    from feature_cases import FEATURE_CASES, call, fixture_names, outputs

    for case in FEATURE_CASES:
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            B = outputs(call(oracle, case, golden))
        for key, b in zip(fixture_names(case, len(B)), B):
            a = golden[key]
            assert a.dtype == b.dtype and a.shape == b.shape, case["name"]
            np.testing.assert_array_equal(a, b, err_msg=case["name"])


def test_product_chroma_filter_matches_reference(ref):
    import librosa_b200 as lb

    for i, kw in enumerate(RP.CHROMA_KW):
        RP.assert_pinned(ref, f"chroma/{i}", lb.filters.chroma(**kw))
    RP.assert_pinned(ref, "hz_to_octs", lb.hz_to_octs(RP.OCTS_F, tuning=0.2, bins_per_octave=24))


def test_griffinlim_bit_exact(ref, oracle):
    S = np.abs(oracle.stft(RP.griffinlim_input(), n_fft=512, hop_length=128))
    RP.assert_pinned(ref, "griffinlim/S", S)
    for i, kw in enumerate(RP.GL_KW):
        RP.assert_pinned(ref, f"griffinlim/{i}", oracle.griffinlim(S, hop_length=128, **kw))


def test_product_host_constants_match_reference(ref):
    """The product's own host-side constant builders (librosa_b200.filters / convert / util) against the
    reference — these feed the GPU plans, so they are pinned as tightly as the oracle."""
    import librosa_b200 as lb

    for i, kw in enumerate(RP.MEL_KW):
        RP.assert_pinned(ref, f"mel/{i}", lb.filters.mel(**kw))
    RP.assert_pinned(ref, "window_sumsquare_hann_50", lb.filters.window_sumsquare(window="hann", n_frames=50))
    for i, w in enumerate(RP.WINDOWS):
        RP.assert_pinned(ref, f"get_window/{i}", lb.filters.get_window(w, 64))
    for htk in (False, True):
        RP.assert_pinned(ref, f"hz_to_mel/{htk}", lb.hz_to_mel(RP.HZ, htk=htk))
        RP.assert_pinned(ref, f"mel_to_hz/{htk}", lb.mel_to_hz(RP.HZ / 50, htk=htk))
    assert ref["hz_to_mel_60"] == lb.hz_to_mel(60.0) and ref["mel_to_hz_20"] == lb.mel_to_hz(20.0)
    x = RP.frame_input()
    for axis in (-1, 0, 1):
        if x.shape[axis] >= 5:
            RP.assert_pinned(ref, f"frame/{axis}", lb.util.frame(x, frame_length=5, hop_length=2, axis=axis))
    RP.assert_pinned(ref, "pad_center", lb.util.pad_center(np.ones(5), size=12))
    RP.assert_pinned(ref, "fix_length", lb.util.fix_length(np.ones(5), size=3))
    assert ref["tiny_float32"] == lb.util.tiny(np.float32(1))


def test_power_to_db_axes_and_float64_bit_exact(ref, oracle):
    """power_to_db with explicit reduction axes, and the float64 behaviour of the whole path (the reference
    computes float64 audio in float64: complex128 STFT, float64 mel / MFCC)."""
    P, y = RP.db_inputs()
    for i, kw in enumerate(RP.DB_KW):
        RP.assert_pinned(ref, f"power_to_db/{i}", oracle.power_to_db(P, **kw))
    for i, kw in enumerate(RP.F64_STFT_KW):
        b = oracle.stft(y, **kw)
        assert b.dtype == np.complex128
        RP.assert_pinned(ref, f"f64/stft/{i}", b)
        RP.assert_pinned(ref, f"f64/istft/{i}", oracle.istft(b, hop_length=kw["hop_length"], n_fft=kw["n_fft"]))
    m_or = oracle.melspectrogram(y=y, sr=16000, n_fft=1024)
    assert m_or.dtype == np.float64
    RP.assert_pinned(ref, "f64/mel", m_or)
    RP.assert_pinned(ref, "f64/mfcc", oracle.mfcc(y=y, sr=16000, n_fft=1024))


def test_feature_inverse_bit_exact(ref, oracle):
    """mel_to_stft (NNLS through SciPy's L-BFGS-B) and mfcc_to_mel restated in the oracle."""
    _, _, mf = RP.inverse_inputs()
    for name in ("float32", "float64"):
        RP.assert_pinned(ref, f"inverse/mel_to_stft_{name}", oracle.mel_to_stft(ref[f"inverse/M_{name}"], n_fft=1024, power=2.0))
    for i, kw in enumerate(RP.MFCC_TO_MEL_KW):
        RP.assert_pinned(ref, f"inverse/mfcc_to_mel/{i}", oracle.mfcc_to_mel(mf, **kw))
