"""Host (no GPU): the NumPy restatements of tests/feature_tail_restate.py, which the GPU tests of the onset, row
normalisation, tuning and polyphase-resampling kernels compare against, reproduce the reference's outputs stored in
tests/golden/features_v1.npz.  Where the fixture's input is stored (the S= onset case) the comparison is bit for bit;
where it is a signal, the spectrogram comes from the CPU oracle (oracle/ref_np.py), whose own agreement with the
reference tests/test_oracle_golden.py checks, and the comparison allows for it."""
import numpy as np
import pytest

import feature_tail_restate as R
import signals
from feature_cases import FEATURE_BY_NAME, case_args

U = 2.0 ** -24


def test_onset_from_db_spectrogram_bit_exact(golden):
    _, kw = case_args(FEATURE_BY_NAME["onset_fromS_db"], golden)
    S = kw["S"]
    env = R.onset_envelope(S[None], lag=1, max_size=1, pad_width=1 + 2048 // (2 * 512), bounds=[0, S.shape[0]])
    np.testing.assert_array_equal(env[0, 0], golden["onset_fromS_db"])


@pytest.mark.parametrize("name,channels,agg", [("onset_stereo_lag2_max3_B", None, True),
                                               ("onset_max4_nmels64_A", None, True),
                                               ("onset_multi_4bands_C", [0, 32, 64, 96, 128], True),
                                               ("onset_multi_noagg_B", None, False)])
def test_onset_from_signal(golden, oracle, name, channels, agg):
    case = FEATURE_BY_NAME[name]
    _, kw = case_args(case, golden)
    y = kw.pop("y")
    lag, max_size = kw.pop("lag", 1), kw.pop("max_size", 1)
    kw.pop("channels", None)
    kw.pop("aggregate", None)
    n_fft, hop = kw.get("n_fft", 2048), kw.get("hop_length", 512)
    kw.setdefault("fmax", 0.5 * kw["sr"])
    S = oracle.power_to_db(oracle.melspectrogram(y=y, **kw)).astype(np.float32)
    bounds = None if not agg else (channels or [0, S.shape[-2]])
    env = R.onset_envelope(S, lag=lag, max_size=max_size, pad_width=lag + n_fft // (2 * hop), bounds=bounds)
    want = golden[name]
    got = env if channels or not agg else env[..., 0, :]
    np.testing.assert_allclose(got, want, rtol=1e-3, atol=1e-3 * float(np.abs(want).max()))


@pytest.mark.parametrize("name,norm", [("chroma_norm1_C", 1), ("chroma_tuning_given_norm2_24_B", 2)])
def test_normalize_chroma(golden, oracle, name, norm):
    case = FEATURE_BY_NAME[name]
    _, kw = case_args(case, golden)
    kw.pop("norm", None)
    raw = oracle.chroma_stft(norm=None, **kw).astype(np.float32)
    got = R.normalize(raw, norm)
    np.testing.assert_allclose(got, golden[name], rtol=1e-4, atol=1e-5)


@pytest.mark.parametrize("name", ["tuning_y_T", "tuning_fromS_stereo_T", "tuning_res05_bpo24_T"])
def test_tuning_histograms(golden, oracle, name):
    import piptrack_oracle as P

    case = FEATURE_BY_NAME[name]
    _, kw = case_args(case, golden)
    resolution, bpo = kw.pop("resolution", 0.01), kw.pop("bins_per_octave", 12)
    n_fft = kw.pop("n_fft", 2048)
    if "y" in kw:
        y = kw.pop("y")
        S = np.abs(oracle.stft(y, n_fft=n_fft, hop_length=kw.pop("hop_length", None) or n_fft // 4))
    else:
        S = kw.pop("S")
    pitch, mag = P.piptrack(S=S, n_fft=n_fft, **kw)
    sel = pitch > 0
    med = np.median(mag[sel])
    k = int(R.float_keys(np.float32(med))[()])
    edges = np.linspace(-0.5, 0.5, int(np.ceil(1.0 / resolution)) + 1)
    h0, h1, h2, h3 = R.tuning_histograms(pitch, mag, prefix0=k >> 21, prefix1=k >> 10, mag_threshold=med,
                                         bins_per_octave=bpo, edges=edges)
    assert h0.sum() == sel.sum() and h1.sum() <= h0[k >> 21] and h2.sum() <= h1[(k >> 10) & 0x7FF]
    assert edges[int(np.argmax(h3))] == golden[name]


@pytest.mark.parametrize("name", ["resample_poly_22050_16000_A", "resample_poly_44100_16000_stereo_B",
                                  "resample_poly_up_8000_22050_A", "resample_poly_nofix_scale_B",
                                  "resample_poly_48000_44100_C"])
def test_resample_poly(golden, name):
    import math

    from librosa_b200.core.audio import _poly_filter

    case = FEATURE_BY_NAME[name]
    kw = case["kw"]
    y = signals.make(case["mix"], case["shape"], seed=case.get("seed", len(name)), sr=kw.get("sr", 22050))
    g = math.gcd(kw["orig_sr"], kw["target_sr"])
    up, down = kw["target_sr"] // g, kw["orig_sr"] // g
    h, n_pre_remove = _poly_filter(up, down)
    n = y.shape[-1]
    n_out = (n * up + down - 1) // down
    n_total = int(np.ceil(n * up / down)) if kw.get("fix", True) else n_out
    y64, scale = R.resample_poly64(y, h, up, down, n_pre_remove, min(n_out, n_total), n_total)
    if kw.get("scale"):
        y64, scale = y64 / np.sqrt(up / down), scale / np.sqrt(up / down)
    # the reference runs upfirdn in float32: its own error is within the bound of the kernel's
    k = -(-len(h) // up) + 1
    err = np.abs(golden[name] - y64)
    assert (err <= 2 * (k + 1) * U * scale + 2 * U * np.abs(y64)).all(), float(err.max())
