"""CPU: iirt's host side against tests/golden/iirt_v1.npz without a GPU — the oracle reproduces every stored
result bit for bit, the filter bank equals the reference's, the kernels' tables (coefficients, initial states,
padding lengths, frame starts, the pairwise-sum program) are what SciPy and NumPy compute, and every error and
refusal comes with the reference's message, in its order, before any device work."""
from __future__ import annotations

import os
import warnings

import numpy as np
import pytest
import scipy.signal

import iirt_cases as IC
import iirt_oracle as IO
import librosa_b200 as lb
from librosa_b200 import filters
from librosa_b200.core import semitone as S

GOLDEN = np.load(os.path.join(os.path.dirname(__file__), "golden", "iirt_v1.npz"))
RUNS = [c for c in IC.CASES if f"{c['name']}/S" in GOLDEN.files and not c["refuse"]]
# plain non-finite audio gets the device's verdict (tests/test_gpu_iirt.py); every other error comes from the host
ERRORS = [c for c in IC.CASES if f"{c['name']}/error" in GOLDEN.files and c["name"] != "not_finite"]


def _plan(case):
    kw, extra = IO.resolved(case)
    y = IC.signal(case["sig"])
    return S.plan(y.shape, sr=kw["sr"], win_length=kw["win_length"], hop_length=kw["hop_length"],
                  center=kw["center"], tuning=kw["tuning"], pad_mode=kw["pad_mode"], res_type=kw["res_type"],
                  kwargs=extra)


@pytest.mark.parametrize("case", RUNS, ids=lambda c: c["name"])
def test_oracle_reproduces_fixture(case):
    name = case["name"]
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        got, bands = IO.iirt(case)
    ref = GOLDEN[f"{name}/S"]
    assert got.dtype == ref.dtype and got.shape == ref.shape and np.array_equal(got, ref)
    if name in IC.WITH_STEPS:
        b = IC.WITH_STEPS[name]
        assert np.array_equal(bands[b], GOLDEN[f"{name}/band{b}"])
        ys = IO.resampled(case, IC.signal(case["sig"]))
        assert ys and all(np.array_equal(v, GOLDEN[f"{name}/y{r:g}"]) for r, v in ys.items())


@pytest.mark.parametrize("cfg", sorted(IC.BANKS))
def test_filter_bank_equals_reference(cfg):
    sos, srs = filters.semitone_filterbank(flayout="sos", **IC.BANKS[cfg])
    assert np.array_equal(np.concatenate(sos), GOLDEN[f"bank/{cfg}/sos"])
    assert [len(s) for s in sos] == list(GOLDEN[f"bank/{cfg}/sections"])
    assert np.array_equal(srs, GOLDEN[f"bank/{cfg}/rates"])


def test_transfer_functions_and_frequencies_equal_reference():
    ba, _ = filters.semitone_filterbank()   # the reference's default layout is "ba"
    assert np.array_equal(np.stack([b for b, _ in ba]), GOLDEN["bank/defaults/b"])
    assert np.array_equal(np.stack([a for _, a in ba]), GOLDEN["bank/defaults/a"])
    assert np.array_equal(np.stack(filters.mr_frequencies(0.3)), GOLDEN["mr_frequencies/0.3"])


@pytest.mark.parametrize("cfg", sorted(IC.BANKS))
def test_kernel_tables(cfg):
    """Coefficients, sosfilt_zi, sections and padlen per band, and the bands grouped by rate in np.unique order."""
    _, bank = S.bank_cached(IC.BANKS[cfg].get("tuning", 0.0), {k: v for k, v in IC.BANKS[cfg].items() if k != "tuning"})
    sos, srs = filters.semitone_filterbank(flayout="sos", **IC.BANKS[cfg])
    assert np.array_equal(bank.rates, np.unique(srs))
    for i, s in enumerate(sos):
        ns = len(s)
        assert bank.info[i, 0] == ns
        # sosfiltfilt's default padlen, as its own error message states it
        with pytest.raises(ValueError, match=f"which is {bank.info[i, 1]}\\."):
            scipy.signal.sosfiltfilt(s, np.zeros(int(bank.info[i, 1])))
        assert np.array_equal(bank.coef[i, :ns, 0:3], s[:, 0:3]) and np.array_equal(bank.coef[i, :ns, 3:5], s[:, 4:6])
        assert np.array_equal(bank.coef[i, :ns, 5:7], scipy.signal.sosfilt_zi(s))
        assert np.all(bank.coef[i, ns:, 0] == 1.0) and not bank.coef[i, ns:, 1:].any() and np.all(s[:, 3] == 1.0)
        assert srs[bank.bands[bank.band_off[bank.rate_of[i]]:bank.band_off[bank.rate_of[i] + 1]]].tolist() == \
            [srs[i]] * int(np.sum(srs == srs[i]))


def test_bank_is_memoised():
    k1, b1 = S.bank_cached(0.0, {})
    k2, b2 = S.bank_cached(0.0, {})
    assert k1 == k2 and b1 is b2
    k3, _ = S.bank_cached(0.0, {"Q": 15})
    assert k3 != k1


@pytest.mark.parametrize("case", RUNS, ids=lambda c: c["name"])
def test_frame_tables(case):
    """Each rate's length, window, factor and starts equal the oracle's; the fix_length case reads past n."""
    kw, _ = IO.resolved(case)
    p = _plan(case)
    assert p.n_frames == GOLDEN[f"{case['name']}/S"].shape[-1]
    fixed = False
    for r in p.rates:
        factor, w, starts, n_fix = IO.frame_starts(r.n, sr=kw["sr"], rate=r.rate, win_length=kw["win_length"],
                                                   hop_length=kw["hop_length"], n_frames=p.n_frames)
        assert (r.factor, r.w) == (factor, w) and np.array_equal(r.starts, starts) and r.starts.dtype == np.int32
        fixed |= n_fix > r.n
        if p.n_frames:
            assert r.starts[-1] + r.w <= max(r.n, n_fix)
    assert fixed == (case["name"] == "fix_length")


@pytest.mark.parametrize("w", [0, 1, 7, 8, 9, 82, 127, 128, 129, 136, 410, 1000, 2048, 4097, 8192, 20000])
def test_leaf_program_is_numpys_pairwise_sum(w):
    """The STMSP kernel's summation order equals np.sum over the window axis, as iirt sums, bit for bit."""
    rng = np.random.default_rng(w)
    leaves = S.pairwise_leaves(w)
    assert S.leaves_depth(leaves) <= lb._native.IIRT_MAX_DEPTH
    assert leaves[:, 1].sum() == w and np.all(leaves[:, 1] <= 128)
    x = (rng.standard_normal((6, w + 3)) * rng.uniform(1e-6, 10, (6, 1))) ** 2
    ref = np.sum(x[:, None, 3:3 + w], axis=-1)[:, 0]
    for k in range(6):
        assert IO.leaf_program_sum(x[k, 3:], leaves) == ref[k]


def test_scratch_budget_and_groups():
    """41 MB of float64 scratch per 10 s clip at the defaults; clips are grouped to fit the pool."""
    p = S.plan((1024, 220500), sr=22050, win_length=2048, hop_length=None, center=True, tuning=0.0,
               pad_mode="constant", res_type="polyphase", kwargs={})
    assert [r.n for r in p.rates] == [8902, 44510, 222548]
    assert [r.rows for r in p.rates] == [8902 + 27, 44510 + 27, 222548 + 27]
    per_clip = p.clip_bytes()
    assert 40e6 < per_clip < 42e6 and p.scratch_bytes(32) == 32 * per_clip
    g = S.group_size(p, 1024, 16384 << 20)
    assert g == (16384 << 20) // per_clip and p.scratch_bytes(g) <= (16384 << 20) + 3 * 32 * 8 * 222575
    assert S.group_size(p, 1024, 1) == 1 and S.group_size(p, 3, 1 << 40) == 3


@pytest.mark.parametrize("case", ERRORS, ids=lambda c: c["name"])
def test_errors_match_reference(case):
    """Raised on the host before any device work; non-finite audio that also fails a later check gets the
    reference's error, util.valid_audio's, first."""
    with pytest.raises(Exception) as e:
        IC.call(lb, case)
    assert f"{type(e.value).__name__}: {e.value}" == str(GOLDEN[f"{case['name']}/error"])


@pytest.mark.parametrize("name,match", [("refuse_default_res_type", "pass res_type='polyphase'"),
                                        ("refuse_ba", "pass flayout='sos'"),
                                        ("refuse_callable_pad", "callable pad_mode"),
                                        ("refuse_pad_wrap", "pads with")])
def test_refusals(name, match):
    with pytest.raises(lb.UnsupportedOnGPU, match=match):
        IC.call(lb, IC.BY_NAME[name])


def test_refusal_of_deep_filters():
    """A design with more sections than the kernel is built for is refused; butter at the default Q (10) is not."""
    sos, _ = filters.semitone_filterbank(flayout="sos", ftype="butter", stopband_attenuation=80)
    assert max(len(s) for s in sos) > lb._native.IIRT_MAX_SECTIONS
    y = IC.signal(IC.BY_NAME["defaults"]["sig"])
    with pytest.raises(lb.UnsupportedOnGPU, match="second-order sections"):
        lb.iirt(y, sr=22050, res_type="polyphase", ftype="butter", stopband_attenuation=80)


def test_resampler_rule():
    """A call whose rates all equal sr accepts any res_type; one that resamples refuses non-polyphase resamplers,
    at the first rate that needs it."""
    p = _plan(IC.BY_NAME["sr_only_no_resample"])
    assert [r.up for r in p.rates] == [0]
    with pytest.raises(lb.UnsupportedOnGPU, match="soxr_vhq"):
        lb.iirt(IC.signal(IC.BY_NAME["defaults"]["sig"]), sr=22050, res_type="soxr_vhq")


def test_empty_signal_padding():
    with pytest.raises(ValueError, match="can't extend empty axis 1"):
        lb.iirt(np.zeros((2, 0), np.float32), sr=22050, res_type="polyphase", pad_mode="edge")


def test_public_names():
    assert lb.iirt is lb.core.iirt is S.iirt
    assert filters.semitone_filterbank and filters.mr_frequencies
