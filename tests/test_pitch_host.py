"""yin / pyin without a GPU: the oracle against the reference's outputs (tests/golden/pitch_v1.npz, bit for bit),
the argument errors and warnings of the public functions, and the exactness of the Viterbi's compact
log-transition table."""
import os
import warnings

import numpy as np
import pytest

import librosa_b200 as lb
import pitch_cases as PC
import pitch_oracle as PO
from librosa_b200.core import pitch as P

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def pitch_golden():
    with np.load(os.path.join(ROOT, "tests", "golden", "pitch_v1.npz")) as z:
        return {k: z[k] for k in z.files}


@pytest.mark.parametrize("name", [c["name"] for c in PC.PITCH_CASES])
def test_oracle_bit_exact(pitch_golden, name):
    case = PC.BY_NAME[name]
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        got = PC.outputs(case, PC.run(PO, case))
    for key, arr in got.items():
        ref = pitch_golden[key]
        assert arr.dtype == ref.dtype and arr.shape == ref.shape, key
        assert arr.tobytes() == ref.tobytes(), key


_YIN_FAIL = [(None, None, 2048), (110, None, 2048), (None, 880, 2048), (-1, 440, 2048), (440, 220, 2048),
             (440, 16000, 2048), (10, 21, 2048)]


@pytest.mark.parametrize("fmin,fmax,frame_length", _YIN_FAIL)
def test_yin_fail(fmin, fmax, frame_length):
    y = PC.tone(110).astype(np.float64)
    with pytest.raises(lb.ParameterError) as got:
        lb.yin(y, fmin=fmin, fmax=fmax, frame_length=frame_length)
    with pytest.raises(PO.ParameterError) as want:
        PO.yin(y, fmin=fmin, fmax=fmax, frame_length=frame_length)
    assert str(got.value) == str(want.value)


@pytest.mark.parametrize("fmin,fmax,frame_length", [(None, None, 2048), (110, None, 2048), (None, 880, 2048)])
def test_pyin_fail(fmin, fmax, frame_length):
    y = PC.tone(110)
    with pytest.raises(lb.ParameterError):
        lb.pyin(y, fmin=fmin, fmax=fmax, frame_length=frame_length)


def test_yin_warn():
    with pytest.warns(UserWarning, match="two periods"):
        P._check_yin_params(sr=22050, fmax=1000, fmin=20, frame_length=2048)


@pytest.mark.parametrize("fn", [lb.yin, lb.pyin])
def test_host_errors(fn):
    y = PC.tone(220)
    with pytest.raises(lb.ParameterError, match="Input is too short"):
        fn(y[:1000], fmin=110, fmax=880, center=False)
    with pytest.raises(lb.UnsupportedOnGPU):
        fn(y, fmin=110, fmax=880, pad_mode=lambda *a, **k: None)
    with pytest.raises(lb.ParameterError, match="floating-point"):
        fn(np.arange(5000), fmin=110, fmax=880)


def test_pyin_viterbi_errors():
    y = PC.tone(220)
    with pytest.raises(lb.ParameterError, match="Invalid transition_min_prob"):
        lb.pyin(y, fmin=110, fmax=880, transition_min_prob=-1.0)
    with pytest.raises(lb.ParameterError, match="Empty transition matrix"):
        lb.pyin(y, fmin=110, fmax=880, transition_min_prob=0.9)


@pytest.mark.parametrize("npb,nbps,tmp,hop,sw", [(601, 10, 1e-4, 512, 0.01), (383, 10, None, 512, 0.01),
                                                  (121, 5, 1e-4, 512, 0.01), (383, 10, 1e-4, 256, 0.2),
                                                  (12, 10, 1e-4, 64, 0.01)])
def test_viterbi_table_exact(npb, nbps, tmp, hop, sw):
    """The kernel's predecessor walk over the class table gives the reference's predecessor sets and values."""
    width = round(35.92 * 12 * hop / 22050) * nbps + 1
    vt = P._viterbi_tables(npb, width, sw, tmp)
    eps = np.finfo(np.float64).tiny
    log_trans = np.log(PO.pyin_transition(npb, nbps, sr=22050, hop_length=hop, switch_prob=sw) + eps)
    thr = PO.log_threshold(tmp, eps)
    preds = PO.predecessors(log_trans, thr)
    hw, S = vt["half_width"], 2 * npb
    for j in range(S):
        q, b = j % npb, int(j >= npb)
        ks, vs = [], []
        for h in range(2):
            ps = range(npb) if vt["full"] else range(max(0, q - hw), min(npb - 1, q + hw) + 1)
            for p in ps:
                d = q - p
                v = vt["ltab"][vt["cls"][p], int(h != b), d + hw] if abs(d) <= hw else np.log(eps)
                if vt["full"] or v >= vt["log_thr"]:
                    ks.append(h * npb + p)
                    vs.append(v)
        assert np.array_equal(ks, preds[j])
        assert np.array_equal(np.array(vs).view(np.int64), log_trans[preds[j], j].view(np.int64))
