"""HMM decoding without a GPU: the ``transition_*`` builders bit for bit against the reference's fixture
(tests/golden/sequence_v1.npz), every error case of tests/sequence_cases.py with the reference's class, message and
order, the refusals raised from shapes and dtypes, and the list of cases fragile under a 1-ulp log difference."""
import os
import warnings

import numpy as np
import pytest

import sequence_cases as SC
import sequence_oracle as SO
import librosa_b200 as lb

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def golden():
    with np.load(os.path.join(ROOT, "tests", "golden", "sequence_v1.npz")) as z:
        return {k: z[k] for k in z.files}


@pytest.mark.parametrize("key", list(SC.BUILDERS))
def test_builders_bit_exact(golden, key):
    got = SC.builder(lb, SC.BUILDERS[key])
    want = golden["builder/" + key]
    assert got.dtype == want.dtype and got.shape == want.shape and got.tobytes() == want.tobytes(), key


@pytest.mark.parametrize("key", list(SC.BUILDER_ERRORS))
def test_builder_errors(golden, key):
    with pytest.raises(lb.ParameterError) as exc:
        SC.builder(lb, SC.BUILDER_ERRORS[key])
    assert f"ParameterError: {exc.value}" == str(golden["builder/" + key + "/error"])


@pytest.mark.parametrize("name", [c["name"] for c in SC.CASES])
def test_errors_before_device_work(golden, name):
    """Every error of a host call is raised on the host, with the reference's class and message."""
    if name + "/error" not in golden:
        pytest.skip("not an error case")
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        got = SC.call(lb, SC.BY_NAME[name])
    assert got.get("error") == str(golden[name + "/error"]), got


def test_zero_steps_2d():
    case = SC.BY_NAME["viterbi/zero_steps"]
    prob, transition, _ = SC.make(case)
    out = lb.sequence.viterbi(prob, transition)
    assert out.shape == (0,) and out.dtype == np.uint16
    with pytest.raises(lb.UnsupportedOnGPU, match="zero frames"):
        lb.sequence.viterbi(prob, transition, return_logp=True)


def test_refusals_from_shapes():
    n = lb.sequence.MAX_STATES + 1
    with pytest.raises(lb.UnsupportedOnGPU, match=f"{n} states"):
        lb.sequence.viterbi(np.zeros((n, 1), np.float32), np.eye(n))
    with pytest.raises(lb.UnsupportedOnGPU, match=f"{n} states"):
        lb.sequence.viterbi_discriminative(np.zeros((n, 1), np.float32), np.eye(n))
    with pytest.raises(lb.UnsupportedOnGPU, match="float32 and float64 only"):
        lb.sequence.viterbi(np.zeros((3, 4), np.int32), np.eye(3))
    with pytest.raises(lb.UnsupportedOnGPU, match="float32 and float64 only"):
        lb.sequence.viterbi_binary(np.zeros((3, 4), np.float16), np.eye(2))


def test_fragile_cases_listed(golden):
    """The oracle reproduces every fixture entry bit for bit, and the cases below the 1-ulp bound are the listed ones."""
    fragile = []
    for case in SC.CASES:
        name = case["name"]
        if name + "/lp_sha256" not in golden:
            continue
        prob, transition, kw = SC.make(case)
        kw.pop("return_logp", None)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            r = SO.run(case["op"], prob, transition, **kw)
        assert SO.digest(r["lp"]) == str(golden[name + "/lp_sha256"]), name
        assert r["states"].tobytes() == golden[name + "/states"].tobytes(), name
        if name + "/logp" in golden:
            assert r["logp"].shape == golden[name + "/logp"].shape, name
            assert np.array_equal(r["logp"], golden[name + "/logp"], equal_nan=True), name
        if r["gap"] < SO.fragile_bound(prob.shape[-1], r["max_abs_lp"], prob.dtype):
            fragile.append(name)
    assert fragile == SC.FRAGILE
