"""CPU checks of the GRU / LSTM test infrastructure (no GPU): the numpy restatement oracle/rnn.py against the
reference's PyTorch-generated cases, rten-vecmath's Sigmoid in the C oracle, and the ONNX reader's STRINGS attributes
(the `activations` attribute of an RNN node)."""
import json
import os

import numpy as np
import pytest

import onnx_writer as W
from oracle import oracle
from oracle import rnn as orn

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "rnn_cases.json")
CASES = ["lstm_forwards", "lstm_initial", "lstm_bidirectional", "gru_forwards", "gru_initial", "gru_bidirectional"]


@pytest.fixture(scope="module")
def golden():
    oracle.build()
    with open(GOLDEN) as f:
        return json.load(f)


@pytest.mark.parametrize("name", CASES)
def test_f32_oracle_reproduces_pytorch_cases(golden, name):
    # = test_rnn_pytorch (src/ops/rnn.rs): Y within expect_equal's 1e-8 + 1e-5 |b|
    op, direction, ins, exp = orn.golden_case(golden[name], name)
    y = (orn.gru if op == "gru" else orn.lstm)(direction=direction, mode="f32", **ins)[0]
    assert y.dtype == np.float32 and y.shape == exp.shape
    assert oracle.expect_equal(y, exp), float(np.max(np.abs(y - exp)))


def test_f64_oracle_is_closer_than_tolerance(golden):
    for name in CASES:
        op, direction, ins, exp = orn.golden_case(golden[name], name)
        y = (orn.gru if op == "gru" else orn.lstm)(direction=direction, mode="f64", **ins)[0]
        assert np.max(np.abs(y - exp)) < 1e-5


def test_reverse_runs_backwards_and_final_state():
    r = oracle.XorShiftRng(7)
    x, w, rr = r.uniform((6, 2, 3)), r.uniform((1, 12, 3)), r.uniform((1, 12, 3))
    yf, hf, _ = orn.lstm(x, w, rr, direction="forward")
    yr, hr, _ = orn.lstm(x[::-1].copy(), w, rr, direction="reverse")
    np.testing.assert_array_equal(yr[::-1], yf)
    np.testing.assert_array_equal(hr, hf)
    yb, hb = orn.gru(x, r.uniform((2, 9, 3)), r.uniform((2, 9, 3)), direction="bidirectional")
    np.testing.assert_array_equal(hb[0], yb[-1, 0])
    np.testing.assert_array_equal(hb[1], yb[0, 1])


def _ulp_distance(a, b):
    a = a.astype(np.float32).view(np.int32).astype(np.int64)
    b = b.astype(np.float32).view(np.int32).astype(np.int64)
    a = np.where(a < 0, -(a & 0x7FFFFFFF), a)
    b = np.where(b < 0, -(b & 0x7FFFFFFF), b)
    return np.abs(a - b)


def test_sigmoid_within_vecmath_bound():
    # rten-vecmath's Sigmoid is stated within 4 ULP of 1 / (1 + exp(-x)) (exp.rs MAX_SIGMOID_ERROR_ULPS), on its test range
    x = np.arange(-6.0, 6.0, 0.001, dtype=np.float32)
    x = np.concatenate([x, np.float32([-30.0, -0.0, 0.0, 1e-30, 30.0, 90.0, 104.5])])
    got = orn.sigmoid(x)
    ref = (1.0 / (1.0 + np.exp(-x.astype(np.float64)))).astype(np.float32)
    assert int(_ulp_distance(got, ref).max()) <= 4
    assert got[np.argmax(x == 0)] == np.float32(0.5)


def test_tf32_truncate_clears_low_bits():
    v = np.float32([1.0 + 2.0 ** -12, -3.0000002, 0.1])
    t = orn.tf32_truncate(v)
    assert np.all(t.view(np.uint32) & 0x1FFF == 0)
    assert t[0] == 1.0 and abs(t[2] - 0.1) < 2.0 ** -10 * 0.1


def _strings_attr(name, values):
    """A STRINGS AttributeProto (type 8, one `strings` entry per value) as a NodeProto `attribute` field: appended to a
    node's bytes, it adds the attribute (protobuf fields may come in any order)."""
    body = W._ld(1, name.encode()) + b"".join(W._ld(9, v.encode()) for v in values) + W._vi(20, 8)
    return W._ld(5, body)


@pytest.fixture(scope="module")
def summary():
    from rten_b200 import _build
    _build.build()
    from rten_b200.model import onnx_summary
    return onnx_summary


def _gru_model(activations=None, **attrs):
    w = np.zeros((1, 12, 3), np.float32)
    node = W.node("GRU", ["x", "w", "r"], ["y", "yh"], hidden_size=4, **attrs)
    if activations is not None:
        node += _strings_attr("activations", activations)
    return W.model([node],
                   [W.tensor("w", w), W.tensor("r", np.zeros((1, 12, 4), np.float32))],
                   [W.value_info("x", W.FLOAT, [5, 1, 3])], [W.value_info("y", W.FLOAT, [5, 1, 1, 4])])


def test_strings_attribute_is_decoded(summary):
    s = summary(_gru_model(activations=["Sigmoid", "Tanh"], direction="forward", linear_before_reset=1))
    n = s["nodes"][0]
    assert n["op"] == "GRU" and n["attrs"] == ["hidden_size", "direction", "linear_before_reset", "activations"]
    assert n["strings"] == {"activations": ["Sigmoid", "Tanh"]}
    assert "strings" not in summary(_gru_model())["nodes"][0]


def test_truncated_strings_payload_is_an_error(summary):
    import rten_b200 as rt
    good = _gru_model(activations=["Sigmoid", "Tanh"])
    cut = good.index(b"Tanh") + 2  # inside the second string
    for bad in (good[:cut], good[:good.index(b"Sigmoid") + 3]):
        with pytest.raises(rt.OpError) as e:
            summary(bad)
        assert e.value.kind == "InvalidValue"
