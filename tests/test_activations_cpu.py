"""CPU checks of the Sigmoid / Silu / HardSigmoid / HardSwish test infrastructure (no GPU): the numpy restatement
oracle/activations.py against the reference's known answers and its stated accuracy, the special values the kernels
must reproduce, and the ONNX reader on a HardSigmoid node."""
import json
import os

import numpy as np
import pytest

import onnx_writer as W
from oracle import activations as oa
from oracle import oracle

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "activation_cases.json")
F32 = np.float32


@pytest.fixture(scope="module", autouse=True)
def _oracle_lib():
    oracle.build()


@pytest.fixture(scope="module")
def golden():
    with open(GOLDEN) as f:
        return json.load(f)


def _bits(a):
    return np.asarray(a, F32).view(np.uint32)


def _ulp_distance(a, b):
    """|a - b| in units in the last place, on the ordered integer line of f32 bit patterns"""
    def ordered(x):
        i = np.asarray(x, F32).view(np.int32).astype(np.int64)
        return np.where(i < 0, -(i & 0x7FFFFFFF), i)
    return np.abs(ordered(a) - ordered(b))


def test_hard_sigmoid_known_answers(golden):
    # = test_hard_sigmoid (src/ops/unary_elementwise.rs)
    c = golden["hard_sigmoid"]
    y = oa.hard_sigmoid(np.array(c["input"], F32), c["alpha"], c["beta"])
    assert oracle.expect_equal(y, np.array(c["expected"], F32), golden["atol"], golden["rtol"])


def test_hard_swish_known_answers(golden):
    # = test_hard_swish (src/ops/unary_elementwise.rs)
    c = golden["hard_swish"]
    y = oa.hard_swish(np.array(c["input"], F32))
    assert oracle.expect_equal(y, np.array(c["expected"], F32), golden["atol"], golden["rtol"])


def _sweep():
    return np.arange(-6.0, 6.0, 0.001, dtype=F32)


def test_sigmoid_and_silu_within_4_ulp_of_the_plain_formula():
    # = test_sigmoid / test_silu (rten-vecmath/src/exp.rs): 4 ULP of 1 / (1 + exp(-x)) and x * that over arange(-6, 6, 0.001)
    x = _sweep()
    e = np.exp(-x.astype(np.float64)).astype(F32)
    ref_sig = F32(1.0) / (F32(1.0) + e)
    ref_silu = x * ref_sig
    assert _ulp_distance(oa.sigmoid(x), ref_sig).max() <= 4
    assert _ulp_distance(oa.silu(x), ref_silu).max() <= 4


def test_special_values():
    inf, nan = np.inf, np.nan
    x = np.array([0.0, -0.0, inf, -inf, nan], F32)
    np.testing.assert_array_equal(oa.sigmoid(x)[:4], np.array([0.5, 0.5, 1.0, 0.0], F32))
    assert np.isnan(oa.sigmoid(x)[4])
    s = oa.silu(x)
    assert _bits(s[0]) == _bits(F32(0.0)) and _bits(s[1]) == _bits(F32(-0.0))
    assert s[2] == inf and np.isnan(s[3]) and np.isnan(s[4])  # Silu(-inf) = -inf / inf
    # Exp is inf from 104 on: Silu(x <= -104) = x / inf = -0.0
    assert _bits(oa.silu(np.array([-104.0, -1000.0], F32))).tolist() == [0x80000000] * 2
    hs = oa.hard_sigmoid(x)
    np.testing.assert_array_equal(hs[:4], np.array([0.5, 0.5, 1.0, 0.0], F32))
    assert np.isnan(hs[4])
    # f32::clamp keeps -0.0 and NaN (fminf / fmaxf would not): HardSigmoid(-0.0) with beta = -0.0 is -0.0
    assert _bits(oa.hard_sigmoid(np.array([-0.0], F32), 0.2, -0.0))[0] == 0x80000000
    hw = oa.hard_swish(np.array([-4.0, -3.0, -0.0, 0.0, inf, -inf, nan], F32))
    assert _bits(hw[0]) == 0x80000000  # -4 * 0.0 = -0.0
    assert _bits(hw[1]) == 0x80000000
    assert _bits(hw[2]) == 0x80000000 and _bits(hw[3]) == 0
    assert hw[4] == inf and np.isnan(hw[5]) and np.isnan(hw[6])  # -inf * 0 = NaN


def test_silu_differs_from_mul_of_sigmoid():
    # Silu rounds once where Mul(x, Sigmoid(x)) rounds twice: the executor's SiluFusion is observable in the last bit
    x = _sweep()
    differ = _bits(oa.silu(x)) != _bits(x * oa.sigmoid(x))
    assert differ.sum() > 100


def test_hard_swish_is_x_times_hard_sigmoid_sixth():
    x = _sweep()
    np.testing.assert_array_equal(_bits(oa.hard_swish(x)), _bits(x * oa.hard_sigmoid(x, F32(1.0) / F32(6.0), 0.5)))


def test_reader_lists_hard_sigmoid_attributes():
    from rten_b200.model import onnx_summary
    nodes = [W.node("HardSigmoid", ["x"], ["y"], alpha=1.0 / 6.0, beta=0.5), W.node("HardSwish", ["y"], ["z"]),
             W.node("Sigmoid", ["z"], ["s"])]
    data = W.model(nodes, [], [W.value_info("x", 1, [1, 4])], [W.value_info("s", 1, [1, 4])])
    s = onnx_summary(data)
    assert [n["op"] for n in s["nodes"]] == ["HardSigmoid", "HardSwish", "Sigmoid"]
    assert s["nodes"][0]["attrs"] == ["alpha", "beta"]
    assert s["nodes"][1]["attrs"] == [] and s["nodes"][2]["attrs"] == []
