"""CPU-only: the torch-exported decoder fixtures (tests/golden/make_torch_decoder_fixtures.py) contain exactly the node
types the executor was built for, and every one of them is a row of the executor's OPS table (rten_b200/csrc/model.cu)."""
import collections
import os
import re

import pytest

from rten_b200.model import onnx_summary

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")

EXPECTED = {
    "torch_gpt2.onnx": {"Add", "Cast", "Concat", "Constant", "ConstantOfShape", "Div", "Gather", "MatMul", "Mul", "Pow", "Range",
                        "ReduceMean", "Reshape", "Shape", "Slice", "Softmax", "Split", "Sqrt", "Squeeze", "Sub", "Tanh",
                        "Transpose", "Unsqueeze", "Where"},
    "torch_llama_block.onnx": {"Cast", "Concat", "Constant", "ConstantOfShape", "Equal", "Expand", "Mul", "Neg", "Reshape", "Slice",
                               "Trilu", "Unsqueeze", "Where"},
}


def onnx_ops():
    """the op types OPS accepts in the ONNX domain"""
    src = open(os.path.join(ROOT, "rten_b200", "csrc", "model.cu")).read()
    table = src[src.index("constexpr OpDef OPS[] = {"):src.index("constexpr const OpDef* row(")]
    return {m.group(1) for m in re.finditer(r'^\s*\{"(\w+)", ([A-Z0-9 |]+),', table, re.M) if "ONNX" in m.group(2)}


@pytest.mark.parametrize("name", sorted(EXPECTED))
def test_fixture_node_types(name):
    s = onnx_summary(open(os.path.join(GOLDEN, name), "rb").read())
    ops = collections.Counter(n["op"] for n in s["nodes"])
    assert set(ops) == EXPECTED[name]
    missing = set(ops) - onnx_ops()
    assert not missing, f"{name}: node types with no ONNX row in OPS: {sorted(missing)}"


def test_gpt2_cache_dims_are_static():
    s = onnx_summary(open(os.path.join(GOLDEN, "torch_gpt2.onnx"), "rb").read())
    for i in s["inputs"]:
        if i["name"].startswith("past_key_values."):
            assert i["dims"][1] == 4 and i["dims"][3] == 16, i
