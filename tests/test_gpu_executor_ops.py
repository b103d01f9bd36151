"""`pytest -m gpu`: the executor's operator table through the model API.  Every operator loads only in the domain the
reference's registry lists it under (src/op_registry/onnx_registry.rs), and an unknown domain keeps its own message."""
import pytest

import onnx_writer as W

pytestmark = pytest.mark.gpu

MICROSOFT = ["MatMulNBits", "GroupQueryAttention", "MultiHeadAttention", "SkipLayerNormalization", "SkipSimplifiedLayerNormalization"]
DEFAULT = ["Conv", "ConvInteger", "ConvTranspose", "Relu", "Clip", "Sigmoid", "HardSigmoid", "HardSwish", "MaxPool", "AveragePool",
           "Resize", "Upsample", "Concat", "GlobalAveragePool", "ReduceMean", "Gemm", "MatMul", "MatMulInteger", "Add", "Mul",
           "Softmax", "LayerNormalization", "RMSNormalization", "SimplifiedLayerNormalization", "Erf", "Gather", "Cast",
           "DynamicQuantizeLinear", "Attention", "RotaryEmbedding", "GRU", "LSTM", "Constant", "Reshape", "Flatten", "Squeeze",
           "Unsqueeze", "Transpose", "Identity"]
OTHER_DOMAIN = [(op, d) for op in MICROSOFT for d in ("", "ai.onnx")] + [(op, "com.microsoft") for op in DEFAULT]


@pytest.fixture(scope="module")
def rt():
    import rten_b200
    import rten_b200.model  # noqa: F401
    return rten_b200


@pytest.fixture(scope="module")
def ctx(rt):
    return rt.Context(0)


def _one_node(op, domain):
    return W.model([W.node(op, ["x"], ["y"], domain=domain)], [], [W.value_info("x", W.FLOAT, [2, 3])],
                   [W.value_info("y", W.FLOAT, [2, 3])], extra_opsets=[("com.microsoft", 1)])


@pytest.mark.parametrize("op,domain", OTHER_DOMAIN)
def test_an_operator_of_the_other_domain_fails_the_load(rt, ctx, op, domain):
    with pytest.raises(rt.OpError) as e:
        rt.model.Model(ctx, _one_node(op, domain))
    want = "unsupported operator " + ("com.microsoft." if domain == "com.microsoft" else "") + op
    assert e.value.kind == "UnsupportedValue" and e.value.msg == want, e.value.msg


@pytest.mark.parametrize("domain", ["", "ai.onnx", "com.microsoft"])
def test_gelu_loads_in_both_domains(rt, ctx, domain):
    assert rt.model.Model(ctx, _one_node("Gelu", domain)).node_ops == ["Gelu"]


def test_an_unknown_domain_keeps_its_message(rt, ctx):
    with pytest.raises(rt.OpError) as e:
        rt.model.Model(ctx, _one_node("MatMul", "com.foobar"))
    assert e.value.kind == "UnsupportedValue" and e.value.msg == "unsupported operator domain 'com.foobar'", e.value.msg
