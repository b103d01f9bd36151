"""The executor's load-time graph rewrites, rule by rule: which nodes a loaded model keeps (Model.node_ops) and which
Concat inputs its producers write in place (Model.summary["concat_in_place"]).  Each case is a small graph that only
loads; the positive cases run end to end in test_gpu_activations, test_gpu_instance_norm and test_gpu_resize_concat."""
import numpy as np
import pytest

import onnx_writer as ow

pytestmark = pytest.mark.gpu
F32 = np.float32


@pytest.fixture(scope="module")
def rt():
    import rten_b200
    import rten_b200.model  # noqa: F401
    return rten_b200


@pytest.fixture(scope="module")
def ctx(rt):
    return rt.Context(0)


def _load(rt, ctx, monkeypatch, nodes, inits, inputs, outputs, env=()):
    """the model of `nodes` with f32 graph inputs {name: shape}, loaded with the switches in `env` set"""
    for k in ("RTEN_B200_NO_GROUP_NORM_FUSION", "RTEN_B200_NO_CONCAT_ELISION"):
        monkeypatch.delenv(k, raising=False)
    for k in env:
        monkeypatch.setenv(k, "1")
    data = ow.model(nodes, inits, [ow.value_info(n, ow.FLOAT, s) for n, s in inputs.items()],
                    [ow.value_info(n, ow.FLOAT, [1]) for n in outputs])
    return rt.model.Model(ctx, data)


X = {"x": [1, 8, 6, 6]}


def _conv(name, x, O=8, C=8):
    r = np.random.default_rng(len(name))
    return ow.node("Conv", [x, f"{name}_w", f"{name}_b"], [name], pads=[1, 1, 1, 1]), \
        [ow.tensor(f"{name}_w", r.standard_normal((O, C, 3, 3)).astype(F32)), ow.tensor(f"{name}_b", r.standard_normal(O).astype(F32))]


# ---- SiluFusion: Mul(x, Sigmoid(x)) -> Silu(x) when the Sigmoid's output has no other use
@pytest.mark.parametrize("order", ["x_first", "sigmoid_first"])
def test_silu_fused_in_either_operand_order(rt, ctx, monkeypatch, order):
    mul_in = ["x", "s"] if order == "x_first" else ["s", "x"]
    nodes = [ow.node("Sigmoid", ["x"], ["s"]), ow.node("Mul", mul_in, ["y"])]
    assert _load(rt, ctx, monkeypatch, nodes, [], X, ["y"]).node_ops == ["Silu"]


def test_silu_not_fused_when_the_sigmoid_has_another_reader(rt, ctx, monkeypatch):
    nodes = [ow.node("Sigmoid", ["x"], ["s"]), ow.node("Mul", ["x", "s"], ["y"]), ow.node("Relu", ["s"], ["z"])]
    assert _load(rt, ctx, monkeypatch, nodes, [], X, ["y", "z"]).node_ops == ["Sigmoid", "Mul", "Relu"]


def test_silu_not_fused_when_the_sigmoid_is_a_graph_output(rt, ctx, monkeypatch):
    nodes = [ow.node("Sigmoid", ["x"], ["s"]), ow.node("Mul", ["x", "s"], ["y"])]
    assert _load(rt, ctx, monkeypatch, nodes, [], X, ["y", "s"]).node_ops == ["Sigmoid", "Mul"]


def test_silu_not_fused_for_another_multiplicand(rt, ctx, monkeypatch):
    nodes = [ow.node("Sigmoid", ["x"], ["s"]), ow.node("Mul", ["w", "s"], ["y"])]
    assert _load(rt, ctx, monkeypatch, nodes, [], {**X, "w": X["x"]}, ["y"]).node_ops == ["Sigmoid", "Mul"]


# ---- Conv + activation -> the activation in the convolution epilogue
@pytest.mark.parametrize("act", ["Relu", "Sigmoid", "HardSigmoid", "HardSwish", "Silu"])
def test_conv_activation_fused(rt, ctx, monkeypatch, act):
    conv, inits = _conv("c", "x")
    if act == "Silu":  # made by SiluFusion first
        nodes = [conv, ow.node("Sigmoid", ["c"], ["s"]), ow.node("Mul", ["c", "s"], ["y"])]
    else:
        nodes = [conv, ow.node(act, ["c"], ["y"], **({"alpha": 0.25, "beta": 0.4} if act == "HardSigmoid" else {}))]
    assert _load(rt, ctx, monkeypatch, nodes, inits, X, ["y"]).node_ops == ["Conv"]


def test_conv_clip_not_fused(rt, ctx, monkeypatch):
    conv, inits = _conv("c", "x")
    inits += [ow.tensor("lo", np.array(0, F32)), ow.tensor("hi", np.array(6, F32))]
    nodes = [conv, ow.node("Clip", ["c", "lo", "hi"], ["y"])]
    assert _load(rt, ctx, monkeypatch, nodes, inits, X, ["y"]).node_ops == ["Conv", "Clip"]


def test_conv_activation_not_fused_when_the_conv_output_is_a_graph_output(rt, ctx, monkeypatch):
    conv, inits = _conv("c", "x")
    nodes = [conv, ow.node("Relu", ["c"], ["y"])]
    assert _load(rt, ctx, monkeypatch, nodes, inits, X, ["y", "c"]).node_ops == ["Conv", "Relu"]


def test_conv_activation_not_fused_when_the_conv_output_is_read_twice(rt, ctx, monkeypatch):
    conv, inits = _conv("c", "x")
    nodes = [conv, ow.node("Relu", ["c"], ["r"]), ow.node("Add", ["r", "c"], ["y"])]
    assert _load(rt, ctx, monkeypatch, nodes, inits, X, ["y"]).node_ops == ["Conv", "Relu", "Add"]


def test_conv_takes_only_the_first_of_two_activations(rt, ctx, monkeypatch):
    conv, inits = _conv("c", "x")
    nodes = [conv, ow.node("Relu", ["c"], ["r"]), ow.node("Sigmoid", ["r"], ["y"])]
    assert _load(rt, ctx, monkeypatch, nodes, inits, X, ["y"]).node_ops == ["Conv", "Sigmoid"]


# ---- MatMul + Add(constant f32 [N]) -> MatMul with a row bias
def _matmul_add(rt, ctx, monkeypatch, bias_shape=(16,), bias_const=True, weight_const=True):
    r = np.random.default_rng(3)
    inputs = {"a": [4, 8]}
    inits = []
    if weight_const:
        inits.append(ow.tensor("w", r.standard_normal((8, 16)).astype(F32)))
    else:
        inputs["w"] = [8, 16]
    if bias_const:
        inits.append(ow.tensor("bias", r.standard_normal(bias_shape).astype(F32)))
    else:
        inputs["bias"] = list(bias_shape)
    nodes = [ow.node("MatMul", ["a", "w"], ["m"]), ow.node("Add", ["m", "bias"], ["y"])]
    return _load(rt, ctx, monkeypatch, nodes, inits, inputs, ["y"]).node_ops


def test_matmul_bias_fused(rt, ctx, monkeypatch):
    assert _matmul_add(rt, ctx, monkeypatch) == ["MatMul"]


@pytest.mark.parametrize("case", [dict(bias_const=False), dict(bias_shape=(17,)), dict(bias_shape=(1, 16)), dict(weight_const=False)],
                         ids=["bias_not_constant", "bias_wrong_length", "bias_2d", "weight_not_constant"])
def test_matmul_bias_not_fused(rt, ctx, monkeypatch, case):
    assert _matmul_add(rt, ctx, monkeypatch, **case) == ["MatMul", "Add"]


# ---- GroupNormFusion: torch's export of nn.GroupNorm (+ activation) -> one GroupNorm node
CHAIN = ["Reshape", "InstanceNormalization", "Reshape", "Mul", "Add"]


def _group_norm(act=None, shared=None, shape_target=False, scale_len=2, env=()):
    """nn.GroupNorm(2, 8) on x [1, 8, 6, 6] as torch exports it; `shared`: an intermediate that an Identity also reads"""
    G, (N, C, H, W) = 2, X["x"]
    r = np.random.default_rng(5)
    inits = [ow.tensor("t1", np.array([0, G, -1], np.int64)), ow.tensor("s", np.ones(scale_len, F32)),
             ow.tensor("b", np.zeros(scale_len, F32)), ow.tensor("g", r.standard_normal((C, 1, 1)).astype(F32)),
             ow.tensor("be", r.standard_normal((C, 1, 1)).astype(F32))]
    nodes = [ow.node("Reshape", ["x", "t1"], ["r1"]), ow.node("InstanceNormalization", ["r1", "s", "b"], ["in"], epsilon=1e-5)]
    if shape_target:
        nodes.append(ow.node("Shape", ["x"], ["t2"]))
    else:
        inits.append(ow.tensor("t2", np.array([N, C, H, W], np.int64)))
    nodes += [ow.node("Reshape", ["in", "t2"], ["r2"]), ow.node("Mul", ["r2", "g"], ["mul"]), ow.node("Add", ["mul", "be"], ["add"])]
    outputs = ["y"]
    if act == "Relu":
        nodes.append(ow.node("Relu", ["add"], ["y"]))
    elif act == "Silu":
        nodes += [ow.node("Sigmoid", ["add"], ["sig"]), ow.node("Mul", ["add", "sig"], ["y"])]
    else:
        outputs = ["add"]
    if shared:
        nodes.append(ow.node("Identity", [shared], ["extra"]))
        outputs.append("extra")
    return nodes, inits, outputs, env


@pytest.mark.parametrize("act", [None, "Relu", "Silu"])
def test_group_norm_fused(rt, ctx, monkeypatch, act):
    nodes, inits, outputs, env = _group_norm(act)
    assert _load(rt, ctx, monkeypatch, nodes, inits, X, outputs, env).node_ops == ["GroupNorm"]


@pytest.mark.parametrize("shared", ["r1", "in", "r2", "mul"])
def test_group_norm_not_fused_when_an_intermediate_has_another_reader(rt, ctx, monkeypatch, shared):
    nodes, inits, outputs, env = _group_norm(shared=shared)
    assert _load(rt, ctx, monkeypatch, nodes, inits, X, outputs, env).node_ops == CHAIN + ["Identity"]


def test_group_norm_keeps_an_activation_whose_input_has_another_reader(rt, ctx, monkeypatch):
    nodes, inits, outputs, env = _group_norm("Relu", shared="add")
    assert _load(rt, ctx, monkeypatch, nodes, inits, X, outputs, env).node_ops == ["GroupNorm", "Relu", "Identity"]


@pytest.mark.parametrize("case, ops", [(dict(shape_target=True), ["Reshape", "InstanceNormalization", "Shape"] + CHAIN[2:]),
                                       (dict(scale_len=4), CHAIN),
                                       (dict(act="Silu", env=["RTEN_B200_NO_GROUP_NORM_FUSION"]), CHAIN + ["Silu"])],
                         ids=["target_from_shape", "scale_length_not_groups", "switched_off"])
def test_group_norm_not_fused(rt, ctx, monkeypatch, case, ops):
    nodes, inits, outputs, env = _group_norm(**case)
    assert _load(rt, ctx, monkeypatch, nodes, inits, X, outputs, env).node_ops == ops


# ---- Concat elision: which inputs of a channel Concat their producers write in place
def _concat_plan(rt, ctx, monkeypatch, concat_inputs, outputs=("y",), nested=False):
    (ca, ia), (cb, ib), (cc, ic) = _conv("ca", "x", 4), _conv("cb", "x", 6), _conv("cc", "x", 2)
    nodes = [ca, cb, cc]
    if nested:
        nodes += [ow.node("Concat", ["ca", "cb"], ["inner"], axis=1), ow.node("Concat", ["inner", "cc"], ["y"], axis=1)]
    else:
        nodes.append(ow.node("Concat", concat_inputs, ["y"], axis=1))
    m = _load(rt, ctx, monkeypatch, nodes, ia + ib + ic, X, list(outputs))
    return m.summary["concat_in_place"]


def test_concat_of_two_convolutions_written_in_place(rt, ctx, monkeypatch):
    assert _concat_plan(rt, ctx, monkeypatch, ["ca", "cb"]) == [{"output": "y", "copied": 0, "in_place": ["ca", "cb"]}]


def test_concat_copies_a_graph_output(rt, ctx, monkeypatch):
    plan = _concat_plan(rt, ctx, monkeypatch, ["ca", "cb"], outputs=("y", "ca"))
    assert plan == [{"output": "y", "copied": 1, "in_place": ["cb"]}]


def test_concat_copies_an_input_named_twice(rt, ctx, monkeypatch):
    plan = _concat_plan(rt, ctx, monkeypatch, ["ca", "cb", "ca"])
    assert plan == [{"output": "y", "copied": 2, "in_place": ["cb"]}]


def test_nested_concat_copies_the_inner_concat(rt, ctx, monkeypatch):
    plan = _concat_plan(rt, ctx, monkeypatch, None, nested=True)
    assert plan == [{"output": "inner", "copied": 0, "in_place": ["ca", "cb"]}, {"output": "y", "copied": 1, "in_place": ["cc"]}]
