"""`pytest -m gpu`: InstanceNormalization and the fused GroupNorm chain (rten_b200_instance_norm / rten_b200_group_norm).

  * bit-exact against tests/instance_norm_ref.py on NCHW and channels-last input, row lengths 49 .. 50176 and a row longer than
    the on-chip path takes, each length on the on-chip and on the streaming path (RTEN_B200_GROUP_NORM_STREAM=1 pins
    the streaming path), in place, one row and many rows, G = 32 with C in {64, 320, 640, 1280}, every activation and
    non-unit InstanceNormalization scale / bias;
  * the error statuses and messages;
  * a CUDA-graph replay of a dense call, and one launch for a dense fused GroupNorm + SiLU;
  * through the executor, models in torch's export shape: an SD-style ResNet block (GroupNorm -> SiLU -> Conv ->
    GroupNorm -> SiLU -> Conv + skip), an attention block and a fast-neural-style residual block -- the fused plan's
    output bit-identical to the node-by-node plan's (RTEN_B200_NO_GROUP_NORM_FUSION=1), and GroupNorm + SiLU within a
    float64-derived bound of torch.nn.functional.group_norm."""

import numpy as np
import pytest

import onnx_writer as ow

pytestmark = pytest.mark.gpu

F32 = np.float32
SPATIAL = {49: (7, 7), 196: (14, 14), 784: (28, 28), 3136: (56, 56), 4096: (64, 64), 40960: (160, 256), 50176: (224, 224),
           70000: (250, 280)}
STREAM_ONLY = 70000  # longer than the on-chip path takes


@pytest.fixture(scope="module")
def rt():
    import rten_b200
    from rten_b200 import _lib
    _lib.load()
    return rten_b200


@pytest.fixture(scope="module")
def on(oracle):
    import instance_norm_ref
    return instance_norm_ref


@pytest.fixture(scope="module")
def ctx(rt):
    return rt.Context(0)


@pytest.fixture(params=["onchip", "stream"])
def path(request, monkeypatch):
    if request.param == "stream":
        monkeypatch.setenv("RTEN_B200_GROUP_NORM_STREAM", "1")
    else:
        monkeypatch.delenv("RTEN_B200_GROUP_NORM_STREAM", raising=False)
    return request.param


def _bits(got, want, what):
    got, want = np.asarray(got), np.asarray(want)
    assert got.shape == want.shape, what
    bad = got.view(np.uint32) != want.view(np.uint32)
    assert not bad.any(), f"{what}: {int(bad.sum())} of {bad.size} elements differ, first at {np.argwhere(bad)[0]}"


def _dev(ctx, x, cl):
    return ctx.to_device(x, channels_last=True) if cl else ctx.to_device(x)


def _x(seed, shape):
    r = np.random.default_rng(seed)
    return (r.standard_normal(shape) * 2 + 0.25).astype(F32)


@pytest.mark.parametrize("L", sorted(SPATIAL))
@pytest.mark.parametrize("cl", [False, True], ids=["nchw", "cl"])
def test_instance_norm_bits(rt, on, ctx, path, L, cl):
    if L == STREAM_ONLY and path == "onchip":
        pytest.skip("a row this long always streams")
    N, C = (2, 3) if L <= 4096 else (1, 2)
    x = _x(L, (N, C) + SPATIAL[L])
    r = np.random.default_rng(L + 1)
    s, b = r.uniform(0.5, 2, C).astype(F32), r.uniform(-1, 1, C).astype(F32)
    y = rt.InstanceNormalization(epsilon=1e-5).run(ctx, _dev(ctx, x, cl), s, b)
    if cl:
        assert y.strides[1] == 1, "the output keeps the channels-last layout"
    _bits(y.numpy(), on.instance_norm(x, s, b, 1e-5), f"InstanceNormalization L={L} {'cl' if cl else 'nchw'} {path}")


@pytest.mark.parametrize("cl", [False, True], ids=["nchw", "cl"])
def test_instance_norm_in_place(rt, on, ctx, path, cl):
    x = _x(5, (2, 8, 28, 28))
    s, b = np.full(8, 1.5, F32), np.full(8, -0.25, F32)
    d = _dev(ctx, x, cl)
    y = rt.InstanceNormalization().run(ctx, d, s, b, out=d)
    assert y is d
    _bits(d.numpy(), on.instance_norm(x, s, b), f"in place {path}")


@pytest.mark.parametrize("shape", [(1, 1, 56, 56), (4, 256, 7, 7), (3, 5), (2, 64, 100)], ids=["one_row", "many_rows", "2d", "3d"])
def test_instance_norm_row_counts(rt, on, ctx, path, shape):
    x = _x(9, shape)
    r = np.random.default_rng(10)
    s, b = r.uniform(0.5, 2, shape[1]).astype(F32), r.uniform(-1, 1, shape[1]).astype(F32)
    _bits(rt.InstanceNormalization().run(ctx, x, s, b).numpy(), on.instance_norm(x, s, b), f"{shape} {path}")


def test_instance_norm_strided_input(rt, on, ctx):
    """any other strides: copied to contiguous, the NCHW path"""
    base = _x(11, (2, 6, 20, 20))
    x = base[:, ::2, :, 1:17]
    s, b = np.linspace(0.5, 2, 3).astype(F32), np.linspace(-1, 1, 3).astype(F32)
    _bits(rt.InstanceNormalization().run(ctx, x, s, b).numpy(), on.instance_norm(np.ascontiguousarray(x), s, b), "strided")


ACTS = {"none": None, "relu": "relu", "sigmoid": "sigmoid", "silu": "silu", "hard_sigmoid": "hard_sigmoid", "hard_swish": "hard_swish"}


def _act(rt, name):
    """(the op's activation argument, the oracle function)"""
    from oracle import activations as A, oracle
    return {None: (rt.ACT_NONE, None), "relu": (rt.ACT_RELU, oracle.relu), "sigmoid": (rt.ACT_SIGMOID, A.sigmoid),
            "silu": (rt.ACT_SILU, A.silu), "hard_sigmoid": ((rt.ACT_HARD_SIGMOID, 0.25, 0.375), lambda v: A.hard_sigmoid(v, 0.25, 0.375)),
            "hard_swish": (rt.ACT_HARD_SWISH, A.hard_swish)}[name]


@pytest.mark.parametrize("C, hw", [(64, 16), (320, 64), (640, 32), (1280, 16), (1280, 8)])
@pytest.mark.parametrize("cl", [False, True], ids=["nchw", "cl"])
def test_group_norm_sd_shapes(rt, on, ctx, path, C, hw, cl):
    G = 32
    x = _x(C + hw, (2, C, hw, hw))
    r = np.random.default_rng(C)
    gamma, beta = (1 + 0.2 * r.standard_normal(C)).astype(F32), (0.2 * r.standard_normal(C)).astype(F32)
    s, b = np.ones(G, F32), np.zeros(G, F32)
    act, fn = _act(rt, "silu")
    y = rt.GroupNorm(G, 1e-5, act).run(ctx, _dev(ctx, x, cl), s, b, gamma, beta)
    _bits(y.numpy(), on.group_norm(x, G, s, b, gamma, beta, 1e-5, fn), f"GroupNorm C={C} {hw}x{hw} {path}")


@pytest.mark.parametrize("act", sorted(ACTS))
@pytest.mark.parametrize("cl", [False, True], ids=["nchw", "cl"])
def test_group_norm_activations_and_scale(rt, on, ctx, path, act, cl):
    G, C = 8, 48
    x = _x(21, (2, C, 12, 10))
    r = np.random.default_rng(22)
    s, b = r.uniform(0.5, 2, G).astype(F32), r.uniform(-1, 1, G).astype(F32)
    gamma, beta = r.standard_normal(C).astype(F32), r.standard_normal(C).astype(F32)
    a, fn = _act(rt, ACTS[act])
    y = rt.GroupNorm(G, 1e-6, a).run(ctx, _dev(ctx, x, cl), s, b, gamma, beta)
    _bits(y.numpy(), on.group_norm(x, G, s, b, gamma, beta, 1e-6, fn), f"GroupNorm {act} {path}")


def test_group_norm_without_affine(rt, on, ctx):
    x = _x(23, (1, 32, 9, 9))
    s, b = np.full(4, 0.5, F32), np.full(4, 0.125, F32)
    _bits(rt.GroupNorm(4).run(ctx, x, s, b).numpy(), on.group_norm(x, 4, s, b), "GroupNorm without gamma / beta")


def test_errors(rt, ctx):
    from rten_b200 import OpError
    IN, ones, zeros = rt.InstanceNormalization(), np.ones(4, F32), np.zeros(4, F32)
    cases = [
        (lambda: IN.run(ctx, np.zeros(4, F32), ones, zeros), "expected input with >= 2 dims"),
        (lambda: IN.run(ctx, np.zeros((1, 4, 3), F32), np.ones(3, F32), zeros), "scale length should match channel count"),
        (lambda: IN.run(ctx, np.zeros((1, 4, 3), F32), ones, np.zeros(5, F32)), "bias length should match channel count"),
        (lambda: rt.GroupNorm(3).run(ctx, np.zeros((1, 4, 3, 3), F32), np.ones(3, F32), np.zeros(3, F32)),
         "Input length must be a multiple of specified dimensions"),
        (lambda: rt.GroupNorm(2).run(ctx, np.zeros((1, 4, 3, 3), F32), np.ones(3, F32), np.zeros(2, F32)),
         "scale length should match channel count"),
        (lambda: rt.GroupNorm(2).run(ctx, np.zeros((1, 4, 3, 3), F32), np.ones(2, F32), np.zeros(2, F32), np.ones(3, F32)),
         "Cannot broadcast inputs"),
    ]
    for fn, msg in cases:
        with pytest.raises(OpError) as e:
            fn()
        assert msg in str(e.value)
    with pytest.raises(OpError) as e:
        IN.run(ctx, np.zeros(4, F32), ones, zeros)
    assert e.value.status == 5  # RTEN_ERR_INVALID_VALUE


def test_graph_capture_and_launch_count(rt, on, ctx):
    x = _x(31, (2, 320, 32, 32))
    G, C = 32, 320
    gamma, beta = np.linspace(0.5, 1.5, C).astype(F32), np.linspace(-0.2, 0.2, C).astype(F32)
    s, b = np.ones(G, F32), np.zeros(G, F32)
    d, dg, db, ds, dbb = (ctx.to_device(a) for a in (x, gamma, beta, s, b))
    op = rt.GroupNorm(G, 1e-5, rt.ACT_SILU)
    ctx.sync()
    n0 = ctx.launches
    eager = op.run(ctx, d, ds, dbb, dg, db)
    ctx.sync()
    assert ctx.launches - n0 == 1, "a dense fused GroupNorm + SiLU is one launch"
    from oracle import activations as A
    want = on.group_norm(x, G, s, b, gamma, beta, 1e-5, A.silu)
    _bits(eager.numpy(), want, "eager")
    ctx.graph_begin()
    out = op.run(ctx, d, ds, dbb, dg, db)
    g = ctx.graph_end()
    out.copy_from(np.full(out.shape, np.nan, F32))
    g.launch()
    ctx.sync()
    _bits(out.numpy(), want, "graph replay")


# ---- through the executor -----------------------------------------------------------------------------------------
def _gn_nodes(tag, x, out, N, C, H, W, G, act="silu", weights=None, seed=0):
    """torch's export of nn.GroupNorm(G, C) (+ SiLU as Mul(x, Sigmoid(x))): nodes and initialisers"""
    r = np.random.default_rng(seed)
    inits = [ow.tensor(f"{tag}_t1", np.array([0, G, -1], np.int64)), ow.tensor(f"{tag}_t2", np.array([N, C, H, W], np.int64)),
             ow.tensor(f"{tag}_s", np.ones(G, F32)), ow.tensor(f"{tag}_b", np.zeros(G, F32)),
             ow.tensor(f"{tag}_g", (1 + 0.2 * r.standard_normal((C, 1, 1))).astype(F32)),
             ow.tensor(f"{tag}_be", (0.2 * r.standard_normal((C, 1, 1))).astype(F32))]
    y = f"{tag}_affine" if act else out
    nodes = [ow.node("Reshape", [x, f"{tag}_t1"], [f"{tag}_r1"]),
             ow.node("InstanceNormalization", [f"{tag}_r1", f"{tag}_s", f"{tag}_b"], [f"{tag}_in"], epsilon=1e-5),
             ow.node("Reshape", [f"{tag}_in", f"{tag}_t2"], [f"{tag}_r2"]),
             ow.node("Mul", [f"{tag}_r2", f"{tag}_g"], [f"{tag}_mul"]),
             ow.node("Add", [f"{tag}_mul", f"{tag}_be"], [y])]
    if act == "silu":
        nodes += [ow.node("Sigmoid", [y], [f"{tag}_sig"]), ow.node("Mul", [y, f"{tag}_sig"], [out])]
    elif act == "relu":
        nodes += [ow.node("Relu", [y], [out])]
    return nodes, inits


def _conv(tag, x, out, C, O, k=3, seed=0):
    r = np.random.default_rng(seed)
    w = (r.standard_normal((O, C, k, k)) / np.sqrt(C * k * k)).astype(F32)
    return [ow.node("Conv", [x, f"{tag}_w", f"{tag}_bias"], [out], pads=[k // 2] * 4)], \
           [ow.tensor(f"{tag}_w", w), ow.tensor(f"{tag}_bias", (0.1 * r.standard_normal(O)).astype(F32))]


def _resnet_block(N, C, H, W):
    n1, i1 = _gn_nodes("gn1", "x", "a1", N, C, H, W, 32, seed=1)
    n2, i2 = _conv("c1", "a1", "h1", C, C, seed=2)
    n3, i3 = _gn_nodes("gn2", "h1", "a2", N, C, H, W, 32, seed=3)
    n4, i4 = _conv("c2", "a2", "h2", C, C, seed=4)
    nodes = n1 + n2 + n3 + n4 + [ow.node("Add", ["h2", "x"], ["y"])]
    return nodes, i1 + i2 + i3 + i4, [N, C, H, W], [N, C, H, W]


def _attention_block(N, C, H, W):
    n1, i1 = _gn_nodes("gn", "x", "h", N, C, H, W, 32, act=None, seed=5)
    r = np.random.default_rng(6)
    wq, wk, wv = ((r.standard_normal((C, C)) / np.sqrt(C)).astype(F32) for _ in range(3))
    inits = i1 + [ow.tensor("seq", np.array([N, C, H * W], np.int64)), ow.tensor("back", np.array([N, C, H, W], np.int64)),
                  ow.tensor("wq", wq), ow.tensor("wk", wk), ow.tensor("wv", wv)]
    nodes = n1 + [ow.node("Reshape", ["h", "seq"], ["hs"]), ow.node("Transpose", ["hs"], ["t"], perm=[0, 2, 1]),
                  ow.node("MatMul", ["t", "wq"], ["q"]), ow.node("MatMul", ["t", "wk"], ["k"]), ow.node("MatMul", ["t", "wv"], ["v"]),
                  ow.node("Transpose", ["k"], ["kt"], perm=[0, 2, 1]), ow.node("MatMul", ["q", "kt"], ["s"]),
                  ow.node("Softmax", ["s"], ["p"], axis=-1), ow.node("MatMul", ["p", "v"], ["o"]),
                  ow.node("Transpose", ["o"], ["ot"], perm=[0, 2, 1]), ow.node("Reshape", ["ot", "back"], ["ob"]),
                  ow.node("Add", ["ob", "x"], ["y"])]
    return nodes, inits, [N, C, H, W], [N, C, H, W]


def _style_block(N, C, H, W):
    r = np.random.default_rng(7)
    n1, i1 = _conv("c1", "x", "h1", C, C, seed=8)
    n2, i2 = _conv("c2", "a1", "h2", C, C, seed=9)
    inits = i1 + i2 + [ow.tensor("s1", r.uniform(0.5, 1.5, C).astype(F32)), ow.tensor("b1", r.uniform(-0.5, 0.5, C).astype(F32)),
                       ow.tensor("s2", r.uniform(0.5, 1.5, C).astype(F32)), ow.tensor("b2", r.uniform(-0.5, 0.5, C).astype(F32))]
    nodes = n1 + [ow.node("InstanceNormalization", ["h1", "s1", "b1"], ["n1"], epsilon=1e-5), ow.node("Relu", ["n1"], ["a1"])] + n2 + \
        [ow.node("InstanceNormalization", ["h2", "s2", "b2"], ["n2"], epsilon=1e-5), ow.node("Add", ["n2", "x"], ["y"])]
    return nodes, inits, [N, C, H, W], [N, C, H, W]


def _gn_silu_model(N, C, H, W):
    nodes, inits = _gn_nodes("gn", "x", "y", N, C, H, W, 32, seed=11)
    return nodes, inits, [N, C, H, W], [N, C, H, W]


def _load(rt, ctx, build, shape, fused, monkeypatch):
    nodes, inits, xs, ys = build(*shape)
    data = ow.model(nodes, inits, [ow.value_info("x", ow.FLOAT, xs)], [ow.value_info("y", ow.FLOAT, ys)], opset=17)
    if fused:
        monkeypatch.delenv("RTEN_B200_NO_GROUP_NORM_FUSION", raising=False)
    else:
        monkeypatch.setenv("RTEN_B200_NO_GROUP_NORM_FUSION", "1")
    from rten_b200.model import Model
    return Model(ctx, data)


@pytest.mark.parametrize("build, shape, groups", [(_resnet_block, (2, 64, 16, 16), 2), (_resnet_block, (1, 320, 32, 32), 2),
                                                  (_attention_block, (1, 128, 16, 16), 1), (_style_block, (1, 32, 56, 56), 0)],
                         ids=["resnet64", "resnet320", "attention", "style"])
@pytest.mark.parametrize("cl", [False, True], ids=["nchw", "cl"])
def test_executor_fused_equals_node_plan(rt, ctx, monkeypatch, build, shape, groups, cl):
    x = _x(41, shape)
    fused = _load(rt, ctx, build, shape, True, monkeypatch)
    plain = _load(rt, ctx, build, shape, False, monkeypatch)
    assert fused.node_ops.count("GroupNorm") == groups
    assert "GroupNorm" not in plain.node_ops and "InstanceNormalization" in plain.node_ops
    yf = fused.run({"x": _dev(ctx, x, cl)})[0].numpy()
    yp = plain.run({"x": _dev(ctx, x, cl)})[0].numpy()
    _bits(yf, yp, f"{build.__name__} fused vs node-by-node")


@pytest.mark.parametrize("shape", [(2, 320, 64, 64), (1, 128, 96, 96)])
def test_executor_group_norm_silu_against_torch(rt, ctx, monkeypatch, shape):
    import torch
    N, C, H, W = shape
    x = _x(51, shape)
    m = _load(rt, ctx, _gn_silu_model, shape, True, monkeypatch)
    assert m.node_ops == ["GroupNorm"]
    got = m.run({"x": x})[0].numpy().astype(np.float64)
    r = np.random.default_rng(11)
    gamma, beta = 1 + 0.2 * r.standard_normal(C), 0.2 * r.standard_normal(C)
    t = torch.nn.functional.group_norm(torch.from_numpy(x.astype(np.float64)), 32, torch.from_numpy(gamma.astype(F32).astype(np.float64)),
                                       torch.from_numpy(beta.astype(F32).astype(np.float64)), 1e-5)
    want = torch.nn.functional.silu(t).numpy()
    # float32 rounding of the statistics grows with the serial fold (2 L / 64 steps), each output step adds an ulp
    L = C // 32 * H * W
    tol = (16 + 2 * L / 64) * np.finfo(F32).eps * (np.abs(t.numpy()) + np.abs(beta).max() + 1)
    assert np.all(np.abs(got - want) <= tol), float(np.max(np.abs(got - want) / tol))
