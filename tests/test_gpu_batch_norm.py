"""`pytest -m gpu`: BatchNormalization (rten_b200_batch_norm) and its load-time fold into a Conv / ConvTranspose.

  * the operator against tests/batch_norm_ref.py bit for bit: NCHW with every P % 4, channels-last with C % 4 == 0 and
    != 0, [N, C], [N, C, L], [N, C, 1] and rank 1, misaligned and strided inputs, in place, an output view with guard
    elements, every activation, NaN / inf / subnormal inputs, var + epsilon subnormal, zero scale, empty tensors;
  * kernel identity: every case runs once under CUPTI in a child process and must run exactly the gn_apply_kernel
    instance `bn_rule` names (no kernel for an empty tensor); the error paths leave the output unallocated;
  * the fold: Conv -> BatchNormalization -> Relu loaded through the executor equals rten_b200_conv2d_act called with the
    oracle's folded weights and Relu, bit for bit and launch for launch, for 1x1, 3x3, strided, depthwise, grouped and
    bias-free convolutions, and ConvTranspose (its Relu a node of its own);
  * no fold where the conditions fail: a second reader of the Conv's output, Conv -> Relu -> BatchNormalization, a
    non-constant mean; the BatchNormalization then runs on gn_apply_kernel;
  * the load errors of training_mode = 1, spatial = 0 and a used running_mean output;
  * a DenseNet-121 in torchvision's layout with its BatchNormalization nodes unfolded, at batch 2 in both f32 modes,
    against a float64 torch forward."""
import json

import numpy as np
import pytest

import batch_norm_ref as ref
import gpu_checks as gc
import onnx_writer as ow
import test_gpu_conv_norm_resize_kernels as ck
import test_gpu_row_kernels as rk

pytestmark = pytest.mark.gpu

F32 = np.float32
ACTS = ("none", "relu", "sigmoid", "silu", "hard_sigmoid", "hard_swish")


@pytest.fixture(scope="module")
def rt():
    import rten_b200
    from rten_b200 import _lib
    _lib.load()
    return rten_b200


@pytest.fixture(scope="module")
def ctx(rt):
    return rt.Context(0)


def _act(rt, name):
    """(the op's activation argument, the oracle function)"""
    from oracle import activations as A, oracle
    return {"none": (rt.ACT_NONE, None), "relu": (rt.ACT_RELU, oracle.relu), "sigmoid": (rt.ACT_SIGMOID, A.sigmoid),
            "silu": (rt.ACT_SILU, A.silu), "hard_sigmoid": ((rt.ACT_HARD_SIGMOID, 0.25, 0.375), lambda v: A.hard_sigmoid(v, 0.25, 0.375)),
            "hard_swish": (rt.ACT_HARD_SWISH, A.hard_swish)}[name]


# ---- the operator -----------------------------------------------------------------------------------------------------
def bn_specs():
    s = lambda x, **kw: dict(x=x, **kw)  # noqa: E731
    return [
        # NCHW, every P % 4: small planes packed several to a block, and planes of more than 128 units one per block row
        s((2, 3, 5, 4)), s((2, 3, 5, 5)), s((2, 3, 3, 6)), s((2, 3, 3, 5), act="relu"), s((2, 3, 17, 17)), s((2, 3, 23, 24)),
        s((4, 64, 14, 14)), s((32, 1024, 7, 7), act="relu"),
        # channels-last, C % 4 == 0 and != 0
        s((2, 8, 5, 7), cl=True), s((2, 6, 5, 7), cl=True, act="silu"), s((1, 64, 14, 14), cl=True, act="relu"),
        # [N, C], [N, C, L], [N, C, 1], rank 1
        s((32, 100)), s((3, 5)), s((4, 6, 33)), s((5, 7, 1)), s((37,)), s((4, 6, 1, 1)),
        # misaligned and strided inputs, in place, an output view with guard elements
        s((2, 3, 8, 8), place="misaligned"), s((2, 8, 5, 5), cl=True, place="misaligned"), s((2, 6, 7, 9), place="strided"),
        s((2, 3, 8, 8), place="in_place"), s((2, 8, 5, 5), cl=True, place="in_place"), s((16, 12), place="in_place"),
        s((2, 3, 8, 8), place="guarded"), s((24, 10), place="guarded"),
        # every activation, NCHW and channels-last
        *[s((2, 4, 6, 6), act=a) for a in ACTS], *[s((2, 12, 3, 5), cl=True, act=a) for a in ACTS],
        # NaN / inf / subnormal inputs, var + epsilon subnormal, zero scale
        s((2, 4, 4, 4), special=True), s((2, 8, 3, 3), cl=True, special=True), s((9, 4), special=True),
        # a large map and a BatchNorm1d head
        s((2, 256, 28, 28), act="relu"), s((2, 256, 28, 28), cl=True, act="relu"), s((32, 4096), act="relu"),
        # empty tensors
        s((0, 3, 4, 4)), s((2, 0)), s((2, 3, 0)),
    ]


def bn_rule(s):
    """rten_b200_batch_norm: [N, C] and every shape with one element per (n, c), rank 1 included, run as one
    channels-last image; dense channels-last 4-D input on the channels-last instance; everything else (NCHW-contiguous
    or copied to it) on the NCHW instance, which packs planes of at most 128 units (float4s when P % 4 == 0 and the
    pointers are 16-byte aligned) several to a block.  An empty tensor launches nothing."""
    x = s["x"]
    if 0 in x:
        return set()
    P = int(np.prod(x[2:])) if len(x) > 2 else 1
    if len(x) == 1 or P == 1 or (s.get("cl") and s.get("place") != "strided"):
        return {("gn_apply_kernel", (1,))}
    return {("gn_apply_kernel", (0,))}


def spec_id(s):
    return " ".join(f"{k}={v}" for k, v in s.items())


def bn_prepare(s):
    r = rk._rng("batch_norm", spec_id(s))
    x = s["x"]
    C = x[1] if len(x) > 1 else 1
    xs = (r.standard_normal(x) * 2 + 0.25).astype(F32)
    scale, bias, mean = r.uniform(0.5, 2, C).astype(F32), r.uniform(-1, 1, C).astype(F32), r.uniform(-0.5, 0.5, C).astype(F32)
    var = r.uniform(0.1, 2, C).astype(F32)
    eps = 1e-5
    if s.get("special"):
        flat = xs.reshape(-1)
        flat[:6] = [np.nan, np.inf, -np.inf, 1e-40, -1e-41, 0.0]
        if C > 1:
            var[0], scale[1] = 0.0, 0.0  # channel 0: var + epsilon subnormal; channel 1: zero scale
        eps = 1e-40
    return dict(x=xs, scale=scale, bias=bias, mean=mean, var=var, eps=eps)


def bn_launch(rt, ctx, s, inp):
    """(the output, the guard elements around an output view or None)"""
    a, _ = _act(rt, s.get("act", "none"))
    op = rt.BatchNormalization(inp["eps"], a)
    x, place = inp["x"], s.get("place")
    p = [inp[k] for k in ("scale", "bias", "mean", "var")]
    cl = bool(s.get("cl"))
    if place == "misaligned":
        n = x.size
        buf = ctx.empty((n + 1,))
        shape = x.shape
        strides = ck._cl_strides(shape, shape[1]) if cl else rt.ops._contig(shape)
        xd = buf.view(shape, strides, 1)
        xd.copy_from(x)
        return op.run(ctx, xd, *p).numpy(), None
    if place == "strided":
        base = ctx.to_device(np.repeat(x, 2, axis=1))
        xd = base.view(x.shape, (base.strides[0], 2 * base.strides[1]) + base.strides[2:])
        return op.run(ctx, xd, *p).numpy(), None
    xd = ctx.to_device(x, channels_last=cl)
    if place == "in_place":
        y = op.run(ctx, xd, *p, out=xd)
        assert y is xd
        return xd.numpy(), None
    if place == "guarded":
        buf = ctx.empty((x.size + 8,))
        buf.copy_from(np.full(x.size + 8, np.nan, F32))
        out = buf.view(x.shape, rt.ops._contig(x.shape), 4)
        op.run(ctx, xd, *p, out=out)
        g = buf.numpy()
        return out.numpy(), np.concatenate([g[:4], g[-4:]])
    y = op.run(ctx, xd, *p)
    if cl and len(x.shape) == 4 and x.size:
        assert y.strides[1] == 1, f"{spec_id(s)}: channels-last in must give channels-last out"
    return y.numpy(), None


def bn_want(rt, s, inp):
    _, fn = _act(rt, s.get("act", "none"))
    return ref.batch_norm(inp["x"], inp["scale"], inp["bias"], inp["mean"], inp["var"], inp["eps"], fn)


def _kernel_probe():
    import rten_b200 as rt
    from rten_b200.model import Model
    ctx = rt.Context(0)
    res = {}
    for s in bn_specs():
        inp = bn_prepare(s)

        def call():
            bn_launch(rt, ctx, s, inp)
            ctx.sync()
        res[spec_id(s)] = sorted(rk.capture_kernels(call)[0])
    for variant in NO_FOLD:
        (_, _, mean, _), _, data = _conv_bn_graph(variant)
        m = Model(ctx, data)
        inputs = _no_fold_inputs(variant, mean)

        def run():
            m.run(inputs)
            ctx.sync()
        res["no fold " + variant] = sorted(rk.capture_kernels(run)[0])
    print(json.dumps({"names": res}))


def test_kernel_identity():
    names = rk.probe_in_child("test_gpu_batch_norm")["names"]
    wrong, seen = [], set()
    for s in bn_specs():
        want = bn_rule(s)
        ran = {ck.kernel_key(n) for n in names[spec_id(s)]} - {None}
        if ran != want:
            wrong.append((spec_id(s), sorted(want), sorted(ran)))
        seen |= ran
    assert not wrong, f"{len(wrong)} cases ran other kernels than the rule names: {wrong[:8]}"
    assert seen == {("gn_apply_kernel", (0,)), ("gn_apply_kernel", (1,))}
    for variant in NO_FOLD:  # the BatchNormalization the fold leaves runs on the NCHW instance (a contiguous input)
        ran = {ck.kernel_key(n) for n in names["no fold " + variant]} - {None}
        assert ran == {("gn_apply_kernel", (0,))}, (variant, ran)


def test_batch_norm_bit_exact(rt, ctx):
    for s in bn_specs():
        inp = bn_prepare(s)
        got, guards = bn_launch(rt, ctx, s, inp)
        gc.assert_bit_exact(got, bn_want(rt, s, inp), spec_id(s))
        if guards is not None:
            assert np.isnan(guards).all(), f"{spec_id(s)}: writes outside the output view"


def test_one_launch_and_graph_replay(rt, ctx):
    x = np.random.default_rng(3).standard_normal((2, 64, 28, 28)).astype(F32)
    p = [np.linspace(0.5, 1.5, 64).astype(F32), np.linspace(-1, 1, 64).astype(F32), np.zeros(64, F32), np.ones(64, F32)]
    d, *pd = (ctx.to_device(a) for a in [x] + p)
    op = rt.BatchNormalization(1e-5, rt.ACT_RELU)
    ctx.sync()
    n0 = ctx.launches
    eager = op.run(ctx, d, *pd)
    ctx.sync()
    assert ctx.launches - n0 == 1
    want = ref.batch_norm(x, *p, 1e-5, lambda v: np.maximum(v, F32(0)))
    gc.assert_bit_exact(eager.numpy(), want, "eager")
    ctx.graph_begin()
    out = op.run(ctx, d, *pd)
    g = ctx.graph_end()
    out.copy_from(np.full(out.shape, np.nan, F32))
    g.launch()
    ctx.sync()
    gc.assert_bit_exact(out.numpy(), want, "graph replay")


def test_errors_leave_the_output_unallocated(rt, ctx):
    import ctypes as C
    one, two = np.ones(1, F32), np.ones(2, F32)
    cases = [(np.float32(1.0).reshape(()), [one] * 4, 5, "Input must have at least 1 dim")]
    for k, name in enumerate(("scale", "bias", "mean", "var")):
        q = [two] * 4
        q[k] = np.ones(3, F32)
        cases.append((np.zeros((1, 2, 3), F32), q, 3, f"{name}.size(0) != channels"))
    cases.append((np.zeros(5, F32), [two] * 4, 3, "scale.size(0) != channels"))  # rank 1 is one channel
    for x, q, status, msg in cases:
        A = rt.ops._Args(ctx)
        o = A.out()
        act = rt.ops._activation(rt.ACT_NONE)
        st = ctx.lib.rten_b200_batch_norm(ctx.handle, A.t(ctx.to_device(x)), *(A.t(v) for v in q), 1e-5, C.byref(act), C.byref(o))
        assert st == status, (msg, st)
        assert ctx.lib.rten_b200_last_error(ctx.handle).decode() == msg
        assert not o.data, f"{msg}: the failed call left its output allocated"


# ---- through the executor ---------------------------------------------------------------------------------------------
def _out(name):
    return ow.value_info(name, ow.FLOAT, ["d"])


def _bn_params(r, C, tag, skip=()):
    """(scale, beta, mean, var) and their initialisers, but for the names in `skip`"""
    scale, beta, mean = r.uniform(0.5, 1.5, C).astype(F32), r.uniform(-0.5, 0.5, C).astype(F32), r.uniform(-0.2, 0.2, C).astype(F32)
    var = r.uniform(0.2, 2, C).astype(F32)
    return (scale, beta, mean, var), [ow.tensor(f"{tag}_{k}", v) for k, v in zip(("s", "b", "m", "v"), (scale, beta, mean, var))
                                      if f"{tag}_{k}" not in skip]


def _bn_node(tag, x, y, eps=1e-5, **attrs):
    return ow.node("BatchNormalization", [x] + [f"{tag}_{k}" for k in ("s", "b", "m", "v")], [y], epsilon=eps, **attrs)


# (name, C_in, C_out, k, stride, groups, bias, transpose, H)
FOLDS = [("1x1", 64, 128, 1, 1, 1, True, False, 28), ("3x3 halo", 64, 64, 3, 1, 1, True, False, 28),
         ("3x3 stride 2", 32, 64, 3, 2, 1, True, False, 29), ("depthwise", 48, 48, 3, 1, 48, True, False, 14),
         ("grouped", 64, 64, 3, 1, 4, True, False, 14), ("no bias", 32, 64, 3, 1, 1, False, False, 14),
         ("ConvTranspose", 32, 16, 4, 2, 1, True, True, 14), ("grouped ConvTranspose", 32, 16, 4, 2, 2, False, True, 14)]


def _fold_case(name, cin, cout, k, st, groups, bias, tr, H):
    r = np.random.default_rng(cin * 7 + cout + k + st + groups)
    w = (r.standard_normal((cin, cout // groups, k, k) if tr else (cout, cin // groups, k, k)) / np.sqrt(cin // groups * k * k)).astype(F32)
    b = (0.1 * r.standard_normal(cout)).astype(F32) if bias else None
    params, inits = _bn_params(r, cout, "bn")
    pad = k // 2 if not tr else 1
    attrs = dict(kernel_shape=[k, k], strides=[st, st], pads=[pad] * 4, group=groups)
    inits += [ow.tensor("w", w)] + ([ow.tensor("cb", b)] if bias else [])
    nodes = [ow.node("ConvTranspose" if tr else "Conv", ["x", "w"] + (["cb"] if bias else []), ["c"], **attrs),
             _bn_node("bn", "c", "n"), ow.node("Relu", ["n"], ["y"])]
    x = r.standard_normal((2, cin, H, H)).astype(F32)
    return x, w, b, params, pad, ow.model(nodes, inits, [ow.value_info("x", ow.FLOAT, list(x.shape))], [_out("y")], opset=17)


@pytest.mark.parametrize("case", FOLDS, ids=[f[0] for f in FOLDS])
@pytest.mark.parametrize("cl", [False, True], ids=["nchw", "cl"])
def test_fold_equals_conv_with_folded_weights(rt, ctx, case, cl):
    from rten_b200.model import Model
    name, cin, cout, k, st, groups, bias, tr, H = case
    x, w, b, (scale, beta, mean, var), pad, data = _fold_case(*case)
    m = Model(ctx, data)
    want_ops = ["ConvTranspose", "Relu"] if tr else ["Conv"]
    assert m.node_ops == want_ops, m.node_ops
    wf, bf = ref.fold_conv(w, b, scale, beta, mean, var, 1e-5, transpose=tr, groups=groups)
    xd = ctx.to_device(x, channels_last=cl)
    ctx.sync()
    n0 = ctx.launches
    got = m.run({"x": xd})[0]
    ctx.sync()
    n_model = ctx.launches - n0
    if tr:
        op = rt.ConvTranspose(groups=groups, strides=(st, st), padding=(pad,) * 4)
        packed = op.prepack(ctx, 1, ctx.to_device(wf))
        ctx.sync()
        n0 = ctx.launches
        want = rt.Relu().run(ctx, op.run(ctx, xd, ctx.to_device(wf), ctx.to_device(bf), packed_w=packed))
    else:
        op = rt.Conv(groups=groups, strides=(st, st), padding=(pad,) * 4, activation=rt.ACT_RELU)
        packed = op.prepack(ctx, 1, ctx.to_device(wf))
        ctx.sync()
        n0 = ctx.launches
        want = op.run(ctx, xd, ctx.to_device(wf), ctx.to_device(bf), packed_w=packed)
    ctx.sync()
    # (the executor hands a channels-last output over as a contiguous copy: one more launch)
    n_direct = ctx.launches - n0 + (1 if cl else 0)
    assert n_model == n_direct, f"{name}: {n_model} launches through the executor, {n_direct} direct"
    gc.assert_bit_exact(got.numpy(), want.numpy(), f"{name} folded")


def _conv_bn_graph(variant):
    """Conv -> BatchNormalization chains the fold must leave alone"""
    r = np.random.default_rng(11)
    C = 32
    w = (r.standard_normal((C, C, 3, 3)) / np.sqrt(9 * C)).astype(F32)
    params, inits = _bn_params(r, C, "bn", skip=("bn_m",) if variant == "input mean" else ())
    inits += [ow.tensor("w", w), ow.tensor("cb", (0.1 * r.standard_normal(C)).astype(F32))]
    conv = ow.node("Conv", ["x", "w", "cb"], ["c"], kernel_shape=[3, 3], pads=[1] * 4)
    outs = [_out("y")]
    ins = [ow.value_info("x", ow.FLOAT, [2, C, 14, 14])]
    if variant == "second reader":
        nodes = [conv, _bn_node("bn", "c", "n"), ow.node("Relu", ["n"], ["a"]), ow.node("Add", ["a", "c"], ["y"])]
    elif variant == "relu before":
        nodes = [conv, ow.node("Relu", ["c"], ["a"]), _bn_node("bn", "a", "y")]
    else:  # the mean is a graph input
        ins.append(ow.value_info("bn_m", ow.FLOAT, [C]))
        nodes = [conv, _bn_node("bn", "c", "y")]
    return params, w, ow.model(nodes, inits, ins, outs, opset=17)


NO_FOLD = ("second reader", "relu before", "input mean")


def _no_fold_inputs(variant, mean):
    x = np.random.default_rng(12).standard_normal((2, 32, 14, 14)).astype(F32)
    return {"x": x} | ({"bn_m": mean} if variant == "input mean" else {})


@pytest.mark.parametrize("variant", NO_FOLD)
def test_no_fold(rt, ctx, variant):
    from rten_b200.model import Model
    (scale, beta, mean, var), w, data = _conv_bn_graph(variant)
    m = Model(ctx, data)
    assert "BatchNormalization" in m.node_ops, m.node_ops
    inputs = _no_fold_inputs(variant, mean)
    got = m.run(inputs)[0].numpy()
    # the same graph's Conv (and Relu) alone, then the operator on its output
    c = m.run(inputs, ["c"] if variant != "relu before" else ["a"])[0].numpy()
    bn = ref.batch_norm(c, scale, beta, mean, var, 1e-5)
    want = (np.maximum(bn, F32(0)) + c).astype(F32) if variant == "second reader" else bn
    gc.assert_bit_exact(got, want, variant)


@pytest.mark.parametrize("attrs, outs, status, msg", [
    (dict(training_mode=1), 1, 6, 'BatchNormalization: error in attribute "training_mode": unsupported value'),
    (dict(spatial=0), 1, 6, 'BatchNormalization: error in attribute "spatial": unsupported value'),
    (dict(), 2, 7, "unsupported output: running_mean"),
], ids=["training_mode", "spatial", "running_mean"])
def test_load_errors(rt, ctx, attrs, outs, status, msg):
    from rten_b200 import OpError
    from rten_b200.model import Model
    r = np.random.default_rng(1)
    _, inits = _bn_params(r, 4, "bn")
    names = ["y", "rm"][:outs]
    node = ow.node("BatchNormalization", ["x"] + [f"bn_{k}" for k in ("s", "b", "m", "v")], names, **attrs)
    data = ow.model([node], inits, [ow.value_info("x", ow.FLOAT, [1, 4, 2, 2])], [_out(n) for n in names],
                    opset=14)
    with pytest.raises(OpError) as e:
        Model(ctx, data)
    assert msg in str(e.value) and e.value.status == status  # RTEN_ERR_UNSUPPORTED_VALUE / _OUTPUT


def test_momentum_is_read_and_ignored(rt, ctx):
    from rten_b200.model import Model
    r = np.random.default_rng(2)
    (scale, beta, mean, var), inits = _bn_params(r, 4, "bn")
    data = ow.model([_bn_node("bn", "x", "y", momentum=0.9)], inits, [ow.value_info("x", ow.FLOAT, [3, 4])],
                    [_out("y")], opset=14)
    x = r.standard_normal((3, 4)).astype(F32)
    gc.assert_bit_exact(Model(ctx, data).run({"x": x})[0].numpy(), ref.batch_norm(x, scale, beta, mean, var), "momentum")


# ---- DenseNet-121 -------------------------------------------------------------------------------------------------------
def densenet121(seed=0, growth=32, blocks=(6, 12, 24, 16), init=64, bn_size=4, classes=1000):
    """torchvision's densenet121 as ONNX nodes with every BatchNormalization unfolded, seeded weights: (model bytes,
    {name: array} of the initialisers)"""
    r = np.random.default_rng(seed)
    nodes, params = [], {}

    def conv(x, y, cin, cout, k, stride=1, pad=0):
        params[y + "_w"] = (r.standard_normal((cout, cin, k, k)) * np.sqrt(2.0 / (cin * k * k))).astype(F32)
        nodes.append(ow.node("Conv", [x, y + "_w"], [y], kernel_shape=[k, k], strides=[stride] * 2, pads=[pad] * 4))

    def bn_relu(x, y, C, relu=True):
        params[y + "_s"] = r.uniform(0.5, 1.5, C).astype(F32)
        params[y + "_b"] = r.uniform(-0.2, 0.2, C).astype(F32)
        params[y + "_m"] = r.uniform(-0.2, 0.2, C).astype(F32)
        params[y + "_v"] = r.uniform(0.5, 2, C).astype(F32)
        out = y + "_bn" if relu else y
        nodes.append(ow.node("BatchNormalization", [x] + [y + k for k in ("_s", "_b", "_m", "_v")], [out], epsilon=1e-5, momentum=0.9))
        if relu:
            nodes.append(ow.node("Relu", [out], [y]))

    conv("x", "conv0", 3, init, 7, 2, 3)
    bn_relu("conv0", "relu0", init)
    nodes.append(ow.node("MaxPool", ["relu0"], ["pool0"], kernel_shape=[3, 3], strides=[2, 2], pads=[1] * 4))
    feats, C = ["pool0"], init
    for bi, n in enumerate(blocks):
        for li in range(n):
            t = f"b{bi}l{li}"
            src = feats[0]
            if len(feats) > 1:
                src = t + "_cat"
                nodes.append(ow.node("Concat", list(feats), [src], axis=1))
            bn_relu(src, t + "_a1", C + li * growth)
            conv(t + "_a1", t + "_c1", C + li * growth, bn_size * growth, 1)
            bn_relu(t + "_c1", t + "_a2", bn_size * growth)
            conv(t + "_a2", t + "_c2", bn_size * growth, growth, 3, 1, 1)
            feats.append(t + "_c2")
        C += n * growth
        nodes.append(ow.node("Concat", list(feats), [f"b{bi}_out"], axis=1))
        if bi < len(blocks) - 1:
            bn_relu(f"b{bi}_out", f"t{bi}_a", C)
            conv(f"t{bi}_a", f"t{bi}_c", C, C // 2, 1)
            nodes.append(ow.node("AveragePool", [f"t{bi}_c"], [f"t{bi}_p"], kernel_shape=[2, 2], strides=[2, 2]))
            C //= 2
            feats = [f"t{bi}_p"]
    bn_relu(f"b{len(blocks) - 1}_out", "norm5", C)
    params["fc_w"] = (r.standard_normal((classes, C)) / np.sqrt(C)).astype(F32)
    params["fc_b"] = (0.01 * r.standard_normal(classes)).astype(F32)
    nodes += [ow.node("GlobalAveragePool", ["norm5"], ["gap"]), ow.node("Flatten", ["gap"], ["flat"], axis=1),
              ow.node("Gemm", ["flat", "fc_w", "fc_b"], ["logits"], transB=1)]
    data = ow.model(nodes, [ow.tensor(k, v) for k, v in params.items()], [ow.value_info("x", ow.FLOAT, [None, 3, 224, 224])],
                    [_out("logits")], opset=17)
    return data, params


def densenet121_torch_params(params, dtype=None, device="cpu", channels_last=False):
    """densenet121's weights as torch tensors on `device` (float64 unless told otherwise), once per model"""
    import torch
    P = {k: torch.from_numpy(v).to(device=device, dtype=dtype or torch.float64) for k, v in params.items()}
    if channels_last:
        P = {k: v.contiguous(memory_format=torch.channels_last) if v.ndim == 4 else v for k, v in P.items()}
    return P


def densenet121_torch(P, x, blocks=(6, 12, 24, 16)):
    """the forward of the same weights with torch's functional ops: P from densenet121_torch_params, x a numpy array
    (taken in P's dtype and device) or a torch tensor"""
    import torch
    import torch.nn.functional as F
    ref_w = P["conv0_w"]

    def bn_relu(v, y, relu=True):
        v = F.batch_norm(v, P[y + "_m"], P[y + "_v"], P[y + "_s"], P[y + "_b"], False, 0.0, 1e-5)
        return F.relu(v) if relu else v

    x = x if isinstance(x, torch.Tensor) else torch.from_numpy(x).to(device=ref_w.device, dtype=ref_w.dtype)
    h = F.conv2d(x, P["conv0_w"], stride=2, padding=3)
    h = F.max_pool2d(bn_relu(h, "relu0"), 3, 2, 1)
    feats = [h]
    for bi, n in enumerate(blocks):
        for li in range(n):
            t = f"b{bi}l{li}"
            a = bn_relu(torch.cat(feats, 1), t + "_a1")
            a = bn_relu(F.conv2d(a, P[t + "_c1_w"]), t + "_a2")
            feats.append(F.conv2d(a, P[t + "_c2_w"], padding=1))
        h = torch.cat(feats, 1)
        if bi < len(blocks) - 1:
            h = F.avg_pool2d(F.conv2d(bn_relu(h, f"t{bi}_a"), P[f"t{bi}_c_w"]), 2, 2)
            feats = [h]
    h = bn_relu(h, "norm5").mean((2, 3))
    y = h @ P["fc_w"].T + P["fc_b"]
    return y.numpy() if y.device.type == "cpu" else y


@pytest.mark.parametrize("tf32, tol", [(False, 1e-4), (True, 1e-2)], ids=["3xtf32", "tf32"])
def test_densenet121(rt, tf32, tol):
    from rten_b200.model import Model
    ctx = gc.new_ctx(rt, tf32=tf32)
    data, params = densenet121()
    m = Model(ctx, data)
    # conv0 and every layer's 1x1 convolution take their BatchNormalization; the rest run standalone with the Relu
    assert m.node_ops.count("BatchNormalization") == 121 - 59, m.node_ops.count("BatchNormalization")
    assert "Relu" not in m.node_ops
    x = np.random.default_rng(7).standard_normal((2, 3, 224, 224)).astype(F32)
    want = densenet121_torch(densenet121_torch_params(params), x)
    got = m.run({"x": ctx.to_device(x, channels_last=True)})[0].numpy()
    err = float(np.abs(got - want).max() / np.abs(want).max())
    assert got.shape == want.shape and err <= tol, f"DenseNet-121 logits: {err:.3e} of the largest |logit|"
