"""`pytest -m gpu`: Sigmoid, Silu, HardSigmoid and HardSwish -- the standalone operators and the activations fused into
the convolution epilogues.

  * the four operators bit-exact against oracle/activations.py over arange(-6, 6, 0.001), special values and denormals,
    in NCHW, channels-last and a width-sliced view, in place, one launch per dense call, under CUDA-graph replay;
  * rten_b200_conv2d_act on every convolution path (implicit GEMM, explicit im2col, small-channel stem, NCHW output,
    depthwise k3 / k5, s1 / s2, dilated, 1x1 on a 1x1 map), with and without bias, in both f32 modes, with the same
    launch plan pinned on both sides: bit-identical to conv2d followed by the standalone operator;
  * the epilogue variants (default, RTEN_B200_NO_PLAIN, RTEN_B200_NO_FAST) give the same bits for every new code;
  * unknown activation kinds, and the new kinds on conv2d_ex and conv_integer_ex, are refused;
  * EfficientNet- and MobileNetV3-style block models through the executor: SiluFusion in both Mul operand orders, a
    Sigmoid with a second consumer left alone, Conv + activation fused, Clip not fused -- equal to the op-by-op calls."""
import re

import numpy as np
import pytest

import gpu_checks as gc

pytestmark = pytest.mark.gpu

F32 = np.float32
SIXTH = F32(1.0) / F32(6.0)


@pytest.fixture(scope="module")
def rt():
    import rten_b200
    from rten_b200 import _lib
    _lib.load()
    return rten_b200


@pytest.fixture(scope="module")
def oa(oracle):
    from oracle import activations
    return activations


def _ops(rt):
    """(name, standalone op, oracle function, conv activation) of every new activation"""
    return [
        ("sigmoid", rt.Sigmoid(), lambda a, x: a.sigmoid(x), rt.ACT_SIGMOID),
        ("silu", rt.Silu(), lambda a, x: a.silu(x), rt.ACT_SILU),
        ("hard_sigmoid", rt.HardSigmoid(), lambda a, x: a.hard_sigmoid(x), (rt.ACT_HARD_SIGMOID, 0.2, 0.5)),
        ("hard_sigmoid_sixth", rt.HardSigmoid(SIXTH, 0.5), lambda a, x: a.hard_sigmoid(x, SIXTH, 0.5),
         (rt.ACT_HARD_SIGMOID, float(SIXTH), 0.5)),
        ("hard_swish", rt.HardSwish(), lambda a, x: a.hard_swish(x), rt.ACT_HARD_SWISH),
    ]


def _inputs():
    """the sweep, special values and denormals, padded with wide-range values to a [2, 5, 31, 40] tensor"""
    sweep = np.arange(-6.0, 6.0, 0.001, dtype=F32)
    special = np.array([0.0, -0.0, np.inf, -np.inf, np.nan, -104.0, 104.0, -103.99, 88.7, -88.7, 1e30, -1e30, 3.0, -3.0,
                        -4.0, 4.0, 1e-30, -1e-30], F32)
    denormal = np.array([1, 2, 0x7FFFFF, 0x80000001, 0x80400000, 0x807FFFFF], np.uint32).view(F32)
    flat = np.concatenate([sweep, special, denormal])
    n = 2 * 5 * 31 * 40
    rest = (np.random.default_rng(5).standard_normal(n - flat.size) * 40).astype(F32)
    return np.concatenate([flat, rest]).reshape(2, 5, 31, 40)


def _layouts(ctx, x):
    out = [("nchw", ctx.to_device(x)), ("cl", ctx.to_device(x, channels_last=True))]
    b, c, h, w = x.shape
    wide = ctx.empty((b, c, h, w + 5), x.dtype)
    wide.copy_from(np.concatenate([np.zeros((b, c, h, 2), x.dtype), x, np.zeros((b, c, h, 3), x.dtype)], axis=3))
    out.append(("sliced", wide.view(x.shape, wide.strides, 2)))
    return out


def test_standalone_ops_bit_exact(rt, oa):
    ctx = rt.Context(0)
    x = _inputs()
    for name, op, ref, _ in _ops(rt):
        want = ref(oa, x)
        for lay, xd in _layouts(ctx, x):
            gc.assert_bit_exact(op.run(ctx, xd).numpy(), want, f"{name} on {lay}")
        # in place, channels-last: the output is the input's buffer and keeps its strides
        xd = ctx.to_device(x, channels_last=True)
        y = op.run(ctx, xd, in_place=True)
        assert y.ptr == xd.ptr and y.strides == xd.strides
        gc.assert_bit_exact(xd.numpy(), want, f"{name} in place")
        # an odd length and an unaligned start: the scalar tail loop
        xs = ctx.to_device(x.reshape(-1)[:1001])
        gc.assert_bit_exact(op.run(ctx, xs.view((999,), (1,), 1)).numpy(), want.reshape(-1)[1:1000], f"{name} unaligned")


def test_one_launch_and_graph_replay(rt, oa):
    ctx = rt.Context(0)
    x = _inputs()
    xd = ctx.to_device(x, channels_last=True)
    for name, op, ref, _ in _ops(rt):
        op.run(ctx, xd)  # (warm: allocations)
        n0 = ctx.launches
        y = op.run(ctx, xd)
        assert ctx.launches - n0 == 1, f"{name}: {ctx.launches - n0} launches"
        assert y.strides == xd.strides
        out = ctx.empty(x.shape, F32, xd.strides)
        ctx.graph_begin()
        _Into(op).run(ctx, xd, out)
        g = ctx.graph_end()
        for rep in range(2):
            out.copy_from(np.full(x.shape, np.nan, F32))
            g.launch()
            ctx.sync()
            gc.assert_bit_exact(out.numpy(), ref(oa, x), f"{name} graph replay {rep}")


class _Into:
    """op.run writing into a given output (the capture needs a fixed destination)"""

    def __init__(self, op):
        self.op = op

    def run(self, ctx, x, out):
        from rten_b200.ops import _Args
        import ctypes as C
        A = _Args(ctx)
        o = A.out(out)
        ctx.check(self.op._call(ctx, A.t(x), C.byref(o)))
        return A.wrap(o, out)


# (name, x shape, w shape, Conv kwargs, layouts): one case per convolution path
CONV_CASES = [
    ("implicit_3x3", (2, 64, 14, 14), (96, 64, 3, 3), dict(padding=(1, 1, 1, 1)), ("cl",)),
    ("expand_1x1_n256", (2, 32, 14, 14), (256, 32, 1, 1), dict(), ("cl",)),
    ("explicit_im2col_c17", (2, 17, 15, 15), (40, 17, 3, 3), dict(padding=(1, 1, 1, 1)), ("cl", "nchw")),
    ("smallc_stem_s2", (2, 3, 32, 32), (16, 3, 3, 3), dict(padding=(1, 1, 1, 1), strides=(2, 2)), ("cl", "nchw")),
    ("depthwise_k3s1", (2, 48, 13, 13), (48, 1, 3, 3), dict(groups=48, padding=(1, 1, 1, 1)), ("cl", "nchw")),
    ("depthwise_k5s2", (2, 40, 15, 15), (40, 1, 5, 5), dict(groups=40, padding=(2, 2, 2, 2), strides=(2, 2)), ("cl", "nchw")),
    ("depthwise_k3_dil2", (2, 24, 12, 12), (24, 1, 3, 3), dict(groups=24, padding=(2, 2, 2, 2), dilations=(2, 2)), ("cl",)),
    ("se_1x1_on_1x1", (4, 64, 1, 1), (16, 64, 1, 1), dict(), ("cl", "nchw")),
    ("se_1x1_on_1x1_expand", (4, 16, 1, 1), (64, 16, 1, 1), dict(), ("cl", "nchw")),
]


@pytest.mark.parametrize("case", CONV_CASES, ids=[c[0] for c in CONV_CASES])
def test_conv2d_act_equals_conv_then_op(rt, oracle, case):
    name, xs, ws, kw, layouts = case
    r = oracle.XorShiftRng(sum(map(ord, name)))
    x, w, b = r.uniform(xs, -4.0, 4.0), r.uniform(ws, -1.0, 1.0) / F32(np.sqrt(np.prod(ws[1:]))), r.uniform(ws[:1], -2.0, 2.0)
    for tf32 in (False, True):
        ctx = gc.new_ctx(rt, tf32=tf32)
        plain = rt.Conv(**kw)
        pk = plain.prepack(ctx, 1, w)
        for lay in layouts:
            xd = ctx.to_device(x, channels_last=lay == "cl")
            for bias in (b, None):
                # the same plan on both sides: 64-column tiles (umma_gemm_kernel), then 128 (umma_wide_kernel)
                for bn in (64, 128):
                    with gc.forced(bn, strict=False):
                        y = plain.run(ctx, xd, w, bias, packed_w=pk)
                        for aname, op, _, act in _ops(rt):
                            got = rt.Conv(**kw, activation=act).run(ctx, xd, w, bias, packed_w=pk).numpy()
                            want = op.run(ctx, y).numpy()
                            gc.assert_bit_exact(got, want, f"{name} {lay} bias={bias is not None} bn={bn} "
                                                           f"{'TF32' if tf32 else '3xTF32'}: conv2d_act({aname})")


def test_residual_then_activation(rt, oracle):
    """residual add before the activation; an NCHW (not pixel-contiguous) output refuses it, as Gelu does"""
    r = oracle.XorShiftRng(3)
    x, w, b = r.uniform((2, 32, 10, 10), -2, 2), r.uniform((32, 32, 3, 3), -0.2, 0.2), r.uniform((32,))
    res = r.uniform((2, 32, 10, 10), -2, 2)
    ctx = rt.Context(0)
    xd, rd = ctx.to_device(x, channels_last=True), ctx.to_device(res, channels_last=True)
    y = rt.Conv(padding=(1, 1, 1, 1), activation=rt.ACT_NONE).run(ctx, xd, w, b, residual=rd)
    for aname, op, _, act in _ops(rt):
        got = rt.Conv(padding=(1, 1, 1, 1), activation=act).run(ctx, xd, w, b, residual=rd).numpy()
        gc.assert_bit_exact(got, op.run(ctx, y).numpy(), f"conv + residual + {aname}")
    x17 = r.uniform((2, 17, 9, 9))
    with pytest.raises(rt.OpError) as e:
        rt.Conv(activation=rt.ACT_SILU).run(ctx, ctx.to_device(x17), r.uniform((8, 17, 1, 1)), residual=r.uniform((2, 8, 9, 9)))
    assert e.value.kind == "UnsupportedValue"


_PLAN_LINE = re.compile(r"\[umma_gemm\] [^\n]*?\bepi=(\w+)")
_KNOBS = {"default": {}, "no_plain": {"RTEN_B200_NO_PLAIN": "1"}, "no_fast": {"RTEN_B200_NO_FAST": "1"}}
_ENV_KEYS = ("RTEN_B200_NO_PLAIN", "RTEN_B200_NO_FAST", "RTEN_B200_NO_WIDE") + gc.FORCE_KEYS


def test_epilogue_variants_agree(rt, oracle):
    """A 1x1 convolution + bias + each new code on umma_gemm_kernel: PlainF32Gelu, FastGelu and Generic (the variants
    with the out-of-line activation call, and the rolled generic loop) give the same bits."""
    r = oracle.XorShiftRng(11)
    x, w, b = r.uniform((8, 64, 28, 28), -3, 3), r.uniform((128, 64, 1, 1), -0.2, 0.2), r.uniform((128,))
    ctx = gc.new_ctx(rt, tf32=True)
    xd = ctx.to_device(x, channels_last=True)
    for aname, _, _, act in _ops(rt):
        ref = None
        for (knob, env), want in zip(_KNOBS.items(), ("PlainF32Gelu", "FastGelu", "Generic")):
            with gc.switches(**{**dict.fromkeys(_ENV_KEYS), **env, "RTEN_B200_NO_WIDE": "1"}):
                out, err = gc.run_verbose(lambda: rt.Conv(activation=act).run(ctx, xd, w, b).numpy())
            epis = _PLAN_LINE.findall(err)
            assert epis and all(v == want for v in epis), f"{aname} ({knob}): ran {epis}, expected {want}"
            if ref is None:
                ref = out
            else:
                gc.assert_bit_exact(out, ref, f"{aname}: {want} vs PlainF32Gelu")


def test_errors(rt, oracle):
    import ctypes as C
    from rten_b200.ops import _Args, _conv_params
    ctx = rt.Context(0)
    r = oracle.XorShiftRng(1)
    x, w = r.uniform((1, 8, 6, 6)), r.uniform((8, 8, 1, 1))
    for kind in (-1, 8, 100):
        with pytest.raises(rt.OpError) as e:
            rt.Conv(activation=kind).run(ctx, x, w)
        assert e.value.kind == "InvalidValue", kind
    # conv2d_ex keeps the codes 0-3: the new kinds go through conv2d_act
    for code in (4, 5, 6, 7, 8, -1):
        A = _Args(ctx)
        o = A.out(None)
        p = _conv_params((0, 0, 0, 0), 1, (1, 1), (1, 1))
        st = ctx.lib.rten_b200_conv2d_ex(ctx.handle, A.t(x), A.t(w), None, None, C.byref(p), None, code, C.byref(o))
        assert st == 5, f"conv2d_ex activation {code}: status {st}"
    xq, wq = r.u8((1, 8, 6, 6)), r.i8((8, 8, 1, 1))
    for act in (rt.ACT_SIGMOID, rt.ACT_SILU, rt.ACT_HARD_SIGMOID, rt.ACT_HARD_SWISH):
        with pytest.raises(rt.OpError) as e:
            rt.ConvIntegerToFloat(activation=act).run(ctx, xq, wq, np.uint8(3), None, np.float32(0.01))
        assert e.value.kind == "UnsupportedValue"


# ---- executor ------------------------------------------------------------------------------------------------------
def _graph(W, nodes, consts, x_shape, y_shape):
    onnx_nodes = [W.node(op, ins, outs, **attrs) for op, ins, outs, attrs in nodes]
    inits = [W.tensor(k, v) for k, v in consts.items()]
    return W.model(onnx_nodes, inits, [W.value_info("x", 1, x_shape)], [W.value_info("y", 1, y_shape)])


def _conv_node(x, w, b, out, **attrs):
    return ("Conv", [x, w, b], [out], attrs)


def _op_by_op(rt, ctx, nodes, consts, x, silu_muls):
    """The graph node by node through the ABI, with Mul(x, Sigmoid(x)) as Silu(x) where the executor must fuse it
    (`silu_muls`: their outputs)"""
    v = {"x": x}
    sigmoid_of = {outs[0]: ins[0] for op, ins, outs, _ in nodes if op == "Sigmoid"}
    for op, ins, outs, attrs in nodes:
        a = [v[i] if i in v else consts[i] for i in ins]
        if op == "Conv":
            pads = attrs.get("pads", [0, 0, 0, 0])
            conv = rt.Conv(groups=attrs.get("group", 1), padding=tuple(pads), strides=tuple(attrs.get("strides", (1, 1))))
            y = conv.run(ctx, a[0], a[1], a[2], packed_w=conv.prepack(ctx, 1, a[1]))
        elif op == "Mul" and outs[0] in silu_muls:
            y = rt.Silu().run(ctx, v[sigmoid_of[ins[0]] if ins[0] in sigmoid_of else sigmoid_of[ins[1]]])
        elif op in ("Mul", "Add"):
            y = (rt.Mul() if op == "Mul" else rt.Add()).run(ctx, a[0], a[1])
        elif op == "Sigmoid":
            y = rt.Sigmoid().run(ctx, a[0])
        elif op == "HardSigmoid":
            y = rt.HardSigmoid(attrs.get("alpha", 0.2), attrs.get("beta", 0.5)).run(ctx, a[0])
        elif op == "HardSwish":
            y = rt.HardSwish().run(ctx, a[0])
        elif op == "Relu":
            y = rt.Relu().run(ctx, a[0])
        elif op == "Clip":
            y = rt.Clip().run(ctx, a[0], a[1], a[2])
        elif op == "GlobalAveragePool":
            y = rt.GlobalAveragePool().run(ctx, a[0])
        elif op == "Flatten":
            t = a[0].numpy()
            y = t.reshape(t.shape[0], -1)
        elif op == "Gemm":
            y = rt.Gemm(transpose_b=True).run(ctx, a[0], a[1], a[2])
        else:
            raise AssertionError(op)
        v[outs[0]] = y
    return v["y"].numpy()


def _efficientnet_blocks(u):
    """stem 3x3 + SiLU, MBConv (expand 1x1 + SiLU, depthwise k5 + SiLU, squeeze-excite with SiLU / Sigmoid, projection,
    residual Add), a Sigmoid with a second consumer, head 1x1 + SiLU, pool, Gemm"""
    consts = {"w0": u(32, 8, 3, 3) * F32(0.3), "b0": u(32), "w1": u(48, 32, 1, 1) * F32(0.2), "b1": u(48),
              "wd": u(48, 1, 5, 5) * F32(0.3), "bd": u(48), "ws1": u(12, 48, 1, 1) * F32(0.3), "bs1": u(12),
              "ws2": u(48, 12, 1, 1) * F32(0.3), "bs2": u(48), "wp": u(32, 48, 1, 1) * F32(0.2), "bp": u(32),
              "wh": u(64, 32, 1, 1) * F32(0.2), "bh": u(64), "fw": u(10, 64), "fb": u(10)}
    nodes = [
        _conv_node("x", "w0", "b0", "c0", kernel_shape=[3, 3], pads=[1, 1, 1, 1]),
        ("Sigmoid", ["c0"], ["s0"], {}), ("Mul", ["c0", "s0"], ["a0"], {}),            # Mul(x, Sigmoid(x))
        _conv_node("a0", "w1", "b1", "c1", kernel_shape=[1, 1]),
        ("Sigmoid", ["c1"], ["s1"], {}), ("Mul", ["s1", "c1"], ["a1"], {}),            # Mul(Sigmoid(x), x)
        _conv_node("a1", "wd", "bd", "d1", kernel_shape=[5, 5], pads=[2, 2, 2, 2], group=48),
        ("Sigmoid", ["d1"], ["sd"], {}), ("Mul", ["d1", "sd"], ["a2"], {}),
        ("GlobalAveragePool", ["a2"], ["g"], {}),
        _conv_node("g", "ws1", "bs1", "e1", kernel_shape=[1, 1]),
        ("Sigmoid", ["e1"], ["se"], {}), ("Mul", ["se", "e1"], ["e1a"], {}),
        _conv_node("e1a", "ws2", "bs2", "e2", kernel_shape=[1, 1]),
        ("Sigmoid", ["e2"], ["gate"], {}),                                             # Conv + Sigmoid
        ("Mul", ["a2", "gate"], ["a3"], {}),                                           # squeeze-excite scale
        _conv_node("a3", "wp", "bp", "p", kernel_shape=[1, 1]),
        ("Add", ["p", "a0"], ["res"], {}),
        ("Sigmoid", ["res"], ["sr"], {}), ("Mul", ["res", "sr"], ["m"], {}),           # sr has a second consumer:
        ("Add", ["m", "sr"], ["h0"], {}),                                              # no fusion
        _conv_node("h0", "wh", "bh", "hc", kernel_shape=[1, 1]),
        ("Sigmoid", ["hc"], ["sh"], {}), ("Mul", ["hc", "sh"], ["ha"], {}),
        ("GlobalAveragePool", ["ha"], ["gp"], {}), ("Flatten", ["gp"], ["f"], {}), ("Gemm", ["f", "fw", "fb"], ["y"], dict(transB=1)),
    ]
    silu_muls = {"a0", "a1", "a2", "e1a", "ha"}
    fused = ["Conv", "Conv", "Conv", "GlobalAveragePool", "Conv", "Conv", "Mul", "Conv", "Add", "Sigmoid", "Mul", "Add",
             "Conv", "GlobalAveragePool", "Flatten", "Gemm"]
    return nodes, consts, silu_muls, fused


def _mobilenet_v3_blocks(u):
    """stem 3x3 s2 + HardSwish, expand 1x1 + Relu, depthwise k3 + HardSwish, squeeze-excite with Relu and
    HardSigmoid(1/6, 0.5), projection, residual Add, Clip (not fused), Mul(Sigmoid(x), x) in both orders, a Sigmoid with
    a second consumer, a default HardSigmoid and a HardSwish after an Add, head 1x1 + HardSwish, pool, Gemm"""
    consts = {"w0": u(16, 8, 3, 3) * F32(0.3), "b0": u(16), "w1": u(48, 16, 1, 1) * F32(0.3), "b1": u(48),
              "wd": u(48, 1, 3, 3) * F32(0.4), "bd": u(48), "ws1": u(16, 48, 1, 1) * F32(0.3), "bs1": u(16),
              "ws2": u(48, 16, 1, 1) * F32(0.3), "bs2": u(48), "wp": u(16, 48, 1, 1) * F32(0.2), "bp": u(16),
              "wq": u(16, 16, 1, 1) * F32(0.3), "bq": u(16), "wh": u(40, 16, 1, 1) * F32(0.3), "bh": u(40),
              "fw": u(10, 40), "fb": u(10), "zero": np.array(0.0, F32), "six": np.array(6.0, F32)}
    nodes = [
        _conv_node("x", "w0", "b0", "c0", kernel_shape=[3, 3], pads=[1, 1, 1, 1], strides=[2, 2]),
        ("HardSwish", ["c0"], ["a0"], {}),
        _conv_node("a0", "w1", "b1", "c1", kernel_shape=[1, 1]), ("Relu", ["c1"], ["a1"], {}),
        _conv_node("a1", "wd", "bd", "d1", kernel_shape=[3, 3], pads=[1, 1, 1, 1], group=48),
        ("HardSwish", ["d1"], ["a2"], {}),
        ("GlobalAveragePool", ["a2"], ["g"], {}),
        _conv_node("g", "ws1", "bs1", "e1", kernel_shape=[1, 1]), ("Relu", ["e1"], ["e1a"], {}),
        _conv_node("e1a", "ws2", "bs2", "e2", kernel_shape=[1, 1]),
        ("HardSigmoid", ["e2"], ["gate"], dict(alpha=float(SIXTH), beta=0.5)),
        ("Mul", ["a2", "gate"], ["a3"], {}),
        _conv_node("a3", "wp", "bp", "p", kernel_shape=[1, 1]),
        ("Add", ["p", "a0"], ["res"], {}),
        _conv_node("res", "wq", "bq", "q", kernel_shape=[1, 1]), ("Clip", ["q", "zero", "six"], ["qc"], {}),
        ("Sigmoid", ["qc"], ["s1"], {}), ("Mul", ["s1", "qc"], ["m1"], {}),             # Mul(Sigmoid(x), x) -> Silu
        ("Sigmoid", ["m1"], ["s2"], {}), ("Mul", ["m1", "s2"], ["m2"], {}),             # Mul(x, Sigmoid(x)) -> Silu
        ("Sigmoid", ["m2"], ["s3"], {}), ("Mul", ["s3", "m2"], ["m3"], {}),             # s3 also feeds the Add:
        ("Add", ["m3", "s3"], ["h0"], {}),                                              # no fusion
        ("HardSigmoid", ["h0"], ["h1"], {}), ("Add", ["h1", "res"], ["h2"], {}), ("HardSwish", ["h2"], ["h3"], {}),
        _conv_node("h3", "wh", "bh", "hc", kernel_shape=[1, 1]), ("HardSwish", ["hc"], ["ha"], {}),
        ("GlobalAveragePool", ["ha"], ["gp"], {}), ("Flatten", ["gp"], ["f"], {}), ("Gemm", ["f", "fw", "fb"], ["y"], dict(transB=1)),
    ]
    silu_muls = {"m1", "m2"}
    fused = ["Conv", "Conv", "Conv", "GlobalAveragePool", "Conv", "Conv", "Mul", "Conv", "Add", "Conv", "Clip", "Silu",
             "Silu", "Sigmoid", "Mul", "Add", "HardSigmoid", "Add", "HardSwish", "Conv", "GlobalAveragePool", "Flatten",
             "Gemm"]
    return nodes, consts, silu_muls, fused


@pytest.mark.parametrize("build", [_efficientnet_blocks, _mobilenet_v3_blocks], ids=["efficientnet", "mobilenet_v3"])
def test_block_model(rt, oracle, build):
    import onnx_writer
    from rten_b200.model import Model
    r = oracle.XorShiftRng(59)
    nodes, consts, silu_muls, fused = build(lambda *s: r.uniform(s, -1.0, 1.0))
    x = r.uniform((2, 8, 12, 12), -3.0, 3.0)
    data = _graph(onnx_writer, nodes, consts, x.shape, (2, 10))
    for tf32 in (False, True):
        ctx = gc.new_ctx(rt, tf32=tf32)
        m = Model(ctx, data)
        assert m.node_ops == fused, m.node_ops
        for cl in (False, True):
            xd = ctx.to_device(x, channels_last=cl)
            got = m.run({"x": xd}, ["y"])[0].numpy()
            want = _op_by_op(rt, ctx, nodes, consts, xd, silu_muls)
            gc.assert_bit_exact(got, want, f"{build.__name__} (cl={cl}, {'TF32' if tf32 else '3xTF32'}) vs op by op")
