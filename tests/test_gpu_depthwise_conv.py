"""`pytest -m gpu`: depthwise Conv / ConvInteger (groups = in channels = out channels) on the direct depthwise kernel,
and Clip.  Everything is bit-exact against oracle/depthwise.py (the reference's depthwise arithmetic) unless stated:

  * the reference's known answer through the C ABI;
  * the sweep of tests/depthwise_sweep.py in NCHW, channels-last, a width-sliced view and 1-D NCW / NWC, in both f32
    modes (identical bits), prepacked and per-call weights; conv2d_ex with a residual and activations 0-3 against the
    oracle followed by rten_b200_add and rten_b200_relu / rten_b200_gelu;
  * ConvInteger, ConvIntegerToFloat and conv_integer_ex (scale_b, bias, residual, Relu, out_range) for every signedness
    pair, with padded cases whose x zero point is not 128 (u8) / 0 (i8), where the GEMM path's padding would differ;
  * one launch per device-resident call; CUDA-graph replay; the benched MobileNetV2 112x112x96 s2 b32 layer;
  * Clip through the ABI (NaN, +-inf, +-0.0, absent bounds, i32, in place), and a MobileNetV2-style ONNX model (1x1
    Conv, Clip, depthwise s2, an s1 block with Add, GlobalAveragePool, Flatten, Gemm; Clip in input and attribute forms
    with absent bounds) equal to the op-by-op ABI calls."""
import numpy as np
import pytest

import depthwise_sweep as sw
import gpu_checks as gc

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def rt():
    import rten_b200
    from rten_b200 import _lib
    _lib.load()
    return rten_b200


@pytest.fixture(scope="module")
def oracle():
    from oracle import oracle as o
    return o


@pytest.fixture(scope="module")
def dw():
    from oracle import depthwise as d
    return d


def _conv(rt, case, cls=None, **kw):
    return (cls or rt.Conv)(groups=sw.shapes(case)[1][0], **sw.op_args(case), **kw)


def _layouts(ctx, x):
    """(name, device tensor) of x in NCHW / NCW, channels-last / NWC and (4-D) a width-sliced NCHW view"""
    out = [("nchw", ctx.to_device(x))]
    if x.ndim == 4:
        out.append(("cl", ctx.to_device(x, channels_last=True)))
        b, c, h, w = x.shape
        wide = ctx.empty((b, c, h, w + 5), x.dtype)
        wide.copy_from(np.concatenate([np.zeros((b, c, h, 2), x.dtype), x, np.zeros((b, c, h, 3), x.dtype)], axis=3))
        out.append(("sliced", wide.view(x.shape, wide.strides, 2)))
    else:
        b, c, w = x.shape
        t = ctx.empty(x.shape, x.dtype, (w * c, 1, c))
        t.copy_from(x)
        out.append(("nwc", t))
    return out


def test_known_answer(rt):
    # src/ops/conv.rs:990-1030 (test_conv_depthwise)
    x = np.array([0.5946, 0.8249, 0.0448, 0.9552, 0.2041, 0.2501, 0.2693, 0.1007, 1.5202, 1.5592, 0.9939, 1.7475],
                 np.float32).reshape(1, 3, 2, 2)
    w = np.array([-0.0862, -0.4111, 0.0813, 0.4993, -0.4641, 0.1715, -0.0532, -0.2429, -0.4325, 0.4273, 0.4180, 0.4338],
                 np.float32).reshape(3, 1, 2, 2)
    bias = np.array([0.1, 0.2, 0.3], np.float32)
    want = np.array([0.09020272 + 0.1, -0.09061745 + 0.2, 1.1822754 + 0.3], np.float32).reshape(1, 3, 1, 1)
    ctx = rt.Context(0)
    got = rt.Conv(groups=3).run(ctx, x, w, bias).numpy()
    assert np.allclose(got, want, atol=1e-4, rtol=0)
    from oracle import depthwise
    gc.assert_bit_exact(got, depthwise.depthwise_conv(x, w, bias), "known answer vs oracle")


@pytest.mark.parametrize("case", sw.SWEEP, ids=sw.IDS)
def test_f32_sweep(rt, oracle, dw, case):
    x, w, b = sw.f32_data(oracle, case)
    want = dw.depthwise_conv(x, w, b, **sw.op_args(case))
    want_nb = dw.depthwise_conv(x, w, None, **sw.op_args(case))
    op = _conv(rt, case)
    for tf32 in (False, True):
        ctx = gc.new_ctx(rt, tf32=tf32)
        pk = op.prepack(ctx, 1, ctx.to_device(w)) if x.ndim == 4 else None
        for name, xd in _layouts(ctx, x):
            what = f"{case[0]} {name} {'TF32' if tf32 else '3xTF32'}"
            y = op.run(ctx, xd, w, b)
            if name in ("cl", "nwc") and x.shape[1] > 1:
                assert y.strides[1] == 1, f"{what}: channels-last in must give channels-last out, got {y.strides}"
            gc.assert_bit_exact(y.numpy(), want, what)
            gc.assert_bit_exact(op.run(ctx, xd, w).numpy(), want_nb, what + " no bias")
            if pk is not None:
                gc.assert_bit_exact(op.run(ctx, xd, w, b, packed_w=pk).numpy(), want, what + " prepacked")


@pytest.mark.parametrize("case", [c for c in sw.SWEEP if c[0] in ("k3s1p1_c17", "k5s2_same_c17", "k3s2_c96_nopad", "1d_k5_c17")],
                         ids=lambda c: c[0])
def test_conv2d_ex_residual_and_activations(rt, oracle, dw, case):
    ctx = rt.Context(0)
    x, w, b = sw.f32_data(oracle, case)
    base = dw.depthwise_conv(x, w, b, **sw.op_args(case))
    res = oracle.XorShiftRng(5).uniform(base.shape, -1.0, 1.0)
    summed = rt.Add().run(ctx, base, res)
    unfused = {0: summed.numpy(), 1: rt.Relu().run(ctx, summed).numpy(), 2: rt.Gelu().run(ctx, summed).numpy(),
               3: rt.Gelu(approximate=True).run(ctx, summed).numpy()}
    for act in range(4):
        op = _conv(rt, case, activation=act)
        for name, xd in _layouts(ctx, x):
            got = op.run(ctx, xd, w, b, residual=res).numpy()
            gc.assert_bit_exact(got, unfused[act], f"{case[0]} {name} act={act}")


PAIRS = [(np.uint8, np.uint8), (np.uint8, np.int8), (np.int8, np.uint8), (np.int8, np.int8)]


def _decode_range(r):
    r = np.asarray(r, np.int32).reshape(-1)
    bits = np.where(r >= 0, r, r ^ np.int32(0x7FFFFFFF)).astype(np.int32)
    return bits.view(np.float32)


@pytest.mark.parametrize("pair", PAIRS, ids=lambda p: f"{np.dtype(p[0]).name}x{np.dtype(p[1]).name}")
@pytest.mark.parametrize("case", sw.SWEEP, ids=sw.IDS)
def test_integer_sweep(rt, dw, case, pair):
    xdt, wdt = pair
    ctx = rt.Context(0)
    x, w = sw.int_data(case, xdt, wdt)
    C = w.shape[0]
    # x zero points: not the GEMM path's pad value (128 for u8, 0 for i8), and that value
    xzs = [np.uint8(37), np.uint8(255), np.uint8(128)] if xdt == np.uint8 else [np.int8(-128), np.int8(12), np.int8(0)]
    wzs = [None, np.array(5 if wdt == np.uint8 else -3, wdt), (np.arange(C) % 200).astype(wdt)]
    g = np.random.default_rng(3)
    scale, scale_b = np.float32(0.0173), np.float32(0.37)
    bias = g.uniform(-1, 1, C).astype(np.float32)
    iop = _conv(rt, case, rt.ConvInteger)
    fop = _conv(rt, case, rt.ConvIntegerToFloat)
    for name, xd in _layouts(ctx, x):
        for xz in xzs:
            for wz in wzs:
                what = f"{case[0]} {name} xz={xz} wz={None if wz is None else wz.reshape(-1)[:2]}"
                acc = dw.depthwise_conv_integer(x, w, xz, wz, **sw.op_args(case))
                gc.assert_bit_exact(iop.run(ctx, xd, w, xz, wz).numpy(), acc, what + " ConvInteger")
                gc.assert_bit_exact(fop.run(ctx, xd, w, xz, wz, scale).numpy(), dw.integer_to_float(acc, scale),
                                    what + " ConvIntegerToFloat")
        # conv_integer_ex: scale_b, bias, residual, Relu and the output range
        xz, wz = xzs[0], wzs[2]
        acc = dw.depthwise_conv_integer(x, w, xz, wz, **sw.op_args(case))
        res = g.uniform(-2, 2, acc.shape).astype(np.float32)
        for act in (0, 1):
            fop.activation = act
            want = dw.integer_to_float(acc, scale, scale_b=scale_b, bias=bias, residual=res, relu=bool(act))
            rng = ctx.to_device(np.zeros((1, 2), np.int32))
            rt.DynamicQuantizeLinear.reset_ranges(ctx, rng)
            got = fop.run(ctx, xd, w, xz, wz, scale, bias=bias, residual=res, scale_b=scale_b, out_range=rng).numpy()
            gc.assert_bit_exact(got, want, f"{case[0]} {name} conv_integer_ex act={act}")
            lo, hi = _decode_range(rng.numpy())
            assert lo == want.min() and hi == want.max(), f"{case[0]} {name}: range ({lo}, {hi}) != ({want.min()}, {want.max()})"
        fop.activation = 0


def test_padded_zero_point_differs_from_gemm_padding(rt, dw):
    """The case the GEMM path got wrong: a padded u8 depthwise ConvInteger with x zero point != 128 gives the
    reference's border values (padding acts as the zero point)."""
    ctx = rt.Context(0)
    x = np.full((1, 2, 3, 3), 10, np.uint8)
    w = np.ones((2, 1, 3, 3), np.uint8)
    got = rt.ConvInteger(groups=2, padding=(1, 1, 1, 1)).run(ctx, x, w, np.uint8(10), None).numpy()
    assert (got == 0).all(), "x == x_zp everywhere: every output, border included, must be 0"
    np.testing.assert_array_equal(got, dw.depthwise_conv_integer(x, w, np.uint8(10), None, padding=(1, 1, 1, 1)))


def test_launch_count(rt, oracle):
    r = oracle.XorShiftRng(9)
    x, w, b = r.uniform((4, 64, 20, 20)), r.uniform((64, 1, 3, 3)), r.uniform((64,))
    op = rt.Conv(groups=64, padding=(1, 1, 1, 1), strides=(2, 2))
    for tf32 in (False, True):
        ctx = gc.new_ctx(rt, tf32=tf32)
        wd, bd = ctx.to_device(w), ctx.to_device(b)
        pk = op.prepack(ctx, 1, wd)
        for cl in (False, True):
            xd = ctx.to_device(x, channels_last=cl)
            for packed in (None, pk):
                op.run(ctx, xd, wd, bd, packed_w=packed)  # (warm: allocations)
                n0 = ctx.launches
                op.run(ctx, xd, wd, bd, packed_w=packed)
                assert ctx.launches - n0 == 1, f"tf32={tf32} cl={cl} packed={packed is not None}: {ctx.launches - n0} launches"
    ctx = rt.Context(0)
    g = np.random.default_rng(1)
    xq = ctx.to_device(g.integers(0, 256, (4, 64, 20, 20)).astype(np.uint8), channels_last=True)
    wq = ctx.to_device(g.integers(-128, 128, (64, 1, 3, 3)).astype(np.int8))
    xz, wz = ctx.to_device(np.array(17, np.uint8)), ctx.to_device(np.arange(64).astype(np.int8))
    sc = ctx.to_device(np.array(0.01, np.float32))
    for fn in (lambda: rt.ConvInteger(groups=64, padding=(1, 1, 1, 1)).run(ctx, xq, wq, xz, wz),
               lambda: rt.ConvIntegerToFloat(groups=64, padding=(1, 1, 1, 1)).run(ctx, xq, wq, xz, wz, sc)):
        fn()
        n0 = ctx.launches
        fn()
        assert ctx.launches - n0 == 1


def test_graph_replay(rt, oracle, dw):
    r = oracle.XorShiftRng(13)
    x, w, b = r.uniform((8, 96, 28, 28)), r.uniform((96, 1, 5, 5)), r.uniform((96,))
    ctx = rt.Context(0)
    xd, wd, bd = ctx.to_device(x, channels_last=True), ctx.to_device(w), ctx.to_device(b)
    op = rt.Conv(groups=96, padding=(2, 2, 2, 2))
    eager = op.run(ctx, xd, wd, bd).numpy()
    out = ctx.empty((8, 96, 28, 28), np.float32, (28 * 28 * 96, 1, 28 * 96, 96))
    ctx.graph_begin()
    op.run(ctx, xd, wd, bd, out=out)
    g = ctx.graph_end()
    for rep in range(2):
        out.copy_from(np.full(out.shape, np.nan, np.float32))
        g.launch()
        ctx.sync()
        gc.assert_bit_exact(out.numpy(), eager, f"graph replay {rep}")
    gc.assert_bit_exact(eager, dw.depthwise_conv(x, w, b, padding=(2, 2, 2, 2)), "eager vs oracle")


def test_benched_mobilenet_v2_layer(rt, oracle, dw):
    """MobileNetV2 112x112x96 k3 s2 p1, b32, channels-last: the layer tools/depthwise_bench.py times."""
    r = oracle.XorShiftRng(21)
    x, w, b = r.uniform((32, 96, 112, 112)), r.uniform((96, 1, 3, 3)), r.uniform((96,))
    want = dw.depthwise_conv(x, w, b, padding=(1, 1, 1, 1), strides=(2, 2))
    for tf32 in (False, True):
        ctx = gc.new_ctx(rt, tf32=tf32)
        got = rt.Conv(groups=96, padding=(1, 1, 1, 1), strides=(2, 2)).run(ctx, ctx.to_device(x, channels_last=True), w, b)
        gc.assert_bit_exact(got.numpy(), want, f"MobileNetV2 112x112x96 s2 b32 {'TF32' if tf32 else '3xTF32'}")


def test_clip_abi(rt, dw):
    ctx = rt.Context(0)
    x = np.array([[np.nan, np.inf, -np.inf, -0.0], [0.0, -1.0, 0.5, 7.0]], np.float32)
    lo, hi = np.float32(0.0), np.float32(6.0)
    for mn, mx in ((lo, hi), (None, hi), (lo, None), (None, None), (np.float32(-0.5), None)):
        got = rt.Clip().run(ctx, x, mn, mx).numpy()
        gc.assert_bit_exact(got, dw.clip(x, mn, mx), f"Clip min={mn} max={mx}")
    # device-resident bounds, in place, on a channels-last tensor
    g = np.random.default_rng(0)
    a = (g.standard_normal((2, 8, 5, 5)) * 8).astype(np.float32)
    ad = ctx.to_device(a, channels_last=True)
    y = rt.Clip().run(ctx, ad, ctx.to_device(np.array(0.0, np.float32)), ctx.to_device(np.array(6.0, np.float32)), in_place=True)
    assert y.ptr == ad.ptr and y.strides == ad.strides
    gc.assert_bit_exact(ad.numpy(), dw.clip(a, lo, hi), "Clip in place")
    xi = np.array([-(2**31), -5, 0, 5, 2**31 - 1], np.int32)
    gc.assert_bit_exact(rt.Clip().run(ctx, xi, np.int32(-2), np.int32(3)).numpy(), dw.clip(xi, np.int32(-2), np.int32(3)), "Clip i32")
    gc.assert_bit_exact(rt.Clip().run(ctx, xi, None, np.int32(3)).numpy(), dw.clip(xi, None, np.int32(3)), "Clip i32 no min")
    with pytest.raises(rt.OpError) as e:
        rt.Clip().run(ctx, x, np.int32(0), None)
    assert e.value.kind == "InvalidValue"


def _mobilenet_block_model(W, consts):
    nodes = [
        W.node("Conv", ["x", "w1", "b1"], ["c1"], kernel_shape=[1, 1]),
        W.node("Clip", ["c1", "zero", "six"], ["r1"]),
        W.node("Conv", ["r1", "wd1", "bd1"], ["d1"], group=32, kernel_shape=[3, 3], pads=[1, 1, 1, 1], strides=[2, 2]),
        W.node("Clip", ["d1"], ["r2"], min=0.0, max=6.0),  # legacy attribute form
        W.node("Conv", ["r2", "w2", "b2"], ["p2"], kernel_shape=[1, 1]),
        W.node("Conv", ["p2", "w3", "b3"], ["c3"], kernel_shape=[1, 1]),
        W.node("Clip", ["c3", "", "six"], ["r3"]),  # absent min
        W.node("Conv", ["r3", "wd2", "bd2"], ["d2"], group=48, kernel_shape=[3, 3], pads=[1, 1, 1, 1]),
        W.node("Clip", ["d2"], ["r4"], max=6.0),  # attribute form, absent min
        W.node("Conv", ["r4", "w4", "b4"], ["p4"], kernel_shape=[1, 1]),
        W.node("Add", ["p2", "p4"], ["s"]),
        W.node("GlobalAveragePool", ["s"], ["gp"]),
        W.node("Flatten", ["gp"], ["f"]),
        W.node("Gemm", ["f", "fw", "fb"], ["y"], transB=1),
    ]
    inits = [W.tensor(k, v) for k, v in consts.items()]
    return W.model(nodes, inits, [W.value_info("x", 1, (2, 16, 12, 12))], [W.value_info("y", 1, (2, 10))])


def test_mobilenet_style_model(rt, oracle):
    import onnx_writer
    from rten_b200.model import Model
    r = oracle.XorShiftRng(41)
    u = lambda *s: r.uniform(s, -1.0, 1.0)  # noqa: E731
    consts = {"w1": u(32, 16, 1, 1) * np.float32(0.5), "b1": u(32), "wd1": u(32, 1, 3, 3), "bd1": u(32),
              "w2": u(24, 32, 1, 1) * np.float32(0.3), "b2": u(24), "w3": u(48, 24, 1, 1) * np.float32(0.3), "b3": u(48),
              "wd2": u(48, 1, 3, 3), "bd2": u(48), "w4": u(24, 48, 1, 1) * np.float32(0.3), "b4": u(24),
              "fw": u(10, 24), "fb": u(10), "zero": np.array(0.0, np.float32), "six": np.array(6.0, np.float32)}
    x = r.uniform((2, 16, 12, 12), -3.0, 3.0)
    for tf32 in (False, True):
        ctx = gc.new_ctx(rt, tf32=tf32)
        m = Model(ctx, _mobilenet_block_model(onnx_writer, consts))
        assert m.node_ops.count("Clip") == 4
        for cl in (False, True):
            xd = ctx.to_device(x, channels_last=cl)
            got = m.run({"x": xd}, ["y"])[0].numpy()

            def conv(t, w, b, **kw):
                op = rt.Conv(**kw)
                return op.run(ctx, t, consts[w], consts[b], packed_w=op.prepack(ctx, 1, consts[w]))

            clip = rt.Clip()
            r1 = clip.run(ctx, conv(xd, "w1", "b1"), consts["zero"], consts["six"])
            r2 = clip.run(ctx, conv(r1, "wd1", "bd1", groups=32, padding=(1, 1, 1, 1), strides=(2, 2)), np.float32(0.0), np.float32(6.0))
            p2 = conv(r2, "w2", "b2")
            r3 = clip.run(ctx, conv(p2, "w3", "b3"), None, consts["six"])
            r4 = clip.run(ctx, conv(r3, "wd2", "bd2", groups=48, padding=(1, 1, 1, 1)), None, np.float32(6.0))
            s = rt.Add().run(ctx, p2, conv(r4, "w4", "b4"))
            gp = rt.GlobalAveragePool().run(ctx, s)
            want = rt.Gemm(transpose_b=True).run(ctx, gp.numpy().reshape(2, 24), consts["fw"], consts["fb"]).numpy()
            gc.assert_bit_exact(got, want, f"MobileNetV2-style model vs op by op (cl={cl}, {'TF32' if tf32 else '3xTF32'})")
