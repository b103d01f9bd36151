"""`pytest -m gpu`: what an onnxruntime-genai int4 decoder needs beyond its layer stack, and the decoder itself.

  * ReduceSum: f32 bit for bit against genai_decoder.reduce_sum_ref (the reference's Sum over each lane, in row-major
    order of the reduced axes) over every axis subset of 1-D to 4-D shapes, keepdims 0 / 1, channels-last and strided
    inputs, lane lengths around the warp / CTA switch (1024) and the CTA stages (4096), misaligned lanes, +-inf, NaN and
    +-3e38; i32 exact with wrap-around; noop_with_empty_axes, a 0-D input, empty inputs, the reference's errors and one
    launch per call;
  * Sub (f32) and i32 Add / Sub / Mul bit for bit against numpy through every broadcast path, in place and strided;
  * shape values on the host: Shape with start / end, Gather of a shape with scalar and vector indices, Cast, and a
    Reshape whose target is Shape -> Gather -> Cast, with no launch for the shape chain;
  * the genai decoder from its file through Model: a prompt with empty past caches, then 8 decode steps fed the previous
    presents and a growing attention_mask.  seqlens_k and total_sequence_length come from the mask subgraph.  Logits and
    presents are bit-identical to the operators called one by one (test_gpu_norms's _decoder_ops for the separate-QKV
    decoder), logits within 2e-4 * max |ref| of the float64 forward, and a step launches exactly two kernels more (the
    ReduceSum and the Sub) than the same decoder fed seqlens_k and total_sequence_length as inputs;
  * ReduceSum, Sub and Shape load only in the default domain."""
import itertools

import numpy as np
import pytest

import genai_decoder as gd
import gpu_checks as gc

pytestmark = pytest.mark.gpu

F32, I32 = np.float32, np.int32


@pytest.fixture(scope="module")
def rt():
    import rten_b200
    from rten_b200 import _lib
    _lib.load()
    return rten_b200


@pytest.fixture(scope="module")
def ctx(rt):
    return rt.Context(0)


def _f32(r, shape):
    return (r.standard_normal(shape) * np.exp2(r.integers(-12, 12, shape))).astype(F32)


def _reduce(rt, ctx, x, axes, keepdims):
    return rt.ReduceSum(axes, keep_dims=bool(keepdims)).run(ctx, x).numpy()


# ---- ReduceSum
@pytest.mark.parametrize("shape", [(70,), (5, 300), (3, 7, 65), (2, 3, 5, 33)])
def test_reduce_sum_every_axis_subset(rt, ctx, shape):
    r = np.random.default_rng(len(shape))
    x = _f32(r, shape)
    xd = ctx.to_device(x)
    nd = len(shape)
    for k in range(nd + 1):
        for axes in itertools.combinations(range(nd), k):
            for keep in (0, 1):
                gc.assert_bit_exact(_reduce(rt, ctx, xd, list(axes), keep), gd.reduce_sum_ref(x, list(axes), keep), f"{shape} {axes} {keep}")
    gc.assert_bit_exact(_reduce(rt, ctx, xd, [-1, 0, -1], 1), gd.reduce_sum_ref(x, [-1, 0], 1), f"{shape} repeated axes")


def test_reduce_sum_strided_and_channels_last(rt, ctx):
    r = np.random.default_rng(7)
    x = _f32(r, (2, 48, 9, 11))
    cl = ctx.to_device(x, channels_last=True)
    big = ctx.to_device(_f32(r, (2, 48, 9, 23)))
    view = big.view((2, 48, 9, 11), (big.strides[0], big.strides[1], big.strides[2], 2), 1)  # every other column, odd base
    xv = big.numpy()[:, :, :, 1::2]
    for axes in ([1], [2, 3], [1, 2, 3], [0, 1], [0, 3], None):
        for keep in (0, 1):
            gc.assert_bit_exact(_reduce(rt, ctx, cl, axes, keep), gd.reduce_sum_ref(x, axes, keep), f"channels-last {axes}")
            gc.assert_bit_exact(_reduce(rt, ctx, view, axes, keep), gd.reduce_sum_ref(xv, axes, keep), f"strided {axes}")


@pytest.mark.parametrize("L", [1, 63, 64, 65, 1023, 1024, 1025, 4095, 4096, 4097, 8197, 100003])
def test_reduce_sum_lane_lengths(rt, ctx, L):
    """the warp kernel up to 1024 elements, the CTA kernel above; contiguous (16-byte loads), misaligned and strided lanes"""
    r = np.random.default_rng(L)
    x = _f32(r, (3, L))
    gc.assert_bit_exact(_reduce(rt, ctx, x, [1], 1), gd.reduce_sum_ref(x, [1], 1), f"L={L} contiguous")
    big = ctx.to_device(_f32(r, (3, L + 1)))
    mis = big.view((3, L), (L + 1, 1), 1)
    gc.assert_bit_exact(_reduce(rt, ctx, mis, [1], 0), gd.reduce_sum_ref(big.numpy()[:, 1:], [1], 0), f"L={L} misaligned")
    xt = np.ascontiguousarray(x.T)  # [L, 3]: lanes down the columns
    gc.assert_bit_exact(_reduce(rt, ctx, xt, [0], 0), gd.reduce_sum_ref(xt, [0], 0), f"L={L} strided")


def test_reduce_sum_special_values(rt, ctx):
    r = np.random.default_rng(9)
    x = _f32(r, (6, 2000))
    x[0, ::7] = 3e38
    x[1, 5] = np.inf
    x[2, 5], x[2, 1999] = np.inf, -np.inf
    x[3, 100] = np.nan
    x[4, :] = -3e38
    x[5, :] = -0.0
    for axes in ([1], [0], None):
        gc.assert_bit_exact(_reduce(rt, ctx, x, axes, 1), gd.reduce_sum_ref(x, axes, 1), f"special {axes}")
    s = x[:, :300]
    gc.assert_bit_exact(_reduce(rt, ctx, s, [1], 1), gd.reduce_sum_ref(s, [1], 1), "special, warp kernel")


def test_reduce_sum_i32_wraps(rt, ctx):
    r = np.random.default_rng(10)
    for shape, axes in (((4, 3000), [1]), ((3000, 4), [0]), ((5, 7, 9), [0, 2]), ((2, 100003), None), ((8, 33), [1])):
        x = r.integers(-2**31, 2**31, shape, dtype=np.int64).astype(I32)
        want = np.sum(x, axis=None if axes is None else tuple(axes), dtype=np.int64, keepdims=True).astype(I32)
        got = _reduce(rt, ctx, x, axes, 1)
        assert got.dtype == I32 and np.array_equal(got, want), (shape, axes)
    mask = np.ones((2, 37), I32)
    assert np.array_equal(_reduce(rt, ctx, mask, [1], 1), [[37], [37]])


def test_reduce_sum_edge_cases_and_errors(rt, ctx):
    gc.assert_bit_exact(_reduce(rt, ctx, np.array(2.5, F32), None, 1), np.array(2.5, F32), "0-D")
    gc.assert_bit_exact(_reduce(rt, ctx, np.array(-0.0, F32), None, 0), np.array(0.0, F32), "0-D -0.0 plus 0")
    e = np.zeros((2, 0, 3), F32)
    gc.assert_bit_exact(_reduce(rt, ctx, e, [1], 1), np.zeros((2, 1, 3), F32), "empty lanes give 0")
    assert _reduce(rt, ctx, e, [0], 0).shape == (0, 3)
    assert np.array_equal(_reduce(rt, ctx, np.zeros((0,), I32), None, 0), np.array(0, I32))
    x = np.arange(6, dtype=F32).reshape(2, 3)
    y = rt.ReduceSum([], noop_with_empty_axes=True).run(ctx, x).numpy()
    gc.assert_bit_exact(y, x, "noop_with_empty_axes")
    for axes, x in (([2], x), ([-3], x), ([0], np.array(1.0, F32))):
        with pytest.raises(rt.OpError) as ei:
            _reduce(rt, ctx, x, axes, 1)
        assert ei.value.kind == "InvalidValue" and "Axis is invalid" in ei.value.msg
    with pytest.raises(rt.OpError) as ei:
        _reduce(rt, ctx, np.zeros((4,), np.int8), None, 1)
    assert ei.value.kind == "UnsupportedType"


def test_reduce_sum_one_launch(rt, ctx):
    r = np.random.default_rng(11)
    for shape, axes, dt in (((64, 300), [1], F32), ((64, 5000), [1], F32), ((5000, 64), [0], F32), ((3, 5, 7, 9), [0, 2], F32),
                            ((64, 300), [1], I32), ((2, 9000), None, I32)):
        x = ctx.to_device(_f32(r, shape) if dt == F32 else r.integers(-100, 100, shape).astype(I32))
        ctx.sync()
        n0 = ctx.launches
        y = rt.ReduceSum(axes).run(ctx, x)
        ctx.sync()
        assert ctx.launches - n0 == 1, (shape, axes, dt)
        del y


# ---- Sub and integer Add / Sub / Mul
BCAST = [((4, 37), (4, 37)), ((4, 37), ()), ((4, 6, 8), (8,)), ((4, 6, 8), (6, 1)), ((3, 1, 5), (1, 4, 1)), ((1,), (2, 3, 3))]


@pytest.mark.parametrize("a_shape,b_shape", BCAST)
def test_sub_and_integer_arithmetic(rt, ctx, a_shape, b_shape):
    r = np.random.default_rng(sum(a_shape) + len(b_shape))
    a, b = _f32(r, a_shape), _f32(r, b_shape)
    gc.assert_bit_exact(rt.Sub().run(ctx, a, b).numpy(), a - b, f"Sub f32 {a_shape} {b_shape}")
    ai = r.integers(-2**31, 2**31, a_shape, dtype=np.int64).astype(I32)
    bi = r.integers(-2**31, 2**31, b_shape, dtype=np.int64).astype(I32)
    with np.errstate(over="ignore"):
        for op, f in ((rt.Add(), np.add), (rt.Sub(), np.subtract), (rt.Mul(), np.multiply)):
            got = op.run(ctx, ai, bi).numpy()
            assert got.dtype == I32 and np.array_equal(got, f(ai, bi)), (type(op).__name__, a_shape, b_shape)


def test_sub_in_place_strided_and_errors(rt, ctx):
    r = np.random.default_rng(12)
    a, b = _f32(r, (6, 40)), _f32(r, (6, 40))
    ad = ctx.to_device(a)
    rt.Sub().run(ctx, ad, b, out=ad)
    gc.assert_bit_exact(ad.numpy(), a - b, "Sub in place")
    t = ctx.to_device(a).permute(1, 0)  # [40, 6] view
    gc.assert_bit_exact(rt.Sub().run(ctx, t, b.T.copy()).numpy(), a.T - b.T, "Sub strided")
    ai = r.integers(-50, 50, (6, 40)).astype(I32)
    ti = ctx.to_device(ai).permute(1, 0)
    assert np.array_equal(rt.Mul().run(ctx, ti, np.array([3], I32)).numpy(), ai.T * 3)
    aid = ctx.to_device(ai)
    rt.Add().run(ctx, aid, ai, out=aid)
    assert np.array_equal(aid.numpy(), 2 * ai)
    with pytest.raises(rt.OpError) as ei:
        rt.Sub().run(ctx, a, ai)
    assert ei.value.kind == "UnsupportedType"


# ---- shape values on the host
def _graph(W, nodes, inits, inputs, outputs, domain_opsets=()):
    return W.model(nodes, [W.tensor(k, v) for k, v in inits.items()], [W.value_info(n, t, s) for n, t, s in inputs],
                   [W.value_info(n, t, []) for n, t in outputs], opset=21, extra_opsets=(("com.microsoft", 1),) + tuple(domain_opsets))


def test_shape_and_gather_of_a_shape(rt, ctx):
    import onnx_writer as W
    from rten_b200.model import Model
    x = np.zeros((2, 3, 5, 7), F32)
    cases = {"s_all": {}, "s_1": dict(start=1), "s_neg": dict(start=-3, end=-1), "s_clamp": dict(start=-9, end=99),
             "s_empty": dict(start=3, end=1)}
    want = {"s_all": [2, 3, 5, 7], "s_1": [3, 5, 7], "s_neg": [3, 5], "s_clamp": [2, 3, 5, 7], "s_empty": []}
    nodes = [W.node("Shape", ["x"], [k], **a) for k, a in cases.items()]
    nodes += [W.node("Gather", ["s_all", "i_scalar"], ["g_scalar"], axis=0), W.node("Gather", ["s_all", "i_vec"], ["g_vec"]),
              W.node("Cast", ["g_vec"], ["g_cast"], to=W.INT32)]
    inits = {"i_scalar": np.array(-1, np.int64), "i_vec": np.array([2, -4, 3], np.int64)}
    outs = list(cases) + ["g_scalar", "g_vec", "g_cast"]
    m = Model(ctx, _graph(W, nodes, inits, [("x", W.FLOAT, list(x.shape))], [(o, W.INT64) for o in outs]))
    xd = ctx.to_device(x)
    ctx.sync()
    n0 = ctx.launches
    got = [t.numpy() for t in m.run({"x": xd}, outs)]
    assert ctx.launches == n0
    for k, g in zip(outs, got):
        assert g.dtype == I32
    for k in cases:
        assert got[outs.index(k)].tolist() == want[k], k
    assert got[outs.index("g_scalar")].shape == () and int(got[outs.index("g_scalar")]) == 7
    assert got[outs.index("g_vec")].tolist() == [5, 2, 7] and got[outs.index("g_cast")].tolist() == [5, 2, 7]
    bad = Model(ctx, _graph(W, [W.node("Shape", ["x"], ["s"]), W.node("Gather", ["s", "i"], ["g"])], {"i": np.array(4, np.int64)},
                            [("x", W.FLOAT, list(x.shape))], [("g", W.INT64)]))
    with pytest.raises(rt.OpError) as ei:
        bad.run({"x": xd}, ["g"])
    assert ei.value.kind == "InvalidValue" and "Entry in `indices` is out of range" in ei.value.msg


def test_reshape_to_a_computed_shape(rt, ctx):
    """Reshape(y, Cast(Gather(Shape(x), [0, 1, 2]))) and Reshape(v, Unsqueeze(Gather(Shape(x), -1))): the targets are
    host values and the whole graph launches nothing; a y the target does not fit fails as Reshape does"""
    import onnx_writer as W
    from rten_b200.model import Model
    nodes = [W.node("Shape", ["x"], ["s"]), W.node("Gather", ["s", "idx"], ["g"]), W.node("Cast", ["g"], ["t"], to=W.INT64),
             W.node("Reshape", ["y", "t"], ["z"]),
             W.node("Gather", ["s", "last"], ["n"]), W.node("Unsqueeze", ["n", "ax0"], ["n1"]), W.node("Reshape", ["v", "n1"], ["flat"])]
    inits = {"idx": np.array([0, 1, 2], np.int64), "last": np.array(-1, np.int64), "ax0": np.array([0], np.int64)}
    m = Model(ctx, _graph(W, nodes, inits, [("x", W.FLOAT, [2, 3, 4]), ("y", W.FLOAT, [6, 4]), ("v", W.FLOAT, [1, 4])],
                    [("z", W.FLOAT), ("flat", W.FLOAT)]))
    x = np.zeros((2, 3, 4), F32)
    y = np.arange(24, dtype=F32).reshape(6, 4)
    v = np.arange(4, dtype=F32).reshape(1, 4)
    xd, yd, vd = ctx.to_device(x), ctx.to_device(y), ctx.to_device(v)
    bad = ctx.to_device(np.zeros((5, 5), F32))
    ctx.sync()
    n0 = ctx.launches
    z, flat = m.run({"x": xd, "y": yd, "v": vd}, ["z", "flat"])
    assert ctx.launches == n0
    gc.assert_bit_exact(z.numpy(), y.reshape(2, 3, 4), "Reshape to Shape(x)")
    gc.assert_bit_exact(flat.numpy(), v.reshape(4), "Reshape to Unsqueeze(Gather(Shape(x)))")
    with pytest.raises(rt.OpError) as ei:
        m.run({"x": xd, "y": bad, "v": vd}, ["z"])
    assert ei.value.kind == "InvalidValue" and "same total elements" in ei.value.msg


def test_new_operators_load_only_in_the_default_domain(rt, ctx):
    import onnx_writer as W
    from rten_b200.model import Model
    for op, ins in (("ReduceSum", ["x"]), ("Sub", ["x", "x"]), ("Shape", ["x"])):
        data = _graph(W, [W.node(op, ins, ["y"], domain="com.microsoft")], {}, [("x", W.FLOAT, [2, 3])], [("y", W.FLOAT)])
        with pytest.raises(rt.OpError) as ei:
            Model(ctx, data)
        assert ei.value.kind == "UnsupportedValue" and f"unsupported operator com.microsoft.{op}" in ei.value.msg
        Model(ctx, _graph(W, [W.node(op, ins, ["y"])], {}, [("x", W.FLOAT, [2, 3])], [("y", W.FLOAT)]))


# ---- the genai decoder
@pytest.mark.parametrize("packed", [(0,), ()], ids=["packed-qkv-layer0", "separate-qkv"])
def test_genai_decoder_generates_through_model(rt, ctx, packed):
    from rten_b200.model import Model
    from test_gpu_norms import DEC as c, _decoder_f64, _decoder_graph, _decoder_ops, _decoder_weights
    B, S, steps = 2, 12, 8
    w = gd.genai_weights(packed)
    m = Model(ctx, gd.genai_graph(w, packed))
    names = gd.output_names()
    r = np.random.default_rng(40)
    ids = r.integers(0, c["V"], (B, S)).astype(I32)
    past = [(np.zeros((B, c["Hkv"], 0, c["D"]), F32),) * 2 for _ in range(c["L"])]
    all_ids, logits = ids, []
    for step in range(steps + 1):
        T = all_ids.shape[1]
        feeds = {"input_ids": ids, "attention_mask": np.ones((B, T), I32)}
        for l in range(c["L"]):
            feeds[f"past_key_values.{l}.key"], feeds[f"past_key_values.{l}.value"] = past[l]
        ctx.sync()
        n0 = ctx.launches
        got = m.run(feeds, names)
        ctx.sync()
        launches = ctx.launches - n0
        got = [t.numpy() for t in got]
        sk, total = np.full((B, 1), T - 1, I32), np.array(T, I32)
        ops_past = [(None, None)] * c["L"] if step == 0 else [(ctx.to_device(p[0]), ctx.to_device(p[1])) for p in past]
        if packed:
            lg, pres = gd.genai_ops(rt, ctx, w, ids, ops_past, sk, total, packed)
        else:
            lg, pres = _decoder_ops(rt, ctx, w, ids, None if step == 0 else ops_past, sk, total)
        gc.assert_bit_exact(got[0], lg.numpy(), f"step {step} logits")
        for l in range(c["L"]):
            gc.assert_bit_exact(got[1 + 2 * l], pres[l][0].numpy(), f"step {step} present.{l}.key")
            gc.assert_bit_exact(got[2 + 2 * l], pres[l][1].numpy(), f"step {step} present.{l}.value")
        assert got[1].shape == (B, c["Hkv"], T, c["D"])
        if not packed and step > 0:
            # the same decoder fed seqlens_k / total_sequence_length as inputs: two launches fewer (no ReduceSum, no Sub)
            plain = Model(ctx, _decoder_graph(_decoder_weights(), B, 1, T - 1))
            pf = {"input_ids": ids, "seqlens_k": sk.reshape(B), "total": total}
            for l in range(c["L"]):
                pf[f"past_key_{l}"], pf[f"past_value_{l}"] = past[l]
            ctx.sync()
            p0 = ctx.launches
            plain.run(pf, ["logits"] + [f"present_{kv}_{l}" for l in range(c["L"]) for kv in ("key", "value")])
            ctx.sync()
            assert launches == ctx.launches - p0 + 2, (launches, ctx.launches - p0)
        logits.append(got[0][:, -1])
        past = [(got[1 + 2 * l], got[2 + 2 * l]) for l in range(c["L"])]
        ids = got[0][:, -1].argmax(-1).astype(I32)[:, None]
        all_ids = np.concatenate([all_ids, ids], 1)
    ref = _decoder_f64(_decoder_weights(), all_ids[:, :-1])
    for step, lg in enumerate(logits):
        t = S - 1 + step
        err = float(np.abs(lg.astype(np.float64) - ref[:, t]).max() / np.abs(ref[:, t]).max())
        assert err <= 2e-4, (step, err)
