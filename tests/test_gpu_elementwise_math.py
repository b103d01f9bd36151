"""`pytest -m gpu`: Div and Pow on the broadcast-arithmetic kernels' Div / Pow family (binary_math_{flat,periodic,nd}_kernel),
Sqrt / Reciprocal / Exp / Tanh / Neg / Abs on unary_kernel, ReduceMean on the ReduceSum kernels, and the executor running
the torch-exported blocks that use them.  Oracles: tests/elementwise_math.py.

  * kernel identity: every case runs once under CUPTI in a child process; the kernel that ran must be the one the rule
    names, and every (kernel, operation) pair must have run at least twice;
  * Div / Pow: bit for bit against the oracle (Pow's general exponents within POW_ULP of the correctly rounded result), on
    dense operands with every n % 4, a misaligned operand, bias rows and position tables, two-sided broadcasts,
    channels-last operands, strided and in-place outputs, signed zeros, inf, NaN and division by zero; the one-element
    divisor / exponent keeps a's shape and runs the flat kernel over a dense a; an empty i32 Div still checks its divisor;
  * i32 Div with a zero divisor or INT_MIN / -1 returns RTEN_ERR_INVALID_VALUE and frees the output it allocated;
  * the unary operators: bit for bit on dense, misaligned, strided and in-place tensors, into strided and offset output
    views (nothing written outside them), with +-0, +-inf and NaN;
  * ReduceMean over the last axis, two non-adjacent axes and every axis, on strided input, for the ReduceSum tests' lane
    lengths; the GlobalAveragePool path the executor keeps for the spatial axes against Sum / len;
  * the five blocks as ONNX graphs: every output equals the oracle run node by node, in both f32 modes."""
import ctypes as C

import numpy as np
import pytest

import elementwise_math as em
import gpu_checks as gc
import test_gpu_glue_kernels as gk
import test_gpu_row_kernels as rk

pytestmark = pytest.mark.gpu

F32, I32 = np.float32, np.int32
INVALID_VALUE = 5
MATH_KERNELS = ("binary_math_flat_kernel", "binary_math_periodic_kernel", "binary_math_nd_kernel")
KERNELS = set(MATH_KERNELS) | {"unary_kernel"}
UNARY_CODES = {"Sqrt": 8, "Reciprocal": 9, "Exp": 10, "Tanh": 11, "Neg": 12, "Abs": 13}


def L(shape, strides=None, off=0):
    return tuple(shape), tuple(strides or gk._contig(shape)), off


# ---- binary cases -----------------------------------------------------------------------------------------------------
def binary_specs(sms):
    big = 8 * sms * gk.BLOCK * 4 + 4 * 37 + 3
    specs = []
    for op in ("Div", "Pow"):
        f = dict(op=op, dtype="f32")
        specs += [dict(f, kind="dense", a=L((n,)), b=L((n,))) for n in (1024, 1025, 1026, 1027)]
        specs += [dict(f, kind="dense", a=L((big,)), b=L((big,))),
                  dict(f, kind="misaligned a", a=L((4, 257), off=1), b=L((4, 257))),
                  dict(f, kind="misaligned a", a=L((2, 64, 32), off=1), b=L((32,))),
                  dict(f, kind="bias", a=L((2, 7, 768)), b=L((768,))),
                  dict(f, kind="bias", a=L((3, 5, 30)), b=L((30,))),
                  dict(f, kind="position", a=L((2, 9, 64)), b=L((9, 64))),
                  dict(f, kind="position", a=L((3, 5, 6)), b=L((5, 6))),
                  dict(f, kind="both broadcast", a=L((2, 1, 12)), b=L((1, 7, 1))),
                  dict(f, kind="channels-last", a=L((2, 8, 5, 7), (280, 1, 56, 8)), b=L((2, 8, 5, 7), (280, 1, 56, 8))),
                  dict(f, kind="channels-last + NCHW", a=L((2, 8, 5, 7), (280, 1, 56, 8)), b=L((2, 8, 5, 7))),
                  dict(f, kind="strided out", a=L((5, 33)), b=L((5, 33)), out=L((5, 33), (37, 1))),
                  dict(f, kind="in place", a=L((7, 129)), b=L((7, 129)), out="a"),
                  dict(f, kind="in place", a=L((4, 96)), b=L((96,)), out="a"),
                  dict(f, kind="specials", a=L((2, 9)), b=L((2, 9))),
                  dict(f, kind="specials", a=L((2, 9), off=1), b=L((2, 9))),
                  # one element: Div multiplies by the reciprocal, both keep a's shape
                  dict(f, kind="scalar", a=L((3, 5, 67)), b=L(())),
                  dict(f, kind="scalar", a=L((1029,)), b=L((1, 1))),
                  dict(f, kind="scalar", a=L((2, 8, 5, 7), (280, 1, 56, 8)), b=L((1,))),
                  dict(f, kind="scalar", a=L((5, 33)), b=L(()), out=L((5, 33), (37, 1))),
                  dict(f, kind="scalar", a=L((4, 40)), b=L((1, 1)), out=L((4, 40), (44, 1), 4))]
        i = dict(op=op, dtype="i32")
        specs += [dict(i, kind="dense", a=L((1027,)), b=L((1027,))), dict(i, kind="dense", a=L((4, 64)), b=L((4, 64))),
                  dict(i, kind="bias", a=L((3, 5, 100)), b=L((100,))), dict(i, kind="bias", a=L((3, 5, 30)), b=L((30,))),
                  dict(i, kind="position", a=L((2, 9, 64)), b=L((9, 64))),
                  dict(i, kind="strided out", a=L((5, 33)), b=L((5, 33)), out=L((5, 33), (37, 1))),
                  dict(i, kind="misaligned a", a=L((4, 257), off=1), b=L((4, 257))),
                  dict(i, kind="both broadcast", a=L((2, 1, 12)), b=L((1, 7, 1))),
                  dict(i, kind="scalar", a=L((3, 70)), b=L(()))]
    return specs


def binary_rule(s):
    """binary_op's output and launch: a one-element b (f32 Div, Pow) is a 0-D scalar, so the output takes a's shape and,
    a dense, a's layout.  A one-element b over dense a and output (b's stride 0 everywhere: a period of 1) runs the flat
    kernel, which reads b once; with a strided output, the strided kernel.  Anything else as for Add
    (tests/test_gpu_glue_kernels.py binary_rule), on the Div / Pow family's kernel of the same layout."""
    t = ("float",) if s["dtype"] == "f32" else ("int",)
    if s["kind"] == "scalar":
        mode = s["op"] + (" by one element" if s["op"] == "Div" and s["dtype"] == "f32" else "")
        return ("binary_math_flat_kernel" if s.get("out") is None else "binary_math_nd_kernel", t), mode
    (k, _), mode = gk.binary_rule(s)
    return (k.replace("binary_", "binary_math_"), t), mode


def _scalar(s):
    return s["kind"] == "scalar" and (s["dtype"] == "f32" or s["op"] == "Pow")


def binary_prepare(s):
    r = rk._rng("math", sorted((k, str(v)) for k, v in s.items()))
    ash, bsh = s["a"][0], s["b"][0]
    if s["dtype"] == "i32":
        if s["op"] == "Div":
            a = r.integers(-2 ** 31, 2 ** 31, ash, dtype=np.int64).astype(I32)
            b = r.integers(-70000, 70000, bsh, dtype=np.int64).astype(I32)
            b[b == 0] = 7
            b.reshape(-1)[:3] = [-3, 3, -1][:b.size]  # truncation toward zero on both signs; x / -1
            a.reshape(-1)[:2] = [-7, 7][:a.size]
        else:
            a = r.integers(-12, 12, ash).astype(I32)
            b = r.integers(-3, 14, bsh).astype(I32)
            a.reshape(-1)[:2] = [46341, 216][:a.size]  # the wrapping square and 216 ^ 4 of the reference's tests
        return dict(a=a, b=b)
    if s["kind"] == "specials":
        a = np.resize(np.array([0.0, -0.0, 1.0, np.inf, -np.inf, np.nan, -2.5, 3e38, 1e-45], F32), ash).astype(F32)
        b = np.resize(np.array([0.0, 0.0, -0.0, np.inf, 2.0, 3.0, 0.0, 1e-3, -0.0], F32), bsh).astype(F32)
        return dict(a=a, b=b)
    if s["op"] == "Div":
        return dict(a=r.uniform(-3, 3, ash).astype(F32), b=r.uniform(0.1, 3, bsh).astype(F32) * r.choice([-1, 1], bsh).astype(F32))
    a = r.uniform(-3, 3, ash).astype(F32)
    b = r.choice(np.array([2.0, 3.0, 0.5, -1.5, 2.7, 0.0, 1.0, -2.0], F32), bsh).astype(F32)
    if s["kind"] == "scalar":
        b = np.full(bsh, 2.0 if len(ash) == 3 else 3.0, F32)  # the norm variance and NewGELU's cube
    return dict(a=a, b=b)


def binary_launch(rt, ctx, s, inp):
    op = {"Div": rt.Div, "Pow": rt.Pow}[s["op"]]()
    fill = np.nan if s["dtype"] == "f32" else -7
    a = gk.placed(ctx, inp["a"], s["a"][1], s["a"][2], fill)
    b = gk.placed(ctx, inp["b"], s["b"][1], s["b"][2], fill, guard=a.base.size)
    out = s.get("out")
    if out == "a":
        assert op.run(ctx, a, b, out=a) is a
        return a.numpy(), None
    if out is not None:
        shape, st, off = out
        o = gk.placed(ctx, np.zeros(shape, inp["a"].dtype), st, off, fill)
        assert op.run(ctx, a, b, out=o) is o
        full = o.base.numpy()
        mask = np.ones(full.shape, bool)
        np.lib.stride_tricks.as_strided(mask[off:], shape, [x * mask.itemsize for x in st])[...] = False
        return o.numpy(), full[mask]
    return op.run(ctx, a, b).numpy(), None


def binary_check(s, inp, got):
    what = gk.spec_id("math", s)
    ref = em.div_ref if s["op"] == "Div" else em.pow_ref
    want = ref(inp["a"], inp["b"])
    assert got.shape == want.shape, f"{what}: shape {got.shape}, the reference's {want.shape}"
    if s["op"] == "Pow" and s["dtype"] == "f32":
        general = np.broadcast_to(em.pow_general(inp["b"].reshape(()) if _scalar(s) else inp["b"]), want.shape)
        gc.assert_bit_exact(np.where(general, 0, got), np.where(general, 0, want), what + " (exponents 2 and 3)")
        worst = int(em.ulp_distance(got[general], want[general]).max()) if general.any() else 0
        assert worst <= em.POW_ULP, f"{what}: powf {worst} ulp from the correctly rounded result"
    else:
        gc.assert_bit_exact(got, want, what)


# ---- unary cases ------------------------------------------------------------------------------------------------------
def unary_specs():
    specs = []
    for op in UNARY_CODES:
        specs += [dict(op=op, kind="dense", shape=(n,)) for n in (4096, 1025, 1026, 1027)]
        specs += [dict(op=op, kind="misaligned", shape=(7, 65)), dict(op=op, kind="strided", shape=(6, 33)),
                  dict(op=op, kind="in place", shape=(5, 129)), dict(op=op, kind="specials", shape=(3, 9)),
                  dict(op=op, kind="strided out", shape=(6, 33)), dict(op=op, kind="offset out", shape=(5, 67))]
    return specs


def unary_prepare(s):
    r = rk._rng("math unary", sorted(s.items()))
    x = r.uniform(-12, 12, s["shape"]).astype(F32)
    if s["op"] in ("Sqrt",):
        x = np.abs(x)
    flat = x.reshape(-1)
    flat[:9] = np.array([0.0, -0.0, np.inf, -np.inf, np.nan, 1e-45, -3.5, 104.0, 0.0004], F32)[:flat.size]
    if s["kind"] == "specials":
        x = np.resize(np.array([0.0, -0.0, np.inf, -np.inf, np.nan, 1e-45, -1e-45, 3e38, -9.02, 0.55, -0.55, 88.7, -104.0], F32),
                      s["shape"]).astype(F32)
    return dict(x=x)


def unary_launch(rt, ctx, s, inp):
    """the result, and whatever the output's buffer holds outside the output view"""
    op = getattr(rt, s["op"])()
    x = inp["x"]
    if s["kind"] in ("strided out", "offset out"):  # a row-padded output at an offset, and a misaligned dense one
        st, off = ((x.shape[1] + 3,) + (1,), 2) if s["kind"] == "strided out" else (gk._contig(x.shape), 1)
        o = gk.placed(ctx, np.zeros(x.shape, F32), st, off)
        assert op.run(ctx, ctx.to_device(x), out=o) is o
        full = o.base.numpy()
        mask = np.ones(full.shape, bool)
        np.lib.stride_tricks.as_strided(mask[off:], x.shape, [v * mask.itemsize for v in st])[...] = False
        return o.numpy(), full[mask]
    if s["kind"] == "misaligned":
        return op.run(ctx, gk.placed(ctx, x, gk._contig(x.shape), 1)).numpy(), None
    if s["kind"] == "strided":
        R, Cn = x.shape
        return op.run(ctx, gk.placed(ctx, x, (Cn + 4, 1))).numpy(), None
    if s["kind"] == "in place":
        d = ctx.to_device(x)
        assert op.run(ctx, d, in_place=True) is d
        return d.numpy(), None
    return op.run(ctx, ctx.to_device(x)).numpy(), None


def unary_rule(s):
    return ("unary_kernel", (UNARY_CODES[s["op"]],)), None


# ---- kernel identity --------------------------------------------------------------------------------------------------
def _cases(sms):
    return [("binary", s) for s in binary_specs(sms)] + [("unary", s) for s in unary_specs()]


def _kernel_probe():
    import json
    import torch
    import rten_b200 as rt
    n_sms = torch.cuda.get_device_properties(0).multi_processor_count
    ctx = rt.Context(0)
    res, retaken = {}, 0
    for fam, s in _cases(n_sms):
        inp = binary_prepare(s) if fam == "binary" else unary_prepare(s)

        def call():
            (binary_launch if fam == "binary" else unary_launch)(rt, ctx, s, inp)
            ctx.sync()
        names, again = rk.capture_kernels(call)
        retaken += again
        res[gk.spec_id(fam, s)] = sorted(names)
    print(json.dumps({"sms": n_sms, "names": res, "retaken": retaken}))


@pytest.fixture(scope="module")
def rt():
    import rten_b200
    from rten_b200 import _lib
    _lib.load()
    return rten_b200


@pytest.fixture(scope="module")
def sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def test_kernel_identity():
    out = rk.probe_in_child("test_gpu_elementwise_math")
    n_sms, names = out["sms"], out["names"]
    seen, wrong = {}, []
    for fam, s in _cases(n_sms):
        sid = gk.spec_id(fam, s)
        want, mode = binary_rule(s) if fam == "binary" else unary_rule(s)
        ran = {rk.kernel_key(n, KERNELS) for n in names[sid]} - {None}
        if ran != {want}:
            wrong.append((sid, want, sorted(ran)))
        for k in ran:
            seen[(k, mode)] = seen.get((k, mode), 0) + 1
    assert not wrong, f"{len(wrong)} cases ran another kernel than the rule names: {wrong[:10]}"
    units = {(k, t, m) for (k, t), m in seen}
    for k in MATH_KERNELS:
        for t in (("float",), ("int",)):
            for m in ("Div", "Pow"):
                assert seen.get(((k, t), m), 0) >= 2, f"{k}<{t[0]}> {m} ran in fewer than two cases"
    for k in ("binary_math_flat_kernel", "binary_math_nd_kernel"):
        assert seen.get(((k, ("float",)), "Div by one element"), 0) >= 2, f"{k}<float> Div by one element"
    for op, code in UNARY_CODES.items():
        assert seen.get((("unary_kernel", (code,)), None), 0) >= 2, f"unary_kernel<{code}> ({op})"
    print(f"{len(units)} (kernel, operation) units ran on {n_sms} SMs")


# ---- numbers ----------------------------------------------------------------------------------------------------------
def test_div_pow_exact(rt, sms):
    ctx = rt.Context(0)
    for s in binary_specs(sms):
        inp = binary_prepare(s)
        got, outside = binary_launch(rt, ctx, s, inp)
        binary_check(s, inp, got)
        if outside is not None:
            untouched = np.isnan(outside).all() if s["dtype"] == "f32" else (outside == -7).all()
            assert untouched, f"{gk.spec_id('math', s)}: writes outside the output view"


def test_div_shapes_and_edges(rt):
    ctx = rt.Context(0)
    a = np.array([1.0, 3.0, 7.0, 10.0], F32)
    y = rt.Div().run(ctx, ctx.to_device(a), ctx.to_device(np.full((1, 1), 3.0, F32))).numpy()
    assert y.shape == (4,)
    gc.assert_bit_exact(y, a * (F32(1) / F32(3)), "Div by a [1, 1] divisor")
    assert rt.Div().run(ctx, ctx.to_device(a), ctx.to_device(np.full((1, 4), 3.0, F32))).numpy().shape == (1, 4)
    assert rt.Pow().run(ctx, ctx.to_device(a), ctx.to_device(np.full((1, 1, 1), 2.0, F32))).numpy().shape == (4,)
    z = rt.Div().run(ctx, ctx.to_device(np.array([1.0, -1.0, 0.0, -0.0], F32)), ctx.to_device(np.array([0.0, 0.0, 0.0, 5.0], F32))).numpy()
    assert z[0] == np.inf and z[1] == -np.inf and np.isnan(z[2]) and z[3] == 0 and np.signbit(z[3])
    with pytest.raises(rt.OpError) as e:
        rt.Pow().run(ctx, ctx.to_device(np.ones(3, I32)), ctx.to_device(np.ones(3, F32)))
    assert e.value.kind == "UnsupportedType"


@pytest.mark.parametrize("b", [np.array([3, 0, 5], I32), np.array(0, I32)], ids=["zero element", "zero scalar"])
def test_i32_div_by_zero_fails_and_frees(rt, b):
    _div_failure(rt, np.array([7, 8, 9], I32), b)


def test_i32_div_overflow_fails_and_frees(rt):
    _div_failure(rt, np.array([5, -2 ** 31, 6], I32), np.array([1, -1, 2], I32))


def test_i32_div_empty_output_still_checks_the_divisor(rt):
    """check_nonzero runs over all of b before the broadcast: Div(a[0, 3], b) fails on a zero in b, as the reference does"""
    ctx = rt.Context(0)
    a = ctx.to_device(np.zeros((0, 3), I32))
    with pytest.raises(rt.OpError) as e:
        rt.Div().run(ctx, a, ctx.to_device(np.array([1, 0, 2], I32)))
    assert e.value.kind == "InvalidValue" and "Divisor contains zero" in str(e.value)
    with pytest.raises(rt.OpError):  # the zero in a strided view of b
        rt.Div().run(ctx, a, gk.placed(ctx, np.array([4, 0, 5], I32), (2,), 1, fill=3))
    assert rt.Div().run(ctx, a, ctx.to_device(np.array([1, -1, 2], I32))).numpy().shape == (0, 3)


def _div_failure(rt, a, b):
    ctx = rt.Context(0)
    A = rt.ops._Args(ctx)
    da, db = ctx.to_device(a), ctx.to_device(b)
    A.keep += [da, db]
    o = A.out()
    st = ctx.lib.rten_b200_div(ctx.handle, A.t(da), A.t(db), C.byref(o))
    assert st == INVALID_VALUE, st
    assert ctx.lib.rten_b200_last_error(ctx.handle).decode() == "Divisor contains zero"
    assert not o.data, "the output the failed call allocated is still set"
    good = rt.Div().run(ctx, da, ctx.to_device(np.array([2, 3, 4], I32))).numpy()
    gc.assert_bit_exact(good, em.div_ref(a, np.array([2, 3, 4], I32)), "i32 Div after a failed call")


def test_unary_exact(rt):
    ctx = rt.Context(0)
    for s in unary_specs():
        inp = unary_prepare(s)
        got, outside = unary_launch(rt, ctx, s, inp)
        gc.assert_bit_exact(got, em.unary_ref(s["op"], inp["x"]), gk.spec_id("unary", s))
        if outside is not None:
            assert np.isnan(outside).all(), f"{gk.spec_id('unary', s)}: writes outside the output view"
    x = np.array([-0.0, 0.0], F32)
    assert np.signbit(rt.Neg().run(ctx, ctx.to_device(x[1:])).numpy()[0])
    assert not np.signbit(rt.Abs().run(ctx, ctx.to_device(x[:1])).numpy()[0])
    assert rt.Reciprocal().run(ctx, ctx.to_device(x)).numpy().tolist() == [-np.inf, np.inf]


LANES = [1, 15, 64, 65, 1000, 1024, 1025, 4096, 4097, 8193]


@pytest.mark.parametrize("L", LANES)
def test_reduce_mean_lanes(rt, L):
    ctx = rt.Context(0)
    r = rk._rng("reduce mean", L)
    x = r.uniform(-2, 2, (3, 2, L)).astype(F32)
    big = r.uniform(-2, 2, (4, 3, L + 3)).astype(F32)
    view = ctx.to_device(big)  # a strided view: every other row, the lane cut short
    xv = big[::2, :, 1:L + 1]
    dv = view.view(xv.shape, (2 * 3 * (L + 3), L + 3, 1), 1)
    for axes in ([-1], [0, 2], None):
        for keep in (True, False):
            got = rt.ReduceMean(axes, keep).run(ctx, ctx.to_device(x)).numpy()
            gc.assert_bit_exact(got, em.reduce_mean_ref(x, axes, keep), f"L={L} {axes} keep={keep}")
            got = rt.ReduceMean(axes, keep).run(ctx, dv).numpy()
            gc.assert_bit_exact(got, em.reduce_mean_ref(xv, axes, keep), f"L={L} strided {axes} keep={keep}")


def test_reduce_mean_edges(rt):
    ctx = rt.Context(0)
    gc.assert_bit_exact(rt.ReduceMean([], False).run(ctx, ctx.to_device(np.array(5.0, F32))).numpy(), np.array(5.0, F32), "0-D")
    e = rt.ReduceMean([1], False).run(ctx, ctx.to_device(np.zeros((3, 0), F32))).numpy()
    assert e.shape == (3,) and np.isnan(e).all()
    with pytest.raises(rt.OpError):
        rt.ReduceMean([2]).run(ctx, ctx.to_device(np.zeros((3, 3), F32)))
    with pytest.raises(rt.OpError) as ei:
        rt.ReduceMean([0]).run(ctx, ctx.to_device(np.zeros(3, I32)))
    assert ei.value.kind == "UnsupportedType"


@pytest.mark.parametrize("hw", [(7, 7), (14, 14), (56, 56)])
def test_spatial_reduce_mean_path_is_sum_over_len(rt, hw):
    """The executor keeps GlobalAveragePool for ReduceMean over an NCHW tensor's spatial axes; its bits against the
    reference's ReduceMean, Sum(lane) / len"""
    ctx = rt.Context(0)
    x = rk._rng("spatial mean", hw).uniform(-2, 2, (2, 13) + hw).astype(F32)
    got = rt.GlobalAveragePool().run(ctx, ctx.to_device(x)).numpy()
    gc.assert_bit_exact(got, em.reduce_mean_ref(x, [2, 3], True), f"GlobalAveragePool {hw} against Sum / len")


# ---- the executor ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(em.block_specs(8)))
@pytest.mark.parametrize("tf32x3", [True, False], ids=["3xTF32", "TF32"])
def test_executor_blocks_node_by_node(rt, name, tf32x3):
    from rten_b200.model import Model
    ctx = rt.Context(0)
    ctx.set_f32_mode(tf32x3)
    H = 768 if name != "attention scale" else 128
    shape = (2, 12, 128, 128) if name == "attention scale" else (4, 33, H)
    spec = em.block_specs(H)[name]
    r = rk._rng("block", name)
    feeds = {"x": r.uniform(-3, 3, shape).astype(F32)}
    extra = {}
    if "mask" in spec[2]:
        extra["mask"] = (2, 1, 1, 128)
        feeds["mask"] = np.where(r.random(extra["mask"]) < 0.2, F32(-10000.0), F32(0.0)).astype(F32)
    m = Model(ctx, em.block_model(spec, shape, extra))
    (y,) = m.run(feeds, ["y"])
    gc.assert_bit_exact(y.numpy(), em.run_nodes(spec[0], spec[1], feeds)["y"], f"{name} ({'3xTF32' if tf32x3 else 'TF32'})")
