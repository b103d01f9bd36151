"""`pytest -m gpu`: Where, the comparisons, the logical operators, Trilu, Expand, Slice and Split (masks.cu, api_masks.cu)
and the executor rows and host shape arithmetic built on them (model.cu).  Oracle: tests/mask_ops.py.

  * kernel identity: every case runs under CUPTI; the kernel that ran must be the one `rule` names, and every (kernel,
    operation) pair must run at least twice, once with a partial last unit (a flat pass whose n is not a multiple of a
    whole grid of 16-byte units, or a row whose length is not a multiple of the 512-element row piece);
  * bit for bit against the oracle on dense operands with every n % 4, misaligned operands, one-element operands (GPT-2's
    0-D finfo.min), the strided bias-window condition broadcast over batch and heads, two-sided broadcasts, strided and
    offset outputs with nothing written outside them, empty tensors, and NaN / +-0 / +-inf / subnormals for comparisons;
  * every error path returns the reference's message and frees the output it allocated;
  * the executor: a shape subgraph of host arithmetic launches nothing, Slice and Split of device tensors launch
    nothing, and a Llama-style mask / rotate_half / repeat_kv block equals the oracle node by node in both f32 modes."""
import json

import numpy as np
import pytest

import gpu_checks as gc
import mask_ops as mo
import onnx_writer as W
import test_gpu_glue_kernels as gk
import test_gpu_row_kernels as rk

pytestmark = pytest.mark.gpu

F32, I32 = np.float32, np.int32
INVALID_VALUE, INCOMPATIBLE, UNSUPPORTED_VALUE = 5, 3, 6
CHUNK = 512  # row elements one CTA covers per unit (masks.cu)

VARIANTS = {"where_flat_kernel": {()}, "where_rows_kernel": {()}, "compare_flat_kernel": {("float",), ("int",)},
            "compare_rows_kernel": {("float",), ("int",)}, "trilu_kernel": {()}, "expand_repeat_kernel": {()},
            "fill_kernel": {()}}
KERNELS = set(VARIANTS)
CMP = ("Equal", "Less", "LessOrEqual", "Greater", "GreaterOrEqual")
LOGICAL = ("And", "Or", "Xor")


def L(shape, strides=None, off=0):
    return tuple(shape), tuple(strides or gk._contig(shape)), off


# ---- the launchers' layout choice, restated (masks.cu Layout) ------------------------------------------------------
def _bstrides(shape, t):
    nd = len(shape)
    sh, st, _ = t
    out = []
    for i in range(nd):
        k = i - (nd - len(sh))
        out.append(st[k] if k >= 0 and sh[k] != 1 else 0)
    return out


def _out_shape(*ts):
    return np.broadcast_shapes(*[t[0] for t in ts])


def layout(shape, sts):
    """(dims, strides per operand) after dropping size-1 dims and merging, as Layout does; the output's strides last"""
    dims, st = [], [[] for _ in sts]
    for i, d in enumerate(shape):
        if d == 1:
            continue
        if dims and all(s[-1] == o[i] * d for s, o in zip(st, sts)):
            dims[-1] *= d
            for s, o in zip(st, sts):
                s[-1] = o[i]
            continue
        dims.append(d)
        for s, o in zip(st, sts):
            s.append(o[i])
    if not dims:
        return [1], [[1] for _ in sts]
    return dims, st


def flat_or_rows(shape, ins, out):
    dims, st = layout(shape, [_bstrides(shape, t) for t in ins] + [list(out[1])])
    flat = len(dims) == 1 and st[-1][0] == 1 and all(s[0] in (0, 1) or dims[0] == 1 for s in st[:-1])
    return ("flat" if flat else "rows"), dims


def rule(s):
    """((kernel, template args), operation) the launch runs"""
    if s["op"] == "Trilu":
        return ("trilu_kernel", ()), "Trilu"
    if s["op"] == "Expand":
        return (("expand_repeat_kernel", ()) if s["fast"] else ("nd_copy_kernel", ("unsigned int",))), "Expand"
    ins = [s["cond"], s["x"], s["y"]] if s["op"] == "Where" else [s["a"]] if s["op"] == "Not" else [s["a"], s["b"]]
    shape = _out_shape(*ins)
    out = s.get("out") or L(shape)
    kind, _ = flat_or_rows(shape, ins, out)
    if s["op"] == "Where":
        return (f"where_{kind}_kernel", ()), "Where"
    t = ("float",) if s.get("dtype", "f32") == "f32" and s["op"] not in LOGICAL + ("Not",) else ("int",)
    return (f"compare_{kind}_kernel", t), s["op"]


def partial(s):
    """the case's last unit is partial: a flat n not a multiple of 4, or a row not a multiple of CHUNK"""
    if s["op"] == "Expand":
        return s["x"][0][-1] % CHUNK != 0 if s["fast"] else True
    if s["op"] == "Trilu":
        return s["x"][0][-1] % CHUNK != 0
    ins = [s["cond"], s["x"], s["y"]] if s["op"] == "Where" else [s["a"]] if s["op"] == "Not" else [s["a"], s["b"]]
    shape = _out_shape(*ins)
    kind, dims = flat_or_rows(shape, ins, s.get("out") or L(shape))
    return dims[-1] % (4 if kind == "flat" else CHUNK) != 0


# ---- cases ---------------------------------------------------------------------------------------------------------
def specs():
    out = []
    for dt in ("f32", "i32"):
        w = dict(op="Where", dtype=dt)
        out += [dict(w, cond=L((n,)), x=L((n,)), y=L((n,))) for n in (1024, 1025, 1026, 1027)]
        out += [dict(w, cond=L((4, 257)), x=L((4, 257), off=1), y=L((4, 257))),  # misaligned x: the flat scalar path
                dict(w, cond=L((2, 3, 64, 64)), x=L((2, 3, 64, 64)), y=L(())),  # GPT-2's 0-D finfo.min
                dict(w, cond=L((1, 1, 48, 48), (0, 0, 1024, 1)), x=L((2, 3, 48, 48)), y=L(())),  # the bias window
                dict(w, cond=L((1, 1, 40, 601), (0, 0, 1024, 1), 3), x=L((2, 2, 40, 601)), y=L(())),
                dict(w, cond=L((2, 1, 7)), x=L((1, 5, 1)), y=L((2, 5, 7))),  # two-sided broadcasts
                dict(w, cond=L((3, 130)), x=L((3, 130)), y=L((130,))),
                dict(w, cond=L((5, 33)), x=L((5, 33)), y=L((5, 33)), out=L((5, 33), (37, 1), 2)),
                dict(w, cond=L((0, 7)), x=L((0, 7)), y=L(()))]
    for op in CMP:
        for dt in ("f32", "i32"):
            c = dict(op=op, dtype=dt)
            out += [dict(c, a=L((1027,)), b=L((1027,))), dict(c, a=L((4, 64)), b=L((4, 64))),
                    dict(c, a=L((2, 9, 520)), b=L((520,))), dict(c, a=L((3, 1, 6)), b=L((1, 5, 1))),
                    dict(c, a=L((5, 33)), b=L(()), out=L((5, 33), (40, 1), 1))]
    for op in LOGICAL:
        c = dict(op=op, dtype="i32")
        out += [dict(c, a=L((1026,)), b=L((1026,))), dict(c, a=L((8, 64)), b=L(())),
                dict(c, a=L((2, 1, 600)), b=L((2, 3, 600))), dict(c, a=L((3, 1)), b=L((1, 5)))]
    c = dict(op="Not", dtype="i32")
    out += [dict(c, a=L((1025,))), dict(c, a=L((64,))), dict(c, a=L((3, 700), (800, 1))), dict(c, a=L((2, 5), (1, 2)))]
    for dt in ("f32", "i32"):
        t = dict(op="Trilu", dtype=dt)
        out += [dict(t, x=L((3, 3)), k=0, upper=True), dict(t, x=L((2, 5, 7)), k=1, upper=False),
                dict(t, x=L((64, 1024)), k=-3, upper=True), dict(t, x=L((2, 96, 96)), k=0, upper=False),
                dict(t, x=L((4, 9), (16, 1), 1), k=2, upper=True), dict(t, x=L((0, 4)), k=0, upper=True)]
        e = dict(op="Expand", dtype=dt)
        out += [dict(e, x=L((2, 2, 1, 24, 32)), shape=(2, 2, 4, 24, 32), fast=True),  # repeat_kv
                dict(e, x=L((1, 1, 700)), shape=(3, 2, 700), fast=True),  # leading broadcast
                dict(e, x=L((4, 1, 200)), shape=(4, 3, 200), fast=True),  # a middle broadcast, a partial row piece
                dict(e, x=L((5, 1)), shape=(5, 6), fast=False),  # trailing broadcast: rows of one element take the strided copy
                dict(e, x=L((3, 1, 4, 1)), shape=(3, 2, 4, 5), fast=False)]  # two broadcast runs: the strided copy
    return out


def _rng(s):
    return rk._rng("mask", sorted((k, str(v)) for k, v in s.items()))


SPECIAL = np.array([np.nan, 0.0, -0.0, np.inf, -np.inf, 1e-45, -1e-45, 1.0, -1.0, 1e-38, 3.0, np.nan], F32)


def _values(r, shape, dt, special=False):
    if dt == "i32":
        return r.integers(-3, 4, shape).astype(I32)
    if special:
        return r.choice(SPECIAL, shape).astype(F32)
    return r.uniform(-2, 2, shape).astype(F32)


def prepare(s):
    r = _rng(s)
    dt = s.get("dtype", "f32")
    if s["op"] == "Where":
        return dict(cond=r.integers(-1, 2, s["cond"][0]).astype(I32), x=_values(r, s["x"][0], dt), y=_values(r, s["y"][0], dt))
    if s["op"] in CMP:
        return dict(a=_values(r, s["a"][0], dt, True), b=_values(r, s["b"][0], dt, True))
    if s["op"] in LOGICAL:
        return dict(a=r.integers(-2, 3, s["a"][0]).astype(I32), b=r.integers(-2, 3, s["b"][0]).astype(I32))
    if s["op"] == "Not":
        return dict(a=r.integers(-2, 3, s["a"][0]).astype(I32))
    return dict(x=_values(r, s["x"][0], dt))


def expected(s, inp):
    op = s["op"]
    if op == "Where":
        return mo.where(inp["cond"], inp["x"], inp["y"])
    if op in CMP:
        return mo.compare(op, inp["a"], inp["b"])
    if op in LOGICAL:
        return mo.logical(op, inp["a"], inp["b"])
    if op == "Not":
        return mo.not_(inp["a"])
    if op == "Trilu":
        return mo.trilu(inp["x"], s["k"], s["upper"])
    return mo.expand(inp["x"], s["shape"])


def place(ctx, s, inp):
    """the inputs as device views placed as the case says, and the given output view (or None)"""
    fill = {np.dtype(F32): np.nan, np.dtype(I32): -7}
    dev = {k: gk.placed(ctx, v, s[k][1], s[k][2], fill[v.dtype]) for k, v in inp.items()}
    out, o = s.get("out"), None
    if out is not None:
        odt = I32 if s["op"] != "Where" else inp["x"].dtype
        o = gk.placed(ctx, np.zeros(out[0], odt), out[1], out[2], fill[np.dtype(odt)])
    return dev, o


def call(rt, ctx, s, dev, o):
    """the operator alone (what the kernel probe profiles)"""
    op = s["op"]
    if op == "Where":
        return rt.Where().run(ctx, dev["cond"], dev["x"], dev["y"], out=o)
    if op in CMP + LOGICAL:
        return getattr(rt, op)().run(ctx, dev["a"], dev["b"], out=o)
    if op == "Not":
        return rt.Not().run(ctx, dev["a"], out=o)
    if op == "Trilu":
        return rt.Trilu(s["upper"]).run(ctx, dev["x"], s["k"], out=o)
    return rt.Expand().run(ctx, dev["x"], s["shape"], out=o)


def launch(rt, ctx, s, inp):
    """(result, the guard elements around a given output view)"""
    dev, o = place(ctx, s, inp)
    res = call(rt, ctx, s, dev, o)
    rest = None
    if o is not None:
        out = s["out"]
        full = o.base.numpy()
        mask = np.ones(full.shape, bool)
        np.lib.stride_tricks.as_strided(mask[out[2]:], out[0], [x * mask.itemsize for x in out[1]])[...] = False
        rest = full[mask]
    return res.numpy(), rest


def _empty(s):
    if s["op"] == "Trilu":
        shape = s["x"][0]
    elif s["op"] == "Expand":
        shape = s["shape"]
    else:
        shape = _out_shape(*[s[k] for k in ("cond", "x", "y", "a", "b") if k in s])
    return int(np.prod(shape)) == 0


def _kernel_probe():
    """run in a child process (tests/test_gpu_row_kernels.py probe_in_child): the kernels each case launched"""
    import rten_b200 as rt
    ctx = gc.new_ctx(rt)
    res, retaken = {}, 0
    for i, s in enumerate(specs()):
        dev, o = place(ctx, s, prepare(s))
        ctx.sync()

        def run():
            call(rt, ctx, s, dev, o)
            ctx.sync()
        names, again = rk.capture_kernels(run)
        retaken += again
        res[str(i)] = sorted(names)
    print(json.dumps({"names": res, "retaken": retaken}))


@pytest.fixture(scope="module")
def rt():
    import rten_b200
    return rten_b200


def test_bit_exact(rt):
    ctx = gc.new_ctx(rt)
    for s in specs():
        inp = prepare(s)
        got, rest = launch(rt, ctx, s, inp)
        what = f"{s['op']} {s}"
        gc.assert_bit_exact(got, expected(s, inp), what)
        if rest is not None:
            assert (np.isnan(rest) if rest.dtype == F32 else rest == -7).all(), f"{what}: wrote outside the output view"


def test_kernel_identity():
    names = rk.probe_in_child("test_gpu_mask_ops")["names"]
    seen, wrong = {}, []
    for i, s in enumerate(specs()):
        ran = {rk.kernel_key(n, KERNELS | {"nd_copy_kernel"}) for n in names[str(i)]} - {None}
        if _empty(s):
            if ran:
                wrong.append((s, "nothing", sorted(ran)))
            continue
        kern, op = rule(s)
        if ran != {kern}:
            wrong.append((s, kern, sorted(ran)))
        seen.setdefault((kern, op), []).append(partial(s))
    assert not wrong, f"{len(wrong)} cases ran another kernel than the rule names: {wrong[:5]}"
    for k, parts in seen.items():
        assert len(parts) >= 2 and any(parts), f"{k}: {len(parts)} cases, partial last unit {any(parts)}"
    ran = {k for k, _ in seen}
    for base, args in VARIANTS.items():
        if base != "fill_kernel":  # (ConstantOfShape's fill: test_constant_of_shape_fill)
            for a in args:
                assert (base, a) in ran, f"{base}{a} never ran"


def _fails(ctx, fn, status, msg):
    with pytest.raises(Exception) as e:
        fn()
    assert e.value.status == status and msg in e.value.msg, (status, msg, e.value.status, e.value.msg)


def test_errors(rt):
    ctx = gc.new_ctx(rt)
    f = np.ones((2, 3), F32)
    _fails(ctx, lambda: rt.Trilu().run(ctx, np.ones((4,), F32)), INVALID_VALUE, "Input must have >= 2 dims")
    _fails(ctx, lambda: rt.Expand().run(ctx, f, (-1, 3)), INVALID_VALUE, "Target shape contains negative values")
    _fails(ctx, lambda: rt.Expand().run(ctx, f, (2, 4)), INCOMPATIBLE, "Cannot broadcast input with target shape")
    _fails(ctx, lambda: rt.Where().run(ctx, np.ones((2, 4), I32), f, f), INCOMPATIBLE, "Cannot broadcast inputs")
    _fails(ctx, lambda: rt.Slice().run(ctx, f, [0], [2], [0], [0]), INVALID_VALUE, "steps must be non-zero")
    _fails(ctx, lambda: rt.Slice().run(ctx, f, [2], [0], [0], [-1]), UNSUPPORTED_VALUE, "negative step")
    _fails(ctx, lambda: rt.Split(0).run(ctx, f, [1, 2]), INVALID_VALUE, "Split sizes do not sum to dimension size")
    _fails(ctx, lambda: rt.Split(1).run(ctx, f, None, 4), INVALID_VALUE, "num_outputs exceeds dim size")
    _fails(ctx, lambda: rt.And().run(ctx, f, f), 2, "unsupported type")


def test_slice_and_split_copies(rt):
    ctx = gc.new_ctx(rt)
    x = np.arange(5 * 12, dtype=F32).reshape(5, 12)
    for args in [([1, -5], [4, 100], [0, 1], [2, 3]), ([-100, 0], [3, 12], None, None), ([2], [1], [1], None)]:
        gc.assert_bit_exact(rt.Slice().run(ctx, ctx.to_device(x), *args).numpy(), mo.slice_(x, *args), f"Slice {args}")
    for axis, sizes, k in [(1, [4, 4, 4], None), (1, None, 5), (0, [0, 5], None), (-1, [12], None)]:
        got = rt.Split(axis).run(ctx, ctx.to_device(x), sizes, k)
        exp = mo.split(x, axis, sizes, k)
        assert len(got) == len(exp)
        for g, e in zip(got, exp):
            gc.assert_bit_exact(g.numpy(), e, f"Split {axis} {sizes} {k}")


# ---- executor ----------------------------------------------------------------------------------------------------
def _i64(v):
    return np.array(v, np.int64)


def test_host_shape_subgraph_launches_nothing(rt):
    """ConstantOfShape(Shape(s)) -> Mul(-1) -> Equal -> Where, Concat, Sub, Div, Slice, Range, Add: all host values"""
    nodes = [W.node("Shape", ["x"], ["s"]),
             W.node("Shape", ["s"], ["ss"]),
             W.node("ConstantOfShape", ["ss"], ["ones"], value=_i64([1])),
             W.node("Mul", ["ones", "m1"], ["neg"]),
             W.node("Equal", ["neg", "target"], ["eq"]),
             W.node("Where", ["eq", "ones", "target"], ["shape"]),
             W.node("Slice", ["s", "st", "en"], ["tail"]),
             W.node("Concat", ["tail", "shape"], ["cat"], axis=0),
             W.node("Sub", ["cat", "one"], ["sub"]),
             W.node("Div", ["sub", "two"], ["div"]),
             W.node("Gather", ["s", "zero"], ["d0"], axis=0),
             W.node("Add", ["d0", "one"], ["lim"]),
             W.node("Range", ["zero", "lim", "one"], ["pos"])]
    inits = [W.tensor("m1", _i64(-1)), W.tensor("target", _i64([-1, 7, -1])), W.tensor("st", _i64([-2])), W.tensor("en", _i64([2 ** 40])),
             W.tensor("one", _i64(1)), W.tensor("two", _i64(2)), W.tensor("zero", _i64(0))]
    data = W.model(nodes, inits, [W.value_info("x", W.FLOAT, [2, 3, 5])], [W.value_info(n, W.INT64, []) for n in ("div", "pos", "shape")])
    from rten_b200.model import Model
    ctx = gc.new_ctx(rt)
    m = Model(ctx, data)
    x = ctx.to_device(np.zeros((2, 3, 5), F32))
    ctx.sync()
    n0 = ctx.launches
    div, pos, shape = [t.numpy() for t in m.run({"x": x}, ["div", "pos", "shape"])]
    ctx.sync()
    assert ctx.launches == n0
    s = np.array([2, 3, 5])
    ones = np.ones(3, np.int64)
    shp = np.where(mo.host_arith("Mul", ones, -1) == np.array([-1, 7, -1]), ones, np.array([-1, 7, -1]))
    cat = np.concatenate([s[-2:], shp])
    assert shape.tolist() == shp.tolist()
    assert div.tolist() == mo.host_arith("Div", mo.host_arith("Sub", cat, 1), 2).tolist()
    assert pos.tolist() == [0, 1, 2]


def test_slice_and_split_views_launch_nothing(rt):
    nodes = [W.node("Split", ["x", "sizes"], ["q", "k", "v"], axis=2),
             W.node("Slice", ["x", "st", "en", "ax", "sp"], ["w"]),
             W.node("Add", ["q", "k"], ["qk"]),
             W.node("Mul", ["v", "w"], ["vw"])]
    inits = [W.tensor("sizes", _i64([8, 8, 8])), W.tensor("st", _i64([0, 0])), W.tensor("en", _i64([2 ** 40, 16])),
             W.tensor("ax", _i64([1, 2])), W.tensor("sp", _i64([1, 2]))]
    data = W.model(nodes, inits, [W.value_info("x", W.FLOAT, [2, 5, 24])],
                   [W.value_info(n, W.FLOAT, []) for n in ("qk", "vw")], opset=14)
    from rten_b200.model import Model
    ctx = gc.new_ctx(rt)
    m = Model(ctx, data)
    x = np.random.default_rng(3).standard_normal((2, 5, 24)).astype(F32)
    xd = ctx.to_device(x)
    ctx.sync()
    n0 = ctx.launches
    qk, vw = [t.numpy() for t in m.run({"x": xd}, ["qk", "vw"])]
    ctx.sync()
    assert ctx.launches - n0 == 2  # the Add and the Mul only
    q, k, v = mo.split(x, 2, [8, 8, 8])
    gc.assert_bit_exact(qk, q + k, "q + k")
    gc.assert_bit_exact(vw, v * mo.slice_(x, [0, 0], [2 ** 31 - 1, 16], [1, 2], [1, 2]), "v * w")


def _llama_block():
    """the Llama mask, rotate_half and repeat_kv code as torch exports it (opset 14), without the slice assignment"""
    B, H, KV, T, D = 2, 4, 2, 6, 8
    nodes = [
        # causal mask: full((T, T), min) -> Trilu(upper, k=1) ; padding mask from attention_mask
        W.node("Shape", ["ids"], ["ids_shape"]),
        W.node("Gather", ["ids_shape", "one"], ["T"], axis=0),
        W.node("Unsqueeze", ["T", "ax0"], ["T1"]),
        W.node("Concat", ["T1", "T1"], ["TT"], axis=0),
        W.node("ConstantOfShape", ["TT"], ["full"], value=np.array([-3.0e38], F32)),
        W.node("Trilu", ["full", "one"], ["causal"], upper=1),
        W.node("Range", ["zero", "T", "one"], ["pos"]),
        W.node("Unsqueeze", ["pos", "ax1"], ["pos_col"]),
        W.node("Greater", ["pos", "pos_col"], ["future"]),
        W.node("Cast", ["future"], ["future_b"], to=9),
        W.node("Equal", ["mask", "zero32"], ["pad"]),
        W.node("Unsqueeze", ["pad", "ax12"], ["pad4"]),
        W.node("Or", ["pad4", "future_b"], ["masked"]),
        W.node("Not", ["masked"], ["keep"]),
        W.node("Where", ["keep", "scores", "minval"], ["scores_m"]),
        W.node("Where", ["future_b", "causal", "zerof"], ["causal_m"]),
        W.node("Add", ["scores_m", "causal_m"], ["att"]),
        # rotate_half
        W.node("Slice", ["q", "zero", "half", "axm1"], ["x1"]),
        W.node("Slice", ["q", "half", "big", "axm1"], ["x2"]),
        W.node("Neg", ["x2"], ["nx2"]),
        W.node("Concat", ["nx2", "x1"], ["rot"], axis=-1),
        # repeat_kv: the expand pattern ConstantOfShape(Shape(s)) -> Mul(-1) -> Equal -> Where -> Expand
        W.node("Unsqueeze", ["kv", "ax2"], ["kv5"]),
        W.node("Shape", ["target"], ["tshape"]),
        W.node("ConstantOfShape", ["tshape"], ["ones"], value=np.array([1], np.int64)),
        W.node("Mul", ["ones", "m1"], ["negs"]),
        W.node("Equal", ["target", "negs"], ["is_neg"]),
        W.node("Where", ["is_neg", "ones", "target"], ["eshape"]),
        W.node("Expand", ["kv5", "eshape"], ["kv_rep"]),
        W.node("Reshape", ["kv_rep", "flat_shape"], ["kv_out"]),
        W.node("Split", ["kv_out", "split2"], ["k_half", "v_half"], axis=1),
        W.node("Sub", ["k_half", "v_half"], ["kv_diff"]),
    ]
    inits = [W.tensor("one", np.array(1, np.int64)), W.tensor("zero", np.array(0, np.int64)), W.tensor("ax0", _i64([0])),
             W.tensor("ax1", _i64([1])), W.tensor("ax12", _i64([1, 2])), W.tensor("ax2", _i64([2])), W.tensor("axm1", _i64([-1])),
             W.tensor("zero32", np.array(0, np.int32)), W.tensor("minval", np.array(-3.0e38, F32)), W.tensor("zerof", np.array(0.0, F32)),
             W.tensor("half", _i64([D // 2])), W.tensor("big", _i64([2 ** 62])), W.tensor("m1", np.array(-1, np.int64)),
             W.tensor("target", _i64([B, KV, H // KV, T, D])), W.tensor("flat_shape", _i64([B, H, T, D])), W.tensor("split2", _i64([H // 2, H // 2]))]
    ins = [W.value_info("ids", W.INT32, [B, T]), W.value_info("mask", W.INT32, [B, T]), W.value_info("scores", W.FLOAT, [B, H, T, T]),
           W.value_info("q", W.FLOAT, [B, H, T, D]), W.value_info("kv", W.FLOAT, [B, KV, T, D])]
    outs = [W.value_info(n, W.FLOAT, []) for n in ("att", "rot", "kv_out", "kv_diff")]
    return W.model(nodes, inits, ins, outs, opset=14), (B, H, KV, T, D)


def test_llama_block_node_by_node(rt):
    from rten_b200.model import Model
    data, (B, H, KV, T, D) = _llama_block()
    r = np.random.default_rng(11)
    mask = np.ones((B, T), I32)
    mask[1, 4:] = 0
    feeds = dict(ids=r.integers(0, 50, (B, T)).astype(I32), mask=mask, scores=r.standard_normal((B, H, T, T)).astype(F32),
                 q=r.standard_normal((B, H, T, D)).astype(F32), kv=r.standard_normal((B, KV, T, D)).astype(F32))
    # the oracle, node by node
    causal = mo.trilu(np.full((T, T), F32(-3.0e38), F32), 1, True)
    pos = mo.range_(0, T, 1, I32)
    future = mo.compare("Greater", pos, pos[:, None])
    pad = mo.compare("Equal", mask, np.int32(0))[:, None, None, :]
    keep = mo.not_(mo.logical("Or", pad, future))
    att = mo.where(keep, feeds["scores"], F32(-3.0e38)) + mo.where(future, causal, F32(0))
    q = feeds["q"]
    rot = np.concatenate([-mo.slice_(q, [D // 2], [2 ** 31 - 1], [-1]), mo.slice_(q, [0], [D // 2], [-1])], -1)
    target = np.array([B, KV, H // KV, T, D])
    eshape = mo.where(mo.compare("Equal", target, mo.host_arith("Mul", np.ones(5), -1)), np.ones(5, I32), target)
    kv_out = mo.expand(feeds["kv"][:, :, None], eshape).reshape(B, H, T, D)
    kh, vh = mo.split(kv_out, 1, [H // 2, H // 2])
    for tf32 in (True, False):
        ctx = gc.new_ctx(rt, tf32=tf32)
        m = Model(ctx, data)
        got = [t.numpy() for t in m.run(feeds, ["att", "rot", "kv_out", "kv_diff"])]
        for g, e, n in zip(got, [att, rot, kv_out, kh - vh], ("att", "rot", "kv_out", "kv_diff")):
            gc.assert_bit_exact(g, e.astype(g.dtype), f"{n} tf32={tf32}")


def test_constant_of_shape_fill(rt):
    """an f32 ConstantOfShape is one fill launch (16-byte stores, then a partial tail); an integer one is a host value"""
    from rten_b200.model import Model
    nodes = [W.node("ConstantOfShape", ["shp"], ["f"], value=np.array([-2.5], F32)), W.node("ConstantOfShape", ["shp"], ["i"], value=_i64([7])),
             W.node("ConstantOfShape", ["shp"], ["z"])]
    data = W.model(nodes, [W.tensor("shp", _i64([3, 1027]))], [], [W.value_info(n, W.FLOAT, []) for n in ("f", "i", "z")])
    ctx = gc.new_ctx(rt)
    m = Model(ctx, data)
    ctx.sync()
    n0 = ctx.launches
    f, i, z = [t.numpy() for t in m.run({}, ["f", "i", "z"])]
    ctx.sync()
    assert ctx.launches - n0 == 2  # the two f32 fills
    gc.assert_bit_exact(f, np.full((3, 1027), -2.5, F32), "f32 fill")
    gc.assert_bit_exact(z, np.zeros((3, 1027), F32), "default fill")
    assert i.dtype == I32 and (i == 7).all() and i.shape == (3, 1027)


def test_onnx_domain_only(rt):
    from rten_b200.model import Model
    ctx = gc.new_ctx(rt)
    for op in ("Where", "Equal", "Expand", "Slice", "Split", "Range", "ConstantOfShape", "Trilu", "Not"):
        data = W.model([W.node(op, ["x"], ["y"], domain="com.microsoft")], [], [W.value_info("x", W.FLOAT, [2])],
                       [W.value_info("y", W.FLOAT, [2])], extra_opsets=[("com.microsoft", 1)])
        with pytest.raises(Exception, match=f"unsupported operator com.microsoft.{op}"):
            Model(ctx, data)


def test_errors_free_outputs_and_leave_the_context_usable(rt):
    """every error path of the C ABI through NULL outputs: the reference's message, and no output left allocated"""
    import ctypes as C
    from rten_b200.ops import _Args
    ctx = gc.new_ctx(rt)
    f = ctx.to_device(np.ones((2, 3), F32))
    i32 = lambda v: (C.c_int32 * max(len(v), 1))(*v)  # noqa: E731
    calls = [
        (lambda A, o: ctx.lib.rten_b200_trilu(ctx.handle, A.t(np.ones(4, F32)), 0, 1, C.byref(o[0])), INVALID_VALUE, "Input must have >= 2 dims"),
        (lambda A, o: ctx.lib.rten_b200_slice(ctx.handle, A.t(f), i32([0]), i32([1]), i32([2]), None, 1, C.byref(o[0])), INVALID_VALUE, "Axis is invalid"),
        (lambda A, o: ctx.lib.rten_b200_slice(ctx.handle, A.t(f), i32([0, 0, 0]), i32([1, 1, 1]), i32([0, 1, 1]), None, 3, C.byref(o[0])),
         INVALID_VALUE, "`axes` length must be <= input rank"),
        (lambda A, o: ctx.lib.rten_b200_slice(ctx.handle, A.t(f), i32([0]), i32([1]), None, None, 1, C.byref(o[0])), INVALID_VALUE,
         "`starts` length must match axis count"),
        (lambda A, o: ctx.lib.rten_b200_split(ctx.handle, A.t(f), 1, i32([4, -1]), 2, 0, o, 4, C.byref(C.c_int32())), INVALID_VALUE,
         "Split sizes must be >= 0"),
        (lambda A, o: ctx.lib.rten_b200_split(ctx.handle, A.t(f), 1, None, 0, 0, o, 4, C.byref(C.c_int32())), INVALID_VALUE, "num_outputs must be > 0"),
        (lambda A, o: ctx.lib.rten_b200_split(ctx.handle, A.t(f), 1, i32([1, 1, 1]), 3, 0, o, 2, C.byref(C.c_int32())), INVALID_VALUE,
         "more pieces than there are outputs"),
        (lambda A, o: ctx.lib.rten_b200_expand(ctx.handle, A.t(f), (C.c_int64 * 2)(2, 4), 2, C.byref(o[0])), INCOMPATIBLE,
         "Cannot broadcast input with target shape"),
        (lambda A, o: ctx.lib.rten_b200_where(ctx.handle, A.t(np.ones((2, 4), I32)), A.t(f), A.t(f), C.byref(o[0])), INCOMPATIBLE,
         "Cannot broadcast inputs"),
    ]
    for fn, status, msg in calls:
        A = _Args(ctx)
        outs = (rt._lib.RtenTensor * 4)()
        st = fn(A, outs)
        err = ctx.lib.rten_b200_last_error(ctx.handle).decode()
        assert st == status and msg in err, (msg, st, err)
        assert all(not o.data for o in outs), f"{msg}: an output is still allocated"
    gc.assert_bit_exact(rt.Not().run(ctx, np.array([0, 3], I32)).numpy(), np.array([1, 0], I32), "after the failures")


@pytest.mark.parametrize("case", ["range delta 0", "negative ConstantOfShape dim", "host Div by zero", "host INT_MIN / -1",
                                  "Split pieces != outputs"])
def test_executor_errors(rt, case):
    from rten_b200.model import Model
    nodes, inits, want = {
        "range delta 0": ([W.node("Range", ["a", "b", "c"], ["y"])], [W.tensor("a", _i64(0)), W.tensor("b", _i64(5)), W.tensor("c", _i64(0))],
                          "delta must be non-zero"),
        "negative ConstantOfShape dim": ([W.node("ConstantOfShape", ["a"], ["y"], value=_i64([1]))], [W.tensor("a", _i64([2, -1]))], "Invalid shape"),
        "host Div by zero": ([W.node("Div", ["a", "b"], ["y"])], [W.tensor("a", _i64([4, 6])), W.tensor("b", _i64([2, 0]))], "Divisor contains zero"),
        "host INT_MIN / -1": ([W.node("Div", ["a", "b"], ["y"])], [W.tensor("a", _i64([-2 ** 31, 6])), W.tensor("b", _i64([-1]))],
                              "Divisor contains zero"),
        "Split pieces != outputs": ([W.node("Split", ["x"], ["y", "z", "w"], axis=1, num_outputs=3)], [W.tensor("x", np.ones((2, 4), F32))],
                                    "2 pieces for 3 outputs"),
    }[case]
    data = W.model(nodes, inits, [], [W.value_info("y", W.INT64, [])], opset=18)
    ctx = gc.new_ctx(rt)
    m = Model(ctx, data)
    with pytest.raises(Exception) as e:
        m.run({}, ["y"])
    assert want in e.value.msg, (case, e.value.msg)


def test_host_div_overflow_is_positional(rt):
    """INT_MIN in a and -1 in b that never meet after broadcasting divide fine"""
    from rten_b200.model import Model
    data = W.model([W.node("Div", ["a", "b"], ["y"])], [W.tensor("a", _i64([[-2 ** 31, 6]])), W.tensor("b", _i64([[3, -1]]))], [],
                   [W.value_info("y", W.INT64, [])])
    ctx = gc.new_ctx(rt)
    y = Model(ctx, data).run({}, ["y"])[0].numpy()
    assert y.tolist() == [[int(-2 ** 31 / 3), -6]]
