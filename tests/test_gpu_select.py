"""`pytest -m gpu`: TopK, ArgMax and ArgMin (topk.cu, reduce.cu's arg-reduce kernels) bit for bit against oracle/select.py,
every kernel path by name, the executor's TopK / ArgMax / ArgMin nodes, and the Generator's device sampling.

  * kernel identity (CUPTI, in a child process): the warp TopK kernel (n <= 1024), the cluster TopK kernel holding its
    slices in shared memory at several cluster sizes, the same kernel re-reading global memory (n = 2^20 + 3), and the
    arg-reduce warp / CTA / cluster kernels, each for the rows that select it;
  * values and indices bit-exact for f32 and i32, k in {0, 1, 2, 8, 50, 100, 1024, 2048} and k = n, largest 0 / 1,
    sorted = 0 (the output is sorted anyway; compared as sets too), a non-last axis, the Generator's strided
    last-position view, heavy ties, one and several NaNs, +-0 and +-inf;
  * the reference's errors, and k > 2048 refused as unsupported;
  * small ONNX graphs: TopK with a constant K, K from Shape -> Gather and the opset-9 `k` attribute; ArgMax / ArgMin with
    keepdims 0 / 1 and a negative axis; select_last_index = 1 refused at load;
  * Generator(ModelDecoder(...)) over the int4 decoder fixture: the device path and the host path (an identity logits
    filter) give the same tokens and the same last_logits for ArgMaxSampler and TopKSampler; TopKSampler's two paths on
    seeded 8 x 128256 logits."""
import json
import os
import re
import sys

import numpy as np
import pytest

import genai_decoder as gd
import gpu_checks as gc
import onnx_writer as W
import test_gpu_row_kernels as rk
from oracle import select as S

pytestmark = pytest.mark.gpu

F32, I32 = np.float32, np.int32
KERNELS = {"topk_warp_kernel", "topk_cluster_kernel", "arg_reduce_warp_kernel", "arg_reduce_cta_kernel",
           "arg_reduce_cluster_kernel"}


@pytest.fixture(scope="module")
def rt():
    import rten_b200
    from rten_b200 import _lib
    _lib.load()
    return rten_b200


@pytest.fixture(scope="module")
def ctx(rt):
    return rt.Context(0)


def _logits(rows, n, seed, dtype=F32):
    r = np.random.default_rng(seed)
    if dtype == I32:
        return r.integers(-2**31, 2**31 - 1, (rows, n), dtype=np.int64).astype(I32)
    return r.standard_normal((rows, n)).astype(F32) * F32(4)


def _check_topk(rt, ctx, x, k, axis=-1, largest=True, what="", xd=None):
    v, i = rt.TopK(axis=axis, largest=largest).run(ctx, x if xd is None else xd, k)
    ev, ei = S.topk(x, k, axis, largest)
    gc.assert_bit_exact(i.numpy(), ei, f"{what} indices")
    gc.assert_bit_exact(v.numpy(), ev, f"{what} values")


# ---- kernel identity --------------------------------------------------------------------------------------------------
_NAME = re.compile(r"::(\w+)<([^<>]*)>\(")


def kernel_key(name):
    """(kernel, template arguments) of a demangled kernel name (`<float, false>` from CUPTI or `<float, (bool)0>`), else
    None.  The kernels live in anonymous namespaces, which test_gpu_row_kernels.kernel_key does not read."""
    for m in _NAME.finditer(name):
        if m.group(1) in KERNELS:
            args = []
            for a in m.group(2).split(","):
                a = re.sub(r"^\(bool\)", "", a.strip())
                args.append({"true": 1, "false": 0, "1": 1, "0": 0}.get(a, a))
            return m.group(1), tuple(args)
    return None


# (label, rows, n, k, expected kernel); "arg" cases run ArgMax
def probe_cases(sms):
    out = [(f"topk warp n={n}", 16, n, 2, ("topk_warp_kernel", ("float",))) for n in (8, 64, 1000)]
    for n in (1025, 32000, 50257, 128256):
        for b in (1, 8, 64):
            out.append((f"topk cluster n={n} B={b}", b, n, 50, ("topk_cluster_kernel", ("float", 0))))
    out.append(("topk gmem n=2^20+3", 2, 2**20 + 3, 100, ("topk_cluster_kernel", ("float", 1))))
    out.append(("topk k=1 -> arg cluster", 8, 128256, 1, ("arg_reduce_cluster_kernel", ("float",))))
    out.append(("arg warp", 64, 1000, "arg", ("arg_reduce_warp_kernel", ("float",))))
    out.append(("arg cta", 4 * sms, 5000, "arg", ("arg_reduce_cta_kernel", ("float",))))
    out.append(("arg cluster", 2, 128256, "arg", ("arg_reduce_cluster_kernel", ("float",))))
    out.append(("arg cluster, strided lanes", 2, 128256, "arg0", ("arg_reduce_cluster_kernel", ("float",))))
    return out


def _kernel_probe():
    import rten_b200 as rt
    import torch
    ctx = rt.Context(0)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    names = {}
    for label, rows, n, k, _ in probe_cases(sms):
        x = ctx.to_device(_logits(rows, n, 5))
        if k == "arg":
            fn = lambda: rt.ArgMax(axis=1).run(ctx, x)
        elif k == "arg0":  # lanes down the columns of [n, rows]: stride `rows`
            x = ctx.to_device(np.ascontiguousarray(_logits(rows, n, 5).T))
            fn = lambda: rt.ArgMax(axis=0).run(ctx, x)
        else:
            fn = lambda: rt.TopK().run(ctx, x, k)
        fn()
        ctx.sync()
        _, got = gc._kernels_launched(fn)
        names[label] = sorted(got)
    print(json.dumps({"sms": sms, "names": names}))


def test_kernel_identity():
    out = rk.probe_in_child("test_gpu_select")
    sms, names = out["sms"], out["names"]
    wrong, seen = [], set()
    for label, _, _, _, want in probe_cases(sms):
        ran = {kernel_key(n) for n in names[label]} - {None}
        seen |= ran
        if ran != {want}:
            wrong.append((label, want, sorted(ran)))
    assert not wrong, wrong
    assert {k for k, _ in seen} == KERNELS


# ---- values -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [F32, I32])
@pytest.mark.parametrize("n", [8, 64, 1000, 1025, 32000, 128256])
def test_topk_bit_exact(rt, ctx, dtype, n):
    for rows in (1, 8) if n > 1024 else (1, 8, 300):
        x = _logits(rows, n, n + rows, dtype)
        xd = ctx.to_device(x)
        ks = sorted({k for k in (0, 1, 2, 8, 50, 100, 1024, 2048) if k <= n} | ({n} if n <= 2048 else set()))
        for k in ks:
            for largest in (True, False):
                _check_topk(rt, ctx, x, k, -1, largest, f"{dtype.__name__} {rows}x{n} k={k} largest={largest}", xd)


def test_topk_many_rows_and_gmem(rt, ctx):
    x = _logits(64, 50257, 3)
    _check_topk(rt, ctx, x, 50, what="64 x 50257")
    x = _logits(2, 2**20 + 3, 4)
    for k in (2, 100, 2048):
        _check_topk(rt, ctx, x, k, what=f"2 x 2^20+3 k={k}")
    _check_topk(rt, ctx, x, 7, largest=False, what="2 x 2^20+3 smallest")


def test_topk_unsorted_as_sets(rt, ctx):
    x = _logits(8, 32000, 9)
    v, i = rt.TopK(sorted=False).run(ctx, x, 50)
    ev, ei = S.topk(x, 50)
    assert all(set(a) == set(b) for a, b in zip(i.numpy().tolist(), ei.tolist()))
    assert all(sorted(a) == sorted(b) for a, b in zip(v.numpy().tolist(), ev.tolist()))


def test_topk_axis_and_strided_views(rt, ctx):
    r = np.random.default_rng(11)
    x = r.standard_normal((3, 2000, 5)).astype(F32)
    for k in (1, 2, 50):
        _check_topk(rt, ctx, x, k, axis=1, what=f"axis 1 k={k}")
        _check_topk(rt, ctx, x, k, axis=-2, largest=False, what=f"axis -2 smallest k={k}")
    _check_topk(rt, ctx, x[:, :4, :], 3, axis=0, what="axis 0")
    # the Generator's last-position view of [B, T, vocab] logits: rows T * vocab apart
    B, T, V = 4, 3, 32000
    lg = r.standard_normal((B, T, V)).astype(F32)
    d = ctx.to_device(lg)
    view = d.view((B, V), (T * V, 1), (T - 1) * V)
    for k in (1, 5, 50):
        _check_topk(rt, ctx, lg[:, -1], k, what=f"last-position view k={k}", xd=view)
    gc.assert_bit_exact(rt.ArgMax(axis=-1, keep_dims=False).run(ctx, view).numpy(), S.arg_max(lg[:, -1], -1, False), "argmax view")
    # lanes that start off a 16-byte boundary take the scalar loads of the arg-reduce kernels
    mis = d.view((B, V - 1), (T * V, 1), 1)
    for op, ref in ((rt.ArgMax, S.arg_max), (rt.ArgMin, S.arg_min)):
        gc.assert_bit_exact(op(axis=1).run(ctx, mis).numpy(), ref(lg[:, 0, 1:], 1), f"{op.__name__} misaligned")


def _special_rows(n, seed):
    r = np.random.default_rng(seed)
    rows = [r.integers(0, 3, n).astype(F32),                                     # a few distinct values
            np.where(r.random(n) < 0.5, F32(0.0), F32(-0.0)).astype(F32),        # +-0 only
            r.choice(np.array([np.inf, -np.inf, 1.0, -1.0], F32), n)]
    one_nan = r.standard_normal(n).astype(F32)
    one_nan[n // 3] = np.nan
    many_nan = r.integers(0, 4, n).astype(F32)
    many_nan[r.random(n) < 0.05] = np.nan
    return np.stack(rows + [one_nan, many_nan])


@pytest.mark.parametrize("n", [64, 1000, 5000, 128256])
def test_special_values(rt, ctx, n):
    x = _special_rows(n, n)
    xd = ctx.to_device(x)
    for k in (1, 2, 50, min(n, 2048)):
        for largest in (True, False):
            _check_topk(rt, ctx, x, k, -1, largest, f"special n={n} k={k} largest={largest}", xd)
    for keep in (True, False):
        gc.assert_bit_exact(rt.ArgMax(axis=1, keep_dims=keep).run(ctx, xd).numpy(), S.arg_max(x, 1, keep), f"argmax n={n}")
        gc.assert_bit_exact(rt.ArgMin(axis=1, keep_dims=keep).run(ctx, xd).numpy(), S.arg_min(x, 1, keep), f"argmin n={n}")
    xi = np.random.default_rng(n).integers(-3, 3, (4, n)).astype(I32)
    xi[0, :2] = [-2**31, 2**31 - 1]
    for k in (1, 2, 50):
        _check_topk(rt, ctx, xi, k, what=f"i32 ties n={n} k={k}")
    gc.assert_bit_exact(rt.ArgMax(axis=-1).run(ctx, xi).numpy(), S.arg_max(xi, -1), f"argmax i32 n={n}")
    gc.assert_bit_exact(rt.ArgMin(axis=-1).run(ctx, xi).numpy(), S.arg_min(xi, -1), f"argmin i32 n={n}")


@pytest.mark.parametrize("shape,axis", [((300, 1000), 1), ((4 * 132, 5000), 1), ((2, 128256), 1), ((1, 128256), -1),
                                        ((1000, 7), 0), ((3, 5, 2000), 1), ((6,), 0),
                                        ((128256, 2), 0), ((5000, 300), 0)])  # strided cluster / CTA lanes
def test_arg_reduce_paths(rt, ctx, shape, axis):
    x = np.random.default_rng(len(shape)).standard_normal(shape).astype(F32)
    x = np.round(x * 2).astype(F32)  # ties everywhere
    xd = ctx.to_device(x)
    for keep in (True, False):
        gc.assert_bit_exact(rt.ArgMax(axis=axis, keep_dims=keep).run(ctx, xd).numpy(), S.arg_max(x, axis, keep), f"argmax {shape}")
        gc.assert_bit_exact(rt.ArgMin(axis=axis, keep_dims=keep).run(ctx, xd).numpy(), S.arg_min(x, axis, keep), f"argmin {shape}")


def test_lanes_past_the_grid(rt, ctx):
    """More lanes than the grid has warps, CTAs or clusters: each loops over several lanes, reusing its shared memory
    (up to 148 SMs: the warp kernels' grids hold at most 9472 lanes, the arg-reduce CTA kernel's 1184, the cluster TopK
    kernel's 65535 clusters)"""
    for rows, n, k in ((10000, 8, 2), (10000, 64, 8), (10000, 16, 1), (2000, 1100, 1)):
        x = _logits(rows, n, rows + n)
        xd = ctx.to_device(x)
        _check_topk(rt, ctx, x, k, what=f"{rows} x {n} k={k}", xd=xd)
        gc.assert_bit_exact(rt.ArgMin(axis=1).run(ctx, xd).numpy(), S.arg_min(x, 1), f"argmin {rows} x {n}")
    ties = np.random.default_rng(1).integers(0, 3, (10000, 64)).astype(F32)
    _check_topk(rt, ctx, ties, 8, what="10000 x 64 ties")
    # 65540 rows of 1025: one-CTA clusters, the grid's 65535 clusters take the last rows on a second pass
    x = _logits(65540, 1025, 12)
    v, i = rt.TopK().run(ctx, x, 2)
    v, i = v.numpy(), i.numpy()
    for lo, hi in ((0, 8), (65528, 65540)):
        ev, ei = S.topk(x[lo:hi], 2)
        gc.assert_bit_exact(i[lo:hi], ei, f"65540 x 1025 rows {lo}:{hi} indices")
        gc.assert_bit_exact(v[lo:hi], ev, f"65540 x 1025 rows {lo}:{hi} values")


def test_errors(rt, ctx):
    x = _logits(2, 10, 1)
    # an axis of 2^31 elements (a zero-stride view of one element): the i32 indices cannot hold it
    one = ctx.to_device(np.zeros(1, F32))
    huge = one.view((2**31,), (0,))
    with pytest.raises(rt.OpError, match="2\\^31"):
        rt.TopK().run(ctx, huge, 2)
    with pytest.raises(rt.OpError, match="2\\^31"):
        rt.ArgMax().run(ctx, huge)
    with pytest.raises(rt.OpError, match="k > dimension size"):
        rt.TopK().run(ctx, x, 11)
    with pytest.raises(rt.OpError, match="2048"):
        rt.TopK().run(ctx, _logits(1, 5000, 1), 2049)
    with pytest.raises(rt.OpError, match="Axis is invalid"):
        rt.TopK().run(ctx, np.array(1.0, F32), 1)
    with pytest.raises(rt.OpError, match="Axis is invalid"):
        rt.ArgMax().run(ctx, np.array(1.0, F32))
    with pytest.raises(rt.OpError, match="empty sequence"):
        rt.ArgMax(axis=1).run(ctx, np.zeros((10, 0, 5), F32))
    assert rt.ArgMax(axis=0, keep_dims=False).run(ctx, np.zeros((10, 0, 5), F32)).shape == (0, 5)
    v, i = rt.TopK().run(ctx, x, 0)
    assert v.shape == (2, 0) and i.shape == (2, 0)


# ---- golden cases through the device ------------------------------------------------------------------------------------
def test_golden_cases(rt, ctx):
    here = os.path.dirname(os.path.abspath(__file__))
    for c in json.load(open(os.path.join(here, "golden", "select_cases.json")))["cases"]:
        x = np.array([np.nan if v == "nan" else v for v in c["input"]], F32).reshape(c["shape"])
        if c["op"] == "TopK":
            run = lambda: rt.TopK(axis=-1 if c["axis"] is None else c["axis"], largest=c["largest"]).run(ctx, x, c["k"])
        else:
            op = rt.ArgMax if c["op"] == "ArgMax" else rt.ArgMin
            run = lambda: (None, op(axis=c["axis"], keep_dims=c["keep_dims"]).run(ctx, x))
        if c["error"]:
            with pytest.raises(rt.OpError, match=c["error"]):
                run()
            continue
        v, i = run()
        gc.assert_bit_exact(i.numpy(), np.array(c["indices"], I32).reshape(c["out_shape"]), c["name"])
        if v is not None:
            want = np.array([np.nan if e == "nan" else e for e in c["values"]], F32).reshape(c["out_shape"])
            gc.assert_bit_exact(v.numpy(), want, c["name"])


# ---- executor -----------------------------------------------------------------------------------------------------------
def _run_graph(rt, ctx, nodes, inits, x, outs, out_types):
    from rten_b200.model import Model
    m = Model(ctx, W.model(nodes, inits, [W.value_info("x", W.FLOAT, list(x.shape))],
                           [W.value_info(n, t, []) for n, t in zip(outs, out_types)]))
    return [t.numpy() for t in m.run({"x": x}, outs)]


def test_executor_topk(rt, ctx):
    x = _logits(4, 3000, 21)
    ev, ei = S.topk(x, 7)
    v, i = _run_graph(rt, ctx, [W.node("TopK", ["x", "k"], ["v", "i"])], [W.tensor("k", np.array([7], np.int64))],
                      x, ["v", "i"], [W.FLOAT, W.INT64])
    gc.assert_bit_exact(v, ev, "constant K values")
    gc.assert_bit_exact(i, ei, "constant K indices")
    # K = x.shape[0] through Shape -> Gather, smallest along axis 0
    ev, ei = S.topk(x, 4, 0, False)
    v, i = _run_graph(rt, ctx, [W.node("Shape", ["x"], ["s"]), W.node("Gather", ["s", "zero"], ["k"], axis=0),
                                W.node("TopK", ["x", "k"], ["v", "i"], axis=0, largest=0)],
                      [W.tensor("zero", np.array([0], np.int64))], x, ["v", "i"], [W.FLOAT, W.INT64])
    gc.assert_bit_exact(v, ev, "Shape -> Gather K values")
    gc.assert_bit_exact(i, ei, "Shape -> Gather K indices")
    # opset 9: k is an attribute
    from rten_b200.model import Model
    m = Model(ctx, W.model([W.node("TopK", ["x"], ["v", "i"], k=3)], [], [W.value_info("x", W.FLOAT, list(x.shape))],
                           [W.value_info("v", W.FLOAT, []), W.value_info("i", W.INT64, [])], opset=9))
    v, i = [t.numpy() for t in m.run({"x": x}, ["v", "i"])]
    ev, ei = S.topk(x, 3)
    gc.assert_bit_exact(v, ev, "opset 9 values")
    gc.assert_bit_exact(i, ei, "opset 9 indices")


def test_executor_arg_reduce(rt, ctx):
    x = np.round(_logits(6, 40, 22)).astype(F32)
    for op, ref in (("ArgMax", S.arg_max), ("ArgMin", S.arg_min)):
        for keep in (0, 1):
            for axis in (-1, 0):
                (y,) = _run_graph(rt, ctx, [W.node(op, ["x"], ["y"], axis=axis, keepdims=keep)], [], x, ["y"], [W.INT64])
                gc.assert_bit_exact(y, ref(x, axis, bool(keep)), f"{op} axis {axis} keepdims {keep}")
    from rten_b200.model import Model
    with pytest.raises(rt.OpError, match="select_last_index"):
        Model(ctx, W.model([W.node("ArgMax", ["x"], ["y"], select_last_index=1)], [], [W.value_info("x", W.FLOAT, [2, 3])],
                           [W.value_info("y", W.INT64, [])]))


# ---- Generator ------------------------------------------------------------------------------------------------------------
def _generate(m, B, prompt, sampler, host, steps):
    from rten_b200.generate import Generator, ModelDecoder
    gen = Generator(ModelDecoder(m, B, 64)).with_prompt(prompt).with_sampler(sampler)
    if host:
        gen = gen.with_logits_filter(lambda logits, prev: logits)
    toks, logits = [], []
    for _ in range(steps):
        toks.append(next(gen))
        logits.append(gen.last_logits)
    return np.stack(toks, 1), logits


class _LogitsModel:
    """A model whose every step returns the next of a list of device logits [B, vocab]"""

    def __init__(self, logits):
        self.logits, self.step = logits, 0
        self.input_names, self.output_names = ["input_ids"], ["logits"]

    def run(self, inputs, outputs):
        self.step += 1
        return {"logits": self.logits[self.step - 1]}


def test_generator_topk_beyond_the_device_k(rt, ctx):
    """TopKSampler(k > 2048) keeps sampling on the host without filters, with the tokens of the filtered host path; k up
    to 2048 samples on the device with the same tokens"""
    from rten_b200.generate import Generator, TopKSampler
    r = np.random.default_rng(5)
    steps = [ctx.to_device(r.standard_normal((4, 32000)).astype(F32)) for _ in range(3)]
    for k in (3000, 2048, 50):
        toks = []
        for host in (False, True):
            gen = Generator(_LogitsModel(steps)).with_prompt(np.zeros((4, 1), I32)).with_sampler(TopKSampler(k, 0.9, 17))
            if host:
                gen = gen.with_logits_filter(lambda logits, prev: logits)
            toks.append(np.stack([next(gen) for _ in steps], 1))
            assert (gen._last_device is None) == (host or k > 2048), k  # which path ran
        assert np.array_equal(toks[0], toks[1]), k


def test_generator_device_sampling(rt, ctx):
    from rten_b200.generate import ArgMaxSampler, TopKSampler
    from rten_b200.model import Model
    from test_gpu_norms import DEC as c
    w = gd.genai_weights()
    m = Model(ctx, gd.genai_graph(w))
    B, steps = 2, 6
    prompt = np.random.default_rng(43).integers(0, c["V"], (B, 3)).astype(I32)
    for make in (ArgMaxSampler, lambda: TopKSampler(5, 0.8, 1234)):
        dt, dl = _generate(m, B, prompt, make(), False, steps)
        ht, hl = _generate(m, B, prompt, make(), True, steps)
        assert np.array_equal(dt, ht), (dt, ht)
        for s, (a, b) in enumerate(zip(dl, hl)):
            gc.assert_bit_exact(a, b, f"step {s} last_logits")


def test_topk_sampler_paths_agree(rt, ctx):
    from rten_b200.generate import TopKSampler
    x = _logits(8, 128256, 77)
    xd = ctx.to_device(x)
    a, b = TopKSampler(50, 0.7, 99), TopKSampler(50, 0.7, 99)
    for _ in range(3):
        assert np.array_equal(a.sample_device(xd), b.sample(x))


if __name__ == "__main__":
    sys.exit(pytest.main([__file__, "-q", "-m", "gpu"]))
