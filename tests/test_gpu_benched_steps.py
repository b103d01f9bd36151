"""`pytest -m gpu`: every operator call of the steps bench.py times, checked from its own inputs inside the replayed graph.

The benched steps -- ResNet-50 b32 and BERT-base b16 x 128 in both f32 modes, GPT-2 int8 b8 prefill of 512 tokens and 8
fused decode steps -- run their runners unmodified, with the autotune-then-capture order of gpu_checks._replayed.  While
a step is captured, a recorder wraps every `run`, `run_projected` and `run_chained` of rten_b200.ops and
`DeviceTensor.assign`, keeping each call's operator, attributes, input and output tensors (views included) and the
launch count before and after it.  After the replay every record is read back and checked against a reference computed
from that record's own inputs:

  * bit for bit against the oracle: LayerNormalization, GatherRows, the embedding Add, MaxPool, DynamicQuantizeLinear,
    MatMulIntegerToFloat with its fused epilogue and QuantizedLinear (the integer product itself is formed exactly in
    float64, benched_step_refs.int_matmul, and scaled by the oracle's cast_scale);
  * bit for bit as copies: the prefill's assigns into the K and V^T caches, and the decode Attention's append (row P is
    this step's key / value, rows before P are the previous step's readback, rows after P keep the NaN written into
    every cache before the prefill);
  * in float64 within a per-element bound (benched_step_refs): every f32 Conv call (run, run_projected, run_chained and
    its second output computed from the kernel's own y), BERT's FusedMatMul with bias, Gelu and residual, the
    GlobalAveragePool, the classifier Gemm, BERT's Attention, the prefill's FusedMatMul -> in-place AddSoftmax ->
    MatMul as one composite record, and the decode Attention (check_attention_decode's 2e-5 max |ref|).

Holding the records keeps the pool from reusing their buffers, so every step is also captured without the recorder:
both captures must issue the same number of launches and give the same output bits, and the unrecorded one keeps the
benched buffer reuse.  Every launch of the recorded step must lie inside a record that has a checker.  BERT's graph is
replayed once more after writing a padding mask (-10000 and -inf) and non-zero token types into its input buffers.
"""
import inspect
import math
import time

import numpy as np
import pytest

import benched_step_refs as R
import gpu_checks as gc

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def rt():
    import rten_b200
    from rten_b200 import _lib
    _lib.load()
    return rten_b200


# ---------------------------------------------------------------------------------------------------------------------
# the recorder


class Record:
    def __init__(self, kind, method, obj, attrs, args, sub_attrs, out, l0, l1):
        self.kind, self.method, self.obj, self.attrs, self.args = kind, method, obj, attrs, args
        self.sub_attrs, self.out, self.l0, self.l1 = sub_attrs, out, l0, l1

    @property
    def launches(self):
        return self.l1 - self.l0

    def __repr__(self):
        return f"{self.kind}.{self.method}"


class Recorder:
    """Wraps the operator entry points while installed; calls made between graph_begin and graph_end become records of
    `captures[-1]`.  A call made inside another recorded call (an operator built on another) belongs to the outer one."""

    def __init__(self):
        self.captures, self.active, self.depth = [], False, 0

    def install(self, mp, O):
        for cls in vars(O).values():
            if isinstance(cls, type) and cls.__module__ == O.__name__:
                for m in ("run", "run_projected", "run_chained"):
                    if m in cls.__dict__:
                        mp.setattr(cls, m, self._wrap(cls.__dict__[m], m))
        mp.setattr(O.DeviceTensor, "assign", self._wrap(O.DeviceTensor.assign, "assign"))
        begin, end = O.Context.graph_begin, O.Context.graph_end

        def graph_begin(ctx):
            begin(ctx)
            self.captures.append([])
            self.active = True

        def graph_end(ctx):
            self.active = False
            return end(ctx)

        mp.setattr(O.Context, "graph_begin", graph_begin)
        mp.setattr(O.Context, "graph_end", graph_end)

    def _wrap(self, fn, method):
        sig = inspect.signature(fn)

        def wrapped(obj, *args, **kwargs):
            if not self.active or self.depth:
                return fn(obj, *args, **kwargs)
            ctx = obj.ctx if method == "assign" else args[0]
            bound = sig.bind(obj, *args, **kwargs)
            bound.apply_defaults()
            named = {k: v for k, v in bound.arguments.items() if k not in ("self", "ctx")}
            # operators passed as arguments (a projection, the chained convolution): their attributes at call time
            sub = {k: dict(vars(v)) for k, v in named.items() if hasattr(v, "run") and not isinstance(v, type)}
            attrs = {} if method == "assign" else dict(vars(obj))
            l0 = ctx.launches
            self.depth += 1
            try:
                out = fn(obj, *args, **kwargs)
            finally:
                self.depth -= 1
            self.captures[-1].append(Record(type(obj).__name__, method, obj, attrs, named, sub, out, l0, ctx.launches))
            return out

        return wrapped


def _capture(ctx, fn):
    ctx.graph_begin()
    out = fn()
    return ctx.graph_end(), out


def _replay(ctx, g, out=None):
    """Replay `g` (after filling `out` with NaN when it is f32) and return the number of launches it issued."""
    if out is not None and out.dtype == np.float32:
        out.copy_from(np.full(out.shape, np.nan, np.float32))
    n = ctx.launches
    g.launch()
    ctx.sync()
    return ctx.launches - n


def _assert_same_bits(a, b, what):
    gc.assert_bit_exact(np.asarray(a), np.asarray(b), what)


# ---------------------------------------------------------------------------------------------------------------------
# checkers: each returns None (bit for bit) or the worst bound ratio, and raises when the record is wrong


def _t(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).to("cuda", torch.float64)


def _h(t):
    return None if t is None else t.numpy()


def _bounded(got, ref, bnd, what):
    import torch
    r = R.ratio(torch.from_numpy(np.ascontiguousarray(got)).to(ref.device), ref, bnd)
    assert r <= 1.0, f"{what}: outside the bound (worst ratio {r:.3f})"
    return r


def _col(b):
    return None if b is None else _t(_h(b)).reshape(1, -1, 1, 1)


def _conv_sum(x, w, attrs):
    return R.conv64(_t(_h(x)), _t(_h(w)), attrs["padding"], attrs["strides"], attrs["dilations"], attrs["groups"])


def chk_conv(env, r):
    a = r.args
    S, A = _conv_sum(a["x"], a["w"], r.attrs)
    res = None if a["residual"] is None else _t(_h(a["residual"]))
    ref, bnd = R.epilogue_ref_and_bound(S, A, env.tf32, _col(a["bias"]), res, r.attrs["activation"])
    return _bounded(_h(r.out), ref, bnd, f"{env.where(r)} Conv")


def _conv_first(env, r, what):
    """The first output of run_projected / run_chained: act(conv(x) + bias [+ residual | + proj(x_proj) + bias_proj])."""
    a = r.args
    S, A = _conv_sum(a["x"], a["w"], r.attrs)
    bias, res = _col(a["bias"]), None
    if a.get("proj") is not None:
        Sp, Ap = _conv_sum(a["x_proj"], a["w_proj"], r.sub_attrs["proj"])
        S, A = S + Sp, A + Ap
        if a["bias_proj"] is not None:
            bias = _col(a["bias_proj"]) if bias is None else bias + _col(a["bias_proj"])
    elif a.get("residual") is not None:
        res = _t(_h(a["residual"]))
    ref, bnd = R.epilogue_ref_and_bound(S, A, env.tf32, bias, res, r.attrs["activation"])
    y = r.out[0] if isinstance(r.out, tuple) else r.out
    return _bounded(_h(y), ref, bnd, f"{env.where(r)} {what} y")


def chk_conv_projected(env, r):
    return _conv_first(env, r, "Conv.run_projected")


def chk_conv_chained(env, r):
    """y as run_projected / run with a residual; z = nxt(y) from the y the kernel stored."""
    worst = _conv_first(env, r, "Conv.run_chained")
    y, z = r.out
    a, na = r.args, r.sub_attrs["nxt"]
    S, A = _conv_sum(y, a["w_next"], na)
    ref, bnd = R.epilogue_ref_and_bound(S, A, env.tf32, _col(a["bias_next"]), None, na["activation"])
    return max(worst, _bounded(_h(z), ref, bnd, f"{env.where(r)} Conv.run_chained z"))


def chk_max_pool(env, r):
    want = env.oracle.max_pool(_h(r.args["x"]), r.attrs["kernel_size"], list(r.attrs["padding"]), r.attrs["strides"])
    _assert_same_bits(_h(r.out), want, f"{env.where(r)} MaxPool")


def chk_global_average_pool(env, r):
    ref, bnd = R.global_average_pool_ref_and_bound(_t(_h(r.args["x"])))
    return _bounded(_h(r.out), ref, bnd, f"{env.where(r)} GlobalAveragePool")


def chk_gemm(env, r):
    at = r.attrs
    a, b = _t(_h(r.args["a"])), _t(_h(r.args["b"]))
    a, b = (a.T if at["transpose_a"] else a), (b.T if at["transpose_b"] else b)
    S, A = R.matmul64(a, b)
    c = r.args["c"]
    bias = None if c is None else at["beta"] * _t(_h(c))
    ref, bnd = R.epilogue_ref_and_bound(S, A, env.tf32, bias, None, R.ACT_NONE, alpha=at["alpha"])
    return _bounded(_h(r.out), ref, bnd, f"{env.where(r)} Gemm")


def chk_gather(env, r):
    _assert_same_bits(_h(r.out), _h(r.args["table"])[_h(r.args["indices"])], f"{env.where(r)} GatherRows")


def chk_add(env, r):
    _assert_same_bits(_h(r.out), env.oracle.add(_h(r.args["a"]), _h(r.args["b"])), f"{env.where(r)} Add")


def chk_layer_norm(env, r):
    want = env.oracle.layer_norm(_h(r.args["x"]), _h(r.args["scale"]), _h(r.args["bias"]), r.attrs["axis"],
                                 r.attrs["epsilon"])
    _assert_same_bits(_h(r.out), want, f"{env.where(r)} LayerNormalization")


def chk_fused_matmul(env, r):
    a = r.args
    S, A = R.matmul64(_t(_h(a["a"])), _t(_h(a["b"])))
    bias = None if a["bias"] is None else _t(_h(a["bias"]))
    res = None if a["residual"] is None else _t(_h(a["residual"]))
    alpha = 1.0 if r.attrs["alpha"] is None else r.attrs["alpha"]
    ref, bnd = R.epilogue_ref_and_bound(S, A, env.tf32, bias, res, r.attrs["activation"], alpha=alpha)
    return _bounded(_h(r.out), ref, bnd, f"{env.where(r)} FusedMatMul")


def chk_dql(env, r):
    y, s, z = env.oracle.dynamic_quantize_linear(_h(r.args["x"]))
    gy, gs, gz = (_h(t) for t in r.out)
    _assert_same_bits(gy, y, f"{env.where(r)} DynamicQuantizeLinear y")
    _assert_same_bits(gs.reshape(-1), np.array([s], np.float32), f"{env.where(r)} DynamicQuantizeLinear scale")
    _assert_same_bits(gz.reshape(-1), np.array([z], np.uint8), f"{env.where(r)} DynamicQuantizeLinear zero point")


def _int8_epilogue(oracle, acc, x_scale, w_scale, bias, residual, act):
    """The oracle's Mul(x_scale, w_scale) -> cast_scale -> Add(bias) -> Add(residual) -> activation, as
    gpu_checks._qlinear_oracle."""
    f32 = np.float32
    scale = np.asarray(w_scale, f32) if x_scale is None else (f32(np.asarray(x_scale).reshape(())) * np.asarray(w_scale, f32)).astype(f32)
    y = oracle.cast_scale(acc, scale)
    if bias is not None:
        y = oracle.add(y, bias)
    if residual is not None:
        y = oracle.add(y, residual.reshape(y.shape))
    if act == R.ACT_GELU_TANH:
        y = oracle.gelu(y, True)
    elif act == R.ACT_GELU:
        y = oracle.gelu(y)
    elif act == R.ACT_RELU:
        y = oracle.relu(y)
    return y


def chk_mmitf(env, r):
    a = r.args
    assert a["b_zero_point"] is None and a["out_range"] is None
    xq = _h(a["a"])
    acc = R.int_matmul(xq.reshape(-1, xq.shape[-1]), _h(a["a_zero_point"]).reshape(()), _h(a["b"]))
    want = _int8_epilogue(env.oracle, acc, _h(a["scale_b"]), _h(a["scale"]), _h(a["bias"]), _h(a["residual"]),
                          r.attrs["activation"])
    got = _h(r.out)
    _assert_same_bits(got.reshape(want.shape), want, f"{env.where(r)} MatMulIntegerToFloat")


def chk_quantized_linear(env, r):
    a, o = r.args, env.oracle
    assert a["w_zero_point"] is None
    x = _h(a["x"])
    h = x if a["ln_scale"] is None else o.layer_norm(x, _h(a["ln_scale"]), _h(a["ln_bias"]), -1, r.attrs["ln_epsilon"])
    xq, xs, xz = o.dynamic_quantize_linear(h)
    acc = R.int_matmul(xq.reshape(-1, xq.shape[-1]), xz, _h(a["w"]))
    want = _int8_epilogue(o, acc, xs, _h(a["w_scale"]), _h(a["bias"]), _h(a["residual"]), r.attrs["activation"])
    _assert_same_bits(_h(r.out).reshape(want.shape), want, f"{env.where(r)} QuantizedLinear")


def chk_assign(env, r):
    _assert_same_bits(_h(r.obj), _h(r.args["src"]), f"{env.where(r)} assign")


def chk_attention(env, r):
    a, at = r.args, r.attrs
    if a["new_key"] is not None:
        return _chk_attention_decode(env, r)
    assert not at["is_causal"] and a["nonpad_kv_seqlen"] is None and not at["softcap"]
    q, k, v = (_h(a[n]) for n in ("query", "key", "value"))
    mask = None if a["attn_mask"] is None else _t(_h(a["attn_mask"]))
    scale = at["scale"] or 1.0 / math.sqrt(q.shape[-1])
    ref, bnd = R.attention_ref_and_bound(_t(q), _t(k), _t(v), mask, scale, env.tf32)
    return _bounded(_h(r.out), ref, bnd, f"{env.where(r)} Attention")


def _chk_attention_decode(env, r):
    """The fused decode step: append at P = nonpad_kv_seqlen - 1, then single-query attention over rows 0 ..= P."""
    a, at = r.args, r.attrs
    lens = _h(a["nonpad_kv_seqlen"])
    P = int(lens[0]) - 1
    assert (lens == P + 1).all() and a["attn_mask"] is None
    K, V = _h(a["key"]), _h(a["value"])
    R.check_cache_append(K, env.prev[a["key"].ptr], _h(a["new_key"])[:, :, 0], P, f"{env.where(r)} key cache")
    R.check_cache_append(V, env.prev[a["value"].ptr], _h(a["new_value"])[:, :, 0], P, f"{env.where(r)} value cache")
    env.prev[a["key"].ptr], env.prev[a["value"].ptr] = K, V
    q = _h(a["query"])
    ref = gc._attention_ref(q, K, V, lens, None, at["scale"])
    err = float(np.abs(_h(r.out) - ref).max())
    worst = err / (2e-5 * float(np.abs(ref).max()))
    assert worst <= 1.0, f"{env.where(r)} decode Attention: error {err:.3e} (ratio {worst:.3f})"
    return worst


def chk_attention_composite(env, parts):
    """FusedMatMul(alpha)(q, k^T) -> AddSoftmax(mask) in place -> MatMul(probs, v): the softmax overwrites the scores,
    so the three calls are checked as one attention against attention_ref_and_bound."""
    mm, sm, pv = parts
    q, kt, v = _h(mm.args["a"]), _h(mm.args["b"]), _h(pv.args["b"])
    ref, bnd = R.attention_ref_and_bound(_t(q), _t(kt).transpose(-1, -2), _t(v), _t(_h(sm.args["y"])),
                                         mm.attrs["alpha"], env.tf32)
    return _bounded(_h(pv.out), ref, bnd, f"{env.where(mm)} FusedMatMul -> AddSoftmax -> MatMul")


CHECKERS = {
    ("Conv", "run"): chk_conv, ("Conv", "run_projected"): chk_conv_projected, ("Conv", "run_chained"): chk_conv_chained,
    ("MaxPool", "run"): chk_max_pool, ("GlobalAveragePool", "run"): chk_global_average_pool, ("Gemm", "run"): chk_gemm,
    ("GatherRows", "run"): chk_gather, ("Add", "run"): chk_add, ("LayerNormalization", "run"): chk_layer_norm,
    ("FusedMatMul", "run"): chk_fused_matmul, ("Attention", "run"): chk_attention,
    ("DynamicQuantizeLinear", "run"): chk_dql, ("MatMulIntegerToFloat", "run"): chk_mmitf,
    ("QuantizedLinear", "run"): chk_quantized_linear, ("DeviceTensor", "assign"): chk_assign,
}


def _units(records):
    """The records as checkable units: single records, and (FusedMatMul, AddSoftmax, MatMul) triples where the softmax
    runs in place on the product and the MatMul reads its result."""
    units, i = [], 0
    while i < len(records):
        r = records[i]
        if r.kind == "FusedMatMul" and i + 2 < len(records):
            sm, pv = records[i + 1], records[i + 2]
            if (sm.kind == "AddSoftmax" and sm.out is r.out and sm.args["x"] is r.out and pv.kind == "MatMul"
                    and pv.args["a"] is r.out):
                units.append((r, sm, pv))
                i += 3
                continue
        units.append((r,))
        i += 1
    return units


class Env:
    """What the checkers share: the oracle, the f32 mode, a name for messages and, for the decode Attention, each
    cache as the previous step left it (keyed by its device address)."""

    def __init__(self, oracle, tf32, name, records, prev=None):
        self.oracle, self.tf32, self.name = oracle, tf32, name
        self.index = {id(r): i for i, r in enumerate(records)}
        self.prev = {} if prev is None else prev

    def where(self, r):
        return f"{self.name} record {self.index[id(r)]}"


def check_records(env, records, launches, stats):
    """Check every record; all `launches` of the replayed step must lie inside checked records."""
    units = _units(records)
    unchecked = sorted({repr(u[0]) for u in units if len(u) == 1 and (u[0].kind, u[0].method) not in CHECKERS})
    assert not unchecked, f"{env.name}: records without a checker: {unchecked}"
    held = sum(r.launches for r in records)
    assert held == launches, f"{env.name}: the records hold {held} of the step's {launches} launches"
    for u in units:
        res = chk_attention_composite(env, u) if len(u) == 3 else CHECKERS[(u[0].kind, u[0].method)](env, u[0])
        if res is None:
            stats["exact"] += 1
        elif res > stats["worst"]:
            stats["worst"], stats["worst_at"] = res, f"{env.where(u[0])}: " + " + ".join(repr(r) for r in u)
        stats["units"] += 1
    stats["records"] += len(records)


def _new_stats():
    return dict(records=0, units=0, exact=0, worst=0.0, worst_at="-")


def _report(name, stats, t0):
    print(f"\n{name}: {stats['records']} records checked ({stats['units']} units), {stats['exact']} bit-exact, worst bound "
          f"ratio {stats['worst']:.3f} ({stats['worst_at']}), {time.time() - t0:.1f} s")


def _two_captures(ctx, O, monkeypatch, fn):
    """The step captured without and with the recorder: (plain graph, its output), (recorded graph, output, records)."""
    g0, out0 = _capture(ctx, fn)
    rec = Recorder()
    with monkeypatch.context() as mp:
        rec.install(mp, O)
        g1, out1 = _capture(ctx, fn)
    assert len(rec.captures) == 1
    return (g0, out0), (g1, out1, rec.captures[0])


def _replay_both(ctx, plain, recorded, what):
    n0 = _replay(ctx, plain[0], plain[1])
    got0 = plain[1].numpy()
    n1 = _replay(ctx, recorded[0], recorded[1])
    got1 = recorded[1].numpy()
    assert n0 == n1, f"{what}: the recorded capture issues {n1} launches, the benched one {n0}"
    _assert_same_bits(got1, got0, f"{what}: recorded vs benched capture output")
    return n1


# ---------------------------------------------------------------------------------------------------------------------
# the benched steps

MODES = [("tf32", True), ("tf32x3", False)]


@pytest.mark.parametrize("mode,tf32", MODES, ids=[m for m, _ in MODES])
def test_resnet50_b32_step(rt, oracle, monkeypatch, mode, tf32):
    from rten_b200 import graphs, ops as O
    t0 = time.time()
    rng = oracle.XorShiftRng(5678)
    spec = graphs.make_resnet50(lambda s: rng.uniform(s))
    x = oracle.XorShiftRng(1234).uniform((32, 3, 224, 224))
    ctx = gc.new_ctx(rt, tf32=tf32)
    runner = graphs.ResNet50Runner(ctx, spec, fuse=True)
    xd = ctx.to_device(x, channels_last=True)
    ctx.set_autotune(True)
    runner.run(xd)
    ctx.sync()
    ctx.set_autotune(False)
    plain, recorded = _two_captures(ctx, O, monkeypatch, lambda: runner.run(xd))
    what = f"ResNet-50 b32 {mode}"
    n = _replay_both(ctx, plain, recorded, what)
    stats = _new_stats()
    check_records(Env(oracle, tf32, what, recorded[2]), recorded[2], n, stats)
    _report(what, stats, t0)


def _bert_masked_inputs(B, S):
    """Padding on half the rows, -10000 on some and -inf on others; token types 0 / 1."""
    r = np.random.default_rng(11)
    mask = np.zeros((B, 1, 1, S), np.float32)
    for b in range(0, B, 2):
        mask[b, 0, 0, S - int(r.integers(1, S // 2)):] = -10000.0 if b % 4 == 0 else -np.inf
    return mask, r.integers(0, 2, (B, S)).astype(np.int32)


@pytest.mark.parametrize("mode,tf32", MODES, ids=[m for m, _ in MODES])
def test_bert_b16_step(rt, oracle, monkeypatch, mode, tf32):
    from rten_b200 import graphs, ops as O
    t0 = time.time()
    rng = oracle.XorShiftRng(5678)
    spec = graphs.make_bert(lambda s: rng.uniform(s))
    B, S = 16, 128
    ids = (oracle.XorShiftRng(1234).u64(B * S) % 30522).astype(np.int32).reshape(B, S)
    ctx = gc.new_ctx(rt, tf32=tf32)
    runner = graphs.BertRunner(ctx, spec, fuse=True)
    di, dt = ctx.to_device(ids), ctx.to_device(np.zeros((B, S), np.int32))
    dm = ctx.to_device(np.zeros((B, 1, 1, S), np.float32))
    ctx.set_autotune(True)
    runner.run(di, dt, dm)
    ctx.sync()
    ctx.set_autotune(False)
    plain, recorded = _two_captures(ctx, O, monkeypatch, lambda: runner.run(di, dt, dm))
    for inputs in ("benched", "masked"):
        if inputs == "masked":
            mask, tt = _bert_masked_inputs(B, S)
            dm.copy_from(mask)
            dt.copy_from(tt)
        what = f"BERT-base b16 x 128 {mode} {inputs} inputs"
        n = _replay_both(ctx, plain, recorded, what)
        stats = _new_stats()
        check_records(Env(oracle, tf32, what, recorded[2]), recorded[2], n, stats)
        _report(what, stats, t0)


def _gpt2_prepare(ctx, O, monkeypatch, runner, prompt, rec):
    """gpu_checks.check_gpt2_b8_baseline's order: autotuned eager prefill, the prefill graph, the fused decode graph
    (autotuned eager pass, then capture).  With `rec`, both captures are recorded."""
    with monkeypatch.context() as mp:
        if rec is not None:
            rec.install(mp, O)
        ctx.set_autotune(True)
        runner.forward(prompt)
        ctx.set_autotune(False)
        runner.reset()
        runner.build_prefill_graph(prompt.shape[1])
        runner.past = prompt.shape[1]
        ctx.set_autotune(True)
        runner.build_decode_graph()
        ctx.set_autotune(False)
    ctx.sync()


def _gpt2_replay(ctx, runner, steps, check=None):
    """NaN into every cache, the graph-replayed prefill, then the decode steps: [(launches, logits)] per step.  `check`
    (step index, launches) runs after each replay, before the next one changes the caches."""
    for d in runner.layers:
        d["k"].copy_from(np.full(d["k"].shape, np.nan, np.float32))
        d["vt"].copy_from(np.full(d["vt"].shape, np.nan, np.float32))
    runner.reset()
    out = []
    for i, ids in enumerate(steps):
        n = ctx.launches
        logits = runner.prefill(ids) if i == 0 else runner.decode_step(ids)
        ctx.sync()
        out.append((ctx.launches - n, logits.numpy().copy()))
        if check is not None:
            check(i, out[-1][0])
    return out


def test_gpt2_int8_b8_steps(rt, oracle, monkeypatch):
    from rten_b200 import graphs, ops as O
    t0 = time.time()
    rng = oracle.XorShiftRng(5678)
    spec = graphs.make_gpt2_int8(lambda s: rng.uniform(s))
    B, T0, nd, M = 8, 512, 8, 576
    ids = (oracle.XorShiftRng(1).u64(B * (T0 + nd)) % 50257).astype(np.int32).reshape(B, T0 + nd)
    steps = [ids[:, :T0]] + [ids[:, T0 + i:T0 + i + 1] for i in range(nd)]
    ctx = gc.new_ctx(rt, tf32=False)
    plain = graphs.GPT2Int8Runner(ctx, spec, B, M, fuse=True)
    _gpt2_prepare(ctx, O, monkeypatch, plain, steps[0], None)
    recorded = graphs.GPT2Int8Runner(ctx, spec, B, M, fuse=True)
    rec = Recorder()
    _gpt2_prepare(ctx, O, monkeypatch, recorded, steps[0], rec)
    assert len(rec.captures) == 2
    want = _gpt2_replay(ctx, plain, steps)
    stats = {"prefill": _new_stats(), "decode": _new_stats()}
    prev = {}  # each cache as the last replayed step left it

    def check_step(i, launches):
        records = rec.captures[min(i, 1)]
        name = "GPT-2 int8 b8 " + ("prefill 512" if i == 0 else f"decode step {i}")
        check_records(Env(oracle, False, name, records, prev), records, launches, stats["prefill" if i == 0 else "decode"])
        if i == 0:
            dh = spec.hidden // spec.heads
            for d in recorded.layers:
                vt = d["vt"].view((B, spec.heads, M, dh), (spec.heads * dh * M, dh * M, 1, M))
                prev[d["k"].ptr], prev[vt.ptr] = d["k"].numpy(), vt.numpy()

    got = _gpt2_replay(ctx, recorded, steps, check_step)
    for i, ((n0, l0), (n1, l1)) in enumerate(zip(want, got)):
        what = "GPT-2 int8 b8 " + ("prefill" if i == 0 else f"decode step {i}")
        assert n0 == n1, f"{what}: the recorded capture issues {n1} launches, the benched one {n0}"
        _assert_same_bits(l1, l0, f"{what}: recorded vs benched capture logits")
    for k, s in stats.items():
        _report(f"GPT-2 int8 b8 {k}", s, t0)
