"""`pytest -m gpu`: RMSNormalization / SimplifiedLayerNormalization and the com.microsoft skip layer norms
(SkipLayerNormalization, SkipSimplifiedLayerNormalization).

  * bit-exact against oracle/norms.py (the out and the input_skip_bias_sum outputs) on the vector path (widths 64, 768,
    896, 2048), the wide CTA-per-row path (1600, 3072, 3584, 4096, 5120, 8192) and the generic path (100, 4100), 1 to
    4096 rows, skip as [B, S, H], [1, S, H] and [S, H], with and without bias / beta, scalar gamma, a strided input, and
    +-inf, NaN, -0.0 and all-zero rows;
  * the kernel each width runs (by name, under CUPTI in a child process) and one launch per dense call;
  * CUDA-graph replay with changed inputs gives the eager bits;
  * every error status and message;
  * through the executor: a two-layer int4 decoder as onnxruntime-genai writes it (MatMulNBits, GroupQueryAttention with
    rotary caches, SkipSimplifiedLayerNormalization with outputs [out, "", "", sum]; a prompt and a decode step), an
    ORT-optimized encoder layer (MultiHeadAttention, SkipLayerNormalization with bias) in both f32 modes, a norm chain
    through SiluFusion, an opset-23 RMSNormalization node and the load failures."""
import json
import os

import numpy as np
import pytest

import gpu_checks as gc

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
F32 = np.float32
VEC, WIDE, GENERIC = (64, 768, 896, 2048), (1600, 3072, 3584, 4096, 5120, 8192), (100, 4100)


@pytest.fixture(scope="module")
def rt():
    import rten_b200
    from rten_b200 import _lib
    _lib.load()
    return rten_b200


@pytest.fixture(scope="module")
def on(oracle):
    from oracle import norms
    return norms


def _bits(got, want, what):
    gc.assert_bit_exact(np.asarray(got), np.asarray(want), what)


def _case(seed, rows, H, skip_kind="bsh", bias=True, beta=True, scalar_gamma=False, special=False):
    """x [B, S, H] (rows = B * S), skip, gamma, beta, bias"""
    r = np.random.default_rng(seed)
    B = 1 if rows < 4 else (rows // 4 if rows % 4 == 0 else 1)
    S = rows // B
    x = (r.standard_normal((B, S, H)) * 2).astype(F32)
    if special:
        x[0, 0, :] = 0.0
        if S > 1:
            x[0, 1, :3] = [np.inf, -0.0, 1e-30]
        if S > 2:
            x[0, 2, 1] = np.nan
        if S > 3:
            x[0, 3, 0] = -np.inf
    skip = {"bsh": (B, S, H), "1sh": (1, S, H), "sh": (S, H)}[skip_kind]
    k = r.standard_normal(skip).astype(F32)
    g = np.array([1.25], F32) if scalar_gamma else (1 + 0.1 * r.standard_normal(H)).astype(F32)
    be = (0.1 * r.standard_normal(H)).astype(F32) if beta else None
    b = (0.1 * r.standard_normal(H)).astype(F32) if bias else None
    return x, k, g, be, b


def _check_skip(rt, on, ctx, x, k, g, be, b, rms, want_sum, what, eps=1e-6):
    op = rt.SkipSimplifiedLayerNormalization(eps) if rms else rt.SkipLayerNormalization(eps)
    args = (x, k, g, b) if rms else (x, k, g, be, b)
    res = op.run(ctx, *args, want_sum=want_sum)
    h = lambda a: a.numpy() if hasattr(a, "numpy") else a
    want, want_s = on.skip_layer_norm(h(x), h(k), h(g), None if rms else h(be), h(b), eps, rms=rms)
    y = res[0] if want_sum else res
    _bits(y.numpy(), want, what)
    if want_sum:
        _bits(res[1].numpy(), want_s, what + " sum")


ROWS = (1, 8, 33)


@pytest.mark.parametrize("H", VEC + WIDE + GENERIC)
def test_skip_norms_bit_exact(rt, on, H):
    ctx = rt.Context(0)
    for rows in ROWS + ((4096,) if H in (768, 4096, 100) else ()):
        for rms in (False, True):
            for i, (skip_kind, bias, beta, sg) in enumerate((("bsh", True, True, False), ("1sh", False, False, True),
                                                              ("sh", True, False, False))):
                x, k, g, be, b = _case(H * 7 + rows + i, rows, H, skip_kind, bias, beta and not rms, sg, special=i == 0)
                xd, kd = ctx.to_device(x), ctx.to_device(k)
                _check_skip(rt, on, ctx, xd, kd, ctx.to_device(g), be if be is None else ctx.to_device(be),
                            b if b is None else ctx.to_device(b), rms, i != 1, f"H={H} rows={rows} rms={rms} case {i}")


@pytest.mark.parametrize("H", VEC + WIDE + GENERIC)
def test_rms_norm_bit_exact(rt, on, H):
    ctx = rt.Context(0)
    for rows in ROWS + ((4096,) if H in (768, 4096, 100) else ()):
        x, _, g, _, _ = _case(H + rows, rows, H, special=True)
        xd = ctx.to_device(x)
        for op in (rt.RMSNormalization(-1, 1e-6), rt.SimplifiedLayerNormalization(-1, 1e-6)):
            _bits(op.run(ctx, xd, ctx.to_device(g)).numpy(), on.rms_norm(x, g, -1, 1e-6), f"RMS H={H} rows={rows}")
        _bits(rt.RMSNormalization().run(ctx, xd, np.array([0.5], F32)).numpy(), on.rms_norm(x, np.array([0.5], F32)),
              f"RMS scalar scale H={H}")


def test_rms_norm_over_two_axes_and_scale_broadcast(rt, on):
    ctx = rt.Context(0)
    x = np.random.default_rng(3).standard_normal((3, 4, 8, 16)).astype(F32)
    s = np.random.default_rng(4).standard_normal((8, 1)).astype(F32)
    _bits(rt.RMSNormalization(-2).run(ctx, x, s).numpy(), on.rms_norm(x, s, -2), "RMS axis -2, broadcast scale")


def test_strided_inputs(rt, on):
    """A row-sliced x and skip (rows farther apart than H), aligned (vector / wide kernels) and not (generic)"""
    ctx = rt.Context(0)
    for H, pad in ((768, 64), (4096, 4), (768, 3)):
        x, k, g, be, b = _case(H, 16, H)
        x2, k2 = x.reshape(-1, H), k.reshape(-1, H)
        xb = ctx.to_device(np.concatenate([x2, np.zeros((16, pad), F32)], axis=1))
        kb = ctx.to_device(np.concatenate([k2, np.ones((16, pad), F32)], axis=1))
        xv, kv = xb.view((16, H), (H + pad, 1), 0), kb.view((16, H), (H + pad, 1), 0)
        for rms in (False, True):
            _check_skip(rt, on, ctx, xv, kv, g, None if rms else be, b, rms, True, f"strided H={H} pad={pad} rms={rms}")
        _bits(rt.RMSNormalization().run(ctx, xv, g).numpy(), on.rms_norm(x2, g), f"RMS strided H={H} pad={pad}")


def test_one_launch_and_graph_replay(rt, on):
    ctx = rt.Context(0)
    for H in (768, 4096, 100):
        x, k, g, be, b = _case(H, 64, H)
        xd, kd, gd, bd = (ctx.to_device(a) for a in (x, k, g, b))
        op = rt.SkipSimplifiedLayerNormalization(1e-6)
        op.run(ctx, xd, kd, gd, bd, want_sum=True)  # (warm: allocations)
        n0 = ctx.launches
        op.run(ctx, xd, kd, gd, bd, want_sum=True)
        assert ctx.launches - n0 == 1, f"H={H}: {ctx.launches - n0} launches"
        n0 = ctx.launches
        rt.RMSNormalization(-1, 1e-6).run(ctx, xd, gd)
        assert ctx.launches - n0 == 1
        ctx.graph_begin()
        y, s = op.run(ctx, xd, kd, gd, bd, want_sum=True)
        graph = ctx.graph_end()
        for rep in range(2):
            x2 = (x * (rep + 2)).astype(F32)
            xd.copy_from(x2)
            graph.launch()
            ctx.sync()
            want, want_s = on.skip_layer_norm(x2, k, g, None, b, 1e-6, rms=True)
            _bits(y.numpy(), want, f"graph replay H={H} rep {rep}")
            _bits(s.numpy(), want_s, f"graph replay sum H={H} rep {rep}")


def _err(rt, fn):
    with pytest.raises(rt.OpError) as e:
        fn()
    return e.value.kind, e.value.msg


def test_errors(rt, on):
    ctx = rt.Context(0)
    z = lambda *s: np.zeros(s, F32)
    for rms in (False, True):
        op = rt.SkipSimplifiedLayerNormalization(1e-5) if rms else rt.SkipLayerNormalization(1e-5)
        for c in json.load(open(os.path.join(HERE, "golden", "norm_cases.json")))["invalid"]:
            got = _err(rt, lambda: op.run(ctx, z(*c["input_shape"]), z(*c["skip_shape"]), z(*c["gamma_shape"])))
            assert got == (c["kind"], c["msg"]), got
        assert _err(rt, lambda: op.run(ctx, z(2, 3, 4), z(2, 4), z(4))) == (
            "IncompatibleInputShapes", "skip must broadcast to input over the batch dimension")
        assert _err(rt, lambda: op.run(ctx, z(2, 3, 4), z(3, 3, 4), z(4))) == (
            "IncompatibleInputShapes", "skip must broadcast to input over the batch dimension")
        assert _err(rt, lambda: op.run(ctx, z(3, 4), z(1, 3, 4), z(4))) == (
            "IncompatibleInputShapes", "skip must broadcast to input over the batch dimension")
        assert _err(rt, lambda: op.run(ctx, z(3, 4), z(3, 4, 1, 1), z(4))) == ("InvalidValue", "skip must be 2 or 3 dimensioned")
        assert _err(rt, lambda: op.run(ctx, z(3, 4), z(3, 4), z(3))) == (
            "InvalidValue", "`scale` is not broadcastable to normalized axes of input")
        assert _err(rt, lambda: op.run(ctx, z(3, 4), z(3, 4), z(1, 4))) == ("CastFailed", "gamma, beta and bias must be 1-D tensors")
        assert _err(rt, lambda: op.run(ctx, z(3, 4), z(3, 4), z(4), bias=z(3))) == (
            "InvalidValue", "bias length must equal the hidden size")
        # oracle: the same message for the same deviation
        with pytest.raises(Exception):
            on.skip_layer_norm(z(3, 4), z(3, 4), z(4), None, z(3), 1e-5, rms=rms)
    assert _err(rt, lambda: rt.SkipLayerNormalization(1e-5).run(ctx, z(3, 4), z(3, 4), z(4), z(3))) == (
        "InvalidValue", "`bias` is not broadcastable to normalized axes of input")
    assert _err(rt, lambda: rt.RMSNormalization(2).run(ctx, z(3, 4), z(4))) == ("InvalidValue", "Axis is invalid")
    assert _err(rt, lambda: rt.RMSNormalization().run(ctx, z(3, 4), z(3))) == (
        "InvalidValue", "`scale` is not broadcastable to normalized axes of input")
    import ctypes as C
    from rten_b200.ops import _Args
    A = _Args(ctx)
    o = A.out()
    st = ctx.lib.rten_b200_skip_layer_norm(ctx.handle, A.t(z(3, 4)), A.t(z(3, 4)), A.t(z(4)), A.t(z(4)), None, 1e-5, 1,
                                           C.byref(o), None)
    assert st == 5 and b"no beta" in ctx.lib.rten_b200_last_error(ctx.handle)


def test_bias_of_one_element(rt, on):
    ctx = rt.Context(0)
    x, k, g, _, _ = _case(9, 8, 768)
    b = np.array([0.375], F32)
    for rms in (False, True):
        _check_skip(rt, on, ctx, x, k, g, None, b, rms, True, f"one-element bias rms={rms}")


# ---- kernel identity (CUPTI in a child process, so that no profiler state stays behind in the test session) ----------
def _kernel_probe():
    import gpu_checks as g
    import rten_b200 as rt
    ctx = rt.Context(0)
    res = {}
    for H in VEC + WIDE + GENERIC:
        x, k, gm, _, b = _case(H, 8, H)
        xd, kd, gd, bd = (ctx.to_device(a) for a in (x, k, gm, b))
        op = rt.SkipSimplifiedLayerNormalization(1e-6)
        _, names = g._kernels_launched(lambda: op.run(ctx, xd, kd, gd, bd, want_sum=True))
        _, rnames = g._kernels_launched(lambda: rt.RMSNormalization().run(ctx, xd, gd))
        res[str(H)] = sorted(names | rnames)
    xb = ctx.to_device(np.zeros((8, 772), F32))
    _, names = g._kernels_launched(lambda: rt.SkipLayerNormalization(1e-6).run(ctx, xb.view((8, 768), (772, 1), 1), xb.view((8, 768), (772, 1), 1), np.ones(768, F32)))
    res["unaligned"] = sorted(names)
    print(json.dumps(res))


def test_kernel_identity():
    import subprocess
    import sys
    code = (f"import sys; sys.path[:0] = [{os.path.dirname(HERE)!r}, {HERE!r}]; "
            "import test_gpu_norms as t; t._kernel_probe()")
    res = subprocess.run([sys.executable, "-s", "-c", code], capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-4000:]
    names = json.loads(res.stdout.strip().splitlines()[-1])
    want = {**{str(h): "norm_vec_kernel" for h in VEC}, **{str(h): "norm_wide_kernel" for h in WIDE},
            **{str(h): "norm_kernel" for h in GENERIC}, "unaligned": "norm_kernel"}
    for key, kname in want.items():
        ks = [n for n in names[key] if "_kernel" in n]  # (the session also lists runtime API calls)
        assert ks and all(kname + "(" in n or kname + "<" in n for n in ks), (key, ks)


# ---- through the executor --------------------------------------------------------------------------------------------
def _model(W, nodes, inits, inputs, outputs, opset=18):
    return W.model(nodes, [W.tensor(k, v) for k, v in inits.items()], [W.value_info(n, 1, s) for n, s in inputs],
                   [W.value_info(n, 1, s) for n, s in outputs], opset=opset, extra_opsets=(("com.microsoft", 1),))


def test_model_decoder_chain(rt, on):
    """Embedding norm, a residual SkipSimplifiedLayerNormalization whose sum feeds the next one, Silu through SiluFusion:
    bit-identical to the operators called one by one, and to the oracle."""
    import onnx_writer as W
    from rten_b200.model import Model
    H, T = 4096, 6
    r = np.random.default_rng(21)
    w = {n: (1 + 0.1 * r.standard_normal(H)).astype(F32) for n in ("g0", "g1", "g2")}
    N = lambda op, i, o, **a: W.node(op, i, o, **a)
    nodes = [N("SimplifiedLayerNormalization", ["x", "g0"], ["h0"], axis=-1, epsilon=1e-5),
             N("SkipSimplifiedLayerNormalization", ["h0", "x", "g1"], ["h1", "", "", "res1"], domain="com.microsoft", epsilon=1e-5),
             N("Sigmoid", ["h1"], ["sg"]), N("Mul", ["h1", "sg"], ["act"]),
             N("SkipSimplifiedLayerNormalization", ["act", "res1", "g2"], ["y", "", "", "res2"], domain="com.microsoft", epsilon=1e-5)]
    data = _model(W, nodes, w, [("x", [1, T, H])], [("y", [1, T, H]), ("res2", [1, T, H])])
    ctx = rt.Context(0)
    m = Model(ctx, data)
    assert "Silu" in m.node_ops and "Sigmoid" not in m.node_ops, m.node_ops
    x = r.standard_normal((1, T, H)).astype(F32)
    y, res2 = (t.numpy() for t in m.run({"x": x}, ["y", "res2"]))
    h0 = rt.SimplifiedLayerNormalization(-1, 1e-5).run(ctx, x, w["g0"])
    h1, res1 = rt.SkipSimplifiedLayerNormalization(1e-5).run(ctx, h0, x, w["g1"], want_sum=True)
    act = rt.Silu().run(ctx, h1)
    y1, r2 = rt.SkipSimplifiedLayerNormalization(1e-5).run(ctx, act, res1, w["g2"], want_sum=True)
    _bits(y, y1.numpy(), "executor y")
    _bits(res2, r2.numpy(), "executor residual")
    o0 = on.rms_norm(x, w["g0"], -1, 1e-5)
    o1, s1 = on.skip_layer_norm(o0, x, w["g1"], None, None, 1e-5, rms=True)
    _bits(h1.numpy(), o1, "oracle h1")
    _bits(res1.numpy(), s1, "oracle res1")


def _rel(got, ref):
    return float(np.abs(np.asarray(got, np.float64) - ref).max() / np.abs(ref).max())


def _layer_norm64(s, g, b=None, eps=1e-5, rms=False):
    m = 0.0 if rms else s.mean(-1, keepdims=True)
    d = s - m
    y = d / np.sqrt((d * d).mean(-1, keepdims=True) + eps) * g
    return y if b is None else y + b


# ---- a two-layer int4 decoder as onnxruntime-genai writes it ---------------------------------------------------------
DEC = dict(L=2, V=128, Hq=4, Hkv=2, D=64, I=512, block=32, maxp=64, eps=1e-5)


def _decoder_weights(seed=31):
    from test_gpu_matmul_nbits import pack_nbits
    c = DEC
    hid = c["Hq"] * c["D"]
    r = np.random.default_rng(seed)
    w = {"embed": r.standard_normal((c["V"], hid)).astype(F32)}

    def q4(name, K, N):
        w["b_" + name] = pack_nbits(r.integers(0, 16, (N, K // c["block"], c["block"])))
        w["s_" + name] = r.uniform(0.005, 0.02, (N, K // c["block"])).astype(F32)

    for l in range(c["L"]):
        for nm, K, N in (("q", hid, hid), ("k", hid, c["Hkv"] * c["D"]), ("v", hid, c["Hkv"] * c["D"]), ("o", hid, hid),
                         ("gate", hid, c["I"]), ("up", hid, c["I"]), ("down", c["I"], hid)):
            q4(f"{nm}{l}", K, N)
        w[f"g_in{l}"] = (1 + 0.1 * r.standard_normal(hid)).astype(F32)
        w[f"g_post{l}"] = (1 + 0.1 * r.standard_normal(hid)).astype(F32)
    w["g_final"] = (1 + 0.1 * r.standard_normal(hid)).astype(F32)
    q4("lm", hid, c["V"])
    half = c["D"] // 2
    ang = np.arange(c["maxp"])[:, None] * (10000.0 ** (-np.arange(half) / half))[None, :]
    w["cos"], w["sin"] = np.cos(ang).astype(F32), np.sin(ang).astype(F32)
    return w


def _decoder_graph(w, B, S, P):
    """embedding Gather -> SimplifiedLayerNormalization; per layer MatMulNBits Q / K / V -> GroupQueryAttention (do_rotary,
    cos / sin caches; past caches when P > 0) -> MatMulNBits O -> SkipSimplifiedLayerNormalization [out, "", "", sum] ->
    MatMulNBits gate / up -> Mul(x, Sigmoid(x)) -> Mul -> MatMulNBits down; the next layer's input norm and the final norm
    are SkipSimplifiedLayerNormalization over the running residual; MatMulNBits lm_head."""
    import onnx_writer as W
    c = DEC
    hid, kvd, L = c["Hq"] * c["D"], c["Hkv"] * c["D"], c["L"]
    ms = dict(domain="com.microsoft")

    def mm(x, nm, out, K, N):
        return W.node("MatMulNBits", [x, "b_" + nm, "s_" + nm], [out], K=K, N=N, bits=4, block_size=c["block"], accuracy_level=4, **ms)

    nodes = [W.node("Gather", ["embed", "input_ids"], ["x0"]),
             W.node("SimplifiedLayerNormalization", ["x0", "g_in0"], ["h0"], axis=-1, epsilon=c["eps"])]
    res, h = "x0", "h0"
    for l in range(L):
        past = [f"past_key_{l}", f"past_value_{l}"] if P else ["", ""]
        nodes += [mm(h, f"q{l}", f"q{l}", hid, hid), mm(h, f"k{l}", f"k{l}", hid, kvd), mm(h, f"v{l}", f"v{l}", hid, kvd),
                  W.node("GroupQueryAttention", [f"q{l}", f"k{l}", f"v{l}"] + past + ["seqlens_k", "total", "cos", "sin"],
                         [f"a{l}", f"present_key_{l}", f"present_value_{l}"], num_heads=c["Hq"], kv_num_heads=c["Hkv"], do_rotary=1,
                         local_window_size=-1, **ms),
                  mm(f"a{l}", f"o{l}", f"o{l}", hid, hid),
                  W.node("SkipSimplifiedLayerNormalization", [f"o{l}", res, f"g_post{l}"], [f"h2_{l}", "", "", f"r2_{l}"],
                         epsilon=c["eps"], **ms),
                  mm(f"h2_{l}", f"gate{l}", f"gt{l}", hid, c["I"]), mm(f"h2_{l}", f"up{l}", f"up{l}", hid, c["I"]),
                  W.node("Sigmoid", [f"gt{l}"], [f"sg{l}"]), W.node("Mul", [f"gt{l}", f"sg{l}"], [f"si{l}"]),
                  W.node("Mul", [f"si{l}", f"up{l}"], [f"m{l}"]), mm(f"m{l}", f"down{l}", f"d{l}", c["I"], hid)]
        last = l + 1 == L
        nodes.append(W.node("SkipSimplifiedLayerNormalization", [f"d{l}", f"r2_{l}", "g_final" if last else f"g_in{l + 1}"],
                            ["hf"] if last else [f"h{l + 1}", "", "", f"r{l + 1}"], epsilon=c["eps"], **ms))
        res, h = f"r{l + 1}", f"h{l + 1}"
    nodes.append(mm("hf", "lm", "logits", hid, c["V"]))
    ins = [W.value_info("input_ids", W.INT32, [B, S])]
    for l in range(L if P else 0):
        ins += [W.value_info(f"past_key_{l}", W.FLOAT, [B, c["Hkv"], P, c["D"]]),
                W.value_info(f"past_value_{l}", W.FLOAT, [B, c["Hkv"], P, c["D"]])]
    ins += [W.value_info("seqlens_k", W.INT32, [B]), W.value_info("total", W.INT32, [])]
    outs = [W.value_info("logits", W.FLOAT, [B, S, c["V"]])]
    for l in range(L):
        outs += [W.value_info(f"present_key_{l}", W.FLOAT, []), W.value_info(f"present_value_{l}", W.FLOAT, [])]
    return W.model(nodes, [W.tensor(k, v) for k, v in w.items()], ins, outs, opset=21, extra_opsets=[("com.microsoft", 1)])


def _decoder_ops(rt, ctx, w, ids, past, sk, total):
    """The same forward, one ops.py call per node (Mul(x, Sigmoid(x)) as Silu, which the executor fuses it into)"""
    c = DEC
    d = {k: ctx.to_device(v) for k, v in w.items()}
    nb = rt.MatMulNBits(block_size=c["block"], accuracy_level=4)
    mm = lambda x, nm: nb.run(ctx, x, d["b_" + nm], d["s_" + nm])
    gqa = rt.GroupQueryAttention(c["Hq"], c["Hkv"], do_rotary=True, local_window_size=-1)
    ssn = rt.SkipSimplifiedLayerNormalization(c["eps"])
    x0 = rt.GatherRows().run(ctx, d["embed"], ids)
    h = rt.SimplifiedLayerNormalization(-1, c["eps"]).run(ctx, x0, d["g_in0"])
    res, presents = x0, []
    for l in range(c["L"]):
        pk, pv = past[l] if past else (None, None)
        a, prk, prv = gqa.run(ctx, mm(h, f"q{l}"), mm(h, f"k{l}"), mm(h, f"v{l}"), sk, total, past_key=pk, past_value=pv,
                              cos_cache=d["cos"], sin_cache=d["sin"])
        presents.append((prk, prv))
        h2, r2 = ssn.run(ctx, mm(a, f"o{l}"), res, d[f"g_post{l}"], want_sum=True)
        m = rt.Mul().run(ctx, rt.Silu().run(ctx, mm(h2, f"gate{l}")), mm(h2, f"up{l}"))
        if l + 1 < c["L"]:
            h, res = ssn.run(ctx, mm(m, f"down{l}"), r2, d[f"g_in{l + 1}"], want_sum=True)
        else:
            h = ssn.run(ctx, mm(m, f"down{l}"), r2, d["g_final"])
    return mm(h, "lm"), presents


def _decoder_f64(w, ids):
    """float64 forward over the whole sequence (dequantized weights, causal attention through ref_gqa)"""
    from test_gpu_group_query_attention import ref_gqa
    from test_gpu_matmul_nbits import dequantize_nbits
    c = DEC
    B, T = ids.shape
    W64 = lambda nm: dequantize_nbits(w["b_" + nm], w["s_" + nm]).astype(np.float64)
    g = lambda nm: w[nm].astype(np.float64)
    x = w["embed"].astype(np.float64)[ids]
    h = _layer_norm64(x, g("g_in0"), eps=c["eps"], rms=True)
    res = x
    for l in range(c["L"]):
        a = ref_gqa(h @ W64(f"q{l}"), h @ W64(f"k{l}"), h @ W64(f"v{l}"), None, None, np.full(B, T - 1, np.int32), T, c["Hq"],
                    c["Hkv"], w["cos"], w["sin"], do_rotary=True)[0]
        res = res + a @ W64(f"o{l}")
        h2 = _layer_norm64(res, g(f"g_post{l}"), eps=c["eps"], rms=True)
        gt = h2 @ W64(f"gate{l}")
        res = res + (gt / (1 + np.exp(-gt)) * (h2 @ W64(f"up{l}"))) @ W64(f"down{l}")
        h = _layer_norm64(res, g("g_final" if l + 1 == c["L"] else f"g_in{l + 1}"), eps=c["eps"], rms=True)
    return h @ W64("lm")


def test_model_genai_int4_decoder(rt):
    """A prompt, then one decode step fed the prompt's present caches, through Model: logits and present caches
    bit-identical to the operators called one by one, and logits within 2e-4 * max |ref| of the float64 forward (the
    single-op MatMulNBits / GroupQueryAttention bound is 2e-5; two layers of seven products and four norms compound it)."""
    from rten_b200.model import Model
    c = DEC
    B, S = 2, 40
    w = _decoder_weights()
    ids = np.random.default_rng(32).integers(0, c["V"], (B, S + 1)).astype(np.int32)
    ref = _decoder_f64(w, ids)
    ctx = rt.Context(0)
    names = ["logits"] + [f"present_{kv}_{l}" for l in range(c["L"]) for kv in ("key", "value")]
    # prompt
    m = Model(ctx, _decoder_graph(w, B, S, 0))
    assert m.node_ops.count("SkipSimplifiedLayerNormalization") == 2 * c["L"] and "Silu" in m.node_ops, m.node_ops
    sk, total = np.full(B, S - 1, np.int32), np.array(S, np.int32)
    got = [t.numpy() for t in m.run({"input_ids": ids[:, :S], "seqlens_k": sk, "total": total}, names)]
    lg, pres = _decoder_ops(rt, ctx, w, ids[:, :S], None, sk, total)
    _bits(got[0], lg.numpy(), "prompt logits")
    for l in range(c["L"]):
        _bits(got[1 + 2 * l], pres[l][0].numpy(), f"prompt present_key_{l}")
        _bits(got[2 + 2 * l], pres[l][1].numpy(), f"prompt present_value_{l}")
    assert _rel(got[0], ref[:, :S]) <= 2e-4, _rel(got[0], ref[:, :S])
    # one decode step
    md = Model(ctx, _decoder_graph(w, B, 1, S))
    sk1, total1 = np.full(B, S, np.int32), np.array(S + 1, np.int32)
    feeds = {"input_ids": ids[:, S:], "seqlens_k": sk1, "total": total1}
    for l in range(c["L"]):
        feeds[f"past_key_{l}"], feeds[f"past_value_{l}"] = got[1 + 2 * l], got[2 + 2 * l]
    got1 = [t.numpy() for t in md.run(feeds, names)]
    past = [(ctx.to_device(got[1 + 2 * l]), ctx.to_device(got[2 + 2 * l])) for l in range(c["L"])]
    lg1, pres1 = _decoder_ops(rt, ctx, w, ids[:, S:], past, sk1, total1)
    _bits(got1[0], lg1.numpy(), "decode logits")
    for l in range(c["L"]):
        _bits(got1[1 + 2 * l], pres1[l][0].numpy(), f"decode present_key_{l}")
        _bits(got1[2 + 2 * l], pres1[l][1].numpy(), f"decode present_value_{l}")
    assert _rel(got1[0], ref[:, S:]) <= 2e-4, _rel(got1[0], ref[:, S:])


def test_model_encoder_layer(rt, on):
    """An ORT-optimized encoder layer: MultiHeadAttention, then SkipLayerNormalization with the residual bias (input 4),
    in both f32 modes: bit-identical to the two operators called one by one, and within 1e-4 (3xTF32) / 1e-2 (single-pass
    TF32, the prefill kernel's 4e-3 attention bound carried through the norm) * max |ref| of a float64 forward."""
    import onnx_writer as W
    from rten_b200.model import Model
    from test_gpu_multi_head_attention import ref_mha
    B, S, Hn, hid, eps = 2, 64, 12, 768, 1e-12
    r = np.random.default_rng(22)
    w = {"g": (1 + 0.1 * r.standard_normal(hid)).astype(F32), "be": (0.1 * r.standard_normal(hid)).astype(F32),
         "bi": (0.1 * r.standard_normal(hid)).astype(F32)}
    nodes = [W.node("MultiHeadAttention", ["x", "x", "x"], ["a"], domain="com.microsoft", num_heads=Hn),
             W.node("SkipLayerNormalization", ["a", "x", "g", "be", "bi"], ["y"], domain="com.microsoft", epsilon=eps)]
    data = _model(W, nodes, w, [("x", [B, S, hid])], [("y", [B, S, hid])])
    x = r.standard_normal((B, S, hid)).astype(F32)
    a64 = ref_mha(x, x, x, H=Hn)[0]
    ref = _layer_norm64(a64 + x.astype(np.float64) + w["bi"], w["g"].astype(np.float64), w["be"].astype(np.float64), eps)
    for tf32, tol in ((False, 1e-4), (True, 1e-2)):
        ctx = gc.new_ctx(rt, tf32=tf32)
        y = Model(ctx, data).run({"x": x}, ["y"])[0].numpy()
        a = rt.MultiHeadAttention(Hn).run(ctx, x, x, x, want_present=False)[0]
        y1 = rt.SkipLayerNormalization(eps).run(ctx, a, x, w["g"], w["be"], w["bi"])
        _bits(y, y1.numpy(), f"encoder layer tf32={tf32}")
        assert _rel(y, ref) <= tol, (tf32, _rel(y, ref))


def test_model_rms_normalization_opset23_and_load_failures(rt, on):
    import onnx_writer as W
    from rten_b200.model import Model
    H = 896
    g = np.linspace(0.5, 1.5, H).astype(F32)
    x = np.random.default_rng(23).standard_normal((3, 5, H)).astype(F32)
    ok = _model(W, [W.node("RMSNormalization", ["x", "g"], ["y"], axis=-1, epsilon=1e-6, stash_type=1)], {"g": g},
                [("x", [3, 5, H])], [("y", [3, 5, H])], opset=23)
    ctx = rt.Context(0)
    _bits(Model(ctx, ok).run({"x": x}, ["y"])[0].numpy(), on.rms_norm(x, g, -1, 1e-6), "opset-23 RMSNormalization")
    bad = {
        "stash_type must be 1": [W.node("RMSNormalization", ["x", "g"], ["y"], stash_type=0)],
        "missing attribute epsilon": [W.node("SkipSimplifiedLayerNormalization", ["x", "x", "g"], ["y"], domain="com.microsoft")],
        "mean and inv_std_var": [W.node("SkipLayerNormalization", ["x", "x", "g"], ["y", "mean"], domain="com.microsoft", epsilon=1e-5)],
        "only the normalized output": [W.node("SimplifiedLayerNormalization", ["x", "g"], ["y", "", "inv_std_var"], epsilon=1e-5)],
    }
    for msg, nodes in bad.items():
        with pytest.raises(rt.OpError) as e:
            Model(ctx, _model(W, nodes, {"g": g}, [("x", [3, 5, H])], [("y", [3, 5, H])]))
        assert e.value.kind == "UnsupportedValue" and msg in e.value.msg, e.value.msg
