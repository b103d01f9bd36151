"""The Attention operator with q_seq > 1 on the calls that need masking or grouped-query heads (causal, a right-padded KV
cache through nonpad_kv_seqlen, q_heads != kv_heads): the streaming wgmma kernel attn_prefill_kernel.

Every GPU assertion rests on `ref_attention`, a vectorised float64 restatement of the reference's own test oracle
(src/ops/attention.rs:1219-1322) restricted to what these calls use; the CPU test checks it against a literal per-row
transcription of that function on the reference's case table.  Bounds: |d| <= 2e-5 * max |ref| in 3xTF32 (the library
default, the decode kernel's stated bound) and 4e-3 * max |ref| in single-pass TF32 (attn_fused's bound)."""
import math

import numpy as np
import pytest

# ---------------------------------------------------------------------------------------------------------------------
# float64 reference


def ref_attention(q, k, v, mask=None, nonpad=None, causal=False, scale=None):
    """softmax(scale q k^T + mask, masked keys -> -inf, NaN -> 0) v, with q [B, qh, T, dh], k / v [B, kvh, L, dh],
    query head h reading kv head h // (qh // kvh).  nonpad [B]: keys >= clamp(nonpad[b], 0, L) are masked; causal: row s
    sees keys 0 ..= s + offset, offset = valid_b - T with nonpad and 0 without."""
    q, k, v = (np.asarray(a, np.float64) for a in (q, k, v))
    B, qh, T, dh = q.shape
    kvh, L = k.shape[1], k.shape[2]
    scale = 1.0 / math.sqrt(dh) if scale is None else scale
    k = np.repeat(k, qh // kvh, axis=1)
    v = np.repeat(v, qh // kvh, axis=1)
    s = scale * np.einsum("bhqd,bhkd->bhqk", q, k)
    if mask is not None:
        s = s + np.asarray(mask, np.float64)
    t = np.arange(L)[None, None, None, :]
    if nonpad is not None:
        valid = np.clip(np.asarray(nonpad, np.int64), 0, L)[:, None, None, None]
        s = np.where(t >= valid, -np.inf, s)
    if causal:
        off = (np.clip(np.asarray(nonpad, np.int64), 0, L) - T) if nonpad is not None else np.zeros(B, np.int64)
        s = np.where(t > np.arange(T)[None, None, :, None] + off[:, None, None, None], -np.inf, s)
    with np.errstate(invalid="ignore"):
        p = np.exp(s - s.max(-1, keepdims=True))
        p = p / p.sum(-1, keepdims=True)
    p = np.where(np.isnan(p), 0.0, p)
    return np.einsum("bhqk,bhkd->bhqd", p, v)


def _loop_attention(q, k, v, mask, nonpad, causal, scale):
    """src/ops/attention.rs:1254-1320 transcribed row by row (float64, no past inputs, no softcap)."""
    B, qh, T, dh = q.shape
    kvh, total = k.shape[1], k.shape[2]
    factor = qh // kvh
    m = None if mask is None else np.broadcast_to(mask, (B, qh, T, total))
    out = np.zeros((B, qh, T, v.shape[3]))
    for b in range(B):
        for n in range(qh):
            hk = n // factor
            for s in range(T):
                scores = [sum(float(q[b, n, s, d]) * float(k[b, hk, t, d]) for d in range(dh)) * scale for t in range(total)]
                if m is not None:
                    scores = [sc + float(m[b, n, s, t]) for t, sc in enumerate(scores)]
                if nonpad is not None:
                    scores = [-math.inf if t >= nonpad[b] else sc for t, sc in enumerate(scores)]
                if causal:
                    offset = nonpad[b] - T if nonpad is not None else 0
                    scores = [-math.inf if t > s + offset else sc for t, sc in enumerate(scores)]
                mx = max(scores)
                if mx == -math.inf:
                    probs = [0.0] * total  # exp(-inf - -inf) = NaN, flushed to zero
                else:
                    e = [math.exp(sc - mx) for sc in scores]
                    probs = [x / sum(e) for x in e]
                for d in range(v.shape[3]):
                    out[b, n, s, d] = sum(p * float(v[b, hk, t, d]) for t, p in enumerate(probs))
    return out


def test_reference_attention_matches_the_row_loop():
    """The reference's nonpad_kv_seqlen case table (src/ops/attention.rs:1745-1768), with grouped-query heads and a float
    mask on top: the vectorised reference equals the row-by-row transcription."""
    rng = np.random.default_rng(5)
    kv_seq, qh, kvh, dh = 5, 4, 2, 3
    for lens, q_seq, causal in (([5, 3], 4, False), ([5, 3], 3, True), ([1], 3, True)):
        B = len(lens)
        q, k, v = rng.standard_normal((B, qh, q_seq, dh)), rng.standard_normal((B, kvh, kv_seq, dh)), rng.standard_normal((B, kvh, kv_seq, dh))
        for mask in (None, rng.uniform(-2, 0, (B, 1, q_seq, kv_seq))):
            got = ref_attention(q, k, v, mask, lens, causal, 0.5)
            want = _loop_attention(q, k, v, mask, lens, causal, 0.5)
            np.testing.assert_allclose(got, want, rtol=1e-12, atol=1e-12)
            if lens == [1]:  # offset 1 - 3: rows 0 and 1 see no key at all
                assert not got[:, :, :2].any() and got[:, :, 2].any()
    # GQA without nonpad, causal top-left with more keys than queries
    q, k, v = rng.standard_normal((1, 6, 4, 2)), rng.standard_normal((1, 3, 7, 2)), rng.standard_normal((1, 3, 7, 2))
    np.testing.assert_allclose(ref_attention(q, k, v, None, None, True, 0.7), _loop_attention(q, k, v, None, None, True, 0.7), rtol=1e-12, atol=1e-12)


# ---------------------------------------------------------------------------------------------------------------------
# GPU


@pytest.fixture(scope="module")
def rt():
    import rten_b200
    from rten_b200 import _lib
    _lib.load()
    return rten_b200


def _ctx(rt, tf32):
    ctx = rt.Context(0)
    ctx.set_f32_mode(not tf32)
    return ctx


def _rel_err(got, ref):
    return float(np.abs(np.asarray(got, np.float64) - ref).max() / max(float(np.abs(ref).max()), 1e-30))


def _kernels(fn):
    import gpu_checks as gc
    return gc._kernels_launched(fn)


def _device_inputs(ctx, q, k, v, v_layout):
    """q, k, v on the device; v natural ([.., L, dh]) or as a [.., L, dh] view of a transposed [.., dh, cap] cache whose
    capacity is L rounded up to 4 positions (rows of whole 16-byte units, as TMA needs them)."""
    B, kvh, L, dh = v.shape
    if v_layout == "transposed":
        cap = -(-L // 4) * 4
        vt = np.zeros((B, kvh, dh, cap), np.float32)
        vt[..., :L] = v.transpose(0, 1, 3, 2)
        dvt = ctx.to_device(vt)
        dv = dvt.view((B, kvh, L, dh), (kvh * dh * cap, dh * cap, 1, cap))
    else:
        dv = ctx.to_device(v)
    return ctx.to_device(q), ctx.to_device(k), dv


# (B, q_heads, kv_heads, q_seq, keys, head size, causal, nonpad, mask shape or None, value layout)
CASES = [
    ("causal, q_seq == keys", (2, 4, 4, 128, 128, 64, True, None, None, "natural")),
    ("causal chunked prefill (offset P)", (2, 4, 4, 64, 300, 64, True, [164, 264], None, "transposed")),
    ("causal, nonpad < q_seq", (2, 4, 4, 100, 160, 64, True, [40, 160], None, "natural")),
    ("non-causal nonpad mix, GQA 8/2, 200 over 1000", (4, 8, 2, 200, 1000, 64, False, [0, 1000, 77, 513], None, "transposed")),
    ("GQA 32/8 head 128, 77 over 333", (1, 32, 8, 77, 333, 128, True, None, None, "natural")),
    ("GQA 12/4, mask [B,1,1,L]", (2, 12, 4, 96, 150, 64, True, None, "b11l", "natural")),
    ("GQA 8/1 head 128, nonpad, mask [1,1,T,L]", (2, 8, 1, 70, 260, 128, True, [250, 130], "11tl", "transposed")),
    ("mask [B,H,T,L] with -inf rows, head 128", (2, 3, 3, 65, 200, 128, True, None, "bhtl", "natural")),
    ("4096 keys, nonpad", (1, 4, 2, 130, 4096, 64, False, [4000], None, "transposed")),
    # fewer queries and keys than one tile and than the 32-key box of V^T: whole tiles of out-of-bounds fill
    ("2 queries over 5 keys, causal nonpad", (2, 2, 1, 2, 5, 64, True, [5, 3], None, "transposed")),
    ("3 queries over 20 keys, head 128", (1, 4, 2, 3, 20, 128, True, None, "b11l", "natural")),
]


def _case_data(seed, B, qh, kvh, T, L, dh, causal, nonpad, mask_kind):
    rng = np.random.default_rng(seed)
    q = rng.uniform(-1, 1, (B, qh, T, dh)).astype(np.float32)
    k = rng.uniform(-1, 1, (B, kvh, L, dh)).astype(np.float32)
    v = rng.uniform(-1, 1, (B, kvh, L, dh)).astype(np.float32)
    mask = None
    if mask_kind == "b11l":
        mask = rng.uniform(-3, 0, (B, 1, 1, L)).astype(np.float32)
    elif mask_kind == "11tl":
        mask = rng.uniform(-3, 0, (1, 1, T, L)).astype(np.float32)
    elif mask_kind == "bhtl":
        mask = rng.uniform(-3, 0, (B, qh, T, L)).astype(np.float32)
        # rows whose maximum lies in their last key tile: the online rescale must shrink what came before
        for s in (3, 40, 64):
            mask[:, :, s, s] = 12.0
        mask[0, 1, 5, :] = -np.inf  # a row masked wholly: zeros, not NaN
        mask[1, 2, 64, :] = -np.inf  # ... alone in its query tile
    return q, k, v, mask


def _run(rt, ctx, q, k, v, mask, nonpad, causal, v_layout, out=None):
    dq, dk, dv = _device_inputs(ctx, q, k, v, v_layout)
    qh, kvh = q.shape[1], k.shape[1]
    op = rt.Attention(is_causal=causal, q_num_heads=qh, kv_num_heads=kvh)
    dm = None if mask is None else ctx.to_device(mask)
    dl = None if nonpad is None else ctx.to_device(np.asarray(nonpad, np.int32))
    return op.run(ctx, dq, dk, dv, attn_mask=dm, nonpad_kv_seqlen=dl, out=out)


@pytest.mark.gpu
@pytest.mark.parametrize("tf32", [False, True], ids=["3xtf32", "tf32"])
@pytest.mark.parametrize("name,case", CASES, ids=[c[0] for c in CASES])
def test_prefill_attention_matches_float64(rt, name, case, tf32):
    B, qh, kvh, T, L, dh, causal, nonpad, mask_kind, v_layout = case
    if tf32 and L > 1024:
        pytest.skip("the TF32 bound is stated for <= 1024 keys")
    q, k, v, mask = _case_data(len(name), B, qh, kvh, T, L, dh, causal, nonpad, mask_kind)
    ref = ref_attention(q, k, v, mask, nonpad, causal)
    ctx = _ctx(rt, tf32)
    got = _run(rt, ctx, q, k, v, mask, nonpad, causal, v_layout).numpy()
    tol = 4e-3 if tf32 else 2e-5
    err = _rel_err(got, ref)
    assert got.shape == ref.shape and np.isfinite(got).all() and err <= tol, f"{name} (tf32={tf32}): rel err {err:.2e} > {tol}"
    dead = np.all(ref == 0.0, axis=-1)  # rows that see no key (or only -inf): exact zeros
    if mask_kind == "bhtl":
        assert dead[0, 1, 5] and dead[1, 2, 64]
    assert not got[dead].any(), f"{name}: fully masked rows are not exact zeros"


@pytest.mark.gpu
def test_prefill_attention_merged_projection_views(rt):
    """Q / K / V as strided [B, nh, S, dh] views of one [B, S, 3H] projection, the output written through a [B, S, H]
    view; 8 x 12 x 4 = 384 CTAs, more than the device has SMs."""
    B, nh, S, dh = 8, 12, 200, 64
    H = nh * dh
    rng = np.random.default_rng(11)
    qkv = rng.uniform(-1, 1, (B, S, 3 * H)).astype(np.float32)
    q, k, v = (qkv[:, :, i * H:(i + 1) * H].reshape(B, S, nh, dh).transpose(0, 2, 1, 3) for i in range(3))
    ref = ref_attention(q, k, v, causal=True)
    for tf32 in (False, True):
        ctx = _ctx(rt, tf32)
        dqkv = ctx.to_device(qkv)
        part = lambda i: dqkv.view((B, nh, S, dh), (S * 3 * H, dh, 3 * H, 1), i * H)
        att = ctx.empty((B, S, H))
        rt.Attention(is_causal=True).run(ctx, part(0), part(1), part(2), out=att.view((B, nh, S, dh), (S * H, dh, H, 1)))
        got = att.numpy().reshape(B, S, nh, dh).transpose(0, 2, 1, 3)
        tol = 4e-3 if tf32 else 2e-5
        assert _rel_err(got, ref) <= tol, f"merged views (tf32={tf32}): rel err {_rel_err(got, ref):.2e}"


def _kernel_probe():
    """Run in a child process (see below): the kernels of (1) the routed calls of CASES in both f32 modes, (2) a q_seq == 1
    call, (3) a non-causal equal-heads call the composed path served before; one CUPTI session each, printed as JSON."""
    import json
    import rten_b200 as rt
    calls = []
    for tf32 in (False, True):
        ctx = _ctx(rt, tf32)
        for name, case in CASES:
            B, qh, kvh, T, L, dh, causal, nonpad, mask_kind, v_layout = case
            calls.append((ctx, *_case_data(len(name), B, qh, kvh, T, L, dh, causal, nonpad, mask_kind), nonpad, causal, v_layout))
    _, routed = _kernels(lambda: [_run(rt, *c).numpy() for c in calls])
    ctx = _ctx(rt, False)
    rng = np.random.default_rng(3)
    q1, k, v = (rng.uniform(-1, 1, s).astype(np.float32) for s in ((2, 4, 1, 64), (2, 2, 50, 64), (2, 2, 50, 64)))
    _, decode = _kernels(lambda: rt.Attention(is_causal=True).run(ctx, ctx.to_device(q1), ctx.to_device(k), ctx.to_device(v),
                                                                  nonpad_kv_seqlen=ctx.to_device(np.array([50, 7], np.int32))).numpy())
    q, kk = rng.uniform(-1, 1, (2, 2, 40, 64)).astype(np.float32), rng.uniform(-1, 1, (2, 2, 50, 64)).astype(np.float32)
    _, composed = _kernels(lambda: rt.Attention().run(ctx, ctx.to_device(q), ctx.to_device(kk), ctx.to_device(kk)).numpy())
    print(json.dumps({"routed": sorted(routed), "decode": sorted(decode), "composed": sorted(composed)}))


@pytest.mark.gpu
def test_prefill_attention_kernel_identity():
    """The routed calls run attn_prefill_kernel (every head size and f32 mode, both value layouts, GQA, masks), q_seq == 1
    still runs attn_decode_kernel, and a call the composed path served before does not reach the new kernel.  The CUPTI
    sessions run in a child process, so that they leave no profiler state behind in the test session."""
    import json
    import os
    import subprocess
    import sys
    here = os.path.dirname(os.path.abspath(__file__))
    code = (f"import sys; sys.path[:0] = [{os.path.dirname(here)!r}, {here!r}]; "
            "import test_gpu_attention_prefill as t; t._kernel_probe()")
    res = subprocess.run([sys.executable, "-s", "-c", code], capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-4000:]
    names = json.loads(res.stdout.strip().splitlines()[-1])
    for dh in (64, 128):
        for x3 in ("true", "false"):
            assert any("attn_prefill_kernel" in n and f"<{dh}, {x3}>" in n for n in names["routed"]), \
                f"no attn_prefill_kernel<{dh}, {x3}> among {names['routed']}"
    assert any("attn_decode_kernel" in n for n in names["decode"]) and not any("attn_prefill_kernel" in n for n in names["decode"]), names["decode"]
    assert not any("attn_prefill_kernel" in n for n in names["composed"]), names["composed"]


@pytest.mark.gpu
def test_prefill_attention_unsupported_layout_keeps_its_error(rt):
    """A layout the prefill kernel does not take (head size 80, causal) keeps the composed path's error."""
    ctx = _ctx(rt, False)
    rng = np.random.default_rng(3)
    q80, k80 = rng.uniform(-1, 1, (1, 2, 8, 80)).astype(np.float32), rng.uniform(-1, 1, (1, 2, 8, 80)).astype(np.float32)
    with pytest.raises(rt.OpError) as e:
        rt.Attention(is_causal=True).run(ctx, ctx.to_device(q80), ctx.to_device(k80), ctx.to_device(k80))
    assert e.value.kind == "UnsupportedValue" and e.value.msg == "causal / padded attention with q_seq > 1: pass the additive mask explicitly"


@pytest.mark.gpu
@pytest.mark.parametrize("tf32", [False, True], ids=["3xtf32", "tf32"])
def test_prefill_attention_is_deterministic(rt, tf32):
    """Three runs of the same call give the same bits (no atomics, no split over CTAs)."""
    import gpu_checks as gc
    B, qh, kvh, T, L, dh = 3, 8, 2, 150, 700, 64
    q, k, v, mask = _case_data(21, B, qh, kvh, T, L, dh, True, None, "b11l")
    ctx = _ctx(rt, tf32)
    outs = [_run(rt, ctx, q, k, v, mask, [700, 150, 333], True, "transposed").numpy() for _ in range(3)]
    for i in (1, 2):
        gc.assert_bit_exact(outs[i], outs[0], f"prefill attention (tf32={tf32}) run {i + 1} vs run 1")


@pytest.mark.gpu
@pytest.mark.parametrize("tf32", [False, True], ids=["3xtf32", "tf32"])
def test_prefill_attention_graph_replay_reads_the_device_lengths(rt, tf32):
    """A causal call with nonpad_kv_seqlen captured in a CUDA graph, replayed after the device lengths were rewritten
    (shorter, longer, past the clamp at both ends), matches an eager call with those lengths bit for bit: the launch
    depends on shapes only and the kernel reads the lengths when it runs."""
    import gpu_checks as gc
    B, qh, kvh, T, L, dh = 3, 8, 2, 96, 400, 128
    q, k, v, _ = _case_data(7, B, qh, kvh, T, L, dh, True, None, None)
    ctx = _ctx(rt, tf32)
    dq, dk, dv = _device_inputs(ctx, q, k, v, "natural")
    dlen = ctx.to_device(np.array([400, 96, 250], np.int32))
    out = ctx.empty((B, qh, T, dh))
    op = rt.Attention(is_causal=True, q_num_heads=qh, kv_num_heads=kvh)
    run = lambda: op.run(ctx, dq, dk, dv, nonpad_kv_seqlen=dlen, out=out)
    run()  # warm-up outside the capture
    ctx.sync()
    ctx.graph_begin()
    run()
    graph = ctx.graph_end()
    tol = 4e-3 if tf32 else 2e-5
    for lens in ([400, 96, 250], [17, 300, 96], [0, 400, 50], [10000, -5, 399]):
        dlen.copy_from(np.array(lens, np.int32))
        graph.launch()
        ctx.sync()
        replayed = out.numpy()
        eager = _run(rt, ctx, q, k, v, None, lens, True, "natural").numpy()
        gc.assert_bit_exact(replayed, eager, f"graph replay (tf32={tf32}) with lengths {lens} vs an eager call")
        err = _rel_err(replayed, ref_attention(q, k, v, None, lens, True))
        assert err <= tol, f"graph replay (tf32={tf32}) with lengths {lens}: rel err {err:.2e}"


@pytest.mark.gpu
@pytest.mark.parametrize("P,T", [(0, 512), (100, 64)], ids=["prefill", "chunked"])
def test_prefill_attention_matches_the_gpt2_runner_composition(rt, P, T):
    """GPT2Int8Runner's cache layout (K [B,nh,M,dh], V^T [B,nh,dh,M], M = 576) and its attention composition (explicit
    additive causal mask, FusedMatMul -> AddSoftmax -> MatMul, 3xTF32): Attention(is_causal, nonpad = P + T) over the
    whole cache agrees within 2e-5 * max |ref|."""
    B, nh, dh, M = 8, 12, 64, 576
    Ltot = P + T
    rng = np.random.default_rng(P + T)
    ctx = _ctx(rt, False)
    kc = np.zeros((B, nh, M, dh), np.float32)
    vt = np.zeros((B, nh, dh, M), np.float32)
    kc[:, :, :Ltot] = rng.uniform(-1, 1, (B, nh, Ltot, dh))
    vt[:, :, :, :Ltot] = rng.uniform(-1, 1, (B, nh, dh, Ltot))
    q = rng.uniform(-1, 1, (B, nh, T, dh)).astype(np.float32)
    dq, dk, dvt = ctx.to_device(q), ctx.to_device(kc), ctx.to_device(vt)
    scale = 1.0 / math.sqrt(dh)
    # the runner's composition
    mask = np.where(np.arange(Ltot)[None, :] <= (P + np.arange(T))[:, None], 0.0, -np.inf).astype(np.float32).reshape(1, 1, T, Ltot)
    kt = dk.view((B, nh, dh, Ltot), (nh * M * dh, M * dh, 1, dh))
    scores = rt.FusedMatMul(scale).run(ctx, dq, kt)
    probs = rt.AddSoftmax().run(ctx, scores, ctx.to_device(mask), in_place=True)
    v = dvt.view((B, nh, Ltot, dh), (nh * dh * M, dh * M, 1, M))
    composed = rt.MatMul().run(ctx, probs, v).numpy()
    # one call over the whole cache, valid length on the device
    vfull = dvt.view((B, nh, M, dh), (nh * dh * M, dh * M, 1, M))
    got = rt.Attention(is_causal=True, q_num_heads=nh, kv_num_heads=nh, scale=scale).run(
        ctx, dq, dk, vfull, nonpad_kv_seqlen=ctx.to_device(np.full((B,), Ltot, np.int32))).numpy()
    err = _rel_err(got, composed)
    assert err <= 2e-5, f"GPT-2 prefill P={P} T={T}: rel err vs the runner's composition {err:.2e}"


def _attention_graph(B, S, E, nh, kvh, dh, seed):
    import onnx_writer as W
    rng = np.random.default_rng(seed)
    w = {"wq": rng.uniform(-0.2, 0.2, (E, nh * dh)), "wk": rng.uniform(-0.2, 0.2, (E, kvh * dh)),
         "wv": rng.uniform(-0.2, 0.2, (E, kvh * dh)), "wo": rng.uniform(-0.2, 0.2, (nh * dh, E))}
    w = {k: v.astype(np.float32) for k, v in w.items()}
    shapes = {"shq": np.array([B, S, nh, dh], np.int64), "shkv": np.array([B, S, kvh, dh], np.int64), "sho": np.array([B, S, nh * dh], np.int64)}
    nodes = [W.node("MatMul", ["x", "wq"], ["q0"]), W.node("MatMul", ["x", "wk"], ["k0"]), W.node("MatMul", ["x", "wv"], ["v0"]),
             W.node("Reshape", ["q0", "shq"], ["q1"]), W.node("Reshape", ["k0", "shkv"], ["k1"]), W.node("Reshape", ["v0", "shkv"], ["v1"]),
             W.node("Transpose", ["q1"], ["q"], perm=[0, 2, 1, 3]), W.node("Transpose", ["k1"], ["k"], perm=[0, 2, 1, 3]),
             W.node("Transpose", ["v1"], ["v"], perm=[0, 2, 1, 3]),
             W.node("Attention", ["q", "k", "v"], ["a"], is_causal=1, q_num_heads=nh, kv_num_heads=kvh),
             W.node("Transpose", ["a"], ["a1"], perm=[0, 2, 1, 3]), W.node("Reshape", ["a1", "sho"], ["a2"]),
             W.node("MatMul", ["a2", "wo"], ["y"])]
    inits = [W.tensor(k, v) for k, v in {**w, **shapes}.items()]
    data = W.model(nodes, inits, [W.value_info("x", W.FLOAT, [B, S, E])], [W.value_info("y", W.FLOAT, [B, S, E])], opset=23)
    return data, w


@pytest.mark.gpu
@pytest.mark.parametrize("nh,kvh", [(4, 4), (8, 2)], ids=["mha", "gqa"])
def test_prefill_attention_through_the_onnx_executor(rt, nh, kvh):
    """An exporter-form opset-23 graph (Q / K / V projections, Reshape / Transpose views, Attention(is_causal=1), merge,
    output projection) through Model.run against its float64 interpretation."""
    from rten_b200.model import Model
    B, S, E, dh = 2, 150, 96, 64
    data, w = _attention_graph(B, S, E, nh, kvh, dh, nh * 10 + kvh)
    x = np.random.default_rng(1).uniform(-1, 1, (B, S, E)).astype(np.float32)
    x64 = x.astype(np.float64)
    heads = lambda y, n: y.reshape(B, S, n, dh).transpose(0, 2, 1, 3)
    a = ref_attention(heads(x64 @ w["wq"], nh), heads(x64 @ w["wk"], kvh), heads(x64 @ w["wv"], kvh), causal=True)
    want = a.transpose(0, 2, 1, 3).reshape(B, S, nh * dh) @ w["wo"].astype(np.float64)
    ctx = _ctx(rt, False)
    m = Model(ctx, data)
    (y,) = m.run({"x": ctx.to_device(x)})
    err = _rel_err(y.numpy(), want)
    assert err <= 2e-5, f"executor Attention {nh}/{kvh}: rel err {err:.2e}"
