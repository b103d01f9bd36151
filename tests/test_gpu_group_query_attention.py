"""RotaryEmbedding and com.microsoft GroupQueryAttention: the rotary / cache-append kernel, the single-query attention
kernel with rotary embedding, cache append and sliding window fused in (decode steps), and the streaming prefill kernel
with a sliding window (prompts).

Every GPU assertion rests on two numpy restatements: `rotary_ref` (the reference's rotary_embedding,
src/ops/embedding.rs:46-207) and `ref_gqa` (GroupQueryAttention::run_impl and gqa_present_cache,
src/ops/attention/contrib.rs:369-810).  The CPU tests check `ref_gqa` against a literal row-by-row transcription of
those functions and `rotary_ref` against the reference's RotaryEmbedding known-answer cases (tests/golden).  In float32
`rotary_ref` rounds every product and sum on its own, as the kernels do, so rotated values and present caches compare
bit for bit.  Attention outputs: |d| <= 2e-5 * max |ref| in 3xTF32 (the prefill and decode kernels' bound) and
4e-3 * max |ref| for the prefill kernel in single-pass TF32."""
import json
import math
import os

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))

# ---------------------------------------------------------------------------------------------------------------------
# numpy restatements


def rotary_ref(x, cos, sin, interleaved, dtype=np.float64):
    """x [..., D] rotated over its first 2 * half elements with cos / sin [..., half] (broadcast against x[..., 0])."""
    x = np.asarray(x).astype(dtype)
    c, s = np.asarray(cos).astype(dtype), np.asarray(sin).astype(dtype)
    half = c.shape[-1]
    rd = 2 * half
    y = x.copy()
    if interleaved:
        x1, x2 = x[..., 0:rd:2], x[..., 1:rd:2]
        y[..., 0:rd:2] = x1 * c - x2 * s
        y[..., 1:rd:2] = x1 * s + x2 * c
    else:
        x1, x2 = x[..., :half], x[..., half:rd]
        y[..., :half] = x1 * c - x2 * s
        y[..., half:rd] = x1 * s + x2 * c
    return y


def _split_qkv(query, key, value, H, Hkv):
    B, S, hid = query.shape
    if key is None:
        D = hid // (H + 2 * Hkv)
        q, k, v = query[..., :H * D], query[..., H * D:(H + Hkv) * D], query[..., (H + Hkv) * D:]
    else:
        D = hid // H
        q, k, v = query, key, value
    return q.reshape(B, S, H, D), k.reshape(B, S, Hkv, D), v.reshape(B, S, Hkv, D), D


def ref_gqa(query, key, value, past_key, past_value, seqlens_k, total, H, Hkv, cos=None, sin=None, position_ids=None, bias=None,
            scale=None, do_rotary=False, interleaved=False, window=-1, dtype=np.float64):
    """(output [B, S, H * D], present_key, present_value [B, Hkv, P + S, D]) of GroupQueryAttention.  `dtype` is the
    precision of the rotary embedding and of the present caches; the attention itself is float64."""
    q, k, v, D = _split_qkv(query, key, value, H, Hkv)
    B, S = q.shape[:2]
    P = 0 if past_key is None else past_key.shape[2]
    T = P + S
    sk = np.asarray(seqlens_k).reshape(B).astype(np.int64)
    first = S == total
    past_len = np.zeros(B, np.int64) if first else sk + 1 - S
    q, k, v = q.astype(dtype), k.astype(dtype), v.astype(dtype)
    if do_rotary:
        pos = np.asarray(position_ids) if position_ids is not None else past_len[:, None] + np.arange(S)[None, :]
        c, s = np.asarray(cos)[pos][:, :, None], np.asarray(sin)[pos][:, :, None]
        q = rotary_ref(q, c, s, interleaved, dtype)
        k = rotary_ref(k, c, s, interleaved, dtype)
    pk = np.zeros((B, Hkv, T, D), dtype)
    pv = np.zeros((B, Hkv, T, D), dtype)
    for b in range(B):
        pl = past_len[b]
        if past_key is not None:
            pk[b, :, :pl] = past_key[b, :, :pl]
            pv[b, :, :pl] = past_value[b, :, :pl]
        pk[b, :, pl:pl + S] = k[b].transpose(1, 0, 2)
        pv[b, :, pl:pl + S] = v[b].transpose(1, 0, 2)
    scale = 1.0 / math.sqrt(D) if scale is None else scale
    out = np.zeros((B, S, H, D))
    g = H // Hkv
    for b in range(B):
        L = sk[b] + 1
        K = np.repeat(pk[b, :, :L].astype(np.float64), g, axis=0)  # [H, L, D]
        V = np.repeat(pv[b, :, :L].astype(np.float64), g, axis=0)
        sc = scale * np.einsum("shd,hld->hsl", q[b].astype(np.float64), K)
        if bias is not None:
            bb = bias[0 if bias.shape[0] == 1 else b][:, :S, :L].astype(np.float64)
            sc = sc + bb
        t = np.arange(L)[None, :]
        causal = past_len[b] + np.arange(S)[:, None] + 1
        start = np.where((window > 0) & (causal > window), causal - window, 0) if window > 0 else np.zeros_like(causal)
        sc = np.where((t < start) | (t >= causal), -np.inf, sc)
        p = np.exp(sc - sc.max(-1, keepdims=True))
        p = p / p.sum(-1, keepdims=True)
        out[b] = np.einsum("hsl,hld->shd", p, V)
    return out.reshape(B, S, H * D), pk, pv


def _loop_gqa(query, key, value, past_key, past_value, seqlens_k, total, H, Hkv, cos, sin, position_ids, bias, scale, do_rotary,
              interleaved, window):
    """GroupQueryAttention::run_impl with gqa_present_cache and rotary_embedding, transcribed row by row (float64)."""
    q, k, v, D = _split_qkv(query, key, value, H, Hkv)
    B, S = q.shape[:2]
    P = 0 if past_key is None else past_key.shape[2]
    T = P + S
    first = S == total

    def past_len(b):
        return 0 if first else int(seqlens_k[b]) + 1 - S

    def rotate(x, b, s):
        if not do_rotary:
            return [float(e) for e in x]
        half = cos.shape[1]
        p = int(position_ids[b][s]) if position_ids is not None else past_len(b) + s
        c, sn = cos[p], sin[p]
        y = [float(e) for e in x]
        for i in range(half):
            if interleaved:
                x1, x2 = float(x[2 * i]), float(x[2 * i + 1])
                y[2 * i], y[2 * i + 1] = x1 * c[i] - x2 * sn[i], x1 * sn[i] + x2 * c[i]
            else:
                x1, x2 = float(x[i]), float(x[half + i])
                y[i], y[half + i] = x1 * c[i] - x2 * sn[i], x1 * sn[i] + x2 * c[i]
        return y

    rq = [[[rotate(q[b, s, h], b, s) for h in range(H)] for s in range(S)] for b in range(B)]
    rk = [[[rotate(k[b, s, h], b, s) for h in range(Hkv)] for s in range(S)] for b in range(B)]

    def present(new, past):
        cache = np.zeros((B, Hkv, T, D))
        for b in range(B):
            pb = past_len(b)
            for h in range(Hkv):
                if past is not None:
                    cache[b, h, :pb] = past[b, h, :pb]
                for s in range(S):
                    cache[b, h, pb + s] = new(b, s, h)
        return cache

    pk = present(lambda b, s, h: rk[b][s][h], past_key)
    pv = present(lambda b, s, h: v[b, s, h], past_value)
    scale = 1.0 / math.sqrt(D) if scale is None else scale
    out = np.zeros((B, S, H * D))
    for b in range(B):
        for n in range(H):
            hk = n // (H // Hkv)
            kv_len = int(seqlens_k[b]) + 1
            for s in range(S):
                row = [scale * sum(rq[b][s][n][d] * pk[b, hk, t, d] for d in range(D)) for t in range(kv_len)]
                seq_causal = past_len(b) + s + 1
                start, width = (seq_causal - window, window) if window > 0 and seq_causal > window else (0, seq_causal)
                if bias is not None:
                    brow = bias[0 if bias.shape[0] == 1 else b, 0 if bias.shape[1] == 1 else n, s]
                    for t in range(start, start + width):
                        row[t] += float(brow[t])
                for t in range(0, start):
                    row[t] = -math.inf
                for t in range(seq_causal, kv_len):
                    row[t] = -math.inf
                mx = max(row)
                e = [math.exp(x - mx) for x in row]
                tot = sum(e)
                for d in range(D):
                    out[b, s, n * D + d] = sum(e[t] / tot * pv[b, hk, t, d] for t in range(kv_len))
    return out, pk, pv


# (name, B, S, P, H, Hkv, D, first, seqlens_k, rotary (None | "halves" | "interleaved"), partial rotary, position_ids,
#  local_window_size, bias (None | "b1" | "1h"), packed QKV)
CPU_CASES = [
    ("first prompt", 2, 4, 0, 4, 2, 4, True, [3, 3], None, False, False, -1, None, False),
    ("first prompt over a non-empty past", 1, 3, 2, 2, 1, 4, True, [4], "halves", False, False, -1, None, False),
    ("right-padded decode", 3, 1, 5, 4, 2, 6, False, [5, 2, 3], "interleaved", False, False, -1, "b1", False),
    ("subsequent prompt", 1, 3, 4, 4, 1, 4, False, [5], "halves", True, True, -1, "1h", True),
    ("window at prefill", 1, 6, 0, 2, 2, 4, True, [5], "interleaved", True, False, 3, None, False),
    ("window at decode", 2, 1, 6, 2, 1, 8, False, [6, 4], "halves", True, True, 2, "b1", True),
]


def _cpu_case(seed, B, S, P, H, Hkv, D, first, sk, rot, partial, use_pos, window, bias_kind, packed):
    rng = np.random.default_rng(seed)
    hid = (H + 2 * Hkv) * D if packed else H * D
    query = rng.standard_normal((B, S, hid))
    key = None if packed else rng.standard_normal((B, S, Hkv * D))
    value = None if packed else rng.standard_normal((B, S, Hkv * D))
    pk = rng.standard_normal((B, Hkv, P, D)) if P else None
    pv = rng.standard_normal((B, Hkv, P, D)) if P else None
    total = S if first else max(sk) + 1
    half = (D // 4) if partial else D // 2
    cos = sin = pos = None
    if rot:
        ang = rng.uniform(0, 6.3, (16, half))
        cos, sin = np.cos(ang), np.sin(ang)
        if use_pos:
            pos = rng.integers(0, 16, (B, S))
    bias = None
    if bias_kind:
        shape = (B, 1, S + 1, P + S + 2) if bias_kind == "b1" else (1, H, S, P + S)
        bias = rng.uniform(-2, 0, shape)
    return (query, key, value, pk, pv, np.array(sk), total, H, Hkv, cos, sin, pos, bias, 0.3, rot is not None, rot == "interleaved", window)


def test_reference_gqa_matches_the_row_loop():
    for i, (name, *case) in enumerate(CPU_CASES):
        args = _cpu_case(i, *case)
        want = _loop_gqa(*args)
        (query, key, value, pk, pv, sk, total, H, Hkv, cos, sin, pos, bias, scale, rot, inter, window) = args
        got = ref_gqa(query, key, value, pk, pv, sk, total, H, Hkv, cos, sin, pos, bias, scale, rot, inter, window)
        for g, w, what in zip(got, want, ("output", "present_key", "present_value")):
            np.testing.assert_allclose(g, w, rtol=1e-12, atol=1e-12, err_msg=f"{name}: {what}")
        for b in range(len(sk)):  # present positions after the new tokens are zeros
            end = case[1] if case[6] else int(sk[b]) + 1
            assert not got[1][b, :, end:].any() and not got[2][b, :, end:].any(), name


def _golden_cases():
    with open(os.path.join(HERE, "golden", "rotary_embedding_cases.json")) as f:
        return json.load(f)["cases"]


def _rotary_ref_op(x, cos, sin, pos, interleaved, num_heads, rd, dtype=np.float64):
    """RotaryEmbedding (src/ops/embedding.rs:46-207) on numpy arrays, via rotary_ref."""
    x = np.asarray(x)
    if x.ndim == 3:
        B, S, hid = x.shape
        xr = x.reshape(B, S, num_heads, hid // num_heads)
    else:
        xr = x.transpose(0, 2, 1, 3)
    B, S, nh, D = xr.shape
    rd = rd or D
    cos, sin = np.asarray(cos), np.asarray(sin)
    if pos is not None:
        cos, sin = cos[np.asarray(pos)], sin[np.asarray(pos)]
    cos, sin = np.broadcast_to(cos, (B, S, rd // 2)), np.broadcast_to(sin, (B, S, rd // 2))
    y = rotary_ref(xr, cos[:, :, None], sin[:, :, None], interleaved, dtype)
    return y.reshape(x.shape) if x.ndim == 3 else y.transpose(0, 2, 1, 3)


def test_rotary_restatement_reproduces_the_known_answers():
    for c in _golden_cases():
        got = _rotary_ref_op(c["input"], c["cos"], c["sin"], c["position_ids"], c["interleaved"], c["num_heads"], c["rotary_embedding_dim"])
        np.testing.assert_allclose(got, np.array(c["expected"]), atol=1e-4, rtol=0, err_msg=c["name"])


# ---------------------------------------------------------------------------------------------------------------------
# GPU


@pytest.fixture(scope="module")
def rt():
    import rten_b200
    from rten_b200 import _lib
    _lib.load()
    return rten_b200


def _ctx(rt, tf32=False):
    ctx = rt.Context(0)
    ctx.set_f32_mode(not tf32)
    return ctx


def _rel_err(got, ref):
    return float(np.abs(np.asarray(got, np.float64) - ref).max() / max(float(np.abs(ref).max()), 1e-30))


def _bits_equal(a, b, what):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    assert a.shape == b.shape, f"{what}: shape {a.shape} vs {b.shape}"
    bad = a.view(np.uint32) != b.view(np.uint32)
    assert not bad.any(), f"{what}: {int(bad.sum())} elements differ, first at {np.argwhere(bad)[0]}"


@pytest.mark.gpu
@pytest.mark.parametrize("case", _golden_cases(), ids=lambda c: c["name"])
def test_rotary_embedding_known_answers_bit_exact(rt, case):
    ctx = _ctx(rt)
    x = np.array(case["input"], np.float32)
    cos, sin = np.array(case["cos"], np.float32), np.array(case["sin"], np.float32)
    pos = None if case["position_ids"] is None else np.array(case["position_ids"], np.int32)
    op = rt.RotaryEmbedding(case["interleaved"], case["num_heads"], case["rotary_embedding_dim"])
    got = op.run(ctx, ctx.to_device(x), ctx.to_device(cos), ctx.to_device(sin), None if pos is None else ctx.to_device(pos)).numpy()
    _bits_equal(got, _rotary_ref_op(x, cos, sin, pos, case["interleaved"], case["num_heads"], case["rotary_embedding_dim"], np.float32), case["name"])
    np.testing.assert_allclose(got, np.array(case["expected"]), atol=1e-4, rtol=0)


@pytest.mark.gpu
@pytest.mark.parametrize("layout", ["3d", "4d", "4d strided"])
@pytest.mark.parametrize("interleaved", [False, True], ids=["halves", "interleaved"])
@pytest.mark.parametrize("rd", [0, 48])
@pytest.mark.parametrize("source", ["position_ids host", "position_ids device", "broadcast cache"])
def test_rotary_embedding_bit_exact(rt, layout, interleaved, rd, source):
    B, S, nh, D, maxp = 3, 37, 5, 64, 200
    rng = np.random.default_rng(hash((layout, interleaved, rd, source)) % 1000)
    half = (rd or D) // 2
    ang = rng.uniform(0, 6.3, (maxp, half))
    cos, sin = np.cos(ang).astype(np.float32), np.sin(ang).astype(np.float32)
    ctx = _ctx(rt)
    pos = None
    if source == "broadcast cache":
        cos, sin = cos[None, :S], sin[None, :S]  # [1, S, half]
    else:
        pos = rng.integers(0, maxp, (B, S)).astype(np.int32)
    if layout == "3d":
        x = rng.standard_normal((B, S, nh * D)).astype(np.float32)
        dx = ctx.to_device(x)
    else:
        x = rng.standard_normal((B, nh, S, D)).astype(np.float32)
        if layout == "4d strided":  # a [B, nh, S, D] view of a [B, S, nh, D] buffer
            dbuf = ctx.to_device(np.ascontiguousarray(x.transpose(0, 2, 1, 3)))
            dx = dbuf.view((B, nh, S, D), (S * nh * D, D, nh * D, 1))
        else:
            dx = ctx.to_device(x)
    dpos = None if pos is None else (pos if source == "position_ids host" else ctx.to_device(pos))
    got = rt.RotaryEmbedding(interleaved, nh, rd).run(ctx, dx, ctx.to_device(cos), ctx.to_device(sin), dpos).numpy()
    _bits_equal(got, _rotary_ref_op(x, cos, sin, pos, interleaved, nh, rd, np.float32), f"RotaryEmbedding {layout} {source}")


@pytest.mark.gpu
def test_rotary_embedding_errors(rt):
    ctx = _ctx(rt)
    x = np.zeros((1, 2, 8), np.float32)
    c = np.zeros((1, 2, 2), np.float32)
    cases = [
        (dict(num_heads=0), (x, c, c, None), "InvalidValue", "num_heads must not be 0 for 3 dimensioned input"),
        (dict(num_heads=3), (x, c, c, None), "InvalidValue", "hidden_size must be divisible by num_heads"),
        (dict(num_heads=2, rotary_embedding_dim=3), (x, c, c, None), "InvalidValue", "rotary_embedding_dim must be a positive even number"),
        (dict(num_heads=2, rotary_embedding_dim=6), (x, c, c, None), "InvalidValue", "rotary_embedding_dim must not exceed head size"),
        (dict(num_heads=2), (x, np.zeros((1, 2, 3), np.float32), c, None), "InvalidValue", "Last dimension of cos cache does not match rotary_embedding_dim/2"),
        (dict(num_heads=2), (x, c, np.zeros((1, 2, 1), np.float32), None), "InvalidValue", "Last dimension of sin cache does not match rotary_embedding_dim/2"),
        (dict(num_heads=2), (x, np.zeros((1, 3, 2), np.float32), c, None), "InvalidValue", "cos/sin cache sequence length must be 1 or match the input"),
        (dict(num_heads=2), (x, np.zeros((2, 2, 2), np.float32), c, None), "InvalidValue", "cos/sin cache batch size must be 1 or match the input"),
        (dict(num_heads=2), (x, np.zeros((2, 2), np.float32), np.zeros((2, 2), np.float32), np.array([[0, 2]], np.int32)), "InvalidValue",
         "Entry in `indices` is out of range"),
        (dict(num_heads=2), (np.zeros((2, 8), np.float32), c, c, None), "IncompatibleInputShapes", "Input processed needs 3-4 dimensions"),
    ]
    for attrs, (xi, ci, si, pi), kind, msg in cases:
        with pytest.raises(rt.OpError) as e:
            rt.RotaryEmbedding(**attrs).run(ctx, xi, ci, si, pi)
        assert (e.value.kind, e.value.msg) == (kind, msg), attrs


# (name, B, S, P, H, Hkv, D, first, seqlens_k, rotary, partial, position_ids, window, bias, packed, aliased present, device lens)
GPU_CASES = [
    ("first prompt, GQA 32/8 D128 halves", 1, 300, 0, 32, 8, 128, True, [299], "halves", False, False, -1, None, False, False, True),
    ("first prompt over a non-empty past", 2, 70, 40, 8, 2, 64, True, [69, 69], "interleaved", False, False, -1, None, False, False, False),
    ("first prompt, packed, bias on batch", 3, 65, 0, 4, 4, 64, True, [64, 64, 64], "halves", True, False, -1, "b1", True, False, True),
    ("subsequent prompt B=1, aliased", 1, 100, 500, 16, 2, 128, False, [599], "halves", False, True, -1, "1h", False, True, True),
    ("subsequent prompt B=1, window < context", 1, 130, 300, 8, 1, 64, False, [420], "interleaved", True, False, 100, None, False, True, False),
    ("subsequent prompt, window > context", 1, 64, 64, 8, 8, 64, False, [127], None, False, False, 1000, "b1", True, False, True),
    ("prefill window < context, no rotary", 2, 200, 0, 4, 1, 128, True, [199, 199], None, False, False, 33, None, False, False, True),
    ("decode, right-padded, aliased, GQA 8", 4, 1, 700, 32, 4, 128, False, [699, 10, 350, 0], "halves", False, False, -1, None, False, True, True),
    ("decode, built present, host lens", 3, 1, 90, 8, 2, 64, False, [89, 50, 1], "interleaved", True, True, -1, "b1", False, False, False),
    ("decode, packed, bias on heads", 2, 1, 257, 16, 16, 64, False, [257, 100], "halves", False, False, -1, "1h", True, True, True),
    ("decode, window < context", 2, 1, 600, 8, 1, 128, False, [600, 300], "halves", True, False, 129, None, False, True, True),
    ("decode, window > context, no rotary", 2, 1, 60, 4, 2, 64, False, [60, 7], None, False, False, 5000, "b1", False, False, True),
    ("decode D64 group 8 position_ids", 3, 1, 33, 16, 2, 64, False, [20, 33, 5], "interleaved", False, True, -1, None, True, True, True),
] + [
    # window starts that are not a multiple of 4: (seqlens_k + 1 - window) % 4 = 3, 2, 1 (the first split masks 1-3 loaded positions)
    (f"decode D{D} window {w}", 2, 1, 600, 8, 2, D, False, [600, 300], "halves", False, False, w, "b1" if D == 64 else None, False, True, True)
    for D in (64, 128) for w in (130, 131, 132)
]


def _gpu_case(seed, B, S, P, H, Hkv, D, first, sk, rot, partial, use_pos, window, bias_kind, packed):
    rng = np.random.default_rng(seed)
    f = np.float32
    hid = (H + 2 * Hkv) * D if packed else H * D
    query = rng.uniform(-1, 1, (B, S, hid)).astype(f)
    key = None if packed else rng.uniform(-1, 1, (B, S, Hkv * D)).astype(f)
    value = None if packed else rng.uniform(-1, 1, (B, S, Hkv * D)).astype(f)
    pk = rng.uniform(-1, 1, (B, Hkv, P, D)).astype(f) if P else None
    pv = rng.uniform(-1, 1, (B, Hkv, P, D)).astype(f) if P else None
    total = S if first else max(sk) + 1
    half = D // 4 if partial else D // 2
    cos = sin = pos = None
    if rot:
        maxp = P + S + 8
        inv = 10000.0 ** (-np.arange(half) / half)
        ang = np.arange(maxp)[:, None] * inv[None, :]
        cos, sin = np.cos(ang).astype(f), np.sin(ang).astype(f)
        if use_pos:
            pos = rng.integers(0, maxp, (B, S)).astype(np.int32)
    bias = None
    if bias_kind:
        shape = (B, 1, S + 3, P + S + 5) if bias_kind == "b1" else (1, H, S, P + S)
        bias = rng.uniform(-2, 0, shape).astype(f)
    return query, key, value, pk, pv, np.array(sk, np.int32), total, cos, sin, pos, bias


def _run_gqa(rt, ctx, data, H, Hkv, rot, window, aliased, dev_lens, sentinel=7.5):
    """Run the operator; returns (out, present_key, present_value, launches, initial present buffers).  aliased: the
    present caches are the past buffers ([B, Hkv, P + S, D], past = the first P positions) holding `sentinel` beyond P."""
    query, key, value, pk, pv, sk, total, cos, sin, pos, bias = data
    B, S = query.shape[:2]
    D = (query.shape[2] // (H + 2 * Hkv)) if key is None else query.shape[2] // H
    P = 0 if pk is None else pk.shape[2]
    T = P + S
    dv = lambda a: None if a is None else ctx.to_device(a)
    inits = []
    args = dict(past_key=dv(pk), past_value=dv(pv), cos_cache=dv(cos), sin_cache=dv(sin), position_ids=dv(pos), attention_bias=dv(bias))
    if aliased:
        bufs = []
        for past in (pk, pv):
            full = np.full((B, Hkv, T, D), sentinel, np.float32)
            full[:, :, :P] = past
            inits.append(full)
            bufs.append(ctx.to_device(full))
        st = (Hkv * T * D, T * D, D, 1)
        args["past_key"], args["past_value"] = (b.view((B, Hkv, P, D), st) for b in bufs)
        args["present_key"], args["present_value"] = bufs
    op = rt.GroupQueryAttention(H, Hkv, do_rotary=rot is not None, rotary_interleaved=rot == "interleaved", local_window_size=window)
    dq, dk, dvv = dv(query), dv(key), dv(value)
    dl = ctx.to_device(sk) if dev_lens else sk
    ctx.sync()
    n0 = ctx.launches
    o, k, v = op.run(ctx, dq, dk, dvv, dl, total, **args)
    n = ctx.launches - n0
    return o.numpy(), k.numpy(), v.numpy(), n, inits


@pytest.mark.gpu
@pytest.mark.parametrize("name,case", [(c[0], c[1:]) for c in GPU_CASES], ids=[c[0] for c in GPU_CASES])
def test_group_query_attention_matches_the_restatement(rt, name, case):
    B, S, P, H, Hkv, D, first, sk, rot, partial, use_pos, window, bias_kind, packed, aliased, dev_lens = case
    data = _gpu_case(len(name), B, S, P, H, Hkv, D, first, sk, rot, partial, use_pos, window, bias_kind, packed)
    query, key, value, pk, pv, skv, total, cos, sin, pos, bias = data
    ref = ref_gqa(query, key, value, pk, pv, skv, total, H, Hkv, cos, sin, pos, bias, None, rot is not None, rot == "interleaved", window)
    ref32 = ref_gqa(query, key, value, pk, pv, skv, total, H, Hkv, cos, sin, pos, bias, None, rot is not None, rot == "interleaved",
                    window, dtype=np.float32)
    decode = S == 1 and not first
    for tf32 in ((False,) if decode else (False, True)):
        ctx = _ctx(rt, tf32)
        out, prk, prv, n, inits = _run_gqa(rt, ctx, data, H, Hkv, rot, window, aliased, dev_lens)
        tol = 4e-3 if tf32 else 2e-5
        err = _rel_err(out, ref[0])
        assert np.isfinite(out).all() and err <= tol, f"{name} (tf32={tf32}): rel err {err:.2e} > {tol}"
        for i, (got, want, what) in enumerate(((prk, ref32[1], "present_key"), (prv, ref32[2], "present_value"))):
            if aliased:
                for b in range(B):
                    L = int(sk[b]) + 1
                    _bits_equal(got[b, :, :L], want[b, :, :L], f"{name}: {what}[{b}] valid positions")
                    _bits_equal(got[b, :, L:], inits[i][b, :, L:], f"{name}: {what}[{b}] positions past seqlens_k + 1 (untouched)")
            else:
                _bits_equal(got, want, f"{name}: {what}")
        # launches: aliased decode = 1; prompts = 2; each + 1 for a built present over a non-empty past
        want_n = (1 if decode else 2) + (0 if aliased or P == 0 else 1)
        assert n == want_n, f"{name}: {n} launches, expected {want_n}"


@pytest.mark.gpu
def test_group_query_attention_rejects_a_present_cache_overlapping_the_past(rt):
    """A present cache in a past buffer's memory but with other strides is refused rather than read and written by one
    kernel at once: a contiguous [B, Hkv, P + 1, D] present_key over a contiguous [B, Hkv, P, D] past, and an in-place
    present_key (the past_key buffer itself) that overlaps past_value."""
    B, H, Hkv, D, P = 2, 4, 2, 64, 10
    ctx = _ctx(rt)
    buf = ctx.empty((B * Hkv * (P + 1) * D,))
    dense = buf.view((B, Hkv, P, D), (Hkv * P * D, P * D, D, 1))
    pres = buf.view((B, Hkv, P + 1, D), (Hkv * (P + 1) * D, (P + 1) * D, D, 1))
    in_place = buf.view((B, Hkv, P, D), (Hkv * (P + 1) * D, (P + 1) * D, D, 1))
    other = ctx.empty((B, Hkv, P + 1, D))
    q, k = ctx.empty((B, 1, H * D)), ctx.empty((B, 1, Hkv * D))
    for past_key, past_value in ((dense, dense), (in_place, dense)):
        with pytest.raises(rt.OpError) as e:
            rt.GroupQueryAttention(H, Hkv).run(ctx, q, k, k, np.array([P, P], np.int32), P + 1, past_key=past_key,
                                                past_value=past_value, present_key=pres, present_value=other)
        assert e.value.kind == "UnsupportedOutput" and "overlap a past cache" in e.value.msg


@pytest.mark.gpu
def test_group_query_attention_first_prompt_ignores_a_non_empty_past(rt):
    """A first prompt given a non-empty past: past_len is 0 (the past is not attended and not copied), and the kernel's
    effective key length S keeps the prefill kernel's offset at 0."""
    B, S, P, H, Hkv, D = 2, 50, 30, 4, 2, 64
    data = _gpu_case(3, B, S, P, H, Hkv, D, True, [S - 1, S + 10], None, False, False, -1, None, False)
    query, key, value, pk, pv, sk, total, *_ = data
    ref = ref_gqa(query, key, value, pk, pv, sk, total, H, Hkv)
    ctx = _ctx(rt)
    out, prk, prv, _, _ = _run_gqa(rt, ctx, data, H, Hkv, None, -1, False, True)
    assert _rel_err(out, ref[0]) <= 2e-5
    assert not prk[:, :, S:].any() and not prv[:, :, S:].any()
    _bits_equal(prk[:, :, :S], key.reshape(B, S, Hkv, D).transpose(0, 2, 1, 3), "present_key new tokens")


@pytest.mark.gpu
def test_group_query_attention_decode_graph_replay(rt):
    """One aliased decode step with device seqlens_k captured in a CUDA graph and replayed while seqlens_k and the
    projections advance on the device gives the bytes of eager calls on an identical cache at every step."""
    import gpu_checks as gc
    B, H, Hkv, D, T = 3, 16, 4, 128, 300
    rng = np.random.default_rng(9)
    ang = np.arange(T)[:, None] * (10000.0 ** (-np.arange(D // 2) / (D // 2)))[None, :]
    cos, sin = np.cos(ang).astype(np.float32), np.sin(ang).astype(np.float32)
    ctx = _ctx(rt)
    caches = []
    for _ in range(2):  # graph, eager
        init = rng.uniform(-1, 1, (2, B, Hkv, T, D)).astype(np.float32) if not caches else caches[0][2]
        kc, vc = ctx.to_device(init[0]), ctx.to_device(init[1])
        caches.append((kc, vc, init))
    st = (Hkv * T * D, T * D, D, 1)
    P = T - 1
    op = rt.GroupQueryAttention(H, Hkv, do_rotary=True)
    dq, dk, dv = ctx.empty((B, 1, H * D)), ctx.empty((B, 1, Hkv * D)), ctx.empty((B, 1, Hkv * D))
    dlen = ctx.to_device(np.array([5, 100, 200], np.int32))
    dcos, dsin = ctx.to_device(cos), ctx.to_device(sin)
    out_g = ctx.empty((B, 1, H * D))

    def step(kc, vc, out=None):
        return op.run(ctx, dq, dk, dv, dlen, T, past_key=kc.view((B, Hkv, P, D), st), past_value=vc.view((B, Hkv, P, D), st),
                      cos_cache=dcos, sin_cache=dsin, present_key=kc, present_value=vc, out=out)

    warm = [ctx.to_device(caches[0][2][i]) for i in range(2)]  # one eager step first: nothing is allocated while capturing
    step(*warm)
    lens = [np.array([5, 100, 200], np.int32) + i for i in range(4)]
    new = [[rng.uniform(-1, 1, s).astype(np.float32) for s in ((B, 1, H * D), (B, 1, Hkv * D), (B, 1, Hkv * D))] for _ in lens]
    for t, a in zip((dq, dk, dv), new[0]):
        t.copy_from(a)
    ctx.sync()
    ctx.graph_begin()
    step(caches[0][0], caches[0][1], out_g)
    graph = ctx.graph_end()
    for i, ln in enumerate(lens):
        dlen.copy_from(ln)
        for t, a in zip((dq, dk, dv), new[i]):
            t.copy_from(a)
        n0 = ctx.launches
        graph.launch()
        assert ctx.launches - n0 == 1, "a replayed decode step is one kernel launch"
        ctx.sync()
        g = out_g.numpy()
        e = step(caches[1][0], caches[1][1])[0].numpy()
        gc.assert_bit_exact(g, e, f"graph replay step {i}: output")
        gc.assert_bit_exact(caches[0][0].numpy(), caches[1][0].numpy(), f"graph replay step {i}: key cache")
        gc.assert_bit_exact(caches[0][1].numpy(), caches[1][1].numpy(), f"graph replay step {i}: value cache")


@pytest.mark.gpu
def test_group_query_attention_errors(rt):
    ctx = _ctx(rt)
    B, S, H, Hkv, D, P = 2, 1, 4, 2, 64, 6
    rng = np.random.default_rng(1)
    q = rng.standard_normal((B, S, H * D)).astype(np.float32)
    k = rng.standard_normal((B, S, Hkv * D)).astype(np.float32)
    pk = rng.standard_normal((B, Hkv, P, D)).astype(np.float32)
    sk = np.array([6, 3], np.int32)
    cs = np.zeros((16, D // 2), np.float32)
    base = dict(query=q, key=k, value=k, seqlens_k=sk, total_sequence_length=7, past_key=pk, past_value=pk)

    def check(kind, msg, attrs=None, **over):
        a = dict(base, **over)
        op = rt.GroupQueryAttention(**dict(dict(num_heads=H, kv_num_heads=Hkv), **(attrs or {})))
        with pytest.raises(rt.OpError) as e:
            op.run(ctx, a.pop("query"), a.pop("key"), a.pop("value"), a.pop("seqlens_k"), a.pop("total_sequence_length"), **a)
        assert (e.value.kind, e.value.msg) == (kind, msg)

    check("InvalidValue", "seqlens_k entry is out of range", seqlens_k=np.array([7, 3], np.int32))
    check("InvalidValue", "seqlens_k entry is out of range", seqlens_k=np.array([-1, 3], np.int32))
    check("InvalidValue", "seqlens_k entry is too small for the query sequence length", query=np.zeros((1, 3, H * D), np.float32),
          key=np.zeros((1, 3, Hkv * D), np.float32), value=np.zeros((1, 3, Hkv * D), np.float32), seqlens_k=np.array([1], np.int32),
          past_key=pk[:1], past_value=pk[:1])
    check("IncompatibleInputShapes", "seqlens_k must have batch_size elements", seqlens_k=np.array([6], np.int32))
    check("InvalidValue", "key and value must both be present or both absent", value=None)
    check("InvalidValue", "past_key and past_value must both be present or both absent", past_value=None)
    check("IncompatibleInputShapes", "past_key/past_value shape does not match", past_value=pk[:, :, :5])
    check("IncompatibleInputShapes", "key and value batch size must match query", key=k[:1], value=k[:1])
    check("IncompatibleInputShapes", "key hidden size must equal kv_num_heads * head_size", key=q, value=q)
    check("InvalidValue", "total_sequence_length must be positive", total_sequence_length=0)
    check("InvalidValue", "sequence_length must be 1 when query is not a prompt", query=np.zeros((B, 0, H * D), np.float32),
          key=np.zeros((B, 0, Hkv * D), np.float32), value=np.zeros((B, 0, Hkv * D), np.float32))
    check("UnsupportedValue", "batch size must be 1 when sequence_length > 1 and a past context is given", query=np.zeros((B, 2, H * D), np.float32),
          key=np.zeros((B, 2, Hkv * D), np.float32), value=np.zeros((B, 2, Hkv * D), np.float32))
    check("IncompatibleInputShapes", "attention_bias shape is incompatible with query/key shapes", attention_bias=np.zeros((B, 1, 1, P), np.float32))
    check("InvalidValue", "num_heads must be a multiple of kv_num_heads", attrs=dict(num_heads=3))
    check("InvalidValue", "num_heads and kv_num_heads must be positive", attrs=dict(kv_num_heads=0))
    check("InvalidValue", "cos_cache and sin_cache are required when do_rotary is set", attrs=dict(do_rotary=True))
    check("InvalidValue", "rotary_embedding_dim must not exceed head size", attrs=dict(do_rotary=True),
          cos_cache=np.zeros((16, D), np.float32), sin_cache=np.zeros((16, D), np.float32))
    check("InvalidValue", "Last dimension of sin cache does not match rotary_embedding_dim/2", attrs=dict(do_rotary=True),
          cos_cache=cs, sin_cache=np.zeros((16, 4), np.float32))
    check("InvalidValue", "Entry in `indices` is out of range", attrs=dict(do_rotary=True), cos_cache=cs[:5], sin_cache=cs[:5])
    check("InvalidValue", "Entry in `indices` is out of range", attrs=dict(do_rotary=True), cos_cache=cs, sin_cache=cs,
          position_ids=np.array([[3], [16]], np.int32))
    check("CastFailed", "conversion error for input 7: expected tensor with 2 dims but has 3 dims", attrs=dict(do_rotary=True),
          cos_cache=cs[None], sin_cache=cs[None])
    check("CastFailed", "conversion error for input 6: expected tensor with 0 dims but has 1 dims", total_sequence_length=np.array([7], np.int32))
    check("UnsupportedValue", "GroupQueryAttention softcap is not supported", attrs=dict(softcap=30.0))
    check("UnsupportedValue", "smooth_softmax is not supported", attrs=dict(smooth_softmax=True))
    q80 = np.zeros((B, S, H * 80), np.float32)
    check("UnsupportedValue", "GroupQueryAttention: the head size must be 64 or 128", query=q80, key=np.zeros((B, S, Hkv * 80), np.float32),
          value=np.zeros((B, S, Hkv * 80), np.float32), past_key=np.zeros((B, Hkv, P, 80), np.float32), past_value=np.zeros((B, Hkv, P, 80), np.float32))
    big = np.zeros((B, Hkv, 8192, D), np.float32)
    check("UnsupportedValue", "GroupQueryAttention: a decode step takes at most 8192 cache positions (past + 1)", past_key=big, past_value=big)


def _gqa_graph(B, S, P, H, Hkv, D, maxp, seed):
    import onnx_writer as W
    rng = np.random.default_rng(seed)
    half = D // 2
    ang = np.arange(maxp)[:, None] * (10000.0 ** (-np.arange(half) / half))[None, :]
    cos, sin = np.cos(ang).astype(np.float32), np.sin(ang).astype(np.float32)
    inits = [W.tensor("cos", cos), W.tensor("sin", sin), W.tensor("shq", np.array([B, S, H * D], np.int64)),
             W.tensor("shk", np.array([B, S, Hkv * D], np.int64))]
    nodes = [
        # the opset-23 form rotates [B, H, S, D] heads with RotaryEmbedding; here only K goes that way, Q rotates in GQA
        W.node("RotaryEmbedding", ["k4", "cos", "sin", "pos"], ["k4r"], interleaved=0),
        W.node("Transpose", ["k4r"], ["k4t"], perm=[0, 2, 1, 3]),
        W.node("Reshape", ["k4t", "shk"], ["k3"]),
        W.node("GroupQueryAttention", ["q", "k3", "v", "past_key", "past_value", "seqlens_k", "total", "cos", "sin", "", ""],
               ["y", "present_key", "present_value"], domain="com.microsoft", num_heads=H, kv_num_heads=Hkv, do_rotary=1,
               local_window_size=-1),
    ]
    ins = [W.value_info("q", W.FLOAT, [B, S, H * D]), W.value_info("k4", W.FLOAT, [B, Hkv, S, D]), W.value_info("v", W.FLOAT, [B, S, Hkv * D]),
           W.value_info("pos", W.INT32, [B, S]), W.value_info("past_key", W.FLOAT, [B, Hkv, P, D]),
           W.value_info("past_value", W.FLOAT, [B, Hkv, P, D]), W.value_info("seqlens_k", W.INT32, [B]), W.value_info("total", W.INT32, [])]
    outs = [W.value_info(n, W.FLOAT, []) for n in ("y", "present_key", "present_value")]
    return W.model(nodes, inits, ins, outs, opset=23, extra_opsets=[("com.microsoft", 1)]), cos, sin


@pytest.mark.gpu
def test_group_query_attention_through_the_onnx_executor(rt):
    """RotaryEmbedding (ai.onnx) on the key heads, then com.microsoft GroupQueryAttention with past / present caches and
    empty optional inputs, through Model.run against the restatements."""
    from rten_b200.model import Model
    import onnx_writer as W
    assert hasattr(W, "INT32")
    B, S, P, H, Hkv, D = 2, 1, 40, 8, 2, 64
    data, cos, sin = _gqa_graph(B, S, P, H, Hkv, D, 64, 4)
    rng = np.random.default_rng(2)
    q = rng.uniform(-1, 1, (B, S, H * D)).astype(np.float32)
    k4 = rng.uniform(-1, 1, (B, Hkv, S, D)).astype(np.float32)
    v = rng.uniform(-1, 1, (B, S, Hkv * D)).astype(np.float32)
    pk = rng.uniform(-1, 1, (B, Hkv, P, D)).astype(np.float32)
    pv = rng.uniform(-1, 1, (B, Hkv, P, D)).astype(np.float32)
    sk = np.array([40, 17], np.int32)
    pos = np.array([[33], [9]], np.int32)
    k4r = _rotary_ref_op(k4, cos, sin, pos, False, 0, 0, np.float32)
    k3 = k4r.transpose(0, 2, 1, 3).reshape(B, S, Hkv * D)
    ref = ref_gqa(q, k3, v, pk, pv, sk, P + S, H, Hkv, cos, sin, None, None, None, True, False, -1)
    ref32 = ref_gqa(q, k3, v, pk, pv, sk, P + S, H, Hkv, cos, sin, None, None, None, True, False, -1, dtype=np.float32)
    ctx = _ctx(rt)
    m = Model(ctx, data)
    feeds = {"q": q, "k4": k4, "v": v, "pos": pos, "past_key": pk, "past_value": pv, "seqlens_k": sk, "total": np.array(P + S, np.int32)}
    y, prk, prv = m.run({n: ctx.to_device(a) for n, a in feeds.items()})
    assert _rel_err(y.numpy(), ref[0]) <= 2e-5
    _bits_equal(prk.numpy(), ref32[1], "executor present_key")
    _bits_equal(prv.numpy(), ref32[2], "executor present_value")
