"""com.microsoft MultiHeadAttention: the rotary / append kernel as its prep (bias adds, present caches), the single-query
attention kernel (one query) and the streaming prefill kernel (more), both with the operator's masking: masked keys
score mask_filter_value, a finite value, and stay in the softmax.

Every GPU assertion rests on the numpy restatement `ref_mha` of MultiHeadAttention::run_impl, sdpa_head,
causal_mask_row and concat_past_kv (src/ops/attention/contrib.rs:56-300, src/ops/attention.rs:470-577).  The CPU tests
check it against a literal row-by-row transcription of those functions and against the reference's MultiHeadAttention
known answers (tests/golden/multihead_attention_cases.json).  Attention outputs: |d| <= 2e-5 * max |ref| in 3xTF32 and
for the single-query kernel, 4e-3 * max |ref| for the prefill kernel in single-pass TF32.  Present caches are the
float32 bias adds and copies, compared bit for bit."""
import json
import math
import os

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))

# ---------------------------------------------------------------------------------------------------------------------
# numpy restatements


def _heads(query, key, value, bias, H):
    """q [B, H, S, D], k [B, H, L, D], v [B, H, L, Dv] after the float32 bias adds."""
    f32 = np.float32
    if query.ndim == 5:
        return tuple(query[:, :, :, i].transpose(0, 2, 1, 3).astype(f32) for i in range(3))
    B, S, hid = query.shape
    if key is None:
        key = value = query
    if bias is not None:
        bias = np.asarray(bias, f32)
        query, key, value = (np.asarray(query, f32) + bias[:hid], np.asarray(key, f32) + bias[hid:2 * hid],
                             np.asarray(value, f32) + bias[2 * hid:])
    L = key.shape[1]
    split = lambda x, n: np.asarray(x, f32).reshape(B, n, H, -1).transpose(0, 2, 1, 3)
    return split(query, S), split(key, L), split(value, L)


def ref_mha(query, key=None, value=None, bias=None, kpm=None, attn_bias=None, past_key=None, past_value=None, H=1, scale=None,
            fill=-10000.0, unidirectional=False):
    """(output [B, S, H * Dv], present_key, present_value) of MultiHeadAttention; the caches in float32, the attention in
    float64."""
    q, k, v = _heads(query, key, value, bias, H)
    P = 0
    if past_key is not None:
        P = past_key.shape[2]
        k = np.concatenate([np.asarray(past_key, np.float32), k], axis=2)
        v = np.concatenate([np.asarray(past_value, np.float32), v], axis=2)
    B, _, S, D = q.shape
    T = k.shape[2]
    sc = np.float32(1.0) / np.sqrt(np.float32(D)) if scale is None else scale
    s = float(sc) * np.einsum("bhsd,bhtd->bhst", q.astype(np.float64), k.astype(np.float64))
    if attn_bias is not None:
        s = s + np.broadcast_to(np.asarray(attn_bias, np.float64), s.shape)
    if unidirectional:
        cols = np.arange(T)[None, :]
        masked_from = np.clip(P + np.arange(S)[:, None] + 1, 0, T)
        s = np.where(cols >= masked_from, fill, s)
    if kpm is not None:
        s = np.where((np.asarray(kpm) == 0)[:, None, None, :], fill, s)
    with np.errstate(invalid="ignore", over="ignore"):
        m = s.max(axis=-1, keepdims=True)
        e = np.exp(s - m)
        p = e / e.sum(axis=-1, keepdims=True)
    p = np.nan_to_num(p, nan=0.0)
    out = np.einsum("bhst,bhtd->bhsd", p, v.astype(np.float64))
    return out.transpose(0, 2, 1, 3).reshape(B, S, -1), k, v


def _loop_mha(query, key, value, bias, kpm, attn_bias, past_key, past_value, H, scale, fill, unidirectional):
    """Row by row as run_impl / sdpa_head / causal_mask_row / concat_past_kv do it (float64 arithmetic)."""
    f32 = np.float32
    if query.ndim == 5:
        B, S, _, _, D = query.shape
        qh = lambda b, h, s: query[b, s, h, 0]
        kn = lambda b, h, t: query[b, t, h, 1]
        vn = lambda b, h, t: query[b, t, h, 2]
        L, Dv = S, D
    else:
        B, S, hid = query.shape
        D = hid // H
        k_, v_ = (query, query) if key is None else (key, value)
        L, Dv = k_.shape[1], v_.shape[2] // H
        add = lambda x, off, n: (lambda b, h, t: np.asarray([f32(x[b, t, h * n + i]) + (f32(bias[off + h * n + i]) if bias is not None else f32(0))
                                                            for i in range(n)], f32))
        qh = add(query, 0, D)
        kn = add(k_, hid, D)
        vn = add(v_, 2 * hid, Dv)
    P = 0 if past_key is None else past_key.shape[2]
    T = P + L
    present_k = np.zeros((B, H, T, D), f32)
    present_v = np.zeros((B, H, T, Dv), f32)
    for b in range(B):
        for h in range(H):
            for t in range(T):
                present_k[b, h, t] = past_key[b, h, t] if t < P else kn(b, h, t - P)
                present_v[b, h, t] = past_value[b, h, t] if t < P else vn(b, h, t - P)
    sc = float(f32(1.0) / math.sqrt(D)) if scale is None else scale
    out = np.zeros((B, S, H * Dv))
    for b in range(B):
        for h in range(H):
            for s in range(S):
                q = np.asarray(qh(b, h, s), np.float64)
                row = [sc * float(np.dot(q, present_k[b, h, t].astype(np.float64))) for t in range(T)]
                if attn_bias is not None:
                    ab = np.broadcast_to(attn_bias, (B, H, S, T))
                    row = [x + float(ab[b, h, s, t]) for t, x in enumerate(row)]
                if unidirectional:
                    for t in range(min(max(P + s + 1, 0), T), T):
                        row[t] = fill
                if kpm is not None:
                    row = [fill if kpm[b, t] == 0 else x for t, x in enumerate(row)]
                m = max(row)
                if m == -math.inf:
                    continue  # every score -inf: NaN, flushed to zeros
                e = [math.exp(x - m) for x in row]
                tot = sum(e)
                out[b, s, h * Dv:(h + 1) * Dv] = sum(e[t] / tot * present_v[b, h, t].astype(np.float64) for t in range(T))
    return out, present_k, present_v


def _random_case(seed, B, S, L, P, H, D, mode, bias, kpm, ab, dtype_bias=np.float32):
    """Inputs of one case.  mode: 'self' (no key), 'sep' (key / value of L positions) or 'packed' ([B, S, H, 3, D]).
    kpm: None, 'interior' (zeros inside the sequence) or 'batch' (batch 0 fully padded).  ab: None or the shape kind of
    attention_bias: '11ST', 'BHST' or 'B1S1'."""
    rng = np.random.default_rng(seed)
    u = lambda *s: rng.uniform(-1, 1, s).astype(np.float32)
    hid = H * D
    if mode == "packed":
        query, key, value, L = u(B, S, H, 3, D), None, None, S
    elif mode == "self":
        query, key, value, L = u(B, S, hid), None, None, S
    else:
        query, key, value = u(B, S, hid), u(B, L, hid), u(B, L, hid)
    T = P + L
    bvec = u(3 * hid) if bias else None
    m = None
    if kpm == "interior":
        m = (rng.uniform(0, 1, (B, T)) > 0.3).astype(np.int32)
        m[:, 0] = 1
    elif kpm == "batch":
        m = np.ones((B, T), np.int32)
        m[0] = 0
    shapes = {"11ST": (1, 1, S, T), "BHST": (B, H, S, T), "B1S1": (B, 1, S, 1)}
    abias = (2 * u(*shapes[ab])) if ab else None
    pk = u(B, H, P, D) if P else None
    pv = u(B, H, P, D) if P else None
    return dict(query=query, key=key, value=value, bias=bvec, kpm=m, attn_bias=abias, past_key=pk, past_value=pv)


def test_reference_mha_matches_the_row_loop():
    cases = [
        (1, 2, 3, 3, 0, 2, 4, "self", False, None, None, False),
        (2, 2, 4, 5, 3, 2, 4, "sep", True, "interior", "11ST", True),
        (3, 1, 1, 1, 6, 3, 4, "sep", True, "batch", "BHST", True),
        (4, 2, 3, 3, 2, 2, 2, "packed", False, "interior", "B1S1", True),
        (5, 2, 5, 2, 0, 1, 4, "sep", False, None, "B1S1", True),
        (6, 1, 3, 4, 1, 2, 4, "sep", True, "batch", None, False),
    ]
    for seed, B, S, L, P, H, D, mode, bias, kpm, ab, uni in cases:
        c = _random_case(seed, B, S, L, P, H, D, mode, bias, kpm, ab)
        for fill in (-10000.0, -math.inf):
            args = (c["query"], c["key"], c["value"], c["bias"], c["kpm"], c["attn_bias"], c["past_key"], c["past_value"])
            want = _loop_mha(*args, H, None, fill, uni)
            got = ref_mha(*args, H=H, fill=fill, unidirectional=uni)
            np.testing.assert_allclose(got[0], want[0], rtol=1e-9, atol=1e-12, err_msg=f"case {seed} fill {fill}")
            assert np.array_equal(got[1], want[1]) and np.array_equal(got[2], want[2]), f"case {seed}: present caches"


def _golden_cases():
    with open(os.path.join(HERE, "golden", "multihead_attention_cases.json")) as f:
        return json.load(f)["cases"]


def _golden_inputs(case):
    def arr(name):
        t = case["inputs"].get(name)
        if t is None:
            return None
        return np.asarray(t["data"], np.int32 if t.get("dtype") == "int32" else np.float32).reshape(t["shape"])
    return dict(query=arr("query"), key=arr("key"), value=arr("value"), bias=arr("bias"), kpm=arr("key_padding_mask"),
                attn_bias=arr("attention_bias"), past_key=arr("past_key"), past_value=arr("past_value"))


@pytest.mark.parametrize("case", _golden_cases(), ids=lambda c: c["name"])
def test_restatement_reproduces_the_known_answers(case):
    a = _golden_inputs(case)
    out, pk, pv = ref_mha(**a, H=case["num_heads"], scale=case["scale"], unidirectional=case["unidirectional"])
    if case["expected"] is not None:
        exp = np.asarray(case["expected"]["data"], np.float64).reshape(case["expected"]["shape"])
        # the reference's expect_equal: |a - b| <= 1e-5 + 1e-4 |b|
        assert np.all(np.abs(out - exp) <= 1e-5 + 1e-4 * np.abs(exp)), f"{case['name']}: {out} vs {exp}"
    if case.get("in_place"):
        P = a["past_key"].shape[2]
        assert pk.shape[2] == P + a["key"].shape[1]
        assert np.array_equal(pk[:, :, :P], a["past_key"]) and np.array_equal(pv[:, :, :P], a["past_value"])


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


def _run_mha(rt, ctx, c, H, uni, present, fill=-10000.0, sentinel=7.5):
    """Run the operator on device tensors.  present: 'none' (not requested), 'new' or 'inplace' (the present caches are
    the past buffers [B, H, P + L + 3, D] holding `sentinel` beyond P).  Returns (out, present_key, present_value,
    launches, initial present buffers)."""
    dv = lambda a: None if a is None else ctx.to_device(a)
    q = c["query"]
    B = q.shape[0]
    D = q.shape[4] if q.ndim == 5 else q.shape[2] // H
    L = q.shape[1] if c["key"] is None else c["key"].shape[1]
    P = 0 if c["past_key"] is None else c["past_key"].shape[2]
    args = dict(bias=dv(c["bias"]), key_padding_mask=dv(c["kpm"]), attention_bias=dv(c["attn_bias"]), past_key=dv(c["past_key"]),
                past_value=dv(c["past_value"]))
    inits = []
    if present == "inplace":
        cap = P + L + 3
        bufs = []
        for past in (c["past_key"], c["past_value"]):
            full = np.full((B, H, cap, D), sentinel, np.float32)
            if P:
                full[:, :, :P] = past
            inits.append(full)
            bufs.append(ctx.to_device(full))
        st = (H * cap * D, cap * D, D, 1)
        args["past_key"], args["past_value"] = (b.view((B, H, P, D), st) for b in bufs)
        args["present_key"], args["present_value"] = (b.view((B, H, P + L, D), st) for b in bufs)
    op = rt.MultiHeadAttention(H, mask_filter_value=fill, unidirectional=uni)
    dq, dk, dvv = dv(q), dv(c["key"]), dv(c["value"])
    ctx.sync()
    n0 = ctx.launches
    o, k, v = op.run(ctx, dq, dk, dvv, want_present=present != "none", **args)
    n = ctx.launches - n0
    if present == "inplace":
        k, v = (b.numpy() for b in bufs)
    else:
        k, v = (None if t is None else t.numpy() for t in (k, v))
    return o.numpy(), k, v, n, inits


# (name, B, S, L, P, H, D, mode, bias, kpm, attention_bias, unidirectional, present)
GPU_CASES = [
    ("self, no mask, D64", 2, 128, 0, 0, 4, 64, "self", False, None, None, False, "none"),
    ("separate L 200 != S 96, bias, interior padding, [1,1,S,T], D128", 2, 96, 200, 0, 2, 128, "sep", True, "interior", "11ST", False, "none"),
    ("packed 5-D, batch fully padded, [B,H,S,T], unidirectional P 0", 2, 130, 0, 0, 3, 64, "packed", False, "batch", "BHST", True, "none"),
    ("separate, past 100, unidirectional, [B,1,S,1], bias, new present", 2, 64, 64, 100, 2, 64, "sep", True, None, "B1S1", True, "new"),
    ("prompt over an in-place cache, P 50, D128, bias, padding", 1, 70, 70, 50, 2, 128, "sep", True, "interior", None, True, "inplace"),
    ("cross-attention S 100 over L 700, interior padding", 1, 100, 700, 0, 2, 64, "sep", False, "interior", "11ST", False, "none"),
    ("causal tail: self 257 unidirectional, D128", 1, 257, 0, 0, 2, 128, "self", False, None, None, True, "none"),
    ("decode: in-place cache of 300, unidirectional, padding", 3, 1, 1, 300, 4, 64, "sep", False, "interior", None, True, "inplace"),
    ("decode: P 447, D128, bias, [B,H,S,T], new present", 2, 1, 1, 447, 2, 128, "sep", True, None, "BHST", True, "new"),
    ("decode: one query over 40 keys, unidirectional, batch padded", 2, 1, 40, 0, 2, 64, "sep", False, "batch", "B1S1", True, "none"),
    ("decode: self, no past, D128", 2, 1, 0, 0, 4, 128, "self", False, None, None, False, "none"),
    ("decode: packed with past 20, [1,1,S,T]", 2, 1, 0, 20, 2, 128, "packed", False, "interior", "11ST", True, "new"),
    ("one query over 8300 positions: the prefill kernel", 1, 1, 1, 8299, 1, 64, "sep", False, "interior", None, True, "new"),
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", GPU_CASES, ids=[c[0] for c in GPU_CASES])
def test_multi_head_attention_matches_the_restatement(rt, case):
    name, B, S, L, P, H, D, mode, bias, kpm, ab, uni, present = case
    c = _random_case(len(name), B, S, L or S, P, H, D, mode, bias, kpm, ab)
    ref = ref_mha(**c, H=H, unidirectional=uni)
    prefill = S > 1 or P + (L or S) > 8192
    prep = bias or P > 0 or present != "none"
    for tf32 in (False, True):
        ctx = _ctx(rt, tf32)
        out, prk, prv, n, inits = _run_mha(rt, ctx, c, H, uni, present)
        tol = 4e-3 if tf32 and prefill else 2e-5
        err = _rel_err(out, ref[0])
        assert np.isfinite(out).all() and err <= tol, f"{name} (tf32={tf32}): rel err {err:.2e} > {tol}"
        T = ref[1].shape[2]
        if present == "new":
            _bits_equal(prk, ref[1], f"{name}: present_key")
            _bits_equal(prv, ref[2], f"{name}: present_value")
        elif present == "inplace":
            for got, want, init, what in ((prk, ref[1], inits[0], "present_key"), (prv, ref[2], inits[1], "present_value")):
                _bits_equal(got[:, :, :T], want, f"{name}: {what} positions < P + L")
                _bits_equal(got[:, :, T:], init[:, :, T:], f"{name}: {what} positions beyond P + L (untouched)")
        else:
            assert prk is None and prv is None
        assert n == 1 + int(prep), f"{name}: {n} launches, expected {1 + int(prep)}"


@pytest.mark.gpu
@pytest.mark.parametrize("S", [1, 128])
def test_finite_fill_keeps_masked_keys(rt, S):
    """Rows whose visible keys are all padded, or biased to -3.4e38, are the mean of v over the masked keys -- the
    skipped causal tail included -- and mask_filter_value = -inf gives zeros instead."""
    B, H, D = 2, 2, 64
    P = 0 if S > 1 else 90
    c = _random_case(5, B, S, S, P, H, D, "sep", False, None, None)
    T = P + S
    kpm = np.ones((B, T), np.int32)
    kpm[0, :P + min(S, 64)] = 0  # batch 0: the keys rows 0-63 (and the decode row) can see are padded
    c["kpm"] = kpm
    ab = np.zeros((B, 1, S, T), np.float32)
    ab[1][:, np.tril(np.ones((S, T), bool), P)] = -3.4e38  # batch 1: every visible key biased down
    c["attn_bias"] = ab
    ctx = _ctx(rt)
    for fill in (-10000.0, -math.inf):
        ref = ref_mha(**c, H=H, unidirectional=True, fill=fill)
        out = _run_mha(rt, ctx, c, H, True, "none", fill=fill)[0]
        if fill == -10000.0:
            # batch 0, first row: uniform weights over every key (v of the whole cache, [H, T, D])
            v = ref[2].astype(np.float64)
            assert np.abs(ref[0][0, 0] - v[0].mean(axis=1).reshape(-1)).max() < 1e-6
            # batch 1, row 0 (S > 1): the mean over the masked (future) keys
            if S > 1:
                assert np.abs(ref[0][1, 0] - v[1][:, 1:].mean(axis=1).reshape(-1)).max() < 1e-6
        else:
            assert not ref[0][0, 0].any()
        err = _rel_err(out, ref[0])
        assert np.isfinite(out).all() and err <= 2e-5, f"S {S} fill {fill}: rel err {err:.2e}"
        if fill == -math.inf:
            assert not out[0, 0].any(), "a fully masked row with fill -inf is zeros"


@pytest.mark.gpu
def test_multi_head_attention_rejects_a_present_cache_overlapping_the_past(rt):
    B, H, D, P = 2, 2, 64, 10
    ctx = _ctx(rt)
    buf = ctx.empty((B * H * (P + 1) * D,))
    past = buf.view((B, H, P, D), (H * P * D, P * D, D, 1))
    pres = buf.view((B, H, P + 1, D), (H * (P + 1) * D, (P + 1) * D, D, 1))
    other = ctx.empty((B, H, P + 1, D))
    q = ctx.empty((B, 1, H * D))
    with pytest.raises(rt.OpError) as e:
        rt.MultiHeadAttention(H).run(ctx, q, q, q, past_key=past, past_value=past, present_key=pres, present_value=other)
    assert e.value.kind == "UnsupportedOutput" and "overlap a past cache" in e.value.msg


@pytest.mark.gpu
def test_multi_head_attention_decode_graph_replay(rt):
    """A decode step over in-place caches with a device-resident key_padding_mask, captured in a CUDA graph and replayed
    while the inputs and the mask change on the device, gives the bytes of eager calls on identical caches."""
    import gpu_checks as gc
    B, H, D, P = 3, 12, 64, 200
    cap = P + 1
    rng = np.random.default_rng(4)
    ctx = _ctx(rt)
    init = rng.uniform(-1, 1, (2, B, H, cap, D)).astype(np.float32)
    caches = [(ctx.to_device(init[0]), ctx.to_device(init[1])) for _ in range(2)]  # graph, eager
    st = (H * cap * D, cap * D, D, 1)
    op = rt.MultiHeadAttention(H, unidirectional=True)
    dq, dk, dv = (ctx.empty((B, 1, H * D)) for _ in range(3))
    dbias = ctx.to_device(rng.uniform(-1, 1, 3 * H * D).astype(np.float32))
    dkpm = ctx.to_device(np.ones((B, cap), np.int32))
    out_g = ctx.empty((B, 1, H * D))

    def step(kc, vc, out=None):
        return op.run(ctx, dq, dk, dv, bias=dbias, key_padding_mask=dkpm, past_key=kc.view((B, H, P, D), st),
                      past_value=vc.view((B, H, P, D), st), present_key=kc, present_value=vc, out=out)

    warm = [ctx.to_device(init[i]) for i in range(2)]  # one eager step first: nothing is allocated while capturing
    step(*warm)
    ctx.sync()
    ctx.graph_begin()
    step(caches[0][0], caches[0][1], out_g)
    graph = ctx.graph_end()
    for i in range(3):
        for t in (dq, dk, dv):
            t.copy_from(rng.uniform(-1, 1, (B, 1, H * D)).astype(np.float32))
        dkpm.copy_from((rng.uniform(0, 1, (B, cap)) > 0.2 * i).astype(np.int32))
        n0 = ctx.launches
        graph.launch()
        assert ctx.launches - n0 == 2, "a replayed decode step with a bias is two kernel launches"
        ctx.sync()
        g = out_g.numpy()
        e = step(*caches[1])[0].numpy()
        gc.assert_bit_exact(g, e, f"graph replay step {i}: output")
        gc.assert_bit_exact(caches[0][0].numpy(), caches[1][0].numpy(), f"graph replay step {i}: key cache")
        gc.assert_bit_exact(caches[0][1].numpy(), caches[1][1].numpy(), f"graph replay step {i}: value cache")


@pytest.mark.gpu
def test_multi_head_attention_errors(rt):
    ctx = _ctx(rt)
    B, S, H, D, P = 2, 3, 2, 64, 4
    z = lambda *s: np.zeros(s, np.float32)
    base = dict(query=z(B, S, H * D), key=z(B, 5, H * D), value=z(B, 5, H * D), past_key=z(B, H, P, D), past_value=z(B, H, P, D))

    def check(kind, msg, heads=H, **over):
        a = dict(base, **over)
        with pytest.raises(rt.OpError) as e:
            rt.MultiHeadAttention(heads).run(ctx, a.pop("query"), **a)
        assert (e.value.kind, e.value.msg) == (kind, msg)

    check("CastFailed", "conversion error for input 6: expected tensor with 4 dims but has 3 dims", past_key=z(B, P, D))
    check("CastFailed", "conversion error for input 7: expected tensor with 4 dims but has 3 dims", past_value=z(B, P, D))
    check("InvalidValue", "query must have 3 or 5 dims", query=z(B, S, H, D))
    check("CastFailed", "conversion error for input 1: expected tensor with 3 dims but has 4 dims", key=z(B, 5, H, D))
    check("CastFailed", "conversion error for input 3: expected tensor with 1 dims but has 2 dims", bias=z(1, 3 * H * D))
    check("CastFailed", "conversion error for input 4: expected tensor with 2 dims but has 1 dims", key_padding_mask=np.ones(9, np.int32))
    check("CastFailed", "conversion error for input 5: expected tensor with 4 dims but has 3 dims", attention_bias=z(1, S, 9))
    check("UnsupportedValue", "past_seq_len is not supported", past_sequence_length=np.array(4, np.int32))
    check("CastFailed", "conversion error for input 8: expected tensor with 0 dims but has 1 dims", past_sequence_length=np.array([4], np.int32))
    check("UnsupportedValue", "cache_indirection is not supported", cache_indirection=np.zeros((B, 1, 9), np.int32))
    check("InvalidValue", "num_heads must be positive", heads=0)
    packed = z(B, S, H, 3, D)
    check("InvalidValue", "key must be None when query is packed", query=packed, past_key=None, past_value=None)
    check("InvalidValue", "value must be None when query is packed", query=packed, key=None, past_key=None, past_value=None)
    check("InvalidValue", "bias is not supported with packed QKV format", query=packed, key=None, value=None, bias=z(3 * H * D))
    check("InvalidValue", "4th dimension of packed qkv input must be 3", query=z(B, S, H, 2, D), key=None, value=None)
    check("InvalidValue", "2nd dimension of packed qkv input must be equal to number of attention heads", query=z(B, S, H + 1, 3, D),
          key=None, value=None)
    check("IncompatibleInputShapes", "Hidden size must be divisible by number of attention heads", query=z(B, S, H * D + 1))
    check("InvalidValue", "value input must be set if key input is present", value=None)
    check("IncompatibleInputShapes", "Key and value batch or sequence lengths do not match", value=z(B, 4, H * D))
    check("IncompatibleInputShapes", "Key and value batch or sequence lengths do not match", key=z(1, 5, H * D))
    check("IncompatibleInputShapes", "Key hidden size does not match query hidden size", key=z(B, 5, H * D + 2))
    check("IncompatibleInputShapes", "Value hidden size must be divisible by number of attention heads", value=z(B, 5, H * D + 1))
    check("IncompatibleInputShapes", "Bias shape does not match QKV hidden sizes", bias=z(3 * H * D + 1))
    check("IncompatibleInputShapes", "past_key/past_value shape does not match key/value shape", past_value=z(B, H, P + 1, D))
    check("InvalidValue", "past_key and past_value must either both be present or both be absent", past_value=None)
    check("IncompatibleInputShapes", "Cannot broadcast inputs", attention_bias=z(1, 1, S, 5))
    check("IncompatibleInputShapes", "key_padding_mask shape does not match key sequence length", key_padding_mask=np.ones((B, 5), np.int32))
    check("UnsupportedValue", "MultiHeadAttention: the head size must be 64 or 128", query=z(B, S, H * 80), key=z(B, 5, H * 80),
          value=z(B, 5, H * 80), past_key=None, past_value=None)
    check("UnsupportedValue", "MultiHeadAttention: the value head size must equal the head size", value=z(B, 5, H * 128),
          past_key=None, past_value=None)


def _mha_graph(B, S, L, P, H, D, bias, extra_attrs=None, extra_inputs=(), extra_outputs=()):
    import onnx_writer as W
    attrs = dict(num_heads=H, unidirectional=1)
    attrs.update(extra_attrs or {})
    if attrs.get("num_heads") is None:
        del attrs["num_heads"]
    nodes = [W.node("MultiHeadAttention", ["q", "k", "v", "bias", "kpm", "", "past_key", "past_value", *extra_inputs],
                    ["y", "present_key", "present_value", *extra_outputs], domain="com.microsoft", **attrs)]
    ins = [W.value_info("q", W.FLOAT, [B, S, H * D]), W.value_info("k", W.FLOAT, [B, L, H * D]), W.value_info("v", W.FLOAT, [B, L, H * D]),
           W.value_info("kpm", W.INT32, [B, P + L]), W.value_info("past_key", W.FLOAT, [B, H, P, D]),
           W.value_info("past_value", W.FLOAT, [B, H, P, D])]
    outs = [W.value_info(n, W.FLOAT, []) for n in ("y", "present_key", "present_value")]
    return W.model(nodes, [W.tensor("bias", bias)], ins, outs, opset=17, extra_opsets=[("com.microsoft", 1)])


@pytest.mark.gpu
def test_multi_head_attention_through_the_onnx_executor(rt):
    """A com.microsoft MultiHeadAttention node with a constant bias, a padding mask, past caches and an empty optional
    input, through Model.run against the direct call; unsupported attributes, inputs and outputs fail at load."""
    from rten_b200.model import Model
    B, S, L, P, H, D = 2, 1, 1, 30, 4, 64
    c = _random_case(8, B, S, L, P, H, D, "sep", True, "interior", None)
    ctx = _ctx(rt)
    m = Model(ctx, _mha_graph(B, S, L, P, H, D, c["bias"]))
    feeds = {"q": c["query"], "k": c["key"], "v": c["value"], "kpm": c["kpm"], "past_key": c["past_key"], "past_value": c["past_value"]}
    y, prk, prv = m.run({n: ctx.to_device(a) for n, a in feeds.items()})
    d = lambda a: ctx.to_device(a)
    o2, k2, v2 = rt.MultiHeadAttention(H, unidirectional=True).run(ctx, d(c["query"]), d(c["key"]), d(c["value"]), bias=d(c["bias"]),
                                                                   key_padding_mask=d(c["kpm"]), past_key=d(c["past_key"]),
                                                                   past_value=d(c["past_value"]))
    _bits_equal(y.numpy(), o2.numpy(), "executor output")
    _bits_equal(prk.numpy(), k2.numpy(), "executor present_key")
    _bits_equal(prv.numpy(), v2.numpy(), "executor present_value")
    ref = ref_mha(**c, H=H, unidirectional=True)
    assert _rel_err(y.numpy(), ref[0]) <= 2e-5
    for kw, msg in ((dict(extra_attrs=dict(num_heads=None)), "missing attribute num_heads"),
                    (dict(extra_attrs=dict(scale=0.0)), "an explicit scale must be positive"),
                    (dict(extra_inputs=("q",)), "inputs 8, 9"),
                    (dict(extra_inputs=("", "kpm")), "inputs 8, 9"),
                    (dict(extra_outputs=("qk",)), "the qk output")):
        with pytest.raises(rt.OpError) as e:
            Model(ctx, _mha_graph(B, S, L, P, H, D, c["bias"], **kw))
        assert e.value.kind == "UnsupportedValue" and msg in e.value.msg, e.value.msg


def _kernel_probe():
    """Run in a child process: the kernels of a prompt without prep, a prompt with a bias, a decode step with a present
    cache and a one-query call over more positions than the single-query kernel takes, one CUPTI session each."""
    import gpu_checks as gc
    import rten_b200 as rt
    ctx = _ctx(rt)
    res = {}
    for name, (B, S, L, P, H, D, mode, bias, present) in {
            "prompt": (2, 64, 64, 0, 2, 64, "self", False, "none"),
            "prompt_bias": (2, 64, 80, 0, 2, 128, "sep", True, "none"),
            "decode": (2, 1, 1, 40, 2, 64, "sep", False, "new"),
            "long_decode": (1, 1, 1, 8299, 1, 64, "sep", False, "none")}.items():
        c = _random_case(1, B, S, L, P, H, D, mode, bias, None, None)
        _, names = gc._kernels_launched(lambda: _run_mha(rt, ctx, c, H, False, present))
        res[name] = sorted(names)
    print(json.dumps(res))


@pytest.mark.gpu
def test_multi_head_attention_kernel_identity():
    """Prompts run attn_prefill_mha_kernel (after rotary_mha_kernel when there is a bias), a decode step runs
    attn_decode_mha_kernel after rotary_mha_kernel, and a one-query call over 8300 positions the prefill kernel.  The
    CUPTI sessions run in a child process, so that they leave no profiler state behind in the test session."""
    import subprocess
    import sys
    code = (f"import sys; sys.path[:0] = [{os.path.dirname(HERE)!r}, {HERE!r}]; "
            "import test_gpu_multi_head_attention as t; t._kernel_probe()")
    res = subprocess.run([sys.executable, "-s", "-c", code], capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-4000:]
    names = json.loads(res.stdout.strip().splitlines()[-1])
    has = lambda key, k: any(k in n for n in names[key])
    assert has("prompt", "attn_prefill_mha_kernel") and not has("prompt", "rotary"), names["prompt"]
    assert has("prompt_bias", "attn_prefill_mha_kernel") and has("prompt_bias", "rotary_mha_kernel"), names["prompt_bias"]
    assert has("decode", "attn_decode_mha_kernel") and has("decode", "rotary_mha_kernel"), names["decode"]
    assert has("long_decode", "attn_prefill_mha_kernel") and not has("long_decode", "attn_decode"), names["long_decode"]
    for key in names:
        assert not has(key, "attn_prefill_kernel<") and not has(key, "attn_decode_kernel<"), names[key]
