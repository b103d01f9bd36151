"""`pytest -m gpu`: KV caches extended in place through the executor (rten_b200_model_run_ex, Model.run with
KvCacheHandles) and generation over a loaded model (Generator(ModelDecoder(...))).

  * the genai decoder (tests/genai_decoder.py) generates 10 tokens through Generator(ModelDecoder) with a capacity that
    fits and with capacity 1, which doubles several times: logits and every present cache bit-identical to the same file
    run step by step with plain rten_b200_model_run (new present caches every step);
  * while capacity lasts every present.N.* is the donated buffer (same data pointer), a decode step launches one kernel
    fewer per GroupQueryAttention node than the copying run (no past-prefix copy), and positions beyond the valid length
    keep a sentinel;
  * the reference's fallbacks give the copying path with identical bits: a past that is also a requested output, a past
    with a later second consumer, a capacity too small, a non-writable past;
  * a Whisper-style decoder self-attention (MultiHeadAttention with bias, unidirectional, past / present) in place over
    several steps: identical bits, the same buffer, no more launches than the copying run;
  * errors: writable inputs with strides that do not fit the capacity, a capacity below the shape, a host tensor;
  * a genai decode step with every input on the device captures into a CUDA graph and replays to the eager bits: no host
    synchronisation anywhere in the step (GroupQueryAttention reads total_sequence_length from the host value the
    Shape -> Gather -> Cast chain computes; a device-resident one is a blocking copy, which capture refuses)."""
import ctypes as C

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


@pytest.fixture(scope="module")
def genai(ctx):
    from rten_b200.model import Model
    w = gd.genai_weights()
    return w, Model(ctx, gd.genai_graph(w))


def _valid(h):
    """the valid prefix of a KvCacheHandle, as numpy"""
    t = h.tensor
    return t.view(t.shape[:2] + (h.seq_len,) + t.shape[3:], t.strides).numpy()


def _plain_step(m, ids, T, past, names):
    feeds = {"input_ids": ids, "attention_mask": np.ones((ids.shape[0], T), I32)}
    feeds.update(past)
    return [t.numpy() for t in m.run(feeds, names)]


@pytest.mark.parametrize("capacity", [64, 1])
def test_generator_over_model_decoder(rt, ctx, genai, capacity):
    from rten_b200.generate import Generator, ModelDecoder
    from test_gpu_norms import DEC as c
    _, m = genai
    B, S, steps = 2, 3, 10
    names = gd.output_names()
    prompt = np.random.default_rng(41).integers(0, c["V"], (B, S)).astype(I32)
    gen = Generator(ModelDecoder(m, B, capacity)).with_prompt(prompt)
    past = {f"past_key_values.{l}.{kv}": np.zeros((B, c["Hkv"], 0, c["D"]), F32) for l in range(c["L"]) for kv in ("key", "value")}
    ids, T, caps = prompt, 0, set()
    for step in range(steps):
        tok = next(gen)
        T += ids.shape[1]
        got = _plain_step(m, ids, T, past, names)
        gc.assert_bit_exact(gen.last_logits, got[0][:, -1], f"capacity {capacity} step {step} logits")
        for i, n in enumerate(names[1:]):
            h = gen.kv_cache[n.replace("present.", "past_key_values.")]
            assert h.seq_len == T and h.capacity >= T + 1
            caps.add(h.capacity)
            gc.assert_bit_exact(_valid(h), got[1 + i], f"capacity {capacity} step {step} {n}")
            past[n.replace("present.", "past_key_values.")] = got[1 + i]
        assert np.array_equal(tok, got[0][:, -1].argmax(-1))
        ids = tok[:, None]
    if capacity == 1:
        assert caps == {6, 12, 24}, caps  # the prompt's new cache (3 positions) doubled, then doubled twice more
    else:
        assert caps == {64}


def _handles(ctx, past, capacity, sentinel=7.0):
    """KvCacheHandles over buffers of `capacity` positions: the valid prefix `past`, then the sentinel"""
    from rten_b200.generate import KvCacheHandle
    out = {}
    for n, p in past.items():
        buf = np.full(p.shape[:2] + (capacity,) + p.shape[3:], sentinel, F32)
        buf[:, :, :p.shape[2]] = p
        out[n] = KvCacheHandle(ctx.to_device(buf), p.shape[2], capacity)
    return out


def test_decode_step_in_place(rt, ctx, genai):
    from rten_b200.generate import KvCacheHandle
    from test_gpu_norms import DEC as c
    _, m = genai
    B, S = 2, 9
    names = gd.output_names()
    r = np.random.default_rng(42)
    empty = {f"past_key_values.{l}.{kv}": np.zeros((B, c["Hkv"], 0, c["D"]), F32) for l in range(c["L"]) for kv in ("key", "value")}
    got = _plain_step(m, r.integers(0, c["V"], (B, S)).astype(I32), S, empty, names)
    past = {n.replace("present.", "past_key_values."): g for n, g in zip(names[1:], got[1:])}
    cap = 16
    for step in range(3):
        ids = r.integers(0, c["V"], (B, 1)).astype(I32)
        P = S + step
        hs = _handles(ctx, past, cap)
        ptrs = {n: h.tensor.ptr for n, h in hs.items()}
        feeds = {"input_ids": ids, "attention_mask": np.ones((B, P + 1), I32)}
        feeds.update(hs)
        dev_past = {n: ctx.to_device(p) for n, p in past.items()}
        ctx.sync()
        n0 = ctx.launches
        out = m.run(feeds, names)
        ctx.sync()
        n_inplace = ctx.launches - n0
        plain_feeds = dict(feeds, **dev_past)
        n0 = ctx.launches
        ref = [t.numpy() for t in m.run(plain_feeds, names)]
        ctx.sync()
        n_copy = ctx.launches - n0
        assert n_inplace == n_copy - c["L"], (n_inplace, n_copy)  # one past-prefix copy fewer per GroupQueryAttention
        gc.assert_bit_exact(out[0].numpy(), ref[0], f"step {step} logits")
        for i, n in enumerate(names[1:]):
            pn = n.replace("present.", "past_key_values.")
            h = out[1 + i]
            assert isinstance(h, KvCacheHandle) and h.tensor.ptr == ptrs[pn] and h.seq_len == P + 1 and h.capacity == cap
            gc.assert_bit_exact(_valid(h), ref[1 + i], f"step {step} {n}")
            full = h.tensor.numpy()
            assert (full[:, :, P + 1:] == 7.0).all(), f"step {step} {n}: positions beyond the valid length were written"
            past[pn] = ref[1 + i]


def _gqa_graph(extra_consumer=False):
    import onnx_writer as W
    H, Hkv, D = 4, 2, 64
    nodes = [W.node("GroupQueryAttention", ["q", "k", "v", "past_key", "past_value", "seqlens_k", "total"], ["y", "present_key", "present_value"],
                    domain="com.microsoft", num_heads=H, kv_num_heads=Hkv)]
    outs = ["y", "present_key", "present_value"]
    if extra_consumer:  # a second consumer of the past that runs after the attention node
        nodes.append(W.node("Identity", ["past_key"], ["past_key_again"]))
        outs.append("past_key_again")
    ins = [W.value_info(n, W.FLOAT, ["b", 1, d]) for n, d in (("q", H * D), ("k", Hkv * D), ("v", Hkv * D))]
    ins += [W.value_info(n, W.FLOAT, ["b", Hkv, "p", D]) for n in ("past_key", "past_value")]
    ins += [W.value_info("seqlens_k", W.INT32, ["b"]), W.value_info("total", W.INT32, [])]
    return W.model(nodes, [], ins, [W.value_info(o, W.FLOAT, []) for o in outs], opset=21, extra_opsets=[("com.microsoft", 1)]), outs


def test_fallbacks_give_the_copying_path(rt, ctx):
    from rten_b200.generate import KvCacheHandle
    from rten_b200.model import Model
    B, H, Hkv, D, P = 2, 4, 2, 64, 20
    r = np.random.default_rng(43)
    x = {"q": r.standard_normal((B, 1, H * D)).astype(F32), "k": r.standard_normal((B, 1, Hkv * D)).astype(F32),
         "v": r.standard_normal((B, 1, Hkv * D)).astype(F32), "seqlens_k": np.full(B, P, I32), "total": np.array(P + 1, I32)}
    past = {n: r.standard_normal((B, Hkv, P, D)).astype(F32) for n in ("past_key", "past_value")}
    for case in ("requested", "second consumer", "too small", "not writable", "in place"):
        data, outs = _gqa_graph(case == "second consumer")
        m = Model(ctx, data)
        if case == "requested":
            outs = outs + ["past_key"]
        ref = [t.numpy() for t in m.run(dict(x, **past), outs)]
        hs = _handles(ctx, past, P if case == "too small" else 32)
        feeds = dict(x, **({n: ctx.to_device(p) for n, p in past.items()} if case == "not writable" else hs))
        got = m.run(feeds, outs)
        for i, o in enumerate(outs):
            g = _valid(got[i]) if isinstance(got[i], KvCacheHandle) else got[i].numpy()
            gc.assert_bit_exact(g, ref[i], f"{case}: {o}")
        key_in_place = isinstance(got[1], KvCacheHandle)
        assert key_in_place == (case == "in place"), case
        assert isinstance(got[2], KvCacheHandle) == (case in ("in place", "requested", "second consumer")), case
        if key_in_place:
            assert got[1].tensor.ptr == hs["past_key"].tensor.ptr


def test_multi_head_attention_decoder_in_place(rt, ctx):
    """Whisper's decoder self-attention: MultiHeadAttention with the QKV bias, unidirectional, past / present caches"""
    import onnx_writer as W
    from rten_b200.generate import KvCacheHandle
    from rten_b200.model import Model
    B, H, D, P0, steps, cap = 2, 6, 64, 5, 4, 16
    r = np.random.default_rng(44)
    bias = (0.1 * r.standard_normal(3 * H * D)).astype(F32)
    nodes = [W.node("MultiHeadAttention", ["q", "k", "v", "bias", "", "", "past_key", "past_value"], ["y", "present_key", "present_value"],
                    domain="com.microsoft", num_heads=H, unidirectional=1)]
    ins = [W.value_info(n, W.FLOAT, ["b", 1, H * D]) for n in ("q", "k", "v")]
    ins += [W.value_info(n, W.FLOAT, ["b", H, "p", D]) for n in ("past_key", "past_value")]
    outs = ["y", "present_key", "present_value"]
    m = Model(ctx, W.model(nodes, [W.tensor("bias", bias)], ins, [W.value_info(o, W.FLOAT, []) for o in outs], opset=21,
                           extra_opsets=[("com.microsoft", 1)]))
    past = {n: r.standard_normal((B, H, P0, D)).astype(F32) for n in ("past_key", "past_value")}
    hs = _handles(ctx, past, cap)
    ptrs = {n: h.tensor.ptr for n, h in hs.items()}
    for step in range(steps):
        x = {n: r.standard_normal((B, 1, H * D)).astype(F32) for n in ("q", "k", "v")}
        dev = {n: ctx.to_device(a) for n, a in x.items()}
        ctx.sync()
        n0 = ctx.launches
        got = m.run(dict(dev, **hs), outs)
        ctx.sync()
        n_inplace = ctx.launches - n0
        n0 = ctx.launches
        ref = [t.numpy() for t in m.run(dict(dev, **{n: ctx.to_device(p) for n, p in past.items()}), outs)]
        ctx.sync()
        assert n_inplace <= ctx.launches - n0
        gc.assert_bit_exact(got[0].numpy(), ref[0], f"MHA step {step} y")
        for i, n in ((1, "past_key"), (2, "past_value")):
            assert isinstance(got[i], KvCacheHandle) and got[i].tensor.ptr == ptrs[n] and got[i].seq_len == P0 + step + 1
            gc.assert_bit_exact(_valid(got[i]), ref[i], f"MHA step {step} present {n}")
            assert (got[i].tensor.numpy()[:, :, P0 + step + 1:] == 7.0).all()
            past[n] = ref[i]
        hs = {"past_key": got[1], "past_value": got[2]}


def test_writable_input_errors(rt, ctx):
    from rten_b200 import _lib
    from rten_b200.generate import KvCacheHandle
    from rten_b200.model import Model
    from rten_b200.ops import _desc
    data, outs = _gqa_graph()
    m = Model(ctx, data)
    B, Hkv, D, P = 2, 2, 64, 4
    buf = ctx.to_device(np.zeros((B, Hkv, 8, D), F32))
    x = {"q": np.zeros((B, 1, 4 * D), F32), "k": np.zeros((B, 1, Hkv * D), F32), "v": np.zeros((B, 1, Hkv * D), F32),
         "seqlens_k": np.full(B, P, I32), "total": np.array(P + 1, I32), "past_value": np.zeros((B, Hkv, P, D), F32)}
    for what, h in (("capacity beyond the buffer's strides", KvCacheHandle(buf, P, 16)),
                    ("capacity below the shape", KvCacheHandle(buf, 8, 6))):
        with pytest.raises(rt.OpError) as ei:
            m.run(dict(x, past_key=h), outs)
        assert ei.value.kind == "InvalidValue" and "writable input 'past_key'" in ei.value.msg, what
    # a writable host tensor, through the C ABI directly
    host = np.zeros((B, Hkv, P, D), F32)
    d = _desc(host.ctypes.data, host.dtype, host.shape, [s // 4 for s in host.strides], -1)
    opts = (_lib.RtenModelInputOpts * 1)()
    opts[0].writable, opts[0].grow_axis, opts[0].capacity = 1, 2, P
    out_t = (_lib.RtenTensor * 1)()
    st = ctx.lib.rten_b200_model_run_ex(m.handle, 1, (C.c_char_p * 1)(b"past_key"), C.byref(d), C.cast(opts, C.c_void_p), 1,
                                        (C.c_char_p * 1)(b"y"), out_t, None)
    assert st == 5 and b"must be device-resident" in ctx.lib.rten_b200_last_error(ctx.handle)


def test_genai_decode_step_captures_without_host_sync(rt, ctx, genai):
    from test_gpu_norms import DEC as c
    _, m = genai
    B, P = 2, 6
    names = gd.output_names()
    r = np.random.default_rng(45)
    feeds = {"input_ids": ctx.to_device(r.integers(0, c["V"], (B, 1)).astype(I32)),
             "attention_mask": ctx.to_device(np.ones((B, P + 1), I32))}
    for l in range(c["L"]):
        for kv in ("key", "value"):
            feeds[f"past_key_values.{l}.{kv}"] = ctx.to_device(r.standard_normal((B, c["Hkv"], P, c["D"])).astype(F32))
    eager = [t.numpy() for t in m.run(feeds, names)]
    ctx.sync()
    ctx.graph_begin()
    try:
        captured = m.run(feeds, names)
    finally:
        g = ctx.graph_end()
    g.launch()
    ctx.sync()
    for i, n in enumerate(names):
        gc.assert_bit_exact(captured[i].numpy(), eager[i], f"graph replay {n}")
