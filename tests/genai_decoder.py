"""Test infrastructure for onnxruntime-genai int4 decoders and ReduceSum.

  * `genai_graph`: an int4 decoder as onnxruntime-genai exports it -- genai's value names (`input_ids` and
    `attention_mask` int64, `past_key_values.N.key|value`, `present.N.key|value`, `logits`), symbolic batch / sequence
    dims so one file serves the prompt and every decode step, and the attention-mask subgraph that computes
    GroupQueryAttention's seqlens_k and total_sequence_length:
        attention_mask - ReduceSum(axes [1], keepdims 1) - Sub(1) - Cast(int32)   -> seqlens_k [B, 1]
                       - Shape - Gather(index 1, axis 0) - Cast(int32)          -> total_sequence_length []
    Layers listed in `packed` run one MatMulNBits over the concatenated Q / K / V weights and a GroupQueryAttention with
    empty key / value inputs; the others project Q, K and V separately.  The weights and the layer body are those of
    test_gpu_norms's two-layer decoder.
  * `genai_ops`: the same forward, one ops.py call per node.
  * `sum_ref` / `reduce_sum_ref`: the reference's ReduceSum restated -- every output is vecmath::Sum (the C oracle's
    rto_sum: 4 x 16 chains over 64-element chunks, then 16-element chunks and the masked tail into chain set 0, lanes
    summed in order) of the reduced elements in row-major order of the reduced axes."""
import numpy as np

F32 = np.float32


def sum_ref(v):
    """rto_sum restated in numpy float32 arithmetic (each addition rounded, in the oracle's order)"""
    v = np.asarray(v, F32).reshape(-1)
    n = v.size
    acc = np.zeros((4, 16), F32)
    i = 0
    with np.errstate(over="ignore", invalid="ignore"):
        while i + 64 <= n:
            acc = acc + v[i:i + 64].reshape(4, 16)
            i += 64
        a0 = ((acc[0] + acc[1]) + acc[2]) + acc[3]
        while i + 16 <= n:
            a0 = a0 + v[i:i + 16]
            i += 16
        a0[:n - i] = a0[:n - i] + v[i:]
        s = F32(0)
        for x in a0:
            s = F32(s + x)
    return s


def resolve_axes(ndim, axes):
    if not axes:
        return list(range(ndim))
    out = []
    for a in axes:
        r = a + ndim if a < 0 else a
        if not 0 <= r < ndim:
            raise ValueError("Axis is invalid")
        out.append(r)
    return sorted(set(out))


def reduce_sum_ref(x, axes=None, keepdims=True, lane_sum=sum_ref):
    """ReduceSum of f32 `x`: the kept axes in order, then the reduced ones in ascending order; each lane summed by
    `lane_sum` (sum_ref, or the oracle's rto_sum)"""
    x = np.asarray(x)
    if x.ndim == 0:
        return np.asarray(lane_sum(x.reshape(1)), F32)
    red = resolve_axes(x.ndim, axes)
    kept = [d for d in range(x.ndim) if d not in red]
    p = np.transpose(x, kept + red)
    ks = [x.shape[d] for d in kept]
    L = int(np.prod([x.shape[d] for d in red], dtype=np.int64))
    lanes = np.ascontiguousarray(p).reshape(int(np.prod(ks, dtype=np.int64)), L)
    y = np.array([lane_sum(l) for l in lanes], F32).reshape(ks)
    if keepdims:
        y = y.reshape([1 if d in red else x.shape[d] for d in range(x.ndim)])
    return y


def genai_weights(packed=(0,)):
    from test_gpu_norms import _decoder_weights
    w = _decoder_weights()
    for l in packed:
        w[f"b_qkv{l}"] = np.concatenate([w[f"b_q{l}"], w[f"b_k{l}"], w[f"b_v{l}"]], 0)
        w[f"s_qkv{l}"] = np.concatenate([w[f"s_q{l}"], w[f"s_k{l}"], w[f"s_v{l}"]], 0)
        for nm in "qkv":
            del w[f"b_{nm}{l}"], w[f"s_{nm}{l}"]
    return w


def genai_graph(w, packed=(0,), cfg=None):
    """`cfg`: the decoder's sizes (test_gpu_norms.DEC's keys), DEC by default"""
    import onnx_writer as W
    from test_gpu_norms import DEC
    c = cfg or DEC
    hid, kvd, L = c["Hq"] * c["D"], c["Hkv"] * c["D"], c["L"]
    ms = dict(domain="com.microsoft")

    def mm(x, nm, out, K, N):
        return W.node("MatMulNBits", [x, "b_" + nm, "s_" + nm], [out], K=K, N=N, bits=4, block_size=c["block"], accuracy_level=4, **ms)

    consts = {"/model/axes_1": np.array([1], np.int64), "/model/one": np.array(1, np.int64), "/model/index_1": np.array(1, np.int64)}
    nodes = [W.node("ReduceSum", ["attention_mask", "/model/axes_1"], ["/model/mask_sum"], keepdims=1),
             W.node("Sub", ["/model/mask_sum", "/model/one"], ["/model/mask_sub"]),
             W.node("Cast", ["/model/mask_sub"], ["seqlens_k"], to=W.INT32),
             W.node("Shape", ["attention_mask"], ["/model/mask_shape"]),
             W.node("Gather", ["/model/mask_shape", "/model/index_1"], ["/model/mask_len"], axis=0),
             W.node("Cast", ["/model/mask_len"], ["total_seq_len"], to=W.INT32),
             W.node("Gather", ["embed", "input_ids"], ["x0"]),
             W.node("SimplifiedLayerNormalization", ["x0", "g_in0"], ["h0"], axis=-1, epsilon=c["eps"])]
    res, h = "x0", "h0"
    for l in range(L):
        past = [f"past_key_values.{l}.key", f"past_key_values.{l}.value", "seqlens_k", "total_seq_len", "cos", "sin"]
        if l in packed:
            nodes += [mm(h, f"qkv{l}", f"qkv{l}", hid, hid + 2 * kvd)]
            qkv = [f"qkv{l}", "", ""]
        else:
            nodes += [mm(h, f"q{l}", f"q{l}", hid, hid), mm(h, f"k{l}", f"k{l}", hid, kvd), mm(h, f"v{l}", f"v{l}", hid, kvd)]
            qkv = [f"q{l}", f"k{l}", f"v{l}"]
        nodes += [W.node("GroupQueryAttention", qkv + past, [f"a{l}", f"present.{l}.key", f"present.{l}.value"], num_heads=c["Hq"],
                         kv_num_heads=c["Hkv"], do_rotary=1, local_window_size=-1, **ms),
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
    ins = [W.value_info("input_ids", W.INT64, ["batch_size", "sequence_length"]),
           W.value_info("attention_mask", W.INT64, ["batch_size", "total_sequence_length"])]
    outs = [W.value_info("logits", W.FLOAT, ["batch_size", "sequence_length", c["V"]])]
    for l in range(L):
        for kv in ("key", "value"):
            ins.append(W.value_info(f"past_key_values.{l}.{kv}", W.FLOAT, ["batch_size", c["Hkv"], "past_sequence_length", c["D"]]))
            outs.append(W.value_info(f"present.{l}.{kv}", W.FLOAT, ["batch_size", c["Hkv"], "total_sequence_length", c["D"]]))
    inits = [W.tensor(k, v) for k, v in {**w, **consts}.items()]
    return W.model(nodes, inits, ins, outs, opset=21, extra_opsets=[("com.microsoft", 1)])


def output_names(cfg=None):
    from test_gpu_norms import DEC
    c = cfg or DEC
    return ["logits"] + [f"present.{l}.{kv}" for l in range(c["L"]) for kv in ("key", "value")]


def genai_ops(rt, ctx, w, ids, past, seqlens_k, total, packed=(0,)):
    """genai_graph's forward, one ops.py call per node (Mul(x, Sigmoid(x)) as the Silu the executor fuses it into)"""
    from test_gpu_norms import DEC as c
    d = {k: ctx.to_device(v) for k, v in w.items()}
    nb = rt.MatMulNBits(block_size=c["block"], accuracy_level=4)
    mm = lambda x, nm: nb.run(ctx, x, d["b_" + nm], d["s_" + nm])
    gqa = rt.GroupQueryAttention(c["Hq"], c["Hkv"], do_rotary=True, local_window_size=-1)
    ssn = rt.SkipSimplifiedLayerNormalization(c["eps"])
    x0 = rt.GatherRows().run(ctx, d["embed"], ids)
    h = rt.SimplifiedLayerNormalization(-1, c["eps"]).run(ctx, x0, d["g_in0"])
    res, presents = x0, []
    for l in range(c["L"]):
        q, k, v = (mm(h, f"qkv{l}"), None, None) if l in packed else (mm(h, f"q{l}"), mm(h, f"k{l}"), mm(h, f"v{l}"))
        a, prk, prv = gqa.run(ctx, q, k, v, seqlens_k, total, past_key=past[l][0], past_value=past[l][1], cos_cache=d["cos"],
                              sin_cache=d["sin"])
        presents.append((prk, prv))
        h2, r2 = ssn.run(ctx, mm(a, f"o{l}"), res, d[f"g_post{l}"], want_sum=True)
        m = rt.Mul().run(ctx, rt.Silu().run(ctx, mm(h2, f"gate{l}")), mm(h2, f"up{l}"))
        if l + 1 < c["L"]:
            h, res = ssn.run(ctx, mm(m, f"down{l}"), r2, d[f"g_in{l + 1}"], want_sum=True)
        else:
            h = ssn.run(ctx, mm(m, f"down{l}"), r2, d["g_final"])
    return mm(h, "lm"), presents
