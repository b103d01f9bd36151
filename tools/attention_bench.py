"""Time the Attention operator's prefill kernel (attn_prefill_kernel: one call, scores kept on chip) against the composed
path it replaces (an explicit additive causal mask, FusedMatMul(Q K^T) -> AddSoftmax -> MatMul(P V), the [B, heads, T, L]
scores through HBM), with CUDA events after warm-up, in both f32 modes, the two implementations alternating.

    python tools/attention_bench.py --out DIR [--repeats 7] [--iters 20]

Shapes: the GPT-2 prefill layer (B 8, 12 heads, head 64, T 512 over a 576-position cache, value cache transposed) and a
grouped-query layer (B 2, 32 / 8 heads, head 128, T = L = 2048, natural value layout; the composed path, which has no
grouped-query form, gets the key / value heads repeated once, outside the timed window).  Prints the card name and power
limit with the numbers and writes one JSON line to DIR/attention_bench.json.  Needs an H100; there is no fallback."""
import argparse
import json
import math
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                               text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


def _shape(rt, ctx, name, B, qh, kvh, dh, T, M, P, v_transposed, rng):
    """(routed call, composed call, their outputs, flops, bytes) of one attention layer.  flops: the causal (query, key)
    pairs (row s sees keys 0 ..= P + s), two products of 2 dh flops each; bytes: Q, K, V read and O written once, the
    least any implementation moves."""
    L = P + T
    q = ctx.to_device(rng.uniform(-1, 1, (B, qh, T, dh)).astype(np.float32))
    kc = ctx.to_device(rng.uniform(-1, 1, (B, kvh, M, dh)).astype(np.float32))
    if v_transposed:
        vt = ctx.to_device(rng.uniform(-1, 1, (B, kvh, dh, M)).astype(np.float32))
        v_all = vt.view((B, kvh, M, dh), (kvh * dh * M, dh * M, 1, M))
    else:
        v_all = ctx.to_device(rng.uniform(-1, 1, (B, kvh, M, dh)).astype(np.float32))
    scale = 1.0 / math.sqrt(dh)
    lens = ctx.to_device(np.full((B,), L, np.int32))
    out_a = ctx.empty((B, qh, T, dh))
    op = rt.Attention(is_causal=True, q_num_heads=qh, kv_num_heads=kvh, scale=scale)
    routed = lambda: op.run(ctx, q, kc, v_all, nonpad_kv_seqlen=lens, out=out_a)
    # the composed path: the caller's additive mask, the key / value heads repeated for grouped-query layers
    mask = ctx.to_device(np.where(np.arange(L)[None, :] <= (P + np.arange(T))[:, None], 0.0, -np.inf).astype(np.float32).reshape(1, 1, T, L))
    if kvh != qh:
        rep = qh // kvh
        k_np = np.repeat(kc.numpy()[:, :, :L], rep, axis=1)
        v_np = np.repeat(v_all.numpy()[:, :, :L], rep, axis=1)
        k_c, v_c = ctx.to_device(np.ascontiguousarray(k_np)), ctx.to_device(np.ascontiguousarray(v_np))
        kt = k_c.view((B, qh, dh, L), (qh * L * dh, L * dh, 1, dh))
        v_l = v_c
    else:
        kt = kc.view((B, qh, dh, L), (qh * M * dh, M * dh, 1, dh))
        v_l = vt.view((B, qh, L, dh), (qh * dh * M, dh * M, 1, M)) if v_transposed else v_all.view((B, qh, L, dh), (qh * M * dh, M * dh, dh, 1))
    scores = ctx.empty((B, qh, T, L))
    out_c = ctx.empty((B, qh, T, dh))
    fmm, asm, mm = rt.FusedMatMul(scale), rt.AddSoftmax(), rt.MatMul()

    def composed():
        fmm.run(ctx, q, kt, out=scores)
        asm.run(ctx, scores, mask, in_place=True)
        mm.run(ctx, scores, v_l, out=out_c)

    pairs = B * qh * sum(min(L, P + s + 1) for s in range(T))
    flops = 4.0 * dh * pairs
    nbytes = 4.0 * (2 * B * qh * T * dh + 2 * B * kvh * L * dh)
    return routed, composed, (out_a, out_c), flops, nbytes


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--out", required=True, help="directory for attention_bench.json")
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("attention_bench: no CUDA device; this benchmark measures the H100 kernels and has no fallback")
    import rten_b200 as rt
    card, power = _card()
    stream = torch.cuda.Stream()
    ctx = rt.Context(0, stream=stream.cuda_stream)
    rng = np.random.default_rng(0)
    shapes = [("gpt2_prefill", dict(B=8, qh=12, kvh=12, dh=64, T=512, M=576, P=0, v_transposed=True)),
              ("gqa_32_8_h128", dict(B=2, qh=32, kvh=8, dh=128, T=2048, M=2048, P=0, v_transposed=False))]
    results = []
    for sname, s in shapes:
        routed, composed, (out_a, out_c), flops, nbytes = _shape(rt, ctx, sname, rng=rng, **s)
        for tf32 in (False, True):
            ctx.set_f32_mode(not tf32)
            mode = "tf32" if tf32 else "3xtf32"
            times = {"prefill_kernel": [], "composed": []}
            with torch.cuda.stream(stream):
                for fn in (routed, composed):
                    for _ in range(a.warmup):
                        fn()
                for _ in range(a.repeats):
                    for impl, fn in (("prefill_kernel", routed), ("composed", composed)):
                        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        e0.record()
                        for _ in range(a.iters):
                            fn()
                        e1.record()
                        e1.synchronize()
                        times[impl].append(e0.elapsed_time(e1) * 1e3 / a.iters)
            ctx.sync()
            ya, yc = out_a.numpy().astype(np.float64), out_c.numpy().astype(np.float64)
            diff = float(np.abs(ya - yc).max() / np.abs(yc).max())
            row = dict(shape=sname, mode=mode, **{k: v for k, v in s.items()}, flops=flops, min_bytes=nbytes, rel_diff_vs_composed=diff)
            for impl, ts in times.items():
                ts = sorted(ts)
                med = ts[len(ts) // 2]
                row[impl] = dict(median_us=med, min_us=ts[0], max_us=ts[-1], tflops=flops / (med * 1e-6) / 1e12)
            row["speedup"] = row["composed"]["median_us"] / row["prefill_kernel"]["median_us"]
            results.append(row)
            print(f"{card} (power limit {power}) {sname:14s} {mode:6s}: prefill kernel {row['prefill_kernel']['median_us']:8.1f} us "
                  f"[{row['prefill_kernel']['min_us']:.1f}, {row['prefill_kernel']['max_us']:.1f}]  composed {row['composed']['median_us']:8.1f} us "
                  f"[{row['composed']['min_us']:.1f}, {row['composed']['max_us']:.1f}]  x{row['speedup']:.2f}  "
                  f"{row['prefill_kernel']['tflops']:.1f} TFLOP/s causal  rel diff {diff:.1e}")
    line = json.dumps(dict(tool="attention_bench", card=card, power_limit=power, repeats=a.repeats, iters=a.iters, results=results))
    print(line)
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "attention_bench.json"), "w") as f:
        f.write(line + "\n")


if __name__ == "__main__":
    main()
