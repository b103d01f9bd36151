"""Time GroupQueryAttention against the composed path a caller had before it (RotaryEmbedding on Q and on K, the new K / V
copied into the cache with rten_b200_copy, then rten_b200_attention), and the Attention decode call alone on the same
cache, with CUDA events after warm-up, the implementations alternating.

    python tools/gqa_bench.py --out DIR [--repeats 7] [--iters 20]

Shapes: a Llama-3-8B layer (32 / 8 heads, head 128, full non-interleaved rotary) as a decode step at batch 8 over a
4096-position cache that the call extends in place, and as a first prompt of 2048 tokens at batch 1; and a head-64
decode step (16 / 2 heads, batch 8, 4096 positions).  For decode steps it prints the share of the data-sheet HBM
bandwidth (3.35 TB/s) that reading the valid K and V bytes once in the measured time amounts to.  Prints the card name
and power limit with the numbers and writes one JSON line to DIR/gqa_bench.json.  Needs an H100; there is no fallback."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet


def _card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                               text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


def _shape(rt, ctx, B, S, P, H, Hkv, D, rng):
    """Callables (gqa, composed, attention alone or None) of one layer step; the caches hold P + S positions, the first P
    valid, and every call writes the S new tokens at P (decode: in place, into the same buffers)."""
    T = P + S
    f = np.float32
    half = D // 2
    ang = np.arange(T)[:, None] * (500000.0 ** (-np.arange(half) / half))[None, :]
    cos, sin = ctx.to_device(np.cos(ang).astype(f)), ctx.to_device(np.sin(ang).astype(f))
    q = ctx.to_device(rng.uniform(-1, 1, (B, S, H * D)).astype(f))
    k = ctx.to_device(rng.uniform(-1, 1, (B, S, Hkv * D)).astype(f))
    v = ctx.to_device(rng.uniform(-1, 1, (B, S, Hkv * D)).astype(f))
    kc = ctx.to_device(rng.uniform(-1, 1, (B, Hkv, T, D)).astype(f))
    vc = ctx.to_device(rng.uniform(-1, 1, (B, Hkv, T, D)).astype(f))
    st = (Hkv * T * D, T * D, D, 1)
    first = P == 0
    seqlens = ctx.to_device(np.full((B,), T - 1, np.int32))
    out_g = ctx.empty((B, S, H * D))
    gqa = rt.GroupQueryAttention(H, Hkv, do_rotary=True)
    past = dict(past_key=kc.view((B, Hkv, P, D), st), past_value=vc.view((B, Hkv, P, D), st)) if P else {}

    def run_gqa():
        gqa.run(ctx, q, k, v, seqlens, T, cos_cache=cos, sin_cache=sin, present_key=kc, present_value=vc, out=out_g, **past)

    plain = rt.GroupQueryAttention(H, Hkv)
    out_p = ctx.empty((B, S, H * D))

    def run_plain():  # the same step without rotary embedding: what the rotation itself costs
        plain.run(ctx, q, k, v, seqlens, T, present_key=kc, present_value=vc, out=out_p, **past)

    # the composed path: RotaryEmbedding (positions P .. P + S - 1), copies into the cache, Attention
    pos = ctx.to_device(np.broadcast_to(P + np.arange(S, dtype=np.int32), (B, S)).copy())
    qr, kr = ctx.empty((B, S, H * D)), ctx.empty((B, S, Hkv * D))
    rq, rk = rt.RotaryEmbedding(False, H), rt.RotaryEmbedding(False, Hkv)
    kr_heads = kr.view((B, Hkv, S, D), (S * Hkv * D, D, Hkv * D, 1))
    vr_heads = v.view((B, Hkv, S, D), (S * Hkv * D, D, Hkv * D, 1))
    k_slot, v_slot = kc.view((B, Hkv, S, D), st, P * D), vc.view((B, Hkv, S, D), st, P * D)
    q_heads = qr.view((B, H, S, D), (S * H * D, D, H * D, 1))
    out_c = ctx.empty((B, H, S, D))
    att = rt.Attention(is_causal=True, q_num_heads=H, kv_num_heads=Hkv)
    lens = ctx.to_device(np.full((B,), T, np.int32))

    def attention():
        att.run(ctx, q_heads, kc, vc, nonpad_kv_seqlen=lens, out=out_c)

    def composed():
        rq.run(ctx, q, cos, sin, pos, out=qr)
        rk.run(ctx, k, cos, sin, pos, out=kr)
        k_slot.assign(kr_heads)
        v_slot.assign(vr_heads)
        attention()

    return run_gqa, composed, (attention if not first else None), (run_plain if not first else None), (out_g, out_c)


def _stats(ts):
    ts = sorted(ts)
    return dict(median_us=ts[len(ts) // 2], min_us=ts[0], max_us=ts[-1])


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--out", required=True, help="directory for gqa_bench.json")
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("gqa_bench: no CUDA device; this benchmark measures the H100 kernels and has no fallback")
    import rten_b200 as rt
    card, power = _card()
    stream = torch.cuda.Stream()
    ctx = rt.Context(0, stream=stream.cuda_stream)
    rng = np.random.default_rng(0)
    shapes = [("llama3_8b_decode", dict(B=8, S=1, P=4095, H=32, Hkv=8, D=128)),
              ("llama3_8b_prompt", dict(B=1, S=2048, P=0, H=32, Hkv=8, D=128)),
              ("h64_decode", dict(B=8, S=1, P=4095, H=16, Hkv=2, D=64))]
    results = []
    for sname, s in shapes:
        run_gqa, composed, attention, run_plain, (out_g, out_c) = _shape(rt, ctx, rng=rng, **s)
        impls = [("gqa", run_gqa), ("composed", composed)]
        impls += [("attention_alone", attention), ("gqa_no_rotary", run_plain)] if attention else []
        times = {n: [] for n, _ in impls}
        with torch.cuda.stream(stream):
            for _, fn in impls:
                for _ in range(a.warmup):
                    fn()
            for _ in range(a.repeats):
                for n, fn in impls:
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(a.iters):
                        fn()
                    e1.record()
                    e1.synchronize()
                    times[n].append(e0.elapsed_time(e1) * 1e3 / a.iters)
        ctx.sync()
        composed()
        run_gqa()
        ctx.sync()
        yg = out_g.numpy().astype(np.float64)
        yc = out_c.numpy().astype(np.float64).transpose(0, 2, 1, 3).reshape(yg.shape)
        diff = float(np.abs(yg - yc).max() / np.abs(yc).max())
        row = dict(shape=sname, **s, rel_diff_vs_composed=diff, **{n: _stats(ts) for n, ts in times.items()})
        row["speedup_vs_composed"] = row["composed"]["median_us"] / row["gqa"]["median_us"]
        msg = (f"{card} (power limit {power}) {sname:17s}: gqa {row['gqa']['median_us']:8.1f} us [{row['gqa']['min_us']:.1f}, "
               f"{row['gqa']['max_us']:.1f}]  composed {row['composed']['median_us']:8.1f} us [{row['composed']['min_us']:.1f}, "
               f"{row['composed']['max_us']:.1f}]  x{row['speedup_vs_composed']:.2f}")
        if attention:
            kv_bytes = 2.0 * 4 * s["B"] * s["Hkv"] * (s["P"] + s["S"]) * s["D"]
            row["kv_bytes"] = kv_bytes
            row["hbm_fraction_of_datasheet"] = kv_bytes / (row["gqa"]["median_us"] * 1e-6) / HBM_BYTES_PER_S
            msg += (f"  attention alone {row['attention_alone']['median_us']:.1f} us [{row['attention_alone']['min_us']:.1f}, "
                    f"{row['attention_alone']['max_us']:.1f}]  gqa without rotary {row['gqa_no_rotary']['median_us']:.1f} us  K+V read once = {row['hbm_fraction_of_datasheet']:.2f} of the 3.35 TB/s data sheet")
        msg += f"  rel diff {diff:.1e}"
        print(msg)
        results.append(row)
    line = json.dumps(dict(tool="gqa_bench", card=card, power_limit=power, repeats=a.repeats, iters=a.iters, results=results))
    print(line)
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "gqa_bench.json"), "w") as f:
        f.write(line + "\n")


if __name__ == "__main__":
    main()
