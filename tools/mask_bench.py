"""Time Where, Equal, Expand and Trilu (masks.cu) at the shapes decoder exports run them: Where over GPT-2 attention
scores (8 x 12 x 512 x 512) with the causal-bias window as the condition (rows of stride 1024 broadcast over batch and
heads) and a 0-D y, dense Where and Equal on 16 x 12 x 128 x 128, Expand for Llama-3-8B's repeat_kv (8 -> 32 heads of
4096 x 128) and Trilu on a 2048 x 2048 matrix.
Each form is captured once as a CUDA graph after warm-up; the L2 cache is flushed before every timed replay, and each of
`--repeats` samples averages `--iters` replays timed with CUDA events (tools/depthwise_bench.py).  The bytes bound of a
row is its inputs read once and its output written once, at 3.35 TB/s.

    python tools/mask_bench.py [--out DIR] [--repeats 7] [--iters 50]

Prints the card name and power limit with the numbers; with --out, writes one JSON line to DIR/mask_bench.json.  Needs
an H100; there is no fallback."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from depthwise_bench import HBM_BYTES_PER_S, _card, _time_graphs  # noqa: E402
from elementwise_math_bench import _stats  # noqa: E402


def _forms(rt, ctx, rng):
    """{row name: (bytes bound, [(form name, callable)])}"""
    f32, i32 = np.float32, np.int32
    rows = {}
    # GPT-2: where(bias[:, :, 0:512, 0:512], w, finfo.min), bias a [1, 1, 1024, 1024] buffer
    bias = ctx.to_device(np.tril(np.ones((1024, 1024), i32))[None, None])
    cond = bias.view((1, 1, 512, 512), (1024 * 1024, 1024 * 1024, 1024, 1))
    w = ctx.to_device(rng.standard_normal((8, 12, 512, 512)).astype(f32))
    mn = ctx.to_device(np.array(np.finfo(f32).min, f32))
    wo = ctx.empty(w.shape, f32)
    rows["Where, GPT-2 scores 8x12x512x512, bias window, 0-D y"] = (
        4 * (512 * 512 + 2 * w.size), [("Where", lambda: rt.Where().run(ctx, cond, w, mn, out=wo))])
    shp = (16, 12, 128, 128)
    c = ctx.to_device(rng.integers(0, 2, shp).astype(i32))
    a, b = (ctx.to_device(rng.standard_normal(shp).astype(f32)) for _ in range(2))
    o, oi = ctx.empty(shp, f32), ctx.empty(shp, i32)
    n = int(np.prod(shp))
    rows["Where, dense 16x12x128x128"] = (16 * n, [("Where", lambda: rt.Where().run(ctx, c, a, b, out=o))])
    rows["Equal, dense 16x12x128x128"] = (12 * n, [("Equal", lambda: rt.Equal().run(ctx, a, b, out=oi))])
    kv = ctx.to_device(rng.standard_normal((1, 8, 1, 4096, 128)).astype(f32))
    ko = ctx.empty((1, 8, 4, 4096, 128), f32)
    rows["Expand, repeat_kv 8 -> 32 heads x 4096 x 128"] = (
        4 * (kv.size + 4 * kv.size), [("Expand", lambda: rt.Expand().run(ctx, kv, (1, 8, 4, 4096, 128), out=ko))])
    t = ctx.to_device(rng.standard_normal((2048, 2048)).astype(f32))
    to = ctx.empty(t.shape, f32)
    rows["Trilu 2048x2048"] = (8 * t.size, [("Trilu", lambda: rt.Trilu(False).run(ctx, t, 0, out=to))])
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    import torch
    import rten_b200 as rt
    name, power = _card()
    print(f"card: {name}; power limit: {power}", flush=True)
    flush = torch.empty(64 * 1024 * 1024, dtype=torch.int32, device="cuda")  # 256 MB > 50 MB L2
    stream = torch.cuda.Stream()
    ctx = rt.Context(0, stream=stream.cuda_stream)
    rows_out = []
    with torch.cuda.stream(stream):
        rows = _forms(rt, ctx, np.random.default_rng(0))
        for rname, (nbytes, forms) in rows.items():
            graphs = {}
            for fname, fn in forms:
                for _ in range(a.warmup):
                    fn()
                ctx.sync()
                ctx.graph_begin()
                fn()
                graphs[fname] = ctx.graph_end()
            stream.synchronize()
            times = _time_graphs(graphs, flush, a.repeats, a.iters)
            t_b = nbytes / HBM_BYTES_PER_S
            row = dict(row=rname, bytes_bound_us=t_b * 1e6)
            for fname, ts in times.items():
                st = _stats(ts)
                st["bytes_share"] = t_b / (st["median_us"] * 1e-6)
                row[fname] = st
                print(f"[{power}] {rname:52s} {st['median_us']:8.1f} us [{st['min_us']:.1f}, {st['max_us']:.1f}]  "
                      f"{100 * st['bytes_share']:3.0f}% of the bytes bound ({t_b * 1e6:.1f} us)", flush=True)
            rows_out.append(row)
    ctx.sync()
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "mask_bench.json"), "w") as f:
            f.write(json.dumps(dict(card=name, power=power, time=time.strftime("%Y-%m-%d %H:%M:%S"), rows=rows_out)) + "\n")


if __name__ == "__main__":
    main()
