"""Time Div, Pow, Tanh and the decomposed norm chains that torch's unfused exports run, at the shapes those exports run
them: Div by a scalar on BERT-base attention scores (16 x 12 x 128 x 128), Pow(x, 3) and Tanh on GPT-2 MLP activations
(8 x 512 x 3072), the RMSNorm chain Pow -> ReduceMean -> Add -> Sqrt -> Reciprocal -> Mul -> Mul at 2048 x 4096 against
rten_b200_rms_norm, and the LayerNorm chain ReduceMean -> Sub -> Pow -> ReduceMean -> Add -> Sqrt -> Div -> Mul -> Add at
16 x 128 x 768 against rten_b200_layer_norm.  The chain-vs-fused rows are the baseline a load-time fusion is measured
against.
Each form is captured once as a CUDA graph after warm-up; forms alternate, the L2 cache is flushed before every timed
replay, and each of `--repeats` samples averages `--iters` replays timed with CUDA events (tools/depthwise_bench.py).
The bytes bound of a row is the least traffic the operation needs -- its input and output once, at 3.35 TB/s; a chain
is held to the bound of the fused operator it stands for.

    python tools/elementwise_math_bench.py [--out DIR] [--repeats 7] [--iters 50]

Prints the card name and power limit with the numbers; with --out, writes one JSON line to DIR/elementwise_math_bench.json.
Needs an H100; there is no fallback."""
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


def _stats(ts):
    ts = sorted(ts)
    return dict(median_us=ts[len(ts) // 2], min_us=ts[0], max_us=ts[-1])


def _forms(rt, ctx, rng):
    """{row name: (bytes bound, [(form name, callable)])}"""
    f32 = np.float32
    dev = lambda a: ctx.to_device(np.asarray(a, f32))  # noqa: E731
    rows = {}
    s = dev(rng.uniform(-8, 8, (16, 12, 128, 128)))
    so, eight = ctx.empty(s.shape, f32), dev(8.0)
    rows["Div by scalar, BERT-base scores 16x12x128x128"] = (8 * s.size, [("Div", lambda: rt.Div().run(ctx, s, eight, out=so))])
    h = dev(rng.uniform(-4, 4, (8, 512, 3072)))
    ho = ctx.empty(h.shape, f32)
    three = dev(3.0)
    rows["GPT-2 MLP 8x512x3072"] = (8 * h.size, [("Pow(x, 3)", lambda: rt.Pow().run(ctx, h, three, out=ho)),
                                                 ("Tanh", lambda: rt.Tanh().run(ctx, h, in_place=True))])
    # RMSNorm chain at 2048 x 4096
    x = dev(rng.uniform(-2, 2, (2048, 4096)))
    g = dev(rng.uniform(0.5, 1.5, (4096,)))
    t1, y = ctx.empty(x.shape, f32), ctx.empty(x.shape, f32)
    ms = ctx.empty((2048, 1), f32)
    two, eps6 = dev(2.0), dev(1e-6)

    def rms_chain():
        rt.Pow().run(ctx, x, two, out=t1)
        rt.ReduceMean([-1], True).run(ctx, t1, out=ms)
        rt.Add().run(ctx, ms, eps6, out=ms)
        rt.Sqrt().run(ctx, ms, in_place=True)
        rt.Reciprocal().run(ctx, ms, in_place=True)
        rt.Mul().run(ctx, x, ms, out=t1)
        rt.Mul().run(ctx, t1, g, out=y)
    rows["RMSNorm 2048x4096"] = (8 * x.size, [("chain", rms_chain),
                                              ("rms_norm", lambda: rt.RMSNormalization(epsilon=1e-6).run(ctx, x, g, out=y))])
    # LayerNorm chain at 16 x 128 x 768
    z = dev(rng.uniform(-2, 2, (16, 128, 768)))
    lg, lb = dev(rng.uniform(0.5, 1.5, (768,))), dev(rng.uniform(-0.2, 0.2, (768,)))
    c, c2, zy = (ctx.empty(z.shape, f32) for _ in range(3))
    mu, var = ctx.empty((16, 128, 1), f32), ctx.empty((16, 128, 1), f32)
    eps12 = dev(1e-12)

    def ln_chain():
        rt.ReduceMean([-1], True).run(ctx, z, out=mu)
        rt.Sub().run(ctx, z, mu, out=c)
        rt.Pow().run(ctx, c, two, out=c2)
        rt.ReduceMean([-1], True).run(ctx, c2, out=var)
        rt.Add().run(ctx, var, eps12, out=var)
        rt.Sqrt().run(ctx, var, in_place=True)
        rt.Div().run(ctx, c, var, out=c2)
        rt.Mul().run(ctx, c2, lg, out=c2)
        rt.Add().run(ctx, c2, lb, out=zy)
    rows["LayerNorm 16x128x768"] = (8 * z.size, [("chain", ln_chain),
                                                 ("layer_norm", lambda: rt.LayerNormalization(epsilon=1e-12).run(ctx, z, lg, lb, out=zy))])
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
                print(f"[{power}] {rname:46s} {fname:10s} {st['median_us']:8.1f} us [{st['min_us']:.1f}, {st['max_us']:.1f}]  "
                      f"{100 * st['bytes_share']:3.0f}% of the bytes bound ({t_b * 1e6:.1f} us)", flush=True)
            rows_out.append(row)
    ctx.sync()
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "elementwise_math_bench.json"), "w") as f:
            f.write(json.dumps(dict(card=name, power=power, time=time.strftime("%Y-%m-%d %H:%M:%S"), rows=rows_out)) + "\n")


if __name__ == "__main__":
    main()
