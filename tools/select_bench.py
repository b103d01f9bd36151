"""Time TopK and ArgMax (topk.cu, reduce.cu's arg-reduce kernels) against torch.topk / torch.argmax, and the Generator's
device sampling against its host path.

Kernels: TopK k = 50 at 1 x 32000, 8 x 32000 and 8 x 128256 (sampling a vocabulary; 8 x 128256 also on rows of four
distinct values, which put nearly every key of each radix pass into the same histogram bins), k = 8 at 4096 x 64 and k = 2 at
4096 x 8 (mixture-of-experts routing), ArgMax at 8 x 128256 and 2048 x 32000, all f32.  Each form is captured once as a
CUDA graph after warm-up; the forms alternate, the L2 cache is flushed before every timed replay, and each of
`--repeats` samples averages `--iters` replays timed with CUDA events (tools/depthwise_bench.py).  The bytes bound counts
the input read once and the outputs written once, at 3.35 TB/s.  Every case also checks that this project's indices
equal torch's (the inputs are continuous random values: no ties), and on the tie-heavy rows the values do.

End to end: tokens/s of Generator(ModelDecoder(...)) over the int4 decoder of tools/genai_decode_bench.py
(Llama-3-8B-shaped layers, --layers of them) at vocabularies 32000 and 128256, B 1 and 8, with TopKSampler(50) and
ArgMaxSampler, sampling on the device (no logits filter) against the host path (an identity logits filter, which makes
the Generator copy the logits and sample in numpy), alternating.

    python tools/select_bench.py [--out DIR] [--repeats 7] [--iters 50] [--layers 4] [--tokens 32] [--no-e2e]

Prints the card name and power limit with the numbers; with --out, writes DIR/select_bench.json.  Needs an H100."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.dirname(os.path.abspath(__file__)), os.path.join(ROOT, "tests")]

from depthwise_bench import HBM_BYTES_PER_S, _card, _time_graphs  # noqa: E402

# (name, rows, n, k or None for ArgMax); "ties" rows hold 4 distinct values, so every radix-select pass bins nearly
# every key into the same few histogram bins (shared-memory atomics on few addresses)
CASES = [("TopK k=50, 1 x 32000", 1, 32000, 50), ("TopK k=50, 8 x 32000", 8, 32000, 50),
         ("TopK k=50, 8 x 128256", 8, 128256, 50), ("TopK k=50, 8 x 128256 ties", 8, 128256, 50),
         ("TopK k=8, 4096 x 64 (MoE)", 4096, 64, 8),
         ("TopK k=2, 4096 x 8 (MoE)", 4096, 8, 2), ("ArgMax, 8 x 128256", 8, 128256, None),
         ("ArgMax, 2048 x 32000", 2048, 32000, None)]


def _stats(ts):
    ts = sorted(ts)
    return dict(median_us=round(ts[len(ts) // 2], 2), min_us=round(ts[0], 2), max_us=round(ts[-1], 2))


def bench_kernels(a, rt, power):
    import torch
    flush = torch.empty(64 * 1024 * 1024, dtype=torch.int32, device="cuda")  # 256 MB > 50 MB L2
    stream = torch.cuda.Stream()
    ctx = rt.Context(0, stream=stream.cuda_stream)
    rng = np.random.default_rng(0)
    rows = []
    for name, B, n, k in CASES:
        x = rng.standard_normal((B, n)).astype(np.float32)
        if name.endswith("ties"):
            x = rng.integers(0, 4, (B, n)).astype(np.float32)
        xd, xt = ctx.to_device(x), torch.from_numpy(x).cuda()
        graphs, outs = {}, {}
        with torch.cuda.stream(stream):
            run_rt = (lambda: rt.TopK().run(ctx, xd, k)) if k else (lambda: (None, rt.ArgMax(axis=1, keep_dims=False).run(ctx, xd)))
            run_t = (lambda: torch.topk(xt, k, dim=1)) if k else (lambda: (None, torch.argmax(xt, dim=1)))
            for _ in range(a.warmup):
                run_rt(), run_t()
            ctx.sync()
            stream.synchronize()
            ctx.graph_begin()
            outs["rten_b200"] = run_rt()
            graphs["rten_b200"] = ctx.graph_end()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=stream):
                outs["torch"] = run_t()
            graphs["torch"] = g
            stream.synchronize()
            times = _time_graphs(graphs, flush, a.repeats, a.iters)
        ctx.sync()
        mine = outs["rten_b200"][1].numpy().reshape(B, -1)
        theirs = outs["torch"][1].cpu().numpy().reshape(B, -1)
        # with ties torch's order among equal values is unspecified: compare this project's values with torch's
        same = bool(np.array_equal(mine, theirs)) if not name.endswith("ties") else bool(np.array_equal(
            outs["rten_b200"][0].numpy().reshape(B, -1), outs["torch"][0].cpu().numpy().reshape(B, -1)))
        kk = k or 1
        nbytes = 4 * B * n + (8 if k else 4) * B * kk
        t_b = nbytes / HBM_BYTES_PER_S * 1e6
        row = dict(case=name, rows=B, n=n, k=k, bytes_bound_us=round(t_b, 2), same_indices=same)
        for form, ts in times.items():
            s = _stats(ts)
            s["bytes_share"] = round(t_b / s["median_us"], 3)
            row[form] = s
        ratio = row["torch"]["median_us"] / row["rten_b200"]["median_us"]
        row["speedup_vs_torch"] = round(ratio, 2)
        print(f"[{power}] {name:28s} rten_b200 {row['rten_b200']['median_us']:7.1f} us "
              f"[{row['rten_b200']['min_us']:.1f}, {row['rten_b200']['max_us']:.1f}]  torch {row['torch']['median_us']:7.1f} us  "
              f"x{ratio:.2f}  bytes bound {t_b:.2f} us ({100 * row['rten_b200']['bytes_share']:.0f}%)  same indices: {same}",
              flush=True)
        rows.append(row)
    return rows


def bench_generator(a, rt, card):
    import genai_decoder as gd
    from genai_decode_bench import weights
    from rten_b200.generate import ArgMaxSampler, Generator, ModelDecoder, TopKSampler
    from rten_b200.model import Model
    rows = []
    for V in (32000, 128256):
        c = dict(L=a.layers, V=V, Hq=32, Hkv=8, D=128, I=14336, block=32, maxp=8192, eps=1e-5)
        w = weights(c)
        ctx = rt.Context(0)
        m = Model(ctx, gd.genai_graph(w, (0,), c))
        del w
        r = np.random.default_rng(3)
        for B in (1, 8):
            prompt = r.integers(0, V, (B, 16)).astype(np.int32)
            for sname, make in (("TopKSampler(50)", lambda: TopKSampler(50, 1.0, 7)), ("ArgMaxSampler", ArgMaxSampler)):
                res = {}
                for _ in range(a.samples):
                    for path in ("device", "host"):
                        gen = Generator(ModelDecoder(m, B, 128)).with_prompt(prompt).with_sampler(make())
                        if path == "host":
                            gen = gen.with_logits_filter(lambda logits, prev: logits)
                        next(gen)
                        ctx.sync()
                        t0 = time.perf_counter()
                        toks = [next(gen) for _ in range(a.tokens)]
                        ctx.sync()
                        res.setdefault(path, []).append(a.tokens * B / (time.perf_counter() - t0))
                        res.setdefault(path + "_tokens", np.stack(toks, 1))
                row = dict(V=V, B=B, sampler=sname, layers=a.layers,
                           same_tokens=bool(np.array_equal(res["device_tokens"], res["host_tokens"])))
                for path in ("device", "host"):
                    v = sorted(res[path])
                    row[path + "_tokens_per_s"] = round(v[len(v) // 2], 1)
                row["speedup"] = round(row["device_tokens_per_s"] / row["host_tokens_per_s"], 2)
                print(f"[{card}] V {V:6d} B {B} {sname:16s} device {row['device_tokens_per_s']:8.1f} tok/s  "
                      f"host {row['host_tokens_per_s']:8.1f} tok/s  x{row['speedup']:.2f}  same tokens: {row['same_tokens']}",
                      flush=True)
                rows.append(row)
        del m, ctx
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--layers", type=int, default=4)
    ap.add_argument("--tokens", type=int, default=32)
    ap.add_argument("--samples", type=int, default=3)
    ap.add_argument("--no-e2e", action="store_true")
    a = ap.parse_args()
    import rten_b200 as rt
    name, power = _card()
    print(f"card: {name}; power limit: {power}", flush=True)
    res = dict(card=name, power=power, time=time.strftime("%Y-%m-%d %H:%M:%S"), kernels=bench_kernels(a, rt, power))
    if not a.no_e2e:
        res["generator"] = bench_generator(a, rt, power)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "select_bench.json"), "w") as f:
            f.write(json.dumps(res) + "\n")


if __name__ == "__main__":
    main()
