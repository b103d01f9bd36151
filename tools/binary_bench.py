"""Time broadcast Add / Sub / Mul (launch_binary in rowops.cu) in each of its layouts at the shapes the benched graphs
run: BERT-base (16 x 128 x 768) residual adds (flat; also with a misaligned operand, which runs the flat kernel
scalar) and its position-table add (periodic), GPT-2 small batch 8 position adds of a decode step (8 x 1 x 768) and of a
512-token prefill (8 x 512 x 768) (periodic), and one large strided case, an NCHW tensor plus a channels-last one
(32 x 64 x 56 x 56).  Every shape runs f32 Add and Mul, f32 Sub and i32 Add.
Each form is captured once as a CUDA graph after warm-up; forms alternate, the L2 cache is flushed before every timed
replay, and each of `--repeats` samples averages `--iters` replays timed with CUDA events (tools/depthwise_bench.py).
The bytes bound counts a, b's distinct elements and the output once, at 3.35 TB/s.

    python tools/binary_bench.py [--lib PATH] [--out DIR] [--repeats 7] [--iters 50]

--lib loads that build of librten_b200.so instead of the tree's, so that two builds (say a change and its parent) can
be timed alternately on one card.  Each line also prints a digest of the form's output: two builds computed the same
bits where their digests agree.  Prints the card name and power limit with the numbers; with --out, writes one JSON
line to DIR/binary_bench.json.  Needs an H100; there is no fallback."""
import argparse
import hashlib
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from depthwise_bench import HBM_BYTES_PER_S, _card, _time_graphs  # noqa: E402

# (name, the kernel layout launch_binary picks, a's shape, b's shape, operand placement)
CASES = [
    ("BERT-base residual", "flat", (16, 128, 768), (16, 128, 768), "dense"),
    ("BERT-base residual, a misaligned", "flat scalar", (16, 128, 768), (16, 128, 768), "a misaligned"),
    ("BERT-base position table", "periodic", (16, 128, 768), (128, 768), "dense"),
    ("GPT-2 B8 decode position", "periodic", (8, 1, 768), (1, 768), "dense"),
    ("GPT-2 B8 prefill position", "periodic", (8, 512, 768), (512, 768), "dense"),
    ("NCHW + channels-last", "strided", (32, 64, 56, 56), (32, 64, 56, 56), "b channels-last"),
]
FORMS = [("f32 Add", np.float32, "Add"), ("f32 Mul", np.float32, "Mul"), ("f32 Sub", np.float32, "Sub"),
         ("i32 Add", np.int32, "Add")]


def _stats(ts):
    ts = sorted(ts)
    return dict(median_us=ts[len(ts) // 2], min_us=ts[0], max_us=ts[-1])


def _operands(ctx, rng, dtype, ash, bsh, placement):
    if dtype == np.int32:
        an, bn = (rng.integers(-2 ** 31, 2 ** 31, s, dtype=np.int64).astype(np.int32) for s in (ash, bsh))
    else:
        an, bn = (rng.uniform(-3, 3, s).astype(np.float32) for s in (ash, bsh))
    if placement == "a misaligned":  # one element past a 16-byte boundary
        buf = ctx.to_device(np.concatenate([np.zeros(1, an.dtype), an.reshape(-1)]))
        return buf.view(ash, tuple(s // an.itemsize for s in an.strides), 1), ctx.to_device(bn)
    return ctx.to_device(an), ctx.to_device(bn, channels_last=placement == "b channels-last")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=None, help="librten_b200.so to load instead of the tree's")
    ap.add_argument("--out", default=None)
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    import torch
    import rten_b200 as rt
    from rten_b200 import _lib
    if a.lib:
        _lib.LIB_PATH = os.path.abspath(a.lib)
    lib = _lib.LIB_PATH
    name, power = _card()
    print(f"card: {name}; power limit: {power}; library: {lib}", flush=True)
    flush = torch.empty(64 * 1024 * 1024, dtype=torch.int32, device="cuda")  # 256 MB > 50 MB L2
    stream = torch.cuda.Stream()
    ctx = rt.Context(0, stream=stream.cuda_stream)
    rng = np.random.default_rng(0)
    ops = {"Add": rt.Add(), "Sub": rt.Sub(), "Mul": rt.Mul()}
    rows_out = []
    for cname, kernel, ash, bsh, placement in CASES:
        outs, graphs, nbytes = {}, {}, {}
        with torch.cuda.stream(stream):
            for fname, dtype, op in FORMS:
                x, y = _operands(ctx, rng, dtype, ash, bsh, placement)
                o = ctx.empty(ash, dtype)
                outs[fname] = (x, y, o)
                for _ in range(a.warmup):
                    ops[op].run(ctx, x, y, out=o)
                ctx.sync()
                ctx.graph_begin()
                ops[op].run(ctx, x, y, out=o)
                graphs[fname] = ctx.graph_end()
                nbytes[fname] = np.dtype(dtype).itemsize * (2 * int(np.prod(ash)) + int(np.prod(bsh)))
            stream.synchronize()
            times = _time_graphs(graphs, flush, a.repeats, a.iters)
        ctx.sync()
        row = dict(case=cname, kernel=kernel, a=list(ash), b=list(bsh), placement=placement)
        for fname, ts in times.items():
            s = _stats(ts)
            t_b = nbytes[fname] / HBM_BYTES_PER_S
            s.update(bytes_bound_us=t_b * 1e6, bytes_share=t_b / (s["median_us"] * 1e-6),
                     digest=hashlib.sha1(outs[fname][2].numpy().tobytes()).hexdigest()[:12])
            row[fname] = s
            print(f"[{power}] {cname:34s} {kernel:11s} {fname:8s} {s['median_us']:8.1f} us [{s['min_us']:.1f}, "
                  f"{s['max_us']:.1f}]  {100 * s['bytes_share']:3.0f}% of the bytes bound ({t_b * 1e6:.1f} us)  "
                  f"digest {s['digest']}", flush=True)
        rows_out.append(row)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "binary_bench.json"), "w") as f:
            f.write(json.dumps(dict(card=name, power=power, lib=lib, time=time.strftime("%Y-%m-%d %H:%M:%S"),
                                    rows=rows_out)) + "\n")


if __name__ == "__main__":
    main()
