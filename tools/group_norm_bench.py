"""Time the fused GroupNorm (+ activation) against the node-by-node plan and torch, at the shapes of the models that use
it: the SD 1.5 U-Net (batch 2; GroupNorm(32) + SiLU at 320 x 64^2, 640 x 32^2, 1280 x 16^2, 1280 x 8^2), the SD VAE
decoder (batch 1; GroupNorm(32) + SiLU at 512 x 64^2, 512 x 128^2, 256 x 256^2, 128 x 512^2) and fast-neural-style
(batch 1; InstanceNorm -- GroupNorm with one channel per group -- + Relu at 32 x 224^2, 64 x 112^2, 128 x 56^2).

Forms, each on channels-last and on NCHW input:
  fused    rten_b200_group_norm: the whole chain in one pass
  unfused  the node-by-node plan the executor runs without the fusion: the first Reshape's copy to contiguous (channels-
           last input only), InstanceNormalization, Mul(gamma), Add(beta), the activation
  torch    F.group_norm + F.silu / F.relu on a tensor in the same memory format
Each form is captured once as a CUDA graph after warm-up; forms alternate, the L2 cache is flushed before every timed
replay, and each of `--repeats` samples averages `--iters` replays timed with CUDA events (tools/depthwise_bench.py).
The bytes bound is x read once and y written once at 3.35 TB/s.

    python tools/group_norm_bench.py [--out DIR] [--repeats 5] [--iters 10]

Prints the card name and power limit with the numbers; with --out, writes one JSON line to DIR/group_norm_bench.json.
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

# (model, N, C, H = W, groups (0: one per channel), activation)
SHAPES = [("SD U-Net", 2, 320, 64, 32, "silu"), ("SD U-Net", 2, 640, 32, 32, "silu"), ("SD U-Net", 2, 1280, 16, 32, "silu"),
          ("SD U-Net", 2, 1280, 8, 32, "silu"),
          ("SD VAE decoder", 1, 512, 64, 32, "silu"), ("SD VAE decoder", 1, 512, 128, 32, "silu"),
          ("SD VAE decoder", 1, 256, 256, 32, "silu"), ("SD VAE decoder", 1, 128, 512, 32, "silu"),
          ("fast-neural-style", 1, 32, 224, 0, "relu"), ("fast-neural-style", 1, 64, 112, 0, "relu"),
          ("fast-neural-style", 1, 128, 56, 0, "relu")]


def _stats(ts):
    ts = sorted(ts)
    return dict(median_us=ts[len(ts) // 2], min_us=ts[0], max_us=ts[-1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    import torch
    import torch.nn.functional as F
    import rten_b200 as rt
    name, power = _card()
    print(f"card: {name}; power limit: {power}", flush=True)
    flush = torch.empty(64 * 1024 * 1024, dtype=torch.int32, device="cuda")  # 256 MB > 50 MB L2
    stream = torch.cuda.Stream()
    ctx = rt.Context(0, stream=stream.cuda_stream)
    rng = np.random.default_rng(0)
    rows_out = []
    eps = 1e-5
    for model, N, C, H, groups, act in SHAPES:
        G = groups or C
        shape = (N, C, H, H)
        numel = N * C * H * H
        xn = rng.standard_normal(shape).astype(np.float32)
        gn, ben = (1 + 0.1 * rng.standard_normal(C)).astype(np.float32), (0.1 * rng.standard_normal(C)).astype(np.float32)
        s, b = ctx.to_device(np.ones(G, np.float32)), ctx.to_device(np.zeros(G, np.float32))
        g, be = ctx.to_device(gn), ctx.to_device(ben)
        g3, be3 = ctx.to_device(gn.reshape(C, 1, 1)), ctx.to_device(ben.reshape(C, 1, 1))
        code = rt.ACT_SILU if act == "silu" else rt.ACT_RELU
        fused, inorm, mul, add = rt.GroupNorm(G, eps, code), rt.InstanceNormalization(eps), rt.Mul(), rt.Add()
        act_op = rt.Silu() if act == "silu" else rt.Relu()
        tact = F.silu if act == "silu" else F.relu
        gt, bet = torch.from_numpy(gn).cuda(), torch.from_numpy(ben).cuda()
        keep = []
        forms, torch_forms = {}, {}
        for layout in ("cl", "nchw"):
            x = ctx.to_device(xn, channels_last=layout == "cl")
            xc = ctx.empty(shape)
            xt = torch.from_numpy(xn).cuda()
            if layout == "cl":
                xt = xt.contiguous(memory_format=torch.channels_last)

            def unfused(x=x, xc=xc, layout=layout):
                if layout == "cl":
                    xc.assign(x)  # the first Reshape makes its input contiguous
                src = xc if layout == "cl" else x
                y = inorm.run(ctx, src.reshape(N, G, numel // (N * G)), s, b)
                y = add.run(ctx, mul.run(ctx, y.reshape(shape), g3), be3)
                keep.append(act_op.run(ctx, y))

            forms[f"fused {layout}"] = lambda x=x: keep.append(fused.run(ctx, x, s, b, g, be))
            forms[f"unfused {layout}"] = unfused
            torch_forms[f"torch {layout}"] = lambda xt=xt: keep.append(tact(F.group_norm(xt, G, gt, bet, eps)))
        graphs = {}
        with torch.cuda.stream(stream):
            for _ in range(a.warmup):
                for f in list(forms.values()) + list(torch_forms.values()):
                    f()
            ctx.sync()
            stream.synchronize()
            keep.clear()
            for fname, f in forms.items():
                ctx.graph_begin()
                f()
                graphs[fname] = ctx.graph_end()
            for fname, f in torch_forms.items():
                tg = torch.cuda.CUDAGraph()
                with torch.cuda.graph(tg, stream=stream):
                    f()
                graphs[fname] = tg
            times = _time_graphs(graphs, flush, a.repeats, a.iters)
        ctx.sync()
        torch.cuda.synchronize()
        t_b = 8 * numel / HBM_BYTES_PER_S
        row = dict(model=model, dims=list(shape), groups=G, act=act, bytes_bound_us=t_b * 1e6)
        for fname, ts in times.items():
            st = _stats(ts)
            st.update(bytes_share=t_b / (st["median_us"] * 1e-6))
            row[fname] = st
            print(f"[{power}] {model:18s} {str(shape):22s} G{G:<4d} {fname:14s} {st['median_us']:9.1f} us [{st['min_us']:.1f}, "
                  f"{st['max_us']:.1f}]  {100 * st['bytes_share']:3.0f}% of the bytes bound ({t_b * 1e6:.1f} us)", flush=True)
        rows_out.append(row)
        keep.clear()
        del graphs
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "group_norm_bench.json"), "w") as f:
            f.write(json.dumps(dict(card=name, power=power, time=time.strftime("%Y-%m-%d %H:%M:%S"), rows=rows_out)) + "\n")


if __name__ == "__main__":
    main()
