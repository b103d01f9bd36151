"""Time Sigmoid / Silu / HardSigmoid / HardSwish, standalone and fused into the convolution epilogue:
  (a) the four standalone operators on a 32x112x112x96 channels-last map, as a share of the bytes bound (x read once,
      y written once, at 3.35 TB/s);
  (b) representative EfficientNet-B0 / MobileNetV3-Large layers, b32, channels-last: rten_b200_conv2d_act (the
      activation in the epilogue, one launch) against rten_b200_conv2d followed by the standalone operator, and against
      torch (cuDNN conv + F.silu / F.hardswish, allow_tf32 matched to the f32 mode), in both f32 modes.
Each form is captured once as a CUDA graph after warm-up; forms alternate, the L2 cache is flushed before every timed
replay, and each of `--repeats` samples averages `--iters` replays timed with CUDA events (tools/depthwise_bench.py).

    python tools/activation_bench.py [--out DIR] [--repeats 7] [--iters 20]

Prints the card name and power limit with the numbers; with --out, writes one JSON line to DIR/activation_bench.json.
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

# (name, batch, C_in, C_out, H = W, k, stride, pad, groups, activation)
LAYERS = [
    ("EfficientNet-B0 expand 1x1 56x56 24->144 + SiLU", 32, 24, 144, 56, 1, 1, 0, 1, "silu"),
    ("EfficientNet-B0 depthwise k5 28x28x240 + SiLU", 32, 240, 240, 28, 5, 1, 2, 240, "silu"),
    ("MobileNetV3-L stem 3x3 s2 224x224 3->16 + HardSwish", 32, 3, 16, 224, 3, 2, 1, 1, "hard_swish"),
]


def _stats(ts):
    ts = sorted(ts)
    return dict(median_us=ts[len(ts) // 2], min_us=ts[0], max_us=ts[-1])


def bench_standalone(a, rt, ctx, stream, flush):
    import torch
    xn = np.random.default_rng(0).standard_normal((32, 96, 112, 112)).astype(np.float32) * 4
    x = ctx.to_device(xn, channels_last=True)
    out = ctx.empty(xn.shape, strides=x.strides)
    ops = {"sigmoid": rt.Sigmoid(), "silu": rt.Silu(), "hard_sigmoid": rt.HardSigmoid(), "hard_swish": rt.HardSwish()}
    from rten_b200.ops import _Args
    import ctypes as C

    def run_into(op):
        A = _Args(ctx)
        o = A.out(out)
        ctx.check(op._call(ctx, A.t(x), C.byref(o)))

    graphs = {}
    with torch.cuda.stream(stream):
        for op in ops.values():
            for _ in range(a.warmup):
                run_into(op)
        ctx.sync()
        for name, op in ops.items():
            ctx.graph_begin()
            run_into(op)
            graphs[name] = ctx.graph_end()
        times = _time_graphs(graphs, flush, a.repeats, a.iters)
    t_bytes = 2.0 * 4 * xn.size / HBM_BYTES_PER_S
    rows = []
    for name, ts in times.items():
        s = _stats(ts)
        s.update(op=name, bytes_bound_us=t_bytes * 1e6, bytes_share=t_bytes / (s["median_us"] * 1e-6))
        rows.append(s)
        print(f"{a.smi} standalone {name:12s} 32x112x112x96: {s['median_us']:8.1f} us [{s['min_us']:.1f}, "
              f"{s['max_us']:.1f}]  {100 * s['bytes_share']:.0f}% of the 3.35 TB/s bytes bound", flush=True)
    return rows


def bench_layers(a, rt, ctx_by_mode, stream, flush):
    import torch
    import torch.nn.functional as F
    rng = np.random.default_rng(1)
    rows = []
    for name, B, ci, co, h, k, s, p, g, act in LAYERS:
        oh = (h + 2 * p - k) // s + 1
        xn = rng.uniform(-1, 1, (B, ci, h, h)).astype(np.float32)
        wn = (rng.standard_normal((co, ci // g, k, k)) / np.sqrt(ci // g * k * k)).astype(np.float32)
        bn = rng.uniform(-0.1, 0.1, (co,)).astype(np.float32)
        code = rt.ACT_SILU if act == "silu" else rt.ACT_HARD_SWISH
        std = rt.Silu() if act == "silu" else rt.HardSwish()
        tfn = F.silu if act == "silu" else F.hardswish
        for mode, ctx in ctx_by_mode.items():
            torch.backends.cudnn.allow_tf32 = mode == "tf32"
            x, w, b = ctx.to_device(xn, channels_last=True), ctx.to_device(wn), ctx.to_device(bn)
            out = ctx.empty((B, co, oh, oh), strides=(oh * oh * co, 1, oh * co, co))
            fused_op = rt.Conv(groups=g, padding=(p, p, p, p), strides=(s, s), activation=code)
            plain_op = rt.Conv(groups=g, padding=(p, p, p, p), strides=(s, s))
            pk = plain_op.prepack(ctx, 1, w)
            xt = torch.from_numpy(xn).cuda().to(memory_format=torch.channels_last)
            wt, bt = torch.from_numpy(wn).cuda(), torch.from_numpy(bn).cuda()
            yt = [None]
            forms = {
                "fused": lambda: fused_op.run(ctx, x, w, b, packed_w=pk, out=out),
                "unfused": lambda: std.run(ctx, plain_op.run(ctx, x, w, b, packed_w=pk, out=out), in_place=True),
            }

            def torch_fwd():
                yt[0] = tfn(F.conv2d(xt, wt, bt, stride=s, padding=p, groups=g))

            graphs = {}
            with torch.cuda.stream(stream):
                for _ in range(a.warmup):
                    for f in forms.values():
                        f()
                    torch_fwd()
                ctx.sync()
                stream.synchronize()
                for fname, f in forms.items():
                    ctx.graph_begin()
                    f()
                    graphs[fname] = ctx.graph_end()
                tg = torch.cuda.CUDAGraph()
                with torch.cuda.graph(tg, stream=stream):
                    torch_fwd()
                graphs["torch"] = tg
                times = _time_graphs(graphs, flush, a.repeats, a.iters)
            ctx.sync()
            torch.cuda.synchronize()
            row = dict(layer=name, mode=mode)
            for fname, ts in times.items():
                row[fname] = _stats(ts)
            rows.append(row)
            fu, un, to = row["fused"], row["unfused"], row["torch"]
            print(f"{a.smi} {name:52s} {mode:6s}: fused {fu['median_us']:8.1f} us [{fu['min_us']:.1f}, {fu['max_us']:.1f}]  "
                  f"unfused {un['median_us']:8.1f} [{un['min_us']:.1f}, {un['max_us']:.1f}]  torch {to['median_us']:8.1f} "
                  f"[{to['min_us']:.1f}, {to['max_us']:.1f}]", flush=True)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    import torch
    import rten_b200 as rt
    name, power = _card()
    a.smi = f"[{power}]"
    print(f"card: {name}; power limit: {power}", flush=True)
    flush = torch.empty(64 * 1024 * 1024, dtype=torch.int32, device="cuda")  # 256 MB > 50 MB L2
    stream = torch.cuda.Stream()
    ctx_by_mode = {}
    for mode in ("tf32", "3xtf32"):
        c = rt.Context(0, stream=stream.cuda_stream)
        c.set_f32_mode(mode == "3xtf32")
        ctx_by_mode[mode] = c
    res = dict(card=name, power=power, time=time.strftime("%Y-%m-%d %H:%M:%S"),
               standalone=bench_standalone(a, rt, ctx_by_mode["tf32"], stream, flush),
               layers=bench_layers(a, rt, ctx_by_mode, stream, flush))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "activation_bench.json"), "w") as f:
            f.write(json.dumps(res) + "\n")


if __name__ == "__main__":
    main()
