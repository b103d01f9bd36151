"""Time the decoder operators and the in-place Concat:
  (a) Resize standalone at DeepLab (b8 x 256 x 33^2 -> 129^2, linear), FPN (b8 x 256 x 32^2 -> 64^2, nearest) and DPT
      (b1 x 256 x 96^2 -> 192^2, linear align_corners) sizes, NCHW and channels-last, against F.interpolate, as a share
      of the bytes bound (input read once + output written once at 3.35 TB/s);
  (b) Concat of two b8 x 64 x 256^2 maps: one rten_b200_concat launch against two rten_b200_copy calls and torch.cat,
      as a share of the bytes bound (every byte read once and written once);
  (c) the U-Net (b8, 64 base channels, 256^2) and the ASPP head of tests/decoder_models.py through the model API,
      channels-last, with the Concat elision on and off (RTEN_B200_NO_CONCAT_ELISION), in both f32 modes: time per run,
      launches, and the bytes the elided Concats would have moved.
(a) and (b) are captured as CUDA graphs after warm-up; forms alternate, the L2 cache is flushed before every timed replay
and each of `--repeats` samples averages `--iters` replays timed with CUDA events (tools/depthwise_bench.py).  (c) is
host-timed around a device synchronise, the two plans alternating.

    python tools/decoder_bench.py [--out DIR] [--repeats 7] [--iters 20]

Prints the card name and power limit with the numbers; with --out, writes one JSON line to DIR/decoder_bench.json.
Needs an H100; there is no fallback."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from depthwise_bench import HBM_BYTES_PER_S, _card, _time_graphs  # noqa: E402

# (name, input shape, output H = W, mode, coordinate transform)
RESIZES = [
    ("DeepLab b8x256x33^2 -> 129^2 linear", (8, 256, 33, 33), 129, "linear", "half_pixel"),
    ("FPN b8x256x32^2 -> 64^2 nearest", (8, 256, 32, 32), 64, "nearest", "asymmetric"),
    ("DPT b1x256x96^2 -> 192^2 linear align_corners", (1, 256, 96, 96), 192, "linear", "align_corners"),
]


def _stats(ts):
    ts = sorted(ts)
    return dict(median_us=ts[len(ts) // 2], min_us=ts[0], max_us=ts[-1])


def _capture_torch(fn, stream):
    import torch
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=stream):
        fn()
    return g


def bench_resize(a, rt, ctx, stream, flush):
    import torch
    import torch.nn.functional as F
    rows = []
    for name, shape, o, mode, cm in RESIZES:
        xn = np.random.default_rng(0).standard_normal(shape).astype(np.float32)
        B, C = shape[:2]
        for cl in (False, True):
            x = ctx.to_device(xn, channels_last=cl)
            out = ctx.empty((B, C, o, o), strides=(o * o * C, 1, o * C, C) if cl else None)
            op = rt.Resize(mode, cm, "floor")
            xt = torch.from_numpy(xn).cuda()
            if cl:
                xt = xt.to(memory_format=torch.channels_last)
            keep = [None]
            kw = dict(mode="bilinear", align_corners=cm == "align_corners") if mode == "linear" else dict(mode="nearest")

            def ours():
                op.run(ctx, x, sizes=[B, C, o, o], out=out)

            def torch_fwd():
                keep[0] = F.interpolate(xt, size=(o, o), **kw)

            with torch.cuda.stream(stream):
                for _ in range(a.warmup):
                    ours()
                    torch_fwd()
                ctx.sync()
                ctx.graph_begin()
                ours()
                graphs = {"rten_b200": ctx.graph_end()}
            graphs["torch"] = _capture_torch(torch_fwd, stream)
            with torch.cuda.stream(stream):
                times = _time_graphs(graphs, flush, a.repeats, a.iters)
            t_bytes = 4.0 * (xn.size + B * C * o * o) / HBM_BYTES_PER_S
            row = dict(case=name, layout="channels_last" if cl else "nchw", bytes_bound_us=t_bytes * 1e6)
            for form, ts in times.items():
                row[form] = _stats(ts)
            row["bytes_share"] = t_bytes / (row["rten_b200"]["median_us"] * 1e-6)
            rows.append(row)
            print(f"{a.smi} Resize {name} {row['layout']:13s}: {row['rten_b200']['median_us']:7.1f} us "
                  f"[{row['rten_b200']['min_us']:.1f}, {row['rten_b200']['max_us']:.1f}] {100 * row['bytes_share']:.0f}% of the bytes bound; "
                  f"F.interpolate {row['torch']['median_us']:.1f} us", flush=True)
    return rows


def bench_concat(a, rt, ctx, stream, flush):
    import torch
    shape = (8, 64, 256, 256)
    rng = np.random.default_rng(1)
    an, bn = rng.standard_normal(shape).astype(np.float32), rng.standard_normal(shape).astype(np.float32)
    rows = []
    for cl in (False, True):
        xa, xb = ctx.to_device(an, channels_last=cl), ctx.to_device(bn, channels_last=cl)
        out = ctx.to_device(np.zeros((8, 128, 256, 256), np.float32), channels_last=cl)
        halves = [out.view(shape, out.strides, k * 64 * out.strides[1]) for k in (0, 1)]
        ta, tb = torch.from_numpy(an).cuda(), torch.from_numpy(bn).cuda()
        if cl:
            ta, tb = ta.to(memory_format=torch.channels_last), tb.to(memory_format=torch.channels_last)
        keep = [None]
        cat = rt.Concat(1)
        forms = {"one_launch": lambda: cat.run(ctx, [xa, xb], out=out),
                 "two_copies": lambda: (halves[0].assign(xa), halves[1].assign(xb))}

        def torch_fwd():
            keep[0] = torch.cat([ta, tb], 1)

        graphs = {}
        with torch.cuda.stream(stream):
            for fn in forms.values():
                for _ in range(a.warmup):
                    fn()
            torch_fwd()
            ctx.sync()
            for name, fn in forms.items():
                ctx.graph_begin()
                fn()
                graphs[name] = ctx.graph_end()
        graphs["torch_cat"] = _capture_torch(torch_fwd, stream)
        with torch.cuda.stream(stream):
            times = _time_graphs(graphs, flush, a.repeats, a.iters)
        t_bytes = 2.0 * 4 * 2 * an.size / HBM_BYTES_PER_S
        row = dict(layout="channels_last" if cl else "nchw", bytes_bound_us=t_bytes * 1e6)
        for form, ts in times.items():
            row[form] = _stats(ts)
        row["bytes_share"] = t_bytes / (row["one_launch"]["median_us"] * 1e-6)
        rows.append(row)
        print(f"{a.smi} Concat 2 x b8x64x256^2 {row['layout']:13s}: one launch {row['one_launch']['median_us']:.1f} us "
              f"({100 * row['bytes_share']:.0f}% of the bytes bound), two copies {row['two_copies']['median_us']:.1f} us, "
              f"torch.cat {row['torch_cat']['median_us']:.1f} us", flush=True)
    return rows


def bench_models(a, rt):
    import decoder_models as D
    from rten_b200.model import Model
    rows = []
    cases = [("U-Net b8 c64 256^2", D.unet(B=8, C=64, H=256, W_=256), 4.0 * 2 * 8 * (128 * 256 * 256 + 256 * 128 * 128)),
             ("ASPP head b8 c256 33^2", D.aspp(B=8, C=256, H=33, W_=33), 4.0 * 2 * 8 * 5 * 256 * 33 * 33)]
    for name, (data, _, shape, n_concat), concat_bytes in cases:
        xn = np.random.default_rng(2).standard_normal(shape).astype(np.float32)
        for tf32 in (True, False):
            plans = {}
            for form in ("elided", "copied"):
                if form == "copied":
                    os.environ["RTEN_B200_NO_CONCAT_ELISION"] = "1"
                try:
                    ctx = rt.Context(0)
                    ctx.set_f32_mode(not tf32)
                    plans[form] = (ctx, Model(ctx, data), ctx.to_device(xn, channels_last=True))
                finally:
                    os.environ.pop("RTEN_B200_NO_CONCAT_ELISION", None)
            launches, outs = {}, {}
            for form, (ctx, m, x) in plans.items():
                for _ in range(a.warmup):
                    m.run({"x": x})
                ctx.sync()
                n0 = ctx.launches
                outs[form] = m.run({"x": x})[0].numpy()
                launches[form] = ctx.launches - n0
            times = {f: [] for f in plans}
            for _ in range(a.repeats):
                for form, (ctx, m, x) in plans.items():
                    ctx.sync()
                    t0 = time.perf_counter()
                    for _ in range(a.iters):
                        m.run({"x": x})
                    ctx.sync()
                    times[form].append((time.perf_counter() - t0) / a.iters * 1e6)
            row = dict(model=name, mode="tf32" if tf32 else "tf32x3", launches=launches, concat_nodes=n_concat,
                       concat_bytes=concat_bytes, identical=bool(np.array_equal(outs["elided"], outs["copied"])))
            for form, ts in times.items():
                row[form] = _stats(ts)
            rows.append(row)
            print(f"{a.smi} {name} {row['mode']:6s}: elided {row['elided']['median_us'] / 1e3:.3f} ms ({launches['elided']} launches), "
                  f"copied {row['copied']['median_us'] / 1e3:.3f} ms ({launches['copied']} launches), Concat traffic avoided "
                  f"{concat_bytes / 1e6:.0f} MB, identical bits: {row['identical']}", flush=True)
    return rows


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--out", default=None, help="directory for decoder_bench.json")
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("decoder_bench: no CUDA device; this benchmark measures the H100 kernels and has no fallback")
    import rten_b200 as rt
    card, a.smi = _card()
    stream = torch.cuda.Stream()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")  # larger than the 50 MB L2
    ctx = rt.Context(0, stream=stream.cuda_stream)
    resize = bench_resize(a, rt, ctx, stream, flush)
    concat = bench_concat(a, rt, ctx, stream, flush)
    models = bench_models(a, rt)
    line = json.dumps(dict(tool="decoder_bench", card=card, nvidia_smi=a.smi, repeats=a.repeats, iters=a.iters, resize=resize,
                           concat=concat, models=models))
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "decoder_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
