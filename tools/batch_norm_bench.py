"""Time BatchNormalization (rten_b200_batch_norm, + Relu) and the load-time fold of a Conv's BatchNormalization.

  standalone  rten_b200_batch_norm + Relu in one pass against torch F.batch_norm + F.relu on a tensor in the same memory
              format, at DenseNet-121 b32's maps (56x56x256, 28x28x512, 14x14x1024, 7x7x1024; NCHW and channels-last)
              and a BatchNorm1d head (32 x 4096); the bytes bound is x read once and y written once at 3.35 TB/s
  fold        ResNet-50 b32 layers through the C ABI, channels-last: Conv, then BatchNormalization + Relu as its own pass,
              against the Conv with the folded weights and Relu in its epilogue (what the executor loads)
  model       DenseNet-121 b32 channels-last through the executor (tests/test_gpu_batch_norm.py's graph, BatchNormalization
              unfolded in the file), single-pass TF32: images/s and launches per run, against torch's float32
              channels-last forward of the same weights with TF32 allowed; host time of `--iters` runs between device
              synchronisations (the executor allocates during a run, so it is not captured as a graph)

Each standalone and fold form is captured once as a CUDA graph after warm-up; forms alternate, the L2 cache is flushed before every timed
replay, and each of `--repeats` samples averages `--iters` replays timed with CUDA events (tools/depthwise_bench.py).

    python tools/batch_norm_bench.py [--out DIR] [--repeats 5] [--iters 10] [--skip-model]

Prints the card name and power limit with the numbers; with --out, writes one JSON line to DIR/batch_norm_bench.json.
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

# (name, shape)
STANDALONE = [("DenseNet-121 b32 56x56x256", (32, 256, 56, 56)), ("DenseNet-121 b32 28x28x512", (32, 512, 28, 28)),
              ("DenseNet-121 b32 14x14x1024", (32, 1024, 14, 14)), ("DenseNet-121 b32 7x7x1024", (32, 1024, 7, 7)),
              ("BatchNorm1d 32 x 4096", (32, 4096))]
# (name, B, C_in, C_out, H, k)
FOLD = [("ResNet-50 b32 56x56 1x1 64->256", 32, 64, 256, 56, 1), ("ResNet-50 b32 56x56 3x3 64->64", 32, 64, 64, 56, 3),
        ("ResNet-50 b32 14x14 3x3 256->256", 32, 256, 256, 14, 3)]


def _stats(ts):
    ts = sorted(ts)
    return dict(median_us=ts[len(ts) // 2], min_us=ts[0], max_us=ts[-1])


def _capture(rt, ctx, stream, forms, torch_forms, flush, a):
    import torch
    graphs = {}
    with torch.cuda.stream(stream):
        for _ in range(a.warmup):
            for f in list(forms.values()) + list(torch_forms.values()):
                f()
        ctx.sync()
        stream.synchronize()
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
    return {f: _stats(ts) for f, ts in times.items()}


def bench_standalone(rt, ctx, stream, flush, a, power):
    import torch
    import torch.nn.functional as F
    rng = np.random.default_rng(0)
    rows = []
    for name, shape in STANDALONE:
        C = shape[1]
        xn = rng.standard_normal(shape).astype(np.float32)
        pn = [rng.uniform(0.5, 1.5, C), rng.uniform(-0.5, 0.5, C), rng.uniform(-0.2, 0.2, C), rng.uniform(0.5, 2, C)]
        pn = [v.astype(np.float32) for v in pn]
        pd = [ctx.to_device(v) for v in pn]
        pt = [torch.from_numpy(v).cuda() for v in pn]
        op = rt.BatchNormalization(1e-5, rt.ACT_RELU)
        keep, forms, torch_forms = [], {}, {}
        for layout in (("cl", "nchw") if len(shape) == 4 else ("nchw",)):
            x = ctx.to_device(xn, channels_last=layout == "cl")
            xt = torch.from_numpy(xn).cuda()
            if layout == "cl":
                xt = xt.contiguous(memory_format=torch.channels_last)
            forms[f"rten {layout}"] = lambda x=x: keep.append(op.run(ctx, x, *pd))
            torch_forms[f"torch {layout}"] = lambda xt=xt: keep.append(F.relu(F.batch_norm(xt, pt[2], pt[3], pt[0], pt[1], False, 0.0, 1e-5)))
        times = _capture(rt, ctx, stream, forms, torch_forms, flush, a)
        keep.clear()
        t_b = 8 * xn.size / HBM_BYTES_PER_S
        row = dict(name=name, dims=list(shape), bytes_bound_us=t_b * 1e6)
        for fname, st in times.items():
            st.update(bytes_share=t_b / (st["median_us"] * 1e-6))
            row[fname] = st
            print(f"[{power}] {name:30s} {fname:11s} {st['median_us']:8.1f} us [{st['min_us']:.1f}, {st['max_us']:.1f}]  "
                  f"{100 * st['bytes_share']:3.0f}% of the bytes bound ({t_b * 1e6:.1f} us)", flush=True)
        rows.append(row)
    return rows


def bench_fold(rt, ctx, stream, flush, a, power):
    import batch_norm_ref as ref
    rng = np.random.default_rng(1)
    rows = []
    for name, B, cin, cout, H, k in FOLD:
        xn = rng.standard_normal((B, cin, H, H)).astype(np.float32)
        w = (rng.standard_normal((cout, cin, k, k)) / np.sqrt(cin * k * k)).astype(np.float32)
        b = (0.1 * rng.standard_normal(cout)).astype(np.float32)
        pn = [v.astype(np.float32) for v in (rng.uniform(0.5, 1.5, cout), rng.uniform(-0.5, 0.5, cout),
                                             rng.uniform(-0.2, 0.2, cout), rng.uniform(0.5, 2, cout))]
        wf, bf = ref.fold_conv(w, b, *pn, 1e-5)
        x = ctx.to_device(xn, channels_last=True)
        wd, bd, wfd, bfd = (ctx.to_device(v) for v in (w, b, wf, bf))
        pd = [ctx.to_device(v) for v in pn]
        pad = (k // 2,) * 4
        conv, conv_act = rt.Conv(padding=pad), rt.Conv(padding=pad, activation=rt.ACT_RELU)
        pw, pwf = conv.prepack(ctx, 1, wd), conv_act.prepack(ctx, 1, wfd)
        bn = rt.BatchNormalization(1e-5, rt.ACT_RELU)
        keep = []

        def unfolded():
            y = conv.run(ctx, x, wd, bd, packed_w=pw)
            keep.append(bn.run(ctx, y, *pd, out=y))

        forms = {"conv + batch_norm": unfolded, "folded conv": lambda: keep.append(conv_act.run(ctx, x, wfd, bfd, packed_w=pwf))}
        launches = {}
        for fname, f in forms.items():
            ctx.sync()
            n0 = ctx.launches
            f()
            ctx.sync()
            launches[fname] = ctx.launches - n0
        times = _capture(rt, ctx, stream, forms, {}, flush, a)
        keep.clear()
        row = dict(name=name, launches=launches)
        for fname, st in times.items():
            row[fname] = st
            print(f"[{power}] {name:34s} {fname:18s} {st['median_us']:8.1f} us [{st['min_us']:.1f}, {st['max_us']:.1f}]  "
                  f"{launches[fname]} launches", flush=True)
        row["saved_us"] = times["conv + batch_norm"]["median_us"] - times["folded conv"]["median_us"]
        rows.append(row)
    return rows


def bench_model(rt, a, power):
    """wall time of whole runs between device synchronisations (the executor allocates per run, so no graph capture)"""
    import torch
    import test_gpu_batch_norm as tb
    from rten_b200.model import Model
    torch.backends.cudnn.allow_tf32 = True
    torch.backends.cuda.matmul.allow_tf32 = True
    B = 32
    ctx = rt.Context(0)
    ctx.set_f32_mode(False)  # single-pass TF32, as torch with TF32 allowed
    data, params = tb.densenet121()
    m = Model(ctx, data)
    xn = np.random.default_rng(2).standard_normal((B, 3, 224, 224)).astype(np.float32)
    x = ctx.to_device(xn, channels_last=True)
    xt = torch.from_numpy(xn).cuda().contiguous(memory_format=torch.channels_last)
    # the weights on the device in channels-last once, as the executor's are: the timed forward launches kernels only
    P = tb.densenet121_torch_params(params, dtype=torch.float32, device="cuda", channels_last=True)

    def ours():
        return m.run({"x": x})[0]

    def torch_fwd():
        with torch.no_grad():
            return tb.densenet121_torch(P, xt)

    for _ in range(a.warmup):
        ours()
        torch_fwd()
    ctx.sync()
    torch.cuda.synchronize()
    n0 = ctx.launches
    y = ours().numpy()
    launches = ctx.launches - n0
    yt = torch_fwd().cpu().numpy()
    diff = float(np.abs(y.astype(np.float64) - yt).max() / np.abs(yt).max())
    times = {"rten executor": [], "torch channels-last": []}
    for _ in range(a.repeats):
        for form, fn in (("rten executor", ours), ("torch channels-last", torch_fwd)):
            ctx.sync()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(a.iters):
                fn()
            ctx.sync()
            torch.cuda.synchronize()
            times[form].append((time.perf_counter() - t0) / a.iters * 1e6)
    row = dict(name="DenseNet-121 b32 channels-last TF32", launches=launches, nodes=len(m.node_ops),
               batch_norm_nodes=m.node_ops.count("BatchNormalization"), rel_diff_vs_torch=diff)
    for fname, ts in times.items():
        st = _stats(ts)
        st.update(images_per_s=B / (st["median_us"] * 1e-6))
        row[fname] = st
        print(f"[{power}] {row['name']} {fname:20s} {st['median_us'] / 1e3:8.2f} ms [{st['min_us'] / 1e3:.2f}, "
              f"{st['max_us'] / 1e3:.2f}]  {st['images_per_s']:7.0f} img/s", flush=True)
    print(f"[{power}] executor: {launches} launches per run, {len(m.node_ops)} nodes, {row['batch_norm_nodes']} "
          f"BatchNormalization nodes left standalone; logits within {diff:.1e} of torch's largest", flush=True)
    return [row]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--skip-model", action="store_true")
    a = ap.parse_args()
    import torch
    import rten_b200 as rt
    name, power = _card()
    print(f"card: {name}; power limit: {power}", flush=True)
    flush = torch.empty(64 * 1024 * 1024, dtype=torch.int32, device="cuda")  # 256 MB > 50 MB L2
    stream = torch.cuda.Stream()
    ctx = rt.Context(0, stream=stream.cuda_stream)
    ctx.set_f32_mode(False)
    res = dict(card=name, power=power, time=time.strftime("%Y-%m-%d %H:%M:%S"))
    res["standalone"] = bench_standalone(rt, ctx, stream, flush, a, power)
    res["fold"] = bench_fold(rt, ctx, stream, flush, a, power)
    res["model"] = "not measured" if a.skip_model else bench_model(rt, a, power)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "batch_norm_bench.json"), "w") as f:
            f.write(json.dumps(res) + "\n")


if __name__ == "__main__":
    main()
