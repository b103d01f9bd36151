"""Time depthwise convolutions against cuDNN, and a whole MobileNetV2 through the ONNX executor:
  (a) rten_b200_conv2d / rten_b200_conv_integer_ex with groups = channels: the direct depthwise kernel, one launch;
  (b) torch.nn.functional.conv2d(groups = C) (cuDNN) on the same channels-last tensors.  The f32 depthwise kernel does
      not use tensor cores, so the mode does not change it; cuDNN runs with allow_tf32 = True.
Each form is captured once as a CUDA graph after warm-up; the two forms alternate, the L2 cache is flushed before every
timed replay, and each of `--repeats` samples averages `--iters` replays timed with CUDA events.

    python tools/depthwise_bench.py [--out DIR] [--repeats 7] [--iters 20] [--model-batch 32]

Per layer: median us and [min, max] per form, the launch count, and the share of the roofline the median reaches.  The
roofline is the larger of two bounds: the bytes bound (x read once, out written once, at 3.35 TB/s) and the FP32-issue
bound (2 * kh * kw instructions per output -- the multiply and the add are separate roundings and cannot fuse -- on
132 SMs x 128 lanes at 1.98 GHz).

Whole model: MobileNetV2 (torchvision layout, batch norm folded into seeded conv weights, ReLU6 as Clip(0, 6)) built
with tests/onnx_writer.py and run through rten_b200_model_* on a channels-last device input, in both f32 modes, against
a torch functional forward with the same weights (cuDNN, channels-last, allow_tf32 matched to the mode); img/s of each.

Prints the card name and power limit with the numbers; with --out, writes one JSON line to DIR/depthwise_bench.json.
Needs an H100; there is no fallback."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

HBM_BYTES_PER_S = 3.35e12
FP32_ISSUE_PER_S = 132 * 128 * 1.98e9
# (name, batch, C, H = W, k, stride, pad, dilation, int8)
LAYERS = [
    ("MobileNetV2 112x112x32 k3 s1", 32, 32, 112, 3, 1, 1, 1, False),
    ("MobileNetV2 112x112x96 k3 s2", 32, 96, 112, 3, 2, 1, 1, False),
    ("MobileNetV2 56x56x144 k3 s1", 32, 144, 56, 3, 1, 1, 1, False),
    ("MobileNetV2 7x7x960 k3 s1", 32, 960, 7, 3, 1, 1, 1, False),
    ("EfficientNet-B0 28x28x240 k5", 32, 240, 28, 5, 1, 2, 1, False),
    ("ConvNeXt-T 56x56x96 k7 p3", 32, 96, 56, 7, 1, 3, 1, False),
    ("ConvNeXt-T 14x14x384 k7 p3", 32, 384, 14, 7, 1, 3, 1, False),
    ("DeepLabV3-MNv3 b8 33x33x960 k5 d2", 8, 960, 33, 5, 1, 4, 2, False),
    ("int8 MobileNetV2 112x112x96 s2", 32, 96, 112, 3, 2, 1, 1, True),
]


def _card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


def _time_graphs(graphs, flush, repeats, iters):
    import torch
    times = {f: [] for f in graphs}
    for _ in range(repeats):
        for form, g in graphs.items():
            tot = 0.0
            for _ in range(iters):
                flush.zero_()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                (g.launch if hasattr(g, "launch") else g.replay)()
                e1.record()
                e1.synchronize()
                tot += e0.elapsed_time(e1) * 1e3
            times[form].append(tot / iters)
    return times


def bench_layers(a, rt, ctx, stream, flush, smi):
    import torch
    import torch.nn.functional as F
    torch.backends.cudnn.allow_tf32 = True
    rng = np.random.default_rng(0)
    results = []
    for name, B, C, h, k, s, p, d, q8 in LAYERS:
        oh = (h + 2 * p - d * (k - 1) - 1) // s + 1
        if q8:
            xn = rng.integers(0, 256, (B, C, h, h)).astype(np.uint8)
            wn = rng.integers(-128, 128, (C, 1, k, k)).astype(np.int8)
        else:
            xn = rng.uniform(-1, 1, (B, C, h, h)).astype(np.float32)
            wn = rng.uniform(-1, 1, (C, 1, k, k)).astype(np.float32)
        bn = rng.uniform(-0.1, 0.1, (C,)).astype(np.float32)
        x = ctx.to_device(xn, channels_last=True)
        w, b = ctx.to_device(wn), ctx.to_device(bn)
        out = ctx.empty((B, C, oh, oh), strides=(oh * oh * C, 1, oh * C, C))
        if q8:
            xz, sc = ctx.to_device(np.array(121, np.uint8)), ctx.to_device(np.array(0.01, np.float32))
            op = rt.ConvIntegerToFloat(groups=C, padding=(p, p, p, p), strides=(s, s), dilations=(d, d))
            pk = None

            def ours():
                op.run(ctx, x, w, xz, None, sc, bias=b, out=out)
            # cuDNN has no u8 x i8 depthwise convolution: it runs the f32 convolution of the dequantised values
            xt = ((torch.from_numpy(xn).cuda().float() - 121.0)).to(memory_format=torch.channels_last)
            wt = torch.from_numpy(wn).cuda().float()
        else:
            op = rt.Conv(groups=C, padding=(p, p, p, p), strides=(s, s), dilations=(d, d))
            pk = op.prepack(ctx, 1, w)

            def ours():
                op.run(ctx, x, w, b, packed_w=pk, out=out)
            xt = torch.from_numpy(xn).cuda().to(memory_format=torch.channels_last)
            wt = torch.from_numpy(wn).cuda()
        bt = torch.from_numpy(bn).cuda()
        yt = [None]

        def cudnn():
            yt[0] = F.conv2d(xt, wt, None if q8 else bt, stride=s, padding=p, dilation=d, groups=C)

        graphs = {}
        with torch.cuda.stream(stream):
            for _ in range(a.warmup):
                ours()
                cudnn()
            ctx.sync()
            stream.synchronize()
            ctx.graph_begin()
            ours()
            graphs["rten_b200"] = ctx.graph_end()
            tg = torch.cuda.CUDAGraph()
            with torch.cuda.graph(tg, stream=stream):
                cudnn()
            graphs["cudnn"] = tg
            launches0 = ctx.launches
            ours()
            ctx.sync()
            launches = ctx.launches - launches0
            times = _time_graphs(graphs, flush, a.repeats, a.iters)
        ctx.sync()
        torch.cuda.synchronize()
        ours_y = out.numpy().astype(np.float64)
        ref_y = yt[0].float().cpu().numpy().astype(np.float64)
        if q8:
            ref_y = ref_y * np.float64(np.float32(0.01)) + bn.reshape(1, -1, 1, 1)
        diff = float(np.abs(ours_y - ref_y).max() / np.abs(ref_y).max())
        n_out = B * C * oh * oh
        nbytes = float(xn.itemsize * xn.size + 4 * n_out)
        t_bytes = nbytes / HBM_BYTES_PER_S
        t_issue = 0.0 if q8 else 2.0 * k * k * n_out / FP32_ISSUE_PER_S
        bound = "FP32 issue" if t_issue > t_bytes else "HBM"
        row = dict(layer=name, batch=B, channels=C, size=h, k=k, stride=s, pad=p, dilation=d, int8=q8, bytes=nbytes,
                   hbm_bound_us=t_bytes * 1e6, fp32_issue_bound_us=t_issue * 1e6, bound=bound, launches=launches,
                   rel_diff_vs_cudnn=diff)
        for form, ts in times.items():
            ts = sorted(ts)
            med = ts[len(ts) // 2]
            row[form] = dict(median_us=med, min_us=ts[0], max_us=ts[-1], roofline_share=max(t_bytes, t_issue) / (med * 1e-6))
        results.append(row)
        o, c = row["rten_b200"], row["cudnn"]
        print(f"{smi} {name:34s}: rten_b200 {o['median_us']:8.1f} us [{o['min_us']:.1f}, {o['max_us']:.1f}] "
              f"({launches} launch, {100 * o['roofline_share']:.0f}% of {bound} roofline)  cudnn {c['median_us']:8.1f} us "
              f"[{c['min_us']:.1f}, {c['max_us']:.1f}] ({100 * c['roofline_share']:.0f}%)  {nbytes / 1e6:.1f} MB  "
              f"rel diff {diff:.1e}", flush=True)
    return results


# ---- MobileNetV2 (torchvision layout: inverted residual settings t, c, n, s) ----------------------------------------
SETTINGS = [(1, 16, 1, 1), (6, 24, 2, 2), (6, 32, 3, 2), (6, 64, 4, 2), (6, 96, 3, 1), (6, 160, 3, 2), (6, 320, 1, 1)]


def mobilenet_v2_layers(seed=0):
    """[(kind, params)] with conv = (w, b, stride, groups, relu6) and the block structure as ("block", [convs], residual)"""
    rng = np.random.default_rng(seed)

    def conv(cin, cout, k, s, g, relu6):
        fan = cin // g * k * k
        w = (rng.standard_normal((cout, cin // g, k, k)) * np.sqrt(2.0 / fan)).astype(np.float32)
        b = rng.uniform(-0.05, 0.05, cout).astype(np.float32)
        return dict(w=w, b=b, s=s, g=g, k=k, relu6=relu6)

    layers = [("conv", conv(3, 32, 3, 2, 1, True))]
    cin = 32
    for t, c, n, s in SETTINGS:
        for i in range(n):
            hid = cin * t
            convs = []
            if t != 1:
                convs.append(conv(cin, hid, 1, 1, 1, True))
            convs.append(conv(hid, hid, 3, s if i == 0 else 1, hid, True))
            convs.append(conv(hid, c, 1, 1, 1, False))
            layers.append(("block", convs, (s if i == 0 else 1) == 1 and cin == c))
            cin = c
    layers.append(("conv", conv(cin, 1280, 1, 1, 1, True)))
    fc_w = (rng.standard_normal((1000, 1280)) * 0.02).astype(np.float32)
    fc_b = np.zeros(1000, np.float32)
    return layers, fc_w, fc_b


def mobilenet_v2_onnx(W, layers, fc_w, fc_b, batch):
    nodes, inits = [], [W.tensor("zero", np.array(0.0, np.float32)), W.tensor("six", np.array(6.0, np.float32))]
    n = [0]

    def conv(x, c):
        i = n[0]
        n[0] += 1
        inits.extend([W.tensor(f"w{i}", c["w"]), W.tensor(f"b{i}", c["b"])])
        p = c["k"] // 2
        nodes.append(W.node("Conv", [x, f"w{i}", f"b{i}"], [f"c{i}"], kernel_shape=[c["k"], c["k"]], pads=[p, p, p, p],
                            strides=[c["s"], c["s"]], group=c["g"]))
        if not c["relu6"]:
            return f"c{i}"
        nodes.append(W.node("Clip", [f"c{i}", "zero", "six"], [f"r{i}"]))
        return f"r{i}"

    x = "x"
    for layer in layers:
        if layer[0] == "conv":
            x = conv(x, layer[1])
        else:
            y = x
            for c in layer[1]:
                y = conv(y, c)
            if layer[2]:
                nodes.append(W.node("Add", [x, y], [f"{y}_add"]))
                y = f"{y}_add"
            x = y
    nodes.append(W.node("GlobalAveragePool", [x], ["gap"]))
    nodes.append(W.node("Flatten", ["gap"], ["flat"]))
    inits.extend([W.tensor("fc_w", fc_w), W.tensor("fc_b", fc_b)])
    nodes.append(W.node("Gemm", ["flat", "fc_w", "fc_b"], ["logits"], transB=1))
    return W.model(nodes, inits, [W.value_info("x", 1, (batch, 3, 224, 224))], [W.value_info("logits", 1, (batch, 1000))])


def mobilenet_v2_torch(x, layers, fc_w, fc_b):
    import torch
    import torch.nn.functional as F
    dev = {}

    def conv(t, c):
        key = id(c)
        if key not in dev:
            dev[key] = (torch.from_numpy(c["w"]).cuda(), torch.from_numpy(c["b"]).cuda())
        w, b = dev[key]
        y = F.conv2d(t, w, b, stride=c["s"], padding=c["k"] // 2, groups=c["g"])
        return torch.clamp(y, 0.0, 6.0) if c["relu6"] else y

    for layer in layers:
        if layer[0] == "conv":
            x = conv(x, layer[1])
        else:
            y = x
            for c in layer[1]:
                y = conv(y, c)
            x = x + y if layer[2] else y
    x = F.adaptive_avg_pool2d(x, 1).flatten(1)
    return F.linear(x, fc_w, fc_b)


def bench_model(a, rt, smi):
    import torch
    import onnx_writer
    from rten_b200.model import Model
    B = a.model_batch
    layers, fc_w, fc_b = mobilenet_v2_layers()
    model_bytes = mobilenet_v2_onnx(onnx_writer, layers, fc_w, fc_b, B)
    xn = np.random.default_rng(1).uniform(-1, 1, (B, 3, 224, 224)).astype(np.float32)
    xt = torch.from_numpy(xn).cuda().to(memory_format=torch.channels_last)
    fw, fb = torch.from_numpy(fc_w).cuda(), torch.from_numpy(fc_b).cuda()
    rows = []
    for tf32 in (True, False):
        mode = "tf32" if tf32 else "tf32x3"
        torch.backends.cudnn.allow_tf32 = tf32
        torch.backends.cuda.matmul.allow_tf32 = tf32
        ctx = rt.Context(0)
        ctx.set_f32_mode(not tf32)
        m = Model(ctx, model_bytes)
        x = ctx.to_device(xn, channels_last=True)

        def ours():
            return m.run({"x": x}, ["logits"])[0]

        def torch_fwd():
            with torch.no_grad():
                return mobilenet_v2_torch(xt, layers, fw, fb)

        for _ in range(a.warmup):
            ours()
            torch_fwd()
        ctx.sync()
        torch.cuda.synchronize()
        n0 = ctx.launches
        y = ours().numpy()
        launches = ctx.launches - n0
        yt = torch_fwd().float().cpu().numpy()
        diff = float(np.abs(y.astype(np.float64) - yt).max() / np.abs(yt).max())
        times = {"rten_b200": [], "torch": []}
        for _ in range(a.repeats):
            for form, fn in (("rten_b200", ours), ("torch", torch_fwd)):
                ctx.sync()
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for _ in range(a.iters):
                    fn()
                ctx.sync()
                torch.cuda.synchronize()
                times[form].append((time.perf_counter() - t0) / a.iters)
        row = dict(model="MobileNetV2", batch=B, mode=mode, launches=launches, rel_diff_vs_torch=diff)
        for form, ts in times.items():
            ts = sorted(ts)
            med = ts[len(ts) // 2]
            row[form] = dict(median_ms=med * 1e3, min_ms=ts[0] * 1e3, max_ms=ts[-1] * 1e3, img_per_s=B / med)
        rows.append(row)
        print(f"{smi} MobileNetV2 b{B} {mode:6s}: rten_b200 {row['rten_b200']['median_ms']:.2f} ms "
              f"({row['rten_b200']['img_per_s']:.0f} img/s, {launches} launches)  torch {row['torch']['median_ms']:.2f} ms "
              f"({row['torch']['img_per_s']:.0f} img/s)  rel diff {diff:.1e}", flush=True)
    return rows


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--out", default=None, help="directory for depthwise_bench.json")
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--model-batch", type=int, default=32)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("depthwise_bench: no CUDA device; this benchmark measures the H100 kernels and has no fallback")
    import rten_b200 as rt
    card, smi = _card()
    stream = torch.cuda.Stream()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")  # larger than the 50 MB L2
    ctx = rt.Context(0, stream=stream.cuda_stream)
    layers = bench_layers(a, rt, ctx, stream, flush, smi)
    model = bench_model(a, rt, smi)
    line = json.dumps(dict(tool="depthwise_bench", card=card, nvidia_smi=smi, repeats=a.repeats, iters=a.iters,
                           layers=layers, model=model))
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "depthwise_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
