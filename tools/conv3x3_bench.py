"""Time ResNet-50's 3x3 convolutions at batch 32 in single-pass TF32, as ResNet50Runner runs them: channels-last
activations, prepacked weights, bias + Relu.

    python tools/conv3x3_bench.py --out DIR [--repeats 7] [--iters 20]

For each of the seven distinct 3x3 layer shapes (four stride 1, three stride 2):
  * autotuned: a fresh context with autotuning on runs the layer once; the saved plans file names the winning plan
    (`-1 bn T`: the halo-reuse kernel, else `bn splitk nbuf` of the implicit-GEMM kernel);
  * stride 1 only: every halo unit shape `-1 bn T` (bn in 32, 64, 128; T in 1, 2) pinned through a plans file in a
    context with autotuning off.  A shape the kernel rejects is reported as such (the launch was re-planned).
Each variant is captured as a CUDA graph and timed as `--repeats` samples of `--iters` replays with CUDA events, the L2
cache flushed before every replay.  Reports median us [min, max], TFLOP/s, its share of the 495 TFLOP/s dense TF32 of
the H100 SXM data sheet and of cuBLAS's 8192^3 TF32 GEMM rate measured in the same run, and the sums weighted by how
many times each shape occurs in the network.  Prints the card name, power limit and max SM clock with the numbers and
writes one JSON line to DIR/conv3x3_bench.json.  Needs an H100; there is no fallback."""
import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

TF32_DENSE = 495e12
# (name, input size, channels, stride, occurrences in ResNet-50): C = N for every 3x3 layer
LAYERS = [("layer1 56x56", 56, 64, 1, 3), ("layer2 28x28", 28, 128, 1, 3), ("layer3 14x14", 14, 256, 1, 5),
          ("layer4 7x7", 7, 512, 1, 2), ("layer2.0 s2", 56, 128, 2, 1), ("layer3.0 s2", 28, 256, 2, 1),
          ("layer4.0 s2", 14, 512, 2, 1)]
HALO_SHAPES = [(bn, T) for T in (1, 2) for bn in (32, 64, 128)]


def _card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def _cublas_tf32(torch, n=8192):
    torch.backends.cuda.matmul.allow_tf32 = True
    a, b = torch.randn(n, n, device="cuda"), torch.randn(n, n, device="cuda")
    for _ in range(3):
        a @ b
    torch.cuda.synchronize()
    best = 1e9
    for _ in range(10):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        a @ b
        e.record()
        torch.cuda.synchronize()
        best = min(best, s.elapsed_time(e))
    return 2.0 * n ** 3 / (best * 1e-3)


def _plans(path):
    """{key: entry} of a plans file (`<key> | <three integers>` per line)."""
    out = {}
    if os.path.exists(path):
        for line in open(path).read().splitlines():
            if "|" in line:
                k, v = line.split("|", 1)
                out[k.strip()] = tuple(int(x) for x in v.split())
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--out", required=True, help="directory for conv3x3_bench.json")
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("conv3x3_bench: no CUDA device; this benchmark measures the H100 kernels and has no fallback")
    import rten_b200 as rt
    smi = _card()
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")  # larger than the 50 MB L2
    cublas = _cublas_tf32(torch)
    tmp = tempfile.mkdtemp(prefix="conv3x3_bench_")
    gen = torch.Generator(device="cuda").manual_seed(0)
    B = a.batch

    def timed(ctx, fn):
        for _ in range(a.warmup):
            fn()
        ctx.sync()
        ctx.graph_begin()
        fn()
        g = ctx.graph_end()
        samples = []
        for _ in range(a.repeats):
            tot = 0.0
            for _ in range(a.iters):
                flush.zero_()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                g.launch()
                e1.record(stream)
                e1.synchronize()
                tot += e0.elapsed_time(e1) * 1e3
            samples.append(tot / a.iters)
        del g
        samples.sort()
        return dict(median_us=samples[len(samples) // 2], min_us=samples[0], max_us=samples[-1])

    results = []
    for name, hw, c, s, count in LAYERS:
        oh = (hw - 1) // s + 1
        x = (torch.rand((B, c, hw, hw), device="cuda", generator=gen) * 2 - 1).contiguous(memory_format=torch.channels_last)
        w = (torch.rand((c, c, 3, 3), device="cuda", generator=gen) * 2 - 1) / (9 * c) ** 0.5
        bias = torch.rand((c,), device="cuda", generator=gen) * 0.2 - 0.1
        out = torch.empty((B, c, oh, oh), device="cuda").contiguous(memory_format=torch.channels_last)
        flops = 2.0 * B * oh * oh * c * c * 9

        def layer_ctx(autotune, plans=None):
            ctx = rt.Context(0, stream=stream.cuda_stream)
            ctx.set_f32_mode(False)
            ctx.set_autotune(autotune)
            if plans:
                ctx.load_plans(plans)
            op = rt.Conv(1, (1, 1), (1, 1, 1, 1), (s, s), activation=rt.ACT_RELU)
            T = lambda t: rt.from_torch(ctx, t)
            xt, wt, bt, ot = T(x), T(w), T(bias), T(out)
            pk = op.prepack(ctx, 1, wt)
            return ctx, lambda: op.run(ctx, xt, wt, bt, packed_w=pk, out=ot)

        # autotuned on a fresh context: the plans file records the winner
        ctx, fn = layer_ctx(True)
        fn()
        ctx.sync()
        tuned_path = os.path.join(tmp, "tuned.plans")
        ctx.save_plans(tuned_path)
        (key, plan), = _plans(tuned_path).items()
        row = dict(layer=name, hw=hw, c=c, stride=s, count=count, flops=flops, key=key,
                   plan=" ".join(map(str, plan)), kernel="halo" if plan[0] < 0 else "implicit-GEMM")
        row["autotuned"] = timed(ctx, fn)
        ctx.close()
        row["halo"] = {}
        if s == 1:
            for bn, T in HALO_SHAPES:
                if c % bn:
                    continue
                pin = os.path.join(tmp, "pinned.plans")
                with open(pin, "w") as f:
                    f.write(f"{key} | -1 {bn} {T}\n")
                ctx, fn = layer_ctx(False, pin)
                fn()
                ctx.sync()
                kept = os.path.join(tmp, "kept.plans")
                ctx.save_plans(kept)
                if _plans(kept).get(key) != (-1, bn, T):
                    row["halo"][f"{bn} {T}"] = "rejected"
                else:
                    row["halo"][f"{bn} {T}"] = timed(ctx, fn)
                ctx.close()
        results.append(row)
        t = row["autotuned"]
        tf = flops / (t["median_us"] * 1e-6)
        line = (f"{name:14s} x{count}: {t['median_us']:7.1f} us [{t['min_us']:.1f}, {t['max_us']:.1f}] {tf / 1e12:6.1f} TFLOP/s "
                f"({100 * tf / TF32_DENSE:.0f}% of 495, {100 * tf / cublas:.0f}% of cuBLAS)  won: {row['kernel']} `{row['plan']}`")
        print(line, flush=True)
        for shape, h in row["halo"].items():
            if h == "rejected":
                print(f"    halo -1 {shape}: rejected", flush=True)
            else:
                tf = flops / (h["median_us"] * 1e-6)
                print(f"    halo -1 {shape}: {h['median_us']:7.1f} us [{h['min_us']:.1f}, {h['max_us']:.1f}] {tf / 1e12:6.1f} TFLOP/s", flush=True)

    s1 = sum(r["count"] * r["autotuned"]["median_us"] for r in results if r["stride"] == 1)
    alls = sum(r["count"] * r["autotuned"]["median_us"] for r in results)
    print(f"card: {smi}; cuBLAS TF32 8192^3: {cublas / 1e12:.1f} TFLOP/s")
    print(f"13 stride-1 layers: {s1:.1f} us per step; all 16 3x3 layers: {alls:.1f} us per step")
    line = json.dumps(dict(tool="conv3x3_bench", nvidia_smi=smi, cublas_tf32_tflops=cublas / 1e12, repeats=a.repeats,
                           iters=a.iters, stride1_sum_us=s1, all_sum_us=alls, results=results))
    print(line)
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "conv3x3_bench.json"), "w") as f:
        f.write(line + "\n")


if __name__ == "__main__":
    main()
