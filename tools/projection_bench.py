"""Time ResNet-50's four projection blocks' last convolution and shortcut at batch 32, in both f32 modes, in two forms:
  (a) two launches: the 1x1 downsample conv writes the shortcut tensor, then c3 (1x1) reads it back as its residual;
  (b) one rten_b200_conv2d_projected call: one GEMM over [t | x] against [W3 | Wd], no shortcut tensor.
Each form is captured once as a CUDA graph after warm-up (autotuned plans); the two forms alternate, the L2 cache is
flushed before every timed replay, and each of `--repeats` samples averages `--iters` replays timed with CUDA events.

    python tools/projection_bench.py --out DIR [--repeats 7] [--iters 20]

Reports median us and [min, max] per form, and the form's algorithmic bytes (every input, weight and output once, the
shortcut tensor written and read in form (a)) over its median time against the 3.35 TB/s of the H100 SXM data sheet.
Prints the card name and power limit with the numbers and writes one JSON line to DIR/projection_bench.json.  Needs an
H100; there is no fallback."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12
# (block input channels, its size, bottleneck width, output channels, shortcut stride)
BLOCKS = [("layer1.0", 64, 56, 64, 256, 1), ("layer2.0", 256, 56, 128, 512, 2), ("layer3.0", 512, 28, 256, 1024, 2),
          ("layer4.0", 1024, 14, 512, 2048, 2)]


def _card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--out", required=True, help="directory for projection_bench.json")
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("projection_bench: no CUDA device; this benchmark measures the H100 kernels and has no fallback")
    import rten_b200 as rt
    card, smi = _card()
    stream = torch.cuda.Stream()
    rng = np.random.default_rng(0)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")  # larger than the 50 MB L2
    B = a.batch
    results = []
    for tf32 in (True, False):
        mode = "tf32" if tf32 else "tf32x3"
        ctx = rt.Context(0, stream=stream.cuda_stream)
        ctx.set_f32_mode(not tf32)
        ctx.set_autotune(True)
        for name, cin, h, wd, cout, s in BLOCKS:
            oh = (h - 1) // s + 1
            x = ctx.to_device(rng.uniform(-1, 1, (B, cin, h, h)).astype(np.float32), channels_last=True)
            t = ctx.to_device(rng.uniform(0, 1, (B, wd, oh, oh)).astype(np.float32), channels_last=True)
            w3 = ctx.to_device((rng.uniform(-1, 1, (cout, wd, 1, 1)) / np.sqrt(wd)).astype(np.float32))
            wdn = ctx.to_device((rng.uniform(-1, 1, (cout, cin, 1, 1)) / np.sqrt(cin)).astype(np.float32))
            b3 = ctx.to_device(rng.uniform(-0.1, 0.1, (cout,)).astype(np.float32))
            bd = ctx.to_device(rng.uniform(-0.1, 0.1, (cout,)).astype(np.float32))
            c3, down = rt.Conv(activation=rt.ACT_RELU), rt.Conv(strides=(s, s))
            pk3, pkd = c3.prepack(ctx, 1, w3), down.prepack(ctx, 1, wdn)
            cl = (oh * oh * cout, 1, oh * cout, cout)
            ident, out_a, out_b = (ctx.empty((B, cout, oh, oh), strides=cl) for _ in range(3))

            def two():
                down.run(ctx, x, wdn, bd, packed_w=pkd, out=ident)
                c3.run(ctx, t, w3, b3, packed_w=pk3, residual=ident, out=out_a)

            def folded():
                c3.run_projected(ctx, t, w3, b3, packed_w=pk3, proj=down, x_proj=x, w_proj=wdn, bias_proj=bd,
                                 packed_w_proj=pkd, out=out_b)

            graphs = {}
            with torch.cuda.stream(stream):
                for form, fn in (("two_launches", two), ("folded", folded)):
                    for _ in range(a.warmup):
                        fn()
                    ctx.sync()
                    ctx.graph_begin()
                    fn()
                    graphs[form] = ctx.graph_end()
                times = {f: [] for f in graphs}
                for _ in range(a.repeats):
                    for form, g in graphs.items():
                        tot = 0.0
                        for _ in range(a.iters):
                            flush.zero_()
                            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                            e0.record()
                            g.launch()
                            e1.record()
                            e1.synchronize()
                            tot += e0.elapsed_time(e1) * 1e3
                        times[form].append(tot / a.iters)
            ctx.sync()
            ya, yb = out_a.numpy().astype(np.float64), out_b.numpy().astype(np.float64)
            diff = float(np.abs(ya - yb).max() / np.abs(ya).max())
            e = 4.0
            n_x, n_t, n_o = B * cin * h * h, B * wd * oh * oh, B * cout * oh * oh
            w_bytes = e * (cout * wd + cout * cin + 2 * cout)
            nbytes = {"folded": e * (n_x + n_t + n_o) + w_bytes, "two_launches": e * (n_x + n_t + 3 * n_o) + w_bytes}
            row = dict(block=name, mode=mode, batch=B, flops=2.0 * B * oh * oh * cout * (wd + cin), rel_diff=diff)
            for form, ts in times.items():
                ts = sorted(ts)
                med = ts[len(ts) // 2]
                row[form] = dict(median_us=med, min_us=ts[0], max_us=ts[-1], bytes=nbytes[form],
                                 hbm_share=nbytes[form] / (med * 1e-6) / HBM_BYTES_PER_S)
            row["speedup"] = row["two_launches"]["median_us"] / row["folded"]["median_us"]
            results.append(row)
            ta, tb = row["two_launches"], row["folded"]
            print(f"{smi} {name} {mode:6s}: two launches {ta['median_us']:7.1f} us [{ta['min_us']:.1f}, {ta['max_us']:.1f}] "
                  f"({ta['bytes'] / 1e6:.0f} MB, {100 * ta['hbm_share']:.0f}% of 3.35 TB/s)  folded {tb['median_us']:7.1f} us "
                  f"[{tb['min_us']:.1f}, {tb['max_us']:.1f}] ({tb['bytes'] / 1e6:.0f} MB, {100 * tb['hbm_share']:.0f}%)  "
                  f"x{row['speedup']:.2f}  rel diff {diff:.1e}", flush=True)
    line = json.dumps(dict(tool="projection_bench", card=card, nvidia_smi=smi, repeats=a.repeats, iters=a.iters, results=results))
    print(line)
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "projection_bench.json"), "w") as f:
        f.write(line + "\n")


if __name__ == "__main__":
    main()
