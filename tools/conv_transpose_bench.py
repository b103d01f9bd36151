"""Time ConvTranspose on decoder-head layers, in both f32 modes, against cuDNN:
  (a) rten_b200_conv_transpose with prepacked weights: one implicit-GEMM launch per stride phase with taps, plus one fill
      launch when a phase has none;
  (b) torch.nn.functional.conv_transpose2d (cuDNN) on the same channels-last tensors, with
      torch.backends.cudnn.allow_tf32 matched to the mode (True for TF32, False for the fp32-grade 3xTF32).
Each form is captured once as a CUDA graph after warm-up (autotuned plans); the two forms alternate, the L2 cache is
flushed before every timed replay, and each of `--repeats` samples averages `--iters` replays timed with CUDA events.

    python tools/conv_transpose_bench.py [--out DIR] [--repeats 7] [--iters 20]

Reports median us and [min, max] per form, the layer's algorithmic FLOPs (2 * B * C_in * H * W * C_out/groups * kh * kw)
and bytes (input, weight, bias and output once), and the share of the roofline the median reaches: the larger of
FLOPs / peak and bytes / 3.35 TB/s over the time, with the bound that sets it named.  The peaks are the H100 SXM data
sheet's dense TF32 tensor rate (494.7 TFLOP/s) for TF32 and a third of it for 3xTF32 (three TF32 products per
product).  Prints the card name and power limit with the numbers; with --out, writes one JSON line to
DIR/conv_transpose_bench.json.  Needs an H100; there is no fallback."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12
TF32_FLOPS = 494.7e12
# (name, batch, C_in, C_out, H = W, k, stride, pad)
LAYERS = [
    ("SAM mask decoder up 1", 1, 256, 64, 64, 2, 2, 0),
    ("SAM mask decoder up 2", 1, 64, 32, 128, 2, 2, 0),
    ("DPT reassemble k4 s4", 1, 48, 48, 37, 4, 4, 0),
    ("DPT reassemble k2 s2", 1, 96, 96, 37, 2, 2, 0),
    ("U-Net decoder", 8, 512, 256, 32, 2, 2, 0),
    ("DCGAN k4 s2 p1", 32, 256, 128, 16, 4, 2, 1),
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


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--out", default=None, help="directory for conv_transpose_bench.json")
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    import torch
    import torch.nn.functional as F
    if not torch.cuda.is_available():
        raise SystemExit("conv_transpose_bench: no CUDA device; this benchmark measures the H100 kernels and has no fallback")
    import rten_b200 as rt
    card, smi = _card()
    stream = torch.cuda.Stream()
    rng = np.random.default_rng(0)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")  # larger than the 50 MB L2
    results = []
    for tf32 in (True, False):
        mode = "tf32" if tf32 else "tf32x3"
        torch.backends.cudnn.allow_tf32 = tf32
        ctx = rt.Context(0, stream=stream.cuda_stream)
        ctx.set_f32_mode(not tf32)
        ctx.set_autotune(True)
        for name, B, cin, cout, h, k, s, p in LAYERS:
            oh = (h - 1) * s + k - 2 * p
            xn = rng.uniform(-1, 1, (B, cin, h, h)).astype(np.float32)
            wn = (rng.uniform(-1, 1, (cin, cout, k, k)) / np.sqrt(cin * k * k / (s * s))).astype(np.float32)
            bn = rng.uniform(-0.1, 0.1, (cout,)).astype(np.float32)
            x = ctx.to_device(xn, channels_last=True)
            w, b = ctx.to_device(wn), ctx.to_device(bn)
            op = rt.ConvTranspose(padding=(p, p, p, p), strides=(s, s))
            pk = op.prepack(ctx, 1, w)
            out = ctx.empty((B, cout, oh, oh), strides=(oh * oh * cout, 1, oh * cout, cout))
            xt = torch.from_numpy(xn).cuda().to(memory_format=torch.channels_last)
            wt, bt = torch.from_numpy(wn).cuda(), torch.from_numpy(bn).cuda()
            yt = [None]

            def ours():
                op.run(ctx, x, w, b, packed_w=pk, out=out)

            def cudnn():
                yt[0] = F.conv_transpose2d(xt, wt, bt, stride=s, padding=p)

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
                times = {f: [] for f in graphs}
                for _ in range(a.repeats):
                    for form, g in graphs.items():
                        tot = 0.0
                        for _ in range(a.iters):
                            flush.zero_()
                            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                            e0.record()
                            (g.launch if form == "rten_b200" else g.replay)()
                            e1.record()
                            e1.synchronize()
                            tot += e0.elapsed_time(e1) * 1e3
                        times[form].append(tot / a.iters)
            ctx.sync()
            torch.cuda.synchronize()
            ours_y = out.numpy().astype(np.float64)
            ref_y = yt[0].float().cpu().numpy().astype(np.float64)
            diff = float(np.abs(ours_y - ref_y).max() / np.abs(ref_y).max())
            flops = 2.0 * B * cin * h * h * cout * k * k
            nbytes = 4.0 * (B * cin * h * h + cin * cout * k * k + cout + B * cout * oh * oh)
            peak = TF32_FLOPS if tf32 else TF32_FLOPS / 3
            t_flops, t_bytes = flops / peak, nbytes / HBM_BYTES_PER_S
            bound = "compute" if t_flops >= t_bytes else "HBM"
            row = dict(layer=name, mode=mode, batch=B, c_in=cin, c_out=cout, size=h, k=k, stride=s, pad=p, flops=flops,
                       bytes=nbytes, bound=bound, launches=launches, rel_diff_vs_cudnn=diff)
            for form, ts in times.items():
                ts = sorted(ts)
                med = ts[len(ts) // 2]
                row[form] = dict(median_us=med, min_us=ts[0], max_us=ts[-1], roofline_share=max(t_flops, t_bytes) / (med * 1e-6))
            results.append(row)
            o, c = row["rten_b200"], row["cudnn"]
            print(f"{smi} {name:22s} {mode:6s}: rten_b200 {o['median_us']:8.1f} us [{o['min_us']:.1f}, {o['max_us']:.1f}] "
                  f"({launches} launches, {100 * o['roofline_share']:.0f}% of {bound} roofline)  cudnn {c['median_us']:8.1f} us "
                  f"[{c['min_us']:.1f}, {c['max_us']:.1f}] ({100 * c['roofline_share']:.0f}%)  "
                  f"{flops / 1e9:.2f} GFLOP {nbytes / 1e6:.1f} MB  rel diff {diff:.1e}", flush=True)
    line = json.dumps(dict(tool="conv_transpose_bench", card=card, nvidia_smi=smi, repeats=a.repeats, iters=a.iters,
                           results=results))
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "conv_transpose_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
