"""Time ResNet-50's three layer-1 chain pairs at batch 32 in single-pass TF32, in two forms:
  (a) two launches: c3 (with its residual, or folded with its projection shortcut) writes y, then the next block's
      first 1x1 convolution reads y back and writes z;
  (b) one rten_b200_conv2d_chained call: z is computed from y's tiles while they are stored, y is not read back.
Each form is captured once as a CUDA graph after warm-up (autotuned plans for form (a)); the two forms alternate, the
L2 cache is flushed before every timed replay, and each of `--repeats` samples averages `--iters` replays timed with
CUDA events.

    python tools/chain_bench.py --out DIR [--repeats 7] [--iters 20]

Reports median us and [min, max] per form, and the form's algorithmic bytes (every input, weight and output once, y
read back in form (a)) over its median time against the 3.35 TB/s of the H100 SXM data sheet.  Prints form (a)'s
launch plans (RTEN_B200_VERBOSE lines of its warm-up), the card name and power limit with the numbers, and writes one
JSON line to DIR/chain_bench.json.  Needs an H100; there is no fallback."""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12
# (pair, c3 input channels, size, c3 output channels, next conv's output channels, projection input channels or 0)
PAIRS = [("layer1.0 -> layer1.1.c1", 64, 56, 256, 64, 64), ("layer1.1 -> layer1.2.c1", 64, 56, 256, 64, 0),
         ("layer1.2 -> layer2.0.c1", 64, 56, 256, 128, 0)]


def _card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


def _plans(fn):
    """fn() once with RTEN_B200_VERBOSE set; returns the [umma_gemm] lines it printed to stderr."""
    with tempfile.TemporaryFile(mode="w+") as f:
        sys.stderr.flush()
        saved = os.dup(2)
        os.dup2(f.fileno(), 2)
        os.environ["RTEN_B200_VERBOSE"] = "1"
        try:
            fn()
        finally:
            os.environ.pop("RTEN_B200_VERBOSE", None)
            os.dup2(saved, 2)
            os.close(saved)
        f.seek(0)
        return [ln.strip() for ln in f if ln.startswith("[umma_gemm]")]


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--out", required=True, help="directory for chain_bench.json")
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("chain_bench: no CUDA device; this benchmark measures the H100 kernels and has no fallback")
    import rten_b200 as rt
    card, smi = _card()
    stream = torch.cuda.Stream()
    rng = np.random.default_rng(0)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")  # larger than the 50 MB L2
    B = a.batch
    results = []
    ctx = rt.Context(0, stream=stream.cuda_stream)
    ctx.set_f32_mode(False)  # single-pass TF32: the only mode that chains
    ctx.set_autotune(True)
    for name, cin, h, cout, n2, cproj in PAIRS:
        dev = lambda arr: ctx.to_device(arr.astype(np.float32))
        t = ctx.to_device(rng.uniform(0, 1, (B, cin, h, h)).astype(np.float32), channels_last=True)
        w3 = dev(rng.uniform(-1, 1, (cout, cin, 1, 1)) / np.sqrt(cin))
        b3 = dev(rng.uniform(-0.1, 0.1, (cout,)))
        w1 = dev(rng.uniform(-1, 1, (n2, cout, 1, 1)) / np.sqrt(cout))
        b1 = dev(rng.uniform(-0.1, 0.1, (n2,)))
        c3, c1 = rt.Conv(activation=rt.ACT_RELU), rt.Conv(activation=rt.ACT_RELU)
        pk3, pk1 = c3.prepack(ctx, 1, w3), c1.prepack(ctx, 1, w1)
        if cproj:
            down = rt.Conv()
            x = ctx.to_device(rng.uniform(-1, 1, (B, cproj, h, h)).astype(np.float32), channels_last=True)
            wd = dev(rng.uniform(-1, 1, (cout, cproj, 1, 1)) / np.sqrt(cproj))
            bd = dev(rng.uniform(-0.1, 0.1, (cout,)))
            pkd = down.prepack(ctx, 1, wd)
            src = dict(proj=down, x_proj=x, w_proj=wd, bias_proj=bd, packed_w_proj=pkd)
        else:
            res = ctx.to_device(rng.uniform(-1, 1, (B, cout, h, h)).astype(np.float32), channels_last=True)
            src = dict(residual=res)
        ycl, zcl = (h * h * cout, 1, h * cout, cout), (h * h * n2, 1, h * n2, n2)
        ya, yb = ctx.empty((B, cout, h, h), strides=ycl), ctx.empty((B, cout, h, h), strides=ycl)
        za, zb = ctx.empty((B, n2, h, h), strides=zcl), ctx.empty((B, n2, h, h), strides=zcl)

        def two():
            if cproj:
                c3.run_projected(ctx, t, w3, b3, packed_w=pk3, out=ya, **src)
            else:
                c3.run(ctx, t, w3, b3, packed_w=pk3, out=ya, **src)
            c1.run(ctx, ya, w1, b1, packed_w=pk1, out=za)

        def chained():
            c3.run_chained(ctx, t, w3, b3, packed_w=pk3, nxt=c1, w_next=w1, bias_next=b1, packed_w_next=pk1, out=yb,
                           out_next=zb, **src)

        graphs, plans = {}, {}
        with torch.cuda.stream(stream):
            for form, fn in (("two_launches", two), ("chained", chained)):
                for _ in range(a.warmup):
                    fn()
                ctx.sync()
                plans[form] = _plans(fn)
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
        same = bool(np.array_equal(ya.numpy(), yb.numpy()) and np.array_equal(za.numpy(), zb.numpy()))
        e = 4.0
        n_t, n_y, n_z = B * cin * h * h, B * cout * h * h, B * n2 * h * h
        n_src = B * cproj * h * h if cproj else n_y  # the projection input, or the residual
        w_bytes = e * (cout * cin + cout * cproj + 2 * cout + n2 * cout + n2)
        base = e * (n_t + n_src + n_y + n_z) + w_bytes
        nbytes = {"chained": base, "two_launches": base + e * n_y}
        row = dict(pair=name, batch=B, bit_identical=same, plans=plans)
        for form, ts in times.items():
            ts = sorted(ts)
            med = ts[len(ts) // 2]
            row[form] = dict(median_us=med, min_us=ts[0], max_us=ts[-1], bytes=nbytes[form],
                             hbm_share=nbytes[form] / (med * 1e-6) / HBM_BYTES_PER_S)
        row["speedup"] = row["two_launches"]["median_us"] / row["chained"]["median_us"]
        results.append(row)
        ta, tb = row["two_launches"], row["chained"]
        for form in plans:
            for ln in plans[form]:
                print(f"  {form}: {ln}")
        print(f"{smi} {name}: two launches {ta['median_us']:7.1f} us [{ta['min_us']:.1f}, {ta['max_us']:.1f}] "
              f"({ta['bytes'] / 1e6:.0f} MB, {100 * ta['hbm_share']:.0f}% of 3.35 TB/s)  chained {tb['median_us']:7.1f} us "
              f"[{tb['min_us']:.1f}, {tb['max_us']:.1f}] ({tb['bytes'] / 1e6:.0f} MB, {100 * tb['hbm_share']:.0f}%)  "
              f"x{row['speedup']:.2f}  bit-identical {same}", flush=True)
    line = json.dumps(dict(tool="chain_bench", card=card, nvidia_smi=smi, repeats=a.repeats, iters=a.iters, results=results))
    print(line)
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "chain_bench.json"), "w") as f:
        f.write(line + "\n")


if __name__ == "__main__":
    main()
