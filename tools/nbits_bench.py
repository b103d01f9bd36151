"""Time MatMulNBits (4-bit block-quantized weights, dequantized on chip) against MatMul on the same weights dequantized
to f32 and prepacked once, with CUDA events after warm-up, in both f32 modes, the two implementations alternating.

    python tools/nbits_bench.py --out DIR [--repeats 5] [--iters 20]

Shapes: the two projections of a Llama-class MLP, (K, N) = (4096, 14336) and (14336, 4096), block 32, at M = 1, 8, 16,
32, 64, 512 and 4096 rows.  At M = 8, 16 and 32 both MatMulNBits kernels are timed as well (the streaming kernel and
the wgmma kernel, forced through RTEN_B200_NBITS_SKINNY_MAX), which is where the threshold T of csrc/nbits.h comes
from.  Each row records the algorithmic bytes (nibbles, scales, A and the output once) and flops (2 M N K), and which
data-sheet roofline (3.35 TB/s HBM3; 67 TFLOP/s FP32 for the streaming kernel, 495 / 3 TFLOP/s TF32 for the wgmma
kernel) bounds it.  Prints the card name and power limit with the numbers and writes one JSON line to
DIR/nbits_bench.json.  Needs an H100; there is no fallback."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM = 3.35e12
FP32 = 67e12
TF32 = 495e12
T_ENV = "RTEN_B200_NBITS_SKINNY_MAX"


def _card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                               text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


def _time(fns, stream, repeats, iters, warmup):
    """{name: sorted per-call µs over the repeats}, the functions alternating inside every repeat.  A function is
    (callable, env value of T_ENV or None)."""
    import torch

    def call(fn, env):
        if env is None:
            os.environ.pop(T_ENV, None)
        else:
            os.environ[T_ENV] = env
        fn()

    times = {k: [] for k in fns}
    with torch.cuda.stream(stream):
        for k, (fn, env) in fns.items():
            for _ in range(warmup):
                call(fn, env)
        for _ in range(repeats):
            for k, (fn, env) in fns.items():
                if env is None:
                    os.environ.pop(T_ENV, None)
                else:
                    os.environ[T_ENV] = env
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(iters):
                    fn()
                e1.record()
                e1.synchronize()
                times[k].append(e0.elapsed_time(e1) * 1e3 / iters)
    os.environ.pop(T_ENV, None)
    return {k: sorted(v) for k, v in times.items()}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--out", required=True, help="directory for nbits_bench.json")
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("nbits_bench: no CUDA device; this benchmark measures the H100 kernels and has no fallback")
    import rten_b200 as rt
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from test_gpu_matmul_nbits import T, dequantize_nbits, pack_nbits
    card, power = _card()
    stream = torch.cuda.Stream()
    ctx = rt.Context(0, stream=stream.cuda_stream)
    rng = np.random.default_rng(0)
    block = 32
    results = []
    for K, N in ((4096, 14336), (14336, 4096)):
        b = pack_nbits(rng.integers(0, 16, (N, K // block, block)))
        s = rng.uniform(0.005, 0.02, (N, K // block)).astype(np.float32)
        db, ds = ctx.to_device(b), ctx.to_device(s)
        w = ctx.to_device(dequantize_nbits(b, s))  # the same values as f32 [K, N]
        mm = rt.MatMul()
        packed = mm.prepack(ctx, 1, w)
        nb = rt.MatMulNBits(block_size=block)
        for M in (1, 8, 16, 32, 64, 512, 4096):
            x = ctx.to_device(rng.uniform(-1, 1, (M, K)).astype(np.float32))
            out_n, out_m = ctx.empty((M, N)), ctx.empty((M, N))
            run_n = lambda: nb.run(ctx, x, db, ds, out=out_n)
            run_m = lambda: mm.run(ctx, x, w, packed_b=packed, out=out_m)
            fns = {"nbits": (run_n, None), "matmul_f32_weights": (run_m, None)}
            if M in (8, 16, 32):
                fns["nbits_skinny"] = (run_n, "32")
                fns["nbits_wgmma"] = (run_n, "0")
            nbytes = K * N / 2 + N * K / block * 4 + M * K * 4 + M * N * 4
            flops = 2.0 * M * N * K
            for tf32 in (False, True):
                ctx.set_f32_mode(not tf32)
                mode = "tf32" if tf32 else "3xtf32"
                iters = a.iters if M < 512 else max(3, a.iters // 4)
                times = _time(fns, stream, a.repeats, iters, a.warmup)
                ctx.sync()
                yn, ym = out_n.numpy().astype(np.float64), out_m.numpy().astype(np.float64)
                diff = float(np.abs(yn - ym).max() / max(np.abs(ym).max(), 1e-30))
                skinny = M <= T
                peak = FP32 if skinny else (TF32 if tf32 else TF32 / 3)
                t_bw, t_fl = nbytes / HBM, flops / peak
                row = dict(K=K, N=N, M=M, block=block, mode=mode, kernel="skinny" if skinny else "wgmma", bytes=nbytes, flops=flops,
                           bound="HBM" if t_bw >= t_fl else "compute", roofline_us=max(t_bw, t_fl) * 1e6, rel_diff_vs_matmul=diff)
                for k, ts in times.items():
                    row[k] = dict(median_us=ts[len(ts) // 2], min_us=ts[0], max_us=ts[-1])
                med = row["nbits"]["median_us"]
                row["speedup_vs_matmul"] = row["matmul_f32_weights"]["median_us"] / med
                row["share_of_roofline"] = row["roofline_us"] / med
                results.append(row)
                extra = "".join(f"  {k[6:]} {row[k]['median_us']:.1f}" for k in ("nbits_skinny", "nbits_wgmma") if k in row)
                print(f"{card} (power limit {power}) K {K:5d} N {N:5d} M {M:4d} {mode:6s}: nbits {med:9.1f} us "
                      f"[{row['nbits']['min_us']:.1f}, {row['nbits']['max_us']:.1f}]  matmul {row['matmul_f32_weights']['median_us']:9.1f} us "
                      f"x{row['speedup_vs_matmul']:.2f}  {row['bound']}-bound roofline {row['roofline_us']:.1f} us "
                      f"({100 * row['share_of_roofline']:.0f}%){extra}  rel diff {diff:.1e}", flush=True)
            del x, out_n, out_m
        del packed, w, db, ds
    line = json.dumps(dict(tool="nbits_bench", card=card, power_limit=power, T=T, repeats=a.repeats, iters=a.iters, results=results))
    print(line)
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "nbits_bench.json"), "w") as f:
        f.write(line + "\n")


if __name__ == "__main__":
    main()
