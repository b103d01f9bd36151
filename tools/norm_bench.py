"""Time LayerNormalization, the skip layer norms and RMSNormalization at LLM / encoder shapes:
  SkipSimplifiedLayerNormalization with the sum output (the decoder residual) against torch (x + skip + bias, then
  F.rms_norm); SkipLayerNormalization with bias and beta against the composed path a caller has without it
  (rten_b200_add x 2 + rten_b200_layer_norm) and against torch (x + skip + bias, then F.layer_norm); RMSNormalization
  against F.rms_norm; plain LayerNormalization (scale and bias) against F.layer_norm.  Shapes: Llama-3-8B decode
  (8 x 4096) and prefill (2048 x 4096, 8 x 512 x 4096), Qwen2-7B (3584), 70B (8192), Phi-3 (3072), BERT-base
  (16 x 128 x 768).
Each form is captured once as a CUDA graph after warm-up; forms alternate, the L2 cache is flushed before every timed
replay, and each of `--repeats` samples averages `--iters` replays timed with CUDA events (tools/depthwise_bench.py).
The bytes bound counts x, skip and out (and the sum for the skip-simplified form) plus gamma / beta / bias once, at
3.35 TB/s.

    python tools/norm_bench.py [--out DIR] [--repeats 7] [--iters 20]

Prints the card name and power limit with the numbers; with --out, writes one JSON line to DIR/norm_bench.json.
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

# (name, x shape)
SHAPES = [
    ("Llama-3-8B decode", (8, 4096)),
    ("Llama-3-8B prefill", (2048, 4096)),
    ("Llama-3-8B prefill b8", (8, 512, 4096)),
    ("Qwen2-7B prefill", (2048, 3584)),
    ("70B prefill", (2048, 8192)),
    ("Phi-3 prefill", (2048, 3072)),
    ("BERT-base", (16, 128, 768)),
]


def _stats(ts):
    ts = sorted(ts)
    return dict(median_us=ts[len(ts) // 2], min_us=ts[0], max_us=ts[-1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
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
    eps = 1e-6
    for sname, shape in SHAPES:
        H = shape[-1]
        numel = int(np.prod(shape))
        xn, kn = (rng.standard_normal(shape).astype(np.float32) for _ in range(2))
        gn, ben, bin_ = ((1 + 0.1 * rng.standard_normal(H)).astype(np.float32), (0.1 * rng.standard_normal(H)).astype(np.float32),
                         (0.1 * rng.standard_normal(H)).astype(np.float32))
        x, k, g, be, bi = (ctx.to_device(v) for v in (xn, kn, gn, ben, bin_))
        xt, kt, gt, bet, bit = (torch.from_numpy(v).cuda() for v in (xn, kn, gn, ben, bin_))
        sso, slo, rms = rt.SkipSimplifiedLayerNormalization(eps), rt.SkipLayerNormalization(eps), rt.RMSNormalization(-1, eps)
        add, ln = rt.Add(), rt.LayerNormalization(-1, eps)
        keep = []
        forms = {
            "skip_simplified+sum": lambda: keep.append(sso.run(ctx, x, k, g, bi, want_sum=True)),
            "skip_layer_norm": lambda: keep.append(slo.run(ctx, x, k, g, be, bi)),
            "composed add+add+layer_norm": lambda: keep.append(ln.run(ctx, add.run(ctx, add.run(ctx, x, k), bi), g, be)),
            "rms_norm": lambda: keep.append(rms.run(ctx, x, g)),
            "layer_norm": lambda: keep.append(ln.run(ctx, x, g, be)),
        }
        torch_forms = {
            "torch skip+rms_norm": lambda: keep.append(F.rms_norm(xt + kt + bit, (H,), gt, eps)),
            "torch skip+layer_norm": lambda: keep.append(F.layer_norm(xt + kt + bit, (H,), gt, bet, eps)),
            "torch rms_norm": lambda: keep.append(F.rms_norm(xt, (H,), gt, eps)),
            "torch layer_norm": lambda: keep.append(F.layer_norm(xt, (H,), gt, bet, eps)),
        }
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
        # bytes the operator has to move: x, skip and out (+ the sum), parameters once
        bound = {
            "skip_simplified+sum": 4 * (4 * numel + 2 * H), "torch skip+rms_norm": 4 * (3 * numel + 2 * H),
            "skip_layer_norm": 4 * (3 * numel + 3 * H), "composed add+add+layer_norm": 4 * (3 * numel + 3 * H),
            "torch skip+layer_norm": 4 * (3 * numel + 3 * H), "rms_norm": 4 * (2 * numel + H), "torch rms_norm": 4 * (2 * numel + H),
            "layer_norm": 4 * (2 * numel + 2 * H), "torch layer_norm": 4 * (2 * numel + 2 * H),
        }
        row = dict(shape=sname, dims=list(shape))
        for fname, ts in times.items():
            s = _stats(ts)
            t_b = bound[fname] / HBM_BYTES_PER_S
            s.update(bytes_bound_us=t_b * 1e6, bytes_share=t_b / (s["median_us"] * 1e-6))
            row[fname] = s
            print(f"[{power}] {sname:22s} {str(shape):16s} {fname:28s} {s['median_us']:8.1f} us [{s['min_us']:.1f}, "
                  f"{s['max_us']:.1f}]  {100 * s['bytes_share']:3.0f}% of the bytes bound ({t_b * 1e6:.1f} us)", flush=True)
        rows_out.append(row)
        keep.clear()
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "norm_bench.json"), "w") as f:
            f.write(json.dumps(dict(card=name, power=power, time=time.strftime("%Y-%m-%d %H:%M:%S"), rows=rows_out)) + "\n")


if __name__ == "__main__":
    main()
