"""Time GRU / LSTM layers: this operator (the cluster-resident recurrence where R fits a cluster), its per-step path
(RTEN_B200_NO_RNN_CLUSTER=1: one recurrent product and one gate launch per step) and torch.nn.GRU / nn.LSTM on cuDNN,
with CUDA events after warm-up, the three arms alternating.  Both f32 modes: 3xTF32 (default) with
torch.backends.cudnn.allow_tf32 off, and single-pass TF32 with it on.  cuDNN's TF32 mode also rounds its recurrent
product to TF32; this operator's recurrence is exact f32 in both modes.

    python tools/rnn_bench.py --out DIR [--repeats 5] [--iters 5]

Layers: the two bidirectional GRU layers of a CRNN text recognizer (H 256, I 256 then 512, T 128, B 64); a
bidirectional LSTM (H 256, I 512, T 128, B 32); a latency-bound LSTM (H 128, I 128, B 1, T 512); and an LSTM above the
cluster bound, which takes the per-step path in both of this operator's arms (H 1024, I 1024, B 16, T 64).  Reports the
median us [min, max] per call, us per step and FLOP/s for 2 T B dirs G H (I + H), with the card's name and power limit,
and writes one JSON line to DIR/rnn_bench.json.  Needs an H100; there is no fallback."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

LAYERS = [("crnn_gru1", "gru", dict(T=128, B=64, I=256, H=256, bidir=True)),
          ("crnn_gru2", "gru", dict(T=128, B=64, I=512, H=256, bidir=True)),
          ("bilstm_256", "lstm", dict(T=128, B=32, I=512, H=256, bidir=True)),
          ("lstm_128_b1", "lstm", dict(T=512, B=1, I=128, H=128, bidir=False)),
          ("lstm_1024", "lstm", dict(T=64, B=16, I=1024, H=1024, bidir=False))]


def _card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                               text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


def flops(op, T, B, I, H, bidir):
    G = 3 if op == "gru" else 4
    return 2 * T * B * (2 if bidir else 1) * G * H * (I + H)


def _layer(rt, ctx, op, T, B, I, H, bidir, rng):
    """Callables (ours, per_step, cudnn) and getters of their Y."""
    import torch
    G = 3 if op == "gru" else 4
    dirs = 2 if bidir else 1
    s = 1.0 / np.sqrt(H)
    f = lambda *shape, k=s: rng.uniform(-k, k, shape).astype(np.float32)  # noqa: E731
    x, w, r, b = f(T, B, I, k=1.0), f(dirs, G * H, I), f(dirs, G * H, H), f(dirs, 2 * G * H)
    direction = "bidirectional" if bidir else "forward"
    o = rt.GRU(direction, H) if op == "gru" else rt.LSTM(direction, H)
    pk = o.prepack(ctx, w)
    dx, dw, dr, db = (ctx.to_device(a) for a in (x, w, r, b))
    res = {}

    def ours():
        res["ours"] = o.run(ctx, dx, dw, dr, b=db, packed_w=pk, outputs=(0,))[0]

    def per_step():
        os.environ["RTEN_B200_NO_RNN_CLUSTER"] = "1"
        try:
            res["per_step"] = o.run(ctx, dx, dw, dr, b=db, packed_w=pk, outputs=(0,))[0]
        finally:
            os.environ.pop("RTEN_B200_NO_RNN_CLUSTER")

    m = (torch.nn.GRU if op == "gru" else torch.nn.LSTM)(I, H, bidirectional=bidir).cuda()
    order = [1, 0, 2] if op == "gru" else [0, 2, 3, 1]  # ONNX gate order -> torch's
    ro = lambda a: torch.from_numpy(np.concatenate([a[i * H:(i + 1) * H] for i in order])).cuda()  # noqa: E731
    with torch.no_grad():
        for d, sfx in enumerate(["", "_reverse"][:dirs]):
            getattr(m, "weight_ih_l0" + sfx).copy_(ro(w[d]))
            getattr(m, "weight_hh_l0" + sfx).copy_(ro(r[d]))
            getattr(m, "bias_ih_l0" + sfx).copy_(ro(b[d][:G * H]))
            getattr(m, "bias_hh_l0" + sfx).copy_(ro(b[d][G * H:]))
    tx = torch.from_numpy(x).cuda()

    def cudnn():
        with torch.no_grad():
            res["cudnn"] = m(tx)[0]

    def outputs():
        y = res["ours"].numpy().reshape(T, dirs, B, H).transpose(0, 2, 1, 3).reshape(T, B, dirs * H)
        return y, res["per_step"].numpy().reshape(y.shape), res["cudnn"].cpu().numpy()
    return ours, per_step, cudnn, outputs


def _stats(ts):
    ts = sorted(ts)
    return dict(median_us=ts[len(ts) // 2], min_us=ts[0], max_us=ts[-1])


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--out", required=True, help="directory for rnn_bench.json")
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("rnn_bench: no CUDA device; this benchmark measures the H100 kernels and has no fallback")
    import rten_b200 as rt
    card, power = _card()
    stream = torch.cuda.Stream()
    ctx = rt.Context(0, stream=stream.cuda_stream)
    rng = np.random.default_rng(0)
    results = []
    for mode in ("3xtf32", "tf32"):
        ctx.set_f32_mode(mode == "3xtf32")
        torch.backends.cuda.matmul.allow_tf32 = mode == "tf32"
        torch.backends.cudnn.allow_tf32 = mode == "tf32"
        for name, op, s in LAYERS:
            with torch.cuda.stream(stream):
                ours, per_step, cudnn, outputs = _layer(rt, ctx, op, rng=rng, **s)
                impls = [("ours", ours), ("per_step", per_step), ("cudnn", cudnn)]
                times = {n: [] for n, _ in impls}
                for _, fn in impls:
                    for _ in range(a.warmup):
                        fn()
                for _ in range(a.repeats):
                    for n, fn in impls:
                        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        e0.record()
                        for _ in range(a.iters):
                            fn()
                        e1.record()
                        e1.synchronize()
                        times[n].append(e0.elapsed_time(e1) * 1e3 / a.iters)
            ctx.sync()
            yo, yp, yc = outputs()
            fl = flops(op, **s)
            row = dict(layer=name, op=op, mode=mode, **s, flop=fl,
                       max_abs_diff_per_step=float(np.abs(yo - yp).max()), max_abs_diff_cudnn=float(np.abs(yo - yc).max()))
            for n, ts in times.items():
                st = _stats(ts)
                st["us_per_step"] = st["median_us"] / s["T"]
                st["tflops"] = fl / (st["median_us"] * 1e-6) / 1e12
                row[n] = st
            print(f"{card} (power limit {power}) {mode:6s} {name:12s}: ours {row['ours']['median_us']:9.1f} us "
                  f"[{row['ours']['min_us']:.1f}, {row['ours']['max_us']:.1f}] ({row['ours']['us_per_step']:.2f} us/step, "
                  f"{row['ours']['tflops']:.2f} TFLOP/s)  per-step {row['per_step']['median_us']:9.1f} us  "
                  f"cuDNN {row['cudnn']['median_us']:9.1f} us  |d| vs cuDNN {row['max_abs_diff_cudnn']:.1e}")
            results.append(row)
    line = json.dumps(dict(tool="rnn_bench", card=card, power_limit=power, repeats=a.repeats, iters=a.iters, results=results))
    print(line)
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "rnn_bench.json"), "w") as f:
        f.write(line + "\n")


if __name__ == "__main__":
    main()
