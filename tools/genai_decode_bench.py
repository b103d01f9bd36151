"""Decode-step time of an onnxruntime-genai int4 decoder through Model: KV caches passed as writable inputs with spare
capacity (the attention nodes append in place) against the copying run (new present caches every step), alternating.

Llama-3-8B-shaped layers -- hidden 4096, 32 / 8 heads of 128, MLP 14336, int4 blocks of 32 -- with seeded weights,
--layers of them (4 by default) plus an int4 lm_head over a 32000-token vocabulary, written as genai writes them
(tests/genai_decoder.py: the attention-mask subgraph, packed QKV in layer 0).  Past caches of P random positions are fed
directly (no prefill).  For B 1 and 8 and P 512, 2048 and 4096 it reports the median [min, max] of --samples samples, each
the mean of --steps decode steps ended by a device synchronise; launches per step; and the HBM-bound share: the int4
weights, their scales and the valid caches read once at 3.35 TB/s, over the in-place step time.  Then Generator
(ModelDecoder) tokens/s over 64 new tokens after a 16-token prompt.  The card's name, power limit and max SM clock are
read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

HBM = 3.35e12


def weights(c, seed=1):
    r = np.random.default_rng(seed)
    hid, kvd = c["Hq"] * c["D"], c["Hkv"] * c["D"]
    w = {"embed": (0.02 * r.standard_normal((c["V"], hid))).astype(np.float32)}

    def q4(nm, K, N):
        w["b_" + nm] = r.integers(0, 256, (N, K // c["block"], c["block"] // 2), dtype=np.uint8)
        w["s_" + nm] = r.uniform(0.002, 0.01, (N, K // c["block"])).astype(np.float32)
    for l in range(c["L"]):
        if l == 0:
            q4("qkv0", hid, hid + 2 * kvd)
        else:
            q4(f"q{l}", hid, hid), q4(f"k{l}", hid, kvd), q4(f"v{l}", hid, kvd)
        q4(f"o{l}", hid, hid), q4(f"gate{l}", hid, c["I"]), q4(f"up{l}", hid, c["I"]), q4(f"down{l}", c["I"], hid)
        w[f"g_in{l}"] = np.ones(hid, np.float32)
        w[f"g_post{l}"] = np.ones(hid, np.float32)
    w["g_final"] = np.ones(hid, np.float32)
    q4("lm", hid, c["V"])
    half = c["D"] // 2
    ang = np.arange(c["maxp"])[:, None] * (500000.0 ** (-np.arange(half) / half))[None, :]
    w["cos"], w["sin"] = np.cos(ang).astype(np.float32), np.sin(ang).astype(np.float32)
    return w


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=4)
    ap.add_argument("--samples", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--batches", default="1,8")
    ap.add_argument("--pasts", default="512,2048,4096")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import rten_b200 as rt
    import genai_decoder as gd
    from rten_b200.generate import Generator, KvCacheHandle, ModelDecoder
    from rten_b200.model import Model
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    c = dict(L=a.layers, V=32000, Hq=32, Hkv=8, D=128, I=14336, block=32, maxp=8192, eps=1e-5)
    w = weights(c)
    wbytes = sum(v.nbytes for k, v in w.items() if k.startswith(("b_", "s_")))
    ctx = rt.Context(0)
    m = Model(ctx, gd.genai_graph(w, (0,), c))
    del w
    names = gd.output_names(c)
    pasts = [f"past_key_values.{l}.{kv}" for l in range(c["L"]) for kv in ("key", "value")]
    r = np.random.default_rng(2)
    rows = []
    for B in [int(x) for x in a.batches.split(",")]:
        for P in [int(x) for x in a.pasts.split(",")]:
            cap = P + 64
            hs, dev = {}, {}
            for n in pasts:
                buf = ctx.to_device((0.1 * r.standard_normal((B, c["Hkv"], cap, c["D"]))).astype(np.float32))
                hs[n] = KvCacheHandle(buf, P, cap)
                dev[n] = buf.view((B, c["Hkv"], P, c["D"]), buf.strides)
            base = {"input_ids": ctx.to_device(r.integers(0, c["V"], (B, 1)).astype(np.int32)),
                    "attention_mask": ctx.to_device(np.ones((B, P + 1), np.int32))}
            feeds = {"in place": dict(base, **hs), "copying": dict(base, **dev)}
            times = {k: [] for k in feeds}
            launches = {}
            for k, f in feeds.items():  # warm-up
                m.run(f, names)
            ctx.sync()
            for _ in range(a.samples):
                for k, f in feeds.items():
                    n0 = ctx.launches
                    t0 = time.perf_counter()
                    for _ in range(a.steps):
                        out = m.run(f, names)
                    ctx.sync()
                    times[k].append((time.perf_counter() - t0) / a.steps * 1e6)
                    launches[k] = (ctx.launches - n0) // a.steps
                    del out
            cache = 2 * c["L"] * B * c["Hkv"] * P * c["D"] * 4
            bound = (wbytes + cache) / HBM * 1e6
            row = {"B": B, "P": P, "launches": launches, "bound_us": round(bound, 1)}
            for k, v in times.items():
                v = sorted(v)
                row[k] = {"median_us": round(v[len(v) // 2], 1), "min": round(v[0], 1), "max": round(v[-1], 1),
                          "hbm_share": round(bound / v[len(v) // 2], 3)}
            rows.append(row)
            print(json.dumps(row), flush=True)
            del hs, dev, feeds
    gen_rows = []
    for B in [int(x) for x in a.batches.split(",")]:
        prompt = r.integers(0, c["V"], (B, 16)).astype(np.int32)
        gen = Generator(ModelDecoder(m, B, 128)).with_prompt(prompt)
        next(gen)
        ctx.sync()
        t0 = time.perf_counter()
        for _ in range(64):
            next(gen)
        ctx.sync()
        dt = time.perf_counter() - t0
        gen_rows.append({"B": B, "tokens_per_s": round(64 * B / dt, 1)})
        print(json.dumps(gen_rows[-1]), flush=True)
    res = {"card": card, "config": c, "weight_bytes": wbytes, "steps": rows, "generator": gen_rows}
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
