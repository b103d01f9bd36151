"""Time com.microsoft MultiHeadAttention against the composed path a caller has without it (rten_b200_add for the q / k /
v bias, the new k / v copied into the cache with rten_b200_copy, then rten_b200_attention with an additive mask built
from the padding and causal masks) and against torch.nn.functional.scaled_dot_product_attention on the same heads
(attention alone: no bias adds, no cache copy), with CUDA events after warm-up, the implementations alternating.  Both
f32 modes are measured: 3xTF32 (default) with torch's allow_tf32 off, and single-pass TF32 with it on.

    python tools/mha_bench.py --out DIR [--repeats 7] [--iters 20]

Shapes: a ViT-B/16 encoder layer (batch 32, 197 tokens, 12 heads of 64, no mask); a BERT-base layer with the q / k / v
bias and a key_padding_mask (batch 16, 128 tokens, the last 16 of every other sequence padded); a Whisper-small decoder
self-attention decode step (batch 8, 12 heads of 64, bias, unidirectional, a 448-position cache extended in place); and
a cross-attention of 448 queries over 1500 encoder positions (batch 4, 12 heads of 64).  Prints the card name and power
limit with the numbers and writes one JSON line to DIR/mha_bench.json.  Needs an H100; there is no fallback."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                               text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


def _shape(rt, ctx, B, S, L, P, H, D, self_attn, bias, kpm, uni, rng):
    """Callables (mha, composed, sdpa) of one layer step and their outputs as [B, S, H * D] numpy getters.  With a past
    (P > 0) the caches hold P + L positions and every call writes the L new ones at P, in place."""
    import torch
    f = np.float32
    T = P + L
    hid = H * D
    q = ctx.to_device(rng.uniform(-1, 1, (B, S, hid)).astype(f))
    k = q if self_attn else ctx.to_device(rng.uniform(-1, 1, (B, L, hid)).astype(f))
    v = q if self_attn else ctx.to_device(rng.uniform(-1, 1, (B, L, hid)).astype(f))
    bvec = ctx.to_device(rng.uniform(-0.1, 0.1, 3 * hid).astype(f)) if bias else None
    mask = None
    if kpm:
        m = np.ones((B, T), np.int32)
        m[1::2, T - 16:] = 0
        mask = ctx.to_device(m)
    args = dict(bias=bvec, key_padding_mask=mask)
    if P:
        kc = ctx.to_device(rng.uniform(-1, 1, (B, H, T, D)).astype(f))
        vc = ctx.to_device(rng.uniform(-1, 1, (B, H, T, D)).astype(f))
        st = (H * T * D, T * D, D, 1)
        args.update(past_key=kc.view((B, H, P, D), st), past_value=vc.view((B, H, P, D), st), present_key=kc, present_value=vc)
    op = rt.MultiHeadAttention(H, unidirectional=uni)
    out_m = ctx.empty((B, S, hid))

    def mha():
        op.run(ctx, q, None if self_attn else k, None if self_attn else v, out=out_m, want_present=bool(P), **args)

    # the composed path
    add = rt.Add()
    qb, kb, vb = (ctx.empty((B, n, hid)) for n in (S, L, L))
    bq, bk, bv = ((bvec.view((hid,), (1,), i * hid)) for i in range(3)) if bias else (None, None, None)
    heads = lambda t, n: t.view((B, H, n, D), (n * hid, D, hid, 1))
    additive = np.zeros((B, 1, S, T), f)
    if kpm:
        additive[:, :, :, :] = np.where(m[:, None, None, :] == 0, -10000.0, 0.0)
    if uni:
        additive[:, :, np.triu(np.ones((S, T), bool), P + 1)] = -10000.0
    dmask = ctx.to_device(additive) if (kpm or uni) else None
    att = rt.Attention()
    out_c = ctx.empty((B, S, hid))
    out_heads = heads(out_c, S)
    if P:
        k_slot, v_slot = kc.view((B, H, L, D), st, P * D), vc.view((B, H, L, D), st, P * D)

    def composed():
        qq, kk, vv = q, k, v
        if bias:
            add.run(ctx, q, bq, out=qb)
            add.run(ctx, k, bk, out=kb)
            add.run(ctx, v, bv, out=vb)
            qq, kk, vv = qb, kb, vb
        if P:
            k_slot.assign(heads(kk, L))
            v_slot.assign(heads(vv, L))
            kh, vh = kc, vc
        else:
            kh, vh = heads(kk, L), heads(vv, L)
        att.run(ctx, heads(qq, S), kh, vh, attn_mask=dmask, out=out_heads)

    # torch SDPA on the same heads (attention alone)
    tq = torch.from_numpy(q.numpy()).cuda().view(B, S, H, D).transpose(1, 2)
    tk = (torch.from_numpy(kc.numpy()).cuda() if P else torch.from_numpy(k.numpy()).cuda().view(B, L, H, D).transpose(1, 2))
    tv = (torch.from_numpy(vc.numpy()).cuda() if P else torch.from_numpy(v.numpy()).cuda().view(B, L, H, D).transpose(1, 2))
    tmask = torch.from_numpy(additive).cuda() if (kpm or uni) else None

    def sdpa():
        torch.nn.functional.scaled_dot_product_attention(tq, tk, tv, attn_mask=tmask)

    return mha, composed, sdpa, (lambda: out_m.numpy(), lambda: out_c.numpy())


def _stats(ts):
    ts = sorted(ts)
    return dict(median_us=ts[len(ts) // 2], min_us=ts[0], max_us=ts[-1])


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--out", required=True, help="directory for mha_bench.json")
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("mha_bench: no CUDA device; this benchmark measures the H100 kernels and has no fallback")
    import rten_b200 as rt
    card, power = _card()
    stream = torch.cuda.Stream()
    ctx = rt.Context(0, stream=stream.cuda_stream)
    rng = np.random.default_rng(0)
    shapes = [("vit_b16_encoder", dict(B=32, S=197, L=197, P=0, H=12, D=64, self_attn=True, bias=False, kpm=False, uni=False)),
              ("bert_base_bias_padding", dict(B=16, S=128, L=128, P=0, H=12, D=64, self_attn=True, bias=True, kpm=True, uni=False)),
              ("whisper_small_decode", dict(B=8, S=1, L=1, P=447, H=12, D=64, self_attn=False, bias=True, kpm=False, uni=True)),
              ("cross_448_over_1500", dict(B=4, S=448, L=1500, P=0, H=12, D=64, self_attn=False, bias=False, kpm=False, uni=False))]
    results = []
    for mode in ("3xtf32", "tf32"):
        ctx.set_f32_mode(mode == "3xtf32")
        torch.backends.cuda.matmul.allow_tf32 = mode == "tf32"
        torch.backends.cudnn.allow_tf32 = mode == "tf32"
        for sname, s in shapes:
            mha, composed, sdpa, (get_m, get_c) = _shape(rt, ctx, rng=rng, **s)
            impls = [("mha", mha), ("composed", composed), ("torch_sdpa", sdpa)]
            times = {n: [] for n, _ in impls}
            with torch.cuda.stream(stream):
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
            ym, yc = get_m().astype(np.float64), get_c().astype(np.float64)
            diff = float(np.abs(ym - yc).max() / np.abs(yc).max())
            row = dict(shape=sname, mode=mode, **s, rel_diff_vs_composed=diff, **{n: _stats(ts) for n, ts in times.items()})
            row["speedup_vs_composed"] = row["composed"]["median_us"] / row["mha"]["median_us"]
            print(f"{card} (power limit {power}) {mode:6s} {sname:23s}: mha {row['mha']['median_us']:8.1f} us "
                  f"[{row['mha']['min_us']:.1f}, {row['mha']['max_us']:.1f}]  composed {row['composed']['median_us']:8.1f} us  "
                  f"torch sdpa {row['torch_sdpa']['median_us']:8.1f} us  x{row['speedup_vs_composed']:.2f} vs composed  rel diff {diff:.1e}")
            results.append(row)
    line = json.dumps(dict(tool="mha_bench", card=card, power_limit=power, repeats=a.repeats, iters=a.iters, results=results))
    print(line)
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "mha_bench.json"), "w") as f:
        f.write(line + "\n")


if __name__ == "__main__":
    main()
