"""`pytest -m gpu`: the single-query attention kernels (skinny.cu attn_decode_kernel / attn_decode_mha_kernel) and the
MatMulNBits kernels (nbits.cu nbits_skinny_kernel / nbits_wgmma_kernel) -- the two kernel families every token of an
int4 decoder runs -- each selected by name and checked bit for bit.

The launchers pick an instance, a split count and a grid from the shapes and the SM count.  The rules are restated below
(`decode_rule`, `decode_splits`, `nbits_rule`); `VARIANTS` lists every instance they pick from
(tests/test_decode_step_kernel_table_cpu.py keeps it equal to the built library's symbols).  `DECODE_EDGES` and
`NBITS_EDGES` list the branches of those rules that a name does not show; the case lists reach each of them, and every
instance at least twice, on 132 and on 114 SMs.

  * kernel identity: every case runs once under CUPTI in a child process; each must run exactly the instance its rule
    names (kernels of other files, such as the rotary / append kernel MultiHeadAttention's bias runs first, are not
    claimed), every entry of `VARIANTS` must have run, and each decode launch must have B * q_heads * nsplit CTAs of
    nw * 32 threads (the grid and block Kineto's trace records for the kernel);
  * decode attention against `decode_model`, a float32 restatement of attn_decode_body's operation order: per warp the
    8-lane fma chains of q . k, the xor-4/2/1 butterfly, `* scale` and `+ mask` as two roundings (cuobjdump -sass shows
    an FMUL by the scale and a separate FADD of the mask in every instance: the mask load sits in its own branch, so
    nvcc does not contract them), MultiHeadAttention's fill, the warp max, oracle rto_reduced_range_exp1 of s - max,
    per-lane sums and the xor-8/16 butterfly; the value product as per-4-position fma chains and an xor-1/2 reduction
    (transposed V) or one 16-position fma chain (natural V); the warp merge and the split merge as fma chains in warp
    and split order; num / den with NaN -> 0.  Every fused multiply-add is oracle/norms.py fma_f32 (exactly rounded).
    Cache positions at or past the valid length, and a transposed V's row padding, hold NaN, so a finite bit-exact
    result also proves the kernel never folds them in; fused appends must write exactly cache row len - 1.  The model
    itself is pinned to float64 attention on the CPU (test_decode_step_kernel_table_cpu.py);
  * MatMulNBits: the skinny kernel against `skinny_model` (each lane's fma chain over its 16-byte units in k order, the
    xor-16/8/4/2/1 butterfly), the wgmma kernel in both f32 modes exactly on integer-valued operands (A in [-8, 8],
    scales 2^e for e in [-3, 0], K = 784: every partial sum is a multiple of 2^-3 below 2^16, exact in TF32 and in f32)
    and within the TF32 bounds of gpu_checks on random ones; outputs into views with an odd row pitch 4 bytes past an
    8-byte boundary (the epilogue's scalar stores), whose surroundings must stay untouched."""
import ctypes
import json
import os
import tempfile

import numpy as np
import pytest

import gpu_checks as gc
import test_gpu_conv_norm_resize_kernels as ck
import test_gpu_row_kernels as rk
from test_gpu_matmul_nbits import _exact, dequantize_nbits, pack_nbits

pytestmark = pytest.mark.gpu

F32, I32 = np.float32, np.int32
FLT_MAX = np.finfo(F32).max
CHUNK = {8: 128, 6: 96}  # cached positions per split: 16 per warp (ATTN_CHUNK)

# ---- the kernels ------------------------------------------------------------------------------------------------------
VARIANTS = {
    "attn_decode_kernel": [(64, 6, 0), (64, 8, 0), (128, 8, 0), (64, 6, 1), (64, 8, 1), (128, 8, 1)],  # <DH, NW, EXT>
    "attn_decode_mha_kernel": [(64, 6), (64, 8), (128, 8)],  # <DH, NW>
    "nbits_skinny_kernel": [(8, 4), (16, 4), (32, 2)],  # <MT, CPW>
    "nbits_wgmma_kernel": [(0,), (1,)],  # <X3>
}
KERNELS = set(VARIANTS)
FAMILY_KERNELS = {"decode": ("attn_decode_kernel", "attn_decode_mha_kernel"),
                  "nbits": ("nbits_skinny_kernel", "nbits_wgmma_kernel")}
DECODE_EDGES = ("one split", "16-split floor", "8192 positions dh 64", "8192 positions dh 128",
                "six warps, more than 64 splits", "empty split", "len 0", "window skip 1", "window skip 2",
                "window skip 3", "more than 1024 pairs, several splits", "transposed V", "natural V", "append",
                "append with rotary", "interleaved rotary", "mask", "GQA group 1", "GQA group 4", "GQA group 8",
                "key padding mask", "vis_end fill")
NBITS_EDGES = tuple(f"skinny {mt} {e}" for mt in (8, 16, 32) for e in ("grid-stride loop", "N % (8 CPW) != 0")) + (
    "K % 32 == 16, K < 1024", "K % 32 == 16, partial last chunk of 1024") + tuple(f"block {b}" for b in (16, 32, 64, 128, 256, 512)) + (
    "wgmma M % 128 != 0", "wgmma partial raster group", "wgmma K > 256, K % 256 != 0", "wgmma K % 32 == 16",
    "wgmma M = 1", "M = 32", "M = 33", "scalar stores")


def kernel_key(name, kernels=KERNELS):
    return ck.kernel_key(name, kernels)


def _cdiv(a, b):
    return -(-a // b)


# ---- decode attention: the launch rule ---------------------------------------------------------------------------------
def _splits_for(cap, bh, sms, chunk):
    """skinny.cu launch_attn_decode splits_for: (nsplit, set by the 16-split floor, raised by the while loop).  The loop
    never raises it (test_decode_step_kernel_table_cpu checks every cache length): the count is at least ceil(cap /
    chunk), so ceil(cap / count) rounded up to 4 stays within a chunk, itself a multiple of 4."""
    ns = _cdiv(cap, chunk)
    floor = min(16, _cdiv(2 * sms, bh))
    ns = max(ns, floor)
    ns = max(1, min(ns, max(1, _cdiv(cap, 16))))
    set_by_floor = ns == floor and floor > _cdiv(cap, chunk)
    before = ns
    while ((_cdiv(cap, ns) + 3) & ~3) > chunk:
        ns += 1
    return ns, set_by_floor, ns > before


def decode_rule(B, q_heads, dh, cap, ext, mha, sms):
    """skinny.cu launch_attn_decode: ((kernel, template arguments), nw, nsplit).  A split covers at most 128 positions
    (rounded to 4), more splits when B * q_heads alone leaves SMs idle (at least min(16, ceil(2 SMs / pairs)), at most one
    per 16 positions); at dh 64 the six-warp variant (96-position splits, four CTAs per SM against three) runs when its
    grid needs fewer waves."""
    bh = B * q_heads
    nw, ns = 8, _splits_for(cap, bh, sms, 128)[0]
    if dh == 64:
        ns6 = _splits_for(cap, bh, sms, 96)[0]
        if _cdiv(bh * ns6, 4 * sms) < _cdiv(bh * ns, 3 * sms):
            nw, ns = 6, ns6
    key = ("attn_decode_mha_kernel", (dh, nw)) if mha else ("attn_decode_kernel", (dh, nw, int(ext)))
    return key, nw, ns


def decode_splits(length, lo, ns):
    """attn_decode_body's split arithmetic for one (batch, head): (base, per, [(l0, l1, skip)] per split) -- the splits
    cover [base, length), base = the window's first position rounded down to 4, per a multiple of 4; `skip` positions of
    a split lie below the window"""
    base = lo & ~3
    per = ((length - base + ns - 1) // ns + 3) & ~3
    out = []
    for sp in range(ns):
        l0 = min(length, base + sp * per)
        l1 = min(length, l0 + per)
        out.append((l0, l1, max(0, lo - l0)))
    return base, per, out


def _dims(s):
    return s["B"], s["qh"], s["kvh"], s["dh"], s["cap"]


def decode_lens(s):
    """valid positions per batch (the appended one included) and the window's first position"""
    B, cap = s["B"], s["cap"]
    lens = np.array(s["lens"] if s.get("lens") is not None else [cap] * B, np.int64)
    lo = np.maximum(0, lens - s["window"]) if s.get("window") else np.zeros(B, np.int64)
    return lens, lo


def _is_ext(s):
    return s["op"] == "gqa"  # GroupQueryAttention's decode step always sets the len offset / floor


def decode_case_rule(s, sms):
    B, qh, kvh, dh, cap = _dims(s)
    key, nw, ns = decode_rule(B, qh, dh, cap, _is_ext(s), s["op"] == "mha", sms)
    bh = B * qh
    edges = set()
    chunk = CHUNK[nw]
    _, by_floor, _ = _splits_for(cap, bh, sms, chunk)
    if ns == 1:
        edges.add("one split")
    if by_floor:
        edges.add("16-split floor")
    if cap == 8192:
        edges.add(f"8192 positions dh {dh}")
    if nw == 6 and ns > 64:
        edges.add("six warps, more than 64 splits")
    lens, lo = decode_lens(s)
    for b in range(B):
        _, _, parts = decode_splits(int(lens[b]), int(lo[b]), ns)
        if ns > 1 and any(l1 == l0 for l0, l1, _ in parts):
            edges.add("empty split")
        if parts[0][2]:
            edges.add(f"window skip {parts[0][2]}")
    if (lens == 0).any():
        edges.add("len 0")
    if bh > 1024 and ns > 1:
        edges.add("more than 1024 pairs, several splits")
    edges.add("transposed V" if s.get("vt") else "natural V")
    if s.get("append") or s["op"] == "gqa":
        edges.add("append with rotary" if s.get("rot") else "append")
    if s.get("rot") == "inter":
        edges.add("interleaved rotary")
    if s.get("mask"):
        edges.add("mask")
    if s["op"] != "mha":
        edges.add(f"GQA group {qh // kvh}")
    if s.get("kpm"):
        edges.add("key padding mask")
    if s.get("L") and s.get("unidir"):
        edges.add("vis_end fill")
    return key, nw, ns, edges


def _batches_for_six_warps(qh, cap, sms):
    """the smallest batch at which `qh` heads over `cap` positions take the six-warp kernel"""
    for B in range(1, 400):
        if decode_rule(B, qh, 64, cap, False, False, sms)[1] == 6:
            return B
    raise AssertionError(f"no batch takes six warps at {qh} heads, {cap} positions, {sms} SMs")


def decode_specs(sms):
    d = lambda op, B, qh, kvh, dh, cap, **kw: dict(op=op, B=B, qh=qh, kvh=kvh, dh=dh, cap=cap, **kw)  # noqa: E731
    six = lambda qh, cap: _batches_for_six_warps(qh, cap, sms)  # noqa: E731
    specs = [
        # ONNX Attention (the plain kernel): both value layouts, masks, nonpad lengths, the fused append, GQA groups
        d("attn", 2, 4, 4, 64, 64, lens=(5, 64), mask=True),  # the floor caps at 4 splits: two empty ones for len 5
        d("attn", 1, 8, 1, 64, 300, lens=(300,), vt=True),
        d("attn", 3, 8, 2, 128, 200, lens=(0, 1, 199), vt=True, mask=True, append=True),  # len 0, len 1
        d("attn", 2, 16, 2, 128, 1000, lens=(777, 1000), append=True),
        d("attn", 2, 2, 2, 128, 8192, lens=(8192, 4099), vt=True, rows=(0, 3)),
        d("attn", 1, 2, 1, 64, 8192, lens=(8190,), mask=True, append=True),
        d("attn", six(12, 576), 12, 12, 64, 576, lens=None, vt=True, rows=(0, 1, -2, -1)),  # GPT-2's decode step
        d("attn", six(12, 576), 12, 4, 64, 576, lens="ragged", mask=True, append=True, rows=(0, 5, -6, -1)),
        d("attn", 1, 1, 1, 64, 7, lens=(7,)),  # one split
        d("attn", 4, 32, 8, 64, 40, lens=(40, 3, 17, 33), vt=True),  # one split of 40 positions
        # GroupQueryAttention (the EXT kernel): natural caches extended in place, rotary, windows
        d("gqa", 2, 8, 2, 64, 130, lens=(70, 130), rot="half"),
        d("gqa", 3, 8, 1, 128, 517, lens=(1, 200, 517), rot="inter", mask=True),
        d("gqa", 2, 4, 4, 64, 400, lens=(400, 122), window=37, rot="half"),  # skip 3, 1
        d("gqa", 2, 4, 1, 128, 300, lens=(90, 300), window=64, mask=True),  # skip 2 (lo 26), 0
        d("gqa", 1, 16, 2, 128, 2500, lens=(2389,), window=1000, rot="inter"),
        d("gqa", six(2, 8155), 2, 1, 64, 8155, lens="ragged", rows=(0, -1)),  # six warps, 85 splits
        d("gqa", six(4, 4000), 4, 1, 64, 4000, lens="ragged", rot="half", rows=(0, 1, -1)),
        # MultiHeadAttention (the MHA kernel): key padding mask and vis_end fill
        d("mha", 2, 4, 4, 64, 100, kpm=True, mask=True),
        d("mha", 1, 2, 2, 128, 333, kpm=True),
        d("mha", 2, 3, 3, 64, 9, L=9, unidir=True),  # no past: vis_end 1
        d("mha", six(12, 576), 12, 12, 64, 576, kpm=True, rows=(0, 1, -1)),
        d("mha", 1, 8, 8, 128, 64, L=64, unidir=True, mask=True),
        d("mha", six(12, 576), 12, 12, 64, 576, L=576, mask=True, rows=(0, 40, -1)),
        # more than 1024 (batch, head) pairs with several splits: the counters grow past their first 1024
        d("attn", 33, 32, 8, 64, 300, lens="ragged", rows=(0, 1, 31, 500, -1)),
        d("gqa", 33, 32, 4, 128, 260, lens="ragged", rot="half", rows=(0, 777, -1)),
    ]
    for s in specs:  # "ragged": one valid length in 1 ..= cap per batch
        if s.get("lens") == "ragged":
            s["lens"] = tuple(int(v) for v in _rng("lens", s["B"], s["cap"]).integers(1, s["cap"] + 1, s["B"]))
    return specs


# ---- decode attention: the model ---------------------------------------------------------------------------------------
_RRE = None


def rre(x):
    """oracle rto_reduced_range_exp1 of every element (the reference's exp polynomial, as math.cuh restates it)"""
    global _RRE
    if _RRE is None:
        from oracle import oracle
        _RRE = oracle.lib().rto_reduced_range_exp1
        _RRE.restype = ctypes.c_float
        _RRE.argtypes = [ctypes.c_float]
    x = np.asarray(x, F32)
    return np.array([_RRE(float(v)) for v in x.ravel()], F32).reshape(x.shape)


def _fma(a, b, c):
    from oracle.norms import fma_f32
    return fma_f32(a, b, c)


def decode_model(q, K, V, lens, lo, scale, nw, ns, vt, mask=None, fill_at=None, fill=0.0, perturb=()):
    """attn_decode_body in float32 for R (batch, head) rows: q [R, dh], K / V [R, cap, dh] (the rows the head reads, the
    appended position already in place), lens / lo [R], mask / fill_at [R, cap] (additive mask; positions that score
    `fill`) or None.  `perturb` names deliberate departures from the kernel's order (the suite checks that each one
    changes the result): "butterfly" swaps two levels of the score butterfly, "mul-add" rounds the score chain's
    product and sum separately, "splits" merges the splits in reverse order."""
    q, K, V = (np.asarray(a, F32) for a in (q, K, V))
    R, cap, dh = K.shape
    P = dh // 8
    C = nw * 16
    lens, lo = np.asarray(lens, np.int64), np.asarray(lo, np.int64)
    base = lo & ~3
    per = ((lens - base + ns - 1) // ns + 3) & ~3
    l0 = np.minimum(lens[:, None], base[:, None] + np.arange(ns)[None, :] * per[:, None])  # [R, ns]
    nl = np.minimum(lens[:, None], l0 + per[:, None]) - l0
    skip = np.maximum(0, lo[:, None] - l0)
    i = np.arange(C)
    inr = i[None, None, :] < nl[:, :, None]  # [R, ns, C]: positions of the split
    valid = inr & (i[None, None, :] >= skip[:, :, None])
    pos = np.where(inr, l0[:, :, None] + i, 0)
    rows = np.arange(R)[:, None, None]
    # scores: lane l8 of a position's 8 runs an fma chain over elements l8 P .. l8 P + P - 1; xor-4/2/1 butterfly
    Kg = K[rows, pos].reshape(R, ns, C, 8, P)
    qr = q.reshape(R, 1, 1, 8, P)
    part = np.zeros((R, ns, C, 8), F32)
    for t in range(P):
        if "mul-add" in perturb:
            part = (qr[..., t] * Kg[..., t] + part).astype(F32)
        else:
            part = _fma(qr[..., t], Kg[..., t], part)
    lanes = np.arange(8)
    for o in ((2, 4, 1) if "butterfly" in perturb else (4, 2, 1)):
        part = part + part[..., lanes ^ o]
    with np.errstate(invalid="ignore", over="ignore"):
        s = np.where(inr, part[..., 0], F32(0)) * F32(scale)
        if mask is not None:
            s = s + np.asarray(mask, F32)[rows, pos]
        if fill_at is not None:
            s = np.where(np.asarray(fill_at)[rows, pos], F32(fill), s)
    s = s.astype(F32).reshape(R, ns, nw, 16)
    vw = valid.reshape(R, ns, nw, 16)
    # softmax pieces per warp: max, exponentials, lane sums (lane `sub` holds positions 4 it + sub), xor-8/16 butterfly
    mw = np.where(vw, s, -FLT_MAX).max(-1)
    e = np.zeros_like(s)
    e[vw] = rre((s - mw[..., None])[vw])
    e4 = e.reshape(R, ns, nw, 4, 4)
    lane = e4[..., 0, :]
    for it in range(1, 4):
        lane = lane + e4[..., it, :]
    sw = (lane[..., 0] + lane[..., 1]) + (lane[..., 2] + lane[..., 3])
    # the warp's unnormalised output
    Vg = V[rows, pos].reshape(R, ns, nw, 16, dh)
    inr4 = inr.reshape(R, ns, nw, 16)
    with np.errstate(invalid="ignore"):
        if vt:  # lane (channel, f4): an fma chain over positions 4 f4 .. 4 f4 + 3, then xor-1/2 over f4
            a = np.zeros((R, ns, nw, 4, dh), F32)
            for c in range(4):
                idx = 4 * np.arange(4) + c
                a = np.where(inr4[..., idx, None], _fma(e[..., idx, None], Vg[..., idx, :], a), a)
            o = (a[..., 0, :] + a[..., 1, :]) + (a[..., 2, :] + a[..., 3, :])
        else:  # lane owns channels: one fma chain over the warp's 16 positions
            o = np.zeros((R, ns, nw, dh), F32)
            for k in range(16):
                o = np.where(vw[..., k, None], _fma(e[..., k, None], Vg[..., k, :], o), o)
    # merge the warps (an fma chain in warp order), then the splits (in split order)
    s_m = np.where(np.arange(nw)[None, None, :] * 16 < nl[:, :, None], mw, -FLT_MAX).astype(F32)
    m = np.maximum(s_m.max(-1), -FLT_MAX).astype(F32)
    ew = rre(s_m - m[..., None])
    den = np.zeros((R, ns), F32)
    num = np.zeros((R, ns, dh), F32)
    for w in range(nw):
        den = _fma(sw[..., w], ew[..., w], den)
        num = _fma(o[..., w, :], ew[..., w, None], num)
    if ns == 1:
        nn, dd = num[:, 0], den[:, 0]
    else:
        mm = np.maximum(m.max(-1), -FLT_MAX).astype(F32)
        es = rre(m - mm[:, None])
        nn, dd = np.zeros((R, dh), F32), np.zeros(R, F32)
        for sp in (reversed(range(ns)) if "splits" in perturb else range(ns)):
            dd = _fma(den[:, sp], es[:, sp], dd)
            nn = _fma(num[:, sp], es[:, sp, None], nn)
    with np.errstate(invalid="ignore", divide="ignore"):
        r = (nn / dd[:, None]).astype(F32)
    return np.where(np.isnan(r), F32(0), r)


# ---- decode attention: cases -------------------------------------------------------------------------------------------
def _rng(*key):
    return rk._rng("decode_step", *key)


def _key(s):
    return sorted((k, str(v)) for k, v in s.items())


def decode_prepare(s):
    """inputs, caches with NaN at and past each batch's valid length (the appended row included: the kernel must take
    the new key / value for it), and the model's view of them"""
    B, qh, kvh, dh, cap = _dims(s)
    r = _rng("decode", _key(s))
    lens, lo = decode_lens(s)
    inp = dict(spec=s, lens=lens, lo=lo)
    inp["q"] = r.uniform(-1, 1, (B, qh, dh)).astype(F32)
    K = r.uniform(-1, 1, (B, kvh, cap, dh)).astype(F32)
    V = r.uniform(-1, 1, (B, kvh, cap, dh)).astype(F32)
    append = s.get("append") or s["op"] == "gqa"
    if s["op"] != "mha":
        for b in range(B):
            K[b, :, max(0, lens[b] - 1 if append else lens[b]):] = np.nan
            V[b, :, max(0, lens[b] - 1 if append else lens[b]):] = np.nan
    inp["K"], inp["V"] = K, V
    if append:
        inp["kn"] = r.uniform(-1, 1, (B, kvh, dh)).astype(F32)
        inp["vn"] = r.uniform(-1, 1, (B, kvh, dh)).astype(F32)
    if s.get("mask"):
        inp["mask"] = r.uniform(-3, 3, (B, qh, cap)).astype(F32)
    if s.get("rot"):
        inp["cos"] = r.uniform(-1, 1, (cap, dh // 2)).astype(F32)
        inp["sin"] = r.uniform(-1, 1, (cap, dh // 2)).astype(F32)
    if s.get("kpm"):
        kpm = (r.random((B, cap)) < 0.7).astype(I32)
        kpm[0, :] = 0  # a fully padded row: every position scores the fill value
        inp["kpm"] = kpm
    return inp


def transposed_v(V):
    """[B, kvh, cap, dh] -> the host buffer of a transposed value cache [B, kvh, dh, pitch]: rows padded with NaN to a
    multiple of 4 past cap, and 4 more"""
    B, kvh, cap, dh = V.shape
    buf = np.full((B, kvh, dh, (cap + 3) // 4 * 4 + 4), np.nan, F32)
    buf[..., :cap] = V.transpose(0, 1, 3, 2)
    return buf


def decode_launch(rt, ctx, inp, out=None, dev=None):
    """run the case once (on the device tensors `dev` of an earlier call, else new ones); (output [B, qh, 1, dh] or
    [B, 1, qh dh], the device tensors: "kc" / "vc" the K and V cache buffers when there are)"""
    s = inp["spec"]
    B, qh, kvh, dh, cap = _dims(s)
    dev = {} if dev is None else dev
    if s["op"] == "attn":
        if not dev:
            dev["kc"] = ctx.to_device(inp["K"])
            if s.get("vt"):
                dev["vc"] = ctx.to_device(transposed_v(inp["V"]))
                pitch = dev["vc"].shape[-1]
                dev["v"] = dev["vc"].view((B, kvh, cap, dh), (kvh * dh * pitch, dh * pitch, 1, pitch))
            else:
                dev["vc"] = dev["v"] = ctx.to_device(inp["V"])
            dev["q"] = ctx.to_device(inp["q"][:, :, None, :])
            if s.get("lens") is not None:
                dev["nonpad_kv_seqlen"] = ctx.to_device(inp["lens"].astype(I32))
            if "mask" in inp:
                dev["attn_mask"] = ctx.to_device(inp["mask"][:, :, None, :])
            if "kn" in inp:
                dev["new_key"] = ctx.to_device(inp["kn"][:, :, None, :])
                dev["new_value"] = ctx.to_device(inp["vn"][:, :, None, :])
        kw = {k: dev[k] for k in ("nonpad_kv_seqlen", "attn_mask", "new_key", "new_value") if k in dev}
        return rt.Attention().run(ctx, dev["q"], dev["kc"], dev["v"], out=out, **kw), dev
    if s["op"] == "gqa":
        kd, vd = ctx.to_device(inp["K"]), ctx.to_device(inp["V"])
    if s["op"] == "gqa":
        kd, vd = ctx.to_device(inp["K"]), ctx.to_device(inp["V"])
        st = (kvh * cap * dh, cap * dh, dh, 1)
        op = rt.GroupQueryAttention(qh, kvh, do_rotary=bool(s.get("rot")), rotary_interleaved=s.get("rot") == "inter",
                                    local_window_size=s.get("window") or -1)
        kw = {}
        if s.get("rot"):
            kw["cos_cache"], kw["sin_cache"] = ctx.to_device(inp["cos"]), ctx.to_device(inp["sin"])
        if "mask" in inp:
            kw["attention_bias"] = ctx.to_device(inp["mask"][:, :, None, :])
        y, _, _ = op.run(ctx, ctx.to_device(inp["q"].reshape(B, 1, qh * dh)), ctx.to_device(inp["kn"].reshape(B, 1, kvh * dh)),
                         ctx.to_device(inp["vn"].reshape(B, 1, kvh * dh)), ctx.to_device((inp["lens"] - 1).astype(I32)), cap,
                         past_key=kd.view((B, kvh, cap - 1, dh), st), past_value=vd.view((B, kvh, cap - 1, dh), st),
                         present_key=kd, present_value=vd, out=out, **kw)
        return y, dict(kc=kd, vc=vd)
    # MultiHeadAttention: a past cache of cap - 1 positions extended in place, or (L) one query over L keys, no past
    op = rt.MultiHeadAttention(qh, unidirectional=bool(s.get("unidir")))
    kw = {}
    if "mask" in inp:
        kw["attention_bias"] = ctx.to_device(inp["mask"][:, :, None, :])
    if "kpm" in inp:
        kw["key_padding_mask"] = ctx.to_device(inp["kpm"])
    q = ctx.to_device(inp["q"].reshape(B, 1, qh * dh))
    if s.get("L"):
        k = ctx.to_device(np.ascontiguousarray(inp["K"].transpose(0, 2, 1, 3).reshape(B, cap, qh * dh)))
        v = ctx.to_device(np.ascontiguousarray(inp["V"].transpose(0, 2, 1, 3).reshape(B, cap, qh * dh)))
        y, _, _ = op.run(ctx, q, k, v, out=out, want_present=False, **kw)
        return y, {}
    kd, vd = ctx.to_device(inp["K"]), ctx.to_device(inp["V"])
    st = (qh * cap * dh, cap * dh, dh, 1)
    y, _, _ = op.run(ctx, q, ctx.to_device(inp["K"][:, :, -1].reshape(B, 1, qh * dh)), ctx.to_device(inp["V"][:, :, -1].reshape(B, 1, qh * dh)),
                     past_key=kd.view((B, qh, cap - 1, dh), st), past_value=vd.view((B, qh, cap - 1, dh), st),
                     present_key=kd, present_value=vd, out=out, **kw)
    return y, dict(kc=kd, vc=vd)


def decode_model_inputs(inp, rows=None):
    """the model's inputs for the (batch, head) rows `rows` (flat b * qh + h; default all): q and the appended key rotated
    as the kernel rotates them, the appended row in place, the window, the mask and MultiHeadAttention's fill"""
    from test_gpu_group_query_attention import rotary_ref
    s = inp["spec"]
    B, qh, kvh, dh, cap = _dims(s)
    lens, lo = inp["lens"], inp["lo"]
    q, K, V = inp["q"].copy(), inp["K"].copy(), inp["V"].copy()
    if s.get("rot"):
        pos = np.clip(lens - 1, 0, cap - 1)
        c, sn = inp["cos"][pos][:, None, None, :], inp["sin"][pos][:, None, None, :]
        inter = s["rot"] == "inter"
        q = rotary_ref(q[:, :, None, :], c, sn, inter, dtype=F32)[:, :, 0]
        inp_kn = rotary_ref(inp["kn"][:, :, None, :], c, sn, inter, dtype=F32)[:, :, 0]
    else:
        inp_kn = inp.get("kn")
    if "kn" in inp:
        for b in range(B):
            if lens[b] > 0:
                K[b, :, lens[b] - 1] = inp_kn[b]
                V[b, :, lens[b] - 1] = inp["vn"][b]
    inp["k_written"] = inp_kn
    rows = np.arange(B * qh) if rows is None else np.asarray(rows) % (B * qh)
    b, h = rows // qh, rows % qh
    hk = h // (qh // kvh)
    mask = inp["mask"][b, h] if "mask" in inp else None
    fill_at = None
    if s["op"] == "mha":
        vis_end = 1 if s.get("L") and s.get("unidir") else cap
        fill_at = np.arange(cap)[None, :] >= vis_end
        if "kpm" in inp:
            fill_at = fill_at | (inp["kpm"][b] == 0)
        fill_at = np.broadcast_to(fill_at, (len(rows), cap))
    scale = F32(1) / np.sqrt(F32(dh))
    return dict(q=q[b, h], K=K[b, hk], V=V[b, hk], lens=lens[b], lo=lo[b], scale=scale, vt=bool(s.get("vt")), mask=mask,
                fill_at=fill_at, fill=F32(-10000.0)), rows


def decode_want(inp, sms, perturb=()):
    s = inp["spec"]
    _, nw, ns, _ = decode_case_rule(s, sms)
    mi, rows = decode_model_inputs(inp, s.get("rows"))
    return decode_model(nw=nw, ns=ns, perturb=perturb, **mi), rows


# ---- MatMulNBits: the launch rule and the model --------------------------------------------------------------------
def nbits_rule(M, K, N, block, x3, sms, skinny_max=32):
    """nbits.cu launch_nbits: up to `skinny_max` rows (32, RTEN_B200_NBITS_SKINNY_MAX) the skinny kernel, 8 / 16 / 32 row
    tiles with 4 / 4 / 2 columns per warp, one CTA per 8 CPW columns up to 2 per SM (a grid-stride loop over the rest);
    above it one wgmma CTA per 128 x 128 output tile.  (instance, tiles, grid, tiles of the busiest CTA)"""
    if M <= skinny_max:
        mt = 8 if M <= 8 else 16 if M <= 16 else 32
        cpw = 2 if mt == 32 else 4
        tiles = _cdiv(N, 8 * cpw)
        grid = min(tiles, 2 * sms)
        return ("nbits_skinny_kernel", (mt, cpw)), tiles, grid, _cdiv(tiles, grid)
    tiles = _cdiv(M, 128) * _cdiv(N, 128)
    return ("nbits_wgmma_kernel", (int(x3),)), tiles, tiles, 1


def nbits_edges(s, sms):
    M, K, N, block = s["M"], s["K"], s["N"], s["block"]
    assert K % block == 0, f"{spec_id('nbits', s)}: K is not a whole number of blocks"
    (k, a), tiles, grid, busiest = nbits_rule(M, K, N, block, s["x3"], sms, s.get("skinny_max", 32))
    e = {f"block {block}"}
    if k == "nbits_skinny_kernel":
        if busiest > 1:
            e.add(f"skinny {a[0]} grid-stride loop")
        if N % (8 * a[1]):
            e.add(f"skinny {a[0]} N % (8 CPW) != 0")
        if K % 32 == 16:
            e.add("K % 32 == 16, K < 1024" if K < 1024 else "K % 32 == 16, partial last chunk of 1024")
    else:
        mtiles = _cdiv(M, 128)
        if M % 128:
            e.add("wgmma M % 128 != 0")
        if mtiles > 8 and mtiles % 8:
            e.add("wgmma partial raster group")
        if K > 256 and K % 256:
            e.add("wgmma K > 256, K % 256 != 0")
        if K % 32 == 16:
            e.add("wgmma K % 32 == 16")
        if M == 1:
            e.add("wgmma M = 1")
    if M in (32, 33) and s.get("skinny_max") is None:
        e.add(f"M = {M}")
    if s.get("view") and k == "nbits_wgmma_kernel":
        e.add("scalar stores")
    return e


def nbits_specs(sms):
    n = lambda M, K, N, block, x3=True, **kw: dict(M=M, K=K, N=N, block=block, x3=x3, **kw)  # noqa: E731
    return [
        # skinny: every tile height, a grid-stride loop and a ragged last column tile, K % 32 == 16 on both sides of 1024
        n(5, 1072, 8520, 16, cols=256), n(3, 48, 70, 16), n(8, 1024, 200, 32, view=True), n(1, 512, 96, 64),
        n(16, 1072, 8520, 16, cols=256), n(9, 2560, 300, 512), n(12, 176, 77, 16), n(13, 1024, 130, 128, view=True),
        n(32, 1072, 4300, 16, cols=256), n(17, 80, 33, 16), n(32, 768, 100, 256), n(2, 3072, 40, 256),
        # wgmma: M = 33 at the threshold, a partial raster group (9 M tiles), M = 1 with the skinny kernel switched off
        n(33, 784, 200, 16, x3=True, exact=True), n(33, 784, 200, 16, x3=False, exact=True),
        n(1100, 784, 136, 16, x3=True, exact=True, view=True), n(1100, 784, 136, 16, x3=False, exact=True, view=True),
        n(1, 784, 130, 16, x3=True, exact=True, skinny_max=0), n(1, 784, 130, 16, x3=False, exact=True, skinny_max=0),
        n(300, 1024, 520, 64, x3=True), n(300, 1024, 520, 64, x3=False, view=True), n(1, 512, 300, 32, x3=False, skinny_max=0),
        n(200, 1296, 264, 16, x3=True),
    ]


def nbits_prepare(s):
    r = _rng("nbits", _key(s))
    M, K, N, block = s["M"], s["K"], s["N"], s["block"]
    if s.get("exact"):  # integers and powers of two: every product and partial sum exact in TF32 and in f32
        a = r.integers(-8, 9, (M, K)).astype(F32)
        sc = np.ldexp(F32(1), r.integers(-3, 1, (N, K // block))).astype(F32)
    else:
        a = r.uniform(-1, 1, (M, K)).astype(F32)
        sc = r.uniform(-0.1, 0.1, (N, K // block)).astype(F32)
    return dict(a=a, b=pack_nbits(r.integers(0, 16, (N, K // block, block))), s=sc)


def nbits_launch(rt, ctx, s, inp):
    """(output, the output buffer outside a view or None)"""
    M, N = s["M"], s["N"]
    ctx.set_f32_mode(s["x3"])
    op = rt.MatMulNBits(block_size=s["block"])
    args = [ctx.to_device(inp["a"]), ctx.to_device(inp["b"]), ctx.to_device(inp["s"])]
    with gc.switches(RTEN_B200_NBITS_SKINNY_MAX=s.get("skinny_max")):
        if not s.get("view"):
            return op.run(ctx, *args).numpy(), None
        pitch = N + 3  # odd row pitch, 4 bytes past an 8-byte boundary
        buf = ctx.to_device(np.full(M * pitch + 8, -7.5, F32))
        y = op.run(ctx, *args, out=buf.view((M, N), (pitch, 1), 1))
        host = buf.numpy()
        inside = np.zeros(host.shape, bool)
        inside[1:1 + M * pitch].reshape(M, pitch)[:, :N] = True
        return y.numpy(), host[~inside]


def _nbits_cols(s):
    c = s.get("cols")
    return np.arange(s["N"]) if c is None else np.r_[0:c, s["N"] - c:s["N"]]


def skinny_model(a, w, cols=None, perturb=()):
    """nbits_skinny_kernel in float32: a [M, K], w [K, N] (dequantized: f32(q - 8) * scale, one rounding).  Lane l of
    the chunk at k0 owns elements k0 + 32 l .. k0 + 32 l + 31 (16 in a last half unit) and runs one fma chain per
    (row, column) over its elements of every chunk in k order; the 32 lane sums meet in an xor-16/8/4/2/1 butterfly."""
    a, w = np.asarray(a, F32), np.asarray(w, F32)
    if cols is not None:
        w = w[:, cols]
    M, K = a.shape
    N = w.shape[1]
    acc = np.zeros((M, N, 32), F32)
    for k0 in range(0, K, 1024):
        for j in range(32):
            k = k0 + 32 * np.arange(32) + j  # per lane
            live = k < K
            kk = np.where(live, k, 0)
            upd = _fma(a[:, None, kk], w[kk].T[None], acc)
            acc = np.where(live[None, None, :], upd, acc)
    lanes = np.arange(32)
    for o in ((8, 16, 4, 2, 1) if "butterfly" in perturb else (16, 8, 4, 2, 1)):
        acc = acc + acc[..., lanes ^ o]
    return acc[..., 0]


# ---- the case families ------------------------------------------------------------------------------------------------
def spec_id(fam, s):
    return fam + " " + " ".join(f"{k}={v}" for k, v in s.items())


def case_unit(fam, s, sms):
    """((kernel, template arguments), the CTAs and threads of a decode launch or None, the edges the case reaches)"""
    if fam == "decode":
        key, nw, ns, edges = decode_case_rule(s, sms)
        return key, (s["B"] * s["qh"] * ns, nw * 32), edges
    key = nbits_rule(s["M"], s["K"], s["N"], s["block"], s["x3"], sms, s.get("skinny_max", 32))[0]
    return key, None, nbits_edges(s, sms)


SPECS = {"decode": decode_specs, "nbits": nbits_specs}
EDGES = {"decode": DECODE_EDGES, "nbits": NBITS_EDGES}


def coverage_gaps(sms):
    """instances that fewer than two cases select, and rule edges no case reaches"""
    picked, reached = {}, set()
    for fam, specs in SPECS.items():
        for s in specs(sms):
            (k, a), _, edges = case_unit(fam, s, sms)
            assert a in VARIANTS[k], f"{spec_id(fam, s)}: the rule names {(k, a)}, which the table lacks"
            assert k in FAMILY_KERNELS[fam], f"{spec_id(fam, s)}: {k} is not a kernel of the family"
            picked[(k, a)] = picked.get((k, a), 0) + 1
            reached |= {(fam, e) for e in edges}
    gaps = [("selected fewer than twice", (k, a)) for k, args in VARIANTS.items() for a in args if picked.get((k, a), 0) < 2]
    return gaps + [("edge never reached", (fam, e)) for fam, es in EDGES.items() for e in es if (fam, e) not in reached]


# ---- fixtures ---------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def rt():
    import rten_b200
    from rten_b200 import _lib
    _lib.load()
    return rten_b200


@pytest.fixture(scope="module")
def sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


# ---- kernel identity --------------------------------------------------------------------------------------------------
def _launches(fn, smem=False):
    """[(name, grid, block)] of the kernels `fn` launches, from Kineto's trace (grid and block: x * y * z, None when the
    trace does not record them); with `smem`, [(name, grid, block, shared memory)], the shared memory Kineto records or
    None.  The capture window is held open around the call as rk._capture does"""
    import time
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        time.sleep(0.005)
        fn()
        torch.cuda.synchronize()
        time.sleep(0.005)
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            events = json.load(f).get("traceEvents", [])
    out = []
    for e in events:
        if e.get("cat") != "kernel":
            continue
        a = e.get("args", {})
        g, b = a.get("grid"), a.get("block")
        launch = (e["name"], int(np.prod(g)) if g else None, int(np.prod(b)) if b else None)
        out.append(launch + (a.get("shared memory"),) if smem else launch)
    return out


def _kernel_probe():
    import torch
    import rten_b200 as rt
    n_sms = torch.cuda.get_device_properties(0).multi_processor_count
    ctx = rt.Context(0)
    res = {}
    for fam, specs in SPECS.items():
        for s in specs(n_sms):
            inp = decode_prepare(s) if fam == "decode" else nbits_prepare(s)

            def call():
                if fam == "decode":
                    decode_launch(rt, ctx, inp)
                else:
                    nbits_launch(rt, ctx, s, inp)
                ctx.sync()
            for _ in range(3):  # a capture with no kernel record at all is taken again (see rk.capture_kernels)
                got = _launches(call)
                if got:
                    break
            res[spec_id(fam, s)] = got
    print(json.dumps({"sms": n_sms, "launches": res}))


def test_kernel_identity():
    out = rk.probe_in_child("test_gpu_decode_step_kernels")
    n_sms, launches = out["sms"], out["launches"]
    seen, wrong, no_grid = {}, [], 0
    for fam, specs in SPECS.items():
        for s in specs(n_sms):
            sid = spec_id(fam, s)
            want, shape, _ = case_unit(fam, s, n_sms)
            ours = [(kernel_key(n), g, b) for n, g, b in launches[sid] if kernel_key(n) is not None]
            ran = {k for k, _, _ in ours}
            if ran != {want} or len(ours) != 1:
                wrong.append((sid, want, [(n, g, b) for n, g, b in launches[sid]]))
                continue
            if shape is not None:
                _, g, b = ours[0]
                if g is None:
                    no_grid += 1
                elif (g, b) != shape:
                    wrong.append((sid, f"grid {shape}", (g, b)))
            seen[want] = seen.get(want, 0) + 1
    assert not wrong, f"{len(wrong)} cases ran other kernels or grids than the rule names: {wrong[:6]}"
    assert no_grid == 0, "the trace recorded no grid for the decode kernels"
    missing = [(k, a) for k, args in VARIANTS.items() for a in args if seen.get((k, a), 0) < 2]
    assert not missing, f"instances that fewer than two cases ran: {missing}"
    assert not coverage_gaps(n_sms)
    print(f"14 of 14 instances ran, each at least twice, on {n_sms} SMs; every decode grid as the rule names")


# ---- numbers: decode attention ----------------------------------------------------------------------------------------
def _check_decode(rt, ctx, s, sms):
    inp = decode_prepare(s)
    s = inp["spec"]
    B, qh, dh = s["B"], s["qh"], s["dh"]
    y, dev = decode_launch(rt, ctx, inp)
    got = y.numpy().reshape(B * qh, dh)
    want, rows = decode_want(inp, sms)
    what = spec_id("decode", s)
    gc.assert_bit_exact(got[rows], want, what)
    if "kc" in dev and s["op"] != "mha":
        # the appended row (rotated key) is the only cache change: every other byte, NaN padding included, is as it was
        kc, vc = dev["kc"].numpy(), dev["vc"].numpy()
        k0, v0 = inp["K"].copy(), inp["V"].copy()
        if "kn" in inp:
            for b in range(B):
                if inp["lens"][b] > 0:
                    k0[b, :, inp["lens"][b] - 1] = inp["k_written"][b]
                    v0[b, :, inp["lens"][b] - 1] = inp["vn"][b]
        if s.get("vt"):
            v0 = transposed_v(v0)
        assert np.array_equal(kc.view(I32), k0.view(I32)), f"{what}: key cache bytes other than the appended row"
        assert np.array_equal(vc.view(I32), v0.view(I32)), f"{what}: value cache bytes other than the appended row"
    return inp, got


def test_decode_bit_exact(rt, sms):
    ctx = rt.Context(0)
    for s in decode_specs(sms):
        _check_decode(rt, ctx, s, sms)


def test_decode_runs_again_and_in_a_graph(rt, sms):
    """The split merge's counters are reset by the last CTA of each (batch, head): the same inputs give the same bits
    twice in a row, and from a captured CUDA graph replayed twice; a small call after the large one too"""
    ctx = rt.Context(0)
    specs = [s for s in decode_specs(sms) if s["op"] == "attn" and not s.get("append")]
    for s in specs[:3] + specs[-1:] + specs[:1]:
        inp = decode_prepare(s)
        B, qh, dh = s["B"], s["qh"], s["dh"]
        y, dev = decode_launch(rt, ctx, inp)
        first = y.numpy()
        again = decode_launch(rt, ctx, inp, dev=dev)[0].numpy()
        gc.assert_bit_exact(again, first, spec_id("decode", s) + ": second run")
        out = ctx.empty((B, qh, 1, dh))
        decode_launch(rt, ctx, inp, out=out, dev=dev)  # (an eager call first: nothing is allocated while capturing)
        ctx.sync()
        ctx.graph_begin()
        decode_launch(rt, ctx, inp, out=out, dev=dev)
        graph = ctx.graph_end()
        for i in range(2):
            out.copy_from(np.zeros((B, qh, 1, dh), F32))
            graph.launch()
            ctx.sync()
            gc.assert_bit_exact(out.numpy(), first, spec_id("decode", s) + f": graph replay {i + 1}")


def test_the_decode_comparison_has_teeth(rt, sms):
    """Each deliberate departure from the kernel's order changes the model's bits on a multi-split case with a mask, so
    the bit-exact comparisons above would see the same slip in the kernel"""
    ctx = rt.Context(0)
    s = decode_specs(sms)[2]  # three batches, several splits, transposed V, mask, append
    inp, got = _check_decode(rt, ctx, s, sms)
    for p in ("butterfly", "mul-add", "splits"):
        want, rows = decode_want(inp, sms, perturb=(p,))
        assert not np.array_equal(got[rows].view(I32), want.view(I32)), f"perturbation {p!r} leaves the model's bits unchanged"


# ---- numbers: MatMulNBits ---------------------------------------------------------------------------------------------
def test_nbits_values(rt, sms):
    ctx = rt.Context(0)
    for s in nbits_specs(sms):
        inp = nbits_prepare(s)
        got, outside = nbits_launch(rt, ctx, s, inp)
        what = spec_id("nbits", s)
        key = nbits_rule(s["M"], s["K"], s["N"], s["block"], s["x3"], sms, s.get("skinny_max", 32))[0]
        w = dequantize_nbits(inp["b"], inp["s"])
        if key[0] == "nbits_skinny_kernel":
            cols = _nbits_cols(s)
            gc.assert_bit_exact(got[:, cols], skinny_model(inp["a"], w, cols), what)
        elif s.get("exact"):
            exact = inp["a"].astype(np.float64) @ w.astype(np.float64)
            assert np.abs(exact).max() < 2 ** 16
            gc.assert_bit_exact(got, exact.astype(F32), what)
        else:
            exact, absum = _exact(inp["a"], inp["b"], inp["s"])
            with gc.bound(not s["x3"]):
                gc.assert_tf32_close(got, exact, absum, what)
        if outside is not None:
            assert (outside == F32(-7.5)).all(), f"{what}: writes outside the output view"


def test_skinny_comparison_has_teeth(rt, sms):
    """Swapping two levels of the lane butterfly changes the model's bits when every lane holds part of the sum"""
    ctx = rt.Context(0)
    s = nbits_specs(sms)[2]  # K = 1024: one 32-element unit per lane
    inp = nbits_prepare(s)
    got, _ = nbits_launch(rt, ctx, s, inp)
    w = dequantize_nbits(inp["b"], inp["s"])
    assert not np.array_equal(got.view(I32), skinny_model(inp["a"], w, perturb=("butterfly",)).view(I32))
