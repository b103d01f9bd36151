"""`pytest -m gpu`: the streaming prefill attention kernels (attn_prefill.cu attn_prefill_kernel / attn_prefill_mha_kernel)
-- the prompt work of Attention with q_seq > 1, GroupQueryAttention and MultiHeadAttention -- each selected by name and
checked bit for bit.

The launcher picks an instance from the head size, the context's f32 mode and the operator, and one CTA per (batch,
query head, 64-query tile); each CTA derives its valid length, causal offset, key range and sliding-window skip from the
device lengths.  That arithmetic is restated below (`prefill_rule`, `cta_tiles`); `VARIANTS` lists every instance
(tests/test_prefill_attention_kernel_table_cpu.py keeps it equal to the built library's symbols), and `EDGES` the
branches a kernel name does not show.  The case list reaches each of them, and every instance at least twice, on 132
and on 114 SMs.

  * kernel identity: every case runs once under CUPTI in a child process; each must run exactly the instance its rule
    names (the rotary / append kernels GroupQueryAttention and MultiHeadAttention launch first are not claimed), every
    entry of `VARIANTS` must have run, and each launch must have B * q_heads * q_tiles CTAs of 160 threads;
  * values against `prefill_model`, a float32 restatement of the consumer warpgroup with every rounding explicit: the
    score fmul by the scale, the mask fadd on visible keys only, -inf (or MultiHeadAttention's fill) elsewhere, the tile
    max from -FLT_MAX (fmaxf ignores NaN), the rescale a = reduced_range_exp(m_old - m_new) of l and o, each thread's
    row sum (l + e0) + e1 over its columns 8 c + 2 t, 8 c + 2 t + 1 in c order and the xor-1 / xor-2 quad sums, the
    output update fma(o, a, pv) (3xTF32) or fmul(o, a) + pv (TF32), MultiHeadAttention's tail of n_tail fill keys
    (the value sum in key order, the fmul / fadd updates), o * (1 / l) with NaN -> 0.  reduced_range_exp is the
    oracle's rto_reduced_range_exp1, vectorised (`rre`; the CPU test pins it to the oracle bit for bit).
    The inputs make every tensor-core product exact: Q and K hold integers in [-1, 1] (exact in TF32, low parts 0,
    every score an exact integer), and V is one-hot -- column d is 1 at one chosen key and 0 elsewhere -- so a tile's
    P V is 0, or the one weight e as the tensor core reads it (hi(e) + tf32(lo(e)) in 3xTF32, tf32(e) in one pass).
    Every column then shows the whole max / rescale chain and denominator, and one key's numerator; the keys are
    chosen at tile edges, the causal diagonal, window boundaries, past the valid length and in MultiHeadAttention's
    tail.  In 3xTF32 some columns hold a second 1 in another key tile, so the f32 fma that merges two tiles'
    products shows too (in one pass the tensor core itself would add them, in its own rounding);
  * padded key positions: with nonpad_kv_seqlen, and in GroupQueryAttention's in-place cache, K and V hold NaN at
    every position at or past the valid length (and a transposed V's row padding too), and the result must equal the
    model on the same data with those positions zeroed: a prompt reads the cache a decode step reads, and gets the same
    answer.
  * deliberate slips in the model (quad sum order, the 3xTF32 merge as multiply-then-add, the window skip rounded up,
    the tail one key short) each change its bits on some case, so the comparisons would see the same slip in the
    kernel; reruns and replayed CUDA graphs reproduce the same bits."""
import json

import numpy as np
import pytest

import gpu_checks as gc
import test_gpu_decode_step_kernels as dk
import test_gpu_row_kernels as rk

pytestmark = pytest.mark.gpu

F32, I32 = np.float32, np.int32
FLT_MAX = np.finfo(F32).max
BM = 64  # query rows per CTA
THREADS = 160  # one consumer warpgroup and one TMA warp

# ---- the kernels ------------------------------------------------------------------------------------------------------
VARIANTS = {
    "attn_prefill_kernel": [(64, 1), (64, 0), (128, 1), (128, 0)],  # <DH, X3>
    "attn_prefill_mha_kernel": [(64, 1), (64, 0), (128, 1), (128, 0)],
}
KERNELS = set(VARIANTS)
EDGES = ("one key tile", "partial last key tile", "fewer keys than the 32-key V^T box", "32-key tiles",
         "q_seq < 64", "partial last query tile", "more CTAs than two waves",
         "causal offset > 0", "causal offset < 0", "len 0", "len clamped to kv_seq", "len clamped to 0",
         "window skips whole tiles", "window start inside a tile", "natural V", "transposed V",
         "mask [B,1,1,L]", "mask [1,1,T,L]", "mask [B,H,T,L]", "fully masked row", "mask -inf", "mask +inf", "mask NaN",
         "mask -FLT_MAX", "GQA group 1", "GQA group 4", "GQA group 8",
         "MHA key padding mask", "MHA bias, key stride 1", "MHA bias, key stride 0", "MHA tail taken, finite fill",
         "MHA tail weightless, fill -inf", "MHA one query over more than 8192 keys",
         "NaN past len, natural V, 3xTF32", "NaN past len, natural V, TF32", "NaN past len, transposed V, 3xTF32",
         "NaN past len, transposed V, TF32", "NaN past len, GroupQueryAttention in-place cache")


def kernel_key(name, kernels=KERNELS):
    return dk.kernel_key(name, kernels)


def _cdiv(a, b):
    return -(-a // b)


# ---- the launch rule --------------------------------------------------------------------------------------------------
def tile_keys(dh, x3):
    """Cfg::BN: 32-key tiles at head size 128 in 3xTF32 (two stages and the low parts would not fit in 227 KB), else 64"""
    return 32 if dh == 128 and x3 else 64


def prefill_supported(B, qh, kvh, S, T, dh, window=0, mha=False, lens=False, v_natural=True, causal_offset=0):
    """attn_prefill_supported, on the shapes (the alignment and TMA checks aside)"""
    if dh not in (64, 128) or window < 0 or min(B, qh, kvh, S, T) < 1 or qh % kvh:
        return False
    if B * qh * _cdiv(S, BM) > 0x7fffffff:
        return False
    return not (mha and (window or lens or not v_natural or causal_offset < 0))


def cta_tiles(lim, off, q0, S, causal, window, BN, perturb=()):
    """attn_prefill_body's per-CTA arithmetic (numpy arrays over CTAs): (kend, ntiles, jlo) -- keys [0, kend) exist for
    some row of the tile, key tiles [jlo, ntiles) are loaded; `perturb` "jlo up" rounds the window skip up"""
    lim, off, q0 = (np.asarray(a, np.int64) for a in (lim, off, q0))
    kend = np.minimum(lim, np.minimum(q0 + BM, S) + off) if causal else lim
    kend = np.maximum(kend, 0)
    ntiles = (kend + BN - 1) // BN
    if window > 0:
        start = np.maximum(q0 + off + 1 - window, 0)
        jlo = np.minimum((start + BN - 1) // BN if "jlo up" in perturb else start // BN, ntiles)
    else:
        jlo = np.zeros_like(ntiles)
    return kend, ntiles, jlo


def _dims(s):
    return s["B"], s["qh"], s["kvh"], s["S"], s["T"], s["dh"]


def case_lens(s):
    """(raw lengths or None, lim [B], off [B]): the valid keys and the causal offset of each batch, as the kernel sees
    them (Attention: nonpad_kv_seqlen clamped to [0, kv_seq], offset lim - q_seq; GroupQueryAttention: its rotary kernel's
    len_eff, a first prompt S, else seqlens_k clamped to [S - 1, T - 1] plus one; MultiHeadAttention: every key, the past
    length as the offset)"""
    B, _, _, S, T, _ = _dims(s)
    if s["op"] == "attn":
        if s.get("lens") is None:
            return None, np.full(B, T, np.int64), np.zeros(B, np.int64)
        raw = np.array(s["lens"], np.int64)
        lim = np.clip(raw, 0, T)
        return raw, lim, lim - S
    if s["op"] == "gqa":
        if not s.get("past"):
            lim = np.full(B, S, np.int64)
        else:
            lim = np.clip(np.array(s["lens"], np.int64) - 1, S - 1, T - 1) + 1
        return None, lim, lim - S
    return None, np.full(B, T, np.int64), np.full(B, s.get("past", 0), np.int64)


def _causal(s):
    return bool(s["op"] == "gqa" or s.get("causal") or s.get("unidir"))


def _window(s):
    return s.get("window", 0) if s["op"] == "gqa" else 0


def _fill(s):
    return F32(s.get("fill", -10000.0))


# with Q, K in [-1, 1] every score is at most dh * scale <= 11.4 in size, and the masks add at most 0: a fill above -60
# leaves e^(fill - row max) above the exp cutoff (-87.3) for every row, so the tail's weight is not zero
_TAIL_FILL_MIN = -60.0


def prefill_rule(s):
    """launch_attn_prefill and the top of attn_prefill_body: ((kernel, (DH, X3)), grid, block, BN, q_tiles, per-CTA
    arrays in blockIdx order).  Block u runs query tile q_tiles - 1 - u % q_tiles (the longest causal tiles first), head
    (u / q_tiles) % q_heads, batch u / (q_tiles q_heads)."""
    B, qh, kvh, S, T, dh = _dims(s)
    x3, mha = int(s["x3"]), s["op"] == "mha"
    raw, lim, off = case_lens(s)
    assert prefill_supported(B, qh, kvh, S, T, dh, _window(s), mha, raw is not None, not s.get("vt"), int(off.min()) if mha else 0)
    BN = tile_keys(dh, x3)
    q_tiles = _cdiv(S, BM)
    grid = B * qh * q_tiles
    u = np.arange(grid)
    c = dict(qt=q_tiles - 1 - u % q_tiles, h=(u // q_tiles) % qh, b=u // (q_tiles * qh))
    c["q0"] = c["qt"] * BM
    c["lim"], c["off"] = lim[c["b"]], off[c["b"]]
    c["kend"], c["ntiles"], c["jlo"] = cta_tiles(c["lim"], c["off"], c["q0"], S, _causal(s), _window(s), BN)
    if mha:
        c["kt"] = np.minimum(c["ntiles"] * BN, c["lim"])
        c["n_tail"] = c["lim"] - c["kt"]
        c["tail_taken"] = (c["n_tail"] > 0) & bool(np.isfinite(_fill(s)) and _fill(s) > _TAIL_FILL_MIN)
    key = ("attn_prefill_mha_kernel" if mha else "attn_prefill_kernel", (dh, x3))
    return key, grid, THREADS, BN, q_tiles, c


def prefill_edges(s, sms):
    B, qh, kvh, S, T, dh = _dims(s)
    key, grid, _, BN, q_tiles, c = prefill_rule(s)
    raw, lim, off = case_lens(s)
    e = set()
    run = c["ntiles"] - c["jlo"]
    if (run == 1).any():
        e.add("one key tile")
    if ((c["kend"] % BN != 0) & (run > 0)).any():
        e.add("partial last key tile")
    if s.get("vt") and T < 32:
        e.add("fewer keys than the 32-key V^T box")
    if BN == 32:
        e.add("32-key tiles")
    if S < BM:
        e.add("q_seq < 64")
    if S > BM and S % BM:
        e.add("partial last query tile")
    if grid > 2 * sms:
        e.add("more CTAs than two waves")
    if _causal(s) and (off > 0).any():
        e.add("causal offset > 0")
    if _causal(s) and (off < 0).any():
        e.add("causal offset < 0")
    if raw is not None:
        if (raw == 0).any():
            e.add("len 0")
        if (raw > T).any():
            e.add("len clamped to kv_seq")
        if (raw < 0).any():
            e.add("len clamped to 0")
    w = _window(s)
    if w:
        if (c["jlo"] > 0).any():
            e.add("window skips whole tiles")
        start = c["q0"] + c["off"] + 1 - w
        if ((start > 0) & (start % BN != 0) & (c["jlo"] > 0)).any():
            e.add("window start inside a tile")
    e.add("transposed V" if s.get("vt") else "natural V")
    if s.get("mask"):
        e.add({"b11l": "mask [B,1,1,L]", "11tl": "mask [1,1,T,L]", "bhtl": "mask [B,H,T,L]"}[s["mask"]])
    if s.get("special"):
        e |= {"fully masked row", "mask -inf", "mask +inf", "mask NaN", "mask -FLT_MAX"}
    if s["op"] != "mha":
        e.add(f"GQA group {qh // kvh}")
    else:
        if s.get("kpm"):
            e.add("MHA key padding mask")
        if s.get("bias"):
            e.add("MHA bias, key stride 0" if s["bias"] == "bcast" else "MHA bias, key stride 1")
        if c["tail_taken"].any():
            e.add("MHA tail taken, finite fill")
        if (c["n_tail"] > 0).any() and _fill(s) == -np.inf:
            e.add("MHA tail weightless, fill -inf")
        if S == 1 and T > 8192:
            e.add("MHA one query over more than 8192 keys")
    if s.get("nan") and (lim < T).any():
        if s["op"] == "gqa":
            e.add("NaN past len, GroupQueryAttention in-place cache")
        else:
            e.add(f"NaN past len, {'transposed' if s.get('vt') else 'natural'} V, {'3xTF32' if s['x3'] else 'TF32'}")
    return e


def prefill_specs(sms=None):
    """the cases (the same on every SM count: the grid depends on the shapes only)"""
    a = lambda B, qh, kvh, S, T, dh, x3, **kw: dict(op="attn", B=B, qh=qh, kvh=kvh, S=S, T=T, dh=dh, x3=x3, **kw)  # noqa: E731
    g = lambda B, qh, kvh, S, past, dh, x3, **kw: dict(op="gqa", B=B, qh=qh, kvh=kvh, S=S, T=past + S, dh=dh, x3=x3, past=past, **kw)  # noqa: E731
    m = lambda B, H, S, L, dh, x3, past=0, **kw: dict(op="mha", B=B, qh=H, kvh=H, S=S, T=past + L, dh=dh, x3=x3, past=past, **kw)  # noqa: E731
    return [
        # Attention: causal, nonpad lengths (clamped, 0, shorter than the queries), GQA, masks, both value layouts
        a(2, 4, 4, 128, 128, 64, 1, causal=True),
        a(2, 4, 4, 64, 300, 64, 0, causal=True, lens=(164, 264), vt=True),  # chunked prefill: offsets 100, 200
        a(2, 4, 4, 100, 160, 128, 1, causal=True, lens=(40, 160)),  # offset -60: rows 0 .. 59 of batch 0 see no key
        a(4, 8, 2, 70, 200, 64, 1, lens=(0, 10000, -5, 77), vt=True, mask="b11l", nan=True),
        a(4, 8, 2, 70, 200, 64, 0, lens=(0, 10000, -5, 77), mask="b11l", nan=True),
        a(2, 8, 1, 65, 260, 128, 0, causal=True, lens=(250, 130), mask="11tl", vt=True, nan=True),
        a(2, 3, 3, 65, 200, 128, 1, causal=True, mask="bhtl", special=True),
        a(2, 2, 1, 2, 5, 64, 1, causal=True, lens=(5, 3), vt=True),  # fewer keys than one tile and than V^T's box
        a(1, 4, 2, 3, 20, 128, 0, causal=True, mask="b11l", vt=True),
        a(4, 32, 8, 130, 330, 64, 1, causal=True, lens=(330, 200, 131, 7), nan=True, ctas=24),  # 384 CTAs
        a(1, 8, 8, 96, 96, 128, 0, causal=True),
        # GroupQueryAttention prompts: first prompts, a chunk over an in-place cache with NaN past its length, windows
        g(2, 8, 2, 150, 0, 64, 1, window=37),  # window start 92 in query tile 2: one whole tile skipped
        g(1, 8, 1, 70, 130, 128, 1, lens=(150,), nan=True, window=100),  # offset 80, window start 45: a 32-key tile skipped
        g(2, 4, 4, 300, 0, 128, 0, window=64, mask="11tl", ctas=16),
        g(1, 4, 1, 66, 60, 64, 0, lens=(120,), nan=True),
        # MultiHeadAttention prompts: the causal tail with a finite fill, padding masks, biases, one query over 8192 keys
        m(2, 4, 200, 200, 64, 1, unidir=True, fill=-1.5),
        m(2, 4, 130, 130, 64, 0, unidir=True, fill=-np.inf, kpm=True),
        m(1, 3, 100, 100, 128, 1, unidir=True, fill=-3.0, bias="bcast"),
        m(2, 2, 80, 150, 128, 0, bias="keys", kpm=True),
        m(1, 2, 1, 8200, 64, 1),
        m(1, 2, 1, 8300, 128, 0, kpm=True),
        m(2, 2, 70, 40, 64, 0, past=30, unidir=True, fill=-2.0),  # offset 30
        m(1, 2, 150, 150, 128, 1, unidir=True, fill=0.0, kpm=True),
    ]


def spec_id(s):
    return " ".join(f"{k}={v}" for k, v in s.items())


def coverage_gaps(sms):
    """instances that fewer than two cases select, and edges no case reaches"""
    picked, reached = {}, set()
    for s in prefill_specs(sms):
        (k, a), *_ = prefill_rule(s)
        assert a in VARIANTS[k], f"{spec_id(s)}: the rule names {(k, a)}, which the table lacks"
        picked[(k, a)] = picked.get((k, a), 0) + 1
        reached |= prefill_edges(s, sms)
    gaps = [("selected fewer than twice", (k, a)) for k, args in VARIANTS.items() for a in args if picked.get((k, a), 0) < 2]
    return gaps + [("edge never reached", e) for e in EDGES if e not in reached]


# ---- the model --------------------------------------------------------------------------------------------------------
_CUTOFF = F32(F32(-126.5) * F32(0.693147180559945309417)) + F32(0.01)


def rre(x):
    """oracle rto_reduced_range_exp1 of every element, vectorised: the fma chain of exp_poly (each fma exactly rounded,
    oracle/norms.py fma_f32), k = cvttps2dq(j) (NaN / out of range -> INT_MIN), r * 2^k through the exponent bits of
    k + 127, 0 below the cutoff"""
    fma = dk._fma
    x = np.asarray(x, F32)
    with np.errstate(all="ignore"):
        magic = F32(12582912.0)
        j = fma(x, F32(1.44269504088896340736), magic)
        j = (j - magic).astype(F32)
        r = fma(j, F32(-6.93145752e-1), x)
        r = fma(j, F32(-1.42860677e-6), r)
        t = np.full(x.shape, F32(1.37805939e-3), F32)
        for c in (8.37312452e-3, 4.16695364e-2, 1.66664720e-1, 4.99999851e-1, 1.0):
            t = fma(t, r, F32(c))
        r = fma(t, r, F32(1.0))
        ok = (j > F32(-2147483904.0)) & (j < F32(2147483648.0))
        k = np.where(ok, np.where(ok, j, 0).astype(np.int64), -(2 ** 31))
        p2 = (((k + 127) & 0xffffffff) << 23 & 0xffffffff).astype(np.uint32).view(F32)
        r = (r * p2).astype(F32)
    return np.where(x < _CUTOFF, F32(0), r).astype(F32)


def _hi(x):
    """what kind::tf32 reads of an f32: the low 13 mantissa bits cleared"""
    return (np.asarray(x, F32).view(np.uint32) & np.uint32(0xffffe000)).view(F32)


def _split(x):
    """(hi, lo as the tensor core reads it): lo = tf32_lo(x) = x - hi, rounded to f32, read as TF32"""
    x = np.asarray(x, F32)
    hi = _hi(x)
    with np.errstate(invalid="ignore"):
        return hi, _hi((x - hi).astype(F32))


def _mm(a, b, x3):
    """a [.., M, K] . b [.., K, N] as wgmma tf32 reads them, the sum in float64 rounded once (exact on the one-hot and
    integer operands of the GPU cases): 3xTF32 lo.hi + hi.lo + hi.hi, else hi.hi"""
    with np.errstate(invalid="ignore", over="ignore"):
        if x3:
            ah, al = (v.astype(np.float64) for v in _split(a))
            bh, bl = (v.astype(np.float64) for v in _split(b))
            return (al @ bh + ah @ bl + ah @ bh).astype(F32)
        return (_hi(a).astype(np.float64) @ _hi(b).astype(np.float64)).astype(F32)


def prefill_model(Q, K, V, lim, off, *, causal, x3, scale, window=0, mask=None, mha=None, ctas=None, perturb=()):
    """attn_prefill_body in float32.  Q [B, qh, S, dh], K / V [B, kvh, T, dh] (what the kernel reads; V at keys >= lim
    is taken as 0), lim / off [B] (valid keys, causal offset), mask broadcastable to [B, qh, S, T] or None, mha None or
    dict(fill, kpm [B, T] or None).  `ctas`: (b, h, qt) triples to model (default all).  Returns (out [B, qh, S, dh]
    with NaN in rows not modelled, the MultiHeadAttention tail flag of each modelled CTA).
    `perturb` names deliberate slips (the suite checks that each one changes the result): "quad" sums the row's quad
    xor-2 first, "mul-add" rounds the 3xTF32 rescale's product before adding, "jlo up" rounds the window skip up,
    "tail short" counts the MultiHeadAttention tail one key short."""
    Q, K, V = (np.asarray(a, F32) for a in (Q, K, V))
    B, qh, S, dh = Q.shape
    kvh, T = K.shape[1], K.shape[2]
    BN = tile_keys(dh, x3)
    scale = F32(scale)
    lim, off = np.asarray(lim, np.int64), np.asarray(off, np.int64)
    if ctas is None:
        ctas = [(b, h, qt) for b in range(B) for h in range(qh) for qt in range(_cdiv(S, BM))]
    cb, ch, cq = (np.array([c[i] for c in ctas], np.int64) for i in range(3))
    hk = ch // (qh // kvh)
    q0 = cq * BM
    lim_c, off_c = lim[cb], off[cb]
    kend, ntiles, jlo = cta_tiles(lim_c, off_c, q0, S, causal, window, BN, perturb)
    r = q0[:, None] + np.arange(BM)[None, :]  # [C, 64] tile rows
    live = r < S
    rc = np.minimum(r, S - 1)  # the mask row a phantom row reads
    Qc = np.where(live[..., None], Q[cb[:, None], ch[:, None], rc], F32(0))  # TMA fills rows past q_seq with 0
    row_lim = np.minimum(lim_c[:, None], r + off_c[:, None] + 1) if causal else np.broadcast_to(lim_c[:, None], r.shape)
    row_lo = r + off_c[:, None] + 1 - window if window > 0 else np.zeros_like(r)
    Mf = None if mask is None else np.broadcast_to(np.asarray(mask, F32), (B, qh, S, T))
    C = len(ctas)
    m = np.full((C, BM), -FLT_MAX, F32)
    l4 = np.zeros((C, BM, 4), F32)  # the row sums of the quad's four threads t
    o = np.zeros((C, BM, dh), F32)
    with np.errstate(all="ignore"):
        for j in range(int(ntiles.max()) if C else 0):
            act = (j >= jlo) & (j < ntiles)
            if not act.any():
                continue
            keys = j * BN + np.arange(BN)
            kk = np.minimum(keys, T - 1)
            Kt = np.where((keys < T)[None, :, None], K[cb[:, None], hk[:, None], kk[None, :]], F32(0))
            Vt = np.where((keys[None, :] < lim_c[:, None])[..., None], V[cb[:, None], hk[:, None], kk[None, :]], F32(0))
            z = (_mm(Qc, Kt.transpose(0, 2, 1), x3) * scale).astype(F32)
            key3 = keys[None, None, :]
            mv = None if Mf is None else Mf[cb[:, None, None], ch[:, None, None], rc[:, :, None], kk[None, None, :]]
            if mha is not None:
                exists = key3 < lim_c[:, None, None]
                vis = key3 < row_lim[..., None]
                if mha.get("kpm") is not None:
                    vis = vis & (np.asarray(mha["kpm"])[cb[:, None], np.minimum(keys[None, :], lim_c[:, None] - 1)] != 0)[:, None, :]
                if mv is not None:
                    z = np.where(exists, (z + mv).astype(F32), z)
                z = np.where(~exists, F32(-np.inf), np.where(vis, z, F32(mha["fill"])))
            else:
                ok = (key3 < row_lim[..., None]) & (key3 >= row_lo[..., None])
                if mv is not None:
                    z = np.where(ok, (z + mv).astype(F32), z)
                z = np.where(ok, z, F32(-np.inf))
            z = z.astype(F32)
            mx = np.fmax(m, np.fmax.reduce(z, axis=-1)).astype(F32)
            a = rre((m - mx).astype(F32))
            e = rre((z - mx[..., None]).astype(F32))
            ln = (l4 * a[..., None]).astype(F32)
            cols = 2 * np.arange(4)
            for c in range(BN // 8):
                ln = ((ln + e[..., 8 * c + cols]).astype(F32) + e[..., 8 * c + cols + 1]).astype(F32)
            pv = _mm(e, Vt, x3)
            if x3:
                on = ((o * a[..., None]).astype(F32) + pv).astype(F32) if "mul-add" in perturb else dk._fma(o, a[..., None], pv)
            else:
                on = ((o * a[..., None]).astype(F32) + pv).astype(F32)
            m = np.where(act[:, None], mx, m)
            l4 = np.where(act[:, None, None], ln, l4)
            o = np.where(act[:, None, None], on, o)
        if "quad" in perturb:
            L = ((l4[..., 0] + l4[..., 2]).astype(F32) + (l4[..., 1] + l4[..., 3]).astype(F32)).astype(F32)
        else:
            L = ((l4[..., 0] + l4[..., 1]).astype(F32) + (l4[..., 2] + l4[..., 3]).astype(F32)).astype(F32)
        flags = np.zeros(C, bool)
        if mha is not None:
            fill = F32(mha["fill"])
            kt = np.minimum(ntiles * BN, lim_c)
            n_tail = lim_c - kt - (1 if "tail short" in perturb else 0)
            mn = np.fmax(m, fill).astype(F32)
            et = rre((fill - mn).astype(F32))
            flags = (n_tail > 0) & (et != 0).any(axis=1)
            for i in np.flatnonzero(flags):
                rows = V[cb[i], hk[i], kt[i]:lim_c[i]]
                vsum = np.add.accumulate(rows, axis=0, dtype=F32)[-1]  # in key order
                at = rre((m[i] - mn[i]).astype(F32))
                L[i] = ((L[i] * at).astype(F32) + (F32(n_tail[i]) * et[i]).astype(F32)).astype(F32)
                o[i] = ((o[i] * at[:, None]).astype(F32) + (et[i][:, None] * vsum[None, :]).astype(F32)).astype(F32)
        inv = (F32(1) / L).astype(F32)
        y = (o * inv[..., None]).astype(F32)
    y = np.where(np.isnan(y), F32(0), y)
    out = np.full((B, qh, S, dh), np.nan, F32)
    for i in range(C):
        n = int(live[i].sum())
        out[cb[i], ch[i], q0[i]:q0[i] + n] = y[i, :n]
    return out, flags


# ---- cases ------------------------------------------------------------------------------------------------------------
def _rng(*key):
    return rk._rng("prefill_attention", *key)


def _key(s):
    return sorted((k, str(v)) for k, v in s.items())


def model_ctas(s):
    """the CTAs the value check models: all, or for a large case (`ctas`: n) n of them spread over the grid, the first
    and last blocks included"""
    key, grid, _, _, _, c = prefill_rule(s)
    idx = np.arange(grid) if not s.get("ctas") else np.unique(np.r_[np.linspace(0, grid - 1, s["ctas"]).astype(np.int64)])
    return [(int(c["b"][u]), int(c["h"][u]), int(c["qt"][u])) for u in idx]


def _targets(s, b, lim, off, BN, r):
    """keys worth a one-hot column in batch b: the first and last keys, tile edges, the valid length and past it, the
    causal diagonal and the window boundaries of a few rows, MultiHeadAttention's tail"""
    S, T = s["S"], s["T"]
    ks = {0, 1, T - 1, lim - 1, lim, lim + 1}
    for j in range(1, _cdiv(T, BN) + 1):
        ks |= {j * BN - 1, j * BN}
    for row in (0, 1, BM - 1, BM, S // 2, S - 1):
        ks |= {row + off, row + off + 1}
        if _window(s):
            ks |= {row + off - _window(s), row + off + 1 - _window(s)}
    ks |= set(int(k) for k in r.integers(0, T, 6))
    ks = sorted(k for k in ks if 0 <= k < T and not (s.get("nan") and k >= lim))
    return ks or [0]


def prefill_prepare(s, sel=0):
    """inputs of one selection of one-hot value columns; NaN in K and V at and past the valid length (`nan`)"""
    B, qh, kvh, S, T, dh = _dims(s)
    r = _rng(_key(s), sel)
    raw, lim, off = case_lens(s)
    BN = tile_keys(dh, s["x3"])
    inp = dict(spec=s, lim=lim, off=off, raw=raw)
    inp["Q"] = r.integers(-1, 2, (B, qh, S, dh)).astype(F32)
    K = r.integers(-1, 2, (B, kvh, T, dh)).astype(F32)
    V = np.zeros((B, kvh, T, dh), F32)
    for b in range(B):
        for h in range(kvh):
            pool = _targets(s, b, int(lim[b]), int(off[b]), BN, r)
            first = [pool[d % len(pool)] for d in range(dh)] if sel == 0 else list(r.choice(pool, dh))
            for d, t in enumerate(first):
                V[b, h, t, d] = 1
                if s["x3"] and d % 3 == 1:  # a second 1 in another key tile: the f32 fma merging two tiles' products
                    far = [k for k in pool if k // BN != t // BN]
                    if far:
                        V[b, h, far[(d + sel) % len(far)], d] = 1
    if s.get("nan"):
        for b in range(B):
            K[b, :, lim[b]:] = np.nan
            V[b, :, lim[b]:] = np.nan
    inp["K"], inp["V"] = K, V
    if s.get("mask"):
        shape = {"b11l": (B, 1, 1, T), "11tl": (1, 1, S, T), "bhtl": (B, qh, S, T)}[s["mask"]]
        mk = r.uniform(-3, 0, shape).astype(F32)
        if s.get("special"):
            mk[0, 0, 5, :] = -np.inf  # a fully masked row: zeros
            mk[0, 1, 7, :] = -FLT_MAX  # every key at -FLT_MAX: the scores stay finite and equal
            mk[0, 2, 30, :T:3] = -np.inf
            mk[1, 0, 30, 10] = np.inf  # +inf: the row's max is +inf, its weights inf - inf = NaN -> zeros
            mk[1, 1, 20, 2] = np.nan  # NaN: the row sum is NaN -> zeros
            mk[1, 2, 40, 17] = -FLT_MAX
            mk[1, 2, 64, :] = -np.inf  # a fully masked row alone in its query tile
        inp["mask"] = mk
    if s["op"] == "mha":
        if s.get("kpm"):
            kpm = (r.random((B, T)) < 0.8).astype(I32)
            kpm[0, : min(T, 40)] = 0  # a run of padded keys at the start
            inp["kpm"] = kpm
        if s.get("bias"):
            inp["mask"] = r.uniform(-2, 1, (B, qh, S, T) if s["bias"] == "keys" else (1, 1, S, 1)).astype(F32)
    return inp


def _rows_of(x, heads, dh):
    """[B, heads, L, dh] -> [B, L, heads dh]"""
    B, _, L, _ = x.shape
    return np.ascontiguousarray(x.transpose(0, 2, 1, 3).reshape(B, L, heads * dh))


def prefill_launch(rt, ctx, inp, out=None, dev=None):
    """run the case once (on the device tensors `dev` of an earlier call, else new ones): (output [B, qh, S, dh] on the
    device, as the operator lays it out; the device tensors)"""
    s = inp["spec"]
    B, qh, kvh, S, T, dh = _dims(s)
    ctx.set_f32_mode(bool(s["x3"]))
    dev = {} if dev is None else dev
    if s["op"] == "attn":
        if not dev:
            dev["q"], dev["k"] = ctx.to_device(inp["Q"]), ctx.to_device(inp["K"])
            if s.get("vt"):
                dev["vc"] = ctx.to_device(dk.transposed_v(inp["V"]))  # rows padded with NaN
                pitch = dev["vc"].shape[-1]
                dev["v"] = dev["vc"].view((B, kvh, T, dh), (kvh * dh * pitch, dh * pitch, 1, pitch))
            else:
                dev["v"] = ctx.to_device(inp["V"])
            if inp["raw"] is not None:
                dev["nonpad_kv_seqlen"] = ctx.to_device(inp["raw"].astype(I32))
            if "mask" in inp:
                dev["attn_mask"] = ctx.to_device(inp["mask"])
        kw = {k: dev[k] for k in ("nonpad_kv_seqlen", "attn_mask") if k in dev}
        op = rt.Attention(is_causal=bool(s.get("causal")), q_num_heads=qh, kv_num_heads=kvh)
        return op.run(ctx, dev["q"], dev["k"], dev["v"], out=out, **kw), dev
    lim = inp["lim"]
    if s["op"] == "gqa":
        P = s["past"]
        op = rt.GroupQueryAttention(qh, kvh, local_window_size=s.get("window") or -1)
        kw = {}
        if "mask" in inp:
            kw["attention_bias"] = ctx.to_device(inp["mask"])
        q = ctx.to_device(_rows_of(inp["Q"], qh, dh))
        if not P:  # a first prompt: the new rows are the whole cache
            k, v = (ctx.to_device(_rows_of(inp[n], kvh, dh)) for n in ("K", "V"))
            y, _, _ = op.run(ctx, q, k, v, ctx.to_device((lim - 1).astype(I32)), S, out=out, **kw)
            return y, {}
        # one batch, a chunk of S rows written at [len - S, len) of an in-place cache of T positions; the tail past len
        # keeps what it held (NaN)
        L0 = int(lim[0]) - S
        kc, vc = inp["K"].copy(), inp["V"].copy()
        k, v = (ctx.to_device(_rows_of(inp[n][:, :, L0:L0 + S], kvh, dh)) for n in ("K", "V"))
        kc[:, :, L0:L0 + S] = np.nan  # the operator writes these rows
        vc[:, :, L0:L0 + S] = np.nan
        kd, vd = ctx.to_device(kc), ctx.to_device(vc)
        st = (kvh * T * dh, T * dh, dh, 1)
        y, _, _ = op.run(ctx, q, k, v, ctx.to_device((lim - 1).astype(I32)), int(lim[0]), past_key=kd.view((B, kvh, P, dh), st),
                         past_value=vd.view((B, kvh, P, dh), st), present_key=kd, present_value=vd, out=out, **kw)
        return y, dict(kc=kd, vc=vd)
    P = s.get("past", 0)
    op = rt.MultiHeadAttention(qh, mask_filter_value=float(_fill(s)), unidirectional=bool(s.get("unidir")))
    kw = {}
    if "mask" in inp:
        kw["attention_bias"] = ctx.to_device(inp["mask"])
    if "kpm" in inp:
        kw["key_padding_mask"] = ctx.to_device(inp["kpm"])
    q = ctx.to_device(_rows_of(inp["Q"], qh, dh))
    k, v = (ctx.to_device(_rows_of(inp[n][:, :, P:], qh, dh)) for n in ("K", "V"))
    if P:
        kw["past_key"], kw["past_value"] = (ctx.to_device(np.ascontiguousarray(inp[n][:, :, :P])) for n in ("K", "V"))
    y, _, _ = op.run(ctx, q, k, v, out=out, want_present=bool(P), **kw)
    return y, {}


def _as_bhsd(y, s):
    B, qh, _, S, _, dh = _dims(s)
    y = y.numpy()
    return y if s["op"] == "attn" else y.reshape(B, S, qh, dh).transpose(0, 2, 1, 3)


def prefill_want(inp, ctas=None, perturb=()):
    s = inp["spec"]
    V = inp["V"].copy()
    for b in range(s["B"]):
        V[b, :, inp["lim"][b]:] = 0  # what the kernel promises: positions at or past the valid length are not read
    mha = dict(fill=_fill(s), kpm=inp.get("kpm")) if s["op"] == "mha" else None
    scale = F32(1) / np.sqrt(F32(s["dh"]))
    return prefill_model(inp["Q"], inp["K"], V, inp["lim"], inp["off"], causal=_causal(s), x3=bool(s["x3"]), scale=scale,
                         window=_window(s), mask=inp.get("mask"), mha=mha, ctas=ctas or model_ctas(s), perturb=perturb)


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
def _kernel_probe():
    import torch
    import rten_b200 as rt
    n_sms = torch.cuda.get_device_properties(0).multi_processor_count
    ctx = rt.Context(0)
    res = {}
    for s in prefill_specs(n_sms):
        inp = prefill_prepare(s)

        def call():
            prefill_launch(rt, ctx, inp)
            ctx.sync()
        for _ in range(3):  # a capture with no kernel record at all is taken again (see rk.capture_kernels)
            got = dk._launches(call)
            if got:
                break
        res[spec_id(s)] = got
    print(json.dumps({"sms": n_sms, "launches": res}))


def test_kernel_identity():
    out = rk.probe_in_child("test_gpu_prefill_attention_kernels")
    n_sms, launches = out["sms"], out["launches"]
    seen, wrong, no_grid = {}, [], 0
    for s in prefill_specs(n_sms):
        sid = spec_id(s)
        want, grid, block, *_ = prefill_rule(s)
        ours = [(kernel_key(n), g, b) for n, g, b in launches[sid] if kernel_key(n) is not None]
        if {k for k, _, _ in ours} != {want} or len(ours) != 1:
            wrong.append((sid, want, launches[sid]))
            continue
        _, g, b = ours[0]
        if g is None:
            no_grid += 1
        elif (g, b) != (grid, block):
            wrong.append((sid, f"grid {(grid, block)}", (g, b)))
        seen[want] = seen.get(want, 0) + 1
    assert not wrong, f"{len(wrong)} cases ran other kernels or grids than the rule names: {wrong[:6]}"
    assert no_grid == 0, "the trace recorded no grid for the prefill kernels"
    missing = [(k, a) for k, args in VARIANTS.items() for a in args if seen.get((k, a), 0) < 2]
    assert not missing, f"instances that fewer than two cases ran: {missing}"
    assert not coverage_gaps(n_sms)
    print(f"8 of 8 instances ran, each at least twice, on {n_sms} SMs; every grid as the rule names")


# ---- values -----------------------------------------------------------------------------------------------------------
def _check(rt, ctx, s, sel=0):
    inp = prefill_prepare(s, sel)
    y, dev = prefill_launch(rt, ctx, inp)
    got = _as_bhsd(y, s)
    want, flags = prefill_want(inp)
    rows = ~np.isnan(want[..., 0])
    what = f"{spec_id(s)} selection {sel}"
    gc.assert_bit_exact(got[rows], want[rows], what)
    if s["op"] == "mha":
        c = prefill_rule(s)[5]
        u = {(int(c["b"][i]), int(c["h"][i]), int(c["qt"][i])): i for i in range(len(c["b"]))}
        taken = np.array([c["tail_taken"][u[t]] for t in model_ctas(s)])
        assert np.array_equal(flags, taken), f"{what}: the tail is taken in CTAs {np.flatnonzero(flags)}, the rule says {np.flatnonzero(taken)}"
    if "kc" in dev:  # the in-place caches: the chunk's rows written, the past below and the NaN tail past len untouched
        gc.assert_bit_exact(dev["kc"].numpy(), inp["K"], what + ": key cache")
        gc.assert_bit_exact(dev["vc"].numpy(), inp["V"], what + ": value cache")
    return inp, got


def test_prefill_bit_exact(rt, sms):
    ctx = rt.Context(0)
    for s in prefill_specs(sms):
        for sel in range(1 if s.get("ctas") or s["T"] > 4096 else 2):
            _check(rt, ctx, s, sel)


def test_the_comparison_has_teeth(rt, sms):
    """Each deliberate slip in the model changes its bits on a case the kernel matches, so the bit-exact comparison
    would see the same slip in the kernel"""
    ctx = rt.Context(0)
    specs = prefill_specs(sms)
    pick = {"quad": specs[0], "mul-add": specs[0], "jlo up": specs[12], "tail short": specs[15]}
    for p, s in pick.items():
        inp, got = _check(rt, ctx, s)
        want, _ = prefill_want(inp, perturb=(p,))
        rows = ~np.isnan(want[..., 0])
        assert not np.array_equal(got[rows].view(I32), want[rows].view(I32)), f"perturbation {p!r} leaves the model's bits unchanged"


def test_reruns_and_graphs(rt, sms):
    """The same inputs give the same bits twice in a row and from a captured CUDA graph replayed twice: a plain
    Attention case with NaN past the valid lengths and a MultiHeadAttention case whose CTAs take the causal tail"""
    ctx = rt.Context(0)
    specs = prefill_specs(sms)
    for s in (specs[3], specs[15]):
        inp = prefill_prepare(s)
        y, dev = prefill_launch(rt, ctx, inp)
        first = y.numpy()
        gc.assert_bit_exact(prefill_launch(rt, ctx, inp, dev=dev)[0].numpy(), first, spec_id(s) + ": second run")
        if s["op"] == "mha":  # the inputs of the graph call stay alive with it
            keep = {n: ctx.to_device(_rows_of(inp[n], s["qh"], s["dh"])) for n in ("Q", "K", "V")}
            op = rt.MultiHeadAttention(s["qh"], mask_filter_value=float(_fill(s)), unidirectional=True)
            call = lambda o: op.run(ctx, keep["Q"], keep["K"], keep["V"], out=o, want_present=False)  # noqa: E731
        else:
            call = lambda o: prefill_launch(rt, ctx, inp, out=o, dev=dev)  # noqa: E731
        out = ctx.empty(first.shape)
        call(out)  # (an eager call first: nothing is allocated while capturing)
        ctx.sync()
        ctx.graph_begin()
        call(out)
        graph = ctx.graph_end()
        for i in range(2):
            out.copy_from(np.zeros(first.shape, F32))
            graph.launch()
            ctx.sync()
            gc.assert_bit_exact(out.numpy(), first, spec_id(s) + f": graph replay {i + 1}")
