"""The Attention operator on encoder shapes (128 keys, head size 64, q_seq a multiple of 128, no causal mask, no
nonpad_kv_seqlen, equal head counts, mask absent or [B,1,1,128]) in the single-pass TF32 mode: the one-kernel path
attn_fused_kernel (QK^T -> masked softmax -> PV inside the SM), the attention of BERT-base.

Two kinds of check:
  * the softmax stage bit for bit.  Q and K hold small integers, exact in TF32, so every score is an exact integer and
    the kernel's z = fl(fl(S * scale) + mask) is exactly what the reference's FusedMatMul(alpha) + AddSoftmax computes.
    V is a one-hot permutation, V[t, d] = 1 where t = perm[64 pass + d], so O[i, d] = P[i, perm[64 pass + d]] with the
    13 low mantissa bits dropped (wgmma reads TF32 operands by truncation): two calls show the whole P.  The expected
    bits are the oracle's AddSoftmax with NaNs flushed to zero, truncated the same way.
  * random data against float64, element by element, inside `ref_and_bound`'s bound (its derivation is there).
"""
import json
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
F32 = np.float32
NO_FUSED = "RTEN_B200_NO_FUSED_ATTN"


def trunc_tf32(x):
    """The value a TF32 tensor-core operand reads: the low 13 of the 23 mantissa bits cleared."""
    x = np.ascontiguousarray(x, F32)
    return (x.view(np.uint32) & np.uint32(0xFFFFE000)).view(F32)


# ---------------------------------------------------------------------------------------------------------------------
# float64 reference and the per-element bound

# (score coefficient, output coefficient) per f32 mode; see ref_and_bound
COEF = {True: (2.0 ** -9 + 2.0 ** -17, 2.0 ** -9 + 2.0 ** -16), False: (2.0 ** -15, 2.0 ** -15)}


def ref_and_bound(q, k, v, mask=None, scale=0.125, causal=False, nonpad=None, tf32=True):
    """O = softmax(scale q k^T + mask) v in float64 (masked keys -> -inf, a row without a finite maximum -> zeros, as the
    reference flushes NaNs), q [B, qh, T, dh], k / v [B, kvh, L, dh], query head h reading kv head h // (qh // kvh);
    and a bound on |O_got - O| element by element for a kernel with TF32 operands and f32 arithmetic elsewhere.

    Scores.  Truncating q and k to TF32 moves each by at most 2^-10 relatively, so each product by 2^-9 + 2^-20; the
    f32 sum of 64 products adds at most 63 * 2^-24 < 2^-18 of sum |q k|, the scale multiply 2^-24.  With
    A_it = scale * sum_d |q_id k_td|, every score is off by at most (2^-9 + 2^-17) A_it.  The f32 mask add and the
    subtraction of the maximum round again, by at most 2^-24 |z| each and |z - max| <= 2 max |z|: in all
    delta_i = (2^-9 + 2^-17) max_t A_it + 2^-22 max_t |z_it| over the keys not masked with -inf.
    Softmax.  Scores each off by at most delta_i move P_t = e^z_t / sum e^z by a factor within e^{+-2 delta_i}:
    |dP_t| <= P_t (e^{2 delta_i} - 1).
    Output.  Truncating P and V to TF32 moves each product by at most 2^-9 + 2^-20 relatively; the f32 sum of 128
    products adds at most 127 * 2^-24 < 2^-17; the softmax's own f32 evaluation (exponential polynomial, 16 lane sums
    of 8 and a sum of 16, reciprocal, product) at most 2^-18.  So
        bound(i, d) = sum_t P_t |v_td| ((e^{2 delta_i} - 1) + 2^-9 + 2^-16).
    The last constant is 2^-16 rather than the 2^-17 of the accumulation alone: the cross term and the softmax's own
    rounding need room too.  In the 3xTF32 mode each operand is split into two TF32 parts and the products lose at most
    3 * 2^-20; 3 * 128 f32 additions stay below 2^-15.4: both coefficients become 2^-15."""
    us, uo = COEF[tf32]
    q, k, v = (np.asarray(a, np.float64) for a in (q, k, v))
    B, qh, T, dh = q.shape
    kvh, L = k.shape[1], k.shape[2]
    k, v = np.repeat(k, qh // kvh, axis=1), np.repeat(v, qh // kvh, axis=1)
    s = scale * np.einsum("bhqd,bhkd->bhqk", q, k)
    a = scale * np.einsum("bhqd,bhkd->bhqk", np.abs(q), np.abs(k))
    z = s if mask is None else s + np.asarray(mask, np.float64)
    t = np.arange(L)[None, None, None, :]
    if nonpad is not None:
        z = np.where(t >= np.clip(np.asarray(nonpad), 0, L)[:, None, None, None], -np.inf, z)
    if causal:
        z = np.where(t > np.arange(T)[None, None, :, None], -np.inf, z)
    with np.errstate(invalid="ignore", over="ignore"):
        p = np.exp(z - z.max(-1, keepdims=True))
        p = p / p.sum(-1, keepdims=True)
    p = np.where(np.isnan(p), 0.0, p)
    live = z > -np.inf
    delta = us * np.where(live, a, 0.0).max(-1) + 2.0 ** -22 * np.where(live, np.abs(z), 0.0).max(-1)
    ref = np.einsum("bhqk,bhkd->bhqd", p, v)
    with np.errstate(over="ignore"):
        bnd = np.einsum("bhqk,bhkd->bhqd", p, np.abs(v)) * (np.expm1(2.0 * delta)[..., None] + uo)
    return ref, bnd


def bound_ratio(got, ref, bnd):
    """max |got - ref| / bound (0 / 0 counts as 0: rows of exact zeros must come back as exact zeros)."""
    err = np.abs(np.asarray(got, np.float64) - ref)
    with np.errstate(invalid="ignore", divide="ignore"):
        r = np.where(err == 0, 0.0, err / bnd)
    return float(r.max())


def emulate(oracle, q, k, v, mask, scale):
    """The kernel's arithmetic in numpy: Q, K truncated to TF32 and summed in f32, z = fl(fl(S * scale) + mask), the
    reference's softmax (NaNs flushed), P and V truncated to TF32 and summed in f32."""
    s = np.matmul(trunc_tf32(q), trunc_tf32(k).swapaxes(-1, -2)) * F32(scale)
    p = oracle.softmax(s, -1, True) if mask is None else oracle.add_softmax(s, mask, flush_nans_to_zero=True)
    return np.matmul(trunc_tf32(p), trunc_tf32(v))


def expected_bits(oracle, q, k, mask, scale, perm, pas):
    """What the kernel must return for integer Q, K and the one-hot V of `one_hot_v(perm, pas)`: the oracle's
    AddSoftmax of the exact f32 scores, NaNs flushed, truncated to TF32, columns perm[64 pas : 64 pas + 64]."""
    s = np.matmul(q.astype(np.float64), k.astype(np.float64).swapaxes(-1, -2))
    assert np.abs(s).max() < 2 ** 24
    z = s.astype(F32) * F32(scale)
    p = oracle.softmax(z, -1, True) if mask is None else oracle.add_softmax(z, mask, flush_nans_to_zero=True)
    cols = perm[..., 64 * pas:64 * pas + 64]  # [B, H, 64]
    return trunc_tf32(np.take_along_axis(p, np.broadcast_to(cols[:, :, None, :], p.shape[:3] + (64,)), axis=-1))


def one_hot_v(perm, pas):
    """V[b, h, t, d] = 1 where t = perm[b, h, 64 pas + d]."""
    B, H, L = perm.shape
    v = np.zeros((B, H, L, 64), F32)
    bi, hi, di = np.meshgrid(np.arange(B), np.arange(H), np.arange(64), indexing="ij")
    v[bi, hi, perm[:, :, 64 * pas:64 * pas + 64], di] = 1.0
    return v


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the bound, the emulation and the expected-bits builder


def _random_case(rng, B, H, S, amp, mask_kind, L=128, dh=64):
    q = rng.uniform(-amp, amp, (B, H, S, dh)).astype(F32)
    k = rng.uniform(-amp, amp, (B, H, L, dh)).astype(F32)
    v = rng.uniform(-1, 1, (B, H, L, dh)).astype(F32)
    mask = None
    if mask_kind:
        mask = rng.uniform(-3, 0, (B, 1, 1, L)).astype(F32)
        mask[rng.random(mask.shape) < 0.1] = -np.inf
    return q, k, v, mask


def test_bound_holds_for_the_emulated_kernel(oracle):
    """300 seeded draws, flat and peaked rows, three scales, with and without a mask holding -inf entries: the emulated
    kernel stays inside the bound everywhere."""
    rng = np.random.default_rng(2024)
    worst = 0.0
    for i in range(300):
        amp = (1.0, 3.0)[i % 2]
        scale = (0.125, 0.1, 0.37)[i % 3]
        q, k, v, mask = _random_case(rng, 2, 2, 8, amp, i % 4 >= 2)
        ref, bnd = ref_and_bound(q, k, v, mask, scale)
        r = bound_ratio(emulate(oracle, q, k, v, mask, scale), ref, bnd)
        assert r <= 1.0, f"draw {i}: the emulated kernel exceeds the bound (ratio {r:.3f})"
        worst = max(worst, r)
    assert worst > 1e-3  # (the bound is not vacuous: the emulation's error uses a visible share of it)


@pytest.mark.parametrize("amp", [1.0, 3.0], ids=["flat", "peaked"])
def test_bound_catches_small_mistakes(oracle, amp):
    """Each mutation of the float64 result a subtly wrong kernel could produce leaves the bound somewhere: one key
    dropped from one row, two adjacent keys' V rows swapped, one batch's mask ignored, the scale applied twice."""
    rng = np.random.default_rng(7)
    B, H, S, scale = 2, 2, 16, 0.125
    q, k, v, mask = _random_case(rng, B, H, S, amp, True)
    mask[np.isinf(mask)] = -1.0
    ref, bnd = ref_and_bound(q, k, v, mask, scale)
    assert bound_ratio(emulate(oracle, q, k, v, mask, scale), ref, bnd) <= 1.0
    # one key of row (0, 0, 0) dropped: the key with its largest probability
    s = scale * (q[0, 0, 0].astype(np.float64) @ k[0, 0].astype(np.float64).T) + mask[0, 0, 0]
    t = int(np.argmax(s))
    dropped = mask.copy()
    dropped[0, 0, 0, t] = -np.inf
    one = ref.copy()
    one[0, 0, 0] = ref_and_bound(q, k, v, dropped, scale)[0][0, 0, 0]
    mut = {"one key dropped": one}
    t2 = min(t, 126)
    sw = v.copy()
    sw[0, 0, [t2, t2 + 1]] = sw[0, 0, [t2 + 1, t2]]
    mut["adjacent V rows swapped"] = ref_and_bound(q, k, sw, mask, scale)[0]
    nomask = mask.copy()
    nomask[1] = 0.0
    mut["one row's mask ignored"] = ref_and_bound(q, k, v, nomask, scale)[0]
    mut["scale applied twice"] = ref_and_bound(q, k, v, mask, scale * scale)[0]
    for name, m in mut.items():
        assert bound_ratio(m, ref, bnd) > 1.0, f"{name} ({'peaked' if amp > 1 else 'flat'} rows) stays inside the bound"


def test_expected_bits_builder(oracle):
    """The expected-bits builder on a small case: integer scores, exact zeros for a fully masked row and for rows with a
    +inf or NaN entry, the permutation read back column by column, and the TF32 truncation."""
    rng = np.random.default_rng(3)
    B, H, S = 4, 2, 8
    q = rng.integers(-16, 17, (B, H, S, 64)).astype(F32)
    k = rng.integers(-16, 17, (B, H, 128, 64)).astype(F32)
    mask = rng.uniform(-3, 0, (B, 1, 1, 128)).astype(F32)
    mask[1] = -np.inf
    mask[2, 0, 0, 5] = np.inf
    mask[3, 0, 0, 9] = np.nan
    perm = np.stack([np.stack([rng.permutation(128) for _ in range(H)]) for _ in range(B)])
    got = np.concatenate([expected_bits(oracle, q, k, mask, 0.37, perm, pas) for pas in (0, 1)], axis=-1)
    assert not got[1:].any(), "rows fully masked or holding +inf / NaN must be zeros"
    z = (np.matmul(q, k.swapaxes(-1, -2)) * F32(0.37) + mask[0:1])[0]
    p = oracle.softmax(z, -1, True)
    cols = np.take_along_axis(p, np.broadcast_to(perm[0][:, None, :], p.shape), -1)
    np.testing.assert_array_equal(got[0], trunc_tf32(cols))
    assert (got[0].view(np.uint32) & 0x1FFF == 0).all()
    # the one-hot V picks exactly those columns
    for pas in (0, 1):
        v = one_hot_v(perm, pas)
        np.testing.assert_array_equal(np.matmul(p[None], v[0:1])[0], cols[..., 64 * pas:64 * pas + 64])


# ---------------------------------------------------------------------------------------------------------------------
# GPU


@pytest.fixture(scope="module")
def rt():
    import rten_b200
    from rten_b200 import _lib
    _lib.load()
    return rten_b200


def _ctx(rt, tf32=True):
    ctx = rt.Context(0)
    ctx.set_f32_mode(not tf32)
    return ctx


def _assert_bits(got, exp, what):
    import gpu_checks
    gpu_checks.assert_bit_exact(got, exp, what)


# ---- the softmax stage bit for bit ------------------------------------------------------------------------------
# (B, heads, q_seq, scale, |Q|, |K| <= amp, mask form, value layout, output through a [B, S, H] view)
EXACT = [
    ("bert flat, no mask", (2, 12, 128, 0.125, 1, "none", "natural", False)),
    ("merged views, peaked, mask [B,1,1,128], scale 0.1", (3, 3, 256, 0.1, 16, "b11k", "merged", True)),
    ("transposed V, peaked, mask [128], scale 0.37, q_seq 512", (4, 1, 512, 0.37, 16, "k", "transposed", False)),
    ("flat, mask [1,1,1,128], scale 0.37", (2, 3, 128, 0.37, 1, "111k", "natural", True)),
    ("bert merged views, peaked, mask row stride 132", (4, 12, 128, 0.125, 16, "b11k_pad", "merged", True)),
    ("flat, -inf / +inf / NaN / f32 min mask, scale 0.1", (4, 3, 256, 0.1, 1, "edge", "natural", False)),
    ("bert merged views, peaked, -inf / +inf / NaN / f32 min mask", (4, 12, 128, 0.125, 16, "edge", "merged", True)),
    ("transposed V, flat, q_seq 512, 12 heads", (1, 12, 512, 0.125, 1, "b11k", "transposed", False)),
    ("transposed V, peaked, -inf / +inf / NaN / f32 min mask, scale 0.37", (4, 3, 128, 0.37, 16, "edge", "transposed", True)),
]


def _exact_data(seed, B, H, S, amp, mask_kind):
    """Integer Q and K (different per batch and head), the mask (different per batch), one permutation per head."""
    rng = np.random.default_rng(seed)
    q = rng.integers(-amp, amp + 1, (B, H, S, 64)).astype(F32)
    k = rng.integers(-amp, amp + 1, (B, H, 128, 64)).astype(F32)
    perm = np.stack([np.stack([rng.permutation(128) for _ in range(H)]) for _ in range(B)])
    mask = None
    if mask_kind in ("b11k", "b11k_pad", "edge"):
        mask = rng.uniform(-3, 0, (B, 1, 1, 128)).astype(F32)
    elif mask_kind in ("k", "111k"):
        mask = rng.uniform(-3, 0, (1, 1, 1, 128)).astype(F32)
    if mask_kind == "edge":  # batch 0: scattered -inf and f32 min; 1: every key -inf; 2: one +inf; 3: one NaN
        mask[0, 0, 0, rng.choice(128, 24, replace=False)] = -np.inf
        mask[0, 0, 0, rng.choice(128, 8, replace=False)] = np.finfo(F32).min
        mask[1] = -np.inf
        mask[2, 0, 0, 77] = np.inf
        mask[3, 0, 0, 3] = np.nan
    return q, k, perm, mask


def _device_mask(ctx, mask, kind):
    if mask is None:
        return None
    if kind == "k":
        return ctx.to_device(mask.reshape(128))
    if kind == "b11k_pad":  # rows 132 floats apart, the gaps NaN: a read past the row shows
        B = mask.shape[0]
        buf = np.full((B, 132), np.nan, F32)
        buf[:, :128] = mask.reshape(B, 128)
        return ctx.to_device(buf).view((B, 1, 1, 128), (132, 132, 132, 1))
    return ctx.to_device(mask)


def _device_qkv(ctx, q, k, v, layout):
    B, H, S, dh = q.shape
    L = k.shape[2]
    if layout == "merged":  # BertRunner's layout: strided views of one [B, S, 3 H dh] projection
        Sm, W = max(S, L), H * dh
        qkv = np.zeros((B, Sm, 3 * W), F32)
        for i, (x, rows) in enumerate(((q, S), (k, L), (v, L))):
            qkv[:, :rows, i * W:(i + 1) * W] = x.transpose(0, 2, 1, 3).reshape(B, rows, W)
        d = ctx.to_device(qkv)
        part = lambda i, rows: d.view((B, H, rows, dh), (Sm * 3 * W, dh, 3 * W, 1), i * W)
        return part(0, S), part(1, L), part(2, L)
    dv = ctx.to_device(v)
    if layout == "transposed":  # V stored as [B, H, dh, L], read by TMA
        dv = ctx.to_device(np.ascontiguousarray(v.transpose(0, 1, 3, 2))).view(v.shape, (H * dh * L, dh * L, 1, L))
    return ctx.to_device(q), ctx.to_device(k), dv


def _run_exact(rt, ctx, case, q, k, v, mask):
    B, H, S, scale, amp, mask_kind, layout, strided = case
    dq, dk, dv = _device_qkv(ctx, q, k, v, layout)
    dm = _device_mask(ctx, mask, mask_kind)
    op = rt.Attention(scale=scale)
    if not strided:
        return op.run(ctx, dq, dk, dv, attn_mask=dm).numpy()
    att = ctx.empty((B, S, H * 64))  # [B, S, H] as BertRunner writes it
    op.run(ctx, dq, dk, dv, attn_mask=dm, out=att.view((B, H, S, 64), (S * H * 64, 64, H * 64, 1)))
    return att.numpy().reshape(B, S, H, 64).transpose(0, 2, 1, 3)


@pytest.mark.gpu
@pytest.mark.parametrize("name,case", EXACT, ids=[c[0] for c in EXACT])
def test_softmax_stage_bit_exact(rt, oracle, monkeypatch, name, case):
    """Both passes of the one-hot V give the oracle's P (NaNs flushed, TF32-truncated) bit for bit, on the fused kernel
    and on the composed TF32 path (FusedMatMul -> AddSoftmax -> MatMul, forced by RTEN_B200_NO_FUSED_ATTN), which sees
    the same exact scores, the same softmax and the same truncated P . V."""
    B, H, S, scale, amp, mask_kind, layout, strided = case
    q, k, perm, mask = _exact_data(len(name), B, H, S, amp, mask_kind)
    ctx = _ctx(rt)
    for pas in (0, 1):
        want = expected_bits(oracle, q, k, mask, scale, perm, pas)
        v = one_hot_v(perm, pas)
        monkeypatch.delenv(NO_FUSED, raising=False)
        fused = _run_exact(rt, ctx, case, q, k, v, mask)
        monkeypatch.setenv(NO_FUSED, "1")
        composed = _run_exact(rt, ctx, case, q, k, v, mask)
        monkeypatch.delenv(NO_FUSED)
        _assert_bits(fused, want, f"{name}, pass {pas}: attn_fused_kernel vs the oracle's P")
        _assert_bits(composed, want, f"{name}, pass {pas}: the composed TF32 path vs the oracle's P")
        if mask_kind == "edge":  # fully masked, +inf, NaN: zero rows; the f32-min batch is a normal softmax
            assert not fused[1:4].any() and fused[0].any()


# ---- random data against float64 --------------------------------------------------------------------------------


@pytest.mark.gpu
@pytest.mark.parametrize("S", [128, 384])
@pytest.mark.parametrize("amp", [1.0, 3.0], ids=["uniform", "peaked"])
def test_random_data_within_the_bound(rt, S, amp):
    """BERT-base's attention (B 16, 12 heads) at q_seq 128 and 384, uniform and peaked rows, a [B,1,1,128] mask with
    -inf entries: every element inside ref_and_bound's TF32 bound, merged-projection views and the [B, S, H] output."""
    B, H = 16, 12
    q, k, v, mask = _random_case(np.random.default_rng(S + int(amp)), B, H, S, amp, True)
    ref, bnd = ref_and_bound(q, k, v, mask)
    ctx = _ctx(rt)
    got = _run_exact(rt, ctx, (B, H, S, 0.125, amp, "b11k", "merged", True), q, k, v, mask)
    r = bound_ratio(got, ref, bnd)
    assert r <= 1.0, f"q_seq {S} amp {amp}: error exceeds the bound (ratio {r:.3f})"


# ---- where each declined call goes ------------------------------------------------------------------------------
# overrides of the base call (B 2, 3 heads, q_seq 128, 128 keys, head size 64, TF32, mask [B,1,1,128]); "prefill" names
# the calls the streaming prefill kernel takes
DECLINED = [
    ("3xtf32", dict(tf32=False)),
    ("causal", dict(causal=True, prefill=True)),
    ("nonpad_kv_seqlen", dict(nonpad=[128, 77], prefill=True)),
    ("q_heads != kv_heads", dict(kvh=1, prefill=True)),
    ("per-head mask [B,H,1,128]", dict(mask="bh1k")),
    ("per-query mask [B,1,S,128]", dict(mask="b1sk")),
    ("mask row stride 130", dict(mask="stride130")),
    ("mask offset by one float", dict(mask="offset1")),
    ("q_seq 64", dict(S=64)),
    ("q_seq 192", dict(S=192)),
    ("96 keys", dict(L=96)),
    ("256 keys", dict(L=256)),
    ("head size 128", dict(dh=128)),
    ("Q offset by one float", dict(q_off=True)),
    ("natural V with row stride 65", dict(v_stride=65)),
    ("output row stride 66", dict(o_stride=66)),
]
SENTINEL = F32(-12345.5)


def _declined(rt, ctx, c, seed):
    """Run one declined call into a sentinel-filled buffer; (the result read back through the caller's view, the whole
    buffer, a mask of the view's elements in it, the float64 reference and bound)."""
    B, H, S, L, dh = 2, 3, c.get("S", 128), c.get("L", 128), c.get("dh", 64)
    kvh = c.get("kvh", H)
    rng = np.random.default_rng(seed)
    q = rng.uniform(-1, 1, (B, H, S, dh)).astype(F32)
    k = rng.uniform(-1, 1, (B, kvh, L, dh)).astype(F32)
    v = rng.uniform(-1, 1, (B, kvh, L, dh)).astype(F32)
    kind = c.get("mask", "b11k")
    mshape = {"bh1k": (B, H, 1, L), "b1sk": (B, 1, S, L)}.get(kind, (B, 1, 1, L))
    mask = rng.uniform(-3, 0, mshape).astype(F32)
    ref, bnd = ref_and_bound(q, k, v, mask, 0.125, c.get("causal", False), c.get("nonpad"), c.get("tf32", True))
    if kind == "stride130":
        buf = np.full((B, 130), np.nan, F32)
        buf[:, :L] = mask.reshape(B, L)
        dm = ctx.to_device(buf).view(mshape, (130, 130, 130, 1))
    elif kind == "offset1":
        dm = ctx.to_device(np.concatenate([[0.0], mask.ravel(), [0.0, 0.0, 0.0]]).astype(F32)).view(mshape, (L, L, L, 1), 1)
    else:
        dm = ctx.to_device(mask)
    if c.get("q_off"):
        dq = ctx.to_device(np.concatenate([[0.0], q.ravel()]).astype(F32)).view(q.shape, (H * S * dh, S * dh, dh, 1), 1)
    else:
        dq = ctx.to_device(q)
    if "v_stride" in c:
        vs = c["v_stride"]
        vb = np.zeros((B, kvh, L, vs), F32)
        vb[..., :dh] = v
        dv = ctx.to_device(vb).view(v.shape, (kvh * L * vs, L * vs, vs, 1))
    else:
        dv = ctx.to_device(v)
    os_ = c.get("o_stride", dh + 4)
    pad = 36  # (16-byte aligned: the view's own layout is the only thing a case changes)
    n = B * H * S * os_
    dbuf = ctx.to_device(np.full(n + 2 * pad, SENTINEL, F32))
    out = dbuf.view((B, H, S, dh), (H * S * os_, S * os_, os_, 1), pad)
    inside = np.zeros(n + 2 * pad, bool)
    inside[pad:pad + n].reshape(B, H, S, os_)[..., :dh] = True
    dl = ctx.to_device(np.asarray(c["nonpad"], np.int32)) if "nonpad" in c else None
    res = rt.Attention(is_causal=c.get("causal", False), q_num_heads=H, kv_num_heads=kvh, scale=0.125).run(
        ctx, dq, ctx.to_device(k), dv, attn_mask=dm, nonpad_kv_seqlen=dl, out=out)
    return res, out, dbuf.numpy(), inside, ref, bnd


@pytest.mark.gpu
@pytest.mark.parametrize("name,c", DECLINED, ids=[d[0] for d in DECLINED])
def test_declined_calls(rt, name, c):
    """Calls the fused kernel declines meet the float64 bound of the path that takes them, and write the caller's `out`
    view and nothing else: the declined branch's scope neither frees nor replaces a tensor it did not allocate."""
    ctx = _ctx(rt, c.get("tf32", True))
    res, out, whole, inside, ref, bnd = _declined(rt, ctx, c, len(name))
    assert res is out
    r = bound_ratio(out.numpy(), ref, bnd)
    assert r <= 1.0, f"{name}: error exceeds the bound (ratio {r:.3f})"
    assert (whole[~inside] == SENTINEL).all(), f"{name}: {int((whole[~inside] != SENTINEL).sum())} elements outside the view written"


def _kernel_probe():
    """In a child process: the kernels each bit-exact case and each declined call (and its base form) launched, one CUPTI session each, as JSON."""
    import gpu_checks as gc
    import rten_b200 as rt
    res = {}
    ctx = _ctx(rt)
    for name, case in EXACT:
        B, H, S, scale, amp, mask_kind, layout, strided = case
        q, k, perm, mask = _exact_data(len(name), B, H, S, amp, mask_kind)
        _, names = gc._kernels_launched(lambda: _run_exact(rt, ctx, case, q, k, one_hot_v(perm, 0), mask))
        res[name] = sorted(names)
    for name, c in [("base", {})] + DECLINED:
        cx = _ctx(rt, c.get("tf32", True))
        _, names = gc._kernels_launched(lambda: _declined(rt, cx, c, len(name)))
        res[name] = sorted(names)
    print(json.dumps(res))


@pytest.mark.gpu
def test_kernel_identity():
    """attn_fused_kernel runs every bit-exact case, and the declined calls' base form, and none of the declined calls;
    the prefill kernel takes the causal, nonpad_kv_seqlen and grouped-query calls.  CUPTI runs in a child process, so no profiler state stays behind."""
    import subprocess
    code = (f"import sys; sys.path[:0] = [{os.path.dirname(HERE)!r}, {HERE!r}]; "
            "import test_gpu_attention_encoder as t; t._kernel_probe()")
    res = subprocess.run([sys.executable, "-s", "-c", code], capture_output=True, text=True, timeout=900)
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-4000:]
    names = json.loads(res.stdout.strip().splitlines()[-1])
    fused = lambda key: any("attn_fused_kernel" in n for n in names[key])
    for name in [e[0] for e in EXACT] + ["base"]:
        assert fused(name), f"{name}: attn_fused_kernel did not run ({names[name]})"
    for name, c in DECLINED:
        assert not fused(name), f"{name}: attn_fused_kernel ran"
        assert any("attn_prefill_kernel" in n for n in names[name]) == c.get("prefill", False), (name, names[name])


# ---- graph replay -----------------------------------------------------------------------------------------------


@pytest.mark.gpu
def test_graph_replay(rt):
    """A fused call captured in a CUDA graph and replayed three times gives the eager call's bits each time."""
    B, H, S = 4, 12, 128
    q, k, perm, mask = _exact_data(5, B, H, S, 16, "edge")
    v = np.random.default_rng(6).uniform(-1, 1, (B, H, 128, 64)).astype(F32)
    ctx = _ctx(rt)
    dq, dk, dv = _device_qkv(ctx, q, k, v, "merged")
    dm = ctx.to_device(mask)
    att = ctx.empty((B, S, H * 64))
    run = lambda: rt.Attention(scale=0.125).run(ctx, dq, dk, dv, attn_mask=dm, out=att.view((B, H, S, 64), (S * H * 64, 64, H * 64, 1)))
    run()
    eager = att.numpy()
    assert np.isfinite(eager).all() and not eager.reshape(B, S, H, 64)[1:4].any()
    ctx.graph_begin()
    run()
    graph = ctx.graph_end()
    for i in range(3):
        att.copy_from(np.full(att.shape, np.nan, F32))
        graph.launch()
        ctx.sync()
        _assert_bits(att.numpy(), eager, f"graph replay {i + 1} vs the eager call")


# ---- fully masked rows on every Attention path ------------------------------------------------------------------
# (B, heads, q_seq, causal, f32 mode TF32, composed forced)
PATHS = [
    ("decode", (3, 4, 1, False, False, False)),
    ("prefill", (3, 4, 128, True, False, False)),
    ("fused", (3, 4, 128, False, True, False)),
    ("composed tf32", (3, 4, 128, False, True, True)),
    ("composed 3xtf32", (3, 4, 128, False, False, False)),
]


@pytest.mark.gpu
@pytest.mark.parametrize("name,p", PATHS, ids=[x[0] for x in PATHS])
def test_fully_masked_rows_are_zeros(rt, monkeypatch, name, p):
    """A mask that is -inf at every key of batch 1 gives exact zeros there on every path; the other batches meet the
    path's bound."""
    B, H, S, causal, tf32, composed = p
    q, k, v, _ = _random_case(np.random.default_rng(len(name)), B, H, S, 1.0, False)
    mask = np.random.default_rng(1).uniform(-3, 0, (B, 1, 1, 128)).astype(F32)
    mask[1] = -np.inf
    ref, bnd = ref_and_bound(q, k, v, mask, 0.125, causal, None, tf32)
    ctx = _ctx(rt, tf32)
    if composed:
        monkeypatch.setenv(NO_FUSED, "1")
    got = rt.Attention(is_causal=causal, scale=0.125).run(ctx, ctx.to_device(q), ctx.to_device(k), ctx.to_device(v),
                                                          attn_mask=ctx.to_device(mask)).numpy()
    assert not got[1].any(), f"{name}: the fully masked batch is not exact zeros"
    r = bound_ratio(got, ref, bnd)
    assert r <= 1.0, f"{name}: error exceeds the bound (ratio {r:.3f})"


@pytest.mark.gpu
def test_fully_masked_batch_through_the_executor(rt):
    """An opset-23 Attention node in a model: a [B,1,1,128] mask that pads out batch 1 entirely gives zeros there."""
    import onnx_writer as W
    from rten_b200.model import Model
    B, H, S = 3, 4, 128
    q, k, v, _ = _random_case(np.random.default_rng(9), B, H, S, 1.0, False)
    mask = np.zeros((B, 1, 1, 128), F32)
    mask[0, ..., 100:] = -np.inf
    mask[1] = -np.inf
    nodes = [W.node("Attention", ["q", "k", "v", "m"], ["y"], scale=0.125)]
    ins = [W.value_info(n, W.FLOAT, list(a.shape)) for n, a in (("q", q), ("k", k), ("v", v), ("m", mask))]
    data = W.model(nodes, [], ins, [W.value_info("y", W.FLOAT, [B, H, S, 64])], opset=23)
    ctx = _ctx(rt)
    (y,) = Model(ctx, data).run({n: ctx.to_device(a) for n, a in (("q", q), ("k", k), ("v", v), ("m", mask))})
    got = y.numpy()
    ref, bnd = ref_and_bound(q, k, v, mask)
    assert not got[1].any(), "the padded batch is not exact zeros"
    r = bound_ratio(got, ref, bnd)
    assert r <= 1.0, f"executor: error exceeds the bound (ratio {r:.3f})"
