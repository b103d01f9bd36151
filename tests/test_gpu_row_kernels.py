"""`pytest -m gpu`: every template instance of the Softmax / AddSoftmax, row normalization (LayerNormalization,
RMSNormalization and the skip layer norms), f32 skinny-GEMM and fused quantized-linear kernels, each selected by name and
checked bit for bit.

The launchers (rowops.cu launch_softmax / launch_norm, skinny.cu launch_skinny_f32 / launch_qlinear) pick an
instance at run time from the row width, the row count, the SM count and pointer alignment.  The rules are restated
below (`*_rule`); `VARIANTS` lists every instance the library compiles (tests/test_row_kernel_table_cpu.py keeps it
equal to the built library's symbols).  The case lists select every instance at least twice, one of them with a
partial last unit (fewer float4s per thread than the instance holds, a row count that leaves dead rows in the last
warp, or a column count that leaves dead columns in the last tile).  Widths derived from the SM count make every
skinny instance loop over a second column tile per CTA, and every double-buffered quantized-linear instance over a
third.

  * kernel identity: every call the numbers tests make of a case (each skinny epilogue, the generic rerun of each row
    case) runs under CUPTI in a child process; the kernel that ran must be the one the rule names, and every instance
    of `VARIANTS` must have run;
  * Softmax / AddSoftmax and the row normalizations: bit-exact against the oracle, and the same bits again with the
    vector kernels switched off (RTEN_B200_NO_VEC_ROWS), with -inf / +inf / NaN / +-3e38 rows, constant rows, eps = 0,
    rows far from zero, broadcast masks, misaligned / in-place / strided inputs and outputs; random rows also against
    float64;
  * skinny GEMM: small-integer operands (every partial sum exact in f32, so the result is the exact product bit for bit
    in any summation order) and U[0, 1) floats against a float64 product under 1e-8 + 1e-5 |ref|, with alpha, bias,
    Gemm's beta * C, an activation, a row-strided A and a strided output, in both f32 modes;
  * quantized linear: bit-exact against the operator chain of the oracle with scalar / per-column weight zero points,
    bias, residual, every activation, rounding ties, all-zero and constant inputs, and the composed chain just past the
    kernel's limits;
  * DynamicQuantizeLinear: degenerate ranges on the one-kernel and three-kernel paths, and the ranged form fed by a
    MatMulIntegerToFloat out_range, before and after re-arming it."""
import json
import os
import re
import subprocess
import sys
import zlib

import numpy as np
import pytest

import gpu_checks as gc

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
F32 = np.float32

# ---- the instances the library compiles, and the launchers' selection rules ------------------------------------------
# The operators of launch_norm and their flag sets FL: RMS 1, skip 2, bias 4, sum output 8
NORM_OPS = {"LayerNormalization": 0, "RMSNormalization": 1,
            "SkipLayerNormalization": 2, "SkipLayerNormalization + bias": 6, "SkipLayerNormalization + sum": 10,
            "SkipLayerNormalization + bias + sum": 14, "SkipSimplifiedLayerNormalization": 3,
            "SkipSimplifiedLayerNormalization + bias": 7, "SkipSimplifiedLayerNormalization + sum": 11,
            "SkipSimplifiedLayerNormalization + bias + sum": 15}
NORM_FLAGS = sorted(NORM_OPS.values())
VARIANTS = {
    # <S (threads per row / 4), FMAX (float4s per thread)>
    "softmax_vec_kernel": [(1, 2), (1, 4), (1, 8), (1, 16), (2, 2), (2, 4), (2, 8), (2, 16),
                           (4, 2), (4, 4), (4, 8), (4, 16), (8, 2), (8, 4), (8, 8), (8, 16)],
    # <S (threads per row / 16), FMAX, FL (the operator's flag set, NORM_FLAGS)>
    "norm_vec_kernel": [(S, fm, fl) for S in (1, 2) for fm in (4, 8, 12, 16) for fl in NORM_FLAGS],
    # <VPT (float4s per thread), FL>
    "norm_wide_kernel": [(vpt, fl) for vpt in (4, 8) for fl in NORM_FLAGS],
    # <MT (rows), CPW (columns per warp)>
    "skinny_f32_kernel": [(8, 1), (8, 2), (16, 1), (16, 2), (32, 1)],
    # <MT, CPW, KI (16-byte chunks per lane / 32), WSIGNED, FLN (float4s per lane of the layer norm), DB (double-buffered)>
    "qlinear_kernel": [(8, 1, 2, 0, 6, 0), (8, 1, 2, 1, 6, 0), (8, 2, 2, 0, 6, 0), (8, 2, 2, 1, 6, 0),
                       (8, 4, 2, 0, 6, 1), (8, 4, 2, 1, 6, 1), (8, 1, 6, 0, 6, 0), (8, 1, 6, 1, 6, 0),
                       (16, 1, 2, 0, 6, 0), (16, 1, 2, 1, 6, 0), (16, 2, 2, 0, 6, 0), (16, 2, 2, 1, 6, 0),
                       (16, 4, 2, 0, 6, 1), (16, 4, 2, 1, 6, 1), (16, 1, 6, 0, 6, 0), (16, 1, 6, 1, 6, 0),
                       (8, 1, 2, 0, 8, 0), (8, 1, 2, 1, 8, 0), (8, 2, 2, 0, 8, 0), (8, 2, 2, 1, 8, 0),
                       (8, 4, 2, 0, 8, 1), (8, 4, 2, 1, 8, 1),
                       (16, 1, 2, 0, 8, 0), (16, 1, 2, 1, 8, 0), (16, 2, 2, 0, 8, 0), (16, 2, 2, 1, 8, 0),
                       (16, 4, 2, 0, 8, 1), (16, 4, 2, 1, 8, 1)],
}
GENERIC = ("softmax_kernel", "norm_kernel")
FAMILY_KERNELS = {"softmax": ("softmax_vec_kernel", "softmax_kernel"), "norm": ("norm_vec_kernel", "norm_wide_kernel", "norm_kernel"),
                  "skinny": ("skinny_f32_kernel",), "qlinear": ("qlinear_kernel",)}

_NAME = re.compile(r"rtb::(\w+)(?:<([^<>]*)>)?\(")


def kernel_key(name, kernels=None):
    """(kernel, template arguments) of a demangled kernel name of `kernels` (default: the four families here), else
    None.  Accepts both spellings of the arguments: `<1, 2>` / `<.., false, ..>` (CUPTI) and `<(int)1, (int)2>` /
    `(bool)0` (cu++filt).  Values become ints, type arguments stay names (`float`, `int`)."""
    kernels = set(VARIANTS) | set(GENERIC) if kernels is None else kernels
    for m in _NAME.finditer(name):
        if m.group(1) in kernels:
            args = []
            for a in (m.group(2).split(",") if m.group(2) else []):
                a = re.sub(r"^\((int|bool)\)", "", a.strip())
                args.append({"true": 1, "false": 0}[a] if a in ("true", "false") else int(a) if re.fullmatch(r"-?\d+", a) else a)
            return m.group(1), tuple(args)
    return None


def softmax_rule(n, rows, sms, vec_ok=True):
    """launch_softmax: the fewest segments S (4 S threads per row, F = n / 16 S float4s each, F <= 16) whose rows give
    every SM 32 warps, or with F <= 2; the generic warp-per-row kernel without an S, on misaligned rows or masks."""
    S = 0
    for c in (1, 2, 4, 8):
        if n % (16 * c) or n // (16 * c) > 16:
            continue
        S = c
        if (rows * 4 * c + 31) // 32 >= 32 * sms or n // (16 * c) <= 2:
            break
    if not S or not vec_ok or rows >= 0x7fffffff:
        return "softmax_kernel", ()
    F = n // (16 * S)
    return "softmax_vec_kernel", (S, 2 if F <= 2 else 4 if F <= 4 else 8 if F <= 8 else 16)


def norm_rule(n, rows, sms, fl, aligned=True):
    """launch_norm, for aligned rows with n % 64 == 0 and n <= 8192: S = 1 (16 threads per row) when n <= 1024 and the
    rows give every SM 32 warps or no S = 2 fits; S = 2 when n % 128 == 0, n <= 2048; F = n / 64 S float4s per thread
    rounded up to 4, 8, 12 or 16.  No S fits (n > 2048, or n / 64 > 16 and odd): one CTA per row, 4 float4s per thread
    up to n = 4096, else 8.  Any other row: the generic warp-per-row kernel."""
    if n % 64 or n > 8192 or not aligned:
        return "norm_kernel", ()
    S = 0
    for c in (1, 2):
        if n % (64 * c) or n // (64 * c) > 16:
            continue
        S = c
        if (rows * 16 * c + 31) // 32 >= 32 * sms:
            break
    if not S:
        return "norm_wide_kernel", (4 if n <= 4096 else 8, fl)
    F = n // (64 * S)
    return "norm_vec_kernel", (S, 4 if F <= 4 else 8 if F <= 8 else 12 if F <= 12 else 16, fl)


def skinny_rule(M, N):
    mt = 8 if M <= 8 else 16 if M <= 16 else 32
    return "skinny_f32_kernel", (mt, 1 if mt == 32 else 2 if N >= 4096 else 1)


def qlinear_rule(M, K, N, ln, signed):
    """launch_qlinear (None: qlinear_supported refuses the shape and the composed operator chain runs)."""
    if not (1 <= M <= 16 and K % 16 == 0 and 16 <= K <= 3072 and (not ln or (K % 128 == 0 and K <= 1024))):
        return None
    mt = 8 if M <= 8 else 16
    ki = 2 if K // 16 <= 64 else 6
    cpw = 1 if ki == 6 else 4 if N >= 8192 else 2 if N >= 2048 else 1
    fln = 8 if ln and K // 128 > 6 else 6
    return "qlinear_kernel", (mt, cpw, ki, int(signed), fln, int(cpw == 4))


def _rng(*key):
    return np.random.default_rng(zlib.crc32(repr(key).encode()))


def _bits(got, want, what):
    gc.assert_bit_exact(np.asarray(got), np.asarray(want), what)


# ---- Softmax / AddSoftmax ---------------------------------------------------------------------------------------------
def softmax_specs(sms):
    big = lambda S: -(-32 * sms * 32 // (4 * S))  # rows at which S segments per row give every SM 32 warps
    shapes = [(16, 7), (32, 5), (48, 9), (64, big(1)), (80, 3), (112, 6), (128, big(1)), (144, 5), (240, 3), (256, big(1)),
              (64, 7), (64, 2), (96, 5), (128, big(2)), (160, 3), (224, 7), (288, 5), (480, 3),
              (128, 7), (128, 30), (192, 5), (256, big(4)), (320, 3), (448, 6), (576, 5), (960, 3),
              (256, 7), (256, 2), (384, 3), (512, 5), (640, 3), (1024, 2), (1152, 3), (2048, 5),
              (1, 4), (100, 6), (4096, 3)]  # generic: n = 1, n % 16 != 0, more than 16 float4s per thread at every S
    specs = [dict(kind="softmax", n=n, rows=rows) for n, rows in shapes]
    for n in (64, 128, 192, 2048):
        for ms in ((2, 1, 1, n), (1, 1, 16, n), (n,), (2, 3, 1, 1)):
            specs.append(dict(kind="add_softmax", x=(2, 3, 16, n), m=ms))
    specs += [dict(kind="add_softmax", x=(2, 2, 3, 4, 128), m=(2, 1, 3, 1, 128)),  # four strided leading mask dims
              dict(kind="add_softmax", x=(2, 2, 3, 4, 320), m=(2, 1, 3, 1, 320)),
              dict(kind="add_softmax_padded_mask", x=(2, 3, 16, 128)),  # mask rows 129 floats apart: generic
              dict(kind="add_softmax_in_place", x=(2, 3, 16, 64), m=(2, 1, 1, 64)),
              dict(kind="softmax_misaligned", n=128, rows=7),
              dict(kind="softmax_in_place", n=256, rows=7),
              dict(kind="softmax_in_place_misaligned", n=192, rows=5),
              # an aligned input into a misaligned output view (generic), and into rows 260 floats apart (the vector
              # kernel into a temporary, then a strided copy); Softmax.run has no `out`, so these call the C ABI
              dict(kind="softmax_out_misaligned", n=128, rows=7),
              dict(kind="softmax_out_strided", n=256, rows=7),
              dict(kind="softmax_axis1", shape=(3, 64, 5))]
    return specs


def softmax_expected(s, sms):
    k = s["kind"]
    if k in ("softmax", "softmax_in_place", "softmax_out_strided"):
        return softmax_rule(s["n"], s["rows"], sms)
    if k in ("softmax_misaligned", "softmax_in_place_misaligned", "softmax_out_misaligned"):
        return softmax_rule(s["n"], s["rows"], sms, vec_ok=False)
    if k == "softmax_axis1":
        return softmax_rule(s["shape"][1], s["shape"][0] * s["shape"][2], sms)
    rows = int(np.prod(s["x"][:-1]))
    return softmax_rule(s["x"][-1], rows, sms, vec_ok=k != "add_softmax_padded_mask")


def _special_rows(x):
    """-inf entries, an all -inf row, +inf, NaN, +-3e38 in the first rows (the last row always stays finite)"""
    n = x.shape[1]
    fill = [lambda v: v.__setitem__(slice(None, None, 3), -np.inf), lambda v: v.fill(-np.inf),
            lambda v: v.__setitem__(n // 2, np.inf), lambda v: v.__setitem__(n - 1, np.nan),
            lambda v: (v.__setitem__(slice(None, None, 2), 3e38), v.__setitem__(slice(1, None, 2), -3e38))]
    for i in range(min(len(fill), x.shape[0] - 1)):
        fill[i](x[i])
    return min(len(fill), x.shape[0] - 1)  # first row of random values


def softmax_prepare(s):
    r = _rng("softmax", sorted(s.items()))
    k = s["kind"]
    if k == "softmax_axis1":
        return dict(x=r.uniform(-4, 4, s["shape"]).astype(F32))
    if k.startswith("softmax"):
        x = r.uniform(-4, 4, (s["rows"], s["n"])).astype(F32)
        return dict(x=x, first=_special_rows(x))
    x = r.uniform(-3, 3, s["x"]).astype(F32)
    first = _special_rows(x.reshape(-1, x.shape[-1]))
    m = r.uniform(-2, 0, s.get("m", (1, 1, 16, s["x"][-1]))).astype(F32)
    return dict(x=x, m=m, first=first)


def softmax_launch(rt, ctx, s, inp, flush=False):
    k = s["kind"]
    x = inp["x"]
    if k == "softmax":
        return rt.Softmax(-1, flush).run(ctx, ctx.to_device(x)).numpy()
    if k == "softmax_axis1":
        return rt.Softmax(1, flush).run(ctx, ctx.to_device(x)).numpy()
    if k in ("softmax_misaligned", "softmax_in_place_misaligned"):
        buf = ctx.to_device(np.concatenate([np.zeros(1, F32), x.reshape(-1), np.zeros(3, F32)]))
        xv = buf.view(x.shape, (x.shape[1], 1), 1)  # 4 bytes past a 16-byte boundary
        y = rt.Softmax(-1, flush).run(ctx, xv, in_place=k == "softmax_in_place_misaligned")
        return y.numpy()
    if k == "softmax_in_place":
        d = ctx.to_device(x)
        assert rt.Softmax(-1, flush).run(ctx, d, in_place=True) is d
        return d.numpy()
    if k in ("softmax_out_misaligned", "softmax_out_strided"):
        import ctypes as C
        from rten_b200.ops import _Args
        rows, n = x.shape
        pad, off = (4, 0) if k == "softmax_out_strided" else (0, 1)
        buf = ctx.to_device(np.full(rows * (n + pad) + 4, 7.0, F32))
        xd = ctx.to_device(x)
        A = _Args(ctx)
        o = A.out(buf.view(x.shape, (n + pad, 1), off))
        ctx.check(ctx.lib.rten_b200_softmax(ctx.handle, A.t(xd), None, -1, int(flush), C.byref(o)))
        full = buf.numpy()
        got = full[off:off + rows * (n + pad)].reshape(rows, n + pad)
        outside = np.concatenate([full[:off], got[:, n:].reshape(-1), full[off + rows * (n + pad):]])
        assert (outside == 7.0).all(), f"{k}: writes outside the output view"
        return np.ascontiguousarray(got[:, :n])
    m = inp["m"]
    if k == "add_softmax_padded_mask":
        n = x.shape[-1]
        mb = ctx.to_device(np.concatenate([m.reshape(16, n), np.zeros((16, 1), F32)], axis=1))
        return rt.AddSoftmax(flush).run(ctx, ctx.to_device(x), mb.view((1, 1, 16, n), (16 * (n + 1), 16 * (n + 1), n + 1, 1))).numpy()
    if k == "add_softmax_in_place":
        d = ctx.to_device(x)
        assert rt.AddSoftmax(flush).run(ctx, d, ctx.to_device(m), in_place=True) is d
        return d.numpy()
    return rt.AddSoftmax(flush).run(ctx, ctx.to_device(x), ctx.to_device(m)).numpy()


def softmax_want(oracle, s, inp, flush):
    x = inp["x"]
    if s["kind"] == "softmax_axis1":
        return oracle.softmax(x, 1, flush)
    if "m" in inp:
        m = inp["m"] if s["kind"] != "add_softmax_padded_mask" else inp["m"].reshape(1, 1, 16, x.shape[-1])
        return oracle.add_softmax(x, m, flush)
    return oracle.softmax(x, -1, flush)


def softmax_f64_check(s, inp, got, what):
    """float64 softmax of the rows that hold random values only, under 1e-8 + 1e-5 |ref|"""
    x = inp["x"].astype(np.float64)
    if s["kind"] == "softmax_axis1":
        e = np.exp(x - x.max(1, keepdims=True))
        gc.assert_reference_rule(got, e / e.sum(1, keepdims=True), what)
        return
    if "m" in inp:
        x = x + (inp["m"] if s["kind"] != "add_softmax_padded_mask" else inp["m"].reshape(1, 1, 16, x.shape[-1]))
    x2 = x.reshape(-1, x.shape[-1])[inp["first"]:]
    e = np.exp(x2 - x2.max(1, keepdims=True))
    gc.assert_reference_rule(got.reshape(-1, x.shape[-1])[inp["first"]:], e / e.sum(1, keepdims=True), what)


# ---- row normalization ------------------------------------------------------------------------------------------------
LN_ARMS = ("scalar scale", "scalar scale + scalar bias", "scale", "scale + bias", "scale + scalar bias", "scale + bias, eps 0")


def norm_specs(sms):
    big = 2 * 32 * sms + 1  # rows at which 16 lanes per row give every SM 32 warps (odd: a dead row in the last warp)
    # For every operator: per vector instance (S = 1, then S = 2; FMAX 4, 8, 12, 16) a row of fewer float4s per thread
    # than the instance holds and a full one; the CTA-per-row kernel at 4 and 8 float4s per thread, partial and full;
    # the generic kernel
    shapes = [(64, 7), (256, big), (320, 3), (512, big), (576, 5), (768, big), (832, 3), (1024, big),
              (128, 6), (512, 3), (768, 5), (1024, 4), (1152, 3), (1536, 2), (1664, 3), (2048, 5),
              (2112, 3), (4096, 3), (5120, 3), (8192, 2), (100, 5)]
    ln = "LayerNormalization"
    specs = [dict(kind="rows", op=op, n=n, rows=rows) for op in NORM_OPS for n, rows in shapes]
    specs += [dict(kind="rows", op=ln, n=n, rows=rows) for n, rows in ((192, 5), (448, 9), (704, 3), (960, 7))]
    return specs + [dict(kind=k, op=ln, n=n, rows=rows) for k, n, rows in (
        ("misaligned x", 768, 5), ("misaligned out", 768, 5), ("strided out", 768, 5), ("in place", 1024, 3))]


def norm_expected(s, sms):
    return norm_rule(s["n"], s["rows"], sms, NORM_OPS[s["op"]], aligned=not s["kind"].startswith("misaligned"))


def norm_prepare(s):
    r = _rng("norm", sorted(s.items()))
    n, rows = s["n"], s["rows"]
    x = (r.standard_normal((rows, n)) * 2).astype(F32)
    specials = [lambda v: v.fill(0.75), lambda v: v.__setitem__(slice(None), (1e4 + r.standard_normal(n)).astype(F32)),
                lambda v: v.__setitem__(1, np.inf), lambda v: v.__setitem__(0, -np.inf), lambda v: v.__setitem__(n // 2, np.nan)]
    first = min(len(specials), rows - 1)
    for i in range(first):
        specials[i](x[i])
    g = (1 + 0.1 * r.standard_normal(n)).astype(F32)
    b = (0.1 * r.standard_normal(n)).astype(F32)
    k = r.standard_normal((rows, n)).astype(F32)  # skip
    bi = (0.1 * r.standard_normal(n)).astype(F32)  # the skip norms' bias
    return dict(x=x, g=g, b=b, k=k, bi=bi, first=first)


def _ln_params(inp, arm):
    gs, bs = np.array([1.25], F32), np.array([0.375], F32)
    return {"scalar scale": (gs, None, None), "scalar scale + scalar bias": (gs, bs, None), "scale": (inp["g"], None, None),
            "scale + bias": (inp["g"], inp["b"], None), "scale + scalar bias": (inp["g"], bs, None),
            "scale + bias, eps 0": (inp["g"], inp["b"], 0.0)}[arm]


def _layer_norm_launch(rt, ctx, s, inp, arm):
    x = inp["x"]
    g, b, eps = _ln_params(inp, arm)
    op = rt.LayerNormalization(-1, eps)
    gd, bd = ctx.to_device(g), None if b is None else ctx.to_device(b)  # (one-element scale / bias: read on the device)
    k = s["kind"]
    rows, n = x.shape
    if k == "misaligned x":
        buf = ctx.to_device(np.concatenate([np.zeros(1, F32), x.reshape(-1), np.zeros(3, F32)]))
        return op.run(ctx, buf.view(x.shape, (n, 1), 1), gd, bd).numpy()
    if k in ("misaligned out", "strided out"):
        pad = 4 if k == "strided out" else 0
        buf = ctx.to_device(np.full(rows * (n + pad) + 4, 7.0, F32))
        view = buf.view(x.shape, (n + pad, 1), 1 if k == "misaligned out" else 0)
        y = op.run(ctx, ctx.to_device(x), gd, bd, out=view)
        assert y is view
        full = buf.numpy()
        off = 1 if k == "misaligned out" else 0
        got = full[off:off + rows * (n + pad)].reshape(rows, n + pad)
        assert (got[:, n:] == 7.0).all() and (full[:off] == 7.0).all(), f"{k}: writes outside the output view"
        return np.ascontiguousarray(got[:, :n])
    if k == "in place":
        d = ctx.to_device(x)
        op.run(ctx, d, gd, bd, out=d)
        return d.numpy()
    return op.run(ctx, ctx.to_device(x), gd, bd).numpy()


def norm_launch(rt, ctx, s, inp, arm="scale + bias"):
    """The operator's output; with the sum output, output and sum stacked"""
    op = s["op"]
    if op == "LayerNormalization":
        return _layer_norm_launch(rt, ctx, s, inp, arm)
    x, g = ctx.to_device(inp["x"]), ctx.to_device(inp["g"])
    if op == "RMSNormalization":
        return rt.RMSNormalization(-1, 1e-5).run(ctx, x, g).numpy()
    skip, bias, want_sum = ctx.to_device(inp["k"]), ctx.to_device(inp["bi"]) if "bias" in op else None, op.endswith("sum")
    if op.startswith("SkipSimplified"):
        res = rt.SkipSimplifiedLayerNormalization(1e-5).run(ctx, x, skip, g, bias, want_sum=want_sum)
    else:
        res = rt.SkipLayerNormalization(1e-5).run(ctx, x, skip, g, ctx.to_device(inp["b"]), bias, want_sum=want_sum)
    return np.stack([t.numpy() for t in res]) if want_sum else res.numpy()


def norm_want(oracle, s, inp, arm="scale + bias"):
    from oracle import norms
    op = s["op"]
    if op == "LayerNormalization":
        g, b, eps = _ln_params(inp, arm)
        return oracle.layer_norm(inp["x"], g, b, -1, eps)
    if op == "RMSNormalization":
        return norms.rms_norm(inp["x"], inp["g"], -1, 1e-5)
    rms = op.startswith("SkipSimplified")
    out, sm = norms.skip_layer_norm(inp["x"], inp["k"], inp["g"], None if rms else inp["b"], inp["bi"] if "bias" in op else None,
                                    1e-5, rms=rms)
    return np.stack([out, sm]) if op.endswith("sum") else out


# ---- skinny f32 GEMM --------------------------------------------------------------------------------------------------
SKINNY_EPILOGUES = ("alpha + bias", "Gemm beta * C", "bias + residual + activation", "row-strided A, strided out")


def wide_n(sms, nt, lo, loops):
    """An output width of at least `lo` columns whose tiles of `nt` columns number more than `loops` x SMs, and whose
    last tile is partial"""
    return nt * max(-(-lo // nt), loops * sms + 9) + nt // 4 + 1


def tiles_per_cta(fam, s, sms):
    """Column tiles the busiest CTA walks.  The skinny GEMM and the double-buffered quantized linear cap their grid
    at 2 CTAs per SM and loop over the tiles beyond it; the other quantized-linear variants take one tile per CTA."""
    want = FAMILIES[fam][1](s, sms)
    if want is None or fam not in ("skinny", "qlinear"):
        return 0
    cpw = want[1][1]
    tiles = -(-s["N"] // (8 * cpw))
    grid = tiles if fam == "qlinear" and cpw != 4 else min(tiles, 2 * sms)
    return -(-tiles // grid)


def skinny_specs(sms):
    shapes = [(1, 4, 7), (8, 1028, 3000), (5, 3076, 1),  # <8, 1>
              (1, 4100, 4097), (8, 1024, 5000),  # <8, 2>
              (9, 1020, 33), (16, 4100, 2500),  # <16, 1>
              (9, 3076, 4100), (16, 1028, wide_n(sms, 16, 4096, 2)),  # <16, 2>
              (17, 1024, 100), (32, 4100, 3001), (24, 4, 9)]  # <32, 1>
    return [dict(kind="skinny", M=M, K=K, N=N) for M, K, N in shapes]


def skinny_expected(s, sms):
    return skinny_rule(s["M"], s["N"])


def skinny_prepare(s, ints=True):
    r = _rng("skinny", sorted(s.items()), ints)
    M, K, N = s["M"], s["K"], s["N"]
    if ints:  # |a|, |b| <= 8: every partial sum is an integer below 2^24, exact in f32 in any order
        f = lambda shape, lim=8: r.integers(-lim, lim + 1, shape).astype(F32)
        return dict(a=f((M, K)), bt=f((N, K)), bias=f(N, 50), c=f((M, N), 50), res=f((M, N), 50), ints=True)
    f = lambda shape: r.random(shape, F32)
    return dict(a=f((M, K)), bt=f((N, K)), bias=f(N), c=f((M, N)), res=f((M, N)), ints=False)


def skinny_launch(rt, ctx, s, inp, epi=SKINNY_EPILOGUES[0]):
    M, K, N = s["M"], s["K"], s["N"]
    btd = ctx.to_device(inp["bt"])
    b = btd.view((K, N), (1, K))  # K-major B, as a prepacked weight is
    if epi == "alpha + bias":
        return rt.FusedMatMul(0.5).run(ctx, ctx.to_device(inp["a"]), b, ctx.to_device(inp["bias"])).numpy()
    if epi == "Gemm beta * C":
        beta = -0.5 if inp["ints"] else 0.5
        return rt.Gemm(2.0, beta, False, True).run(ctx, ctx.to_device(inp["a"]), btd, ctx.to_device(inp["c"])).numpy()
    if epi == "bias + residual + activation":
        act = rt.ACT_GELU if inp["ints"] else rt.ACT_RELU
        return rt.FusedMatMul(None, activation=act).run(ctx, ctx.to_device(inp["a"]), b, ctx.to_device(inp["bias"]),
                                                        residual=ctx.to_device(inp["res"])).numpy()
    abuf = ctx.to_device(np.concatenate([inp["a"], np.full((M, 4), np.nan, F32)], axis=1))
    obuf = ctx.to_device(np.full((M, N + 3), 7.0, F32))
    y = rt.FusedMatMul(None).run(ctx, abuf.view((M, K), (K + 4, 1)), b, out=obuf.view((M, N), (N + 3, 1)))
    full = obuf.numpy()
    assert (full[:, N:] == 7.0).all(), "writes outside the strided output view"
    assert y.shape == (M, N)
    return np.ascontiguousarray(full[:, :N])


def skinny_want64(inp, epi):
    """the exact result in float64 (before the activation), and whether the activation is Gelu"""
    p = inp["a"].astype(np.float64) @ inp["bt"].astype(np.float64).T
    if epi == "alpha + bias":
        return 0.5 * p + inp["bias"]
    if epi == "Gemm beta * C":
        return 2.0 * p + (-0.5 if inp["ints"] else 0.5) * inp["c"].astype(np.float64)
    if epi == "bias + residual + activation":
        return p + inp["res"] + inp["bias"]
    return p


# ---- fused quantized linear -------------------------------------------------------------------------------------------
def qlinear_specs(sms):
    # (K, N, layer norm) pairs per instance group; the first of each pair takes the smaller M of the MT, the second the
    # larger; N % (8 CPW) != 0 in at least one of each pair.  The second width of each double-buffered pair has more
    # than 4 x SMs tiles, so that CTAs walk three tiles: t0, then t1 (loaded while t0 is multiplied), then t0 again.
    db = wide_n(sms, 32, 8192, 4)
    pairs = [((768, 777, True), (256, 64, False)),  # CPW 1, KI 2, FLN 6
             ((768, 2304, False), (512, 3075, True)),  # CPW 2
             ((768, 8197, False), (640, db, True)),  # CPW 4 (double-buffered)
             ((1040, 500, False), (3072, 1001, False)),  # KI 6
             ((896, 96, True), (1024, 1003, True)),  # FLN 8, CPW 1
             ((1024, 3000, True), (896, 2048, True)),  # FLN 8, CPW 2
             ((896, 8200, True), (1024, db, True))]  # FLN 8, CPW 4
    specs = []
    for ms in ((1, 8), (9, 16)):
        for signed in (True, False):
            for pair in pairs:
                for M, (K, N, ln) in zip(ms, pair):
                    specs.append(dict(kind="rand", M=M, K=K, N=N, ln=ln, signed=signed))
    specs += [dict(kind="rand", M=1, K=768, N=50257, ln=True, signed=True),  # a vocabulary-sized output
              dict(kind="ties", M=1, K=256, N=100, ln=False, signed=True), dict(kind="ties", M=9, K=512, N=2100, ln=False, signed=False),
              dict(kind="zeros", M=1, K=768, N=300, ln=False, signed=True), dict(kind="zeros", M=12, K=1024, N=2100, ln=False, signed=False),
              dict(kind="const", M=1, K=768, N=300, ln=False, signed=True), dict(kind="const", M=5, K=896, N=500, ln=True, signed=False),
              dict(kind="mixed", M=9, K=768, N=777, ln=False, signed=True),
              # just past the kernel's limits: the composed chain
              dict(kind="rand", M=4, K=3088, N=300, ln=False, signed=True), dict(kind="rand", M=17, K=768, N=300, ln=True, signed=True),
              dict(kind="rand", M=8, K=960, N=300, ln=True, signed=False)]
    for i, s in enumerate(specs):  # the epilogue operands rotate over the cases, on coprime periods
        s.update(wz=(None, "scalar", "vec")[i % 3], act=i % 4, res=i % 5 in (1, 3), bias=i % 7 < 4, scalar_scale=i % 11 == 0,
                 ln_beta=i % 13 < 8)
    return specs


def qlinear_expected(s, sms):
    return qlinear_rule(s["M"], s["K"], s["N"], s["ln"], s["signed"])


def qlinear_prepare(s):
    r = _rng("qlinear", sorted(s.items()))
    M, K, N = s["M"], s["K"], s["N"]
    k = s["kind"]
    if k == "ties":  # range [-100, 155]: scale 255 / 255 = 1, zero point 100, and x * (1 / scale) = j + 0.5 exactly
        x = (r.integers(-100, 155, (M, K)) + 0.5).astype(F32)
        x[0, :2] = (-100.0, 155.0)
    elif k == "zeros":
        x = np.zeros((M, K), F32)
    elif k == "const":
        x = np.full((M, K), 2.5 if s["ln"] is False else -1.5, F32)
    else:
        x = r.uniform(-2, 3, (M, K)).astype(F32)
        if k == "mixed":
            x[0] = 0.0
            x[3] = 0.625
    ln = None
    if s["ln"]:
        ln = (r.uniform(0.5, 1.5, K).astype(F32), r.uniform(-0.5, 0.5, K).astype(F32) if s["ln_beta"] else None)
    wq = r.integers(-128, 128, (K, N)).astype(np.int8) if s["signed"] else r.integers(0, 256, (K, N)).astype(np.uint8)
    wdt = wq.dtype
    ws = np.asarray(r.uniform(0.001, 0.05, () if s["scalar_scale"] else (N,)), F32)
    wz = {None: None, "scalar": np.array(r.integers(-20, 20) if s["signed"] else r.integers(100, 150), wdt),
          "vec": (r.integers(-20, 20, N) if s["signed"] else r.integers(100, 150, N)).astype(wdt)}[s["wz"]]
    bias = r.uniform(-1, 1, N).astype(F32) if s["bias"] else None
    res = r.uniform(-1, 1, (M, N)).astype(F32) if s["res"] else None
    return dict(x=x, ln=ln, wq=wq, ws=ws, wz=wz, bias=bias, res=res)


def qlinear_launch(rt, ctx, s, inp):
    dev = lambda a: None if a is None else ctx.to_device(a)
    dw = ctx.to_device(inp["wq"])
    pk = rt.MatMulInteger().prepack(ctx, 1, dw)
    ln = inp["ln"]
    return rt.QuantizedLinear(s["act"], 1e-5).run(
        ctx, dev(inp["x"]), dw, dev(inp["ws"]), packed_w=pk, w_zero_point=dev(inp["wz"]), bias=dev(inp["bias"]),
        residual=dev(inp["res"]), ln_scale=dev(ln[0]) if ln else None, ln_bias=dev(ln[1]) if ln else None).numpy()


def qlinear_want(oracle, s, inp):
    return gc._qlinear_oracle(oracle, inp["x"], inp["ln"], inp["wq"], inp["wz"], inp["ws"], inp["bias"], inp["res"], s["act"], 1e-5)


FAMILIES = {
    "softmax": (softmax_specs, softmax_expected, softmax_prepare, softmax_launch),
    "norm": (norm_specs, norm_expected, norm_prepare, norm_launch),
    "skinny": (skinny_specs, skinny_expected, skinny_prepare, skinny_launch),
    "qlinear": (qlinear_specs, qlinear_expected, qlinear_prepare, qlinear_launch),
}


def spec_id(fam, s):
    return fam + " " + " ".join(f"{k}={v}" for k, v in s.items())


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


# ---- kernel identity (CUPTI in a child process, so that no profiler state stays behind in the test session) ----------
def probe_runs(fam, s, sms):
    """(label, expected kernel, launch keywords, vector rows off) of every call the identity probe captures for a
    case: each skinny epilogue, and for the row kernels the rerun with RTEN_B200_NO_VEC_ROWS that the numbers tests
    compare against"""
    want = FAMILIES[fam][1](s, sms)
    if fam == "skinny":
        return [(f"epi={e}", want, dict(epi=e), False) for e in SKINNY_EPILOGUES]
    if fam in ("softmax", "norm"):
        return [("", want, {}, False), ("no vector rows", (FAMILY_KERNELS[fam][-1], ()), {}, True)]
    return [("", want, {}, False)]


def coverage_gaps(sms):
    """What the case lists fail to reach on a device with `sms` SMs: instances selected by fewer than two cases,
    skinny instances never looping over a second tile, double-buffered instances never reaching a third tile"""
    picked, loops = {}, {}
    for fam, (specs, expected, _, _) in FAMILIES.items():
        for s in specs(sms):
            want = expected(s, sms)
            if want is None or want[0] in GENERIC:
                continue
            assert want[1] in VARIANTS[want[0]], f"{spec_id(fam, s)}: the rule names {want}, which the table lacks"
            picked[want] = picked.get(want, 0) + 1
            loops[want] = max(loops.get(want, 0), tiles_per_cta(fam, s, sms))
    gaps = [("selected fewer than twice", (b, a)) for b, args in VARIANTS.items() for a in args if picked.get((b, a), 0) < 2]
    gaps += [("no case loops over a second tile", ("skinny_f32_kernel", a)) for a in VARIANTS["skinny_f32_kernel"]
             if loops.get(("skinny_f32_kernel", a), 0) < 2]
    gaps += [("no case reaches a third tile", ("qlinear_kernel", a)) for a in VARIANTS["qlinear_kernel"]
             if a[5] and loops.get(("qlinear_kernel", a), 0) < 3]
    return gaps


def _capture(fn):
    """Names of the kernels `fn` launches, under CUPTI (torch.profiler).  Kineto keeps only the activity records
    whose timestamps, converted from the GPU clock, fall inside the capture window (libkineto's
    CuptiActivityProfiler::outOfRange); the kernels of a short call end microseconds before the window would close,
    so the window is held open a few milliseconds on both sides of the call."""
    import time
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        time.sleep(0.005)
        fn()
        torch.cuda.synchronize()
        time.sleep(0.005)
    return {e.name for e in prof.events()}


def _kernel_probe():
    import torch
    import gpu_checks as g
    import rten_b200 as rt
    n_sms = torch.cuda.get_device_properties(0).multi_processor_count
    ctx = g.new_ctx(rt, tf32=True)
    res, retaken = {}, 0
    for fam, (specs, _, prepare, launch) in FAMILIES.items():
        for s in specs(n_sms):
            inp = prepare(s)
            for label, _, kw, no_vec in probe_runs(fam, s, n_sms):
                def call():
                    launch(rt, ctx, s, inp, **kw)
                    ctx.sync()
                with gc.switches(RTEN_B200_NO_VEC_ROWS=1 if no_vec else None):
                    names, again = capture_kernels(call)
                retaken += again
                res[spec_id(fam, s) + " " + label] = sorted(names)
    print(json.dumps({"sms": n_sms, "names": res, "retaken": retaken}))


def capture_kernels(call):
    """(names of the kernels `call` launches, captures taken again).  Every call launches kernels.  A capture with no
    kernel record at all (seen, rarely, before the window was widened in _capture) is taken again, at most twice."""
    for attempt in range(3):
        names = _capture(call)
        if any("_kernel" in n for n in names):
            break
    return names, attempt


def probe_in_child(module):
    """`module._kernel_probe()` in a child process, so that no profiler state stays behind in the test session: the JSON
    line it prints last"""
    code = (f"import sys; sys.path[:0] = [{os.path.dirname(HERE)!r}, {HERE!r}]; "
            f"import {module} as t; t._kernel_probe()")
    res = subprocess.run([sys.executable, "-s", "-c", code], capture_output=True, text=True, timeout=1200)
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-4000:]
    return json.loads(res.stdout.strip().splitlines()[-1])


def test_kernel_identity():
    out = probe_in_child("test_gpu_row_kernels")
    n_sms, names = out["sms"], out["names"]
    seen, wrong = set(), []
    for fam, (specs, _, _, _) in FAMILIES.items():
        for s in specs(n_sms):
            for label, want, _, _ in probe_runs(fam, s, n_sms):
                sid = spec_id(fam, s) + " " + label
                ran = {kernel_key(n) for n in names[sid]} - {None}
                ran = {k for k in ran if k[0] in FAMILY_KERNELS[fam]}
                if ran != ({want} if want is not None else set()):
                    wrong.append((sid, want, sorted(ran), [n for n in names[sid] if "kernel" in n]))
                if fam == "skinny" and any("umma_" in n for n in names[sid]):
                    wrong.append((sid, "no wgmma GEMM", [n for n in names[sid] if "umma_" in n]))
                seen |= ran
    assert not wrong, f"{len(wrong)} calls ran another kernel than the rule names: {wrong[:10]}"
    missing = [(base, a) for base, args in VARIANTS.items() for a in args if (base, a) not in seen]
    assert not missing, f"instances that no case ran: {missing}"
    gaps = coverage_gaps(n_sms)
    assert not gaps, f"on {n_sms} SMs: {gaps}"
    total = sum(len(v) for v in VARIANTS.values())
    print(f"{total} of {total} instances ran ({', '.join(f'{b}: {len(v)}' for b, v in VARIANTS.items())}) on {n_sms} SMs; "
          f"{len(names)} captures, {out['retaken']} taken again")


# ---- numbers ----------------------------------------------------------------------------------------------------------
def test_softmax_bit_exact(rt, oracle, sms):
    ctx = rt.Context(0)
    for s in softmax_specs(sms):
        inp = softmax_prepare(s)
        sid = spec_id("softmax", s)
        for flush in (False, True):
            want = softmax_want(oracle, s, inp, flush)
            got = softmax_launch(rt, ctx, s, inp, flush)
            _bits(got, want, f"{sid} flush={flush}")
            with gc.switches(RTEN_B200_NO_VEC_ROWS=1):
                _bits(softmax_launch(rt, ctx, s, inp, flush), got, f"{sid} flush={flush}: generic kernel")
        softmax_f64_check(s, inp, got, f"{sid}: float64")


def test_layer_norm_bit_exact(rt, oracle, sms):
    ctx = rt.Context(0)
    for s in norm_specs(sms):
        if s["op"] != "LayerNormalization":
            continue
        inp = norm_prepare(s)
        sid = spec_id("norm", s)
        for arm in LN_ARMS:
            got = norm_launch(rt, ctx, s, inp, arm)
            _bits(got, norm_want(oracle, s, inp, arm), f"{sid} {arm}")
            with gc.switches(RTEN_B200_NO_VEC_ROWS=1):
                _bits(norm_launch(rt, ctx, s, inp, arm), got, f"{sid} {arm}: generic kernel")
            if arm == "scale + bias" and inp["first"] < s["rows"]:
                x = inp["x"][inp["first"]:].astype(np.float64)
                d = x - x.mean(1, keepdims=True)
                ref = d / np.sqrt((d * d).mean(1, keepdims=True) + 1e-5) * inp["g"] + inp["b"]
                err = float(np.abs(got[inp["first"]:] - ref).max())
                assert err <= 1e-5 * float(np.abs(ref).max()), f"{sid}: float64 error {err:.3e}"
        if s["kind"] == "rows" and inp["first"] > 0:
            # a constant row: (x - mean) = 0 exactly, so the output row is the bias; with eps = 0 it is NaN (0 * inf)
            y = norm_launch(rt, ctx, s, inp, "scale + bias")
            _bits(y[0], inp["b"], f"{sid}: constant row")
            assert np.isnan(norm_launch(rt, ctx, s, inp, "scale + bias, eps 0")[0]).all(), f"{sid}: constant row, eps 0"


def test_rms_and_skip_norms_bit_exact(rt, oracle, sms):
    """RMSNormalization and the eight forms of the skip layer norms (output, and the sum output where one is asked
    for): bit-exact against oracle/norms.py, and the same bits again from the generic kernel"""
    ctx = rt.Context(0)
    for s in norm_specs(sms):
        if s["op"] == "LayerNormalization":
            continue
        inp = norm_prepare(s)
        sid = spec_id("norm", s)
        got = norm_launch(rt, ctx, s, inp)
        _bits(got, norm_want(oracle, s, inp), sid)
        with gc.switches(RTEN_B200_NO_VEC_ROWS=1):
            _bits(norm_launch(rt, ctx, s, inp), got, f"{sid}: generic kernel")


@pytest.mark.parametrize("tf32", [False, True], ids=["3xTF32", "TF32"])
def test_skinny_gemm(rt, oracle, sms, tf32):
    """The skinny kernel computes in exact f32 FMAs whatever the mode."""
    ctx = gc.new_ctx(rt, tf32=tf32)
    for s in skinny_specs(sms):
        sid = spec_id("skinny", s)
        for ints in (True, False):
            inp = skinny_prepare(s, ints)
            for epi in SKINNY_EPILOGUES:
                got = skinny_launch(rt, ctx, s, inp, epi)
                want = skinny_want64(inp, epi)
                what = f"{sid} {epi} {'small integers' if ints else 'U[0, 1)'}"
                if ints:
                    w32 = want.astype(F32)
                    assert np.array_equal(w32.astype(np.float64), want), f"{what}: the integer reference is not exact in f32"
                    _bits(got, oracle.gelu(w32) if epi == "bias + residual + activation" else w32, what)
                else:
                    gc.assert_reference_rule(got, want, what)


def test_quantized_linear_bit_exact(rt, oracle, sms):
    ctx = rt.Context(0)
    for s in qlinear_specs(sms):
        inp = qlinear_prepare(s)
        _bits(qlinear_launch(rt, ctx, s, inp), qlinear_want(oracle, s, inp), spec_id("qlinear", s))


# ---- DynamicQuantizeLinear --------------------------------------------------------------------------------------------
def _dql_bits(got, want, what):
    y, sc, zp = got
    ey, es, ez = want
    _bits(sc.numpy(), np.float32(es), what + " scale")
    _bits(zp.numpy(), np.uint8(ez), what + " zero point")
    _bits(y.numpy(), ey, what + " y")


def test_dynamic_quantize_linear_degenerate_ranges(rt, oracle):
    """(<= 16384 elements: one kernel; more: range, then quantisation)"""
    ctx = rt.Context(0)
    for n in (1000, 16384, 16385, 40000):
        for name, v in (("zeros", 0.0), ("constant positive", 3.25), ("constant negative", -2.0), ("-0.0 only", -0.0)):
            x = np.full(n, v, F32)
            _dql_bits(rt.DynamicQuantizeLinear().run(ctx, ctx.to_device(x)), oracle.dynamic_quantize_linear(x), f"DQL {name} n={n}")


def test_dynamic_quantize_linear_producer_range(rt, oracle):
    """DynamicQuantizeLinear(value_range=...) over a range a MatMulIntegerToFloat epilogue accumulated: the bits of the
    plain operator on the same output; re-armed and refilled by a second product with a smaller output, the stale
    extremes of the first must be gone."""
    ctx = rt.Context(0)
    r = _rng("dql range")
    a8 = ctx.to_device(r.integers(0, 256, (64, 256)).astype(np.uint8))
    b8 = ctx.to_device(r.integers(-128, 128, (256, 384)).astype(np.int8))
    scale = r.uniform(0.001, 0.01, 384).astype(F32)
    rng = ctx.to_device(np.zeros(2, np.int32))
    for rep, sc in enumerate((scale, (scale * 0.25).astype(F32))):
        rt.DynamicQuantizeLinear.reset_ranges(ctx, rng)
        y = rt.MatMulIntegerToFloat().run(ctx, a8, b8, np.uint8(3), None, ctx.to_device(sc), out_range=rng)
        plain = rt.DynamicQuantizeLinear().run(ctx, y)
        ranged = rt.DynamicQuantizeLinear().run(ctx, y, value_range=rng)
        yh = y.numpy()
        _dql_bits(ranged, oracle.dynamic_quantize_linear(yh), f"ranged DQL, product {rep}")
        for got, want, what in zip(ranged, plain, ("y", "scale", "zero point")):
            _bits(got.numpy(), want.numpy(), f"ranged vs plain DQL {what}, product {rep}")
