"""`pytest -m gpu`: the kernels of rowops.cu that stage the operands and epilogue vectors of the tensor-core GEMM --
DynamicQuantizeLinear, the integer zero points, explicit and small-channel convolution staging, the strided copy, the
3xTF32 operand split -- and the executor glue around them (Cast int32 -> float, Clip, the ConvTranspose weight pack and
empty-phase fill), each selected by name and checked bit for bit.

The launchers pick a kernel at run time from shapes, strides, pointer alignment and the f32 mode.  The rules are
restated below (`*_rule`); `VARIANTS` lists every instance they pick from (tests/test_staging_kernel_table_cpu.py keeps it
equal to the built library's symbols; tests/test_kernel_names_cpu.py checks that every kernel of the library is in this
table or another by-name table).  `MODES` lists the runtime branches a name does not show.  The case lists reach every (kernel, mode) at least
twice, once with a partial last unit (a block with idle threads, a warp-per-row block with idle rows or lanes, a scalar
tail after the vector blocks).

A case launches several staging kernels (DynamicQuantizeLinear's range, then its quantisation; a convolution's weight
sums, zero points and im2col).  Each rule names the kernels of its family a case must run, and the identity test
requires exactly those of the family, no more and no fewer.

  * kernel identity: every case runs once under CUPTI in a child process; every entry of `VARIANTS` must have run;
  * strided copy: `DeviceTensor.assign` and `.numpy()` on views whose shapes, strides and offsets make
    launch_nd_copy's widening land on 1, 2, 4, 8 and 16 bytes, compared as bit patterns (NaN payloads, -0.0,
    subnormals), with the bytes around an assigned view untouched;
  * DynamicQuantizeLinear: bit-exact against oracle.dynamic_quantize_linear on the one-CTA kernel, the three-kernel
    path on aligned and misaligned inputs, rows written into a pre-padded buffer (128-bit and scalar groups), and the
    ranged form with a producer-accumulated range; NaN, +-inf, subnormal-only, -0.0-only inputs and exact .5 ties;
  * zero points, im2col<u8> and the 8-bit small-channel path: MatMulInteger / ConvInteger against the oracle's exact
    integer arithmetic, with scalar, vector, strided and 0-d zero points, and pads, groups and dilations;
  * f32 staging and the 3xTF32 split: MatMul, Conv and ConvTranspose on integer-valued operands whose products sum
    exactly in f32 in any order (checked on the inputs: sum_k |a_k| |b_k| < 2^24), so every plan and both f32 modes must
    give the exact product.  In 3xTF32 mode one operand carries up to 16 significant bits (a nonzero low part) and the
    other at most 11, so the dropped lo * lo term is zero; in TF32 mode both carry at most 11;
  * Cast int32 -> float through the executor and Clip on f32 / i32, against numpy."""
import json

import numpy as np
import pytest

import gpu_checks as gc
import test_gpu_row_kernels as rk

pytestmark = pytest.mark.gpu

F32, I32, U8, I8, U32 = np.float32, np.int32, np.uint8, np.int8, np.uint32
BLOCK = 256  # threads per block of the grid-stride launches (ew_grid)

# ---- the kernels, and the launchers' selection rules ------------------------------------------------------------------
VARIANTS = {
    "dql_small_kernel": [()], "minmax_init_kernel": [()], "minmax_kernel": [()], "dql_quantize_kernel": [()],
    "dql_quantize_rows_kernel": [()], "range_reset_kernel": [()],
    "rowsum8_kernel": [()], "zp_to_i32_kernel": [()], "fill8_kernel": [()],
    "im2col_kernel": [("float",), ("unsigned char",)], "smallc_pad_kernel": [()], "smallc_pack_w_kernel": [()],
    "smallc8_pad_kernel": [()], "smallc8_pack_w_kernel": [()],
    "nd_copy_kernel": [("unsigned char",), ("unsigned short",), ("unsigned int",), ("uint2",), ("uint4",)],
    "tf32x3_split_kernel": [()], "tf32x3_split_vec_kernel": [()], "tf32x3_lo_flat_kernel": [()],
    "cast_scale_kernel": [()], "clip_kernel": [("float",), ("int",)],
    "conv_transpose_pack_kernel": [()], "conv_transpose_fill_kernel": [()],
}
COPY_TYPES = {1: ("unsigned char",), 2: ("unsigned short",), 4: ("unsigned int",), 8: ("uint2",), 16: ("uint4",)}
# The runtime branches a name does not show: each (kernel, mode) is a unit of coverage.  A key is a kernel, or a
# (kernel, template arguments) pair where the instances differ.  The scalar split kernel takes role 2 (low parts only)
# nowhere: every role-2 split has a 16-byte aligned, TMA-addressable source whose K is a multiple of 32, which the vector
# or the flat kernel takes.
MODES = {
    "minmax_kernel": ("float4 body", "scalar only"),
    "dql_quantize_kernel": ("512-element warp blocks", "scalar only"),
    "dql_quantize_rows_kernel": ("128-bit groups", "scalar groups"),
    "rowsum8_kernel": ("signed", "unsigned"),
    "zp_to_i32_kernel": ("i8 scalar", "i8 vector", "u8 scalar", "u8 vector"),
    ("im2col_kernel", ("unsigned char",)): ("pad 128 (u8 image)", "pad 0 (i8 image)"),
    "tf32x3_split_kernel": ("role 0", "role 1"),
    "tf32x3_split_vec_kernel": ("role 0", "role 1", "role 2"),
    "conv_transpose_fill_kernel": ("channels-last, bias", "channels-last, no bias", "NCHW, bias", "NCHW, no bias"),
    "clip_kernel": ("given bounds", "default bounds"),
}
FAMILY_KERNELS = {
    "copy": ("nd_copy_kernel",),
    "dql": ("dql_small_kernel", "minmax_init_kernel", "minmax_kernel", "dql_quantize_kernel", "dql_quantize_rows_kernel",
            "range_reset_kernel"),
    "int8": ("rowsum8_kernel", "zp_to_i32_kernel", "fill8_kernel", "im2col_kernel", "smallc8_pad_kernel",
             "smallc8_pack_w_kernel"),
    "f32": ("tf32x3_split_kernel", "tf32x3_split_vec_kernel", "tf32x3_lo_flat_kernel", "im2col_kernel", "smallc_pad_kernel",
            "smallc_pack_w_kernel", "conv_transpose_pack_kernel", "conv_transpose_fill_kernel"),
    "cast": ("cast_scale_kernel",),
    "clip": ("clip_kernel",),
}
KERNELS = set(VARIANTS)


def _modes(k, a):
    return MODES.get((k, a), MODES.get(k, (None,)))


def units():
    return [(k, a, m) for k, args in VARIANTS.items() for a in args for m in _modes(k, a)]


def _contig(shape):
    st, s = [], 1
    for d in reversed(shape):
        st.append(s)
        s *= d
    return tuple(reversed(st))


def _span(shape, strides):
    return 1 + sum((d - 1) * s for d, s in zip(shape, strides)) if int(np.prod(shape)) else 0


def _r4(n):
    return (n + 3) // 4 * 4


def _part(n, unit=BLOCK):
    return n % unit != 0


# A unit a rule names: (kernel, template arguments, mode, partial last unit)
def U(k, a=(), mode=None, partial=False):
    return (k, a, mode, bool(partial))


# ---- strided copy -----------------------------------------------------------------------------------------------------
def copy_layouts(s):
    """(shape, source strides, source offset, destination strides, destination offset) in elements, as launch_nd_copy
    sees them: `.numpy()` copies the view into a fresh contiguous buffer, `assign` copies a contiguous tensor (or a view)
    into the view.  Every buffer starts 16-byte aligned (the memory pool hands out 256-byte aligned blocks)."""
    shape = s["shape"]
    v = (s["view"], s["off"])
    c = (_contig(shape), 0)
    src, dst = (v, c) if s["op"] == "numpy" else (s.get("src", c), v)
    return shape, src[0], src[1], dst[0], dst[1]


def copy_rule(s):
    """launch_nd_copy's widening loop: while both sides are unit-stride along the last dim, the last dim's bytes, both
    base addresses and every other stride of both sides (size-1 dims included) are multiples of twice the element
    size, the element doubles, up to 16 bytes; then nd_copy_kernel of that width, one element per thread."""
    shape, ss, so, ds, do = copy_layouts(s)
    es = 4 if s["dtype"] == "f32" else 1
    shape, ss, ds = list(shape), list(ss), list(ds)
    n = int(np.prod(shape))
    sa, da = so * es, do * es  # byte offsets from 16-byte aligned bases
    if ss[-1] == 1 and ds[-1] == 1:
        while es < 16:
            ok = (shape[-1] * es) % (2 * es) == 0 and (sa | da) % (2 * es) == 0
            ok = ok and all((ss[i] * es) % (2 * es) == 0 and (ds[i] * es) % (2 * es) == 0 for i in range(len(shape) - 1))
            if not ok:
                break
            shape[-1] //= 2
            for i in range(len(shape) - 1):
                ss[i] //= 2
                ds[i] //= 2
            n //= 2
            es *= 2
    return [U("nd_copy_kernel", COPY_TYPES[es], None, _part(n))]


def copy_specs(sms):
    u8, f = dict(dtype="u8"), dict(dtype="f32")
    return [
        # 1 byte: u8 with an odd inner extent
        dict(u8, op="numpy", shape=(5, 7), view=(9, 1), off=0), dict(u8, op="assign", shape=(3, 4, 13), view=(64, 16, 1), off=3),
        dict(u8, op="numpy", shape=(1, 5, 16), view=(3, 20, 1), off=0),  # a size-1 dim with an odd stride: no widening
        # 2 bytes: u8 with an inner extent = 2 mod 4
        dict(u8, op="numpy", shape=(6, 10), view=(12, 1), off=0), dict(u8, op="assign", shape=(7, 30), view=(34, 1), off=2),
        # 4 bytes: f32 with an odd inner extent; a size-1 dim with an odd stride; a million elements
        dict(f, op="numpy", shape=(9, 7), view=(8, 1), off=0), dict(f, op="assign", shape=(5, 3, 7), view=(32, 8, 1), off=1),
        dict(f, op="numpy", shape=(4, 1, 12), view=(16, 7, 1), off=0),
        dict(f, op="numpy", shape=(1000, 1001), view=(1003, 1), off=0),
        # 8 bytes: f32 with an inner extent = 2 mod 4, or 4-byte-aligned bases
        dict(f, op="numpy", shape=(6, 10), view=(12, 1), off=0), dict(f, op="assign", shape=(4, 3, 6), view=(40, 12, 1), off=2),
        dict(f, op="assign", shape=(5, 12), view=(14, 1), off=2),
        # 16 bytes: f32 with inner % 4 == 0 on 16-byte aligned bases; u8 with inner % 16 == 0
        dict(f, op="numpy", shape=(8, 12), view=(16, 1), off=0), dict(f, op="assign", shape=(3, 5, 16), view=(100, 20, 1), off=4),
        dict(u8, op="numpy", shape=(9, 32), view=(48, 1), off=0), dict(u8, op="assign", shape=(4, 5, 64), view=(400, 80, 1), off=16),
        # an outer stride of 0: one source row broadcast into every destination row
        dict(f, op="assign", shape=(6, 12), view=(16, 1), off=0, src=((0, 1), 0)),
        dict(u8, op="assign", shape=(5, 24), view=(32, 1), off=8, src=((0, 1), 0)),
    ]


def _bits_of(s, shape, r):
    """random bit patterns of the case's type: f32 patterns include NaN payloads, -0.0 and subnormals"""
    if s["dtype"] == "u8":
        return r.integers(0, 256, shape, dtype=np.int64).astype(U8)
    x = r.integers(0, 2 ** 32, shape, dtype=np.uint64).astype(U32)
    flat = x.reshape(-1)
    special = np.array([0x7fc00001, 0xffa00002, 0x7f800001, 0x80000000, 0x00000001, 0x807fffff, 0x7f800000, 0xff800000], U32)
    flat[:: max(1, flat.size // 16)][:special.size] = special[:flat[:: max(1, flat.size // 16)].size]
    return x


def _as_dev(a):
    return a.view(F32) if a.dtype == U32 else a


def _placed_bits(ctx, arr, strides, off, fill, guard=3):
    """`arr` (u8 or u32 bit patterns) on the device as the view (strides, off) of a buffer filled with `fill`"""
    host = np.full(off + max(_span(arr.shape, strides), 1) + guard, fill, arr.dtype)
    np.lib.stride_tricks.as_strided(host[off:], arr.shape, [st * arr.itemsize for st in strides])[...] = arr
    return ctx.to_device(_as_dev(host)).view(arr.shape, strides, off), host


def copy_prepare(s):
    r = _rng(sorted((k, str(v)) for k, v in s.items()))
    shape = s["shape"]
    src_strides = s.get("src", (None,))[0]
    if src_strides is not None:  # a broadcast source: its own (smaller) extent
        return dict(x=_bits_of(s, tuple(1 if st == 0 else d for d, st in zip(shape, src_strides)), r))
    return dict(x=_bits_of(s, shape, r))


def copy_launch(rt, ctx, s, inp):
    """(the destination's bits, the expected bits)"""
    x = inp["x"]
    fill = U8(0xA5) if s["dtype"] == "u8" else U32(0x7fbadbad)
    if s["op"] == "numpy":
        v, _ = _placed_bits(ctx, x, s["view"], s["off"], fill)
        got = v.numpy()
        return got.view(U32) if s["dtype"] == "f32" else got, x
    if "src" in s:
        st, off = s["src"]
        src, _ = _placed_bits(ctx, x, st, off, fill)
        src = src.view(s["shape"], st, off)
        full = np.broadcast_to(x, s["shape"])
    else:
        src, full = ctx.to_device(_as_dev(x)), x
    dst, host = _placed_bits(ctx, np.zeros(s["shape"], x.dtype), s["view"], s["off"], fill)
    dst.assign(src)
    want = host.copy()
    np.lib.stride_tricks.as_strided(want[s["off"]:], s["shape"], [st * want.itemsize for st in s["view"]])[...] = full
    got = dst.base.numpy()
    return got.view(U32) if s["dtype"] == "f32" else got, want


# ---- DynamicQuantizeLinear --------------------------------------------------------------------------------------------
def _ordered(v):
    """float_to_ordered (rowops.cu) of an f32: the i32 whose order is the float's"""
    b = np.array([v], F32).view(I32)[0]
    return int(b) if b >= 0 else int(b ^ 0x7fffffff)


def dql_layout(s):
    """(x shape, x strides, x offset in floats; for row output: the padded buffer's shape and the interior's offset)"""
    if s["kind"] == "flat":
        return (s["n"],), (1,), s.get("off", 0), None
    B, C, H, W = s["shape"]
    t, l, b, r = s["pad"]
    Hp, Wp = H + t + b, W + l + r + s.get("wextra", 0)
    return (B, C, H, W), (H * W * C, 1, W * C, C), 0, dict(shape=(B, C, Hp, Wp), strides=(Hp * Wp * C, 1, Wp * C, C),
                                                           off=(t * Wp + l) * C + s.get("yoff", 0))


def dql_rule(s):
    """rten_b200_dynamic_quantize_linear_ranged: without a producer range or a row output, n <= 16384 runs the one-CTA
    kernel; otherwise minmax_init + minmax (no pass at all with `value_range`), then the quantisation: row by row into
    the given pre-padded channels-last output (`out=`), else flat.  minmax reads float4s when x is 16-byte aligned; the
    flat quantisation takes 512-element warp blocks when x is 16-byte and y 4-byte aligned; the row quantisation takes a
    16-element group as one 128-bit load and store when the group is whole and both its addresses are 16-byte
    aligned."""
    shape, _, xoff, y = dql_layout(s)
    n = int(np.prod(shape))
    ranged = s.get("ranged", False)
    if not ranged and y is None and n <= 16384:
        return [U("dql_small_kernel", partial=_part(n, 1024))]
    out = []
    if ranged:
        out.append(U("range_reset_kernel", partial=True))  # (one pair: 127 idle threads)
    else:
        x_al = xoff % 4 == 0
        out += [U("minmax_init_kernel", partial=True),
                U("minmax_kernel", mode="float4 body" if x_al else "scalar only",
                  partial=(n % 4 != 0 or _part(n // 4)) if x_al else _part(n))]
    if y is None:
        al = xoff % 4 == 0
        out.append(U("dql_quantize_kernel", mode="512-element warp blocks" if al else "scalar only",
                     partial=n % 512 != 0 if al else _part(n)))
        return out
    B, C, H, W = shape
    row_len, rows = W * C, B * H
    groups = (row_len + 15) // 16
    r = np.arange(rows)[:, None]
    g = np.arange(groups)[None, :]
    xa = (r * row_len + g * 16) * 4
    ya = y["off"] + (r // H) * y["strides"][0] + (r % H) * y["strides"][2] + g * 16
    vec = (row_len - g * 16 >= 16) & (xa % 16 == 0) & (ya % 16 == 0)
    part = _part(rows * groups)
    if vec.any():
        out.append(U("dql_quantize_rows_kernel", mode="128-bit groups", partial=part))
    if not vec.all():
        out.append(U("dql_quantize_rows_kernel", mode="scalar groups", partial=part))
    return out


def dql_specs(sms):
    specs = [dict(kind="flat", n=n, values="rand") for n in (1, 1000, 16384, 16385, 512 * 80, 512 * 81 + 1, 512 * 90 + 511)]
    specs += [dict(kind="flat", n=n, off=off, values="rand") for n, off in ((20000, 1), (40001, 2), (16387, 3))]
    specs += [dict(kind="flat", n=n, values=v) for n in (777, 30001)
              for v in ("nan", "inf", "-inf", "subnormal", "-0.0", "ties")]
    # channels-last x into the interior of a pre-padded buffer: row_len = W C
    specs += [dict(kind="rows", shape=(2, 32, 6, 5), pad=(1, 1, 1, 1), values="rand"),     # 160: 128-bit groups
              dict(kind="rows", shape=(2, 64, 14, 14), pad=(1, 1, 1, 1), values="rand"),   # 896
              dict(kind="rows", shape=(2, 3, 50, 50), pad=(3, 3, 3, 3), values="rand"),    # 150: a scalar last group
              dict(kind="rows", shape=(1, 12, 30, 11), pad=(1, 2, 1, 0), values="rand"),   # 132
              dict(kind="rows", shape=(2, 16, 20, 9), pad=(1, 1, 1, 1), yoff=4, values="rand"),  # pitch, offset 4-aligned
              dict(kind="rows", shape=(1, 20, 24, 22), pad=(0, 1, 0, 1), wextra=1, values="rand"),  # pitch 20 * 25
              dict(kind="rows", shape=(2, 5, 40, 41), pad=(2, 2, 2, 2), values="nan")]
    # ranged: value_range from a MatMulIntegerToFloat out_range, re-armed by reset_ranges
    specs += [dict(kind="flat", n=64 * 384, ranged=True, values="product"), dict(kind="flat", n=72 * 100, ranged=True, values="product"),
              dict(kind="rows", shape=(1, 384, 8, 8), pad=(1, 1, 1, 1), ranged=True, values="product"),
              dict(kind="rows", shape=(1, 102, 16, 4), pad=(1, 1, 1, 1), ranged=True, values="product")]
    return specs


def dql_prepare(s):
    r = _rng(sorted((k, str(v)) for k, v in s.items()))
    shape = dql_layout(s)[0]
    n = int(np.prod(shape))
    v = s["values"]
    if v == "product":  # the GEMM's operands: y = (a - 3) b * scale, [M, N]
        N = shape[1] if s["kind"] == "rows" else {64 * 384: 384, 72 * 100: 100}[n]
        M = n // N
        return dict(a=r.integers(0, 256, (M, 256)).astype(U8), b=r.integers(-128, 128, (256, N)).astype(I8),
                    scale=r.uniform(0.001, 0.01, N).astype(F32))
    x = r.uniform(-3, 5, n).astype(F32)
    if v == "nan":
        x[r.integers(0, n, max(1, n // 50))] = np.nan
    elif v == "inf":
        x[r.integers(0, n, 3)] = np.inf
    elif v == "-inf":
        x[r.integers(0, n, 3)] = -np.inf
    elif v == "subnormal":  # only subnormals: 1 / scale overflows to +inf
        x = (r.integers(1, 2 ** 23, n).astype(U32) | (r.integers(0, 2, n).astype(U32) << 31)).view(F32)
    elif v == "-0.0":
        x = np.full(n, -0.0, F32)
    elif v == "ties":  # range [0, 255]: scale 1, zero point 0, every k + 0.5 a tie
        x = (r.integers(0, 255, n) + np.where(r.random(n) < 0.5, 0.5, 0.0)).astype(F32)
        x[0], x[1] = 0.0, 255.0
    if s["kind"] == "flat":
        return dict(x=x)
    B, C, H, W = shape
    return dict(x=x.reshape(B, H, W, C).transpose(0, 3, 1, 2))  # NCHW values, channels-last in memory


def dql_launch(rt, ctx, s, inp):
    """((y, scale, zero point), the x the oracle quantises, the padded buffer outside the interior or None)"""
    shape, xs, xoff, y = dql_layout(s)
    op = rt.DynamicQuantizeLinear()
    rng = None
    if s.get("ranged"):
        rng = ctx.to_device(np.zeros(2, I32))
        rt.DynamicQuantizeLinear.reset_ranges(ctx, rng)
        prod = rt.MatMulIntegerToFloat().run(ctx, ctx.to_device(inp["a"]), ctx.to_device(inp["b"]), U8(3), None,
                                            ctx.to_device(inp["scale"]), out_range=rng)
        xd = prod.view(shape, xs)
        xh = xd.numpy()
    else:
        xh = inp["x"]
        if s["kind"] == "flat":
            host = np.full(xoff + xh.size + 1, 7.0, F32)
            host[xoff:xoff + xh.size] = xh
            xd = ctx.to_device(host).view(shape, xs, xoff)
        else:
            xd = ctx.to_device(np.ascontiguousarray(xh.transpose(0, 2, 3, 1))).view(shape, xs)
    if y is None:
        return op.run(ctx, xd, value_range=rng), xh, None
    full = ctx.to_device(np.full(int(np.prod(y["shape"])) + 16, 0xEE, U8))
    yv = full.view(shape, y["strides"], y["off"])
    res = op.run(ctx, xd, value_range=rng, out=yv)
    assert res[0] is yv
    buf = full.numpy()
    mask = np.ones(buf.shape, bool)
    np.lib.stride_tricks.as_strided(mask[y["off"]:], shape, y["strides"])[...] = False
    return res, xh, buf[mask]


def dql_check(oracle, s, inp, got):
    (y, sc, zp), xh, outside = got
    ey, es, ez = oracle.dynamic_quantize_linear(np.ascontiguousarray(xh))
    what = spec_id("dql", s)
    gc.assert_bit_exact(sc.numpy(), np.float32(es), what + " scale")
    gc.assert_bit_exact(zp.numpy(), np.uint8(ez), what + " zero point")
    gc.assert_bit_exact(y.numpy(), ey, what + " y")
    if outside is not None:
        assert (outside == 0xEE).all(), f"{what}: writes outside the output's interior"
    if s["values"] == "subnormal":
        with np.errstate(over="ignore", divide="ignore"):
            assert np.isinf(np.float32(1) / np.float32(es)), f"{what}: the scale's reciprocal is finite"
    return ey


# ---- integer GEMM / convolution: zero points, im2col<u8>, the 8-bit small-channel path --------------------------------
def conv_geometry(s):
    B, C, H, W = s["x"]
    O, Cg, kh, kw = s["w"]
    t, l, b, r = s.get("pads", (0, 0, 0, 0))
    sy, sx = s.get("strides", (1, 1))
    dy, dx = s.get("dil", (1, 1))
    OH = (H + t + b - dy * (kh - 1) - 1) // sy + 1
    OW = (W + l + r - dx * (kw - 1) - 1) // sx + 1
    return B, C, H, W, O, Cg, kh, kw, t, l, b, r, sy, sx, dx, OH, OW


def conv_path(s, esize):
    """api_conv.cu's choice for a (non-depthwise) convolution: implicit GEMM when Cg esize % 16 == 0 and >= 32; the
    small-channel path when groups == 1, dilation_x == 1 and (f32) Cg <= 4, kw <= 8, or (8-bit) Cg <= 16, kw <= 8 with
    no weight zero point; else explicit im2col.  The cases keep to shapes launch_umma_gemm takes, so that neither of the
    first two falls through to the explicit path."""
    B, C, H, W, O, Cg, kh, kw, *_, dx, OH, OW = conv_geometry(s)
    groups = C // Cg
    if (Cg * esize) % 16 == 0 and Cg * esize >= 32:
        return "implicit"
    small = Cg <= 4 and kw * 4 <= 32 if esize == 4 else Cg <= 16 and kw <= 8 and s.get("wzp") is None
    if groups == 1 and dx == 1 and small:
        return "smallc"
    return "explicit"


def _zp_unit(signed, zp):
    scalar = zp in ("scalar", "0-d")
    n = 1 if scalar else zp[1]
    return U("zp_to_i32_kernel", mode=("i8 " if signed else "u8 ") + ("scalar" if scalar else "vector"), partial=_part(n, 128))


def _rowsum_unit(signed, rows, K):
    return U("rowsum8_kernel", mode="signed" if signed else "unsigned", partial=rows % 8 != 0 or K % 32 != 0)


def int8_rule(s):
    """MatMulInteger (api_ops.cu): an x zero point without prepacked weights sums B's columns (rowsum8 over the K-major
    copy, N rows); a weight zero point turns into i32 (zp_to_i32, every length) and sums A's rows (M rows).
    ConvInteger (api_conv.cu): an x zero point sums the packed weight's rows (O rows of kh kw Cg); a weight zero point
    turns into i32.  Implicit path: a u8 image with padding is copied into a buffer filled with 128 first (fill8), and a
    weight zero point adds the window-sum GEMM against a row of ones (fill8).  Small-channel path: smallc8_pad and
    smallc8_pack_w.  Explicit path: im2col<u8>, padding with 128 for u8 images and 0 for i8; a weight zero point sums
    the im2col rows (rowsum8 over B OH OW rows of kh kw Cg)."""
    xs, ws = s["xt"] == "i8", s["wt"] == "i8"
    out = []
    if s["op"] == "matmul":
        M, K, N = s["mkn"]
        if s.get("xzp"):
            out.append(_rowsum_unit(ws, N, K))
        if s.get("wzp"):
            out += [_zp_unit(ws, s["wzp"]), _rowsum_unit(xs, M, K)]
        return out
    B, C, H, W, O, Cg, kh, kw, t, l, b, r, sy, sx, dx, OH, OW = conv_geometry(s)
    Kd = kh * kw * Cg
    if s.get("xzp"):
        out.append(_rowsum_unit(ws, O, Kd))
    if s.get("wzp"):
        out.append(_zp_unit(ws, s["wzp"]))
    path = conv_path(s, 1)
    padded = (t | l | b | r) != 0
    if path == "implicit":
        if not xs and padded:
            out.append(U("fill8_kernel", partial=_part(B * (H + t + b) * (W + l + r) * C)))
        if s.get("wzp"):
            out.append(U("fill8_kernel", partial=_part(Kd)))
    elif path == "smallc":
        Hp, Wp = H + t + b, max(W + l + r, (OW - 1) * sx + 8)
        out += [U("smallc8_pad_kernel", partial=_part(B * Hp * Wp)), U("smallc8_pack_w_kernel", partial=_part(O * kh * 128))]
    else:
        kpad = (Kd + 15) // 16 * 16
        out.append(U("im2col_kernel", ("unsigned char",), "pad 0 (i8 image)" if xs else "pad 128 (u8 image)",
                     _part(B * OH * OW * kpad // 16) or kpad > Kd))
        if s.get("wzp"):
            out.append(_rowsum_unit(xs, B * OH * OW, Kd))
    return out


def int8_specs(sms):
    mm = lambda mkn, xt, wt, **kw: dict(op="matmul", mkn=mkn, xt=xt, wt=wt, **kw)  # noqa: E731
    cv = lambda x, w, xt="u8", wt="i8", **kw: dict(op="conv", x=x, w=w, xt=xt, wt=wt, **kw)  # noqa: E731
    return [
        # MatMulInteger: unprepacked weights with an x zero point (column sums); weight zero points of every form
        mm((64, 256, 384), "u8", "i8", xzp=True), mm((50, 70, 33), "u8", "u8", xzp=True),
        mm((37, 96, 72), "u8", "i8", xzp=True, wzp=("vec", 72)), mm((40, 20, 9), "i8", "u8", wzp=("strided", 9)),
        mm((33, 64, 16), "u8", "i8", wzp="0-d"), mm((64, 45, 130), "i8", "i8", xzp=True, wzp=("strided", 130)),
        mm((48, 17, 8), "u8", "u8", wzp="0-d"), mm((45, 33, 12), "u8", "u8", wzp="0-d"),
        mm((36, 40, 30), "i8", "u8", wzp=("vec", 30)),
        # ConvInteger, implicit path: a weight zero point (fill8 + the window-sum GEMM), u8 padding (fill8)
        cv((1, 32, 9, 9), (40, 32, 3, 3), pads=(1, 1, 1, 1), wzp=("vec", 40)),
        cv((2, 64, 7, 6), (24, 64, 1, 1), xt="i8", wzp="0-d"),
        cv((1, 48, 10, 11), (16, 48, 3, 3), pads=(1, 0, 1, 2), xzp=True),
        # explicit path: groups, dilation_x = 2, asymmetric pads; a weight zero point (rowsum8 over im2col rows, kpad > Kd)
        cv((1, 17, 12, 13), (20, 17, 3, 3), pads=(1, 1, 1, 1), xzp=True, wzp=("strided", 20)),
        cv((2, 12, 9, 10), (18, 6, 3, 3), pads=(0, 1, 2, 1), strides=(2, 1), xt="i8", wzp=("vec", 18)),
        cv((1, 3, 15, 16), (8, 3, 3, 3), pads=(2, 1, 0, 3), dil=(1, 2), xzp=True),
        cv((1, 6, 11, 11), (8, 3, 2, 2), xt="i8", wt="u8", xzp=True),
        # the 8-bit stem (small-channel path): C = 1, 3, 16; kw = 7 and 8; a non-contiguous OIHW weight view
        cv((2, 3, 30, 31), (16, 3, 7, 7), pads=(3, 3, 3, 3), strides=(2, 2), xzp=True, wview=True),
        cv((1, 1, 20, 21), (8, 1, 7, 8), pads=(3, 3, 4, 4), strides=(2, 2)),
        cv((1, 16, 18, 17), (12, 16, 3, 7), pads=(1, 3, 1, 3), xzp=True, wview=True),
        cv((1, 3, 14, 14), (9, 3, 5, 8), xt="i8", strides=(1, 2)),
        # the same stem with a weight zero point: im2col<u8>
        cv((2, 3, 30, 31), (16, 3, 7, 7), pads=(3, 3, 3, 3), strides=(2, 2), xzp=True, wzp="0-d", wview=True),
        cv((1, 16, 18, 17), (12, 16, 3, 7), pads=(1, 3, 1, 3), wzp=("vec", 12)),
    ]


def int8_prepare(s):
    r = _rng(sorted((k, str(v)) for k, v in s.items()))
    lo = lambda t: (-128, 128) if t == "i8" else (0, 256)  # noqa: E731
    dt = lambda t: I8 if t == "i8" else U8  # noqa: E731
    if s["op"] == "matmul":
        M, K, N = s["mkn"]
        xshape, wshape, nz = (M, K), (K, N), N
    else:
        xshape, wshape, nz = s["x"], s["w"], s["w"][0]
    x = r.integers(*lo(s["xt"]), xshape).astype(dt(s["xt"]))
    w = r.integers(*lo(s["wt"]), wshape).astype(dt(s["wt"]))
    xz = dt(s["xt"])(r.integers(*lo(s["xt"]))) if s.get("xzp") else None
    wz = None
    if s.get("wzp"):
        full = r.integers(*lo(s["wt"]), 2 * nz).astype(dt(s["wt"]))
        wz = {"scalar": full[:1], "0-d": np.array(full[0]), "vec": full[:nz]}.get(
            s["wzp"] if isinstance(s["wzp"], str) else s["wzp"][0], full[::2])  # "strided": a host view with stride 2
    return dict(x=x, w=w, xz=xz, wz=wz)


def int8_launch(rt, ctx, s, inp):
    if s["op"] == "matmul":
        return rt.MatMulInteger().run(ctx, ctx.to_device(inp["x"]), ctx.to_device(inp["w"]), inp["xz"], inp["wz"]).numpy()
    B, C, H, W, O, Cg, kh, kw, t, l, b, r, sy, sx, dx, OH, OW = conv_geometry(s)
    w = inp["w"]
    if s.get("wview"):  # OIHW strides of a (O, C + 1, kh, kw + 2) buffer
        host = np.zeros((O, Cg + 1, kh, kw + 2), w.dtype)
        host[:, :Cg, :, :kw] = w
        wd = ctx.to_device(host).view(w.shape, ((Cg + 1) * kh * (kw + 2), kh * (kw + 2), kw + 2, 1))
    else:
        wd = ctx.to_device(w)
    op = rt.ConvInteger(groups=C // Cg, dilations=s.get("dil", (1, 1)), padding=s.get("pads", (0, 0, 0, 0)),
                        strides=s.get("strides", (1, 1)))
    return op.run(ctx, ctx.to_device(inp["x"]), wd, inp["xz"], inp["wz"]).numpy()


def int8_want(oracle, s, inp):
    wz = None if inp["wz"] is None else np.ascontiguousarray(inp["wz"]).reshape(inp["wz"].shape)  # (keeps a 0-d one 0-d)
    if s["op"] == "matmul":
        return oracle.matmul_integer(inp["x"], inp["w"], inp["xz"], wz)
    B, C, H, W, O, Cg, *_ = conv_geometry(s)
    return oracle.conv_integer(inp["x"], inp["w"], inp["xz"], wz, padding=s.get("pads", (0, 0, 0, 0)), groups=C // Cg,
                               strides=s.get("strides", (1, 1)), dilations=s.get("dil", (1, 1)))


# ---- f32 staging and the 3xTF32 split ---------------------------------------------------------------------------------
def _split_unit(d0, rows, s1_ok, role):
    """launch_tf32x3_split over `rows` rows of d0 elements padded to d0p = d0 rounded up to 4, from a 16-byte aligned
    source whose row stride is a multiple of 4 (`s1_ok`: the role-2 source's rows are dense)"""
    d0p = _r4(d0)
    n = rows * d0p
    if role == 2 and d0 % 4 == 0 and s1_ok:
        return U("tf32x3_lo_flat_kernel", partial=(n // 4) % 128 != 0)
    if d0 % 4 == 0:
        return U("tf32x3_split_vec_kernel", mode=f"role {role}", partial=_part(n // 4))
    return U("tf32x3_split_kernel", mode=f"role {role}", partial=_part(n))


def _gemm_splits(K, M, N, a_dense):
    """launch_tf32x3 (umma_gemm.cu) after to_kmajor has made both operands TMA-addressable (16-byte aligned, row stride a
    multiple of 4; a copy with rows padded to K rounded up to 4 when they were not): B is split [hi | lo | hi] (role 1);
    A, when K % 32 == 0, keeps its hi parts in place and has only its low parts written (role 2: the flat kernel on
    dense rows, the vector kernel on padded ones), else is split [lo | hi | hi] (role 0)."""
    a = _split_unit(K, M, a_dense, 2 if K % 32 == 0 else 0)
    return [a, _split_unit(K, N, True, 1)]


def f32_rule(s):
    """MatMul (M > 32: no skinny kernel) and Conv in 3xTF32 mode run the splits of launch_tf32x3; in TF32 mode none.
    Conv (api_conv.cu conv_path): explicit path: im2col<float> into rows of kpad = Kd rounded up to 4, then A = the
    im2col rows (dense when kpad == Kd) and B = the packed weights of each group; small-channel path: smallc_pad and
    smallc_pack_w, and in 3xTF32 mode the low parts of the padded copy (the flat kernel) and B = the [O, kh, 32] packed
    weights (role 1, 32 wide).  ConvTranspose (api_conv.cu conv_transpose_core): without prepacked weights each phase's
    sub-kernel is packed (conv_transpose_pack); when a phase has no taps, one fill writes the bias (or 0) into every such
    phase, visiting channels fastest for a channels-last output; the phases' convolutions are not claimed here."""
    x3 = s["mode"] == "3xTF32"
    if s["op"] == "matmul":
        M, K, N = s["mkn"]
        a_dense = s["a"] != "sliced" or K % 4 != 0  # a sliced A keeps its padded rows; an unaddressable one is copied
        return _gemm_splits(K, M, N, a_dense) if x3 else []
    if s["op"] == "convt":
        B, C, H, W = s["x"]
        _, Og, kh, kw = s["w"]
        sy, sx = s["strides"]
        O, Cg = Og * s.get("groups", 1), C // s.get("groups", 1)
        OH, OW = (H - 1) * sy + kh, (W - 1) * sx + kw
        mode = ("channels-last" if s["cl"] else "NCHW") + (", bias" if s["bias"] else ", no bias")
        return [U("conv_transpose_pack_kernel", partial=_part(O * Cg)),
                U("conv_transpose_fill_kernel", mode=mode, partial=_part(B * O * OH * OW))]
    B, C, H, W, O, Cg, kh, kw, t, l, b, r, sy, sx, dx, OH, OW = conv_geometry(s)
    groups = C // Cg
    Kd = kh * kw * Cg
    path = conv_path(s, 4)
    if path == "smallc":
        Wp = (OW - 1) * sx + 8
        out = [U("smallc_pad_kernel", partial=_part(B * H * Wp)), U("smallc_pack_w_kernel", partial=_part(O * kh * 32))]
        if x3:
            out += [_split_unit(B * H * Wp * 4, 1, True, 2), _split_unit(32, O * kh, True, 1)]
        return out
    assert path == "explicit", s
    kpad = _r4(Kd)
    out = [U("im2col_kernel", ("float",), None, _part(B * OH * OW * kpad // 4) or kpad > Kd)]
    if x3:
        out += _gemm_splits(Kd, B * OH * OW, O // groups, True)
    return out


def f32_specs(sms):
    mm = lambda mkn, a, mode, wide, pre=False: dict(op="matmul", mkn=mkn, a=a, prepacked=pre, mode=mode, wide=wide)  # noqa: E731
    cv = lambda x, w, mode, wide, **kw: dict(op="conv", x=x, w=w, mode=mode, wide=wide, **kw)  # noqa: E731
    ct = lambda x, w, strides, cl, bias, mode, **kw: dict(op="convt", x=x, w=w, strides=strides, cl=cl, bias=bias, mode=mode,  # noqa: E731
                                                         wide="a" if mode == "3xTF32" else None, **kw)
    x3, t1 = "3xTF32", "TF32"
    return [
        # MatMul: K % 4 != 0, K % 32 != 0, K % 32 == 0 with dense / sliced / misaligned A, per-call and prepacked B
        mm((40, 37, 48), "dense", x3, "a"), mm((64, 37, 20), "dense", x3, "b", True), mm((33, 22, 36), "sliced", x3, "a"),
        mm((129, 100, 72), "dense", x3, "a"), mm((70, 100, 40), "sliced", x3, "b", True), mm((100, 52, 24), "misaligned", x3, "b"),
        mm((64, 64, 48), "dense", x3, "a"), mm((97, 64, 40), "sliced", x3, "a"), mm((200, 96, 24), "misaligned", x3, "a", True),
        mm((48, 128, 36), "sliced", x3, "b", True), mm((40, 32, 20), "dense", x3, "b"),
        mm((64, 37, 48), "dense", t1, None), mm((80, 64, 40), "sliced", t1, None, True),
        # Conv, explicit path: C = 17; Cg = 6 with groups; C = 3 with dilation_x = 2; C = 3 with a 9 x 9 kernel
        cv((1, 17, 10, 11), (12, 17, 3, 3), x3, "a", pads=(1, 1, 1, 1)),
        cv((2, 12, 9, 8), (10, 6, 3, 3), x3, "b", pads=(1, 0, 1, 2)),
        cv((1, 3, 16, 15), (8, 3, 3, 3), x3, "a", pads=(1, 2, 1, 2), dil=(1, 2)),
        cv((1, 3, 20, 21), (6, 3, 9, 9), x3, "b", pads=(4, 4, 4, 4), strides=(2, 2)),
        cv((1, 8, 9, 9), (16, 4, 2, 4), x3, "a"),  # Kd = 32: the flat low-part kernel on im2col rows
        cv((1, 17, 10, 11), (12, 17, 3, 3), t1, None, pads=(1, 1, 1, 1)),
        cv((1, 3, 16, 15), (8, 3, 3, 3), t1, None, dil=(1, 2)),
        # the f32 RGB stem (small-channel path): C = 1, 3, 4; 7 x 7 stride 2; a strided weight view
        cv((2, 3, 32, 30), (16, 3, 7, 7), x3, "a", pads=(3, 3, 3, 3), strides=(2, 2), wview=True),
        cv((1, 1, 29, 31), (8, 1, 7, 7), x3, "b", pads=(3, 3, 3, 3), strides=(2, 2)),
        cv((1, 4, 24, 25), (12, 4, 7, 7), x3, "a", pads=(3, 3, 3, 3), strides=(2, 2), wview=True),
        cv((1, 3, 32, 30), (16, 3, 7, 7), t1, None, pads=(3, 3, 3, 3), strides=(2, 2), wview=True),
        # ConvTranspose without prepacked weights, stride > kernel extent: phases with no taps
        ct((1, 4, 5, 6), (4, 3, 2, 2), (3, 3), False, True, x3), ct((2, 6, 4, 5), (6, 5, 2, 1), (3, 2), True, True, x3),
        ct((1, 5, 6, 5), (5, 4, 1, 2), (2, 3), False, False, t1), ct((1, 8, 5, 4), (8, 3, 2, 2), (4, 3), True, False, x3),
        ct((2, 3, 4, 4), (3, 7, 1, 1), (2, 2), True, True, t1), ct((1, 2, 7, 3), (2, 5, 2, 2), (3, 4), False, False, x3),
        ct((1, 3, 6, 6), (3, 9, 2, 2), (3, 3), True, False, t1), ct((1, 4, 4, 5), (4, 2, 1, 2), (2, 3), False, True, t1),
    ]


def _ints(r, shape, kind):
    """integer-valued f32: "wide" up to 16 significant bits (a nonzero low part in 3xTF32), "narrow" within 11 bits
    and small, "tf32" within 11 bits"""
    if kind == "wide":
        return r.integers(-(2 ** 16) + 1, 2 ** 16, shape).astype(F32)
    if kind == "narrow":
        return r.integers(-2, 3, shape).astype(F32)
    return r.integers(-1023, 1024, shape).astype(F32)


def f32_prepare(s):
    r = _rng(sorted((k, str(v)) for k, v in s.items()))
    ka = "wide" if s["wide"] == "a" else "narrow" if s["wide"] == "b" else "tf32"
    kb = "wide" if s["wide"] == "b" else "narrow" if s["wide"] == "a" else "narrow"
    if s["op"] == "matmul":
        M, K, N = s["mkn"]
        return dict(a=_ints(r, (M, K), ka), b=_ints(r, (K, N), kb))
    if s["op"] == "convt":
        O = s["w"][1] * s.get("groups", 1)
        return dict(x=_ints(r, s["x"], ka), w=_ints(r, s["w"], kb), bias=_ints(r, (O,), "tf32") if s["bias"] else None)
    return dict(x=_ints(r, s["x"], ka), w=_ints(r, s["w"], kb))


def _exact(s, inp):
    """the exact int64 result, and the largest sum_k |a_k| |b_k| of an output"""
    if s["op"] == "matmul":
        a, b = inp["a"].astype(np.int64), inp["b"].astype(np.int64)
        return a @ b, (np.abs(a) @ np.abs(b)).max()
    import torch
    x, w = torch.from_numpy(inp["x"].astype(np.float64)), torch.from_numpy(inp["w"].astype(np.float64))
    if s["op"] == "convt":
        f = lambda u, v: torch.nn.functional.conv_transpose2d(u, v, stride=s["strides"], groups=s.get("groups", 1))  # noqa: E731
    else:
        B, C, H, W, O, Cg, kh, kw, t, l, b, r, sy, sx, dx, OH, OW = conv_geometry(s)
        f = lambda u, v: torch.nn.functional.conv2d(torch.nn.functional.pad(u, (l, r, t, b)), v, stride=(sy, sx),  # noqa: E731
                                                    dilation=s.get("dil", (1, 1)), groups=C // Cg)
    y, bound = f(x, w).numpy(), f(x.abs(), w.abs()).numpy().max()
    if s["op"] == "convt" and inp["bias"] is not None:
        y = y + inp["bias"].astype(np.float64)[None, :, None, None]
        bound += np.abs(inp["bias"]).max()
    assert np.array_equal(y, np.round(y)), "float64 lost an integer"
    return y.astype(np.int64), bound


def f32_launch(rt, ctx, s, inp):
    ctx.set_f32_mode(s["mode"] == "3xTF32")
    try:
        if s["op"] == "matmul":
            M, K, N = s["mkn"]
            a = inp["a"]
            if s["a"] == "sliced":  # A[:, :K] of an [M, K + 4] buffer
                host = np.full((M, K + 4), np.nan, F32)
                host[:, :K] = a
                ad = ctx.to_device(host).view((M, K), (K + 4, 1))
            elif s["a"] == "misaligned":  # 4 bytes past a 16-byte boundary
                host = np.full(M * K + 1, np.nan, F32)
                host[1:] = a.reshape(-1)
                ad = ctx.to_device(host).view((M, K), (K, 1), 1)
            else:
                ad = ctx.to_device(a)
            op = rt.MatMul()
            bd = ctx.to_device(inp["b"])
            pb = op.prepack(ctx, 1, bd) if s["prepacked"] else None
            return op.run(ctx, ad, bd, packed_b=pb).numpy()
        xd = ctx.to_device(inp["x"], channels_last=s["op"] == "convt" and s["cl"])
        if s["op"] == "convt":
            op = rt.ConvTranspose(groups=s.get("groups", 1), strides=s["strides"])
            return op.run(ctx, xd, ctx.to_device(inp["w"]), inp["bias"]).numpy()
        B, C, H, W, O, Cg, kh, kw, *_ = conv_geometry(s)
        w = inp["w"]
        if s.get("wview"):
            host = np.full((O, Cg + 2, kh, kw + 1), np.nan, F32)
            host[:, :Cg, :, :kw] = w
            wd = ctx.to_device(host).view(w.shape, ((Cg + 2) * kh * (kw + 1), kh * (kw + 1), kw + 1, 1))
        else:
            wd = ctx.to_device(w)
        op = rt.Conv(groups=C // Cg, dilations=s.get("dil", (1, 1)), padding=s.get("pads", (0, 0, 0, 0)),
                     strides=s.get("strides", (1, 1)))
        return op.run(ctx, xd, wd).numpy()
    finally:
        ctx.set_f32_mode(True)


# ---- Cast int32 -> float, Clip ----------------------------------------------------------------------------------------
def cast_rule(s):
    return [U("cast_scale_kernel", partial=_part(s["n"]))]


def cast_specs(sms):
    return [dict(n=n) for n in (1, 300, 4096, 100003)]


def cast_prepare(s):
    r = _rng("cast", s["n"])
    x = r.integers(-2 ** 31, 2 ** 31, s["n"], dtype=np.int64).astype(I32)
    edges = [2 ** 24, 2 ** 24 + 1, 2 ** 24 + 3, -(2 ** 24) - 1, 2 ** 25 + 2, 2 ** 25 + 6, 2 ** 31 - 1, -2 ** 31, 2 ** 31 - 64,
             2 ** 31 - 65, 2 ** 31 - 128, -(2 ** 31) + 64, -(2 ** 31) + 65, 0, -1, 1, 16777217 * 3]
    x[:min(len(edges), x.size)] = np.array(edges[:x.size], np.int64).astype(I32)
    return dict(x=x)


def cast_launch(rt, ctx, s, inp):
    import onnx_writer as W
    from rten_b200.model import Model
    g = W.model([W.node("Cast", ["x"], ["y"], to=W.FLOAT)], [], [W.value_info("x", W.INT32, [s["n"]])],
                [W.value_info("y", W.FLOAT, [s["n"]])])
    (y,) = Model(ctx, g).run({"x": inp["x"]}, ["y"])
    return y.numpy()


def clip_rule(s):
    mode = "default bounds" if s["min"] is None and s["max"] is None else "given bounds"
    return [U("clip_kernel", ("float",) if s["dtype"] == "f32" else ("int",), mode, _part(s["n"]))]


def clip_specs(sms):
    f, i = dict(dtype="f32"), dict(dtype="i32")
    return [dict(f, n=1000, min=-1.5, max=2.0), dict(f, n=1024, min=0.0, max=None), dict(f, n=77, min=None, max=-0.0),
            dict(f, n=4096, min=None, max=None), dict(f, n=333, min=None, max=None), dict(f, n=64, min=3.0, max=1.0),
            dict(i, n=1000, min=-100, max=50), dict(i, n=2048, min=None, max=7), dict(i, n=513, min=-2 ** 31, max=None),
            dict(i, n=256, min=None, max=None), dict(i, n=999, min=None, max=None), dict(i, n=100, min=9, max=-9)]


def clip_prepare(s):
    r = _rng("clip", sorted((k, str(v)) for k, v in s.items()))
    n = s["n"]
    if s["dtype"] == "f32":
        x = r.uniform(-4, 4, n).astype(F32)
        sp = np.array([np.nan, -np.nan, np.inf, -np.inf, -0.0, 0.0, 3.4e38, -3.4e38, 1e-45], F32)
    else:
        x = r.integers(-2 ** 31, 2 ** 31, n, dtype=np.int64).astype(I32)
        sp = np.array([-2 ** 31, 2 ** 31 - 1, 0, -1, 1, -100, 50], I32)
    x[:min(n, sp.size)] = sp[:min(n, sp.size)]
    return dict(x=x)


def clip_launch(rt, ctx, s, inp):
    t = F32 if s["dtype"] == "f32" else I32
    mn = None if s["min"] is None else np.array(s["min"], t)
    mx = None if s["max"] is None else np.array(s["max"], t)
    return rt.Clip().run(ctx, ctx.to_device(inp["x"]), mn, mx).numpy()


def clip_ref(x, mn, mx):
    """src/ops/unary_elementwise.rs Clip: x.max(min).min(max) with `a > b ? a : b` and `a < b ? a : b` (so NaN becomes
    min, and -0.0 clipped at min = +0.0 becomes +0.0: -0.0 > +0.0 is false); missing bounds are the type's finite
    extremes"""
    t = x.dtype.type
    lo = t(mn) if mn is not None else (t(-np.finfo(F32).max) if t is F32 else t(-2 ** 31))
    hi = t(mx) if mx is not None else (t(np.finfo(F32).max) if t is F32 else t(2 ** 31 - 1))
    with np.errstate(invalid="ignore"):
        v = np.where(x > lo, x, lo).astype(x.dtype)
        return np.where(v < hi, v, hi).astype(x.dtype)


# ---- the case families ------------------------------------------------------------------------------------------------
RULES = {"copy": copy_rule, "dql": dql_rule, "int8": int8_rule, "f32": f32_rule, "cast": cast_rule, "clip": clip_rule}
SPECS = {"copy": copy_specs, "dql": dql_specs, "int8": int8_specs, "f32": f32_specs, "cast": cast_specs, "clip": clip_specs}
PREPARE = {"copy": copy_prepare, "dql": dql_prepare, "int8": int8_prepare, "f32": f32_prepare, "cast": cast_prepare,
           "clip": clip_prepare}
LAUNCH = {"copy": copy_launch, "dql": dql_launch, "int8": int8_launch, "f32": f32_launch, "cast": cast_launch,
          "clip": clip_launch}


def spec_id(fam, s):
    return fam + " " + " ".join(f"{k}={v}" for k, v in s.items())


def claimed(fam, s):
    """the kernels whose launches a case's rule accounts for: its family's, except that a ConvTranspose's phase
    convolutions (which may split or im2col) are not restated here"""
    if fam == "f32" and s["op"] == "convt":
        return {"conv_transpose_pack_kernel", "conv_transpose_fill_kernel"}
    return set(FAMILY_KERNELS[fam])


def case_units(fam, s):
    """{(kernel, arguments, mode): partial} of a case (a kernel launched twice counts once, partial if either is)"""
    out = {}
    for k, a, m, p in RULES[fam](s):
        out[(k, a, m)] = out.get((k, a, m), False) or p
    return out


def _rng(*key):
    return rk._rng("staging", *key)


def coverage_gaps(sms):
    """(kernel, arguments, mode) units that fewer than two cases select, or that no case selects with a partial last
    unit"""
    picked, part = {}, set()
    for fam, specs in SPECS.items():
        for s in specs(sms):
            for (k, a, m), p in case_units(fam, s).items():
                assert a in VARIANTS[k] and m in _modes(k, a), f"{spec_id(fam, s)}: the rule names {(k, a, m)}, which the table lacks"
                assert k in FAMILY_KERNELS[fam], f"{spec_id(fam, s)}: {k} is not a kernel of the family"
                picked[(k, a, m)] = picked.get((k, a, m), 0) + 1
                if p:
                    part.add((k, a, m))
    gaps = [("selected fewer than twice", u) for u in units() if picked.get(u, 0) < 2]
    return gaps + [("never with a partial last unit", u) for u in units() if u not in part]


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
    res, retaken = {}, 0
    for fam, specs in SPECS.items():
        for s in specs(n_sms):
            inp = PREPARE[fam](s)

            def call():
                LAUNCH[fam](rt, ctx, s, inp)
                ctx.sync()
            names, again = rk.capture_kernels(call)
            retaken += again
            res[spec_id(fam, s)] = sorted(names)
    print(json.dumps({"sms": n_sms, "names": res, "retaken": retaken}))


def test_kernel_identity():
    out = rk.probe_in_child("test_gpu_staging_kernels")
    n_sms, names = out["sms"], out["names"]
    seen, wrong = {}, []
    for fam, specs in SPECS.items():
        for s in specs(n_sms):
            sid = spec_id(fam, s)
            want = case_units(fam, s)
            ran = {rk.kernel_key(n, KERNELS) for n in names[sid]} - {None}
            ran = {k for k in ran if k[0] in claimed(fam, s)}
            if ran != {(k, a) for k, a, _ in want}:
                wrong.append((sid, sorted({(k, a) for k, a, _ in want}), sorted(ran)))
            for k, a, m in want:
                if (k, a) in ran:
                    seen[(k, a, m)] = seen.get((k, a, m), 0) + 1
    assert not wrong, f"{len(wrong)} cases ran other kernels than the rule names: {wrong[:8]}"
    missing = [u for u in units() if seen.get(u, 0) < 2]
    assert not missing, f"kernels (and modes) that fewer than two cases ran: {missing}"
    assert not coverage_gaps(n_sms)
    print(f"{len(units())} kernel units each ran at least twice on {n_sms} SMs; {len(names)} captures, "
          f"{out['retaken']} taken again")
    for u in units():
        print(f"  {u[0]}{'<' + ', '.join(u[1]) + '>' if u[1] else ''} {u[2] or ''}: {seen[u]} cases")


# ---- numbers ----------------------------------------------------------------------------------------------------------
def test_strided_copy_bits(rt, sms):
    ctx = rt.Context(0)
    for s in copy_specs(sms):
        got, want = copy_launch(rt, ctx, s, copy_prepare(s))
        assert got.dtype == want.dtype and np.array_equal(got, want), (
            f"{spec_id('copy', s)}: {int((got != want).sum())} elements differ in their bits")


def test_dynamic_quantize_linear_bit_exact(rt, oracle, sms):
    """Bit-exact against oracle.dynamic_quantize_linear: NaN quantises to 0 (the reference's SIMD body: the conversion
    gives INT_MIN, then saturates), every positive x of an input of subnormals only to 0 (1 / scale = +inf), and exact
    .5 ties to even."""
    ctx = rt.Context(0)
    for s in dql_specs(sms):
        inp = dql_prepare(s)
        ey = dql_check(oracle, s, inp, dql_launch(rt, ctx, s, inp))
        if s["values"] == "nan":
            x = inp["x"].reshape(-1) if s["kind"] == "flat" else inp["x"].transpose(0, 2, 3, 1).reshape(-1)
            assert (ey.transpose(0, 2, 3, 1).reshape(-1) if ey.ndim == 4 else ey)[np.isnan(x)].max() == 0


def test_zero_points_and_int8_staging_exact(rt, oracle, sms):
    ctx = rt.Context(0)
    for s in int8_specs(sms):
        inp = int8_prepare(s)
        gc.assert_bit_exact(int8_launch(rt, ctx, s, inp), int8_want(oracle, s, inp), spec_id("int8", s))


def test_f32_staging_exact(rt, sms):
    """Integer-valued operands: the exact product, converted to f32 once, in both f32 modes.  This rests on wgmma's
    f32 accumulation adding integer-valued terms exactly while every partial sum stays below 2^24 (exact TF32 products,
    a 24-bit accumulator significand)."""
    ctx = rt.Context(0)
    for s in f32_specs(sms):
        inp = f32_prepare(s)
        exact, bound = _exact(s, inp)
        assert bound < 2 ** 24, f"{spec_id('f32', s)}: sum |a||b| = {bound} is not exact in f32"
        if s["mode"] == "TF32":
            for v in inp.values():
                assert v is None or (np.abs(v) < 2 ** 11).all(), "a TF32 operand with more than 11 significant bits"
        gc.assert_bit_exact(f32_launch(rt, ctx, s, inp), exact.astype(F32), spec_id("f32", s))


def test_cast_int32_to_float(rt, sms):
    """Cast int32 -> float rounds to nearest, ties to even: 2^24 + 1 -> 2^24, 2^24 + 3 -> 2^24 + 4, INT_MAX -> 2^31"""
    ctx = rt.Context(0)
    for s in cast_specs(sms):
        inp = cast_prepare(s)
        gc.assert_bit_exact(cast_launch(rt, ctx, s, inp), inp["x"].astype(F32), spec_id("cast", s))


def test_clip_exact(rt, sms):
    ctx = rt.Context(0)
    for s in clip_specs(sms):
        inp = clip_prepare(s)
        got = clip_launch(rt, ctx, s, inp)
        want = clip_ref(inp["x"], s["min"], s["max"])
        gc.assert_bit_exact(got, want, spec_id("clip", s))
        if s["dtype"] == "f32" and s["min"] is not None and (s["max"] is None or s["min"] <= s["max"]):
            assert (got[:2] == np.float32(s["min"])).all(), f"{spec_id('clip', s)}: NaN is not clipped to min"


def test_clip_reference_expectations(rt):
    """The reference's own Clip unit tests (src/ops/unary_elementwise.rs), through the kernel: NaN -> min, -0.0 at
    min = +0.0 -> +0.0, min > max -> max everywhere"""
    ctx = rt.Context(0)
    x = np.array([np.nan, -0.0, -5.0, 0.5, 10.0], F32)
    got = rt.Clip().run(ctx, ctx.to_device(x), np.array(0.0, F32), np.array(6.0, F32)).numpy()
    assert got[0] == 0.0 and got[1] == 0.0 and not np.signbit(got[1]) and got[2] == 0.0 and got[3] == 0.5 and got[4] == 6.0, got
    assert (rt.Clip().run(ctx, ctx.to_device(x[2:]), np.array(3.0, F32), np.array(1.0, F32)).numpy() == 1.0).all()
    i = np.array([-2 ** 31, 2 ** 31 - 1, 0], I32)
    assert (rt.Clip().run(ctx, ctx.to_device(i)).numpy() == i).all()
