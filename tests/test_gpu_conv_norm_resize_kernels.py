"""`pytest -m gpu`: the depthwise convolution, GroupNorm / InstanceNormalization, Resize / Concat, ReduceSum / ReduceMean
and rotary-embedding kernels (depthwise.cu, groupnorm.cu, resize.cu, reduce.cu, rotary.cu), each selected by name and
checked bit for bit.

The launchers pick an instance and a runtime mode from the element type, strides, pointer alignment, shapes and the SM
count.  The rules are restated below (`*_rule`); `VARIANTS` lists every instance they pick from
(tests/test_conv_norm_resize_kernel_table_cpu.py keeps it equal to the built library's symbols).  A rule returns the
units a case runs -- (kernel, template arguments, partial last unit) -- and the runtime modes it reaches.  The case lists
select every instance at least twice, once with a partial last unit: a partial last channel slice (threads whose channel
vector starts past C), a partial last run or quad, a ragged last ring chunk or lane, idle threads of the last block, or
a grid-stride loop that runs past the grid.  `MODES` lists the runtime branches a name does not show; each must be
reached (for depthwise, by an f32 case and by an 8-bit one).

  * kernel identity: every case runs once under CUPTI in a child process; each case must run exactly the instances of
    `VARIANTS` its rule names, no more and no fewer (kernels of other files, such as the strided copy of a channels-last
    read-back or of the channels-last GroupNorm stream, are not claimed), and every entry of `VARIANTS` must have run;
  * depthwise Conv / ConvInteger / ConvIntegerToFloat against oracle/depthwise.py: several channel slices with a
    partial last one, a halved slice for 7x7 and 15x15 kernels, weights read through the read-only cache when even one
    vector's taps exceed 48 KB (1-D NWC convolutions with 3073 to 12289 taps), a 17-channel slice of a 20-channel
    channels-last buffer in and out (the 4-channel vector's tail) whose other channels must stay untouched, every 8-bit
    signedness pair on the vector, scalar and planar bodies with zero points, scale_b, bias, residual, Relu and the
    output range;
  * GroupNorm / InstanceNormalization against tests/instance_norm_ref.py, on chip and streaming
    (RTEN_B200_GROUP_NORM_STREAM), NCHW and channels-last, vector and scalar, at the 128- and 1024-thread clamps, with
    more than 65535 planes and more than 65535 channels-last images;
  * Resize against oracle/resize.py on each kernel, nearest and linear, with a partial last quad and outputs into a
    channel slice or a padded row; Concat of f32 / i32 / i8 / u8 through each copy unit and more than 16 sources;
  * ReduceSum / ReduceMean against genai_decoder.reduce_sum_ref (ReduceMean: that sum / L in f32), i32 against the
    wrapped exact sum, contiguous and strided or misaligned, short and long lanes, more outputs than the grid;
  * RotaryEmbedding and GroupQueryAttention's cache build against test_gpu_group_query_attention.rotary_ref in float32
    (bit-exact: the kernel rounds each product and sum, as numpy's float32 does); MultiHeadAttention's bias add into
    the present key and value caches, exactly.

For the cases that loop past the grid, the value tests compare the head and tail of the output only."""
import json
import re

import numpy as np
import pytest

import gpu_checks as gc
import test_gpu_row_kernels as rk

pytestmark = pytest.mark.gpu

F32, I32, U8, I8 = np.float32, np.int32, np.uint8, np.int8
SMEM_MAX = 48 * 1024  # depthwise.cu kSmemMax

# ---- the kernels ------------------------------------------------------------------------------------------------------
_T8 = {"u8": "unsigned char", "i8": "signed char"}
PAIRS8 = ("u8u8", "u8i8", "i8u8", "i8i8")  # (x type, w type)
OUT_CODE = {"f32": 0, "i32": 1, "qf32": 2, "act": 3}  # depthwise.cu OUT_*


def _dw_types(x):
    return ("float", "float") if x == "f32" else (_T8[x[:2]], _T8[x[2:]])


VARIANTS = {
    # <XT, WT, OUT, VEC>
    "depthwise_cl_kernel": [("float", "float", o, v) for o in (0, 3) for v in (1, 4)]
                           + [_dw_types(p) + (o, v) for p in PAIRS8 for o in (1, 2) for v in (1, 4)],
    # <XT, WT, OUT>
    "depthwise_planar_kernel": [("float", "float", 0), ("float", "float", 3)] + [_dw_types(p) + (o,) for p in PAIRS8 for o in (1, 2)],
    "gn_onchip_kernel": [(0,), (1,)], "gn_stats_kernel": [()], "gn_apply_kernel": [(0,), (1,)],  # <CL>
    "resize_cl4_kernel": [(0,), (1,)],  # <LINEAR>
    "resize_kernel": [(lin, row) for lin in (0, 1) for row in (0, 1)],  # <LINEAR, ROW>
    "concat_kernel": [("uint4",), ("unsigned int",), ("unsigned char",)],
    "reduce_sum_warp_kernel": [(t, v) for t in ("float", "int") for v in (0, 1)],  # <T, VEC>
    "reduce_sum_cta_kernel": [(t, v) for t in ("float", "int") for v in (0, 1)],
    "rotary_kernel": [()], "rotary_mha_kernel": [()],
}
KERNELS = set(VARIANTS)
FAMILY_KERNELS = {
    "dw": ("depthwise_cl_kernel", "depthwise_planar_kernel"),
    "gn": ("gn_onchip_kernel", "gn_stats_kernel", "gn_apply_kernel"),
    "resize": ("resize_cl4_kernel", "resize_kernel"),
    "concat": ("concat_kernel",),
    "reduce": ("reduce_sum_warp_kernel", "reduce_sum_cta_kernel"),
    "rotary": ("rotary_kernel", "rotary_mha_kernel"),
}
# The runtime branches a name does not show.  Depthwise modes are required of an f32 case and of an 8-bit one.
DW_MODES = ("one slice", "several slices", "partial last slice", "halved slice", "weights through the read-only cache",
            "several runs per CTA", "4-channel tail")
MODES = {
    "dw": tuple(f"{t} {m}" for t in ("f32", "8-bit") for m in DW_MODES),
    "gn": ("on chip NCHW vec", "on chip NCHW scalar", "on chip channels-last", "on chip 128 threads", "on chip 1024 threads",
           "stream NCHW vec", "stream NCHW scalar", "stream channels-last vec", "stream channels-last scalar",
           "stream channels-last vec, C / G % 4 != 0", "more than 65535 planes", "more than 65535 images"),
    "resize": ("cl4", "channel fastest", "row vec", "row scalar", "row partial quad", "past the grid"),
    "concat": ("16-byte units", "element units", "more than 16 sources", "past the grid"),
    "reduce": ("warp", "CTA", "vec", "scalar", "misaligned", "warp past the grid", "CTA past the grid", "ReduceMean"),
    "rotary": ("RotaryEmbedding", "interleaved", "position ids", "GroupQueryAttention", "MultiHeadAttention"),
}

_NAME = re.compile(r"(\w+)(?:<([^<>]*)>)?\(")


def kernel_key(name, kernels=KERNELS):
    """(kernel, template arguments) of a demangled kernel name of `kernels`, else None.  Reads the anonymous namespace
    in both spellings (`rtb::(anonymous namespace)::` from CUPTI, `rtb::<unnamed>::` from cu++filt), names without
    template arguments, and both spellings of the arguments (`<float, true>`, `<float, (bool)1>`, `(int)4`).  Values
    become ints, type arguments stay names (`signed char`, `uint4`)."""
    for m in _NAME.finditer(name):
        if m.group(1) in kernels:
            args = []
            for a in (m.group(2).split(",") if m.group(2) else []):
                a = re.sub(r"^\((int|bool)\)", "", a.strip())
                args.append({"true": 1, "false": 0}[a] if a in ("true", "false") else int(a) if re.fullmatch(r"-?\d+", a) else a)
            return m.group(1), tuple(args)
    return None


def U(k, a=(), partial=False):
    return (k, tuple(a), bool(partial))


def _cdiv(a, b):
    return -(-a // b)


def _grid(items, sms):
    """resize.cu grid_for: one 256-thread block per 256 items, at most 8 per SM"""
    return max(1, min(_cdiv(items, 256), 8 * sms))


def _loops(items, sms):
    """a block with idle threads, or a grid-stride loop past the grid"""
    return items % 256 != 0 or items > 256 * _grid(items, sms)


# ---- depthwise convolution --------------------------------------------------------------------------------------------
def dw_geometry(s):
    """(B, C, H, W, kh, kw, pt, pl, pb, pr, sy, sx, OH, OW); a 1-D case is 2-D over H = 1"""
    shape = s["x"]
    one_d = len(shape) == 3
    B, C, W = shape[0], shape[1], shape[-1]
    H = 1 if one_d else shape[2]
    kh, kw = (1, s["k"][0]) if one_d else s["k"]
    p = s.get("pads", (0, 0) if one_d else (0, 0, 0, 0))
    pt, pl, pb, pr = (0, p[0], 0, p[1]) if one_d else p
    st = s.get("strides", (1,) if one_d else (1, 1))
    sy, sx = (1, st[0]) if one_d else st
    OH = (H + pt + pb - kh) // sy + 1
    OW = (W + pl + pr - kw) // sx + 1
    return B, C, H, W, kh, kw, pt, pl, pb, pr, sy, sx, OH, OW


def dw_pixel_stride(s):
    """the channels-last pixel stride of x and of the output (a channel slice: the buffer's channel count)"""
    return s.get("cb", s["x"][1])


def dw_rule(s, sms):
    """depthwise.cu launch_typed: channel stride 1 and C > 1 take the channels-last body, 4-channel vectors when every
    pixel stride of x and the output is a multiple of 4 (and both are aligned), else 1; a slice of nv vectors (at most 64,
    the slices balanced) x 256 / nv pixels per pass, nv halved while the slice's weights exceed 48 KB, and read through
    the read-only cache when even one vector's do; up to 8 passes (runs) per CTA while the grid still gives every SM 8
    CTAs.  Otherwise one thread per output (the planar body)."""
    B, C, H, W, kh, kw, pt, pl, pb, pr, sy, sx, OH, OW = dw_geometry(s)
    xt, wt = _dw_types(s["dt"])
    out = OUT_CODE[s["out"]]
    cls = "f32" if s["dt"] == "f32" else "8-bit"
    if s["layout"] == "nchw" or C == 1:
        n = B * C * OH * OW
        return [U("depthwise_planar_kernel", (xt, wt, out), n % 256 != 0)], set()
    vec = dw_pixel_stride(s) % 4 == 0
    V = 4 if vec else 1
    es = 4 if s["dt"] == "f32" else 1
    taps = kh * kw
    nvec = _cdiv(C, V)
    nv = nv0 = _cdiv(nvec, _cdiv(nvec, 64))
    while nv > 1 and taps * V * nv * es > SMEM_MAX:
        nv = (nv + 1) // 2
    use_smem = taps * V * nv * es <= SMEM_MAX
    ppb = 256 // nv
    gy = _cdiv(C, V * nv)
    npix = B * OH * OW
    groups = _cdiv(npix, ppb)
    runs = 8
    while runs > 1 and groups * gy < runs * sms * 8:
        runs //= 2
    idle_slice = gy * V * nv - C >= V  # channel vectors of the last slice that start past C (n <= 0)
    partial = idle_slice or npix % ppb != 0 or groups % runs != 0 or 256 % nv != 0 or C % V != 0
    modes = {"several slices" if gy > 1 else "one slice"}
    if idle_slice:
        modes.add("partial last slice")
    if nv < nv0:
        modes.add("halved slice")
    if not use_smem:
        modes.add("weights through the read-only cache")
    if runs > 1:
        modes.add("several runs per CTA")
    if V == 4 and C % 4:
        modes.add("4-channel tail")
    return [U("depthwise_cl_kernel", (xt, wt, out, V), partial)], {f"{cls} {m}" for m in modes}


def dw_specs(sms):
    f = lambda x, k, layout, out="f32", **kw: dict(dt="f32", out=out, x=x, k=k, layout=layout, **kw)  # noqa: E731
    specs = [
        # f32 and f32 + activations 4-7: planar, scalar and vector channels-last bodies
        f((2, 17, 9, 11), (3, 3), "nchw", pads=(1, 1, 1, 1)), f((1, 5, 8, 8), (5, 5), "nchw", out="act", act=5, strides=(2, 2)),
        f((2, 3, 7, 9), (3, 3), "nchw", out="act", act=7, pads=(1, 0, 1, 2)), f((1, 9, 6, 13), (3, 1), "nchw", pads=(1, 0, 1, 0)),
        f((2, 17, 9, 11), (3, 3), "cl", pads=(1, 1, 1, 1)), f((1, 6, 10, 10), (3, 3), "cl", out="act", act=4, strides=(2, 2)),
        f((2, 3, 12), (5,), "cl", out="act", act=6, pads=(2, 1)),
        f((2, 20, 9, 9), (3, 3), "cl", pads=(1, 1, 1, 1)), f((1, 8, 7, 7), (5, 5), "cl", out="act", act=5, pads=(2, 2, 2, 2)),
        f((2, 12, 16), (3,), "cl", out="act", act=7, strides=(2,)),
        # several slices: C = 130 at VEC = 1 (a partial last slice), C = 260 at VEC = 4 (one idle vector), C = 960
        f((1, 130, 6, 7), (3, 3), "cl", pads=(1, 1, 1, 1)), f((1, 260, 5, 6), (3, 3), "cl", pads=(1, 1, 1, 1)),
        f((1, 960, 4, 4), (3, 3), "cl", pads=(1, 1, 1, 1)),
        # halved slice: 7 x 7 at 63 vectors (nv 63 -> 32: two slices, the last partial), 15 x 15 at VEC = 1
        f((1, 252, 9, 9), (7, 7), "cl", pads=(3, 3, 3, 3)), f((1, 66, 16, 17), (15, 15), "cl", pads=(7, 7, 7, 7), strides=(2, 2)),
        # weights through the read-only cache: 1-D NWC, one vector's 3073 (VEC = 4) / 12289 (VEC = 1) taps beyond 48 KB
        f((1, 4, 3075), (3073,), "cl"), f((1, 3, 12291), (12289,), "cl", out="act", act=5),
        # several runs per CTA
        f((1, 16, 400, 400), (3, 3), "cl", pads=(1, 1, 1, 1)),
        # a 17-channel slice of a 20-channel channels-last buffer, in and out, with a residual: the 4-channel tail
        f((2, 17, 9, 11), (3, 3), "slice", cb=20, pads=(1, 1, 1, 1), res=True),
        f((1, 17, 12), (5,), "slice", cb=20, pads=(2, 2), res=True, out="act", act=4),
        f((1, 6, 7, 5), (3, 3), "slice", cb=8, strides=(2, 1), res=True),
    ]
    # every 8-bit pair and output on the vector, scalar and planar bodies
    for p in PAIRS8:
        for out in ("i32", "qf32"):
            q = dict(dt=p, out=out)
            specs += [dict(q, x=(2, 20, 7, 9), k=(3, 3), layout="cl", pads=(1, 1, 1, 1)),
                      dict(q, x=(1, 17, 8, 7), k=(3, 3), layout="slice", cb=20, pads=(0, 1, 2, 1), res=out == "qf32"),
                      dict(q, x=(2, 17, 9, 8), k=(5, 5), layout="cl", strides=(2, 2), pads=(2, 2, 2, 2)),
                      dict(q, x=(2, 3, 14), k=(3,), layout="cl", pads=(1, 1)),
                      dict(q, x=(2, 17, 6, 7), k=(3, 3), layout="nchw", pads=(1, 1, 1, 1)),
                      dict(q, x=(1, 5, 13), k=(5,), layout="nchw", strides=(2,))]
    # 8-bit modes
    specs += [dict(dt="u8i8", out="qf32", x=(1, 260, 5, 6), k=(3, 3), layout="cl", pads=(1, 1, 1, 1)),
              dict(dt="i8u8", out="i32", x=(1, 130, 4, 5), k=(3, 3), layout="cl"),
              dict(dt="i8i8", out="qf32", x=(1, 256, 17, 17), k=(15, 15), layout="cl", pads=(7, 7, 7, 7), strides=(4, 4)),
              dict(dt="u8u8", out="i32", x=(1, 8, 12291), k=(12289,), layout="cl"),
              dict(dt="u8i8", out="i32", x=(1, 16, 400, 400), k=(3, 3), layout="cl", pads=(1, 1, 1, 1))]
    return specs


def dw_prepare(s):
    B, C, H, W, kh, kw, *_ = dw_geometry(s)
    r = _rng("dw", sorted((k, str(v)) for k, v in s.items()))
    one_d = len(s["x"]) == 3
    wshape = (C, 1, kw) if one_d else (C, 1, kh, kw)
    OH, OW = dw_geometry(s)[-2:]
    oshape = (B, C, OW) if one_d else (B, C, OH, OW)
    if s["dt"] == "f32":
        big = kh * kw > 1000  # long sums: small integers keep every partial sum exact and far from overflow
        x = (r.integers(-3, 4, s["x"]) if big else r.uniform(-2, 2, s["x"])).astype(F32)
        w = (r.integers(-2, 3, wshape) if big else r.uniform(-1, 1, wshape)).astype(F32)
        inp = dict(x=x, w=w, b=r.uniform(-1, 1, C).astype(F32))
    else:
        lo = lambda t: (-128, 128) if t == "i8" else (0, 256)  # noqa: E731
        dt = lambda t: I8 if t == "i8" else U8  # noqa: E731
        xt, wt = s["dt"][:2], s["dt"][2:]
        inp = dict(x=r.integers(*lo(xt), s["x"]).astype(dt(xt)), w=r.integers(*lo(wt), wshape).astype(dt(wt)),
                   xz=dt(xt)(r.integers(*lo(xt))), wz=r.integers(*lo(wt), C).astype(dt(wt)),
                   scale=F32(0.0173), scale_b=F32(0.37), b=r.uniform(-1, 1, C).astype(F32))
    if s.get("res"):
        inp["res"] = r.uniform(-2, 2, oshape).astype(F32)
    return inp


def _cl_strides(shape, cb):
    """channels-last strides of `shape` with a pixel stride of cb channels"""
    if len(shape) == 3:
        B, C, W = shape
        return (W * cb, 1, cb)
    B, C, H, W = shape
    return (H * W * cb, 1, W * cb, cb)


def _placed(ctx, arr, cb, fill):
    """(a channels-last view of arr's channels at the front of a cb-channel buffer filled with `fill`, the buffer)"""
    full_shape = (arr.shape[0], cb) + arr.shape[2:]
    host = np.full(full_shape, fill, arr.dtype)
    host[:, :arr.shape[1]] = arr
    buf = ctx.empty(full_shape, arr.dtype, _cl_strides(full_shape, cb))
    buf.copy_from(host)
    return buf.view(arr.shape, _cl_strides(arr.shape, cb)), buf


def dw_launch(rt, ctx, s, inp):
    """(the output, and for a channel slice the output buffer's other channels)"""
    B, C, H, W, kh, kw, pt, pl, pb, pr, sy, sx, OH, OW = dw_geometry(s)
    one_d = len(s["x"]) == 3
    kw_ = dict(groups=C, padding=(pl, pr) if one_d else (pt, pl, pb, pr), strides=(sx,) if one_d else (sy, sx),
               dilations=(1,) if one_d else (1, 1))
    x = inp["x"]
    out = None
    if s["layout"] == "nchw":
        xd = ctx.to_device(x)
    elif s["layout"] == "cl":
        xd = ctx.empty(x.shape, x.dtype, _cl_strides(x.shape, C))
        xd.copy_from(x)
    else:
        xd, _ = _placed(ctx, x, s["cb"], x.dtype.type(7))
        oshape = (B, C, OW) if one_d else (B, C, OH, OW)
        out, obuf = _placed(ctx, np.zeros(oshape, F32 if s["out"] != "i32" else I32), s["cb"], np.nan if s["out"] != "i32" else -7)
    res = inp.get("res")
    if s["out"] in ("f32", "act"):
        y = rt.Conv(activation=s.get("act", 0), **kw_).run(ctx, xd, inp["w"], inp["b"], residual=res, out=out)
    elif s["out"] == "i32":
        y = rt.ConvInteger(**kw_).run(ctx, xd, inp["w"], inp["xz"], inp["wz"], out=out)
    else:
        rng = ctx.to_device(np.zeros(2, I32))
        rt.DynamicQuantizeLinear.reset_ranges(ctx, rng)
        y = rt.ConvIntegerToFloat(activation=1, **kw_).run(ctx, xd, inp["w"], inp["xz"], inp["wz"], inp["scale"], out=out,
                                                           bias=inp["b"], residual=res, scale_b=inp["scale_b"], out_range=rng)
        inp["range"] = rng
    if out is None:
        return y.numpy(), None
    whole = obuf.numpy()
    return y.numpy(), whole[:, C:]


def dw_want(s, inp):
    from oracle import activations as A
    from oracle import depthwise as D
    B, C, H, W, kh, kw, pt, pl, pb, pr, sy, sx, OH, OW = dw_geometry(s)
    one_d = len(s["x"]) == 3
    kw_ = dict(padding=(pl, pr) if one_d else (pt, pl, pb, pr), strides=(sx,) if one_d else (sy, sx),
               dilations=(1,) if one_d else (1, 1))
    if s["dt"] == "f32":
        y = D.depthwise_conv(inp["x"], inp["w"], inp["b"], **kw_)
        if "res" in inp:
            y = (y + inp["res"]).astype(F32)
        act = s.get("act", 0)
        fn = {0: lambda v: v, 4: A.sigmoid, 5: A.silu, 6: A.hard_sigmoid, 7: A.hard_swish}[act]
        return np.asarray(fn(y), F32)
    acc = D.depthwise_conv_integer(inp["x"], inp["w"], inp["xz"], inp["wz"], **kw_)
    if s["out"] == "i32":
        return acc
    return D.integer_to_float(acc, inp["scale"], scale_b=inp["scale_b"], bias=inp["b"], residual=inp.get("res"), relu=True)


# ---- GroupNorm / InstanceNormalization -------------------------------------------------------------------------------
def gn_rule(s, sms):
    """groupnorm.cu launch_group_norm: rows of L = (C / G) P elements up to 51200 (and no RTEN_B200_GROUP_NORM_STREAM)
    run on chip, one CTA per row of clamp(ceil(L / 16) rounded up to a warp, 128, 1024) threads, 16-byte copies for NCHW
    rows with L % 4 == 0.  Longer rows stream: the statistics per row (8192-float ring chunks; channels-last rows are
    copied to [N, C, P] first), then the output pass: NCHW with one y block row per (n, c) plane up to 65535 (then a
    loop) and float4s when P % 4 == 0; channels-last with one y block row per image up to 65535 and k pixels per sweep,
    float4s when C % 4 == 0."""
    N, C = s["x"][:2]
    P = int(np.prod(s["x"][2:]))
    G = s["G"]
    cg, cl = C // G, s["cl"]
    L = cg * P
    if L <= 51200 and not s["stream"]:
        threads = min(1024, max(128, _cdiv(_cdiv(L, 16), 32) * 32))
        modes = {"on chip channels-last" if cl else "on chip NCHW vec" if L % 4 == 0 else "on chip NCHW scalar"}
        if threads in (128, 1024):
            modes.add(f"on chip {threads} threads")
        return [U("gn_onchip_kernel", (int(cl),), L % threads != 0)], modes
    out = [U("gn_stats_kernel", (), L % 8192 != 0 or L % 64 != 0)]
    bw = 8 * sms
    if not cl:
        vec = P % 4 == 0
        n4, planes = (P // 4 if vec else P), N * C
        gy = min(planes, 65535)
        gx = max(1, min(_cdiv(n4, 1024), _cdiv(bw, gy)))
        modes = {"stream NCHW vec" if vec else "stream NCHW scalar"}
        if planes > 65535:
            modes.add("more than 65535 planes")
        return out + [U("gn_apply_kernel", (0,), n4 % (256 * gx) != 0 or planes > gy)], modes
    vec = C % 4 == 0
    CU, gy = (C // 4 if vec else C), min(N, 65535)
    k = max(1, (bw // gy) * 256 // CU)
    k = min(k, max(1, _cdiv(P, 4)))
    modes = {"stream channels-last vec" if vec else "stream channels-last scalar"}
    if vec and cg % 4:
        modes.add("stream channels-last vec, C / G % 4 != 0")
    if N > 65535:
        modes.add("more than 65535 images")
    return out + [U("gn_apply_kernel", (1,), (CU * k) % 256 != 0 or P % k != 0 or N > gy)], modes


def gn_specs(sms):
    g = lambda x, G, cl, stream, **kw: dict(x=x, G=G, cl=cl, stream=stream, **kw)  # noqa: E731
    specs = []
    for stream in (False, True):
        specs += [g((2, 8, 10, 10), 4, False, stream, affine=True), g((1, 6, 7, 7), 2, False, stream, act=5),
                  g((2, 12, 9, 9), 3, True, stream, affine=True), g((2, 12, 5, 5), 4, True, stream, act=5),
                  g((2, 6, 7, 7), 3, True, stream, affine=True), g((1, 10, 5, 6), 5, True, stream)]
    specs += [
        # the on-chip thread-count clamps: L = 2048 (128) is the top of the 128 clamp, 16384 and 39996 give 1024
        g((2, 32, 64, 64), 8, False, False, affine=True), g((1, 4, 99, 101), 1, False, False),
        g((1, 3, 97, 101), 1, False, False, act=5), g((1, 64, 32, 32), 2, True, False, affine=True),
        g((1, 16, 8, 16), 8, False, False),
        # long rows stream on their own: several ring chunks and a ragged last one
        g((1, 4, 170, 170), 2, False, False, affine=True), g((1, 8, 120, 120), 2, True, False, act=5),
        # more than 65535 planes and channels-last images, tiny spatial size: InstanceNormalization streaming
        g((2, 33000, 1, 3), 33000, False, True, inst=True), g((1, 65600, 2, 2), 65600, False, True, inst=True),
        g((65600, 4, 1, 2), 4, True, True, inst=True), g((65600, 3, 1, 2), 3, True, True, inst=True),
    ]
    return specs


def gn_prepare(s):
    r = _rng("gn", sorted((k, str(v)) for k, v in s.items()))
    C, G = s["x"][1], s["G"]
    inp = dict(x=(r.standard_normal(s["x"]) * 2 + 0.25).astype(F32), s=r.uniform(0.5, 2, G).astype(F32),
               b=r.uniform(-1, 1, G).astype(F32))
    if s.get("affine"):
        inp["gamma"], inp["beta"] = r.uniform(0.5, 1.5, C).astype(F32), r.uniform(-0.5, 0.5, C).astype(F32)
    return inp


def gn_launch(rt, ctx, s, inp):
    xd = ctx.to_device(inp["x"], channels_last=s["cl"])
    with gc.switches(RTEN_B200_GROUP_NORM_STREAM=1 if s["stream"] else None):
        if s.get("inst"):
            y = rt.InstanceNormalization(epsilon=1e-5).run(ctx, xd, inp["s"], inp["b"])
        else:
            y = rt.GroupNorm(s["G"], 1e-5, s.get("act", 0)).run(ctx, xd, inp["s"], inp["b"], inp.get("gamma"), inp.get("beta"))
        ctx.sync()
    if s["cl"]:
        assert y.strides[1] == 1, f"{spec_id('gn', s)}: channels-last in must give channels-last out"
    return y.numpy()


def gn_want(s, inp, part=slice(None)):
    import instance_norm_ref as on
    from oracle import activations as A
    x = inp["x"][part]
    if s.get("inst"):
        return on.instance_norm(x, inp["s"], inp["b"], 1e-5)
    return on.group_norm(x, s["G"], inp["s"], inp["b"], inp.get("gamma"), inp.get("beta"), 1e-5,
                         A.silu if s.get("act") == 5 else None)


# ---- Resize -----------------------------------------------------------------------------------------------------------
def resize_geometry(s):
    B, C, H, W = s["x"]
    return B, C, H, W, int(np.floor(H * s["sc"][0])), int(np.floor(W * s["sc"][1]))


def resize_out_strides(s):
    """the output's strides and offset: a channels-last slice of a `cb`-channel buffer from channel `c0`, an NCHW
    buffer with rows padded to `owp`, or None (the allocated output follows the input's layout)"""
    B, C, H, W, OH, OW = resize_geometry(s)
    if "cb" in s:
        return _cl_strides((B, C, OH, OW), s["cb"]), s.get("c0", 0)
    if "owp" in s:
        return (C * OH * s["owp"], OH * s["owp"], s["owp"], 1), 0
    return (_cl_strides((B, C, OH, OW), C) if s["cl"] else gc_contig((B, C, OH, OW))), 0


def gc_contig(shape):
    st, n = [], 1
    for d in reversed(shape):
        st.append(n)
        n *= d
    return tuple(reversed(st))


def resize_rule(s, sms):
    """resize.cu launch_resize: channel stride 1 on both sides, C % 4 == 0 and 16-byte pixels and bases: one thread per
    4 channels of a pixel (resize_cl4_kernel); channel-contiguous outputs otherwise: one element per thread, channel
    fastest; any other layout: 4 consecutive output columns per thread, one float4 store when the output's rows are
    contiguous, its other strides multiples of 4 and its base 16-byte aligned (`vec`), else scalar stores."""
    B, C, H, W, OH, OW = resize_geometry(s)
    lin = int(s["mode"] == "linear")
    os_, off = resize_out_strides(s)
    xs1 = 1 if s["cl"] else H * W
    xpix = C if s["cl"] else 1
    cl4 = xs1 == 1 and os_[1] == 1 and C % 4 == 0 and xpix % 4 == 0 and os_[3] % 4 == 0 and off % 4 == 0
    total = B * C * OH * OW
    if cl4:
        n = total // 4
        return [U("resize_cl4_kernel", (lin,), _loops(n, sms))], {"cl4"} | ({"past the grid"} if n > 256 * 8 * sms else set())
    if os_[1] == 1 and C > 1:
        return [U("resize_kernel", (lin, 0), _loops(total, sms))], {"channel fastest"} | (
            {"past the grid"} if total > 256 * 8 * sms else set())
    vec = os_[3] == 1 and all(v % 4 == 0 for v in os_[:3]) and off % 4 == 0
    n = B * C * OH * _cdiv(OW, 4)
    modes = {"row vec" if vec else "row scalar"} | ({"row partial quad"} if OW % 4 else set())
    if n > 256 * 8 * sms:
        modes.add("past the grid")
    return [U("resize_kernel", (lin, 1), _loops(n, sms) or OW % 4 != 0)], modes


def resize_specs(sms):
    rz = lambda x, sc, mode, cl, **kw: dict(x=x, sc=sc, mode=mode, cl=cl, **kw)  # noqa: E731
    specs = []
    for mode in ("nearest", "linear"):
        specs += [
            rz((2, 8, 7, 9), (2, 2), mode, True), rz((1, 12, 5, 6), (1.5, 2.5), mode, True, coord="align_corners"),
            rz((1, 8, 6, 6), (2, 2), mode, True, cb=12, c0=4),  # a channel slice of a wider buffer: still 16-byte pixels
            rz((2, 3, 7, 9), (2, 2), mode, True), rz((1, 6, 5, 5), (2, 3), mode, True, cb=10, c0=2),
            rz((1, 5, 6, 7), (3, 2), mode, True, coord="asymmetric"),
            rz((2, 3, 8, 8), (2, 2), mode, False), rz((1, 2, 5, 7), (1.5, 1.5), mode, False),  # OW 16, 10 (partial quad)
            rz((1, 3, 5, 7), (2, 1.5), mode, False, owp=12), rz((2, 2, 4, 5), (2, 2), mode, False, owp=12),  # 10: padded rows
            rz((1, 3, 9, 9), (0.5, 0.5), mode, False, coord="pytorch_half_pixel"),
            rz((1, 32, 128, 128), (2, 2), mode, True), rz((1, 8, 256, 256), (2, 2), mode, False),  # past the grid
        ]
    return specs


def resize_prepare(s):
    r = _rng("resize", sorted((k, str(v)) for k, v in s.items()))
    return dict(x=r.uniform(-2, 2, s["x"]).astype(F32))


def _nearest(s):
    return "round_prefer_floor" if s["mode"] == "linear" else s.get("nearest_mode", "round_prefer_ceil")


def resize_launch(rt, ctx, s, inp):
    """(output, the output buffer outside the view or None)"""
    B, C, H, W, OH, OW = resize_geometry(s)
    xd = ctx.to_device(inp["x"], channels_last=s["cl"])
    op = rt.Resize(s["mode"], s.get("coord", "half_pixel"), _nearest(s))
    scales = [1, 1, s["sc"][0], s["sc"][1]]
    if "cb" not in s and "owp" not in s:
        return op.run(ctx, xd, scales=scales).numpy(), None
    os_, off = resize_out_strides(s)
    n = off + 1 + sum((d - 1) * st for d, st in zip((B, C, OH, OW), os_))
    buf = ctx.to_device(np.full(n + 8, np.nan, F32))
    y = op.run(ctx, xd, scales=scales, out=buf.view((B, C, OH, OW), os_, off))
    host = buf.numpy()
    mask = np.ones(host.shape, bool)
    np.lib.stride_tricks.as_strided(mask[off:], (B, C, OH, OW), [st * 1 for st in os_])[...] = False
    return y.numpy(), host[mask]


def resize_want(s, inp):
    from oracle import resize as R
    return R.resize(inp["x"], scales=[1, 1, s["sc"][0], s["sc"][1]], mode=s["mode"], coord_mode=s.get("coord", "half_pixel"),
                    nearest_mode=_nearest(s))


# ---- Concat -----------------------------------------------------------------------------------------------------------
_ES = {"f32": 4, "i32": 4, "i8": 1, "u8": 1}


def concat_rule(s, sms):
    """api_conv.cu rten_b200_concat over contiguous inputs: the dimensions inside the axis merge into it, so each source
    is [outer, ext inner] (start inner in the output); 16-byte units when every ext inner is a multiple of 16 bytes,
    else the element's own size (f32 / i32: 4 bytes, 8-bit: 1); one launch of up to 16 sources, y blocks per source,
    grid-stride x blocks (at most 8 per SM) over the most units any source has."""
    es = _ES[s["dt"]]
    ax = s["axis"]
    inner = int(np.prod(s["shapes"][0][ax + 1:]))
    outer = int(np.prod(s["shapes"][0][:ax]))
    v = 16 // es
    vec = all((sh[ax] * inner) % v == 0 for sh in s["shapes"])
    unit = v if vec else 1
    ns = [outer * sh[ax] * inner // unit for sh in s["shapes"]]
    t = ("uint4",) if vec else ("unsigned int",) if es == 4 else ("unsigned char",)
    most = max(ns)
    partial = any(n % 256 for n in ns) or most > 256 * _grid(most, sms)
    modes = {"16-byte units" if vec else "element units"}
    if len(ns) > 16:
        modes.add("more than 16 sources")
    if most > 256 * 8 * sms:
        modes.add("past the grid")
    return [U("concat_kernel", t, partial)], modes


def concat_specs(sms):
    c = lambda dt, shapes, axis: dict(dt=dt, shapes=tuple(tuple(x) for x in shapes), axis=axis)  # noqa: E731
    return [
        c("f32", [(2, 8, 5, 5), (2, 4, 5, 5)], 1), c("f32", [(6, 10), (2, 10)], 0), c("f32", [(3, 7), (3, 5)], 1),
        c("f32", [(2, 3, 5), (2, 1, 5), (2, 2, 5)], 1),
        c("i32", [(4, 3, 6), (4, 5, 6)], 1), c("i32", [(2, 4, 8), (2, 4, 8)], 2),
        c("i8", [(5, 16), (5, 32)], 1), c("i8", [(5, 7), (5, 9)], 1), c("u8", [(3, 20), (3, 12)], 1),
        c("u8", [(4, 3, 16), (4, 1, 16)], 1),
        c("f32", [(4, 3)] * 20, 1), c("i8", [(2, 16)] * 18, 1), c("u8", [(3, 5)] * 17, 0),
        c("f32", [(2048, 1200), (2048, 400)], 1), c("i32", [(1500, 1001), (1500, 3)], 1),
    ]


def concat_prepare(s):
    r = _rng("concat", sorted((k, str(v)) for k, v in s.items()))
    if s["dt"] == "f32":
        return dict(xs=[r.uniform(-4, 4, sh).astype(F32) for sh in s["shapes"]])
    t = {"i32": I32, "i8": I8, "u8": U8}[s["dt"]]
    info = np.iinfo(t)
    return dict(xs=[r.integers(info.min, int(info.max) + 1, sh).astype(t) for sh in s["shapes"]])


def concat_launch(rt, ctx, s, inp):
    return rt.Concat(s["axis"]).run(ctx, [ctx.to_device(x) for x in inp["xs"]]).numpy()


# ---- ReduceSum / ReduceMean -------------------------------------------------------------------------------------------
def reduce_params(s):
    """api_rows.cu reduce_run's lane description: (L, outputs, vec) -- reduced dimensions of size > 1 merged where dense,
    vec when they form one unit-stride run, the base is 16-byte aligned and every kept stride is a multiple of 4"""
    shape, axes = s["x"], s["axes"]
    strides = s.get("strides") or gc_contig(shape)
    off = s.get("off", 0)
    L, nout, rs, rx, ox = 1, 1, [], [], []
    for i, (d, st) in enumerate(zip(shape, strides)):
        if i in axes:
            L *= d
            if d == 1:
                continue
            if rx and rx[-1] == st * d:
                rs[-1] *= d
                rx[-1] = st
            else:
                rs.append(d)
                rx.append(st)
        else:
            nout *= d
            if d > 1:
                ox.append(st)
    vec = (not rx or (len(rx) == 1 and rx[0] == 1)) and off % 4 == 0 and all(v % 4 == 0 for v in ox)
    return L, nout, vec


def reduce_rule(s, sms):
    """reduce.cu launch_typed: lanes of up to 1024 elements one warp per output (8 per CTA, at most 8 CTAs per SM, a
    grid-stride loop over the rest), longer lanes one CTA per output (at most 8 per SM); VEC: the lane read as 16-byte
    vectors"""
    L, nout, vec = reduce_params(s)
    t = "float" if s["dt"] == "f32" else "int"
    modes = {"vec" if vec else "misaligned" if s.get("off", 0) % 4 else "scalar"}
    if s.get("mean"):
        modes.add("ReduceMean")
    if L <= 1024:
        grid = min(8 * sms, _cdiv(nout, 8))
        modes.add("warp")
        if nout > 8 * grid:
            modes.add("warp past the grid")
        return [U("reduce_sum_warp_kernel", (t, int(vec)), nout % 8 != 0 or nout > 8 * grid or L % 64 != 0)], modes
    grid = min(8 * sms, nout)
    modes.add("CTA")
    if nout > grid:
        modes.add("CTA past the grid")
    return [U("reduce_sum_cta_kernel", (t, int(vec)), L % 4096 != 0 or L % 64 != 0 or nout > grid)], modes


def reduce_specs(sms):
    rd = lambda dt, x, axes, **kw: dict(dt=dt, x=x, axes=tuple(axes), **kw)  # noqa: E731
    warp_many, cta_many = 8 * sms * 8 + 500, 8 * sms + 50
    specs = []
    for dt in ("f32", "i32"):
        m = dict(mean=True) if dt == "f32" else {}
        specs += [
            rd(dt, (64, 300), [1]), rd(dt, (50, 77), [1], **m), rd(dt, (30, 64), [0]), rd(dt, (4, 6, 50), [0, 2], **m),
            rd(dt, (16, 200), [1], strides=(200, 1), off=1),  # misaligned: 4 bytes past a 16-byte boundary
            rd(dt, (12, 5000), [1], **m), rd(dt, (8, 4097), [1]), rd(dt, (3000, 6), [0], **m), rd(dt, (2, 70, 70), [1, 2]),
            rd(dt, (6, 4100), [1], strides=(4100, 1), off=2),
            rd(dt, (warp_many, 40), [1], **m), rd(dt, (warp_many, 33), [1]),
            rd(dt, (cta_many, 1500), [1], **m), rd(dt, (cta_many, 1030), [1]),
        ]
    return specs


def reduce_prepare(s):
    r = _rng("reduce", sorted((k, str(v)) for k, v in s.items()))
    shape = s["x"]
    n = s.get("off", 0) + int(np.prod(shape))
    buf = r.uniform(-3, 3, n).astype(F32) if s["dt"] == "f32" else r.integers(-2 ** 31, 2 ** 31, n, dtype=np.int64).astype(I32)
    return dict(buf=buf)


def _reduce_x(s, inp):
    off = s.get("off", 0)
    return inp["buf"][off:].reshape(s["x"])


def reduce_launch(rt, ctx, s, inp):
    op = (rt.ReduceMean if s.get("mean") else rt.ReduceSum)(axes=list(s["axes"]))
    off = s.get("off", 0)
    d = ctx.to_device(inp["buf"])
    xd = d.view(s["x"], gc_contig(s["x"]), off) if off else d.view(s["x"], gc_contig(s["x"]))
    return op.run(ctx, xd).numpy()


def reduce_want(s, x):
    import genai_decoder as gd
    axes = list(s["axes"])
    if s["dt"] == "i32":
        t = np.sum(x.astype(np.int64), axis=tuple(axes), keepdims=True)
        return ((t + 2 ** 31) % 2 ** 32 - 2 ** 31).astype(I32)
    y = gd.reduce_sum_ref(x, axes)
    if s.get("mean"):
        L = int(np.prod([x.shape[a] for a in axes]))
        y = (y / F32(L)).astype(F32)
    return y


# ---- rotary embedding -------------------------------------------------------------------------------------------------
def rotary_rule(s, sms):
    """rotary.cu launch_rotary: one warp per row (8 per CTA) of Q, the new K and V, and the built cache positions; lanes
    stride over the row's D elements.  MultiHeadAttention's prep (bias adds, no rotation) is rotary_mha_kernel."""
    if s["op"] == "rope":
        B, H, S, D = s["bhsd"]
        rows = B * H * S
        modes = {"RotaryEmbedding"} | ({"interleaved"} if s["inter"] else set()) | ({"position ids"} if s.get("pos") else set())
        return [U("rotary_kernel", (), rows % 8 != 0 or D % 32 != 0)], modes
    if s["op"] == "gqa":
        B, S, H, Hkv, D = s["dims"]
        rows = B * S * H + 2 * B * S * Hkv  # Q, new K and V; the prompt fills the whole cache
        return [U("rotary_kernel", (), rows % 8 != 0 or D % 32 != 0)], {"GroupQueryAttention"} | (
            {"interleaved"} if s["inter"] else set())
    B, S, H, D = s["dims"]
    rows = 3 * B * S * H
    return [U("rotary_mha_kernel", (), rows % 8 != 0 or D % 32 != 0)], {"MultiHeadAttention"}


def rotary_specs(sms):
    return [
        dict(op="rope", bhsd=(2, 3, 5, 16), inter=False, form="bhsd"), dict(op="rope", bhsd=(1, 4, 7, 64), inter=True, form="bhsd"),
        dict(op="rope", bhsd=(2, 2, 9, 48), inter=False, form="bsh"), dict(op="rope", bhsd=(3, 2, 6, 32), inter=True, form="bsh"),
        dict(op="rope", bhsd=(2, 3, 5, 40), inter=False, form="bhsd", pos=True),
        dict(op="rope", bhsd=(1, 2, 11, 64), inter=True, form="bsh", pos=True),
        dict(op="gqa", dims=(2, 5, 4, 2, 64), inter=False), dict(op="gqa", dims=(1, 7, 6, 2, 64), inter=True),
        dict(op="mha", dims=(2, 5, 3, 64)), dict(op="mha", dims=(1, 8, 2, 64)),
    ]


def rotary_prepare(s):
    r = _rng("rotary", sorted((k, str(v)) for k, v in s.items()))
    if s["op"] == "rope":
        B, H, S, D = s["bhsd"]
        inp = dict(x=r.uniform(-2, 2, (B, H, S, D)).astype(F32))
        if s.get("pos"):
            inp["cos"], inp["sin"] = r.uniform(-1, 1, (32, D // 2)).astype(F32), r.uniform(-1, 1, (32, D // 2)).astype(F32)
            inp["pos"] = r.integers(0, 32, (B, S)).astype(I32)
        else:
            inp["cos"], inp["sin"] = r.uniform(-1, 1, (B, S, D // 2)).astype(F32), r.uniform(-1, 1, (B, S, D // 2)).astype(F32)
        return inp
    if s["op"] == "gqa":
        B, S, H, Hkv, D = s["dims"]
        return dict(q=r.uniform(-1, 1, (B, S, H * D)).astype(F32), k=r.uniform(-1, 1, (B, S, Hkv * D)).astype(F32),
                    v=r.uniform(-1, 1, (B, S, Hkv * D)).astype(F32), cos=r.uniform(-1, 1, (S + 3, D // 2)).astype(F32),
                    sin=r.uniform(-1, 1, (S + 3, D // 2)).astype(F32))
    B, S, H, D = s["dims"]
    return dict(q=r.uniform(-1, 1, (B, S, H * D)).astype(F32), k=r.uniform(-1, 1, (B, S, H * D)).astype(F32),
                v=r.uniform(-1, 1, (B, S, H * D)).astype(F32), bias=r.uniform(-1, 1, 3 * H * D).astype(F32))


def rotary_launch(rt, ctx, s, inp):
    if s["op"] == "rope":
        B, H, S, D = s["bhsd"]
        x = inp["x"] if s["form"] == "bhsd" else inp["x"].transpose(0, 2, 1, 3).reshape(B, S, H * D)
        op = rt.RotaryEmbedding(interleaved=s["inter"], num_heads=0 if s["form"] == "bhsd" else H)
        y = op.run(ctx, ctx.to_device(np.ascontiguousarray(x)), inp["cos"], inp["sin"], inp.get("pos"))
        return (y.numpy(),)
    if s["op"] == "gqa":
        B, S, H, Hkv, D = s["dims"]
        op = rt.GroupQueryAttention(H, Hkv, do_rotary=True, rotary_interleaved=s["inter"])
        _, pk, pv = op.run(ctx, inp["q"], inp["k"], inp["v"], np.full(B, S - 1, I32), S,
                           cos_cache=inp["cos"], sin_cache=inp["sin"])
        return pk.numpy(), pv.numpy()
    B, S, H, D = s["dims"]
    _, pk, pv = rt.MultiHeadAttention(H).run(ctx, inp["q"], inp["k"], inp["v"], bias=inp["bias"])
    return pk.numpy(), pv.numpy()


def rotary_want(s, inp):
    from test_gpu_group_query_attention import rotary_ref
    if s["op"] == "rope":
        B, H, S, D = s["bhsd"]
        c, sn = (inp["cos"][inp["pos"]], inp["sin"][inp["pos"]]) if s.get("pos") else (inp["cos"], inp["sin"])
        y = rotary_ref(inp["x"], c[:, None], sn[:, None], s["inter"], dtype=F32)
        return (y if s["form"] == "bhsd" else y.transpose(0, 2, 1, 3).reshape(B, S, H * D),)
    if s["op"] == "gqa":
        B, S, H, Hkv, D = s["dims"]
        k = inp["k"].reshape(B, S, Hkv, D).transpose(0, 2, 1, 3)
        v = inp["v"].reshape(B, S, Hkv, D).transpose(0, 2, 1, 3)
        return rotary_ref(k, inp["cos"][None, None, :S], inp["sin"][None, None, :S], s["inter"], dtype=F32), v
    B, S, H, D = s["dims"]
    hd = H * D
    k = (inp["k"] + inp["bias"][hd:2 * hd]).astype(F32).reshape(B, S, H, D).transpose(0, 2, 1, 3)
    v = (inp["v"] + inp["bias"][2 * hd:]).astype(F32).reshape(B, S, H, D).transpose(0, 2, 1, 3)
    return k, v


# ---- the case families ------------------------------------------------------------------------------------------------
RULES = {"dw": dw_rule, "gn": gn_rule, "resize": resize_rule, "concat": concat_rule, "reduce": reduce_rule, "rotary": rotary_rule}
SPECS = {"dw": dw_specs, "gn": gn_specs, "resize": resize_specs, "concat": concat_specs, "reduce": reduce_specs,
         "rotary": rotary_specs}
PREPARE = {"dw": dw_prepare, "gn": gn_prepare, "resize": resize_prepare, "concat": concat_prepare, "reduce": reduce_prepare,
           "rotary": rotary_prepare}
LAUNCH = {"dw": dw_launch, "gn": gn_launch, "resize": resize_launch, "concat": concat_launch, "reduce": reduce_launch,
          "rotary": rotary_launch}
def spec_id(fam, s):
    return fam + " " + " ".join(f"{k}={v}" for k, v in s.items())


def _rng(*key):
    return rk._rng("conv_norm_resize", *key)


def coverage_gaps(sms):
    """instances that fewer than two cases select or none with a partial last unit, and runtime modes no case reaches"""
    picked, part, modes = {}, set(), set()
    for fam, specs in SPECS.items():
        for s in specs(sms):
            units, ms = RULES[fam](s, sms)
            for k, a, p in units:
                assert a in VARIANTS[k], f"{spec_id(fam, s)}: the rule names {(k, a)}, which the table lacks"
                assert k in FAMILY_KERNELS[fam], f"{spec_id(fam, s)}: {k} is not a kernel of the family"
                picked[(k, a)] = picked.get((k, a), 0) + 1
                if p:
                    part.add((k, a))
            modes |= {(fam, m) for m in ms}
    inst = [(k, a) for k, args in VARIANTS.items() for a in args]
    gaps = [("selected fewer than twice", u) for u in inst if picked.get(u, 0) < 2]
    gaps += [("never with a partial last unit", u) for u in inst if u not in part]
    return gaps + [("mode never reached", (fam, m)) for fam, ms in MODES.items() for m in ms if (fam, m) not in modes]


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
    out = rk.probe_in_child("test_gpu_conv_norm_resize_kernels")
    n_sms, names = out["sms"], out["names"]
    seen, wrong = {}, []
    for fam, specs in SPECS.items():
        for s in specs(n_sms):
            sid = spec_id(fam, s)
            want = {(k, a) for k, a, _ in RULES[fam](s, n_sms)[0]}
            ran = {kernel_key(n) for n in names[sid]} - {None}
            if ran != want:
                wrong.append((sid, sorted(want), sorted(ran)))
            for u in want & ran:
                seen[u] = seen.get(u, 0) + 1
    assert not wrong, f"{len(wrong)} cases ran other kernels than the rule names: {wrong[:8]}"
    missing = [(k, a) for k, args in VARIANTS.items() for a in args if seen.get((k, a), 0) < 2]
    assert not missing, f"instances that fewer than two cases ran: {missing}"
    assert not coverage_gaps(n_sms)
    total = sum(len(v) for v in VARIANTS.values())
    print(f"{total} of {total} instances ran, each at least twice, on {n_sms} SMs; {len(names)} captures, "
          f"{out['retaken']} taken again")


# ---- numbers ----------------------------------------------------------------------------------------------------------
def test_depthwise_bit_exact(rt, sms):
    ctx = rt.Context(0)
    for s in dw_specs(sms):
        inp = dw_prepare(s)
        got, outside = dw_launch(rt, ctx, s, inp)
        want = dw_want(s, inp)
        what = spec_id("dw", s)
        gc.assert_bit_exact(got, want, what)
        if outside is not None:
            fill = -7 if s["out"] == "i32" else np.nan
            assert (np.isnan(outside) if s["out"] != "i32" else outside == fill).all(), f"{what}: writes outside the slice"
        if s["out"] == "qf32":
            r = np.asarray(inp["range"].numpy(), I32).reshape(-1)
            lo, hi = np.where(r >= 0, r, r ^ np.int32(0x7FFFFFFF)).astype(I32).view(F32)
            assert lo == want.min() and hi == want.max(), f"{what}: range ({lo}, {hi}) != ({want.min()}, {want.max()})"


def test_group_norm_bit_exact(rt, sms):
    ctx = rt.Context(0)
    for s in gn_specs(sms):
        inp = gn_prepare(s)
        got = gn_launch(rt, ctx, s, inp)
        what = spec_id("gn", s)
        N = s["x"][0]
        if s.get("inst") and (N > 65535 or s["x"][1] > 65535):  # the head and the tail of the grid loop
            if N > 65535:
                for part in (slice(0, 64), slice(N - 64, N)):
                    gc.assert_bit_exact(got[part], gn_want(s, inp, part), what)
            else:
                x = inp["x"]
                C = s["x"][1]
                for cs in (slice(0, 64), slice(C - 64, C)):
                    sub = dict(inp, x=x[:, cs], s=inp["s"][cs], b=inp["b"][cs])
                    gc.assert_bit_exact(got[:, cs], gn_want(s, sub), what)
            continue
        gc.assert_bit_exact(got, gn_want(s, inp), what)


def test_resize_bit_exact(rt, sms):
    ctx = rt.Context(0)
    for s in resize_specs(sms):
        inp = resize_prepare(s)
        got, outside = resize_launch(rt, ctx, s, inp)
        gc.assert_bit_exact(got, resize_want(s, inp), spec_id("resize", s))
        if outside is not None:
            assert np.isnan(outside).all(), f"{spec_id('resize', s)}: writes outside the output view"


def test_concat_bit_exact(rt, sms):
    from oracle import resize as R
    ctx = rt.Context(0)
    for s in concat_specs(sms):
        inp = concat_prepare(s)
        got = concat_launch(rt, ctx, s, inp)
        want = R.concat(inp["xs"], s["axis"])
        assert got.dtype == want.dtype and got.shape == want.shape, spec_id("concat", s)
        assert np.array_equal(got.view(np.uint8), np.ascontiguousarray(want).view(np.uint8)), spec_id("concat", s)


def test_reduce_sum_bit_exact(rt, sms):
    ctx = rt.Context(0)
    for s in reduce_specs(sms):
        inp = reduce_prepare(s)
        got = reduce_launch(rt, ctx, s, inp)
        x = _reduce_x(s, inp)
        what = spec_id("reduce", s)
        if s["x"][0] > 1000 and s["axes"] == (1,):  # the head and the tail of the grid loop
            for part in (slice(0, 64), slice(s["x"][0] - 64, s["x"][0])):
                gc.assert_bit_exact(got[part], reduce_want(s, x[part]), what)
            continue
        gc.assert_bit_exact(got, reduce_want(s, x), what)


def test_rotary_bit_exact(rt, sms):
    ctx = rt.Context(0)
    for s in rotary_specs(sms):
        inp = rotary_prepare(s)
        for i, (g, w) in enumerate(zip(rotary_launch(rt, ctx, s, inp), rotary_want(s, inp))):
            gc.assert_bit_exact(g, np.asarray(w, F32), f"{spec_id('rotary', s)} output {i}")
