"""`pytest -m gpu`: every pooling, GlobalAveragePool, broadcast Add / Mul / Sub and row gather / scatter kernel of
rowops.cu, each selected by name and checked bit for bit; and the executor's MaxPool / AveragePool ceil_mode and
auto_pad, which load as the reference reads them.

The launchers (launch_maxpool / launch_avgpool, launch_row_mean, launch_binary, launch_gather_rows /
launch_scatter_rows, behind the entry points of api_conv.cu and api_rows.cu) pick a kernel at run
time from the operands' strides, the channel count and pointer alignment.  The rules are restated below (`*_rule`);
`VARIANTS` lists every kernel they pick from (tests/test_glue_kernel_table_cpu.py keeps it equal to the built library's
symbols).  Some kernels also take a runtime mode the name does not show: the thread mapping of maxpool_kernel /
avgpool_kernel (`channels_fastest`, from the output's layout) and the operation (Add, Sub or Mul) of the three
broadcast-arithmetic kernels.  The case lists reach every (kernel, mode) at least twice, one of them with a partial last
unit (a block with idle threads or rows, or a scalar tail).

  * kernel identity: every case runs once under CUPTI in a child process; the kernel that ran must be the one the rule
    names, and every kernel of `VARIANTS` must have run;
  * MaxPool: bit-exact against the oracle (a fold from -inf with `v > m ? v : m`) on ResNet's stem, YOLO's SPPF and
    U-Net's pools, channels-last with C % 4 != 0, channel-sliced, spatially strided and misaligned inputs, asymmetric
    pads, windows entirely in the padding, NaN / +-inf / +-0 inputs;
  * AveragePool: the kernel each layout selects, and windows that reach into the end padding, as the executor pads a
    ceil-mode pool;
  * GlobalAveragePool: bit-exact against the oracle's Sum order over lengths that stop at every stage of the
    reference's fold, four layouts and row counts that leave idle lanes, with +-inf, inf - inf and NaN rows;
  * Add / Mul / Sub: exactly the correctly rounded f32 result (float64, rounded once), on dense operands with every
    n % 4, a misaligned operand, bias rows, position tables, two-sided broadcasts, channels-last operands, strided and
    in-place outputs, signed zeros, inf - inf and NaN; f32 Sub and i32 on the same kernels, i32 wrapping mod 2^32;
  * Gather / Scatter: both gather kernels with column-sliced, misaligned and row-padded tables, negative indices,
    3-D and empty index tensors; scatter into a strided table from strided updates.  Indices stay in range: the gather
    kernels do not bounds-check (the reference returns an error), so an out-of-range index is a contract for the
    caller to keep, not a case to run.

The executor's pools (rten_b200/csrc/model.cu fill_pool_attrs) are run from small ONNX graphs: ceil_mode, auto_pad
SAME_UPPER / VALID, the refused SAME_LOWER and a read Indices output.  Their output shapes are checked against
`pool_out_size`, a restatement of the reference's output_size_and_padding_for_axis (src/ops/pooling.rs), and their
values against the oracle pools given the explicit pads that produce that shape."""
import numpy as np
import pytest

import gpu_checks as gc
import test_gpu_row_kernels as rk

pytestmark = pytest.mark.gpu

F32, I32 = np.float32, np.int32

# ---- the kernels, and the launchers' selection rules ------------------------------------------------------------------
BIN_TYPES = [("float",), ("int",)]  # <T>: the operation is a runtime argument
VARIANTS = {
    "maxpool_cl4_kernel": [()], "maxpool_kernel": [()], "avgpool_cl4_kernel": [()], "avgpool_kernel": [()],
    "row_mean_kernel": [()], "row_mean_thread_kernel": [()],
    "binary_flat_kernel": BIN_TYPES, "binary_periodic_kernel": BIN_TYPES, "binary_nd_kernel": BIN_TYPES,
    "gather_rows_kernel": [()], "gather_rows_vec_kernel": [()], "scatter_rows_kernel": [()],
}
# the runtime modes a kernel's name does not show: each (kernel, mode) is a unit of coverage
MODES = {"maxpool_kernel": ("rows fastest", "channels fastest"), "avgpool_kernel": ("rows fastest", "channels fastest"),
         "binary_flat_kernel": ("Add", "Sub", "Mul"), "binary_periodic_kernel": ("Add", "Sub", "Mul"),
         "binary_nd_kernel": ("Add", "Sub", "Mul")}
FAMILY_KERNELS = {"pool": ("maxpool_cl4_kernel", "maxpool_kernel", "avgpool_cl4_kernel", "avgpool_kernel"),
                  "gap": ("row_mean_kernel", "row_mean_thread_kernel"),
                  "binary": ("binary_flat_kernel", "binary_periodic_kernel", "binary_nd_kernel"),
                  "gather": ("gather_rows_kernel", "gather_rows_vec_kernel", "scatter_rows_kernel")}
KERNELS = set(VARIANTS)
BLOCK = 256  # threads per block of the elementwise launches (ew_grid)


def _contig(shape):
    st, s = [], 1
    for d in reversed(shape):
        st.append(s)
        s *= d
    return tuple(reversed(st))


def _dense(shape, strides):
    """the view covers its span exactly (no gaps, no overlap)"""
    n = int(np.prod(shape))
    span = 1 + sum((d - 1) * s for d, s in zip(shape, strides)) if n else 0
    return span == n and all(s > 0 or d == 1 for d, s in zip(shape, strides))


# 4-D layouts of an NCHW tensor: (strides, offset in floats) of the view a test hands the entry point
def layout4(shape, name):
    B, C, H, W = shape
    if name == "nchw":
        return _contig(shape), 0
    if name == "cl":
        return (H * W * C, 1, W * C, C), 0
    if name == "cl_off1":  # channels-last, 4 bytes past a 16-byte boundary
        return (H * W * C, 1, W * C, C), 1
    if name == "cslice_nchw":  # channels 2 .. 2 + C of a (B, C + 5, H, W) tensor
        return ((C + 5) * H * W, H * W, W, 1), 2 * H * W
    if name == "cslice_cl":  # channels 4 .. 4 + C of a channels-last (B, C + 8, H, W) tensor
        return (H * W * (C + 8), 1, W * (C + 8), C + 8), 4
    if name == "sstride_nchw":  # x[:, :, ::2, ::2] of a (B, C, 2H, 2W) tensor
        return (C * 4 * H * W, 4 * H * W, 4 * W, 2), 0
    if name == "sstride_cl":  # the same of a channels-last tensor
        return (4 * H * W * C, 1, 4 * W * C, 2 * C), 0
    if name == "wcrop_nchw":  # x[..., :W] of a (B, C, H, W + 3) tensor: (h, w) strides that are not one stride
        return (C * H * (W + 3), H * (W + 3), W + 3, 1), 0
    if name == "wcrop_cl":  # the same of a channels-last tensor
        return (H * (W + 2) * C, 1, (W + 2) * C, C), 0
    raise ValueError(name)


def placed(ctx, arr, strides, off=0, fill=np.nan, guard=0):
    """`arr` on the device as the view (strides, off) of a buffer whose other elements hold `fill`, with `guard` more
    of them after the view's span"""
    arr = np.asarray(arr)
    span = 1 + sum((d - 1) * s for d, s in zip(arr.shape, strides)) if arr.size else 0
    host = np.full(off + max(span, 1) + guard, fill, arr.dtype)
    np.lib.stride_tricks.as_strided(host[off:], arr.shape, [s * arr.itemsize for s in strides])[...] = arr
    return ctx.to_device(host).view(arr.shape, strides, off)


def pool_rule(s):
    """launch_maxpool / launch_avgpool: the channels-last kernel (one thread per pixel and 4 channels) when input and
    output are channels-last, C % 4 == 0, every other stride a multiple of 4 and both bases 16-byte aligned; else the
    generic kernel, its thread mapping channels-fastest when the output is (pool2d allocates it in the input's layout)."""
    B, C, H, W = s["shape"]
    xs, off = layout4(s["shape"], s["layout"])
    oh, ow = pool_windows(s)
    cl = xs[1] == 1 and C > 1  # layout_like
    ys = (C * oh * ow, 1, ow * C, C) if cl else (C * oh * ow, oh * ow, ow, 1)
    base = "maxpool" if s["op"] == "max" else "avgpool"
    if (xs[1] == 1 and ys[1] == 1 and C % 4 == 0 and all(v % 4 == 0 for v in (xs[0], xs[2], xs[3], ys[0], ys[2], ys[3]))
            and off % 4 == 0):
        return (base + "_cl4_kernel", ()), None
    return (base + "_kernel", ()), "channels fastest" if ys[1] == 1 else "rows fastest"


def gap_rule(s):
    """launch_row_mean (after rten_b200_global_average_pool copies an input whose (h, w) strides are not one stride
    to a contiguous tensor): one thread per row when rows are adjacent (s_inner == 1) and a row's elements are not
    (kstride != 1) -- channels-last; else one warp per row."""
    B, C, H, W = s["shape"]
    xs, _ = layout4(s["shape"], s["layout"])
    if xs[2] != W * xs[3]:
        xs = _contig(s["shape"])
    return ("row_mean_thread_kernel" if xs[1] == 1 and xs[3] != 1 else "row_mean_kernel", ()), None


def _aligned(off):
    return off % 4 == 0


def binary_layouts(s):
    """(shape, strides, offset) of a, b and the output; the output's as binary_op allocates it unless given"""
    a, b = s["a"], s["b"]
    nd = max(len(a[0]), len(b[0]))
    same = len(a[0]) == len(b[0]) and _dense(a[0], a[1]) and all(
        x == y and (x == 1 or sa == sb) for x, y, sa, sb in zip(a[0], b[0], a[1], b[1]))
    shape = tuple(max(x, y) for x, y in zip((1,) * (nd - len(a[0])) + tuple(a[0]), (1,) * (nd - len(b[0])) + tuple(b[0])))
    out = s.get("out")
    if out == "a":
        out = a
    elif out is None:
        out = (shape, tuple(a[1]) if same else _contig(shape), 0)
    return a, b, out, same, shape


def _binary_aligned(s):
    a, b, out, _, _ = binary_layouts(s)
    return _aligned(a[2]) and _aligned(b[2]) and _aligned(out[2])


def binary_rule(s):
    """binary_op hands launch_binary dense operands and output of one layout as one [n] view with unit strides, anything
    else with its broadcast strides.  For every type and operation, launch_binary runs the flat kernel when a, b and the
    output are dense row-major over the iteration space; the periodic kernel when a and the output are and b is a dense
    block of the trailing dims repeated over the leading ones, whose length (the period) is a multiple of 4, with
    16-byte aligned bases; else the strided kernel."""
    a, b, out, same, shape = binary_layouts(s)
    t = ("float",) if s["dtype"] == "f32" else ("int",)
    if same and all(d == 1 or so == sa for d, so, sa in zip(shape, out[1], a[1])):
        return ("binary_flat_kernel", t), s["op"]
    nd = len(shape)

    def bstrides(v):  # binary_op's broadcast strides: 0 over a missing or size-1 dim
        return [0] * (nd - len(v[0])) + [st if d != 1 else 0 for d, st in zip(v[0], v[1])]
    sa, sb = bstrides(a), bstrides(b)
    n, period, dense, bcast = 1, 0, True, False
    for i in range(nd - 1, -1, -1):
        if shape[i] != 1:
            dense = dense and sa[i] == n and out[1][i] == n
            if not bcast and sb[i] == n:
                pass
            elif sb[i] == 0:
                if not bcast:
                    period = n
                bcast = True
            else:
                dense = False
        n *= shape[i]
    if dense and not bcast:
        return ("binary_flat_kernel", t), s["op"]
    if dense and period % 4 == 0 and n < 2 ** 31 - 1 and _binary_aligned(s):
        return ("binary_periodic_kernel", t), s["op"]
    return ("binary_nd_kernel", t), s["op"]


def gather_rule(s):
    """launch_gather_rows: one float4 per thread when the table's columns are adjacent, the width and the row stride
    are multiples of 4 and the table is 16-byte aligned; else one element per thread.  Scatter: one kernel.  No launch
    at all for an empty index tensor."""
    nidx = int(np.prod(s["idx"]))
    width = s["table"][1]
    if nidx * width == 0:
        return None, None
    if s["kind"] == "scatter":
        return ("scatter_rows_kernel", ()), None
    ts, off = table_layout(s)
    vec = ts[1] == 1 and width % 4 == 0 and ts[0] % 4 == 0 and nidx * width < 2 ** 31 - 1 and off % 4 == 0
    return ("gather_rows_vec_kernel" if vec else "gather_rows_kernel", ()), None


# ---- the reference's pool output size ---------------------------------------------------------------------------------
def pool_out_size(n, k, s, ps, pe, ceil=False, same=False):
    """(output size, start pad, end pad) along one axis: src/ops/pooling.rs output_size_and_padding_for_axis, dilation
    1.  SAME (auto_pad SAME_UPPER / SAME_LOWER): ceil(n / s) windows, the odd unit of padding at the end.  Fixed pads:
    floor or ceil of the window count; in ceil mode a last window that would start inside the end padding is dropped."""
    if same:
        out = -(-n // s)
        total = max((out - 1) * s + k - n, 0)
        return out, total // 2, -(-total // 2)
    if n + ps + pe < k:
        raise ValueError("Input too small for kernel size")
    windows = n + ps + pe - k
    out = (-(-windows // s) if ceil else windows // s) + 1
    if ceil and (out - 1) * s >= n + ps:
        out -= 1
    return out, ps, pe


def pool_windows(s):
    B, C, H, W = s["shape"]
    (kh, kw), (t, l, b, r), (sy, sx) = s["k"], s["pads"], s["strides"]
    return pool_out_size(H, kh, sy, t, b)[0], pool_out_size(W, kw, sx, l, r)[0]


# ---- case lists -------------------------------------------------------------------------------------------------------
def pool_specs(sms):
    stem = dict(shape=(1, 64, 112, 112), k=(3, 3), pads=(1, 1, 1, 1), strides=(2, 2))
    sppf = dict(shape=(1, 32, 20, 20), k=(5, 5), pads=(2, 2, 2, 2), strides=(1, 1))
    unet = dict(shape=(2, 16, 24, 24), k=(2, 2), pads=(0, 0, 0, 0), strides=(2, 2))
    odd = dict(shape=(2, 6, 13, 11), k=(3, 3), pads=(1, 1, 1, 1), strides=(2, 2))
    k3s2 = lambda C, H, W, pads=(1, 1, 1, 1): dict(shape=(2, C, H, W), k=(3, 3), pads=pads, strides=(2, 2))  # noqa: E731
    specs = [dict(op="max", layout="cl", values="rand", **stem), dict(op="max", layout="nchw", values="rand", **stem),
             dict(op="max", layout="cl", values="rand", **sppf), dict(op="max", layout="nchw", values="rand", **sppf),
             dict(op="max", layout="nchw", values="rand", **unet), dict(op="max", layout="cl", values="rand", **unet),
             # channels-last, C % 4 != 0: the generic kernel, channels fastest
             dict(op="max", layout="cl", values="rand", **odd), dict(op="max", layout="cl", values="rand", **k3s2(3, 17, 17)),
             dict(op="max", layout="cl_off1", values="rand", **k3s2(8, 15, 15)),  # misaligned: the generic kernel
             dict(op="max", layout="cslice_cl", values="rand", **k3s2(8, 14, 15)),
             dict(op="max", layout="cslice_nchw", values="rand", **k3s2(5, 14, 15)),
             dict(op="max", layout="sstride_cl", values="rand", **k3s2(12, 9, 10)),
             dict(op="max", layout="sstride_nchw", values="rand", **k3s2(5, 9, 10)),
             # asymmetric pads; pads >= the kernel (a window entirely in the padding: -inf)
             dict(op="max", layout="nchw", values="rand", **k3s2(4, 12, 13, (0, 1, 2, 0))),
             dict(op="max", layout="cl", values="rand", **k3s2(4, 12, 13, (2, 0, 1, 2))),
             dict(op="max", layout="nchw", values="rand", shape=(1, 3, 5, 6), k=(2, 2), pads=(2, 3, 2, 2), strides=(1, 2)),
             dict(op="max", layout="cl", values="rand", shape=(1, 8, 5, 6), k=(2, 3), pads=(3, 2, 2, 3), strides=(2, 1)),
             # NaN, +-inf, +-0 on both mappings and the channels-last kernel
             dict(op="max", layout="cl", values="special", **k3s2(8, 11, 12)),
             dict(op="max", layout="nchw", values="special", **k3s2(5, 11, 12)),
             dict(op="max", layout="cl", values="special", shape=(2, 5, 6, 7), k=(2, 2), pads=(0, 0, 0, 0), strides=(1, 1)),
             dict(op="max", layout="nchw", values="zeros", shape=(1, 4, 6, 6), k=(2, 2), pads=(0, 0, 0, 0), strides=(2, 2)),
             dict(op="max", layout="cl", values="zeros", shape=(1, 8, 6, 6), k=(3, 3), pads=(1, 1, 1, 1), strides=(2, 2))]
    # AveragePool: each kernel and mapping twice, and windows that run past the end padding (the ceil-mode windows)
    for cip in (False, True):
        specs += [dict(op="avg", layout="cl", values="rand", cip=cip, **k3s2(8, 14, 14)),
                  dict(op="avg", layout="nchw", values="rand", cip=cip, **k3s2(5, 14, 14, (1, 1, 2, 2))),
                  dict(op="avg", layout="cl", values="rand", cip=cip, **k3s2(6, 13, 12, (0, 0, 2, 1))),
                  dict(op="avg", layout="cslice_cl", values="rand", cip=cip, shape=(1, 8, 12, 12), k=(3, 3), pads=(0, 0, 1, 1),
                       strides=(2, 2))]
    return specs


GAP_LENGTHS = {1: (1, 1), 15: (3, 5), 16: (4, 4), 17: (1, 17), 49: (7, 7), 63: (7, 9), 64: (8, 8), 65: (5, 13), 80: (8, 10),
               100: (10, 10), 143: (11, 13), 196: (14, 14), 784: (28, 28), 3136: (56, 56), 12544: (112, 112)}


def gap_specs(sms):
    """Every length: one row, NCHW; B * C = 26 (not a multiple of 8), channels-last; B * C = 150 (not a multiple of 8
    or 128), NCHW with special rows.  The lengths up to 3136 also: a channel slice of each layout and a view whose
    (h, w) strides are not one stride, channels-last then NCHW, with special rows; 12544 keeps to NCHW and one
    channels-last case."""
    specs = []
    for n, (H, W) in GAP_LENGTHS.items():
        specs += [dict(layout="nchw", shape=(1, 1, H, W), special=False),
                  dict(layout="cl", shape=(2, 13, H, W), special=n != 12544),
                  dict(layout="nchw", shape=(2, 75, H, W), special=True)]
        if n <= 3136:
            specs += [dict(layout="cslice_nchw", shape=(2, 13, H, W), special=True),
                      dict(layout="cslice_cl", shape=(3, 50, H, W), special=True),
                      dict(layout="wcrop_cl", shape=(2, 13, H, W), special=True),
                      dict(layout="wcrop_nchw", shape=(1, 9, H, W), special=False)]
    return specs


def binary_specs(sms):
    L = lambda shape, strides=None, off=0: (tuple(shape), tuple(strides or _contig(shape)), off)  # noqa: E731
    big = 8 * sms * BLOCK * 4 + 4 * 37 + 3  # more float4s than the capped grid has threads: a second grid-stride pass
    specs = []
    for op in ("Add", "Mul"):
        f = dict(op=op, dtype="f32")
        specs += [dict(f, kind="dense", a=L((n,)), b=L((n,))) for n in (1024, 1025, 1026, 1027)]
        specs += [dict(f, kind="dense", a=L((big,)), b=L((big,))),
                  dict(f, kind="dense", a=L((2, 3, 4, 5)), b=L((2, 3, 4, 5))),
                  dict(f, kind="misaligned a", a=L((4, 257), off=1), b=L((4, 257))),
                  dict(f, kind="misaligned a", a=L((2, 64, 32), off=1), b=L((32,))),
                  dict(f, kind="bias", a=L((2, 7, 768)), b=L((768,))),
                  dict(f, kind="bias", a=L((3, 5, 100)), b=L((100,))),
                  dict(f, kind="bias", a=L((3, 5, 30)), b=L((30,))),  # C % 4 != 0: strided
                  dict(f, kind="bias", a=L((big // 1024 + 1, 1024)), b=L((1024,))),
                  dict(f, kind="position", a=L((2, 9, 64)), b=L((9, 64))),
                  dict(f, kind="position", a=L((3, 5, 6)), b=L((5, 6))),  # period 30: strided
                  dict(f, kind="both broadcast", a=L((2, 1, 12)), b=L((1, 7, 1))),
                  dict(f, kind="both broadcast", a=L((3, 1, 5)), b=L((1, 4, 1))),
                  dict(f, kind="channels-last", a=L((2, 8, 5, 7), (280, 1, 56, 8)), b=L((2, 8, 5, 7), (280, 1, 56, 8))),
                  dict(f, kind="channels-last + NCHW", a=L((2, 8, 5, 7), (280, 1, 56, 8)), b=L((2, 8, 5, 7))),
                  dict(f, kind="strided out", a=L((5, 33)), b=L((5, 33)), out=L((5, 33), (37, 1))),
                  dict(f, kind="strided out", a=L((6, 64)), b=L((64,)), out=L((6, 64), (68, 1), 4)),
                  dict(f, kind="in place", a=L((7, 129)), b=L((7, 129)), out="a"),
                  dict(f, kind="in place", a=L((4, 96)), b=L((96,)), out="a"),
                  dict(f, kind="specials", a=L((2, 9)), b=L((2, 9))),
                  dict(f, kind="specials", a=L((2, 9), off=1), b=L((2, 9)))]
    sub = dict(op="Sub", dtype="f32")
    specs += [dict(sub, kind="dense", a=L((1027,)), b=L((1027,))), dict(sub, kind="dense", a=L((4, 64)), b=L((4, 64))),
              dict(sub, kind="bias", a=L((3, 5, 100)), b=L((100,))), dict(sub, kind="position", a=L((2, 9, 64)), b=L((9, 64))),
              dict(sub, kind="specials", a=L((2, 9)), b=L((2, 9))), dict(sub, kind="specials", a=L((2, 9)), b=L((9,))),
              dict(sub, kind="misaligned a", a=L((4, 257), off=1), b=L((4, 257))),
              dict(sub, kind="position", a=L((3, 5, 6)), b=L((5, 6)))]  # period 30: strided
    for op in ("Add", "Sub", "Mul"):
        i = dict(op=op, dtype="i32")
        specs += [dict(i, kind="dense", a=L((1027,)), b=L((1027,))), dict(i, kind="wrap", a=L((2, 8)), b=L((2, 8))),
                  dict(i, kind="bias", a=L((3, 5, 100)), b=L((100,))), dict(i, kind="wrap", a=L((2, 8)), b=L((8,))),
                  dict(i, kind="strided out", a=L((5, 33)), b=L((5, 33)), out=L((5, 33), (37, 1))),
                  dict(i, kind="misaligned a", a=L((4, 257), off=1), b=L((4, 257))),
                  dict(i, kind="both broadcast", a=L((2, 1, 12)), b=L((1, 7, 1)))]
    return specs


def table_layout(s):
    """(strides, offset) of the table view.  The view starts 4 R W floats into its buffer, so that a negative index
    that were not counted from the end would read the buffer's filler, not memory outside it."""
    R, Wd = s["table"]
    st, off = {"dense": ((Wd, 1), 0), "off1": ((Wd, 1), 1), "colslice": ((2 * Wd, 2), 0), "transposed": ((1, R), 0),
               "rowpad": ((Wd + 4, 1), 0), "rowpad3": ((Wd + 3, 1), 0)}[s["tlayout"]]
    return st, off + 4 * R * Wd


def gather_specs(sms):
    g = lambda table, tl, idx, neg=True: dict(kind="gather", table=table, tlayout=tl, idx=idx, neg=neg)  # noqa: E731
    return [g((50, 12), "dense", (7,)), g((50, 12), "rowpad", (2, 3)), g((64, 768), "dense", (2, 5, 3)),  # vector
            g((1000, 16), "dense", (300,)), g((50, 13), "dense", (7,)), g((50, 13), "dense", (2, 3, 2)),
            g((40, 12), "colslice", (9,)), g((40, 12), "transposed", (5,)), g((40, 12), "off1", (2, 4)),
            g((40, 12), "rowpad3", (6,)), g((50, 12), "dense", (0,)), g((50, 13), "dense", (2, 0, 3)),
            dict(kind="scatter", table=(40, 12), tlayout="rowpad3", idx=(5,), neg=True, ulayout="rowpad"),
            dict(kind="scatter", table=(30, 13), tlayout="colslice", idx=(7,), neg=True, ulayout="transposed"),
            dict(kind="scatter", table=(64, 16), tlayout="dense", idx=(20,), neg=True, ulayout="dense")]


# ---- partial last units -----------------------------------------------------------------------------------------------
def partial(fam, s):
    """the case leaves a unit of its kernel partly idle: a block with idle threads, a warp-per-row block with idle
    warps, a thread-per-row block with idle threads, a scalar tail after the float4s"""
    want, _ = RULES[fam](s)
    if want is None:
        return False
    k = want[0]
    if fam == "pool":
        B, C = s["shape"][:2]
        oh, ow = pool_windows(s)
        items = B * C * oh * ow // (4 if "cl4" in k else 1)
        return items % BLOCK != 0
    if fam == "gap":
        rows = s["shape"][0] * s["shape"][1]
        return rows % (8 if k == "row_mean_kernel" else 128) != 0
    if fam == "binary":
        n = int(np.prod(binary_layouts(s)[4]))
        if k == "binary_flat_kernel" and _binary_aligned(s):
            return n % 4 != 0
        return (n // 4 if k == "binary_periodic_kernel" else n) % BLOCK != 0
    n = int(np.prod(s["idx"])) * s["table"][1]
    return (n // 4 if k == "gather_rows_vec_kernel" else n) % BLOCK != 0


RULES = {"pool": pool_rule, "gap": gap_rule, "binary": binary_rule, "gather": gather_rule}
SPECS = {"pool": pool_specs, "gap": gap_specs, "binary": binary_specs, "gather": gather_specs}


def spec_id(fam, s):
    return fam + " " + " ".join(f"{k}={v}" for k, v in s.items())


def units():
    return [(k, a, m) for k, args in VARIANTS.items() for a in args for m in MODES.get(k, (None,))]


def coverage_gaps(sms):
    """(kernel, arguments, mode) units that fewer than two cases select, or that no case selects with a partial last
    unit"""
    picked, part = {}, set()
    for fam, specs in SPECS.items():
        for s in specs(sms):
            want, mode = RULES[fam](s)
            if want is None:
                continue
            assert want[1] in VARIANTS[want[0]], f"{spec_id(fam, s)}: the rule names {want}, which the table lacks"
            u = (want[0], want[1], mode)
            picked[u] = picked.get(u, 0) + 1
            if partial(fam, s):
                part.add(u)
    gaps = [("selected fewer than twice", u) for u in units() if picked.get(u, 0) < 2]
    return gaps + [("never with a partial last unit", u) for u in units() if u not in part]


# ---- inputs, launches, references -------------------------------------------------------------------------------------
def _rng(*key):
    return rk._rng("glue", *key)


def _special_values(r, shape):
    return r.choice(np.array([np.nan, np.inf, -np.inf, 0.0, -0.0, 1.5, -1.5, 1e38, -1e38], F32), shape)


def pool_prepare(s):
    r = _rng(sorted(s.items()))
    if s["values"] == "special":
        x = _special_values(r, s["shape"])
    elif s["values"] == "zeros":  # +0 / -0 only: the first of two equal values is kept
        x = np.where(r.random(s["shape"]) < 0.5, F32(0.0), F32(-0.0)).astype(F32)
    else:
        x = r.uniform(-4, 4, s["shape"]).astype(F32)
    return dict(x=x)


def pool_launch(rt, ctx, s, inp):
    xs, off = layout4(s["shape"], s["layout"])
    xd = placed(ctx, inp["x"], xs, off, fill=3.0e38)  # a read outside the view wins every max and shifts every mean
    if s["op"] == "max":
        return rt.MaxPool(s["k"], s["pads"], s["strides"]).run(ctx, xd).numpy()
    return rt.AveragePool(s["k"], s["pads"], s["strides"], s["cip"]).run(ctx, xd).numpy()


def pool_want(oracle, s, inp):
    if s["op"] == "max":
        return oracle.max_pool(inp["x"], s["k"], list(s["pads"]), s["strides"])
    from oracle import resize
    return resize.average_pool(inp["x"], s["k"], s["pads"], s["strides"], s["cip"])


def gap_prepare(s):
    r = _rng(sorted(s.items()))
    B, C, H, W = s["shape"]
    x = r.uniform(-2, 2, s["shape"]).astype(F32)
    if s["special"]:
        rows = x.reshape(B * C, H * W)  # (a view: writes reach x)
        n = H * W
        rows[0, n // 2] = np.inf
        rows[1, 0], rows[1, n - 1] = np.inf, -np.inf  # inf - inf: NaN (for n == 1: -inf)
        rows[2, (n * 2) // 3] = np.nan
        rows[3, n - 1] = -np.inf
    return dict(x=x)


def gap_launch(rt, ctx, s, inp):
    xs, off = layout4(s["shape"], s["layout"])
    return rt.GlobalAveragePool().run(ctx, placed(ctx, inp["x"], xs, off)).numpy()


def gap_want(oracle, s, inp):
    return oracle.global_average_pool(inp["x"])


def _wrap_cases(r, shape):
    """i32 operands at the wrap edges: INT_MAX + 1, INT_MIN - 1, INT_MIN * -1, 65536 * 65536, around random values"""
    a = r.integers(-2 ** 31, 2 ** 31, shape, dtype=np.int64).astype(I32)
    b = r.integers(-2 ** 31, 2 ** 31, shape, dtype=np.int64).astype(I32)
    fa, fb = a.reshape(-1), b.reshape(-1)  # (views: b may broadcast, so only its own elements are set)
    edges = [(2 ** 31 - 1, 1), (-2 ** 31, -1), (-2 ** 31, 1), (65536, 65536), (2 ** 31 - 1, -1), (-1, -2 ** 31)]
    for i, (x, y) in enumerate(edges[:min(fa.size, fb.size)]):
        fa[i], fb[i] = x, y
    return a, b


def binary_prepare(s):
    r = _rng(sorted((k, str(v)) for k, v in s.items()))
    ash, bsh = s["a"][0], s["b"][0]
    if s["dtype"] == "i32":
        if s["kind"] == "wrap":
            a, b = _wrap_cases(r, ash)
            b = b.reshape(-1)[:int(np.prod(bsh))].reshape(bsh)
        else:
            a = r.integers(-2 ** 31, 2 ** 31, ash, dtype=np.int64).astype(I32)
            b = r.integers(-2 ** 31, 2 ** 31, bsh, dtype=np.int64).astype(I32)
        return dict(a=a, b=b)
    if s["kind"] == "specials":
        sv = np.array([0.0, -0.0, -0.0, np.inf, np.inf, np.nan, -np.inf, 3e38, 1e-45], F32)
        a = np.resize(sv, ash).astype(F32)
        b = np.resize(np.array([-0.0, -0.0, 0.0, -np.inf, np.inf, 1.0, 0.0, 3e38, 1e-45], F32), bsh).astype(F32)
        return dict(a=a, b=b)
    return dict(a=r.uniform(-3, 3, ash).astype(F32), b=r.uniform(-3, 3, bsh).astype(F32))


def binary_launch(rt, ctx, s, inp):
    """the result, and whatever the output's buffer holds outside the output view"""
    op = {"Add": rt.Add, "Sub": rt.Sub, "Mul": rt.Mul}[s["op"]]()
    fill = np.nan if s["dtype"] == "f32" else -7
    a = placed(ctx, inp["a"], s["a"][1], s["a"][2], fill)
    # (b's buffer extends as far as a's: an offset of a used for b reads filler, not memory outside the buffer)
    b = placed(ctx, inp["b"], s["b"][1], s["b"][2], fill, guard=a.base.size)
    out = s.get("out")
    if out == "a":
        y = op.run(ctx, a, b, out=a)
        assert y is a
        return a.numpy(), None
    if out is not None:
        shape, st, off = out
        o = placed(ctx, np.zeros(shape, inp["a"].dtype), st, off, fill)
        assert op.run(ctx, a, b, out=o) is o
        full = o.base.numpy()
        mask = np.ones(full.shape, bool)
        np.lib.stride_tricks.as_strided(mask[off:], shape, [x * mask.itemsize for x in st])[...] = False
        return o.numpy(), full[mask]
    return op.run(ctx, a, b).numpy(), None


def binary_want(s, inp):
    a, b = inp["a"], inp["b"]
    if s["dtype"] == "i32":
        a64, b64 = a.astype(np.int64), b.astype(np.int64)
        v = {"Add": a64 + b64, "Sub": a64 - b64, "Mul": a64 * b64}[s["op"]]
        return (((v + 2 ** 31) % 2 ** 32) - 2 ** 31).astype(I32)  # reduced mod 2^32 into [INT_MIN, INT_MAX]
    a64, b64 = a.astype(np.float64), b.astype(np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        v = {"Add": a64 + b64, "Sub": a64 - b64, "Mul": a64 * b64}[s["op"]]
        return v.astype(F32)  # exact in float64, then one rounding: the correctly rounded f32 result


def gather_prepare(s):
    r = _rng(sorted((k, str(v)) for k, v in s.items()))
    R, Wd = s["table"]
    table = r.uniform(-1, 1, (R, Wd)).astype(F32)
    idx = r.integers(0, R, s["idx"]).astype(I32)
    if s["neg"] and idx.size:
        flat = idx.reshape(-1)
        if s["kind"] == "scatter":  # distinct rows: half of them named from the end
            flat[:] = r.permutation(R)[:flat.size]
        flat[::2] -= R
        flat[0] = -1 if s["kind"] == "gather" else flat[0]
    upd = r.uniform(-1, 1, (int(np.prod(s["idx"])), Wd)).astype(F32)
    return dict(table=table, idx=idx, upd=upd)


def gather_launch(rt, ctx, s, inp):
    ts, off = table_layout(s)
    t = placed(ctx, inp["table"], ts, off)
    if s["kind"] == "gather":
        return rt.GatherRows().run(ctx, t, ctx.to_device(inp["idx"])).numpy(), None
    n, Wd = inp["upd"].shape
    us = {"dense": (Wd, 1), "rowpad": (Wd + 4, 1), "transposed": (1, n)}[s["ulayout"]]
    u = placed(ctx, inp["upd"], us)
    assert rt.ScatterRows().run(ctx, t, ctx.to_device(inp["idx"]), u) is t
    full = t.base.numpy()
    mask = np.ones(full.shape, bool)
    np.lib.stride_tricks.as_strided(mask[off:], t.shape, [x * mask.itemsize for x in ts])[...] = False
    return t.numpy(), full[mask]


def gather_want(s, inp):
    if s["kind"] == "gather":
        return inp["table"][inp["idx"]]
    want = inp["table"].copy()
    want[inp["idx"]] = inp["upd"]
    return want


def launch_case(rt, ctx, fam, s, inp):
    return {"pool": pool_launch, "gap": gap_launch, "binary": binary_launch, "gather": gather_launch}[fam](rt, ctx, s, inp)


PREPARE = {"pool": pool_prepare, "gap": gap_prepare, "binary": binary_prepare, "gather": gather_prepare}


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
    import json
    import torch
    import rten_b200 as rt
    n_sms = torch.cuda.get_device_properties(0).multi_processor_count
    ctx = rt.Context(0)
    res, retaken = {}, 0
    for fam, specs in SPECS.items():
        for s in specs(n_sms):
            inp = PREPARE[fam](s)

            def call():
                launch_case(rt, ctx, fam, s, inp)
                ctx.sync()
            names, again = rk.capture_kernels(call)
            retaken += again
            res[spec_id(fam, s)] = sorted(names)
    print(json.dumps({"sms": n_sms, "names": res, "retaken": retaken}))


def test_kernel_identity():
    out = rk.probe_in_child("test_gpu_glue_kernels")
    n_sms, names = out["sms"], out["names"]
    seen, wrong = {}, []
    for fam, specs in SPECS.items():
        for s in specs(n_sms):
            sid = spec_id(fam, s)
            want, mode = RULES[fam](s)
            ran = {rk.kernel_key(n, KERNELS) for n in names[sid]} - {None}
            ran = {k for k in ran if k[0] in FAMILY_KERNELS[fam]}
            if ran != ({want} if want is not None else set()):
                wrong.append((sid, want, sorted(ran), [n for n in names[sid] if "kernel" in n]))
            for k in ran:
                seen[(k[0], k[1], mode)] = seen.get((k[0], k[1], mode), 0) + 1
    assert not wrong, f"{len(wrong)} cases ran another kernel than the rule names: {wrong[:10]}"
    missing = [u for u in units() if seen.get(u, 0) < 2]
    assert not missing, f"kernels (and modes) that fewer than two cases ran: {missing}"
    assert not coverage_gaps(n_sms)
    print(f"{len(units())} kernel units each ran at least twice ({min(seen.values())} to {max(seen.values())} cases) on "
          f"{n_sms} SMs; {len(names)} captures, {out['retaken']} taken again")


# ---- numbers ----------------------------------------------------------------------------------------------------------
def test_max_pool_bit_exact(rt, oracle, sms):
    """Bit-exact against oracle.max_pool: a fold from -inf with `v > m ? v : m` in (ky, kx) order, the reference's
    `acc.max(x)` for NaN inputs (a NaN never replaces the running maximum; an all-NaN window gives -inf).  For +0 / -0
    the oracle's rule keeps the first of two equal values, and so must the kernels; Rust leaves f32::max(+0, -0)
    unspecified, so the reference itself may return either zero there."""
    ctx = rt.Context(0)
    for s in pool_specs(sms):
        if s["op"] != "max":
            continue
        inp = pool_prepare(s)
        got = pool_launch(rt, ctx, s, inp)
        want = pool_want(oracle, s, inp)
        gc.assert_bit_exact(got, want, spec_id("pool", s))
        if s["pads"][0] >= s["k"][0] or s["pads"][1] >= s["k"][1]:
            assert np.isneginf(got).any(), f"{spec_id('pool', s)}: no window lies entirely in the padding"


def test_average_pool_windows(rt, oracle, sms):
    """The AveragePool cases of the identity test, bit-exact against oracle/resize.py average_pool, including windows
    that reach into the end padding, as the executor pads a ceil-mode pool"""
    ctx = rt.Context(0)
    for s in pool_specs(sms):
        if s["op"] == "avg":
            inp = pool_prepare(s)
            gc.assert_bit_exact(pool_launch(rt, ctx, s, inp), pool_want(oracle, s, inp), spec_id("pool", s))


def test_global_average_pool_bit_exact(rt, oracle, sms):
    ctx = rt.Context(0)
    for s in gap_specs(sms):
        inp = gap_prepare(s)
        got = gap_launch(rt, ctx, s, inp)
        gc.assert_bit_exact(got, gap_want(oracle, s, inp), spec_id("gap", s))
        if s["special"] and s["shape"][2] * s["shape"][3] > 1:
            g = got.reshape(-1)
            assert g[0] == np.inf and np.isnan(g[1]) and np.isnan(g[2]) and g[3] == -np.inf, spec_id("gap", s)


def test_binary_ops_exact(rt, sms):
    ctx = rt.Context(0)
    for s in binary_specs(sms):
        inp = binary_prepare(s)
        got, outside = binary_launch(rt, ctx, s, inp)
        gc.assert_bit_exact(got, binary_want(s, inp), spec_id("binary", s))
        if outside is not None:
            untouched = np.isnan(outside).all() if s["dtype"] == "f32" else (outside == -7).all()
            assert untouched, f"{spec_id('binary', s)}: writes outside the output view"


def test_binary_signed_zeros_and_wrap_edges(rt):
    """The edges by name: -0 + -0 = -0, -0 + +0 = +0, inf + -inf and inf - inf = NaN, on the flat, periodic and
    strided f32 kernels; i32 INT_MAX + 1 = INT_MIN, INT_MIN - 1 = INT_MAX, INT_MIN * -1 = INT_MIN, 65536 * 65536 = 0 on
    the flat and the strided kernel"""
    ctx = rt.Context(0)
    z = np.array([-0.0, -0.0, np.inf, 5.0], F32)
    w = np.array([-0.0, 0.0, -np.inf, np.nan], F32)
    # [4] + [4]; [3, 4] + [4]; [4, 1] + [4, 3]: element i of every output row is z[i] + w[i]
    for name, a, b, pick in (("flat", z, w, lambda y: y), ("periodic", np.tile(z, (3, 1)), w, lambda y: y[2]),
                             ("strided", z[:, None], np.repeat(w[:, None], 3, 1), lambda y: y[:, 2])):
        y = pick(rt.Add().run(ctx, ctx.to_device(a), ctx.to_device(b)).numpy())
        assert np.signbit(y[0]) and y[0] == 0 and not np.signbit(y[1]) and y[1] == 0, (name, y)
        assert np.isnan(y[2]) and np.isnan(y[3]), (name, y)
    for name, b in (("flat", np.full(5, np.inf, F32)), ("strided", np.full((2, 5), np.inf, F32))):
        d = rt.Sub().run(ctx, ctx.to_device(np.full(5, np.inf, F32)), ctx.to_device(b)).numpy()
        assert np.isnan(d).all(), (f"inf - inf on the {name} kernel", d)
    imax, imin = 2 ** 31 - 1, -2 ** 31
    cases = (("Add", imax, 1, imin), ("Sub", imin, 1, imax), ("Mul", imin, -1, imin), ("Mul", 65536, 65536, 0))
    for op, x, y, want in cases:
        for kernel, a, b in (("flat", np.full(5, x, I32), np.full(5, y, I32)), ("strided", np.full((3, 5), x, I32), np.full(5, y, I32))):
            got = getattr(rt, op)().run(ctx, ctx.to_device(a), ctx.to_device(b)).numpy()
            assert (got == want).all(), f"i32 {op} {x}, {y} on the {kernel} kernel: {got.reshape(-1)[:3]}, want {want}"


def test_gather_scatter_rows(rt, sms):
    ctx = rt.Context(0)
    for s in gather_specs(sms):
        inp = gather_prepare(s)
        got, outside = gather_launch(rt, ctx, s, inp)
        gc.assert_bit_exact(got, gather_want(s, inp), spec_id("gather", s))
        if outside is not None:
            assert np.isnan(outside).all(), f"{spec_id('gather', s)}: writes outside the table view"


# ---- the executor's pools: ceil_mode and auto_pad ---------------------------------------------------------------------
def pool_graph(op, shape, **attrs):
    import onnx_writer as W
    outs = attrs.pop("outputs", ["y"])
    nodes = [W.node(op, ["x"], outs, **attrs)]
    graph_outs = [W.value_info(o, W.FLOAT, ["n", "c", "h", "w"]) for o in outs if o]
    return W.model(nodes, [], [W.value_info("x", W.FLOAT, list(shape))], graph_outs)


# (op, input shape, attributes): each ceil / SAME case names a size where the rule differs from the floor formula
EXECUTOR_POOLS = [
    ("MaxPool", (1, 8, 54, 55), dict(kernel_shape=[3, 3], strides=[2, 2], ceil_mode=1)),  # 54 -> 27 (floor: 26), 55 -> 27
    ("MaxPool", (2, 4, 13, 16), dict(kernel_shape=[3, 3], strides=[2, 2], pads=[1, 1, 1, 1], ceil_mode=1)),
    ("MaxPool", (1, 3, 6, 7), dict(kernel_shape=[2, 2], strides=[3, 3], pads=[1, 1, 2, 2], ceil_mode=1)),  # drop rule
    ("MaxPool", (1, 3, 8, 9), dict(kernel_shape=[3, 2], strides=[2, 3], pads=[0, 0, 2, 2], ceil_mode=1)),  # drop rule
    ("MaxPool", (1, 3, 4, 6), dict(kernel_shape=[2, 2], strides=[2, 2], pads=[0, 0, 2, 2], ceil_mode=1)),  # ceil < floor
    ("MaxPool", (1, 4, 13, 13), dict(kernel_shape=[3, 3], strides=[2, 2], auto_pad="SAME_UPPER")),
    ("MaxPool", (1, 4, 12, 14), dict(kernel_shape=[3, 3], strides=[2, 2], auto_pad="SAME_UPPER", pads=[5, 5, 5, 5])),
    ("MaxPool", (1, 4, 12, 13), dict(kernel_shape=[3, 3], strides=[2, 2], auto_pad="VALID")),
    ("MaxPool", (1, 4, 12, 13), dict(kernel_shape=[2, 2], strides=[2, 2], auto_pad="NOTSET", ceil_mode=1)),
    ("AveragePool", (1, 8, 54, 55), dict(kernel_shape=[3, 3], strides=[2, 2], ceil_mode=1, count_include_pad=0)),
    ("AveragePool", (1, 8, 54, 55), dict(kernel_shape=[3, 3], strides=[2, 2], ceil_mode=1, count_include_pad=1)),
    ("AveragePool", (1, 3, 6, 7), dict(kernel_shape=[2, 2], strides=[3, 3], pads=[1, 1, 2, 2], ceil_mode=1, count_include_pad=1)),
    ("AveragePool", (2, 4, 11, 10), dict(kernel_shape=[3, 3], strides=[2, 2], auto_pad="SAME_UPPER", count_include_pad=0)),
    ("AveragePool", (2, 4, 11, 10), dict(kernel_shape=[3, 3], strides=[2, 2], auto_pad="SAME_UPPER", count_include_pad=1)),
    ("AveragePool", (1, 4, 12, 13), dict(kernel_shape=[3, 3], strides=[2, 2], auto_pad="VALID", count_include_pad=1)),
]


def executor_pool_expect(shape, attrs):
    """(output H, W, the explicit pads [t, l, b, r] under which the floor formula gives them)"""
    k, st = attrs["kernel_shape"], attrs.get("strides", [1, 1])
    same = attrs.get("auto_pad") in ("SAME_UPPER", "SAME_LOWER")
    p = attrs.get("pads", [0, 0, 0, 0]) if not same else [0, 0, 0, 0]
    res = [pool_out_size(shape[2 + i], k[i], st[i], p[i], p[2 + i], bool(attrs.get("ceil_mode", 0)), same) for i in range(2)]
    (oh, pt, _), (ow, pl, _) = res
    # the end pad that makes floor((n + ps + pe - k) / s) + 1 the size (the kernels never read it)
    pb, pr = ((o - 1) * st[i] + k[i] - shape[2 + i] - ps for i, (o, ps, _) in enumerate(res))
    return oh, ow, [pt, pl, pb, pr]


def _pool_case_id(op, shape, attrs):
    short = {"kernel_shape": "k", "strides": "s", "pads": "p", "ceil_mode": "ceil", "auto_pad": "", "count_include_pad": "cip"}
    return "-".join([op, "x".join(map(str, shape[2:]))] + [short[k] + ("x".join(map(str, v)) if isinstance(v, list) else str(v))
                                                          for k, v in attrs.items()])


@pytest.mark.parametrize("op,shape,attrs", EXECUTOR_POOLS, ids=[_pool_case_id(*c) for c in EXECUTOR_POOLS])
def test_executor_pool_ceil_mode_and_auto_pad(rt, oracle, op, shape, attrs):
    from oracle import resize
    from rten_b200.model import Model
    ctx = rt.Context(0)
    what = f"{op} {shape} {attrs}"
    x = _rng(what).uniform(-3, 3, shape).astype(F32)
    (y,) = Model(ctx, pool_graph(op, shape, **dict(attrs))).run({"x": x}, ["y"])
    oh, ow, pads = executor_pool_expect(shape, attrs)
    assert y.shape == (shape[0], shape[1], oh, ow), f"{what}: output shape {y.shape}, the reference's {(oh, ow)}"
    k, st = attrs["kernel_shape"], attrs.get("strides", [1, 1])
    if op == "MaxPool":
        want = oracle.max_pool(x, k, pads, st)
    else:
        want = resize.average_pool(x, k, pads, st, bool(attrs.get("count_include_pad", 0)))
    gc.assert_bit_exact(y.numpy(), want, what)


def test_executor_pool_load_failures(rt):
    from rten_b200.model import Model
    ctx = rt.Context(0)
    shape = (1, 4, 8, 8)
    bad = {
        "SAME_LOWER is not supported": ("MaxPool", dict(kernel_shape=[3, 3], auto_pad="SAME_LOWER")),
        "auto_pad: unsupported value": ("AveragePool", dict(kernel_shape=[3, 3], auto_pad="SAME")),
        "Indices output": ("MaxPool", dict(kernel_shape=[2, 2], strides=[2, 2], outputs=["y", "idx"])),
    }
    for msg, (op, attrs) in bad.items():
        with pytest.raises(rt.OpError, match=msg):
            Model(ctx, pool_graph(op, shape, **attrs))
    # an AveragePool with ceil_mode = 1 loads (the reference implements it)
    Model(ctx, pool_graph("AveragePool", shape, kernel_shape=[3, 3], strides=[2, 2], ceil_mode=1))
