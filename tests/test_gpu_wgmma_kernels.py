"""`pytest -m gpu`: the wgmma GEMM / implicit-GEMM convolution kernels (umma_gemm.cu umma_gemm_kernel, umma_kernel.cuh
umma_wide_kernel, umma_halo.cu umma_halo_kernel), each selected by name and checked bit for bit.

The launchers pick the epilogue variant (`pick_epilogue`), the tile width and split-K (`plan_valid`, pinned here with
RTEN_B200_FORCE_BN / FORCE_SPLITK / FORCE_STRICT), the conv pixel box (`conv_tile`), the chained instance and, under
RTEN_B200_HALO=1, the halo unit shape (`halo_params`, `halo_model_shape`).  The rules are restated below with the C++
function each follows; `VARIANTS` lists every instance they pick from (tests/test_wgmma_kernel_table_cpu.py keeps it
equal to the built library's symbols).  `EDGES` lists the branches a kernel name does not show; the case list reaches
each of them, and every instance at least twice, on 132 and on 114 SMs.  No entry point sets a row bias (EpilogueDesc
bias_kind 2): `pick_epilogue` restates it, but no case can reach it.

  * kernel identity: every case runs once under CUPTI in a child process and must run exactly the instance its rule
    names, with the grid min(units, SMs) and the kernel's block, and print the `[umma_gemm]` / `[umma_halo]` line the
    rule gives (epi, bn, splitk, units, chain; bn, T, R, tb, units);
  * values against `wgmma_model`, a float32 restatement: the accumulator is the exact product of the TF32-truncated
    operands (3xTF32: lo*hi + hi*lo + hi*hi, no lo*lo; integers: exact i32 with wrap-around and the zero-point terms),
    rounded once, then GenericEpi's order one rounded operation at a time.  The operands are dyadic on a grid where every
    product term is a multiple of 2^-q and the sum of |terms| of every output stays below 2^(22 - q): every partial sum,
    in any K order, split or tensor-core accumulation order, is exact, so the kernel's result has exactly one correct
    set of bits.  Bias, residual, alpha, beta, the scales and the chained convolution's y are full-mantissa floats, so
    every epilogue rounding, and the TF32 read of the staged y, is observable;
  * every output is a view into a NaN-filled buffer with padding on all sides, and A, B and the conv input are views
    with NaN past K (or C): a bit-exact result inside and NaN outside shows nothing outside the views is read or written;
  * each case runs twice, and a few (the largest split-K, one per kernel) are replayed from a CUDA graph into a
    re-poisoned output: the same bits each time.

Full-mantissa operands cannot be checked bit for bit: `test_full_mantissa_within_the_tf32_bound` keeps one such case per
kernel on the TF32 / 3xTF32 bound against float64."""
import json
import re

import numpy as np
import pytest

import gpu_checks as gc
import test_gpu_conv_norm_resize_kernels as ck
import test_gpu_decode_step_kernels as dk
import test_gpu_row_kernels as rk

pytestmark = pytest.mark.gpu

F32 = np.float32
EPIS = ("Generic", "Fast", "FastGelu", "PlainF32", "PlainF32Gelu", "PlainI8", "PlainI8Gelu")  # enum Epi, in order

# ---- the kernels ------------------------------------------------------------------------------------------------------
VARIANTS = {
    "umma_gemm_kernel": [(0, e) for e in EPIS[:5]] + [(1, e) for e in ("Generic", "Fast", "FastGelu", "PlainI8", "PlainI8Gelu")],
    "umma_wide_kernel": [("PlainF32", 0), ("PlainF32Gelu", 0), ("PlainF32", 64), ("PlainF32", 128)],  # <Epi, CHAIN_N2>
    "umma_halo_kernel": [(32, 1), (64, 1), (32, 2), (64, 2), (128, 2)],  # <N, T>
}
KERNELS = set(VARIANTS)
NUM_THREADS, WIDE_THREADS, HALO_THREADS = 416, 384, 384
EDGES = (
    "M tail", "N % 32 != 0", "N % 4 != 0", "K % 32 != 0", "k_blocks > stages", "units > SMs", "split-K 2", "largest split-K",
    "batched, A broadcast", "batched, B broadcast", "direct stores", "alpha != 1", "r_scale != 1", "residual TMA-staged",
    "residual not TMA-staged", "NaN through act 0", "Relu drops NaN", "out_range",
    *(f"act {a}" for a in range(8)),
    *(f"integer {s}" for s in ("u8 x u8", "u8 x i8", "i8 x u8", "i8 x i8")),
    "za scalar (za8)", "za vector", "zb scalar", "zb vector", "scale scalar", "scale vector", "scale_b", "raw i32 output",
    "conv padding", "conv stride 2", "conv dilation", "conv tile overhang", "conv projection", "3xTF32 two-plane",
    "3xTF32 three-segment", "wide bn 128", "wide bn 256", "chain 64", "chain 128",
    "halo T = 1", "halo T = 2", "halo tb > 1", "halo partial last group", "halo row strips", "halo 1x3", "halo 3x1",
    "halo 5x5", "halo asymmetric padding", "halo bias + Relu")


def _epi_arg(a):
    """an Epi template argument in any spelling ((rtb::Epi)3, rtb::Epi::PlainF32, 3) as its name"""
    a = str(a).strip()
    m = re.fullmatch(r"\(?(?:rtb::)?Epi\)?\s*(\d+)", a.replace("(rtb::Epi)", "Epi ")) or re.fullmatch(r"(\d+)", a)
    if m:
        return EPIS[int(m.group(1))]
    m = re.fullmatch(r"(?:rtb::)?Epi::(\w+)", a)
    return m.group(1) if m else a


def kernel_key(name, kernels=KERNELS):
    """(kernel, template arguments) as in ck.kernel_key, with the Epi argument as its name in both spellings: the cast
    `(rtb::Epi)3` (cu++filt, CUPTI) and the enumerator `rtb::Epi::PlainF32`"""
    k = ck.kernel_key(name.replace("rtb::Epi::", "EPI__"), kernels)
    if k is None:
        return None
    base, args = k
    args = tuple(_epi_arg(str(a).replace("EPI__", "Epi::")) if isinstance(a, str) else a for a in args)
    if base == "umma_wide_kernel" and len(args) == 1:
        args += (0,)
    if base == "umma_wide_kernel":
        args = (args[0] if isinstance(args[0], str) else EPIS[args[0]], args[1])
    if base == "umma_gemm_kernel" and not isinstance(args[1], str):
        args = (args[0], EPIS[args[1]])
    return base, args


def _cdiv(a, b):
    return -(-a // b)


# ---- the rules --------------------------------------------------------------------------------------------------------
def pick_epilogue(kind, N, tma_store, res_tma, splitk, e, no_fast=False, no_plain=False):
    """umma_gemm.cu pick_epilogue.  Fast: a TMA store, N % 32 == 0, no row bias, the residual (if any) TMA-staged (column
    vectors are 16-byte aligned copies here); RTEN_B200_NO_FAST sends everything to Generic.  Plain (unless
    RTEN_B200_NO_PLAIN): f32 with alpha = 1, no range and r_scale = 1; integer with a scale, no vector zero point of A, no
    zero point of B and no split-K.  Gelu variants for act > 1."""
    fast = tma_store and N % 32 == 0 and not no_fast and e.get("bias_kind", 0) != 2 and (not e.get("r") or res_tma)
    if not fast:
        return "Generic"
    gelu = e.get("act", 0) > 1
    if not no_plain:
        if kind == 0 and e.get("alpha", 1.0) == 1.0 and not e.get("range") and (not e.get("r") or e.get("r_scale", 1.0) == 1.0):
            return "PlainF32Gelu" if gelu else "PlainF32"
        if kind == 1 and e.get("scale") and not e.get("za") and not e.get("zb") and splitk == 1:
            return "PlainI8Gelu" if gelu else "PlainI8"
    return "FastGelu" if gelu else "Fast"


def generic_res_tma(epi, kind, act, res_tma):
    """umma_gemm.cu launch_plan: the generic epilogue takes a TMA-staged residual only on its f32, act <= Relu path"""
    return res_tma and not (epi == "Generic" and (kind == 1 or act > 1))


def conv_tile(B, OH, OW, sy, sx):
    """umma_gemm.cu pick_conv_tile: the output-pixel box (tw, th, tb) of at most 128 pixels that wastes the fewest MMA rows
    (ties: the wider box); a box row spans at most 256 input pixels"""
    best, tw, th, tb = -1.0, 1, 1, 1
    for w in range(1, min(OW, 128) + 1):
        if w * sx > 256:
            break
        for h in range(1, min(OH, 128 // w) + 1):
            if h * sy > 256:
                break
            b = min(B, 128 // (w * h))
            if b < 1:
                continue
            tiles = _cdiv(OW, w) * _cdiv(OH, h) * _cdiv(B, b)
            eff = B * OH * OW / (tiles * 128.0)
            if eff > best + 1e-9 or (eff > best - 1e-9 and w > tw):
                best, tw, th, tb = eff, w, h, b
    return tw, th, tb


SPLITS = (1, 2, 3, 4, 5, 6, 8, 10, 12, 16)


def plan_valid(bn, sk, k_blocks, tiles, N, step, wide_ok, act, sms):
    """umma_gemm.cu plan_shape and enumerate_plans: bn 32 / 64 on umma_gemm_kernel (a multiple of the step: 32 with a TMA
    store, else 16), bn 128 / 256 on umma_wide_kernel only with the plain f32 epilogue and no split-K, bn 256 only for
    act <= Relu; a bn above round_up(N, step) is not enumerated (except 32); split-K from SPLITS with at least 4 K blocks
    per split, no empty split, fewer than 2 * SMs tiles, and 2 * tiles counters at most 65536"""
    nmax = _cdiv(N, step) * step
    if bn > nmax and bn != 32:
        return False
    if bn > 64:
        if bn not in (128, 256) or not wide_ok or sk != 1 or (bn == 256 and act > 1):
            return False
    elif bn % 32 or bn % step:
        return False
    if sk > 1:
        kb_per = _cdiv(k_blocks, sk)
        if k_blocks // sk < 4 or (sk - 1) * kb_per >= k_blocks or tiles >= 2 * sms or tiles * 2 > 1 << 16:
            return False
    return sk in SPLITS


def largest_splitk(k_blocks, tiles, N, step, sms):
    return max(sk for sk in SPLITS if plan_valid(32, sk, k_blocks, tiles, N, step, False, 0, sms))


# halo_params constants (umma_halo.cu)
HALO_SHAPES = ((32, 1), (32, 2), (64, 1), (64, 2), (128, 2))
HALO_FIXED_BYTES = 1024 + 2048 + 2 * 128 * 128
HALO_SMEM_MAX = 227 * 1024
HB_MAX = 8


def halo_params(B, C, OH, OW, N, kh, kw, pt, pl, bn, T):
    """umma_halo.cu halo_params for a stride-1, undilated f32 conv with at most a column bias and Relu: None where the
    kernel cannot take it, else R (rows per unit), tb (images per unit: whole images when OH P <= 128 T slots, else strips
    of R rows), P = OW + kw - 1, the units and the weight stages that fit beside the two patches"""
    if (bn, T) not in HALO_SHAPES or kh * kw < 2 or kh * kw > 32 or C % 32 or C < 32 or N < bn or N % bn:
        return None
    P = OW + kw - 1
    if P > 256:
        return None
    if OH * P <= T * 128:
        R, tb = OH, min(1 + (T * 128 - OH * P) // ((OH + kh - 1) * P), B)
    else:
        R, tb = (T * 128) // P, 1
        if R < 1:
            return None
    nr = R + kh - 1
    if nr > 256 or tb > 256:
        return None
    alloc = T * 128 + (kh - 1) * P + kw - 1
    loaded = tb * nr * P
    patch = _cdiv(max(alloc, loaded) * 128, 1024) * 1024
    budget = HALO_SMEM_MAX - HALO_FIXED_BYTES - 2 * patch
    if bn * 128 * 3 > budget:
        return None
    strips = _cdiv(OH, R)
    return dict(bn=bn, T=T, R=R, tb=tb, P=P, nr=nr, strips=strips, units=strips * _cdiv(B, tb) * (N // bn),
                b_stages=min(HB_MAX, budget // (bn * 128)), patch_tx=loaded * 128, c_blocks=C // 32, taps=kh * kw)


def halo_model_shape(B, C, OH, OW, N, kh, kw, pt, pl, sms):
    """umma_halo.cu halo_model_shape: the shape of HALO_SHAPES (in that order, the first of equal costs) with the
    smallest waves x (max(MMA clocks, operand bytes / 55) + epilogue + 800)"""
    best, pick = 1e30, None
    for bn, T in HALO_SHAPES:
        p = halo_params(B, C, OH, OW, N, kh, kw, pt, pl, bn, T)
        if p is None:
            continue
        waves = float(_cdiv(p["units"], sms))
        mma = p["c_blocks"] * p["taps"] * (8.0 * T * max(16.0, bn / 2.0) + 60.0)
        ingest = p["c_blocks"] * (float(p["patch_tx"]) + p["taps"] * bn * 128.0) / 55.0
        epi = T * 128 * bn * 4 / 16.0
        cost = waves * (max(mma, ingest) + epi + 800.0) + 4000.0
        if cost < best:
            best, pick = cost, p
    return pick


# ---- the cases --------------------------------------------------------------------------------------------------------
def _conv_out(s):
    (pt, pl, pb, pr), (kh, kw), st, d = s["pads"], s["k"], s.get("stride", 1), s.get("dil", 1)
    return (s["H"] + pt + pb - d * (kh - 1) - 1) // st + 1, (s["W"] + pl + pr - d * (kw - 1) - 1) // st + 1


def _mm(name, M, K, N, **kw):
    return dict(name=name, op="mm", M=M, K=K, N=N, **kw)


def _conv(name, B, C, H, W, O, k=(1, 1), pads=(0, 0, 0, 0), **kw):
    return dict(name=name, op="conv", B=B, C=C, H=H, W=W, O=O, k=k, pads=pads, **kw)


def _int(name, M, K, N, sa, sb, **kw):
    return dict(name=name, op="mmi", M=M, K=K, N=N, sa=sa, sb=sb, **kw)


def _halo(name, B, C, H, W, O, k, pads, **kw):
    return dict(name=name, op="halo", B=B, C=C, H=H, W=W, O=O, k=k, pads=pads, **kw)


def specs(sms):
    big_m = 128 * (sms // 2 + 7)  # > SMs / 2 row tiles: with 2+ column tiles, more units than SMs
    return [
        # narrow f32: every epilogue variant, tails, ring wrap, split-K, batches, direct stores
        _mm("plain bias", 200, 96, 64, bn=64, bias=True),
        _mm("plain bias+res relu, K tail", 130, 72, 96, bn=32, bias=True, res=True, act=1),
        _mm("generic N tail", 300, 64, 40, bn=64, bias=True),
        # N % 4 != 0 into rows padded to a multiple of 4: direct stores (a TMA store would write the padding)
        _mm("generic N tail, res relu", 257, 128, 50, bn=32, res=True, act=1),
        _mm("fast alpha", 160, 64, 64, bn=64, alpha=0.7, bias=True, res=True, act=1),
        _mm("fastgelu alpha", 140, 96, 64, bn=32, alpha=0.7, bias=True, act=2),
        _mm("fastgelu tanh alpha", 150, 64, 128, bn=64, alpha=1.5, act=3),
        _mm("plaingelu tanh", 180, 64, 96, bn=32, bias=True, act=3),
        _mm("plaingelu erf persistent", big_m, 64, 128, bn=64, bias=True, act=2),
        dict(name="gemm beta full C", op="gemm", M=190, K=64, N=64, bn=64, alpha=1.0, beta=1.3),
        dict(name="gemm alpha beta, broadcast C", op="gemm", M=150, K=40, N=64, bn=32, alpha=0.6, beta=0.6, c="row"),
        dict(name="gemm alpha, full C, N tail", op="gemm", M=96, K=64, N=48, bn=64, alpha=1.25, beta=1.0),
        _mm("direct stores", 170, 64, 64, bn=32, bias=True, act=1, out="odd"),
        _mm("direct stores gelu", 133, 64, 96, bn=64, bias=True, act=3, out="odd"),
        _mm("nan through act 0", 100, 64, 64, bn=64, bias=True, nan=True),
        _mm("relu drops nan", 100, 64, 64, bn=32, bias=True, act=1, nan=True),
        _mm("split-K 2", 256, 512, 64, bn=64, sk=2, bias=True, res=True, act=1),
        _mm("largest split-K, K = 8192", 256, 8192, 64, bn=32, sk="max", bias=True),
        _mm("split-K fast", 200, 1024, 64, bn=32, sk=4, alpha=0.7, bias=True),
        _mm("persistent plain", big_m, 320, 256, bn=32, bias=True, res=True, act=1),
        _mm("batched, B broadcast", 130, 64, 64, bn=64, batch=(2, 3), bcast="B", bias=True),
        _mm("batched, A broadcast", 140, 64, 96, bn=32, batch=(3, 2), bcast="A", act=1),
        _mm("3xTF32 two-plane", 150, 64, 64, bn=64, x3=True),
        _mm("3xTF32 three-segment", 140, 44, 64, bn=32, x3=True, bias=True),
        # convolutions on umma_gemm_kernel / umma_wide_kernel
        _conv("conv 3x3 pad, sigmoid", 2, 32, 10, 11, 64, k=(3, 3), pads=(1, 1, 1, 1), bn=64, bias=True, act=4),
        _conv("conv 3x3 stride 2, silu", 3, 64, 13, 13, 32, k=(3, 3), pads=(1, 1, 1, 1), stride=2, bn=32, bias=True, act=5),
        _conv("conv 3x3 dilation 2, hardsigmoid", 2, 32, 12, 12, 64, k=(3, 3), pads=(2, 2, 2, 2), dil=2, bn=32, act=(6, 0.15, 0.45)),
        _conv("conv 1x1 overhang, hardswish", 3, 32, 9, 13, 32, bn=32, bias=True, act=7),
        _conv("conv 1x1 res relu", 2, 64, 12, 12, 96, bn=32, bias=True, res=True, act=1),
        _conv("conv 1x1 3xTF32 two-plane", 2, 32, 8, 8, 32, bn=32, x3=True, bias=True),
        _conv("conv 1x1 3xTF32 three-segment", 2, 36, 8, 8, 64, bn=64, x3=True),
        _conv("conv projection", 2, 64, 14, 14, 128, bn=64, bias=True, act=1, proj=(64, 2)),
        _conv("conv projection wide", 2, 32, 8, 8, 128, bn=128, bias=True, act=1, proj=(96, 1)),
        # wide
        _mm("wide 128 bias res", 260, 96, 256, bn=128, bias=True, res=True, act=1),
        _mm("wide 256 relu", 200, 64, 512, bn=256, bias=True, act=1),
        _mm("wide 128 gelu", 150, 64, 160, bn=128, bias=True, act=2),
        _conv("wide 128 conv gelu tanh", 2, 32, 9, 9, 256, bn=128, bias=True, act=3),
        dict(name="wide 256 gemm full C", op="gemm", M=300, K=64, N=256, bn=256, alpha=1.0, beta=1.0),
        _conv("wide 256 conv stride 2", 2, 32, 15, 15, 256, k=(3, 3), pads=(1, 1, 1, 1), stride=2, bn=256, bias=True),
        _mm("wide 128 persistent", big_m, 64, 256, bn=128, bias=True),
        # chained 1x1 convolutions
        _conv("chain 64", 2, 64, 10, 10, 128, bn=128, bias=True, act=1, chain=(64, 1)),
        _conv("chain 64 residual", 2, 32, 9, 9, 64, bn=128, bias=True, res=True, act=1, chain=(64, 0)),
        _conv("chain 128", 3, 32, 8, 8, 256, bn=128, bias=True, act=1, chain=(128, 1)),
        _conv("chain 128 projection", 2, 64, 8, 8, 96, bn=128, bias=True, act=0, chain=(128, 0), proj=(32, 1)),
        # integer
        _int("i8 raw, za8 + zb vector", 200, 256, 64, 0, 1, za="scalar", zb="vector", bn=64),
        _int("i8 raw, za vector, N tail", 150, 200, 48, 1, 0, za="vector", bn=64),
        _int("i8 raw u8 x u8", 130, 128, 64, 0, 0, bn=32),
        _int("i8 raw i8 x i8, zb scalar", 140, 384, 64, 1, 1, zb="scalar", bn=32),
        _int("i8 float plain", 200, 256, 64, 0, 1, za="scalar", scale="vector", scale_b=True, bias=True, res=True, act=1,
             range=True, bn=64),
        _int("i8 float plain gelu", 150, 128, 96, 1, 1, scale="scalar", bias=True, act=2, bn=32),
        _int("i8 float plain gelu tanh range", 170, 256, 64, 0, 1, za="scalar", scale="vector", act=3, range=True, bn=32),
        _int("i8 float fastgelu zb", 130, 256, 64, 0, 1, za="scalar", zb="vector", scale="vector", scale_b=True, bias=True,
             act=2, bn=64),
        _int("i8 float fast split-K", 200, 2048, 64, 0, 1, za="scalar", scale="vector", bias=True, res=True, act=1, sk=2, bn=32),
        _int("i8 float fastgelu zb scalar", 140, 128, 64, 1, 0, zb="scalar", scale="scalar", act=3, bn=32),
        _int("i8 float generic", 160, 256, 40, 0, 1, za="scalar", scale="vector", scale_b=True, bias=True, res=True, act=1,
             range=True, bn=64),
        _int("i8 float persistent", big_m, 128, 128, 0, 1, za="scalar", scale="vector", bias=True, bn=32),
        # halo (RTEN_B200_HALO=1: the model's unit shape)
        _halo("halo 3x3 strips", 2, 32, 24, 24, 32, (3, 3), (1, 1, 1, 1), bias=True, act=1),
        _halo("halo 3x3 tb", 7, 32, 5, 5, 64, (3, 3), (1, 1, 1, 1), bias=True),
        _halo("halo 5x5", 3, 32, 12, 12, 64, (5, 5), (2, 2, 2, 2), bias=True),
        _halo("halo asym pad", 4, 64, 7, 7, 128, (3, 3), (0, 1, 2, 1), bias=True, act=1),
        _halo("halo 1x3 tb", 32, 32, 8, 8, 256, (1, 3), (0, 1, 0, 1), bias=True, act=1),
        _halo("halo 1x3 strips", 8, 32, 56, 56, 32, (1, 3), (0, 1, 0, 1)),
        _halo("halo 3x1 strips", 1, 32, 56, 56, 256, (3, 1), (1, 0, 1, 0), bias=True, act=1),
        _halo("halo 3x1 n64", 4, 32, 56, 56, 64, (3, 1), (1, 0, 1, 0), bias=True),
        _halo("halo 3x1 t2", 2, 32, 56, 56, 256, (3, 1), (1, 0, 1, 0), act=1),
        _halo("halo 1x3 t2 n64", 8, 32, 56, 56, 64, (1, 3), (0, 1, 0, 1), bias=True),
        _halo("halo 1x3 n128", 4, 32, 56, 56, 256, (1, 3), (0, 1, 0, 1), bias=True, act=1),
        _halo("halo 3x1 n128", 8, 32, 40, 40, 256, (3, 1), (1, 0, 1, 0)),
    ]


def spec_id(s):
    return s["name"]


def _geom(s):
    """(kind, M, N, K elements, k_blocks, tiles_m, batch, conv tile or None)"""
    op = s["op"]
    kind = 1 if op == "mmi" else 0
    kelems = 128 if kind else 32
    if op in ("conv", "halo"):
        OH, OW = _conv_out(s)
        C = s["C"]
        Cx = 3 * _cdiv(C, 4) * 4 if s.get("x3") else C
        kh, kw = s["k"]
        kb = kh * kw * _cdiv(Cx, kelems)
        if s.get("proj"):
            Cp = s["proj"][0]
            kb += (3 * Cp if s.get("x3") else Cp) // kelems
        st = s.get("stride", 1)
        tw, th, tb = conv_tile(s["B"], OH, OW, st, st)
        tiles_m = _cdiv(OW, tw) * _cdiv(OH, th) * _cdiv(s["B"], tb)
        return kind, s["B"] * OH * OW, s["O"], kb, tiles_m, 1, (tw, th, tb)
    K = 3 * _cdiv(s["K"], 4) * 4 if s.get("x3") else s["K"]
    batch = int(np.prod(s.get("batch", (1,))))
    return kind, s["M"], s["N"], _cdiv(K, kelems), _cdiv(s["M"], 128), batch, None


def _epi_desc(s):
    op = s["op"]
    e = dict(act=s.get("act", 0) if not isinstance(s.get("act"), tuple) else s["act"][0], alpha=s.get("alpha", 1.0),
             bias_kind=1 if s.get("bias") else 0)
    if op == "gemm":
        e.update(r=True, r_scale=s["beta"], r_row=s.get("c") != "row")
    elif s.get("res"):
        e.update(r=True, r_scale=1.0, r_row=True)
    if op == "mmi":
        e.update(scale=bool(s.get("scale")), za=s.get("za") == "vector", za8=s.get("za") == "scalar", zb=bool(s.get("zb")),
                 range=bool(s.get("range")))
    return e


def case_rule(s, sms):
    """dict(key: the instance, grid, block, line: what the verbose line must show, edges)"""
    op = s["op"]
    kind, M, N, kb, tiles_m, batch, tile = _geom(s)
    e = _epi_desc(s)
    edges = set()
    if op == "halo":
        OH, OW = _conv_out(s)
        kh, kw = s["k"]
        p = halo_model_shape(s["B"], s["C"], OH, OW, N, kh, kw, s["pads"][0], s["pads"][1], sms)
        assert p is not None, f"{s['name']}: the halo kernel cannot take it"
        edges |= {f"halo T = {p['T']}", "halo bias + Relu" if s.get("bias") and e["act"] == 1 else ""}
        if p["tb"] > 1:
            edges.add("halo tb > 1")
            if s["B"] % p["tb"]:
                edges.add("halo partial last group")
        if p["R"] < OH:
            edges.add("halo row strips")
        edges.add({(1, 3): "halo 1x3", (3, 1): "halo 3x1", (5, 5): "halo 5x5"}.get((kh, kw), ""))
        pt, pl, pb, pr = s["pads"]
        if pt != pb or pl != pr:
            edges.add("halo asymmetric padding")
        if p["units"] > sms:
            edges.add("units > SMs")
        return dict(key=("umma_halo_kernel", (p["bn"], p["T"])), grid=min(p["units"], sms), block=HALO_THREADS,
                    line=dict(bn=p["bn"], T=p["T"], R=p["R"], tb=p["tb"], P=p["P"], units=p["units"]), edges=edges - {""})
    odd = s.get("out") == "odd"
    tma_store = not odd and N % 4 == 0  # prepare_launch: unit column stride, N % 4 == 0, TMA-addressable rows
    step = 32 if tma_store else 16
    res_tma = bool(e.get("r")) and tma_store and (kind == 0 or e.get("scale")) and e.get("r_row", True) and N % 32 == 0
    chain = s.get("chain")
    bn = s["bn"]
    tiles_n = 1 if chain else _cdiv(N, bn)
    tiles = tiles_m * tiles_n * batch
    sk = s.get("sk", 1)
    if sk == "max":
        sk = largest_splitk(kb, tiles, N, step, sms)
    epi = pick_epilogue(kind, N, tma_store, res_tma, sk, e)
    wide_ok = pick_epilogue(kind, N, tma_store, res_tma, 1, e) in ("PlainF32", "PlainF32Gelu")
    # (a chained launch has a fixed plan, bn = 128 over every column, which enumerate_plans does not rank)
    assert chain or plan_valid(bn, sk, kb, tiles, N, step, wide_ok, e["act"], sms), f"{s['name']}: no valid plan bn={bn} splitk={sk}"
    units = tiles * sk
    if bn > 64:
        assert epi in ("PlainF32", "PlainF32Gelu")
        key = ("umma_wide_kernel", ("PlainF32", chain[0]) if chain else (epi, 0))
        block = WIDE_THREADS
        edges.add(f"wide bn {bn}")
        if chain:
            edges.add(f"chain {chain[0]}")
    else:
        key = ("umma_gemm_kernel", (kind, epi))
        block = NUM_THREADS
    # the edges
    if M % 128 and op != "conv":
        edges.add("M tail")
    if N % 32:
        edges.add("N % 32 != 0")
    if op in ("mm", "gemm") and s["K"] % 32:
        edges.add("K % 32 != 0")
    if kb > 8:
        edges.add("k_blocks > stages")
    if units > sms:
        edges.add("units > SMs")
    if sk == 2:
        edges.add("split-K 2")
    if s.get("sk") == "max" and sk == largest_splitk(kb, tiles, N, step, sms):
        edges.add("largest split-K")
    if s.get("batch"):
        edges.add(f"batched, {s['bcast']} broadcast")
    if not tma_store:
        edges.add("direct stores")
    if N % 4:
        edges.add("N % 4 != 0")
    if e["alpha"] != 1.0:
        edges.add("alpha != 1")
    if e.get("r") and e.get("r_scale", 1.0) != 1.0:
        edges.add("r_scale != 1")
    if e.get("r"):
        edges.add("residual TMA-staged" if generic_res_tma(epi, kind, e["act"], res_tma) else "residual not TMA-staged")
    if s.get("nan"):
        edges.add("Relu drops NaN" if e["act"] == 1 else "NaN through act 0")
    edges.add(f"act {e['act']}")
    if op == "mmi":
        edges.add(f"integer {'i8' if s['sa'] else 'u8'} x {'i8' if s['sb'] else 'u8'}")
        edges |= {x for x, on in (("za scalar (za8)", s.get("za") == "scalar"), ("za vector", s.get("za") == "vector"),
                                   ("zb scalar", s.get("zb") == "scalar"), ("zb vector", s.get("zb") == "vector"),
                                   ("scale scalar", s.get("scale") == "scalar"), ("scale vector", s.get("scale") == "vector"),
                                   ("scale_b", s.get("scale_b")), ("raw i32 output", not s.get("scale")),
                                   ("out_range", s.get("range"))) if on}
    if op == "conv":
        OH, OW = _conv_out(s)
        if any(s["pads"]):
            edges.add("conv padding")
        if s.get("stride", 1) == 2:
            edges.add("conv stride 2")
        if s.get("dil", 1) > 1:
            edges.add("conv dilation")
        tw, th, tb = tile
        if OW % tw or OH % th or s["B"] % tb:
            edges.add("conv tile overhang")
        if s.get("proj"):
            edges.add("conv projection")
    if s.get("x3"):
        C = s["C"] if op == "conv" else s["K"]
        edges.add("3xTF32 two-plane" if C % 32 == 0 else "3xTF32 three-segment")
    line = dict(epi=epi, bn=bn, splitk=sk, units=units, tma_store=int(tma_store), chain=chain[0] if chain else 0)
    return dict(key=key, grid=min(units, sms), block=block, line=line, edges=edges)


def coverage_gaps(sms):
    """instances that fewer than two cases select, and edges no case reaches"""
    picked, reached = {}, set()
    for s in specs(sms):
        r = case_rule(s, sms)
        k = r["key"]
        assert k[1] in VARIANTS[k[0]], f"{spec_id(s)}: the rule names {k}, which the table lacks"
        picked[k] = picked.get(k, 0) + 1
        reached |= r["edges"]
    gaps = [("selected fewer than twice", (k, a)) for k, args in VARIANTS.items() for a in args if picked.get((k, a), 0) < 2]
    return gaps + [("edge never reached", e) for e in EDGES if e not in reached]


# ---- inputs -----------------------------------------------------------------------------------------------------------
def _rng(*key):
    return rk._rng("wgmma", *key)


def _grid(r, shape, lim, den):
    """multiples of 1/den in [-lim/den, lim/den]"""
    return (r.integers(-lim, lim + 1, shape) / den).astype(F32)


def _x3_operand(r, shape):
    """hi + lo: hi a multiple of 2^-4 in [-1/4, 1/4], lo = sign(hi) * (0 .. 3) * 2^-16 where hi != 0.  hi is the TF32
    truncation of the sum (lo is below its last TF32 bit), and lo a 2-bit value: both lo parts of a product are
    non-zero on most terms, and a lo * lo term would be a multiple of 2^-32"""
    hi = (r.integers(-4, 5, shape) / 16).astype(F32)
    lo = (np.sign(hi) * r.integers(0, 4, shape) * 2.0 ** -16).astype(F32)
    return (hi + lo).astype(F32)


def prepare(s):
    """host inputs.  f32 products: A, B (conv x, w) multiples of 2^-4 (|.| <= 1, or <= 1/2 and 1/4 for long K and the
    chained convolutions); 3xTF32: `_x3_operand`; integers: any 8-bit values.  Bias, residual, C and scales are
    full-mantissa floats."""
    r = _rng(spec_id(s))
    op = s["op"]
    inp = {}
    u = lambda *sh: r.uniform(-1, 1, sh).astype(F32)  # noqa: E731
    if op == "mmi":
        M, K, N = s["M"], s["K"], s["N"]
        inp["a"] = (r.integers(-128, 128, (M, K)).astype(np.int8) if s["sa"] else r.integers(0, 256, (M, K)).astype(np.uint8))
        inp["b"] = (r.integers(-128, 128, (K, N)).astype(np.int8) if s["sb"] else r.integers(0, 256, (K, N)).astype(np.uint8))
        zdt = lambda signed: np.int8 if signed else np.uint8  # noqa: E731
        zr = lambda signed, n: (r.integers(-128, 128, n) if signed else r.integers(0, 256, n)).astype(zdt(signed))  # noqa: E731
        if s.get("za"):
            inp["za"] = zr(s["sa"], 1)[0] if s["za"] == "scalar" else zr(s["sa"], M)
        if s.get("zb"):
            inp["zb"] = zr(s["sb"], 1)[0] if s["zb"] == "scalar" else zr(s["sb"], N)
        if s.get("scale"):
            inp["scale"] = (r.uniform(0.001, 0.01, ()) if s["scale"] == "scalar" else r.uniform(0.001, 0.01, N)).astype(F32)
        if s.get("scale_b"):
            inp["scale_b"] = F32(r.uniform(0.5, 2.0))
        if s.get("bias"):
            inp["bias"] = u(N)
        if s.get("res"):
            inp["res"] = u(M, N)
        return inp
    if op in ("mm", "gemm"):
        M, K, N = s["M"], s["K"], s["N"]
        za = zb = ()
        if s.get("batch"):
            za, zb = (tuple(s["batch"]), ()) if s["bcast"] == "B" else ((), tuple(s["batch"]))
        if s.get("x3"):
            inp["a"], inp["b"] = _x3_operand(r, za + (M, K)), _x3_operand(r, zb + (K, N))
        else:
            lim = 8 if K > 1024 else 16
            inp["a"], inp["b"] = _grid(r, za + (M, K), lim, 16), _grid(r, zb + (K, N), lim, 16)
        if s.get("bias"):
            inp["bias"] = u(N)
            if s.get("nan"):
                inp["bias"][::7] = np.nan
        outer = np.broadcast_shapes(za, zb)
        if s.get("res"):
            inp["res"] = u(*outer, M, N)
        if op == "gemm":
            inp["c"] = u(N) if s.get("c") == "row" else u(M, N)
        return inp
    # convolutions
    B, C, H, W, O = s["B"], s["C"], s["H"], s["W"], s["O"]
    kh, kw = s["k"]
    chain = s.get("chain")
    if s.get("x3"):
        inp["x"], inp["w"] = _x3_operand(r, (B, C, H, W)), _x3_operand(r, (O, C, kh, kw))
    elif chain:
        inp["x"], inp["w"] = _grid(r, (B, C, H, W), 4, 16), _grid(r, (O, C, kh, kw), 4, 16)
    else:
        inp["x"], inp["w"] = _grid(r, (B, C, H, W), 16, 16), _grid(r, (O, C, kh, kw), 16, 16)
    OH, OW = _conv_out(s)
    if chain:
        # y = act(acc + residual + bias) with |acc| < 4 and |bias| in [16, 32): |y| >= 8 or y = 0, so TF32(y) is a
        # multiple of 2^-7; W2 multiples of 2^-4 in [-1/16, 1/16]
        mag = r.uniform(16, 32, O).astype(F32)
        inp["bias"] = (np.where(r.integers(0, 2, O) == 1, mag, -mag)).astype(F32)
        inp["w2"] = _grid(r, (chain[0], O, 1, 1), 1, 16)
        inp["b2"] = u(chain[0])
    elif s.get("bias"):
        inp["bias"] = u(O)
    if s.get("res"):
        inp["res"] = u(B, O, OH, OW)
    if s.get("proj"):
        Cp, ps = s["proj"]
        Hp, Wp = (OH - 1) * ps + 1, (OW - 1) * ps + 1
        if s.get("x3"):
            inp["xp"], inp["wp"] = _x3_operand(r, (B, Cp, Hp, Wp)), _x3_operand(r, (O, Cp, 1, 1))
        else:
            inp["xp"], inp["wp"] = _grid(r, (B, Cp, Hp, Wp), 4 if chain else 16, 16), _grid(r, (O, Cp, 1, 1), 4 if chain else 16, 16)
        inp["bp"] = u(O)
    return inp


# ---- the model --------------------------------------------------------------------------------------------------------
def tf32_trunc(a, rne=False):
    """wgmma's TF32 read: the 13 low mantissa bits dropped (`rne`: rounded to nearest even instead)"""
    from oracle.rnn import tf32_truncate
    if not rne:
        return tf32_truncate(a)
    b = np.ascontiguousarray(a, F32).view(np.uint32).astype(np.uint64)
    b = (b + 0xFFF + ((b >> 13) & 1)) & 0xFFFFE000
    return b.astype(np.uint32).view(F32)


def x3_parts(a, rne=False):
    hi = tf32_trunc(a, rne)
    lo = tf32_trunc((np.asarray(a, F32) - hi).astype(F32), rne)
    return hi, lo


def lsb_exp(v):
    """the exponent of the lowest set bit over the non-zero finite values of v (None if there are none)"""
    v = np.abs(np.asarray(v, np.float64))
    v = v[np.isfinite(v) & (v != 0)]
    if not v.size:
        return None
    m, e = np.frexp(v)
    mi = (m * 2.0 ** 53).astype(np.uint64)
    tz = np.log2((mi & (~mi + np.uint64(1))).astype(np.float64)).astype(np.int64)
    return int((e - 53 + tz).min())


def _conv_f64(x, w, pads, stride, dil):
    """float64 conv of x [B, C, H, W] and w [O, C, kh, kw] as [B, OH, OW, O]"""
    B, C, H, W = x.shape
    O, _, kh, kw = w.shape
    pt, pl, pb, pr = pads
    xp = np.zeros((B, H + pt + pb, W + pl + pr, C))
    xp[:, pt:pt + H, pl:pl + W] = x.transpose(0, 2, 3, 1)
    OH = (H + pt + pb - dil * (kh - 1) - 1) // stride + 1
    OW = (W + pl + pr - dil * (kw - 1) - 1) // stride + 1
    out = np.zeros((B, OH, OW, O))
    for ky in range(kh):
        for kx in range(kw):
            win = xp[:, ky * dil:ky * dil + stride * (OH - 1) + 1:stride, kx * dil:kx * dil + stride * (OW - 1) + 1:stride]
            out += win @ w[:, :, ky, kx].astype(np.float64).T
    return out


def _product(s, a, b, pads=None, stride=1, dil=1):
    """float64 a . b: matmul (broadcast batches) or conv"""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return _conv_f64(a, b, pads, stride, dil) if pads is not None else np.matmul(a, b)


def exact_accumulator(s, a, b, pads=None, stride=1, dil=1, x3=False, perturb=()):
    """(float32 accumulator, the exactness margin: log2(2^22 / (2^q max sum |terms|)), > 0 when exact in every order).
    The kernel's terms: TF32(a) TF32(b), or in 3xTF32 lo(a) hi(b) + hi(a) lo(b) + hi(a) hi(b)."""
    rne = "tf32-rne" in perturb
    if x3:
        (ha, la), (hb, lb) = x3_parts(a, rne), x3_parts(b, rne)
        pairs = [(la, hb), (ha, lb), (ha, hb)] + ([(la, lb)] if "four-product" in perturb else [])
    else:
        pairs = [(tf32_trunc(a, rne), tf32_trunc(b, rne))]
    acc = sum(_product(s, x, y, pads, stride, dil) for x, y in pairs)
    mag = sum(_product(s, np.abs(x), np.abs(y), pads, stride, dil) for x, y in pairs[:3])
    qs = [-(lsb_exp(x) + lsb_exp(y)) for x, y in pairs[:3] if lsb_exp(x) is not None and lsb_exp(y) is not None]
    q = max(qs) if qs else 0
    margin = 22 - q - float(np.log2(max(float(mag.max()), 2.0 ** -60)))
    return acc, margin


def _kblock(a, b, which, op_conv=False):
    """a, b with K block 0 (the first 32 K elements) dropped or doubled (matmul operands only)"""
    a = np.array(a, F32)
    f = F32(0) if which == "drop" else F32(2)
    a[..., :32] *= f
    return a, b


def _act(x, act, alpha=0.2, beta=0.5):
    from oracle import activations as oa
    from oracle import oracle
    x = np.asarray(x, F32)
    if act == 0:
        return x
    if act == 1:
        with np.errstate(invalid="ignore"):
            return np.where(x > 0, x, F32(0)).astype(F32)
    if act in (2, 3):
        return oracle.gelu(x, act == 3).reshape(x.shape)
    return {4: oa.sigmoid, 5: oa.silu, 6: lambda v: oa.hard_sigmoid(v, alpha, beta), 7: oa.hard_swish}[act](x)


def _fma(a, b, c):
    from oracle.norms import fma_f32
    return np.asarray(fma_f32(a, b, c), F32)


def epilogue_f32(acc, e, bias=None, r=None, perturb=()):
    """GenericEpi (f32): acc * alpha, fma(r_scale, r, .), + bias, + row bias (0), act -- each rounded"""
    x = np.asarray(acc, F32)
    alpha, rs = F32(e.get("alpha", 1.0)), F32(e.get("r_scale", 1.0))
    b = F32(0) if bias is None else np.asarray(bias, F32)
    with np.errstate(invalid="ignore"):
        if "alpha-after-fma" in perturb and r is not None:
            x = (_fma(rs, r, x) * alpha).astype(F32)
        elif "bias-before-residual" in perturb and r is not None:
            x = ((x * alpha).astype(F32) + b).astype(F32)
            x = _fma(rs, r, x)
            b = F32(0)
        else:
            x = (x * alpha).astype(F32)
            if r is not None:
                x = _fma(rs, r, x)
        x = ((x + b).astype(F32) + F32(0)).astype(F32)
    return _act(x, e.get("act", 0), *e.get("act_ab", (0.2, 0.5)))


def epilogue_i8(c, e, scale=None, scale_b=None, bias=None, r=None, perturb=()):
    """GenericEpi (integer): the i32 result, or (float)c * (scale_b * scale) rounded twice, + bias, + r, act"""
    c = np.asarray(c, np.int64).astype(np.uint64).astype(np.uint32).view(np.int32)
    if scale is None:
        return c
    sc = np.asarray(scale, F32)
    if scale_b is not None:
        if "scale-unrounded" in perturb:
            sc = np.float64(scale_b) * sc.astype(np.float64)
        else:
            sc = (F32(scale_b) * sc).astype(F32)
    x = (c.astype(F32) * sc).astype(F32)
    if bias is not None:
        x = (x + bias).astype(F32)
    if r is not None:
        x = (x + r).astype(F32)
    return _act(x, e.get("act", 0))


def encode_range(y):
    """umma_kernel.cuh f32_to_ordered of (min, max)"""
    v = np.array([np.min(y), np.max(y)], F32).view(np.int32).astype(np.int64)
    return np.where(v >= 0, v, v ^ 0x7FFFFFFF).astype(np.int32)


def wgmma_model(s, inp, perturb=()):
    """(outputs as the call returns them, exactness margin)"""
    op = s["op"]
    e = _epi_desc(s)
    act = s.get("act", 0)
    if isinstance(act, tuple):
        e["act_ab"] = act[1:]
    if op == "mmi":
        a, b = inp["a"].astype(np.int64), inp["b"].astype(np.int64)
        za = np.asarray(inp.get("za", 0), np.int64)
        zb = np.asarray(inp.get("zb", 0), np.int64)
        if "kblock-drop" in perturb or "kblock-double" in perturb:
            a = a.copy()
            a[:, :128] *= 0 if "kblock-drop" in perturb else 2
        za_col = za.reshape(-1, 1) if za.ndim else za
        c = (a - za_col) @ (b - zb)
        y = epilogue_i8(c, e, inp.get("scale"), inp.get("scale_b"), inp.get("bias"), inp.get("res"), perturb)
        out = [y]
        if s.get("range"):
            out.append(encode_range(y))
        return out, 22.0  # (integer arithmetic is exact)
    if op in ("mm", "gemm"):
        a, b = inp["a"], inp["b"]
        if "kblock-drop" in perturb or "kblock-double" in perturb:
            a, b = _kblock(a, b, "drop" if "kblock-drop" in perturb else "double")
        acc, margin = exact_accumulator(s, a, b, x3=s.get("x3", False), perturb=perturb)
        r = inp.get("c") if op == "gemm" else inp.get("res")
        if op == "gemm":
            e["alpha"] = s["alpha"]
        return [epilogue_f32(acc.astype(F32), e, inp.get("bias"), r, perturb)], margin
    pads, st, dil = s["pads"], s.get("stride", 1), s.get("dil", 1)
    x, w = inp["x"], inp["w"]
    if "kblock-drop" in perturb or "kblock-double" in perturb:
        x = np.array(x, F32)
        x[:, :min(32, x.shape[1])] *= F32(0 if "kblock-drop" in perturb else 2)
    acc, margin = exact_accumulator(s, x, w, pads, st, dil, x3=s.get("x3", False), perturb=perturb)
    bias = inp.get("bias")
    if s.get("proj"):
        Cp, ps = s["proj"]
        accp, mp = exact_accumulator(s, inp["xp"], inp["wp"], (0, 0, 0, 0), ps, 1, x3=s.get("x3", False), perturb=perturb)
        acc = acc + accp  # one accumulator over both K ranges
        margin = min(margin, mp) - 1
        bias = (bias + inp["bp"]).astype(F32) if bias is not None else inp["bp"]  # column_bias: bias + bias2, rounded
    res = inp["res"].transpose(0, 2, 3, 1) if s.get("res") else None
    y = epilogue_f32(acc.astype(F32), e, bias, res, perturb)
    outs = [y.transpose(0, 3, 1, 2)]
    if s.get("chain"):
        N2, act2 = s["chain"]
        accz, mz = exact_accumulator(s, y.transpose(0, 3, 1, 2), inp["w2"], (0, 0, 0, 0), 1, 1, perturb=perturb)
        z = epilogue_f32(accz.astype(F32), dict(act=act2), inp["b2"])
        outs.append(z.transpose(0, 3, 1, 2))
        margin = min(margin, mz)
    return outs, margin


# ---- device placement -------------------------------------------------------------------------------------------------
def _nan_buffer(ctx, shape, strides, off, size, dtype=F32, values=None):
    """a view (shape, strides, off) of a device buffer of `size` NaNs (integers: 0x7F bytes), holding `values`"""
    fill = np.nan if np.dtype(dtype).kind == "f" else (np.iinfo(dtype).max if np.dtype(dtype).kind == "i" else 0x7F)
    buf = np.full(size, fill, dtype)
    if values is not None:
        buf[_view_index(shape, strides, off)] = values
    d = ctx.to_device(buf)
    return d.view(tuple(shape), tuple(strides), off), d, buf


def _view_index(shape, strides, off):
    idx = np.full(tuple(shape), off, np.int64)
    for i, (n, st) in enumerate(zip(shape, strides)):
        idx = idx + (np.arange(n) * st).reshape([-1 if j == i else 1 for j in range(len(shape))])
    return idx


def _dense_strides(shape, pad_last):
    """row-major strides with the last dim padded to a multiple of 4 plus `pad_last`"""
    st, acc = [], 1
    for i, n in enumerate(reversed(shape)):
        st.append(acc)
        acc *= (_cdiv(n, 4) * 4 + pad_last) if i == 0 else n
    return tuple(reversed(st)), acc


def _matrix_strides(shape):
    """(strides, buffer size) of [.., rows, K] matrices: rows padded past K with 4 to 7 elements (a multiple of 16
    bytes), each matrix followed by a spare row and each outer batch by another, so that no batch dims collapse"""
    *outer, rows, k = shape
    kp = _cdiv(k, 4) * 4 + 4
    st = [1, kp]
    span = rows * kp  # elements one entry of the dim below occupies
    for n in reversed(outer):
        st.append(span + kp)
        span = n * (span + kp)
    st = tuple(reversed(st))
    return st, 1 + sum((n - 1) * x for n, x in zip(shape, st)) + 4


class Placed:
    """the device operands of one case, and its NaN-padded outputs (views into poisoned buffers)"""

    def __init__(self, ctx, s, inp):
        self.args, self.outs = {}, []
        op = s["op"]
        if op in ("mm", "gemm", "mmi"):
            a, b = inp["a"], inp["b"]
            # A: rows padded past K with NaN, batches a row apart more (no flattening); B as a K-major view
            ast, asz = _matrix_strides(a.shape)
            self.args["a"] = _nan_buffer(ctx, a.shape, ast, 0, asz, a.dtype, a)[0]
            bst, bsz = _matrix_strides(np.swapaxes(b, -1, -2).shape)
            bst = bst[:-2] + (bst[-1], bst[-2])
            self.args["b"] = _nan_buffer(ctx, b.shape, bst, 0, bsz, b.dtype, b)[0]
            for k in ("bias", "res", "c", "za", "zb", "scale", "scale_b"):
                if k in inp:
                    self.args[k] = ctx.to_device(np.asarray(inp[k]))
            outer = np.broadcast_shapes(a.shape[:-2], b.shape[:-2])
            oshape = tuple(outer) + (s["M"], s["N"])
            dt = np.int32 if op == "mmi" and not s.get("scale") else F32
        else:
            x = inp["x"]
            self.args["x"] = self._nhwc(ctx, x, 4)
            for k in ("bias", "bp", "b2"):
                if k in inp:
                    self.args[k] = ctx.to_device(inp[k])
            if "res" in inp:
                self.args["res"] = ctx.to_device(inp["res"], channels_last=True)
            if "xp" in inp:
                self.args["xp"] = self._nhwc(ctx, inp["xp"], 4)
            OH, OW = _conv_out(s)
            oshape = (s["B"], s["O"], OH, OW)
            dt = F32
        self.outs.append(self._out(ctx, oshape, dt, odd=s.get("out") == "odd", conv=op not in ("mm", "gemm", "mmi")))
        if s.get("chain"):
            OH, OW = _conv_out(s)
            self.outs.append(self._out(ctx, (s["B"], s["chain"][0], OH, OW), F32, conv=True))
        if s.get("range"):
            self.rng = ctx.to_device(np.array([2 ** 31 - 1, -2 ** 31], np.int32))

    @staticmethod
    def _nhwc(ctx, x, cpad):
        """x [B, C, H, W] as a channels-last view whose pixels are C + cpad (rounded to 4) floats apart, NaN between"""
        B, C, H, W = x.shape
        cs = _cdiv(C, 4) * 4 + cpad
        strides = (H * W * cs, 1, W * cs, cs)
        return _nan_buffer(ctx, x.shape, strides, 0, B * H * W * cs, F32, x)[0]

    @staticmethod
    def _out(ctx, shape, dt, odd=False, conv=False):
        """(view, device buffer, index of the view) in a NaN buffer with 4 elements before and after, rows (pixels)
        padded by 4 (odd: by 1, which no TMA store can write)"""
        if conv:
            B, C, H, W = shape
            cs = C + (1 if odd else 4)
            strides, size = (H * W * cs, 1, W * cs, cs), B * H * W * cs
        else:
            st, size = _dense_strides(shape, 4)
            if odd:
                n = shape[-1] + 1
                st = tuple((int(np.prod(shape[i + 1:-1])) * n) if i < len(shape) - 1 else 1 for i in range(len(shape)))
                size = int(np.prod(shape[:-1])) * n
            strides = st
        view, dev, _ = _nan_buffer(ctx, shape, strides, 4, size + 8, dt)
        return view, dev, _view_index(shape, strides, 4), size + 8

    def poison(self):
        for view, dev, _, size in self.outs:
            fill = np.nan if dev.dtype.kind == "f" else np.iinfo(dev.dtype).max
            dev.copy_from(np.full(size, fill, dev.dtype))
        if getattr(self, "rng", None) is not None:
            self.rng.copy_from(np.array([2 ** 31 - 1, -2 ** 31], np.int32))

    def read(self):
        """(the outputs as host arrays, the changes outside the views: [(output, element offset from the view's first
        element, value)])"""
        got, clean = [], []
        for i, (view, dev, idx, size) in enumerate(self.outs):
            full = dev.numpy()
            got.append(full[idx])
            mask = np.ones(size, bool)
            mask[idx.ravel()] = False
            bad = mask & ~(np.isnan(full) if dev.dtype.kind == "f" else full == np.iinfo(dev.dtype).max)
            clean += [(i, int(j) - 4, full[j].item()) for j in np.flatnonzero(bad)]
        if getattr(self, "rng", None) is not None:
            got.append(self.rng.numpy())
        return got, clean


def _env(s):
    if s["op"] == "halo":
        return dict(RTEN_B200_HALO=1, RTEN_B200_FORCE_BN=None, RTEN_B200_FORCE_SPLITK=None, RTEN_B200_FORCE_STRICT=None)
    sk = s.get("sk", 1)
    env = dict(RTEN_B200_HALO=None, RTEN_B200_FORCE_BN=s["bn"], RTEN_B200_FORCE_STRICT=1)
    env["RTEN_B200_FORCE_SPLITK"] = sk if sk != "max" else None
    return env


def run_case(rt, ctx, s, pl, sms):
    """one call of the case's operator into pl's outputs (the plan pinned by `_env`)"""
    op, a = s["op"], pl.args
    ctx.set_f32_mode(bool(s.get("x3")))
    env = _env(s)
    if s.get("sk") == "max":
        kind, M, N, kb, tiles_m, batch, _ = _geom(s)
        env["RTEN_B200_FORCE_SPLITK"] = largest_splitk(kb, tiles_m * _cdiv(N, s["bn"]) * batch, N, 32, sms)
    out = pl.outs[0][0]
    act = s.get("act", 0)
    with gc.switches(**env):
        if op == "mm":
            rt.FusedMatMul(s.get("alpha"), activation=act).run(ctx, a["a"], a["b"], a.get("bias"), residual=a.get("res"), out=out)
        elif op == "gemm":
            rt.Gemm(s["alpha"], s["beta"]).run(ctx, a["a"], a["b"], a["c"], out=out)
        elif op == "mmi":
            if s.get("scale"):
                rt.MatMulIntegerToFloat(act).run(ctx, a["a"], a["b"], a.get("za"), a.get("zb"), a["scale"], out=out,
                                                 bias=a.get("bias"), residual=a.get("res"), scale_b=a.get("scale_b"),
                                                 out_range=getattr(pl, "rng", None))
            else:
                rt.MatMulInteger().run(ctx, a["a"], a["b"], a.get("za"), a.get("zb"), out=out)
        else:
            inp = pl.inp
            st, d = s.get("stride", 1), s.get("dil", 1)
            conv = rt.Conv(1, (d, d), s["pads"], (st, st), activation=act)
            if s.get("chain"):
                N2, act2 = s["chain"]
                nxt = rt.Conv(1, (1, 1), (0, 0, 0, 0), (1, 1), activation=act2)
                kw = {}
                if s.get("proj"):
                    kw = dict(proj=rt.Conv(1, (1, 1), (0, 0, 0, 0), (s["proj"][1],) * 2), x_proj=a["xp"], w_proj=inp["wp"],
                              bias_proj=a["bp"])
                conv.run_chained(ctx, a["x"], inp["w"], a.get("bias"), residual=a.get("res"), nxt=nxt, w_next=inp["w2"],
                                 bias_next=a["b2"], out=out, out_next=pl.outs[1][0], **kw)
            elif s.get("proj"):
                proj = rt.Conv(1, (1, 1), (0, 0, 0, 0), (s["proj"][1],) * 2)
                conv.run_projected(ctx, a["x"], inp["w"], a.get("bias"), proj=proj, x_proj=a["xp"], w_proj=inp["wp"],
                                   bias_proj=a["bp"], out=out)
            else:
                conv.run(ctx, a["x"], inp["w"], a.get("bias"), residual=a.get("res"), out=out)


def place(ctx, s, inp):
    pl = Placed(ctx, s, inp)
    pl.inp = inp
    return pl


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


@pytest.fixture(autouse=True)
def _clean_env():
    keys = ("RTEN_B200_NO_FAST", "RTEN_B200_NO_PLAIN", "RTEN_B200_NO_WIDE", "RTEN_B200_NO_HALO", "RTEN_B200_NO_CHAIN",
            "RTEN_B200_X3_THREE_PLANES", "RTEN_B200_TUNE_FILE", "RTEN_B200_HALO") + gc.FORCE_KEYS
    with gc.switches(**dict.fromkeys(keys)):
        yield


# ---- kernel identity --------------------------------------------------------------------------------------------------
_GEMM_LINE = re.compile(r"\[umma_gemm\] [^\n]*?\bbn=(\d+) splitk=(\d+) units=(\d+) [^\n]*?\btma_store=(\d) [^\n]*?\bepi=(\w+)( chain=\d+)?")
_HALO_LINE = re.compile(r"\[umma_halo\] [^\n]*?: bn=(\d+) T=(\d+) R=(\d+) tb=(\d+) P=(\d+) units=(\d+)")


def parse_lines(err):
    gemm = [dict(bn=int(b), splitk=int(k), units=int(u), tma_store=int(t), epi=e, chain=int(c.split("=")[1]) if c else 0)
            for b, k, u, t, e, c in _GEMM_LINE.findall(err)]
    halo = [dict(bn=int(b), T=int(t), R=int(r), tb=int(tb), P=int(p), units=int(u)) for b, t, r, tb, p, u in _HALO_LINE.findall(err)]
    return gemm, halo


def _kernel_probe():
    import torch
    import rten_b200 as rt
    n_sms = torch.cuda.get_device_properties(0).multi_processor_count
    ctx = rt.Context(0)
    res = {}
    for s in specs(n_sms):
        pl = place(ctx, s, prepare(s))

        def call():
            run_case(rt, ctx, s, pl, n_sms)
            ctx.sync()
        for _ in range(3):  # a capture with no kernel record at all is taken again (see rk.capture_kernels)
            got, err = gc.run_verbose(lambda: dk._launches(call))
            if got:
                break
        res[spec_id(s)] = dict(launches=got, err=err)
    print(json.dumps({"sms": n_sms, "runs": res}))


def check_identity(s, r, run):
    """None when the recorded launches and verbose line are what rule `r` names, else a description"""
    ours = [(kernel_key(n), g, b) for n, g, b in run["launches"] if kernel_key(n) is not None]
    if [k for k, _, _ in ours] != [r["key"]]:
        return f"ran {[k for k, _, _ in ours]}, rule {r['key']}"
    _, g, b = ours[0]
    if (g is not None and g != r["grid"]) or (b is not None and b != r["block"]):
        return f"grid {g} block {b}, rule {r['grid']} / {r['block']}"
    gemm, halo = parse_lines(run["err"])
    lines = halo if r["key"][0] == "umma_halo_kernel" else gemm
    if lines != [r["line"]]:
        return f"printed {lines}, rule {r['line']}"
    return None


def test_kernel_identity():
    out = rk.probe_in_child("test_gpu_wgmma_kernels")
    n_sms, runs = out["sms"], out["runs"]
    seen, wrong = {}, []
    for s in specs(n_sms):
        r = case_rule(s, n_sms)
        err = check_identity(s, r, runs[spec_id(s)])
        if err:
            wrong.append((spec_id(s), err))
            continue
        seen.setdefault(r["key"], []).append(spec_id(s))
    assert not wrong, f"{len(wrong)} cases ran other kernels, grids or plans than the rule names: {wrong[:8]}"
    missing = [(k, a) for k, args in VARIANTS.items() for a in args if len(seen.get((k, a), ())) < 2]
    assert not missing, f"instances that fewer than two cases ran: {missing}"
    assert not coverage_gaps(n_sms)
    for k, args in VARIANTS.items():
        for a in args:
            print(f"  {k}<{', '.join(map(str, a))}>: {'; '.join(seen[(k, a)])}")
    print(f"19 of 19 instances ran, each at least twice, on {n_sms} SMs")


# ---- values -----------------------------------------------------------------------------------------------------------
def _check(got, want, what):
    for i, (g, w) in enumerate(zip(got, want)):
        gc.assert_bit_exact(g, w, f"{what}: output {i}")


def test_values_bit_exact(rt, sms):
    ctx = rt.Context(0)
    worst, failed = 99.0, []
    for s in specs(sms):
        inp = prepare(s)
        want, margin = wgmma_model(s, inp)
        assert margin > 0, f"{spec_id(s)}: the data is not exact in every order (margin {margin:.2f} bits)"
        worst = min(worst, margin)
        pl = place(ctx, s, inp)
        for attempt in ("first run", "rerun"):
            pl.poison()
            run_case(rt, ctx, s, pl, sms)
            got, clean = pl.read()
            try:
                _check(got, want, f"{spec_id(s)} ({attempt})")
            except AssertionError as ex:
                failed.append(str(ex))
            if clean:
                failed.append(f"{spec_id(s)} ({attempt}): {len(clean)} values outside the output views changed: {clean[:8]}")
    assert not failed, f"{len(failed)} failures: " + "\n".join(failed)
    print(f"{len(specs(sms))} cases bit-exact, twice each; smallest exactness margin {worst:.1f} bits")


def graph_cases(sms):
    """the largest split-K case and one case per kernel"""
    ss = specs(sms)
    pick = [next(s for s in ss if s.get("sk") == "max")]
    for base in VARIANTS:
        pick.append(next(s for s in ss if case_rule(s, sms)["key"][0] == base and s not in pick))
    return pick


def test_graph_replay(rt, sms):
    ctx = rt.Context(0)
    for s in graph_cases(sms):
        inp = prepare(s)
        want, _ = wgmma_model(s, inp)
        pl = place(ctx, s, inp)
        run_case(rt, ctx, s, pl, sms)  # (first run outside the capture: one-time weight packing and splits)
        ctx.sync()
        with gc.switches(**_env(s)):
            ctx.graph_begin()
            run_case(rt, ctx, s, pl, sms)
            graph = ctx.graph_end()
        for i in range(2):
            pl.poison()
            ctx.sync()
            graph.launch()
            ctx.sync()
            got, clean = pl.read()
            _check(got, want, f"{spec_id(s)}: graph replay {i + 1}")
            assert not clean, f"{spec_id(s)}: graph replay {i + 1} wrote outside the output views: {clean[:8]}"


def test_full_mantissa_within_the_tf32_bound(rt, sms):
    """Full-mantissa operands: the result depends on the K order, so it is held to the TF32 (3xTF32) bound against
    float64 -- one case per kernel, and a 3xTF32 one"""
    ctx = rt.Context(0)
    r = _rng("full mantissa")
    cases = [(s, x3) for s, x3 in ((_mm("full narrow", 300, 200, 96, bn=64, bias=True), False),
                                   (_mm("full narrow x3", 300, 200, 96, bn=64, bias=True, x3=True), True),
                                   (_mm("full wide", 260, 256, 256, bn=128, bias=True), False),
                                   (_halo("full halo", 2, 32, 20, 20, 64, (3, 3), (1, 1, 1, 1), bias=True), False))]
    for s, x3 in cases:
        s = dict(s, x3=x3)
        inp = prepare(dict(s, x3=False))
        for k in ("a", "b", "x", "w"):
            if k in inp:
                inp[k] = r.uniform(-1, 1, inp[k].shape).astype(F32)
        pl = place(ctx, s, inp)
        run_case(rt, ctx, s, pl, sms)
        got, clean = pl.read()
        assert not clean, clean[:8]
        if s["op"] == "mm":
            exact = _product(s, inp["a"], inp["b"]) + inp["bias"]
            absum = _product(s, np.abs(inp["a"]), np.abs(inp["b"]))
        else:
            exact = (_conv_f64(inp["x"], inp["w"], s["pads"], 1, 1) + inp["bias"]).transpose(0, 3, 1, 2)
            absum = _conv_f64(np.abs(inp["x"]), np.abs(inp["w"]), s["pads"], 1, 1).transpose(0, 3, 1, 2)
        with gc.bound(not x3):
            worst = gc.assert_tf32_close(got[0], exact, absum, spec_id(s))
        print(f"  {spec_id(s)}: error / bound {worst:.3f}")
