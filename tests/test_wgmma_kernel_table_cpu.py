"""CPU-only: the kernel table of tests/test_gpu_wgmma_kernels.py is exactly the set of wgmma GEMM, wide-tile and halo
kernel instances compiled into the library (its sm_90a symbols, demangled), its case list selects every instance at
least twice and reaches every edge on an H100 SXM and PCIe, every case's data is exact in every accumulation order, the
float32 model agrees with a float64 restatement, and each plausible wrong order of operations changes the model's bits
on the case data -- so the GPU test's bit-for-bit comparison would see it in a kernel."""
import numpy as np
import pytest

import test_gpu_wgmma_kernels as wk
from test_row_kernel_table_cpu import compiled_instances, lib_path  # noqa: F401  (lib_path: a fixture)


def test_variant_table_matches_the_library(lib_path):  # noqa: F811
    found = compiled_instances(lib_path, wk.KERNELS, wk.kernel_key)
    for base, args in wk.VARIANTS.items():
        assert len(set(args)) == len(args), f"{base}: duplicate entries in the table"
        assert set(args) == found.get(base, set()), (
            f"{base}: compiled but not in the table {sorted(found.get(base, set()) - set(args), key=str)}, "
            f"in the table but not compiled {sorted(set(args) - found.get(base, set()), key=str)}")
    assert sum(len(v) for v in wk.VARIANTS.values()) == 19


@pytest.mark.parametrize("sms", [132, 114])
def test_cases_reach_every_kernel(sms):
    assert not wk.coverage_gaps(sms)


@pytest.mark.parametrize("sms", [132, 114])
def test_every_case_is_exact_in_every_order(sms):
    """From the data, not assumed: every product term of every case is a multiple of 2^-q and the sum of |terms| of
    every output is below 2^(22 - q) (two bits below the f32 significand)"""
    for s in wk.specs(sms):
        _, margin = wk.wgmma_model(s, wk.prepare(s))
        assert margin > 0, f"{s['name']}: margin {margin:.2f} bits"


def test_exactness_margin_detects_inexact_data():
    s = wk._mm("probe", 130, 64, 64, bn=64)
    inp = wk.prepare(s)
    assert wk.wgmma_model(s, inp)[1] > 0
    inp["a"] = (inp["a"] + np.float32(2.0 ** -20)).astype(np.float32)  # 24-bit operands: TF32 truncation is not exact
    inp["a"] = wk.tf32_trunc(inp["a"]) + np.float32(2.0 ** -12)
    assert wk.wgmma_model(s, inp)[1] < 0


def _f64_model(s, inp):
    """float64: the exact product of the full operands and the epilogue in float64"""
    from scipy.special import erf
    e = wk._epi_desc(s)
    if s["op"] == "gemm":
        acc = np.matmul(inp["a"].astype(np.float64), inp["b"].astype(np.float64))
        return s["alpha"] * acc + s["beta"] * inp["c"].astype(np.float64)
    acc = np.matmul(inp["a"].astype(np.float64), inp["b"].astype(np.float64))
    x = e["alpha"] * acc + (inp["res"] if "res" in inp else 0) + (inp["bias"] if "bias" in inp else 0)
    act = e["act"]
    if act == 1:
        x = np.maximum(x, 0)
    elif act == 2:
        x = 0.5 * x * (1 + erf(x / np.sqrt(2)))
    elif act == 3:
        x = 0.5 * x * (1 + np.tanh(np.sqrt(2 / np.pi) * (x + 0.044715 * x ** 3)))
    return x


@pytest.mark.parametrize("name", ["plain bias", "fast alpha", "fastgelu alpha", "plaingelu tanh", "gemm beta full C",
                                  "3xTF32 two-plane", "batched, A broadcast"])
def test_model_against_float64(name):
    s = next(c for c in wk.specs(132) if c["name"] == name)
    inp = wk.prepare(s)
    got = wk.wgmma_model(s, inp)[0][0]
    want = _f64_model(s, inp)
    assert got.dtype == np.float32 and np.isfinite(got).all()
    assert np.abs(got - want).max() <= 1e-5 * max(1.0, np.abs(want).max()), np.abs(got - want).max()


def test_integer_model_against_exact_product():
    s = next(c for c in wk.specs(132) if c["name"] == "i8 raw, za8 + zb vector")
    inp = wk.prepare(s)
    a = inp["a"].astype(np.int64) - int(inp["za"])
    b = inp["b"].astype(np.int64) - inp["zb"].astype(np.int64)
    np.testing.assert_array_equal(wk.wgmma_model(s, inp)[0][0], (a @ b).astype(np.int32))


# each deliberate slip, and a case whose data must show it
SLIPS = {"bias-before-residual": "plain bias+res relu, K tail", "alpha-after-fma": "fast alpha",
         "tf32-rne": "3xTF32 two-plane", "four-product": "3xTF32 three-segment", "kblock-drop": "split-K 2",
         "kblock-double": "plain bias", "scale-unrounded": "i8 float plain"}


@pytest.mark.parametrize("slip", sorted(SLIPS))
def test_each_slip_changes_the_bits(slip):
    s = next(c for c in wk.specs(132) if c["name"] == SLIPS[slip])
    inp = wk.prepare(s)
    good = wk.wgmma_model(s, inp)[0]
    bad = wk.wgmma_model(s, inp, perturb=(slip,))[0]
    assert any(not np.array_equal(np.asarray(g).view(np.int32), np.asarray(b, g.dtype).view(np.int32))
               for g, b in zip(good, bad)), f"{slip} leaves the bits of {s['name']} unchanged"


def test_tf32_read_of_the_chained_y_is_observable():
    """the chained z depends on TF32(y): rounding y to nearest instead of truncating changes z"""
    s = next(c for c in wk.specs(132) if c["name"] == "chain 64")
    inp = wk.prepare(s)
    good, bad = wk.wgmma_model(s, inp)[0], wk.wgmma_model(s, inp, perturb=("tf32-rne",))[0]
    assert not np.array_equal(good[1], bad[1])


def test_the_worked_anchors():
    # pick_epilogue: the variant of each operand combination
    pe = wk.pick_epilogue
    assert pe(0, 64, True, True, 1, dict(act=1, r=True)) == "PlainF32"
    assert pe(0, 64, True, True, 1, dict(act=2, alpha=0.5)) == "FastGelu"
    assert pe(0, 40, True, False, 1, dict(act=0)) == "Generic"
    assert pe(0, 64, False, False, 1, dict(act=0)) == "Generic"
    assert pe(0, 64, True, True, 1, dict(act=0, bias_kind=2)) == "Generic"
    assert pe(1, 64, True, False, 2, dict(act=1, scale=True)) == "Fast"  # PlainI8 takes no split-K
    assert pe(1, 64, True, False, 1, dict(act=3, scale=True, za8=True)) == "PlainI8Gelu"
    assert pe(1, 64, True, False, 1, dict(act=1, scale=True, zb=True)) == "Fast"
    assert pe(0, 64, True, True, 1, dict(act=1), no_plain=True) == "Fast"
    assert pe(0, 64, True, True, 1, dict(act=1), no_fast=True) == "Generic"
    # bn 256 only for act <= Relu; wide only without split-K
    assert wk.plan_valid(256, 1, 4, 2, 512, 32, True, 1, 132) and not wk.plan_valid(256, 1, 4, 2, 512, 32, True, 2, 132)
    assert wk.plan_valid(128, 1, 4, 2, 512, 32, True, 2, 132) and not wk.plan_valid(128, 2, 64, 2, 512, 32, True, 0, 132)
    assert wk.largest_splitk(256, 2, 64, 32, 132) == 16 and wk.largest_splitk(16, 2, 64, 32, 132) == 4
    # pick_conv_tile: ResNet-50 layer-1 at batch 32 fills every 128-row tile (784 M tiles, test_gpu_wide_tiles.py); of
    # the boxes that do, the first 8 pixels wide wins (8 x 1 x 16)
    tw, th, tb = wk.conv_tile(32, 56, 56, 1, 1)
    assert (tw, th, tb) == (8, 1, 16) and (56 // tw) * (56 // th) * (32 // tb) == 784
    # halo_params: tests/test_gpu_halo_wide.py WIDE_CASES (T = 2) and test_gpu_plan_space.py HALO_CASES (T = 1)
    hp = lambda B, C, H, W, N, kh, kw, bn, T: wk.halo_params(B, C, H, W, N, kh, kw, 0, 0, bn, T)  # noqa: E731
    for args, want in (((7, 64, 7, 7, 128, 3, 3), (7, 3)), ((2, 32, 28, 28, 128, 3, 3), (8, 1)),
                       ((1, 32, 5, 158, 128, 3, 3), (1, 1)), ((3, 32, 12, 12, 64, 5, 5), (12, 1)),
                       ((2, 32, 9, 13, 64, 4, 8), (9, 1))):
        p = hp(*args, 32, 2)
        assert (p["R"], p["tb"]) == want, (args, p)
    assert hp(1, 32, 5, 158, 128, 3, 3, 128, 2) is None and hp(1, 32, 4, 254, 64, 3, 3, 32, 2) is None
    assert hp(2, 64, 14, 14, 192, 3, 3, 128, 2) is None and hp(2, 64, 14, 14, 192, 3, 3, 64, 2) is not None
    for args, want in (((7, 64, 5, 5, 64, 3, 3), (5, 2)), ((8, 64, 4, 4, 64, 3, 3), (4, 3)), ((11, 64, 3, 3, 64, 3, 3), (3, 5)),
                       ((4, 64, 16, 16, 32, 3, 3), (7, 1)), ((2, 32, 6, 126, 64, 3, 3), (1, 1))):
        p = hp(*args, 32, 1)
        assert (p["R"], p["tb"]) == want, (args, p)


def test_kernel_key_spellings():
    k = wk.kernel_key
    assert k("void rtb::umma_gemm_kernel<(int)0, (rtb::Epi)3>(rtb::TmaMaps, rtb::KParams)") == ("umma_gemm_kernel", (0, "PlainF32"))
    assert k("void rtb::umma_gemm_kernel<1, rtb::Epi::PlainI8Gelu>(rtb::TmaMaps, rtb::KParams)") == ("umma_gemm_kernel", (1, "PlainI8Gelu"))
    assert k("void rtb::umma_gemm_kernel<1, (rtb::Epi)0>(rtb::TmaMaps, rtb::KParams)") == ("umma_gemm_kernel", (1, "Generic"))
    assert k("void rtb::umma_wide_kernel<(rtb::Epi)3, (int)128>(rtb::TmaMaps, rtb::KParams)") == ("umma_wide_kernel", ("PlainF32", 128))
    assert k("void rtb::umma_wide_kernel<rtb::Epi::PlainF32Gelu, 0>(rtb::TmaMaps, rtb::KParams)") == ("umma_wide_kernel", ("PlainF32Gelu", 0))
    assert k("void rtb::(anonymous namespace)::umma_halo_kernel<64, 2>(CUtensorMap_st, CUtensorMap_st, "
             "rtb::(anonymous namespace)::HaloParams)") == ("umma_halo_kernel", (64, 2))
    assert k("void rtb::<unnamed>::umma_halo_kernel<(int)32, (int)1>(CUtensorMap_st, CUtensorMap_st, "
             "rtb::<unnamed>::HaloParams)") == ("umma_halo_kernel", (32, 1))
    # the out-of-line act4 cloned into a kernel names that kernel: no new key
    assert k("[clone void rtb::umma_gemm_kernel<(int)1, (rtb::Epi)6>(rtb::TmaMaps, rtb::KParams)] rtb::act4(float4, int, "
             "float, float)") == ("umma_gemm_kernel", (1, "PlainI8Gelu"))
    assert k("void rtb::<unnamed>::skinny_f32_kernel<(int)16, (int)2>(rtb::<unnamed>::SkinnyF32Params)") is None
