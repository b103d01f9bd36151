"""CPU-only: the kernel table of tests/test_gpu_conv_norm_resize_kernels.py is exactly the set of depthwise, GroupNorm,
Resize / Concat, ReduceSum and rotary kernel instances compiled into the library (its sm_90a symbols, demangled), and its
case lists select every instance at least twice, once with a partial last unit, and reach every runtime mode.  An
instance added without a test, or one removed, fails here before any GPU time is spent."""
import pytest

import test_gpu_conv_norm_resize_kernels as ck
from test_row_kernel_table_cpu import compiled_instances, lib_path  # noqa: F401  (lib_path: a fixture)


def test_variant_table_matches_the_library(lib_path):  # noqa: F811
    found = compiled_instances(lib_path, ck.KERNELS, ck.kernel_key)
    for base, args in ck.VARIANTS.items():
        assert len(set(args)) == len(args), f"{base}: duplicate entries in the table"
        assert set(args) == found.get(base, set()), (
            f"{base}: compiled but not in the table {sorted(found.get(base, set()) - set(args))}, "
            f"in the table but not compiled {sorted(set(args) - found.get(base, set()))}")
    # 30 depthwise, 5 GroupNorm, 9 Resize / Concat, 8 ReduceSum, 2 rotary
    assert sum(len(v) for v in ck.VARIANTS.values()) == 54


@pytest.mark.parametrize("sms", [132, 114])
def test_cases_reach_every_kernel(sms):
    """The rules over the case lists for an H100 SXM (132 SMs) and PCIe (114 SMs): every instance at least twice, once
    with a partial last unit, and every runtime mode"""
    assert not ck.coverage_gaps(sms)


def test_kernel_key_spellings():
    k = ck.kernel_key
    assert k("void rtb::(anonymous namespace)::depthwise_cl_kernel<signed char, unsigned char, 2, 4>(rtb::DepthwiseParams, "
             "int, int, int, long long)") == ("depthwise_cl_kernel", ("signed char", "unsigned char", 2, 4))
    assert k("void rtb::<unnamed>::depthwise_cl_kernel<signed char, unsigned char, (int)2, (int)4>(rtb::DepthwiseParams, "
             "int, int, int, long long)") == ("depthwise_cl_kernel", ("signed char", "unsigned char", 2, 4))
    assert k("rtb::gn_stats_kernel(const float *, rtb::GroupNormParams, long long, int, float2 *)") == ("gn_stats_kernel", ())
    assert k("rtb::(anonymous namespace)::rotary_kernel(rtb::(anonymous namespace)::RotaryParams)") == ("rotary_kernel", ())
    assert k("void rtb::gn_apply_kernel<true>(rtb::GroupNormParams, const float2 *, int, int)") == ("gn_apply_kernel", (1,))
    assert k("void rtb::gn_apply_kernel<(bool)0>(rtb::GroupNormParams, const float2 *, int, int)") == ("gn_apply_kernel", (0,))
    assert k("void rtb::<unnamed>::reduce_sum_cta_kernel<float, (bool)1>(rtb::ReduceParams)") == ("reduce_sum_cta_kernel", ("float", 1))
    assert k("void rtb::(anonymous namespace)::concat_kernel<uint4>(rtb::ConcatParams)") == ("concat_kernel", ("uint4",))
    assert k("void rtb::<unnamed>::concat_kernel<unsigned int>(rtb::ConcatParams)") == ("concat_kernel", ("unsigned int",))
    assert k("void rtb::nd_copy_kernel<unsigned int>(const T1 *, T1 *, rtb::NdParams)") is None
    assert k("void rtb::<unnamed>::arg_reduce_cta_kernel<float>(rtb::SelectParams)") is None
