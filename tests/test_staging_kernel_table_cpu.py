"""CPU-only: the kernel table of tests/test_gpu_staging_kernels.py is exactly the set of operand-staging kernels compiled
into the library (its sm_90a symbols, demangled), its case lists select every kernel and mode at least twice, once with a
partial last unit.  (tests/test_kernel_names_cpu.py checks that every kernel of the library is in one by-name table.)"""
import pytest

import test_gpu_row_kernels as rk
import test_gpu_staging_kernels as sk
from test_row_kernel_table_cpu import compiled_instances, lib_path  # noqa: F401  (lib_path: a fixture)


def test_variant_table_matches_the_library(lib_path):  # noqa: F811
    found = compiled_instances(lib_path, sk.KERNELS)
    for base, args in sk.VARIANTS.items():
        assert len(set(args)) == len(args), f"{base}: duplicate entries in the table"
        assert set(args) == found.get(base, set()), (
            f"{base}: compiled but not in the table {sorted(found.get(base, set()) - set(args))}, "
            f"in the table but not compiled {sorted(set(args) - found.get(base, set()))}")
    assert sum(len(v) for v in sk.VARIANTS.values()) == 28


@pytest.mark.parametrize("sms", [132, 114])
def test_cases_reach_every_kernel(sms):
    """The rules over the case lists for an H100 SXM (132 SMs) and PCIe (114 SMs): every kernel instance and runtime
    mode at least twice, once with a partial last unit"""
    assert not sk.coverage_gaps(sms)


def test_kernel_key_spellings():
    k = sk.KERNELS
    assert rk.kernel_key("void rtb::nd_copy_kernel<uint2>(const T1 *, T1 *, rtb::NdParams)", k) == ("nd_copy_kernel", ("uint2",))
    assert rk.kernel_key("void rtb::im2col_kernel<unsigned char>(const T1 *, T1 *, rtb::Im2ColParams, T1)", k) == (
        "im2col_kernel", ("unsigned char",))
    assert rk.kernel_key("void rtb::clip_kernel<int>(const T1 *, T1 *, long long, const T1 *, const T1 *, T1, T1)", k) == (
        "clip_kernel", ("int",))
    assert rk.kernel_key("rtb::tf32x3_lo_flat_kernel(const float4 *, float4 *, long long)", k) == ("tf32x3_lo_flat_kernel", ())
    assert rk.kernel_key("void rtb::binary_flat_kernel<float>(const T1 *, const T1 *, T1 *, long long, int, int, int)", k) is None
