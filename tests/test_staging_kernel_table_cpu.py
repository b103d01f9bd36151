"""CPU-only: the kernel table of tests/test_gpu_staging_kernels.py is exactly the set of operand-staging kernels compiled
into the library (its sm_90a symbols, demangled), its case lists select every kernel and mode at least twice, once with a
partial last unit, and every kernel defined in rowops.cu is in exactly one of the four by-name tables (row kernels, glue,
elementwise math, staging).  A kernel added to rowops.cu without a by-name test fails here before any GPU time is spent."""
import os
import re

import pytest

import test_gpu_elementwise_math as em
import test_gpu_glue_kernels as gk
import test_gpu_row_kernels as rk
import test_gpu_staging_kernels as sk
from test_row_kernel_table_cpu import compiled_instances, lib_path  # noqa: F401  (lib_path: a fixture)

ROWOPS = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "rten_b200", "csrc", "rowops.cu")


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


_GLOBAL = re.compile(r"__global__\s+(?:void\s+)?(?:__launch_bounds__\([^)]*\)\s*)?(?:void\s+)?(\w+)\s*\(")


def global_kernels(path):
    """the names of the `__global__` functions defined in a CUDA source"""
    with open(path) as f:
        return set(_GLOBAL.findall(f.read()))


def _tables():
    return {"row kernels": set(rk.VARIANTS) | set(rk.GENERIC), "glue": set(gk.VARIANTS), "elementwise math": set(em.KERNELS),
            "staging": set(sk.VARIANTS)}


def unlisted(path):
    """(kernels of `path` in no by-name table, kernels in more than one)"""
    tables = _tables()
    names = global_kernels(path)
    homes = {n: [t for t, ks in tables.items() if n in ks] for n in names}
    return sorted(n for n, h in homes.items() if not h), sorted(n for n, h in homes.items() if len(h) > 1)


def test_every_rowops_kernel_is_tested_by_name():
    names = global_kernels(ROWOPS)
    assert len(names) >= 40, f"the parser found only {sorted(names)}"
    missing, twice = unlisted(ROWOPS)
    assert not missing, f"kernels of rowops.cu no by-name test covers: {missing}"
    assert not twice, f"kernels of rowops.cu in more than one by-name table: {twice}"


def test_the_completeness_check_reports_a_new_kernel(tmp_path):
    with open(ROWOPS) as f:
        src = f.read()
    extra = tmp_path / "rowops.cu"
    extra.write_text(src + "\nnamespace rtb {\n__global__ void __launch_bounds__(128) staged_new_kernel(const float* x) {}\n}\n")
    assert unlisted(str(extra))[0] == ["staged_new_kernel"]
