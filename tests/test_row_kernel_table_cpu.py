"""CPU-only: the variant table of tests/test_gpu_row_kernels.py is exactly the set of Softmax, row normalization,
skinny-GEMM and quantized-linear kernel instances compiled into the library (its sm_90a symbols, demangled), and its
case lists select every instance at least twice.  An instance added without a test, or one removed, fails here before
any GPU time is spent."""
import os
import subprocess

import pytest

import test_gpu_row_kernels as rk


@pytest.fixture(scope="module")
def lib_path():
    from rten_b200 import _build
    return _build.build()


def _cuda_tool(name):
    from rten_b200 import _build
    return os.path.join(os.path.dirname(_build._nvcc()), name)


def compiled_instances(lib, kernels=None, key=None):
    """{kernel: its compiled template argument tuples} over the kernels `key` (default rk.kernel_key) accepts
    (`kernels`, default the four families of tests/test_gpu_row_kernels.py)"""
    syms = subprocess.run([_cuda_tool("cuobjdump"), "-symbols", lib], capture_output=True, text=True, check=True).stdout
    mangled = [ln.split()[-1] for ln in syms.splitlines() if "STT_FUNC" in ln]
    names = subprocess.run([_cuda_tool("cu++filt")], input="\n".join(mangled), capture_output=True, text=True, check=True).stdout
    found = {}
    for name in names.splitlines():
        k = (key or rk.kernel_key)(name, kernels)
        if k is not None:
            found.setdefault(k[0], set()).add(k[1])
    return found


def test_variant_table_matches_the_library(lib_path):
    found = compiled_instances(lib_path)
    for base, args in rk.VARIANTS.items():
        assert len(set(args)) == len(args), f"{base}: duplicate entries in the table"
        assert set(args) == found.get(base, set()), (
            f"{base}: compiled but not in the table {sorted(found.get(base, set()) - set(args))}, "
            f"in the table but not compiled {sorted(set(args) - found.get(base, set()))}")
    for base in rk.GENERIC:
        assert found.get(base) == {()}, f"{base} is not compiled"
    assert sum(len(v) for v in rk.VARIANTS.values()) == 149


@pytest.mark.parametrize("sms", [132, 114])
def test_cases_reach_every_instance(sms):
    """The rules over the case lists for an H100 SXM (132 SMs) and PCIe (114 SMs): every instance at least twice, every
    skinny instance over two column tiles per CTA, every double-buffered quantized-linear instance over three."""
    assert not rk.coverage_gaps(sms)


def test_quantized_linear_operand_combinations():
    """The epilogue operands of the quantized-linear cases vary independently: every pair of residual and activation,
    of weight zero point and bias, and (on the cases with a layer norm) of weight zero point and layer-norm bias."""
    specs = rk.qlinear_specs(132)
    pairs = lambda a, b, ss: {(s[a], s[b]) for s in ss}
    assert pairs("res", "act", specs) == {(r, a) for r in (False, True) for a in range(4)}
    assert pairs("wz", "bias", specs) == {(w, b) for w in (None, "scalar", "vec") for b in (False, True)}
    assert pairs("wz", "ln_beta", [s for s in specs if s["ln"]]) == {(w, b) for w in (None, "scalar", "vec") for b in (False, True)}
    assert {s["scalar_scale"] for s in specs} == {False, True}


def test_kernel_key_spellings():
    assert rk.kernel_key("void rtb::softmax_vec_kernel<4, 2>(rtb::SoftmaxParams)") == ("softmax_vec_kernel", (4, 2))
    assert rk.kernel_key("void rtb::softmax_vec_kernel<(int)4, (int)2>(rtb::SoftmaxParams)") == ("softmax_vec_kernel", (4, 2))
    assert rk.kernel_key("void rtb::qlinear_kernel<16, 4, 2, true, 8, true>(rtb::QLinearParams)") == ("qlinear_kernel", (16, 4, 2, 1, 8, 1))
    assert rk.kernel_key("void rtb::qlinear_kernel<(int)8, (int)1, (int)6, (bool)0, (int)6, (bool)0>(rtb::QLinearParams)") == (
        "qlinear_kernel", (8, 1, 6, 0, 6, 0))
    assert rk.kernel_key("rtb::norm_kernel(rtb::NormParams)") == ("norm_kernel", ())
    assert rk.kernel_key("void rtb::norm_vec_kernel<1, 4, 2>(rtb::NormParams)") == ("norm_vec_kernel", (1, 4, 2))
    assert rk.kernel_key("void rtb::norm_wide_kernel<(int)8, (int)15>(rtb::NormParams)") == ("norm_wide_kernel", (8, 15))
