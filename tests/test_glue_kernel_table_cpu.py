"""CPU-only: the kernel table of tests/test_gpu_glue_kernels.py is exactly the set of pooling, GlobalAveragePool,
broadcast-arithmetic and row gather / scatter kernels compiled into the library (its sm_90a symbols, demangled), its
case lists select every kernel and mode at least twice, and its restatement of the reference's pool output size agrees
with torch's.  A kernel added without a test, or one removed, fails here before any GPU time is spent."""
import pytest

import test_gpu_glue_kernels as gk
from test_row_kernel_table_cpu import compiled_instances, lib_path  # noqa: F401  (lib_path: a fixture)


def test_variant_table_matches_the_library(lib_path):  # noqa: F811
    found = compiled_instances(lib_path, gk.KERNELS)
    for base, args in gk.VARIANTS.items():
        assert len(set(args)) == len(args), f"{base}: duplicate entries in the table"
        assert set(args) == found.get(base, set()), (
            f"{base}: compiled but not in the table {sorted(found.get(base, set()) - set(args))}, "
            f"in the table but not compiled {sorted(set(args) - found.get(base, set()))}")
    assert sum(len(v) for v in gk.VARIANTS.values()) == 15


@pytest.mark.parametrize("sms", [132, 114])
def test_cases_reach_every_kernel(sms):
    """The rules over the case lists for an H100 SXM (132 SMs) and PCIe (114 SMs): every kernel instance, and every
    thread mapping and operation of the kernels that take one at run time, at least twice, once with a partial last
    unit"""
    assert not gk.coverage_gaps(sms)


def test_kernel_key_spellings():
    k = gk.KERNELS
    assert gk.rk.kernel_key("void rtb::binary_flat_kernel<float>(const T1 *, const T1 *, T1 *, long long, int, int, int)", k) == (
        "binary_flat_kernel", ("float",))
    assert gk.rk.kernel_key("void rtb::binary_periodic_kernel<int>(const int *, const int *, int *, unsigned int, unsigned int, "
                            "int, int)", k) == ("binary_periodic_kernel", ("int",))
    assert gk.rk.kernel_key("rtb::maxpool_cl4_kernel(const float *, float *, rtb::PoolParams)", k) == ("maxpool_cl4_kernel", ())
    assert gk.rk.kernel_key("void rtb::softmax_vec_kernel<4, 2>(rtb::SoftmaxParams)", k) is None


def test_pool_output_size_matches_torch():
    """pool_out_size against torch.nn.functional.max_pool2d's output shapes: floor and ceil mode (torch drops a last
    window that would start in the end padding as the reference does) over symmetric pads up to half the kernel, and
    SAME as an unpadded floor pool over the input padded by the pads it returns"""
    import torch
    import torch.nn.functional as F
    checked = 0
    for n in range(1, 21):
        x = torch.zeros(1, 1, n, 1)
        for k in range(1, 6):
            for s in range(1, 5):
                for p in range(0, k // 2 + 1):
                    for ceil in (False, True):
                        if n + 2 * p < k:
                            with pytest.raises(ValueError):
                                gk.pool_out_size(n, k, s, p, p, ceil)
                            continue
                        want = F.max_pool2d(x, (k, 1), (s, 1), (p, 0), ceil_mode=ceil).shape[2]
                        assert gk.pool_out_size(n, k, s, p, p, ceil) == (want, p, p), (n, k, s, p, ceil)
                        checked += 1
                out, ps, pe = gk.pool_out_size(n, k, s, 5, 5, same=True)
                assert out == -(-n // s) and pe - ps in (0, 1), (n, k, s)
                xp = F.pad(x, (0, 0, ps, pe))
                assert F.max_pool2d(xp, (k, 1), (s, 1)).shape[2] == out, (n, k, s, "SAME")
    assert checked > 1000


def test_executor_pool_pads_give_the_reference_size():
    """The explicit pads the executor tests hand the oracle give, under the floor formula, the reference's size"""
    for op, shape, attrs in gk.EXECUTOR_POOLS:
        oh, ow, (t, l, b, r) = gk.executor_pool_expect(shape, attrs)
        k, st = attrs["kernel_shape"], attrs.get("strides", [1, 1])
        assert (shape[2] + t + b - k[0]) // st[0] + 1 == oh and (shape[3] + l + r - k[1]) // st[1] + 1 == ow, (op, shape, attrs)
