"""CPU-only: the numpy oracle of the mask and layout operators (tests/mask_ops.py) reproduces the expected values in
tests/golden/mask_ops_cases.json, the kernel table of tests/test_gpu_mask_ops.py is exactly the set of masks.cu kernels
compiled into the library, and every `__global__` kernel of masks.cu is in that table."""
import os

import numpy as np
import pytest

import mask_ops as mo
import test_gpu_mask_ops as gm
from test_row_kernel_table_cpu import compiled_instances, lib_path  # noqa: F401  (lib_path: a fixture)
from test_kernel_names_cpu import library_kernels

MASKS = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "rten_b200", "csrc", "masks.cu")


def _arr(v, dtype):
    return np.array(v, np.int32 if dtype == "i32" else np.float32)


def _run(c):
    dt = c.get("dtype", "f32")
    op = c["op"]
    if op == "Where":
        return mo.where(np.array(c["cond"], np.int32), _arr(c["x"], dt), _arr(c["y"], dt))
    if op in ("Equal", "Less", "LessOrEqual", "Greater", "GreaterOrEqual"):
        return mo.compare(op, _arr(c["a"], dt), _arr(c["b"], dt))
    if op in ("And", "Or", "Xor"):
        return mo.logical(op, _arr(c["a"], dt), _arr(c["b"], dt))
    if op == "Not":
        return mo.not_(_arr(c["a"], dt))
    if op == "Trilu":
        return mo.trilu(np.array(c["input"], np.int32), c["k"], c["upper"])
    if op == "Expand":
        return mo.expand(_arr(c["input"], dt), c["shape"])
    if op == "Split":
        return mo.split(_arr(c["input"], dt), c["axis"], c["split"], c["num_outputs"])
    if op == "Slice":
        return mo.slice_(_arr(c["input"], dt), c["starts"], c["ends"], c["axes"], c["steps"])
    if op == "ConstantOfShape":
        return mo.constant_of_shape(c["value"], c["shape"], np.int32 if dt == "i32" else np.float32)
    if op == "Range":
        return mo.range_(c["start"], c["limit"], c["delta"], np.int32 if dt == "i32" else np.float32)
    raise KeyError(op)


@pytest.mark.parametrize("case", mo.cases(), ids=lambda c: f"{c['op']}: {c['name']}")
def test_oracle_reproduces_the_reference_cases(case):
    if "error" in case:
        with pytest.raises(mo.OpFailed) as e:
            _run(case)
        assert str(e.value) == case["error"]
        return
    got = _run(case)
    if isinstance(got, list):
        assert len(got) == len(case["expected"])
        for g, e in zip(got, case["expected"]):
            np.testing.assert_array_equal(g, np.array(e, g.dtype))
    else:
        np.testing.assert_array_equal(got, np.array(case["expected"], got.dtype))


def test_comparison_oracle_is_ieee():
    a = np.array([np.nan, 0.0, -0.0, np.inf, 1e-45, 1e-45], np.float32)
    b = np.array([np.nan, -0.0, 0.0, np.inf, 0.0, 1e-45], np.float32)
    assert mo.compare("Equal", a, b).tolist() == [0, 1, 1, 1, 0, 1]
    assert mo.compare("Greater", a, b).tolist() == [0, 0, 0, 0, 1, 0]


def test_host_arithmetic_rules():
    assert mo.host_arith("Add", [2 ** 31 - 1], [1]).tolist() == [-2 ** 31]
    assert mo.host_arith("Mul", [65536], [65536]).tolist() == [0]
    assert mo.host_arith("Div", [-7, 7], [2, -2]).tolist() == [-3, -3]
    assert mo.host_arith("Sub", [2 ** 40], [0]).tolist() == [2 ** 31 - 1]  # int64 saturated as the loader does
    with pytest.raises(mo.OpFailed, match="Divisor contains zero"):
        mo.host_arith("Div", [1, 2], [1, 0])


def test_kernel_table_matches_the_library(lib_path):  # noqa: F811
    found = compiled_instances(lib_path, gm.KERNELS)
    for base, args in gm.VARIANTS.items():
        assert set(args) == found.get(base, set()), (base, sorted(found.get(base, set())), sorted(args))
    assert set(found) == set(gm.VARIANTS)


def test_every_masks_kernel_is_in_the_table():
    names = set(library_kernels([MASKS]))
    assert len(names) >= 6, sorted(names)
    assert names == set(gm.VARIANTS), (sorted(names - set(gm.VARIANTS)), sorted(set(gm.VARIANTS) - names))
