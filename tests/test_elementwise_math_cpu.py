"""CPU-only: the numpy oracles of tests/elementwise_math.py (Div, Pow, Sqrt, Reciprocal, Exp, Tanh, Neg, Abs, ReduceMean)
against the expected values of the reference's own unit tests and against the reference's rules stated one by one, and
the C ABI of the new entry points (declared in include/rten_b200.h, bound in rten_b200/_lib.py, exported by the
library)."""
import ctypes

import numpy as np
import pytest

import elementwise_math as em
import genai_decoder as gd

F32, I32 = np.float32, np.int32
NEW_ENTRY_POINTS = ["rten_b200_div", "rten_b200_pow", "rten_b200_sqrt", "rten_b200_reciprocal", "rten_b200_exp",
                    "rten_b200_tanh", "rten_b200_neg", "rten_b200_abs", "rten_b200_reduce_mean"]


@pytest.mark.parametrize("i", range(len(em.REFERENCE_CASES)))
def test_oracles_give_the_reference_tests_values(i):
    op, a, b, want = em.REFERENCE_CASES[i]
    got = em.reference_case_ref(op, a, b, want)
    assert got.shape == want.shape and got.dtype == want.dtype, (op, got.shape, want.shape)
    np.testing.assert_array_equal(got, want)


def test_div_by_one_element_is_a_times_the_reciprocal_with_a_shape():
    a = np.array([1.0, 3.0, 7.0, 1e-3], F32)
    got = em.div_ref(a, np.full((1, 1), 3.0, F32))
    assert got.shape == (4,)  # a's shape, not the broadcast [1, 4]
    np.testing.assert_array_equal(got.view(I32), (a * (F32(1) / F32(3))).view(I32))
    # two roundings differ from one somewhere: 7 * (1 / 3) is not 7 / 3 in f32
    assert (got != a / F32(3)).any()
    # a divisor of more than one element divides, with the broadcast shape
    assert em.div_ref(a, np.full((1, 4), 3.0, F32)).shape == (1, 4)
    with np.errstate(divide="ignore", invalid="ignore"):
        sp = em.div_ref(np.array([1.0, -1.0, 0.0, np.inf], F32), np.array([0.0, 0.0, 0.0, -0.0], F32))
    assert sp[0] == np.inf and sp[1] == -np.inf and np.isnan(sp[2]) and sp[3] == -np.inf


def test_i32_div_truncates_and_refuses_zero_and_overflow():
    got = em.div_ref(np.array([7, -7, 7, -7, em.IMIN], I32), np.array([2, 2, -2, -2, 1], I32))
    np.testing.assert_array_equal(got, np.array([3, -3, -3, 3, em.IMIN], I32))
    with pytest.raises(em.DivError):
        em.div_ref(np.array([1, 2], I32), np.array([1, 0], I32))
    with pytest.raises(em.DivError):
        em.div_ref(np.array([em.IMIN], I32), np.array(-1, I32))
    # a one-element i32 divisor broadcasts (no reciprocal path for integers)
    assert em.div_ref(np.array([4, 6], I32), np.full((1, 1), 2, I32)).shape == (1, 2)


def test_pow_fast_paths_and_i32_rules():
    x = np.array([1.1, -3.7, 1e20, -0.0, np.inf], F32)
    with np.errstate(over="ignore"):
        np.testing.assert_array_equal(em.pow_ref(x, F32(2)).view(I32), (x * x).view(I32))
        np.testing.assert_array_equal(em.pow_ref(x, F32(3)).view(I32), ((x * x) * x).view(I32))
    assert em.pow_ref(x, np.ones((1, 1), F32)).shape == (5,)  # map_in: the base's shape
    assert em.pow_ref(x, np.ones((1, 5), F32)).shape == (1, 5)
    got = em.pow_ref(np.array([3, -3, 7, 2, 1, -1, 0, 5], I32), np.array([0, 5, 13, 31, -3, -3, -1, -2], I32))
    want = [1, -243, (7 ** 13 + 2 ** 31) % 2 ** 32 - 2 ** 31, em.IMIN, 1, -1, em.IMAX, 0]
    np.testing.assert_array_equal(got, np.array(want, I32))
    assert em.pow_general(np.array([2, 3, 2.5, -2], F32)).tolist() == [False, False, True, True]


def test_unary_oracles():
    x = np.array([4.0, 2.0, -0.0, 0.0, -1.0, np.inf, -np.inf, np.nan, 1e-40], F32)
    with np.errstate(all="ignore"):
        sq = em.unary_ref("Sqrt", x)
        assert sq[0] == 2 and np.signbit(sq[2]) and sq[2] == 0 and np.isnan(sq[4]) and sq[5] == np.inf and np.isnan(sq[6])
        rc = em.unary_ref("Reciprocal", x)
        assert rc[0] == 0.25 and rc[2] == -np.inf and rc[3] == np.inf and rc[5] == 0 and np.signbit(rc[6])
    ng = em.unary_ref("Neg", x)
    assert np.signbit(ng[3]) and not np.signbit(ng[2]) and ng[5] == -np.inf
    ab = em.unary_ref("Abs", x)
    assert not np.signbit(ab).any() and ab[6] == np.inf
    e = em.unary_ref("Exp", np.array([0.0, 1.0, 104.0, -104.0, 88.0], F32))
    assert e[0] == 1 and abs(float(e[1]) - np.e) < 1e-6 and e[2] == np.inf and e[3] == 0 and np.isfinite(e[4])
    t = em.unary_ref("Tanh", np.array([0.0, -0.0, 9.1, -9.1, 0.3], F32))
    # (tanh.rs returns 0 - |x| for x <= 0: Tanh(-0) is +0)
    assert t[0] == 0 and not np.signbit(t[1]) and t[2] == 1 and t[3] == -1 and abs(float(t[4]) - np.tanh(0.3)) < 1e-6


def test_reduce_mean_oracle():
    r = np.random.default_rng(3)
    x = r.uniform(-2, 2, (3, 5, 70)).astype(F32)
    for axes in ([-1], [0, 2], None):
        got = em.reduce_mean_ref(x, axes, False)
        n = x.size // got.size
        np.testing.assert_array_equal(got, gd.reduce_sum_ref(x, axes, False) / F32(n))
        np.testing.assert_allclose(got, x.astype(np.float64).mean(axis=None if axes is None else tuple(axes)), rtol=1e-5, atol=1e-6)
    assert np.isnan(em.reduce_mean_ref(np.zeros((0,), F32), [0], False))  # an empty lane


def test_ulp_distance():
    one = F32(1)
    assert em.ulp_distance(np.array([one]), np.array([np.nextafter(one, F32(2))]))[0] == 1
    assert em.ulp_distance(np.array([F32(-0.0)]), np.array([F32(0.0)]))[0] == 0
    assert em.ulp_distance(np.array([np.nextafter(F32(0), F32(1))]), np.array([np.nextafter(F32(0), F32(-1))]))[0] == 2
    assert em.ulp_distance(np.array([F32(np.nan)]), np.array([F32(1)]))[0] > em.POW_ULP


def test_blocks_run_node_by_node():
    """every block's node list runs through the oracles and ends in y"""
    r = np.random.default_rng(0)
    for name, spec in em.block_specs(16).items():
        feeds = {"x": r.uniform(-2, 2, (3, 16)).astype(F32)}
        for e in spec[2]:
            feeds[e] = r.uniform(-1, 0, (3, 16)).astype(F32)
        vals = em.run_nodes(spec[0], spec[1], feeds)
        assert vals["y"].shape == (3, 16) and np.isfinite(vals["y"]).all(), name


def test_abi_declares_and_binds_the_new_entry_points():
    from test_abi_cpu import header_symbols
    from rten_b200 import _build, _lib
    syms = set(header_symbols())
    for s in NEW_ENTRY_POINTS:
        assert s in syms, f"{s} is not declared in include/rten_b200.h"
        assert s in _lib.declared_symbols(), f"{s} has no signature in rten_b200/_lib.py"
        assert hasattr(ctypes.CDLL(_build.build()), s), f"{s} is not exported"
