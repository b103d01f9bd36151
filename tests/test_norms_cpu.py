"""CPU checks of the RMSNormalization / skip layer norm restatement (oracle/norms.py) that the GPU tests compare against
bit for bit: the reference's known answers (tests/golden/norm_cases.json: the contrib.rs shape, optional-output and
invalid cases, norm.rs test_rms_normalization), and its Normalize arms and fused multiply-add against the C oracle's
LayerNormalization."""
import ctypes as C
import json
import os

import numpy as np
import pytest

from oracle import norms, oracle

HERE = os.path.dirname(os.path.abspath(__file__))
CASES = json.load(open(os.path.join(HERE, "golden", "norm_cases.json")))
f32 = np.float32


def eq_1e4(a, b):
    """src/ops/mod.rs expect_eq_1e4: atol 1e-4, rtol 0"""
    return np.asarray(a).shape == np.asarray(b).shape and bool(np.all(np.abs(np.asarray(a) - np.asarray(b)) <= 1e-4))


def arr(v, shape=None):
    return None if v is None else (np.asarray(v, f32) if shape is None else np.asarray(v, f32).reshape(shape))


@pytest.mark.parametrize("i", range(len(CASES["shape_cases"])))
def test_skip_layer_norm_shape_cases(i):
    c = CASES["shape_cases"][i]
    out, s = norms.skip_layer_norm(arr(c["input"], c["input_shape"]), arr(c["skip"], c["skip_shape"]), arr(c["gamma"]),
                                   arr(c["beta"]), arr(c["bias"]), c["epsilon"], rms=c["op"] == "simplified")
    assert eq_1e4(out, arr(c["expected"], c["input_shape"]))


@pytest.mark.parametrize("op", ["standard", "simplified"])
def test_skip_layer_norm_optional_outputs(op):
    c = next(c for c in CASES["optional_outputs"] if c["op"] == op)
    out, s = norms.skip_layer_norm(arr(c["input"]), arr(c["skip"]), arr(c["gamma"]), arr(c["beta"]), arr(c["bias"]),
                                   c["epsilon"], rms=op == "simplified")
    assert np.array_equal(s, arr(c["expected_sum"]))
    assert eq_1e4(out, arr(c["expected"]))


@pytest.mark.parametrize("rms", [False, True])
@pytest.mark.parametrize("i", range(len(CASES["invalid"])))
def test_skip_layer_norm_invalid(i, rms):
    c = CASES["invalid"][i]
    with pytest.raises(oracle.OpError) as e:
        norms.skip_layer_norm(np.zeros(c["input_shape"], f32), np.zeros(c["skip_shape"], f32), np.zeros(c["gamma_shape"], f32),
                              None, None, 1e-5, rms=rms)
    assert (e.value.kind, e.value.msg) == (c["kind"], c["msg"])


def test_skip_layer_norm_bias_length():
    """The one deviation: the reference panics inside add_in_place"""
    with pytest.raises(oracle.OpError) as e:
        norms.skip_layer_norm(np.zeros((2, 4), f32), np.zeros((2, 4), f32), np.ones(4, f32), None, np.ones(3, f32), 1e-5)
    assert (e.value.kind, e.value.msg) == ("InvalidValue", "bias length must equal the hidden size")


def test_rms_normalization_formula():
    c = CASES["rms"]
    assert eq_1e4(norms.rms_norm(arr(c["input"]), arr(c["scale"]), c["axis"], c["epsilon"]), arr(c["expected"]))


def test_rms_scale_broadcast_errors():
    with pytest.raises(oracle.OpError) as e:
        norms.rms_norm(np.ones((2, 3), f32), np.ones(4, f32))
    assert e.value.msg == "`scale` is not broadcastable to normalized axes of input"
    with pytest.raises(oracle.OpError) as e:
        norms.rms_norm(np.ones((2, 3), f32), np.ones(3, f32), axis=2)
    assert e.value.msg == "Axis is invalid"


def test_fma_f32_is_exactly_rounded():
    """Against exact rational arithmetic on products that straddle float32 rounding boundaries"""
    from fractions import Fraction
    r = np.random.default_rng(7)
    a = r.standard_normal(4000).astype(f32)
    b = (r.standard_normal(4000) * 1e-3).astype(f32)
    c = r.standard_normal(4000).astype(f32)
    got = norms.fma_f32(a, b, c)
    for x, y, z, g in zip(a, b, c, got):
        exact = Fraction(float(x)) * Fraction(float(y)) + Fraction(float(z))
        lo = np.float32(float(exact))
        cands = [np.nextafter(lo, np.float32(-np.inf)), lo, np.nextafter(lo, np.float32(np.inf))]
        best = min(cands, key=lambda v: (abs(Fraction(float(v)) - exact), int(np.float32(v).view(np.int32)) & 1))
        assert g == best, (x, y, z, g, best)


def _sum(rows):
    f = oracle.lib().rto_sum
    return np.array([f(r.ctypes.data_as(C.POINTER(C.c_float)), r.size) for r in np.ascontiguousarray(rows)], f32)


@pytest.mark.parametrize("n", [64, 100, 768])
def test_normalize_arms_match_the_c_layer_norm(n):
    """The numpy arms (with fma_f32) reproduce rto_layer_norm's three arms bit for bit, given its statistics"""
    r = oracle.XorShiftRng(11)
    x = r.uniform((9, n), -3.0, 3.0)
    x[0] = 0.0
    x[1, :3] = [-0.0, 1e-30, -1e-30]
    g, b = r.uniform((n,), 0.5, 1.5), r.uniform((n,), -0.5, 0.5)
    f = norms._sum_square_sub()
    with np.errstate(invalid="ignore"):
        mean = _sum(x) / f32(n)
        var = np.array([f(row.ctypes.data_as(C.POINTER(C.c_float)), n, m) for row, m in zip(x, mean)], f32) / f32(n)
        for gamma, gs, beta, bs in ((None, 2.0, None, 0.5), (None, 2.0, None, 0.0), (g, 1.0, None, 0.0), (g, 1.0, b, 0.0),
                                    (None, 1.5, b, 0.0), (g, 1.0, None, 0.25)):
            rstd = f32(gs) / np.sqrt(var + f32(1e-5))
            want = oracle.layer_norm(x, g if gamma is not None else f32(gs), b if beta is not None else (f32(bs) if bs else None),
                                     -1, 1e-5)
            got = norms.normalize_arms(x, mean, rstd, gamma, beta, bs)
            assert np.array_equal(got.view(np.int32), want.view(np.int32)), (gamma is None, beta is None, bs)


def test_rms_special_rows():
    """All-zero rows normalise to zeros (only epsilon keeps rstd finite); an inf makes rstd 0, so only its own element
    becomes inf * 0 = NaN; a NaN poisons its row; -0.0 keeps its sign under the multiply arm"""
    x = np.zeros((3, 64), f32)
    x[1, 5] = np.inf
    x[2, 0] = np.nan
    x[0, 1] = -0.0
    g = np.ones(64, f32)
    with np.errstate(invalid="ignore"):
        y = norms.rms_norm(x, g, -1, 1e-6)
    assert np.all(y[0] == 0) and np.signbit(y[0, 1])
    assert np.isnan(y[1, 5]) and np.all(np.delete(y[1], 5) == 0)
    assert np.all(np.isnan(y[2]))
