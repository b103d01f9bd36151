"""CPU checks of the depthwise convolution and Clip restatements (oracle/depthwise.py) and of their C ABI surface:

  * the reference's known answer `test_conv_depthwise` (src/ops/conv.rs:990-1030);
  * the f32 oracle against a float64 7-deep loop (the reference's reference_conv, padded taps skipped) within 1e-5, and
    the integer oracle exactly, on the sweep of tests/depthwise_sweep.py, for every signedness pair, x zero points
    0 / 12 / 255 (u8) or -128 (i8) and w zero points absent, scalar or per channel;
  * the f32 oracle's tap order: bias first, then (ky, kx), padded taps skipped (-0.0 and infinite weights);
  * the Clip rule: NaN, +-inf, +-0.0, missing bounds, i32;
  * the ABI table and the ONNX summary of a Clip node."""
import ctypes
import json
import os

import numpy as np
import pytest

import depthwise_sweep as sw

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def oracle():
    from oracle import oracle as o
    return o


@pytest.fixture(scope="module")
def dw():
    from oracle import depthwise as d
    return d


def test_known_answer(dw):
    # src/ops/conv.rs:990-1030 (test_conv_depthwise): groups = 3, one input channel per output channel
    x = np.array([0.5946, 0.8249, 0.0448, 0.9552, 0.2041, 0.2501, 0.2693, 0.1007, 1.5202, 1.5592, 0.9939, 1.7475],
                 np.float32).reshape(1, 3, 2, 2)
    w = np.array([-0.0862, -0.4111, 0.0813, 0.4993, -0.4641, 0.1715, -0.0532, -0.2429, -0.4325, 0.4273, 0.4180, 0.4338],
                 np.float32).reshape(3, 1, 2, 2)
    bias = np.array([0.1, 0.2, 0.3], np.float32)
    want = np.array([0.09020272 + 0.1, -0.09061745 + 0.2, 1.1822754 + 0.3], np.float32).reshape(1, 3, 1, 1)
    got = dw.depthwise_conv(x, w, bias)
    assert got.dtype == np.float32 and got.shape == (1, 3, 1, 1)
    assert np.allclose(got, want, atol=1e-4, rtol=0)


@pytest.mark.parametrize("case", sw.SWEEP, ids=sw.IDS)
def test_f32_oracle_against_float64_loop(oracle, dw, case):
    x, w, b = sw.f32_data(oracle, case)
    for bias in (b, None):
        got = dw.depthwise_conv(x, w, bias, **sw.op_args(case))
        want = sw.loop_reference(x, w, bias, case)
        assert got.shape == want.shape and got.dtype == np.float32
        assert np.allclose(got, want, atol=1e-5, rtol=1e-5), f"{case[0]}: max err {np.abs(got - want).max()}"


PAIRS = [(np.uint8, np.uint8), (np.uint8, np.int8), (np.int8, np.uint8), (np.int8, np.int8)]


@pytest.mark.parametrize("pair", PAIRS, ids=lambda p: f"{np.dtype(p[0]).name}x{np.dtype(p[1]).name}")
@pytest.mark.parametrize("case", sw.SWEEP, ids=sw.IDS)
def test_integer_oracle_against_loop(dw, case, pair):
    xdt, wdt = pair
    x, w = sw.int_data(case, xdt, wdt)
    C = w.shape[0]
    xzs = [0, 12, 255] if xdt == np.uint8 else [0, 12, -128]
    wz_forms = [None, np.array(7 if wdt == np.uint8 else -3, wdt),
                np.arange(C).astype(np.int64).__mod__(200).astype(wdt)]
    for xz in xzs:
        for wz in wz_forms:
            got = dw.depthwise_conv_integer(x, w, np.array(xz, xdt), wz, **sw.op_args(case))
            want = sw.loop_reference(x, w, None, case, x_zp=xz, w_zp=wz)
            assert got.dtype == np.int32
            np.testing.assert_array_equal(got, want, err_msg=f"{case[0]} xz={xz} wz={wz}")


def test_f32_order_bias_then_taps_skipping_padding(dw):
    # a padded tap is skipped, not multiplied by 0: an infinite weight on a tap that only ever reads padding leaves
    # the output finite, and an output whose taps are all padding is the bias itself (-0.0 included)
    x = np.ones((1, 2, 1, 1), np.float32)
    w = np.zeros((2, 1, 3, 3), np.float32)
    w[:, 0, 1, 1] = 2.0
    w[:, 0, 0, 0] = np.inf
    bias = np.array([-0.0, 1.5], np.float32)
    y = dw.depthwise_conv(x, w, bias, padding=(1, 1, 1, 1))
    np.testing.assert_array_equal(y.reshape(-1), [2.0, 3.5])
    y = dw.depthwise_conv(x, w, bias, padding=(3, 3, 3, 3))  # 5x5 outputs; the corners see only padding
    assert np.signbit(y[0, 0, 0, 0]) and y[0, 0, 0, 0] == 0.0
    assert y[0, 1, 0, 0] == 1.5 and y[0, 0, 2, 2] == 2.0 and y[0, 1, 2, 2] == 3.5
    # no bias: +0.0 start, so (+0.0) + (-0.0 * 1) = +0.0
    xz = np.full((1, 1, 1, 1), -0.0, np.float32)
    y = dw.depthwise_conv(xz, np.ones((1, 1, 1, 1), np.float32), None, padding=(0, 0, 0, 0))
    assert not np.signbit(y.reshape(-1)[0])
    # ky-major order: the sum is formed bias, then (0,0), (0,1), (1,0), (1,1), each rounded
    x = np.array([1e8, 1.0, -1e8, 1.0], np.float32).reshape(1, 1, 2, 2)
    y = dw.depthwise_conv(x, np.ones((1, 1, 2, 2), np.float32), np.array([0.5], np.float32))
    acc = np.float32(0.5)
    for v in x.reshape(-1):
        acc = np.float32(acc + np.float32(v * np.float32(1.0)))
    assert y.reshape(-1)[0] == acc


def test_integer_to_float_rounding_order(dw):
    acc = np.array([[[[7, -3]], [[1 << 24 | 1, 0]]]], np.int32)  # [1, 2, 1, 2]
    got = dw.integer_to_float(acc, np.float32(0.1), scale_b=np.float32(3.0), bias=np.array([0.25, -1.0], np.float32),
                              relu=True)
    sv = np.float32(np.float32(3.0) * np.float32(0.1))
    want = acc.astype(np.float32) * sv + np.array([0.25, -1.0], np.float32).reshape(1, 2, 1, 1)
    want = np.where(want > 0, want, np.float32(0))
    np.testing.assert_array_equal(got, want)


def test_clip_rule(dw):
    x = np.array([np.nan, np.inf, -np.inf, -0.0, 0.0, -1.0, 0.5, 7.0], np.float32)
    y = dw.clip(x, np.float32(0.0), np.float32(6.0))
    np.testing.assert_array_equal(y, [0.0, 6.0, 0.0, 0.0, 0.0, 0.0, 0.5, 6.0])
    assert not np.signbit(y[3]), "-0.0 clipped at min = +0.0 is +0.0 (x > min is false)"
    y = dw.clip(x, None, np.float32(6.0))  # NaN becomes the missing min: f32::MIN
    assert y[0] == np.finfo(np.float32).min and y[2] == np.finfo(np.float32).min and y[1] == 6.0
    y = dw.clip(x, np.float32(-0.5), None)
    assert y[0] == -0.5 and y[1] == np.finfo(np.float32).max and np.signbit(y[3]) and y[5] == -0.5
    y = dw.clip(x)
    assert y[0] == np.finfo(np.float32).min and y[1] == np.finfo(np.float32).max
    xi = np.array([-(2**31), -5, 0, 5, 2**31 - 1], np.int32)
    np.testing.assert_array_equal(dw.clip(xi, np.int32(-2), np.int32(3)), [-2, -2, 0, 3, 3])
    np.testing.assert_array_equal(dw.clip(xi, None, np.int32(3)), [-(2**31), -5, 0, 3, 3])


def test_clip_in_the_abi_table():
    from rten_b200 import _build, _lib
    src = open(os.path.join(ROOT, "include", "rten_b200.h")).read()
    assert "rten_b200_clip(" in src
    assert "rten_b200_clip" in _lib.declared_symbols()
    lib = ctypes.CDLL(_build.build())
    assert hasattr(lib, "rten_b200_clip")
    import rten_b200 as rt
    assert hasattr(rt, "Clip")


def test_onnx_summary_of_a_clip_node():
    import sys
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    import onnx_writer as ow
    from rten_b200 import _lib
    nodes = [ow.node("Clip", ["x", "lo", ""], ["y"], name="relu6"), ow.node("Clip", ["y"], ["z"], name="legacy", min=0.0, max=6.0)]
    model = ow.model(nodes, [ow.tensor("lo", np.array(0.0, np.float32))], [ow.value_info("x", 1, [1, 4])],
                     [ow.value_info("z", 1, [1, 4])])
    lib = _lib.load()
    buf = ctypes.create_string_buffer(1 << 16)
    need = ctypes.c_size_t(0)
    assert lib.rten_b200_onnx_summary(model, len(model), buf, len(buf), ctypes.byref(need)) == 0
    s = json.loads(buf.value.decode())
    assert "Clip" in json.dumps(s)
