"""CPU checks of the Resize / Upsample / AveragePool / Concat test infrastructure (no GPU): the numpy restatement
oracle/resize.py against the reference's own test tables (tests/golden/resize_cases.json) and against
torch.nn.functional.interpolate / avg_pool2d as a second witness, the output-size and error cases, and the ONNX writer /
reader round trip of the new nodes and their attributes."""
import json
import os

import numpy as np
import pytest

import onnx_writer as W
from oracle import resize as R

HERE = os.path.dirname(os.path.abspath(__file__))
F32 = np.float32


@pytest.fixture(scope="module")
def golden():
    with open(os.path.join(HERE, "golden", "resize_cases.json")) as f:
        return json.load(f)


def _arr(shape, data):
    return np.array(data, F32).reshape(shape)


def test_resize_nearest_tables(golden):
    g = golden["resize_nearest"]
    for c in g["cases"]:
        y = R.resize(_arr(c["shape"], c["input"]), scales=c["scales"], mode="nearest", coord_mode=g["coord_mode"],
                     nearest_mode=g["nearest_mode"])
        assert list(y.shape) == c["expected_shape"]
        assert np.array_equal(y, _arr(c["expected_shape"], c["expected"]))


def test_resize_nearest_mode_table(golden):
    g = golden["resize_nearest_mode"]
    x = _arr(g["shape"], g["input"])
    for c in g["cases"]:
        y = R.resize(x, scales=g["scales"], mode="nearest", coord_mode=g["coord_mode"], nearest_mode=c["nearest_mode"])
        assert np.array_equal(y, _arr(g["expected_shape"], c["expected"])), c["nearest_mode"]


def test_resize_bilinear_tables(golden):
    g = golden["resize_bilinear"]
    x = _arr(g["shape"], g["input"])
    for c in g["cases"]:
        y = R.resize(x, scales=c["scales"], mode="linear", coord_mode=c["coord_mode"], nearest_mode=g["nearest_mode"])
        assert list(y.shape) == c["expected_shape"]
        np.testing.assert_allclose(y, _arr(c["expected_shape"], c["expected"]), atol=g["atol"], rtol=0)
    g = golden["resize_non_integer_scale"]
    x = _arr(g["shape"], g["input"])
    for c in g["cases"]:
        y = R.resize(x, scales=g["scales"], mode=c["mode"], coord_mode=g["coord_mode"], nearest_mode=g["nearest_mode"])
        np.testing.assert_allclose(y, _arr(g["expected_shape"], c["expected"]), atol=g["atol"], rtol=0)


def test_upsample_tables(golden):
    g = golden["upsample"]
    x = _arr(g["shape"], g["input"])
    for c in g["cases"]:
        np.testing.assert_allclose(R.upsample(x, g["scales"], c["mode"]), _arr(g["expected_shape"], c["expected"]),
                                   atol=g["atol"], rtol=0)


def test_resize_scales_sizes_and_errors(golden):
    for c in golden["resize_scales_sizes"]["cases"]:
        x = np.ones(c["shape"], F32)
        if "error" in c:
            with pytest.raises(R.ResizeError) as e:
                R.resize(x, scales=c.get("scales"), sizes=c.get("sizes"), mode="linear")
            assert [e.value.kind, str(e.value)] == c["error"]
        else:
            assert list(R.resize(x, scales=c.get("scales"), sizes=c.get("sizes"), mode="linear").shape) == c["expected_shape"]


def test_output_size_arithmetic():
    # floor(in as f32 * scale) in f32: 10 * 0.7f32 = 7.0000005 -> 7; 5 * 1.7 -> 8; 1 / scale and in / out are f32 quotients
    sizes, inv = R.calc_output_size([1, 3, 10, 5], scales=[1, 1, 0.7, 1.7])
    assert sizes == [1, 3, 7, 8]
    assert inv[2] == F32(1.0) / F32(0.7) and inv[3] == F32(1.0) / F32(1.7)
    sizes, inv = R.calc_output_size([1, 3, 10, 5], sizes=[1, 3, 33, 1])
    assert sizes == [1, 3, 33, 1] and inv[2] == F32(10) / F32(33) and inv[3] == F32(5.0)
    with pytest.raises(R.ResizeError):
        R.calc_output_size([1, 3, 10, 5], sizes=[1, 3, -1, 5])


def test_one_pixel_align_corners_is_nan_like_the_reference():
    # dest * (in - 1) / (out - 1) = 0 * 3 / 0: NaN survives f32::clamp, indexes pixel 0, and poisons the bilinear weight
    x = np.arange(8, dtype=F32).reshape(1, 1, 2, 4)
    assert np.isnan(R.resize(x, sizes=[1, 1, 2, 1], mode="linear", coord_mode="align_corners")).all()
    y = R.resize(x, sizes=[1, 1, 2, 1], mode="nearest", coord_mode="align_corners")
    assert np.array_equal(y.reshape(-1), [0, 4])


@pytest.mark.parametrize("scale", [2.0, 0.5, 1.7, (2.0, 3.0)])
@pytest.mark.parametrize("align", [False, True])
def test_linear_against_torch(scale, align):
    import torch
    import torch.nn.functional as TF
    rng = np.random.default_rng(7)
    x = rng.standard_normal((2, 3, 9, 11)).astype(F32)
    sy, sx = scale if isinstance(scale, tuple) else (scale, scale)
    y = R.resize(x, scales=[1, 1, sy, sx], mode="linear", coord_mode="align_corners" if align else "half_pixel")
    want = TF.interpolate(torch.from_numpy(x), size=y.shape[2:], scale_factor=None, mode="bilinear", align_corners=align)
    if not align:  # torch derives its scale from the sizes unless told the factor
        want = TF.interpolate(torch.from_numpy(x), scale_factor=(sy, sx), mode="bilinear", align_corners=False,
                              recompute_scale_factor=False)
    # torch rounds the coordinate of a non-dyadic scale differently (its 1 / 1.7 weights differ in the last bits)
    tol = 1e-5 if scale == 1.7 else 1e-6
    np.testing.assert_allclose(y, want.numpy(), atol=tol, rtol=tol)


@pytest.mark.parametrize("scale", [2.0, 3.0, 0.5])
def test_nearest_asymmetric_floor_against_torch(scale):
    import torch
    import torch.nn.functional as TF
    x = np.random.default_rng(8).standard_normal((2, 3, 8, 6)).astype(F32)
    y = R.resize(x, scales=[1, 1, scale, scale], mode="nearest", coord_mode="asymmetric", nearest_mode="floor")
    want = TF.interpolate(torch.from_numpy(x), scale_factor=scale, mode="nearest")
    assert np.array_equal(y, want.numpy())


def test_average_pool_tables(golden):
    g = golden["average_pool"]
    x = _arr(g["shape"], g["input"])
    for c in g["cases"]:
        y = R.average_pool(x, c["kernel"], strides=c["strides"])
        np.testing.assert_allclose(y, _arr(c["expected_shape"], c["expected"]), atol=g["atol"], rtol=0)
    g = golden["average_pool_padding"]
    x = np.broadcast_to(np.array(g["rows"], F32), (1, g["channels"], 4, 4))
    for key, cip in (("expected", False), ("expected_include_pad", True)):
        y = R.average_pool(x, g["kernel"], g["pads"], g["strides"], cip)
        np.testing.assert_allclose(y, np.broadcast_to(np.array(g[key], F32), y.shape), atol=g["atol"], rtol=0)


@pytest.mark.parametrize("cip", [False, True])
def test_average_pool_against_torch(cip):
    import torch
    import torch.nn.functional as TF
    x = np.random.default_rng(9).standard_normal((2, 5, 9, 10)).astype(F32)
    y = R.average_pool(x, (3, 3), (1, 1, 1, 1), (2, 2), cip)
    want = TF.avg_pool2d(torch.from_numpy(x), 3, 2, 1, count_include_pad=cip)
    np.testing.assert_allclose(y, want.numpy(), atol=1e-6, rtol=1e-6)


def test_concat_tables(golden):
    g = golden["concat"]
    t = {k: _arr(g[k]["shape"], g[k]["data"]) for k in ("a", "b")}
    for c in g["cases"]:
        y = R.concat([t[k] for k in c["inputs"]], c["axis"])
        assert np.array_equal(y, _arr(c["expected_shape"], c["expected"]))
    c = g["int_with_empty"]
    assert R.concat([np.array(v, np.int32) for v in c["inputs"]], c["axis"]).tolist() == c["expected"]
    for c in g["errors"]:
        with pytest.raises(R.ResizeError) as e:
            R.concat([np.zeros(s, F32) for s in c["shapes"]], c["axis"])
        assert [e.value.kind, str(e.value)] == c["error"]


def test_onnx_round_trip_of_the_new_nodes():
    from rten_b200 import _build
    _build.build()
    from rten_b200.model import onnx_summary
    nodes = [
        W.node("Resize", ["x", "", "scales"], ["r"], mode="linear", coordinate_transformation_mode="align_corners",
               nearest_mode="floor"),
        W.node("Upsample", ["x", "scales"], ["u"], mode="nearest"),
        W.node("AveragePool", ["r"], ["p"], kernel_shape=[2, 2], strides=[2, 2], pads=[0, 0, 0, 0], count_include_pad=1),
        W.node("Concat", ["p", "x"], ["y"], axis=1),
    ]
    data = W.model(nodes, [W.tensor("scales", np.array([1, 1, 2, 2], F32))], [W.value_info("x", W.FLOAT, [1, 4, 8, 8])],
                   [W.value_info("y", W.FLOAT, [1, 8, 8, 8])])
    s = onnx_summary(data)
    assert [n["op"] for n in s["nodes"]] == ["Resize", "Upsample", "AveragePool", "Concat"]
    assert s["nodes"][0]["inputs"] == ["x", "", "scales"]
    assert set(s["nodes"][0]["attrs"]) == {"mode", "coordinate_transformation_mode", "nearest_mode"}
    assert set(s["nodes"][2]["attrs"]) == {"kernel_shape", "strides", "pads", "count_include_pad"}
    assert s["initializers"][0]["dims"] == [4] and s["initializers"][0]["data_type"] == W.FLOAT
