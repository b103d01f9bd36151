"""CPU-only: the ReduceSum restatement the GPU tests compare against, and the onnxruntime-genai decoder file they load.

  * genai_decoder.sum_ref is the C oracle's rto_sum bit for bit at every length 0-300 and on long lanes, with mixed
    magnitudes, -0.0, +-inf and NaN;
  * genai_decoder.reduce_sum_ref with sum_ref gives the bits it gives with rto_sum in every branch of the reference's
    `reduce`: contiguous inner chunks, a single axis, permuted multi-axis slices, all axes, negative and repeated axes,
    keepdims 0 / 1, a 0-D input and empty reductions;
  * the genai-shaped decoder reads back with genai's names and int64 types, the attention-mask subgraph and the int64
    constants it needs."""
import ctypes as C

import numpy as np
import pytest

import genai_decoder as gd
import onnx_writer as W

F32 = np.float32


@pytest.fixture(scope="module")
def rto_sum(oracle):
    f = oracle.lib().rto_sum

    def s(v):
        v = np.ascontiguousarray(v, F32).reshape(-1)
        return F32(f(v.ctypes.data_as(C.POINTER(C.c_float)), v.size))
    return s


def _bits(a, b):
    return np.asarray(a, F32).view(np.uint32).tobytes() == np.asarray(b, F32).view(np.uint32).tobytes()


def _lane(r, n):
    v = (r.standard_normal(n) * np.exp2(r.integers(-20, 20, n))).astype(F32)
    if n > 3:
        v[r.integers(0, n)] = -0.0
    return v


def test_sum_ref_is_the_oracle_sum(rto_sum):
    r = np.random.default_rng(5)
    for n in list(range(0, 301)) + [1023, 1024, 1025, 4095, 4096, 4097, 8193, 70001]:
        v = _lane(r, n)
        assert _bits(gd.sum_ref(v), rto_sum(v)), n
    special = np.array([3e38, 3e38, -3e38, 1.0, -0.0] * 20, F32)
    for v in (special, np.array([np.inf, -np.inf] + [1.0] * 70, F32), np.array([1.0] * 65 + [np.nan], F32), np.array([-0.0], F32)):
        assert _bits(gd.sum_ref(v), rto_sum(v))


@pytest.mark.parametrize("keepdims", [0, 1])
def test_reduce_sum_ref_branches(rto_sum, keepdims):
    r = np.random.default_rng(6)
    x = (r.standard_normal((3, 5, 7, 70)) * 100).astype(F32)
    cases = [(x, [3]), (x, [2, 3]), (x, [-1, -2]), (x, [1]), (x, [0, 2]), (x, [1, 3]), (x, [0, 1, 2]), (x, None), (x, [2, 2, -2]),
             (np.ascontiguousarray(x.transpose(0, 2, 3, 1)).transpose(0, 3, 1, 2), [1, 2, 3]),
             (r.standard_normal((2, 0, 3)).astype(F32), [1]), (r.standard_normal((2, 0, 3)).astype(F32), [0])]
    for a, axes in cases:
        got = gd.reduce_sum_ref(a, axes, keepdims)
        want = gd.reduce_sum_ref(a, axes, keepdims, lane_sum=rto_sum)
        ref = np.sum(a.astype(np.float64), axis=tuple(gd.resolve_axes(a.ndim, axes)), keepdims=bool(keepdims))
        assert got.shape == ref.shape, (axes, got.shape, ref.shape)
        assert _bits(got, want), axes
        assert np.allclose(got, ref, rtol=1e-5, atol=1e-2), axes
    assert _bits(gd.reduce_sum_ref(np.array(-0.0, F32)), F32(0.0))
    with pytest.raises(ValueError, match="Axis is invalid"):
        gd.reduce_sum_ref(x, [4])


def test_genai_decoder_file():
    from rten_b200.model import onnx_summary
    from test_gpu_norms import DEC as c
    s = onnx_summary(gd.genai_graph(gd.genai_weights()))
    ops = [n["op"] for n in s["nodes"]]
    assert ops[:6] == ["ReduceSum", "Sub", "Cast", "Shape", "Gather", "Cast"], ops
    assert ops.count("GroupQueryAttention") == c["L"] and ops.count("MatMulNBits") == 1 + 3 + 4 * c["L"] + 1, ops
    gqa = [n for n in s["nodes"] if n["op"] == "GroupQueryAttention"]
    assert gqa[0]["inputs"][:3] == ["qkv0", "", ""] and gqa[1]["inputs"][:3] == ["q1", "k1", "v1"]
    assert all(g["inputs"][5:7] == ["seqlens_k", "total_seq_len"] for g in gqa)
    ins = {v["name"]: v["elem_type"] for v in s["inputs"]}
    assert ins["input_ids"] == W.INT64 and ins["attention_mask"] == W.INT64
    assert ins["past_key_values.0.key"] == W.FLOAT and ins[f"past_key_values.{c['L'] - 1}.value"] == W.FLOAT
    assert [v["name"] for v in s["outputs"]] == gd.output_names()
    inits = {t["name"]: t for t in s["initializers"]}
    assert inits["/model/axes_1"]["data_type"] == W.INT64 and inits["/model/axes_1"]["dims"] == [1]
    assert inits["/model/index_1"]["data_type"] == W.INT64 and inits["/model/index_1"]["dims"] == []
    assert inits["/model/one"]["data_type"] == W.INT64
    cast = [n for n in s["nodes"] if n["op"] == "Cast"]
    assert [n["outputs"] for n in cast] == [["seqlens_k"], ["total_seq_len"]]
