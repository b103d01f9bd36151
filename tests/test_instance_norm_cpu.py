"""CPU checks of the InstanceNormalization / GroupNorm restatement (tests/instance_norm_ref.py) that the GPU tests
compare against bit for bit: the reference's known answer (tests/golden/instance_norm_cases.json, norm.rs test_instance_normalization),
its error messages, its statistics against the C oracle's LayerNormalization -- which folds a row in the same order and
takes a scalar scale and bias through the same Normalize arm -- and the GroupNorm chain against its own node-by-node
restatement."""
import json
import os

import numpy as np
import pytest

import instance_norm_ref as ref
from oracle import activations, oracle

HERE = os.path.dirname(os.path.abspath(__file__))
CASES = json.load(open(os.path.join(HERE, "golden", "instance_norm_cases.json")))
f32 = np.float32


@pytest.mark.parametrize("i", range(len(CASES["cases"])))
def test_instance_norm_reference_case(i):
    c = CASES["cases"][i]
    got = ref.instance_norm(np.asarray(c["input"], f32), np.asarray(c["scale"], f32), np.asarray(c["bias"], f32), c["epsilon"])
    want = np.asarray(c["expected"], f32)
    assert got.shape == want.shape
    assert np.all(np.abs(got - want) <= c["atol"])


@pytest.mark.parametrize("L", [1, 16, 49, 63, 64, 100, 196, 784, 4096, 4100])
def test_instance_norm_rows_are_layer_norm_rows(L):
    """Each (n, c) lane is LayerNormalization of that lane with scalar scale[c] and bias[c]: same fold order (full
    64-element chunks, 16-element chunks, masked tail), same arm, same bits."""
    r = np.random.default_rng(L)
    x = (r.standard_normal((2, 3, L)) * 3 + 0.5).astype(f32)
    scale, bias = r.uniform(0.5, 2, 3).astype(f32), r.uniform(-1, 1, 3).astype(f32)
    got = ref.instance_norm(x, scale, bias, 1e-3)
    for n in range(2):
        for c in range(3):
            want = oracle.layer_norm(x[n, c], scale[c:c + 1], bias[c:c + 1], -1, 1e-3)
            assert got[n, c].tobytes() == want.tobytes()


def test_instance_norm_spatial_dims_are_one_lane():
    r = np.random.default_rng(3)
    x = r.standard_normal((2, 4, 5, 7)).astype(f32)
    s, b = r.standard_normal(4).astype(f32), r.standard_normal(4).astype(f32)
    assert ref.instance_norm(x, s, b).tobytes() == ref.instance_norm(x.reshape(2, 4, 35), s, b).reshape(x.shape).tobytes()


@pytest.mark.parametrize("x_shape, s_len, b_len, msg", [
    ((4,), 4, 4, "expected input with >= 2 dims"),
    ((1, 4, 3), 3, 4, "scale length should match channel count"),
    ((1, 4, 3), 4, 5, "bias length should match channel count"),
])
def test_instance_norm_errors(x_shape, s_len, b_len, msg):
    with pytest.raises(oracle.OpError) as e:
        ref.instance_norm(np.zeros(x_shape, f32), np.ones(s_len, f32), np.zeros(b_len, f32))
    assert e.value.kind == "InvalidValue" and msg in str(e.value)


@pytest.mark.parametrize("act", [None, activations.silu, activations.sigmoid])
def test_group_norm_is_the_node_chain(act):
    r = np.random.default_rng(7)
    N, C, H, W, G = 2, 12, 5, 6, 3
    x = r.standard_normal((N, C, H, W)).astype(f32)
    s, b = r.uniform(0.5, 1.5, G).astype(f32), r.uniform(-0.5, 0.5, G).astype(f32)
    gamma, beta = r.standard_normal(C).astype(f32), r.standard_normal(C).astype(f32)
    got = ref.group_norm(x, G, s, b, gamma, beta, 1e-6, act)
    y = ref.instance_norm(x.reshape(N, G, -1), s, b, 1e-6).reshape(x.shape)
    y = y * gamma.reshape(1, C, 1, 1)
    y = y + beta.reshape(1, C, 1, 1)
    if act is not None:
        y = act(y)
    assert got.dtype == f32 and got.tobytes() == np.asarray(y, f32).tobytes()


def test_group_norm_channels_not_divisible():
    with pytest.raises(oracle.OpError) as e:
        ref.group_norm(np.zeros((1, 6, 2, 2), f32), 4, np.ones(4, f32), np.zeros(4, f32))
    assert "Input length must be a multiple of specified dimensions" in str(e.value)
