"""CPU checks of the BatchNormalization restatement (tests/batch_norm_ref.py) that the GPU tests compare against bit for
bit: the reference's known answers (tests/golden/batch_norm_cases.json, norm.rs test_batch_norm), its error messages,
its arithmetic against a float64 evaluation, and the load-time Conv / ConvTranspose fold against the unfolded pair."""
import json
import os

import numpy as np
import pytest

import batch_norm_ref as ref
from oracle.oracle import OpError

HERE = os.path.dirname(os.path.abspath(__file__))
CASES = json.load(open(os.path.join(HERE, "golden", "batch_norm_cases.json")))
f32 = np.float32


@pytest.mark.parametrize("i", range(len(CASES["cases"])))
def test_batch_norm_reference_case(i):
    c = CASES["cases"][i]
    got = ref.batch_norm(np.asarray(c["input"], f32), *(np.asarray(c[k], f32) for k in ("scale", "bias", "mean", "var")),
                         c["epsilon"])
    want = np.asarray(c["expected"], f32)
    assert got.shape == want.shape
    assert np.all(np.abs(got - want) <= CASES["atol"])


def test_batch_norm_errors():
    p = [np.ones(2, f32)] * 4
    with pytest.raises(OpError) as e:
        ref.batch_norm(np.float32(1.0), *p)
    assert (e.value.kind, e.value.msg) == ("InvalidValue", "Input must have at least 1 dim")
    for k, name in enumerate(("scale", "bias", "mean", "var")):
        q = list(p)
        q[k] = np.ones(3, f32)
        with pytest.raises(OpError) as e:
            ref.batch_norm(np.ones((2, 2, 3), f32), *q)
        assert (e.value.kind, e.value.msg) == ("IncompatibleInputShapes", f"{name}.size(0) != channels")


@pytest.mark.parametrize("shape", [(2, 5, 3, 7), (4, 6), (3, 4, 9), (11,)])
def test_batch_norm_is_one_fma_per_element(shape):
    """y is the float64 value of (x - mean) * s + bias with x - mean and s rounded to float32, rounded once"""
    r = np.random.default_rng(len(shape))
    x = r.standard_normal(shape).astype(f32)
    C = shape[1] if len(shape) > 1 else 1
    scale, bias, mean = (r.standard_normal(C).astype(f32) for _ in range(3))
    var = r.uniform(0, 2, C).astype(f32)
    got = ref.batch_norm(x, scale, bias, mean, var, 1e-3)
    s = (scale / np.sqrt(var + f32(1e-3))).astype(f32)
    cs = (1, C) + (1,) * (len(shape) - 2) if len(shape) > 1 else (1,)
    d = (x - mean.reshape(cs)).astype(f32)
    exact = d.astype(np.float64) * s.reshape(cs).astype(np.float64) + bias.reshape(cs).astype(np.float64)
    assert np.all(np.abs(got.astype(np.float64) - exact) <= np.spacing(np.abs(exact).astype(f32)).astype(np.float64) / 2)


def test_activation_follows():
    from oracle import activations
    x = np.linspace(-3, 3, 24, dtype=f32).reshape(2, 3, 4)
    p = [np.array(v, f32) for v in ([1, 2, 3], [0.5, -0.5, 0], [0, 1, -1], [1, 0.5, 2])]
    y = ref.batch_norm(x, *p)
    assert ref.batch_norm(x, *p, activation=activations.silu).tobytes() == activations.silu(y).tobytes()


def _conv64(x, w, b, groups, transpose):
    import torch
    import torch.nn.functional as F
    t = lambda a: torch.from_numpy(np.asarray(a, np.float64))  # noqa: E731
    f = F.conv_transpose2d if transpose else F.conv2d
    return f(t(x), t(w), None if b is None else t(b), groups=groups).numpy()


@pytest.mark.parametrize("cin,cout,groups,transpose,bias", [(6, 8, 1, False, True), (6, 8, 1, False, False),
                                                           (6, 8, 2, False, True), (8, 8, 8, False, True),
                                                           (6, 8, 1, True, True), (6, 8, 2, True, False)])
def test_fold_equals_conv_then_batch_norm(cin, cout, groups, transpose, bias):
    """The folded convolution computes the convolution followed by the normalization, up to the rounding of w * s"""
    r = np.random.default_rng(cin * cout + groups + transpose)
    x = r.standard_normal((2, cin, 5, 5)).astype(f32)
    w = r.standard_normal((cin, cout // groups, 3, 3) if transpose else (cout, cin // groups, 3, 3)).astype(f32)
    b = r.standard_normal(cout).astype(f32) if bias else None
    scale, beta, mean = (r.standard_normal(cout).astype(f32) for _ in range(3))
    var = r.uniform(0.1, 2, cout).astype(f32)
    wf, bf = ref.fold_conv(w, b, scale, beta, mean, var, 1e-5, transpose=transpose, groups=groups)
    assert wf.shape == w.shape and bf.shape == (cout,)
    got = _conv64(x, wf, bf, groups, transpose)
    y = _conv64(x, w, b, groups, transpose)
    s = (scale.astype(np.float64) / np.sqrt(var.astype(np.float64) + 1e-5))[None, :, None, None]
    want = (y - mean[None, :, None, None]) * s + beta[None, :, None, None]
    assert np.abs(got - want).max() <= 1e-5 * (1 + np.abs(want).max())
    # the folded bias is the operator applied to the convolution bias
    b0 = np.zeros(cout, f32) if b is None else b
    assert bf.tobytes() == ref.batch_norm(b0[None, :], scale, beta, mean, var, 1e-5)[0].tobytes()
