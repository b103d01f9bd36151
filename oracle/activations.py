"""Numpy restatement of the reference's Sigmoid, Silu, HardSigmoid and HardSwish (float32, element by element).

  Sigmoid     rten-vecmath/src/exp.rs:201-212            1 / (1 + Exp(0 - x))
  Silu        exp.rs:217-228, src/ops/unary_elementwise.rs:685-687
                                                         x / (1 + Exp(0 - x)): one division, not x * Sigmoid(x)
  HardSigmoid src/ops/unary_elementwise.rs:437-449       clamp(alpha * x + beta, 0, 1)
  HardSwish   src/ops/unary_elementwise.rs:457-469       x * clamp((1/6 as f32) * x + 0.5, 0, 1)

numpy's float32 +, -, * and / are single, exactly rounded operations, like Rust's (which never contracts a * b + c
into a fused multiply-add), and Exp is the C oracle's rto_exp (oracle.exp).  clamp is Rust's f32::clamp: `<` / `>`
comparisons, so NaN passes through and -0.0 stays -0.0 (np.clip / np.minimum would not keep both)."""
from __future__ import annotations

import numpy as np

from . import oracle

_F32 = np.float32


def sigmoid(x):
    x = np.asarray(x, _F32)
    return (_F32(1.0) / (_F32(1.0) + oracle.exp(_F32(0.0) - x))).astype(_F32)


def silu(x):
    x = np.asarray(x, _F32)
    with np.errstate(invalid="ignore"):  # Silu(-inf) = -inf / inf = NaN, as in the reference
        return (x / (_F32(1.0) + oracle.exp(_F32(0.0) - x))).astype(_F32)


def clamp01(v):
    """f32::clamp(v, 0.0, 1.0)"""
    v = np.array(v, _F32, copy=True)
    v[v < _F32(0.0)] = _F32(0.0)
    v[v > _F32(1.0)] = _F32(1.0)
    return v


def hard_sigmoid(x, alpha=0.2, beta=0.5):
    x = np.asarray(x, _F32)
    return clamp01(_F32(alpha) * x + _F32(beta))


def hard_swish(x):
    x = np.asarray(x, _F32)
    with np.errstate(invalid="ignore"):  # HardSwish(-inf) = -inf * 0 = NaN, as in the reference
        return (x * hard_sigmoid(x, _F32(1.0) / _F32(6.0), 0.5)).astype(_F32)
