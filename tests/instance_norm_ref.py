"""Test infrastructure: restatement of the reference's InstanceNormalization and of the GroupNorm node chain torch
exports, float32, bit for bit, built on the C oracle's folds and oracle/norms.py's exactly rounded fused multiply-add.

  instance_norm  src/ops/norm.rs instance_normalization: x made contiguous, each (n, c) lane of L elements normalised
                 with mean = Sum / L, var = SumSquareSub(mean) / L (the C oracle's rto_sum / rto_sum_square_sub, the
                 reference's fold_unroll<4> x 16-lane order), rstd = scale[c] / sqrt(var + epsilon),
                 y = fma(x - mean, rstd, bias[c]) (Normalize's arm 0)
  group_norm     Reshape(x, [N, G, -1]) -> InstanceNormalization -> Reshape back -> Mul(gamma[c]) -> Add(beta[c]) ->
                 activation, each step rounded on its own

Errors mirror the reference's OpError kinds and messages."""
from __future__ import annotations

import ctypes as C
from typing import Optional

import numpy as np

from oracle import oracle
from oracle.norms import fma_f32
from oracle.oracle import OpError

_F32 = np.float32


def _folds():
    lib = oracle.lib()
    fq = lib.rto_sum_square_sub
    fq.restype = C.c_float
    fq.argtypes = [C.POINTER(C.c_float), C.c_size_t, C.c_float]
    return lib.rto_sum, fq


def instance_norm(x, scale, bias, epsilon: Optional[float] = None):
    """InstanceNormalization (src/ops/norm.rs instance_normalization_in_place)"""
    x = np.ascontiguousarray(x, _F32)
    scale, bias = np.asarray(scale, _F32), np.asarray(bias, _F32)
    if scale.ndim != 1 or bias.ndim != 1:
        raise OpError("CastFailed", "scale and bias must be 1-D tensors")
    if x.ndim < 2:
        raise OpError("InvalidValue", "expected input with >= 2 dims")
    chans = x.shape[1]
    if scale.shape[0] != chans:
        raise OpError("InvalidValue", "scale length should match channel count")
    if bias.shape[0] != chans:
        raise OpError("InvalidValue", "bias length should match channel count")
    eps = _F32(1e-5 if epsilon is None else epsilon)
    if x.size == 0:
        return np.empty_like(x)
    rows = x.reshape(x.shape[0] * chans, -1)
    L = rows.shape[1]
    fs, fq = _folds()
    ptr = lambda r: r.ctypes.data_as(C.POINTER(C.c_float))  # noqa: E731
    mean = np.array([fs(ptr(r), L) for r in rows], _F32) / _F32(L)
    var = np.array([fq(ptr(r), L, float(m)) for r, m in zip(rows, mean)], _F32) / _F32(L)
    ch = np.arange(len(rows)) % chans
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        rstd = scale[ch] / np.sqrt(var + eps)
        y = fma_f32(rows - mean[:, None], rstd[:, None], np.broadcast_to(bias[ch][:, None], rows.shape))
    return y.reshape(x.shape)


def group_norm(x, groups: int, inst_scale, inst_bias, gamma=None, beta=None, epsilon: Optional[float] = None,
               activation=None):
    """The GroupNorm node chain: InstanceNormalization of x as [N, groups, -1], then * gamma[c], + beta[c] and the
    activation (None, or a function of one float32 array such as oracle.activations.silu)"""
    x = np.ascontiguousarray(x, _F32)
    if x.ndim < 2:
        raise OpError("InvalidValue", "expected input with >= 2 dims")
    chans = x.shape[1]
    if groups <= 0 or chans % groups:
        raise OpError("InvalidValue", "Input length must be a multiple of specified dimensions")
    y = instance_norm(x.reshape(x.shape[0], groups, -1), inst_scale, inst_bias, epsilon).reshape(x.shape)
    cshape = (1, chans) + (1,) * (x.ndim - 2)
    with np.errstate(invalid="ignore", over="ignore"):
        if gamma is not None:
            y = (y * np.asarray(gamma, _F32).reshape(cshape)).astype(_F32)
        if beta is not None:
            y = (y + np.asarray(beta, _F32).reshape(cshape)).astype(_F32)
    return y if activation is None else np.asarray(activation(y), _F32)
