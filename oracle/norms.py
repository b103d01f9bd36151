"""Restatement of the reference's RMSNormalization / SimplifiedLayerNormalization and the com.microsoft skip layer norms
(SkipLayerNormalization, SkipSimplifiedLayerNormalization), float32, bit for bit.

  rms_norm         src/ops/norm.rs rms_normalization -> layer_normalization_impl with DynamicRootMeanSquare:
                   mean 0, variance = SumSquare / n, rstd = scale / sqrt(variance + epsilon), no bias
  skip_layer_norm  src/ops/norm/contrib.rs skip_layer_normalization: s = add(x, skip), then add_in_place(s, bias) -- two
                   rounded adds -- and layer_normalization_impl over the last axis (Dynamic, or DynamicRootMeanSquare
                   for the simplified operator); output 3 (input_skip_bias_sum) is s

SumSquare (rten-vecmath/src/sum.rs) is SumSquareSub at offset 0 -- x - 0 is x for every x -- so the statistic is the C
oracle's rto_sum_square_sub(row, n, 0), in the reference's fold_unroll<4> x 16-lane order.  The statistics of the
centring variant and its output are the C oracle's rto_layer_norm.  The RMS output goes through Normalize's three arms
(rten-vecmath/src/normalize.rs:101-169) with mean 0, restated here with numpy float32 operations and an exactly rounded
fused multiply-add (`fma_f32`).

Errors mirror the reference's OpError kinds and messages.  Deviation: a bias whose length is neither the hidden size nor
1 raises InvalidValue "bias length must equal the hidden size" -- the reference panics inside add_in_place."""
from __future__ import annotations

import ctypes as C
from typing import Optional

import numpy as np

from . import oracle
from .oracle import OpError

_F32 = np.float32


def fma_f32(a, b, c):
    """float32 a * b + c with one rounding.  The float64 product of two float32 values is exact; the float64 sum is
    rounded to odd (moved one ulp towards the exact sum when it is inexact and even), which makes the final rounding to
    float32 the correctly rounded fused result (53 >= 24 + 2 bits)."""
    a64, b64, c64 = (np.asarray(v, _F32).astype(np.float64) for v in (a, b, c))
    p = a64 * b64
    with np.errstate(invalid="ignore", over="ignore"):
        s = p + c64
        bb = s - p
        err = (p - (s - bb)) + (c64 - bb)  # TwoSum: s + err == p + c64 exactly (finite s)
        odd = (s.view(np.int64) & 1) == 1
        fix = np.isfinite(s) & (err != 0) & ~odd
        s = np.where(fix, np.nextafter(s, np.where(err > 0, np.inf, -np.inf)), s)
        return s.astype(_F32)


def _sum_square_sub():
    f = oracle.lib().rto_sum_square_sub
    f.restype = C.c_float
    f.argtypes = [C.POINTER(C.c_float), C.c_size_t, C.c_float]
    return f


def sum_square(rows):
    """SumSquare of each row of a [rows, n] float32 array"""
    rows = np.ascontiguousarray(rows, _F32)
    f = _sum_square_sub()
    return np.array([f(r.ctypes.data_as(C.POINTER(C.c_float)), r.size, 0.0) for r in rows], _F32)


def normalize_arms(x, mean, rstd, gamma=None, beta=None, beta_scalar=0.0):
    """Normalize's three arms over [rows, n]: mean / rstd per row, gamma / beta per element or None"""
    x = np.asarray(x, _F32)
    mean = np.asarray(mean, _F32)[:, None]
    rstd = np.asarray(rstd, _F32)[:, None]
    bs = _F32(beta_scalar)
    with np.errstate(invalid="ignore", over="ignore"):
        d = x - mean
        if gamma is None and beta is None:
            return fma_f32(d, rstd, bs)
        if gamma is not None and beta is None and bs == 0:
            return d * (np.asarray(gamma, _F32)[None, :] * rstd)
        g = np.ones(x.shape[1], _F32) if gamma is None else np.asarray(gamma, _F32)
        b = np.zeros(x.shape[1], _F32) if beta is None else np.asarray(beta, _F32)
        return fma_f32(d, g[None, :] * rstd, np.broadcast_to(b + bs, x.shape))


def _param(p, nshape, err):
    """scale.item() for one element, else broadcast to the normalized shape (layer_normalization_impl)"""
    p = np.asarray(p, _F32)
    if p.size == 1:
        return None, float(p.reshape(-1)[0])
    try:
        return np.ascontiguousarray(np.broadcast_to(p, nshape)).reshape(-1), 1.0
    except ValueError:
        raise OpError("InvalidValue", err)


def _rms_rows(x2, gamma, gamma_scalar, eps):
    """RMSNormalization of the rows of a [rows, n] array; gamma per element (flattened) or None"""
    n = x2.shape[1]
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        var = sum_square(x2) / _F32(n)
        rstd = _F32(gamma_scalar) / np.sqrt(var + _F32(eps))
    return normalize_arms(x2, np.zeros(len(x2), _F32), rstd, gamma, None, 0.0)


def rms_norm(x, scale, axis: int = -1, epsilon: Optional[float] = None):
    """RMSNormalization / SimplifiedLayerNormalization (src/ops/norm.rs rms_normalization)"""
    x = np.ascontiguousarray(x, _F32)
    eps = 1e-5 if epsilon is None else float(epsilon)
    ax = oracle._resolve_axis(x.ndim, axis)
    nshape = x.shape[ax:]
    g, gs = _param(scale, nshape, "`scale` is not broadcastable to normalized axes of input")
    n = int(np.prod(nshape))
    if x.size == 0:
        return np.empty_like(x)
    return _rms_rows(x.reshape(-1, n), g, gs, eps).reshape(x.shape)


def skip_layer_norm(x, skip, gamma, beta=None, bias=None, epsilon: float = 1e-5, rms: bool = False):
    """(output, input_skip_bias_sum) of SkipLayerNormalization (rms False) / SkipSimplifiedLayerNormalization (rms True)"""
    x = np.asarray(x, _F32)
    skip = np.asarray(skip, _F32)
    for t in (gamma, beta, bias):
        if t is not None and np.asarray(t).ndim != 1:
            raise OpError("CastFailed", "gamma, beta and bias must be 1-D tensors")
    if x.ndim not in (2, 3):
        raise OpError("InvalidValue", "input must be 2 or 3 dimensioned")
    if skip.ndim not in (2, 3):
        raise OpError("InvalidValue", "skip must be 2 or 3 dimensioned")
    ok = skip.shape[-2:] == x.shape[-2:] and skip.ndim <= x.ndim
    if ok and skip.ndim == 3:
        ok = skip.shape[0] in (1, x.shape[0])
    if not ok:
        raise OpError("IncompatibleInputShapes", "skip must broadcast to input over the batch dimension")
    H = x.shape[-1]
    if bias is not None and np.asarray(bias).shape[0] not in (H, 1):
        raise OpError("InvalidValue", "bias length must equal the hidden size")
    s = x + np.broadcast_to(skip, x.shape)
    if bias is not None:
        s = s + np.asarray(bias, _F32)
    s = np.ascontiguousarray(s, _F32)
    if rms:
        g, gs = _param(gamma, (H,), "`scale` is not broadcastable to normalized axes of input")
        if s.size == 0:
            return np.empty_like(s), s
        return _rms_rows(s.reshape(-1, H), g, gs, epsilon).reshape(s.shape), s
    return oracle.layer_norm(s, gamma, beta, -1, epsilon), s
