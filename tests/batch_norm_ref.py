"""Test infrastructure: restatement of the reference's BatchNormalization in float32, bit for bit, and of the executor's
load-time fold of a BatchNormalization into the Conv / ConvTranspose before it.

  batch_norm  src/ops/norm.rs batch_norm_in_place (normalize_each_channel -> normalize_slice -> Normalize's arm for a
              static mean and variance, rten-vecmath/src/normalize.rs): per channel c, the channel being axis 1 of a
              rank >= 2 input and the whole of a rank-1 input,
                s = scale[c] / sqrt(var[c] + epsilon)      (a rounded add, a correctly rounded sqrt and division)
                y = fma(x - mean[c], s, bias[c])           (the subtraction rounded, then one fused multiply-add)
              then the activation, if any
  fold_conv   the folded convolution's weights and bias:
                w'[co, ..] = w[co, ..] * s[co]             (ConvTranspose: weight axis 1, co = g (C_out / G) + j)
                b'[co] = fma(bias[co] - mean[co], s[co], beta[co])   (bias 0 without one)

Errors mirror the reference's OpError kinds and messages."""
from __future__ import annotations

from typing import Optional

import numpy as np

from oracle.norms import fma_f32
from oracle.oracle import OpError

_F32 = np.float32


def channel_scale(scale, var, epsilon: Optional[float] = None):
    """s = scale / sqrt(var + epsilon), float32, each step rounded"""
    eps = _F32(1e-5 if epsilon is None else epsilon)
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        return (np.asarray(scale, _F32) / np.sqrt(np.asarray(var, _F32) + eps)).astype(_F32)


def batch_norm(x, scale, bias, mean, var, epsilon: Optional[float] = None, activation=None):
    """BatchNormalization (src/ops/norm.rs batch_norm), then `activation` (None, or a function of one float32 array such
    as oracle.activations.silu)"""
    x = np.asarray(x, _F32)
    params = [np.asarray(p, _F32) for p in (scale, bias, mean, var)]
    if x.ndim < 1:
        raise OpError("InvalidValue", "Input must have at least 1 dim")
    chans = x.shape[1] if x.ndim >= 2 else 1
    for name, p in zip(("scale", "bias", "mean", "var"), params):
        if p.shape[0] != chans:
            raise OpError("IncompatibleInputShapes", f"{name}.size(0) != channels")
    scale, bias, mean, var = params
    s = channel_scale(scale, var, epsilon)
    cshape = (1, chans) + (1,) * (x.ndim - 2) if x.ndim >= 2 else (1,)
    with np.errstate(invalid="ignore", over="ignore"):
        d = (x - mean.reshape(cshape)).astype(_F32)
        y = fma_f32(d, np.broadcast_to(s.reshape(cshape), x.shape), np.broadcast_to(bias.reshape(cshape), x.shape))
    y = np.asarray(y, _F32).reshape(x.shape)
    return y if activation is None else np.asarray(activation(y), _F32)


def fold_conv(w, b, scale, beta, mean, var, epsilon: Optional[float] = None, transpose: bool = False, groups: int = 1):
    """(w', b') of a Conv (w [C_out, C_in / G, k..]) or ConvTranspose (w [C_in, C_out / G, k..]) with bias b (or None)
    followed by BatchNormalization(scale, beta, mean, var, epsilon)"""
    w = np.asarray(w, _F32)
    s = channel_scale(scale, var, epsilon)
    if transpose:
        cin, cpg = w.shape[:2]
        co = (np.arange(cin) // (cin // groups))[:, None] * cpg + np.arange(cpg)[None, :]  # [C_in, C_out / G]
        sw = s[co].reshape(co.shape + (1,) * (w.ndim - 2))
    else:
        sw = s.reshape((-1,) + (1,) * (w.ndim - 1))
    with np.errstate(invalid="ignore", over="ignore"):
        wf = (w * sw).astype(_F32)
        b = np.zeros(len(s), _F32) if b is None else np.asarray(b, _F32)
        bf = fma_f32((b - np.asarray(mean, _F32)).astype(_F32), s, np.asarray(beta, _F32))
    return wf, np.asarray(bf, _F32)
