"""Depthwise convolution and Clip on the CPU, restated from the reference's arithmetic.

TEST INFRASTRUCTURE ONLY, like oracle.py.

Depthwise convolution (src/ops/conv/depthwise.rs, selected at src/ops/conv.rs:269-284 when in channels == out
channels == groups and the convolution is not the pointwise case): every output starts from bias[c] (or +0.0), then for
ky, then kx, ascending, `out += x * w` as a separate multiply and add, over the taps that fall inside the image only.
numpy's float32 `*` and `+` are separate, exactly rounded operations, so the restatement below -- vectorised over every
output per tap, in that tap order, with padded taps left out by a mask -- gives the reference's bits by construction.

The integer kernel sums (x - x_zp) * (w - w_zp[c]) in wrapping i32 over the same taps: padding acts as x_zp.

Clip (src/ops/unary_elementwise.rs:249-309): x.max(min).min(max) with `a > b ? a : b` / `a < b ? a : b`.
"""
from __future__ import annotations

import numpy as np

from .oracle import OpError


def _geometry(x, w, padding, strides, dilations):
    """(x 4-D, w 4-D, OH, OW, pads [t, l, b, r], strides, dilations); a 3-D x / w is a 1-D convolution over H = 1."""
    if x.ndim == 3:
        x, w = x[:, :, None, :], w[:, :, None, :]
        padding = padding if isinstance(padding, str) else [0, padding[0], 0, padding[1]]
        strides, dilations = (1, strides[0]), (1, dilations[0])
    B, C, H, W = x.shape
    if w.shape[0] != C or w.shape[1] != 1:
        raise OpError("InvalidValue", "not a depthwise kernel ([C, 1, kh, kw])")
    kh, kw = w.shape[2], w.shape[3]
    if isinstance(padding, str):  # Padding::Same (src/ops/pooling.rs:63-137)
        pads = []
        for n, k, s, d in ((H, kh, strides[0], dilations[0]), (W, kw, strides[1], dilations[1])):
            o = -(-n // s)
            tot = max((o - 1) * s + (k - 1) * d + 1 - n, 0)
            pads.append((tot // 2, tot - tot // 2))
        pads = [pads[0][0], pads[1][0], pads[0][1], pads[1][1]]
    else:
        pads = list(padding)
    pt, pl, pb, pr = pads
    OH = (H + pt + pb - dilations[0] * (kh - 1) - 1) // strides[0] + 1
    OW = (W + pl + pr - dilations[1] * (kw - 1) - 1) // strides[1] + 1
    return x, w, OH, OW, pads, strides, dilations


def _taps(x, OH, OW, pads, strides, dilations, kh, kw):
    """Per tap (ky, kx) in the reference's order: (ky, kx, x values at every output [B, C, OH, OW], valid [OH, OW])."""
    H, W = x.shape[2], x.shape[3]
    oy, ox = np.arange(OH), np.arange(OW)
    for ky in range(kh):
        iy = oy * strides[0] - pads[0] + ky * dilations[0]
        vy = (iy >= 0) & (iy < H)
        for kx in range(kw):
            ix = ox * strides[1] - pads[1] + kx * dilations[1]
            vx = (ix >= 0) & (ix < W)
            xs = x[:, :, np.clip(iy, 0, H - 1)][:, :, :, np.clip(ix, 0, W - 1)]
            yield ky, kx, xs, vy[:, None] & vx[None, :]


def depthwise_conv(x, w, bias=None, padding=(0, 0, 0, 0), strides=(1, 1), dilations=(1, 1)):
    """f32 depthwise convolution: x [B, C, H, W] (or [B, C, W]), w [C, 1, kh, kw] (or [C, 1, kw]), bias [C]."""
    x3 = np.asarray(x).ndim == 3
    x, w, OH, OW, pads, strides, dilations = _geometry(np.asarray(x, np.float32), np.asarray(w, np.float32), padding,
                                                       strides, dilations)
    B, C = x.shape[0], x.shape[1]
    out = np.zeros((B, C, OH, OW), np.float32)
    if bias is not None:
        out[...] = np.asarray(bias, np.float32)[None, :, None, None]
    for ky, kx, xs, valid in _taps(x, OH, OW, pads, strides, dilations, w.shape[2], w.shape[3]):
        prod = xs * w[:, 0, ky, kx][None, :, None, None]
        out = np.where(valid[None, None], out + prod, out)
    return out[:, :, 0, :] if x3 else out


def depthwise_conv_integer(x, w, x_zero_point=None, w_zero_point=None, padding=(0, 0, 0, 0), strides=(1, 1),
                           dilations=(1, 1)):
    """ConvInteger, depthwise: wrapping i32 sums of (x - x_zp) * (w - w_zp[c]) over the taps inside the image only."""
    x, w = np.asarray(x), np.asarray(w)
    if x.dtype not in (np.uint8, np.int8) or w.dtype not in (np.uint8, np.int8):
        raise OpError("UnsupportedType")
    x3 = x.ndim == 3
    xz = 0 if x_zero_point is None else int(np.asarray(x_zero_point).reshape(-1)[0])
    C = w.shape[0]
    wz = np.zeros(C, np.int64) if w_zero_point is None else np.broadcast_to(np.asarray(w_zero_point).astype(np.int64).reshape(-1), (C,))
    x, w, OH, OW, pads, strides, dilations = _geometry(x.astype(np.int64) - xz, w.astype(np.int64), padding, strides,
                                                       dilations)
    wd = w - wz[:, None, None, None]
    acc = np.zeros((x.shape[0], C, OH, OW), np.int64)
    for ky, kx, xs, valid in _taps(x, OH, OW, pads, strides, dilations, w.shape[2], w.shape[3]):
        acc += np.where(valid[None, None], xs * wd[:, 0, ky, kx][None, :, None, None], 0)
    out = ((acc + 2**31) % 2**32 - 2**31).astype(np.int32)  # (a wrapped sum is the wrapped sum of the products)
    return out[:, :, 0, :] if x3 else out


def integer_to_float(acc, scale, scale_b=None, bias=None, residual=None, relu=False):
    """ConvIntegerToFloat's output and the nodes conv_integer_ex folds, each as its own f32 operation: f32(acc) *
    (scale_b * scale), + bias[c], + residual, Relu."""
    sv = np.float32(np.asarray(scale, np.float32).reshape(-1)[0])
    if scale_b is not None:
        sv = np.float32(np.float32(np.asarray(scale_b, np.float32).reshape(-1)[0]) * sv)
    y = np.asarray(acc).astype(np.float32) * sv
    shape = [1] * y.ndim
    shape[1] = -1
    if bias is not None:
        y = y + np.asarray(bias, np.float32).reshape(shape)
    if residual is not None:
        y = y + np.asarray(residual, np.float32)
    if relu:
        y = np.where(y > 0, y, np.float32(0))
    return y.astype(np.float32)


def clip(x, min=None, max=None):
    """x.max(min).min(max) for f32 or i32; a missing bound is the type's finite minimum / maximum."""
    x = np.asarray(x)
    info = np.finfo(x.dtype) if x.dtype.kind == "f" else np.iinfo(x.dtype)
    lo = x.dtype.type(info.min if min is None else np.asarray(min).reshape(-1)[0])
    hi = x.dtype.type(info.max if max is None else np.asarray(max).reshape(-1)[0])
    with np.errstate(invalid="ignore"):
        v = np.where(x > lo, x, lo)
        return np.where(v < hi, v, hi).astype(x.dtype)
