"""Numpy restatement of the reference's Resize, AveragePool and Concat (float32).

  calc_output_size   src/ops/resize.rs:273-308   floor(in as f32 * scale) and 1 / scale, or in as f32 / out as f32
  resize_impl        resize.rs:350-407           1-D to 4-D inputs expanded to NCHW (NCHW; NCW before NHW; HW; W)
  input_coord        resize.rs:48-75             per coordinate transform, the operation order as written there
  nearest_resize     resize.rs:110-161           clamp, then the rounding of `round_coord`
  bilinear_resize    resize.rs:167-243           clamp, (i1, i2 = min(i1 + 1, in - 1), w = c - i1), lerp along x then y
  lerp               resize.rs:102-104           (1 - w) * a + w * b: two rounded products, one rounded sum
  average_pool       src/ops/pooling.rs:263-333, 391-417   sum of the taps inside the image from 0, one division
  concat             src/ops/concat.rs:20-85

numpy's float32 +, -, * and / are single, exactly rounded operations, like Rust's (which never contracts a * b + c into
a fused multiply-add); every product and sum below is its own np.float32 operation.  clamp is Rust's f32::clamp (`<` /
`>` comparisons): a NaN coordinate -- align_corners with a 1-pixel output is 0 * (in - 1) / 0 -- passes through, indexes
pixel 0 (`NaN as usize`) and makes the bilinear weight, hence the output, NaN, exactly as the reference does."""
from __future__ import annotations

import numpy as np

_F32 = np.float32

MODES = ("nearest", "linear")
COORD_MODES = ("half_pixel", "asymmetric", "align_corners", "pytorch_half_pixel")
NEAREST_MODES = ("floor", "ceil", "round_prefer_floor", "round_prefer_ceil")


class ResizeError(ValueError):
    """kind = the reference's OpError variant"""

    def __init__(self, kind, msg):
        super().__init__(msg)
        self.kind = kind


def _as_i32(v):
    """Rust's `f32 as i32`: truncating, saturating, NaN -> 0"""
    if np.isnan(v):
        return 0
    return int(np.clip(np.float64(v), -2.0 ** 31, 2.0 ** 31 - 1))


def calc_output_size(in_shape, scales=None, sizes=None):
    """-> (sizes, inv_scales) per axis"""
    target = scales if scales is not None else sizes
    if target is None:
        raise ResizeError("MissingInputs", "missing inputs")
    if len(target) != len(in_shape):
        raise ResizeError("IncompatibleInputShapes", "scales/sizes length should equal input rank")
    out, inv = [], []
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        for n, t in zip(in_shape, target):
            if scales is not None:
                s = _F32(t)
                out.append(_as_i32(np.floor(_F32(n) * s)))
                inv.append(_F32(1.0) / s)
            else:
                out.append(int(t))
                inv.append(_F32(n) / _F32(int(t)))
    if any(o < 0 for o in out):
        raise ResizeError("InvalidValue", "scales/sizes must be positive")
    return out, inv


def input_coord(dest, scale, mode, length_original, length_resized):
    """dest: float32 array of output coordinates"""
    dest = np.asarray(dest, _F32)
    scale = _F32(scale)
    half = _F32(0.5)
    with np.errstate(divide="ignore", invalid="ignore"):
        if mode == "half_pixel":
            return scale * (dest + half) - half
        if mode == "asymmetric":
            return scale * dest
        if mode == "align_corners":
            return dest * _F32(length_original - 1) / _F32(length_resized - 1)
        if mode == "pytorch_half_pixel":
            if length_resized > 1:
                return scale * (dest + half) - half
            return np.zeros_like(dest)
    raise ValueError(mode)


def _clamp(c, length):
    hi = _F32(length) - _F32(1.0)
    c = np.where(c < _F32(0.0), _F32(0.0), c)
    return np.where(c > hi, hi, c).astype(_F32)


def _as_usize(c):
    with np.errstate(invalid="ignore"):
        return np.where(np.isnan(c), 0, np.trunc(c)).astype(np.int64)


def _round_half_away(c):
    # f32::round on a non-negative coordinate
    f = np.floor(c)
    return np.where(c - f >= _F32(0.5), f + _F32(1.0), f).astype(_F32)


def round_coord(c, nearest_mode):
    if nearest_mode == "ceil":
        return _as_usize(np.ceil(c))
    if nearest_mode == "floor":
        return _as_usize(c)
    fract = c - np.trunc(c)
    tie = np.ceil(c) if nearest_mode == "round_prefer_ceil" else np.floor(c)
    return _as_usize(np.where(fract == _F32(0.5), tie, _round_half_away(c)))


def _coords(n_out, inv_scale, coord_mode, n_in):
    dest = np.arange(n_out, dtype=np.int64).astype(_F32)
    return _clamp(input_coord(dest, inv_scale, coord_mode, n_in, n_out), n_in)


def _lerp(a, b, w):
    one = _F32(1.0)
    with np.errstate(invalid="ignore"):
        return ((one - w) * a).astype(_F32) + (w * b).astype(_F32)


def resize_4d(x, out_hw, inv_scale, mode, coord_mode, nearest_mode):
    x = np.asarray(x, _F32)
    B, C, H, W = x.shape
    OH, OW = out_hw
    if B * C * OH * OW == 0:
        return np.zeros((B, C, OH, OW), _F32)
    cy = _coords(OH, inv_scale[0], coord_mode, H)
    cx = _coords(OW, inv_scale[1], coord_mode, W)
    if mode == "nearest":
        iy, ix = round_coord(cy, nearest_mode), round_coord(cx, nearest_mode)
        return np.ascontiguousarray(x[:, :, iy][:, :, :, ix])
    y1, x1 = _as_usize(cy), _as_usize(cx)
    y2, x2 = np.minimum(y1 + 1, H - 1), np.minimum(x1 + 1, W - 1)
    wy = (cy - y1.astype(_F32)).astype(_F32)[None, None, :, None]
    wx = (cx - x1.astype(_F32)).astype(_F32)[None, None, None, :]
    top = _lerp(x[:, :, y1][:, :, :, x1], x[:, :, y1][:, :, :, x2], wx)
    bottom = _lerp(x[:, :, y2][:, :, :, x1], x[:, :, y2][:, :, :, x2], wx)
    return _lerp(top, bottom, wy).astype(_F32)


def resize(x, scales=None, sizes=None, mode="nearest", coord_mode="half_pixel", nearest_mode="round_prefer_floor"):
    x = np.asarray(x, _F32)
    out, inv = calc_output_size(x.shape, scales, sizes)
    ins = list(x.shape)
    one = _F32(1.0)

    def run(x4, y, xw):
        hw = (out[y] if y is not None else 1, out[xw])
        sc = (inv[y] if y is not None else one, inv[xw])
        return resize_4d(x4, hw, sc, mode, coord_mode, nearest_mode).reshape(out)

    if ins == out:
        return x.copy()
    if x.ndim == 4 and ins[:2] == out[:2]:
        return run(x, 2, 3)
    if x.ndim == 3 and ins[:2] == out[:2]:  # NCW
        return run(x.reshape(ins[0], ins[1], 1, ins[2]), None, 2)
    if x.ndim == 3 and ins[0] == out[0]:  # NHW
        return run(x.reshape(ins[0], 1, ins[1], ins[2]), 1, 2)
    if x.ndim == 2:
        return run(x.reshape(1, 1, ins[0], ins[1]), 0, 1)
    if x.ndim == 1:
        return run(x.reshape(1, 1, 1, ins[0]), None, 0)
    raise ResizeError("UnsupportedValue", "Only 1D to 4D inputs are supported with up to two resized dimensions")


def upsample(x, scales, mode="nearest"):
    return resize(x, scales=scales, mode=mode, coord_mode="asymmetric", nearest_mode="floor")


def average_pool(x, kernel, pads=(0, 0, 0, 0), strides=(1, 1), count_include_pad=False):
    """pads = (top, left, bottom, right)"""
    x = np.asarray(x, _F32)
    B, C, H, W = x.shape
    kh, kw = kernel
    pt, pl, pb, pr = pads
    sy, sx = strides
    OH = (H + pt + pb - kh) // sy + 1
    OW = (W + pl + pr - kw) // sx + 1
    out = np.zeros((B, C, OH, OW), _F32)
    for oy in range(OH):
        for ox in range(OW):
            acc = np.zeros((B, C), _F32)
            taps = 0
            for ky in range(kh):
                for kx in range(kw):
                    iy, ix = oy * sy + ky - pt, ox * sx + kx - pl
                    if 0 <= iy < H and 0 <= ix < W:
                        acc = (acc + x[:, :, iy, ix]).astype(_F32)
                        taps += 1
            with np.errstate(divide="ignore", invalid="ignore"):
                out[:, :, oy, ox] = acc / _F32(kh * kw if count_include_pad else taps)
    return out


def concat(inputs, axis):
    first = np.asarray(inputs[0])
    if not -first.ndim <= axis < first.ndim:
        raise ResizeError("InvalidValue", "Axis is invalid")
    axis %= first.ndim
    for t in inputs[1:]:
        t = np.asarray(t)
        if t.ndim != first.ndim:
            raise ResizeError("IncompatibleInputShapes", "Tensors must have the same number of dimensions")
        if any(d != axis and a != b for d, (a, b) in enumerate(zip(first.shape, t.shape))):
            raise ResizeError("IncompatibleInputShapes", "Dimensions must be the same except for concat axis")
    return np.concatenate([np.asarray(t) for t in inputs], axis=axis)
