"""numpy restatements of the mask and layout operators (rten_b200/csrc/masks.cu, api_masks.cu) and of the executor's
host-value rules (model.cu), checked against the reference's own unit-test values in tests/golden/mask_ops_cases.json.

  * where(cond, x, y): cond (i32) != 0 picks x, broadcasting the three (src/ops/binary_elementwise.rs where_op);
  * compare(op, a, b): i32 0 / 1, IEEE comparisons (NaN false, -0 == +0) (boolean_op); logical(op, a, b) / not_:
    nonzero is true (logical_boolean_op, unary_elementwise.rs not);
  * trilu(x, k, upper): (i, j) kept when i + k - j <= 0 (upper) or >= 0 (src/ops/trilu.rs);
  * expand(x, shape): bidirectional broadcast (src/ops/layout.rs expand);
  * slice_ranges / slice_(x, ...): the clamped ranges of src/ops/slice.rs, positive steps;
  * split(x, axis, sizes, num_outputs): src/ops/split.rs;
  * constant_of_shape(value, shape, dtype): src/ops/generate.rs constant_of_shape;
  * range_(start, limit, delta): the serial `val = val + delta` of src/ops/generate.rs range, in the inputs' type;
  * host_arith(op, a, b): the executor's host shape arithmetic, i32 wrapping, Div truncating."""
import json
import os

import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "mask_ops_cases.json")
I32 = np.int32


class OpFailed(Exception):
    pass


def where(cond, x, y):
    try:
        np.broadcast_shapes(np.shape(cond), np.shape(x), np.shape(y))
    except ValueError:
        raise OpFailed("Cannot broadcast inputs")
    return np.where(np.asarray(cond) != 0, x, y).astype(np.result_type(x, y))


def compare(op, a, b):
    f = {"Equal": np.equal, "Less": np.less, "LessOrEqual": np.less_equal, "Greater": np.greater,
         "GreaterOrEqual": np.greater_equal}[op]
    with np.errstate(invalid="ignore"):
        return f(a, b).astype(I32)


def logical(op, a, b):
    f = {"And": np.logical_and, "Or": np.logical_or, "Xor": np.logical_xor}[op]
    return f(np.asarray(a) != 0, np.asarray(b) != 0).astype(I32)


def not_(x):
    return (np.asarray(x) == 0).astype(I32)


def trilu(x, k=0, upper=True):
    x = np.asarray(x)
    if x.ndim < 2:
        raise OpFailed("Input must have >= 2 dims")
    i = np.arange(x.shape[-2])[:, None]
    j = np.arange(x.shape[-1])[None, :]
    delta = i + k - j
    keep = delta <= 0 if upper else delta >= 0
    return np.where(keep, x, np.zeros((), x.dtype)).astype(x.dtype)


def expand(x, shape):
    x = np.asarray(x)
    if any(int(d) < 0 for d in shape):
        raise OpFailed("Target shape contains negative values")
    try:
        out = np.broadcast_shapes(x.shape, tuple(int(d) for d in shape))
    except ValueError:
        raise OpFailed("Cannot broadcast input with target shape")
    return np.broadcast_to(x, out).copy()


def slice_ranges(shape, starts, ends, axes=None, steps=None):
    nd = len(shape)
    if axes is not None and len(axes) > nd:
        raise OpFailed("`axes` length must be <= input rank")
    n = len(axes) if axes is not None else nd
    if len(starts) != n:
        raise OpFailed("`starts` length must match axis count")
    if len(ends) != n:
        raise OpFailed("`ends` length must match axis count")
    if steps is not None:
        if len(steps) != n:
            raise OpFailed("`steps` length must match axis count")
        if any(s == 0 for s in steps):
            raise OpFailed("steps must be non-zero")
    out = [(0, d, 1) for d in shape]
    for i in range(n):
        a = i if axes is None else (axes[i] + nd if axes[i] < 0 else axes[i])
        if not 0 <= a < nd:
            raise OpFailed("Axis is invalid")
        d, s = shape[a], 1 if steps is None else steps[i]
        b, e = min(d, max(-d, starts[i])), min(d, max(-d, ends[i]))
        b, e = b + d if b < 0 else b, e + d if e < 0 else e
        out[a] = (b, max(0, -(-(e - b) // s)) if e > b else 0, s)
    return out


def slice_(x, starts, ends, axes=None, steps=None):
    x = np.asarray(x)
    r = slice_ranges(x.shape, starts, ends, axes, steps)
    return x[tuple(slice(b, b + n * s, s) for b, n, s in r)].copy()


def split(x, axis, sizes=None, num_outputs=None):
    x = np.asarray(x)
    a = axis + x.ndim if axis < 0 else axis
    if not 0 <= a < x.ndim:
        raise OpFailed("Axis is invalid")
    dim = x.shape[a]
    if sizes is not None:
        if any(s < 0 for s in sizes):
            raise OpFailed("Split sizes must be >= 0")
        if sum(sizes) != dim:
            raise OpFailed("Split sizes do not sum to dimension size")
        pieces, at = [], 0
        for s in sizes:
            pieces.append((at, s))
            at += s
    else:
        if num_outputs <= 0:
            raise OpFailed("num_outputs must be > 0")
        if num_outputs > dim:
            raise OpFailed("num_outputs exceeds dim size")
        c = -(-dim // num_outputs)
        pieces = [(at, min(c, dim - at)) for at in range(0, dim, c)]
    return [np.take(x, np.arange(b, b + n), axis=a) for b, n in pieces]


def range_(start, limit, delta, dtype):
    t = np.dtype(dtype).type
    start, limit, delta = t(start), t(limit), t(delta)
    if delta == 0:
        raise OpFailed("delta must be non-zero")
    out, v = [], start
    while (delta > 0 and v < limit) or (delta < 0 and v > limit):
        out.append(v)
        v = t(v + delta)
    return np.array(out, dtype)


def constant_of_shape(value, shape, dtype):
    if any(int(d) < 0 for d in shape):
        raise OpFailed("Invalid shape")
    return np.full(tuple(int(d) for d in shape), value, dtype)


def sat32(v):
    return np.clip(np.asarray(v, np.int64), -2 ** 31, 2 ** 31 - 1).astype(I32)


def host_arith(op, a, b):
    a, b = sat32(a).astype(np.int64), sat32(b).astype(np.int64)
    if op == "Div":
        if (b == 0).any() or ((b == -1).any() and (a == -2 ** 31).any()):
            raise OpFailed("Divisor contains zero")
        a, b = np.broadcast_arrays(a, b)
        q = np.abs(a) // np.abs(b) * np.sign(a) * np.sign(b)
        return q.astype(I32)
    r = {"Add": np.add, "Sub": np.subtract, "Mul": np.multiply}[op](a, b)
    return (((r + 2 ** 31) % 2 ** 32) - 2 ** 31).astype(I32)


def cases():
    with open(GOLDEN) as f:
        return json.load(f)["cases"]
