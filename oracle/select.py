"""numpy restatement of the order behind TopK, ArgMax and ArgMin (src/ops/reduce.rs topk, arg_max, arg_min).

Every element of a lane gets a 64-bit composite key and each operator takes the largest keys (rten_b200/csrc/select.cuh
builds the same keys on the device):
  * the 32-bit value key orders the values as the reference's cmp_nan_greater does: NaN above every number, all NaNs
    alike, -0.0 equal to +0.0;
  * TopK, largest: (value key, -index); smallest: (NaN last, then -value key, -index).  Ties, and several NaNs, come in
    ascending index order.  The reference's comparator is not consistent between two NaNs (each compares greater than
    the other), so its order among several NaNs is unspecified; ascending index is this project's definition;
  * ArgMax / ArgMin: Iterator::max_by keeps the LAST of equal elements but never lets go of a NaN, so the index is the
    first NaN's, else the last maximum's (minimum's): (value key, +index) for numbers, (NaN, -index) for NaNs.
Errors carry the reference's messages (ValueError)."""
import numpy as np

U32 = np.uint64(0xFFFFFFFF)


def value_key(x):
    """uint64 array of 32-bit order keys: larger key = greater under cmp_nan_greater"""
    x = np.asarray(x)
    if x.dtype == np.int32:
        return (x.view(np.uint32) ^ np.uint32(0x80000000)).astype(np.uint64)
    u = np.asarray(x, np.float32).view(np.uint32).copy()
    u[u == np.uint32(0x80000000)] = 0
    neg = (u & np.uint32(0x80000000)) != 0
    k = np.where(neg, ~u, u | np.uint32(0x80000000)).astype(np.uint64)
    k[np.isnan(np.asarray(x, np.float32))] = U32
    return k


def _isnan(x):
    x = np.asarray(x)
    return np.isnan(x) if x.dtype.kind == "f" else np.zeros(x.shape, bool)


def composite(x, mode, axis):
    """the composite keys of x's lanes along `axis` (moved last): mode 'largest', 'smallest', 'argmax' or 'argmin'"""
    x = np.moveaxis(np.asarray(x), axis, -1)
    k, nan = value_key(x), _isnan(x)
    idx = np.broadcast_to(np.arange(x.shape[-1], dtype=np.uint64), x.shape)
    if mode == "smallest":
        k = np.where(nan, np.uint64(0), U32 - k)
    elif mode == "argmin":
        k = np.where(nan, U32, U32 - k)
    later = (mode in ("argmax", "argmin")) & ~nan
    lo = np.where(later, idx, U32 - idx)
    return (k << np.uint64(32)) | lo


def _axis(ndim, axis):
    if ndim == 0 or not -ndim <= axis < ndim:
        raise ValueError("Axis is invalid")
    return axis % ndim


def topk(x, k, axis=-1, largest=True):
    """(values, i32 indices), best first"""
    x = np.asarray(x)
    if k < 0:
        raise ValueError("k must be positive")
    a = _axis(x.ndim, axis)
    if k > 0 and k > x.shape[a]:
        raise ValueError("k > dimension size")
    c = composite(x, "largest" if largest else "smallest", a)
    order = np.argsort(c, axis=-1, kind="stable")[..., ::-1][..., :k]
    vals = np.take_along_axis(np.moveaxis(x, a, -1), order, -1)
    return np.moveaxis(vals, -1, a), np.moveaxis(order.astype(np.int32), -1, a)


def _arg(x, axis, keepdims, mode):
    x = np.asarray(x)
    a = _axis(x.ndim, axis)
    if x.shape[a] == 0:
        raise ValueError("Cannot select index from empty sequence")
    c = composite(x, mode, a)
    out = (np.argmax(c, axis=-1) if c.size else np.zeros(c.shape[:-1], np.int64)).astype(np.int32)
    return np.expand_dims(out, a) if keepdims else out


def arg_max(x, axis=0, keepdims=True):
    return _arg(x, axis, keepdims, "argmax")


def arg_min(x, axis=0, keepdims=True):
    return _arg(x, axis, keepdims, "argmin")
