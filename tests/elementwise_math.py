"""Test infrastructure for Div, Pow, Sqrt, Reciprocal, Exp, Tanh, Neg, Abs and ReduceMean: numpy restatements of the
reference's operators (src/ops/binary_elementwise.rs, unary_elementwise.rs, reduce.rs), the expected values of the
reference's own unit tests for them, and the torch-exported blocks that use them as small ONNX graphs.

  * `div_ref`: f32 a / b correctly rounded; a one-element b is a * (1 / b), two roundings, with a's shape; i32 truncates
    toward zero and raises DivError on a zero divisor or INT_MIN / -1.
  * `pow_ref`: FastPow.  f32 exponent 2 is x * x, 3 is x * x * x; other exponents give the correctly rounded result
    (float64 pow, rounded once), which the device's powf matches within POW_ULP.  i32 exponents >= 0 wrap, negative ones
    go through f32 with a saturating conversion.  A one-element exponent keeps the base's shape.
  * `UNARY`: Sqrt / Reciprocal / Neg / Abs in float32 arithmetic, Exp / Tanh through the C oracle's rto_exp / rto_tanh.
  * `reduce_mean_ref`: genai_decoder.reduce_sum_ref (the reference's Sum over each lane) divided by the lane length."""
import numpy as np

import genai_decoder as gd

F32, I32 = np.float32, np.int32
IMIN, IMAX = -2 ** 31, 2 ** 31 - 1

# The largest error of CUDA's powf, in ulp of the exact result: the CUDA C++ Programming Guide's table of single-precision
# standard functions gives 4 (full range).
POW_ULP = 4


class DivError(ValueError):
    """The reference's InvalidValue("Divisor contains zero")"""


def _scalar_b(b):
    return np.asarray(b).size == 1


def div_ref(a, b):
    a, b = np.asarray(a), np.asarray(b)
    if a.dtype == F32:
        with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
            if _scalar_b(b):
                return (a * (F32(1) / b.reshape(()))).astype(F32)
            return (a / b).astype(F32)
    a64, b64 = np.broadcast_arrays(a.astype(np.int64), b.astype(np.int64))
    if (b == 0).any() or ((a64 == IMIN) & (b64 == -1)).any():
        raise DivError("Divisor contains zero")
    q = np.abs(a64) // np.abs(b64)
    return (np.sign(a64) * np.sign(b64) * q).astype(I32)


def _pow_f32(x, e):
    """FastPow of float32 arrays (broadcast): exact products for 2 and 3, the correctly rounded pow for the rest"""
    x, e = np.broadcast_arrays(np.asarray(x, F32), np.asarray(e, F32))
    with np.errstate(all="ignore"):
        general = np.power(x.astype(np.float64), e.astype(np.float64)).astype(F32)
        return np.where(e == 2, x * x, np.where(e == 3, (x * x) * x, general)).astype(F32)


def pow_ref(a, b):
    a, b = np.asarray(a), np.asarray(b)
    if _scalar_b(b):
        b = b.reshape(())
    if a.dtype == F32:
        return _pow_f32(a, b).reshape(np.broadcast_shapes(a.shape, b.shape))
    x, e = np.broadcast_arrays(a.astype(np.int64), b.astype(np.int64))
    out = np.empty(x.shape, np.int64)
    for i, (xv, ev) in enumerate(zip(x.reshape(-1), e.reshape(-1))):
        if ev >= 0:
            out.reshape(-1)[i] = pow(int(xv), int(ev), 2 ** 32)
        else:
            v = float(_pow_f32(F32(xv), F32(ev)))
            out.reshape(-1)[i] = 0 if v != v else int(min(max(v, IMIN), IMAX))
    return ((out + 2 ** 31) % 2 ** 32 - 2 ** 31).astype(I32)


def pow_general(b):
    """the elements whose exponent takes powf (not 2 or 3)"""
    return (np.asarray(b) != 2) & (np.asarray(b) != 3)


def ulp_distance(got, want):
    """|got - want| in float32 units in the last place (NaN == NaN, +0 == -0), as int64"""
    def key(v):
        i = np.asarray(v, F32).view(np.int32).astype(np.int64)
        return np.where(i < 0, -(i & 0x7fffffff), i)
    d = np.abs(key(got) - key(want))
    both_nan = np.isnan(got) & np.isnan(want)
    return np.where(both_nan, 0, np.where(np.isnan(got) | np.isnan(want), 2 ** 40, d))


def _oracle():
    from oracle import oracle
    return oracle


UNARY = {
    "Sqrt": lambda x: np.sqrt(np.asarray(x, F32)),
    "Reciprocal": lambda x: F32(1) / np.asarray(x, F32),
    "Exp": lambda x: _oracle().exp(np.asarray(x, F32)),
    "Tanh": lambda x: _oracle().tanh(np.asarray(x, F32)),
    "Neg": lambda x: -np.asarray(x, F32),
    "Abs": lambda x: np.abs(np.asarray(x, F32)),
}


def unary_ref(op, x):
    with np.errstate(all="ignore"):
        return np.asarray(UNARY[op](x), F32).reshape(np.shape(x))


def reduce_mean_ref(x, axes=None, keepdims=True):
    x = np.asarray(x, F32)
    red = gd.resolve_axes(x.ndim, axes) if x.ndim else []
    n = int(np.prod([x.shape[a] for a in red])) if red else 1
    with np.errstate(all="ignore"):
        return (np.asarray(gd.reduce_sum_ref(x, axes, keepdims), F32) / F32(n)).astype(F32)


# ---- the reference's unit tests (binary_elementwise.rs test_div / test_pow, reduce.rs test_reduce_mean) ------------
# (op, a, b or axes, expected) -- values as the reference's tests state them
REFERENCE_CASES = [
    ("Div", np.array([[10, 20], [30, 40]], F32), np.array([[1, 2], [3, 4]], F32), np.array([[10, 10], [10, 10]], F32)),
    ("Div", np.array([[10, 20], [30, 40]], F32), np.array(10, F32), np.array([[1, 2], [3, 4]], F32)),
    ("Div", np.array([1, 2, 3, 4], I32), np.array([2, 2, 2, 2], I32), np.array([0, 1, 1, 2], I32)),
    ("Div", np.array([1, 2, 3, 4], I32), np.array(2, I32), np.array([0, 1, 1, 2], I32)),
    ("Pow", np.array([2, 3, 4], F32), np.array(2, F32), np.array([4, 9, 16], F32)),
    ("Pow", np.array([2, 3, 4], F32), np.array(3, F32), np.array([8, 27, 64], F32)),
    ("Pow", np.array([2, 3, 4], F32), np.array([1, 2, 3], F32), np.array([2, 9, 64], F32)),
    ("Pow", np.array(4, I32), np.array(2, I32), np.array(16, I32)),
    ("Pow", np.array(2, I32), np.array(3, I32), np.array(8, I32)),
    ("Pow", np.array(4097, I32), np.array(2, I32), np.array(4097 * 4097, I32)),
    ("Pow", np.array(46340, I32), np.array(2, I32), np.array(46340 * 46340, I32)),
    ("Pow", np.array(46341, I32), np.array(2, I32), np.array((46341 * 46341) - 2 ** 32, I32)),
    ("Pow", np.array(216, I32), np.array(4, I32), np.array(-2118184960, I32)),
    ("Pow", np.array(2, I32), np.array(-1, I32), np.array(0, I32)),
    ("ReduceMean", np.arange(1, 10, dtype=F32).reshape(3, 3), ([-1], False), np.array([2, 5, 8], F32)),
    ("ReduceMean", np.arange(1, 10, dtype=F32).reshape(3, 3), ([-1], True), np.array([[2], [5], [8]], F32)),
    ("ReduceMean", np.arange(1, 10, dtype=F32).reshape(3, 3), ([0], False), np.array([4, 5, 6], F32)),
    ("ReduceMean", np.arange(1, 10, dtype=F32).reshape(3, 3), (None, False), np.array(5, F32)),
    ("ReduceMean", np.array([5, 1, 20, 2, 30, 1, 40, 2, 55, 1, 60, 2], F32).reshape(3, 2, 2), ([1], False),
     np.array([[12.5, 1.5], [35, 1.5], [57.5, 1.5]], F32)),
    ("ReduceMean", np.array(5, F32), ([], False), np.array(5, F32)),
]


def reference_case_ref(op, a, b, want):
    """the oracle's answer for one REFERENCE_CASES entry"""
    if op == "Div":
        return div_ref(a, b)
    if op == "Pow":
        return pow_ref(a, b)
    axes, keep = b
    return reduce_mean_ref(a, axes, keep)


# ---- the torch-exported blocks, as node lists on a device input x [.., H] ---------------------------------------------
def block_specs(H):
    """{name: (nodes [(op, inputs, outputs, attributes)], constants {name: array}, extra f32 graph inputs)} of the five
    blocks as torch.onnx.export writes them at opset 13 (no MatMul: the attention block starts from the scores)"""
    g = np.linspace(0.5, 1.5, H, dtype=F32)
    bta = np.linspace(-0.2, 0.2, H, dtype=F32)
    half, one, two = F32(0.5), F32(1), F32(2)
    return {
        "attention scale": ([("Div", ["x", "sqrt_d"], ["s"], {}), ("Add", ["s", "mask"], ["m"], {}),
                             ("Softmax", ["m"], ["y"], {"axis": -1})],
                            {"sqrt_d": F32(8.0)}, ["mask"]),
        "erf gelu": ([("Div", ["x", "sqrt2"], ["d"], {}), ("Erf", ["d"], ["e"], {}), ("Add", ["e", "one"], ["p"], {}),
                      ("Mul", ["x", "p"], ["q"], {}), ("Mul", ["q", "half"], ["y"], {})],
                     {"sqrt2": F32(1.4142135381698608), "one": one, "half": half}, []),
        "layer norm": ([("ReduceMean", ["x"], ["mu"], {"axes": [-1]}), ("Sub", ["x", "mu"], ["c"], {}),
                        ("Pow", ["c", "two"], ["c2"], {}), ("ReduceMean", ["c2"], ["var"], {"axes": [-1]}),
                        ("Add", ["var", "eps"], ["ve"], {}), ("Sqrt", ["ve"], ["sd"], {}), ("Div", ["c", "sd"], ["xn"], {}),
                        ("Mul", ["xn", "g"], ["xg"], {}), ("Add", ["xg", "b"], ["y"], {})],
                       {"two": two, "eps": F32(1e-12), "g": g, "b": bta}, []),
        "rms norm": ([("Pow", ["x", "two"], ["x2"], {}), ("ReduceMean", ["x2"], ["ms"], {"axes": [-1]}),
                      ("Add", ["ms", "eps"], ["me"], {}), ("Sqrt", ["me"], ["r"], {}), ("Reciprocal", ["r"], ["ir"], {}),
                      ("Mul", ["x", "ir"], ["xn"], {}), ("Mul", ["xn", "g"], ["y"], {})],
                     {"two": two, "eps": F32(1e-6), "g": g}, []),
        "new gelu": ([("Pow", ["x", "three"], ["x3"], {}), ("Mul", ["x3", "k"], ["kx3"], {}), ("Add", ["x", "kx3"], ["inner"], {}),
                      ("Mul", ["inner", "s2pi"], ["t"], {}), ("Tanh", ["t"], ["th"], {}), ("Add", ["th", "one"], ["p"], {}),
                      ("Mul", ["x", "half"], ["hx"], {}), ("Mul", ["hx", "p"], ["y"], {})],
                     {"three": F32(3), "k": F32(0.044715), "s2pi": F32(np.sqrt(2.0 / np.pi)), "one": one, "half": half}, []),
    }


def block_model(spec, x_shape, extra_shapes):
    """the ONNX model (opset 13) of one block_specs entry: x and the extra inputs f32 graph inputs, output y"""
    import onnx_writer as W
    nodes, consts, extra = spec
    onnx_nodes = [W.node(op, ins, outs, **attrs) for op, ins, outs, attrs in nodes]
    inits = [W.tensor(k, np.asarray(v)) for k, v in consts.items()]
    ins = [W.value_info("x", W.FLOAT, list(x_shape))] + [W.value_info(e, W.FLOAT, list(extra_shapes[e])) for e in extra]
    return W.model(onnx_nodes, inits, ins, [W.value_info("y", W.FLOAT, list(x_shape))], opset=13)


def run_nodes(nodes, consts, feeds):
    """the reference's op-by-op execution of a node list, every value computed by its operator's oracle"""
    vals = {**{k: np.asarray(v) for k, v in consts.items()}, **feeds}
    for op, ins, outs, attrs in nodes:
        x = [vals[i] for i in ins]
        if op == "Div":
            y = div_ref(*x)
        elif op == "Pow":
            y = pow_ref(*x)
        elif op in UNARY:
            y = unary_ref(op, x[0])
        elif op == "ReduceMean":
            y = reduce_mean_ref(x[0], attrs.get("axes"), bool(attrs.get("keepdims", 1)))
        elif op in ("Add", "Sub", "Mul"):
            a, b = (np.asarray(v, F32) for v in x)
            with np.errstate(all="ignore"):
                y = {"Add": a + b, "Sub": a - b, "Mul": a * b}[op].astype(F32)
        elif op == "Erf":
            y = _oracle().erf(np.asarray(x[0], F32))
        elif op == "Softmax":
            y = _oracle().softmax(np.asarray(x[0], F32), attrs.get("axis", -1))
        else:
            raise NotImplementedError(op)
        vals[outs[0]] = np.asarray(y)
    return vals
