"""GRU and LSTM on the CPU, restated from the reference's order of operations (src/ops/rnn.rs gru / lstm).

TEST INFRASTRUCTURE ONLY, like oracle.py.

Per direction and step (direction 1 of a bidirectional layer, and a reverse layer, run t = T - 1 .. 0):
  GRU : gates = x_t W^T (+ Wb); s = h R^T (+ Rb); z, r = sigmoid(gates + s); h~ = tanh(gates_h + s_h * r);
        h = (1 - z) * h~ + z * h
  LSTM: gates = ((x_t W^T (+ Wb)) + h R^T) (+ Rb); i, o, f = sigmoid; c~ = tanh; c = f * c + i * c~; h = o * tanh(c)
Gate order is ONNX's: z, r, h (GRU) and i, o, f, c (LSTM).

mode "f32": float32 throughout, products as float32 matrix products, sigmoid and tanh by rten-vecmath's recipes
(sigmoid below on rten_oracle.c's rto_exp, and rto_tanh) except the LSTM's last tanh, which is a float32 tanh as the reference's
f32::tanh.  mode "f64": float64 throughout with exact sigmoid / tanh: the value the f32 computations approximate.
tf32_input (f64 mode): x and W enter the input projection with their low 13 mantissa bits cleared, as the tensor cores'
single TF32 pass reads them; the recurrence stays exact.
"""
from __future__ import annotations

import numpy as np

from . import oracle

_DIRECTIONS = ("forward", "reverse", "bidirectional")


def sigmoid(x):
    """rten-vecmath's Sigmoid (exp.rs): reciprocal(1 + Exp(neg(x))) with neg = 0 - x and reciprocal = an exact 1 / x.
    numpy's float32 subtraction, addition and division are single, exactly rounded operations, so this is the recipe
    applied to the oracle's Exp (rto_exp)."""
    f32 = np.float32
    x = np.asarray(x, f32)
    e = oracle.exp(f32(0.0) - x)
    return (f32(1.0) / (f32(1.0) + e)).astype(f32)


def tf32_truncate(a):
    a = np.ascontiguousarray(a, np.float32)
    return (a.view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)


class _Math:
    def __init__(self, mode: str):
        if mode not in ("f32", "f64"):
            raise ValueError(mode)
        self.f64 = mode == "f64"
        self.dt = np.float64 if self.f64 else np.float32

    def cast(self, a):
        return None if a is None else np.asarray(a, np.float32).astype(self.dt)

    def sigmoid(self, x):
        return 1.0 / (1.0 + np.exp(-x)) if self.f64 else sigmoid(x)

    def tanh(self, x):
        return np.tanh(x) if self.f64 else oracle.tanh(x)

    def std_tanh(self, x):
        return np.tanh(x)


def _run(G, x, w, r, b, h0, c0, direction, mode, tf32_input):
    if direction not in _DIRECTIONS:
        raise ValueError(direction)
    m = _Math(mode)
    x32, w32 = np.asarray(x, np.float32), np.asarray(w, np.float32)
    if tf32_input:
        x32, w32 = tf32_truncate(x32), tf32_truncate(w32)
    X, W, R, Bi = m.cast(x32), m.cast(w32), m.cast(r), m.cast(b)
    T, B, _ = X.shape
    dirs = 2 if direction == "bidirectional" else 1
    H = W.shape[1] // G
    h = m.cast(h0) if h0 is not None else np.zeros((dirs, B, H), m.dt)
    h = h.copy()
    c = None
    if G == 4:
        c = (m.cast(c0) if c0 is not None else np.zeros((dirs, B, H), m.dt)).copy()
    Y = np.zeros((T, dirs, B, H), m.dt)
    for d in range(dirs):
        rev = (d == 0 and direction == "reverse") or d == 1
        Wb = Bi[d, :G * H] if Bi is not None else None
        Rb = Bi[d, G * H:] if Bi is not None else None
        for t in (range(T - 1, -1, -1) if rev else range(T)):
            gates = X[t] @ W[d].T
            if Wb is not None:
                gates = gates + Wb
            if G == 3:
                s = h[d] @ R[d].T
                if Rb is not None:
                    s = s + Rb
                zr = m.sigmoid(gates[:, :2 * H] + s[:, :2 * H])
                z, rr = zr[:, :H], zr[:, H:]
                ht = m.tanh(gates[:, 2 * H:] + s[:, 2 * H:] * rr)
                h[d] = (1 - z) * ht + z * h[d]
            else:
                gates = gates + h[d] @ R[d].T
                if Rb is not None:
                    gates = gates + Rb
                iof = m.sigmoid(gates[:, :3 * H])
                i, o, f = iof[:, :H], iof[:, H:2 * H], iof[:, 2 * H:]
                cc = m.tanh(gates[:, 3 * H:])
                c[d] = f * c[d] + i * cc
                h[d] = o * m.std_tanh(c[d])
            Y[t, d] = h[d]
    return Y, h, c


def gru(x, w, r, b=None, initial_h=None, direction="forward", mode="f32", tf32_input=False):
    """(Y [T, dirs, B, H], Y_h [dirs, B, H])"""
    Y, h, _ = _run(3, x, w, r, b, initial_h, None, direction, mode, tf32_input)
    return Y, h


def lstm(x, w, r, b=None, initial_h=None, initial_c=None, direction="forward", mode="f32", tf32_input=False):
    """(Y [T, dirs, B, H], Y_h [dirs, B, H], Y_c [dirs, B, H])"""
    return _run(4, x, w, r, b, initial_h, initial_c, direction, mode, tf32_input)


# ---- the reference's PyTorch-generated cases (pytorch-ref-tests/rnn.json, tests/golden/rnn_cases.json) ----------------
def _reorder(a, G):
    """PyTorch gate order -> ONNX: LSTM (i, f, c, o) -> (i, o, f, c); GRU (r, z, n) -> (z, r, n), along axis 0."""
    parts = np.split(np.asarray(a, np.float32), G, axis=0)
    order = (0, 3, 1, 2) if G == 4 else (1, 0, 2)
    return np.concatenate([parts[i] for i in order], axis=0)


def golden_case(case: dict, name: str):
    """(op, direction, inputs dict, expected Y [T, dirs, 1, H]) of one case, in ONNX layout."""
    op = "lstm" if name.startswith("lstm") else "gru"
    G = 4 if op == "lstm" else 3
    t = lambda v: np.asarray(v[1], np.float32).reshape(v[0])  # noqa: E731
    p = case["params"]
    bidir = "weight_ih_l0_reverse" in p
    sfx = ["", "_reverse"] if bidir else [""]
    w = np.stack([_reorder(t(p["weight_ih_l0" + s]), G) for s in sfx])
    r = np.stack([_reorder(t(p["weight_hh_l0" + s]), G) for s in sfx])
    b = np.stack([np.concatenate([_reorder(t(p["bias_ih_l0" + s]), G), _reorder(t(p["bias_hh_l0" + s]), G)]) for s in sfx])
    x = t(case["input"])[:, None, :]
    exp = t(case["output"])
    T = exp.shape[0]
    exp = exp.reshape(T, len(sfx), 1, -1)
    ins = {"x": x, "w": w, "r": r, "b": b}
    if "initial_hidden" in case:
        ins["initial_h"] = t(case["initial_hidden"])[:, None, :]
    if "initial_cell" in case:
        ins["initial_c"] = t(case["initial_cell"])[:, None, :]
    return op, "bidirectional" if bidir else "forward", ins, exp
