"""`pytest -m gpu`: whole models in the form torch.onnx.export writes at opset 13, run by the executor with every
decomposed block left as it is (no fusion matches them), against a float64 torch forward of the same weights.

  * a two-layer BERT-style encoder: Q / K / V MatMul + Add, Reshape / Transpose head split, MatMul -> Div(sqrt(d)) ->
    Add(an additive f32 mask input) -> Softmax -> MatMul, the decomposed LayerNorm (ReduceMean -> Sub -> Pow(2) ->
    ReduceMean -> Add(eps) -> Sqrt -> Div -> Mul -> Add) after attention and after the FFN, and the Erf Gelu with Div;
  * a GPT-2-style pre-LN block: the decomposed LayerNorm, causal attention scaled by Div, and NewGELU (Pow(x, 3) -> Mul
    -> Add -> Mul -> Tanh -> Add -> Mul -> Mul).

Both in both f32 modes, within the tolerance the repository states for encoder layers (tests/test_gpu_norms.py
test_model_encoder_layer): 1e-4 (3xTF32) and 1e-2 (single-pass TF32) of the largest |output|."""
import numpy as np
import pytest

import gpu_checks as gc

pytestmark = pytest.mark.gpu

F32 = np.float32
B, S, H, NH, FFN = 2, 64, 256, 4, 1024
DH = H // NH
TOL = {True: 1e-4, False: 1e-2}  # 3xTF32, TF32


@pytest.fixture(scope="module")
def rt():
    import rten_b200
    import rten_b200.model  # noqa: F401
    return rten_b200


def _weights(seed, names):
    r = np.random.default_rng(seed)
    w = {}
    for name, (i, o) in names.items():
        w["w" + name] = (r.standard_normal((i, o)) / np.sqrt(i)).astype(F32)
        w["b" + name] = (0.1 * r.standard_normal(o)).astype(F32)
    return w, r


class _Graph:
    def __init__(self):
        self.nodes, self.consts = [], {}

    def n(self, op, ins, outs, **attrs):
        self.nodes.append((op, ins, outs, attrs))
        return outs[0]

    def layer_norm(self, p, x, g, b, eps):
        """LayerNorm as torch exports it below opset 17"""
        mu = self.n("ReduceMean", [x], [p + "mu"], axes=[-1])
        d = self.n("Sub", [x, mu], [p + "d"])
        var = self.n("ReduceMean", [self.n("Pow", [d, "two"], [p + "d2"])], [p + "var"], axes=[-1])
        sd = self.n("Sqrt", [self.n("Add", [var, eps], [p + "ve"])], [p + "sd"])
        xn = self.n("Div", [d, sd], [p + "xn"])
        return self.n("Add", [self.n("Mul", [xn, g], [p + "xg"]), b], [p + "ln"])

    def linear(self, p, x, name):
        return self.n("Add", [self.n("MatMul", [x, "w" + name], [p + name + "0"]), "b" + name], [p + name])

    def attention(self, p, x, mask):
        heads = {}
        for t in "qkv":
            r = self.n("Reshape", [self.linear(p, x, p + t), "shape_heads"], [p + t + "r"])
            heads[t] = self.n("Transpose", [r], [p + t + "h"], perm=[0, 2, 3, 1] if t == "k" else [0, 2, 1, 3])
        s = self.n("Div", [self.n("MatMul", [heads["q"], heads["k"]], [p + "s0"]), "sqrt_d"], [p + "s1"])
        pr = self.n("Softmax", [self.n("Add", [s, mask], [p + "s2"])], [p + "p"], axis=-1)
        c = self.n("Transpose", [self.n("MatMul", [pr, heads["v"]], [p + "c0"])], [p + "c1"], perm=[0, 2, 1, 3])
        return self.linear(p, self.n("Reshape", [c, "shape_merge"], [p + "c2"]), p + "o")

    def model(self, inputs, output):
        import onnx_writer as W
        self.consts.update(shape_heads=np.array([0, 0, NH, DH], np.int64), shape_merge=np.array([0, 0, H], np.int64),
                           sqrt_d=F32(np.sqrt(DH)), two=F32(2), one=F32(1), half=F32(0.5))
        return W.model([W.node(op, i, o, **a) for op, i, o, a in self.nodes],
                       [W.tensor(k, np.asarray(v)) for k, v in self.consts.items()],
                       [W.value_info(k, W.FLOAT, list(v)) for k, v in inputs.items()],
                       [W.value_info(output, W.FLOAT, [B, S, H])], opset=13)


def bert_encoder():
    """(model bytes, weights) of the two-layer encoder; the output is `l1_out`"""
    g = _Graph()
    x = "x"
    for l in range(2):
        p = f"l{l}_"
        w, r = _weights(100 + l, {p + "q": (H, H), p + "k": (H, H), p + "v": (H, H), p + "o": (H, H), p + "f1": (H, FFN),
                                  p + "f2": (FFN, H)})
        for ln in ("ln1", "ln2"):
            w[p + ln + "g"] = (1 + 0.1 * r.standard_normal(H)).astype(F32)
            w[p + ln + "b"] = (0.1 * r.standard_normal(H)).astype(F32)
        g.consts.update(w)
        a = g.n("Add", [g.attention(p, x, "mask"), x], [p + "res1"])
        h = g.layer_norm(p + "ln1_", a, p + "ln1g", p + "ln1b", "eps")
        f = g.linear(p, h, p + "f1")
        e = g.n("Add", [g.n("Erf", [g.n("Div", [f, "sqrt2"], [p + "gd"])], [p + "ge"]), "one"], [p + "gp"])
        f2 = g.n("Mul", [g.n("Mul", [f, e], [p + "gq"]), "half"], [p + "gelu"])
        o = g.n("Add", [g.linear(p, f2, p + "f2"), h], [p + "res2"])
        x = g.layer_norm(p + "ln2_", o, p + "ln2g", p + "ln2b", "eps")
    g.consts.update(eps=F32(1e-12), sqrt2=F32(1.4142135381698608))
    return g.model({"x": (B, S, H), "mask": (B, 1, 1, S)}, x), g.consts, x


def gpt2_block():
    g = _Graph()
    p = "b_"
    w, r = _weights(200, {p + "q": (H, H), p + "k": (H, H), p + "v": (H, H), p + "o": (H, H), p + "fc": (H, FFN),
                          p + "proj": (FFN, H)})
    for ln in ("ln1", "ln2"):
        w[p + ln + "g"] = (1 + 0.1 * r.standard_normal(H)).astype(F32)
        w[p + ln + "b"] = (0.1 * r.standard_normal(H)).astype(F32)
    g.consts.update(w)
    h = g.layer_norm(p + "ln1_", "x", p + "ln1g", p + "ln1b", "eps")
    r1 = g.n("Add", ["x", g.attention(p, h, "causal")], [p + "res1"])
    h2 = g.layer_norm(p + "ln2_", r1, p + "ln2g", p + "ln2b", "eps")
    u = g.linear(p, h2, p + "fc")
    inner = g.n("Add", [u, g.n("Mul", [g.n("Pow", [u, "three"], [p + "u3"]), "k"], [p + "ku3"])], [p + "inner"])
    th = g.n("Tanh", [g.n("Mul", [inner, "s2pi"], [p + "t"])], [p + "th"])
    gl = g.n("Mul", [g.n("Mul", [u, "half"], [p + "hu"]), g.n("Add", [th, "one"], [p + "p1"])], [p + "gelu"])
    out = g.n("Add", [r1, g.linear(p, gl, p + "proj")], [p + "out"])
    g.consts.update(eps=F32(1e-5), three=F32(3), k=F32(0.044715), s2pi=F32(np.sqrt(2.0 / np.pi)),
                    causal=np.triu(np.full((S, S), -10000.0, F32), 1).reshape(1, 1, S, S))
    return g.model({"x": (B, S, H)}, out), g.consts, out


# ---- float64 torch forwards ------------------------------------------------------------------------------------------
def _t(w):
    import torch
    return {k: torch.from_numpy(np.asarray(v, np.float64)) for k, v in w.items() if np.asarray(v).dtype == F32}


def _ln64(x, g, b, eps):
    mu = x.mean(-1, keepdim=True)
    d = x - mu
    return d / ((d * d).mean(-1, keepdim=True) + eps).sqrt() * g + b


def _attn64(w, p, x, mask):
    def heads(t):
        return (x @ w["w" + p + t] + w["b" + p + t]).reshape(B, S, NH, DH).transpose(1, 2)
    s = heads("q") @ heads("k").transpose(-1, -2) / np.sqrt(DH) + mask
    c = (s.softmax(-1) @ heads("v")).transpose(1, 2).reshape(B, S, H)
    return c @ w["w" + p + "o"] + w["b" + p + "o"]


def bert64(consts, x, mask):
    import torch
    w = _t(consts)
    x, mask = torch.from_numpy(x.astype(np.float64)), torch.from_numpy(mask.astype(np.float64))
    for l in range(2):
        p = f"l{l}_"
        h = _ln64(_attn64(w, p, x, mask) + x, w[p + "ln1g"], w[p + "ln1b"], 1e-12)
        f = h @ w["w" + p + "f1"] + w["b" + p + "f1"]
        f = 0.5 * f * (1 + torch.erf(f / np.sqrt(2.0)))
        x = _ln64(f @ w["w" + p + "f2"] + w["b" + p + "f2"] + h, w[p + "ln2g"], w[p + "ln2b"], 1e-12)
    return x.numpy()


def gpt2_64(consts, x):
    import torch
    w, p = _t(consts), "b_"
    x = torch.from_numpy(x.astype(np.float64))
    r1 = x + _attn64(w, p, _ln64(x, w[p + "ln1g"], w[p + "ln1b"], 1e-5), w["causal"])
    u = _ln64(r1, w[p + "ln2g"], w[p + "ln2b"], 1e-5) @ w["w" + p + "fc"] + w["b" + p + "fc"]
    gl = 0.5 * u * (1 + torch.tanh(np.sqrt(2.0 / np.pi) * (u + 0.044715 * u ** 3)))
    return (r1 + gl @ w["w" + p + "proj"] + w["b" + p + "proj"]).numpy()


def _rel(got, ref):
    return float(np.abs(np.asarray(got, np.float64) - ref).max() / np.abs(ref).max())


UNFUSED = {"Div", "Pow", "Sqrt", "ReduceMean", "Sub"}


@pytest.mark.parametrize("tf32x3", [True, False], ids=["3xTF32", "TF32"])
def test_bert_encoder_opset13(rt, tf32x3):
    from rten_b200.model import Model
    data, consts, out = bert_encoder()
    r = np.random.default_rng(7)
    x = r.standard_normal((B, S, H)).astype(F32)
    mask = np.zeros((B, 1, 1, S), F32)
    mask[1, ..., S - 17:] = -10000.0  # the second sequence right-padded
    ctx = gc.new_ctx(rt, tf32=not tf32x3)
    m = Model(ctx, data)
    assert UNFUSED | {"Erf"} <= set(m.node_ops), m.node_ops
    (y,) = m.run({"x": x, "mask": mask}, [out])
    rel = _rel(y.numpy(), bert64(consts, x, mask))
    assert rel <= TOL[tf32x3], f"BERT encoder ({'3xTF32' if tf32x3 else 'TF32'}): {rel:.2e} of max |ref|"


@pytest.mark.parametrize("tf32x3", [True, False], ids=["3xTF32", "TF32"])
def test_gpt2_block_opset13(rt, tf32x3):
    from rten_b200.model import Model
    data, consts, out = gpt2_block()
    x = np.random.default_rng(8).standard_normal((B, S, H)).astype(F32)
    ctx = gc.new_ctx(rt, tf32=not tf32x3)
    m = Model(ctx, data)
    assert UNFUSED | {"Tanh"} <= set(m.node_ops), m.node_ops
    (y,) = m.run({"x": x}, [out])
    rel = _rel(y.numpy(), gpt2_64(consts, x))
    assert rel <= TOL[tf32x3], f"GPT-2 block ({'3xTF32' if tf32x3 else 'TF32'}): {rel:.2e} of max |ref|"
