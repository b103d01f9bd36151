"""GRU and LSTM on the GPU: the input projection on the wgmma GEMM, the recurrence on rnn_cluster_kernel (one launch)
or, above the cluster bound or with RTEN_B200_NO_RNN_CLUSTER=1, on the per-step path (recurrent product + gate kernel).

References: the reference's PyTorch-generated cases (tests/golden/rnn_cases.json) with its expect_equal rule, and the
numpy restatement oracle/rnn.py.  Accuracy rule of the parity matrix: the GPU's largest error against the float64
restatement may exceed the float32 restatement's by at most FLOOR.  In single-pass TF32 the float64 restatement reads
x and W truncated to TF32 in the input projection (the recurrence is exact f32 in both modes)."""
import json
import os

import numpy as np
import pytest

import gpu_checks as gc
from oracle import oracle
from oracle import rnn as orn

HERE = os.path.dirname(os.path.abspath(__file__))
FLOOR = 3e-5  # absolute, on outputs in [-1, 1]: f32 FMA-chain / 3xTF32 rounding beyond the f32 restatement's own


@pytest.fixture(scope="module")
def rt():
    import rten_b200
    from rten_b200 import _lib
    _lib.load()
    return rten_b200


def _ctx(rt, tf32=False):
    ctx = rt.Context(0)
    ctx.set_f32_mode(not tf32)
    return ctx


def _run(rt, ctx, op, ins, direction, per_step=False, outputs=None, packed=False):
    G = 3 if op == "gru" else 4
    H = ins["w"].shape[1] // G
    o = rt.GRU(direction, H) if op == "gru" else rt.LSTM(direction, H)
    kw = {k: v for k, v in ins.items() if k not in ("x", "w", "r")}
    if outputs is not None:
        kw["outputs"] = outputs
    if packed:
        kw["packed_w"] = o.prepack(ctx, ins["w"])
    with gc.switches(RTEN_B200_NO_RNN_CLUSTER=1 if per_step else None):
        res = o.run(ctx, ins["x"], ins["w"], ins["r"], **kw)
    return [None if t is None else t.numpy() for t in res]


def _case(op, T, B, I, H, direction, bias=True, init=True, seed=0):
    r = np.random.default_rng(seed)
    G = 3 if op == "gru" else 4
    dirs = 2 if direction == "bidirectional" else 1
    s = 1.0 / np.sqrt(H)
    f = lambda *shape, k=s: r.uniform(-k, k, shape).astype(np.float32)  # noqa: E731
    ins = {"x": f(T, B, I, k=1.0), "w": f(dirs, G * H, I), "r": f(dirs, G * H, H)}
    if bias:
        ins["b"] = f(dirs, 2 * G * H)
    if init:
        ins["initial_h"] = f(dirs, B, H, k=0.5)
        if op == "lstm":
            ins["initial_c"] = f(dirs, B, H, k=0.5)
    return ins


def _oracle(op, ins, direction, mode, tf32_input=False):
    fn = orn.gru if op == "gru" else orn.lstm
    out = fn(direction=direction, mode=mode, tf32_input=tf32_input, **ins)
    return [o for o in out if o is not None]


def _max_err(got, ref):
    return max(float(np.abs(np.asarray(g, np.float64) - np.asarray(e, np.float64)).max()) for g, e in zip(got, ref) if g is not None)


def _check_rule(got, op, ins, direction, tf32, what):
    exact = _oracle(op, ins, direction, "f64")
    f32 = _oracle(op, ins, direction, "f32")
    ref = _oracle(op, ins, direction, "f64", tf32_input=True) if tf32 else exact
    base = _max_err(f32, exact)
    err = _max_err(got, ref)
    assert err <= base + FLOOR, f"{what}: GPU error {err:.3e} > f32 restatement's {base:.3e} + {FLOOR:.0e}"
    return err


# ---------------------------------------------------------------------------------------------------------------------
GOLDEN = ["lstm_forwards", "lstm_initial", "lstm_bidirectional", "gru_forwards", "gru_initial", "gru_bidirectional"]


@pytest.mark.gpu
@pytest.mark.parametrize("tf32", [False, True], ids=["tf32x3", "tf32"])
@pytest.mark.parametrize("per_step", [False, True], ids=["cluster", "per_step"])
def test_golden_cases(rt, per_step, tf32):
    import gpu_checks as gc
    with open(os.path.join(HERE, "golden", "rnn_cases.json")) as f:
        cases = json.load(f)
    ctx = _ctx(rt, tf32)
    for name in GOLDEN:
        op, direction, ins, exp = orn.golden_case(cases[name], name)
        y = _run(rt, ctx, op, ins, direction, per_step)[0]
        if tf32:
            # |d| <= 2^-9 sum_k |x_k w_k| per pre-activation, through the bounded gates: stated on Y with the largest sum
            absum = max(float(np.abs(ins["x"]).sum(-1).max() * np.abs(ins["w"]).max()), 1.0)
            gc.assert_tf32_close(y, exp.astype(np.float64), np.full(exp.shape, absum), f"{name} ({'per-step' if per_step else 'cluster'})")
        else:
            # expect_equal's rule with atol 1e-7 instead of 1e-8: a few outputs lie near 0 after cancellation, where the
            # 3xTF32 projection's last-bit differences from an f32 GEMM exceed 1e-8 + 1e-5 |b| (seen: 4e-8 at 1.3e-3)
            assert oracle.expect_equal(y, exp, atol=1e-7), f"{name}: max |d| = {float(np.abs(y - exp).max()):.3e}"


PARITY = [(op, B, H) for op in ("gru", "lstm") for B in (1, 7, 64) for H in (5, 64, 256, 1024)]


@pytest.mark.gpu
@pytest.mark.parametrize("tf32", [False, True], ids=["tf32x3", "tf32"])
@pytest.mark.parametrize("op,B,H", PARITY)
def test_parity_matrix(rt, op, B, H, tf32):
    """forward / reverse / bidirectional and bias / initial state vary across the matrix; I != H throughout.  H = 1024
    takes the per-step path on its own (its R does not fit a cluster)."""
    k = PARITY.index((op, B, H))
    direction = ("forward", "reverse", "bidirectional")[k % 3]
    T = 9 if H < 1024 else 5
    ins = _case(op, T, B, H + 3 if H != 64 else 40, H, direction, bias=k % 2 == 0, init=k % 4 < 2, seed=k)
    ctx = _ctx(rt, tf32)
    got = _run(rt, ctx, op, ins, direction)
    _check_rule(got, op, ins, direction, tf32, f"{op} {direction} B={B} H={H}")
    if H <= 64:  # the per-step path at a cluster-sized shape
        got = _run(rt, ctx, op, ins, direction, per_step=True)
        _check_rule(got, op, ins, direction, tf32, f"{op} {direction} B={B} H={H} per-step")


@pytest.mark.gpu
@pytest.mark.parametrize("op", ["gru", "lstm"])
def test_each_output_alone(rt, op):
    ctx = _ctx(rt)
    ins = _case(op, 6, 3, 20, 16, "bidirectional", seed=3)
    full = _run(rt, ctx, op, ins, "bidirectional", packed=True)
    for i in range(len(full)):
        got = _run(rt, ctx, op, ins, "bidirectional", outputs=(i,), packed=True)
        assert all(g is None for j, g in enumerate(got) if j != i)
        np.testing.assert_array_equal(got[i], full[i])
    # sequence_lens is accepted and ignored, as the reference ignores it
    seq = np.array([1, 2, 3], np.int32)
    got = _run(rt, ctx, op, dict(ins, sequence_lens=seq), "bidirectional", packed=True)
    for g, e in zip(got, full):
        np.testing.assert_array_equal(g, e)


@pytest.mark.gpu
@pytest.mark.parametrize("op", ["gru", "lstm"])
def test_long_sequence(rt, op):
    """T = 2048 at H = 256: the error does not grow across steps beyond the f32 restatement's."""
    ins = _case(op, 2048, 2, 64, 256, "forward", seed=11)
    ctx = _ctx(rt)
    got = _run(rt, ctx, op, ins, "forward", packed=True)
    _check_rule(got, op, ins, "forward", False, f"{op} T=2048")


@pytest.mark.gpu
@pytest.mark.parametrize("op", ["gru", "lstm"])
def test_launch_counts_graph_replay_and_determinism(rt, op):
    """Device-resident, packed W: the cluster path is the projection GEMM's launches + 1; the per-step path adds the
    state init and T * (dirs + 1).  A captured call replays to the eager call's bits; repeated calls are identical."""
    T, B, I, H = 12, 4, 64, 32
    ctx = _ctx(rt)
    ins = _case(op, T, B, I, H, "bidirectional", seed=5)
    o = rt.GRU("bidirectional", H) if op == "gru" else rt.LSTM("bidirectional", H)
    pk = o.prepack(ctx, ins["w"])
    d = {k: ctx.to_device(v) for k, v in ins.items()}
    args = dict(b=d["b"], initial_h=d["initial_h"], packed_w=pk)
    if op == "lstm":
        args["initial_c"] = d["initial_c"]
    # the projection GEMM alone: MatMul of x [T * B, I] with the same packed matrix
    xd = d["x"].reshape(T * B, I)
    rt.MatMul().run(ctx, xd, ins["w"].reshape(-1, I).T.copy(), packed_b=pk)
    n0 = ctx.launches
    rt.MatMul().run(ctx, xd, ins["w"].reshape(-1, I).T.copy(), packed_b=pk)
    n_gemm = ctx.launches - n0

    def call():
        return o.run(ctx, d["x"], d["w"], d["r"], **args)

    eager = [t.numpy() for t in call()]
    n0 = ctx.launches
    again = [t.numpy() for t in call()]
    assert ctx.launches - n0 == n_gemm + 1, f"cluster path: {ctx.launches - n0} launches, expected {n_gemm + 1}"
    for a, b in zip(eager, again):
        np.testing.assert_array_equal(a, b)
    with gc.switches(RTEN_B200_NO_RNN_CLUSTER=1):
        n0 = ctx.launches
        per = [t.numpy() for t in call()]
        assert ctx.launches - n0 == n_gemm + 1 + T * 3, f"per-step path: {ctx.launches - n0} launches"
    _check_rule(per, op, ins, "bidirectional", False, "per-step")
    ctx.sync()
    ctx.graph_begin()
    cap = call()
    graph = ctx.graph_end()
    for _ in range(2):
        graph.launch()
        ctx.sync()
        for a, b in zip(cap, eager):
            np.testing.assert_array_equal(a.numpy(), b)


@pytest.mark.gpu
def test_errors(rt):
    ctx = _ctx(rt)
    z = lambda *s: np.zeros(s, np.float32)  # noqa: E731
    H, I, B, T = 4, 3, 2, 5

    def check(op, kind, msg, direction="forward", lbr=True, **over):
        G = 3 if op == "gru" else 4
        a = dict(x=z(T, B, I), w=z(1, G * H, I), r=z(1, G * H, H))
        a.update(over)
        o = rt.GRU(direction, H, lbr) if op == "gru" else rt.LSTM(direction, H)
        with pytest.raises(rt.OpError) as e:
            o.run(ctx, a.pop("x"), a.pop("w"), a.pop("r"), **a)
        assert (e.value.kind, e.value.msg) == (kind, msg)

    check("gru", "UnsupportedValue", "`linear_before_reset=0` is not supported", lbr=False)
    check("gru", "InvalidValue", "input must have 3 dims (seq, batch, input)", x=z(T, I))
    check("gru", "InvalidValue", "weights must have 3 dims (dir, hidden x 3, input)", w=z(12, I))
    check("gru", "InvalidValue", "recurrent_weights must have 3 dims", r=z(12, H))
    check("gru", "InvalidValue", "bias must have 2 dims (dir, hidden x 6)", b=z(24))
    check("gru", "InvalidValue", "initial_hidden must have 3 dims", initial_h=z(B, H))
    check("gru", "InvalidValue", "weights dim 1 must be 3 * hidden_size", w=z(1, 13, I))
    check("gru", "InvalidValue", "bias must have shape [directions, 2 * gates * hidden_size]", b=z(1, 23))
    check("lstm", "InvalidValue", "input must have 3 dims (seq, batch, input)", x=z(T, I))
    check("lstm", "InvalidValue", "weights must have 3 dims (dir, hidden x 4, input)", w=z(16, I))
    check("lstm", "InvalidValue", "recurrent_weights must have 3 dims (dir, hidden x 4, hidden)", r=z(16, H))
    check("lstm", "InvalidValue", "weights dim 1 must be 4 * hidden_size", w=z(1, 18, I))
    check("lstm", "InvalidValue", "bias must have 2 dims", b=z(32))
    check("lstm", "InvalidValue", "bias dim 1 must be 8 * hidden_size", b=z(1, 36))
    check("lstm", "InvalidValue", "bias must have shape [directions, 2 * gates * hidden_size]", b=z(1, 40))
    check("lstm", "InvalidValue", "initial_hidden must have 3 dims", initial_h=z(B, H))
    check("lstm", "InvalidValue", "initial_cell must have 3 dims", initial_c=z(B, H))
    check("lstm", "InvalidValue", "initial_cell must have shape [directions, batch, hidden_size]", initial_c=z(1, B + 1, H))
    check("lstm", "UnsupportedValue", "LSTM peephole weights are not supported", peephole=z(1, 12))
    check("lstm", "InvalidValue", "weights dim 0 must be the number of directions", direction="bidirectional")
    check("gru", "InvalidValue", "weights dim 2 must be the input size", w=z(1, 12, I + 1))
    check("gru", "InvalidValue", "recurrent_weights must have shape [directions, gates * hidden_size, hidden_size]", r=z(1, 12, H + 1))
    check("gru", "InvalidValue", "initial_hidden must have shape [directions, batch, hidden_size]", initial_h=z(1, B, H + 1))
    check("gru", "CastFailed", "sequence_lens must be i32", sequence_lens=z(B))


# ---------------------------------------------------------------------------------------------------------------------
# Whole model: a small CRNN recognizer through the ONNX executor
def _strings_attr(name, values):
    """A STRINGS AttributeProto as a NodeProto `attribute` field, appended to a node's bytes (fields may come in any
    order)."""
    import onnx_writer as W
    body = W._ld(1, name.encode()) + b"".join(W._ld(9, v.encode()) for v in values) + W._vi(20, 8)
    return W._ld(5, body)


def _crnn(op, H1=12, H2=10, C=4, classes=7, seed=2, extra_attrs=None, extra_inputs=()):
    import onnx_writer as W
    r = np.random.default_rng(seed)
    G = 3 if op == "GRU" else 4
    f = lambda *s, k=0.3: r.uniform(-k, k, s).astype(np.float32)  # noqa: E731
    wts = {"cw": f(C, 1, 3, 3), "cb": f(C), "w1": f(2, G * H1, C * 4), "r1": f(2, G * H1, H1), "b1": f(2, 2 * G * H1),
           "w2": f(2, G * H2, 2 * H1), "r2": f(2, G * H2, H2), "b2": f(2, 2 * G * H2), "fc": f(2 * H2, classes)}
    attrs = dict(hidden_size=H1, direction="bidirectional")
    if op == "GRU":
        attrs["linear_before_reset"] = 1
    attrs1 = dict(attrs, **(extra_attrs or {}))
    activations = attrs1.pop("activations", None)
    attrs2 = dict(attrs, hidden_size=H2)
    nodes = [W.node("Conv", ["x", "cw", "cb"], ["c"], pads=[1, 1, 1, 1]), W.node("Relu", ["c"], ["cr"]),
             W.node("MaxPool", ["cr"], ["p"], kernel_shape=[2, 2], strides=[2, 2]),
             W.node("Transpose", ["p"], ["pt"], perm=[3, 0, 1, 2]), W.node("Reshape", ["pt", "s1"], ["seq"]),
             W.node(op, ["seq", "w1", "r1", "b1", *extra_inputs], ["y1"], **attrs1)
             + (_strings_attr("activations", activations) if activations is not None else b""),
             W.node("Transpose", ["y1"], ["y1t"], perm=[0, 2, 1, 3]), W.node("Reshape", ["y1t", "s2"], ["seq2"]),
             W.node(op, ["seq2", "w2", "r2", "b2"], ["y2", "y2h"], **attrs2),
             W.node("Transpose", ["y2"], ["y2t"], perm=[0, 2, 1, 3]), W.node("Reshape", ["y2t", "s3"], ["seq3"]),
             W.node("MatMul", ["seq3", "fc"], ["logits"])]
    inits = [W.tensor(k, v) for k, v in wts.items()]
    inits += [W.tensor("s1", np.array([0, 0, -1], np.int64)), W.tensor("s2", np.array([0, 0, -1], np.int64)),
              W.tensor("s3", np.array([0, 0, -1], np.int64))]
    if extra_inputs:
        inits.append(W.tensor("P", f(2, 3 * H1)))
    data = W.model(nodes, inits, [W.value_info("x", W.FLOAT, [2, 1, 8, 16])],
                   [W.value_info("logits", W.FLOAT, [8, 2, classes]), W.value_info("y2h", W.FLOAT, [2, 2, H2])])
    return data, wts


def _torch_crnn(op, wts, x):
    import torch
    t = lambda a: torch.from_numpy(np.asarray(a, np.float64))  # noqa: E731
    c = torch.nn.functional.conv2d(t(x), t(wts["cw"]), t(wts["cb"]), padding=1)
    p = torch.nn.functional.max_pool2d(torch.relu(c), 2, 2)
    seq = p.permute(3, 0, 1, 2).reshape(p.shape[3], p.shape[0], -1)
    G = 3 if op == "GRU" else 4
    order = [1, 0, 2] if G == 3 else [0, 2, 3, 1]  # ONNX (z, r, h) / (i, o, f, c) -> torch (r, z, n) / (i, f, g, o)

    def layer(seq, w, r, b):
        H = r.shape[2]
        m = (torch.nn.GRU if G == 3 else torch.nn.LSTM)(w.shape[2], H, bidirectional=True).double()
        ro = lambda a: np.concatenate([a[i * H:(i + 1) * H] for i in order])  # noqa: E731
        with torch.no_grad():
            for d, sfx in enumerate(["", "_reverse"]):
                getattr(m, "weight_ih_l0" + sfx).copy_(t(ro(w[d])))
                getattr(m, "weight_hh_l0" + sfx).copy_(t(ro(r[d])))
                getattr(m, "bias_ih_l0" + sfx).copy_(t(ro(b[d][:G * H])))
                getattr(m, "bias_hh_l0" + sfx).copy_(t(ro(b[d][G * H:])))
            y, st = m(seq)
        hn = st if G == 3 else st[0]
        return y, hn

    y1, _ = layer(seq, wts["w1"], wts["r1"], wts["b1"])
    y2, h2 = layer(y1, wts["w2"], wts["r2"], wts["b2"])
    return (y2 @ t(wts["fc"])).numpy(), h2.numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("op", ["GRU", "LSTM"])
def test_crnn_through_the_onnx_executor(rt, op):
    from rten_b200.model import Model
    ctx = _ctx(rt)
    data, wts = _crnn(op)
    x = np.random.default_rng(9).uniform(0, 1, (2, 1, 8, 16)).astype(np.float32)
    m = Model(ctx, data)
    assert m.node_ops.count(op) == 2
    logits, yh = (t.numpy() for t in m.run({"x": x}, ["logits", "y2h"]))
    exp_logits, exp_h = _torch_crnn(op, wts, x)
    assert logits.shape == exp_logits.shape and yh.shape == exp_h.shape
    assert float(np.abs(logits - exp_logits).max()) < 1e-4
    assert float(np.abs(yh - exp_h).max()) < 1e-4
    refused = [dict(activation_alpha=[0.5]), dict(activation_beta=[0.5]), dict(activations=["Relu", "Tanh", "Tanh"][:3 if op == "LSTM" else 2]),
               dict(clip=1.0), dict(layout=1), dict(hidden_size=None)]
    if op == "LSTM":
        refused.append(dict(input_forget=1))
    for extra in refused:
        attrs = {k: v for k, v in extra.items() if v is not None}
        d, _ = _crnn(op, extra_attrs=attrs)
        if "hidden_size" in extra:
            d = d.replace(b"\n\x0bhidden_size", b"\n\x0bhidden_sizX", 1)
        with pytest.raises(rt.OpError) as e:
            Model(ctx, d)
        assert e.value.kind == "UnsupportedValue", (extra, e.value.msg)
    # the default activations, repeated per direction, load
    dflt = ["Sigmoid", "Tanh"] if op == "GRU" else ["Sigmoid", "Tanh", "Tanh"]
    Model(ctx, _crnn(op, extra_attrs=dict(activations=dflt * 2))[0])
    if op == "LSTM":
        with pytest.raises(rt.OpError) as e:
            Model(ctx, _crnn(op, extra_inputs=["", "", "", "P"])[0])
        assert e.value.kind == "UnsupportedValue" and "peephole" in e.value.msg


# ---------------------------------------------------------------------------------------------------------------------
def _kernel_probe():
    """Run in a child process: the kernels of a cluster-sized call and of an H = 1024 call, one CUPTI session each."""
    import gpu_checks as gc
    import rten_b200 as rt
    ctx = _ctx(rt)
    res = {}
    for name, (op, B, H) in {"gru256": ("gru", 8, 256), "lstm256": ("lstm", 3, 256), "lstm1024": ("lstm", 4, 1024)}.items():
        ins = _case(op, 4, B, 64, H, "bidirectional", seed=1)
        _, names = gc._kernels_launched(lambda: _run(rt, ctx, op, ins, "bidirectional"))
        res[name] = sorted(names)
    print(json.dumps(res))


@pytest.mark.gpu
def test_kernel_identity():
    import subprocess
    import sys
    code = (f"import sys; sys.path[:0] = [{os.path.dirname(HERE)!r}, {HERE!r}]; "
            "import test_gpu_rnn as t; t._kernel_probe()")
    res = subprocess.run([sys.executable, "-s", "-c", code], capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-4000:]
    names = json.loads(res.stdout.strip().splitlines()[-1])
    has = lambda key, k: any(k in n for n in names[key])  # noqa: E731
    for key in ("gru256", "lstm256"):
        assert has(key, "rnn_cluster_kernel") and not has(key, "rnn_step_gates_kernel"), names[key]
    assert has("lstm1024", "rnn_step_gates_kernel") and not has("lstm1024", "rnn_cluster_kernel"), names["lstm1024"]
    # the per-step path sets its state buffers from h0 / c0 (or zeros) first
    assert has("lstm1024", "rnn_state_init_kernel") and not has("lstm256", "rnn_state_init_kernel"), names["lstm1024"]
