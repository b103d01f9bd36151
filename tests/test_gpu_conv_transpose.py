"""`pytest -m gpu`: rten_b200_conv_transpose -- ConvTranspose as stride-phase convolutions on the implicit-GEMM conv
kernel, one launch per phase with taps and one fill launch for the phases without.

  * the reference's known answers (tests/golden/conv_transpose_cases.json) through the C ABI;
  * the sweep of tests/conv_transpose_sweep.py (groups up to groups = channels, dilation, asymmetric pads, output
    padding, SAME, 1-D; implicit and explicit channel counts; tap-less phases) in NCHW and channels-last, against
    float64: 3xTF32 within 1e-8 + 1e-5*|b|, single-pass TF32 within 2^-9 * conv_transpose(|x|, |w|);
  * prepacked and per-call weights give the same bits; the launch count of a prepacked channels-last TF32 call;
  * a captured CUDA graph replays to the eager result; errors carry the reference's status and message;
  * Model: Conv -> Relu -> ConvTranspose(bias) -> Add equals the op-by-op result; output_shape fails the load."""
import json
import os

import numpy as np
import pytest

import conv_transpose_sweep as sw
import gpu_checks as gc

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = json.load(open(os.path.join(HERE, "golden", "conv_transpose_cases.json")))


@pytest.fixture(scope="module")
def rt():
    import rten_b200
    from rten_b200 import _lib
    _lib.load()
    return rten_b200


@pytest.fixture(scope="module")
def oracle():
    from oracle import oracle as o
    return o


def _dev(ctx, a, cl):
    """Device copy of a 3-D / 4-D array, channels-last when `cl`."""
    if not cl or a.ndim == 4:
        return ctx.to_device(a, channels_last=cl)
    b, c, w = a.shape
    t = ctx.empty(a.shape, a.dtype, (w * c, 1, c))
    t.copy_from(a)
    return t


def _op(rt, case):
    return rt.ConvTranspose(**sw.op_args(case))


@pytest.mark.parametrize("c", GOLDEN["cases"], ids=lambda c: c["name"])
def test_golden_case(rt, c):
    ctx = rt.Context(0)
    x = np.asarray(c["input"], np.float32).reshape(c["input_shape"])
    w = np.asarray(c["kernel"], np.float32).reshape(c["kernel_shape"])
    b = None if c["bias"] is None else np.asarray(c["bias"], np.float32)
    op = rt.ConvTranspose(groups=c["groups"], dilations=c["dilations"], padding=c["padding"], strides=c["strides"],
                          output_padding=c["output_padding"])
    y = op.run(ctx, x, w, b).numpy()
    assert list(y.shape) == c["expected_shape"]
    if c["expected"] is not None:
        gc.assert_reference_rule(y.reshape(-1), np.asarray(c["expected"]), c["name"])


@pytest.mark.parametrize("tf32", [False, True], ids=["3xTF32", "TF32"])
@pytest.mark.parametrize("case", sw.SWEEP, ids=[c[0] for c in sw.SWEEP])
def test_sweep_against_float64(rt, oracle, case, tf32):
    ctx = gc.new_ctx(rt, tf32=tf32)
    x, w, b = sw.case_data(oracle, case)
    want, absum = sw.torch_f64(x, w, b, case)
    op = _op(rt, case)
    pk = op.prepack(ctx, 1, ctx.to_device(w))
    for cl in (False, True):
        xd = _dev(ctx, x, cl)
        got = op.run(ctx, xd, w, b).numpy()
        what = f"{case[0]} cl={cl} {'TF32' if tf32 else '3xTF32'}"
        if tf32:
            gc.assert_tf32_close(got, want, absum, what)
        else:
            gc.assert_reference_rule(got, want, what)
        y = op.run(ctx, xd, w, b, packed_w=pk)
        if cl and x.shape[1] > 1:
            assert y.strides[1] == 1, f"{what}: channels-last input must give channels-last output, got {y.strides}"
        gc.assert_bit_exact(y.numpy(), got, f"{what}: prepacked vs per-call weights")


def _phase_counts(case, x_shape, w_shape):
    """(phases with a convolution, phases without) of a 2-D case, restating the decomposition's rules."""
    from oracle.conv_transpose import output_size_and_padding
    _, _, _, k, s, d, pad, op, _ = case
    (OH, OW), pads = output_size_and_padding(x_shape[2:], k, pad, s, d, op)
    import math

    def live(n_in, n_out, kk, ss, dd, p, q):
        taps = [t for t in range(kk - 1, -1, -1) if (t * dd) % ss == (q + p) % ss]
        n = -(-(n_out - q) // ss)
        if not taps or n <= 0:
            return False
        e0 = (q + p - taps[0] * dd) // ss
        last = n - 1 + e0 + (len(taps) - 1) * (dd // math.gcd(dd, ss))
        return max(e0, 0) <= min(last, n_in - 1)

    ly = [live(x_shape[2], OH, k[0], s[0], d[0], pads[0], q) for q in range(min(s[0], OH))]
    lx = [live(x_shape[3], OW, k[1], s[1], d[1], pads[1], q) for q in range(min(s[1], OW))]
    n_live = sum(a and b for a in ly for b in lx)
    return n_live, len(ly) * len(lx) - n_live


@pytest.mark.parametrize("case", [c for c in sw.SWEEP if len(c[1]) == 4 and c[8] == 1 and c[1][1] % 8 == 0],
                         ids=lambda c: c[0])
def test_launch_count(rt, oracle, case):
    """Channels-last, single-pass TF32, prepacked, groups 1: (phases with taps) + (1 if any phase has none)."""
    ctx = gc.new_ctx(rt, tf32=True)
    x, w, b = sw.case_data(oracle, case)
    op = _op(rt, case)
    pk = op.prepack(ctx, 1, ctx.to_device(w))
    xd, wd, bd = ctx.to_device(x, channels_last=True), ctx.to_device(w), ctx.to_device(b)
    op.run(ctx, xd, wd, bd, packed_w=pk)
    ctx.sync()
    n_live, n_empty = _phase_counts(case, x.shape, w.shape)
    before = ctx.launches
    op.run(ctx, xd, wd, bd, packed_w=pk)
    ctx.sync()
    assert ctx.launches - before == n_live + (1 if n_empty else 0), (case[0], n_live, n_empty)


@pytest.mark.parametrize("tf32", [False, True], ids=["3xTF32", "TF32"])
def test_graph_replay(rt, oracle, tf32):
    case = sw.SWEEP[1]
    ctx = gc.new_ctx(rt, tf32=tf32)
    x, w, b = sw.case_data(oracle, case)
    op = _op(rt, case)
    pk = op.prepack(ctx, 1, ctx.to_device(w))
    xd, wd, bd = ctx.to_device(x, channels_last=True), ctx.to_device(w), ctx.to_device(b)
    eager = op.run(ctx, xd, wd, bd, packed_w=pk).numpy()
    out, g = gc._replayed(ctx, lambda: op.run(ctx, xd, wd, bd, packed_w=pk))
    gc.assert_bit_exact(out.numpy(), eager, f"graph replay ({'TF32' if tf32 else '3xTF32'})")


def test_large_layers_against_float64(rt, oracle):
    """The benchmarked decoder shapes (smaller batch): SAM k2 s2 and DCGAN k4 s2 p1, channels-last, both modes."""
    cases = [("SAM 256->64 k2 s2", (1, 256, 16, 16), 64, (2, 2), (2, 2), (1, 1), (0, 0, 0, 0), (0, 0), 1),
             ("DCGAN 256->128 k4 s2 p1", (2, 256, 8, 8), 128, (4, 4), (2, 2), (1, 1), (1, 1, 1, 1), (0, 0), 1),
             ("DPT 48 k4 s4", (1, 48, 13, 13), 48, (4, 4), (4, 4), (1, 1), (0, 0, 0, 0), (0, 0), 1)]
    for tf32 in (False, True):
        ctx = gc.new_ctx(rt, tf32=tf32)
        for case in cases:
            x, w, b = sw.case_data(oracle, case)
            want, absum = sw.torch_f64(x, w, b, case)
            op = _op(rt, case)
            pk = op.prepack(ctx, 1, ctx.to_device(w))
            got = op.run(ctx, ctx.to_device(x, channels_last=True), w, b, packed_w=pk).numpy()
            if tf32:
                gc.assert_tf32_close(got, want, absum, case[0])
            else:
                gc.assert_reference_rule(got, want, case[0])


def test_errors(rt):
    ctx = rt.Context(0)
    x = np.zeros((1, 4, 3, 3), np.float32)
    w = np.zeros((4, 2, 2, 2), np.float32)

    def err(fn):
        with pytest.raises(rt.OpError) as e:
            fn()
        return e.value.kind, e.value.msg

    T = rt.ConvTranspose
    cases = [
        (lambda: T(strides=(2, 2)).run(ctx, np.zeros((1, 3, 3, 3), np.float32), w),
         ("IncompatibleInputShapes", "Input channels does not match kernel input channels")),
        (lambda: T(groups=3, strides=(2, 2)).run(ctx, x, w), ("InvalidValue", "Input channel count not divisible by groups")),
        (lambda: T(groups=0).run(ctx, x, w), ("InvalidValue", "Group count must be > 0")),
        (lambda: T(strides=(2, 2)).run(ctx, x, w, np.zeros(3, np.float32)), ("IncompatibleInputShapes", "bias.size(0) != out_channels")),
        (lambda: T(strides=(2,)).run(ctx, x, w), ("InvalidValue", "expected 2 stride values")),
        (lambda: T(dilations=(1,)).run(ctx, x, w), ("InvalidValue", "expected 2 dilation values")),
        (lambda: T(output_padding=(1,)).run(ctx, x, w), ("InvalidValue", "expected 2 output_padding values")),
        (lambda: T(padding=(0, 0)).run(ctx, x, w), ("InvalidValue", "Wrong number of pad values")),
        (lambda: T(strides=(0, 0)).run(ctx, x, w), ("InvalidValue", "Strides must be > 0")),
        (lambda: T(dilations=(0, 1)).run(ctx, x, w), ("InvalidValue", "Dilations must be > 0")),
        (lambda: T().run(ctx, x, np.zeros((4, 2, 0, 2), np.float32)), ("InvalidValue", "Kernel size must be > 0")),
        (lambda: T().run(ctx, np.zeros((1, 4, 0, 3), np.float32), w), ("InvalidValue", "Input width and height must be > 0")),
        (lambda: T(padding=(4, 4, 4, 4)).run(ctx, x, w), ("InvalidValue", "Input is too small")),
        (lambda: T(padding="same", strides=(3, 3)).run(ctx, x, np.zeros((4, 2, 1, 1), np.float32)), ("InvalidValue", "Input is too small")),
        (lambda: T().run(ctx, x, np.zeros((4, 2, 2), np.float32)), ("InvalidValue", "kernel must have 4 dims (COHW)")),
        (lambda: T(strides=(2,), dilations=(1,), padding=(0, 0)).run(ctx, np.zeros((1, 4, 3), np.float32), w),
         ("InvalidValue", "kernel must have 3 dims (OCW)")),
        (lambda: T(strides=(2,), dilations=(1,), padding=(0, 0, 0, 0)).run(ctx, np.zeros((1, 4, 3), np.float32), w[:, :, 0]),
         ("InvalidValue", "expected 2 pad values")),
        (lambda: T(strides=(2, 2), dilations=(1,), padding=(0, 0)).run(ctx, np.zeros((1, 4, 3), np.float32), w[:, :, 0]),
         ("InvalidValue", "expected 1 stride value")),
        (lambda: T(strides=(2,), dilations=(1,), padding=(0, 0), output_padding=(0, 0)).run(ctx, np.zeros((1, 4, 3), np.float32), w[:, :, 0]),
         ("InvalidValue", "expected 1 output_padding value")),
        (lambda: T().run(ctx, x.astype(np.int32), w), ("UnsupportedType", "unsupported type")),
    ]
    for fn, want in cases:
        assert err(fn) == want
    # batch 0: an empty output of the right shape
    y = T(strides=(2, 2)).run(ctx, np.zeros((0, 4, 3, 3), np.float32), w)
    assert y.shape == (0, 2, 6, 6)
    # a prepacked weight built for other strides is refused
    pk = T(strides=(2, 2)).prepack(ctx, 1, w)
    assert err(lambda: T(strides=(3, 3)).run(ctx, x, w, packed_w=pk))[0] == "InvalidValue"


def _model_bytes(onnx_writer, consts, output_shape=None):
    ct_attrs = dict(strides=[2, 2], pads=[1, 1, 1, 1], kernel_shape=[4, 4], output_padding=[1, 1])
    if output_shape is not None:
        ct_attrs["output_shape"] = output_shape
    W = onnx_writer
    nodes = [W.node("Conv", ["x", "w1", "b1"], ["c"], pads=[1, 1, 1, 1], kernel_shape=[3, 3]),
             W.node("Relu", ["c"], ["r"]),
             W.node("ConvTranspose", ["r", "wt", "bt"], ["t"], **ct_attrs),
             W.node("Add", ["t", "res"], ["y"])]
    inits = [W.tensor(k, v) for k, v in consts.items()]
    return W.model(nodes, inits, [W.value_info("x", 1, (2, 8, 6, 6)), W.value_info("res", 1, (2, 8, 13, 13))],
                   [W.value_info("y", 1, (2, 8, 13, 13))])


def test_model_conv_relu_conv_transpose_add(rt, oracle):
    import onnx_writer
    from rten_b200.model import Model
    r = oracle.XorShiftRng(31)
    x = r.uniform((2, 8, 6, 6))
    consts = {"w1": r.uniform((16, 8, 3, 3)) / np.float32(8.0), "b1": r.uniform((16,)),
              "wt": r.uniform((16, 8, 4, 4)) / np.float32(8.0), "bt": r.uniform((8,))}
    res = r.uniform((2, 8, 13, 13))
    ctx = rt.Context(0)
    m = Model(ctx, _model_bytes(onnx_writer, consts))
    assert m.node_ops == ["Conv", "ConvTranspose", "Add"]
    got = m.run({"x": x, "res": res}, ["y"])[0].numpy()
    c = rt.Conv(padding=(1, 1, 1, 1), activation=rt.ACT_RELU).run(ctx, x, consts["w1"], consts["b1"])
    ct = rt.ConvTranspose(strides=(2, 2), padding=(1, 1, 1, 1), output_padding=(1, 1))
    t = ct.run(ctx, c, consts["wt"], consts["bt"], packed_w=ct.prepack(ctx, 1, consts["wt"]))
    want = rt.Add().run(ctx, t, res).numpy()
    gc.assert_bit_exact(got, want, "Model Conv -> Relu -> ConvTranspose -> Add vs op by op")
    with pytest.raises(rt.OpError) as e:
        Model(ctx, _model_bytes(onnx_writer, consts, output_shape=[13, 13]))
    assert e.value.kind == "UnsupportedValue"
