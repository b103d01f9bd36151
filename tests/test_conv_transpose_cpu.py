"""ConvTranspose without a GPU: the CPU restatement of the reference (oracle/conv_transpose.py) against the reference's
known answers (tests/golden/conv_transpose_cases.json) and float64 torch, the stride-phase decomposition the CUDA path
uses (restated with oracle.conv) against it, and the C-ABI parameter struct."""
import ctypes
import json
import os

import numpy as np
import pytest

import conv_transpose_sweep as sw
from oracle import oracle
from oracle.conv_transpose import conv_transpose, output_size_and_padding

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = json.load(open(os.path.join(HERE, "golden", "conv_transpose_cases.json")))


def _rule(got, want, what):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    assert got.shape == want.shape, f"{what}: shape {got.shape} != {want.shape}"
    bad = np.abs(got - want) > 1e-8 + 1e-5 * np.abs(want)
    assert not bad.any(), f"{what}: {int(bad.sum())} of {bad.size} elements outside 1e-8 + 1e-5*|want|"


def golden_args(c):
    x = np.asarray(c["input"], np.float32).reshape(c["input_shape"])
    w = np.asarray(c["kernel"], np.float32).reshape(c["kernel_shape"])
    b = None if c["bias"] is None else np.asarray(c["bias"], np.float32)
    return x, w, b, dict(padding=c["padding"], groups=c["groups"], strides=tuple(c["strides"]),
                         dilations=tuple(c["dilations"]), output_padding=tuple(c["output_padding"]))


@pytest.mark.parametrize("c", GOLDEN["cases"], ids=lambda c: c["name"])
def test_oracle_reproduces_golden_case(c):
    x, w, b, kw = golden_args(c)
    y = conv_transpose(x, w, b, **kw)
    assert list(y.shape) == c["expected_shape"]
    if c["expected"] is not None:
        _rule(y.reshape(-1), c["expected"], c["name"])


@pytest.mark.parametrize("row", GOLDEN["output_size_and_padding"], ids=lambda r: str(r.get("error", r.get("expected_shape"))))
def test_oracle_output_size_and_padding(row):
    args = (row["input_shape"], row["kernel_shape"], row["padding"], row["strides"], row["dilations"], row["output_padding"])
    if "error" in row:
        with pytest.raises(oracle.OpError) as e:
            output_size_and_padding(*args)
        assert [e.value.kind, e.value.msg] == row["error"]
    else:
        shape, pads = output_size_and_padding(*args)
        assert [list(shape), pads] == [row["expected_shape"], row["expected_pads"]]


@pytest.mark.parametrize("case", sw.SWEEP, ids=[c[0] for c in sw.SWEEP])
def test_oracle_matches_torch_float64(case):
    x, w, b = sw.case_data(oracle, case)
    want, _ = sw.torch_f64(x, w, b, case)
    _rule(conv_transpose(x, w, b, **sw.op_args(case)), want, case[0])


@pytest.mark.parametrize("case", sw.SWEEP, ids=[c[0] for c in sw.SWEEP])
def test_phase_decomposition_matches_oracle(case):
    """The CUDA path's arithmetic plan: one stride-1 convolution per phase with taps (oracle.conv), bias elsewhere."""
    x, w, b = sw.case_data(oracle, case)
    kw = sw.op_args(case)
    want = conv_transpose(x, w, b, **kw)
    if x.ndim == 3:
        pad = kw["padding"]
        kw = dict(groups=kw["groups"], strides=(1,) + kw["strides"], dilations=(1,) + kw["dilations"],
                  output_padding=(0,) + kw["output_padding"], padding=pad if pad == "same" else (0, pad[0], 0, pad[1]))
        got = sw.phase_decomposition(oracle, x[:, :, None, :], w[:, :, None, :], b, **kw)[:, :, 0, :]
    else:
        got = sw.phase_decomposition(oracle, x, w, b, **kw)
    _rule(got, want, case[0])


def test_tap_less_phases_hold_the_bias():
    """k = 1, s = 2: three of four phases receive no tap, only the bias."""
    r = oracle.XorShiftRng(7)
    x, w, b = r.uniform((1, 4, 3, 3)), r.uniform((4, 2, 1, 1)), r.uniform((2,))
    y = conv_transpose(x, w, b, strides=(2, 2), output_padding=(1, 1))
    assert y.shape == (1, 2, 6, 6)
    mask = np.ones((6, 6), bool)
    mask[0::2, 0::2] = False
    assert (y[0][:, mask] == b[:, None]).all()


@pytest.mark.parametrize("kw, err", [
    (dict(w_shape=(3, 2, 2, 2)), ("IncompatibleInputShapes", "Input channels does not match kernel input channels")),
    (dict(groups=3), ("InvalidValue", "Input channel count not divisible by groups")),
    (dict(groups=0), ("InvalidValue", "Group count must be > 0")),
    (dict(bias=np.zeros(3, np.float32)), ("IncompatibleInputShapes", "bias.size(0) != out_channels")),
    (dict(strides=(2,)), ("InvalidValue", "expected 2 stride values")),
    (dict(dilations=(1, 1, 1)), ("InvalidValue", "expected 2 dilation values")),
    (dict(output_padding=(1,)), ("InvalidValue", "expected 2 output_padding values")),
    (dict(padding=(0, 0)), ("InvalidValue", "Wrong number of pad values")),
    (dict(w_shape=(4, 2, 2)), ("InvalidValue", "kernel must have 4 dims (COHW)")),
])
def test_oracle_errors(kw, err):
    x = np.zeros((1, 4, 3, 3), np.float32)
    w = np.zeros(kw.pop("w_shape", (4, 2, 2, 2)), np.float32)
    args = dict(strides=(2, 2))
    args.update(kw)
    with pytest.raises(oracle.OpError) as e:
        conv_transpose(x, w, **args)
    assert (e.value.kind, e.value.msg) == err


def test_oracle_1d_errors():
    x, w = np.zeros((1, 4, 3), np.float32), np.zeros((4, 2, 2), np.float32)
    for kw, msg in [(dict(strides=(2, 2)), "expected 1 stride value"), (dict(strides=(2,), padding=(0, 0, 0, 0)), "expected 2 pad values"),
                    (dict(strides=(2,), dilations=(1, 1)), "expected 1 dilation value"),
                    (dict(strides=(2,), dilations=(1,), output_padding=(0, 0)), "expected 1 output_padding value")]:
        kw.setdefault("dilations", (1,))
        kw.setdefault("padding", (0, 0))
        with pytest.raises(oracle.OpError) as e:
            conv_transpose(x, w, **kw)
        assert e.value.msg == msg
    with pytest.raises(oracle.OpError) as e:
        conv_transpose(x, np.zeros((4, 2, 1, 2), np.float32), strides=(2,), dilations=(1,), padding=(0, 0))
    assert e.value.msg == "kernel must have 3 dims (OCW)"


def test_params_struct_matches_header():
    from rten_b200._lib import RtenConvTransposeParams
    # pads[4], auto_pad_same, groups, strides[2], dilations[2], output_padding[2], n_pads, n_strides, n_dilations,
    # n_output_padding: all int32
    assert ctypes.sizeof(RtenConvTransposeParams) == 16 + 4 + 4 + 8 + 8 + 8 + 4 * 4
    src = open(os.path.join(os.path.dirname(HERE), "include", "rten_b200.h")).read()
    end = src.index("} rten_conv_transpose_params;")
    body = src[src.rindex("typedef struct {", 0, end) + len("typedef struct {"):end]
    header = [f.strip().rstrip(";").split()[1] for f in body.strip().splitlines()]
    ours = [n + (f"[{t._length_}]" if hasattr(t, "_length_") else "") for n, t in RtenConvTransposeParams._fields_]
    assert header == ours
