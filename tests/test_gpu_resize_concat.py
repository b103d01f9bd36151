"""GPU checks of Resize, Concat, AveragePool and the executor's in-place Concat: every operator bit-exact against
oracle/resize.py across modes, layouts, ranks and output strides; the decoder models of tests/decoder_models.py through
the model API in both f32 modes, with the Concat elision on and off giving identical bits."""
import itertools
import json

import numpy as np
import pytest

import decoder_models as D
import gpu_checks
from oracle import resize as R

pytestmark = pytest.mark.gpu
F32 = np.float32


@pytest.fixture(scope="module")
def rt():
    import rten_b200
    import rten_b200.model  # noqa: F401
    return rten_b200


@pytest.fixture(scope="module")
def ctx(rt):
    return rt.Context(0)


def _rand(shape, seed=0):
    return np.random.default_rng(seed).standard_normal(shape).astype(F32)


def _sliced(ctx, x):
    """x as a non-contiguous device view: the odd columns and rows of a buffer twice as large in H and W"""
    big = np.zeros(x.shape[:2] + (2 * x.shape[2], 2 * x.shape[3]), F32)
    big[:, :, 1::2, 1::2] = x
    t = ctx.to_device(big)
    s = t.strides
    return t.view(x.shape, (s[0], s[1], 2 * s[2], 2 * s[3]), s[2] + s[3])


def _layouts(ctx, x):
    yield "nchw", ctx.to_device(x)
    yield "channels_last", ctx.to_device(x, channels_last=True)
    yield "sliced", _sliced(ctx, x)


TARGETS = [dict(scales=[1, 1, 2, 2]), dict(scales=[1, 1, 0.5, 0.5]), dict(scales=[1, 1, 1.7, 1.7]), dict(scales=[1, 1, 2, 3]),
           dict(sizes=[2, None, 1, 1]), dict(sizes=[2, None, 13, 1]), dict(sizes=[2, None, 5, 9])]
MODES = [("nearest", nm) for nm in R.NEAREST_MODES] + [("linear", "floor")]


@pytest.mark.parametrize("channels", [1, 3, 4, 6, 64])
def test_resize_bit_exact(rt, ctx, channels):
    x = _rand((2, channels, 7, 9), channels)
    for (mode, nm), cm, tgt in itertools.product(MODES, R.COORD_MODES, TARGETS):
        tgt = {k: [channels if v is None else v for v in vs] for k, vs in tgt.items()}
        want = R.resize(x, mode=mode, coord_mode=cm, nearest_mode=nm, **tgt)
        op = rt.Resize(mode, cm, nm)
        for name, xd in _layouts(ctx, x):
            got = op.run(ctx, xd, **tgt)
            if name == "channels_last" and channels > 1:
                assert got.strides[1] == 1, "a channels-last input gives a channels-last output"
            gpu_checks.assert_bit_exact(got.numpy(), want, f"Resize {mode}/{nm}/{cm} {tgt} {name} C={channels}")


def test_resize_into_a_strided_output(rt, ctx):
    x = _rand((2, 8, 6, 5), 1)
    want = R.resize(x, scales=[1, 1, 2, 2], mode="linear")
    for cl in (False, True):
        # the output is channels [4, 12) of a 16-channel buffer
        buf = ctx.to_device(np.full((2, 16, 12, 10), 7.0, F32), channels_last=cl)
        out = buf.view(want.shape, buf.strides, 4 * buf.strides[1])
        rt.Resize("linear").run(ctx, ctx.to_device(x, channels_last=cl), scales=[1, 1, 2, 2], out=out)
        full = buf.numpy()
        gpu_checks.assert_bit_exact(full[:, 4:12], want, f"Resize into a slice (channels_last={cl})")
        assert (full[:, :4] == 7.0).all() and (full[:, 12:] == 7.0).all()


def test_resize_ranks_copy_and_errors(rt, ctx):
    for shape, scales in [((9,), [2.5]), ((4, 6), [2, 0.5]), ((2, 3, 5), [1, 1, 3]), ((2, 3, 5), [1, 2, 2]), ((2, 3, 4, 5), [1, 1, 1, 1])]:
        x = _rand(shape, len(shape))
        for mode in ("nearest", "linear"):
            got = rt.Resize(mode).run(ctx, x, scales=scales).numpy()
            gpu_checks.assert_bit_exact(got, R.resize(x, scales=scales, mode=mode), f"Resize rank {len(shape)} {mode}")
    assert rt.Resize().run(ctx, _rand((1, 1, 2, 2)), scales=[1, 1, 0, 0]).shape == (1, 1, 0, 0)
    for scales, kind in [([1, 1, 1], "IncompatibleInputShapes"), ([1, 1, -1, 1], "InvalidValue"), ([2, 1, 3, 3], "UnsupportedValue")]:
        with pytest.raises(rt.OpError) as e:
            rt.Resize("linear").run(ctx, _rand((1, 1, 2, 2)), scales=scales)
        assert e.value.kind == kind


@pytest.mark.parametrize("case", [((8, 256, 33, 33), [8, 256, 129, 129], "linear", "half_pixel"),
                                  ((8, 256, 32, 32), [8, 256, 64, 64], "nearest", "asymmetric"),
                                  ((1, 256, 96, 96), [1, 256, 192, 192], "linear", "align_corners")])
def test_resize_benched_sizes(rt, ctx, case):
    shape, sizes, mode, cm = case
    x = _rand(shape, 3)
    want = R.resize(x, sizes=sizes, mode=mode, coord_mode=cm, nearest_mode="floor")
    for cl in (False, True):
        got = rt.Resize(mode, cm, "floor").run(ctx, ctx.to_device(x, channels_last=cl), sizes=sizes).numpy()
        gpu_checks.assert_bit_exact(got, want, f"Resize {shape} -> {sizes} channels_last={cl}")


@pytest.mark.parametrize("dtype", [np.float32, np.int32, np.int8, np.uint8])
def test_concat_bit_exact(rt, ctx, dtype):
    rng = np.random.default_rng(5)

    def arr(shape):
        return rng.integers(-100, 100, shape).astype(dtype) if dtype != np.uint8 else rng.integers(0, 200, shape).astype(dtype)

    base = [2, 4, 6, 8]
    for axis, counts in itertools.product(range(-1, 4), [(4, 8), (3, 1, 5, 2, 7), tuple(range(1, 21))]):
        xs = []
        for n in counts:
            s = list(base)
            s[axis] = n
            xs.append(arr(s))
        before = ctx.launches
        got = rt.Concat(axis).run(ctx, [ctx.to_device(a) for a in xs])
        launches = ctx.launches - before
        assert launches == (len(xs) + 15) // 16, f"Concat of {len(xs)}: {launches} launches"
        gpu_checks.assert_bit_exact(got.numpy(), R.concat(xs, axis), f"Concat {np.dtype(dtype).name} axis {axis} x{len(xs)}")


def test_concat_layouts_and_in_place_inputs(rt, ctx):
    a, b, c = _rand((2, 8, 5, 6), 1), _rand((2, 3, 5, 6), 2), _rand((2, 5, 5, 6), 3)
    want = R.concat([a, b, c], 1)
    got = rt.Concat(1).run(ctx, [ctx.to_device(t, channels_last=True) for t in (a, b, c)])
    assert got.strides[1] == 1, "channels-last inputs give a channels-last output"
    gpu_checks.assert_bit_exact(got.numpy(), want, "Concat channels-last, misaligned slices")
    got = rt.Concat(1).run(ctx, [_sliced(ctx, a), ctx.to_device(b, channels_last=True), ctx.to_device(c)])
    gpu_checks.assert_bit_exact(got.numpy(), want, "Concat mixed layouts")
    # inputs that already are their slice of the output are not copied
    for cl in (False, True):
        out = ctx.to_device(np.zeros(want.shape, F32), channels_last=cl)
        views = [out.view(t.shape, out.strides, o * out.strides[1]) for t, o in ((a, 0), (b, 8), (c, 11))]
        views[0].copy_from(a) if views[0].is_contiguous() else rt.Resize().run(ctx, a, scales=[1, 1, 1, 1], out=views[0])
        rt.Resize().run(ctx, c, scales=[1, 1, 1, 1], out=views[2])
        before = ctx.launches
        rt.Concat(1).run(ctx, [views[0], ctx.to_device(b), views[2]], out=out)
        assert ctx.launches - before == 1
        gpu_checks.assert_bit_exact(out.numpy(), want, "Concat with two inputs in place")
        before = ctx.launches
        rt.Concat(1).run(ctx, views, out=out)
        assert ctx.launches - before == 0, "every input in place: nothing to launch"
    with pytest.raises(rt.OpError) as e:
        rt.Concat(0).run(ctx, [_rand((5, 10)), _rand((5, 11))])
    assert e.value.kind == "IncompatibleInputShapes"
    with pytest.raises(rt.OpError) as e:
        rt.Concat(2).run(ctx, [_rand((5, 10)), _rand((5, 10))])
    assert e.value.kind == "InvalidValue"


@pytest.mark.parametrize("count_include_pad", [False, True])
def test_average_pool_bit_exact(rt, ctx, count_include_pad):
    for channels, kernel, pads, strides in [(5, (2, 2), (0, 0, 0, 0), (2, 2)), (8, (3, 3), (1, 1, 1, 1), (1, 1)),
                                            (8, (3, 2), (1, 0, 1, 1), (2, 3)), (3, (5, 5), (2, 2, 2, 2), (3, 3))]:
        x = _rand((2, channels, 11, 13), channels)
        want = R.average_pool(x, kernel, pads, strides, count_include_pad)
        for name, xd in _layouts(ctx, x):
            got = rt.AveragePool(kernel, pads, strides, count_include_pad).run(ctx, xd).numpy()
            gpu_checks.assert_bit_exact(got, want, f"AveragePool k{kernel} p{pads} s{strides} {name}")


def _run_model(rt, data, x, tf32, elide, outputs=None):
    with gpu_checks.switches(RTEN_B200_NO_CONCAT_ELISION=None if elide else 1):
        ctx = gpu_checks.new_ctx(rt, tf32)
        model = rt.model.Model(ctx, data)
    xd = ctx.to_device(x, channels_last=True)
    model.run({"x": xd}, outputs)  # (first run: weights split / plans made)
    before = ctx.launches
    outs = [o.numpy() for o in model.run({"x": xd}, outputs)]
    return outs, ctx.launches - before, model.summary


@pytest.mark.parametrize("tf32", [True, False])
@pytest.mark.parametrize("name", sorted(D.MODELS))
def test_decoder_models(rt, name, tf32):
    data, forward, shape, n_concat = D.MODELS[name]()
    x = _rand(shape, 11)
    want = forward(x)
    on, launches_on, summary_on = _run_model(rt, data, x, tf32, True)
    off, launches_off, summary_off = _run_model(rt, data, x, tf32, False)
    tol = 2e-2 if tf32 else 1e-4
    for g, g_off, w in zip(on, off, want):
        assert g.shape == w.shape
        assert np.abs(g - w).max() <= tol * np.abs(w).max(), f"{name}: error {np.abs(g - w).max():.3e} vs scale {np.abs(w).max():.3e}"
        gpu_checks.assert_bit_exact(g, g_off, f"{name}: elision on vs off")
    plan = summary_on["concat_in_place"]
    assert "concat_in_place" not in summary_off
    fully = [p for p in plan if p["copied"] == 0]
    expect = {"unet": 2, "aspp": 1, "sppf": 1, "densenet": 1, "fpn": 0, "skip_and_output": 0, "upsample_concat": 1}[name]
    assert len(fully) == expect, json.dumps(plan)
    if name == "upsample_concat":  # the Resize by scales computes its output size as the operator does
        assert any(v.startswith("resize") for v in plan[0]["in_place"]), json.dumps(plan)
    assert launches_off - launches_on >= len(fully), f"{name}: {launches_on} launches with elision, {launches_off} without"
    if name == "skip_and_output":
        assert len(plan) == 1 and plan[0]["copied"] == 1 and len(plan[0]["in_place"]) == 1  # the graph output is copied
    if name == "densenet":
        # each Concat of the chain takes the previous Concat's output (copied) and one convolution (in place)
        assert [p["copied"] for p in plan] == [0, 1, 1]


def test_a_requested_intermediate_that_lives_in_a_concat_buffer(rt):
    data, forward, shape, _ = D.unet()
    x = _rand(shape, 12)
    names = [n["outputs"][0] for n in rt.model.onnx_summary(data)["nodes"] if n["op"] == "ConvTranspose"]
    on, _, _ = _run_model(rt, data, x, True, True, outputs=names)
    off, _, _ = _run_model(rt, data, x, True, False, outputs=names)
    for a, b in zip(on, off):
        gpu_checks.assert_bit_exact(a, b, "ConvTranspose output requested from inside a Concat buffer")
