"""`pytest -m gpu`: the seven epilogue variants of umma_gemm_kernel compute the same bits.  Each launch runs three times:
with the default choice, under RTEN_B200_NO_PLAIN (the plain variants give way to Fast / FastGelu) and under
RTEN_B200_NO_FAST (everything on Generic).  The variant that ran is read from the RTEN_B200_VERBOSE plan line (`epi=`),
and so are the work units: every variant runs at least one launch with more units than SMs, so the staging ring and
the barrier phases carry over from one unit to the next.  f32 outputs, i32 outputs and the *ToFloat output ranges must
be bit-identical across the three runs.  Each variant is also held bit for bit against a float32 model of its
roundings, on data whose products are exact, by tests/test_gpu_wgmma_kernels.py; the cases here stay for the agreement
of the variants on full-mantissa data and the benched shapes."""
import re

import numpy as np
import pytest

import gpu_checks as gc

pytestmark = pytest.mark.gpu

_PLAN_LINE = re.compile(r"\[umma_gemm\] [^\n]*?\bsplitk=(\d+) units=(\d+) [^\n]*?\bepi=(\w+)")
KNOBS = {"default": {}, "no_plain": {"RTEN_B200_NO_PLAIN": "1"}, "no_fast": {"RTEN_B200_NO_FAST": "1"}}
VARIANTS = ("Generic", "Fast", "FastGelu", "PlainF32", "PlainF32Gelu", "PlainI8", "PlainI8Gelu")
_ENV_KEYS = ("RTEN_B200_NO_PLAIN", "RTEN_B200_NO_FAST", "RTEN_B200_NO_WIDE") + gc.FORCE_KEYS


@pytest.fixture(scope="module")
def rt():
    import rten_b200
    from rten_b200 import _lib
    _lib.load()
    return rten_b200


def _under(env, run):
    """run() with `env` and RTEN_B200_VERBOSE set, on umma_gemm_kernel only (no wide-tile plans): its outputs and the
    (splitk, units, epi) of every GEMM launch."""
    with gc.switches(**{**dict.fromkeys(_ENV_KEYS), **env, "RTEN_B200_NO_WIDE": "1"}):
        outs, err = gc.run_verbose(run)
    plans = [(int(s), int(u), v) for s, u, v in _PLAN_LINE.findall(err)]
    return outs, plans


def _range_buf(ctx):
    return ctx.to_device(np.array([2 ** 31 - 1, -2 ** 31], np.int32))  # (min, max) before any output is folded in


def _cases(rt, oracle, ctx):
    """(name, run, variant expected per knob setting); run() returns a list of numpy arrays."""
    r = oracle.XorShiftRng(2024)
    f = lambda *s: ctx.to_device(r.uniform(s, -1, 1))
    a, b, bias, res = f(4100, 256), f(256, 512), f(512), f(4100, 512)
    cases = []

    def mm(alpha=None, act=rt.ACT_NONE, residual=None, out=None):
        return lambda: [rt.FusedMatMul(alpha, activation=act).run(ctx, a, b, bias, residual=residual, out=out).numpy()]

    cases.append(("FusedMatMul + bias + residual + Relu", mm(act=rt.ACT_RELU, residual=res), ("PlainF32", "Fast", "Generic")))
    cases.append(("FusedMatMul + bias + Gelu", mm(act=rt.ACT_GELU), ("PlainF32Gelu", "FastGelu", "Generic")))
    cases.append(("FusedMatMul alpha = 0.5 + bias + residual + Relu", mm(0.5, rt.ACT_RELU, res), ("Fast", "Fast", "Generic")))
    cases.append(("FusedMatMul alpha = 0.5 + bias + ApproxGelu", mm(0.5, rt.ACT_GELU_TANH), ("FastGelu", "FastGelu", "Generic")))
    c = f(4100, 512)
    cases.append(("Gemm(1, 0.5) + full C", lambda: [rt.Gemm(1.0, 0.5).run(ctx, a, b, c).numpy()], ("Fast", "Fast", "Generic")))
    # an output whose rows are 513 floats apart: no TMA store, so the generic epilogue stores directly
    wide = ctx.to_device(np.zeros((4100, 513), np.float32))
    view = wide.view((4100, 512), (513, 1))
    cases.append(("FusedMatMul + bias into a strided view",
                  lambda: [mm(act=rt.ACT_RELU, out=view)()[0], wide.numpy()], ("Generic", "Generic", "Generic")))
    # ResNet-50 bottleneck expansion at batch 32: 1x1 conv + bias + residual + Relu (25088 rows)
    x = ctx.to_device(r.uniform((32, 64, 28, 28), -1, 1), channels_last=True)
    w = r.uniform((256, 64, 1, 1), -1, 1) / np.float32(8.0)
    cb, cres = r.uniform((256,), -1, 1), ctx.to_device(r.uniform((32, 256, 28, 28), -1, 1), channels_last=True)
    conv = rt.Conv(1, (1, 1), (0, 0, 0, 0), (1, 1), activation=rt.ACT_RELU)
    pk = conv.prepack(ctx, 1, w)
    cases.append(("Conv 1x1 + bias + residual + Relu", lambda: [conv.run(ctx, x, w, cb, packed_w=pk, residual=cres).numpy()],
                  ("PlainF32", "Fast", "Generic")))

    # integer kind: u8 activations, i8 weights
    a8, b8 = ctx.to_device(r.u8((8200, 512))), ctx.to_device(r.i8((512, 256)))
    az, bz = ctx.to_device(r.u8((8200,))), ctx.to_device(r.i8((256,)))
    az1 = np.uint8(117)
    scale, scale_b = ctx.to_device(r.uniform((256,), 0.001, 0.01)), np.float32(0.037)
    bias8, res8 = ctx.to_device(r.uniform((256,), -1, 1)), ctx.to_device(r.uniform((8200, 256), -1, 1))
    cases.append(("MatMulInteger, vector zero points", lambda: [rt.MatMulInteger().run(ctx, a8, b8, az, bz).numpy()],
                  ("Fast", "Fast", "Generic")))

    def mmf(act, b_zero_point=None):
        def run():
            rng = _range_buf(ctx)
            y = rt.MatMulIntegerToFloat(act).run(ctx, a8, b8, az1, b_zero_point, scale, bias=bias8, residual=res8,
                                                 scale_b=scale_b, out_range=rng)
            return [y.numpy(), rng.numpy()]
        return run

    cases.append(("MatMulIntegerToFloat + scale_b + bias + residual + Relu + out_range", mmf(rt.ACT_RELU),
                  ("PlainI8", "Fast", "Generic")))
    cases.append(("MatMulIntegerToFloat + scale_b + bias + residual + Gelu + out_range", mmf(rt.ACT_GELU),
                  ("PlainI8Gelu", "FastGelu", "Generic")))
    cases.append(("MatMulIntegerToFloat, vector b_zero_point + Gelu + out_range", mmf(rt.ACT_GELU, bz),
                  ("FastGelu", "FastGelu", "Generic")))
    xq = ctx.to_device(r.u8((16, 64, 28, 28)), channels_last=True)
    wq = r.i8((128, 64, 3, 3))
    cres8 = ctx.to_device(r.uniform((16, 128, 28, 28), -1, 1), channels_last=True)
    cbias8 = r.uniform((128,), -1, 1)
    cq = rt.ConvIntegerToFloat(1, (1, 1), (1, 1, 1, 1), (1, 1), activation=rt.ACT_RELU)
    pkq = cq.prepack(ctx, 1, wq)

    def convq():
        rng = _range_buf(ctx)
        y = cq.run(ctx, xq, wq, np.uint8(121), None, np.float32(0.0042), packed_w=pkq, bias=cbias8, residual=cres8,
                   scale_b=np.float32(0.0371), out_range=rng)
        return [y.numpy(), rng.numpy()]

    cases.append(("ConvIntegerToFloat 3x3 + scale_b + bias + residual + Relu + out_range", convq,
                  ("PlainI8", "Fast", "Generic")))
    return cases


def test_epilogue_variants_agree(rt, oracle):
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    ctx = gc.new_ctx(rt, tf32=True)
    persistent = set()  # variants seen on a launch with more work units than SMs
    for name, run, expect in _cases(rt, oracle, ctx):
        ref = None
        for (knob, env), want in zip(KNOBS.items(), expect):
            outs, plans = _under(env, run)
            assert plans, f"{name} ({knob}): no GEMM launch line was printed"
            assert all(v == want for _, _, v in plans), f"{name} ({knob}): ran {plans}, expected epi={want}"
            persistent.update(v for _, u, v in plans if u > sms)
            for o in outs:
                assert o.dtype != np.float32 or np.isfinite(o).all(), f"{name} ({knob}): non-finite output"
            if ref is None:
                ref = outs
            else:
                for i, (o, o0) in enumerate(zip(outs, ref)):
                    gc.assert_bit_exact(o, o0, f"{name}: output {i} under {knob} vs {expect[0]}")
        print(f"  {name}: {' / '.join(expect)} bit-identical; units {[u for _, u, _ in plans]} on {sms} SMs")
    missing = [v for v in VARIANTS if v not in persistent]
    assert not missing, f"variants never run on more work units than SMs: {missing}"


def test_epilogue_variants_splitk(rt, oracle):
    """Forced split-K (two CTAs per tile, the last to arrive sums in split order and runs the epilogue): the same bits
    from PlainF32, Fast and Generic, and from Fast and Generic for the integer kind (PlainI8 takes no split-K)."""
    ctx = gc.new_ctx(rt, tf32=True)
    r = oracle.XorShiftRng(77)
    a, b = ctx.to_device(r.uniform((256, 4096), -1, 1)), ctx.to_device(r.uniform((4096, 256), -1, 1))
    bias, res = ctx.to_device(r.uniform((256,), -1, 1)), ctx.to_device(r.uniform((256, 256), -1, 1))
    a8, b8 = ctx.to_device(r.u8((256, 4096))), ctx.to_device(r.i8((4096, 256)))
    scale = ctx.to_device(r.uniform((256,), 0.0001, 0.001))

    def mmf():
        rng = _range_buf(ctx)
        y = rt.MatMulIntegerToFloat(rt.ACT_RELU).run(ctx, a8, b8, np.uint8(3), None, scale, bias=bias, residual=res,
                                                     out_range=rng)
        return [y.numpy(), rng.numpy()]

    cases = [("FusedMatMul + bias + residual + Relu",
              lambda: [rt.FusedMatMul(None, activation=rt.ACT_RELU).run(ctx, a, b, bias, residual=res).numpy()],
              ("PlainF32", "Fast", "Generic")),
             ("MatMulIntegerToFloat + bias + residual + Relu + out_range", mmf, ("Fast", "Fast", "Generic"))]
    split = {"RTEN_B200_FORCE_SPLITK": "2", "RTEN_B200_FORCE_STRICT": "1"}
    for name, run, expect in cases:
        ref = None
        for (knob, env), want in zip(KNOBS.items(), expect):
            outs, plans = _under({**env, **split}, run)
            assert plans and all(s == 2 and v == want for s, _, v in plans), \
                f"{name} ({knob}): ran {plans}, expected split-K 2 with epi={want}"
            if ref is None:
                ref = outs
            else:
                for i, (o, o0) in enumerate(zip(outs, ref)):
                    gc.assert_bit_exact(o, o0, f"{name} split-K: output {i} under {knob} vs {expect[0]}")
