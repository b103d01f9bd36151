"""`pytest -m gpu`: the 8192^3 GEMMs that bench.py times (TF32 MatMul with a K-major B, MatMulInteger u8 x i8), computed
the way it computes them -- autotuned plan, then a CUDA-graph replay -- and checked against float64 products on the
GPU; and ResNet-50 b32 determinism once its launch plans are fixed.

At this size a work unit runs 256 f32 K blocks (the operand ring wraps many times) and every CTA runs about 15 units.
A dropped or repeated 32-wide K block moves a result on signed data by about sqrt(32) ~ 6, which the single-pass TF32
bound (2^-9 * sum |a b| ~ 10) cannot see; the uniform [0, 1) run (bound 0.2 % of the result against 0.4 % for one
block) and the 3xTF32 run (bound 2^-18 * sum |a b| ~ 0.02) can."""
import numpy as np
import pytest

import gpu_checks as gc
from gpu_checks import forced

pytestmark = pytest.mark.gpu

N = 8192


@pytest.fixture(scope="module")
def rt():
    import rten_b200
    from rten_b200 import _lib
    _lib.load()
    return rten_b200


def _as_benched(ctx, fn):
    """bench.py's secondary_numbers: one eager launch (autotunes the plan), then the launch captured and replayed."""
    ctx.set_autotune(True)
    fn()
    ctx.sync()
    ctx.set_autotune(False)
    ctx.graph_begin()
    fn()
    g = ctx.graph_end()
    return g


def _replay(ctx, g, out_t):
    import torch
    out_t.fill_(float("nan") if out_t.is_floating_point() else -1)
    torch.cuda.synchronize()
    g.launch()
    ctx.sync()
    return out_t.clone()


def _tf32_ratio(got, a_t, bs_t, rel):
    """Largest |got - a @ b| / (rel * |a| @ |b| + 1e-6) with b = bs_t^T, in float64 on the GPU."""
    a64, b64 = a_t.double(), bs_t.double().t()
    err = (got.double() - a64 @ b64).abs_()
    bound = (a64.abs_() @ b64.abs_()).mul_(rel).add_(1e-6)
    return float(err.div_(bound).max())


def _f32_gemm(rt, tf32, uniform, forced_bns=()):
    """MatMul 8192^3 as benched: a [M, K]; b a K-major view of [N, K] storage.  Returns the error / bound ratio of the
    replayed result and checks it bit for bit against the forced plans of `forced_bns`."""
    import torch
    gen = torch.Generator(device="cuda").manual_seed(8192 + 2 * uniform + tf32)
    draw = torch.rand if uniform else torch.randn
    a_t = draw(N, N, device="cuda", generator=gen)
    bs_t = draw(N, N, device="cuda", generator=gen)
    o_t = torch.empty(N, N, device="cuda")
    torch.cuda.synchronize()
    ctx = gc.new_ctx(rt, tf32=tf32)
    a, b, o = rt.from_torch(ctx, a_t), rt.from_torch(ctx, bs_t).permute(1, 0), rt.from_torch(ctx, o_t)
    run = lambda: rt.MatMul().run(ctx, a, b, out=o)
    g = _as_benched(ctx, run)
    got = _replay(ctx, g, o_t)
    del g
    what = f"MatMul {N}^3 {'tf32' if tf32 else 'tf32x3'} {'U[0, 1)' if uniform else 'randn'}"
    for bn in forced_bns:
        o_t.fill_(float("nan"))
        torch.cuda.synchronize()
        with forced(bn):
            hit0, _ = ctx.forced_plan_counts()
            run()
            ctx.sync()
            hit1, _ = ctx.forced_plan_counts()
        assert hit1 == hit0 + 1, f"{what}: the forced bn={bn} plan was not taken"
        same = got.view(torch.int32) == o_t.view(torch.int32)
        assert bool(same.all()), f"{what}: replayed plan vs forced bn={bn}: {int((~same).sum())} elements differ"
    ratio = _tf32_ratio(got, a_t, bs_t, 2.0 ** -9 if tf32 else 2.0 ** -18)
    assert ratio <= 1.0, f"{what}: error {ratio:.2f}x the bound"
    del ctx
    return what, ratio


def test_bench_gemm_tf32(rt):
    what, ratio = _f32_gemm(rt, tf32=True, uniform=False, forced_bns=(256, 128, 64))
    print(f"{what}: error / bound {ratio:.3f}; bit-identical to forced bn = 256, 128, 64")
    what, ratio = _f32_gemm(rt, tf32=True, uniform=True)
    print(f"{what}: error / bound {ratio:.3f}")


def test_bench_gemm_tf32x3(rt):
    what, ratio = _f32_gemm(rt, tf32=False, uniform=False)
    print(f"{what}: error / bound {ratio:.3f}")


def test_bench_gemm_int8(rt):
    """MatMulInteger u8 x i8 (K-major B view, no zero points) against a float64 product of the same integers: every
    partial sum is below 8192 * 255 * 128 < 2^53, so float64 is exact in any summation order."""
    import torch
    gen = torch.Generator(device="cuda").manual_seed(88)
    a_t = torch.randint(0, 255, (N, N), device="cuda", dtype=torch.uint8, generator=gen)
    bs_t = torch.randint(-128, 127, (N, N), device="cuda", dtype=torch.int8, generator=gen)
    o_t = torch.empty(N, N, device="cuda", dtype=torch.int32)
    torch.cuda.synchronize()
    ctx = gc.new_ctx(rt)
    a, b, o = rt.from_torch(ctx, a_t), rt.from_torch(ctx, bs_t).permute(1, 0), rt.from_torch(ctx, o_t)
    g = _as_benched(ctx, lambda: rt.MatMulInteger().run(ctx, a, b, out=o))
    got = _replay(ctx, g, o_t)
    del g
    want = (a_t.double() @ bs_t.double().t()).to(torch.int32)
    same = got == want
    assert bool(same.all()), f"MatMulInteger {N}^3: {int((~same).sum())} of {same.numel()} elements differ"
    print(f"MatMulInteger {N}^3 u8 x i8: bit-exact")
    del ctx


def test_resnet50_plans_pinned(rt, oracle, tmp_path):
    """ResNet-50 fp32 b32, TF32, with bench.py's weights and input (make_spec / make_inputs): once the launch plans are
    fixed the step is deterministic.  Two replays of one graph agree bit for bit, and a second context that loads the
    first one's plans (no autotuning) reproduces its logits bit for bit."""
    from rten_b200 import graphs
    rng = oracle.XorShiftRng(5678)
    spec = graphs.make_resnet50(lambda s: rng.uniform(s))
    x = oracle.XorShiftRng(1234).uniform((32, 3, 224, 224))
    plans = str(tmp_path / "resnet50_b32_tf32.plans")

    def replays(ctx, count):
        runner = graphs.ResNet50Runner(ctx, spec, fuse=True)
        xd = ctx.to_device(x, channels_last=True)
        runner.run(xd)  # eager pass: autotunes if enabled, warms the buffer pool
        ctx.sync()
        ctx.set_autotune(False)
        ctx.graph_begin()
        out = runner.run(xd)
        g = ctx.graph_end()
        got = []
        for _ in range(count):
            out.copy_from(np.full(out.shape, np.nan, np.float32))
            g.launch()
            ctx.sync()
            got.append(out.numpy())
        return got

    ctx1 = gc.new_ctx(rt, tf32=True)
    ctx1.set_autotune(True)
    first, second = replays(ctx1, 2)
    gc.assert_bit_exact(second, first, "ResNet-50 b32 tf32: second replay vs first")
    ctx1.save_plans(plans)
    del ctx1
    ctx2 = gc.new_ctx(rt, tf32=True)
    ctx2.load_plans(plans)
    (pinned,) = replays(ctx2, 1)
    gc.assert_bit_exact(pinned, first, "ResNet-50 b32 tf32: context with the loaded plans vs the autotuning context")
    assert np.isfinite(first).all()
    with open(plans) as f:
        n_plans = len(f.readlines())
    print(f"ResNet-50 b32 tf32: logits bit-identical across replays and across contexts sharing one plan file "
          f"({n_plans} plans)")
