"""`pytest -m gpu`: the halo-reuse kernel's 256-slot units (T = 2: two consumer warpgroups of 128 slots each), pinned
through a plans file per tile width bn, on geometries the ResNet-50 layers and the 128-slot cases of
test_gpu_plan_space.py do not reach.  For each accepted shape: the [umma_halo] line names it, the result is within the
float64 TF32 bound, bit-identical to the 128-slot plan `-1 32 1` of the same problem, or to its first 256-slot plan where
no 128-slot unit holds a row (every halo shape accumulates in one order), and two CUDA-graph replays into a NaN-poisoned output give the eager run's bits.  A shape the geometry cannot take
(a patch that no longer fits in shared memory, bn not dividing N) must be rejected and the launch re-planned."""
import pytest

import gpu_checks as gc
import test_gpu_plan_space as ps

pytestmark = pytest.mark.gpu

# (test id, ConvF32 arguments, whether a 128-slot unit exists (a row of P <= 128 slots), {bn: (R, tb) the [umma_halo]
# line must show at T = 2, or None: the entry is rejected})
WIDE_CASES = [
    # 7x7 maps: P = 9, tb = 1 + (256 - 63) / 81 = 3 images per unit, 7 images -> a last unit of one
    ("7x7-maps-tb3", dict(xs=(7, 64, 7, 7), ws=(128, 64, 3, 3), pad=1, seed=61), True, {32: (7, 3), 64: (7, 3), 128: (7, 3)}),
    # 28x28: P = 30, strips of 256 / 30 = 8 rows, the last one 4 rows
    ("28x28-strips", dict(xs=(2, 32, 28, 28), ws=(128, 32, 3, 3), pad=1, seed=62), True, {32: (8, 1), 64: (8, 1), 128: (8, 1)}),
    # P = 160: one row per unit fits 256 slots but not 128; at bn = 128 three weight stages no longer fit beside the
    # two patches (2 x 73 KB)
    ("p160", dict(xs=(1, 32, 5, 158), ws=(128, 32, 3, 3), pad=1, seed=63), False, {32: (1, 1), 64: (1, 1), 128: None}),
    # P = 256: the two patches of one row alone exceed shared memory
    ("p256", dict(xs=(1, 32, 4, 254), ws=(64, 32, 3, 3), pad=1, seed=64), False, {32: None, 64: None}),
    ("5x5-window", dict(xs=(3, 32, 12, 12), ws=(64, 32, 5, 5), pad=2, seed=65), True, {32: (12, 1), 64: (12, 1)}),
    ("4x8-window", dict(xs=(2, 32, 12, 20), ws=(64, 32, 4, 8), pad=0, seed=66), True, {32: (9, 1), 64: (9, 1)}),
    # N = 192: a multiple of 64, not of 128
    ("n192", dict(xs=(2, 64, 14, 14), ws=(192, 64, 3, 3), pad=1, seed=67), True, {32: (14, 1), 64: (14, 1), 128: None}),
]


@pytest.fixture(scope="module")
def rt():
    import rten_b200
    from rten_b200 import _lib
    _lib.load()
    return rten_b200


@pytest.fixture(autouse=True)
def _clean_env():
    with gc.switches(**dict.fromkeys(ps._ENV)):
        yield


@pytest.mark.parametrize("name,kw,t1,want", WIDE_CASES, ids=[c[0] for c in WIDE_CASES])
def test_halo_256_slot_units(rt, tmp_path, name, kw, t1, want):
    import torch
    prob = ps.ConvF32(f"halo-wide {name}", True, **kw)
    _, key = ps._candidates(rt, prob, tmp_path)
    ctx = gc.new_ctx(rt, tf32=True)
    run = prob.build(rt, ctx)
    exact, absum = prob.exact()
    # the bits every halo shape must give: the 128-slot plan's where the geometry has one, else the first 256-slot plan's
    ref, worst = None, 0.0
    outs, err = ps._pin(ctx, run, prob, key, (-1, 32, 1), tmp_path)
    if t1:
        assert ps._ran(err, (-1, 32, 1), prob.name)[1] == 1
        ref = (outs[0], "-1 32 1")
    else:
        assert ps._STALE in err and not ps._HALO.search(err), \
            f"{prob.name}: no 128-slot unit holds a row of this map, yet `-1 32 1` ran: {err.strip()}"
    ran = []
    for bn, shape in want.items():
        plan = (-1, bn, 2)
        outs, err = ps._pin(ctx, run, prob, key, plan, tmp_path)
        if shape is None:
            assert ps._STALE in err and len(ps._GEMM.findall(err)) == 1 and not ps._HALO.search(err), \
                f"{prob.name}: `-1 {bn} 2` cannot fit this geometry and must be re-planned; printed: {err.strip()}"
            continue
        _, T, R, tb, P = ps._ran(err, plan, prob.name)
        assert T == 2 and (R, tb) == shape, f"{prob.name}: bn={bn} ran T={T} R={R} tb={tb}, expected T=2 and {shape}"
        with gc.bound(True):
            worst = max(worst, gc.assert_tf32_close(outs[0], exact, absum, f"{prob.name}: {plan}"))
        if ref is None:
            ref = (outs[0], f"-1 {bn} 2")
        gc.assert_bit_exact(outs[0], ref[0], f"{prob.name}: {plan} vs {ref[1]}")
        # two graph replays of the pinned plan into a NaN-poisoned output
        ctx.graph_begin()
        run()
        g = ctx.graph_end()
        for i in range(2):
            prob.poison()
            torch.cuda.synchronize()
            g.launch()
            ctx.sync()
            gc.assert_bit_exact(ps._np(prob.out), outs[0], f"{prob.name}: {plan}, graph replay {i}")
        del g
        ran.append(f"bn={bn} R={R} tb={tb} P={P}")
    del run
    ctx.close()
    print(f"\n  {prob.name}: T=2 {ran}; worst err/bound {worst:.3f}")
