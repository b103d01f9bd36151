"""`pytest -m gpu`: the wide-tile GEMM / conv kernel (umma_wide_kernel: 128 x 128 and 128 x 256 tiles for launches with
the plain f32 epilogue).  Each case is forced onto a wide plan and onto a 64-column plan of umma_gemm_kernel: the wide
result must meet the TF32 (or 3xTF32) bound against float64, the wide kernel must have run (forced-plan counter, and
CUPTI kernel records where the session has them), and both plans must agree bit for bit (same K order, same epilogue
roundings).  The persistent-schedule cases launch more work units than the device has SMs, so every CTA carries its
pipeline state from one unit to the next.  Both wide instances and the chained ones are also held bit for bit against
an exact product, with CUPTI required to show them, by tests/test_gpu_wgmma_kernels.py; the cases here stay for the
agreement of wide and narrow plans on full-mantissa data and the benched shapes."""
import re

import numpy as np
import pytest

import gpu_checks as gc
from gpu_checks import bound, forced

pytestmark = pytest.mark.gpu

# the plan line launch_plan prints under RTEN_B200_VERBOSE
_PLAN_LINE = re.compile(r"\[umma_gemm\] [^\n]*?\bbn=(\d+) [^\n]*?\bunits=(\d+) ")


@pytest.fixture(scope="module")
def rt():
    import rten_b200
    from rten_b200 import _lib
    _lib.load()
    return rten_b200


def _with_plan_lines(fn):
    """`fn()` with RTEN_B200_VERBOSE=1, and the (bn, units) of every GEMM launch it printed to stderr."""
    out, err = gc.run_verbose(fn)
    return out, [(int(b), int(u)) for b, u in _PLAN_LINE.findall(err)]


def _wide_vs_narrow(ctx, run, bn, what, seen, log=False, repeats=1):
    """Output of `run` on a forced wide plan and its largest difference from the forced 64-column plan.  Under
    FORCE_STRICT a forced-plan hit means a bn > 64 plan was launched, and only umma_wide_kernel runs those.  CUPTI must
    agree: no umma_gemm_kernel in the session, and umma_wide_kernel among its umma_ records.  (Inside the whole GPU
    suite a session can miss the records of kernels launched with launch attributes while keeping others; `seen`
    counts the sessions that did record the wide kernel.)  With `log` the (bn, units) of the wide launches are
    returned too.  `repeats` > 1 runs the wide plan that many times in all, and every run must give the same bits."""
    plans = None
    with forced(bn):
        hit0, _ = ctx.forced_plan_counts()
        if log:
            (wide, names), plans = _with_plan_lines(lambda: gc._kernels_launched(run))
        else:
            wide, names = gc._kernels_launched(run)
        hit1, _ = ctx.forced_plan_counts()
        again = [run() for _ in range(repeats - 1)]
    assert hit1 > hit0, f"{what}: the forced bn={bn} plan was not taken"
    umma = [n for n in names if "umma_" in n]
    assert not any("umma_gemm_kernel" in n for n in umma), f"{what}: the 64-column kernel ran ({umma})"
    if umma:
        assert any("umma_wide_kernel" in n for n in umma), f"{what}: umma_wide_kernel did not run ({umma})"
        seen.append(what)
    for i, out in enumerate(again):
        gc.assert_bit_exact(out, wide, f"{what}: wide (bn={bn}) run {i + 2} vs run 1")
    with forced(64):
        narrow = run()
    diff = float(np.abs(wide.astype(np.float64) - narrow).max())
    gc.assert_bit_exact(wide, narrow, f"{what}: wide (bn={bn}) vs 64-column plan")
    return wide, diff, plans


def _case(ctx, run, bn, what, exact, absum, seen, log=False, repeats=1, extra_abs=0.0):
    got, diff, plans = _wide_vs_narrow(ctx, run, bn, what, seen, log, repeats)
    worst = gc.assert_tf32_close(got, exact, absum, what, extra_abs=extra_abs)
    return dict(what=what, diff=diff, worst=worst, plans=plans)


def _exact_product(a, b):
    """float64 a @ b and |a| @ |b| (numpy broadcasting), computed on the GPU."""
    import torch
    ta = torch.from_numpy(np.ascontiguousarray(a)).to("cuda", torch.float64)
    tb = torch.from_numpy(np.ascontiguousarray(b)).to("cuda", torch.float64)
    return torch.matmul(ta, tb).cpu().numpy(), torch.matmul(ta.abs(), tb.abs()).cpu().numpy()


def _matmul(rt, oracle, ctx, bn, ashape, bshape, seed, seen, residual=False, in_place=False, a_pad=0, **kw):
    """FusedMatMul + bias [+ residual].  `in_place`: the residual tensor is also the output.  `a_pad`: A's matrices
    sit `a_pad` rows apart in a larger buffer, so the batch does not flatten into one matrix."""
    r = oracle.XorShiftRng(seed)
    a, b, bias = r.uniform(ashape), r.uniform(bshape), r.uniform((bshape[-1],))
    exact, absum = _exact_product(a, b)
    exact = exact + bias
    if a_pad:
        store = np.zeros(ashape[:-2] + (ashape[-2] + a_pad, ashape[-1]), np.float32)
        store[..., :ashape[-2], :] = a
        ds = ctx.to_device(store)
        da = ds.view(ashape, ds.strides)
    else:
        da = ctx.to_device(a)
    db, dbias = ctx.to_device(b), ctx.to_device(bias)
    what = f"FusedMatMul {ashape}x{bshape} + bias"
    if a_pad:
        what += f" (A rows {a_pad} apart between batches)"
    if not residual:
        run = lambda: rt.FusedMatMul(None).run(ctx, da, db, dbias).numpy()
    else:
        res = r.uniform(exact.shape)
        exact = exact + res
        dres = ctx.to_device(res)
        what += " + residual" + (", in place" if in_place else "")

        def run():
            if in_place:
                dres.copy_from(res)
            out = rt.FusedMatMul(None).run(ctx, da, db, dbias, residual=dres, out=dres if in_place else None)
            assert not in_place or out is dres
            return out.numpy()
    return _case(ctx, run, bn, what, exact, absum, seen, **kw)


def _gemm_c(rt, oracle, ctx, bn, m, k, n, seed, seen, **kw):
    """Gemm(alpha = 1, beta = 1) with a full [M, N] C: the wide kernel stages C through its residual map."""
    r = oracle.XorShiftRng(seed)
    a, b, c = r.uniform((m, k)), r.uniform((k, n)), r.uniform((m, n))
    exact, absum = _exact_product(a, b)
    da, db, dc = ctx.to_device(a), ctx.to_device(b), ctx.to_device(c)
    what = f"Gemm(1, 1) {m}x{k}x{n} + full C"
    return _case(ctx, lambda: rt.Gemm(1.0, 1.0).run(ctx, da, db, dc).numpy(), bn, what, exact + c, absum, seen, **kw)


def _conv(rt, oracle, ctx, bn, xs, ws, pads, strides, residual, seed, seen, bias=True, **kw):
    r = oracle.XorShiftRng(seed)
    x = r.uniform(xs)
    w = r.uniform(ws, -1, 1) / np.float32(np.sqrt(ws[1] * ws[2] * ws[3]))
    b = r.uniform((ws[0],)) if bias else None
    op = rt.Conv(1, (1, 1), pads, strides, activation=1)
    xd = ctx.to_device(x, channels_last=True)
    pk = op.prepack(ctx, 1, w)
    exact, absum = gc._conv_exact(x, w, b, pads, 1, strides, (1, 1), device="cuda")
    kwargs = {"packed_w": pk}
    if residual:
        res = r.uniform(exact.shape)
        kwargs["residual"] = ctx.to_device(res, channels_last=True)
        exact = exact + res
    what = f"Conv{'' if bias else ' (no bias)'} + Relu x{xs} w{ws} pads={pads} s={strides} residual={residual}"
    return _case(ctx, lambda: op.run(ctx, xd, w, b, **kwargs).numpy(), bn, what, np.maximum(exact, 0), absum, seen, **kw)


def _gelu(rt, oracle, ctx, bn, seed, seen, approx=False):
    from scipy.special import erf
    r = oracle.XorShiftRng(seed)
    a, b, bias = r.uniform((256, 384), -1, 1), r.uniform((384, 384), -1, 1), r.uniform((384,), -1, 1)
    da, db, dbias = ctx.to_device(a), ctx.to_device(b), ctx.to_device(bias)
    act = rt.ACT_GELU_TANH if approx else rt.ACT_GELU
    what = f"FusedMatMul 256x384x384 + bias + {'ApproxGelu' if approx else 'Gelu'}"
    x, absum = _exact_product(a, b)
    x = x + bias
    if approx:
        exact = 0.5 * x * (1.0 + np.tanh(np.sqrt(2.0 / np.pi) * (x + 0.044715 * x ** 3)))
    else:
        exact = 0.5 * x * (1.0 + erf(x / np.sqrt(2.0)))
    # both Gelu forms have slopes below 1.13: the product's bound carries over, plus the f32 evaluation of Gelu itself
    return _case(ctx, lambda: rt.FusedMatMul(None, activation=act).run(ctx, da, db, dbias).numpy(), bn, what, exact,
                 1.13 * absum, seen, extra_abs=1e-6 * float(np.abs(exact).max()))


def _summary(title, rows, seen):
    print(f"{title}: {len(rows)} cases, largest |wide - 64-column plan| = {max(r['diff'] for r in rows)}, worst error / "
          f"bound = {max(r['worst'] for r in rows):.3f}; CUPTI showed umma_wide_kernel in {len(seen)} of them")


@pytest.mark.parametrize("tf32", [True, False], ids=["tf32", "tf32x3"])
@pytest.mark.parametrize("bn", [128, 256])
def test_wide_tiles(rt, oracle, bn, tf32):
    ctx = gc.new_ctx(rt, tf32=tf32)
    rows, seen = [], []
    with bound(tf32):
        # ragged M, batched z dims with a broadcast B, and N that the last tile overhangs by whole 32-column chunks
        n_over = 160 if bn == 128 else 288
        rows.append(_matmul(rt, oracle, ctx, bn, (130, 256), (256, n_over), seed=1, seen=seen))
        rows.append(_matmul(rt, oracle, ctx, bn, (2, 3, 200, 96), (96, 2 * bn), seed=2, seen=seen))
        rows.append(_matmul(rt, oracle, ctx, bn, (2, 130, 64), (2, 64, n_over), seed=3, seen=seen))
        # one 128-row tile that is mostly (M = 40, above the skinny path's 32) or half (M = 64: the second warpgroup's
        # rows are all outside) empty
        rows.append(_matmul(rt, oracle, ctx, bn, (40, 256), (256, 2 * bn), seed=8, seen=seen))
        rows.append(_matmul(rt, oracle, ctx, bn, (64, 256), (256, 2 * bn), seed=9, seen=seen))
        # MatMul + residual (BERT's output projections), one work unit
        rows.append(_matmul(rt, oracle, ctx, bn, (128, 192), (192, bn), seed=10, seen=seen, residual=True))
        # ResNet-50 bottleneck expansion: 1x1 conv + residual + Relu; a stride-2 3x3 conv
        rows.append(_conv(rt, oracle, ctx, bn, (4, 512, 14, 14), (1024, 512, 1, 1), (0, 0, 0, 0), (1, 1), True, seed=4, seen=seen))
        rows.append(_conv(rt, oracle, ctx, bn, (4, 128, 28, 28), (256, 128, 3, 3), (1, 1, 1, 1), (2, 2), False, seed=5, seen=seen))
        if bn == 128:
            rows.append(_gelu(rt, oracle, ctx, bn, seed=6, seen=seen))
            rows.append(_gelu(rt, oracle, ctx, bn, seed=7, seen=seen, approx=True))
    _summary(f"bn={bn} {'tf32' if tf32 else 'tf32x3'}", rows, seen)


@pytest.mark.parametrize("tf32", [True, False], ids=["tf32", "tf32x3"])
@pytest.mark.parametrize("bn", [128, 256])
def test_wide_tiles_persistent(rt, oracle, bn, tf32):
    """Persistent schedules: every launch has more work units than the device has SMs, so CTAs run several units in
    turn and carry the operand ring's stage and phases, the staging-buffer parity, the residual barrier phases, the
    residual prefetch of the next unit and the shared bias vector from one unit to the next.  The unit counts are read
    from the launches themselves (RTEN_B200_VERBOSE), not inferred from the shapes."""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    ctx = gc.new_ctx(rt, tf32=tf32)
    rows, seen = [], []
    kw = dict(seen=seen, log=True)
    with bound(tf32):
        # ragged last M tile; 17 K blocks, which neither ring size (4 or 6 stages) divides, so every unit starts at a
        # different stage and phase; three runs that must agree bit for bit
        rows.append(_matmul(rt, oracle, ctx, bn, (4100, 544), (544, 2048), seed=11, residual=True, repeats=3, **kw))
        # K ends inside the last 32-element block: the TMA zero-fills its tail (K % 4 == 0 keeps A addressable)
        rows.append(_matmul(rt, oracle, ctx, bn, (4100, 532), (532, 2048), seed=12, residual=True, **kw))
        # 16 batch entries in the launch's z coordinate (A's matrices are not uniformly strided), B broadcast
        rows.append(_matmul(rt, oracle, ctx, bn, (16, 520, 256), (256, 512), seed=13, a_pad=8, **kw))
        # Gemm's C as the residual
        rows.append(_gemm_c(rt, oracle, ctx, bn, 4100, 512, 2048, seed=14, **kw))
        # ResNet-50 layer-1 expansion at batch 32 (784 M tiles of 8 x 8 x 2 pixels); three runs that must agree
        rows.append(_conv(rt, oracle, ctx, bn, (32, 64, 56, 56), (256, 64, 1, 1), (0, 0, 0, 0), (1, 1), True, seed=15,
                          repeats=3, **kw))
        # odd batch: the last box of images runs past the 65th; no bias, so the bias vector is all zeros
        rows.append(_conv(rt, oracle, ctx, bn, (65, 64, 28, 28), (512, 64, 3, 3), (1, 1, 1, 1), (2, 2), False, seed=16,
                          bias=False, **kw))
        # the output overwrites the residual: each residual chunk is read before the chunk is stored
        rows.append(_matmul(rt, oracle, ctx, bn, (4100, 544), (544, 2048), seed=17, residual=True, in_place=True, **kw))
    for row in rows:
        assert row["plans"], f"{row['what']}: no GEMM launch line was printed"
        for launched_bn, units in row["plans"]:
            assert launched_bn == bn, f"{row['what']}: launched bn={launched_bn}, forced {bn}"
            assert units > sms, f"{row['what']}: {units} work units on {sms} SMs: no CTA runs a second unit"
        print(f"  {row['what']}: units {[u for _, u in row['plans']]} on {sms} SMs, |wide - 64-column| = {row['diff']}, "
              f"error / bound = {row['worst']:.3f}")
    most = max(u for row in rows for _, u in row["plans"])
    assert most >= 2 * sms, f"bn={bn}: no case launches 2x as many units as SMs (most: {most})"
    _summary(f"persistent bn={bn} {'tf32' if tf32 else 'tf32x3'}", rows, seen)


def test_wide_gelu_epilogue(rt, oracle):
    """The wide kernel's Gelu epilogue (erf and tanh forms) must be BIT-IDENTICAL to the Gelu operator applied to the
    same product: FusedMatMul(bias, Gelu) vs FusedMatMul(bias) -> Gelu, both on a forced 128-column plan (same
    accumulation order), over more work units than SMs, with rows of zeros, zero biases and amplitudes of 1, 6 and 40."""
    ctx = gc.new_ctx(rt, tf32=True)
    r = oracle.XorShiftRng(2718)
    n = 0
    for (m, k, nn), amp in [((2200, 64, 1024), 1.0), ((2200, 128, 1024), 6.0), ((2200, 32, 1024), 40.0)]:
        a = (r.uniform((m, k), -1, 1) * amp).astype(np.float32)
        a[:4] = 0.0  # rows of exact zeros: Gelu(bias) alone
        b = r.uniform((k, nn), -1, 1)
        bias = r.uniform((nn,), -1, 1)
        bias[:3] = 0.0
        da, db, dbias = ctx.to_device(a), ctx.to_device(b), ctx.to_device(bias)
        for act, approx in ((rt.ACT_GELU, False), (rt.ACT_GELU_TANH, True)):
            what = f"wide Gelu epilogue (approximate={approx}) {m}x{k}x{nn} amp {amp}"
            with forced(128):
                hit0, _ = ctx.forced_plan_counts()
                fused = rt.FusedMatMul(None, activation=act).run(ctx, da, db, dbias).numpy()
                plain = rt.FusedMatMul(None).run(ctx, da, db, dbias)
                hit1, _ = ctx.forced_plan_counts()
            assert hit1 == hit0 + 2, f"{what}: the forced bn=128 plan was not taken"
            two = rt.Gelu(approximate=approx).run(ctx, plain).numpy()
            gc.assert_bit_exact(fused, two, what)
            n += 1
    print(f"{n} fused-vs-operator comparisons bit-identical on 128-column tiles")


def test_wide_tiles_refused(rt, oracle):
    """Launches outside the wide kernel's epilogue (alpha != 1; erf or tanh Gelu at 256 columns; Gemm's C scaled by
    beta != 1, or broadcast so that it has no residual map) never take a forced wide plan: they fall back to a valid
    plan and count a miss, or fail under FORCE_STRICT."""
    ctx = gc.new_ctx(rt)
    r = oracle.XorShiftRng(7)
    a, b, bias = r.uniform((256, 128)), r.uniform((128, 256)), r.uniform((256,))
    c_full, c_row = r.uniform((256, 256)), r.uniform((256,))
    cases = [(128, lambda: rt.FusedMatMul(0.5).run(ctx, a, b, bias).numpy(), "alpha = 0.5"),
             (256, lambda: rt.FusedMatMul(None, activation=rt.ACT_GELU).run(ctx, a, b, bias).numpy(), "Gelu"),
             (256, lambda: rt.FusedMatMul(None, activation=rt.ACT_GELU_TANH).run(ctx, a, b, bias).numpy(), "ApproxGelu"),
             (128, lambda: rt.Gemm(1.0, 0.5).run(ctx, a, b, c_full).numpy(), "Gemm beta = 0.5, full C"),
             (128, lambda: rt.Gemm(1.0, 1.0).run(ctx, a, b, c_row).numpy(), "Gemm broadcast (N,) C")]
    for bn, run, what in cases:
        with forced(bn, strict=False):
            _, miss0 = ctx.forced_plan_counts()
            out, names = gc._kernels_launched(run)
            _, miss1 = ctx.forced_plan_counts()
        assert miss1 == miss0 + 1, f"{what}: forced bn={bn} should have recorded a miss ({miss0} -> {miss1})"
        assert not any("umma_wide_kernel" in n for n in names), f"{what}: took a wide plan"
        assert np.isfinite(out).all()
        with forced(bn, strict=True):
            with pytest.raises(rt.OpError):
                run()
