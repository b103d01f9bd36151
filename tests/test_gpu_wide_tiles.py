"""`pytest -m gpu`: the wide-tile GEMM / conv kernel (umma_wide_kernel: 128 x 128 and 128 x 256 tiles for launches with
the plain f32 epilogue).  Each case is forced onto a wide plan and onto a 64-column plan of umma_gemm_kernel: the wide
result must meet the TF32 (or 3xTF32) bound against float64, the wide kernel must have run (forced-plan counter, and
CUPTI kernel records where the session has them), and both plans must agree bit for bit (same K order, same epilogue
roundings)."""
import contextlib
import os

import numpy as np
import pytest

import gpu_checks as gc

pytestmark = pytest.mark.gpu

KEYS = ("RTEN_B200_FORCE_BN", "RTEN_B200_FORCE_SPLITK", "RTEN_B200_FORCE_STRICT")


@pytest.fixture(scope="module")
def rt():
    import rten_b200
    from rten_b200 import _lib
    _lib.load()
    return rten_b200


@contextlib.contextmanager
def forced(bn, strict=True):
    for k in KEYS:
        os.environ.pop(k, None)
    os.environ["RTEN_B200_FORCE_BN"] = str(bn)
    os.environ["RTEN_B200_FORCE_SPLITK"] = "1"
    if strict:
        os.environ["RTEN_B200_FORCE_STRICT"] = "1"
    try:
        yield
    finally:
        for k in KEYS:
            os.environ.pop(k, None)


@contextlib.contextmanager
def bound(tf32):
    saved = gc.TF32_REL
    gc.TF32_REL = 2.0 ** -9 if tf32 else 2.0 ** -18
    try:
        yield
    finally:
        gc.TF32_REL = saved


def _wide_vs_narrow(ctx, run, bn, what, seen):
    """Output of `run` on a forced wide plan and its largest difference from the forced 64-column plan.  Under
    FORCE_STRICT a forced-plan hit means a bn > 64 plan was launched, and only umma_wide_kernel runs those.  CUPTI must
    agree: no umma_gemm_kernel in the session, and umma_wide_kernel among its umma_ records.  (Inside the whole GPU
    suite a session can miss the records of kernels launched with launch attributes while keeping others; `seen`
    counts the sessions that did record the wide kernel.)"""
    with forced(bn):
        hit0, _ = ctx.forced_plan_counts()
        wide, names = gc._kernels_launched(run)
        hit1, _ = ctx.forced_plan_counts()
    assert hit1 > hit0, f"{what}: the forced bn={bn} plan was not taken"
    umma = [n for n in names if "umma_" in n]
    assert not any("umma_gemm_kernel" in n for n in umma), f"{what}: the 64-column kernel ran ({umma})"
    if umma:
        assert any("umma_wide_kernel" in n for n in umma), f"{what}: umma_wide_kernel did not run ({umma})"
        seen.append(what)
    with forced(64):
        narrow = run()
    diff = float(np.abs(wide.astype(np.float64) - narrow).max())
    gc.assert_bit_exact(wide, narrow, f"{what}: wide (bn={bn}) vs 64-column plan")
    return wide, diff


def _matmul(rt, oracle, ctx, bn, ashape, bshape, seed, seen):
    r = oracle.XorShiftRng(seed)
    a, b, bias = r.uniform(ashape), r.uniform(bshape), r.uniform((bshape[-1],))
    da, db, dbias = ctx.to_device(a), ctx.to_device(b), ctx.to_device(bias)
    what = f"FusedMatMul {ashape}x{bshape} + bias"
    got, diff = _wide_vs_narrow(ctx, lambda: rt.FusedMatMul(None).run(ctx, da, db, dbias).numpy(), bn, what, seen)
    exact = np.matmul(a.astype(np.float64), b.astype(np.float64)) + bias
    absum = np.matmul(np.abs(a).astype(np.float64), np.abs(b).astype(np.float64))
    gc.assert_tf32_close(got, exact, absum, what)
    return diff


def _conv(rt, oracle, ctx, bn, xs, ws, pads, strides, residual, seed, seen):
    r = oracle.XorShiftRng(seed)
    x = r.uniform(xs)
    w = r.uniform(ws, -1, 1) / np.float32(np.sqrt(ws[1] * ws[2] * ws[3]))
    b = r.uniform((ws[0],))
    op = rt.Conv(1, (1, 1), pads, strides, activation=1)
    xd = ctx.to_device(x, channels_last=True)
    pk = op.prepack(ctx, 1, w)
    exact, absum = gc._conv_exact(x, w, b, pads, 1, strides, (1, 1))
    kw = {"packed_w": pk}
    if residual:
        res = r.uniform(exact.shape)
        kw["residual"] = ctx.to_device(res, channels_last=True)
        exact = exact + res
    what = f"Conv + Relu x{xs} w{ws} pads={pads} s={strides} residual={residual}"
    got, diff = _wide_vs_narrow(ctx, lambda: op.run(ctx, xd, w, b, **kw).numpy(), bn, what, seen)
    gc.assert_tf32_close(got, np.maximum(exact, 0), absum, what)
    return diff


def _gelu(rt, oracle, ctx, bn, seed, seen):
    from scipy.special import erf
    r = oracle.XorShiftRng(seed)
    a, b, bias = r.uniform((256, 384), -1, 1), r.uniform((384, 384), -1, 1), r.uniform((384,), -1, 1)
    da, db, dbias = ctx.to_device(a), ctx.to_device(b), ctx.to_device(bias)
    what = "FusedMatMul 256x384x384 + bias + Gelu"
    got, diff = _wide_vs_narrow(ctx, lambda: rt.FusedMatMul(None, activation=rt.ACT_GELU).run(ctx, da, db, dbias).numpy(), bn, what, seen)
    x = np.matmul(a.astype(np.float64), b.astype(np.float64)) + bias
    exact = 0.5 * x * (1.0 + erf(x / np.sqrt(2.0)))
    absum = np.matmul(np.abs(a).astype(np.float64), np.abs(b).astype(np.float64))
    # Gelu's slope is below 1.13: the product's bound carries over, plus the f32 evaluation of Gelu itself
    gc.assert_tf32_close(got, exact, 1.13 * absum, what, extra_abs=1e-6 * float(np.abs(exact).max()))
    return diff


@pytest.mark.parametrize("tf32", [True, False], ids=["tf32", "tf32x3"])
@pytest.mark.parametrize("bn", [128, 256])
def test_wide_tiles(rt, oracle, bn, tf32):
    ctx = gc.new_ctx(rt, tf32=tf32)
    diffs, seen = [], []
    with bound(tf32):
        # ragged M, batched z dims with a broadcast B, and N that the last tile overhangs by whole 32-column chunks
        n_over = 160 if bn == 128 else 288
        diffs.append(_matmul(rt, oracle, ctx, bn, (130, 256), (256, n_over), seed=1, seen=seen))
        diffs.append(_matmul(rt, oracle, ctx, bn, (2, 3, 200, 96), (96, 2 * bn), seed=2, seen=seen))
        diffs.append(_matmul(rt, oracle, ctx, bn, (2, 130, 64), (2, 64, n_over), seed=3, seen=seen))
        # ResNet-50 bottleneck expansion: 1x1 conv + residual + Relu; a stride-2 3x3 conv
        diffs.append(_conv(rt, oracle, ctx, bn, (4, 512, 14, 14), (1024, 512, 1, 1), (0, 0, 0, 0), (1, 1), True, seed=4, seen=seen))
        diffs.append(_conv(rt, oracle, ctx, bn, (4, 128, 28, 28), (256, 128, 3, 3), (1, 1, 1, 1), (2, 2), False, seed=5, seen=seen))
        if bn == 128:
            diffs.append(_gelu(rt, oracle, ctx, bn, seed=6, seen=seen))
    print(f"bn={bn} {'tf32' if tf32 else 'tf32x3'}: {len(diffs)} cases, largest |wide - 64-column plan| = {max(diffs)}; "
          f"CUPTI showed umma_wide_kernel in {len(seen)} of them")


def test_wide_tiles_refused(rt, oracle):
    """Launches outside the wide kernel's epilogue (alpha != 1; Gelu at 256 columns) never take a forced wide plan: they
    fall back to a valid plan and count a miss, or fail under FORCE_STRICT."""
    ctx = gc.new_ctx(rt)
    r = oracle.XorShiftRng(7)
    a, b, bias = r.uniform((256, 128)), r.uniform((128, 256)), r.uniform((256,))
    cases = [(128, lambda: rt.FusedMatMul(0.5).run(ctx, a, b, bias).numpy(), "alpha = 0.5"),
             (256, lambda: rt.FusedMatMul(None, activation=rt.ACT_GELU).run(ctx, a, b, bias).numpy(), "Gelu")]
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
