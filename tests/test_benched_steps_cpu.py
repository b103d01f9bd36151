"""The references and bounds of tests/test_gpu_benched_steps.py on the CPU (benched_step_refs):

  * float32 emulations of the kernels -- TF32-truncated operands (or the 3xTF32 split), f32 accumulation block by block,
    f32 epilogue roundings -- stay inside each bound in both f32 modes, and use a visible share of it;
  * small slips land outside: one K block dropped, the bias added twice, the residual omitted for one row, one head's
    mask ignored, the V rows of two adjacent keys swapped, one channel of a chained convolution computed from the wrong
    y, a cache row written one position off;
  * the torch attention bound is test_gpu_attention_encoder.ref_and_bound, and the exact integer product gives the
    oracle's MatMulInteger / MatMulIntegerToFloat bits;
  * the recorder and the grouping of the in-place attention triple, on a stand-in operator module."""
import types

import numpy as np
import pytest
import torch

import benched_step_refs as R
import test_gpu_attention_encoder as tae
import test_gpu_benched_steps as steps

F32 = np.float32
MODES = [("tf32", True), ("tf32x3", False)]
KB = 32  # K block of the emulated accumulation


def _tf32(x):
    return (np.ascontiguousarray(x, F32).view(np.uint32) & np.uint32(0xFFFFE000)).view(F32)


def emulate_matmul(a, b, tf32, drop_block=None):
    """a [M, K] @ b [K, N] as the tensor cores compute it: TF32-truncated operands (3xTF32: lo.hi + hi.lo + hi.hi of
    the truncated splits), each K block's products summed exactly and added to an f32 accumulator."""
    a, b = np.asarray(a, F32), np.asarray(b, F32)
    if tf32:
        parts = [(_tf32(a), _tf32(b))]
    else:
        ah, bh = _tf32(a), _tf32(b)
        parts = [(_tf32(a - ah), bh), (ah, _tf32(b - bh)), (ah, bh)]
    acc = np.zeros((a.shape[0], b.shape[1]), F32)
    for i, k0 in enumerate(range(0, a.shape[1], KB)):
        if i == drop_block:
            continue
        for pa, pb in parts:
            acc = (acc + pa[:, k0:k0 + KB].astype(np.float64) @ pb[k0:k0 + KB].astype(np.float64)).astype(F32)
    return acc


def emulate_epilogue(acc, bias=None, residual=None, act=R.ACT_NONE, alpha=1.0):
    """The epilogue one f32 rounding at a time: alpha, + bias, + residual, then the activation (rounded once)."""
    y = (acc * F32(alpha)).astype(F32)
    if bias is not None:
        y = (y + bias).astype(F32)
    if residual is not None:
        y = (y + residual).astype(F32)
    if act == R.ACT_RELU:
        return np.maximum(y, F32(0))
    if act in (R.ACT_GELU, R.ACT_GELU_TANH):
        return R.gelu64(torch.from_numpy(y.astype(np.float64)), act == R.ACT_GELU_TANH).numpy().astype(F32)
    return y


def _im2col(x, k, pad, stride):
    """NCHW x -> [B * OH * OW, C * k * k] rows in OIHW weight order, and (B, OH, OW)."""
    B, C, H, W = x.shape
    xp = np.pad(x, ((0, 0), (0, 0), (pad, pad), (pad, pad)))
    win = np.lib.stride_tricks.sliding_window_view(xp, (k, k), axis=(2, 3))[:, :, ::stride, ::stride]
    OH, OW = win.shape[2], win.shape[3]
    return np.ascontiguousarray(win.transpose(0, 2, 3, 1, 4, 5)).reshape(B * OH * OW, C * k * k), (B, OH, OW)


def emulate_conv(x, w, pad, stride, tf32, drop_block=None):
    """The convolution as the implicit GEMM it is, through emulate_matmul: NCHW f32, no bias."""
    cols, (B, OH, OW) = _im2col(x, w.shape[2], pad, stride)
    acc = emulate_matmul(cols, w.reshape(w.shape[0], -1).T, tf32, drop_block)
    return acc.reshape(B, OH, OW, -1).transpose(0, 3, 1, 2)


def _d(a):
    return torch.from_numpy(np.asarray(a, np.float64))


def _ratio(got, ref, bnd):
    return R.ratio(_d(got), ref, bnd)


def _gemm_case(seed, M=48, K=320, N=40):
    r = np.random.default_rng(seed)
    a = r.uniform(-1, 1, (M, K)).astype(F32)
    b = (r.uniform(-1, 1, (K, N)) / np.sqrt(K)).astype(F32)
    return a, b, r.uniform(-0.1, 0.1, N).astype(F32), r.uniform(-1, 1, (M, N)).astype(F32)


def _conv_block(seed, B=2, C=32, S=8):
    """A bottleneck tail in miniature: t -> c3 (1x1) + shortcut x, relu -> y; y -> c1 of the next block, relu -> z."""
    r = np.random.default_rng(seed)
    t = np.maximum(r.uniform(-1, 1, (B, C, S, S)), 0).astype(F32)
    x = r.uniform(-1, 2, (B, 4 * C, S, S)).astype(F32)
    w3 = (r.uniform(-1, 1, (4 * C, C, 1, 1)) / np.sqrt(C)).astype(F32)
    w1 = (r.uniform(-1, 1, (C, 4 * C, 1, 1)) / np.sqrt(4 * C)).astype(F32)
    w2 = (r.uniform(-1, 1, (C, C, 3, 3)) / np.sqrt(9 * C)).astype(F32)
    b3, b1 = r.uniform(-0.1, 0.1, 4 * C).astype(F32), r.uniform(-0.1, 0.1, C).astype(F32)
    return t, x, w3, b3, w1, b1, w2


def _col(b):
    return _d(b).reshape(1, -1, 1, 1)


def _attention_case(seed, amp, B=2, H=2, T=16, L=128):
    r = np.random.default_rng(seed)
    q, k = (r.uniform(-amp, amp, (B, H, n, 64)).astype(F32) for n in (T, L))
    v = r.uniform(-1, 1, (B, H, L, 64)).astype(F32)
    mask = np.zeros((B, 1, 1, L), F32)
    mask[0, 0, 0, L - 40:] = -10000.0
    mask[1, 0, 0, L - 25:] = -np.inf
    return q, k, v, mask


def _emulated_cases(tf32, seed):
    """[(name, emulated output, float64 reference, bound)] over every bound kind the GPU test uses."""
    out = []
    a, b, bias, res = _gemm_case(seed)
    S, A = R.matmul64(_d(a), _d(b))
    acc = emulate_matmul(a, b, tf32)
    for name, kw in (("bias + Gelu", dict(bias=bias, act=R.ACT_GELU)), ("bias + residual", dict(bias=bias, residual=res)),
                     ("bias + tanh Gelu", dict(bias=bias, act=R.ACT_GELU_TANH)), ("alpha", dict(alpha=0.125))):
        ref, bnd = R.epilogue_ref_and_bound(S, A, tf32, None if kw.get("bias") is None else _d(kw["bias"]),
                                            None if kw.get("residual") is None else _d(kw["residual"]),
                                            kw.get("act", R.ACT_NONE), kw.get("alpha", 1.0))
        out.append((f"FusedMatMul {name}", emulate_epilogue(acc, **kw), ref, bnd))
    t, x, w3, b3, w1, b1, w2 = _conv_block(seed)
    S3, A3 = R.conv64(_d(t), _d(w3), (0, 0, 0, 0), (1, 1))
    y = emulate_epilogue(emulate_conv(t, w3, 0, 1, tf32), b3[None, :, None, None], x, R.ACT_RELU)
    ref, bnd = R.epilogue_ref_and_bound(S3, A3, tf32, _col(b3), _d(x), R.ACT_RELU)
    out.append(("chained y", y, ref, bnd))
    Sz, Az = R.conv64(_d(y), _d(w1), (0, 0, 0, 0), (1, 1))
    z = emulate_epilogue(emulate_conv(y, w1, 0, 1, tf32), b1[None, :, None, None], None, R.ACT_RELU)
    ref, bnd = R.epilogue_ref_and_bound(Sz, Az, tf32, _col(b1), None, R.ACT_RELU)
    out.append(("chained z", z, ref, bnd))
    S2, A2 = R.conv64(_d(t), _d(w2), (1, 1, 1, 1), (2, 2))
    c2 = emulate_epilogue(emulate_conv(t, w2, 1, 2, tf32), b1[None, :, None, None], None, R.ACT_RELU)
    ref, bnd = R.epilogue_ref_and_bound(S2, A2, tf32, _col(b1), None, R.ACT_RELU)
    out.append(("3x3 stride 2", c2, ref, bnd))
    xp, wd = x[:, :16], (w3[:, :16] / F32(2)).astype(F32)  # a projection shortcut of 16 input channels
    Sp, Ap = R.conv64(_d(xp), _d(wd), (0, 0, 0, 0), (1, 1))
    both = emulate_conv(np.concatenate([t, xp], 1), np.concatenate([w3, wd], 1), 0, 1, tf32)
    yp = emulate_epilogue(emulate_epilogue(both, b3[None, :, None, None]), b1[0], None, R.ACT_RELU)
    ref, bnd = R.epilogue_ref_and_bound(S3 + Sp, A3 + Ap, tf32, _col(b3) + float(b1[0]), None, R.ACT_RELU)
    out.append(("projected", yp, ref, bnd))
    gap = (x.astype(F32).reshape(x.shape[0], x.shape[1], -1).cumsum(-1, dtype=F32)[..., -1:] / F32(x.shape[2] * x.shape[3]))
    ref, bnd = R.global_average_pool_ref_and_bound(_d(x))
    out.append(("GlobalAveragePool", gap.astype(F32).reshape(ref.shape), ref, bnd))
    return out


@pytest.mark.parametrize("mode,tf32", MODES, ids=[m for m, _ in MODES])
def test_emulated_kernels_stay_inside_the_bounds(mode, tf32):
    """Six seeds of every case: each inside its bound; every GEMM / convolution case uses a visible share of it."""
    worst = {}
    for seed in range(6):
        for name, got, ref, bnd in _emulated_cases(tf32, seed):
            r = _ratio(got, ref, bnd)
            assert r <= 1.0, f"{mode} seed {seed} {name}: the emulated kernel leaves the bound (ratio {r:.3f})"
            worst[name] = max(worst.get(name, 0.0), r)
    for name, r in worst.items():
        if name != "GlobalAveragePool":
            assert r > 0.02, f"{mode} {name}: the emulation uses only {r:.4f} of the bound"


def test_attention_bound_is_ref_and_bound():
    """The torch restatement gives ref_and_bound's numbers: masks with -10000 and -inf, a causal [1, 1, T, L] mask, a
    fully masked row, both modes."""
    for tf32 in (True, False):
        for amp in (1.0, 3.0):
            q, k, v, mask = _attention_case(5, amp)
            causal = np.where(np.arange(128)[None, :] <= np.arange(16)[:, None] + 100, 0, -np.inf).astype(F32)[None, None]
            full = mask.copy()
            full[1] = -np.inf
            for m in (None, mask, causal, full):
                want = tae.ref_and_bound(q, k, v, m, 0.125, tf32=tf32)
                got = R.attention_ref_and_bound(_d(q), _d(k), _d(v), None if m is None else _d(m), 0.125, tf32)
                for w, g in zip(want, got):
                    np.testing.assert_allclose(g.numpy(), w, rtol=1e-9, atol=1e-300)


@pytest.mark.parametrize("amp", [1.0, 3.0], ids=["flat", "peaked"])
def test_emulated_attention_stays_inside_the_bound(oracle, amp):
    """test_gpu_attention_encoder.emulate (the fused kernel's arithmetic) against the torch bound, the benched masks."""
    worst = 0.0
    for seed in range(4):
        q, k, v, mask = _attention_case(seed, amp)
        ref, bnd = R.attention_ref_and_bound(_d(q), _d(k), _d(v), _d(mask), 0.125, True)
        r = _ratio(tae.emulate(oracle, q, k, v, mask, 0.125), ref, bnd)
        assert r <= 1.0, f"seed {seed}: the emulated attention leaves the bound (ratio {r:.3f})"
        worst = max(worst, r)
    assert worst > 1e-3


@pytest.mark.parametrize("mode,tf32", MODES, ids=[m for m, _ in MODES])
def test_small_slips_leave_the_bounds(mode, tf32):
    a, b, bias, res = _gemm_case(1)
    S, A = R.matmul64(_d(a), _d(b))
    ref, bnd = R.epilogue_ref_and_bound(S, A, tf32, _d(bias), _d(res))
    acc = emulate_matmul(a, b, tf32)
    no_res = res.copy()
    no_res[7] = 0
    slips = {
        "one K block dropped": emulate_epilogue(emulate_matmul(a, b, tf32, drop_block=3), bias, res),
        "bias added twice": emulate_epilogue(emulate_epilogue(acc, bias), bias, res),
        "residual omitted for one row": emulate_epilogue(acc, bias, no_res),
    }
    for name, got in slips.items():
        assert _ratio(got, ref, bnd) > 1.0, f"{mode}: {name} stays inside the bound"
    # one channel of the chained next convolution computed from the block's input instead of its output y
    t, x, w3, b3, w1, b1, _ = _conv_block(2)
    y = emulate_epilogue(emulate_conv(t, w3, 0, 1, tf32), b3[None, :, None, None], x, R.ACT_RELU)
    z = emulate_epilogue(emulate_conv(y, w1, 0, 1, tf32), b1[None, :, None, None], None, R.ACT_RELU)
    wrong = emulate_epilogue(emulate_conv(x, w1, 0, 1, tf32), b1[None, :, None, None], None, R.ACT_RELU)
    z[:, 5] = wrong[:, 5]
    Sz, Az = R.conv64(_d(y), _d(w1), (0, 0, 0, 0), (1, 1))
    ref, bnd = R.epilogue_ref_and_bound(Sz, Az, tf32, _col(b1), None, R.ACT_RELU)
    assert _ratio(z, ref, bnd) > 1.0, f"{mode}: a chained channel from the wrong y stays inside the bound"
    # attention: one head's mask ignored; two adjacent keys' V rows swapped
    for amp in (1.0, 3.0):
        q, k, v, mask = _attention_case(3, amp)
        qd, kd, vd, md = _d(q), _d(k), _d(v), _d(mask)
        ref, bnd = R.attention_ref_and_bound(qd, kd, vd, md, 0.125, tf32)
        unmasked = ref.clone()
        unmasked[0, 1] = R.attention_ref_and_bound(qd, kd, vd, None, 0.125, tf32)[0][0, 1]
        p = torch.softmax(0.125 * qd[0, 0, 0] @ kd[0, 0].T + md[0, 0, 0], -1)
        t = min(int(p.argmax()), 126)
        sw = vd.clone()
        sw[0, 0, [t, t + 1]] = sw[0, 0, [t + 1, t]]
        swapped = R.attention_ref_and_bound(qd, kd, sw, md, 0.125, tf32)[0]
        for name, got in (("one head's mask ignored", unmasked), ("adjacent V rows swapped", swapped)):
            assert R.ratio(got, ref, bnd) > 1.0, f"{mode} amp {amp}: {name} stays inside the bound"


def test_cache_append_rule():
    """check_cache_append passes the right append and refuses a row written one position late or early, a changed
    earlier row and a written later row."""
    r = np.random.default_rng(4)
    B, H, M, d, P = 2, 3, 12, 8, 6
    prev = np.full((B, H, M, d), np.nan, F32)
    prev[:, :, :P] = r.uniform(-1, 1, (B, H, P, d))
    new = r.uniform(-1, 1, (B, H, d)).astype(F32)
    good = prev.copy()
    good[:, :, P] = new
    R.check_cache_append(good, prev, new, P, "right row")
    bad = {}
    for shift in (1, -1):
        b = prev.copy()
        b[:, :, P + shift] = new
        bad[f"shifted by {shift}"] = b
    b = good.copy()
    b[1, 2, 0, 3] += 1
    bad["earlier row changed"] = b
    b = good.copy()
    b[0, 0, M - 1] = 0
    bad["later row written"] = b
    b = good.copy()
    b[1, 0, P] = np.roll(new[1, 0], 1)
    bad["one head's row permuted"] = b
    for name, post in bad.items():
        with pytest.raises(AssertionError):
            R.check_cache_append(post, prev, new, P, name)


def test_int_matmul_is_the_oracle_product(oracle):
    """The exact float64 product and the oracle's cast_scale give the oracle's MatMulInteger and MatMulIntegerToFloat
    bits: u8 activations with their zero point, i8 weights, per-column and scalar scales."""
    rng = oracle.XorShiftRng(31)
    for M, K, N in ((5, 96, 40), (33, 768, 130)):
        a, b = rng.u8((M, K)), rng.i8((K, N))
        for zp in (np.uint8(0), np.uint8(131)):
            acc = R.int_matmul(a, zp, b)
            np.testing.assert_array_equal(acc, oracle.matmul_integer(a, b, zp, None))
            for scale in (rng.uniform((N,), 0.001, 0.05), rng.uniform((), 0.001, 0.05)):
                gotf = steps._int8_epilogue(oracle, acc, None, scale, None, None, R.ACT_NONE)
                want = oracle.matmul_integer_to_float(a, b, zp, None, scale)
                np.testing.assert_array_equal(gotf.view(np.int32), want.view(np.int32))


# ---- the recorder on a stand-in operator module ---------------------------------------------------------------------


def _fake_ops():
    """A module shaped like rten_b200.ops: a context whose launches count, operators that launch, in-place softmax."""
    O = types.ModuleType("fake_ops")

    class Context:
        def __init__(self):
            self.launches = 0

        def graph_begin(self):
            pass

        def graph_end(self):
            return "graph"

    class DeviceTensor:
        def __init__(self, ctx, name):
            self.ctx, self.name = ctx, name

        def assign(self, src):
            self.ctx.launches += 1

    class FusedMatMul:
        def __init__(self, alpha=None):
            self.alpha = alpha

        def run(self, ctx, a, b, bias=None):
            ctx.launches += 1
            return DeviceTensor(ctx, "scores")

    class AddSoftmax:
        def run(self, ctx, x, y, in_place=False):
            ctx.launches += 1
            return x

    class MatMul:
        def run(self, ctx, a, b, out=None):
            ctx.launches += 2
            return out

    class Outer:  # an operator built on another: one record
        def run(self, ctx, a):
            return FusedMatMul().run(ctx, a, a)

    for c in (Context, DeviceTensor, FusedMatMul, AddSoftmax, MatMul, Outer):
        c.__module__ = O.__name__
        setattr(O, c.__name__, c)
    return O


def test_recorder_and_units(monkeypatch):
    O = _fake_ops()
    ctx = O.Context()
    q, kt, v, out, mask = (O.DeviceTensor(ctx, n) for n in ("q", "kt", "v", "out", "mask"))
    rec = steps.Recorder()
    with monkeypatch.context() as mp:
        rec.install(mp, O)
        O.FusedMatMul(0.5).run(ctx, q, kt)  # outside the capture: not recorded
        ctx.graph_begin()
        s = O.FusedMatMul(0.5).run(ctx, q, kt)
        p = O.AddSoftmax().run(ctx, s, mask, in_place=True)
        O.MatMul().run(ctx, p, v, out=out)
        O.Outer().run(ctx, q)
        out.assign(q)
        ctx.graph_end()
    records = rec.captures[0]
    assert [repr(r) for r in records] == ["FusedMatMul.run", "AddSoftmax.run", "MatMul.run", "Outer.run",
                                          "DeviceTensor.assign"]
    assert [r.launches for r in records] == [1, 1, 2, 1, 1] and ctx.launches == 7
    assert records[0].attrs == {"alpha": 0.5} and records[0].args["bias"] is None and records[2].args["out"] is out
    assert records[4].obj is out and records[4].args["src"] is q
    units = steps._units(records)
    assert [len(u) for u in units] == [3, 1, 1]
    # a softmax that is not in place on the product is not part of an attention triple
    records[1].out = O.DeviceTensor(ctx, "copy")
    assert [len(u) for u in steps._units(records)] == [1, 1, 1, 1, 1]
