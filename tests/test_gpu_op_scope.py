"""`pytest -m gpu`: a call that fails after it has allocated its outputs returns them.

Each case calls the C ABI with outputs whose `data` is NULL and fails only after the call allocated them.  It checks the
status and message, that every output the call was asked to allocate has `data` NULL again, and that the next valid
call of the same operator on that context gives the bits a fresh context gives.  One more case runs Attention through
a one-kernel branch that allocates its output and then declines the shape: the result is the composed path's."""
import ctypes as C

import numpy as np
import pytest

import gpu_checks as gc

pytestmark = pytest.mark.gpu

F32 = np.float32
INCOMPATIBLE_SHAPES, INVALID_VALUE, UNSUPPORTED_VALUE, UNSUPPORTED_OUTPUT = 3, 5, 6, 7


@pytest.fixture(scope="module")
def rt():
    import rten_b200
    from rten_b200 import _lib
    _lib.load()
    return rten_b200


def _arg(A, t):
    """`t`'s descriptor for a call, with `t` kept alive (and its memory out of the pool) for as long as the call's `A`"""
    A.keep.append(t)
    return A.t(t)


def _check_failure(ctx, st, status, msg, outs):
    assert st == status, f"status {st}, expected {status}: {ctx.lib.rten_b200_last_error(ctx.handle).decode()}"
    assert ctx.lib.rten_b200_last_error(ctx.handle).decode() == msg
    for o in outs:
        assert not o.data, "an output the failed call allocated is still set"


def _same_as_fresh(rt, ctx, run, what):
    """`run(ctx)` gives the same bits on the context a call failed on as on a fresh one."""
    gc.assert_bit_exact(run(ctx), run(rt.Context(0)), what)


def _softmax_case(rt, oracle, host):
    ctx = rt.Context(0)
    r = oracle.XorShiftRng(11)
    x, bad_mask, mask = r.uniform((4, 8)), r.uniform((3, 8)), r.uniform((1, 8))
    dev = (lambda a: a) if host else ctx.to_device
    A = rt.ops._Args(ctx)
    o = A.out()
    st = ctx.lib.rten_b200_softmax(ctx.handle, _arg(A, dev(x)), _arg(A, dev(bad_mask)), -1, 0, C.byref(o))
    _check_failure(ctx, st, INCOMPATIBLE_SHAPES, "Cannot broadcast inputs", [o])
    _same_as_fresh(rt, ctx, lambda c: rt.AddSoftmax().run(c, x, mask).numpy(), "Softmax after a failed call")


def test_softmax_device(rt, oracle):
    _softmax_case(rt, oracle, host=False)


def test_softmax_host(rt, oracle):
    _softmax_case(rt, oracle, host=True)


def test_matmul_residual(rt, oracle):
    ctx = rt.Context(0)
    r = oracle.XorShiftRng(12)
    a, b, res = r.uniform((32, 64)), r.uniform((64, 48)), r.uniform((32, 48))
    A = rt.ops._Args(ctx)
    o = A.out()
    st = ctx.lib.rten_b200_matmul_ex(ctx.handle, _arg(A, ctx.to_device(a)), _arg(A, ctx.to_device(b)), None, None, 1.0,
                                     _arg(A, ctx.to_device(r.uniform((32, 47)))), 0, C.byref(o))
    _check_failure(ctx, st, INCOMPATIBLE_SHAPES, "residual shape does not match output", [o])

    def run(c):
        B = rt.ops._Args(c)
        out = B.out()
        c.check(c.lib.rten_b200_matmul_ex(c.handle, _arg(B, c.to_device(a)), _arg(B, c.to_device(b)), None, None, 1.0,
                                          _arg(B, c.to_device(res)), 0, C.byref(out)))
        return B.wrap(out, None).numpy()

    _same_as_fresh(rt, ctx, run, "matmul_ex after a failed call")


def test_conv_residual(rt, oracle):
    ctx = rt.Context(0)
    r = oracle.XorShiftRng(13)
    x, w, res = r.uniform((1, 16, 6, 6)), r.uniform((32, 16, 1, 1)), r.uniform((1, 32, 6, 6))
    p = rt.ops._conv_params((0, 0, 0, 0), 1, (1, 1), (1, 1))
    A = rt.ops._Args(ctx)
    o = A.out()
    st = ctx.lib.rten_b200_conv2d_ex(ctx.handle, _arg(A, ctx.to_device(x)), A.t(w), None, None, C.byref(p),
                                     _arg(A, ctx.to_device(r.uniform((1, 32, 5, 5)))), 0, C.byref(o))
    _check_failure(ctx, st, INCOMPATIBLE_SHAPES, "residual shape does not match output", [o])

    def run(c):
        B = rt.ops._Args(c)
        out = B.out()
        c.check(c.lib.rten_b200_conv2d_ex(c.handle, _arg(B, c.to_device(x)), B.t(w), None, None, C.byref(p),
                                          _arg(B, c.to_device(res)), 0, C.byref(out)))
        return B.wrap(out, None).numpy()

    _same_as_fresh(rt, ctx, run, "conv2d_ex after a failed call")


def test_resize_empty_input(rt, oracle):
    ctx = rt.Context(0)
    A = rt.ops._Args(ctx)
    o = A.out()
    p = rt.ops.RtenResizeParams()
    p.n, p.use_sizes = 4, 1
    for i, v in enumerate((1, 2, 4, 4)):
        p.sizes[i] = v
    st = ctx.lib.rten_b200_resize(ctx.handle, _arg(A, ctx.empty((1, 2, 0, 3))), C.byref(p), C.byref(o))
    _check_failure(ctx, st, INVALID_VALUE, "cannot resize an empty input", [o])
    x = oracle.XorShiftRng(14).uniform((1, 2, 3, 3))
    _same_as_fresh(rt, ctx, lambda c: rt.Resize().run(c, c.to_device(x), sizes=(1, 2, 6, 6)).numpy(), "Resize after a failed call")


def test_dynamic_quantize_linear_strided_output(rt, oracle):
    ctx = rt.Context(0)
    x = oracle.XorShiftRng(15).uniform((8, 16), -2, 2)
    y = ctx.empty((8, 32), np.uint8).view((8, 16), (32, 1))
    A = rt.ops._Args(ctx)
    yo, s, z = A.out(y), A.out(), A.out()
    st = ctx.lib.rten_b200_dynamic_quantize_linear_ranged(ctx.handle, _arg(A, ctx.to_device(x)), None, C.byref(yo), C.byref(s),
                                                          C.byref(z), None)
    _check_failure(ctx, st, UNSUPPORTED_OUTPUT, "quantized output must be contiguous", [s, z])

    def run(c):
        q, qs, qz = rt.DynamicQuantizeLinear().run(c, c.to_device(x))
        return np.concatenate([q.numpy().ravel().view(np.uint8), qs.numpy().ravel().view(np.uint8), qz.numpy().ravel()])

    _same_as_fresh(rt, ctx, run, "DynamicQuantizeLinear after a failed call")


def test_multi_head_attention_misaligned_query(rt, oracle):
    ctx = rt.Context(0)
    r = oracle.XorShiftRng(16)
    B, S, H, D = 1, 4, 2, 64
    q = r.uniform((B, S, H * D))
    buf = ctx.empty((B * S * H * D + 1,))
    buf.copy_from(np.concatenate([np.zeros(1, F32), q.ravel()]))
    qv = buf.view((B, S, H * D), (S * H * D, H * D, 1), offset_elems=1)
    A = rt.ops._Args(ctx)
    o, pk, pv = A.out(), A.out(), A.out()
    p = rt.ops.RtenMhaParams(H, 0.0, -10000.0, 0)
    st = ctx.lib.rten_b200_multi_head_attention(ctx.handle, A.t(qv), None, None, None, None, None, None, None, None, None,
                                                C.byref(p), C.byref(o), C.byref(pk), C.byref(pv))
    _check_failure(ctx, st, UNSUPPORTED_VALUE,
                   "MultiHeadAttention: query, key, value, the caches and the output need 16-byte aligned rows", [o, pk, pv])

    def run(c):
        out, k, v = rt.MultiHeadAttention(H).run(c, c.to_device(q))
        return np.concatenate([out.numpy().ravel(), k.numpy().ravel(), v.numpy().ravel()])

    _same_as_fresh(rt, ctx, run, "MultiHeadAttention after a failed call")


def test_attention_declined_branch(rt, oracle):
    """TF32 mode with 64 keys: the fused encoder branch allocates the output, its kernel takes 128 keys only, and the
    call composes MatMul -> Softmax -> MatMul instead."""
    ctx = rt.Context(0)
    ctx.set_f32_mode(False)
    r = oracle.XorShiftRng(17)
    B, Hh, Sq, Sk, D = 1, 2, 64, 64, 64
    q, k, v = (ctx.to_device(r.uniform(s)) for s in ((B, Hh, Sq, D), (B, Hh, Sk, D), (B, Hh, Sk, D)))
    scale = 1.0 / np.sqrt(F32(D))
    A = rt.ops._Args(ctx)
    o = A.out()
    p = rt.ops.RtenAttentionParams(0, Hh, Hh, float(scale), 0.0)
    ctx.check(ctx.lib.rten_b200_attention(ctx.handle, A.t(q), A.t(k), A.t(v), None, None, C.byref(p), None, None, C.byref(o)))
    got = A.wrap(o, None).numpy()
    kt = k.permute(0, 1, 3, 2)
    A2 = rt.ops._Args(ctx)
    s, y = A2.out(), A2.out()
    ctx.check(ctx.lib.rten_b200_matmul_ex(ctx.handle, A2.t(q), A2.t(kt), None, None, float(scale), None, 0, C.byref(s)))
    ctx.check(ctx.lib.rten_b200_softmax(ctx.handle, C.byref(s), None, -1, 1, C.byref(s)))
    ctx.check(ctx.lib.rten_b200_matmul_ex(ctx.handle, C.byref(s), A2.t(v), None, None, 1.0, None, 0, C.byref(y)))
    exp = A2.wrap(y, None).numpy()
    ctx.free(s.data)
    gc.assert_bit_exact(got, exp, "Attention through a declined one-kernel branch")
