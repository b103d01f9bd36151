"""Float64 references and per-element error bounds for the operator calls of the benched steps
(tests/test_gpu_benched_steps.py), and the cache-append rule.  tests/test_benched_steps_cpu.py holds float32 emulations
of the kernels inside these bounds and shows that small slips land outside them.

Everything takes torch float64 tensors on any device, so the GPU test computes its references on the GPU."""
import math

import numpy as np
import torch
import torch.nn.functional as F

ACT_NONE, ACT_RELU, ACT_GELU, ACT_GELU_TANH = 0, 1, 2, 3

# operand rounding of one GEMM / convolution: single-pass TF32 (True) or 3xTF32 (False), relative to sum |a b|
GEMM_COEF = {True: 2.0 ** -9, False: 2.0 ** -18}
# max |d/dx gelu(x)| over the reals: 1.1289 at x = sqrt(2) (erf form); the tanh form's maximum is 1.1289 too
GELU_SLOPE = 1.13


def ratio(got, ref, bnd):
    """max |got - ref| / bnd (0 / 0 counts as 0, so an exact zero must come back as an exact zero; a NaN where the
    reference is finite counts as infinitely far)."""
    err = (got.to(torch.float64) - ref).abs()
    r = torch.where(err == 0, torch.zeros_like(err), err / bnd)
    r = torch.nan_to_num(r, nan=math.inf)
    return float(r.max()) if r.numel() else 0.0


def gelu64(x, approximate):
    if approximate:
        return 0.5 * x * (1.0 + torch.tanh(math.sqrt(2.0 / math.pi) * (x + 0.044715 * x ** 3)))
    return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))


def epilogue_ref_and_bound(acc, absacc, tf32, bias=None, residual=None, act=ACT_NONE, alpha=1.0):
    """out = act(alpha S + bias + residual) in float64 from the exact product S = sum_k a_k b_k (`acc`) and
    A = sum_k |a_k b_k| (`absacc`), and a bound on |out_got - out| element by element for a kernel that multiplies
    TF32 operands (or 3xTF32 splits), accumulates in f32 and runs its epilogue in f32.

    Product.  Each TF32 operand is truncated by less than 2^-10 of itself, so each product moves by less than
    2^-9 |a b| (2^-18 |a b| after the three-part 3xTF32 split): |S_got - S| <= c A, c = 2^-9 or 2^-18.  The tensor
    cores' f32 accumulation is not in this sum.  It is no worst-case bound: K = 4608 f32 additions could in principle
    reach K 2^-24 A.  In practice its error stays inside c A at the benched depths, and the ratio the test prints shows
    the margin: the largest, 0.81, is a 3xTF32 ResNet-50 convolution on an H100 80GB HBM3 at 700 W.
    Epilogue.  The scale multiply, the bias add and the residual add (a projected convolution adds two biases) round in
    f32: at most four roundings of values no larger than M = |alpha| A + |bias| + |residual|, so the pre-activation
    is off by at most c |alpha| A + 2^-21 M.  Relu has slope 1 and Gelu at most 1.13.  Gelu's own f32 evaluation
    (0.5 x (1 + erf) loses 1 + erf's cancellation for negative x) adds at most 2^-21 (|out| + |x|), and the stored
    output one more rounding, 2^-23 |out|."""
    s = alpha * acc
    m = abs(alpha) * absacc
    for t in (bias, residual):
        if t is not None:
            s = s + t
            m = m + t.abs()
    pre = GEMM_COEF[tf32] * abs(alpha) * absacc + 2.0 ** -21 * m
    if act == ACT_RELU:
        ref, bnd = s.clamp_min(0.0), pre
    elif act in (ACT_GELU, ACT_GELU_TANH):
        ref = gelu64(s, act == ACT_GELU_TANH)
        bnd = GELU_SLOPE * pre + 2.0 ** -21 * (ref.abs() + s.abs())
    else:
        assert act == ACT_NONE, f"activation {act} has no bound here"
        ref, bnd = s, pre
    return ref, bnd + 2.0 ** -23 * ref.abs()


def matmul64(a, b):
    """(S, A) of a @ b, batched over leading dimensions."""
    return a @ b, a.abs() @ b.abs()


def conv64(x, w, pads, strides, dilations=(1, 1), groups=1):
    """(S, A) of the convolution of NCHW x with OIHW w (pads [top, left, bottom, right]), no bias."""
    xp = F.pad(x, (pads[1], pads[3], pads[0], pads[2]))
    kw = dict(stride=tuple(strides), dilation=tuple(dilations), groups=groups)
    return F.conv2d(xp, w, None, **kw), F.conv2d(xp.abs(), w.abs(), None, **kw)


def global_average_pool_ref_and_bound(x):
    """mean over H, W of NCHW x -> [B, C, 1, 1], and its bound: an f32 sum of n = H W terms and the division round
    at most n + 1 times, each by 2^-24 of a value no larger than sum |x|: (n + 1) 2^-24 mean |x|, plus 2^-23 |out|."""
    n = x.shape[2] * x.shape[3]
    ref = x.mean((2, 3), keepdim=True)
    return ref, (n + 1) * 2.0 ** -24 * x.abs().mean((2, 3), keepdim=True) + 2.0 ** -23 * ref.abs()


# (score coefficient, output coefficient) per f32 mode, as test_gpu_attention_encoder.COEF
ATTN_COEF = {True: (2.0 ** -9 + 2.0 ** -17, 2.0 ** -9 + 2.0 ** -16), False: (2.0 ** -15, 2.0 ** -15)}


def attention_ref_and_bound(q, k, v, mask=None, scale=0.125, tf32=True):
    """test_gpu_attention_encoder.ref_and_bound (its docstring derives the bound) in torch: O = softmax(scale q k^T +
    mask) v for q [B, h, T, d], k / v [B, h, L, d] and an additive mask broadcast to [B, h, T, L]; rows without a finite
    maximum give zeros.  The CPU companion checks that both give the same numbers."""
    us, uo = ATTN_COEF[tf32]
    s = scale * (q @ k.transpose(-1, -2))
    a = scale * (q.abs() @ k.abs().transpose(-1, -2))
    z = s if mask is None else s + mask
    live = z > -math.inf
    p = torch.softmax(z, -1)
    p = torch.nan_to_num(p, nan=0.0)
    delta = (us * torch.where(live, a, 0.0).amax(-1)
             + 2.0 ** -22 * torch.where(live, z.abs(), 0.0).amax(-1))
    ref = p @ v
    bnd = (p @ v.abs()) * (torch.expm1(2.0 * delta)[..., None] + uo)
    return ref, bnd


def int_matmul(a, a_zero_point, b):
    """sum_k (a[m, k] - a_zero_point) b[k, n] exactly, as int32 numpy: the u8 / i8 values are exact in float64 and
    every partial sum stays below 2^53, so a float64 product gives the exact integers MatMulInteger computes."""
    dev = "cuda" if torch.cuda.is_available() else "cpu"
    at = torch.from_numpy(np.ascontiguousarray(a)).to(dev, torch.float64) - float(a_zero_point)
    bt = torch.from_numpy(np.ascontiguousarray(b)).to(dev, torch.float64)
    return (at @ bt).cpu().numpy().astype(np.int32)


def check_cache_append(post, prev, new, P, what):
    """A KV cache [B, heads, M, d] after the step that appends position P (same P for every batch row): row P holds
    `new` [B, heads, d] bit for bit, rows before P are unchanged from `prev` (the cache read back after the previous
    step), and rows after P still hold NaN.  Raises AssertionError naming the first rule that fails."""
    bits = lambda t: np.ascontiguousarray(t, np.float32).view(np.int32)
    assert np.array_equal(bits(post[:, :, P]), bits(new)), f"{what}: row {P} is not the appended key / value"
    assert np.array_equal(bits(post[:, :, :P]), bits(prev[:, :, :P])), f"{what}: rows before {P} changed"
    assert np.isnan(post[:, :, P + 1:]).all(), f"{what}: a row after {P} was written"
