"""Host-side mirror of RTen's operator interface for the hot path, over the C ABI.

Each class below corresponds to the reference operator of the same name and keeps its attribute
names (src/ops/matmul.rs, conv.rs, norm.rs, attention.rs, unary_elementwise.rs, quantize.rs):
`op.run(ctx, *inputs) -> outputs` plays `Operator::run(&OpRunContext)` (src/operator.rs:498),
`op.prepack(ctx, index, input)` plays `Operator::prepack` (:587-601), and failures raise `OpError`
carrying the reference's `OpError` variant and message.

Inputs may be numpy arrays (host tensors: the library stages them through HBM inside the call)
or `DeviceTensor`s (resident in HBM).  Outputs are `DeviceTensor`s allocated from the context's
pool; `.numpy()` copies them back.  Nothing here computes: no CUDA library => exception.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional, Sequence

import numpy as np

from . import _lib
from ._lib import (RTEN_DEVICE_HOST, RTEN_F32, RTEN_I8, RTEN_I32, RTEN_U8, RtenActivation, RtenAttentionParams, RtenConvParams,
                   RtenConvTransposeParams, RtenGqaParams, RtenMhaParams, RtenResizeParams, RtenTensor, RtenRnnParams)

_NP2RT = {np.dtype(np.float32): RTEN_F32, np.dtype(np.int32): RTEN_I32, np.dtype(np.int8): RTEN_I8,
          np.dtype(np.uint8): RTEN_U8}
_RT2NP = {v: k for k, v in _NP2RT.items()}

ACT_NONE, ACT_RELU, ACT_GELU, ACT_GELU_TANH = 0, 1, 2, 3
# activations fused into a Conv epilogue through Conv(activation=...) only (rten_b200_conv2d_act); ACT_HARD_SIGMOID takes
# (alpha, beta): pass (ACT_HARD_SIGMOID, alpha, beta), or the code alone for the ONNX defaults
ACT_SIGMOID, ACT_SILU, ACT_HARD_SIGMOID, ACT_HARD_SWISH = 4, 5, 6, 7


class OpError(Exception):
    """`OpError` (src/operator.rs:116-144)."""

    def __init__(self, status: int, msg: str):
        self.status = status
        self.kind = _lib.STATUS_NAMES.get(status, str(status))
        self.msg = msg
        super().__init__(f"{self.kind}: {msg}")


class Context:
    """One per host thread / stream (= OpRunContext + BufferPool, src/operator.rs:328-390)."""

    def __init__(self, device: int = 0, stream: Optional[int] = None, workspace_bytes: int = 0):
        self.lib = _lib.load()
        h = C.c_void_p()
        st = self.lib.rten_b200_ctx_create(device, C.c_void_p(stream) if stream else None, workspace_bytes, C.byref(h))
        if st != 0:
            raise OpError(st, "rten_b200_ctx_create failed: an H100 (sm_90a) with a working driver is required")
        self.handle = h
        self.device = device

    def close(self):
        if getattr(self, "handle", None):
            self.lib.rten_b200_ctx_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def check(self, st: int):
        if st != 0:
            raise OpError(st, self.lib.rten_b200_last_error(self.handle).decode())

    def sync(self):
        self.check(self.lib.rten_b200_sync(self.handle))

    def set_f32_mode(self, tf32x3: bool):
        """True (the library default): 3xTF32 error-compensated products, f32-grade accuracy at 1/3 of the tensor rate.
        False: single-pass TF32 -- an explicit opt-in to 10-bit operand mantissas."""
        self.check(self.lib.rten_b200_set_f32_mode(self.handle, 1 if tf32x3 else 0))

    def forced_plan_counts(self):
        """(matched, unmatched) launches under the RTEN_B200_FORCE_* sweep knobs."""
        a, b = C.c_uint64(), C.c_uint64()
        self.check(self.lib.rten_b200_debug_forced_plans(self.handle, C.byref(a), C.byref(b)))
        return int(a.value), int(b.value)

    def set_autotune(self, enable: bool = True):
        """Time candidate launch plans the first time each MatMul / Conv problem is seen (outside graph capture)."""
        self.check(self.lib.rten_b200_set_autotune(self.handle, 1 if enable else 0))

    def save_plans(self, path: str):
        self.check(self.lib.rten_b200_save_plans(self.handle, path.encode()))

    def load_plans(self, path: str):
        self.check(self.lib.rten_b200_load_plans(self.handle, path.encode()))

    @property
    def launches(self) -> int:
        return int(self.lib.rten_b200_launch_count(self.handle))

    # ---- memory
    def alloc(self, nbytes: int) -> int:
        p = C.c_void_p()
        self.check(self.lib.rten_b200_alloc(self.handle, nbytes, C.byref(p)))
        return p.value

    def free(self, ptr: int):
        self.check(self.lib.rten_b200_free(self.handle, C.c_void_p(ptr)))

    def pinned_empty(self, shape, dtype) -> np.ndarray:
        """Pinned host array (for asynchronous staging of host tensors)."""
        dtype = np.dtype(dtype)
        n = int(np.prod(shape)) * dtype.itemsize
        p = C.c_void_p()
        self.check(self.lib.rten_b200_host_alloc(self.handle, max(n, 16), C.byref(p)))
        buf = (C.c_uint8 * max(n, 1)).from_address(p.value)
        arr = np.frombuffer(buf, dtype=dtype, count=int(np.prod(shape))).reshape(shape)
        return arr

    def empty(self, shape, dtype=np.float32, strides=None) -> "DeviceTensor":
        dtype = np.dtype(dtype)
        shape = tuple(int(s) for s in shape)
        n = int(np.prod(shape)) if len(shape) else 1
        ptr = self.alloc(max(n, 1) * dtype.itemsize)
        if strides is None:
            strides = _contig(shape)
        return DeviceTensor(self, ptr, shape, tuple(strides), dtype, owner=True)

    def to_device(self, arr, channels_last: bool = False) -> "DeviceTensor":
        arr = np.asarray(arr)
        strides = None
        if channels_last and arr.ndim == 4:
            b, c, h, w = arr.shape
            strides = (h * w * c, 1, w * c, c)
        t = self.empty(arr.shape, arr.dtype, strides)
        t.copy_from(arr)
        return t

    # ---- CUDA graph over an op list
    def graph_begin(self):
        self.check(self.lib.rten_b200_graph_begin(self.handle))

    def graph_end(self) -> "Graph":
        g = C.c_void_p()
        self.check(self.lib.rten_b200_graph_end(self.handle, C.byref(g)))
        return Graph(self, g)


class Graph:
    def __init__(self, ctx: Context, handle):
        self.ctx, self.handle = ctx, handle

    def launch(self):
        self.ctx.check(self.ctx.lib.rten_b200_graph_launch(self.ctx.handle, self.handle))

    def __del__(self):
        try:
            if self.handle and self.ctx.handle:
                self.ctx.lib.rten_b200_graph_destroy(self.handle)
        except Exception:
            pass


def _contig(shape):
    s, out = 1, []
    for d in reversed(shape):
        out.append(s)
        s *= d
    return tuple(reversed(out))


class DeviceTensor:
    """A strided tensor resident in HBM (element strides, like rten-tensor layouts)."""

    def __init__(self, ctx: Context, ptr: int, shape, strides, dtype, owner: bool, base=None):
        self.ctx, self.ptr, self.shape, self.strides, self.dtype = ctx, ptr, tuple(shape), tuple(strides), np.dtype(dtype)
        self.owner = owner
        self.base = base  # keeps the owning tensor alive for views

    def __del__(self):
        try:
            if self.owner and self.ptr and self.ctx.handle:
                self.ctx.lib.rten_b200_free(self.ctx.handle, C.c_void_p(self.ptr))
        except Exception:
            pass

    @property
    def ndim(self):
        return len(self.shape)

    @property
    def size(self):
        return int(np.prod(self.shape)) if self.shape else 1

    def desc(self) -> RtenTensor:
        return _desc(self.ptr, self.dtype, self.shape, self.strides, self.ctx.device)

    def view(self, shape, strides, offset_elems: int = 0) -> "DeviceTensor":
        return DeviceTensor(self.ctx, self.ptr + offset_elems * self.dtype.itemsize, shape, strides, self.dtype, False,
                            base=self.base if self.base is not None else self)

    def permute(self, *axes) -> "DeviceTensor":
        return self.view([self.shape[a] for a in axes], [self.strides[a] for a in axes])

    def reshape(self, *shape) -> "DeviceTensor":
        assert self.is_contiguous(), "reshape needs a contiguous tensor"
        shape = tuple(shape[0]) if len(shape) == 1 and not isinstance(shape[0], int) else tuple(shape)
        assert int(np.prod(shape)) == self.size
        return self.view(shape, _contig(shape))

    def is_contiguous(self) -> bool:
        return all(s == 1 or st == c for s, st, c in zip(self.shape, self.strides, _contig(self.shape)))

    def copy_from(self, arr: np.ndarray):
        arr = np.ascontiguousarray(arr, dtype=self.dtype).reshape(np.shape(arr))  # (ascontiguousarray turns 0-d into 1-d)
        assert arr.shape == self.shape
        src = _desc(arr.ctypes.data, arr.dtype, arr.shape, _contig(arr.shape), RTEN_DEVICE_HOST)
        dst = self.desc()
        self.ctx.check(self.ctx.lib.rten_b200_copy(self.ctx.handle, C.byref(src), C.byref(dst)))

    def assign(self, src: "DeviceTensor"):
        """Strided device-to-device copy of `src` (same shape) into this view (e.g. appending to a KV cache)."""
        assert tuple(src.shape) == tuple(self.shape) and src.dtype == self.dtype
        a, b = src.desc(), self.desc()
        self.ctx.check(self.ctx.lib.rten_b200_copy(self.ctx.handle, C.byref(a), C.byref(b)))

    def numpy(self) -> np.ndarray:
        out = np.empty(self.shape, self.dtype)
        dst = _desc(out.ctypes.data, out.dtype, out.shape, _contig(out.shape), RTEN_DEVICE_HOST)
        src = self.desc()
        self.ctx.check(self.ctx.lib.rten_b200_copy(self.ctx.handle, C.byref(src), C.byref(dst)))
        return out


def from_torch(ctx: Context, t) -> DeviceTensor:
    """Borrow a CUDA torch tensor's storage (torch is plumbing for device memory only)."""
    import torch

    dt = {torch.float32: np.float32, torch.int32: np.int32, torch.int8: np.int8, torch.uint8: np.uint8}[t.dtype]
    return DeviceTensor(ctx, t.data_ptr(), tuple(t.shape), tuple(t.stride()), dt, owner=False, base=t)


def _desc(ptr, dtype, shape, strides, device) -> RtenTensor:
    d = RtenTensor()
    d.data = ptr
    d.dtype = _NP2RT[np.dtype(dtype)]
    d.ndim = len(shape)
    for i, (s, st) in enumerate(zip(shape, strides)):
        d.shape[i] = int(s)
        d.strides[i] = int(st)
    d.device = device
    return d


class _Args:
    """Keeps numpy inputs alive for the duration of a call and builds descriptors."""

    def __init__(self, ctx: Context):
        self.ctx = ctx
        self.keep = []

    def t(self, x):
        if x is None:
            return None
        if isinstance(x, DeviceTensor):
            d = x.desc()
        else:
            a = np.asarray(x)
            if a.dtype not in _NP2RT:
                raise OpError(2, f"unsupported dtype {a.dtype}")
            if any(s < 0 for s in a.strides):
                a = np.ascontiguousarray(a)
            self.keep.append(a)
            d = _desc(a.ctypes.data, a.dtype, a.shape, [s // a.itemsize for s in a.strides], RTEN_DEVICE_HOST)
        self.keep.append(d)
        return C.byref(d)

    def out(self, into: Optional[DeviceTensor] = None):
        d = into.desc() if into is not None else RtenTensor()
        self.keep.append(d)
        return d

    def wrap(self, d: RtenTensor, into: Optional[DeviceTensor]) -> DeviceTensor:
        if into is not None:
            return into
        shape = tuple(d.shape[i] for i in range(d.ndim))
        strides = tuple(d.strides[i] for i in range(d.ndim))
        return DeviceTensor(self.ctx, d.data, shape, strides, _RT2NP[d.dtype], owner=True)


class Packed:
    """`PrepackedInput` (src/operator.rs:25-31)."""

    def __init__(self, ctx: Context, handle):
        self.ctx, self.handle = ctx, handle

    def __del__(self):
        try:
            if self.handle and self.ctx.handle:
                self.ctx.lib.rten_b200_packed_free(self.ctx.handle, self.handle)
        except Exception:
            pass


def _ph(p: Optional[Packed]):
    return p.handle if p is not None else None


# =========================================================================================
# Operators
# =========================================================================================
class Gemm:
    """src/ops/matmul.rs:106-147; ONNX defaults alpha = beta = 1 (src/op_registry/onnx_registry.rs:1184-1196)."""

    def __init__(self, alpha=1.0, beta=1.0, transpose_a=False, transpose_b=False):
        self.alpha, self.beta, self.transpose_a, self.transpose_b = alpha, beta, transpose_a, transpose_b

    def run(self, ctx, a, b, c=None, out=None):
        A = _Args(ctx)
        o = A.out(out)
        ctx.check(ctx.lib.rten_b200_gemm(ctx.handle, A.t(a), A.t(b), A.t(c), self.alpha, self.beta, int(self.transpose_a),
                                         int(self.transpose_b), C.byref(o)))
        return A.wrap(o, out)


class MatMul:
    """src/ops/matmul.rs:387-434"""

    def prepack_inputs(self):
        return [1]

    def prepack(self, ctx, index, value):
        if index != 1:
            return None
        A = _Args(ctx)
        h = C.c_void_p()
        ctx.check(ctx.lib.rten_b200_prepack_b(ctx.handle, A.t(value), C.byref(h)))
        return Packed(ctx, h)

    def run(self, ctx, a, b, packed_b: Optional[Packed] = None, out=None):
        A = _Args(ctx)
        o = A.out(out)
        ctx.check(ctx.lib.rten_b200_matmul(ctx.handle, A.t(a), A.t(b), _ph(packed_b), None, 1.0, C.byref(o)))
        return A.wrap(o, out)


class FusedMatMul(MatMul):
    """src/ops/matmul.rs:459-507: optional `alpha`, row bias as third input.  `activation` / `residual`
    are this backend's epilogue extensions (0 = reference behaviour)."""

    def __init__(self, alpha: Optional[float] = None, activation: int = ACT_NONE):
        self.alpha, self.activation = alpha, activation

    def run(self, ctx, a, b, bias=None, packed_b: Optional[Packed] = None, residual=None, out=None):
        A = _Args(ctx)
        o = A.out(out)
        ctx.check(ctx.lib.rten_b200_matmul_ex(ctx.handle, A.t(a), A.t(b), _ph(packed_b), A.t(bias),
                                              1.0 if self.alpha is None else self.alpha, A.t(residual), self.activation,
                                              C.byref(o)))
        return A.wrap(o, out)


class MatMulInteger(MatMul):
    """src/ops/matmul.rs:649-697"""

    def run(self, ctx, a, b, a_zero_point=None, b_zero_point=None, packed_b: Optional[Packed] = None, out=None):
        A = _Args(ctx)
        o = A.out(out)
        ctx.check(ctx.lib.rten_b200_matmul_integer(ctx.handle, A.t(a), A.t(b), _ph(packed_b), A.t(a_zero_point),
                                                   A.t(b_zero_point), None, C.byref(o)))
        return A.wrap(o, out)


class MatMulIntegerToFloat(MatMul):
    """src/ops/matmul.rs:776-811 (inputs: a, b, a_zero_point, b_zero_point, scale)"""

    def __init__(self, activation: int = ACT_NONE):
        self.activation = activation

    def run(self, ctx, a, b, a_zero_point, b_zero_point, scale, packed_b: Optional[Packed] = None, out=None, bias=None,
            residual=None, scale_b=None, out_range=None):
        """`bias` / `residual` / `self.activation`: the Add / Add / Gelu nodes that follow the operator in a quantised
        transformer, folded into the epilogue with the same f32 roundings (rten_b200_matmul_integer_ex)."""
        if scale is None:
            raise OpError(4, "missing inputs")
        A = _Args(ctx)
        o = A.out(out)
        ctx.check(ctx.lib.rten_b200_matmul_integer_ex(ctx.handle, A.t(a), A.t(b), _ph(packed_b), A.t(a_zero_point),
                                                      A.t(b_zero_point), A.t(scale), A.t(scale_b), A.t(bias), A.t(residual),
                                                      self.activation, A.t(out_range), C.byref(o)))
        return A.wrap(o, out)


class MatMulNBits:
    """src/ops/matmul/contrib.rs:119-195 (com.microsoft MatMulNBits): a [..., M, K] f32 times a 4-bit block-quantized
    b u8 [N, k_blocks, block_size / 2] with f32 scales [N, k_blocks] (or 1-D [N * k_blocks]).  `accuracy_level` 0-4 is
    accepted and, as the reference allows, every level computes in f32: the context's f32 mode for more than 32 rows,
    exact f32 FMAs for up to 32."""

    def __init__(self, bits: int = 4, block_size: int = 32, accuracy_level: int = 0):
        if not 0 <= int(accuracy_level) <= 4:
            raise OpError(5, "accuracy_level must be 0-4")
        self.bits, self.block_size, self.accuracy_level = int(bits), int(block_size), int(accuracy_level)

    def run(self, ctx, a, b, scales, out=None):
        A = _Args(ctx)
        o = A.out(out)
        ctx.check(ctx.lib.rten_b200_matmul_nbits(ctx.handle, A.t(a), A.t(b), A.t(scales), self.bits, self.block_size, C.byref(o)))
        return A.wrap(o, out)


class QuantizedLinear:
    """[LayerNormalization] -> DynamicQuantizeLinear -> Mul -> MatMulIntegerToFloat -> Add(bias) -> Add(residual) -> activation
    as one call (rten_b200_quantized_linear): the skinny-M decode kernel for <= 16 rows, the operator chain otherwise;
    bit-identical to the separate operators either way."""

    def __init__(self, activation: int = ACT_NONE, ln_epsilon: Optional[float] = None):
        self.activation, self.ln_epsilon = activation, ln_epsilon

    def run(self, ctx, x, w, w_scale, packed_w: Optional[Packed] = None, w_zero_point=None, bias=None, residual=None,
            ln_scale=None, ln_bias=None, out=None):
        A = _Args(ctx)
        o = A.out(out)
        ctx.check(ctx.lib.rten_b200_quantized_linear(ctx.handle, A.t(x), A.t(ln_scale), A.t(ln_bias),
                                                     -1.0 if self.ln_epsilon is None else float(self.ln_epsilon), A.t(w), _ph(packed_w),
                                                     A.t(w_zero_point), A.t(w_scale), A.t(bias), A.t(residual), self.activation, C.byref(o)))
        return A.wrap(o, out)


class Attention:
    """src/ops/attention.rs:645-905 (ONNX `Attention`) on 4-D inputs; attributes as the reference's.

    q_seq == 1 runs the decode kernel.  q_seq > 1 with `is_causal`, `nonpad_kv_seqlen` or q_heads != kv_heads runs the
    streaming prefill kernel (device tensors, head size 64 or 128): causal row s attends to keys 0 ..= s + offset, with
    offset = valid - q_seq when `nonpad_kv_seqlen` is given (valid = nonpad_kv_seqlen[b] clamped to [0, total_seq] on
    the device) and 0 otherwise; query head h reads kv head h // (q_heads // kv_heads); fully masked rows are zeros.  Its
    products follow the context's f32 mode (3xTF32 by default, one TF32 pass after `set_f32_mode(False)`)."""

    def __init__(self, is_causal=False, kv_num_heads=None, q_num_heads=None, scale: Optional[float] = None, softcap: float = 0.0):
        self.is_causal, self.kv_num_heads, self.q_num_heads, self.scale, self.softcap = is_causal, kv_num_heads, q_num_heads, scale, softcap

    def run(self, ctx, query, key, value, attn_mask=None, nonpad_kv_seqlen=None, new_key=None, new_value=None, out=None):
        """`new_key` / `new_value`: this step's key / value [batch, kv_heads, 1, head], appended to the caches `key` /
        `value` at position nonpad_kv_seqlen[b] - 1 by the same kernel (q_seq = 1 only)."""
        A = _Args(ctx)
        o = A.out(out)
        p = RtenAttentionParams(int(bool(self.is_causal)), int(self.q_num_heads or 0), int(self.kv_num_heads or 0),
                                float(self.scale) if self.scale else 0.0, float(self.softcap))
        ctx.check(ctx.lib.rten_b200_attention(ctx.handle, A.t(query), A.t(key), A.t(value), A.t(attn_mask), A.t(nonpad_kv_seqlen),
                                              C.byref(p), A.t(new_key), A.t(new_value), C.byref(o)))
        return A.wrap(o, out)


class RotaryEmbedding:
    """src/ops/embedding.rs:209-252 (ai.onnx RotaryEmbedding): input [batch, seq, hidden] (`num_heads` heads) or
    [batch, heads, seq, head]; cos / sin [batch|1, seq|1, dim / 2], or [max_pos, dim / 2] tables gathered by
    `position_ids`.  Rotated values equal a float32 restatement bit for bit (no fused multiply-add)."""

    def __init__(self, interleaved: bool = False, num_heads: int = 0, rotary_embedding_dim: int = 0):
        self.interleaved, self.num_heads, self.rotary_embedding_dim = bool(interleaved), int(num_heads), int(rotary_embedding_dim)

    def run(self, ctx, input, cos, sin, position_ids=None, out=None):
        A = _Args(ctx)
        o = A.out(out)
        ctx.check(ctx.lib.rten_b200_rotary_embedding(ctx.handle, A.t(input), A.t(cos), A.t(sin), A.t(position_ids), int(self.interleaved),
                                                     self.num_heads, self.rotary_embedding_dim, C.byref(o)))
        return A.wrap(o, out)


class GroupQueryAttention:
    """src/ops/attention/contrib.rs:419-810 (com.microsoft GroupQueryAttention); attribute names and defaults as the
    reference's.  Decode steps (one query, not a first prompt) run the single-query attention kernel with the rotary
    embedding and the cache append fused in; prompts run the rotary / append kernel and the streaming prefill kernel."""

    def __init__(self, num_heads: int, kv_num_heads: int, scale: Optional[float] = None, do_rotary: bool = False,
                 rotary_interleaved: bool = False, local_window_size: int = -1, softcap: float = 0.0, smooth_softmax: bool = False):
        self.num_heads, self.kv_num_heads, self.scale = int(num_heads), int(kv_num_heads), scale
        self.do_rotary, self.rotary_interleaved = bool(do_rotary), bool(rotary_interleaved)
        self.local_window_size, self.softcap, self.smooth_softmax = int(local_window_size), float(softcap), bool(smooth_softmax)

    def run(self, ctx, query, key, value, seqlens_k, total_sequence_length, past_key=None, past_value=None, cos_cache=None,
            sin_cache=None, position_ids=None, attention_bias=None, out=None, present_key=None, present_value=None):
        """Returns (output, present_key, present_value).  `key` / `value` None: `query` is packed QKV.  `present_key` /
        `present_value` may be views of the `past_key` / `past_value` buffers (same data pointer and strides, S more
        positions): then only the new tokens are written into them."""
        if self.smooth_softmax:
            raise OpError(6, "smooth_softmax is not supported")
        A = _Args(ctx)
        o, pk, pv = A.out(out), A.out(present_key), A.out(present_value)
        p = RtenGqaParams(self.num_heads, self.kv_num_heads, float(self.scale) if self.scale else 0.0, int(self.do_rotary),
                          int(self.rotary_interleaved), self.local_window_size, self.softcap)
        total = total_sequence_length
        if not isinstance(total, (DeviceTensor, np.ndarray)):
            total = np.asarray(total, np.int32)
        ctx.check(ctx.lib.rten_b200_group_query_attention(
            ctx.handle, A.t(query), A.t(key), A.t(value), A.t(past_key), A.t(past_value), A.t(seqlens_k), A.t(total), A.t(cos_cache),
            A.t(sin_cache), A.t(position_ids), A.t(attention_bias), C.byref(p), C.byref(o), C.byref(pk), C.byref(pv)))
        return A.wrap(o, out), A.wrap(pk, present_key), A.wrap(pv, present_value)


class MultiHeadAttention:
    """src/ops/attention/contrib.rs:43-300 (com.microsoft MultiHeadAttention); attribute names and defaults as the
    reference's.  Masked keys (unidirectional, key_padding_mask) score `mask_filter_value` and stay in the softmax.  One
    query runs the single-query attention kernel, more the streaming prefill kernel; a bias, a past cache or a present
    output adds one launch of the rotary / append kernel before it."""

    def __init__(self, num_heads: int, scale: Optional[float] = None, mask_filter_value: float = -10000.0, unidirectional: bool = False):
        self.num_heads, self.scale = int(num_heads), scale
        self.mask_filter_value, self.unidirectional = float(mask_filter_value), bool(unidirectional)

    def run(self, ctx, query, key=None, value=None, bias=None, key_padding_mask=None, attention_bias=None, past_key=None,
            past_value=None, past_sequence_length=None, cache_indirection=None, out=None, present_key=None, present_value=None,
            want_present: bool = True):
        """Returns (output, present_key, present_value); the present caches are None with `want_present=False`.
        `present_key` / `present_value` may be views of the `past_key` / `past_value` buffers (same data pointer and
        strides, L more positions): then only the new positions are written into them."""
        A = _Args(ctx)
        o = A.out(out)
        pk = A.out(present_key) if want_present else None
        pv = A.out(present_value) if want_present else None
        p = RtenMhaParams(self.num_heads, float(self.scale) if self.scale else 0.0, self.mask_filter_value, int(self.unidirectional))
        ctx.check(ctx.lib.rten_b200_multi_head_attention(
            ctx.handle, A.t(query), A.t(key), A.t(value), A.t(bias), A.t(key_padding_mask), A.t(attention_bias), A.t(past_key),
            A.t(past_value), A.t(past_sequence_length), A.t(cache_indirection), C.byref(p), C.byref(o),
            C.byref(pk) if want_present else None, C.byref(pv) if want_present else None))
        return (A.wrap(o, out), A.wrap(pk, present_key) if want_present else None,
                A.wrap(pv, present_value) if want_present else None)


_RNN_DIRECTIONS = {"forward": 0, "reverse": 1, "bidirectional": 2}


class _Rnn:
    """Shared plumbing of GRU / LSTM (src/ops/rnn.rs).  `direction` is "forward", "reverse" or "bidirectional";
    `hidden_size` is informative (H is read from the weights, as the reference does)."""

    def __init__(self, direction: str = "forward", hidden_size: int = 0):
        if direction not in _RNN_DIRECTIONS:
            raise OpError(5, f"unsupported direction {direction!r}")
        self.direction, self.hidden_size = direction, int(hidden_size)

    def prepack(self, ctx, w) -> Packed:
        """W [dirs, G * H, I] packed for the input projection (the [I, dirs * G * H] matrix the GEMM reads)."""
        wa = np.ascontiguousarray(w.numpy() if isinstance(w, DeviceTensor) else np.asarray(w, np.float32))
        A = _Args(ctx)
        h = C.c_void_p()
        ctx.check(ctx.lib.rten_b200_prepack_b(ctx.handle, A.t(wa.reshape(-1, wa.shape[-1]).T), C.byref(h)))
        return Packed(ctx, h)


class GRU(_Rnn):
    """src/ops/rnn.rs gru: input projection on the wgmma GEMM, the recurrence in one cluster-resident kernel (or one
    launch pair per step for large hidden sizes).  Only linear_before_reset = 1 is supported, as in the reference."""

    def __init__(self, direction: str = "forward", hidden_size: int = 0, linear_before_reset: bool = True):
        super().__init__(direction, hidden_size)
        self.linear_before_reset = bool(linear_before_reset)

    def run(self, ctx, x, w, r, b=None, sequence_lens=None, initial_h=None, packed_w: Optional[Packed] = None,
            outputs=(0, 1)):
        """Returns (Y, Y_h); an output whose index is not in `outputs` is not computed and comes back as None.
        sequence_lens is accepted and ignored, as the reference ignores it."""
        A = _Args(ctx)
        y, yh = A.out(), A.out()
        p = RtenRnnParams(_RNN_DIRECTIONS[self.direction], self.hidden_size, int(self.linear_before_reset))
        ctx.check(ctx.lib.rten_b200_gru(ctx.handle, A.t(x), A.t(w), _ph(packed_w), A.t(r), A.t(b), A.t(sequence_lens),
                                        A.t(initial_h), C.byref(p), C.byref(y) if 0 in outputs else None,
                                        C.byref(yh) if 1 in outputs else None))
        return tuple(A.wrap(o, None) if i in outputs else None for i, o in enumerate((y, yh)))


class LSTM(_Rnn):
    """src/ops/rnn.rs lstm, on the same kernels as GRU.  Peephole weights (input 7) are refused."""

    def run(self, ctx, x, w, r, b=None, sequence_lens=None, initial_h=None, initial_c=None, peephole=None,
            packed_w: Optional[Packed] = None, outputs=(0, 1, 2)):
        """Returns (Y, Y_h, Y_c); outputs not in `outputs` are None.  sequence_lens is accepted and ignored."""
        A = _Args(ctx)
        y, yh, yc = A.out(), A.out(), A.out()
        p = RtenRnnParams(_RNN_DIRECTIONS[self.direction], self.hidden_size, 1)
        ctx.check(ctx.lib.rten_b200_lstm(ctx.handle, A.t(x), A.t(w), _ph(packed_w), A.t(r), A.t(b), A.t(sequence_lens),
                                         A.t(initial_h), A.t(initial_c), A.t(peephole), C.byref(p),
                                         C.byref(y) if 0 in outputs else None, C.byref(yh) if 1 in outputs else None,
                                         C.byref(yc) if 2 in outputs else None))
        return tuple(A.wrap(o, None) if i in outputs else None for i, o in enumerate((y, yh, yc)))


def _conv_params(padding, groups, strides, dilations) -> RtenConvParams:
    p = RtenConvParams()
    if isinstance(padding, str):
        if padding.lower() != "same":
            raise OpError(5, "unknown padding mode")
        p.auto_pad_same = 1
    else:
        pads = list(padding)
        if len(pads) == 2:  # 1-D [start, end]
            pads = [pads[0], pads[1], 0, 0]
        if len(pads) != 4:
            raise OpError(5, "Wrong number of pad values")
        for i in range(4):
            p.pads[i] = int(pads[i])
    p.groups = int(groups)
    p.n_strides = len(strides)
    p.n_dilations = len(dilations)
    for i in range(min(2, len(strides))):
        p.strides[i] = int(strides[i])
    for i in range(min(2, len(dilations))):
        p.dilations[i] = int(dilations[i])
    return p


def _activation(activation) -> RtenActivation:
    """An ACT_* code, or (kind, alpha, beta), as the rten_activation struct.  A bare code takes HardSigmoid's ONNX
    defaults (0.2, 0.5), which the other kinds ignore."""
    kind, alpha, beta = tuple(activation) if isinstance(activation, (tuple, list)) else (activation, 0.2, 0.5)
    return RtenActivation(int(kind), float(alpha), float(beta))


class Conv:
    """src/ops/conv.rs:367-419: attributes groups, dilations, padding ('same' or [t,l,b,r]), strides.  `activation`: an
    ACT_* code or (kind, alpha, beta), applied in the convolution's epilogue (run / run_projected / run_chained take the
    codes ACT_NONE .. ACT_GELU_TANH; run takes every kind)."""

    def __init__(self, groups=1, dilations=(1, 1), padding=(0, 0, 0, 0), strides=(1, 1), activation=ACT_NONE):
        self.groups, self.dilations, self.padding, self.strides = groups, tuple(dilations), padding, tuple(strides)
        self.activation = activation

    def prepack(self, ctx, index, value):
        if index != 1:
            return None
        A = _Args(ctx)
        h = C.c_void_p()
        ctx.check(ctx.lib.rten_b200_prepack_conv_weight(ctx.handle, A.t(value), self.groups, C.byref(h)))
        return Packed(ctx, h)

    def run(self, ctx, x, w, bias=None, packed_w: Optional[Packed] = None, residual=None, out=None):
        A = _Args(ctx)
        o = A.out(out)
        p = _conv_params(self.padding, self.groups, self.strides, self.dilations)
        act = _activation(self.activation)
        ctx.check(ctx.lib.rten_b200_conv2d_act(ctx.handle, A.t(x), A.t(w), _ph(packed_w), A.t(bias), C.byref(p),
                                               A.t(residual), C.byref(act), C.byref(o)))
        return A.wrap(o, out)

    def run_projected(self, ctx, x, w, bias=None, packed_w: Optional[Packed] = None, *, proj: "Conv", x_proj, w_proj,
                      bias_proj=None, packed_w_proj: Optional[Packed] = None, out=None):
        """act(self(x, w, bias) + proj(x_proj, w_proj, bias_proj)) with this op's activation: a residual block's last
        convolution and its projection shortcut (rten_b200_conv2d_projected)."""
        A = _Args(ctx)
        o = A.out(out)
        p = _conv_params(self.padding, self.groups, self.strides, self.dilations)
        pp = _conv_params(proj.padding, proj.groups, proj.strides, proj.dilations)
        ctx.check(ctx.lib.rten_b200_conv2d_projected(ctx.handle, A.t(x), A.t(w), _ph(packed_w), A.t(bias), C.byref(p),
                                                     A.t(x_proj), A.t(w_proj), _ph(packed_w_proj), A.t(bias_proj),
                                                     C.byref(pp), self.activation, C.byref(o)))
        return A.wrap(o, out)

    def run_chained(self, ctx, x, w, bias=None, packed_w: Optional[Packed] = None, residual=None, *, nxt: "Conv", w_next,
                    bias_next=None, packed_w_next: Optional[Packed] = None, proj: Optional["Conv"] = None, x_proj=None,
                    w_proj=None, bias_proj=None, packed_w_proj: Optional[Packed] = None, out=None, out_next=None):
        """(y, z): y = act(self(x, w, bias) [+ residual | + proj(x_proj, w_proj, bias_proj)]) with this op's activation,
        z = nxt(y, w_next, bias_next) with nxt's -- a residual block's last convolution and the next block's first
        (rten_b200_conv2d_chained)."""
        A = _Args(ctx)
        o, o2 = A.out(out), A.out(out_next)
        p = _conv_params(self.padding, self.groups, self.strides, self.dilations)
        pn = _conv_params(nxt.padding, nxt.groups, nxt.strides, nxt.dilations)
        pp = _conv_params(proj.padding, proj.groups, proj.strides, proj.dilations) if proj is not None else None
        ctx.check(ctx.lib.rten_b200_conv2d_chained(ctx.handle, A.t(x), A.t(w), _ph(packed_w), A.t(bias), C.byref(p),
                                                   A.t(residual), A.t(x_proj), A.t(w_proj), _ph(packed_w_proj),
                                                   A.t(bias_proj), C.byref(pp) if pp is not None else None,
                                                   self.activation, A.t(w_next), _ph(packed_w_next), A.t(bias_next),
                                                   C.byref(pn), nxt.activation, C.byref(o), C.byref(o2)))
        return A.wrap(o, out), A.wrap(o2, out_next)


def _conv_transpose_params(padding, groups, strides, dilations, output_padding) -> RtenConvTransposeParams:
    p = RtenConvTransposeParams()
    if isinstance(padding, str):
        if padding.lower() != "same":
            raise OpError(5, "unknown padding mode")
        p.auto_pad_same = 1
    else:
        pads = list(padding)
        p.n_pads = len(pads)
        for i in range(min(4, len(pads))):
            p.pads[i] = int(pads[i])
    p.groups = int(groups)
    for arr, vals, n in ((p.strides, strides, "n_strides"), (p.dilations, dilations, "n_dilations"),
                         (p.output_padding, output_padding or (), "n_output_padding")):
        setattr(p, n, len(vals))
        for i in range(min(2, len(vals))):
            arr[i] = int(vals[i])
    return p


class ConvTranspose:
    """src/ops/conv_transpose.rs:412-440: attributes groups, dilations, padding ('same' or [t, l, b, r]; 1-D: [start,
    end]), strides and output_padding (None: zeros).  Weights are [C_in, C_out / groups, kh, kw] (1-D: [C_in,
    C_out / groups, kw])."""

    def __init__(self, groups=1, dilations=(1, 1), padding=(0, 0, 0, 0), strides=(1, 1), output_padding=None):
        self.groups, self.dilations, self.padding, self.strides = groups, tuple(dilations), padding, tuple(strides)
        self.output_padding = None if output_padding is None else tuple(output_padding)

    def _params(self):
        return _conv_transpose_params(self.padding, self.groups, self.strides, self.dilations, self.output_padding)

    def prepack(self, ctx, index, value):
        """The per-phase sub-kernels of the weight (input 1), built once."""
        if index != 1:
            return None
        A = _Args(ctx)
        h = C.c_void_p()
        p = self._params()
        ctx.check(ctx.lib.rten_b200_prepack_conv_transpose_weight(ctx.handle, A.t(value), C.byref(p), C.byref(h)))
        return Packed(ctx, h)

    def run(self, ctx, x, w, bias=None, packed_w: Optional[Packed] = None, out=None):
        A = _Args(ctx)
        o = A.out(out)
        p = self._params()
        ctx.check(ctx.lib.rten_b200_conv_transpose(ctx.handle, A.t(x), A.t(w), _ph(packed_w), A.t(bias), C.byref(p),
                                                   C.byref(o)))
        return A.wrap(o, out)


class ConvInteger(Conv):
    """src/ops/conv.rs:477-533"""

    def run(self, ctx, x, w, x_zero_point=None, w_zero_point=None, packed_w: Optional[Packed] = None, out=None):
        A = _Args(ctx)
        o = A.out(out)
        p = _conv_params(self.padding, self.groups, self.strides, self.dilations)
        ctx.check(ctx.lib.rten_b200_conv_integer(ctx.handle, A.t(x), A.t(w), _ph(packed_w), A.t(x_zero_point),
                                                 A.t(w_zero_point), None, C.byref(p), C.byref(o)))
        return A.wrap(o, out)


class ConvIntegerToFloat(Conv):
    """src/ops/conv.rs:535-587"""

    def run(self, ctx, x, w, x_zero_point, w_zero_point, scale, packed_w: Optional[Packed] = None, out=None,
            bias=None, residual=None, scale_b=None, out_range=None):
        """`bias` / `residual` / `self.activation` = the Add(bias), Add(identity), Relu nodes that follow the operator in
        a quantised ResNet, executed in the epilogue with the same f32 roundings (rten_b200_conv_integer_ex)."""
        if scale is None:
            raise OpError(4, "missing inputs")
        A = _Args(ctx)
        o = A.out(out)
        p = _conv_params(self.padding, self.groups, self.strides, self.dilations)
        ctx.check(ctx.lib.rten_b200_conv_integer_ex(ctx.handle, A.t(x), A.t(w), _ph(packed_w), A.t(x_zero_point),
                                                    A.t(w_zero_point), A.t(scale), A.t(scale_b), C.byref(p), A.t(bias),
                                                    A.t(residual), self.activation, A.t(out_range), C.byref(o)))
        return A.wrap(o, out)


class Softmax:
    """src/ops/norm.rs:843-899; `in_place` = run_in_place on input 0."""

    def __init__(self, axis=-1, flush_nans_to_zero=False):
        self.axis, self.flush_nans_to_zero = axis, flush_nans_to_zero

    def run(self, ctx, x, in_place=False, out=None):
        A = _Args(ctx)
        into = x if (in_place and isinstance(x, DeviceTensor)) else out
        o = A.out(into)
        ctx.check(ctx.lib.rten_b200_softmax(ctx.handle, A.t(x), None, self.axis, int(self.flush_nans_to_zero), C.byref(o)))
        return A.wrap(o, into)


class AddSoftmax:
    """src/ops/attention.rs:72-165: the larger input is QK; the other is broadcast to it."""

    def __init__(self, flush_nans_to_zero=False):
        self.flush_nans_to_zero = flush_nans_to_zero

    def run(self, ctx, x, y, in_place=False):
        nx = x.size if isinstance(x, DeviceTensor) else np.asarray(x).size
        ny = y.size if isinstance(y, DeviceTensor) else np.asarray(y).size
        qk, m = (x, y) if nx > ny else (y, x)
        A = _Args(ctx)
        into = qk if (in_place and isinstance(qk, DeviceTensor)) else None
        o = A.out(into)
        ctx.check(ctx.lib.rten_b200_softmax(ctx.handle, A.t(qk), A.t(m), -1, int(self.flush_nans_to_zero), C.byref(o)))
        return A.wrap(o, into)


class LayerNormalization:
    """src/ops/norm.rs:531-569"""

    def __init__(self, axis=-1, epsilon: Optional[float] = None):
        self.axis, self.epsilon = axis, epsilon

    def run(self, ctx, x, scale, bias=None, out=None):
        A = _Args(ctx)
        o = A.out(out)
        ctx.check(ctx.lib.rten_b200_layer_norm(ctx.handle, A.t(x), A.t(scale), A.t(bias), self.axis,
                                               -1.0 if self.epsilon is None else float(self.epsilon), C.byref(o)))
        return A.wrap(o, out)


class RMSNormalization:
    """src/ops/norm.rs rms_normalization: LayerNormalization without centring, rstd = scale / sqrt(mean(x^2) + epsilon)"""

    def __init__(self, axis=-1, epsilon: Optional[float] = None):
        self.axis, self.epsilon = axis, epsilon

    def run(self, ctx, x, scale, out=None):
        A = _Args(ctx)
        o = A.out(out)
        ctx.check(ctx.lib.rten_b200_rms_norm(ctx.handle, A.t(x), A.t(scale), self.axis,
                                             -1.0 if self.epsilon is None else float(self.epsilon), C.byref(o)))
        return A.wrap(o, out)


class SimplifiedLayerNormalization(RMSNormalization):
    """src/ops/norm/contrib.rs: ONNX Runtime's name for RMSNormalization"""


class SkipLayerNormalization:
    """src/ops/norm/contrib.rs (com.microsoft): LayerNormalization of (x + skip) + bias over the last axis.
    `run(..., want_sum=True)` also returns that sum (the operator's output 3, input_skip_bias_sum)."""

    _rms = 0

    def __init__(self, epsilon: float):
        self.epsilon = float(epsilon)

    def _run(self, ctx, x, skip, gamma, beta, bias, want_sum):
        A = _Args(ctx)
        o = A.out()
        s = A.out() if want_sum else None
        ctx.check(ctx.lib.rten_b200_skip_layer_norm(ctx.handle, A.t(x), A.t(skip), A.t(gamma), A.t(beta), A.t(bias),
                                                    self.epsilon, self._rms, C.byref(o), C.byref(s) if want_sum else None))
        return (A.wrap(o, None), A.wrap(s, None)) if want_sum else A.wrap(o, None)

    def run(self, ctx, x, skip, gamma, beta=None, bias=None, want_sum=False):
        return self._run(ctx, x, skip, gamma, beta, bias, want_sum)


class SkipSimplifiedLayerNormalization(SkipLayerNormalization):
    """src/ops/norm/contrib.rs (com.microsoft): RMSNormalization of (x + skip) + bias over the last axis (no beta)."""

    _rms = 1

    def run(self, ctx, x, skip, gamma, bias=None, want_sum=False):
        return self._run(ctx, x, skip, gamma, None, bias, want_sum)


class InstanceNormalization:
    """src/ops/norm.rs instance_normalization: each (n, c) lane normalised over its spatial elements, scale / bias [C].
    `run(..., out=x)` normalises in place."""

    def __init__(self, epsilon: Optional[float] = None):
        self.epsilon = epsilon

    def run(self, ctx, x, scale, bias, out=None):
        A = _Args(ctx)
        o = A.out(out)
        ctx.check(ctx.lib.rten_b200_instance_norm(ctx.handle, A.t(x), A.t(scale), A.t(bias),
                                                  -1.0 if self.epsilon is None else float(self.epsilon), C.byref(o)))
        return A.wrap(o, out)


class GroupNorm:
    """torch's exported GroupNorm chain in one pass: Reshape [N, groups, -1] -> InstanceNormalization(inst_scale,
    inst_bias) -> Reshape back -> Mul(gamma) -> Add(beta) -> activation (an ACT_* code or (kind, alpha, beta)), each step
    rounded as the node chain rounds it (rten_b200_group_norm)."""

    def __init__(self, groups: int, epsilon: Optional[float] = None, activation=ACT_NONE):
        self.groups, self.epsilon, self.activation = int(groups), epsilon, activation

    def run(self, ctx, x, inst_scale, inst_bias, gamma=None, beta=None, out=None):
        A = _Args(ctx)
        o = A.out(out)
        act = _activation(self.activation)
        ctx.check(ctx.lib.rten_b200_group_norm(ctx.handle, A.t(x), self.groups, A.t(inst_scale), A.t(inst_bias), A.t(gamma),
                                               A.t(beta), -1.0 if self.epsilon is None else float(self.epsilon), C.byref(act),
                                               C.byref(o)))
        return A.wrap(o, out)


class BatchNormalization:
    """src/ops/norm.rs batch_norm: y = fma(x - mean[c], scale[c] / sqrt(var[c] + epsilon), bias[c]) over channel axis 1
    (a rank-1 x is one channel), then the activation (an ACT_* code or (kind, alpha, beta)); rten_b200_batch_norm.
    `run(..., out=x)` normalises in place."""

    def __init__(self, epsilon: Optional[float] = None, activation=ACT_NONE):
        self.epsilon, self.activation = epsilon, activation

    def run(self, ctx, x, scale, bias, mean, var, out=None):
        A = _Args(ctx)
        o = A.out(out)
        act = _activation(self.activation)
        ctx.check(ctx.lib.rten_b200_batch_norm(ctx.handle, A.t(x), A.t(scale), A.t(bias), A.t(mean), A.t(var),
                                               -1.0 if self.epsilon is None else float(self.epsilon), C.byref(act),
                                               C.byref(o)))
        return A.wrap(o, out)


class _Unary:
    fn = ""

    def run(self, ctx, x, in_place=False, out=None):
        A = _Args(ctx)
        into = x if (in_place and isinstance(x, DeviceTensor)) else out
        o = A.out(into)
        ctx.check(self._call(ctx, A.t(x), C.byref(o)))
        return A.wrap(o, into)


class Erf(_Unary):
    """src/ops/unary_elementwise.rs:384-387"""

    def _call(self, ctx, x, o):
        return ctx.lib.rten_b200_erf(ctx.handle, x, o)


class Gelu(_Unary):
    """src/ops/unary_elementwise.rs:399-435"""

    def __init__(self, approximate=False):
        self.approximate = approximate

    def _call(self, ctx, x, o):
        return ctx.lib.rten_b200_gelu(ctx.handle, x, int(self.approximate), o)


class Relu(_Unary):
    def _call(self, ctx, x, o):
        return ctx.lib.rten_b200_relu(ctx.handle, x, o)


class Sigmoid(_Unary):
    """rten-vecmath/src/exp.rs:201-212: 1 / (1 + exp(0 - x))"""

    def _call(self, ctx, x, o):
        return ctx.lib.rten_b200_sigmoid(ctx.handle, x, o)


class Silu(_Unary):
    """exp.rs:217-228: x / (1 + exp(0 - x)), one division -- what the reference runs for Mul(x, Sigmoid(x))"""

    def _call(self, ctx, x, o):
        return ctx.lib.rten_b200_silu(ctx.handle, x, o)


class HardSigmoid(_Unary):
    """src/ops/unary_elementwise.rs:437-449: clamp(alpha * x + beta, 0, 1)"""

    def __init__(self, alpha=0.2, beta=0.5):
        self.alpha, self.beta = alpha, beta

    def _call(self, ctx, x, o):
        return ctx.lib.rten_b200_hard_sigmoid(ctx.handle, x, float(self.alpha), float(self.beta), o)


class HardSwish(_Unary):
    """src/ops/unary_elementwise.rs:457-469: x * clamp(x / 6 + 0.5, 0, 1)"""

    def _call(self, ctx, x, o):
        return ctx.lib.rten_b200_hard_swish(ctx.handle, x, o)


class Sqrt(_Unary):
    """src/ops/unary_elementwise.rs:743-745: IEEE square root (f32)"""

    def _call(self, ctx, x, o):
        return ctx.lib.rten_b200_sqrt(ctx.handle, x, o)


class Reciprocal(_Unary):
    """src/ops/unary_elementwise.rs:607-609: 1 / x, IEEE (f32)"""

    def _call(self, ctx, x, o):
        return ctx.lib.rten_b200_reciprocal(ctx.handle, x, o)


class Exp(_Unary):
    """rten-vecmath/src/exp.rs Exp (f32): inf from 104 on, 0 from -104 down"""

    def _call(self, ctx, x, o):
        return ctx.lib.rten_b200_exp(ctx.handle, x, o)


class Tanh(_Unary):
    """rten-vecmath/src/tanh.rs Tanh (f32)"""

    def _call(self, ctx, x, o):
        return ctx.lib.rten_b200_tanh(ctx.handle, x, o)


class Neg(_Unary):
    """src/ops/unary_elementwise.rs:550-555: -x, the sign bit flipped (f32)"""

    def _call(self, ctx, x, o):
        return ctx.lib.rten_b200_neg(ctx.handle, x, o)


class Abs(_Unary):
    """src/ops/unary_elementwise.rs:195-220: the sign bit cleared (f32)"""

    def _call(self, ctx, x, o):
        return ctx.lib.rten_b200_abs(ctx.handle, x, o)


class Clip:
    """src/ops/unary_elementwise.rs:249-333: x.max(min).min(max), f32 or i32; `min` / `max` are scalars of x's type (or
    None: the type's finite extreme), read on the device.  `in_place` = run_in_place on input 0."""

    def run(self, ctx, x, min=None, max=None, in_place=False, out=None):
        A = _Args(ctx)
        into = x if (in_place and isinstance(x, DeviceTensor)) else out
        o = A.out(into)
        ctx.check(ctx.lib.rten_b200_clip(ctx.handle, A.t(x), A.t(min), A.t(max), C.byref(o)))
        return A.wrap(o, into)


class DynamicQuantizeLinear:
    """src/ops/quantize.rs:436-468 -> (y u8, y_scale f32 scalar, y_zero_point u8 scalar)"""

    def run(self, ctx, x, comm: Optional["Comm"] = None, value_range=None, out=None):
        """`comm`: batch-sharded run -- the quantisation range is all-reduced over the ranks (min, max) first.
        `value_range`: i32[2] device tensor filled by the producer of x (`out_range=` of the *IntegerToFloat operators):
        the operator then skips its own min / max pass.  `out`: u8 destination view, e.g. the interior of a spatially
        pre-padded channels-last buffer (rows at arbitrary pitches)."""
        A = _Args(ctx)
        y, s, z = A.out(out), A.out(), A.out()
        ctx.check(ctx.lib.rten_b200_dynamic_quantize_linear_ranged(ctx.handle, A.t(x), A.t(value_range), C.byref(y), C.byref(s),
                                                                   C.byref(z), comm.handle if comm is not None else None))
        return A.wrap(y, out), A.wrap(s, None), A.wrap(z, None)

    @staticmethod
    def reset_ranges(ctx, ranges: "DeviceTensor"):
        """Re-arm a [n, 2] i32 tensor of producer-computed ranges (one launch) before the producers run."""
        d = ranges.desc()
        ctx.check(ctx.lib.rten_b200_range_reset(ctx.handle, C.byref(d)))


class Comm:
    """Cross-rank communicator of a batch-sharded run (rten_b200_comm_*; NCCL resolved at run time)."""

    def __init__(self, ctx: Context, unique_id: bytes, rank: int, world: int):
        assert len(unique_id) == 128
        self.ctx, self.rank, self.world = ctx, rank, world
        h = C.c_void_p()
        buf = C.create_string_buffer(unique_id, 128)
        ctx.check(ctx.lib.rten_b200_comm_create(ctx.handle, buf, rank, world, C.byref(h)))
        self.handle = h

    @staticmethod
    def unique_id() -> bytes:
        buf = C.create_string_buffer(128)
        st = _lib.load().rten_b200_comm_unique_id(buf)
        if st != 0:
            raise OpError(st, "libnccl.so.2 could not be loaded")
        return buf.raw

    @property
    def uses_peer_memory(self) -> bool:
        """True: quantisation ranges travel through NVLink peer mailboxes (one kernel per exchange); False: NCCL."""
        return bool(self.ctx.lib.rten_b200_comm_uses_peer_memory(self.handle))

    def timeouts(self) -> int:
        return int(self.ctx.lib.rten_b200_comm_timeouts(self.handle))

    def close(self):
        if getattr(self, "handle", None):
            self.ctx.lib.rten_b200_comm_destroy(self.handle)
            self.handle = None


class Add:
    def run(self, ctx, a, b, out=None):
        A = _Args(ctx)
        o = A.out(out)
        ctx.check(ctx.lib.rten_b200_add(ctx.handle, A.t(a), A.t(b), C.byref(o)))
        return A.wrap(o, out)


class Mul:
    """src/ops/binary_elementwise.rs Mul (f32, broadcasting)."""

    def run(self, ctx, a, b, out=None):
        A = _Args(ctx)
        o = A.out(out)
        ctx.check(ctx.lib.rten_b200_mul(ctx.handle, A.t(a), A.t(b), C.byref(o)))
        return A.wrap(o, out)


class Sub:
    """src/ops/binary_elementwise.rs Sub (f32 or wrapping i32, broadcasting)."""

    def run(self, ctx, a, b, out=None):
        A = _Args(ctx)
        o = A.out(out)
        ctx.check(ctx.lib.rten_b200_sub(ctx.handle, A.t(a), A.t(b), C.byref(o)))
        return A.wrap(o, out)


class Div:
    """src/ops/binary_elementwise.rs:600-638 Div (f32, or truncating i32 that refuses a zero divisor and INT_MIN / -1,
    broadcasting).  A one-element f32 divisor is a * (1 / b), with a's shape."""

    def run(self, ctx, a, b, out=None):
        A = _Args(ctx)
        o = A.out(out)
        ctx.check(ctx.lib.rten_b200_div(ctx.handle, A.t(a), A.t(b), C.byref(o)))
        return A.wrap(o, out)


class Pow:
    """src/ops/binary_elementwise.rs:965-1029 Pow (FastPow; f32 ^ f32 or i32 ^ i32, broadcasting).  A one-element
    exponent maps the base (a's shape)."""

    def run(self, ctx, a, b, out=None):
        A = _Args(ctx)
        o = A.out(out)
        ctx.check(ctx.lib.rten_b200_pow(ctx.handle, A.t(a), A.t(b), C.byref(o)))
        return A.wrap(o, out)


class Where:
    """src/ops/binary_elementwise.rs where_op: cond (i32, nonzero is true) ? x : y, the three broadcast together; x and y
    both f32 or both i32."""

    def run(self, ctx, cond, x, y, out=None):
        A = _Args(ctx)
        o = A.out(out)
        ctx.check(ctx.lib.rten_b200_where(ctx.handle, A.t(cond), A.t(x), A.t(y), C.byref(o)))
        return A.wrap(o, out)


class _Compare:
    """binary_elementwise.rs boolean_op / logical_boolean_op: i32 0 / 1 of a (op) b, broadcasting.  The comparisons take
    f32 or i32 (IEEE: NaN compares false, -0 == +0), the logical operators i32 with nonzero as true."""
    _fn = ""

    def run(self, ctx, a, b, out=None):
        A = _Args(ctx)
        o = A.out(out)
        ctx.check(getattr(ctx.lib, self._fn)(ctx.handle, A.t(a), A.t(b), C.byref(o)))
        return A.wrap(o, out)


class Equal(_Compare):
    _fn = "rten_b200_equal"


class Less(_Compare):
    _fn = "rten_b200_less"


class LessOrEqual(_Compare):
    _fn = "rten_b200_less_or_equal"


class Greater(_Compare):
    _fn = "rten_b200_greater"


class GreaterOrEqual(_Compare):
    _fn = "rten_b200_greater_or_equal"


class And(_Compare):
    _fn = "rten_b200_and"


class Or(_Compare):
    _fn = "rten_b200_or"


class Xor(_Compare):
    _fn = "rten_b200_xor"


class Not:
    """src/ops/unary_elementwise.rs not: i32 1 where x == 0, else 0."""

    def run(self, ctx, x, out=None):
        A = _Args(ctx)
        o = A.out(out)
        ctx.check(ctx.lib.rten_b200_not(ctx.handle, A.t(x), C.byref(o)))
        return A.wrap(o, out)


class Trilu:
    """src/ops/trilu.rs: the upper (or lower) triangle of every matrix over the last two dims, shifted by k; f32 or i32."""

    def __init__(self, upper: bool = True):
        self.upper = bool(upper)

    def run(self, ctx, x, k: int = 0, out=None):
        A = _Args(ctx)
        o = A.out(out)
        ctx.check(ctx.lib.rten_b200_trilu(ctx.handle, A.t(x), int(k), int(self.upper), C.byref(o)))
        return A.wrap(o, out)


def _ints(ctype, v):
    return None if v is None else (ctype * max(len(v), 1))(*[int(i) for i in v])


class Expand:
    """src/ops/layout.rs expand: x (f32 or i32) broadcast bidirectionally with the target `shape`."""

    def run(self, ctx, x, shape, out=None):
        A = _Args(ctx)
        o = A.out(out)
        ctx.check(ctx.lib.rten_b200_expand(ctx.handle, A.t(x), _ints(C.c_int64, shape), len(shape), C.byref(o)))
        return A.wrap(o, out)


class Slice:
    """src/ops/slice.rs slice, copied: starts / ends (and axes, steps when given) of equal length; positive steps only."""

    def run(self, ctx, x, starts, ends, axes=None, steps=None, out=None):
        A = _Args(ctx)
        o = A.out(out)
        ctx.check(ctx.lib.rten_b200_slice(ctx.handle, A.t(x), _ints(C.c_int32, starts), _ints(C.c_int32, ends), _ints(C.c_int32, axes),
                                          _ints(C.c_int32, steps), len(starts), C.byref(o)))
        return A.wrap(o, out)


class Split:
    """src/ops/split.rs split, copied: by `split` sizes when given, else into num_outputs pieces of ceil(n / k)."""

    def __init__(self, axis: int = 0, num_outputs: Optional[int] = None):
        self.axis, self.num_outputs = int(axis), num_outputs

    def run(self, ctx, x, split=None, num_outputs: Optional[int] = None):
        A = _Args(ctx)
        k = num_outputs if num_outputs is not None else self.num_outputs
        cap = len(split) if split is not None else int(k or 0)
        outs = (RtenTensor * max(cap, 1))()
        A.keep.append(outs)
        n = C.c_int32(0)
        ctx.check(ctx.lib.rten_b200_split(ctx.handle, A.t(x), self.axis, _ints(C.c_int32, split), len(split) if split is not None else 0,
                                          int(k or 0), outs, cap, C.byref(n)))
        return [A.wrap(outs[i], None) for i in range(n.value)]


TOPK_MAX_K = 2048  # the largest k rten_b200_topk takes (RTEN_ERR_UNSUPPORTED_VALUE above)


class TopK:
    """src/ops/reduce.rs topk (f32 or i32): the k largest (or smallest) elements along `axis` and their i32 indices,
    best first, ties by ascending index; NaN is above every number in both directions, -0.0 equals +0.0.  The output is
    always sorted (`sorted` is accepted for the ONNX attribute).  k <= TOPK_MAX_K."""

    def __init__(self, axis: int = -1, largest: bool = True, sorted: bool = True):
        self.axis, self.largest, self.sorted = int(axis), bool(largest), bool(sorted)

    def run(self, ctx, x, k: int, values_out=None, indices_out=None):
        A = _Args(ctx)
        v, i = A.out(values_out), A.out(indices_out)
        ctx.check(ctx.lib.rten_b200_topk(ctx.handle, A.t(x), int(k), self.axis, int(self.largest), int(self.sorted),
                                         C.byref(v), C.byref(i)))
        return A.wrap(v, values_out), A.wrap(i, indices_out)


class ArgMax:
    """src/ops/reduce.rs arg_max (f32 or i32 -> i32): the first NaN's index, else the last maximum's."""
    _fn = "rten_b200_arg_max"

    def __init__(self, axis: int = 0, keep_dims: bool = True):
        self.axis, self.keep_dims = int(axis), bool(keep_dims)

    def run(self, ctx, x, out=None):
        A = _Args(ctx)
        o = A.out(out)
        ctx.check(getattr(ctx.lib, self._fn)(ctx.handle, A.t(x), self.axis, int(self.keep_dims), C.byref(o)))
        return A.wrap(o, out)


class ArgMin(ArgMax):
    """src/ops/reduce.rs arg_min (f32 or i32 -> i32): the first NaN's index, else the last minimum's."""
    _fn = "rten_b200_arg_min"


class ReduceSum:
    """src/ops/reduce.rs ReduceSum (f32 or wrapping i32): axes None or empty reduces every axis, unless
    noop_with_empty_axes, which makes it a copy."""

    def __init__(self, axes=None, keep_dims: bool = True, noop_with_empty_axes: bool = False):
        self.axes = None if axes is None else [int(a) for a in axes]
        self.keep_dims, self.noop_with_empty_axes = keep_dims, noop_with_empty_axes

    def run(self, ctx, x, out=None):
        if not self.axes and self.noop_with_empty_axes:
            src = x if isinstance(x, DeviceTensor) else ctx.to_device(np.asarray(x))
            y = out if out is not None else ctx.empty(src.shape, src.dtype)
            y.assign(src)
            return y
        A = _Args(ctx)
        o = A.out(out)
        ax = (C.c_int32 * max(len(self.axes or []), 1))(*(self.axes or []))
        ctx.check(ctx.lib.rten_b200_reduce_sum(ctx.handle, A.t(x), ax, len(self.axes or []), int(self.keep_dims), C.byref(o)))
        return A.wrap(o, out)


class ReduceMean(ReduceSum):
    """src/ops/reduce.rs:524-541 ReduceMean (f32): each lane's ReduceSum divided by its length; an empty lane is NaN"""

    def run(self, ctx, x, out=None):
        if not self.axes and self.noop_with_empty_axes:
            return super().run(ctx, x, out)
        A = _Args(ctx)
        o = A.out(out)
        ax = (C.c_int32 * max(len(self.axes or []), 1))(*(self.axes or []))
        ctx.check(ctx.lib.rten_b200_reduce_mean(ctx.handle, A.t(x), ax, len(self.axes or []), int(self.keep_dims), C.byref(o)))
        return A.wrap(o, out)


class MaxPool:
    """src/ops/pooling.rs MaxPool: kernel_size, padding [t,l,b,r], strides."""

    def __init__(self, kernel_size, padding=(0, 0, 0, 0), strides=(1, 1)):
        self.kernel_size, self.padding, self.strides = tuple(kernel_size), tuple(padding), tuple(strides)

    def run(self, ctx, x, out=None):
        A = _Args(ctx)
        o = A.out(out)
        k = (C.c_int32 * 2)(*self.kernel_size)
        p = (C.c_int32 * 4)(*self.padding)
        s = (C.c_int32 * 2)(*self.strides)
        ctx.check(ctx.lib.rten_b200_max_pool(ctx.handle, A.t(x), k, p, s, C.byref(o)))
        return A.wrap(o, out)


class AveragePool:
    """src/ops/pooling.rs AveragePool: kernel_size, padding [t,l,b,r], strides, count_include_pad."""

    def __init__(self, kernel_size, padding=(0, 0, 0, 0), strides=(1, 1), count_include_pad=False):
        self.kernel_size, self.padding, self.strides = tuple(kernel_size), tuple(padding), tuple(strides)
        self.count_include_pad = bool(count_include_pad)

    def run(self, ctx, x, out=None):
        A = _Args(ctx)
        o = A.out(out)
        k = (C.c_int32 * 2)(*self.kernel_size)
        p = (C.c_int32 * 4)(*self.padding)
        s = (C.c_int32 * 2)(*self.strides)
        ctx.check(ctx.lib.rten_b200_average_pool(ctx.handle, A.t(x), k, p, s, int(self.count_include_pad), C.byref(o)))
        return A.wrap(o, out)


RESIZE_MODES = {"nearest": 0, "linear": 1}
RESIZE_COORD_MODES = {"half_pixel": 0, "asymmetric": 1, "align_corners": 2, "pytorch_half_pixel": 3}
RESIZE_NEAREST_MODES = {"floor": 0, "ceil": 1, "round_prefer_floor": 2, "round_prefer_ceil": 3}


class Resize:
    """src/ops/resize.rs Resize: `scales` or `sizes`, one value per input axis (the ONNX defaults: nearest, half_pixel,
    round_prefer_floor)."""

    def __init__(self, mode="nearest", coord_mode="half_pixel", nearest_mode="round_prefer_floor"):
        self.mode, self.coord_mode, self.nearest_mode = mode, coord_mode, nearest_mode

    def run(self, ctx, x, scales=None, sizes=None, out=None):
        if scales is None and sizes is None:
            raise OpError(4, "missing inputs")
        A = _Args(ctx)
        o = A.out(out)
        p = RtenResizeParams()
        p.mode = RESIZE_MODES[self.mode]
        p.coord_mode = RESIZE_COORD_MODES[self.coord_mode]
        p.nearest_mode = RESIZE_NEAREST_MODES[self.nearest_mode]
        target = list(scales if scales is not None else sizes)
        p.n = len(target)
        p.use_sizes = int(scales is None)
        for i, v in enumerate(target[:4]):
            if scales is not None:
                p.scales[i] = float(v)
            else:
                p.sizes[i] = int(v)
        ctx.check(ctx.lib.rten_b200_resize(ctx.handle, A.t(x), C.byref(p), C.byref(o)))
        return A.wrap(o, out)


class Upsample(Resize):
    """src/ops/resize.rs:616-643 Upsample: Resize by scales with the asymmetric transform and floor rounding."""

    def __init__(self, mode="nearest"):
        super().__init__(mode, "asymmetric", "floor")

    def run(self, ctx, x, scales, out=None):
        return super().run(ctx, x, scales=scales, out=out)


class Concat:
    """src/ops/concat.rs Concat along `axis`."""

    def __init__(self, axis):
        self.axis = int(axis)

    def run(self, ctx, inputs, out=None):
        A = _Args(ctx)
        o = A.out(out)
        refs = [A.t(t) for t in inputs]
        arr = (C.POINTER(RtenTensor) * max(len(refs), 1))(*[C.cast(r, C.POINTER(RtenTensor)) for r in refs])
        ctx.check(ctx.lib.rten_b200_concat(ctx.handle, arr, len(refs), self.axis, C.byref(o)))
        return A.wrap(o, out)


class GlobalAveragePool:
    def run(self, ctx, x, out=None):
        A = _Args(ctx)
        o = A.out(out)
        ctx.check(ctx.lib.rten_b200_global_average_pool(ctx.handle, A.t(x), C.byref(o)))
        return A.wrap(o, out)


class ScatterRows:
    """table[indices[r], :] = updates[r, :] in place (2-D f32 table, distinct i32 indices)."""

    def run(self, ctx, table: "DeviceTensor", indices, updates):
        A = _Args(ctx)
        t = table.desc()
        ctx.check(ctx.lib.rten_b200_scatter_rows(ctx.handle, C.byref(t), A.t(indices), A.t(updates)))
        return table


class GatherRows:
    """Gather(axis=0) of a 2-D table with i32 indices (embedding lookup; src/ops/gather.rs)."""

    def run(self, ctx, table, indices, out=None):
        A = _Args(ctx)
        o = A.out(out)
        ctx.check(ctx.lib.rten_b200_gather_rows(ctx.handle, A.t(table), A.t(indices), C.byref(o)))
        return A.wrap(o, out)
