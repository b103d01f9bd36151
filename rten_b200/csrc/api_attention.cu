// Attention entry points of the C ABI (include/rten_b200.h):
//   rten_b200_attention               : the reference's `Attention` operator (src/ops/attention.rs:645-905) on 4-D inputs
//   rten_b200_rotary_embedding        : ai.onnx RotaryEmbedding (src/ops/embedding.rs:46-252)
//   rten_b200_group_query_attention   : com.microsoft GroupQueryAttention (src/ops/attention/contrib.rs:369-417,
//                                       :438-810), the attention operator of quantized decoder-only LLM exports
//   rten_b200_multi_head_attention    : com.microsoft MultiHeadAttention (src/ops/attention/contrib.rs:56-300), the
//                                       attention of ONNX Runtime's optimized encoder and encoder-decoder exports
// Validation restates the reference's checks and messages on everything the host can see.  The work runs on four
// kernels: the single-query attention kernel for a decode step (skinny.cu, with GroupQueryAttention's rotary embedding,
// cache append and sliding window fused in), the streaming prefill kernel (attn_prefill.cu) for prompts, the fused
// encoder kernel (attn_fused.cu) and the rotary / cache-append kernel (rotary.cu).  Attention composes this library's
// MatMul and Softmax for the calls none of them serves.  Every launch is filled in from head-row views (RotaryRows) of
// its operands.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstring>
#include <string>
#include <vector>

#include "api_util.h"
#include "attn_fused.h"
#include "attn_prefill.h"
#include "rotary.h"
#include "skinny.h"

using namespace rtb;

namespace {

// ---- head-row views: element (b, s, h, i) of an operand, s a query or key position

// [b, s, h, d] head rows of a [B, S, heads * D] tensor (head h at columns h * D ..), starting at head h0
RotaryRows rows3(const rten_tensor* t, int64_t D, int64_t h0) {
    RotaryRows r;
    r.p = (float*)t->data + h0 * D * t->strides[2];
    r.sb = t->strides[0];
    r.ss = t->strides[1];
    r.sh = D * t->strides[2];
    r.sd = t->strides[2];
    return r;
}

// a [B, heads, T, D] tensor (a cache, or Attention's q / k / v / output) as rows indexed (b, t, h)
RotaryRows cache_rows(const rten_tensor* t) {
    RotaryRows r;
    r.p = (float*)t->data;
    r.sb = t->strides[0];
    r.ss = t->strides[2];
    r.sh = t->strides[1];
    r.sd = t->strides[3];
    return r;
}

// component c (0 = q, 1 = k, 2 = v) of a packed [B, S, heads, 3, D] tensor
RotaryRows packed_rows(const rten_tensor* t, int c) {
    RotaryRows r;
    r.p = (float*)t->data + c * t->strides[3];
    r.sb = t->strides[0];
    r.ss = t->strides[1];
    r.sh = t->strides[2];
    r.sd = t->strides[4];
    return r;
}

// dense scratch: [B, S, heads, D], or [B, heads, S, D] (a cache) when `heads_outer`
RotaryRows dense_rows(void* p, int64_t S, int64_t heads, int64_t D, bool heads_outer) {
    RotaryRows r;
    r.p = (float*)p;
    r.sb = S * heads * D;
    r.ss = heads_outer ? D : heads * D;
    r.sh = heads_outer ? S * D : D;
    return r;
}

// ---- launch parts built from views

// rows of n positions as the (d, s, h, b) operand of a TMA map (head dimension contiguous)
OperandDesc operand(const RotaryRows& r, int64_t D, int64_t n, int64_t heads, int64_t B) {
    OperandDesc d;
    d.base = r.p;
    d.dims[0] = D;
    d.dims[1] = n;
    d.dims[2] = heads;
    d.dims[3] = B;
    d.strides[1] = r.ss;
    d.strides[2] = r.sh;
    d.strides[3] = r.sb;
    return d;
}

// a 4-D [b, h, s, d] value tensor stored transposed (key dimension contiguous) as the (s, d, h, b) operand of a TMA map
OperandDesc transposed_operand(const rten_tensor* t) {
    OperandDesc d;
    d.base = t->data;
    d.dims[0] = t->shape[2];
    d.dims[1] = t->shape[3];
    d.dims[2] = t->shape[1];
    d.dims[3] = t->shape[0];
    d.strides[1] = t->strides[3];
    d.strides[2] = t->strides[1];
    d.strides[3] = t->strides[0];
    return d;
}

// a single-query launch: q rows (b, 0, h), k / v caches of `cap` positions as rows (b, l, kv_h)
AttnDecodeLaunch decode_launch(int64_t B, int64_t qh, int64_t kvh, int64_t D, int64_t cap, const RotaryRows& q, const RotaryRows& k,
                               const RotaryRows& v) {
    AttnDecodeLaunch L;
    L.B = (int)B;
    L.q_heads = (int)qh;
    L.kv_heads = (int)kvh;
    L.dh = (int)D;
    L.kv_cap = (int)cap;
    L.q = q.p;
    L.q_b = q.sb;
    L.q_h = q.sh;
    L.k = k.p;
    L.k_b = k.sb;
    L.k_h = k.sh;
    L.k_l = k.ss;
    L.v = v.p;
    L.v_b = v.sb;
    L.v_h = v.sh;
    L.v_l = v.ss;
    L.v_d = v.sd;
    return L;
}

void decode_out(AttnDecodeLaunch& L, const RotaryRows& o) {
    L.out = o.p;
    L.o_b = o.sb;
    L.o_h = o.sh;
}

// q, k and the output of a streaming launch (the prefill or the fused encoder kernel): S queries over T keys
template <class Launch>
void stream_io(Launch& A, int64_t B, int64_t qh, int64_t kvh, int64_t S, int64_t T, int64_t D, const RotaryRows& q, const RotaryRows& k,
               const RotaryRows& o) {
    A.B = (int)B;
    A.q_seq = (int)S;
    A.kv_seq = (int)T;
    A.dh = (int)D;
    A.q = operand(q, D, S, qh, B);
    A.k = operand(k, D, T, kvh, B);
    A.out = o.p;
    A.o_b = o.sb;
    A.o_h = o.sh;
    A.o_s = o.ss;
}

// a prefill launch in the context's f32 mode, the value rows in their natural layout
AttnPrefillLaunch prefill_launch(rten_ctx* ctx, int64_t B, int64_t qh, int64_t kvh, int64_t S, int64_t T, int64_t D, float scale,
                                 const RotaryRows& q, const RotaryRows& k, const RotaryRows& v, const RotaryRows& o) {
    AttnPrefillLaunch A;
    stream_io(A, B, qh, kvh, S, T, D, q, k, o);
    A.q_heads = (int)qh;
    A.kv_heads = (int)kvh;
    A.v = operand(v, D, T, kvh, B);
    A.scale = scale;
    A.x3 = ctx->f32_mode == RTEN_F32_TF32 ? 0 : 1;
    return A;
}

long long bstride(const rten_tensor* t, int i) { return t->shape[i] == 1 ? 0 : t->strides[i]; }

// the (b, h, s, t) element strides of a 4-D additive mask, 0 on its size-1 (broadcast) dimensions; all 0 without one
void mask_strides(const rten_tensor* m, long long* ms) {
    for (int i = 0; i < 4; i++) ms[i] = m ? bstride(m, i) : 0;
}

void set_mask(AttnDecodeLaunch& L, const rten_tensor* m, const long long* ms) {
    L.mask = m ? (const float*)m->data : nullptr;
    L.m_b = ms[0];
    L.m_h = ms[1];
    L.m_l = ms[3];
}

void set_mask(AttnPrefillLaunch& A, const rten_tensor* m, const long long* ms) {
    A.mask = m ? (const float*)m->data : nullptr;
    A.m_b = ms[0];
    A.m_h = ms[1];
    A.m_s = ms[2];
}

// the cache fields of a rotary / append launch: the new K / V rows (null: none) appended to the present caches kc / vc
// of T positions, and for build_k / build_v the past caches pk / pv (null: none) copied below them, the tail zeroed
void cache_prep(RotaryLaunch& R, int64_t B, int64_t S, int64_t H, int64_t Hkv, int64_t D, int64_t T, const RotaryRows& k_new,
                const RotaryRows& v_new, const RotaryRows& kc, const RotaryRows& vc, const rten_tensor* pk, const rten_tensor* pv,
                bool build_k, bool build_v) {
    R.B = (int)B;
    R.S = (int)S;
    R.D = (int)D;
    R.H = (int)H;
    R.Hkv = (int)Hkv;
    R.T = (int)T;
    R.k_new = k_new;
    R.v_new = v_new;
    R.k_cache = kc;
    R.v_cache = vc;
    R.build_k = build_k;
    R.build_v = build_v;
    if (pk) {
        R.k_past = cache_rows(pk);
        R.v_past = cache_rows(pv);
    }
}

// ---- inputs and outputs

// device view of an input whose last dimension is contiguous (a contiguous copy when it is not)
rten_status in_last_contiguous(OpScope& sc, const rten_tensor* t, rten_tensor* v) {
    rten_status s = sc.in(t, v);
    if (s == RTEN_OK && v->strides[v->ndim - 1] != 1 && v->shape[v->ndim - 1] > 1) {
        rten_tensor c;
        s = sc.contiguous(v, &c);
        *v = c;
    }
    return s;
}

// [first, last) byte range a tensor spans
void byte_span(const rten_tensor* t, uintptr_t* a, uintptr_t* b) {
    *a = reinterpret_cast<uintptr_t>(t->data);
    *b = *a + (uintptr_t)span_elems(t) * dtype_size(t->dtype);
}

// The [B, heads, T, D] present caches (null: not requested) of `op`.  Each one is either its past cache itself -- same
// data and strides, extended in place (*alias_k / *alias_v) -- or lies outside the memory of every past cache it is not:
// otherwise one launch would read and write the same memory.
rten_status present_caches(rten_ctx* ctx, const char* op, const rten_tensor* present_key, const rten_tensor* present_value,
                           const rten_tensor* past_key, const rten_tensor* past_value, int64_t B, int64_t heads, int64_t T, int64_t D,
                           bool* alias_k, bool* alias_v) {
    auto aliased = [](const rten_tensor* pres, const rten_tensor* past) {
        if (!pres || !past || !pres->data || pres->data != past->data || pres->device < 0 || past->device < 0 || pres->ndim != 4) return false;
        for (int i = 0; i < 4; i++)
            if (pres->strides[i] != past->strides[i]) return false;
        return true;
    };
    *alias_k = aliased(present_key, past_key);
    *alias_v = aliased(present_value, past_value);
    for (const rten_tensor* pres : {present_key, present_value})
        for (const rten_tensor* past : {past_key, past_value}) {
            if (!pres || !past || !pres->data || pres->device < 0 || past->device < 0 || aliased(pres, past)) continue;
            uintptr_t a0, a1, b0, b1;
            rten_tensor pshape = *pres;
            pshape.ndim = 4;
            pshape.shape[0] = B;
            pshape.shape[1] = heads;
            pshape.shape[2] = T;
            pshape.shape[3] = D;
            byte_span(&pshape, &a0, &a1);
            byte_span(past, &b0, &b1);
            if (a0 < b1 && b0 < a1)
                return fail(ctx, RTEN_ERR_UNSUPPORTED_OUTPUT,
                            (std::string(op) + ": present_key / present_value overlap a past cache without being that buffer (same data and strides)").c_str());
        }
    return RTEN_OK;
}

// the value of a 0-D / 1-element i32 tensor, wherever it lives (device: one synchronous 4-byte copy)
rten_status read_scalar_i32(rten_ctx* ctx, const rten_tensor* t, int32_t* v) {
    if (t->device < 0) {
        *v = *(const int32_t*)t->data;
        return RTEN_OK;
    }
    RTB_CUDA(ctx, cudaMemcpyAsync(v, t->data, 4, cudaMemcpyDeviceToHost, ctx->stream));
    RTB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return RTEN_OK;
}

int32_t host_i32(const rten_tensor* t, int64_t i0, int64_t i1) {
    const int64_t s0 = t->ndim > 0 ? t->strides[0] : 0, s1 = t->ndim > 1 ? t->strides[1] : 0;
    return ((const int32_t*)t->data)[i0 * s0 + i1 * s1];
}

// ---- rotary tables

// position_ids as a device view.  Held by the host, every entry must index both tables (negative entries count from the
// end, as Gather reads them), and the resolved positions are staged contiguously for the kernels.
rten_status position_view(rten_ctx* ctx, OpScope& sc, const rten_tensor* pos, int64_t cos_rows, int64_t sin_rows, rten_tensor* view) {
    if (pos->device >= 0) return sc.in(pos, view);
    const int64_t n0 = pos->shape[0], n1 = pos->shape[1];
    std::vector<int32_t> res((size_t)std::max<int64_t>(n0 * n1, 1));
    for (int64_t i = 0; i < n0; i++)
        for (int64_t j = 0; j < n1; j++) {
            const int64_t q = host_i32(pos, i, j);
            for (int64_t rows : {cos_rows, sin_rows})
                if (q < -rows || q >= rows) return fail(ctx, RTEN_ERR_INVALID_VALUE, "Entry in `indices` is out of range");
            res[(size_t)(i * n1 + j)] = (int32_t)(q < 0 ? q + cos_rows : q);
        }
    void* d = nullptr;
    RTB_TRY(temp_alloc(ctx, res.size() * 4, &d));
    RTB_CUDA(ctx, cudaMemcpyAsync(d, res.data(), res.size() * 4, cudaMemcpyHostToDevice, ctx->stream));
    sc.host_involved = true;
    *view = *pos;
    view->data = d;
    view->device = ctx->device;
    view->strides[0] = n1;
    view->strides[1] = 1;
    return RTEN_OK;
}

// rows of the contiguous [max_pos, half] tables cos / sin gathered by position: pos[b, s] (a device view), or
// past_len(b) + s without one
RotaryTable position_table(const rten_tensor& cos, const rten_tensor& sin, int64_t half, int interleaved, const rten_tensor* pos) {
    RotaryTable tab;
    tab.cos = (const float*)cos.data;
    tab.sin = (const float*)sin.data;
    tab.half = (int)half;
    tab.interleaved = interleaved ? 1 : 0;
    tab.by_pos = 1;
    tab.max_pos = (int)std::min(cos.shape[0], sin.shape[0]);
    if (pos) {
        tab.pos = (const int32_t*)pos->data;
        tab.p_b = bstride(pos, 0);
        tab.p_s = bstride(pos, 1);
    }
    return tab;
}

// src/ops/embedding.rs:20-44 on a [cb, cs, half] cache
rten_status cache_dims(rten_ctx* ctx, int ndim, const int64_t* shape, int64_t B, int64_t S, int64_t half, const char* bad_last_dim) {
    if (ndim != 3) return fail(ctx, RTEN_ERR_INVALID_VALUE, "cos/sin cache must be a 3D tensor");
    if (shape[2] != half) return fail(ctx, RTEN_ERR_INVALID_VALUE, bad_last_dim);
    if (shape[1] != 1 && shape[1] != S) return fail(ctx, RTEN_ERR_INVALID_VALUE, "cos/sin cache sequence length must be 1 or match the input");
    if (shape[0] != 1 && shape[0] != B) return fail(ctx, RTEN_ERR_INVALID_VALUE, "cos/sin cache batch size must be 1 or match the input");
    return RTEN_OK;
}

// the reference's failed conversion of an input to a tensor view of fixed rank (src/operator.rs InputCastFailed)
rten_status rank_fail(rten_ctx* ctx, int index, int expected, int actual) {
    ctx->err = "conversion error for input " + std::to_string(index) + ": expected tensor with " + std::to_string(expected) +
               " dims but has " + std::to_string(actual) + " dims";
    return RTEN_ERR_CAST_FAILED;
}

const char* const COS_LAST = "Last dimension of cos cache does not match rotary_embedding_dim/2";
const char* const SIN_LAST = "Last dimension of sin cache does not match rotary_embedding_dim/2";

}  // namespace

extern "C" {

rten_status rten_b200_attention(rten_ctx* ctx, const rten_tensor* query, const rten_tensor* key, const rten_tensor* value,
                                const rten_tensor* attn_mask, const rten_tensor* nonpad_kv_seqlen, const rten_attention_params* prm,
                                const rten_tensor* new_key, const rten_tensor* new_value, rten_tensor* out) {
    RTB_TRY(check_ctx(ctx));
    if (!query || !key || !value || !prm || !out) return fail(ctx, RTEN_ERR_MISSING_INPUTS, "missing inputs");
    if (query->dtype != RTEN_F32 || key->dtype != RTEN_F32 || value->dtype != RTEN_F32)
        return fail(ctx, RTEN_ERR_UNSUPPORTED_TYPE, "unsupported type");
    if (query->ndim != 4) return fail(ctx, RTEN_ERR_INVALID_VALUE, "query must have 3 or 4 dimensions");  // (3-D: split heads first)
    if (key->ndim != 4 || value->ndim != 4)
        return fail(ctx, RTEN_ERR_INCOMPATIBLE_SHAPES, "query, key and value must have the same rank");
    const int64_t B = query->shape[0], qh = query->shape[1], qs = query->shape[2], dh = query->shape[3];
    const int64_t kvh = key->shape[1], total = key->shape[2];
    if (key->shape[0] != B || value->shape[0] != B)
        return fail(ctx, RTEN_ERR_INCOMPATIBLE_SHAPES, "query, key and value must have the same batch size");
    if (value->shape[1] != kvh || value->shape[2] != total)
        return fail(ctx, RTEN_ERR_INCOMPATIBLE_SHAPES, "key and value must have the same number of heads and sequence length");
    if (key->shape[3] != dh) return fail(ctx, RTEN_ERR_INCOMPATIBLE_SHAPES, "key head size must match query head size");
    if (qh == 0 || kvh == 0 || qh % kvh) return fail(ctx, RTEN_ERR_INCOMPATIBLE_SHAPES, "q_num_heads must be a positive multiple of kv_num_heads");
    const int64_t dv = value->shape[3];
    if (nonpad_kv_seqlen) {
        if (nonpad_kv_seqlen->dtype != RTEN_I32) return fail(ctx, RTEN_ERR_UNSUPPORTED_TYPE, "unsupported type");
        if (nonpad_kv_seqlen->ndim != 1 || nonpad_kv_seqlen->shape[0] != B)
            return fail(ctx, RTEN_ERR_INCOMPATIBLE_SHAPES, "nonpad_kv_seqlen must have batch_size elements");
    }
    if (prm->softcap > 0.0f) return fail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "attention softcap is not supported");
    if ((new_key == nullptr) != (new_value == nullptr))
        return fail(ctx, RTEN_ERR_INVALID_VALUE, "past_key and past_value must either both be present or both be absent");
    const float scale = prm->scale > 0.0f ? prm->scale : 1.0f / std::sqrt((float)dh);
    // mask: float, broadcastable to (batch, q_heads, q_seq, total_seq)
    long long ms[4] = {0, 0, 0, 0};
    if (attn_mask) {
        if (attn_mask->dtype != RTEN_F32) return fail(ctx, RTEN_ERR_INVALID_VALUE, "attn_mask must have a float or bool (int32) type");
        if (attn_mask->ndim > 4) return fail(ctx, RTEN_ERR_INCOMPATIBLE_SHAPES, "Cannot broadcast inputs");
        const int64_t target[4] = {B, qh, qs, total};
        for (int i = 0; i < 4; i++) {
            const int mi = i - (4 - attn_mask->ndim);
            if (mi < 0 || attn_mask->shape[mi] == 1)
                ms[i] = 0;
            else if (attn_mask->shape[mi] == target[i])
                ms[i] = attn_mask->strides[mi];
            else
                return fail(ctx, RTEN_ERR_INCOMPATIBLE_SHAPES, "Cannot broadcast inputs");
        }
    }
    const bool resident = query->device >= 0 && key->device >= 0 && value->device >= 0 && (!attn_mask || attn_mask->device >= 0) &&
                          (!nonpad_kv_seqlen || nonpad_kv_seqlen->device >= 0) && (!new_key || (new_key->device >= 0 && new_value->device >= 0)) &&
                          (out->data == nullptr || out->device >= 0);
    const RotaryRows qr = cache_rows(query), kr = cache_rows(key), vr = cache_rows(value);
    if (qs == 1 && dv == dh && resident && query->strides[3] == 1 && key->strides[3] == 1) {
        AttnDecodeLaunch L = decode_launch(B, qh, kvh, dh, total, qr, kr, vr);
        L.len = nonpad_kv_seqlen ? (const int32_t*)nonpad_kv_seqlen->data : nullptr;
        set_mask(L, attn_mask, ms);
        L.scale = scale;
        bool ok = true;
        if (new_key) {
            // [batch, kv_heads, 1, head] (or [batch, kv_heads, head]) views of the projection output
            auto nk = [&](const rten_tensor* t, const float** p, long long* sb, long long* sh) {
                if (t->dtype != RTEN_F32) return false;
                if (t->ndim == 4 && t->shape[0] == B && t->shape[1] == kvh && t->shape[2] == 1 && t->shape[3] == dh && t->strides[3] == 1) {
                    *p = (const float*)t->data;
                    *sb = t->strides[0];
                    *sh = t->strides[1];
                    return true;
                }
                if (t->ndim == 3 && t->shape[0] == B && t->shape[1] == kvh && t->shape[2] == dh && t->strides[2] == 1) {
                    *p = (const float*)t->data;
                    *sb = t->strides[0];
                    *sh = t->strides[1];
                    return true;
                }
                return false;
            };
            ok = nk(new_key, &L.k_new, &L.kn_b, &L.kn_h) && nk(new_value, &L.v_new, &L.vn_b, &L.vn_h);
            if (!ok) return fail(ctx, RTEN_ERR_INCOMPATIBLE_SHAPES, "new key / value must be [batch, kv_heads, 1, head_size]");
        }
        // the kernel reads nonpad_kv_seqlen with unit stride
        const bool unit_len = !nonpad_kv_seqlen || nonpad_kv_seqlen->strides[0] == 1 || B == 1;
        if (unit_len && attn_decode_supported(L)) {
            OpScope sc(ctx);
            rten_tensor ov;
            const int64_t oshape[4] = {B, qh, 1, dh};
            RTB_TRY(sc.out(out, RTEN_F32, 4, oshape, &ov, nullptr));
            if (ov.strides[3] != 1) return fail(ctx, RTEN_ERR_UNSUPPORTED_OUTPUT, "output head dimension must be contiguous");
            decode_out(L, cache_rows(&ov));
            return sc.finish(launch_attn_decode(ctx, L));
        }
    }
    // The one-kernel branches below allocate `out` in a scope of their own: a branch whose kernel declines the layout
    // leaves that scope without finishing it, which returns the output, and the next branch starts from `out` as given.
    // ---- encoder shapes (128 keys, head size 64, value tensor stored transposed): one fused kernel per layer where available
    // (single-pass TF32 products: only when the context opted in to that mode)
    if (resident && ctx->f32_mode == RTEN_F32_TF32 && !new_key && !nonpad_kv_seqlen && !prm->is_causal && qh == kvh && dv == dh &&
        query->strides[3] == 1 && key->strides[3] == 1 && (value->strides[2] == 1 || value->strides[3] == 1) &&
        (!attn_mask || (ms[1] == 0 && ms[2] == 0 && (ms[3] == 1 || total == 1)))) {
        OpScope sc(ctx);
        rten_tensor ov;
        const int64_t oshape[4] = {B, qh, qs, dh};
        RTB_TRY(sc.out(out, RTEN_F32, 4, oshape, &ov, nullptr));
        AttnFusedLaunch L;
        stream_io(L, B, qh, kvh, qs, total, dh, qr, kr, cache_rows(&ov));
        L.heads = (int)qh;
        if (value->strides[3] == 1 && value->strides[2] != 1) {  // natural layout: the kernel transposes the tile itself
            L.v = vr.p;
            L.v_b = vr.sb;
            L.v_h = vr.sh;
            L.v_s = vr.ss;
        } else {
            L.vt = transposed_operand(value);
        }
        L.mask = attn_mask ? (const float*)attn_mask->data : nullptr;
        L.m_b = ms[0];
        L.scale = scale;
        if (ov.strides[3] == 1 && attn_fused_supported(L)) return sc.finish(launch_attn_fused(ctx, L));
    }
    // ---- causal, right-padded (nonpad_kv_seqlen) or grouped-query calls with q_seq > 1: the streaming prefill kernel
    // (head size 64 / 128, f32 products in the context's mode); other layouts keep the errors below
    if (qs > 1 && resident && !new_key && (prm->is_causal || nonpad_kv_seqlen || qh != kvh) && dv == dh && (dh == 64 || dh == 128) &&
        query->strides[3] == 1 && key->strides[3] == 1 && (value->strides[2] == 1 || value->strides[3] == 1) &&
        (!attn_mask || ms[3] == 1 || total == 1) && (!nonpad_kv_seqlen || nonpad_kv_seqlen->strides[0] == 1 || B == 1)) {
        OpScope sc(ctx);
        rten_tensor ov;
        const int64_t oshape[4] = {B, qh, qs, dh};
        RTB_TRY(sc.out(out, RTEN_F32, 4, oshape, &ov, nullptr));
        AttnPrefillLaunch L = prefill_launch(ctx, B, qh, kvh, qs, total, dh, scale, qr, kr, vr, cache_rows(&ov));
        L.v_natural = value->strides[3] == 1;
        if (!L.v_natural) L.v = transposed_operand(value);
        L.len = nonpad_kv_seqlen ? (const int32_t*)nonpad_kv_seqlen->data : nullptr;
        L.causal = prm->is_causal ? 1 : 0;
        set_mask(L, attn_mask, ms);
        if (ov.strides[3] == 1 && attn_prefill_supported(L)) return sc.finish(launch_attn_prefill(ctx, L));
    }
    // ---- general path: scale * Q K^T (+ mask) -> Softmax (NaNs flushed) -> . V  with this library's operators.
    // Causal masking / externally managed caches with q_seq > 1 need the mask spelled out by the caller.
    if (new_key) return fail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "the fused cache append needs q_seq = 1 and head size 64 or 128");
    if ((prm->is_causal && (qs > 1 || nonpad_kv_seqlen)) || nonpad_kv_seqlen)
        return fail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "causal / padded attention with q_seq > 1: pass the additive mask explicitly");
    if (qh != kvh) return fail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "grouped-query attention with q_seq > 1 is not supported");
    rten_tensor kt = *key;  // K^T view
    kt.shape[2] = dh;
    kt.shape[3] = total;
    kt.strides[2] = key->strides[3];
    kt.strides[3] = key->strides[2];
    Intermediate scores(ctx);
    RTB_TRY(rten_b200_matmul_ex(ctx, query, &kt, nullptr, nullptr, scale, nullptr, 0, &scores));
    RTB_TRY(rten_b200_softmax(ctx, &scores, attn_mask, -1, 1, &scores));
    return rten_b200_matmul(ctx, &scores, value, nullptr, nullptr, 1.0f, out);
}

rten_status rten_b200_rotary_embedding(rten_ctx* ctx, const rten_tensor* input, const rten_tensor* cos, const rten_tensor* sin,
                                       const rten_tensor* position_ids, int interleaved, int num_heads, int rotary_embedding_dim,
                                       rten_tensor* out) {
    RTB_TRY(check_ctx(ctx));
    if (!input || !cos || !sin || !out) return fail(ctx, RTEN_ERR_MISSING_INPUTS, "missing inputs");
    if (input->dtype != RTEN_F32 || cos->dtype != RTEN_F32 || sin->dtype != RTEN_F32 || (position_ids && position_ids->dtype != RTEN_I32))
        return fail(ctx, RTEN_ERR_UNSUPPORTED_TYPE, "unsupported type");
    // [batch, seq, heads, head_size] view of the input
    int64_t B, S, H, D;
    if (input->ndim == 3) {
        if (num_heads <= 0) return fail(ctx, RTEN_ERR_INVALID_VALUE, "num_heads must not be 0 for 3 dimensioned input");
        if (input->shape[2] % num_heads) return fail(ctx, RTEN_ERR_INVALID_VALUE, "hidden_size must be divisible by num_heads");
        B = input->shape[0];
        S = input->shape[1];
        H = num_heads;
        D = input->shape[2] / num_heads;
    } else if (input->ndim == 4) {
        B = input->shape[0];
        H = input->shape[1];
        S = input->shape[2];
        D = input->shape[3];
    } else {
        return fail(ctx, RTEN_ERR_INCOMPATIBLE_SHAPES, "Input processed needs 3-4 dimensions");
    }
    const int64_t rd = rotary_embedding_dim == 0 ? D : rotary_embedding_dim;
    if (rd <= 0 || rd % 2) return fail(ctx, RTEN_ERR_INVALID_VALUE, "rotary_embedding_dim must be a positive even number");
    if (rd > D) return fail(ctx, RTEN_ERR_INVALID_VALUE, "rotary_embedding_dim must not exceed head size");
    const int64_t half = rd / 2;
    OpScope sc(ctx);
    rten_tensor xv, cv, sv, pv;
    RTB_TRY(sc.in(input, &xv));
    RTB_TRY(sc.in(cos, &cv));
    RTB_TRY(sc.in(sin, &sv));
    RotaryTable tab;
    if (position_ids) {
        // the caches are gathered by position: [max_pos, half] tables, gathered to [pb, ps, half]
        if (position_ids->ndim != 2) return rank_fail(ctx, 3, 2, position_ids->ndim);
        if (cos->ndim != 2 || sin->ndim != 2) return fail(ctx, RTEN_ERR_INVALID_VALUE, "cos/sin cache must be a 3D tensor");
        RTB_TRY(position_view(ctx, sc, position_ids, cos->shape[0], sin->shape[0], &pv));
        const int64_t gc[3] = {position_ids->shape[0], position_ids->shape[1], cos->shape[1]};
        const int64_t gs[3] = {position_ids->shape[0], position_ids->shape[1], sin->shape[1]};
        RTB_TRY(cache_dims(ctx, 3, gc, B, S, half, COS_LAST));
        RTB_TRY(cache_dims(ctx, 3, gs, B, S, half, SIN_LAST));
        if (cos->shape[0] < 1 || sin->shape[0] < 1) return fail(ctx, RTEN_ERR_INVALID_VALUE, "Entry in `indices` is out of range");
        rten_tensor cc, scc;
        RTB_TRY(sc.contiguous(&cv, &cc));
        RTB_TRY(sc.contiguous(&sv, &scc));
        tab = position_table(cc, scc, half, interleaved, &pv);
    } else {
        RTB_TRY(cache_dims(ctx, cos->ndim, cos->shape, B, S, half, COS_LAST));
        RTB_TRY(cache_dims(ctx, sin->ndim, sin->shape, B, S, half, SIN_LAST));
        rten_tensor cc = cv, scc = sv;
        if (cv.strides[2] != 1 && half > 1) RTB_TRY(sc.contiguous(&cv, &cc));
        if (sv.strides[2] != 1 && half > 1) RTB_TRY(sc.contiguous(&sv, &scc));
        tab.cos = (const float*)cc.data;
        tab.sin = (const float*)scc.data;
        tab.half = (int)half;
        tab.interleaved = interleaved ? 1 : 0;
        tab.c_b = bstride(&cc, 0);
        tab.c_s = bstride(&cc, 1);
        tab.s_b = bstride(&scc, 0);
        tab.s_s = bstride(&scc, 1);
    }
    rten_tensor ov;
    RTB_TRY(sc.out(out, RTEN_F32, input->ndim, input->shape, &ov, nullptr));
    RotaryLaunch L;
    L.B = (int)B;
    L.S = (int)S;
    L.H = (int)H;
    L.D = (int)D;
    L.rot = tab;
    L.x = input->ndim == 3 ? rows3(&xv, D, 0) : cache_rows(&xv);
    L.y = input->ndim == 3 ? rows3(&ov, D, 0) : cache_rows(&ov);
    return sc.finish(B * S * H * D > 0 ? launch_rotary(ctx, L) : RTEN_OK);
}

rten_status rten_b200_group_query_attention(rten_ctx* ctx, const rten_tensor* query, const rten_tensor* key, const rten_tensor* value,
                                            const rten_tensor* past_key, const rten_tensor* past_value, const rten_tensor* seqlens_k,
                                            const rten_tensor* total_sequence_length, const rten_tensor* cos, const rten_tensor* sin,
                                            const rten_tensor* position_ids, const rten_tensor* attention_bias, const rten_gqa_params* prm,
                                            rten_tensor* out, rten_tensor* present_key, rten_tensor* present_value) {
    RTB_TRY(check_ctx(ctx));
    if (!query || !seqlens_k || !total_sequence_length || !prm || !out || !present_key || !present_value)
        return fail(ctx, RTEN_ERR_MISSING_INPUTS, "missing inputs");
    for (const rten_tensor* t : {query, key, value, past_key, past_value, cos, sin, attention_bias})
        if (t && t->dtype != RTEN_F32) return fail(ctx, RTEN_ERR_UNSUPPORTED_TYPE, "unsupported type");
    for (const rten_tensor* t : {seqlens_k, total_sequence_length, position_ids})
        if (t && t->dtype != RTEN_I32) return fail(ctx, RTEN_ERR_UNSUPPORTED_TYPE, "unsupported type");
    // tensor views of fixed rank, converted in the reference's order (past caches first, in `run`)
    {
        const rten_tensor* ts[] = {past_key, past_value, query, key, value, total_sequence_length, cos, sin, position_ids, attention_bias};
        const int idx[] = {3, 4, 0, 1, 2, 6, 7, 8, 9, 10}, rank[] = {4, 4, 3, 3, 3, 0, 2, 2, 2, 4};
        for (int i = 0; i < 10; i++)
            if (ts[i] && ts[i]->ndim != rank[i]) return rank_fail(ctx, idx[i], rank[i], ts[i]->ndim);
    }
    if (prm->softcap > 0.0f) return fail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "GroupQueryAttention softcap is not supported");
    // seqlens_k: [batch] (or [batch, 1])
    int sl_nd = seqlens_k->ndim;
    while (sl_nd > 1 && seqlens_k->shape[sl_nd - 1] == 1) sl_nd--;
    if (sl_nd != 1) return fail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "seqlens_k must be a vector");
    const int64_t H = prm->num_heads, Hkv = prm->kv_num_heads;
    if (H <= 0 || Hkv <= 0) return fail(ctx, RTEN_ERR_INVALID_VALUE, "num_heads and kv_num_heads must be positive");
    if (H % Hkv) return fail(ctx, RTEN_ERR_INVALID_VALUE, "num_heads must be a multiple of kv_num_heads");
    const int64_t B = query->shape[0], S = query->shape[1];
    int64_t D;
    const bool packed = !key && !value;
    if (key && value) {
        if (query->shape[2] % H) return fail(ctx, RTEN_ERR_INCOMPATIBLE_SHAPES, "query hidden size must be divisible by num_heads");
        D = query->shape[2] / H;
        if (key->shape[0] != B || value->shape[0] != B) return fail(ctx, RTEN_ERR_INCOMPATIBLE_SHAPES, "key and value batch size must match query");
        if (key->shape[1] != value->shape[1] || key->shape[2] != value->shape[2])
            return fail(ctx, RTEN_ERR_INCOMPATIBLE_SHAPES, "key and value must have the same shape");
        if (key->shape[2] != Hkv * D) return fail(ctx, RTEN_ERR_INCOMPATIBLE_SHAPES, "key hidden size must equal kv_num_heads * head_size");
        if (key->shape[1] != S) return fail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "key sequence length must match query sequence length");
    } else if (packed) {
        if (query->shape[2] % (H + 2 * Hkv))
            return fail(ctx, RTEN_ERR_INCOMPATIBLE_SHAPES, "packed query hidden size must be divisible by num_heads + 2 * kv_num_heads");
        D = query->shape[2] / (H + 2 * Hkv);
    } else {
        return fail(ctx, RTEN_ERR_INVALID_VALUE, "key and value must both be present or both absent");
    }
    if (seqlens_k->shape[0] != B) return fail(ctx, RTEN_ERR_INCOMPATIBLE_SHAPES, "seqlens_k must have batch_size elements");
    int32_t total = 0;
    RTB_TRY(read_scalar_i32(ctx, total_sequence_length, &total));
    if (total <= 0) return fail(ctx, RTEN_ERR_INVALID_VALUE, "total_sequence_length must be positive");
    int64_t P = 0;
    if (past_key && past_value) {
        const int64_t* a = past_key->shape;
        const int64_t* v = past_value->shape;
        if (a[0] != B || v[0] != B || a[1] != Hkv || v[1] != Hkv || a[3] != D || v[3] != D || a[2] != v[2])
            return fail(ctx, RTEN_ERR_INCOMPATIBLE_SHAPES, "past_key/past_value shape does not match");
        P = a[2];
    } else if (past_key || past_value) {
        return fail(ctx, RTEN_ERR_INVALID_VALUE, "past_key and past_value must both be present or both absent");
    }
    const int64_t T = P + S;
    const bool first = S == total;
    const bool subsequent = S > 1 && S != total;
    if (subsequent && B != 1)
        return fail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "batch size must be 1 when sequence_length > 1 and a past context is given");
    if (!first && !subsequent && S != 1) return fail(ctx, RTEN_ERR_INVALID_VALUE, "sequence_length must be 1 when query is not a prompt");
    const bool host_lens = seqlens_k->device < 0;
    if (host_lens) {
        for (int64_t b = 0; b < B; b++) {
            const int64_t len = host_i32(seqlens_k, b, 0);
            if (len < 0 || len >= T) return fail(ctx, RTEN_ERR_INVALID_VALUE, "seqlens_k entry is out of range");
            if (len + 1 < S) return fail(ctx, RTEN_ERR_INVALID_VALUE, "seqlens_k entry is too small for the query sequence length");
        }
    }
    if (attention_bias) {
        const int64_t* s = attention_bias->shape;
        if ((s[0] != 1 && s[0] != B) || (s[1] != 1 && s[1] != H) || s[2] < S || s[3] < T)
            return fail(ctx, RTEN_ERR_INCOMPATIBLE_SHAPES, "attention_bias shape is incompatible with query/key shapes");
    }
    const float scale = prm->scale > 0.0f ? prm->scale : 1.0f / std::sqrt((float)D);
    int64_t half = 0;
    if (prm->do_rotary) {
        if (!cos || !sin) return fail(ctx, RTEN_ERR_INVALID_VALUE, "cos_cache and sin_cache are required when do_rotary is set");
        const int64_t rd = cos->shape[1] == 0 ? D : 2 * cos->shape[1];
        if (rd <= 0 || rd % 2) return fail(ctx, RTEN_ERR_INVALID_VALUE, "rotary_embedding_dim must be a positive even number");
        if (rd > D) return fail(ctx, RTEN_ERR_INVALID_VALUE, "rotary_embedding_dim must not exceed head size");
        half = rd / 2;
        if (!position_ids && (first || host_lens)) {  // positions past_len(b) + s, gathered from both tables
            for (int64_t b = 0; b < B; b++) {
                const int64_t last = (first ? 0 : host_i32(seqlens_k, b, 0) + 1 - S) + S - 1;
                if (last >= cos->shape[0] || last >= sin->shape[0]) return fail(ctx, RTEN_ERR_INVALID_VALUE, "Entry in `indices` is out of range");
            }
        }
    }
    if (D != 64 && D != 128) return fail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "GroupQueryAttention: the head size must be 64 or 128");
    const bool decode = S == 1 && !first;
    if (decode && T > ATTN_DECODE_MAX_CACHE)
        return fail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, ("GroupQueryAttention: a decode step takes at most " + std::to_string(ATTN_DECODE_MAX_CACHE) +
                                                      " cache positions (past + 1)").c_str());
    bool alias_k, alias_v;
    RTB_TRY(present_caches(ctx, "GroupQueryAttention", present_key, present_value, past_key, past_value, B, Hkv, T, D, &alias_k, &alias_v));

    // ---- device views
    OpScope sc(ctx);
    rten_tensor qv, kv, vv, pkv, pvv, slv, cv, snv, posv, biasv;
    RTB_TRY(sc.in(query, &qv));
    if (key) RTB_TRY(sc.in(key, &kv));
    if (value) RTB_TRY(sc.in(value, &vv));
    if (past_key) RTB_TRY(sc.in(past_key, &pkv));
    if (past_value) RTB_TRY(sc.in(past_value, &pvv));
    RTB_TRY(sc.in(seqlens_k, &slv));
    if (attention_bias) RTB_TRY(in_last_contiguous(sc, attention_bias, &biasv));
    RotaryTable tab;
    if (prm->do_rotary) {
        RTB_TRY(sc.in(cos, &cv));
        RTB_TRY(sc.in(sin, &snv));
        rten_tensor cc, scc;
        RTB_TRY(sc.contiguous(&cv, &cc));
        RTB_TRY(sc.contiguous(&snv, &scc));
        if (position_ids) {
            RTB_TRY(position_view(ctx, sc, position_ids, cos->shape[0], sin->shape[0], &posv));
            const int64_t gc[3] = {position_ids->shape[0], position_ids->shape[1], half};
            RTB_TRY(cache_dims(ctx, 3, gc, B, S, half, COS_LAST));
        }
        if (cos->shape[1] != half) return fail(ctx, RTEN_ERR_INVALID_VALUE, COS_LAST);
        if (sin->shape[1] != half) return fail(ctx, RTEN_ERR_INVALID_VALUE, SIN_LAST);
        if (cos->shape[0] < 1 || sin->shape[0] < 1) return fail(ctx, RTEN_ERR_INVALID_VALUE, "Entry in `indices` is out of range");
        tab = position_table(cc, scc, half, prm->rotary_interleaved, position_ids ? &posv : nullptr);
    }
    rten_tensor ov, pk, pv;
    const int64_t oshape[3] = {B, S, H * D}, cshape[4] = {B, Hkv, T, D};
    RTB_TRY(sc.out(out, RTEN_F32, 3, oshape, &ov, nullptr));
    RTB_TRY(sc.out(present_key, RTEN_F32, 4, cshape, &pk, nullptr));
    RTB_TRY(sc.out(present_value, RTEN_F32, 4, cshape, &pv, nullptr));
    if (ov.strides[2] != 1 || pk.strides[3] != 1 || pv.strides[3] != 1)
        return fail(ctx, RTEN_ERR_UNSUPPORTED_OUTPUT, "GroupQueryAttention: the outputs need a contiguous last dimension");
    if (B * S == 0 || H * D == 0) return sc.finish(RTEN_OK);

    const RotaryRows qr = rows3(&qv, D, 0), orows = rows3(&ov, D, 0);
    const RotaryRows kr = packed ? rows3(&qv, D, H) : rows3(&kv, D, 0);
    const RotaryRows vr = packed ? rows3(&qv, D, H + Hkv) : rows3(&vv, D, 0);
    const RotaryRows kc = cache_rows(&pk), vc = cache_rows(&pv);
    long long ms[4];
    mask_strides(attention_bias ? &biasv : nullptr, ms);
    const int window = prm->local_window_size > 0 ? prm->local_window_size : 0;
    RotaryLaunch R;  // the fields both rotary / append launches share
    R.rot = tab;
    R.seqlens = (const int32_t*)slv.data;
    R.sl_s = slv.strides[0];
    R.first = first ? 1 : 0;
    // the present caches' past prefix and zero tail, unless the present cache is the past buffer (or there is no past)
    RotaryLaunch Rb = R;
    cache_prep(Rb, B, S, H, Hkv, D, T, RotaryRows(), RotaryRows(), kc, vc, past_key ? &pkv : nullptr, &pvv, !alias_k, !alias_v);
    const bool build = P > 0 && (Rb.build_k || Rb.build_v);

    if (decode) {
        AttnDecodeLaunch L = decode_launch(B, H, Hkv, D, T, qr, kc, vc);
        L.len = (const int32_t*)slv.data;
        L.len_s = slv.strides[0];
        L.len_add = 1;
        L.len_min = 1;
        L.window = window;
        set_mask(L, attention_bias ? &biasv : nullptr, ms);
        L.k_new = kr.p;
        L.kn_b = kr.sb;
        L.kn_h = kr.sh;
        L.v_new = vr.p;
        L.vn_b = vr.sb;
        L.vn_h = vr.sh;
        L.scale = scale;
        if (prm->do_rotary) {
            L.rot_cos = tab.cos;
            L.rot_sin = tab.sin;
            L.rot_half = tab.half;
            L.rot_interleaved = tab.interleaved;
            L.rot_max_pos = tab.max_pos;
            L.rot_pos = tab.pos;
            L.rot_pos_b = tab.p_b;
        }
        decode_out(L, orows);
        if (qr.sd == 1 && kr.sd == 1 && vr.sd == 1 && attn_decode_supported(L)) {
            if (build) RTB_TRY(launch_rotary(ctx, Rb));
            return sc.finish(launch_attn_decode(ctx, L));
        }
        // (a layout the single-query kernel cannot read: the prompt path below serves one query as well)
    }

    // ---- prompt: rotary + append, then the streaming prefill kernel over the present caches
    void* qs = nullptr;
    void* le = nullptr;
    RTB_TRY(temp_alloc(ctx, (size_t)(B * S * H * D) * 4, &qs));
    RTB_TRY(temp_alloc(ctx, (size_t)B * 4, &le));
    cache_prep(R, B, S, H, Hkv, D, T, kr, vr, kc, vc, nullptr, nullptr, false, false);
    R.x = qr;
    R.y = dense_rows(qs, S, H, D, false);
    R.len_eff = (int32_t*)le;
    AttnPrefillLaunch A = prefill_launch(ctx, B, H, Hkv, S, T, D, scale, R.y, kc, vc, orows);
    A.len = (const int32_t*)le;
    A.causal = 1;
    A.window = window;
    set_mask(A, attention_bias ? &biasv : nullptr, ms);
    if (!attn_prefill_supported(A))
        return fail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "GroupQueryAttention: the present caches and the output need 16-byte aligned rows");
    if (build) RTB_TRY(launch_rotary(ctx, Rb));
    RTB_TRY(launch_rotary(ctx, R));
    return sc.finish(launch_attn_prefill(ctx, A));
}

rten_status rten_b200_multi_head_attention(rten_ctx* ctx, const rten_tensor* query, const rten_tensor* key, const rten_tensor* value,
                                           const rten_tensor* bias, const rten_tensor* key_padding_mask, const rten_tensor* attention_bias,
                                           const rten_tensor* past_key, const rten_tensor* past_value, const rten_tensor* past_sequence_length,
                                           const rten_tensor* cache_indirection, const rten_mha_params* prm, rten_tensor* out,
                                           rten_tensor* present_key, rten_tensor* present_value) {
    RTB_TRY(check_ctx(ctx));
    if (!query || !prm || !out) return fail(ctx, RTEN_ERR_MISSING_INPUTS, "missing inputs");
    for (const rten_tensor* t : {query, key, value, bias, attention_bias, past_key, past_value})
        if (t && t->dtype != RTEN_F32) return fail(ctx, RTEN_ERR_UNSUPPORTED_TYPE, "unsupported type");
    for (const rten_tensor* t : {key_padding_mask, past_sequence_length, cache_indirection})
        if (t && t->dtype != RTEN_I32) return fail(ctx, RTEN_ERR_UNSUPPORTED_TYPE, "unsupported type");
    // inputs as the reference reads them: past caches (in `run`), query, then inputs 1-5, 8, 9 (in `run_impl`)
    if (past_key && past_key->ndim != 4) return rank_fail(ctx, 6, 4, past_key->ndim);
    if (past_value && past_value->ndim != 4) return rank_fail(ctx, 7, 4, past_value->ndim);
    if (query->ndim != 3 && query->ndim != 5) return fail(ctx, RTEN_ERR_INVALID_VALUE, "query must have 3 or 5 dims");
    {
        const rten_tensor* ts[] = {key, value, bias, key_padding_mask, attention_bias};
        const int rank[] = {3, 3, 1, 2, 4};
        for (int i = 0; i < 5; i++)
            if (ts[i] && ts[i]->ndim != rank[i]) return rank_fail(ctx, i + 1, rank[i], ts[i]->ndim);
    }
    if (past_sequence_length) {
        if (past_sequence_length->ndim != 0) return rank_fail(ctx, 8, 0, past_sequence_length->ndim);
        return fail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "past_seq_len is not supported");
    }
    if (cache_indirection) {
        if (cache_indirection->ndim != 3) return rank_fail(ctx, 9, 3, cache_indirection->ndim);
        return fail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "cache_indirection is not supported");
    }
    const int64_t H = prm->num_heads;
    if (H <= 0) return fail(ctx, RTEN_ERR_INVALID_VALUE, "num_heads must be positive");
    const bool packed = query->ndim == 5;
    const int64_t B = query->shape[0], S = query->shape[1];
    int64_t D, Dv, L, hidden = 0;
    if (packed) {  // [B, S, H, 3, D]
        if (key) return fail(ctx, RTEN_ERR_INVALID_VALUE, "key must be None when query is packed");
        if (value) return fail(ctx, RTEN_ERR_INVALID_VALUE, "value must be None when query is packed");
        if (bias) return fail(ctx, RTEN_ERR_INVALID_VALUE, "bias is not supported with packed QKV format");
        if (query->shape[3] != 3) return fail(ctx, RTEN_ERR_INVALID_VALUE, "4th dimension of packed qkv input must be 3");
        if (query->shape[2] != H)
            return fail(ctx, RTEN_ERR_INVALID_VALUE, "2nd dimension of packed qkv input must be equal to number of attention heads");
        D = Dv = query->shape[4];
        L = S;
    } else {
        hidden = query->shape[2];
        if (hidden % H) return fail(ctx, RTEN_ERR_INCOMPATIBLE_SHAPES, "Hidden size must be divisible by number of attention heads");
        D = hidden / H;
        if (key && !value) return fail(ctx, RTEN_ERR_INVALID_VALUE, "value input must be set if key input is present");
        const rten_tensor* k = key ? key : query;  // (no key: key = value = query, a given value is ignored)
        const rten_tensor* v = key ? value : query;
        if (k->shape[0] != B || v->shape[0] != B || v->shape[1] != k->shape[1])
            return fail(ctx, RTEN_ERR_INCOMPATIBLE_SHAPES, "Key and value batch or sequence lengths do not match");
        if (k->shape[2] != hidden) return fail(ctx, RTEN_ERR_INCOMPATIBLE_SHAPES, "Key hidden size does not match query hidden size");
        if (v->shape[2] % H) return fail(ctx, RTEN_ERR_INCOMPATIBLE_SHAPES, "Value hidden size must be divisible by number of attention heads");
        Dv = v->shape[2] / H;
        L = k->shape[1];
        if (bias && bias->shape[0] != 2 * hidden + v->shape[2])
            return fail(ctx, RTEN_ERR_INCOMPATIBLE_SHAPES, "Bias shape does not match QKV hidden sizes");
    }
    int64_t P = 0;
    if (past_key && past_value) {
        const int64_t* a = past_key->shape;
        const int64_t* v = past_value->shape;
        if (a[0] != B || v[0] != B || a[1] != H || v[1] != H || a[3] != D || v[3] != Dv || a[2] != v[2])
            return fail(ctx, RTEN_ERR_INCOMPATIBLE_SHAPES, "past_key/past_value shape does not match key/value shape");
        P = a[2];
    } else if (past_key || past_value) {
        return fail(ctx, RTEN_ERR_INVALID_VALUE, "past_key and past_value must either both be present or both be absent");
    }
    const int64_t T = P + L;
    if (attention_bias) {
        const int64_t target[4] = {B, H, S, T};
        for (int i = 0; i < 4; i++)
            if (attention_bias->shape[i] != target[i] && attention_bias->shape[i] != 1)
                return fail(ctx, RTEN_ERR_INCOMPATIBLE_SHAPES, "Cannot broadcast inputs");
    }
    if (key_padding_mask && (key_padding_mask->shape[0] != B || key_padding_mask->shape[1] != T))
        return fail(ctx, RTEN_ERR_INCOMPATIBLE_SHAPES, "key_padding_mask shape does not match key sequence length");
    if (D != 64 && D != 128) return fail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "MultiHeadAttention: the head size must be 64 or 128");
    if (Dv != D) return fail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "MultiHeadAttention: the value head size must equal the head size");
    if (T == 0 && B * S > 0) return fail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "MultiHeadAttention: there must be at least one key position");
    const float scale = prm->scale > 0.0f ? prm->scale : 1.0f / std::sqrt((float)D);
    // present caches: the past buffer itself (in place) or new memory
    bool alias_k, alias_v;
    RTB_TRY(present_caches(ctx, "MultiHeadAttention", present_key, present_value, past_key, past_value, B, H, T, D, &alias_k, &alias_v));

    // ---- device views (head dimension contiguous)
    OpScope sc(ctx);
    rten_tensor qv, kv, vv, bv, mv, abv, pkv, pvv;
    RTB_TRY(in_last_contiguous(sc, query, &qv));
    if (key) RTB_TRY(in_last_contiguous(sc, key, &kv));
    if (key) RTB_TRY(in_last_contiguous(sc, value, &vv));
    if (bias) RTB_TRY(in_last_contiguous(sc, bias, &bv));
    if (key_padding_mask) RTB_TRY(in_last_contiguous(sc, key_padding_mask, &mv));
    if (attention_bias) RTB_TRY(sc.in(attention_bias, &abv));
    if (past_key) RTB_TRY(in_last_contiguous(sc, past_key, &pkv));
    if (past_value) RTB_TRY(in_last_contiguous(sc, past_value, &pvv));
    rten_tensor ov, pk, pv;
    const int64_t oshape[3] = {B, S, H * D}, cshape[4] = {B, H, T, D};
    RTB_TRY(sc.out(out, RTEN_F32, 3, oshape, &ov, nullptr));
    if (present_key) RTB_TRY(sc.out(present_key, RTEN_F32, 4, cshape, &pk, nullptr));
    if (present_value) RTB_TRY(sc.out(present_value, RTEN_F32, 4, cshape, &pv, nullptr));
    if (ov.strides[2] != 1 || (present_key && pk.strides[3] != 1) || (present_value && pv.strides[3] != 1))
        return fail(ctx, RTEN_ERR_UNSUPPORTED_OUTPUT, "MultiHeadAttention: the outputs need a contiguous last dimension");
    if (B * S == 0) return sc.finish(RTEN_OK);

    // head rows (b, s, h, i) of q and of the new k / v
    const RotaryRows qr = packed ? packed_rows(&qv, 0) : rows3(&qv, D, 0);
    const RotaryRows kr = packed ? packed_rows(&qv, 1) : key ? rows3(&kv, D, 0) : qr;
    const RotaryRows vr = packed ? packed_rows(&qv, 2) : key ? rows3(&vv, D, 0) : qr;
    const RotaryRows orows = rows3(&ov, D, 0);
    // prep (one rotary / append launch) when there is a bias to add or a cache to build; else q / k / v are read in place
    const bool prep = bias || P > 0 || present_key || present_value;
    RotaryRows qa = qr;  // what the attention kernel reads
    RotaryRows kc = kr;  // [B, H, T, D] caches as rows (b, t, h); without prep the inputs' rows (T = L)
    RotaryRows vc = vr;
    RotaryLaunch R;
    if (prep) {
        auto scratch = [&](size_t n, void** p) { return temp_alloc(ctx, n * 4, p); };
        void* qs = nullptr;
        void* ks = nullptr;
        void* vs = nullptr;
        const size_t ncache = (size_t)(B * H * T * D);
        if (bias) RTB_TRY(scratch((size_t)(B * S * H * D), &qs));
        if (!present_key) RTB_TRY(scratch(ncache, &ks));
        if (!present_value) RTB_TRY(scratch(ncache, &vs));
        kc = present_key ? cache_rows(&pk) : dense_rows(ks, T, H, D, true);
        vc = present_value ? cache_rows(&pv) : dense_rows(vs, T, H, D, true);
        if (bias) {
            R.x = qr;
            R.y = dense_rows(qs, S, H, D, false);
            qa = R.y;
            const float* bb = (const float*)bv.data;
            R.x_bias = bb;
            R.k_bias = bb + hidden;
            R.v_bias = bb + 2 * hidden;
        }
        cache_prep(R, B, S, H, H, D, T, kr, vr, kc, vc, P > 0 ? &pkv : nullptr, &pvv, P > 0 && !alias_k, P > 0 && !alias_v);
        R.mha = 1;
        R.S_kv = (int)L;
        R.past = (int)P;
    }
    long long ms[4];
    mask_strides(attention_bias ? &abv : nullptr, ms);
    const int32_t* kpm_d = key_padding_mask ? (const int32_t*)mv.data : nullptr;
    const long long kpm_b = key_padding_mask ? mv.strides[0] : 0;
    const float fill = prm->mask_filter_value;

    if (S == 1) {
        AttnDecodeLaunch A = decode_launch(B, H, H, D, T, qa, kc, vc);
        set_mask(A, attention_bias ? &abv : nullptr, ms);
        A.scale = scale;
        decode_out(A, orows);
        A.mha = 1;
        A.vis_end = prm->unidirectional ? (int)P + 1 : (int)T;
        A.fill = fill;
        A.kpm = kpm_d;
        A.kpm_b = kpm_b;
        if (attn_decode_supported(A)) {
            if (prep) RTB_TRY(launch_rotary(ctx, R));
            return sc.finish(launch_attn_decode(ctx, A));
        }
        // (a cache longer than the single-query kernel takes: the prefill kernel serves one query as well)
    }
    AttnPrefillMha M;
    M.causal_offset = (int)P;
    M.fill = fill;
    M.kpm = kpm_d;
    M.kpm_b = kpm_b;
    M.v_rows = vc.p;
    M.v_b = vc.sb;
    M.v_h = vc.sh;
    M.v_t = vc.ss;
    if (attention_bias) M.m_t = ms[3];
    AttnPrefillLaunch A = prefill_launch(ctx, B, H, H, S, T, D, scale, qa, kc, vc, orows);
    A.causal = prm->unidirectional ? 1 : 0;
    set_mask(A, attention_bias ? &abv : nullptr, ms);
    A.mha = &M;
    if (qa.sd != 1 || kc.sd != 1 || vc.sd != 1 || !attn_prefill_supported(A))
        return fail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "MultiHeadAttention: query, key, value, the caches and the output need 16-byte aligned rows");
    if (prep) RTB_TRY(launch_rotary(ctx, R));
    return sc.finish(launch_attn_prefill(ctx, A));
}

}  // extern "C"
