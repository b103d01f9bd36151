// Fused operator entry points of the C ABI for the autoregressive decode path (include/rten_b200.h):
//   rten_b200_quantized_linear : [LayerNormalization] -> DynamicQuantizeLinear -> MatMulIntegerToFloat -> Add -> Add -> act
//   rten_b200_attention        : the reference's `Attention` operator (src/ops/attention.rs:645-905) on 4-D inputs
//   rten_b200_matmul_skinny    : used internally by MatMul / Gemm dispatch for M <= 32 (exact f32 FMA arithmetic)
// Each one has a hand-written skinny-M kernel (skinny.cu) for the decode shapes and otherwise composes the public
// operators of this library, so every shape the operator chain accepts is served with identical results.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstring>

#include "api_util.h"
#include "attn_fused.h"
#include "attn_prefill.h"
#include "rowops.h"
#include "skinny.h"

using namespace rtb;

namespace {

void free_if(rten_ctx* ctx, rten_tensor& t) {
    if (t.data) rten_b200_free(ctx, t.data);
    t.data = nullptr;
}

rten_tensor empty_tensor() {
    rten_tensor t;
    memset(&t, 0, sizeof(t));
    return t;
}

// a 4-D [b, h, s, d] tensor as the (d, s, h, b) operand of a TMA map, or (s, d, h, b) when `transposed` (key dimension
// contiguous: a value tensor stored transposed)
OperandDesc attn_operand(const rten_tensor* t, bool transposed) {
    OperandDesc d;
    d.base = t->data;
    d.dims[0] = transposed ? t->shape[2] : t->shape[3];
    d.dims[1] = transposed ? t->shape[3] : t->shape[2];
    d.dims[2] = t->shape[1];
    d.dims[3] = t->shape[0];
    d.strides[0] = 1;
    d.strides[1] = transposed ? t->strides[3] : t->strides[2];
    d.strides[2] = t->strides[1];
    d.strides[3] = t->strides[0];
    return d;
}

// An output a one-kernel attention branch allocated but cannot write (its layout does not fit the kernel): back to the
// pool, so that the branches below start from the caller's `out` as it was.
void give_back_output(rten_ctx* ctx, OpScope& sc, rten_tensor* out, const rten_tensor& ov) {
    if (out->data == ov.data && sc.allocated.size()) {
        pool_free(ctx, ov.data);
        out->data = nullptr;
        sc.allocated.clear();
    }
}

}  // namespace

extern "C" {

rten_status rten_b200_quantized_linear(rten_ctx* ctx, const rten_tensor* x, const rten_tensor* ln_scale, const rten_tensor* ln_bias,
                                       float ln_epsilon, const rten_tensor* w, const rten_packed* pw, const rten_tensor* w_zp,
                                       const rten_tensor* w_scale, const rten_tensor* bias, const rten_tensor* residual,
                                       int activation, rten_tensor* out) {
    if (!ctx) return RTEN_ERR_INVALID_VALUE;
    if (!x || !w || !w_scale || !out) return fail(ctx, RTEN_ERR_MISSING_INPUTS, "missing inputs");
    if (x->dtype != RTEN_F32 || w_scale->dtype != RTEN_F32) return fail(ctx, RTEN_ERR_UNSUPPORTED_TYPE, "unsupported type");
    if (w->dtype != RTEN_I8 && w->dtype != RTEN_U8) return fail(ctx, RTEN_ERR_UNSUPPORTED_TYPE, "unsupported type");
    if (w->ndim != 2) return fail(ctx, RTEN_ERR_INVALID_VALUE, "the weight must be a matrix");
    if (activation < 0 || activation > 3) return fail(ctx, RTEN_ERR_INVALID_VALUE, "unknown activation");
    if (ln_bias && !ln_scale) return fail(ctx, RTEN_ERR_MISSING_INPUTS, "missing inputs");
    if (x->ndim < 1) return fail(ctx, RTEN_ERR_INVALID_VALUE, "Inputs must have >= 1 dimensions");
    const int64_t K = x->shape[x->ndim - 1], N = w->shape[1];
    if (K != w->shape[0])
        return fail(ctx, RTEN_ERR_INCOMPATIBLE_SHAPES, "Columns of first matrix does not match rows of second matrix");
    int64_t M = 1;
    for (int i = 0; i + 1 < x->ndim; i++) M *= x->shape[i];

    // ---- fast path: every operand resident, rows uniformly strided, M <= 16
    bool fast = x->device >= 0 && pw && pw->kind == 0 && pw->dtype == w->dtype && pw->K == K && pw->N == N && pw->colsum &&
                w_scale->device >= 0 && (!bias || bias->device >= 0) && (!residual || residual->device >= 0) &&
                (!w_zp || w_zp->device >= 0) && (!ln_scale || ln_scale->device >= 0) && (!ln_bias || ln_bias->device >= 0) &&
                (out->data == nullptr || out->device >= 0) && M >= 1 && N >= 1;
    // x rows: [.., K] with unit inner stride and one uniform row stride
    int64_t xs = K;
    if (fast) {
        if (x->strides[x->ndim - 1] != 1 && K > 1) fast = false;
        if (x->ndim >= 2) {
            xs = x->strides[x->ndim - 2];
            int64_t expect = xs * x->shape[x->ndim - 2];
            for (int i = x->ndim - 3; i >= 0 && fast; i--) {
                if (x->shape[i] != 1 && x->strides[i] != expect) fast = false;
                expect *= x->shape[i];
            }
        }
    }
    auto vec_ok = [&](const rten_tensor* t, int64_t n) {
        return t->dtype == RTEN_F32 && ((t->ndim == 1 && t->shape[0] == n && (t->strides[0] == 1 || n == 1)) || (numel(t) == 1 && n == 1));
    };
    if (fast && ln_scale && !vec_ok(ln_scale, K)) fast = false;
    if (fast && ln_bias && !vec_ok(ln_bias, K)) fast = false;
    if (fast && bias && !vec_ok(bias, N)) fast = false;
    if (fast && !(numel(w_scale) == 1 || vec_ok(w_scale, N))) fast = false;
    if (fast && w_zp && !((w_zp->dtype == w->dtype) && (numel(w_zp) == 1 || (w_zp->ndim == 1 && w_zp->shape[0] == N)))) fast = false;
    if (fast && residual) {
        if (residual->dtype != RTEN_F32 || numel(residual) != M * N || !is_contiguous(residual)) fast = false;
    }
    if (fast) {
        QLinearLaunch L;
        L.x = (const float*)x->data;
        L.xs = xs;
        L.M = (int)M;
        L.K = (int)K;
        L.N = (int)N;
        L.has_ln = ln_scale ? 1 : 0;
        L.ln_gamma = ln_scale ? (const float*)ln_scale->data : nullptr;
        L.ln_beta = ln_bias ? (const float*)ln_bias->data : nullptr;
        L.ln_eps = ln_epsilon < 0.0f ? 1e-5f : ln_epsilon;
        L.w = pw->data;
        L.ldw = pw->ld;
        L.w_signed = pw->dtype == RTEN_I8;
        L.colsum = pw->colsum;
        L.w_scale = (const float*)w_scale->data;
        L.w_scale_len = (int)numel(w_scale);
        L.bias = bias ? (const float*)bias->data : nullptr;
        L.residual = residual ? (const float*)residual->data : nullptr;
        L.rs = N;
        L.act = activation;
        if (qlinear_supported(L)) {
            OpScope sc(ctx);
            rten_tensor ov;
            int64_t oshape[RTEN_MAX_DIMS];
            for (int i = 0; i + 1 < x->ndim; i++) oshape[i] = x->shape[i];
            oshape[x->ndim - 1] = N;
            rten_status st = sc.out(out, RTEN_F32, x->ndim, oshape, &ov, nullptr);
            if (st == RTEN_OK && !is_contiguous(&ov)) st = fail(ctx, RTEN_ERR_UNSUPPORTED_OUTPUT, "output tensor must be contiguous");
            if (st == RTEN_OK && w_zp) {
                int32_t* zb = nullptr;
                const int len = (int)numel(w_zp);
                st = temp_alloc(ctx, (size_t)len * 4, (void**)&zb);
                if (st == RTEN_OK) st = launch_zp_to_i32(ctx, w_zp->data, w_zp->dtype == RTEN_I8, len, w_zp->ndim == 0 ? 0 : w_zp->strides[0], zb);
                L.zb = zb;
                L.zb_len = len;
            }
            if (st == RTEN_OK) {
                L.out = (float*)ov.data;
                L.os = N;
                st = launch_qlinear(ctx, L);
            }
            return sc.finish(st);
        }
    }

    // ---- general path: the operator chain, through this library's own entry points
    rten_tensor h = empty_tensor(), q = empty_tensor(), qs = empty_tensor(), qz = empty_tensor();
    const rten_tensor* cur = x;
    rten_status st = RTEN_OK;
    if (ln_scale) {
        st = rten_b200_layer_norm(ctx, x, ln_scale, ln_bias, -1, ln_epsilon, &h);
        cur = &h;
    }
    if (st == RTEN_OK) st = rten_b200_dynamic_quantize_linear(ctx, cur, &q, &qs, &qz, nullptr);
    if (st == RTEN_OK) st = rten_b200_matmul_integer_ex(ctx, &q, w, pw, &qz, w_zp, w_scale, &qs, bias, residual, activation, nullptr, out);
    free_if(ctx, h);
    free_if(ctx, q);
    free_if(ctx, qs);
    free_if(ctx, qz);
    return st;
}

rten_status rten_b200_attention(rten_ctx* ctx, const rten_tensor* query, const rten_tensor* key, const rten_tensor* value,
                                const rten_tensor* attn_mask, const rten_tensor* nonpad_kv_seqlen, const rten_attention_params* prm,
                                const rten_tensor* new_key, const rten_tensor* new_value, rten_tensor* out) {
    if (!ctx) return RTEN_ERR_INVALID_VALUE;
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
    if (qs == 1 && dv == dh && resident && query->strides[3] == 1 && key->strides[3] == 1) {
        AttnDecodeLaunch L;
        L.B = (int)B;
        L.q_heads = (int)qh;
        L.kv_heads = (int)kvh;
        L.dh = (int)dh;
        L.kv_cap = (int)total;
        L.q = (const float*)query->data;
        L.q_b = query->strides[0];
        L.q_h = query->strides[1];
        L.k = (float*)key->data;
        L.k_b = key->strides[0];
        L.k_h = key->strides[1];
        L.k_l = key->strides[2];
        L.v = (float*)value->data;
        L.v_b = value->strides[0];
        L.v_h = value->strides[1];
        L.v_l = value->strides[2];
        L.v_d = value->strides[3];
        L.len = nonpad_kv_seqlen ? (const int32_t*)nonpad_kv_seqlen->data : nullptr;
        if (nonpad_kv_seqlen && nonpad_kv_seqlen->strides[0] != 1 && B > 1) L.dh = 0;  // (forces the general path)
        L.mask = attn_mask ? (const float*)attn_mask->data : nullptr;
        L.m_b = ms[0];
        L.m_h = ms[1];
        L.m_l = ms[3];
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
        if (attn_decode_supported(L)) {
            OpScope sc(ctx);
            rten_tensor ov;
            const int64_t oshape[4] = {B, qh, 1, dh};
            rten_status st = sc.out(out, RTEN_F32, 4, oshape, &ov, nullptr);
            if (st == RTEN_OK && ov.strides[3] != 1) st = fail(ctx, RTEN_ERR_UNSUPPORTED_OUTPUT, "output head dimension must be contiguous");
            if (st == RTEN_OK) {
                L.out = (float*)ov.data;
                L.o_b = ov.strides[0];
                L.o_h = ov.strides[1];
                st = launch_attn_decode(ctx, L);
            }
            return sc.finish(st);
        }
    }
    // ---- encoder shapes (128 keys, head size 64, value tensor stored transposed): one fused kernel per layer where available
    // (single-pass TF32 products: only when the context opted in to that mode)
    if (resident && ctx->f32_mode == RTEN_F32_TF32 && !new_key && !nonpad_kv_seqlen && !prm->is_causal && qh == kvh && dv == dh &&
        query->strides[3] == 1 && key->strides[3] == 1 && (value->strides[2] == 1 || value->strides[3] == 1) &&
        (!attn_mask || (ms[1] == 0 && ms[2] == 0 && (ms[3] == 1 || total == 1)))) {
        AttnFusedLaunch L;
        L.B = (int)B;
        L.heads = (int)qh;
        L.q_seq = (int)qs;
        L.kv_seq = (int)total;
        L.dh = (int)dh;
        L.q = attn_operand(query, false);
        L.k = attn_operand(key, false);
        if (value->strides[3] == 1 && value->strides[2] != 1) {  // natural layout: the kernel transposes the tile itself
            L.v = (const float*)value->data;
            L.v_b = value->strides[0];
            L.v_h = value->strides[1];
            L.v_s = value->strides[2];
        } else {
            L.vt = attn_operand(value, true);
        }
        L.mask = attn_mask ? (const float*)attn_mask->data : nullptr;
        L.m_b = ms[0];
        L.scale = scale;
        OpScope sc(ctx);
        rten_tensor ov;
        const int64_t oshape[4] = {B, qh, qs, dh};
        rten_status st = sc.out(out, RTEN_F32, 4, oshape, &ov, nullptr);
        if (st == RTEN_OK) {
            L.out = (float*)ov.data;
            L.o_b = ov.strides[0];
            L.o_h = ov.strides[1];
            L.o_s = ov.strides[2];
            if (ov.strides[3] == 1 && attn_fused_supported(L)) return sc.finish(launch_attn_fused(ctx, L));
            give_back_output(ctx, sc, out, ov);  // compose below
        }
        st = sc.finish(st);
        if (st != RTEN_OK) return st;
    }
    // ---- causal, right-padded (nonpad_kv_seqlen) or grouped-query calls with q_seq > 1: the streaming prefill kernel
    // (head size 64 / 128, f32 products in the context's mode); other layouts keep the errors below
    if (qs > 1 && resident && !new_key && (prm->is_causal || nonpad_kv_seqlen || qh != kvh) && dv == dh && (dh == 64 || dh == 128) &&
        query->strides[3] == 1 && key->strides[3] == 1 && (value->strides[2] == 1 || value->strides[3] == 1) &&
        (!attn_mask || ms[3] == 1 || total == 1) && (!nonpad_kv_seqlen || nonpad_kv_seqlen->strides[0] == 1 || B == 1)) {
        AttnPrefillLaunch L;
        L.B = (int)B;
        L.q_heads = (int)qh;
        L.kv_heads = (int)kvh;
        L.q_seq = (int)qs;
        L.kv_seq = (int)total;
        L.dh = (int)dh;
        L.q = attn_operand(query, false);
        L.k = attn_operand(key, false);
        L.v_natural = value->strides[3] == 1;
        L.v = attn_operand(value, !L.v_natural);
        L.len = nonpad_kv_seqlen ? (const int32_t*)nonpad_kv_seqlen->data : nullptr;
        L.causal = prm->is_causal ? 1 : 0;
        L.mask = attn_mask ? (const float*)attn_mask->data : nullptr;
        L.m_b = ms[0];
        L.m_h = ms[1];
        L.m_s = ms[2];
        L.scale = scale;
        L.x3 = ctx->f32_mode == RTEN_F32_TF32 ? 0 : 1;
        OpScope sc(ctx);
        rten_tensor ov;
        const int64_t oshape[4] = {B, qh, qs, dh};
        rten_status st = sc.out(out, RTEN_F32, 4, oshape, &ov, nullptr);
        if (st == RTEN_OK) {
            L.out = (float*)ov.data;
            L.o_b = ov.strides[0];
            L.o_h = ov.strides[1];
            L.o_s = ov.strides[2];
            if (ov.strides[3] == 1 && attn_prefill_supported(L)) return sc.finish(launch_attn_prefill(ctx, L));
            give_back_output(ctx, sc, out, ov);
        }
        st = sc.finish(st);
        if (st != RTEN_OK) return st;
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
    rten_tensor scores = empty_tensor();
    rten_status st = rten_b200_matmul_ex(ctx, query, &kt, nullptr, nullptr, scale, nullptr, 0, &scores);
    if (st == RTEN_OK) st = rten_b200_softmax(ctx, &scores, attn_mask, -1, 1, &scores);
    if (st == RTEN_OK) st = rten_b200_matmul(ctx, &scores, value, nullptr, nullptr, 1.0f, out);
    free_if(ctx, scores);
    return st;
}

}  // extern "C"
