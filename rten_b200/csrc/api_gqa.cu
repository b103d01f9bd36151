// Entry points of the C ABI for rotary-embedded grouped-query attention and multi-head attention (include/rten_b200.h):
//   rten_b200_rotary_embedding        : ai.onnx RotaryEmbedding (src/ops/embedding.rs:46-252)
//   rten_b200_group_query_attention   : com.microsoft GroupQueryAttention (src/ops/attention/contrib.rs:369-417,
//                                       :438-810), the attention operator of quantized decoder-only LLM exports
//   rten_b200_multi_head_attention    : com.microsoft MultiHeadAttention (src/ops/attention/contrib.rs:56-300), the
//                                       attention of ONNX Runtime's optimized encoder and encoder-decoder exports
// Validation restates the reference's checks and messages on everything the host can see.  The work runs on three
// kernels: the rotary / cache-append kernel (rotary.cu), the single-query attention kernel for a decode step
// (skinny.cu, with the rotary embedding, cache append and sliding window fused in) and the streaming prefill kernel
// (attn_prefill.cu) for prompts.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstring>
#include <string>
#include <vector>

#include "api_util.h"
#include "attn_prefill.h"
#include "rotary.h"
#include "skinny.h"

using namespace rtb;

namespace {

constexpr int GQA_DECODE_MAX_CACHE = 8192;  // the single-query kernel's 64 splits x 128 positions

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

// a [B, heads, T, D] cache as rows indexed (b, t, h)
RotaryRows cache_rows(const rten_tensor* t) {
    RotaryRows r;
    r.p = (float*)t->data;
    r.sb = t->strides[0];
    r.ss = t->strides[2];
    r.sh = t->strides[1];
    r.sd = t->strides[3];
    return r;
}

long long bstride(const rten_tensor* t, int i) { return t->shape[i] == 1 ? 0 : t->strides[i]; }

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

// position_ids held by the host: every entry must index both tables (negative entries count from the end, as Gather
// reads them); the resolved positions are staged contiguously for the kernels
rten_status stage_positions(rten_ctx* ctx, OpScope& sc, const rten_tensor* pos, int64_t cos_rows, int64_t sin_rows, rten_tensor* view) {
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

// [first, last) byte range a tensor spans
void byte_span(const rten_tensor* t, uintptr_t* a, uintptr_t* b) {
    *a = reinterpret_cast<uintptr_t>(t->data);
    *b = *a + (uintptr_t)span_elems(t) * dtype_size(t->dtype);
}

const char* const COS_LAST = "Last dimension of cos cache does not match rotary_embedding_dim/2";
const char* const SIN_LAST = "Last dimension of sin cache does not match rotary_embedding_dim/2";

}  // namespace

extern "C" {

rten_status rten_b200_rotary_embedding(rten_ctx* ctx, const rten_tensor* input, const rten_tensor* cos, const rten_tensor* sin,
                                       const rten_tensor* position_ids, int interleaved, int num_heads, int rotary_embedding_dim,
                                       rten_tensor* out) {
    if (!ctx) return RTEN_ERR_INVALID_VALUE;
    if (!input || !cos || !sin || !out) return fail(ctx, RTEN_ERR_MISSING_INPUTS, "missing inputs");
    if (input->dtype != RTEN_F32 || cos->dtype != RTEN_F32 || sin->dtype != RTEN_F32 || (position_ids && position_ids->dtype != RTEN_I32))
        return fail(ctx, RTEN_ERR_UNSUPPORTED_TYPE, "unsupported type");
    // [batch, seq, heads, head_size] view of the input
    int64_t B, S, H, D;
    RotaryRows x;
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
    rten_status st = sc.in(input, &xv);
    if (st == RTEN_OK) st = sc.in(cos, &cv);
    if (st == RTEN_OK) st = sc.in(sin, &sv);
    if (st != RTEN_OK) return sc.finish(st);
    RotaryTable tab;
    tab.half = (int)half;
    tab.interleaved = interleaved ? 1 : 0;
    if (position_ids) {
        // the caches are gathered by position: [max_pos, half] tables, gathered to [pb, ps, half]
        if (position_ids->ndim != 2) return sc.finish(rank_fail(ctx, 3, 2, position_ids->ndim));
        if (cos->ndim != 2 || sin->ndim != 2) return sc.finish(fail(ctx, RTEN_ERR_INVALID_VALUE, "cos/sin cache must be a 3D tensor"));
        if (position_ids->device < 0) {
            st = stage_positions(ctx, sc, position_ids, cos->shape[0], sin->shape[0], &pv);
        } else {
            st = sc.in(position_ids, &pv);
        }
        if (st != RTEN_OK) return sc.finish(st);
        const int64_t gc[3] = {position_ids->shape[0], position_ids->shape[1], cos->shape[1]};
        const int64_t gs[3] = {position_ids->shape[0], position_ids->shape[1], sin->shape[1]};
        st = cache_dims(ctx, 3, gc, B, S, half, COS_LAST);
        if (st == RTEN_OK) st = cache_dims(ctx, 3, gs, B, S, half, SIN_LAST);
        if (st == RTEN_OK && (cos->shape[0] < 1 || sin->shape[0] < 1)) st = fail(ctx, RTEN_ERR_INVALID_VALUE, "Entry in `indices` is out of range");
        if (st != RTEN_OK) return sc.finish(st);
        rten_tensor cc, scc;
        st = sc.contiguous(&cv, &cc);
        if (st == RTEN_OK) st = sc.contiguous(&sv, &scc);
        if (st != RTEN_OK) return sc.finish(st);
        tab.cos = (const float*)cc.data;
        tab.sin = (const float*)scc.data;
        tab.by_pos = 1;
        tab.max_pos = (int)std::min(cos->shape[0], sin->shape[0]);
        tab.pos = (const int32_t*)pv.data;
        tab.p_b = bstride(&pv, 0);
        tab.p_s = bstride(&pv, 1);
    } else {
        st = cache_dims(ctx, cos->ndim, cos->shape, B, S, half, COS_LAST);
        if (st == RTEN_OK) st = cache_dims(ctx, sin->ndim, sin->shape, B, S, half, SIN_LAST);
        if (st != RTEN_OK) return sc.finish(st);
        rten_tensor cc = cv, scc = sv;
        if (cv.strides[2] != 1 && half > 1) st = sc.contiguous(&cv, &cc);
        if (st == RTEN_OK && sv.strides[2] != 1 && half > 1) st = sc.contiguous(&sv, &scc);
        if (st != RTEN_OK) return sc.finish(st);
        tab.cos = (const float*)cc.data;
        tab.sin = (const float*)scc.data;
        tab.c_b = bstride(&cc, 0);
        tab.c_s = bstride(&cc, 1);
        tab.s_b = bstride(&scc, 0);
        tab.s_s = bstride(&scc, 1);
    }
    rten_tensor ov;
    st = sc.out(out, RTEN_F32, input->ndim, input->shape, &ov, nullptr);
    if (st != RTEN_OK) return sc.finish(st);
    if (input->ndim == 3) {
        x = rows3(&xv, D, 0);
    } else {
        x = cache_rows(&xv);
    }
    RotaryLaunch L;
    L.B = (int)B;
    L.S = (int)S;
    L.H = (int)H;
    L.D = (int)D;
    L.rot = tab;
    L.x = x;
    L.y = input->ndim == 3 ? rows3(&ov, D, 0) : cache_rows(&ov);
    if (B * S * H * D > 0) st = launch_rotary(ctx, L);
    return sc.finish(st);
}

rten_status rten_b200_group_query_attention(rten_ctx* ctx, const rten_tensor* query, const rten_tensor* key, const rten_tensor* value,
                                            const rten_tensor* past_key, const rten_tensor* past_value, const rten_tensor* seqlens_k,
                                            const rten_tensor* total_sequence_length, const rten_tensor* cos, const rten_tensor* sin,
                                            const rten_tensor* position_ids, const rten_tensor* attention_bias, const rten_gqa_params* prm,
                                            rten_tensor* out, rten_tensor* present_key, rten_tensor* present_value) {
    if (!ctx) return RTEN_ERR_INVALID_VALUE;
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
    if (decode && T > GQA_DECODE_MAX_CACHE)
        return fail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "GroupQueryAttention: a decode step takes at most 8192 cache positions (past + 1)");

    // ---- device views
    // an aliased present cache is the past buffer itself (same data and strides) with room for the new positions
    auto aliased = [&](const rten_tensor* pres, const rten_tensor* past) {
        if (!past || !pres->data || pres->data != past->data || pres->device < 0 || past->device < 0 || pres->ndim != 4) return false;
        for (int i = 0; i < 4; i++)
            if (pres->strides[i] != past->strides[i]) return false;
        return true;
    };
    const bool alias_k = aliased(present_key, past_key), alias_v = aliased(present_value, past_value);
    // a present cache in the memory of a past cache without being that same buffer would be read and written by one
    // kernel at once
    for (const rten_tensor* pres : {present_key, present_value})
        for (const rten_tensor* past : {past_key, past_value}) {
            if (!past || !pres->data || pres->device < 0 || past->device < 0 || (pres == present_key ? alias_k : alias_v)) continue;
            if (pres->data == past->data && aliased(pres, past)) continue;
            uintptr_t a0, a1, b0, b1;
            rten_tensor pshape = *pres;
            pshape.ndim = 4;
            pshape.shape[0] = B;
            pshape.shape[1] = Hkv;
            pshape.shape[2] = T;
            pshape.shape[3] = D;
            byte_span(&pshape, &a0, &a1);
            byte_span(past, &b0, &b1);
            if (a0 < b1 && b0 < a1)
                return fail(ctx, RTEN_ERR_UNSUPPORTED_OUTPUT,
                            "GroupQueryAttention: present_key / present_value overlap a past cache without being that buffer (same data and strides)");
        }
    OpScope sc(ctx);
    rten_tensor qv, kv, vv, pkv, pvv, slv, cv, snv, posv, biasv;
    rten_status st = sc.in(query, &qv);
    if (st == RTEN_OK && key) st = sc.in(key, &kv);
    if (st == RTEN_OK && value) st = sc.in(value, &vv);
    if (st == RTEN_OK && past_key) st = sc.in(past_key, &pkv);
    if (st == RTEN_OK && past_value) st = sc.in(past_value, &pvv);
    if (st == RTEN_OK) st = sc.in(seqlens_k, &slv);
    if (st == RTEN_OK && attention_bias) {
        st = sc.in(attention_bias, &biasv);
        if (st == RTEN_OK && biasv.strides[3] != 1 && biasv.shape[3] > 1) {
            rten_tensor c;
            st = sc.contiguous(&biasv, &c);
            biasv = c;
        }
    }
    RotaryTable tab;
    if (st == RTEN_OK && prm->do_rotary) {
        st = sc.in(cos, &cv);
        if (st == RTEN_OK) st = sc.in(sin, &snv);
        rten_tensor cc, scc;
        if (st == RTEN_OK) st = sc.contiguous(&cv, &cc);
        if (st == RTEN_OK) st = sc.contiguous(&snv, &scc);
        if (st == RTEN_OK && position_ids)
            st = position_ids->device < 0 ? stage_positions(ctx, sc, position_ids, cos->shape[0], sin->shape[0], &posv) : sc.in(position_ids, &posv);
        if (st == RTEN_OK && position_ids) {
            const int64_t gc[3] = {position_ids->shape[0], position_ids->shape[1], half};
            st = cache_dims(ctx, 3, gc, B, S, half, COS_LAST);
        }
        if (st == RTEN_OK && cos->shape[1] != half) st = fail(ctx, RTEN_ERR_INVALID_VALUE, COS_LAST);
        if (st == RTEN_OK && sin->shape[1] != half) st = fail(ctx, RTEN_ERR_INVALID_VALUE, SIN_LAST);
        if (st == RTEN_OK && (cos->shape[0] < 1 || sin->shape[0] < 1)) st = fail(ctx, RTEN_ERR_INVALID_VALUE, "Entry in `indices` is out of range");
        tab.cos = (const float*)cc.data;
        tab.sin = (const float*)scc.data;
        tab.half = (int)half;
        tab.interleaved = prm->rotary_interleaved ? 1 : 0;
        tab.by_pos = 1;
        tab.max_pos = (int)std::min(cos->shape[0], sin->shape[0]);
        if (position_ids) {
            tab.pos = (const int32_t*)posv.data;
            tab.p_b = bstride(&posv, 0);
            tab.p_s = bstride(&posv, 1);
        }
    }
    rten_tensor ov, pk, pv;
    const int64_t oshape[3] = {B, S, H * D}, cshape[4] = {B, Hkv, T, D};
    if (st == RTEN_OK) st = sc.out(out, RTEN_F32, 3, oshape, &ov, nullptr);
    if (st == RTEN_OK) st = sc.out(present_key, RTEN_F32, 4, cshape, &pk, nullptr);
    if (st == RTEN_OK) st = sc.out(present_value, RTEN_F32, 4, cshape, &pv, nullptr);
    if (st == RTEN_OK && (ov.strides[2] != 1 || pk.strides[3] != 1 || pv.strides[3] != 1))
        st = fail(ctx, RTEN_ERR_UNSUPPORTED_OUTPUT, "GroupQueryAttention: the outputs need a contiguous last dimension");
    if (st != RTEN_OK) return sc.finish(st);
    if (B * S == 0 || H * D == 0) return sc.finish(RTEN_OK);

    const RotaryRows qr = rows3(&qv, D, 0);
    const RotaryRows kr = packed ? rows3(&qv, D, H) : rows3(&kv, D, 0);
    const RotaryRows vr = packed ? rows3(&qv, D, H + Hkv) : rows3(&vv, D, 0);
    const int window = prm->local_window_size > 0 ? prm->local_window_size : 0;
    RotaryLaunch R;  // the rotary / append kernel's common fields
    R.B = (int)B;
    R.S = (int)S;
    R.D = (int)D;
    R.H = (int)H;
    R.Hkv = (int)Hkv;
    R.T = (int)T;
    R.rot = tab;
    R.k_cache = cache_rows(&pk);
    R.v_cache = cache_rows(&pv);
    R.seqlens = (const int32_t*)slv.data;
    R.sl_s = slv.strides[0];
    R.first = first ? 1 : 0;
    // the present caches' past prefix and zero tail, unless the present cache is the past buffer (or there is no past)
    RotaryLaunch Rb = R;
    Rb.build_k = !alias_k;
    Rb.build_v = !alias_v;
    if (past_key) {
        Rb.k_past = cache_rows(&pkv);
        Rb.v_past = cache_rows(&pvv);
    }
    const bool build = P > 0 && (Rb.build_k || Rb.build_v);

    if (decode) {
        AttnDecodeLaunch L;
        L.B = (int)B;
        L.q_heads = (int)H;
        L.kv_heads = (int)Hkv;
        L.dh = (int)D;
        L.kv_cap = (int)T;
        L.q = qr.p;
        L.q_b = qr.sb;
        L.q_h = qr.sh;
        L.k = (float*)pk.data;
        L.k_b = pk.strides[0];
        L.k_h = pk.strides[1];
        L.k_l = pk.strides[2];
        L.v = (float*)pv.data;
        L.v_b = pv.strides[0];
        L.v_h = pv.strides[1];
        L.v_l = pv.strides[2];
        L.v_d = pv.strides[3];
        L.len = (const int32_t*)slv.data;
        L.len_s = slv.strides[0];
        L.len_add = 1;
        L.len_min = 1;
        L.window = window;
        if (attention_bias) {
            L.mask = (const float*)biasv.data;
            L.m_b = bstride(&biasv, 0);
            L.m_h = bstride(&biasv, 1);
            L.m_l = biasv.strides[3];
        }
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
        L.out = (float*)ov.data;
        L.o_b = ov.strides[0];
        L.o_h = D;
        if (qr.sd == 1 && kr.sd == 1 && vr.sd == 1 && attn_decode_supported(L)) {
            if (build) st = launch_rotary(ctx, Rb);
            if (st == RTEN_OK) st = launch_attn_decode(ctx, L);
            return sc.finish(st);
        }
        // (a layout the single-query kernel cannot read: the prompt path below serves one query as well)
    }

    // ---- prompt: rotary + append, then the streaming prefill kernel over the present caches
    void* qs = nullptr;
    void* le = nullptr;
    st = temp_alloc(ctx, (size_t)(B * S * H * D) * 4, &qs);
    if (st == RTEN_OK) st = temp_alloc(ctx, (size_t)B * 4, &le);
    if (st != RTEN_OK) return sc.finish(st);
    R.x = qr;
    R.y.p = (float*)qs;
    R.y.sb = S * H * D;
    R.y.ss = H * D;
    R.y.sh = D;
    R.y.sd = 1;
    R.k_new = kr;
    R.v_new = vr;
    R.len_eff = (int32_t*)le;
    AttnPrefillLaunch A;
    A.B = (int)B;
    A.q_heads = (int)H;
    A.kv_heads = (int)Hkv;
    A.q_seq = (int)S;
    A.kv_seq = (int)T;
    A.dh = (int)D;
    A.q.base = qs;
    A.q.dims[0] = D;
    A.q.dims[1] = S;
    A.q.dims[2] = H;
    A.q.dims[3] = B;
    A.q.strides[0] = 1;
    A.q.strides[1] = H * D;
    A.q.strides[2] = D;
    A.q.strides[3] = S * H * D;
    auto cache_desc = [](const rten_tensor& t) {
        OperandDesc d;
        d.base = t.data;
        d.dims[0] = t.shape[3];
        d.dims[1] = t.shape[2];
        d.dims[2] = t.shape[1];
        d.dims[3] = t.shape[0];
        d.strides[0] = 1;
        d.strides[1] = t.strides[2];
        d.strides[2] = t.strides[1];
        d.strides[3] = t.strides[0];
        return d;
    };
    A.k = cache_desc(pk);
    A.v = cache_desc(pv);
    A.v_natural = true;
    A.len = (const int32_t*)le;
    A.causal = 1;
    A.window = window;
    if (attention_bias) {
        A.mask = (const float*)biasv.data;
        A.m_b = bstride(&biasv, 0);
        A.m_h = bstride(&biasv, 1);
        A.m_s = biasv.strides[2];
    }
    A.scale = scale;
    A.x3 = ctx->f32_mode == RTEN_F32_TF32 ? 0 : 1;
    A.out = (float*)ov.data;
    A.o_b = ov.strides[0];
    A.o_h = D;
    A.o_s = ov.strides[1];
    if (!attn_prefill_supported(A))
        return sc.finish(fail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "GroupQueryAttention: the present caches and the output need 16-byte aligned rows"));
    if (build) st = launch_rotary(ctx, Rb);
    if (st == RTEN_OK) st = launch_rotary(ctx, R);
    if (st == RTEN_OK) st = launch_attn_prefill(ctx, A);
    return sc.finish(st);
}

rten_status rten_b200_multi_head_attention(rten_ctx* ctx, const rten_tensor* query, const rten_tensor* key, const rten_tensor* value,
                                           const rten_tensor* bias, const rten_tensor* key_padding_mask, const rten_tensor* attention_bias,
                                           const rten_tensor* past_key, const rten_tensor* past_value, const rten_tensor* past_sequence_length,
                                           const rten_tensor* cache_indirection, const rten_mha_params* prm, rten_tensor* out,
                                           rten_tensor* present_key, rten_tensor* present_value) {
    if (!ctx) return RTEN_ERR_INVALID_VALUE;
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

    // ---- present caches: the past buffer itself (in place), new memory, or refused when they overlap a past cache
    auto aliased = [&](const rten_tensor* pres, const rten_tensor* past) {
        if (!pres || !past || !pres->data || pres->data != past->data || pres->device < 0 || past->device < 0 || pres->ndim != 4) return false;
        for (int i = 0; i < 4; i++)
            if (pres->strides[i] != past->strides[i]) return false;
        return true;
    };
    const bool alias_k = aliased(present_key, past_key), alias_v = aliased(present_value, past_value);
    for (const rten_tensor* pres : {present_key, present_value})
        for (const rten_tensor* past : {past_key, past_value}) {
            if (!pres || !past || !pres->data || pres->device < 0 || past->device < 0 || aliased(pres, past)) continue;
            uintptr_t a0, a1, b0, b1;
            rten_tensor pshape = *pres;
            pshape.ndim = 4;
            pshape.shape[0] = B;
            pshape.shape[1] = H;
            pshape.shape[2] = T;
            pshape.shape[3] = D;
            byte_span(&pshape, &a0, &a1);
            byte_span(past, &b0, &b1);
            if (a0 < b1 && b0 < a1)
                return fail(ctx, RTEN_ERR_UNSUPPORTED_OUTPUT,
                            "MultiHeadAttention: present_key / present_value overlap a past cache without being that buffer (same data and strides)");
        }

    // ---- device views (head dimension contiguous)
    OpScope sc(ctx);
    auto view = [&](const rten_tensor* t, rten_tensor* v) {
        rten_status s = sc.in(t, v);
        if (s == RTEN_OK && v->strides[v->ndim - 1] != 1 && v->shape[v->ndim - 1] > 1) {
            rten_tensor c;
            s = sc.contiguous(v, &c);
            *v = c;
        }
        return s;
    };
    rten_tensor qv, kv, vv, bv, mv, abv, pkv, pvv;
    rten_status st = view(query, &qv);
    if (st == RTEN_OK && key) st = view(key, &kv);
    if (st == RTEN_OK && key) st = view(value, &vv);
    if (st == RTEN_OK && bias) st = view(bias, &bv);
    if (st == RTEN_OK && key_padding_mask) st = view(key_padding_mask, &mv);
    if (st == RTEN_OK && attention_bias) st = sc.in(attention_bias, &abv);
    if (st == RTEN_OK && past_key) st = view(past_key, &pkv);
    if (st == RTEN_OK && past_value) st = view(past_value, &pvv);
    rten_tensor ov, pk, pv;
    const int64_t oshape[3] = {B, S, H * D}, cshape[4] = {B, H, T, D};
    if (st == RTEN_OK) st = sc.out(out, RTEN_F32, 3, oshape, &ov, nullptr);
    if (st == RTEN_OK && present_key) st = sc.out(present_key, RTEN_F32, 4, cshape, &pk, nullptr);
    if (st == RTEN_OK && present_value) st = sc.out(present_value, RTEN_F32, 4, cshape, &pv, nullptr);
    if (st == RTEN_OK && (ov.strides[2] != 1 || (present_key && pk.strides[3] != 1) || (present_value && pv.strides[3] != 1)))
        st = fail(ctx, RTEN_ERR_UNSUPPORTED_OUTPUT, "MultiHeadAttention: the outputs need a contiguous last dimension");
    if (st != RTEN_OK) return sc.finish(st);
    if (B * S == 0) return sc.finish(RTEN_OK);

    // head rows (b, s, h, i) of q and of the new k / v
    RotaryRows qr, kr, vr;
    if (packed) {
        auto comp = [&](int c) {
            RotaryRows r;
            r.p = (float*)qv.data + c * qv.strides[3];
            r.sb = qv.strides[0];
            r.ss = qv.strides[1];
            r.sh = qv.strides[2];
            r.sd = qv.strides[4];
            return r;
        };
        qr = comp(0);
        kr = comp(1);
        vr = comp(2);
    } else {
        qr = rows3(&qv, D, 0);
        kr = key ? rows3(&kv, D, 0) : qr;
        vr = key ? rows3(&vv, D, 0) : qr;
    }
    // prep (one rotary / append launch) when there is a bias to add or a cache to build; else q / k / v are read in place
    const bool prep = bias || P > 0 || present_key || present_value;
    RotaryRows qa = qr;    // what the attention kernel reads
    RotaryRows kc, vc;     // [B, H, T, D] caches as rows (b, t, h) when prepped
    RotaryLaunch R;
    if (prep) {
        auto scratch = [&](size_t n, void** p) { return temp_alloc(ctx, n * 4, p); };
        void* qs = nullptr;
        void* ks = nullptr;
        void* vs = nullptr;
        const size_t ncache = (size_t)(B * H * T * D);
        if (bias) st = scratch((size_t)(B * S * H * D), &qs);
        if (st == RTEN_OK && !present_key) st = scratch(ncache, &ks);
        if (st == RTEN_OK && !present_value) st = scratch(ncache, &vs);
        if (st != RTEN_OK) return sc.finish(st);
        auto dense_cache = [&](void* p) {
            RotaryRows r;
            r.p = (float*)p;
            r.sb = H * T * D;
            r.ss = D;
            r.sh = T * D;
            r.sd = 1;
            return r;
        };
        kc = present_key ? cache_rows(&pk) : dense_cache(ks);
        vc = present_value ? cache_rows(&pv) : dense_cache(vs);
        R.B = (int)B;
        R.S = (int)S;
        R.D = (int)D;
        R.H = (int)H;
        R.Hkv = (int)H;
        R.T = (int)T;
        if (bias) {
            R.x = qr;
            R.y.p = (float*)qs;
            R.y.sb = S * H * D;
            R.y.ss = H * D;
            R.y.sh = D;
            R.y.sd = 1;
            qa = R.y;
            const float* bb = (const float*)bv.data;
            R.x_bias = bb;
            R.k_bias = bb + hidden;
            R.v_bias = bb + 2 * hidden;
        }
        R.k_new = kr;
        R.v_new = vr;
        R.k_cache = kc;
        R.v_cache = vc;
        R.build_k = P > 0 && !alias_k;
        R.build_v = P > 0 && !alias_v;
        if (P > 0) {
            R.k_past = cache_rows(&pkv);
            R.v_past = cache_rows(&pvv);
        }
        R.mha = 1;
        R.S_kv = (int)L;
        R.past = (int)P;
    } else {
        kc = kr;  // (b, t, h) rows of the inputs: T = L
        vc = vr;
    }
    const int32_t* kpm_d = key_padding_mask ? (const int32_t*)mv.data : nullptr;
    const long long kpm_b = key_padding_mask ? mv.strides[0] : 0;
    const float fill = prm->mask_filter_value;

    if (S == 1) {
        AttnDecodeLaunch A;
        A.B = (int)B;
        A.q_heads = (int)H;
        A.kv_heads = (int)H;
        A.dh = (int)D;
        A.kv_cap = (int)T;
        A.q = qa.p;
        A.q_b = qa.sb;
        A.q_h = qa.sh;
        A.k = kc.p;
        A.k_b = kc.sb;
        A.k_h = kc.sh;
        A.k_l = kc.ss;
        A.v = vc.p;
        A.v_b = vc.sb;
        A.v_h = vc.sh;
        A.v_l = vc.ss;
        A.v_d = 1;
        if (attention_bias) {
            A.mask = (const float*)abv.data;
            A.m_b = bstride(&abv, 0);
            A.m_h = bstride(&abv, 1);
            A.m_l = bstride(&abv, 3);
        }
        A.scale = scale;
        A.out = (float*)ov.data;
        A.o_b = ov.strides[0];
        A.o_h = D;
        A.mha = 1;
        A.vis_end = prm->unidirectional ? (int)P + 1 : (int)T;
        A.fill = fill;
        A.kpm = kpm_d;
        A.kpm_b = kpm_b;
        if (attn_decode_supported(A)) {
            if (prep) st = launch_rotary(ctx, R);
            if (st == RTEN_OK) st = launch_attn_decode(ctx, A);
            return sc.finish(st);
        }
        // (a cache longer than the single-query kernel takes: the prefill kernel serves one query as well)
    }
    auto rows_desc = [](const RotaryRows& r, int64_t D_, int64_t n, int64_t heads, int64_t batch) {
        OperandDesc d;
        d.base = r.p;
        d.dims[0] = D_;
        d.dims[1] = n;
        d.dims[2] = heads;
        d.dims[3] = batch;
        d.strides[0] = 1;
        d.strides[1] = r.ss;
        d.strides[2] = r.sh;
        d.strides[3] = r.sb;
        return d;
    };
    AttnPrefillMha M;
    M.causal_offset = (int)P;
    M.fill = fill;
    M.kpm = kpm_d;
    M.kpm_b = kpm_b;
    M.v_rows = vc.p;
    M.v_b = vc.sb;
    M.v_h = vc.sh;
    M.v_t = vc.ss;
    AttnPrefillLaunch A;
    A.B = (int)B;
    A.q_heads = (int)H;
    A.kv_heads = (int)H;
    A.q_seq = (int)S;
    A.kv_seq = (int)T;
    A.dh = (int)D;
    A.q = rows_desc(qa, D, S, H, B);
    A.k = rows_desc(kc, D, T, H, B);
    A.v = rows_desc(vc, D, T, H, B);
    A.v_natural = true;
    A.causal = prm->unidirectional ? 1 : 0;
    if (attention_bias) {
        A.mask = (const float*)abv.data;
        A.m_b = bstride(&abv, 0);
        A.m_h = bstride(&abv, 1);
        A.m_s = bstride(&abv, 2);
        M.m_t = bstride(&abv, 3);
    }
    A.scale = scale;
    A.x3 = ctx->f32_mode == RTEN_F32_TF32 ? 0 : 1;
    A.out = (float*)ov.data;
    A.o_b = ov.strides[0];
    A.o_h = D;
    A.o_s = ov.strides[1];
    A.mha = &M;
    if (qa.sd != 1 || kc.sd != 1 || vc.sd != 1 || !attn_prefill_supported(A))
        return sc.finish(fail(ctx, RTEN_ERR_UNSUPPORTED_VALUE,
                              "MultiHeadAttention: query, key, value, the caches and the output need 16-byte aligned rows"));
    if (prep) st = launch_rotary(ctx, R);
    if (st == RTEN_OK) st = launch_attn_prefill(ctx, A);
    return sc.finish(st);
}

}  // extern "C"
