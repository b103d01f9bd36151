// Launcher of the streaming prefill attention kernel (attn_prefill.cu): the ONNX Attention operator for q_seq >= 2 with
// causal masking, a right-padded KV cache (nonpad_kv_seqlen) and grouped-query heads, scores kept on chip.
#pragma once
#include <cstdint>

#include "umma_gemm.h"

namespace rtb {

// out[b, h, s, :] = softmax_t(scale * Q[b, h, s] . K[b, hk, t] + mask[b, h, s, t], masked t -> -inf) . V[b, hk, t, :]
// with hk = h / (q_heads / kv_heads), the NaN of a fully masked row flushed to 0, and t masked when
//   t >= valid_b                  (valid_b = clamp(len[b], 0, kv_seq), or kv_seq when len is null), or
//   t > s + offset, causal only   (offset = valid_b - q_seq with len, 0 without).
// com.microsoft MultiHeadAttention's scores (contrib.rs:56-300): every key t < kv_seq exists; after the bias, a key is
// MASKED -- its score replaced by the finite `fill`, so it still counts in the softmax -- when t > s + causal_offset
// (causal) or key_padding_mask[b, t] == 0.  The value rows (the same tensor as `v`) are read again with plain loads
// for the keys above every row's causal diagonal when their weight e^(fill - row max) is not zero.
struct AttnPrefillMha {
    int causal_offset = 0;
    float fill = -10000.0f;
    const int32_t* kpm = nullptr;  // key_padding_mask i32 [B, kv_seq] (row stride kpm_b, keys contiguous) or null
    long long kpm_b = 0;
    long long m_t = 1;             // the mask's key stride (0: broadcast over keys)
    const float* v_rows = nullptr;  // value element (b, kv_h, t, d) at v_rows + b v_b + kv_h v_h + t v_t + d
    long long v_b = 0, v_h = 0, v_t = 0;
};

struct AttnPrefillLaunch {
    int B = 0, q_heads = 0, kv_heads = 0, q_seq = 0, kv_seq = 0, dh = 0;
    OperandDesc q;  // (d, s, h, b): head dimension contiguous
    OperandDesc k;  // (d, t, kv_h, b)
    OperandDesc v;  // v_natural: (d, t, kv_h, b); else (t, d, kv_h, b), the value tensor stored transposed
    bool v_natural = true;
    const int32_t* len = nullptr;  // nonpad_kv_seqlen [B] (read on the device) or null
    int causal = 0;
    int window = 0;  // > 0: keys t < s + offset + 1 - window are masked too (sliding window; key tiles wholly below skipped)
    const float* mask = nullptr;  // additive, element strides m_b / m_h / m_s (0 = broadcast), key dimension contiguous
    long long m_b = 0, m_h = 0, m_s = 0;
    float scale = 1.0f;
    int x3 = 1;  // 1: both products in 3xTF32 (lo*hi + hi*lo + hi*hi); 0: one TF32 pass
    float* out = nullptr;  // element strides o_b, o_h, o_s; head dimension contiguous
    long long o_b = 0, o_h = 0, o_s = 0;
    const AttnPrefillMha* mha = nullptr;  // set: MultiHeadAttention masking (no len, no window, natural value layout)
};
bool attn_prefill_supported(const AttnPrefillLaunch& L);
rten_status launch_attn_prefill(rten_ctx* ctx, const AttnPrefillLaunch& L);

}  // namespace rtb
