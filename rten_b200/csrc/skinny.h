// Launchers of the skinny-M (M <= 32) kernels of skinny.cu: HBM-streaming vector-matrix products for autoregressive
// decode (rten-gemm's gemv path, rten-gemm/src/lib.rs:668-747, kernels rten-gemm/src/kernels/simd_generic.rs:14-197 f32,
// :795-1129 int8) with the operators around them fused in, and single-query attention over a KV cache
// (src/ops/attention.rs:518-560 sdpa_head, :645-905 Attention with an externally managed cache).
#pragma once
#include <cstdint>

#include "common.h"

namespace rtb {

// [LayerNormalization] -> DynamicQuantizeLinear -> Mul(x_scale, w_scale) -> MatMulIntegerToFloat -> Add(bias) ->
// Add(residual) -> activation, for an f32 input of M <= 16 rows.  Every stage performs the same exactly rounded
// operations as the separate operators (bit-identical results).
struct QLinearLaunch {
    const float* x = nullptr;  // [M, K], row stride xs (elements), 16-byte aligned rows
    long long xs = 0;
    int M = 0, K = 0, N = 0;
    int has_ln = 0;  // LayerNormalization over the last axis first (gamma required, beta optional)
    const float* ln_gamma = nullptr;
    const float* ln_beta = nullptr;
    float ln_eps = 1e-5f;
    const void* w = nullptr;  // [N, ldw] 8-bit, K-major (rten_b200_prepack_b layout)
    long long ldw = 0;
    int w_signed = 1;
    const int32_t* colsum = nullptr;  // sum_k w[n, k]
    const int32_t* zb = nullptr;      // weight zero point(s) as i32: scalar or [N]; null = 0
    int zb_len = 0;
    const float* w_scale = nullptr;  // scalar or [N]
    int w_scale_len = 0;
    const float* bias = nullptr;      // [N] or null
    const float* residual = nullptr;  // [M, N] (row stride rs) or null
    long long rs = 0;
    int act = 0;
    float* out = nullptr;  // [M, N], row stride os
    long long os = 0;
};
// true if the fused kernel can serve the problem (M <= 16, K % 16 == 0, alignment, LayerNorm width limits)
bool qlinear_supported(const QLinearLaunch& L);
rten_status launch_qlinear(rten_ctx* ctx, const QLinearLaunch& L);

// D[m, n] = act(alpha * sum_k A[m, k] * B[n, k] + bias[n] + residual[m, n]) in exact f32 FMA arithmetic, M <= 32.
struct SkinnyF32Launch {
    const float* a = nullptr;  // [M, K] row stride as, 16-byte aligned rows
    long long as = 0;
    const float* b = nullptr;  // [N, K] K-major, row stride bs
    long long bs = 0;
    int M = 0, N = 0, K = 0;
    float alpha = 1.0f;
    const float* bias = nullptr;  // [N] or null
    const float* residual = nullptr;
    long long rs = 0;
    float r_scale = 1.0f;
    int act = 0;
    float* out = nullptr;
    long long os = 0;
};
bool skinny_f32_supported(const SkinnyF32Launch& L);
rten_status launch_skinny_f32(rten_ctx* ctx, const SkinnyF32Launch& L);

// Single-query attention (q_seq = 1) over a cache of `kv_cap` positions of which len[b] are valid:
//   out[b, h, :] = softmax(scale * q[b, h, :] . K[b, hk, l, :] (+ mask[b, h, l]))_{l < len[b]} . V[b, hk, l, :]
// Optional fused cache append: k_new / v_new [B, kv_heads, dh] are written at position len[b] - 1 first, k_new rotated
// like q when a rotary table is given.
struct AttnDecodeCore {
    int B = 0, q_heads = 0, kv_heads = 0, dh = 0, kv_cap = 0;
    const float* q = nullptr;  // element strides: q_b, q_h (dh contiguous)
    long long q_b = 0, q_h = 0;
    float* k = nullptr;  // cache: strides k_b, k_h, k_l (dh contiguous)
    long long k_b = 0, k_h = 0, k_l = 0;
    float* v = nullptr;  // cache: strides v_b, v_h, v_l, v_d  (v_l == 1: transposed cache [.., dh, cap]; v_d == 1: natural)
    long long v_b = 0, v_h = 0, v_l = 0, v_d = 0;
    const int32_t* len = nullptr;  // [B] valid positions INCLUDING the appended one; null = kv_cap for every batch
    const float* mask = nullptr;   // additive, strides m_b, m_h, m_l (0 = broadcast) or null
    long long m_b = 0, m_h = 0, m_l = 0;
    const float* k_new = nullptr;  // strides kn_b, kn_h
    long long kn_b = 0, kn_h = 0;
    const float* v_new = nullptr;
    long long vn_b = 0, vn_h = 0;
    float scale = 1.0f;
    float* out = nullptr;  // strides o_b, o_h (dh contiguous)
    long long o_b = 0, o_h = 0;
};
// GroupQueryAttention's additions; with their defaults the plain kernel runs, compiled from the same code as before
struct AttnDecodeExt {
    long long len_s = 1;           // element stride of len
    int len_add = 0, len_min = 0;  // valid positions = clamp(len[b * len_s] + len_add, len_min, kv_cap)
    int window = 0;                // > 0: positions below (valid positions) - window are masked (natural value layout only)
    // rotary embedding of q and k_new at position rot_pos[b * rot_pos_b] (null: valid positions - 1), clamped to
    // [0, rot_max_pos - 1]; rot_cos / rot_sin [rot_max_pos, rot_half] contiguous, null = no rotation
    const float* rot_cos = nullptr;
    const float* rot_sin = nullptr;
    int rot_half = 0, rot_interleaved = 0, rot_max_pos = 0;
    const int32_t* rot_pos = nullptr;
    long long rot_pos_b = 0;
    // MultiHeadAttention (mha = 1, none of the fields above): positions l >= vis_end, and positions whose
    // kpm[b * kpm_b + l] is 0, score `fill` in place of scale * q.k + mask
    int mha = 0;
    int vis_end = 0;
    float fill = 0.0f;
    const int32_t* kpm = nullptr;
    long long kpm_b = 0;
};
struct AttnDecodeLaunch : AttnDecodeCore, AttnDecodeExt {};
constexpr int ATTN_DECODE_MAX_CACHE = 8192;  // kv_cap limit: 64 splits of the kernel's 128-position chunks
bool attn_decode_supported(const AttnDecodeLaunch& L);
rten_status launch_attn_decode(rten_ctx* ctx, const AttnDecodeLaunch& L);

}  // namespace rtb
