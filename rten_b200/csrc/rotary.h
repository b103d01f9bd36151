// Launcher of the rotary embedding / KV-cache append kernel (rotary.cu): ai.onnx RotaryEmbedding
// (src/ops/embedding.rs:46-252) and the steps of com.microsoft GroupQueryAttention around its attention kernel
// (src/ops/attention/contrib.rs:369-417 gqa_present_cache, :438-810 run_impl): rotary of Q and of the new K, the new
// tokens written into the present caches, and the present caches' past prefix and zero tail.
#pragma once
#include <cstdint>

#include "common.h"

namespace rtb {

// Element (b, s, h, i) of a strided tensor of head rows lies at p + b * sb + s * ss + h * sh + i * sd.
struct RotaryRows {
    float* p = nullptr;
    long long sb = 0, ss = 0, sh = 0, sd = 1;
};

// Where the cos / sin entries of row (b, s) come from.
struct RotaryTable {
    const float* cos = nullptr;  // null: rows are copied unrotated
    const float* sin = nullptr;
    int half = 0;  // rotary_dim / 2
    int interleaved = 0;
    // by_pos = 0: cos + b * c_b + s * c_s and sin + b * s_b + s * s_s (0 strides broadcast), entries contiguous
    long long c_b = 0, c_s = 0, s_b = 0, s_s = 0;
    // by_pos = 1: row q of [max_pos, half] tables, q = pos[b * p_b + s * p_s] if pos, else past_len(b) + s, clamped to
    // [0, max_pos - 1] on the device
    int by_pos = 0, max_pos = 0;
    const int32_t* pos = nullptr;
    long long p_b = 0, p_s = 0;
};

// One launch, one warp per head row, over up to five row streams (a null pointer turns its stream off):
//   x -> y        [B, S, H, D]: rotated (RotaryEmbedding, GroupQueryAttention's Q)
//   k_new -> k_cache, v_new -> v_cache  [B, S, Hkv, D] -> present [B, Hkv, T, D] (ss = the position stride) at
//                 position past_len(b) + s; K rotated, V copied
//   build_k / build_v: the present caches' other positions: past[b, :, t] for t < past_len(b), zero from
//                 past_len(b) + S on (the positions of the new tokens are left to the append)
// and writes len_eff[b] = past_len(b) + S when len_eff is set.  past_len(b) = 0 for a first prompt (or without
// seqlens), else clamp(seqlens[b], S - 1, T - 1) + 1 - S, read on the device.
struct RotaryCore {
    int B = 0, S = 0, D = 0, H = 0, Hkv = 0, T = 0;
    RotaryTable rot;
    RotaryRows x, y;
    RotaryRows k_new, v_new, k_cache, v_cache, k_past, v_past;
    int build_k = 0, build_v = 0;
    const int32_t* seqlens = nullptr;
    long long sl_s = 1;
    int first = 0;
    int32_t* len_eff = nullptr;
};
// MultiHeadAttention's prep (mha = 1; no rotation, seqlens and len_eff unused): the new K / V streams have S_kv rows per
// batch, past_len(b) = past for every batch (present caches of T = past + S_kv positions), and each stream may add a
// bias vector -- element h * D + i to element i of a head-h row, one rounded f32 add (null: none)
struct RotaryMha {
    int mha = 0;
    int S_kv = 0;
    int past = 0;
    const float* x_bias = nullptr;
    const float* k_bias = nullptr;
    const float* v_bias = nullptr;
};
struct RotaryLaunch : RotaryCore, RotaryMha {};
rten_status launch_rotary(rten_ctx* ctx, const RotaryLaunch& L);

}  // namespace rtb
