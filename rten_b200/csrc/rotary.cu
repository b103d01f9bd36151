// Rotary embedding and KV-cache append (rotary.h): one warp per head row, lanes striding over the row's elements.
// Every row is read and written once; rotated elements use rotary_elem (rotary.cuh), whose arithmetic is the
// reference's exactly rounded products and sums.
#include <cuda_runtime.h>

#include <algorithm>

#include "rotary.cuh"
#include "rotary.h"

namespace rtb {

namespace {

constexpr int RT_WARPS = 8;

struct RotaryParams {
    RotaryCore L;
    long long nq, nk, nv, nb, nbuilt;  // rows of the Q, new K, new V streams, of one built cache, of all built caches
};

__device__ __forceinline__ int past_len(const RotaryCore& L, int b) {
    if (L.first || !L.seqlens) return 0;
    const int sk = min(max(L.seqlens[(long long)b * L.sl_s], L.S - 1), L.T - 1);
    return sk + 1 - L.S;
}

// cos / sin rows of token (b, s)
__device__ __forceinline__ void table_rows(const RotaryCore& L, int b, int s, const float** c, const float** sn) {
    const RotaryTable& t = L.rot;
    if (!t.by_pos) {
        *c = t.cos + (long long)b * t.c_b + (long long)s * t.c_s;
        *sn = t.sin + (long long)b * t.s_b + (long long)s * t.s_s;
        return;
    }
    int q = t.pos ? t.pos[(long long)b * t.p_b + (long long)s * t.p_s] : past_len(L, b) + s;
    q = min(max(q, 0), t.max_pos - 1);
    *c = t.cos + (long long)q * t.half;
    *sn = t.sin + (long long)q * t.half;
}

// one row: dst = rotate(src) (rotate: the table is set) or a copy of src (src null: zeros)
__device__ __forceinline__ void row_op(const RotaryCore& L, const float* src, long long xd, float* dst, long long yd, bool rotate,
                                       int b, int s, int lane) {
    const float* c = nullptr;
    const float* sn = nullptr;
    if (rotate) table_rows(L, b, s, &c, &sn);
    for (int i = lane; i < L.D; i += 32) {
        float v = 0.0f;
        if (src) v = rotate ? rotary_elem(src, xd, i, c, sn, L.rot.half, L.rot.interleaved) : src[i * xd];
        dst[i * yd] = v;
    }
}

// one MultiHeadAttention row: dst = src + bias (bias: the row's head slice, one rounded add per element), a copy of src
// (bias null) or zeros (src null)
__device__ __forceinline__ void row_bias(const RotaryCore& L, const float* src, long long xd, float* dst, long long yd, const float* bias,
                                         int lane) {
    for (int i = lane; i < L.D; i += 32) {
        float v = 0.0f;
        if (src) v = bias ? __fadd_rn(src[i * xd], bias[i]) : src[i * xd];
        dst[i * yd] = v;
    }
}

// MHA: MultiHeadAttention's prep (no rotation, no len_eff): bias adds, the new rows counted by S_kv, the past length
// M.past for every batch
template <bool MHA>
__device__ __forceinline__ void rotary_body(const RotaryParams& p, const RotaryMha& M) {
    const RotaryCore& L = p.L;
    const bool rot = !MHA && L.rot.cos != nullptr;
    const int S_new = MHA ? M.S_kv : L.S;
    if (!MHA && L.len_eff && blockIdx.x == 0)
        for (int b = threadIdx.x; b < L.B; b += blockDim.x) L.len_eff[b] = past_len(L, b) + L.S;
    const int lane = threadIdx.x & 31;
    long long r = (long long)blockIdx.x * RT_WARPS + (threadIdx.x >> 5);
    if (r < p.nq) {  // Q: row (b, s, h)
        const int h = (int)(r % L.H), s = (int)(r / L.H % L.S), b = (int)(r / ((long long)L.H * L.S));
        const float* src = L.x.p + b * L.x.sb + s * L.x.ss + h * L.x.sh;
        float* dst = L.y.p + b * L.y.sb + s * L.y.ss + h * L.y.sh;
        if constexpr (MHA) row_bias(L, src, L.x.sd, dst, L.y.sd, M.x_bias ? M.x_bias + (long long)h * L.D : nullptr, lane);
        else row_op(L, src, L.x.sd, dst, L.y.sd, rot, b, s, lane);
        return;
    }
    r -= p.nq;
    if (r < p.nk + p.nv) {  // new K / V: row (b, s, h) -> present (b, h, past_len(b) + s)
        const bool is_k = r < p.nk;
        if (!is_k) r -= p.nk;
        const RotaryRows& src = is_k ? L.k_new : L.v_new;
        const RotaryRows& dst = is_k ? L.k_cache : L.v_cache;
        const int h = (int)(r % L.Hkv), s = (int)(r / L.Hkv % S_new), b = (int)(r / ((long long)L.Hkv * S_new));
        const int t = (MHA ? M.past : past_len(L, b)) + s;
        const float* sp = src.p + b * src.sb + s * src.ss + h * src.sh;
        float* dp = dst.p + b * dst.sb + (long long)t * dst.ss + h * dst.sh;
        if constexpr (MHA) {
            const float* bias = is_k ? M.k_bias : M.v_bias;
            row_bias(L, sp, src.sd, dp, dst.sd, bias ? bias + (long long)h * L.D : nullptr, lane);
        } else {
            row_op(L, sp, src.sd, dp, dst.sd, rot && is_k, b, s, lane);
        }
        return;
    }
    r -= p.nk + p.nv;
    if (r < p.nbuilt) {  // present position (b, h, t) other than the new tokens: past prefix or zero
        bool is_k = L.build_k && r < p.nb;
        if (L.build_k && !is_k) r -= p.nb;
        const RotaryRows& past = is_k ? L.k_past : L.v_past;
        const RotaryRows& dst = is_k ? L.k_cache : L.v_cache;
        const int t = (int)(r % L.T), h = (int)(r / L.T % L.Hkv), b = (int)(r / ((long long)L.T * L.Hkv));
        const int pl = MHA ? M.past : past_len(L, b);
        if (t >= pl && t < pl + S_new) return;
        const float* src = t < pl ? past.p + b * past.sb + (long long)t * past.ss + h * past.sh : nullptr;
        float* dp = dst.p + b * dst.sb + (long long)t * dst.ss + h * dst.sh;
        if constexpr (MHA) row_bias(L, src, past.sd, dp, dst.sd, nullptr, lane);
        else row_op(L, src, past.sd, dp, dst.sd, false, b, 0, lane);
    }
}

__global__ void __launch_bounds__(RT_WARPS * 32) rotary_kernel(const __grid_constant__ RotaryParams p) { rotary_body<false>(p, RotaryMha()); }
__global__ void __launch_bounds__(RT_WARPS * 32) rotary_mha_kernel(const __grid_constant__ RotaryParams p, const __grid_constant__ RotaryMha m) {
    rotary_body<true>(p, m);
}

}  // namespace

rten_status launch_rotary(rten_ctx* ctx, const RotaryLaunch& L) {
    RotaryParams p;
    p.L = L;
    p.nq = L.y.p ? (long long)L.B * L.S * L.H : 0;
    const long long s_new = L.mha ? L.S_kv : L.S;
    p.nk = L.k_new.p ? (long long)L.B * s_new * L.Hkv : 0;
    p.nv = L.v_new.p ? (long long)L.B * s_new * L.Hkv : 0;
    p.nb = (long long)L.B * L.Hkv * L.T;
    p.nbuilt = (L.build_k ? p.nb : 0) + (L.build_v ? p.nb : 0);
    const long long rows = p.nq + p.nk + p.nv + p.nbuilt;
    const long long grid = std::max<long long>(1, (rows + RT_WARPS - 1) / RT_WARPS);
    if (grid > 0x7fffffffll) return fail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "rotary embedding: too many rows for one launch");
    if (L.mha) return launch(ctx, "rotary launch", rotary_mha_kernel, {(unsigned)grid, RT_WARPS * 32}, p, L);
    return launch(ctx, "rotary launch", rotary_kernel, {(unsigned)grid, RT_WARPS * 32}, p);
}

}  // namespace rtb
