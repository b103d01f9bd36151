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
    RotaryLaunch L;
    long long nq, nk, nv, nb, nbuilt;  // rows of the Q, new K, new V streams, of one built cache, of all built caches
};

__device__ __forceinline__ int past_len(const RotaryLaunch& L, int b) {
    if (L.first || !L.seqlens) return 0;
    const int sk = min(max(L.seqlens[(long long)b * L.sl_s], L.S - 1), L.T - 1);
    return sk + 1 - L.S;
}

// cos / sin rows of token (b, s)
__device__ __forceinline__ void table_rows(const RotaryLaunch& L, int b, int s, const float** c, const float** sn) {
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
__device__ __forceinline__ void row_op(const RotaryLaunch& L, const float* src, long long xd, float* dst, long long yd, bool rotate,
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

__global__ void __launch_bounds__(RT_WARPS * 32) rotary_kernel(const __grid_constant__ RotaryParams p) {
    const RotaryLaunch& L = p.L;
    const bool rot = L.rot.cos != nullptr;
    if (L.len_eff && blockIdx.x == 0)
        for (int b = threadIdx.x; b < L.B; b += blockDim.x) L.len_eff[b] = past_len(L, b) + L.S;
    const int lane = threadIdx.x & 31;
    long long r = (long long)blockIdx.x * RT_WARPS + (threadIdx.x >> 5);
    if (r < p.nq) {  // Q: row (b, s, h)
        const int h = (int)(r % L.H), s = (int)(r / L.H % L.S), b = (int)(r / ((long long)L.H * L.S));
        row_op(L, L.x.p + b * L.x.sb + s * L.x.ss + h * L.x.sh, L.x.sd, L.y.p + b * L.y.sb + s * L.y.ss + h * L.y.sh, L.y.sd, rot, b,
               s, lane);
        return;
    }
    r -= p.nq;
    if (r < p.nk + p.nv) {  // new K / V: row (b, s, h) -> present (b, h, past_len(b) + s)
        const bool is_k = r < p.nk;
        if (!is_k) r -= p.nk;
        const RotaryRows& src = is_k ? L.k_new : L.v_new;
        const RotaryRows& dst = is_k ? L.k_cache : L.v_cache;
        const int h = (int)(r % L.Hkv), s = (int)(r / L.Hkv % L.S), b = (int)(r / ((long long)L.Hkv * L.S));
        const int t = past_len(L, b) + s;
        row_op(L, src.p + b * src.sb + s * src.ss + h * src.sh, src.sd, dst.p + b * dst.sb + (long long)t * dst.ss + h * dst.sh, dst.sd,
               rot && is_k, b, s, lane);
        return;
    }
    r -= p.nk + p.nv;
    if (r < p.nbuilt) {  // present position (b, h, t) other than the new tokens: past prefix or zero
        bool is_k = L.build_k && r < p.nb;
        if (L.build_k && !is_k) r -= p.nb;
        const RotaryRows& past = is_k ? L.k_past : L.v_past;
        const RotaryRows& dst = is_k ? L.k_cache : L.v_cache;
        const int t = (int)(r % L.T), h = (int)(r / L.T % L.Hkv), b = (int)(r / ((long long)L.T * L.Hkv));
        const int pl = past_len(L, b);
        if (t >= pl && t < pl + L.S) return;
        const float* src = t < pl ? past.p + b * past.sb + (long long)t * past.ss + h * past.sh : nullptr;
        row_op(L, src, past.sd, dst.p + b * dst.sb + (long long)t * dst.ss + h * dst.sh, dst.sd, false, b, 0, lane);
    }
}

}  // namespace

rten_status launch_rotary(rten_ctx* ctx, const RotaryLaunch& L) {
    RotaryParams p;
    p.L = L;
    p.nq = L.y.p ? (long long)L.B * L.S * L.H : 0;
    p.nk = L.k_new.p ? (long long)L.B * L.S * L.Hkv : 0;
    p.nv = L.v_new.p ? (long long)L.B * L.S * L.Hkv : 0;
    p.nb = (long long)L.B * L.Hkv * L.T;
    p.nbuilt = (L.build_k ? p.nb : 0) + (L.build_v ? p.nb : 0);
    const long long rows = p.nq + p.nk + p.nv + p.nbuilt;
    const long long grid = std::max<long long>(1, (rows + RT_WARPS - 1) / RT_WARPS);
    if (grid > 0x7fffffffll) return fail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "rotary embedding: too many rows for one launch");
    rotary_kernel<<<(unsigned)grid, RT_WARPS * 32, 0, ctx->stream>>>(p);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail_cuda(ctx, e, "rotary launch");
    count_launch(ctx);
    return RTEN_OK;
}

}  // namespace rtb
