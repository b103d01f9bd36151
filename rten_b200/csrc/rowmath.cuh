// Device helpers shared by the row kernels (rowops.cu) and the fused skinny-M kernels (skinny.cu): the exact scalar
// recipes of DynamicQuantizeLinear (src/ops/quantize.rs:352-434, rten-vecmath/src/quantize.rs:38-77), the fold step
// of Sum / SumSquareSub (rten-vecmath/src/sum.rs:22-35,111-130) and Normalize's output arms.
#pragma once
#include <cstdint>

namespace rtb {

__device__ __forceinline__ int float_to_ordered(float f) {
    int i = __float_as_int(f);
    return i >= 0 ? i : i ^ 0x7fffffff;
}
__device__ __forceinline__ float ordered_to_float(int i) { return __int_as_float(i >= 0 ? i : i ^ 0x7fffffff); }

__device__ __forceinline__ void dql_params(const int* mm, float& scale, float& inv_scale, int& zp) {
    const float x_min = ordered_to_float(mm[0]), x_max = ordered_to_float(mm[1]);
    const float lo = fminf(x_min, 0.0f), hi = fmaxf(x_max, 0.0f);
    scale = __fdiv_rn(__fsub_rn(hi, lo), 255.0f);
    const float min_scaled = __fdiv_rn(lo, scale);
    float z = __fsub_rn(0.0f, min_scaled);
    z = fminf(fmaxf(z, 0.0f), 255.0f);  // clamp (NaN -> 0 after the cast below)
    z = rintf(z);                       // round_ties_even
    zp = (z != z) ? 0 : (int)z;
    inv_scale = __fdiv_rn(1.0f, scale);
}

__device__ __forceinline__ int rne_i32_x86(float v) {
    if (!(v >= -2147483648.0f && v < 2147483648.0f)) return (int)0x80000000;
    return __float2int_rn(v);
}
__device__ __forceinline__ uint8_t quant1(float x, float inv_scale, int zp) {
    // saturate_u8(round(x * inv_scale) + zp): the rounded value is clamped to [-256, 511] first -- anything outside
    // saturates the same way -- so that the sum stays in 32 bits (zp is in [0, 255])
    int r = rne_i32_x86(__fmul_rn(x, inv_scale));
    r = max(-256, min(511, r));
    return (uint8_t)max(0, min(255, r + zp));
}

template <bool SQSUB>
__device__ __forceinline__ float fold_step(float acc, float x, float off) {
    if (SQSUB) {
        const float d = __fsub_rn(x, off);
        return __fmaf_rn(d, d, acc);
    }
    return __fadd_rn(acc, x);
}

__device__ __forceinline__ float4 add4(float4 a, float4 b) {
    return make_float4(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y), __fadd_rn(a.z, b.z), __fadd_rn(a.w, b.w));
}

// Normalize's three arms (rten-vecmath/src/normalize.rs:101-169): 0 = scalar scale and bias, 1 = per-element scale, no
// bias; 2 = the general one (g = 1 without a per-element scale, b = 0 without a per-element bias)
__device__ __forceinline__ float norm_arm(int mode, float a, float mean, float rstd, float g, float b, float beta_scalar) {
    if (mode == 0) return __fmaf_rn(__fsub_rn(a, mean), rstd, beta_scalar);
    if (mode == 1) return __fmul_rn(__fsub_rn(a, mean), __fmul_rn(g, rstd));
    return __fmaf_rn(__fsub_rn(a, mean), __fmul_rn(g, rstd), __fadd_rn(b, beta_scalar));
}
__device__ __forceinline__ float4 norm_arm4(int mode, float4 a, float mean, float rstd, float4 g, float4 b, float bs) {
    return make_float4(norm_arm(mode, a.x, mean, rstd, g.x, b.x, bs), norm_arm(mode, a.y, mean, rstd, g.y, b.y, bs),
                       norm_arm(mode, a.z, mean, rstd, g.z, b.z, bs), norm_arm(mode, a.w, mean, rstd, g.w, b.w, bs));
}

// Sum / SumSquareSub of one row held in registers as float4s, in the reference's fold_unroll<4> x 16-lane order (see
// norm_vec_kernel in rowops.cu for the thread <-> chain mapping): thread (c = lane & 15, segment seg) of a row
// that spans 16 S lanes holds the float4s f = c + 16 (seg F + k), k < F.  Every lane of the row returns the total.
template <int S, bool SQSUB, int FMAX = 16>
__device__ __forceinline__ float ln_vec_fold(const float4 (&v)[FMAX], int F, float off, int c, int seg) {
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int sg = 0; sg < S; sg++) {
        if (sg > 0) {
            const float4 in = make_float4(__shfl_up_sync(0xffffffffu, acc.x, 16), __shfl_up_sync(0xffffffffu, acc.y, 16),
                                          __shfl_up_sync(0xffffffffu, acc.z, 16), __shfl_up_sync(0xffffffffu, acc.w, 16));
            if (seg == sg) acc = in;
        }
        if (seg == sg) {
#pragma unroll
            for (int k = 0; k < FMAX; k++) {
                if (k < F) {
                    acc.x = fold_step<SQSUB>(acc.x, v[k].x, off);
                    acc.y = fold_step<SQSUB>(acc.y, v[k].y, off);
                    acc.z = fold_step<SQSUB>(acc.z, v[k].z, off);
                    acc.w = fold_step<SQSUB>(acc.w, v[k].w, off);
                }
            }
        }
    }
    // u = c >> 2 selects the unrolled accumulator, l = 4 (c & 3) + j the lane: threads c, c + 4, c + 8, c + 12 -> thread c (< 4)
    float4 r = acc;
#pragma unroll
    for (int u = 1; u < 4; u++) {
        r.x = __fadd_rn(r.x, __shfl_down_sync(0xffffffffu, acc.x, 4 * u));
        r.y = __fadd_rn(r.y, __shfl_down_sync(0xffffffffu, acc.y, 4 * u));
        r.z = __fadd_rn(r.z, __shfl_down_sync(0xffffffffu, acc.z, 4 * u));
        r.w = __fadd_rn(r.w, __shfl_down_sync(0xffffffffu, acc.w, 4 * u));
    }
    float s = 0.0f;
#pragma unroll
    for (int q = 0; q < 4; q++) {
        const float in = __shfl_up_sync(0xffffffffu, s, 1);
        if (c == q) {
            if (q > 0) s = in;
            s = __fadd_rn(__fadd_rn(__fadd_rn(__fadd_rn(s, r.x), r.y), r.z), r.w);
        }
    }
    // thread c = 3 of the row's LAST segment holds the total
    const int lane = threadIdx.x & 31;
    const int base = (lane / (16 * S)) * (16 * S);
    return __shfl_sync(0xffffffffu, s, base + (S - 1) * 16 + 3);
}

// The same fold over a row staged in shared memory as F * 16 float4s (n = 64 F), by one whole warp: lane c = lane & 15
// walks the float4s f = c + 16 k, k < F -- its four chains in ascending i -- and lanes 16..31 repeat lanes 0..15.
// Every lane returns the total.
template <bool SQSUB>
__device__ __forceinline__ float ln_smem_fold(const float4* s4, int F, float off) {
    const int c = threadIdx.x & 15;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int k = 0; k < F; k++) {
        const float4 v = s4[c + 16 * k];
        acc.x = fold_step<SQSUB>(acc.x, v.x, off);
        acc.y = fold_step<SQSUB>(acc.y, v.y, off);
        acc.z = fold_step<SQSUB>(acc.z, v.z, off);
        acc.w = fold_step<SQSUB>(acc.w, v.w, off);
    }
    float4 r = acc;  // acc[0][l] = ((acc[0][l] + acc[1][l]) + acc[2][l]) + acc[3][l], as in ln_vec_fold
#pragma unroll
    for (int u = 1; u < 4; u++) {
        r.x = __fadd_rn(r.x, __shfl_down_sync(0xffffffffu, acc.x, 4 * u));
        r.y = __fadd_rn(r.y, __shfl_down_sync(0xffffffffu, acc.y, 4 * u));
        r.z = __fadd_rn(r.z, __shfl_down_sync(0xffffffffu, acc.z, 4 * u));
        r.w = __fadd_rn(r.w, __shfl_down_sync(0xffffffffu, acc.w, 4 * u));
    }
    float s = 0.0f;
#pragma unroll
    for (int q = 0; q < 4; q++) {
        const float in = __shfl_up_sync(0xffffffffu, s, 1);
        if (c == q) {
            if (q > 0) s = in;
            s = __fadd_rn(__fadd_rn(__fadd_rn(__fadd_rn(s, r.x), r.y), r.z), r.w);
        }
    }
    return __shfl_sync(0xffffffffu, s, 3);
}

// ln_smem_fold for any n, in two steps so that the 64 chains can run over a row that arrives chunk by chunk
// (groupnorm.cu).  smem_fold_chunks adds F full 64-element chunks (F * 16 float4s at s4) to the running chains `acc`
// (lane c = lane & 15 owns chains 4c .. 4c + 3); smem_fold_finish then combines the chains and folds the rem < 64
// elements after the last full chunk -- its full 16-element chunks, then the masked tail -- into acc[0], and sums the
// 16 lanes in order (simd_fold_unroll4 in rowops.cu, over shared memory).  A whole warp calls both; every lane returns
// the total.  (ln_smem_fold is the rem = 0 case; it stays as it is so that the kernels using it keep their code.)
template <bool SQSUB>
__device__ __forceinline__ void smem_fold_chunks(float4& acc, const float4* s4, int F, float off) {
    const int c = threadIdx.x & 15;
#pragma unroll 4
    for (int k = 0; k < F; k++) {
        const float4 v = s4[c + 16 * k];
        acc.x = fold_step<SQSUB>(acc.x, v.x, off);
        acc.y = fold_step<SQSUB>(acc.y, v.y, off);
        acc.z = fold_step<SQSUB>(acc.z, v.z, off);
        acc.w = fold_step<SQSUB>(acc.w, v.w, off);
    }
}

template <bool SQSUB>
__device__ __forceinline__ float smem_fold_finish(float4 acc, const float* t, int rem, float off) {
    const int c = threadIdx.x & 15;
    float4 r = acc;  // acc[0][l] = ((acc[0][l] + acc[1][l]) + acc[2][l]) + acc[3][l]: thread c < 4 holds l = 4c .. 4c + 3
#pragma unroll
    for (int u = 1; u < 4; u++) {
        r.x = __fadd_rn(r.x, __shfl_down_sync(0xffffffffu, acc.x, 4 * u));
        r.y = __fadd_rn(r.y, __shfl_down_sync(0xffffffffu, acc.y, 4 * u));
        r.z = __fadd_rn(r.z, __shfl_down_sync(0xffffffffu, acc.z, 4 * u));
        r.w = __fadd_rn(r.w, __shfl_down_sync(0xffffffffu, acc.w, 4 * u));
    }
    if (c < 4) {
        for (int i = 4 * c; i < rem; i += 16) {  // element i of the remainder goes to lane l = i % 16
            r.x = fold_step<SQSUB>(r.x, t[i], off);
            if (i + 1 < rem) r.y = fold_step<SQSUB>(r.y, t[i + 1], off);
            if (i + 2 < rem) r.z = fold_step<SQSUB>(r.z, t[i + 2], off);
            if (i + 3 < rem) r.w = fold_step<SQSUB>(r.w, t[i + 3], off);
        }
    }
    float s = 0.0f;
#pragma unroll
    for (int q = 0; q < 4; q++) {
        const float in = __shfl_up_sync(0xffffffffu, s, 1);
        if (c == q) {
            if (q > 0) s = in;
            s = __fadd_rn(__fadd_rn(__fadd_rn(__fadd_rn(s, r.x), r.y), r.z), r.w);
        }
    }
    return __shfl_sync(0xffffffffu, s, 3);
}

}  // namespace rtb
