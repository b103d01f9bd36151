// ReduceSum (src/ops/reduce.rs reduce / reduce_sum).  Every output is one lane: the reduced elements in row-major order of
// the reduced axes.  The reference sums each lane with vecmath::Sum, its 64-chain fold (rten-vecmath/src/sum.rs), in
// every branch of `reduce`: the contiguous inner chunks, the single-axis lanes and the permuted multi-axis slices all
// present the elements in that order.  So the kernels gather a lane into shared memory in that order -- straight from
// the strided input, no permuted copy -- and fold it there with smem_fold_chunks / smem_fold_finish (rowmath.cuh), the
// fold InstanceNormalization uses.
//   - lanes of up to RW_MAX elements: one warp per output, the whole lane staged at once (reduce_sum_warp_kernel);
//   - longer lanes: one CTA per output (reduce_sum_cta_kernel).  Warps 1.. stage the next RC_CHUNK elements of the lane
//     while warp 0 folds the current ones into its 64 chains; RC_CHUNK is a multiple of 64, so the chunks of the fold
//     never straddle two stages.
// i32 sums wrap, and every order gives the same result: the threads add their own elements and the partial sums are
// combined in any order, in registers.
#include <cuda_runtime.h>

#include <algorithm>
#include <type_traits>

#include "common.h"
#include "reduce.h"
#include "rowmath.cuh"

namespace rtb {

namespace {

constexpr int RW_WARPS = 8, RW_MAX = 1024;         // warp kernel: 8 outputs per CTA, lanes up to 1024 elements
constexpr int RC_THREADS = 256, RC_CHUNK = 4096;  // CTA kernel: two 16 KB stages

// offset of element j of a lane, relative to the lane's first element
__device__ __forceinline__ long long lane_off(const ReduceParams& p, long long j) {
    long long off = 0;
#pragma unroll 1
    for (int k = p.nr - 1; k >= 0; k--) {
        const long long s = p.rs[k], q = j / s;
        off += (j - q * s) * p.rx[k];
        j = q;
    }
    return off;
}

__device__ __forceinline__ void out_offs(const ReduceParams& p, long long o, long long& xo, long long& yo) {
    xo = 0, yo = 0;
#pragma unroll 1
    for (int k = p.no - 1; k >= 0; k--) {
        const long long s = p.os[k], q = o / s, i = o - q * s;
        xo += i * p.ox[k];
        yo += i * p.oy[k];
        o = q;
    }
}

template <typename T>
using Vec4 = typename std::conditional<std::is_same<T, float>::value, float4, int4>::type;

// s[i] = element j0 + i of the lane at x, i < n, by threads t = 0 .. nt - 1
template <typename T, bool VEC>
__device__ __forceinline__ void stage(const ReduceParams& p, const T* x, long long j0, int n, T* s, int t, int nt) {
    if (VEC) {
        const int n4 = n >> 2;
        for (int i = t; i < n4; i += nt) reinterpret_cast<Vec4<T>*>(s)[i] = reinterpret_cast<const Vec4<T>*>(x + j0)[i];
        for (int i = 4 * n4 + t; i < n; i += nt) s[i] = x[j0 + i];
    } else {
        for (int i = t; i < n; i += nt) s[i] = x[lane_off(p, j0 + i)];
    }
}

// this thread's wrapping sum of the lane elements j = t, t + nt, ...
template <bool VEC>
__device__ __forceinline__ unsigned int_partial(const ReduceParams& p, const int* x, int t, int nt) {
    unsigned s = 0;
    if (VEC) {
        const long long n4 = p.L >> 2;
        for (long long i = t; i < n4; i += nt) {
            const int4 v = reinterpret_cast<const int4*>(x)[i];
            s += (unsigned)v.x + (unsigned)v.y + (unsigned)v.z + (unsigned)v.w;
        }
        for (long long j = 4 * n4 + t; j < p.L; j += nt) s += (unsigned)x[j];
    } else {
        for (long long j = t; j < p.L; j += nt) s += (unsigned)x[lane_off(p, j)];
    }
    return s;
}

__device__ __forceinline__ unsigned warp_sum(unsigned s) {
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) s += __shfl_xor_sync(0xffffffffu, s, d);
    return s;
}

template <typename T, bool VEC>
__global__ void __launch_bounds__(RW_WARPS * 32) reduce_sum_warp_kernel(const ReduceParams p) {
    constexpr bool F32 = std::is_same<T, float>::value;
    __shared__ __align__(16) T buf[RW_WARPS][F32 ? RW_MAX : 4];
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int L = (int)p.L;
    for (long long o = (long long)blockIdx.x * RW_WARPS + w; o < p.nout; o += (long long)gridDim.x * RW_WARPS) {
        long long xo, yo;
        out_offs(p, o, xo, yo);
        const T* x = static_cast<const T*>(p.x) + xo;
        if constexpr (F32) {
            stage<float, VEC>(p, x, 0, L, buf[w], lane, 32);
            __syncwarp();
            const int F = L >> 6;
            float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
            smem_fold_chunks<false>(acc, reinterpret_cast<const float4*>(buf[w]), F, 0.0f);
            const float s = smem_fold_finish<false>(acc, buf[w] + 64 * F, L - 64 * F, 0.0f);
            if (lane == 0) static_cast<float*>(p.y)[yo] = s;
            __syncwarp();  // (the next output reuses the buffer)
        } else {
            const unsigned s = warp_sum(int_partial<VEC>(p, x, lane, 32));
            if (lane == 0) static_cast<int*>(p.y)[yo] = (int)s;
        }
    }
}

template <typename T, bool VEC>
__global__ void __launch_bounds__(RC_THREADS) reduce_sum_cta_kernel(const ReduceParams p) {
    constexpr bool F32 = std::is_same<T, float>::value;
    __shared__ __align__(16) T ring[2][F32 ? RC_CHUNK : RC_THREADS / 32];
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (long long o = blockIdx.x; o < p.nout; o += gridDim.x) {
        long long xo, yo;
        out_offs(p, o, xo, yo);
        const T* x = static_cast<const T*>(p.x) + xo;
        if constexpr (F32) {
            const long long nch = (p.L + RC_CHUNK - 1) / RC_CHUNK;
            stage<float, VEC>(p, x, 0, (int)min((long long)RC_CHUNK, p.L), ring[0], threadIdx.x, RC_THREADS);
            __syncthreads();
            float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
            float total = 0.0f;
            for (long long k = 0; k < nch; k++) {
                if (w > 0 && k + 1 < nch) {
                    const long long j0 = (k + 1) * RC_CHUNK;
                    stage<float, VEC>(p, x, j0, (int)min((long long)RC_CHUNK, p.L - j0), ring[(k + 1) & 1], threadIdx.x - 32,
                                      RC_THREADS - 32);
                }
                if (w == 0) {
                    const int len = (int)min((long long)RC_CHUNK, p.L - k * RC_CHUNK), F = len >> 6;
                    const float* s = ring[k & 1];
                    smem_fold_chunks<false>(acc, reinterpret_cast<const float4*>(s), F, 0.0f);
                    if (k + 1 == nch) total = smem_fold_finish<false>(acc, s + 64 * F, len - 64 * F, 0.0f);
                }
                __syncthreads();
            }
            if (threadIdx.x == 0) static_cast<float*>(p.y)[yo] = total;
        } else {
            const unsigned s = warp_sum(int_partial<VEC>(p, x, threadIdx.x, RC_THREADS));
            if (lane == 0) ring[0][w] = (int)s;
            __syncthreads();
            if (w == 0) {
                unsigned t = lane < RC_THREADS / 32 ? (unsigned)ring[0][lane] : 0u;
                t = warp_sum(t);
                if (lane == 0) static_cast<int*>(p.y)[yo] = (int)t;
            }
            __syncthreads();
        }
    }
}

template <typename T>
rten_status launch_typed(rten_ctx* ctx, const ReduceParams& p) {
    const long long cap = (long long)ctx->num_sms * 8;
    if (p.L <= RW_MAX) {
        const LaunchShape s{dim3((unsigned)std::min(cap, (p.nout + RW_WARPS - 1) / RW_WARPS)), dim3(RW_WARPS * 32)};
        return p.vec ? launch(ctx, "reduce_sum launch", reduce_sum_warp_kernel<T, true>, s, p)
                     : launch(ctx, "reduce_sum launch", reduce_sum_warp_kernel<T, false>, s, p);
    }
    const LaunchShape s{dim3((unsigned)std::min(cap, p.nout)), dim3(RC_THREADS)};
    return p.vec ? launch(ctx, "reduce_sum launch", reduce_sum_cta_kernel<T, true>, s, p)
                 : launch(ctx, "reduce_sum launch", reduce_sum_cta_kernel<T, false>, s, p);
}

}  // namespace

rten_status launch_reduce_sum(rten_ctx* ctx, int dtype, const ReduceParams& p) {
    if (p.nout == 0) return RTEN_OK;
    return dtype == RTEN_F32 ? launch_typed<float>(ctx, p) : launch_typed<int>(ctx, p);
}

}  // namespace rtb
