// ReduceSum and ReduceMean (src/ops/reduce.rs reduce / reduce_sum / reduce_mean).  Every output is one lane: the reduced elements in row-major order of
// the reduced axes.  The reference sums each lane with vecmath::Sum, its 64-chain fold (rten-vecmath/src/sum.rs), in
// every branch of `reduce`: the contiguous inner chunks, the single-axis lanes and the permuted multi-axis slices all
// present the elements in that order.  So the kernels gather a lane into shared memory in that order -- straight from
// the strided input, no permuted copy -- and fold it there with smem_fold_chunks / smem_fold_finish (rowmath.cuh), the
// fold InstanceNormalization uses.  ReduceMean is the same fold with one division by the lane length at the store.
//   - lanes of up to RW_MAX elements: one warp per output, the whole lane staged at once (reduce_sum_warp_kernel);
//   - longer lanes: one CTA per output (reduce_sum_cta_kernel).  Warps 1.. stage the next RC_CHUNK elements of the lane
//     while warp 0 folds the current ones into its 64 chains; RC_CHUNK is a multiple of 64, so the chunks of the fold
//     never straddle two stages.
// i32 sums wrap, and every order gives the same result: the threads add their own elements and the partial sums are
// combined in any order, in registers.
//
// ArgMax, ArgMin and TopK with k = 1 (arg_reduce_*_kernel) take the largest composite key of each lane (select.cuh), a
// total order, so partial maxima combine in any order.  Short lanes: one warp per output; long lanes: one CTA per
// output, or, when the outputs are too few to give every SM one, one thread-block cluster per output whose CTAs take
// contiguous slices of the lane and combine their maxima through distributed shared memory.
#include <cooperative_groups.h>
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
            if (lane == 0) static_cast<float*>(p.y)[yo] = p.mean ? __fdiv_rn(s, (float)p.L) : s;
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
            if (threadIdx.x == 0) static_cast<float*>(p.y)[yo] = p.mean ? __fdiv_rn(total, (float)p.L) : total;
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

// ---- arg-reduce --------------------------------------------------------------------------------------------------------
constexpr int AC_THREADS = 256, AC_MIN_SLICE = 2048;  // CTA / cluster kernels; a cluster gives each CTA >= AC_MIN_SLICE

// this thread's largest key among the lane elements j = j0 + t, j0 + t + nt, ... < j1
template <typename T>
__device__ __forceinline__ uint64_t arg_partial(const SelectParams& a, const T* x, long long j0, long long j1, int t, int nt) {
    const ReduceParams& p = a.r;
    const bool contig = p.nr == 0 || p.rx[0] == 1;
    uint64_t best = 0;  // below or equal to every key
    auto take = [&](T v, long long j) {
        const uint64_t k = sel_key(v, (uint32_t)j, a.mode);
        best = k > best ? k : best;
    };
    if (contig && (reinterpret_cast<uintptr_t>(x + j0) & 15) == 0) {  // 16-byte loads: four elements in flight each
        const long long n4 = (j1 - j0) >> 2;
        const Vec4<T>* x4 = reinterpret_cast<const Vec4<T>*>(x + j0);
        for (long long q = t; q < n4; q += nt) {
            const Vec4<T> v = x4[q];
            const long long j = j0 + 4 * q;
            take(v.x, j), take(v.y, j + 1), take(v.z, j + 2), take(v.w, j + 3);
        }
        j0 += 4 * n4;
    }
    for (long long j = j0 + t; j < j1; j += nt) {
        const uint64_t k = sel_key(contig ? x[j] : x[lane_off(p, j)], (uint32_t)j, a.mode);
        best = k > best ? k : best;
    }
    return best;
}

template <typename T>
__device__ __forceinline__ void arg_store(const SelectParams& a, const T* x, long long yo, uint64_t best) {
    const uint32_t i = sel_index<T>(best, a.mode);
    static_cast<int*>(a.r.y)[yo] = (int)i;
    if (a.vals) static_cast<T*>(a.vals)[yo] = x[lane_off(a.r, i)];
}

// the CTA's largest key, in every thread
__device__ __forceinline__ uint64_t block_max_u64(uint64_t v, uint64_t* part) {
    v = warp_max_u64(v);
    if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = v;
    __syncthreads();
    v = (threadIdx.x & 31) < AC_THREADS / 32 ? part[threadIdx.x & 31] : 0;
    v = warp_max_u64(v);
    __syncthreads();  // (part is reused)
    return v;
}

template <typename T>
__global__ void __launch_bounds__(RW_WARPS * 32) arg_reduce_warp_kernel(const SelectParams a) {
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (long long o = (long long)blockIdx.x * RW_WARPS + w; o < a.r.nout; o += (long long)gridDim.x * RW_WARPS) {
        long long xo, yo;
        out_offs(a.r, o, xo, yo);
        const T* x = static_cast<const T*>(a.r.x) + xo;
        const uint64_t best = warp_max_u64(arg_partial<T>(a, x, 0, a.r.L, lane, 32));
        if (lane == 0) arg_store<T>(a, x, yo, best);
    }
}

template <typename T>
__global__ void __launch_bounds__(AC_THREADS) arg_reduce_cta_kernel(const SelectParams a) {
    __shared__ uint64_t part[AC_THREADS / 32];
    for (long long o = blockIdx.x; o < a.r.nout; o += gridDim.x) {
        long long xo, yo;
        out_offs(a.r, o, xo, yo);
        const T* x = static_cast<const T*>(a.r.x) + xo;
        const uint64_t best = block_max_u64(arg_partial<T>(a, x, 0, a.r.L, threadIdx.x, AC_THREADS), part);
        if (threadIdx.x == 0) arg_store<T>(a, x, yo, best);
    }
}

// one cluster per output: CTA `rank` takes elements [rank * S, (rank + 1) * S) of the lane, rank 0 combines
template <typename T>
__global__ void __launch_bounds__(AC_THREADS) arg_reduce_cluster_kernel(const SelectParams a) {
    namespace cg = cooperative_groups;
    cg::cluster_group cl = cg::this_cluster();
    const int C = (int)cl.num_blocks(), rank = (int)cl.block_rank();
    __shared__ uint64_t part[AC_THREADS / 32];
    __shared__ uint64_t cta_best;
    const long long S = ((a.r.L + C - 1) / C + 3) & ~3LL, j0 = min(a.r.L, rank * S), j1 = min(a.r.L, j0 + S);
    for (long long o = blockIdx.x / C; o < a.r.nout; o += gridDim.x / C) {
        long long xo, yo;
        out_offs(a.r, o, xo, yo);
        const T* x = static_cast<const T*>(a.r.x) + xo;
        const uint64_t best = block_max_u64(arg_partial<T>(a, x, j0, j1, threadIdx.x, AC_THREADS), part);
        if (threadIdx.x == 0) cta_best = best;
        cl.sync();
        if (rank == 0 && threadIdx.x < 32) {
            uint64_t v = threadIdx.x < C ? *cl.map_shared_rank(&cta_best, (int)threadIdx.x) : 0;
            v = warp_max_u64(v);
            if (threadIdx.x == 0) arg_store<T>(a, x, yo, v);
        }
        cl.sync();  // rank 0 has read every CTA's cta_best
    }
}

template <typename T>
rten_status launch_arg_typed(rten_ctx* ctx, const SelectParams& a) {
    const ReduceParams& p = a.r;
    const long long cap = (long long)ctx->num_sms * 8;
    if (p.L <= RW_MAX) {
        const LaunchShape s{dim3((unsigned)std::min(cap, (p.nout + RW_WARPS - 1) / RW_WARPS)), dim3(RW_WARPS * 32)};
        return launch(ctx, "arg_reduce launch", arg_reduce_warp_kernel<T>, s, a);
    }
    // a cluster per lane while the lanes leave SMs idle, each CTA with at least AC_MIN_SLICE elements
    long long C = std::min({16LL, (ctx->num_sms + p.nout - 1) / p.nout, (p.L + AC_MIN_SLICE - 1) / AC_MIN_SLICE});
    if (C >= 2) {
        LaunchShape s{dim3(1), dim3(AC_THREADS)};
        C = cluster_size_fit<arg_reduce_cluster_kernel<T>>((int)C, s);
        s.grid = dim3((unsigned)(std::min(p.nout, 65535LL) * C));
        s.cluster = (int)C;
        return launch(ctx, "arg_reduce launch", arg_reduce_cluster_kernel<T>, s, a);
    }
    const LaunchShape s{dim3((unsigned)std::min(cap, p.nout)), dim3(AC_THREADS)};
    return launch(ctx, "arg_reduce launch", arg_reduce_cta_kernel<T>, s, a);
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

rten_status launch_arg_reduce(rten_ctx* ctx, int dtype, const SelectParams& a) {
    if (a.r.nout == 0) return RTEN_OK;
    return dtype == RTEN_F32 ? launch_arg_typed<float>(ctx, a) : launch_arg_typed<int>(ctx, a);
}

}  // namespace rtb
