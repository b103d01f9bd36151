// InstanceNormalization (src/ops/norm.rs instance_normalization: normalize_each_channel -> normalize_slice) and the
// GroupNorm chain torch exports -- Reshape [N, G, -1], InstanceNormalization, Reshape back, Mul(gamma), Add(beta) and an
// optional activation -- as one normalization pass.  Bit-identical to the reference: the statistics of each row in the
// Sum / SumSquareSub fold order (fold_unroll<4> over 16 lanes: 64 serial chains, then the 16-element chunks and the
// masked tail), the output through Normalize's arm 0, then the Mul, the Add and the activation each rounded on its own.
//
// Rows are few and long (N * G of them, (C / G) * H * W elements each), so the kernels parallelise over a row's
// elements, not over rows:
//   gn_onchip_kernel  L <= ONCHIP_MAX: one CTA per row loads it once into shared memory (cp.async, all warps), one warp
//                     folds it there twice, then all warps normalise it from shared memory: one read and one write of x.
//                     Channels-last input is gathered slab by slab -- pixels x (C / G) channels -- into logical (c, p)
//                     order, and scattered back on the way out.
//   streaming         longer rows: gn_stats_kernel streams each row through a shared-memory ring filled by every warp
//                     of its CTA, once per statistic, while one warp folds; gn_apply_kernel then normalises the whole
//                     tensor over all SMs.  Two reads of x for the statistics, one read and one write for the output.
//                     Channels-last rows are first copied to [N, C, P] order (one more read and write of x) so that the
//                     fold reads them in logical order with full sectors; a per-channel sweep of the channels-last data
//                     would use 4 bytes of every 32-byte sector and rely on L2 to keep the rest for the next channel,
//                     which a 4 MB row spread over 32 CTAs does not fit.
// The fold of one row is serial: 2 ceil(L / 64) dependent adds / FMAs per lane, which bounds a long row's time no
// matter how fast it arrives.
//
// BatchNormalization (src/ops/norm.rs batch_norm_in_place: normalize_each_channel with MeanNormalize::Static) is the
// output pass alone, gn_apply_kernel with G = C and its constants per channel: mean[c], and
// scale[c] / sqrt(var[c] + epsilon) computed by each thread as the reference computes it, then Normalize's arm 0.
// The mean and variance are kernel arguments of their own, so GroupNormParams and the other kernels stay as they were.
#include <cuda_runtime.h>

#include <algorithm>
#include <climits>
#include <cstdint>
#include <cstdlib>

#include "common.h"
#include "groupnorm.h"
#include "math.cuh"
#include "rowmath.cuh"
#include "rowops.h"

namespace rtb {

constexpr int ONCHIP_MAX = 51200;  // floats of a row the on-chip path takes (200 KB of shared memory)
constexpr int RING_CHUNK = 8192;   // floats per ring stage (a multiple of 64: chunks start on a fold chunk)
constexpr int RING_STAGES = 6;     // 192 KB of shared memory, five stages in flight while one is folded
constexpr int STATS_THREADS = 512;
constexpr int APPLY_THREADS = 256;

__device__ __forceinline__ void cp_async4(void* s, const void* g) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;\n" ::"r"((unsigned)__cvta_generic_to_shared(s)), "l"(g));
}
__device__ __forceinline__ void cp_async16(void* s, const void* g) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"((unsigned)__cvta_generic_to_shared(s)), "l"(g));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N)); }

// one output element: Normalize's arm 0 with the row's instance-norm bias, then gamma, beta and the activation
__device__ __forceinline__ float gn_out(const GroupNormParams& p, float v, float mean, float rstd, float ib, float gm, float bt) {
    float y = __fmaf_rn(__fsub_rn(v, mean), rstd, ib);
    if (p.gamma) y = __fmul_rn(y, gm);
    if (p.beta) y = __fadd_rn(y, bt);
    return apply_act(y, p.act, p.act_alpha, p.act_beta);
}

// (mean, rstd) of a row of n elements staged at s, by one whole warp
__device__ __forceinline__ float2 smem_row_stats(const float* s, int n, float eps, float scale) {
    const int F = n / 64;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    smem_fold_chunks<false>(acc, reinterpret_cast<const float4*>(s), F, 0.0f);
    const float mean = __fdiv_rn(smem_fold_finish<false>(acc, s + 64 * F, n - 64 * F, 0.0f), (float)n);
    acc = make_float4(0.f, 0.f, 0.f, 0.f);
    smem_fold_chunks<true>(acc, reinterpret_cast<const float4*>(s), F, mean);
    const float var = __fdiv_rn(smem_fold_finish<true>(acc, s + 64 * F, n - 64 * F, mean), (float)n);
    return make_float2(mean, __fdiv_rn(scale, __fsqrt_rn(__fadd_rn(var, eps))));
}

// One CTA per row (n, g).  vec: the row starts 16-byte aligned and L % 4 == 0 (NCHW only).
template <bool CL>
__global__ void __launch_bounds__(1024) gn_onchip_kernel(const GroupNormParams p, int vec) {
    extern __shared__ float4 srow4[];
    float* srow = reinterpret_cast<float*>(srow4);
    __shared__ float2 stat;
    const int g = (int)(blockIdx.x % (unsigned)p.G);
    const long long n = blockIdx.x / (unsigned)p.G;
    const int cg = p.C / p.G, P = (int)p.P, L = cg * P, t = threadIdx.x, nt = blockDim.x;
    const float* xr;  // NCHW: the row; channels-last: channel g cg of pixel 0 of image n
    float* yr;
    if (CL) {
        xr = p.x + n * P * p.C + (long long)g * cg;
        yr = p.y + n * P * p.C + (long long)g * cg;
        for (int j = t; j < L; j += nt) {  // j = pixel * cg + channel: consecutive threads read consecutive addresses
            const int px = j / cg, cl = j - px * cg;
            cp_async4(srow + cl * P + px, xr + (long long)px * p.C + cl);
        }
    } else {
        xr = p.x + (long long)blockIdx.x * L;
        yr = p.y + (long long)blockIdx.x * L;
        if (vec) {
            for (int f = t; f < L / 4; f += nt) cp_async16(srow4 + f, xr + 4 * f);
        } else {
            for (int i = t; i < L; i += nt) cp_async4(srow + i, xr + i);
        }
    }
    cp_async_commit();
    cp_async_wait<0>();
    __syncthreads();
    if (t < 32) {
        const float2 st = smem_row_stats(srow, L, p.eps, __ldg(p.inst_scale + g));
        if (t == 0) stat = st;
    }
    __syncthreads();
    const float mean = stat.x, rstd = stat.y, ib = __ldg(p.inst_bias + g);
    if (CL) {
        for (int j = t; j < L; j += nt) {
            const int px = j / cg, cl = j - px * cg, c = g * cg + cl;
            yr[(long long)px * p.C + cl] = gn_out(p, srow[cl * P + px], mean, rstd, ib, p.gamma ? __ldg(p.gamma + c) : 1.0f,
                                                  p.beta ? __ldg(p.beta + c) : 0.0f);
        }
    } else {
        for (int i = t; i < L; i += nt) {
            const int c = g * cg + i / P;
            yr[i] = gn_out(p, srow[i], mean, rstd, ib, p.gamma ? __ldg(p.gamma + c) : 1.0f, p.beta ? __ldg(p.beta + c) : 0.0f);
        }
    }
}

// Statistics of row blockIdx.x of xs ([N * G, L], contiguous): every warp fills the ring, warp 0 folds it.
// vec: rows start 16-byte aligned (L % 4 == 0).
__global__ void __launch_bounds__(STATS_THREADS) gn_stats_kernel(const float* __restrict__ xs, const GroupNormParams p, long long L,
                                                                 int vec, float2* __restrict__ stats) {
    extern __shared__ float4 ring4[];
    float* ring = reinterpret_cast<float*>(ring4);
    const float* xr = xs + (long long)blockIdx.x * L;
    const int t = threadIdx.x;
    const long long nchunk = (L + RING_CHUNK - 1) / RING_CHUNK;
    auto load = [&](long long k) {
        if (k < nchunk) {
            float* dst = ring + (k % RING_STAGES) * RING_CHUNK;
            const float* src = xr + k * RING_CHUNK;
            const int len = (int)(L - k * RING_CHUNK < RING_CHUNK ? L - k * RING_CHUNK : RING_CHUNK);
            if (vec) {
                for (int f = t; f < len / 4; f += STATS_THREADS) cp_async16(dst + 4 * f, src + 4 * f);
            } else {
                for (int i = t; i < len; i += STATS_THREADS) cp_async4(dst + i, src + i);
            }
        }
        cp_async_commit();  // (an empty group past the end keeps the wait counts uniform)
    };
    float mean = 0.0f, total = 0.0f;
    for (int pass = 0; pass < 2; pass++) {
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int k = 0; k < RING_STAGES - 1; k++) load(k);
        for (long long k = 0; k < nchunk; k++) {
            cp_async_wait<RING_STAGES - 2>();
            __syncthreads();  // chunk k has landed for every thread; stage (k - 1) % RING_STAGES has been folded
            load(k + RING_STAGES - 1);
            if (t < 32) {
                const float* s = ring + (k % RING_STAGES) * RING_CHUNK;
                const int len = (int)(L - k * RING_CHUNK < RING_CHUNK ? L - k * RING_CHUNK : RING_CHUNK);
                const int F = len / 64;
                if (pass == 0) smem_fold_chunks<false>(acc, reinterpret_cast<const float4*>(s), F, 0.0f);
                else smem_fold_chunks<true>(acc, reinterpret_cast<const float4*>(s), F, mean);
                if (k == nchunk - 1)
                    total = pass == 0 ? smem_fold_finish<false>(acc, s + 64 * F, len - 64 * F, 0.0f)
                                      : smem_fold_finish<true>(acc, s + 64 * F, len - 64 * F, mean);
            }
        }
        cp_async_wait<0>();
        __syncthreads();  // the ring is free for the next pass
        if (pass == 0) mean = __fdiv_rn(total, (float)L);
    }
    if (t == 0) {
        const int g = (int)(blockIdx.x % (unsigned)p.G);
        const float var = __fdiv_rn(total, (float)L);
        stats[blockIdx.x] = make_float2(mean, __fdiv_rn(__ldg(p.inst_scale + g), __fsqrt_rn(__fadd_rn(var, p.eps))));
    }
}

// (mean, rstd) of row `row` = (n, g): the statistics pass's, or BatchNormalization's constants of channel g (bn_mean set)
__device__ __forceinline__ float2 row_stats(const GroupNormParams& p, const float2* __restrict__ stats, const float* __restrict__ bn_mean,
                                            const float* __restrict__ bn_var, long long row, int g) {
    if (!bn_mean) return stats[row];
    return make_float2(__ldg(bn_mean + g), __fdiv_rn(__ldg(p.inst_scale + g), __fsqrt_rn(__fadd_rn(__ldg(bn_var + g), p.eps))));
}

// The output of the streaming path, and BatchNormalization, over all SMs.  NCHW, k == 0: blockIdx.y walks the (n, c)
// planes, threads the plane's pixels.  NCHW, k > 0 (planes of at most blockDim.x / k units): each block takes k whole
// planes at a time, thread t unit t % n4 of plane t / n4, so small planes do not leave most of a block idle.
// Channels-last: blockIdx.y walks the images; thread i of an image keeps the channel unit i % CU (CU = C / 4 float4s
// with vec, else C floats) and walks the pixels i / CU, i / CU + k, ...  vec: 16-byte accesses.  bn_mean / bn_var:
// BatchNormalization's mean and variance (G = C, no `stats`), else null.
template <bool CL>
__global__ void __launch_bounds__(APPLY_THREADS) gn_apply_kernel(const GroupNormParams p, const float2* __restrict__ stats, int vec,
                                                                 int k, const float* __restrict__ bn_mean, const float* __restrict__ bn_var) {
    const int cg = p.C / p.G;
    const long long P = p.P;
    if (!CL) {
        const long long n4 = vec ? P / 4 : P;
        // unit f of plane `plane`
        auto unit = [&](long long plane, long long f, float2 st, float ib, float gm, float bt) {
            const float* xp = p.x + plane * P;
            float* yp = p.y + plane * P;
            if (vec) {
                float4 v = reinterpret_cast<const float4*>(xp)[f];
                v.x = gn_out(p, v.x, st.x, st.y, ib, gm, bt);
                v.y = gn_out(p, v.y, st.x, st.y, ib, gm, bt);
                v.z = gn_out(p, v.z, st.x, st.y, ib, gm, bt);
                v.w = gn_out(p, v.w, st.x, st.y, ib, gm, bt);
                reinterpret_cast<float4*>(yp)[f] = v;
            } else {
                yp[f] = gn_out(p, xp[f], st.x, st.y, ib, gm, bt);
            }
        };
        auto plane_consts = [&](long long plane, float2* st, float* ib, float* gm, float* bt) {
            const int c = (int)(plane % p.C);
            *st = row_stats(p, stats, bn_mean, bn_var, (plane / p.C) * p.G + c / cg, c / cg);
            *ib = __ldg(p.inst_bias + c / cg), *gm = p.gamma ? __ldg(p.gamma + c) : 1.0f, *bt = p.beta ? __ldg(p.beta + c) : 0.0f;
        };
        float2 st;
        float ib, gm, bt;
        if (k > 0) {
            const int lp = (int)(threadIdx.x / n4), f = (int)(threadIdx.x - lp * n4);
            if (lp >= k) return;
            for (long long plane = (long long)blockIdx.x * k + lp; plane < p.N * p.C; plane += (long long)gridDim.x * k) {
                plane_consts(plane, &st, &ib, &gm, &bt);
                unit(plane, f, st, ib, gm, bt);
            }
            return;
        }
        for (long long plane = blockIdx.y; plane < p.N * p.C; plane += gridDim.y) {
            plane_consts(plane, &st, &ib, &gm, &bt);
            for (long long f = (long long)blockIdx.x * blockDim.x + threadIdx.x; f < n4; f += (long long)gridDim.x * blockDim.x)
                unit(plane, f, st, ib, gm, bt);
        }
        return;
    }
    const int CU = vec ? p.C / 4 : p.C, W = vec ? 4 : 1;
    const int i0 = blockIdx.x * blockDim.x + threadIdx.x;
    if (i0 >= CU * k) return;
    const int cu = i0 % CU;
    for (long long n = blockIdx.y; n < p.N; n += gridDim.y) {
        float mean[4], rstd[4], ib[4], gm[4], bt[4];
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const int c = cu * W + (j < W ? j : 0);
            const float2 st = row_stats(p, stats, bn_mean, bn_var, n * p.G + c / cg, c / cg);
            mean[j] = st.x, rstd[j] = st.y;
            ib[j] = __ldg(p.inst_bias + c / cg);
            gm[j] = p.gamma ? __ldg(p.gamma + c) : 1.0f;
            bt[j] = p.beta ? __ldg(p.beta + c) : 0.0f;
        }
        const float* xi = p.x + n * P * p.C;
        float* yi = p.y + n * P * p.C;
        for (long long px = i0 / CU; px < P; px += k) {
            if (vec) {
                float4 v = reinterpret_cast<const float4*>(xi)[px * CU + cu];
                v.x = gn_out(p, v.x, mean[0], rstd[0], ib[0], gm[0], bt[0]);
                v.y = gn_out(p, v.y, mean[1], rstd[1], ib[1], gm[1], bt[1]);
                v.z = gn_out(p, v.z, mean[2], rstd[2], ib[2], gm[2], bt[2]);
                v.w = gn_out(p, v.w, mean[3], rstd[3], ib[3], gm[3], bt[3]);
                reinterpret_cast<float4*>(yi)[px * CU + cu] = v;
            } else {
                yi[px * CU + cu] = gn_out(p, xi[px * CU + cu], mean[0], rstd[0], ib[0], gm[0], bt[0]);
            }
        }
    }
}

// gn_apply_kernel over the whole tensor: NCHW one (n, c) plane per block row -- or, for BatchNormalization's planes of
// at most half a block, whole planes packed into each block -- channels-last k pixels per sweep
static rten_status launch_apply(rten_ctx* ctx, const GroupNormParams& p, const float2* stats, const float* bn_mean = nullptr,
                                const float* bn_var = nullptr) {
    auto al16 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
    const long long blocks_wanted = 8LL * ctx->num_sms;
    if (!p.channels_last) {
        const int vec = p.P % 4 == 0 && al16(p.x) && al16(p.y);
        const long long n4 = vec ? p.P / 4 : p.P, planes = p.N * p.C;
        if (bn_mean && n4 <= APPLY_THREADS / 2) {
            const long long k = APPLY_THREADS / n4, gx = std::min<long long>((planes + k - 1) / k, 4 * blocks_wanted);
            return launch(ctx, "batch_norm launch", gn_apply_kernel<false>, {dim3((unsigned)gx), dim3(APPLY_THREADS)}, p, stats, vec,
                          (int)k, bn_mean, bn_var);
        }
        const long long gy = std::min<long long>(planes, 65535);
        const long long gx = std::max<long long>(1, std::min<long long>((n4 + APPLY_THREADS * 4 - 1) / (APPLY_THREADS * 4),
                                                                        (blocks_wanted + gy - 1) / gy));
        return launch(ctx, "group_norm apply launch", gn_apply_kernel<false>, {dim3((unsigned)gx, (unsigned)gy), dim3(APPLY_THREADS)}, p,
                      stats, vec, 0, bn_mean, bn_var);
    }
    const int vec = p.C % 4 == 0 && al16(p.x) && al16(p.y);
    const long long CU = vec ? p.C / 4 : p.C, gy = std::min<long long>(p.N, 65535);
    // k pixels per sweep: about blocks_wanted CTAs in all, each thread walking at least four pixels
    long long k = std::max<long long>(1, (blocks_wanted / gy) * APPLY_THREADS / CU);
    k = std::min<long long>(k, std::max<long long>(1, (p.P + 3) / 4));
    const long long gx = (CU * k + APPLY_THREADS - 1) / APPLY_THREADS;
    return launch(ctx, "group_norm apply launch", gn_apply_kernel<true>, {dim3((unsigned)gx, (unsigned)gy), dim3(APPLY_THREADS)}, p,
                  stats, vec, (int)k, bn_mean, bn_var);
}

rten_status launch_batch_norm(rten_ctx* ctx, const GroupNormParams& p, const float* mean, const float* var) {
    if (p.N == 0 || p.C == 0 || p.P == 0) return RTEN_OK;
    return launch_apply(ctx, p, nullptr, mean, var);
}

rten_status launch_group_norm(rten_ctx* ctx, const GroupNormParams& p) {
    if (p.N == 0 || p.C == 0 || p.P == 0) return RTEN_OK;
    const int cg = p.C / p.G;
    const long long L = (long long)cg * p.P, rows = p.N * p.G;
    if (rows > INT_MAX || L > INT_MAX / 2 || p.P * p.C > INT_MAX)
        return fail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "normalization rows beyond 2^30 elements are not supported");
    auto al16 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
    const bool cl = p.channels_last != 0;
    if (L <= ONCHIP_MAX && !getenv("RTEN_B200_GROUP_NORM_STREAM")) {
        const int threads = (int)std::min<long long>(1024, std::max<long long>(128, ((L + 15) / 16 + 31) / 32 * 32));
        const size_t smem = (size_t)(L + 3) / 4 * 16;
        const int vec = !cl && L % 4 == 0 && al16(p.x) && al16(p.y);
        const LaunchShape s{dim3((unsigned)rows), dim3((unsigned)threads), smem, smem > 48 * 1024 ? (int)smem : 0};
        return cl ? launch(ctx, "group_norm launch", gn_onchip_kernel<true>, s, p, vec)
                  : launch(ctx, "group_norm launch", gn_onchip_kernel<false>, s, p, vec);
    }
    // streaming: the statistics from [N, C, P] rows, then the output pass
    const float* xs = p.x;
    if (cl) {
        void* xc = nullptr;
        RTB_TRY(temp_alloc(ctx, (size_t)(p.N * p.C * p.P) * 4, &xc));
        const long long shape[3] = {p.N, p.C, p.P}, ss[3] = {p.P * p.C, 1, p.C}, ds[3] = {p.C * p.P, p.P, 1};
        RTB_TRY(launch_nd_copy(ctx, 4, p.x, xc, 3, shape, ss, ds));
        xs = (const float*)xc;
    }
    float2* stats = nullptr;
    RTB_TRY(temp_alloc(ctx, (size_t)rows * sizeof(float2), (void**)&stats));
    const size_t ring = (size_t)RING_STAGES * RING_CHUNK * 4;
    RTB_TRY(launch(ctx, "group_norm stats launch", gn_stats_kernel, {dim3((unsigned)rows), dim3(STATS_THREADS), ring, (int)ring}, xs, p, L,
                   (int)(L % 4 == 0 && al16(xs)), stats));
    return launch_apply(ctx, p, stats);
}

}  // namespace rtb
