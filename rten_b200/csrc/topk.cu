// TopK for k >= 2 (src/ops/reduce.rs topk): the k largest composite keys of each lane (select.cuh), written largest
// first with their indices and the elements' values.  k = 1 runs on the arg-reduce kernels (reduce.cu).
//   - lanes of up to TW_MAX elements: one warp per lane bitonic-sorts the lane's composite keys in shared memory and
//     writes the first k (topk_warp_kernel);
//   - longer lanes: one thread-block cluster of C CTAs per lane (topk_cluster_kernel).  CTA `rank` holds the 32-bit
//     value keys (the composite key's high word) of its contiguous slice of the lane in shared memory, read from global
//     memory once.  A radix select in four 8-bit passes finds the k-th largest key T: each pass every CTA histograms
//     its keys that match the digits found so far, and every CTA sums the cluster's histograms through distributed
//     shared memory.  Keys above T are all taken; ties at T are taken lowest index first, which a prefix over the CTAs'
//     tie counts assigns (CTA rank order is index order).  The k selected composite keys are written into rank 0's
//     shared memory, which sorts them and writes the outputs.  A lane longer than C slices of shared memory runs the
//     same kernel with GMEM = true: every pass reads the slice from global memory again.
#include <cooperative_groups.h>
#include <cuda_runtime.h>

#include <algorithm>

#include "common.h"
#include "reduce.h"

namespace rtb {

namespace {

namespace cg = cooperative_groups;

constexpr int TW_WARPS = 4, TW_MAX = 1024;  // warp kernel: a lane of up to 1024 keys per warp, 8 KB each
constexpr int TC_THREADS = 512, TC_WARPS = TC_THREADS / 32;
constexpr int TC_SLICE = 40960;     // value keys per CTA in shared memory (160 KB)
constexpr int TC_MIN_SLICE = 2048;  // a cluster gives each CTA at least this many elements

__device__ __forceinline__ int pow2_ceil(int n) { return n <= 1 ? 1 : 1 << (32 - __clz(n - 1)); }

// bitonic sort of s[0, N), N a power of two, largest first, by threads t = 0 .. nt - 1; sync() between stages
template <typename Sync>
__device__ __forceinline__ void bitonic_desc(uint64_t* s, int N, int t, int nt, Sync sync) {
    for (int size = 2; size <= N; size <<= 1) {
        for (int stride = size >> 1; stride > 0; stride >>= 1) {
            for (int q = t; q < (N >> 1); q += nt) {
                const int i = 2 * q - (q & (stride - 1)), j = i + stride;
                const uint64_t a = s[i], b = s[j];
                if ((a < b) == ((i & size) == 0)) s[i] = b, s[j] = a;
            }
            sync();
        }
    }
}

template <typename T>
__device__ __forceinline__ void topk_store(const SelectParams& p, const T* x, long long yo, int i, uint64_t key) {
    const uint32_t j = ~(uint32_t)key;
    static_cast<int*>(p.r.y)[yo + i * p.ys] = (int)j;
    static_cast<T*>(p.vals)[yo + i * p.ys] = x[j * p.r.rx[0]];
}

template <typename T>
__global__ void __launch_bounds__(TW_WARPS * 32) topk_warp_kernel(const SelectParams p) {
    __shared__ uint64_t buf[TW_WARPS][TW_MAX];
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int n = (int)p.r.L, N = pow2_ceil(n);
    uint64_t* s = buf[w];
    for (long long o = (long long)blockIdx.x * TW_WARPS + w; o < p.r.nout; o += (long long)gridDim.x * TW_WARPS) {
        long long xo, yo;
        out_offs(p.r, o, xo, yo);
        const T* x = static_cast<const T*>(p.r.x) + xo;
        // padding keys are 0, below every element's key (whose low word ~index is never 0)
        for (int i = lane; i < N; i += 32) s[i] = i < n ? sel_key(x[i * p.r.rx[0]], (uint32_t)i, p.mode) : 0;
        __syncwarp();
        bitonic_desc(s, N, lane, 32, [] { __syncwarp(); });
        for (int i = lane; i < p.k; i += 32) topk_store<T>(p, x, yo, i, s[i]);
        __syncwarp();  // (the next lane reuses the buffer)
    }
}

template <typename T, bool GMEM>
__global__ void __launch_bounds__(TC_THREADS) topk_cluster_kernel(const SelectParams p) {
    cg::cluster_group cl = cg::this_cluster();
    const int C = (int)cl.num_blocks(), rank = (int)cl.block_rank();
    const int tid = threadIdx.x, w = tid >> 5, lane = tid & 31;
    extern __shared__ uint32_t keys[];                      // this CTA's slice of value keys (GMEM = false)
    __shared__ uint32_t hist[2][256], tot[256];             // per-pass histograms (double buffered), the cluster's sums
    __shared__ uint32_t wabove[TC_WARPS], wtie[TC_WARPS];   // per warp: keys above T, keys equal to T
    __shared__ uint32_t counts[2];                          // this CTA: keys above T, keys equal to T
    __shared__ uint32_t found_bin, found_above, base_above, base_tie;
    __shared__ uint64_t sel[TOPK_MAX_K];                    // rank 0: the k selected composite keys
    const long long n = p.r.L, S = (n + C - 1) / C, xs = p.r.rx[0];
    const long long j0 = min(n, rank * S);
    const int m = (int)(min(n, j0 + S) - j0);
    const int k = p.k, mode = p.mode;
    // warp w owns slice positions [w * R, w * R + R), R a multiple of 32
    const int R = ((m + TC_WARPS - 1) / TC_WARPS + 31) & ~31;
    const int w0 = min(m, w * R), w1 = min(m, w0 + R);
    for (long long o = blockIdx.x / C; o < p.r.nout; o += gridDim.x / C) {
        long long xo, yo;
        out_offs(p.r, o, xo, yo);
        const T* x = static_cast<const T*>(p.r.x) + xo + j0 * xs;
        auto key = [&](int i) -> uint32_t { return GMEM ? sel_high(x[i * xs], mode) : keys[i]; };
        if (!GMEM)
            for (int i = tid; i < m; i += TC_THREADS) keys[i] = sel_high(x[i * xs], mode);
        // ---- radix select: prefix holds the digits of T found so far, krem the keys still to take at or below it
        uint32_t prefix = 0, mask = 0;
        int krem = k;
#pragma unroll 1
        for (int pass = 0; pass < 4; pass++) {
            const int shift = 24 - 8 * pass;
            uint32_t* h = hist[pass & 1];
            if (tid < 256) h[tid] = 0;
            __syncthreads();
            for (int i = tid; i < m; i += TC_THREADS) {
                const uint32_t kk = key(i);
                if ((kk & mask) == prefix) atomicAdd(&h[(kk >> shift) & 255], 1u);
            }
            cl.sync();  // every histogram of this pass is complete
            if (tid < 256) {
                uint32_t t = 0;
                for (int q = 0; q < C; q++) t += cl.map_shared_rank(h, q)[tid];
                tot[tid] = t;
            }
            __syncthreads();
            if (w == 0) {
                // lane l holds bins 8l .. 8l + 7; `above` counts the keys in higher bins
                uint32_t b[8], lsum = 0;
#pragma unroll
                for (int q = 0; q < 8; q++) lsum += (b[q] = tot[8 * lane + q]);
                uint32_t incl = lsum;  // inclusive sum over lanes >= lane
#pragma unroll
                for (int d = 1; d < 32; d <<= 1) {
                    const uint32_t v = __shfl_down_sync(0xffffffffu, incl, d);
                    if (lane + d < 32) incl += v;
                }
                uint32_t above = incl - lsum;
#pragma unroll
                for (int q = 7; q >= 0; q--) {
                    if (above < (uint32_t)krem && above + b[q] >= (uint32_t)krem) found_bin = 8 * lane + q, found_above = above;
                    above += b[q];
                }
            }
            __syncthreads();
            prefix |= found_bin << shift;
            mask |= 255u << shift;
            krem -= (int)found_above;
        }
        // ---- T = prefix: every key above it is taken, and the krem ties at T of lowest index
        const uint32_t T_ = prefix;
        uint32_t na = 0, nt = 0;
        for (int i0 = w0; i0 < w1; i0 += 32) {
            const int i = i0 + lane;
            const uint32_t kk = i < w1 ? key(i) : 0;
            na += __popc(__ballot_sync(0xffffffffu, i < w1 && kk > T_));
            nt += __popc(__ballot_sync(0xffffffffu, i < w1 && kk == T_));
        }
        if (lane == 0) wabove[w] = na, wtie[w] = nt;
        __syncthreads();
        if (tid == 0) {
            uint32_t a = 0, t = 0;
            for (int q = 0; q < TC_WARPS; q++) a += wabove[q], t += wtie[q];
            counts[0] = a, counts[1] = t;
        }
        cl.sync();  // every CTA's counts are visible
        if (tid == 0) {
            uint32_t a = 0, t = 0;
            for (int q = 0; q < rank; q++) {
                const uint32_t* c = cl.map_shared_rank(counts, q);
                a += c[0], t += c[1];
            }
            base_above = a, base_tie = t;
        }
        __syncthreads();
        // this warp's first output position among the keys above T, and its first tie ordinal
        uint32_t a = base_above, t = base_tie;
        for (int q = 0; q < w; q++) a += wabove[q], t += wtie[q];
        uint64_t* dst = cl.map_shared_rank(sel, 0);
        for (int i0 = w0; i0 < w1; i0 += 32) {
            const int i = i0 + lane;
            const uint32_t kk = i < w1 ? key(i) : 0;
            const unsigned ba = __ballot_sync(0xffffffffu, i < w1 && kk > T_);
            const unsigned bt = __ballot_sync(0xffffffffu, i < w1 && kk == T_);
            const unsigned lt = (1u << lane) - 1;
            const uint64_t ck = ((uint64_t)kk << 32) | ~(uint32_t)(j0 + i);
            if ((ba >> lane) & 1) dst[a + __popc(ba & lt)] = ck;
            if ((bt >> lane) & 1) {
                const uint32_t ord = t + __popc(bt & lt);
                if (ord < (uint32_t)krem) dst[(k - krem) + ord] = ck;
            }
            a += __popc(ba), t += __popc(bt);
        }
        cl.sync();  // the k keys are in rank 0's sel
        if (rank == 0) {
            const int N = pow2_ceil(k);
            for (int i = k + tid; i < N; i += TC_THREADS) sel[i] = 0;
            __syncthreads();
            bitonic_desc(sel, N, tid, TC_THREADS, [] { __syncthreads(); });
            const T* xl = static_cast<const T*>(p.r.x) + xo;
            for (int i = tid; i < k; i += TC_THREADS) topk_store<T>(p, xl, yo, i, sel[i]);
        }
        cl.sync();  // rank 0 is done with sel before the next lane writes it
    }
}

template <typename T>
rten_status launch_topk_typed(rten_ctx* ctx, const SelectParams& p) {
    const long long n = p.r.L, rows = p.r.nout;
    if (n <= TW_MAX) {
        const long long cap = (long long)ctx->num_sms * 16;
        const LaunchShape s{dim3((unsigned)std::min(cap, (rows + TW_WARPS - 1) / TW_WARPS)), dim3(TW_WARPS * 32)};
        return launch(ctx, "topk launch", topk_warp_kernel<T>, s, p);
    }
    // enough clusters to cover the SMs, each CTA with at least TC_MIN_SLICE elements; as many CTAs as the slices in
    // shared memory need, or 16 re-reading global memory
    int C = (int)std::min({16LL, (ctx->num_sms + rows - 1) / rows, (n + TC_MIN_SLICE - 1) / TC_MIN_SLICE});
    C = std::max(C, 1);
    const size_t full = (size_t)TC_SLICE * 4;
    const int C16 = cluster_size_fit<topk_cluster_kernel<T, false>>(16, LaunchShape{dim3(16), dim3(TC_THREADS), full, (int)full});
    const long long need = (n + TC_SLICE - 1) / TC_SLICE;
    LaunchShape s{dim3(1), dim3(TC_THREADS)};
    if (need <= C16) {
        C = std::min(std::max(C, (int)need), C16);
        s.smem = (size_t)((n + C - 1) / C) * 4;
        s.smem_optin = (int)s.smem;
        s.grid = dim3((unsigned)(std::min(rows, 65535LL) * C));
        s.cluster = C;
        return launch(ctx, "topk launch", topk_cluster_kernel<T, false>, s, p);
    }
    C = C16;
    s.grid = dim3((unsigned)(std::min(rows, 65535LL) * C));
    s.cluster = C;
    return launch(ctx, "topk launch", topk_cluster_kernel<T, true>, s, p);
}

}  // namespace

rten_status launch_topk(rten_ctx* ctx, int dtype, const SelectParams& p) {
    if (p.r.nout == 0 || p.k == 0) return RTEN_OK;
    if (p.k == 1) return launch_arg_reduce(ctx, dtype, p);
    if (p.k > TOPK_MAX_K) return fail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "TopK: k > 2048 is not supported");
    return dtype == RTEN_F32 ? launch_topk_typed<float>(ctx, p) : launch_topk_typed<int>(ctx, p);
}

}  // namespace rtb
