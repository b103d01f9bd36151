// ReduceSum and the arg-reduce family (reduce.cu), TopK (topk.cu).  All pointers are device pointers; all launches go to
// ctx->stream.
#pragma once
#include <map>
#include <mutex>

#include "common.h"
#include "select.cuh"

namespace rtb {

// y[o] = the sum of the L elements x[xoff(o) + roff(j)], j < L, one output per o < nout, where
//   xoff(o) = sum_k idx_k(o) ox[k] over the kept dims (shape os, row-major),
//   roff(j) = sum_k idx_k(j) rx[k] over the reduced dims (shape rs, row-major, ascending axis order),
//   yoff(o) = sum_k idx_k(o) oy[k].
// f32 sums are the reference's Sum (rten-vecmath/src/sum.rs) over the elements in j order, bit for bit; i32 sums wrap.
// L = 0 gives 0.  vec: nr == 1, rx[0] == 1 and every lane starts 16-byte aligned (16-byte loads).  mean (f32):
// ReduceMean, each sum divided by (float)L, IEEE (src/ops/reduce.rs reduce_mean; L = 0 gives NaN).
struct ReduceParams {
    const void* x = nullptr;
    void* y = nullptr;
    long long nout = 0, L = 0;
    int no = 0, nr = 0;
    long long os[RTEN_MAX_DIMS], ox[RTEN_MAX_DIMS], oy[RTEN_MAX_DIMS];
    long long rs[RTEN_MAX_DIMS], rx[RTEN_MAX_DIMS];
    int vec = 0, mean = 0;
};
rten_status launch_reduce_sum(rten_ctx* ctx, int dtype, const ReduceParams& p);

// TopK, ArgMax and ArgMin over one axis: r addresses the lanes as for ReduceSum (r.nr <= 1: the lane is the L elements
// x[xoff(o) + j * rx[0]]), r.y receives the i32 indices.  Each output row takes the k largest composite keys of its
// lane under `mode` (select.cuh), largest first: index i of row o goes to yoff(o) + i * ys, and with vals != null the
// element's value is copied there too.  ArgMax / ArgMin are k = 1 with mode SEL_ARGMAX / SEL_ARGMIN.  1 <= k <= L.
struct SelectParams {
    ReduceParams r;
    void* vals = nullptr;
    int k = 1, mode = SEL_LARGEST;
    long long ys = 0;
};
constexpr int TOPK_MAX_K = 2048;
// k = 1 (reduce.cu): one warp per lane up to 1024 elements, else one CTA per lane, or one cluster per lane when the
// lanes are too few to fill the SMs
rten_status launch_arg_reduce(rten_ctx* ctx, int dtype, const SelectParams& p);
// any k <= TOPK_MAX_K (topk.cu); k = 1 runs launch_arg_reduce
rten_status launch_topk(rten_ctx* ctx, int dtype, const SelectParams& p);

// the x and y offsets of output o
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

// The largest cluster of at most `want` CTAs that the current device can schedule with this launch shape (16-CTA
// clusters need the non-portable size and a GPC with 16 free SMs).  For `want` > 8 the answer is asked once per kernel
// and device, for the largest shared memory the caller launches the kernel with (s), and kept under a lock.
template <auto KERN>
int cluster_size_fit(int want, const LaunchShape& s) {
    if (want <= 8) return want;
    static std::mutex mu;
    static std::map<int, bool> fits16;  // device -> a 16-CTA cluster fits
    int dev = 0;
    cudaGetDevice(&dev);
    std::lock_guard<std::mutex> lock(mu);
    auto it = fits16.find(dev);
    if (it == fits16.end()) {
        auto kern = KERN;
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3(16);
        cfg.blockDim = s.block;
        cfg.dynamicSmemBytes = s.smem;
        cudaLaunchAttribute attr[1];
        attr[0].id = cudaLaunchAttributeClusterDimension;
        attr[0].val.clusterDim = {16u, 1, 1};
        cfg.attrs = attr;
        cfg.numAttrs = 1;
        int active = 0;
        cudaError_t e = s.smem_optin > 0 ? cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, s.smem_optin)
                                         : cudaSuccess;
        if (e == cudaSuccess) e = cudaFuncSetAttribute(kern, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
        if (e == cudaSuccess) e = cudaOccupancyMaxActiveClusters(&active, kern, &cfg);
        cudaGetLastError();
        it = fits16.emplace(dev, e == cudaSuccess && active >= 1).first;
    }
    return it->second ? want : 8;
}

}  // namespace rtb
