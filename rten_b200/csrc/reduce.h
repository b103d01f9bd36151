// ReduceSum (reduce.cu).  All pointers are device pointers; all launches go to ctx->stream.
#pragma once
#include "common.h"

namespace rtb {

// y[o] = the sum of the L elements x[xoff(o) + roff(j)], j < L, one output per o < nout, where
//   xoff(o) = sum_k idx_k(o) ox[k] over the kept dims (shape os, row-major),
//   roff(j) = sum_k idx_k(j) rx[k] over the reduced dims (shape rs, row-major, ascending axis order),
//   yoff(o) = sum_k idx_k(o) oy[k].
// f32 sums are the reference's Sum (rten-vecmath/src/sum.rs) over the elements in j order, bit for bit; i32 sums wrap.
// L = 0 gives 0.  vec: nr == 1, rx[0] == 1 and every lane starts 16-byte aligned (16-byte loads).
struct ReduceParams {
    const void* x = nullptr;
    void* y = nullptr;
    long long nout = 0, L = 0;
    int no = 0, nr = 0;
    long long os[RTEN_MAX_DIMS], ox[RTEN_MAX_DIMS], oy[RTEN_MAX_DIMS];
    long long rs[RTEN_MAX_DIMS], rx[RTEN_MAX_DIMS];
    int vec = 0;
};
rten_status launch_reduce_sum(rten_ctx* ctx, int dtype, const ReduceParams& p);

}  // namespace rtb
