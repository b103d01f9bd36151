// Rotary position embedding of one element (src/ops/embedding.rs:46-207), shared by the rotary / cache-append kernel
// (rotary.cu) and the single-query attention kernel (skinny.cu).  Rows are head vectors of `d` elements; the first
// 2 * half are rotated, the rest copied.  The arithmetic is the reference's two products and one sum, each rounded on
// its own (no fused multiply-add), so rotated values equal a float32 restatement bit for bit.
#pragma once

namespace rtb {

// element i of the rotated row x (element stride xd) with the cos / sin row c / s of `half` entries
__device__ __forceinline__ float rotary_elem(const float* x, long long xd, int i, const float* c, const float* s, int half,
                                             int interleaved) {
    if (i >= 2 * half) return x[i * xd];
    int p, i1, i2;
    bool second;
    if (interleaved) {  // pairs (2p, 2p + 1)
        p = i >> 1;
        i1 = 2 * p;
        i2 = i1 + 1;
        second = i & 1;
    } else {  // halves (p, p + half)
        second = i >= half;
        p = second ? i - half : i;
        i1 = p;
        i2 = p + half;
    }
    const float x1 = x[i1 * xd], x2 = x[i2 * xd], cs = c[p], sn = s[p];
    return second ? __fadd_rn(__fmul_rn(x1, sn), __fmul_rn(x2, cs)) : __fsub_rn(__fmul_rn(x1, cs), __fmul_rn(x2, sn));
}

}  // namespace rtb
