// Per-call scope used by every operator entry point: stages host tensors through HBM, allocates /
// validates outputs, and at the end copies host outputs back and releases temporaries.
#pragma once
#include <vector>

#include "common.h"

struct rten_packed {
    int kind = 0;   // 0: MatMul B, 1: Conv weight
    int dtype = RTEN_F32;
    // matmul: B [K, N] stored K-major as [N, ld]
    int64_t K = 0, N = 0, ld = 0;
    // conv: [O, kh*kw, Cg] (K-major, pitch per tap = Cg)
    int64_t O = 0, Cg = 0, kh = 0, kw = 0;
    int groups = 1;
    void* data = nullptr;
    int32_t* colsum = nullptr;  // int8: sum over K per output column / channel
    void* x3 = nullptr;         // f32: [hi | lo | hi] copy for the 3xTF32 mode, built by the first launch that needs it (cudaMalloc)
    // conv transpose (kind 2): W [C_in, C_out/groups, kh, kw] with O = C_out, Cg = C_in/groups, kh, kw, groups as above;
    // one conv-weight pack (kind 1) per residue phase (ry, rx) of the strides, row-major, null where it has no taps
    int64_t sy = 1, sx = 1, dy = 1, dx = 1;
    std::vector<rten_packed*> phases;
};

namespace rtb {

struct OpScope {
    rten_ctx* ctx;
    bool host_involved = false;
    struct Copyback {
        void* host;
        void* dev;
        size_t bytes;
    };
    std::vector<Copyback> copybacks;
    std::vector<rten_tensor*> allocated;

    explicit OpScope(rten_ctx* c) : ctx(c) { cudaSetDevice(c->device); }

    // device view of an input (H2D copy of the spanned region for host tensors)
    rten_status in(const rten_tensor* t, rten_tensor* view);
    // device view of an output; allocates when o->data == NULL (optionally with the given strides)
    rten_status out(rten_tensor* o, int dtype, int ndim, const int64_t* shape, rten_tensor* view,
                    const int64_t* preferred_strides);
    // contiguous device copy (no-op when already contiguous)
    rten_status contiguous(const rten_tensor* v, rten_tensor* c);
    rten_status finish(rten_status st);
};

// a tensor with no data, shape or strides, for an entry point to allocate
inline rten_tensor empty_tensor() {
    rten_tensor t;
    memset(&t, 0, sizeof(t));
    return t;
}

// releases a temporary an entry point allocated
inline void free_if(rten_ctx* ctx, rten_tensor& t) {
    if (t.data) rten_b200_free(ctx, t.data);
    t.data = nullptr;
}

}  // namespace rtb
