// Per-call scope used by every operator entry point: stages host tensors through HBM, allocates /
// validates outputs, and at the end copies host outputs back and releases temporaries.
#pragma once
#include <memory>
#include <vector>

#include "common.h"
#include "rowops.h"

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

// a pack under construction, freed unless released to the caller
struct PackedFree {
    rten_ctx* ctx;
    void operator()(rten_packed* p) const { rten_b200_packed_free(ctx, p); }
};
using PackedPtr = std::unique_ptr<rten_packed, PackedFree>;

// An entry point opens one scope after its argument checks and returns success only through `return sc.finish(...)`.
// Any other return from inside the scope is a failure: the destructor then frees the outputs the call allocated (their
// `data` back to NULL), releases the temporaries and synchronises when a host tensor was staged.  Scopes do not nest
// (the temporaries live on the context): an entry point calls another only after its own scope has closed.
struct OpScope {
    rten_ctx* ctx;
    bool host_involved = false;
    bool finished = false;
    struct Copyback {
        void* host;
        void* dev;
        size_t bytes;
    };
    std::vector<Copyback> copybacks;
    std::vector<rten_tensor*> allocated;

    explicit OpScope(rten_ctx* c) : ctx(c) { cudaSetDevice(c->device); }
    OpScope(const OpScope&) = delete;
    OpScope& operator=(const OpScope&) = delete;
    // (any failing status takes finish's failure path, which leaves the context's error message as it is)
    ~OpScope() {
        if (!finished) finish(RTEN_ERR_CUDA);
    }

    // device view of an input (H2D copy of the spanned region for host tensors)
    rten_status in(const rten_tensor* t, rten_tensor* view);
    // device view of an output; allocates when o->data == NULL (optionally with the given strides)
    rten_status out(rten_tensor* o, int dtype, int ndim, const int64_t* shape, rten_tensor* view,
                    const int64_t* preferred_strides);
    // contiguous device copy (no-op when already contiguous)
    rten_status contiguous(const rten_tensor* v, rten_tensor* c);
    // success: host outputs copied back; failure: allocated outputs freed.  Either way the temporaries are released.
    rten_status finish(rten_status st);
};

// copies the device view `src` into the device view `dst` of the same shape
inline rten_status copy_view(rten_ctx* ctx, const rten_tensor& src, const rten_tensor& dst) {
    long long shape[RTEN_MAX_DIMS], ss[RTEN_MAX_DIMS], ds[RTEN_MAX_DIMS];
    for (int i = 0; i < src.ndim; i++) {
        shape[i] = src.shape[i];
        ss[i] = src.strides[i];
        ds[i] = dst.strides[i];
    }
    return launch_nd_copy(ctx, dtype_size(src.dtype), src.data, dst.data, src.ndim, shape, ss, ds);
}

inline rten_status check_ctx(rten_ctx* ctx) { return ctx ? RTEN_OK : RTEN_ERR_INVALID_VALUE; }

// An intermediate of a composed operator: starts with no data, shape or strides for an entry point to allocate, and goes
// back to the pool when it goes out of scope.
struct Intermediate : rten_tensor {
    rten_ctx* ctx;
    explicit Intermediate(rten_ctx* c) : rten_tensor(), ctx(c) {}
    Intermediate(const Intermediate&) = delete;
    Intermediate& operator=(const Intermediate&) = delete;
    ~Intermediate() {
        if (data) rten_b200_free(ctx, data);
    }
};

}  // namespace rtb
