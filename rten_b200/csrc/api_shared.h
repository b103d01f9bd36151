// Helpers shared by the operator entry points (api_ops.cu: MatMul family, api_conv.cu: Conv family and pooling,
// api_rows.cu: row / elementwise operators, api_rnn.cu: GRU / LSTM).
#pragma once
#include <algorithm>
#include <cstdint>

#include "api_util.h"
#include "umma_gemm.h"

namespace rtb {
namespace api {

inline int64_t round_up(int64_t v, int64_t m) { return (v + m - 1) / m * m; }

// ---------------------------------------------------------------------------------------
// K-major 2-level operand: rows x K with element strides.  Packs into an aligned workspace when
// TMA cannot address the original (k stride != 1, misaligned base / pitch).
// ---------------------------------------------------------------------------------------
struct Mat {
    const void* base;
    int64_t rows, K;
    int64_t rs, ks;       // element strides
    int64_t z0 = 1, z1 = 1;  // batch dims (z0 inner)
    int64_t zs0 = 0, zs1 = 0;
};

rten_status to_kmajor(rten_ctx* ctx, int esize, const Mat& m, OperandDesc* od);

inline rten_status check_zero_point(rten_ctx* ctx, const rten_tensor* zp, int64_t expected, int want_dtype) {
    if (!zp) return RTEN_OK;
    if (zp->dtype != want_dtype) return fail(ctx, RTEN_ERR_CAST_FAILED, "zero point type does not match its tensor");
    if (zp->ndim == 0) return RTEN_OK;
    if (zp->ndim == 1) {
        if (zp->shape[0] != expected) return fail(ctx, RTEN_ERR_INVALID_VALUE, "Zero point has incorrect size");
        return RTEN_OK;
    }
    return fail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "Only scalar or vector zero points are supported");
}

// ---------------------------------------------------------------------------------------
// Conv geometry (src/ops/pooling.rs:63-159)
// ---------------------------------------------------------------------------------------
inline rten_status axis_out(rten_ctx* ctx, int64_t in, int64_t k, int64_t stride, bool same, int64_t ps, int64_t pe,
                     int64_t dil, int64_t* out, int64_t* p0, int64_t* p1) {
    if (dil <= 0) return fail(ctx, RTEN_ERR_INVALID_VALUE, "Dilations must be > 0");
    if (k <= 0) return fail(ctx, RTEN_ERR_INVALID_VALUE, "Kernel size must be > 0");
    if (stride <= 0) return fail(ctx, RTEN_ERR_INVALID_VALUE, "Strides must be > 0");
    if (same) {
        const int64_t o = (in + stride - 1) / stride;
        int64_t total = (o - 1) * stride + (k - 1) * dil + 1 - in;
        if (total < 0) total = 0;
        *out = o;
        *p0 = total / 2;
        *p1 = (total + 1) / 2;
        return RTEN_OK;
    }
    const int64_t padded = in + ps + pe;
    const int64_t dk = k + (k - 1) * (dil - 1);
    if (padded < dk) return fail(ctx, RTEN_ERR_INVALID_VALUE, "Input too small for kernel size");
    *out = (padded - dil * (k - 1) - 1) / stride + 1;
    *p0 = ps;
    *p1 = pe;
    return RTEN_OK;
}

// Validated geometry of a transposed convolution (2-D form: a 1-D one runs over a height-1 image)
struct ConvTShape {
    rten_tensor x, w;
    bool one_d = false;
    int64_t B, C, H, W, O, Og, Cg, kh, kw, OH, OW, sy, sx, dy, dx, pt, pl, pb, pr;
    int groups;
};

// ConvTranspose's argument checks on `w` (and `x` when given) and its output geometry (api_conv.cu)
rten_status conv_transpose_shape(rten_ctx* ctx, const rten_tensor* xp, const rten_tensor& w0, const rten_tensor* bias,
                                 const rten_conv_transpose_params* cp, ConvTShape& S);
// Resize's output sizes `osz` on `x` and the input / output size ratio `inv` of each axis (api_conv.cu)
rten_status resize_output_size(rten_ctx* ctx, const rten_tensor& x, const rten_resize_params* p, int64_t osz[4], float inv[4]);

}  // namespace api
}  // namespace rtb
