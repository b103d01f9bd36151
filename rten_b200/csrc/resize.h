// Resize (nearest / bilinear over the last two axes of an NCHW view) and Concat kernels (resize.cu).  All pointers are
// device pointers; launches go to ctx->stream.
#pragma once
#include <cstdint>

#include "common.h"

namespace rtb {

struct ResizeParams {
    int mode, coord_mode, nearest_mode;  // rten_resize_mode / rten_resize_coord_mode / rten_resize_nearest_mode
    int B, C, H, W, OH, OW;
    float inv_y, inv_x;  // output -> input scale per axis (src/ops/resize.rs:287-298)
    const float* x;
    long long xs[4];  // element strides (b, c, h, w)
    float* out;
    long long os[4];
};
rten_status launch_resize(rten_ctx* ctx, const ResizeParams& p);

constexpr int kConcatMaxSources = 16;
constexpr int kConcatMaxDims = RTEN_MAX_DIMS;

// One source of a Concat launch: `n` elements of `ext` positions along the concat axis, stored at dst_off in the output
struct ConcatSource {
    const void* src;
    long long n, ext, dst_off;
    long long strides[kConcatMaxDims];
};
// Shape / strides in elements of `esize` bytes (1, 4 or 16: the entry point widens the element when every slice allows)
struct ConcatParams {
    int esize, ndim, axis, nsrc;
    void* out;
    long long shape[kConcatMaxDims], out_strides[kConcatMaxDims];
    ConcatSource s[kConcatMaxSources];
};
rten_status launch_concat(rten_ctx* ctx, const ConcatParams& p);

}  // namespace rtb
