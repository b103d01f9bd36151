// Depthwise convolution (groups = in channels = out channels) as one direct kernel launch (depthwise.cu).  All pointers
// are device pointers; the launch goes to ctx->stream.
#pragma once
#include <cstdint>

#include "common.h"

namespace rtb {

struct DepthwiseParams {
    int x_dtype, w_dtype;  // RTEN_F32 for both, or RTEN_U8 / RTEN_I8 each (ConvInteger)
    int B, C, H, W, OH, OW, kh, kw, sy, sx, dy, dx, pt, pl;
    const void* x;
    long long xs[4];  // element strides of x (b, c, h, w)
    const void* w;
    long long ws_c, ws_h, ws_w;  // element strides of the weight's channel, row and column ([C, 1, kh, kw] or its pack)
    void* out;                   // f32, or i32 for ConvInteger without a scale
    long long os[4];
    const float* bias = nullptr;  // [C], bias_stride apart
    long long bias_stride = 1;
    const float* res = nullptr;  // residual laid out like out (its own strides)
    long long rs[4] = {0, 0, 0, 0};
    int act = 0;  // apply_act code (integer outputs: 0 or 1)
    float act_alpha = 0.0f, act_beta = 0.0f;  // HardSigmoid's (act 6)
    // ConvInteger: zero points in their own 8-bit type, read on the device; w_zp one per channel (w_zp_stride apart) or a
    // scalar (stride 0)
    const void* x_zp = nullptr;
    const void* w_zp = nullptr;
    long long w_zp_stride = 0;
    const float* scale = nullptr;    // scalar: f32 output = f32(acc) * (scale_b * scale)
    const float* scale_b = nullptr;  // optional scalar
    int* range = nullptr;            // optional (min, max) of the f32 output, ordered-int encoded
};

rten_status launch_depthwise(rten_ctx* ctx, const DepthwiseParams& p);

}  // namespace rtb
