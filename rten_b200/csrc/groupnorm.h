// InstanceNormalization, the GroupNorm chain torch exports and BatchNormalization (groupnorm.cu).  All pointers are
// device pointers; all launches go to ctx->stream.
#pragma once
#include "common.h"

namespace rtb {

// Rows r = (n, g), n < N, g < G, each the L = cg * P elements of channels g cg .. g cg + cg - 1 in logical (c, p) order.
// Every output element is, each step rounded on its own:
//   y = fma(x - mean, rstd, inst_bias[g]), rstd = inst_scale[g] / sqrt(var + eps)   (Normalize's arm 0)
//   y = y * gamma[c]  (when gamma),  y = y + beta[c]  (when beta),  y = act(y)
// with mean and var in the reference's Sum / SumSquareSub fold order.  x and y are [N, C, P] (channels_last 0) or
// [N, P, C] (channels_last 1), dense; y may be x.
struct GroupNormParams {
    const float* x = nullptr;
    float* y = nullptr;
    const float* inst_scale = nullptr;  // [G]
    const float* inst_bias = nullptr;   // [G]
    const float* gamma = nullptr;       // [C], or null
    const float* beta = nullptr;        // [C], or null
    long long N = 0;
    int C = 0, G = 0;
    long long P = 0;
    int channels_last = 0;
    float eps = 1e-5f;
    int act = 0;  // rten_activation_kind
    float act_alpha = 0.0f, act_beta = 0.0f;
};
rten_status launch_group_norm(rten_ctx* ctx, const GroupNormParams& p);
// BatchNormalization: G = C and no statistics pass; channel c's mean is mean[c] ([C]) and its rstd is
// inst_scale[c] / sqrt(var[c] + eps), each step rounded on its own; inst_bias[c] is the operator's bias.  One launch of
// the output pass.  Any N, C, P whose channel count fits an int.
rten_status launch_batch_norm(rten_ctx* ctx, const GroupNormParams& p, const float* mean, const float* var);

}  // namespace rtb
