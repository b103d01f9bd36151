// Launchers of the recurrent kernels of GRU and LSTM (rnn.cu; src/ops/rnn.rs gru / lstm).  The input projection
// x . W^T of every time step runs before them as one GEMM (api_rnn.cu); these kernels add the biases and the recurrent
// product h . R^T step by step and apply the gate arithmetic.
#pragma once
#include <cstdint>

#include "common.h"

namespace rtb {

// One GRU (G = 3, gates z, r, h) or LSTM (G = 4, gates i, o, f, c) layer over T steps.  Element strides throughout.
struct RnnLaunch {
    int gru = 0;
    int T = 0, B = 0, H = 0, dirs = 1;
    int reverse = 0;            // direction = reverse (dirs == 1); with dirs == 2 direction 1 always runs backwards
    const float* xp = nullptr;  // [T, B, dirs * G * H] contiguous: x . W^T without bias
    const float* r = nullptr;   // R [dirs, G * H, H]
    long long r_d = 0, r_row = 0, r_k = 0;
    const float* bias = nullptr;  // [dirs, 2 * G * H] (input biases, then recurrent biases) or null
    long long b_d = 0, b_k = 0;
    const float* h0 = nullptr;  // [dirs, B, H] or null (zeros)
    long long h0_d = 0, h0_b = 0, h0_k = 0;
    const float* c0 = nullptr;  // LSTM only, as h0
    long long c0_d = 0, c0_b = 0, c0_k = 0;
    float* y = nullptr;  // [T, dirs, B, H] or null
    long long y_t = 0, y_d = 0, y_b = 0, y_k = 0;
    float* yh = nullptr;  // [dirs, B, H] or null
    long long yh_d = 0, yh_b = 0, yh_k = 0;
    float* yc = nullptr;  // LSTM only, as yh
    long long yc_d = 0, yc_b = 0, yc_k = 0;
};

// The whole recurrence in ONE launch of rnn_cluster_kernel: one thread-block cluster per (direction, batch slice), its
// CTAs holding R's rows in shared memory for all T steps and exchanging h through distributed shared memory.
// RTEN_ERR_UNSUPPORTED_VALUE (ctx->err untouched) when R does not fit the cluster's shared memory or the cluster does
// not schedule; the caller then takes the per-step path.
rten_status launch_rnn_cluster(rten_ctx* ctx, const RnnLaunch& L);

// Per-step path.  State buffers h / c [dirs, B, ld] (ld >= H; c: LSTM only; either may be null in the init), set by
// launch_rnn_state_init from h0 / c0 (or zeros), which with T == 0 also writes Y_h / Y_c.  Step `s` (0-based, s < T)
// reads the recurrent product rec [dirs, B, G * H] (h . R^T without bias, contiguous), updates h / c in place and
// writes Y (and Y_h / Y_c when s == T - 1).
rten_status launch_rnn_state_init(rten_ctx* ctx, const RnnLaunch& L, float* h, float* c, int ld);
rten_status launch_rnn_step_gates(rten_ctx* ctx, const RnnLaunch& L, int s, const float* rec, float* h, float* c, int ld);

}  // namespace rtb
