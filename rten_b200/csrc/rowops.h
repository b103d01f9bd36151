// Launchers of the HBM-bound kernels (rowops.cu).  All pointers are device pointers; all launches
// go to ctx->stream.
#pragma once
#include <cstdint>

#include "common.h"

namespace rtb {

enum {
    UNARY_ERF = 0,
    UNARY_GELU = 1,
    UNARY_APPROX_GELU = 2,
    UNARY_RELU = 3,
    UNARY_SIGMOID = 4,
    UNARY_SILU = 5,
    UNARY_HARD_SIGMOID = 6,  // alpha * x + beta, clamped
    UNARY_HARD_SWISH = 7,
    UNARY_SQRT = 8,        // __fsqrt_rn
    UNARY_RECIPROCAL = 9,  // 1 / x, IEEE
    UNARY_EXP = 10,        // exp_ref
    UNARY_TANH = 11,       // tanh_ref
    UNARY_NEG = 12,        // -x (the sign bit flipped)
    UNARY_ABS = 13         // the sign bit cleared
};

// Softmax over the last (contiguous) axis of x viewed as [rows, n]; optional mask broadcast over
// up to 4 leading dims: row index is decomposed over lead[0..nlead) (row-major), mask element =
// mask[sum idx_d * mstride[d] + i * mstride_last].
rten_status launch_softmax(rten_ctx* ctx, const float* x, float* y, long long rows, int n, int flush_nan,
                           const float* mask, int nlead, const long long* lead, const long long* mstride,
                           long long mstride_last);
// LayerNormalization, RMSNormalization / SimplifiedLayerNormalization and the skip layer norms
// (SkipLayerNormalization, SkipSimplifiedLayerNormalization) over rows of n floats: s = (x + skip) + bias (skip and bias
// optional), normalised with mean and variance (rms = 0) or with the root mean square and no centring (rms = 1).  y and
// sum are dense [rows, n]; sum (the rounded s) is written when not null.  y may be x when there is no skip (in-place
// LayerNormalization); it never aliases skip, bias or sum.
struct NormParams {
    const float* x = nullptr;     // row r at x + r * xs (elements contiguous)
    const float* skip = nullptr;  // row r at skip + (r % skip_rows) * ss, or null
    const float* bias = nullptr;  // element i at bias[i * bias_inc] (bias_inc 0: one value for the row), or null
    const float* gamma = nullptr;     // [n], or null: the device scalar gamma_sp
    const float* gamma_sp = nullptr;
    const float* beta = nullptr;      // [n], or null: the device scalar beta_sp, or null: 0
    const float* beta_sp = nullptr;
    float* y = nullptr;
    float* sum = nullptr;
    long long rows = 0, skip_rows = 1, xs = 0, ss = 0;
    int n = 0, bias_inc = 1, rms = 0;
    float eps = 1e-5f;
};
rten_status launch_norm(rten_ctx* ctx, const NormParams& p);
// y[row] = Sum(x_row) / n in the reference's Sum order; row r starts at
// x + (r / rows_inner) * s_outer + (r % rows_inner) * s_inner, elements kstride apart.
rten_status launch_row_mean(rten_ctx* ctx, const float* x, float* y, long long rows, int n, long long rows_inner,
                            long long s_outer, long long s_inner, long long kstride);
// y may be x; alpha / beta are read by UNARY_HARD_SIGMOID only
rten_status launch_unary(rten_ctx* ctx, int op, const float* x, float* y, long long n, float alpha = 0.0f, float beta = 0.0f);
// Clip of n contiguous f32 (or i32) elements; y may be x; mn / mx: device scalars of the same type, or null
rten_status launch_clip(rten_ctx* ctx, int is_i32, const void* x, void* y, long long n, const void* mn, const void* mx);
rten_status launch_nd_copy(rten_ctx* ctx, int esize, const void* src, void* dst, int ndim, const long long* shape,
                           const long long* sstride, const long long* dstride);
// d = a (op) b over the iteration space `shape`, element strides sa / sb / sd (0 where an operand broadcasts): f32
// (__fadd_rn / __fsub_rn / __fmul_rn / __fdiv_rn, Pow as FastPow, then Relu when `relu`) or i32 (Add / Sub / Mul / Pow
// wrapping, Div truncating).  The flat kernel when a, b and d are dense row-major over `shape` (so a dense view of any
// layout runs flat when passed as [n] with unit strides), the periodic one when a and d are and b is a dense block of
// the trailing dims repeated over the leading ones (period a multiple of 4, fewer than 2^31 elements, 16-byte aligned
// bases), else the strided one.  Div, Pow and BIN_RCP_MUL run on kernels of their own (binary_math_*) with the same
// three layouts, so that Add / Sub / Mul keep their code and registers; a one-element b over dense a and d also runs
// their flat kernel, which reads b once.
//   BIN_RCP_MUL (f32): a * (1 / b), two roundings -- the reference's Div by a one-element divisor.
//   BIN_POW: f32 ^ f32 and i32 ^ i32 (src/ops/binary_elementwise.rs FastPow): exponent 2 is x * x, 3 is x * x * x
//     (rounded left to right), any other f32 exponent powf; a non-negative i32 exponent wraps, a negative one goes
//     through f32 and back with Rust's saturating `as i32`.
//   i32 BIN_DIV: a zero divisor or INT_MIN / -1 sets *err to 1 (err must then be a device int the caller zeroed) and
//     stores 0 there; err is read by i32 Div only.
enum BinaryOp { BIN_ADD = 0, BIN_SUB = 1, BIN_MUL = 2, BIN_DIV = 3, BIN_POW = 4, BIN_RCP_MUL = 5 };
rten_status launch_binary(rten_ctx* ctx, int dtype, int op, int relu, const void* a, const void* b, void* d, int ndim,
                          const long long* shape, const long long* sa, const long long* sb, const long long* sd,
                          int* err = nullptr);
rten_status launch_minmax(rten_ctx* ctx, const float* x, long long n, int* mm /* 2 ordered ints */);
// `xch` (batch-sharded runs): the kernel first exchanges the local range in `mm` with the other ranks (comm_device.cuh)
struct RangeExchange;
rten_status launch_dql_quantize(rten_ctx* ctx, const float* x, uint8_t* y, long long n, int* mm,
                                float* scale_out, uint8_t* zp_out, const RangeExchange* xch = nullptr);
rten_status launch_rowsum8(rten_ctx* ctx, const void* a, int is_signed, long long rows, int K, long long ld, int* out);
rten_status launch_zp_to_i32(rten_ctx* ctx, const void* zp, int is_signed, int n, long long zs, int* out);
rten_status launch_fill8(rten_ctx* ctx, void* p, long long n, uint8_t v);
rten_status launch_cast_scale(rten_ctx* ctx, const int* in, float* out, long long n, int cols, const float* scale,
                              int scale_len);

struct Im2ColParams {
    int B, C, H, W, OH, OW, kh, kw, sy, sx, dy, dx, pt, pl;
    int c0;    // first input channel (group offset)
    int kpad;  // output row pitch in elements (>= kh*kw*C, zero filled beyond)
    long long xs_b, xs_c, xs_h, xs_w;  // input element strides
};
rten_status launch_im2col(rten_ctx* ctx, int esize, const void* x, void* out, const Im2ColParams& p, int pad_value);

rten_status launch_smallc_pad(rten_ctx* ctx, const float* x, float* xp, int B, int C, int H, int W, int Wp, int pl,
                              long long xs_b, long long xs_c, long long xs_h, long long xs_w);
rten_status launch_smallc_pack_w(rten_ctx* ctx, const float* w, float* wp, int O, int C, int kh, int kw, long long ws_o,
                                 long long ws_c, long long ws_h, long long ws_w);

struct PoolParams {
    int B, C, H, W, OH, OW, kh, kw, sy, sx, pt, pl;
    long long xs_b, xs_c, xs_h, xs_w, ys_b, ys_c, ys_h, ys_w;
    int channels_fastest;  // thread -> element mapping that keeps warps coalesced for NHWC memory
};
rten_status launch_maxpool(rten_ctx* ctx, const float* x, float* y, const PoolParams& p);
rten_status launch_avgpool(rten_ctx* ctx, const float* x, float* y, const PoolParams& p, int count_include_pad);
rten_status launch_gather_rows(rten_ctx* ctx, const float* table, const int* idx, float* out, long long nidx,
                               int width, long long t_rs, long long t_cs, long long rows);

// 3xTF32 operand split: dst contiguous [d3][d2][d1][3 * d0p]; role 0 = [lo|hi|hi], 1 = [hi|lo|hi]
rten_status launch_tf32x3_split(rten_ctx* ctx, const float* x, float* y, const long long dims[4], const long long strides[4],
                                long long d0p, int role);

rten_status launch_dql_small(rten_ctx* ctx, const float* x, uint8_t* y, int n, float* scale_out, uint8_t* zp_out);

rten_status launch_scatter_rows(rten_ctx* ctx, float* table, const int* idx, const float* src, long long nidx, int width,
                                long long t_rs, long long t_cs, long long s_rs, long long s_cs, long long rows);

rten_status launch_range_reset(rten_ctx* ctx, int* mm, int pairs);

rten_status launch_smallc8_pad(rten_ctx* ctx, const void* x, void* xp, int B, int C, int H, int W, int Hp, int Wp, int pt,
                               int pl, long long xs_b, long long xs_c, long long xs_h, long long xs_w, int pad_value);
rten_status launch_smallc8_pack_w(rten_ctx* ctx, const void* w, void* wp, int O, int C, int kh, int kw, long long ws_o,
                                  long long ws_c, long long ws_h, long long ws_w);

// ConvTranspose as stride-phase convolutions (api_conv.cu).  Sub-kernel of one residue phase: taps ky0, ky0 - step_y, ...
// (Th of them) and kx0, kx0 - step_x, ... (Tw) of W [C_in, Og, kh, kw], written as the [O = groups*Og, Th, Tw, Cg] pack
struct ConvTransposePack {
    int O, Og, Cg, Th, Tw, ky0, kx0, step_y, step_x;
    long long ws_i, ws_o, ws_h, ws_w;  // W element strides
};
rten_status launch_conv_transpose_pack(rten_ctx* ctx, const float* w, float* dst, const ConvTransposePack& p);
// bias[o] (or 0 without one) into every output element of a phase without a convolution: phase (qy, qx) has one iff
// bit qy of live_y and bit qx of live_x are set (strides up to 256)
struct ConvTransposeFill {
    int B, O, OH, OW, sy, sx;
    long long s_b, s_o, s_h, s_w;  // output element strides
    uint32_t live_y[8], live_x[8];
};
rten_status launch_conv_transpose_fill(rten_ctx* ctx, float* out, const float* bias, const ConvTransposeFill& p);

rten_status launch_dql_quantize_rows(rten_ctx* ctx, const float* x, uint8_t* y, long long rows, int row_len, int rows_inner,
                                     long long y_inner, long long y_outer, int* mm, float* scale_out, uint8_t* zp_out,
                                     const RangeExchange* xch = nullptr);

}  // namespace rtb
