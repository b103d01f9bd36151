// Launch interface of the wgmma GEMM / implicit-GEMM-conv kernel (umma_gemm.cu).
//
// Computes, per batch z:   D[m, n] = epilogue( sum_k A[m, k] * B[n, k] )
// with BOTH operands K-major in global memory (k contiguous), fetched by TMA into 128B-swizzled
// shared-memory tiles and multiplied by wgmma (tf32 for f32 data, s8/u8 for
// u8/i8 data) with the accumulator in registers.
//
// The A operand is either a plain (k, m, z0, z1) tensor or an NHWC activation tensor addressed
// as an implicit im2col matrix: row = output pixel (b, oy, ox), k = (ky, kx, c).
#pragma once
#include <cuda.h>

#include <cstdint>

#include "common.h"

namespace rtb {

// Up-to-rank-4 strided operand description in ELEMENTS (inner dim has stride 1).
struct OperandDesc {
    const void* base = nullptr;
    int64_t dims[4] = {1, 1, 1, 1};     // dims[0] = innermost (k or c)
    int64_t strides[4] = {1, 0, 0, 0};  // elements; strides[0] must be 1
};

struct EpilogueDesc {
    void* d = nullptr;
    int d_is_i32 = 0;  // output element type: 0 f32, 1 i32
    // plain mode: offset = z0*s_z0 + z1*s_z1 + m*s_row + n*s_col
    // conv  mode: offset = b*s_z0 + oy*s_row + ox*s_z1 + n*s_col     (s_z1 plays the x stride)
    int64_t s_z0 = 0, s_z1 = 0, s_row = 0, s_col = 1;
    // optional residual / Gemm "C" term: v += r_scale * R[...] with its own (broadcastable) strides
    const float* r = nullptr;
    float r_scale = 1.0f;
    int64_t r_z0 = 0, r_z1 = 0, r_row = 0, r_col = 0;
    const float* bias = nullptr;
    int bias_kind = 0;  // 1: per column n, 2: per row m
    const float* bias2 = nullptr;  // bias_kind 1, plain f32 epilogue only: a second column bias, added to `bias` first
    float alpha = 1.0f;
    int act = 0;  // apply_act code (math.cuh): 0 none, 1 relu, 2 gelu(erf), 3 gelu(tanh), 4-7 sigmoid, silu, hard
                  // sigmoid (act_alpha, act_beta), hard swish
    // integer path: C = acc - za[m % za_len]*colsum[n] - zb[n % zb_len]*rowsum[m] + K*za*zb
    const int32_t* za = nullptr;
    int za_len = 0;
    // ... or ONE 8-bit zero point read in place (a DynamicQuantizeLinear output used as it is: no conversion launch)
    const uint8_t* za8 = nullptr;
    int za8_signed = 0;
    const int32_t* zb = nullptr;
    int zb_len = 0;
    const int32_t* rowsum = nullptr;  // sum_k A[m,k]   (needed iff zb != null)
    const int32_t* colsum = nullptr;  // sum_k B[n,k]   (needed iff za != null)
    const float* scale = nullptr;     // cast_scale fused: f32 out = f32(C) * scale[n % scale_len]
    int scale_len = 0;
    // optional: running (min, max) of the f32 OUTPUT of this launch, as two order-preserving int encodings updated with
    // atomicMin / atomicMax -- the range the next DynamicQuantizeLinear needs, computed while the data is in registers
    int* range = nullptr;
    const float* scale2 = nullptr;    // optional scalar factor: the effective scale is fmul(scale2[0], scale[n]) -- the
                                      // graph's Mul(x_scale, w_scale) node folded into the epilogue, same rounding
    // HardSigmoid's alpha / beta (act 6).  Last in the struct, which is last in KParams: the kernel parameter offsets
    // of every other field stay where they were.
    float act_alpha = 0.0f, act_beta = 0.0f;
};

struct ConvGeom {
    int B = 0, H = 0, W = 0, C = 0;  // NHWC input (C = channels of this group)
    int OH = 0, OW = 0;
    int kh = 1, kw = 1, sy = 1, sx = 1, dy = 1, dx = 1, pt = 0, pl = 0;
};

struct GemmLaunch {
    int kind = 0;      // 0: f32 data via kind::tf32; 1: 8-bit integers via kind::i8
    int a_signed = 0;  // kind 1: A is i8 (else u8)
    int b_signed = 1;  // kind 1: B is i8 (else u8)
    int M = 0, N = 0, K = 0;
    int z0 = 1, z1 = 1;  // batch dims (plain mode)
    int conv = 0;        // A addressed as implicit im2col of an NHWC tensor
    ConvGeom g;
    OperandDesc a;  // plain: (k, m, z0, z1); conv: (c, x, y, b)
    OperandDesc b;  // plain: (k, n, z0, z1) (stride 0 = broadcast); conv: (c, o, tap, 1)
    EpilogueDesc epi;
    // 3xTF32 (RTEN_F32_TF32X3), set by the caller that owns a constant B: slot caching the split copy of `b`
    // ([hi | lo | hi] along K) across launches -- weights are split once, not per call (owned by the rten_packed)
    void** b_x3_slot = nullptr;
    // optional: low parts of A already computed by the caller, laid out exactly like `a` (same dims / strides) -- the
    // small-channel stem splits its padded NHWC4 copy once instead of the 8x larger overlapping window view
    const void* a_lo_base = nullptr;
    // internal (launch_tf32x3 -> kernel): two-plane A -- `a` is the original tensor (segments 1, 2), `a_lo` its low parts
    int x3_cb = 0;
    OperandDesc a_lo;
    // optional projection source of a 1x1, unpadded conv launch (`proj.C` > 0): a second 1x1, unpadded convolution
    // into the same output pixels, summed in the same accumulator -- D = act(A*B + A_proj*B_proj + bias + epi.bias2).
    // Its K blocks follow the main ones.  Runs only with the plain f32 epilogue (else RTEN_ERR_UNSUPPORTED_VALUE).
    struct Projection {
        int C = 0;       // channels of a (a multiple of 32)
        int stride = 1;  // pixel (ox, oy) reads a at (ox * stride, oy * stride)
        OperandDesc a;   // (c, x, y, b) of the NHWC input
        OperandDesc b;   // (c, o, 1, 1)
        void** b_x3_slot = nullptr;  // as b_x3_slot above
        int x3_cb = 0;               // internal, as x3_cb / a_lo above
        OperandDesc a_lo;
    } proj;
    // optional chained 1x1 convolution of the output (`chain.N2` > 0): z = act(D * W^T + bias) over N2 columns, computed
    // from the output tile while it is staged for its store, so D is not read back.  Runs only for a conv launch in
    // single-pass TF32 with the plain f32 epilogue (no Gelu), N % 32 == 0, N <= 256, N2 in {64, 128}, TMA-addressable
    // w and z (else RTEN_ERR_UNSUPPORTED_VALUE).
    struct Chain {
        int N2 = 0;
        OperandDesc w;  // (c, o, 1, 1): dims {N, N2}, K-major
        const float* bias = nullptr;
        int act = 0;    // 0 none, 1 relu
        OperandDesc z;  // (n, x, y, b) of the NHWC output: dims {N2, OW, OH, B}
    } chain;
};

// Returns RTEN_OK and enqueues the kernel, or RTEN_ERR_UNSUPPORTED_VALUE (without touching ctx->err
// semantics of the caller) when the operands violate a TMA constraint -- the caller then packs
// the operand into an aligned K-major workspace and retries.
rten_status launch_umma_gemm(rten_ctx* ctx, const GemmLaunch& L);

// Tiled, 128B-swizzled rank-4 tensor map over `od` (cuTensorMapEncodeTiled through the runtime's driver entry point).
bool encode_map(rten_ctx* ctx, CUtensorMap* map, const OperandDesc& od, int esize, bool is_f32, const uint32_t box[4],
                const uint32_t estr[4]);

// Stride-1 convolutions with a kh x kw > 1 window on the halo-reuse kernel (umma_halo.cu): one activation patch per
// channel block in shared memory, every filter tap a shifted window of it.  Its unit shapes {bn, T}: bn output channels
// x T tiles of 128 pixel slots (T = 1: one m64 half per consumer warpgroup, bn <= 64; T = 2: two halves).
constexpr int HALO_SHAPES[5][2] = {{32, 1}, {32, 2}, {64, 1}, {64, 2}, {128, 2}};
bool halo_shape_fits(const GemmLaunch& L, int bn, int T);  // the halo kernel can run L with unit shape (bn, T)
// The unit shape the halo kernel's cost model ranks first for L; false if no shape fits.
bool halo_model_shape(rten_ctx* ctx, const GemmLaunch& L, int& bn, int& T);
// RTEN_ERR_UNSUPPORTED_VALUE if the shape does not fit L.
rten_status launch_umma_halo_conv(rten_ctx* ctx, const GemmLaunch& L, int bn, int T, bool verbose);

// The plans file (RTEN_B200_TUNE_FILE, rten_b200_save_plans / rten_b200_load_plans): ctx->tune_cache as text.
void tune_cache_load(rten_ctx* ctx, const char* path);
void tune_cache_save(rten_ctx* ctx, const char* path);

// true if `od` can be fed to TMA directly (16-B aligned base and strides, inner stride 1).
bool tma_compatible(const OperandDesc& od, int esize, int rank);

}  // namespace rtb
