/*
 * rten_b200.h -- C ABI of librten_b200.so: the H100 (sm_90a) operator execution backend for RTen.
 *
 * This is the drop-in boundary for ONE path of robertknight/rten: `Operator::run` /
 * `run_in_place` / `prepack` (src/operator.rs:486-613) of the dense operators of ResNet-50 /
 * BERT-base / GPT-2, replacing rten-gemm's packed GEMM (rten-gemm/src/lib.rs:199-391) and the
 * rten-vecmath row kernels.  A Rust `impl Operator` shim fills `rten_tensor` descriptors from
 * `ValueView`s (src/value.rs:299) and calls one function below per operator (INTEGRATION.md).
 *
 * Conventions
 *  - Every entry point takes a context (one per host thread / stream: rten's ops are `Send + Sync`
 *    and `Model::run` may be re-entered concurrently, src/operator.rs:622).
 *  - `rten_tensor.strides` are ELEMENT strides like rten-tensor layouts; arbitrary (non-negative)
 *    strides are accepted, including the permuted views `TransformInputs` hands to MatMul
 *    (src/ops/transform_inputs.rs:23-34).
 *  - `device >= 0`: `data` is a device pointer on that CUDA ordinal (buffers resident in HBM).
 *    `device == RTEN_DEVICE_HOST`: `data` is host memory; the library stages it through HBM on the
 *    context's stream (host<->device copies are part of the call) -- this is how an unmodified
 *    rten `Vec<T>`-backed tensor crosses the boundary.
 *  - Output tensors: `out->data == NULL` => the library allocates from the context pool (plays
 *    `ctx.pool()`, src/operator.rs:360) on device and fills shape/strides/device; the caller later
 *    returns it with rten_b200_free().  Otherwise `out` must already have the result shape.
 *  - Calls enqueue work on the context stream and return without synchronising unless a host
 *    tensor is involved; asynchronous CUDA errors surface on the next call or rten_b200_sync().
 *  - Errors: status codes mirror `OpError` (src/operator.rs:116-144); rten_b200_last_error()
 *    returns the reference's static message string for that error.  When a call fails, every output it
 *    allocated (`data == NULL` on entry) is freed and its `data` is NULL again: nothing is left to release.
 *  - No CPU fallback exists: without an H100 + driver every op fails with RTEN_ERR_CUDA.
 */
#ifndef RTEN_B200_H
#define RTEN_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define RTEN_MAX_DIMS 8
#define RTEN_DEVICE_HOST (-1)

/* = `DataType` (src/value.rs:20-40) */
typedef enum { RTEN_F32 = 0, RTEN_I32 = 1, RTEN_I8 = 2, RTEN_U8 = 3 } rten_dtype;

typedef struct {
    void* data;
    int32_t dtype; /* rten_dtype */
    int32_t ndim;
    int64_t shape[RTEN_MAX_DIMS];
    int64_t strides[RTEN_MAX_DIMS]; /* elements */
    int32_t device;                 /* RTEN_DEVICE_HOST or CUDA ordinal */
    int32_t _reserved;
} rten_tensor;

/* = `OpError` variants (src/operator.rs:116-144) + device errors */
typedef enum {
    RTEN_OK = 0,
    RTEN_ERR_CAST_FAILED = 1,
    RTEN_ERR_UNSUPPORTED_TYPE = 2,
    RTEN_ERR_INCOMPATIBLE_SHAPES = 3, /* IncompatibleInputShapes(&'static str) */
    RTEN_ERR_MISSING_INPUTS = 4,
    RTEN_ERR_INVALID_VALUE = 5,      /* InvalidValue(&'static str) */
    RTEN_ERR_UNSUPPORTED_VALUE = 6,  /* UnsupportedValue(&'static str) */
    RTEN_ERR_UNSUPPORTED_OUTPUT = 7, /* UnsupportedOutput(&'static str) */
    RTEN_ERR_CUDA = 100,
    RTEN_ERR_NCCL = 101
} rten_status;

typedef struct rten_ctx rten_ctx;
/* = `PrepackedInput` (src/operator.rs:25-31): a weight re-laid out once for the tensor cores. */
typedef struct rten_packed rten_packed;

/* fp32 GEMM/Conv arithmetic mode (SURVEY.md hard part A). */
typedef enum {
    RTEN_F32_TF32 = 0,  /* single wgmma tf32 pass: operands rounded to 10 mantissa bits.  EXPLICIT OPT-IN
                           (rten_b200_set_f32_mode or env RTEN_B200_F32_MODE=tf32); tolerance |d| <= 2^-9 sum_k |a_k b_k| */
    RTEN_F32_TF32X3 = 1 /* DEFAULT: 3-pass error-compensated split (hi*hi + hi*lo + lo*hi, f32 accumulation): meets the
                           reference's own f32 tolerance (rten-tensor/src/test_util.rs:47-92) at 1/3 of the tensor rate */
} rten_f32_mode;

/* Activation fused into an operator's epilogue (the node that follows it in the graph), applied after the bias and the
 * residual add with the standalone operator's exact f32 roundings: the fused result is bit-identical to the operator
 * chain.  Codes 0-3 are the `int activation` of the *_ex functions. */
typedef enum {
    RTEN_ACT_NONE = 0,
    RTEN_ACT_RELU = 1,
    RTEN_ACT_GELU = 2,         /* erf form */
    RTEN_ACT_GELU_TANH = 3,    /* tanh approximation */
    RTEN_ACT_SIGMOID = 4,      /* rten_b200_sigmoid */
    RTEN_ACT_SILU = 5,         /* rten_b200_silu */
    RTEN_ACT_HARD_SIGMOID = 6, /* rten_b200_hard_sigmoid with (alpha, beta) */
    RTEN_ACT_HARD_SWISH = 7    /* rten_b200_hard_swish */
} rten_activation_kind;
typedef struct {
    int32_t kind; /* rten_activation_kind */
    float alpha;  /* RTEN_ACT_HARD_SIGMOID only (ONNX defaults 0.2, 0.5); ignored otherwise */
    float beta;
} rten_activation;

/* ---- context, memory, diagnostics ----------------------------------------------------------- */
rten_status rten_b200_ctx_create(int device, void* cuda_stream_or_null, size_t workspace_bytes, rten_ctx** out);
void rten_b200_ctx_destroy(rten_ctx* ctx);
const char* rten_b200_last_error(rten_ctx* ctx);
rten_status rten_b200_sync(rten_ctx* ctx);
rten_status rten_b200_set_f32_mode(rten_ctx* ctx, int mode /* rten_f32_mode */);
/* Plan autotuning (off by default; env RTEN_B200_AUTOTUNE=1 turns it on at context creation).  When on, the FIRST
 * MatMul / Conv launch of every distinct problem (shape, layout, epilogue) outside graph capture times the cost
 * model's best launch plans on the device and caches the winner in the context -- the role rten-gemm's per-arch
 * kernel selection and blocking heuristics play (rten-gemm/src/lib.rs:199-391), decided by measurement.  Integer
 * results do not depend on the plan; f32 results stay within the TF32 tolerance but may differ in the last bits
 * between plans (split-K changes the summation order).  Measured plans are used for the rest of the context's life
 * even after autotuning is switched off again, and env RTEN_B200_TUNE_FILE=<path> keeps them across processes
 * (read at context creation, rewritten at destruction when new problems were measured). */
rten_status rten_b200_set_autotune(rten_ctx* ctx, int enable);
rten_status rten_b200_save_plans(rten_ctx* ctx, const char* path);
rten_status rten_b200_load_plans(rten_ctx* ctx, const char* path);
/* Caching, stream-ordered device allocator = `BufferPool` (src/buffer_pool.rs:1-140). */
rten_status rten_b200_alloc(rten_ctx* ctx, size_t bytes, void** dev_ptr);
rten_status rten_b200_free(rten_ctx* ctx, void* dev_ptr);
/* Pinned host buffers for callers that want asynchronous staging of host tensors. */
rten_status rten_b200_host_alloc(rten_ctx* ctx, size_t bytes, void** host_ptr);
rten_status rten_b200_host_free(rten_ctx* ctx, void* host_ptr);
/* Copies between host and device tensors of identical shape (strided on both sides). */
rten_status rten_b200_copy(rten_ctx* ctx, const rten_tensor* src, rten_tensor* dst);
/* Number of CUDA kernels this context has launched so far (bench.py `gpu_launches`). */
uint64_t rten_b200_launch_count(rten_ctx* ctx);
const char* rten_b200_version(void);
/* Debug aid for plan sweeps (env RTEN_B200_FORCE_BN / _SPLITK): how many tensor-core launches
 * found a valid plan matching every forced field, and how many fell back to the cost model's choice because none did.
 * With env RTEN_B200_FORCE_STRICT=1 such a launch fails with RTEN_ERR_INVALID_VALUE instead. */
rten_status rten_b200_debug_forced_plans(rten_ctx* ctx, uint64_t* matched, uint64_t* unmatched);
/* Capture everything enqueued between begin/end into a CUDA graph; replay with graph_launch.
 * (launch-bound op lists: the `Graph::run_plan` loop, src/graph.rs:880-1286, as one graph) */
typedef struct rten_graph rten_graph;
rten_status rten_b200_graph_begin(rten_ctx* ctx);
rten_status rten_b200_graph_end(rten_ctx* ctx, rten_graph** out);
rten_status rten_b200_graph_launch(rten_ctx* ctx, rten_graph* g);
void rten_b200_graph_destroy(rten_graph* g);

/* ---- prepack == `Operator::prepack` (src/operator.rs:587-601) ------------------------------- */
/* MatMul/FusedMatMul/MatMulInteger input 1 (src/ops/matmul.rs:410-420,687-697): B [K,N] (f32, i8 or
 * u8) -> K-major [N,K] tensor-core layout (+ per-column sums for the int8 zero-point epilogue). */
rten_status rten_b200_prepack_b(rten_ctx* ctx, const rten_tensor* b, rten_packed** out);
/* Conv/ConvInteger kernel OIHW (the reference prepacks it per call, src/ops/conv.rs:302-315):
 * -> [O, kh, kw, C/g] K-major (+ per-output-channel sums for ConvInteger). */
rten_status rten_b200_prepack_conv_weight(rten_ctx* ctx, const rten_tensor* w, int groups, rten_packed** out);
void rten_b200_packed_free(rten_ctx* ctx, rten_packed* p);

/* ---- operators == `Operator::run` ------------------------------------------------------------ */
/* Gemm (src/ops/matmul.rs:32-167): out = alpha * op(a) @ op(b) + beta * broadcast(c). */
rten_status rten_b200_gemm(rten_ctx* ctx, const rten_tensor* a, const rten_tensor* b, const rten_tensor* c_or_null,
                           float alpha, float beta, int trans_a, int trans_b, rten_tensor* out);

/* MatMul (src/ops/matmul.rs:390-434) / FusedMatMul (:462-507): numpy-matmul broadcasting; optional row
 * bias over N; alpha scales the product before the bias is added.  `packed_b_or_null` = the
 * PrepackedInput for input 1 (then `b` is only consulted for its shape). */
rten_status rten_b200_matmul(rten_ctx* ctx, const rten_tensor* a, const rten_tensor* b,
                             const rten_packed* packed_b_or_null, const rten_tensor* row_bias_or_null, float alpha,
                             rten_tensor* out);
/* Extension used by whole-model runners: fused activation after bias (rten_activation_kind 0 none, 1 relu, 2 gelu(erf),
 * 3 gelu(tanh)) and optional residual add (same shape as out) before the activation. */
rten_status rten_b200_matmul_ex(rten_ctx* ctx, const rten_tensor* a, const rten_tensor* b,
                                const rten_packed* packed_b_or_null, const rten_tensor* row_bias_or_null, float alpha,
                                const rten_tensor* residual_or_null, int activation, rten_tensor* out);

/* MatMulInteger (src/ops/matmul.rs:582-697): a u8|i8, b u8|i8, zero points scalar or vector, out i32
 * exact.  `scale_or_null` != NULL => MatMulIntegerToFloat (:776-811): out f32 = f32(acc) * scale
 * (scalar or per column). */
rten_status rten_b200_matmul_integer(rten_ctx* ctx, const rten_tensor* a, const rten_tensor* b,
                                     const rten_packed* packed_b_or_null, const rten_tensor* a_zero_point_or_null,
                                     const rten_tensor* b_zero_point_or_null, const rten_tensor* scale_or_null,
                                     rten_tensor* out);
/* MatMulIntegerToFloat followed by the graph's Add(bias [N]), Add(residual, same shape as the output) and activation
 * (rten_activation) in the epilogue, as separate exactly rounded f32 operations in that order -- bit-identical to the
 * unfused operators.  Requires `scale`. */
rten_status rten_b200_matmul_integer_ex(rten_ctx* ctx, const rten_tensor* a, const rten_tensor* b, const rten_packed* packed_b,
                                        const rten_tensor* a_zero_point, const rten_tensor* b_zero_point,
                                        const rten_tensor* scale, const rten_tensor* scale_b_or_null /* scalar: effective scale = scale_b * scale */,
                                        const rten_tensor* bias, const rten_tensor* residual, int activation,
                                        rten_tensor* out_range_or_null, rten_tensor* out);

/* MatMulNBits (src/ops/matmul/contrib.rs:21-195, ONNX Runtime's com.microsoft.MatMulNBits): a f32 [..., M, K] (at
 * least 2 dims, the leading dims flatten into rows) times a 4-bit block-quantized B: b u8 [N, k_blocks, blob_bytes] with
 * block = 2 * blob_bytes elements (a power of two >= 16), byte j of a block holding element 2j in its low nibble and
 * 2j + 1 in its high nibble, zero point 8; scales f32 [N, k_blocks], or 1-D [N * k_blocks] with k_blocks =
 * K / block_size.  out f32 [..., M, N] = a . w with w[k, n] = f32(nibble - 8) * scales[n, k / block] (one f32 rounding);
 * K == 0 gives zeros.  Only bits = 4.  Errors as the reference's, plus RTEN_ERR_INCOMPATIBLE_SHAPES for 2-D scales that
 * are not [N, k_blocks].  Rows = prod(leading dims) * M <= 32 (T): a streaming kernel reads every column's nibbles and
 * scales from HBM once and computes in exact f32 FMA arithmetic; more rows: a wgmma kernel dequantizes the nibbles into
 * its shared-memory B tiles and follows the context's f32 mode (3xTF32 default, one TF32 pass opt-in).  B is never
 * expanded to f32 in HBM.  Device-resident a / b / scales with 16-byte aligned rows (K % 32 == 0 for b) take exactly one
 * kernel launch and no host synchronisation (capturable in a CUDA graph); other layouts are first copied. */
rten_status rten_b200_matmul_nbits(rten_ctx* ctx, const rten_tensor* a, const rten_tensor* b, const rten_tensor* scales,
                                   int bits, int block_size, rten_tensor* out);

/* Conv (src/ops/conv.rs:124-419).  x NCHW (or NCW), w OIHW, bias [O].  pads = {top,left,bottom,right};
 * auto_pad_same != 0 => `Padding::Same` (pads ignored).  n_spatial = 1 or 2 gives the expected
 * number of stride/dilation values (error strings as the reference). */
typedef struct {
    int32_t pads[4];
    int32_t auto_pad_same;
    int32_t groups;
    int32_t strides[2];
    int32_t dilations[2];
    int32_t n_strides;   /* number of valid entries in strides (reference validates == spatial dims) */
    int32_t n_dilations; /* idem */
} rten_conv_params;
rten_status rten_b200_conv2d(rten_ctx* ctx, const rten_tensor* x, const rten_tensor* w,
                             const rten_packed* packed_w_or_null, const rten_tensor* bias_or_null,
                             const rten_conv_params* p, rten_tensor* out);
/* Extension: fused residual add (same shape as out) + activation, codes 0-3 of rten_activation_kind (any other code:
 * RTEN_ERR_INVALID_VALUE; conv2d_act takes the others).
 *
 * Depthwise convolutions -- the reference's condition (src/ops/conv.rs:248-284): not the pointwise case (1x1, no
 * padding, strides and dilations 1, groups 1), and in channels == out channels == groups, which includes 1-channel
 * convolutions with groups 1 -- of conv2d, conv2d_ex, conv_integer and conv_integer_ex (and the separate calls of
 * conv2d_projected / conv2d_chained and the stride phases of conv_transpose) run on a direct depthwise kernel in ONE
 * launch over all batches and channels, for x in any strides (NCHW and channels-last without a copy) and w as given or
 * its rten_b200_prepack_conv_weight(groups = C) handle; zero points are read in place on the device, so a
 * device-resident call is exactly one launch and can be captured in a CUDA graph.  Its arithmetic is the reference's
 * depthwise executor's (src/ops/conv/depthwise.rs), per output and in its order:
 *   f32: bias[c] (or +0.0), then for ky, then kx, ascending, out = out + x * w with the product and the sum each rounded
 *        (no fused multiply-add) over the taps inside the image only -- padded taps are skipped, not multiplied by 0 --
 *        then the residual add and activation.  Bit-identical to the reference in both f32 modes (no tensor cores).
 *   ConvInteger: wrapping i32 sums of (x - x_zero_point) * (w - w_zero_point[c]) over the taps inside the image only, so
 *        padding acts as x_zero_point.  The GEMM path of other convolutions pads with the reference's literal 0 in the
 *        shifted-i8 domain (128 for u8 images) instead: a padded depthwise ConvInteger whose x zero point is not 128
 *        (u8) / 0 (i8) gives the reference's depthwise border values, which that path would not.  The f32 output of
 *        conv_integer_ex is formed as its GEMM epilogue forms it. */
rten_status rten_b200_conv2d_ex(rten_ctx* ctx, const rten_tensor* x, const rten_tensor* w,
                                const rten_packed* packed_w_or_null, const rten_tensor* bias_or_null,
                                const rten_conv_params* p, const rten_tensor* residual_or_null, int activation,
                                rten_tensor* out);
/* Extension: conv2d_ex with any rten_activation (NULL: none) -- Conv followed by Relu, Gelu, Sigmoid, Silu (the
 * reference's fusion of Mul(x, Sigmoid(x))), HardSigmoid or HardSwish in the convolution's epilogue, on every path
 * (implicit GEMM, small-channel stem, explicit im2col, NCHW outputs, depthwise), bit-identical to conv2d_ex followed by
 * the standalone operator.  An unknown kind is RTEN_ERR_INVALID_VALUE.  Kinds above Relu after a residual need a
 * pixel-contiguous output (else RTEN_ERR_UNSUPPORTED_VALUE), as Gelu always has. */
rten_status rten_b200_conv2d_act(rten_ctx* ctx, const rten_tensor* x, const rten_tensor* w,
                                 const rten_packed* packed_w_or_null, const rten_tensor* bias_or_null,
                                 const rten_conv_params* p, const rten_tensor* residual_or_null,
                                 const rten_activation* act_or_null, rten_tensor* out);
/* Extension: act(Conv(x, w, bias, p) + Conv(x_proj, w_proj, bias_proj, p_proj)) -- the ONNX pattern Conv, Conv -> Add
   (-> Relu) of a residual block with a projection shortcut.  Both outputs must have the same shape
   (RTEN_ERR_INCOMPATIBLE_SHAPES); all tensors are f32 (RTEN_ERR_UNSUPPORTED_TYPE); otherwise the checks of conv2d_ex.
   Two 1x1 convolutions (groups 1, no padding or dilation) over channels-last, 16-byte addressable inputs whose channel
   counts are multiples of 32 run as one GEMM over both inputs, and the projection is never written; any other pair
   runs as the two calls conv2d_ex(x_proj) and conv2d_ex(x, residual = that result). */
rten_status rten_b200_conv2d_projected(rten_ctx* ctx, const rten_tensor* x, const rten_tensor* w,
                                       const rten_packed* packed_w_or_null, const rten_tensor* bias_or_null,
                                       const rten_conv_params* p, const rten_tensor* x_proj, const rten_tensor* w_proj,
                                       const rten_packed* packed_w_proj_or_null, const rten_tensor* bias_proj_or_null,
                                       const rten_conv_params* p_proj, int activation, rten_tensor* out);
/* Extension: out = act(Conv(x, w, bias, p) [+ residual | + Conv(x_proj, w_proj, bias_proj, p_proj)]) and
   out_next = activation_next(Conv(out, w_next, bias_next, p_next)) -- a residual block's last convolution and the next
   block's first.  residual and x_proj are exclusive (RTEN_ERR_INVALID_VALUE); mismatched projection or residual shapes
   return RTEN_ERR_INCOMPATIBLE_SHAPES; all tensors are f32 (RTEN_ERR_UNSUPPORTED_TYPE); otherwise the checks of
   conv2d_ex / conv2d_projected.  In single-pass TF32, a 1x1 convolution (groups 1, no padding or dilation; a projection
   as conv2d_projected folds it) over channels-last, 16-byte addressable inputs with up to 256 output channels, a
   multiple of 32, followed by a 1x1, stride-1, unpadded convolution to 64 or 128 channels, runs as one launch that
   computes out_next from out's tiles while they are stored, so out is not read back.  Any other pair runs as the calls
   conv2d_ex (or conv2d_projected) then conv2d_ex(out, w_next), with the same results. */
rten_status rten_b200_conv2d_chained(rten_ctx* ctx, const rten_tensor* x, const rten_tensor* w,
                                     const rten_packed* packed_w_or_null, const rten_tensor* bias_or_null,
                                     const rten_conv_params* p, const rten_tensor* residual_or_null,
                                     const rten_tensor* x_proj_or_null, const rten_tensor* w_proj_or_null,
                                     const rten_packed* packed_w_proj_or_null, const rten_tensor* bias_proj_or_null,
                                     const rten_conv_params* p_proj_or_null, int activation, const rten_tensor* w_next,
                                     const rten_packed* packed_w_next_or_null, const rten_tensor* bias_next_or_null,
                                     const rten_conv_params* p_next, int activation_next, rten_tensor* out,
                                     rten_tensor* out_next);
/* ConvTranspose (src/ops/conv_transpose.rs:226-410), f32.  x NCHW (or NCW), w [C_in, C_out/groups, kh, kw] (or
 * [C_in, C_out/groups, kw]), bias [C_out]; the output layout follows the input (channels-last in, channels-last out).
 * pads = {top, left, bottom, right} (1-D: {start, end}); auto_pad_same != 0 => `Padding::Same` (output = input * stride,
 * pads ignored).  The n_* counts give how many entries of each array are set: the reference checks them against the
 * spatial rank (n_output_padding = 0: the attribute is absent, zeros).  Errors and messages as the reference
 * (conv_transpose.rs:144-345); batch 0 gives an empty output.  Strides above 256 return RTEN_ERR_UNSUPPORTED_VALUE.
 *
 * Computed as stride-phase convolutions: output rows o = q + s*j of phase q = o mod s (per axis) receive the taps k
 * with k*d = q + pad (mod s), so each phase with taps is an ordinary stride-1 convolution with a reversed sub-kernel,
 * run on the implicit-GEMM conv kernel and stored through a strided view of the output; every phase without taps gets
 * the bias (or 0) from one fill launch.  prepack builds the sub-kernels of every residue phase once (they depend only
 * on the weight, groups, strides and dilations); a channels-last, single-pass TF32 call with prepacked weights and
 * groups 1 is (phases with taps) + (1 if a phase has none) launches. */
typedef struct {
    int32_t pads[4];
    int32_t auto_pad_same;
    int32_t groups;
    int32_t strides[2];
    int32_t dilations[2];
    int32_t output_padding[2];
    int32_t n_pads;
    int32_t n_strides;
    int32_t n_dilations;
    int32_t n_output_padding;
} rten_conv_transpose_params;
rten_status rten_b200_conv_transpose(rten_ctx* ctx, const rten_tensor* x, const rten_tensor* w,
                                     const rten_packed* packed_w_or_null, const rten_tensor* bias_or_null,
                                     const rten_conv_transpose_params* p, rten_tensor* out);
rten_status rten_b200_prepack_conv_transpose_weight(rten_ctx* ctx, const rten_tensor* w, const rten_conv_transpose_params* p,
                                                    rten_packed** out);
/* ConvInteger (src/ops/conv.rs:421-533); scale_or_null != NULL => ConvIntegerToFloat (:535-587). */
rten_status rten_b200_conv_integer(rten_ctx* ctx, const rten_tensor* x, const rten_tensor* w,
                                   const rten_packed* packed_w_or_null, const rten_tensor* x_zero_point_or_null,
                                   const rten_tensor* w_zero_point_or_null, const rten_tensor* scale_or_null,
                                   const rten_conv_params* p, rten_tensor* out);
/* ConvIntegerToFloat with the graph nodes around it folded into the kernel epilogue, each as the same exactly rounded
 * f32 operation the separate operator would perform (bit-identical results): the Mul that forms the scale
 * (`scale_b_or_null`: scalar, effective scale = scale_b * scale), then Add(bias [O]), Add(residual, same shape as the
 * output) and Relu (activation 0 / 1).  Requires `scale`. */
rten_status rten_b200_conv_integer_ex(rten_ctx* ctx, const rten_tensor* x, const rten_tensor* w, const rten_packed* packed_w,
                                      const rten_tensor* x_zero_point, const rten_tensor* w_zero_point,
                                      const rten_tensor* scale, const rten_tensor* scale_b_or_null,
                                      const rten_conv_params* params, const rten_tensor* bias, const rten_tensor* residual,
                                      int activation, rten_tensor* out_range_or_null, rten_tensor* out);

/* ---- autoregressive decode path (rten-generate's loop: one token per sequence and step) -------------------------- */
/* The per-token linear layer of a dynamically quantised transformer as ONE call:
 *   [LayerNormalization(x, ln_scale, ln_bias, axis -1)] -> DynamicQuantizeLinear -> Mul(x_scale, w_scale) ->
 *   MatMulIntegerToFloat(x_q, w, x_zp, w_zero_point, scale) -> Add(bias) -> Add(residual) -> activation
 * -- the node chain `tools/ort-quantize.py` + RTen's fusions (src/optimize/fusions.rs:966-1058) leave around every
 * MatMul of GPT-2.  x [.., K] f32, w [K, N] i8 | u8 (packed_w = its rten_b200_prepack_b handle), w_scale scalar or [N].
 * For M = prod(leading dims) <= 16 this is the skinny-M kernel that plays rten-gemm's gemv path
 * (rten-gemm/src/lib.rs:668-747, kernels simd_generic.rs:795-1129): the weights stream from HBM exactly once, the
 * quantised activations live in shared memory, nothing else is launched.  Larger M runs the separate operators.  Either
 * way every stage performs the operators' exactly rounded arithmetic: results are bit-identical to the unfused graph. */
rten_status rten_b200_quantized_linear(rten_ctx* ctx, const rten_tensor* x, const rten_tensor* ln_scale_or_null,
                                       const rten_tensor* ln_bias_or_null, float ln_epsilon, const rten_tensor* w,
                                       const rten_packed* packed_w_or_null, const rten_tensor* w_zero_point_or_null,
                                       const rten_tensor* w_scale, const rten_tensor* bias_or_null,
                                       const rten_tensor* residual_or_null, int activation, rten_tensor* out);
/* Attention (src/ops/attention.rs:645-905, the ONNX `Attention` operator) on 4-D inputs: query [batch, q_heads, q_seq,
 * head], key / value [batch, kv_heads, total_seq, head] with any strides (a transposed value cache is just a view),
 * attn_mask float broadcastable to [batch, q_heads, q_seq, total_seq], nonpad_kv_seqlen i32 [batch] = number of valid
 * key / value positions when the caller manages a right-padded KV cache (`:817-832`; read on the device, so a decode
 * step stays a fixed launch list).  out [batch, q_heads, q_seq, head]; fully masked rows give zeros (sdpa_head :548-552).
 * q_seq = 1 (decode) with head size 64 / 128 is ONE kernel: scores, softmax and the value product stream the cache once,
 * split over the sequence to fill the SMs.  `new_key` / `new_value` [batch, kv_heads, 1, head] (optional) are written
 * into the caches at position nonpad_kv_seqlen[b] - 1 by the same kernel first (the cache append of rten-generate,
 * rten-generate/src/generator.rs:858-886, without a separate launch).
 * q_seq > 1 with is_causal, nonpad_kv_seqlen or q_heads != kv_heads (prompt / chunked prefill): ONE streaming kernel
 * with the scores kept on chip, for device-resident f32 tensors of head size 64 / 128 (value head size equal), the
 * head dimension contiguous in query, key and out, value with either of its last two dimensions contiguous, and any
 * attn_mask with a contiguous key dimension.  Query row s attends to keys 0 ..= s + offset when causal (offset =
 * valid_b - q_seq with nonpad_kv_seqlen, 0 without) and to keys below valid_b otherwise, where valid_b =
 * clamp(nonpad_kv_seqlen[b], 0, total_seq): read on the device, an out-of-range entry is clamped, not reported.  Both
 * products follow the context's f32 mode: 3xTF32 (default) or one TF32 pass.  Query head h reads kv head
 * h / (q_heads / kv_heads).  Other shapes compose MatMul / Softmax / MatMul; causal, padded or grouped-query calls with
 * q_seq > 1 that the kernel cannot take fail with RTEN_ERR_UNSUPPORTED_VALUE. */
typedef struct {
    int32_t is_causal;
    int32_t q_num_heads;  /* informative for 4-D inputs */
    int32_t kv_num_heads;
    float scale;          /* <= 0: 1 / sqrt(head size) */
    float softcap;        /* > 0 unsupported */
} rten_attention_params;
rten_status rten_b200_attention(rten_ctx* ctx, const rten_tensor* query, const rten_tensor* key, const rten_tensor* value,
                                const rten_tensor* attn_mask_or_null, const rten_tensor* nonpad_kv_seqlen_or_null,
                                const rten_attention_params* params, const rten_tensor* new_key_or_null,
                                const rten_tensor* new_value_or_null, rten_tensor* out);

/* RotaryEmbedding (src/ops/embedding.rs:46-252, the ai.onnx operator): input f32 [batch, seq, hidden] (num_heads heads of
 * hidden / num_heads) or [batch, heads, seq, head] with any strides; the first rotary_embedding_dim elements of every head
 * (0: the whole head) are rotated, the rest copied.  cos / sin [batch|1, seq|1, dim / 2], or with position_ids i32
 * [batch|1, seq|1] tables [max_pos, dim / 2] gathered by position.  Pairs (2i, 2i + 1) when interleaved, else
 * (i, i + dim / 2); y1 = x1 cos - x2 sin, y2 = x1 sin + x2 cos with each product and sum rounded to f32 on its own (no
 * fused multiply-add: bit-identical to a float32 restatement).  out has the input's shape and must not overlap it.
 * Host-resident position_ids are checked (the reference's Gather error); device-resident ones are clamped to
 * [0, max_pos - 1] on the device, nothing is reported.  One kernel launch. */
rten_status rten_b200_rotary_embedding(rten_ctx* ctx, const rten_tensor* input, const rten_tensor* cos, const rten_tensor* sin,
                                       const rten_tensor* position_ids_or_null, int interleaved, int num_heads,
                                       int rotary_embedding_dim, rten_tensor* out);

/* GroupQueryAttention (com.microsoft; src/ops/attention/contrib.rs:369-417, :438-810): the attention operator of ONNX
 * Runtime's int4 LLM exports.  query [B, S, H * D], key / value [B, S, Hkv * D] (both NULL: query is packed QKV
 * [B, S, (H + 2 Hkv) * D]); past_key / past_value [B, Hkv, P, D] (optional); seqlens_k i32 [B] or [B, 1] = total length
 * - 1; total_sequence_length i32 scalar; cos / sin [max_pos, rotary_dim / 2] and position_ids i32 [B, S] for do_rotary;
 * attention_bias [B|1, H|1, >= S, >= P + S] added to the scores.  Outputs: out [B, S, H * D] and the present caches
 * present_key / present_value [B, Hkv, P + S, D].
 * S == total_sequence_length is a first prompt (past_len(b) = 0); otherwise past_len(b) = seqlens_k[b] + 1 - S, and S > 1
 * needs B == 1.  Q and the new K are rotated (rotary_dim = 2 cos.shape[1] <= D, interleaved pairs or halves, the
 * RotaryEmbedding arithmetic above) at position position_ids[b, s], else past_len(b) + s.  The present cache holds
 * past[b, :, :past_len(b)], then the S new tokens, then zeros.  Query row s attends to keys [start, past_len(b) + s + 1)
 * with start = past_len(b) + s + 1 - local_window_size when local_window_size > 0 and that is positive, else 0; query
 * head h reads kv head h / (H / Hkv); scale <= 0 means 1 / sqrt(D).
 * In-place present cache (the reference's run_in_place): present_key / present_value whose data pointer and strides
 * equal past_key's / past_value's (the past buffer, with room for S more positions) receive only the new tokens; the
 * prefix is already there and positions past past_len(b) + S are left untouched.  Otherwise (data == NULL or another
 * buffer) the present cache is built whole, zeros included.  A present cache that overlaps a past cache's memory without
 * being that buffer (same data pointer and strides) fails with RTEN_ERR_UNSUPPORTED_OUTPUT.
 * Host-resident seqlens_k / position_ids are checked with the reference's errors; device-resident ones are read only on
 * the device (seqlens_k clamped to [S - 1, P + S - 1], positions to [0, max_pos - 1], nothing reported), so a step is a
 * fixed launch list.  total_sequence_length decides the prompt kind and is read on the host: if it is device-resident
 * that is one synchronous 4-byte copy, and such a call cannot be captured in a CUDA graph.
 * Paths (head size 64 or 128, device-resident tensors with 16-byte aligned rows and contiguous heads):
 *  - decode step (S == 1, not a first prompt), P + 1 <= 8192: ONE single-query kernel launch rotates q and the new key
 *    itself, appends the new key / value to the present caches and streams them once -- plus one launch that copies the
 *    past prefix when the present caches are not the past buffers and P > 0.
 *  - prompts: the rotary / append kernel (rotated Q to a scratch, new K / V into the present caches) and the streaming
 *    prefill attention kernel (causal, key tiles below every row's window skipped), products in the context's f32 mode
 *    -- plus the past-prefix launch as above.
 * Other head sizes, longer decode caches and softcap > 0 fail with RTEN_ERR_UNSUPPORTED_VALUE; there is no composed
 * fallback.  (smooth_softmax and head_sink are not parameters: the reference rejects them.) */
typedef struct {
    int32_t num_heads;
    int32_t kv_num_heads;
    float scale;               /* <= 0: 1 / sqrt(head size) */
    int32_t do_rotary;
    int32_t rotary_interleaved;
    int32_t local_window_size; /* <= 0: no sliding window */
    float softcap;             /* > 0 unsupported */
} rten_gqa_params;
rten_status rten_b200_group_query_attention(rten_ctx* ctx, const rten_tensor* query, const rten_tensor* key_or_null,
                                            const rten_tensor* value_or_null, const rten_tensor* past_key_or_null,
                                            const rten_tensor* past_value_or_null, const rten_tensor* seqlens_k,
                                            const rten_tensor* total_sequence_length, const rten_tensor* cos_or_null,
                                            const rten_tensor* sin_or_null, const rten_tensor* position_ids_or_null,
                                            const rten_tensor* attention_bias_or_null, const rten_gqa_params* params,
                                            rten_tensor* out, rten_tensor* present_key, rten_tensor* present_value);

/* MultiHeadAttention (com.microsoft; src/ops/attention/contrib.rs:56-300): the attention of ONNX Runtime's optimized
 * encoder and encoder-decoder exports.  query [B, S, H * D], or packed QKV [B, S, H, 3, D] (key, value and bias NULL);
 * key [B, L, H * D] and value [B, L, H * Dv] (key NULL: key = value = query, a given value is ignored); bias
 * [2 H D + H Dv], its three slices added to q, k and v (one rounded f32 add each) before the heads are split;
 * key_padding_mask i32 [B, P + L]; attention_bias f32 broadcastable to [B, H, S, P + L] (any dimension may be 1,
 * the key dimension included); past_key / past_value [B, H, P, D].  Outputs: out [B, S, H * Dv] and, when not NULL,
 * present_key / present_value [B, H, P + L, D] = concat(past, new k / v).
 * scores = scale q k^T (scale <= 0: 1 / sqrt(D)), then in this order: + attention_bias; with unidirectional, keys
 * t > P + s REPLACED by mask_filter_value; keys with key_padding_mask[b, t] == 0 REPLACED by mask_filter_value;
 * softmax with NaN flushed to 0; times v.  A finite mask_filter_value keeps masked keys in the softmax: a row whose
 * keys are all masked is the mean of v over all keys.
 * past_sequence_length and cache_indirection (inputs 8 and 9) fail with the reference's errors, as does every shape
 * error it raises, with its messages.
 * In-place present caches as for GroupQueryAttention: present_key / present_value whose data pointer and strides equal
 * past_key's / past_value's (the past buffer with room for L more positions) receive only the new positions; positions
 * beyond P + L stay untouched.  A present cache overlapping a past cache without being that buffer fails with
 * RTEN_ERR_UNSUPPORTED_OUTPUT.  Host-resident tensors are staged; nothing is read back to the host, so a
 * device-resident call can be captured in a CUDA graph.
 * Paths (head size 64 or 128 with Dv == D; device-resident tensors with 16-byte aligned rows):
 *  - prep, when there is a bias, a past cache or a present output: ONE launch of the rotary / append kernel adds the
 *    bias to q (into a scratch buffer), writes k' and v' into the present caches (or scratch caches when a present
 *    output is not requested) and copies the past prefix unless the caches are in place.
 *  - S == 1: the single-query attention kernel (caches up to 8192 positions; longer ones take the prefill kernel).
 *  - S >= 2: the streaming prefill attention kernel, products in the context's f32 mode.  q / k / v are read in place
 *    through strided views when there is no prep, and out is written in place.  Key tiles above every row's causal
 *    diagonal are skipped and added back as masked keys; their values are read only when their weight is not 0.
 *  Launches: one without prep, two with it.
 * Other head sizes and Dv != D fail with RTEN_ERR_UNSUPPORTED_VALUE; there is no composed fallback. */
typedef struct {
    int32_t num_heads;
    float scale;             /* <= 0: 1 / sqrt(head size) */
    float mask_filter_value; /* the score of a masked key (the reference's default: -10000) */
    int32_t unidirectional;
} rten_mha_params;
rten_status rten_b200_multi_head_attention(rten_ctx* ctx, const rten_tensor* query, const rten_tensor* key_or_null,
                                           const rten_tensor* value_or_null, const rten_tensor* bias_or_null,
                                           const rten_tensor* key_padding_mask_or_null, const rten_tensor* attention_bias_or_null,
                                           const rten_tensor* past_key_or_null, const rten_tensor* past_value_or_null,
                                           const rten_tensor* past_sequence_length_or_null, const rten_tensor* cache_indirection_or_null,
                                           const rten_mha_params* params, rten_tensor* out, rten_tensor* present_key_or_null,
                                           rten_tensor* present_value_or_null);

/* GRU and LSTM (src/ops/rnn.rs gru / lstm), f32.  x [T, B, I]; w [dirs, G * H, I] and r [dirs, G * H, H] with G = 3
 * (GRU gates z, r, h) or 4 (LSTM gates i, o, f, c), in that ONNX order; bias [dirs, 2 * G * H] (input biases, then
 * recurrent biases); initial_h (and initial_c) [dirs, B, H].  Outputs y [T, dirs, B, H], y_h [dirs, B, H] and y_c
 * [dirs, B, H]; every optional input and output may be NULL.  dirs = 2 for bidirectional; direction 1 of a
 * bidirectional layer and a reverse layer run t = T - 1 .. 0, and y stays indexed by t.  H is read from w, as the
 * reference does (params->hidden_size is informative).  sequence_lens (i32) is accepted and ignored, as the reference
 * ignores it: every sequence runs all T steps.
 * Arithmetic, in the reference's order with every operation rounded on its own:
 *   GRU : gx = x W^T (+ Wb); s = h R^T (+ Rb); z, r = sigmoid(gx + s); h~ = tanh(gx_h + r s_h); h = (1 - z) h~ + z h
 *   LSTM: g = ((x W^T (+ Wb)) + h R^T) (+ Rb); i, o, f = sigmoid(g); c~ = tanh(g_c); c = f c + i c~; h = o tanhf(c)
 * sigmoid = 1 / (1 + exp(-x)) and tanh are rten-vecmath's recipes; the LSTM's last tanh is a correctly rounded tanhf
 * (the reference's f32::tanh).  GRU requires linear_before_reset = 1 (0 fails with RTEN_ERR_UNSUPPORTED_VALUE, as in the
 * reference); a non-NULL LSTM peephole input fails with RTEN_ERR_UNSUPPORTED_VALUE.  Every shape error the reference
 * raises comes back with its message; mismatched dimensions it does not check fail with RTEN_ERR_INVALID_VALUE.
 * Paths:
 *  - input projection: ONE wgmma GEMM [T * B, I] x [dirs * G * H, I]^T for every step and direction, in the context's
 *    f32 mode.  packed_w_or_null = rten_b200_prepack_b of w viewed as [I, dirs * G * H] (the transpose of w reshaped to
 *    [dirs * G * H, I]); in 3xTF32 mode its split copy is cached with the handle.
 *  - recurrence, cluster path: ONE launch of rnn_cluster_kernel.  A thread-block cluster per (direction, batch slice)
 *    keeps its direction's R in shared memory for all T steps, split over its CTAs by hidden unit; each step every CTA
 *    computes its gates' h R^T as exact f32 FMA chains (in both f32 modes), applies the gate arithmetic and pushes its
 *    slice of h to every CTA of the cluster through distributed shared memory, then crosses one cluster barrier.  The
 *    cluster size is the smallest of 1, 2, 4, 8, 16 CTAs whose shared memory holds R (16 needs the non-portable size
 *    and is checked with cudaOccupancyMaxActiveClusters).  This covers H <= 256 for GRU and LSTM at any B and I: up to
 *    H = 336 (LSTM) / 388 (GRU) with 8-CTA clusters, and H = 468 / 544 where 16-CTA clusters schedule; H need not be a
 *    multiple of 4.
 *  - recurrence, per-step path (larger H, or env RTEN_B200_NO_RNN_CLUSTER=1 for comparison): per step and direction
 *    the recurrent product on the skinny f32 kernel (B <= 32: exact f32; R is copied once into zero-padded 16-byte
 *    rows when its rows are not) or else on the wgmma GEMM in 3xTF32 in both f32 modes (R split once per call), then
 *    one gate kernel for all directions.
 * Launches of a device-resident call with contiguous x and packed w: cluster path 2 (plus the TF32 low-part split of
 * x in 3xTF32 mode); per-step path 2 + T * (dirs + 1) with R in 16-byte rows and B <= 32 (plus one launch per step and
 * direction for the 3xTF32 split of h on the wgmma GEMM).
 * Nothing is read back to the host, so such a call can be captured in a CUDA graph. */
typedef struct {
    int32_t direction;           /* 0 forward, 1 reverse, 2 bidirectional */
    int32_t hidden_size;         /* informative */
    int32_t linear_before_reset; /* GRU: must be 1 */
} rten_rnn_params;
rten_status rten_b200_gru(rten_ctx* ctx, const rten_tensor* x, const rten_tensor* w, const rten_packed* packed_w_or_null,
                          const rten_tensor* r, const rten_tensor* bias_or_null, const rten_tensor* sequence_lens_or_null,
                          const rten_tensor* initial_h_or_null, const rten_rnn_params* params, rten_tensor* y_or_null,
                          rten_tensor* y_h_or_null);
rten_status rten_b200_lstm(rten_ctx* ctx, const rten_tensor* x, const rten_tensor* w, const rten_packed* packed_w_or_null,
                           const rten_tensor* r, const rten_tensor* bias_or_null, const rten_tensor* sequence_lens_or_null,
                           const rten_tensor* initial_h_or_null, const rten_tensor* initial_c_or_null,
                           const rten_tensor* peephole_or_null, const rten_rnn_params* params, rten_tensor* y_or_null,
                           rten_tensor* y_h_or_null, rten_tensor* y_c_or_null);

/* Softmax (src/ops/norm.rs:825-899) and AddSoftmax (src/ops/attention.rs:30-165) when mask != NULL
 * (mask broadcast to x, added lane-wise before the softmax over `axis`; AddSoftmax uses axis -1).
 * `out` may alias `x` (= run_in_place). */
rten_status rten_b200_softmax(rten_ctx* ctx, const rten_tensor* x, const rten_tensor* mask_or_null, int axis,
                              int flush_nans_to_zero, rten_tensor* out);
/* LayerNormalization (src/ops/norm.rs:437-569); epsilon < 0 => default 1e-5. */
rten_status rten_b200_layer_norm(rten_ctx* ctx, const rten_tensor* x, const rten_tensor* scale,
                                 const rten_tensor* bias_or_null, int axis, float epsilon, rten_tensor* out);
/* RMSNormalization / SimplifiedLayerNormalization (src/ops/norm.rs rms_normalization): layer_normalization_impl with
 * DynamicRootMeanSquare -- mean 0, rstd = scale / sqrt(SumSquare / n + epsilon), no bias.  `scale` broadcasts to the
 * normalized axes [axis, ndim), or is a scalar when it has one element; epsilon < 0 => default 1e-5.  `out` must be
 * contiguous (allocated when out->data == NULL).  Bit-identical to the reference. */
rten_status rten_b200_rms_norm(rten_ctx* ctx, const rten_tensor* x, const rten_tensor* scale, int axis, float epsilon,
                               rten_tensor* out);
/* com.microsoft SkipLayerNormalization (rms == 0) and SkipSimplifiedLayerNormalization (rms != 0), src/ops/norm/contrib.rs:
 * s = (x + skip) + bias, two rounded adds; out = LayerNormalization (or RMSNormalization) of s over the last axis with
 * gamma and, for SkipLayerNormalization only, beta (beta_or_null must be NULL when rms != 0).  x is [B, S, H] or [S, H];
 * skip has the same trailing two dims and broadcasts over the batch ([B, S, H], [1, S, H] or [S, H]); gamma, beta and
 * bias are 1-D.  sum_out_or_null receives s (the operator's output 3, input_skip_bias_sum).  The reference's error
 * statuses and messages, with one deviation: a bias whose length is neither H nor 1 returns RTEN_ERR_INVALID_VALUE
 * (the reference panics).  Outputs must be contiguous.  Bit-identical to the reference, one kernel launch for dense
 * device-resident operands (capturable in a CUDA graph), no temporary beyond the outputs. */
rten_status rten_b200_skip_layer_norm(rten_ctx* ctx, const rten_tensor* x, const rten_tensor* skip, const rten_tensor* gamma,
                                      const rten_tensor* beta_or_null, const rten_tensor* bias_or_null, float epsilon, int rms,
                                      rten_tensor* out, rten_tensor* sum_out_or_null);
/* InstanceNormalization (src/ops/norm.rs instance_normalization): each (n, c) lane of x [N, C, ...] normalised over its
 * L elements, mean = Sum / L and var = SumSquareSub(mean) / L in the reference's fold order, then
 * y = fma(x - mean, scale[c] / sqrt(var + epsilon), bias[c]).  scale and bias are 1-D [C]; epsilon < 0 => default 1e-5.
 * The reference's statuses and messages: "expected input with >= 2 dims", "scale length should match channel count",
 * "bias length should match channel count".  NCHW-contiguous and dense channels-last 4-D x are read as they are and the
 * output keeps x's layout; x in any other strides is copied to contiguous first.  `out` may alias `x` (run_in_place).
 * Bit-identical to the reference.  One kernel launch for rows up to 51200 elements, else two (three for channels-last). */
rten_status rten_b200_instance_norm(rten_ctx* ctx, const rten_tensor* x, const rten_tensor* scale, const rten_tensor* bias,
                                    float epsilon, rten_tensor* out);
/* GroupNorm as torch exports it, in one normalization pass: exactly the result of
 *   Reshape(x, [N, groups, -1]) -> InstanceNormalization(inst_scale, inst_bias, epsilon) -> Reshape to x's shape
 *   -> Mul(gamma [C, 1, ..]) -> Add(beta [C, 1, ..]) -> activation
 * each step rounded on its own: the InstanceNormalization value of row (n, g) -- the channels g C/groups ..
 * (g + 1) C/groups - 1 of image n in (c, spatial) order -- then y * gamma[c] (when gamma), + beta[c] (when beta), then
 * the activation (NULL or RTEN_ACT_NONE: none), computed as the standalone operator computes it.  inst_scale and
 * inst_bias are 1-D [groups]; gamma and beta have C elements, one per channel.  C % groups != 0 returns
 * RTEN_ERR_INVALID_VALUE "Input length must be a multiple of specified dimensions", as the Reshape does; gamma or beta
 * with another length returns RTEN_ERR_INCOMPATIBLE_SHAPES "Cannot broadcast inputs"; otherwise the errors of
 * rten_b200_instance_norm against [N, groups, L].  Layouts, aliasing and launches as rten_b200_instance_norm. */
rten_status rten_b200_group_norm(rten_ctx* ctx, const rten_tensor* x, int groups, const rten_tensor* inst_scale,
                                 const rten_tensor* inst_bias, const rten_tensor* gamma_or_null, const rten_tensor* beta_or_null,
                                 float epsilon, const rten_activation* act_or_null, rten_tensor* out);
/* BatchNormalization in inference mode (src/ops/norm.rs batch_norm_in_place): per channel c,
 *   s = scale[c] / sqrt(var[c] + epsilon)        (a rounded add, a correctly rounded sqrt and division)
 *   y = fma(x - mean[c], s, bias[c])             (the subtraction rounded, then one fused multiply-add)
 * then the activation (NULL or RTEN_ACT_NONE: none), computed as the standalone operator computes it.  The channel is
 * axis 1 of x when x has rank >= 2; a rank-1 x is one channel.  scale, bias, mean and var are 1-D [C]; epsilon < 0 =>
 * default 1e-5.  The reference's statuses and messages: rank 0 returns RTEN_ERR_INVALID_VALUE "Input must have at least
 * 1 dim"; a parameter of another length returns RTEN_ERR_INCOMPATIBLE_SHAPES "scale.size(0) != channels" (bias, mean,
 * var alike).  NCHW-contiguous x (any rank) and dense channels-last 4-D x are read as they are and the output keeps x's
 * layout; x in any other strides is copied to contiguous first.  `out` may alias `x` (run_in_place).  Bit-identical to
 * the reference; one kernel launch for dense device-resident operands, capturable in a CUDA graph. */
rten_status rten_b200_batch_norm(rten_ctx* ctx, const rten_tensor* x, const rten_tensor* scale, const rten_tensor* bias,
                                 const rten_tensor* mean, const rten_tensor* var, float epsilon,
                                 const rten_activation* act_or_null, rten_tensor* out);
/* Clip (src/ops/unary_elementwise.rs:249-333), f32 or i32: x.max(min).min(max) with `a > b ? a : b` comparisons, so
 * NaN becomes min and -0.0 clipped at min = 0 becomes +0.0.  min / max are scalar tensors of x's type (NULL: the type's
 * finite minimum / maximum), read on the device: no host synchronisation, capturable in a CUDA graph.  `out` may alias
 * `x`.  One kernel launch for dense device-resident x. */
rten_status rten_b200_clip(rten_ctx* ctx, const rten_tensor* x, const rten_tensor* min_or_null, const rten_tensor* max_or_null,
                           rten_tensor* out);
/* Erf / Gelu (src/ops/unary_elementwise.rs:384-435); approximate != 0 => tanh form. */
rten_status rten_b200_erf(rten_ctx* ctx, const rten_tensor* x, rten_tensor* out);
rten_status rten_b200_gelu(rten_ctx* ctx, const rten_tensor* x, int approximate, rten_tensor* out);
/* Sigmoid, Silu, HardSigmoid and HardSwish, f32, bit-identical to the reference, every operation a separate exactly
 * rounded one (no fused multiply-add):
 *   Sigmoid     1 / (1 + exp(0 - x))                   rten-vecmath/src/exp.rs:201-212
 *   Silu        x / (1 + exp(0 - x)): ONE division, not x * Sigmoid(x) (exp.rs:217-228; the reference's optimizer
 *               rewrites Mul(x, Sigmoid(x)) into it)
 *   HardSigmoid clamp(alpha * x + beta, 0, 1)          src/ops/unary_elementwise.rs:437-449 (ONNX defaults 0.2, 0.5)
 *   HardSwish   x * clamp(x / 6 + 0.5, 0, 1)           :457-469, with 1/6 rounded to f32 and multiplied
 * exp is rten-vecmath's Exp (inf from 104 on), so Silu(x <= -104) = -0.0 and Silu(-inf) = NaN.  clamp is f32::clamp
 * (comparisons): NaN passes through and -0.0 stays -0.0, so HardSwish(-4) = -0.0.  x in any strides; `out` may alias
 * `x` (run_in_place).  One kernel launch for dense device-resident x, capturable in a CUDA graph. */
rten_status rten_b200_sigmoid(rten_ctx* ctx, const rten_tensor* x, rten_tensor* out);
rten_status rten_b200_silu(rten_ctx* ctx, const rten_tensor* x, rten_tensor* out);
rten_status rten_b200_hard_sigmoid(rten_ctx* ctx, const rten_tensor* x, float alpha, float beta, rten_tensor* out);
rten_status rten_b200_hard_swish(rten_ctx* ctx, const rten_tensor* x, rten_tensor* out);
/* Sqrt, Reciprocal, Exp, Tanh, Neg and Abs, f32 only, bit-identical to the reference including +-0, +-inf and NaN:
 *   Sqrt        IEEE square root (x.sqrt())             src/ops/unary_elementwise.rs:743-745
 *   Reciprocal  1 / x, IEEE division                    :607-609 (1 / +-0 = +-inf)
 *   Exp         rten-vecmath's Exp (inf from 104 on, 0 from -104 down)   :391, rten-vecmath/src/exp.rs
 *   Tanh        rten-vecmath's Tanh                      :758, rten-vecmath/src/tanh.rs
 *   Neg         -x, the sign bit flipped (-(+0) = -0)    :550-555
 *   Abs         the sign bit cleared                      :195-220
 * x in any strides; `out` may alias `x` (run_in_place).  One kernel launch for dense device-resident x, capturable in a
 * CUDA graph.  None of them is a convolution-epilogue activation. */
rten_status rten_b200_sqrt(rten_ctx* ctx, const rten_tensor* x, rten_tensor* out);
rten_status rten_b200_reciprocal(rten_ctx* ctx, const rten_tensor* x, rten_tensor* out);
rten_status rten_b200_exp(rten_ctx* ctx, const rten_tensor* x, rten_tensor* out);
rten_status rten_b200_tanh(rten_ctx* ctx, const rten_tensor* x, rten_tensor* out);
rten_status rten_b200_neg(rten_ctx* ctx, const rten_tensor* x, rten_tensor* out);
rten_status rten_b200_abs(rten_ctx* ctx, const rten_tensor* x, rten_tensor* out);
/* Communicator of a batch-sharded run (one process per GPU).  The reference has no counterpart (single process, rayon
 * threads); it exists so that DynamicQuantizeLinear can use the range of the WHOLE tensor when the batch is split over
 * ranks.  NCCL (libnccl.so.2) is resolved with dlopen at the first call; rank 0 creates the 128-byte id, the host
 * distributes it (any side channel), every rank calls comm_create with the same id. */
typedef struct rten_comm rten_comm;
rten_status rten_b200_comm_unique_id(void* id_out_128_bytes);
rten_status rten_b200_comm_create(rten_ctx* ctx, const void* id_128_bytes, int rank, int world_size, rten_comm** out);
void rten_b200_comm_destroy(rten_comm* comm);
/* 1: the range exchange runs as one kernel over NVLink peer memory (mailboxes opened through CUDA IPC at comm_create);
 * 0: the peers' memory could not be opened (or RTEN_B200_NCCL_RANGES=1) and two ncclAllReduce calls are used.  Both are exact. */
int rten_b200_comm_uses_peer_memory(const rten_comm* comm);
/* Exchanges that gave up waiting for a peer (~30 s) since comm_create: 0 in a healthy run, -1 if the device cannot be read. */
int rten_b200_comm_timeouts(const rten_comm* comm);

/* DynamicQuantizeLinear (src/ops/quantize.rs:352-468): y u8, scale f32 scalar, zero_point u8 scalar.
 * comm_or_null (a rten_comm*): when the batch is sharded over ranks, the local (min, max) is all-reduced over the ranks
 * first -- integer min / max on an order-preserving encoding, exact -- so every rank picks the unsharded tensor's scale
 * and zero point (SURVEY.md 8e) and the sharded outputs stay bit-identical to the unsharded reference's. */
rten_status rten_b200_dynamic_quantize_linear(rten_ctx* ctx, const rten_tensor* x, rten_tensor* y,
                                              rten_tensor* scale, rten_tensor* zero_point, void* comm_or_null);
/* Producer-computed ranges.  `out_range_or_null` of the *_integer_ex functions is a device i32[2] in which the kernel
 * epilogue accumulates (min, max) of the f32 output it writes (order-preserving integer encoding, atomicMin / atomicMax:
 * exact, order independent); `rten_b200_range_reset` re-arms any number of such pairs in one launch; the ranged
 * DynamicQuantizeLinear then skips its own pass over x.  Same bits as the plain operator (NaN inputs excepted). */
rten_status rten_b200_range_reset(rten_ctx* ctx, rten_tensor* ranges_i32_n_by_2);
rten_status rten_b200_dynamic_quantize_linear_ranged(rten_ctx* ctx, const rten_tensor* x, const rten_tensor* range_or_null,
                                                     rten_tensor* y, rten_tensor* scale, rten_tensor* zero_point,
                                                     void* comm_or_null);

/* ---- residency glue (SURVEY.md 8f-1) so whole models stay in HBM ------------------------------ */
rten_status rten_b200_relu(rten_ctx* ctx, const rten_tensor* x, rten_tensor* out);
/* Add, Sub and Mul (src/ops/binary_elementwise.rs) with numpy broadcasting: f32 (each result rounded once) or i32
 * (wrapping); a and b of the same type. */
rten_status rten_b200_add(rten_ctx* ctx, const rten_tensor* a, const rten_tensor* b, rten_tensor* out);
rten_status rten_b200_sub(rten_ctx* ctx, const rten_tensor* a, const rten_tensor* b, rten_tensor* out);
rten_status rten_b200_mul(rten_ctx* ctx, const rten_tensor* a, const rten_tensor* b, rten_tensor* out);
/* Div (src/ops/binary_elementwise.rs:600-638) with numpy broadcasting, a and b of the same type:
 *   f32: a / b, IEEE-rounded; x / 0 is +-inf or NaN.  A b of exactly one element (any rank) is the reference's
 *        "division as multiplication-by-reciprocal": a * (1 / b), two roundings, and the output takes a's shape, not
 *        the broadcast one (Div(a[4], b[1, 1]) is [4]).  b is read on the device.
 *   i32: truncates toward zero.  A zero divisor returns RTEN_ERR_INVALID_VALUE "Divisor contains zero", as the reference
 *        does, and so does INT_MIN / -1 (an overflow panic in Rust).  An i32 Div SYNCHRONISES with the host: the
 *        kernel's flag is read back after the launch (so it cannot be captured in a CUDA graph).  On an error the
 *        outputs the call allocated are freed.  Every element of b is checked, also when the output is empty (the
 *        reference checks b before broadcasting). */
rten_status rten_b200_div(rten_ctx* ctx, const rten_tensor* a, const rten_tensor* b, rten_tensor* out);
/* Pow (src/ops/binary_elementwise.rs:965-1029, FastPow) with numpy broadcasting, base a and exponent b:
 *   f32 ^ f32: exponent 2 is x * x, 3 is x * x * x (rounded left to right), both bit-identical to the reference; any
 *              other exponent is CUDA's powf, within its documented 4 ulp of the exact result (the reference's is libm's).
 *   i32 ^ i32: exponents >= 0 wrap (wrapping_pow); a negative one is computed as f32 powf(x, e) and converted back with
 *              Rust's saturating `as i32` (NaN -> 0): 1 ^ -n = 1, 0 ^ -n = INT32_MAX, |x| >= 2 gives 0.
 * A one-element exponent (any rank) maps the base: the output takes a's shape (the reference's map_in).  Mixed types
 * (the reference's i32 ^ f32) return RTEN_ERR_UNSUPPORTED_TYPE: that case is left out. */
rten_status rten_b200_pow(rten_ctx* ctx, const rten_tensor* a, const rten_tensor* b, rten_tensor* out);
/* Where (src/ops/binary_elementwise.rs where_op): out = cond != 0 ? x : y, with cond, x and y broadcast together
 * (numpy rules; RTEN_ERR_INCOMPATIBLE_SHAPES "Cannot broadcast inputs" otherwise).  cond is i32 (ONNX bool maps to
 * i32), x and y are both f32 or both i32; the elements are copied as bits.  Any layouts: dense operands of the output's
 * shape (a one-element operand is read once per thread) run one flat pass; strided windows and broadcasts run a pass over
 * the output's rows.  An allocated output is contiguous; a given `out` may be any strided view (not aliasing an input). */
rten_status rten_b200_where(rten_ctx* ctx, const rten_tensor* cond, const rten_tensor* x, const rten_tensor* y, rten_tensor* out);
/* Equal, Less, LessOrEqual, Greater, GreaterOrEqual (binary_elementwise.rs boolean_op): i32 0 / 1 of a (op) b, a and b
 * both f32 or both i32, broadcast as Where broadcasts.  f32 comparisons are IEEE: NaN compares false, -0 == +0, and
 * subnormals are not flushed. */
rten_status rten_b200_equal(rten_ctx* ctx, const rten_tensor* a, const rten_tensor* b, rten_tensor* out);
rten_status rten_b200_less(rten_ctx* ctx, const rten_tensor* a, const rten_tensor* b, rten_tensor* out);
rten_status rten_b200_less_or_equal(rten_ctx* ctx, const rten_tensor* a, const rten_tensor* b, rten_tensor* out);
rten_status rten_b200_greater(rten_ctx* ctx, const rten_tensor* a, const rten_tensor* b, rten_tensor* out);
rten_status rten_b200_greater_or_equal(rten_ctx* ctx, const rten_tensor* a, const rten_tensor* b, rten_tensor* out);
/* And, Or, Xor (logical_boolean_op) and Not (unary_elementwise.rs not): i32 inputs, nonzero is true, i32 0 / 1 out;
 * the binary ones broadcast as Where broadcasts.  Other types: RTEN_ERR_UNSUPPORTED_TYPE. */
rten_status rten_b200_and(rten_ctx* ctx, const rten_tensor* a, const rten_tensor* b, rten_tensor* out);
rten_status rten_b200_or(rten_ctx* ctx, const rten_tensor* a, const rten_tensor* b, rten_tensor* out);
rten_status rten_b200_xor(rten_ctx* ctx, const rten_tensor* a, const rten_tensor* b, rten_tensor* out);
rten_status rten_b200_not(rten_ctx* ctx, const rten_tensor* x, rten_tensor* out);
/* Trilu (src/ops/trilu.rs), f32 or i32, over every matrix of the last two dims: element (i, j) is kept when
 * i + k - j <= 0 (upper != 0) or >= 0 (upper == 0), else 0.  x with fewer than 2 dims: RTEN_ERR_INVALID_VALUE "Input
 * must have >= 2 dims".  x and out may be any strided views. */
rten_status rten_b200_trilu(rten_ctx* ctx, const rten_tensor* x, int64_t k, int upper, rten_tensor* out);
/* Expand (src/ops/layout.rs expand): x (f32 or i32) broadcast with the n-dim target `shape` (bidirectionally, numpy
 * rules).  A negative target dim: RTEN_ERR_INVALID_VALUE "Target shape contains negative values"; shapes that do not
 * broadcast: RTEN_ERR_INCOMPATIBLE_SHAPES "Cannot broadcast input with target shape".  A dense x broadcast over one run
 * of adjacent dims into a dense output, with repeated rows of at least 128 elements (repeat_kv's [b, kv, 1, l, d] ->
 * [b, kv, n, l, d], or a leading broadcast), runs the repeat kernel, 16 bytes per thread when the rows allow; anything
 * else is a strided copy. */
rten_status rten_b200_expand(rten_ctx* ctx, const rten_tensor* x, const int64_t* shape, int n, rten_tensor* out);
/* Slice (src/ops/slice.rs) of a 4-byte-element x, copied into out: n entries of starts and ends, and of axes and steps
 * when not NULL (axes default to 0 .. n - 1, steps to 1).  Ranges clamp as the reference's SliceRange::clamp, negative
 * starts / ends count from the end.  Errors (RTEN_ERR_INVALID_VALUE): "`axes` length must be <= input rank", "`starts`
 * length must match axis count", "steps must be non-zero", "Axis is invalid".  A negative step is
 * RTEN_ERR_UNSUPPORTED_VALUE: the library's strides are non-negative. */
rten_status rten_b200_slice(rten_ctx* ctx, const rten_tensor* x, const int32_t* starts, const int32_t* ends, const int32_t* axes,
                            const int32_t* steps, int n, rten_tensor* out);
/* Split (src/ops/split.rs) of a 4-byte-element x along `axis` into copies: by the n_split sizes of `split` when not NULL,
 * else into num_outputs pieces of ceil(dim / num_outputs) (the last one shorter, and fewer pieces when they run out).
 * outs has room for n_outs tensors; *n_pieces gets the number written.  Errors (RTEN_ERR_INVALID_VALUE): "Split sizes
 * must be >= 0", "Split sizes do not sum to dimension size", "num_outputs must be > 0", "num_outputs exceeds dim
 * size", "Axis is invalid", and more pieces than n_outs.  On an error every output the call allocated is freed. */
rten_status rten_b200_split(rten_ctx* ctx, const rten_tensor* x, int axis, const int32_t* split, int n_split, int num_outputs,
                            rten_tensor* outs, int n_outs, int32_t* n_pieces);
/* ReduceSum (src/ops/reduce.rs), f32 or i32, one launch.  `axes` (n_axes values in [-ndim, ndim - 1], duplicates
 * allowed) are the reduced axes; n_axes = 0 reduces every axis.  keep_dims != 0 keeps them as size-1 axes.  Each f32
 * output is the reference's Sum (the 64-chain fold of rten-vecmath/src/sum.rs) of its elements taken in row-major order
 * of the reduced axes, bit for bit, whatever the input's strides; i32 sums wrap.  An empty reduction gives 0; a 0-D
 * input (n_axes = 0) gives its value plus 0. */
rten_status rten_b200_reduce_sum(rten_ctx* ctx, const rten_tensor* x, const int32_t* axes, int n_axes, int keep_dims, rten_tensor* out);
/* ReduceMean (src/ops/reduce.rs:524-541), f32 only, one launch: each output is rten_b200_reduce_sum's Sum of its lane
 * divided by the lane length as f32 (one IEEE division).  An empty lane gives NaN.  Axes, keep_dims, strides and a 0-D
 * input as rten_b200_reduce_sum. */
rten_status rten_b200_reduce_mean(rten_ctx* ctx, const rten_tensor* x, const int32_t* axes, int n_axes, int keep_dims,
                                  rten_tensor* out);
/* TopK (src/ops/reduce.rs topk), f32 or i32 x in any strides: the k largest (largest != 0) or smallest elements along
 * `axis` (in [-ndim, ndim - 1]), values (x's type) and i32 indices, both with x's shape but k along the axis, best first.
 * Order: NaN is above every number for both directions (so largest = 0 takes NaNs last); -0.0 and +0.0 are equal;
 * equal values, and several NaNs, come in ascending index order.  Values are copied bit for bit.  `sorted` is accepted
 * and ignored: the output is always sorted.  k = 0 gives empty outputs.  Errors: a 0-D x or an axis out of range
 * "Axis is invalid", k < 0 "k must be positive", k > the axis size "k > dimension size" (RTEN_ERR_INVALID_VALUE);
 * k > 2048 or an axis of 2^31 or more elements RTEN_ERR_UNSUPPORTED_VALUE.  Outputs are the caller's (data set, any
 * strides) or allocated (data NULL); one or two launches.  k = 1 runs on the ArgMax kernels. */
rten_status rten_b200_topk(rten_ctx* ctx, const rten_tensor* x, int64_t k, int axis, int largest, int sorted,
                           rten_tensor* values_out, rten_tensor* indices_out);
/* ArgMax / ArgMin (src/ops/reduce.rs arg_max / arg_min: Iterator::max_by), f32 or i32 x in any strides, i32 indices,
 * one launch.  The index of the first NaN of a lane if it holds one, else of the LAST maximum (ArgMax) or minimum
 * (ArgMin); -0.0 and +0.0 are equal.  keep_dims != 0 keeps the axis with size 1.  Errors: a 0-D x or an axis out of
 * range "Axis is invalid", an empty lane "Cannot select index from empty sequence" (RTEN_ERR_INVALID_VALUE); an axis
 * of 2^31 or more elements RTEN_ERR_UNSUPPORTED_VALUE.  Outputs as for rten_b200_reduce_sum. */
rten_status rten_b200_arg_max(rten_ctx* ctx, const rten_tensor* x, int axis, int keep_dims, rten_tensor* out);
rten_status rten_b200_arg_min(rten_ctx* ctx, const rten_tensor* x, int axis, int keep_dims, rten_tensor* out);
/* MaxPool 2-D (src/ops/pooling.rs): kernel {kh,kw}; pads/strides as conv; padding never wins. */
rten_status rten_b200_max_pool(rten_ctx* ctx, const rten_tensor* x, const int32_t kernel[2], const int32_t pads[4],
                               const int32_t strides[2], rten_tensor* out);
rten_status rten_b200_global_average_pool(rten_ctx* ctx, const rten_tensor* x, rten_tensor* out);
/* AveragePool 2-D (src/ops/pooling.rs:263-333, 391-417), f32 NCHW in any strides; the output layout follows the input.
 * Per output: the sum, from +0.0, of the taps inside the image in (ky, kx) order, each add rounded, then ONE division by
 * kh * kw (count_include_pad != 0) or by the number of taps inside the image.  Bit-identical to the reference.  There
 * is no ceil_mode parameter (rten_b200_max_pool has none either): the model executor rejects ceil_mode = 1. */
rten_status rten_b200_average_pool(rten_ctx* ctx, const rten_tensor* x, const int32_t kernel[2], const int32_t pads[4],
                                   const int32_t strides[2], int count_include_pad, rten_tensor* out);
/* Resize (src/ops/resize.rs), f32: nearest or bilinear resampling of the last two axes.  The target is `scales`
 * (output size floor(in as f32 * scale), output -> input scale 1 / scale) or, with use_sizes != 0, `sizes` (scale
 * in as f32 / out as f32), `n` values each, one per input axis (resize.rs:273-308).  1-D to 4-D inputs of which at most
 * the last two axes change, expanded to NCHW as the reference does (resize.rs:350-407: NCHW; NCW before NHW; HW; W); an
 * output shape equal to the input's is a copy; an empty output comes back empty.  Errors as the
 * reference: n != rank RTEN_ERR_INCOMPATIBLE_SHAPES "scales/sizes length should equal input rank", a negative size
 * RTEN_ERR_INVALID_VALUE "scales/sizes must be positive", anything else RTEN_ERR_UNSUPPORTED_VALUE "Only 1D to 4D
 * inputs are supported with up to two resized dimensions".
 * Every coordinate, weight and blend is computed on the device in f32 with separately rounded operations in the
 * reference's order (x direction first, then y): the result is bit-identical to it, including NaN for a bilinear
 * align_corners output of one pixel along a resized axis (its coordinate is 0 / 0 there too).
 * x in any strides.  A library-allocated output follows the input's layout (channels-last in, channels-last out); a
 * caller's `out` is written through its strides.  One kernel launch: channels-last with C % 4 == 0 and 16-byte
 * addressable pixels moves one float4 of channels per thread; other layouts produce runs of 4 output columns per
 * thread, stored as a float4 when the output row is aligned. */
typedef enum { RTEN_RESIZE_NEAREST = 0, RTEN_RESIZE_LINEAR = 1 } rten_resize_mode;
typedef enum {
    RTEN_RESIZE_HALF_PIXEL = 0,
    RTEN_RESIZE_ASYMMETRIC = 1,
    RTEN_RESIZE_ALIGN_CORNERS = 2,
    RTEN_RESIZE_PYTORCH_HALF_PIXEL = 3
} rten_resize_coord_mode;
typedef enum {
    RTEN_RESIZE_FLOOR = 0,
    RTEN_RESIZE_CEIL = 1,
    RTEN_RESIZE_ROUND_PREFER_FLOOR = 2,
    RTEN_RESIZE_ROUND_PREFER_CEIL = 3
} rten_resize_nearest_mode;
typedef struct {
    int32_t mode;         /* rten_resize_mode */
    int32_t coord_mode;   /* rten_resize_coord_mode */
    int32_t nearest_mode; /* rten_resize_nearest_mode (nearest only) */
    int32_t n;            /* entries of scales / sizes that are set */
    float scales[4];
    int64_t sizes[4];
    int32_t use_sizes;
} rten_resize_params;
rten_status rten_b200_resize(rten_ctx* ctx, const rten_tensor* x, const rten_resize_params* p, rten_tensor* out);
/* Concat (src/ops/concat.rs): `n` >= 1 inputs of one type (f32, i32, i8 or u8) and rank, equal in every dimension but
 * `axis` (negative counts from the end); errors as `concatenated_shape` (concat.rs:20-47).  Inputs and `out` in any
 * strides; a library-allocated output follows the layout of input 0 (channels-last in, channels-last out).  ONE kernel
 * launch per 16 inputs copies every slice, in 16-byte units when every slice is 16-byte addressable and the innermost
 * dimension is contiguous on both sides.  An input that already is its slice of `out` (same address and strides) is
 * skipped: a caller that had the producers write into `out` pays nothing for it. */
rten_status rten_b200_concat(rten_ctx* ctx, const rten_tensor* const* inputs, int n, int axis, rten_tensor* out);
/* Gather along axis 0 of a 2-D table with i32 indices (embedding lookups, src/ops/gather.rs). */
rten_status rten_b200_gather_rows(rten_ctx* ctx, const rten_tensor* table, const rten_tensor* indices_i32,
                                  rten_tensor* out);
/* table[indices[r], :] = updates[r, :] in place (ScatterElements / ScatterND restricted to whole rows of a 2-D f32 table,
 * distinct indices): the KV-cache append when the write position is a device-resident value, so that a decode step is
 * a fixed list of launches and can be replayed as a CUDA graph. */
rten_status rten_b200_scatter_rows(rten_ctx* ctx, rten_tensor* table, const rten_tensor* indices, const rten_tensor* updates);

/* ---- model loading and graph execution (SURVEY.md 8f-3 / 8f-4) ------------------------------------------------- */
/* `Model::load` + `Graph::run_plan` (src/model.rs, src/graph.rs:880-1286) for the hot-path operator set: the ONNX file is
 * decoded by a hand-written wire-format reader (rten-onnx/src/onnx.rs), int64 tensors become i32 as in rten's loader,
 * constants are uploaded to HBM once, Mul(x, Sigmoid(x)) becomes Silu (SiluFusion: either operand order, only when the
 * Sigmoid has no other consumer), then Conv + {Relu, Sigmoid, Silu, HardSigmoid, HardSwish} and MatMul + Add(bias) are
 * fused at load (the subset of src/optimize.rs these models need; Clip is not fused), constant weights are prepacked
 * once (`Operator::prepack`, src/graph.rs:488-565).
 * A run executes the nodes in topological order, one operator call of this library each; temporaries are reference
 * counted and return to the context pool after their last consumer; Relu / Clip / Gelu / Erf / Sigmoid / HardSigmoid /
 * HardSwish / Softmax run in place when the
 * executor holds the last reference to their input (src/graph.rs:973-1049); Reshape / Flatten / Squeeze / Unsqueeze /
 * Transpose / Identity are views.  A Concat over axis 1 whose input channel counts the file determines is written in
 * place: each input produced by Conv (with its fused activation), ConvTranspose, MaxPool, AveragePool, Resize or
 * Upsample -- unless it is a graph output, feeds the Concat twice, already feeds another such Concat, or its channel
 * slice would not start 16-byte aligned -- gets a strided view of its slice of the Concat's buffer as `out`; the Concat
 * node copies the remaining inputs in one launch, and launches nothing when there are none.  Results are bit-identical
 * to the copying plan; env RTEN_B200_NO_CONCAT_ELISION=1 at load selects that plan for comparisons, and
 * rten_b200_model_summary lists the plan under "concat_in_place".  Operators: Conv, ConvInteger, ConvTranspose (constant weights prepacked at load; a
 * node that sets output_shape fails the load), Relu, Clip, Sigmoid, HardSigmoid (alpha / beta, defaults 0.2 / 0.5),
 * HardSwish, MaxPool, AveragePool (ceil_mode = 1 fails the load), Resize and Upsample (scales / sizes must be constants;
 * the attribute checks and defaults of the reference's reader: antialias, exclude_outside, extrapolation_value,
 * keep_aspect_ratio_policy and cubic_coeff_a at their defaults, cubic computed as linear), Concat (a missing axis fails
 * the load), GlobalAveragePool, ReduceMean (spatial axes), ReduceSum (f32 / i32; axes from the attribute or a host-known
 * input 1), Gemm, MatMul, MatMulInteger, Add, Sub and Mul (f32, or i32 wrapping), Softmax, LayerNormalization,
 * RMSNormalization and SimplifiedLayerNormalization (stash_type 1), SkipLayerNormalization and
 * SkipSimplifiedLayerNormalization (com.microsoft; outputs 0 and 3: a missing epsilon or a named mean / inv_std_var output
 * fails the load), Gelu, Erf, Gather (rows of a 2-D table; or, on the host, a host-known vector with host-known indices),
 * Cast (i32 -> f32; an integer Cast of a host-known value stays on the host), Shape (start / end; a host value),
 * DynamicQuantizeLinear, Attention (4-D), MatMulNBits (com.microsoft, bits 4; constant B / scales used in place),
 * RotaryEmbedding, GroupQueryAttention (com.microsoft; output and present_key / present_value, inputs 12-15 rejected;
 * a present cache is a new buffer, so a decode step also copies the past -- two launches, not one -- unless the past is
 * a writable input with capacity, see rten_b200_model_run_ex),
 * MultiHeadAttention (com.microsoft; outputs 0-2; a missing num_heads, an explicit scale <= 0, inputs 8 / 9 and the
 * qk output 3 fail the load; present caches as for GroupQueryAttention), GRU / LSTM (outputs 0-2; constant W prepacked at
 * load; activation_alpha / activation_beta, non-default activations, clip != 0, layout != 0, LSTM input_forget != 0, a
 * missing hidden_size and a non-empty peephole input fail the load), Constant and the view operators.  MatMulNBits,
 * GroupQueryAttention, MultiHeadAttention and the two Skip norms are com.microsoft operators, Gelu is both, every other
 * one is of the default domain ("" or "ai.onnx"); any other (domain, operator) pair fails the LOAD with
 * RTEN_ERR_UNSUPPORTED_VALUE ("unsupported operator <name>", "com.microsoft.<name>" in that domain), and any other
 * domain with "unsupported operator domain '<domain>'".
 * Host values: Shape, a Gather of a host-known vector on axis 0 with host-known indices (scalar or vector, negative
 * indices from the end), an integer Cast and Reshape / Flatten / Squeeze / Unsqueeze / Identity of a host-known value
 * are computed on the host -- no launch, no device memory -- and may be a Reshape target or an axes input.  An operator
 * taking one as a tensor gets a host tensor: GroupQueryAttention reads total_sequence_length from it without a copy back
 * (onnxruntime-genai's attention-mask subgraph), the others stage it. */
typedef struct rten_model rten_model;
rten_status rten_b200_model_load(rten_ctx* ctx, const void* onnx_bytes, size_t len, rten_model** out);
void rten_b200_model_free(rten_model* model);
int32_t rten_b200_model_num_inputs(const rten_model* model);
int32_t rten_b200_model_num_outputs(const rten_model* model);
const char* rten_b200_model_input_name(const rten_model* model, int32_t index);
const char* rten_b200_model_output_name(const rten_model* model, int32_t index);
int32_t rten_b200_model_num_nodes(const rten_model* model); /* after the load-time fusions */
const char* rten_b200_model_node_op(const rten_model* model, int32_t index);
const char* rten_b200_model_summary(const rten_model* model); /* JSON: the decoded file (before fusion) + "concat_in_place" */
/* Inputs by name (device tensors, or host tensors staged for the run; integer inputs are i32).  Outputs by name: any
 * value of the graph may be requested (`Model::run` with arbitrary output nodes); each comes back as a contiguous device
 * tensor the caller owns (rten_b200_free). */
rten_status rten_b200_model_run(rten_model* model, int32_t n_inputs, const char* const* input_names, const rten_tensor* inputs,
                                int32_t n_outputs, const char* const* output_names, rten_tensor* outputs);
/* rten_b200_model_run with writable inputs (the reference's owned inputs with spare capacity, run_in_place).
 * opts_or_null[i] describes inputs[i].  A writable input must be device-resident and have the strides of a dense tensor
 * whose grow_axis has `capacity` positions (grow_axis -1: dense as it is); anything else fails with
 * RTEN_ERR_INVALID_VALUE.  The caller keeps the buffer: the run never frees it.
 * GroupQueryAttention (past inputs 3 / 4) and MultiHeadAttention (6 / 7) write their present cache into the past's
 * buffer -- only the new positions, nothing beyond P + new -- when the past is a writable input with grow_axis 2, the
 * node is its last consumer, it is not a requested output and the capacity holds P + S (GQA) or P + L (MHA).  Otherwise
 * the node builds a new present cache as rten_b200_model_run does.  A requested output that is such a present cache
 * comes back as the view of the input's buffer (not contiguous: the input's strides), and output_alias_or_null[i] is the
 * index of that input; every other output is handed over as by rten_b200_model_run, with output_alias -1. */
typedef struct {
    int32_t writable;  /* the run may write into this input's buffer and return it as an output */
    int32_t grow_axis; /* the axis `capacity` extends (-1: none) */
    int64_t capacity;  /* positions along grow_axis the buffer holds (>= shape[grow_axis]) */
} rten_model_input_opts;
rten_status rten_b200_model_run_ex(rten_model* model, int32_t n_inputs, const char* const* input_names, const rten_tensor* inputs,
                                   const rten_model_input_opts* opts_or_null, int32_t n_outputs, const char* const* output_names,
                                   rten_tensor* outputs, int32_t* output_alias_or_null);
/* The reader alone -- no context, no GPU: JSON description (opset, nodes with operator / inputs / outputs / attribute
 * names, initialisers with type and shape, graph inputs / outputs) of an ONNX file.  `needed` receives the size of the
 * full text incl. the terminator. */
rten_status rten_b200_onnx_summary(const void* onnx_bytes, size_t len, char* json_out, size_t capacity, size_t* needed);

#ifdef __cplusplus
}
#endif
#endif /* RTEN_B200_H */
