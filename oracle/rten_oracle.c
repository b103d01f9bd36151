/*
 * rten_oracle.c -- CPU restatement of robertknight/rten's operator hot path.
 *
 * THIS IS TEST INFRASTRUCTURE, NOT THE PRODUCT.  Only tests/, __graft_entry__.smoke()
 * and bench.py's cpu_baseline / --impl reference legs may load it.  The product path
 * (rten_b200/, librten_b200.so) never links or calls anything in oracle/.
 *
 * The reference is Rust (edition 2024); no cargo/rustc exists in the build image, so
 * oracle/_ref cannot be built (see oracle/Makefile).  Every function below
 * restates the reference algorithm and cites the file:line (relative to the rten tree,
 * commit c7f7bad) it follows.  Parity pin: the golden vectors the reference's own tests
 * hold for this path (tests/test_oracle_golden.py).
 *
 * Numeric conventions: the reference's x86-64 host path is the AVX-512 one
 * (rten-simd/src/dispatch.rs:39-56): 16 f32 lanes, fused mul_add
 * (rten-simd/src/arch/x86_64/avx512.rs:260).  `fmaf` below is that fused op; V=16 is
 * the lane count used wherever the reference reduces across SIMD lanes.
 *
 * Build: gcc -O3 -march=x86-64-v3 -fopenmp -ffp-contract=off -shared -fPIC (oracle/Makefile).
 * -ffp-contract=off matters: only explicit fmaf() may fuse, exactly as in the reference.
 */
#include <math.h>
#include <stddef.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <float.h>
#ifdef _OPENMP
#include <omp.h>
#endif

/* Threads a GEMM / im2col may use from where it is called.  Level 0 (not inside a parallel region): every thread
 * of the runtime; level 1 (inside the per-image team loop of rto_conv_f32): the team size g_team; deeper: 1.
 * `work` (multiply-adds) bounds the count so tiny problems do not pay the fork/join of 100+ threads. */
static int g_team = 1;
static int threads_for(size_t work) {
#ifdef _OPENMP
    int level = omp_get_level();
    int nt = level == 0 ? omp_get_max_threads() : (level == 1 ? g_team : 1);
    size_t cap = work / 131072;
    if (cap < 1) cap = 1;
    if ((size_t)nt > cap) nt = (int)cap;
    return nt < 1 ? 1 : nt;
#else
    (void)work;
    return 1;
#endif
}

#define V 16 /* AVX-512 f32 lanes */

/* ------------------------------------------------------------------------------------
 * RNG -- rten-tensor/src/rng.rs:16-32 (XorShift64), :49-66 (integer narrowing),
 *        rten-gemm/src/reduced_range_rng.rs:37-57.
 * ---------------------------------------------------------------------------------- */
static inline uint64_t xorshift_next(uint64_t *state) {
    uint64_t t = *state;
    t ^= t << 13;
    t ^= t >> 7;
    t ^= t << 17;
    *state = t;
    return t;
}

void rto_rng_u64(uint64_t *state, uint64_t *out, size_t n) {
    for (size_t i = 0; i < n; i++) out[i] = xorshift_next(state);
}

/* next_f32: top 40 bits scaled by 2^-40 (rng.rs:26-32). */
void rto_rng_f32(uint64_t *state, float *out, size_t n) {
    const float scale = 1.0f / (float)(1ull << 40);
    for (size_t i = 0; i < n; i++) {
        uint64_t v = xorshift_next(state) >> (64 - 40);
        out[i] = (float)v * scale;
    }
}

void rto_rng_u8(uint64_t *state, uint8_t *out, size_t n, int reduce_range) {
    for (size_t i = 0; i < n; i++) {
        uint64_t v = xorshift_next(state);
        out[i] = reduce_range ? (uint8_t)(v % 128) : (uint8_t)v;
    }
}

void rto_rng_i8(uint64_t *state, int8_t *out, size_t n, int reduce_range) {
    for (size_t i = 0; i < n; i++) {
        uint64_t v = xorshift_next(state);
        out[i] = reduce_range ? (int8_t)((int16_t)(v % 128) - 64) : (int8_t)(uint8_t)v;
    }
}

void rto_rng_i32(uint64_t *state, int32_t *out, size_t n) {
    for (size_t i = 0; i < n; i++) out[i] = (int32_t)(uint32_t)xorshift_next(state);
}

/* ------------------------------------------------------------------------------------
 * exp -- rten-vecmath/src/exp.rs:8-25 (constants), :61-127 (Exp), :140-191
 *        (ReducedRangeExp).
 * ---------------------------------------------------------------------------------- */
#define INV_LOG2 1.44269504088896340736f /* f32::consts::LOG2_E */
#define ROUNDING_MAGIC 12582912.0f
#define LOG2_HI (-6.93145752e-1f)
#define LOG2_LO (-1.42860677e-6f)
#define EXP_POLY_0 1.0f
#define EXP_POLY_1 1.0f
#define EXP_POLY_2 4.99999851e-1f
#define EXP_POLY_3 1.66664720e-1f
#define EXP_POLY_4 4.16695364e-2f
#define EXP_POLY_5 8.37312452e-3f
#define EXP_POLY_6 1.37805939e-3f

static inline float bits_f32(uint32_t u) {
    float f;
    memcpy(&f, &u, 4);
    return f;
}

/* AVX `cvttps2dq`: out-of-range / NaN -> 0x80000000 (rten-simd to_int_trunc). */
static inline int32_t trunc_i32(float x) {
    if (!(x > -2147483904.0f && x < 2147483648.0f)) return INT32_MIN;
    return (int32_t)x;
}

static inline float exp_poly(float x, float *j_out) {
    float j = fmaf(x, INV_LOG2, ROUNDING_MAGIC);
    j = j - ROUNDING_MAGIC;
    float r = fmaf(j, LOG2_HI, x);
    r = fmaf(j, LOG2_LO, r);
    float tmp = EXP_POLY_6;
    tmp = fmaf(tmp, r, EXP_POLY_5);
    tmp = fmaf(tmp, r, EXP_POLY_4);
    tmp = fmaf(tmp, r, EXP_POLY_3);
    tmp = fmaf(tmp, r, EXP_POLY_2);
    tmp = fmaf(tmp, r, EXP_POLY_1);
    *j_out = j;
    return fmaf(tmp, r, EXP_POLY_0);
}

/* exp.rs:61-127 */
float rto_exp1(float x) {
    float j;
    float r = exp_poly(x, &j);
    int32_t k = trunc_i32(j);
    uint32_t ia = (k > 0) ? 0u : 0x83000000u;
    uint32_t is = ia + 0x7f000000u;
    uint32_t it = ((uint32_t)k << 23) - ia;
    r = r * bits_f32(is);
    r = r * bits_f32(it);
    if (x >= 104.0f) r = INFINITY;
    if (x <= -104.0f) r = 0.0f;
    return r;
}

/* exp.rs:140-191; EXP_LOWER_CUTOFF = -126.5*ln2 + 0.01 (exp.rs:131). */
float rto_reduced_range_exp1(float x) {
    const float cutoff = -126.5f * 0.693147180559945309417f + 0.01f;
    float j;
    float r = exp_poly(x, &j);
    int32_t k = trunc_i32(j);
    uint32_t kp = (uint32_t)(k + 127) << 23;
    r = r * bits_f32(kp);
    if (x < cutoff) r = 0.0f;
    return r;
}

void rto_exp(const float *x, float *y, size_t n) {
#pragma omp parallel for schedule(static) if (n > 65536)
    for (size_t i = 0; i < n; i++) y[i] = rto_exp1(x[i]);
}

/* ------------------------------------------------------------------------------------
 * erf / gelu / tanh -- rten-vecmath/src/erf.rs:23-100, tanh.rs:12-66,
 *   poly_eval: rten-simd/src/ops.rs:571-577 (Horner with mul_add, final mul by x),
 *   reciprocal = 1/x exact divide (ops.rs:639), neg = 0 - x (ops.rs:644).
 * ---------------------------------------------------------------------------------- */
float rto_erf1(float x0) {
    int neg = x0 < 0.0f;
    float x = fabsf(x0);
    const float p = 0.3275911f;
    const float a0 = 0.254829592f, a1 = -0.284496736f, a2 = 1.421413741f, a3 = -1.453152027f,
                a4 = 1.061405429f;
    float t = 1.0f / fmaf(x, p, 1.0f);
    float y = a4;
    y = fmaf(y, t, a3);
    y = fmaf(y, t, a2);
    y = fmaf(y, t, a1);
    y = fmaf(y, t, a0);
    float at = y * t;
    float x_m2 = 0.0f - (x * x);
    float e = rto_reduced_range_exp1(x_m2);
    float r = 1.0f - at * e;
    return neg ? (0.0f - r) : r;
}

float rto_gelu1(float x) {
    const float sqrt_2_rcp = 0.70710678118654752440f; /* 1/SQRT_2, erf.rs:58 */
    float half_x = x * 0.5f;
    float y = x * sqrt_2_rcp;
    y = rto_erf1(y) + 1.0f;
    return half_x * y;
}

float rto_tanh1(float x) {
    int x_negative = x <= 0.0f;
    float abs_x = fabsf(x);
    const float P1 = 0.999999940395355224609375f, P3 = -0.33332359790802001953125f,
                P5 = 0.13310669362545013427734375f, P7 = -5.21197654306888580322265625e-2f,
                P9 = 1.5497927553951740264892578125e-2f;
    float x_sqr = x * x;
    float ys = fmaf(P9, x_sqr, P7);
    ys = fmaf(ys, x_sqr, P5);
    ys = fmaf(ys, x_sqr, P3);
    ys = fmaf(ys, x_sqr, P1);
    ys = ys * abs_x;
    float x2 = abs_x * 2.0f;
    float e = rto_exp1(x2);
    float ym = (e - 1.0f) / (e + 1.0f);
    float y = (abs_x >= 9.02f) ? 1.0f : ym;
    if (abs_x <= 0.55f) y = ys;
    if (abs_x <= 0.0004f) y = abs_x;
    return x_negative ? (0.0f - y) : y;
}

float rto_approx_gelu1(float x) {
    const float sqrt_2_pi = 0.7978845608028654f; /* erf.rs:79 */
    float half_x = x * 0.5f;
    float x_cubed = (x * x) * x;
    float y = fmaf(x_cubed, 0.044715f, x);
    y = y * sqrt_2_pi;
    y = rto_tanh1(y);
    y = y + 1.0f;
    return half_x * y;
}

#define UNARY(name, fn)                                                   \
    void name(const float *x, float *y, size_t n) {                       \
        _Pragma("omp parallel for schedule(static) if (n > 65536)")       \
        for (size_t i = 0; i < n; i++) y[i] = fn(x[i]);                   \
    }
UNARY(rto_erf, rto_erf1)
UNARY(rto_gelu, rto_gelu1)
UNARY(rto_approx_gelu, rto_approx_gelu1)
UNARY(rto_tanh, rto_tanh1)

/* Relu -- src/ops/unary_elementwise.rs (Relu = max(x, 0)); NaN handling follows
 * x86 maxps(x, 0): returns the second operand when either is NaN -> 0. */
void rto_relu(const float *x, float *y, size_t n) {
#pragma omp parallel for schedule(static) if (n > 65536)
    for (size_t i = 0; i < n; i++) y[i] = x[i] > 0.0f ? x[i] : 0.0f;
}

/* ------------------------------------------------------------------------------------
 * Lane-wise SIMD folds -- rten-simd/src/iter.rs:70-120 (fold, fold_unroll<4>):
 * 4 accumulators of V lanes over 4V-element chunks, acc0=((acc0+acc1)+acc2)+acc3, then
 * remaining full V chunks into acc0, masked tail, then lanes summed in order
 * (`to_array().into_iter().sum()`).
 * ---------------------------------------------------------------------------------- */
typedef float (*fold_fn)(float acc, float x, float param);
static inline float fold_add(float acc, float x, float p) { (void)p; return acc + x; }
static inline float fold_sqsub(float acc, float x, float p) {
    float d = x - p;
    return fmaf(d, d, acc);
}

static inline float simd_fold_unroll4(const float *x, size_t n, fold_fn f, float param) {
    float acc[4][V];
    for (int u = 0; u < 4; u++)
        for (int l = 0; l < V; l++) acc[u][l] = 0.0f;
    size_t i = 0;
    for (; i + 4 * V <= n; i += 4 * V)
        for (int u = 0; u < 4; u++)
            for (int l = 0; l < V; l++) acc[u][l] = f(acc[u][l], x[i + u * V + l], param);
    for (int u = 1; u < 4; u++)
        for (int l = 0; l < V; l++) acc[0][l] = acc[0][l] + acc[u][l];
    for (; i + V <= n; i += V)
        for (int l = 0; l < V; l++) acc[0][l] = f(acc[0][l], x[i + l], param);
    for (size_t l = 0; i + l < n; l++) acc[0][l] = f(acc[0][l], x[i + l], param);
    float s = 0.0f;
    for (int l = 0; l < V; l++) s += acc[0][l];
    return s;
}

/* rten-vecmath/src/sum.rs:22-35 */
float rto_sum(const float *x, size_t n) { return simd_fold_unroll4(x, n, fold_add, 0.0f); }
/* rten-vecmath/src/sum.rs:111-130 */
float rto_sum_square_sub(const float *x, size_t n, float offset) {
    return simd_fold_unroll4(x, n, fold_sqsub, offset);
}

/* ------------------------------------------------------------------------------------
 * Softmax -- rten-vecmath/src/softmax.rs:60-101 (3 passes), :176-228 (max, exp+sum with
 * per-lane partial sums, masked tail), optional mask add first
 * (src/ops/attention.rs:53-66: `*qk += m` then Softmax in place).
 * ---------------------------------------------------------------------------------- */
static void softmax_lane(const float *x, const float *mask, float *y, size_t n, int flush_nan) {
    if (mask)
        for (size_t i = 0; i < n; i++) y[i] = x[i] + mask[i];
    else if (y != x)
        memcpy(y, x, n * sizeof(float));
    /* max: fold_unroll<4> with max; x86 maxps(max, x) semantics irrelevant without NaN. */
    float m = -FLT_MAX; /* f32::MIN */
    for (size_t i = 0; i < n; i++) m = (m > y[i]) ? m : y[i]; /* maxps(a=max,b=x): a>b?a:b */
    float lanes[V];
    for (int l = 0; l < V; l++) lanes[l] = 0.0f;
    for (size_t i = 0; i < n; i++) {
        float e = rto_reduced_range_exp1(y[i] - m);
        y[i] = e;
        lanes[i % V] = lanes[i % V] + e;
    }
    float s = 0.0f;
    for (int l = 0; l < V; l++) s += lanes[l];
    float inv = 1.0f / s;
    for (size_t i = 0; i < n; i++) {
        float v = y[i] * inv;
        if (flush_nan && v != v) v = 0.0f;
        y[i] = v;
    }
}

/* x: [rows, n]; mask: NULL or [mask_rows, n] broadcast by row % mask_rows is NOT assumed --
 * caller passes an already broadcast mask of the same shape (or NULL). */
void rto_softmax(const float *x, const float *mask, float *y, size_t rows, size_t n,
                 int flush_nan) {
#pragma omp parallel for schedule(static) if (rows * n > 65536)
    for (size_t r = 0; r < rows; r++)
        softmax_lane(x + r * n, mask ? mask + r * n : NULL, y + r * n, n, flush_nan);
}

/* ------------------------------------------------------------------------------------
 * LayerNormalization -- src/ops/norm.rs:103-161 (normalize_slice), :456-529;
 * rten-vecmath/src/normalize.rs:101-169 (three match arms).
 *   gamma == NULL  -> scalar scale `gamma_scalar` (norm.rs:468-470 `scale.item()`)
 *   beta  == NULL  -> scalar bias `beta_scalar`
 * ---------------------------------------------------------------------------------- */
void rto_layer_norm(const float *x, float *y, size_t rows, size_t n, const float *gamma,
                    float gamma_scalar, const float *beta, float beta_scalar, float eps) {
#pragma omp parallel for schedule(static) if (rows * n > 65536)
    for (size_t r = 0; r < rows; r++) {
        const float *xr = x + r * n;
        float *yr = y + r * n;
        float mean = rto_sum(xr, n) / (float)n;
        float var = rto_sum_square_sub(xr, n, mean) / (float)n;
        float rstd = gamma_scalar / sqrtf(var + eps);
        if (!gamma && !beta) {
            /* (None, None, scale, bias) arm */
            for (size_t i = 0; i < n; i++) yr[i] = fmaf(xr[i] - mean, rstd, beta_scalar);
        } else if (gamma && !beta && beta_scalar == 0.0f) {
            /* (Some(scale), None, const_scale, 0.) arm: mul only */
            for (size_t i = 0; i < n; i++) yr[i] = (xr[i] - mean) * (gamma[i] * rstd);
        } else {
            for (size_t i = 0; i < n; i++) {
                float sv = (gamma ? gamma[i] : 1.0f) * rstd;
                float bv = (beta ? beta[i] : 0.0f) + beta_scalar;
                yr[i] = fmaf(xr[i] - mean, sv, bv);
            }
        }
    }
}

/* ------------------------------------------------------------------------------------
 * f32 GEMM -- rten-gemm/src/lib.rs:794-1093 (gemm_impl), :1128-1256 (gemm_block, bias
 * after the first depth block), rten-gemm/src/kernels/simd_generic.rs:285-414
 * (micro-kernel: per K block a fused-multiply-add chain over ascending k starting from 0,
 * then the alpha/beta write-back special cases), block sizes lib.rs:630-663 (kc=256 for
 * f32; MR x NR = 6 x 32 for AVX-512, x86_64.rs:271-274 -- tile shape does not change the
 * per-element arithmetic).
 *
 * A: [M,K] with element strides (a_rs, a_cs); B: [K,N] strides (b_rs, b_cs);
 * C: [M,N] row-major contiguous.  bias_kind: 0 none, 1 row (len N), 2 column (len M).
 * beta == 0 must not read C (lib.rs gemm_uninit; tests.rs:631-674).
 * M == 1 uses the gemv restatement below (lib.rs:876-891).
 * ---------------------------------------------------------------------------------- */
#define KC 256
#define MR 6
#define NR 32

/* gemv -- lib.rs:668-747 + simd_generic.rs:14-103 (row-major B: K chunks of 8, each
 * chunk an fma chain from 0 scaled by alpha then added with the effective beta), bias
 * last.  Deviation (documented): the reference's scalar tail-column path
 * (simd_generic.rs:87-102, unfused `acc += a*b`) depends on the rayon thread count via
 * its column-block split; this restatement uses the fused chain for every column. */
static void gemv_f32(size_t N, size_t K, const float *a, ptrdiff_t a_cs, const float *b,
                     ptrdiff_t b_rs, ptrdiff_t b_cs, float *c, float alpha, float beta,
                     const float *bias, int bias_kind) {
    size_t kblk = (b_rs == 1) ? 512 : 8;
#pragma omp parallel for schedule(static) if (N * K > 262144)
    for (size_t j = 0; j < N; j++) {
        float eff_beta = beta;
        float out = 0.0f;
        for (size_t k0 = 0; k0 < K; k0 += kblk) {
            size_t k1 = k0 + kblk < K ? k0 + kblk : K;
            float acc = 0.0f;
            for (size_t k = k0; k < k1; k++) acc = fmaf(a[k * a_cs], b[k * b_rs + j * b_cs], acc);
            if (alpha != 1.0f) acc = acc * alpha;
            if (eff_beta == 0.0f)
                out = acc;
            else if (eff_beta == 1.0f)
                out = (k0 == 0 ? c[j] : out) + acc;
            else
                out = fmaf((k0 == 0 ? c[j] : out), eff_beta, acc);
            eff_beta = 1.0f;
        }
        if (K == 0) out = (beta == 0.0f) ? 0.0f : c[j] * beta;
        if (bias_kind == 1) out = out + bias[j];
        if (bias_kind == 2) out = out + bias[0];
        c[j] = out;
    }
}

void rto_gemm_f32(size_t M, size_t N, size_t K, const float *a, ptrdiff_t a_rs, ptrdiff_t a_cs,
                  const float *b, ptrdiff_t b_rs, ptrdiff_t b_cs, float *c, float alpha,
                  float beta, const float *bias, int bias_kind) {
    if (M == 0 || N == 0) return;
    if (K == 0) { /* lib.rs:843-873 */
        for (size_t i = 0; i < M; i++)
            for (size_t j = 0; j < N; j++) {
                float v = (beta == 0.0f) ? 0.0f : c[i * N + j] * beta;
                if (bias_kind == 1) v = v + bias[j];
                if (bias_kind == 2) v = v + bias[i];
                c[i * N + j] = v;
            }
        return;
    }
    if (M == 1) {
        gemv_f32(N, K, a, a_cs, b, b_rs, b_cs, c, alpha, beta, bias, bias_kind);
        return;
    }
    size_t n_col_tiles = (N + NR - 1) / NR;
    /* row blocks of mc = 66 rows (row_block_size: 64 rounded up to a multiple of MR, lib.rs:660-663); column tiles x
     * row blocks are distributed over threads like the reference's nested rayon loops (lib.rs:943-1018). */
    const size_t MC = 66;
    size_t n_row_blocks = (M + MC - 1) / MC;
    int nt = threads_for(M * N * K);
#pragma omp parallel if (nt > 1) num_threads(nt)
    {
        static __thread float *bp_buf = NULL;
        if (!bp_buf) bp_buf = (float *)aligned_alloc(64, (size_t)KC * NR * sizeof(float));
        float *bp = bp_buf;
#pragma omp for schedule(dynamic, 1) collapse(2)
        for (size_t jt = 0; jt < n_col_tiles; jt++)
            for (size_t ib = 0; ib < n_row_blocks; ib++) {
                size_t j0 = jt * NR;
                size_t nj = (N - j0 < NR) ? N - j0 : NR;
                size_t r0 = ib * MC, r1 = (r0 + MC < M) ? r0 + MC : M;
                for (size_t k0 = 0; k0 < K; k0 += KC) {
                    size_t kc = (K - k0 < KC) ? K - k0 : KC;
                    /* pack B panel (zero padded lanes are computed but never stored) */
                    for (size_t k = 0; k < kc; k++) {
                        const float *brow = b + (k0 + k) * b_rs + j0 * b_cs;
                        float *dst = bp + k * NR;
                        if (b_cs == 1) {
                            memcpy(dst, brow, nj * sizeof(float));
                        } else {
                            for (size_t j = 0; j < nj; j++) dst[j] = brow[j * b_cs];
                        }
                        for (size_t j = nj; j < NR; j++) dst[j] = 0.0f;
                    }
                    float eff_beta = (k0 == 0) ? beta : 1.0f;
                    for (size_t i0 = r0; i0 < r1; i0 += MR) {
                        size_t mi = (r1 - i0 < MR) ? r1 - i0 : MR;
                        float acc[MR][NR];
                        for (size_t i = 0; i < MR; i++)
                            for (size_t j = 0; j < NR; j++) acc[i][j] = 0.0f;
                        for (size_t k = 0; k < kc; k++) {
                            const float *bk = bp + k * NR;
                            for (size_t i = 0; i < mi; i++) {
                                float av = a[(i0 + i) * a_rs + (k0 + k) * a_cs];
#pragma omp simd
                                for (size_t j = 0; j < NR; j++) acc[i][j] = fmaf(av, bk[j], acc[i][j]);
                            }
                        }
                        for (size_t i = 0; i < mi; i++) {
                            float *crow = c + (i0 + i) * N + j0;
                            for (size_t j = 0; j < nj; j++) {
                                float t = acc[i][j], o;
                                if (eff_beta == 0.0f && alpha == 1.0f)
                                    o = t;
                                else if (eff_beta == 1.0f && alpha == 1.0f)
                                    o = crow[j] + t;
                                else if (eff_beta == 0.0f)
                                    o = t * alpha;
                                else
                                    o = fmaf(t, alpha, crow[j] * eff_beta);
                                if (k0 == 0) {
                                    if (bias_kind == 1) o = o + bias[j0 + j];
                                    if (bias_kind == 2) o = o + bias[i0 + i];
                                }
                                crow[j] = o;
                            }
                        }
                    }
                }
            }
    }
}

/* float64 "truth" GEMM used for error budgeting of the TF32 GPU path, and the
 * sum(|a||b|) bound the tolerance is stated against (2^-9 sum |a||b| in the single-pass TF32 mode). */
void rto_gemm_f64(size_t M, size_t N, size_t K, const float *a, ptrdiff_t a_rs, ptrdiff_t a_cs,
                  const float *b, ptrdiff_t b_rs, ptrdiff_t b_cs, double *c, double *cabs) {
#pragma omp parallel for schedule(static) if (M * N * K > 262144)
    for (size_t i = 0; i < M; i++)
        for (size_t j = 0; j < N; j++) {
            double s = 0.0, sa = 0.0;
            for (size_t k = 0; k < K; k++) {
                double p = (double)a[i * a_rs + k * a_cs] * (double)b[k * b_rs + j * b_cs];
                s += p;
                sa += fabs(p);
            }
            c[i * N + j] = s;
            if (cabs) cabs[i * N + j] = sa;
        }
}

/* ------------------------------------------------------------------------------------
 * int8 GEMM -- u8 x i8 -> i32, exact with wrap-around.
 * rten-gemm/src/kernels/generic.rs:327-355 (direct definition) ==
 * rten-gemm/src/kernels/simd_generic.rs:676-746 (dot - rowsum*zb - colsum*za + K*za*zb);
 * i32 arithmetic wraps (Rust release `+=` on the VNNI path is non-saturating).
 * a_zp: NULL or len M; b_zp: NULL or len N.
 * ---------------------------------------------------------------------------------- */
void rto_gemm_u8i8(size_t M, size_t N, size_t K, const uint8_t *a, ptrdiff_t a_rs,
                   ptrdiff_t a_cs, const int8_t *b, ptrdiff_t b_rs, ptrdiff_t b_cs, int32_t *c,
                   const uint8_t *a_zp, const int8_t *b_zp) {
    int nt = threads_for(M * N * K);
#pragma omp parallel if (nt > 1) num_threads(nt)
    {
        int16_t *bcol = (int16_t *)malloc((K ? K : 1) * sizeof(int16_t));
#pragma omp for schedule(static)
        for (size_t j = 0; j < N; j++) {
            int32_t zb = b_zp ? (int32_t)b_zp[j] : 0;
            for (size_t k = 0; k < K; k++) bcol[k] = (int16_t)((int32_t)b[k * b_rs + j * b_cs] - zb);
            for (size_t i = 0; i < M; i++) {
                int32_t za = a_zp ? (int32_t)a_zp[i] : 0;
                uint32_t acc = 0; /* unsigned: defined wrap-around */
                const uint8_t *ar = a + i * a_rs;
                if (a_cs == 1) {
                    for (size_t k = 0; k < K; k++)
                        acc += (uint32_t)(((int32_t)ar[k] - za) * (int32_t)bcol[k]);
                } else {
                    for (size_t k = 0; k < K; k++)
                        acc += (uint32_t)(((int32_t)ar[k * a_cs] - za) * (int32_t)bcol[k]);
                }
                c[i * N + j] = (int32_t)acc;
            }
        }
        free(bcol);
    }
}

/* cast_scale -- src/ops/matmul.rs:734-773: f32(acc) * scale, scalar or per column. */
void rto_cast_scale(const int32_t *in, float *out, size_t rows, size_t cols, const float *scale,
                    size_t scale_len) {
#pragma omp parallel for schedule(static) if (rows * cols > 65536)
    for (size_t r = 0; r < rows; r++)
        for (size_t j = 0; j < cols; j++)
            out[r * cols + j] = (float)in[r * cols + j] * scale[scale_len == 1 ? 0 : j];
}

/* ------------------------------------------------------------------------------------
 * Conv -- src/ops/conv.rs:124-365 (conv_impl: per group, per image GEMM of
 * W[O/g, (C/g)*kh*kw] @ im2col[(c,ky,kx), (oy,ox)] with column bias),
 * src/ops/conv/im2col.rs:43-108 (row r = (c*kh + ky)*kw + kx; col n = oy*ow + ox;
 * iy = oy*sy - pad_top + ky*dy; ix = ox*sx - pad_left + kx*dx; out of range -> 0),
 * pointwise fast path conv.rs:33-87 (same arithmetic: plain GEMM on X[n] as [C, H*W]).
 * Depthwise (conv.rs:269-284) is out of scope (SURVEY.md 2, row 3) and is computed here
 * through the same im2col+GEMM definition.
 * Output size: src/ops/pooling.rs:63-159 is restated host-side (oracle.py); this
 * function receives explicit out_h/out_w and the 4 fixed pads.
 * ---------------------------------------------------------------------------------- */
static void im2col_f32(const float *x, size_t C, size_t H, size_t W, size_t kh, size_t kw,
                       size_t oh, size_t ow, int pt, int pl, int sy, int sx, int dy, int dx,
                       float *col) {
    size_t Ncol = oh * ow;
    int nt = threads_for(C * kh * kw * Ncol * 8);
#pragma omp parallel for collapse(3) schedule(static) if (nt > 1) num_threads(nt)
    for (size_t c = 0; c < C; c++)
        for (size_t ky = 0; ky < kh; ky++)
            for (size_t kx = 0; kx < kw; kx++) {
                float *dst = col + ((c * kh + ky) * kw + kx) * Ncol;
                for (size_t oy = 0; oy < oh; oy++) {
                    long iy = (long)oy * sy - pt + (long)ky * dy;
                    for (size_t ox = 0; ox < ow; ox++) {
                        long ix = (long)ox * sx - pl + (long)kx * dx;
                        float v = 0.0f;
                        if (iy >= 0 && iy < (long)H && ix >= 0 && ix < (long)W)
                            v = x[(c * H + (size_t)iy) * W + (size_t)ix];
                        dst[oy * ow + ox] = v;
                    }
                }
            }
}

static void conv_f32_one(const float *xi, const float *wg, const float *bg, float *yo, size_t cg, size_t og,
                         size_t H, size_t W, size_t kh, size_t kw, size_t oh, size_t ow, const int *pads,
                         const int *strides, const int *dil, int pointwise) {
    size_t Kd = cg * kh * kw, Ncol = oh * ow;
    if (pointwise) {
        rto_gemm_f32(og, Ncol, Kd, wg, (ptrdiff_t)Kd, 1, xi, (ptrdiff_t)Ncol, 1, yo, 1.0f, 0.0f, bg, bg ? 2 : 0);
    } else {
        /* per-thread scratch that only grows: a fresh multi-megabyte malloc per image and layer means mmap + page
         * faults every time, which serialises many-core hosts on the kernel's address-space lock */
        static __thread float *col_buf = NULL;
        static __thread size_t col_cap = 0;
        size_t need = Kd * Ncol;
        if (need > col_cap) {
            free(col_buf);
            col_buf = (float *)malloc(need * sizeof(float));
            col_cap = need;
        }
        float *col = col_buf;
        im2col_f32(xi, cg, H, W, kh, kw, oh, ow, pads[0], pads[1], strides[0], strides[1], dil[0], dil[1], col);
        rto_gemm_f32(og, Ncol, Kd, wg, (ptrdiff_t)Kd, 1, col, (ptrdiff_t)Ncol, 1, yo, 1.0f, 0.0f, bg, bg ? 2 : 0);
    }
}

/* The reference parallelises over batch items with rayon (conv.rs:317-321) AND inside each GEMM (lib.rs:943-1018,
 * work stealing).  Here: two OpenMP levels -- teams over (image, group), and the column tiles x row blocks of each
 * GEMM over the threads of a team -- same arithmetic whatever the split. */
void rto_conv_f32(const float *x, const float *w, const float *bias, float *y, size_t B,
                  size_t C, size_t H, size_t W, size_t O, size_t kh, size_t kw, size_t oh,
                  size_t ow, const int *pads, const int *strides, const int *dil,
                  size_t groups) {
    size_t cg = C / groups, og = O / groups;
    size_t Kd = cg * kh * kw, Ncol = oh * ow;
    int pointwise = (kh == 1 && kw == 1 && pads[0] == 0 && pads[1] == 0 && pads[2] == 0 &&
                     pads[3] == 0 && strides[0] == 1 && strides[1] == 1);
    size_t units = B * groups;
    int nthreads = 1, in_par = 0;
#ifdef _OPENMP
    nthreads = omp_get_max_threads();
    in_par = omp_in_parallel();
#endif
    if (units > 1 && nthreads > 1 && !in_par) {
        /* teams: `outer` images in flight, each GEMM / im2col inside uses nthreads / outer threads */
        int outer = (size_t)nthreads < units ? nthreads : (int)units;
#ifdef _OPENMP
        omp_set_max_active_levels(2);
#endif
        /* threads inside each image's GEMM only when there are few images: nested teams are re-created for every
         * GEMM call by the OpenMP runtime, which costs more than it gains once >= 8 images run side by side */
        g_team = units >= 8 ? 1 : nthreads / outer;
        if (g_team < 1) g_team = 1;
#pragma omp parallel for schedule(dynamic, 1) collapse(2) num_threads(outer)
        for (size_t n = 0; n < B; n++)
            for (size_t g = 0; g < groups; g++)
                conv_f32_one(x + (n * C + g * cg) * H * W, w + g * og * Kd, bias ? bias + g * og : NULL,
                             y + (n * O + g * og) * Ncol, cg, og, H, W, kh, kw, oh, ow, pads, strides, dil, pointwise);
        g_team = 1;
    } else {
        for (size_t n = 0; n < B; n++)
            for (size_t g = 0; g < groups; g++)
                conv_f32_one(x + (n * C + g * cg) * H * W, w + g * og * Kd, bias ? bias + g * og : NULL,
                             y + (n * O + g * og) * Ncol, cg, og, H, W, kh, kw, oh, ow, pads, strides, dil, pointwise);
    }
}

/* ConvInteger -- src/ops/conv.rs:421-475: kernel is the GEMM LHS (u8 after shift-cast),
 * image is the RHS (i8 after shift-cast); x_zp scalar replicated per column, w_zp per
 * output channel.  Padded taps are packed as literal 0 in the shifted-i8 domain and
 * still receive the -x_zp correction (rten-gemm/src/im2col.rs:340-358, x86 path
 * CAST_B_U8 = false) -- SURVEY.md gotcha G3.  Inputs here are ALREADY shift-cast
 * (w: u8, x: i8); oracle.py performs the casts of data and zero points
 * (src/shift_cast.rs:39-50). */
void rto_conv_u8i8(const int8_t *x, const uint8_t *w, int32_t *y, size_t B, size_t C, size_t H,
                   size_t W, size_t O, size_t kh, size_t kw, size_t oh, size_t ow,
                   const int *pads, const int *strides, const int *dil, size_t groups,
                   int8_t x_zp, const uint8_t *w_zp) {
    size_t cg = C / groups, og = O / groups;
    size_t Kd = cg * kh * kw, Ncol = oh * ow;
#pragma omp parallel for schedule(dynamic, 1) collapse(2)
    for (size_t n = 0; n < B; n++)
        for (size_t g = 0; g < groups; g++) {
            const int8_t *xi = x + (n * C + g * cg) * H * W;
            int8_t *col = (int8_t *)malloc((Kd * Ncol) ? (Kd * Ncol) : 1);
            for (size_t c = 0; c < cg; c++)
                for (size_t ky = 0; ky < kh; ky++)
                    for (size_t kx = 0; kx < kw; kx++) {
                        int8_t *dst = col + ((c * kh + ky) * kw + kx) * Ncol;
                        for (size_t oy = 0; oy < oh; oy++) {
                            long iy = (long)oy * strides[0] - pads[0] + (long)ky * dil[0];
                            for (size_t ox = 0; ox < ow; ox++) {
                                long ix = (long)ox * strides[1] - pads[1] + (long)kx * dil[1];
                                int8_t v = 0; /* literal 0 in the shifted domain (G3) */
                                if (iy >= 0 && iy < (long)H && ix >= 0 && ix < (long)W)
                                    v = xi[(c * H + (size_t)iy) * W + (size_t)ix];
                                dst[oy * ow + ox] = v;
                            }
                        }
                    }
            int8_t *bz = (int8_t *)malloc(Ncol ? Ncol : 1);
            memset(bz, x_zp, Ncol);
            rto_gemm_u8i8(og, Ncol, Kd, w + g * og * Kd, (ptrdiff_t)Kd, 1, col, (ptrdiff_t)Ncol,
                          1, y + (n * O + g * og) * Ncol, w_zp ? w_zp + g * og : NULL, bz);
            free(bz);
            free(col);
        }
}

/* ------------------------------------------------------------------------------------
 * DynamicQuantizeLinear -- src/ops/quantize.rs:352-434; element quantisation
 * rten-vecmath/src/quantize.rs:38-77: i32 rne(x * inv_scale) + zp, then saturate to u8
 * (AVX cvtps2dq: NaN / out of range -> INT32_MIN, which saturates to 0).
 * ---------------------------------------------------------------------------------- */
static inline int32_t rne_i32(float v) {
    if (!(v >= -2147483648.0f && v < 2147483648.0f)) return INT32_MIN;
    return (int32_t)lrintf(v); /* default rounding mode: ties to even */
}

void rto_quantize_u8(const float *x, uint8_t *y, size_t n, float inv_scale, uint8_t zp) {
#pragma omp parallel for schedule(static) if (n > 65536)
    for (size_t i = 0; i < n; i++) {
        int64_t q = (int64_t)rne_i32(x[i] * inv_scale) + (int64_t)zp;
        /* i32 add wraps in the reference only for |x*inv_scale| ~ 2^31; saturate chain
         * i32 -> i16 -> u8 equals clamp(q, 0, 255) for all non-wrapping inputs. */
        if (q < 0) q = 0;
        if (q > 255) q = 255;
        y[i] = (uint8_t)q;
    }
}

void rto_dynamic_quantize_linear(const float *x, size_t n, uint8_t *y, float *scale_out,
                                 uint8_t *zp_out) {
    if (n == 0) { /* quantize.rs:378-386 */
        *scale_out = 1.0f;
        *zp_out = 0;
        return;
    }
    float x_min = INFINITY, x_max = -INFINITY;
#pragma omp parallel for reduction(min : x_min) reduction(max : x_max) if (n > 65536)
    for (size_t i = 0; i < n; i++) {
        if (x[i] < x_min) x_min = x[i];
        if (x[i] > x_max) x_max = x[i];
    }
    const float q_min = 0.0f, q_max = 255.0f;
    float x_min_adj = x_min < q_min ? x_min : q_min;
    float x_max_adj = x_max > q_min ? x_max : q_min;
    float x_range = x_max_adj - x_min_adj;
    float scale = x_range / q_max;
    float min_scaled = x_min_adj / scale;
    float initial_zp = q_min - min_scaled;
    float clipped = initial_zp < q_min ? q_min : (initial_zp > q_max ? q_max : initial_zp);
    float rounded = nearbyintf(clipped); /* round_ties_even */
    float sat = rounded < 0.0f ? 0.0f : (rounded > 255.0f ? 255.0f : rounded);
    uint8_t zp = (sat != sat) ? 0 : (uint8_t)sat; /* `as u8`: NaN -> 0 */
    *scale_out = scale;
    *zp_out = zp;
    float inv_scale = 1.0f / scale; /* quantize.rs:210 */
    rto_quantize_u8(x, y, n, inv_scale, zp);
}

/* ------------------------------------------------------------------------------------
 * Residency glue (SURVEY.md 8f-1), restated for whole-model parity of ResNet-50/BERT:
 *   MaxPool  -- src/ops/pooling.rs (max over in-range taps; padding never wins: -inf)
 *   GlobalAveragePool -- src/ops/pooling.rs:516-521 (vecmath::Sum / len)
 *   Add      -- src/ops/binary_elementwise.rs (same-shape or per-channel; host broadcasts)
 * ---------------------------------------------------------------------------------- */
void rto_maxpool2d(const float *x, float *y, size_t B, size_t C, size_t H, size_t W, size_t kh,
                   size_t kw, size_t oh, size_t ow, const int *pads, const int *strides) {
#pragma omp parallel for schedule(static)
    for (size_t nc = 0; nc < B * C; nc++) {
        const float *xi = x + nc * H * W;
        float *yo = y + nc * oh * ow;
        for (size_t oy = 0; oy < oh; oy++)
            for (size_t ox = 0; ox < ow; ox++) {
                float m = -INFINITY;
                for (size_t ky = 0; ky < kh; ky++)
                    for (size_t kx = 0; kx < kw; kx++) {
                        long iy = (long)oy * strides[0] - pads[0] + (long)ky;
                        long ix = (long)ox * strides[1] - pads[1] + (long)kx;
                        if (iy >= 0 && iy < (long)H && ix >= 0 && ix < (long)W) {
                            float v = xi[(size_t)iy * W + (size_t)ix];
                            m = v > m ? v : m;
                        }
                    }
                yo[oy * ow + ox] = m;
            }
    }
}

void rto_global_avgpool(const float *x, float *y, size_t BC, size_t HW) {
#pragma omp parallel for schedule(static)
    for (size_t i = 0; i < BC; i++) {
        y[i] = rto_sum(x + i * HW, HW) / (float)HW;
    }
}

void rto_add(const float *a, const float *b, float *y, size_t n) {
#pragma omp parallel for schedule(static) if (n > 65536)
    for (size_t i = 0; i < n; i++) y[i] = a[i] + b[i];
}

/* torchrun exports OMP_NUM_THREADS=1; the CPU baseline legs ask for all host cores explicitly. */
void rto_set_num_threads(int n) {
#ifdef _OPENMP
    if (n > 0) omp_set_num_threads(n);
#else
    (void)n;
#endif
}

int rto_num_threads(void) {
#ifdef _OPENMP
    return omp_get_max_threads();
#else
    return 1;
#endif
}
