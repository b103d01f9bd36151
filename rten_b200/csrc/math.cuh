// Device restatement of rten-vecmath's scalar recipes (SURVEY.md Appendix A).  Same operation
// order, fused multiply-adds and exact IEEE division as the reference's AVX-512 path, so the
// elementwise results are bit-identical to it:
//   ReducedRangeExp / Exp : rten-vecmath/src/exp.rs:61-191
//   Erf / Gelu / ApproxGelu: rten-vecmath/src/erf.rs:23-100
//   Tanh                  : rten-vecmath/src/tanh.rs:12-66
// Compile WITHOUT --use_fast_math (division and fmaf must stay IEEE).
#pragma once
#include <cstdint>

namespace rtb {

__device__ __forceinline__ float exp_poly(float x, float& j) {
    const float inv_log2 = 1.44269504088896340736f;
    const float magic = 12582912.0f;
    j = __fmaf_rn(x, inv_log2, magic);
    j = __fsub_rn(j, magic);
    float r = __fmaf_rn(j, -6.93145752e-1f, x);
    r = __fmaf_rn(j, -1.42860677e-6f, r);
    float t = 1.37805939e-3f;
    t = __fmaf_rn(t, r, 8.37312452e-3f);
    t = __fmaf_rn(t, r, 4.16695364e-2f);
    t = __fmaf_rn(t, r, 1.66664720e-1f);
    t = __fmaf_rn(t, r, 4.99999851e-1f);
    t = __fmaf_rn(t, r, 1.0f);
    return __fmaf_rn(t, r, 1.0f);
}

// x86 cvttps2dq semantics: NaN / out of range -> INT_MIN
__device__ __forceinline__ int trunc_i32_x86(float x) {
    if (!(x > -2147483904.0f && x < 2147483648.0f)) return (int)0x80000000;
    return __float2int_rz(x);
}

__device__ __forceinline__ float reduced_range_exp(float x) {
    const float cutoff = -126.5f * 0.693147180559945309417f + 0.01f;
    float j;
    float r = exp_poly(x, j);
    int k = trunc_i32_x86(j);
    float p2 = __int_as_float((int)((unsigned)(k + 127) << 23));
    r = __fmul_rn(r, p2);
    return (x < cutoff) ? 0.0f : r;
}

__device__ __forceinline__ float exp_ref(float x) {
    float j;
    float r = exp_poly(x, j);
    int k = trunc_i32_x86(j);
    unsigned ia = (k > 0) ? 0u : 0x83000000u;
    unsigned is = ia + 0x7f000000u;
    unsigned it = ((unsigned)k << 23) - ia;
    r = __fmul_rn(r, __uint_as_float(is));
    r = __fmul_rn(r, __uint_as_float(it));
    if (x >= 104.0f) r = __int_as_float(0x7f800000);
    if (x <= -104.0f) r = 0.0f;
    return r;
}

__device__ __forceinline__ float erf_ref(float x0) {
    bool neg = x0 < 0.0f;
    float x = fabsf(x0);
    float t = __fdiv_rn(1.0f, __fmaf_rn(x, 0.3275911f, 1.0f));
    float y = 1.061405429f;
    y = __fmaf_rn(y, t, -1.453152027f);
    y = __fmaf_rn(y, t, 1.421413741f);
    y = __fmaf_rn(y, t, -0.284496736f);
    y = __fmaf_rn(y, t, 0.254829592f);
    float at = __fmul_rn(y, t);
    float xm2 = __fsub_rn(0.0f, __fmul_rn(x, x));
    float e = reduced_range_exp(xm2);
    float r = __fsub_rn(1.0f, __fmul_rn(at, e));
    return neg ? __fsub_rn(0.0f, r) : r;
}

__device__ __forceinline__ float gelu_ref(float x) {
    float half_x = __fmul_rn(x, 0.5f);
    float y = __fmul_rn(x, 0.70710678118654752440f);
    y = __fadd_rn(erf_ref(y), 1.0f);
    return __fmul_rn(half_x, y);
}

// ---- two lanes at a time: a pair type with the scalar IEEE operations applied to each half, so gelu_ref_x2 is
// bit-identical to two gelu_ref calls (sm_90 has no packed f32x2 arithmetic; the pairs keep the code shared)
struct f32x2 {
    float x, y;
};
__device__ __forceinline__ f32x2 pack2(float a, float b) { return {a, b}; }
__device__ __forceinline__ void unpack2(f32x2 p, float& a, float& b) {
    a = p.x;
    b = p.y;
}
__device__ __forceinline__ f32x2 fma2(f32x2 a, f32x2 b, f32x2 c) { return {__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y)}; }
__device__ __forceinline__ f32x2 mul2(f32x2 a, f32x2 b) { return {__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)}; }
__device__ __forceinline__ f32x2 add2(f32x2 a, f32x2 b) { return {__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)}; }
__device__ __forceinline__ f32x2 splat2(float c) { return pack2(c, c); }

// (a0, a1) += (b0, b1) on f32 bit patterns, each half rounded to nearest like a scalar add
__device__ __forceinline__ void add_f32x2(uint32_t& a0, uint32_t& a1, float b0, float b1) {
    a0 = __float_as_uint(__fadd_rn(__uint_as_float(a0), b0));
    a1 = __float_as_uint(__fadd_rn(__uint_as_float(a1), b1));
}
// (a0, a1) *= (b0, b1) on f32 bit patterns, each half rounded to nearest like a scalar multiply
__device__ __forceinline__ void mul_f32x2(uint32_t& a0, uint32_t& a1, float b0, float b1) {
    a0 = __float_as_uint(__fmul_rn(__uint_as_float(a0), b0));
    a1 = __float_as_uint(__fmul_rn(__uint_as_float(a1), b1));
}

// reduced_range_exp of two lanes (same roundings as the scalar recipe)
__device__ __forceinline__ void reduced_range_exp_x2(float& x0, float& x1) {
    const f32x2 x = pack2(x0, x1);
    const float magic = 12582912.0f;
    f32x2 j = fma2(x, splat2(1.44269504088896340736f), splat2(magic));
    j = add2(j, splat2(-magic));
    f32x2 r = fma2(j, splat2(-6.93145752e-1f), x);
    r = fma2(j, splat2(-1.42860677e-6f), r);
    f32x2 q = splat2(1.37805939e-3f);
    q = fma2(q, r, splat2(8.37312452e-3f));
    q = fma2(q, r, splat2(4.16695364e-2f));
    q = fma2(q, r, splat2(1.66664720e-1f));
    q = fma2(q, r, splat2(4.99999851e-1f));
    q = fma2(q, r, splat2(1.0f));
    q = fma2(q, r, splat2(1.0f));
    float j0, j1;
    unpack2(j, j0, j1);
    const float p0 = __int_as_float((int)((unsigned)(trunc_i32_x86(j0) + 127) << 23));
    const float p1 = __int_as_float((int)((unsigned)(trunc_i32_x86(j1) + 127) << 23));
    float e0, e1;
    unpack2(mul2(q, pack2(p0, p1)), e0, e1);
    const float cutoff = -126.5f * 0.693147180559945309417f + 0.01f;
    x0 = (x0 < cutoff) ? 0.0f : e0;
    x1 = (x1 < cutoff) ? 0.0f : e1;
}

__device__ __forceinline__ void gelu_ref_x2(float& x0, float& x1) {
    const f32x2 x = pack2(x0, x1);
    const f32x2 half_x = mul2(x, splat2(0.5f));
    const f32x2 y = mul2(x, splat2(0.70710678118654752440f));
    float y0, y1;
    unpack2(y, y0, y1);
    // ---- erf_ref(y)
    const float a0 = fabsf(y0), a1 = fabsf(y1);
    const f32x2 ax = pack2(a0, a1);
    float d0, d1;
    unpack2(fma2(ax, splat2(0.3275911f), splat2(1.0f)), d0, d1);
    const f32x2 t = pack2(__frcp_rn(d0), __frcp_rn(d1));  // == __fdiv_rn(1.0f, d): both are the correctly rounded quotient
    f32x2 pl = splat2(1.061405429f);
    pl = fma2(pl, t, splat2(-1.453152027f));
    pl = fma2(pl, t, splat2(1.421413741f));
    pl = fma2(pl, t, splat2(-0.284496736f));
    pl = fma2(pl, t, splat2(0.254829592f));
    const f32x2 at = mul2(pl, t);
    const f32x2 xm2 = mul2(pack2(-a0, -a1), ax);  // 0 - x*x: the negation of the rounded product, exactly
    // ---- reduced_range_exp(xm2)
    const float magic = 12582912.0f;
    f32x2 j = fma2(xm2, splat2(1.44269504088896340736f), splat2(magic));
    j = add2(j, splat2(-magic));
    f32x2 r = fma2(j, splat2(-6.93145752e-1f), xm2);
    r = fma2(j, splat2(-1.42860677e-6f), r);
    f32x2 q = splat2(1.37805939e-3f);
    q = fma2(q, r, splat2(8.37312452e-3f));
    q = fma2(q, r, splat2(4.16695364e-2f));
    q = fma2(q, r, splat2(1.66664720e-1f));
    q = fma2(q, r, splat2(4.99999851e-1f));
    q = fma2(q, r, splat2(1.0f));
    q = fma2(q, r, splat2(1.0f));
    float j0, j1, m0, m1;
    unpack2(j, j0, j1);
    unpack2(xm2, m0, m1);
    const float p0 = __int_as_float((int)((unsigned)(trunc_i32_x86(j0) + 127) << 23));
    const float p1 = __int_as_float((int)((unsigned)(trunc_i32_x86(j1) + 127) << 23));
    float e0, e1;
    unpack2(mul2(q, pack2(p0, p1)), e0, e1);
    const float cutoff = -126.5f * 0.693147180559945309417f + 0.01f;
    e0 = (m0 < cutoff) ? 0.0f : e0;
    e1 = (m1 < cutoff) ? 0.0f : e1;
    // ---- 1 - at * e (two roundings), sign, + 1, * x / 2
    float r0, r1;
    unpack2(fma2(mul2(at, pack2(e0, e1)), splat2(-1.0f), splat2(1.0f)), r0, r1);
    r0 = (y0 < 0.0f) ? __fsub_rn(0.0f, r0) : r0;
    r1 = (y1 < 0.0f) ? __fsub_rn(0.0f, r1) : r1;
    unpack2(mul2(half_x, add2(pack2(r0, r1), splat2(1.0f))), x0, x1);
}

__device__ __forceinline__ float tanh_ref(float x) {
    bool neg = x <= 0.0f;
    float ax = fabsf(x);
    float x2 = __fmul_rn(x, x);
    float ys = __fmaf_rn(1.5497927553951740264892578125e-2f, x2, -5.21197654306888580322265625e-2f);
    ys = __fmaf_rn(ys, x2, 0.13310669362545013427734375f);
    ys = __fmaf_rn(ys, x2, -0.33332359790802001953125f);
    ys = __fmaf_rn(ys, x2, 0.999999940395355224609375f);
    ys = __fmul_rn(ys, ax);
    float e = exp_ref(__fmul_rn(ax, 2.0f));
    float ym = __fdiv_rn(__fsub_rn(e, 1.0f), __fadd_rn(e, 1.0f));
    float y = (ax >= 9.02f) ? 1.0f : ym;
    if (ax <= 0.55f) y = ys;
    if (ax <= 0.0004f) y = ax;
    return neg ? __fsub_rn(0.0f, y) : y;
}

__device__ __forceinline__ float approx_gelu_ref(float x) {
    float half_x = __fmul_rn(x, 0.5f);
    float x3 = __fmul_rn(__fmul_rn(x, x), x);
    float y = __fmaf_rn(x3, 0.044715f, x);
    y = __fmul_rn(y, 0.7978845608028654f);
    y = tanh_ref(y);
    y = __fadd_rn(y, 1.0f);
    return __fmul_rn(half_x, y);
}

// Sigmoid / Silu (rten-vecmath/src/exp.rs:201-228): 1 / (1 + exp(0 - x)) and x / (1 + exp(0 - x)) -- Silu is ONE
// division, not x * Sigmoid(x).  exp_ref is inf from 104 on, so Silu(x <= -104) = -0 and Silu(-inf) = -inf / inf = NaN.
__device__ __forceinline__ float sigmoid_ref(float x) {
    return __fdiv_rn(1.0f, __fadd_rn(1.0f, exp_ref(__fsub_rn(0.0f, x))));
}
__device__ __forceinline__ float silu_ref(float x) { return __fdiv_rn(x, __fadd_rn(1.0f, exp_ref(__fsub_rn(0.0f, x)))); }

// Rust's f32::clamp(0, 1): `<` / `>` comparisons, so NaN passes through and -0.0 stays -0.0 (fminf / fmaxf would not)
__device__ __forceinline__ float clamp01_ref(float v) {
    if (v < 0.0f) v = 0.0f;
    if (v > 1.0f) v = 1.0f;
    return v;
}
// HardSigmoid / HardSwish (src/ops/unary_elementwise.rs:437-469): product and sum each rounded (Rust does not contract)
__device__ __forceinline__ float hard_sigmoid_ref(float x, float alpha, float beta) {
    return clamp01_ref(__fadd_rn(__fmul_rn(alpha, x), beta));
}
__device__ __forceinline__ float hard_swish_ref(float x) { return __fmul_rn(x, hard_sigmoid_ref(x, 1.0f / 6.0f, 0.5f)); }

// Activation codes of the fused epilogues: 0 none, 1 Relu, 2 Gelu, 3 Gelu (tanh), 4 Sigmoid, 5 Silu, 6 HardSigmoid
// (alpha, beta), 7 HardSwish.  Codes 0-3 only: the decode GEMV kernels (skinny.cu), whose operators take no others.
__device__ __forceinline__ float apply_act(float v, int act) {
    switch (act) {
        case 1: return v > 0.0f ? v : 0.0f;
        case 2: return gelu_ref(v);
        case 3: return approx_gelu_ref(v);
        default: return v;
    }
}
// Every code; alpha / beta are read by code 6 only.
__device__ __forceinline__ float apply_act(float v, int act, float alpha, float beta) {
    switch (act) {
        case 4: return sigmoid_ref(v);
        case 5: return silu_ref(v);
        case 6: return hard_sigmoid_ref(v, alpha, beta);
        case 7: return hard_swish_ref(v);
        default: return apply_act(v, act);
    }
}

}  // namespace rtb
