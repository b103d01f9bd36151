// Depthwise convolution: out[b, c, oy, ox] of a convolution with groups = in channels = out channels, every batch and
// channel in one launch.  The arithmetic restates the reference's depthwise executor (src/ops/conv/depthwise.rs) per
// output, in its order:
//   f32 : acc = bias[c] (or +0.0), then for ky, then kx, ascending, over the taps that fall inside the image only:
//         acc = acc + x * w, the product and the sum each rounded (no fused multiply-add), so results are bit-identical
//         to it whatever the context's f32 mode (no tensor cores are used).  The residual add and activation of
//         conv2d_ex follow, as the GEMM epilogue performs them.
//   int : acc += (x - x_zp) * (w - w_zp[c]) in wrapping i32, again over the taps inside the image only -- padding acts
//         as x_zp, not as the GEMM path's literal 0 in the shifted-i8 domain.  Then either the i32 itself, or
//         ConvIntegerToFloat's f32(acc) * (scale_b * scale) + bias + residual, Relu, with the GEMM epilogue's roundings
//         and its optional output range.
// Two bodies:
//   channels-last (channel stride 1): a CTA owns a slice of `nv` channel vectors of VEC channels and passes over
//         `runs` groups of 256 / nv consecutive output pixels; the slice's weights are staged in shared memory once, as
//         [tap][channel], so a thread reads one vector of x and one of w per tap.  VEC = 4 (16-byte f32 / 4-byte 8-bit
//         loads) when every pixel stride and base allows it, else 1.
//   otherwise (NCHW and any other strides): one thread per output, consecutive threads along x; weights read through
//         the read-only cache (one channel per warp, almost always).
#include <cuda_runtime.h>

#include <climits>
#include <cstdint>
#include <type_traits>

#include "depthwise.h"
#include "math.cuh"

namespace rtb {
namespace {

constexpr int kThreads = 256;
constexpr int kSmemMax = 48 * 1024;  // weights of a channel slice; larger kernels shrink the slice

// f32 conv; ConvInteger; ConvIntegerToFloat; f32 conv followed by Sigmoid, Silu, HardSigmoid or HardSwish (apply_act
// codes 4-7: a kernel of their own, since their exp and divisions in every output loop slow the codes 0-3 by ~2%)
enum { OUT_F32 = 0, OUT_I32 = 1, OUT_QF32 = 2, OUT_F32_ACT = 3 };
__host__ __device__ constexpr bool f32_out(int out) { return out == OUT_F32 || out == OUT_F32_ACT; }

template <int OUT>
using AccT = typename std::conditional<f32_out(OUT), float, unsigned>::type;

__device__ __forceinline__ int ordered_f32(float f) {  // the encoding of EpilogueDesc::range
    const int i = __float_as_int(f);
    return i >= 0 ? i : i ^ 0x7fffffff;
}

// n (<= VEC) consecutive elements from q, the rest 0; a whole vector is one 16-byte (f32) or 4-byte (8-bit) load
template <typename T, int VEC, bool LDG>
__device__ __forceinline__ void load_vec(const T* q, int n, T (&v)[VEC]) {
    if constexpr (VEC == 4) {
        if (n == 4) {
            if constexpr (sizeof(T) == 4) {
                const float4 f = LDG ? __ldg(reinterpret_cast<const float4*>(q)) : *reinterpret_cast<const float4*>(q);
                v[0] = f.x;
                v[1] = f.y;
                v[2] = f.z;
                v[3] = f.w;
            } else {
                const unsigned u = LDG ? __ldg(reinterpret_cast<const unsigned*>(q)) : *reinterpret_cast<const unsigned*>(q);
#pragma unroll
                for (int k = 0; k < 4; k++) v[k] = (T)(uint8_t)(u >> (8 * k));
            }
            return;
        }
    }
#pragma unroll
    for (int k = 0; k < VEC; k++) v[k] = k < n ? (LDG ? __ldg(q + k) : q[k]) : T(0);
}

template <int OUT, typename XT, typename WT, int VEC>
__device__ __forceinline__ void mac(AccT<OUT> (&acc)[VEC], const XT (&xv)[VEC], const WT (&wv)[VEC], int xz,
                                    const int (&wz)[VEC]) {
#pragma unroll
    for (int k = 0; k < VEC; k++) {
        if constexpr (f32_out(OUT))
            acc[k] = __fadd_rn(acc[k], __fmul_rn(xv[k], wv[k]));
        else  // |x - xz|, |w - wz| <= 255: the product is exact, the sum wraps
            acc[k] += (unsigned)(((int)xv[k] - xz) * ((int)wv[k] - wz[k]));
    }
}

template <int OUT, int VEC>
__device__ __forceinline__ void init_acc(const DepthwiseParams& p, int c0, int n, AccT<OUT> (&acc)[VEC]) {
#pragma unroll
    for (int k = 0; k < VEC; k++) {
        if constexpr (f32_out(OUT))
            acc[k] = (p.bias && k < n) ? __ldg(p.bias + (long long)(c0 + k) * p.bias_stride) : 0.0f;
        else
            acc[k] = 0u;
    }
}

template <int OUT, typename XT, typename WT, int VEC>
__device__ __forceinline__ void zero_points(const DepthwiseParams& p, int c0, int n, int& xz, int (&wz)[VEC]) {
    xz = 0;
#pragma unroll
    for (int k = 0; k < VEC; k++) wz[k] = 0;
    if constexpr (!f32_out(OUT)) {
        if (p.x_zp) xz = (int)__ldg(reinterpret_cast<const XT*>(p.x_zp));
        if (p.w_zp) {
#pragma unroll
            for (int k = 0; k < VEC; k++)
                if (k < n) wz[k] = (int)__ldg(reinterpret_cast<const WT*>(p.w_zp) + (long long)(c0 + k) * p.w_zp_stride);
        }
    }
}

// The epilogue of n channels from c0 at output pixel (b, oy, ox); folds f32 outputs into (lo, hi) for the range
template <int OUT, int VEC>
__device__ __forceinline__ void epilogue(const DepthwiseParams& p, AccT<OUT> (&acc)[VEC], int b, int c0, int oy, int ox,
                                         int n, float& lo, float& hi) {
    const long long ooff = (long long)b * p.os[0] + (long long)c0 * p.os[1] + (long long)oy * p.os[2] + (long long)ox * p.os[3];
    const long long roff = (long long)b * p.rs[0] + (long long)c0 * p.rs[1] + (long long)oy * p.rs[2] + (long long)ox * p.rs[3];
    uint32_t y[VEC];
    float sv = 0.0f;
    if constexpr (OUT == OUT_QF32) {
        sv = __ldg(p.scale);
        if (p.scale_b) sv = __fmul_rn(__ldg(p.scale_b), sv);
    }
#pragma unroll
    for (int k = 0; k < VEC; k++) {
        if constexpr (OUT == OUT_I32) {
            y[k] = acc[k];
        } else {
            float v;
            if constexpr (f32_out(OUT)) {
                v = acc[k];
            } else {
                v = __fmul_rn(__int2float_rn((int)acc[k]), sv);
                if (p.bias && k < n) v = __fadd_rn(v, __ldg(p.bias + (long long)(c0 + k) * p.bias_stride));
            }
            if (p.res && k < n) v = __fadd_rn(v, __ldg(p.res + roff + k * p.rs[1]));
            if constexpr (OUT == OUT_F32_ACT)
                v = apply_act(v, p.act, p.act_alpha, p.act_beta);
            else
                v = apply_act(v, p.act);
            if constexpr (OUT == OUT_QF32) {
                if (k < n) {
                    lo = fminf(lo, v);
                    hi = fmaxf(hi, v);
                }
            }
            y[k] = __float_as_uint(v);
        }
    }
    uint32_t* o = reinterpret_cast<uint32_t*>(p.out) + ooff;
    if (VEC == 4 && n == 4) {  // (the vector body has a channel stride of 1 and 16-byte aligned pixels)
        *reinterpret_cast<uint4*>(o) = make_uint4(y[0], y[1], y[2], y[3]);
    } else {
#pragma unroll
        for (int k = 0; k < VEC; k++)
            if (k < n) o[k * p.os[1]] = y[k];
    }
}

// the warp's (lo, hi) into the launch-wide range; every lane of the warp calls it
__device__ __forceinline__ void range_commit(int* range, float lo, float hi) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        lo = fminf(lo, __shfl_xor_sync(0xffffffffu, lo, o));
        hi = fmaxf(hi, __shfl_xor_sync(0xffffffffu, hi, o));
    }
    if ((threadIdx.x & 31) == 0 && lo <= hi) {
        atomicMin(&range[0], ordered_f32(lo));
        atomicMax(&range[1], ordered_f32(hi));
    }
}

// (b, a, r) of index i over [.., A, R] with r fastest
__device__ __forceinline__ void split3(long long i, int R, int A, bool narrow, int& b, int& a, int& r) {
    if (narrow) {
        unsigned u = (unsigned)i;
        r = (int)(u % (unsigned)R);
        u /= (unsigned)R;
        a = (int)(u % (unsigned)A);
        b = (int)(u / (unsigned)A);
    } else {
        r = (int)(i % R);
        i /= R;
        a = (int)(i % A);
        b = (int)(i / A);
    }
}

template <typename XT, typename WT, int OUT, int VEC>
__global__ void __launch_bounds__(kThreads) depthwise_cl_kernel(const DepthwiseParams p, int nv, int runs, int use_smem, long long npix) {
    extern __shared__ __align__(16) uint8_t smem[];
    WT* sw = reinterpret_cast<WT*>(smem);
    const int csl = VEC * nv, taps = p.kh * p.kw, ppb = kThreads / nv;
    const int cbase = blockIdx.y * csl;
    const WT* wg = reinterpret_cast<const WT*>(p.w);
    if (use_smem) {  // the slice's weights as [tap][channel]
        for (int i = threadIdx.x; i < taps * csl; i += kThreads) {
            const int t = i / csl, cl = i - t * csl, c = cbase + cl, ky = t / p.kw, kx = t - ky * p.kw;
            sw[i] = c < p.C ? wg[(long long)c * p.ws_c + (long long)ky * p.ws_h + (long long)kx * p.ws_w] : WT(0);
        }
        __syncthreads();
    }
    const int cv = threadIdx.x % nv, lane = threadIdx.x / nv;
    const int c0 = cbase + cv * VEC;
    const int n = min(VEC, p.C - c0);
    float lo = INFINITY, hi = -INFINITY;
    int xz, wz[VEC];
    zero_points<OUT, XT, WT, VEC>(p, c0, n > 0 ? n : 0, xz, wz);
    // `runs` groups of ppb consecutive pixels per CTA: the slice's weights are staged once for all of them
    for (int r = 0; r < runs; r++) {
        const long long pix = ((long long)blockIdx.x * runs + r) * ppb + lane;
        if (lane >= ppb || n <= 0 || pix >= npix) continue;
        int b, oy, ox;
        split3(pix, p.OW, p.OH, npix <= INT_MAX, b, oy, ox);
        AccT<OUT> acc[VEC];
        init_acc<OUT, VEC>(p, c0, n, acc);
        const XT* xb = reinterpret_cast<const XT*>(p.x) + (long long)b * p.xs[0] + (long long)c0 * p.xs[1];
        const int iy0 = oy * p.sy - p.pt, ix0 = ox * p.sx - p.pl;
        for (int ky = 0; ky < p.kh; ky++) {
            const int iy = iy0 + ky * p.dy;
            if (iy < 0 || iy >= p.H) continue;
            const XT* xr = xb + (long long)iy * p.xs[2];
            for (int kx = 0; kx < p.kw; kx++) {
                const int ix = ix0 + kx * p.dx;
                if (ix < 0 || ix >= p.W) continue;
                XT xv[VEC];
                load_vec<XT, VEC, true>(xr + (long long)ix * p.xs[3], n, xv);
                WT wv[VEC];
                if (use_smem) {
                    load_vec<WT, VEC, false>(sw + (ky * p.kw + kx) * csl + cv * VEC, VEC, wv);
                } else {
#pragma unroll
                    for (int k = 0; k < VEC; k++)
                        wv[k] = k < n ? __ldg(wg + (long long)(c0 + k) * p.ws_c + (long long)ky * p.ws_h + (long long)kx * p.ws_w)
                                      : WT(0);
                }
                mac<OUT, XT, WT, VEC>(acc, xv, wv, xz, wz);
            }
        }
        epilogue<OUT, VEC>(p, acc, b, c0, oy, ox, n, lo, hi);
    }
    if constexpr (OUT == OUT_QF32)
        if (p.range) range_commit(p.range, lo, hi);
}

template <typename XT, typename WT, int OUT>
__global__ void __launch_bounds__(kThreads) depthwise_planar_kernel(const DepthwiseParams p, long long n_out) {
    const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
    float lo = INFINITY, hi = -INFINITY;
    if (i < n_out) {
        const bool narrow = n_out <= INT_MAX;
        int bc, oy, ox;
        split3(i, p.OW, p.OH, narrow, bc, oy, ox);
        const int c = bc % p.C, b = bc / p.C;
        AccT<OUT> acc[1];
        init_acc<OUT, 1>(p, c, 1, acc);
        int xz, wz[1];
        zero_points<OUT, XT, WT, 1>(p, c, 1, xz, wz);
        const XT* xb = reinterpret_cast<const XT*>(p.x) + (long long)b * p.xs[0] + (long long)c * p.xs[1];
        const WT* wc = reinterpret_cast<const WT*>(p.w) + (long long)c * p.ws_c;
        const int iy0 = oy * p.sy - p.pt, ix0 = ox * p.sx - p.pl;
        for (int ky = 0; ky < p.kh; ky++) {
            const int iy = iy0 + ky * p.dy;
            if (iy < 0 || iy >= p.H) continue;
            const XT* xr = xb + (long long)iy * p.xs[2];
            for (int kx = 0; kx < p.kw; kx++) {
                const int ix = ix0 + kx * p.dx;
                if (ix < 0 || ix >= p.W) continue;
                const XT xv[1] = {__ldg(xr + (long long)ix * p.xs[3])};
                const WT wv[1] = {__ldg(wc + (long long)ky * p.ws_h + (long long)kx * p.ws_w)};
                mac<OUT, XT, WT, 1>(acc, xv, wv, xz, wz);
            }
        }
        epilogue<OUT, 1>(p, acc, b, c, oy, ox, 1, lo, hi);
    }
    if constexpr (OUT == OUT_QF32)
        if (p.range) range_commit(p.range, lo, hi);
}

bool aligned(const void* ptr, int bytes) { return (reinterpret_cast<uintptr_t>(ptr) % bytes) == 0; }

template <typename XT, typename WT, int OUT>
rten_status launch_typed(rten_ctx* ctx, const DepthwiseParams& p) {
    const long long npix = (long long)p.B * p.OH * p.OW;
    const int taps = p.kh * p.kw;
    if (p.xs[1] == 1 && p.C > 1) {
        // 4-channel vectors when x's and the output's pixels are whole vectors (a channel tail is handled in the kernel)
        const int xe = (int)sizeof(XT);
        const bool vec = p.os[1] == 1 && aligned(p.x, 4 * xe) && aligned(p.out, 16) && p.xs[0] % 4 == 0 && p.xs[2] % 4 == 0 &&
                         p.xs[3] % 4 == 0 && p.os[0] % 4 == 0 && p.os[2] % 4 == 0 && p.os[3] % 4 == 0;
        const int VEC = vec ? 4 : 1;
        // a slice of nv channel vectors (at most 64, slices balanced) x 256 / nv pixels per pass; the weight slice must
        // fit in shared memory, else it is read through the read-only cache
        const int nvec = (p.C + VEC - 1) / VEC, nslices = (nvec + 63) / 64;
        int nv = (nvec + nslices - 1) / nslices;
        while (nv > 1 && (long long)taps * VEC * nv * (int)sizeof(WT) > kSmemMax) nv = (nv + 1) / 2;
        const long long smem = (long long)taps * VEC * nv * (int)sizeof(WT);
        const int use_smem = smem <= kSmemMax;
        const int ppb = kThreads / nv;
        const long long gy = (p.C + (long long)VEC * nv - 1) / ((long long)VEC * nv);
        // passes per CTA: up to 8, while the grid still gives every SM several CTAs
        const long long groups = (npix + ppb - 1) / ppb;
        int runs = 8;
        while (runs > 1 && groups * gy < (long long)runs * ctx->num_sms * 8) runs /= 2;
        const long long gx = (groups + runs - 1) / runs;
        if (gx > INT_MAX || gy > 65535) return fail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "depthwise convolution is too large");
        const dim3 grid((unsigned)gx, (unsigned)gy);
        const size_t sb = use_smem ? (size_t)smem : 0;
        auto kern = vec ? depthwise_cl_kernel<XT, WT, OUT, 4> : depthwise_cl_kernel<XT, WT, OUT, 1>;
        return launch(ctx, "depthwise convolution launch", kern, {grid, kThreads, sb}, p, nv, runs, use_smem, npix);
    }
    const long long n = npix * p.C;
    const long long g = (n + kThreads - 1) / kThreads;
    if (g > INT_MAX) return fail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "depthwise convolution is too large");
    return launch(ctx, "depthwise convolution launch", depthwise_planar_kernel<XT, WT, OUT>, {(unsigned)g, kThreads}, p, n);
}

template <typename XT, typename WT>
rten_status launch_int(rten_ctx* ctx, const DepthwiseParams& p) {
    return p.scale ? launch_typed<XT, WT, OUT_QF32>(ctx, p) : launch_typed<XT, WT, OUT_I32>(ctx, p);
}

template <typename XT>
rten_status launch_int_w(rten_ctx* ctx, const DepthwiseParams& p) {
    return p.w_dtype == RTEN_I8 ? launch_int<XT, int8_t>(ctx, p) : launch_int<XT, uint8_t>(ctx, p);
}

}  // namespace

rten_status launch_depthwise(rten_ctx* ctx, const DepthwiseParams& p) {
    if ((long long)p.B * p.C * p.OH * p.OW == 0) return RTEN_OK;
    if (p.x_dtype == RTEN_F32)
        return p.act > 3 ? launch_typed<float, float, OUT_F32_ACT>(ctx, p) : launch_typed<float, float, OUT_F32>(ctx, p);
    return p.x_dtype == RTEN_I8 ? launch_int_w<int8_t>(ctx, p) : launch_int_w<uint8_t>(ctx, p);
}

}  // namespace rtb
