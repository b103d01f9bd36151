// Resize and Concat: the operators of a segmentation / detection decoder that only move and blend f32 values, so both are
// bytes-bound and bit-identical to the reference (src/ops/resize.rs, src/ops/concat.rs).
//
// Resize arithmetic, per output pixel and axis, all in f32 on the device with explicitly rounded operations (nvcc must
// not contract a multiply into the add that follows: the reference is Rust, which never does):
//   c  = input_coord(o)                           resize.rs:48-75, the operation order as written there
//   c  = clamp(c, 0, in as f32 - 1)               f32::clamp: a NaN coordinate (align_corners with a 1-pixel output is
//                                                 0 * (in - 1) / 0) stays NaN, indexes pixel 0 and makes the linear
//                                                 weight, hence the output, NaN -- as the reference's does
//   nearest: round_coord(c)                       resize.rs:121-141
//   linear : i1 = c as usize, i2 = min(i1 + 1, in - 1), w = c - i1; lerp(a, b, w) = (1 - w) * a + w * b as two rounded
//            products and a rounded sum, along x first, then y    resize.rs:102-104, 191-235
#include "resize.h"

#include <algorithm>

namespace rtb {
namespace {

__device__ __forceinline__ float input_coord(int dest, float scale, int mode, int len_in, int len_out) {
    switch (mode) {
        case RTEN_RESIZE_ASYMMETRIC:
            return __fmul_rn(scale, (float)dest);
        case RTEN_RESIZE_ALIGN_CORNERS:
            return __fdiv_rn(__fmul_rn((float)dest, (float)(len_in - 1)), (float)(len_out - 1));
        case RTEN_RESIZE_PYTORCH_HALF_PIXEL:
            if (len_out <= 1) return 0.0f;
            // fallthrough
        default:  // half_pixel
            return __fsub_rn(__fmul_rn(scale, __fadd_rn((float)dest, 0.5f)), 0.5f);
    }
}

// the clamped input coordinate of output position `dest` (NaN passes through, as f32::clamp lets it)
__device__ __forceinline__ float clamped_coord(int dest, float scale, int mode, int len_in, int len_out) {
    float c = input_coord(dest, scale, mode, len_in, len_out);
    const float hi = __fsub_rn((float)len_in, 1.0f);
    if (c < 0.0f) c = 0.0f;
    if (c > hi) c = hi;
    return c;
}

// `f32 as usize` of a clamped coordinate: truncation, NaN -> 0
__device__ __forceinline__ int as_index(float c) { return __float2int_rz(c); }

__device__ __forceinline__ int nearest_index(float c, int nearest_mode) {
    switch (nearest_mode) {
        case RTEN_RESIZE_CEIL: return as_index(ceilf(c));
        case RTEN_RESIZE_FLOOR: return as_index(c);
        default: {
            // f32::round rounds halves away from zero: the two round_prefer modes take the half cases themselves
            const float fract = __fsub_rn(c, truncf(c));
            if (fract == 0.5f) return as_index(nearest_mode == RTEN_RESIZE_ROUND_PREFER_CEIL ? ceilf(c) : floorf(c));
            return as_index(roundf(c));
        }
    }
}

struct LinearTap {
    int i1, i2;
    float w;
};
__device__ __forceinline__ LinearTap linear_tap(float c, int len_in) {
    LinearTap t;
    t.i1 = as_index(c);
    t.i2 = min(t.i1 + 1, len_in - 1);
    t.w = __fsub_rn(c, (float)t.i1);
    return t;
}

__device__ __forceinline__ float lerp(float a, float b, float w) {
    return __fadd_rn(__fmul_rn(__fsub_rn(1.0f, w), a), __fmul_rn(w, b));
}
__device__ __forceinline__ float bilerp(float tl, float tr, float bl, float br, float wx, float wy) {
    return lerp(lerp(tl, tr, wx), lerp(bl, br, wx), wy);
}

// Channels-last: one thread per (output pixel, 4 channels).  Coordinates and weights are computed once per thread and
// shared by its channels; adjacent threads cover adjacent channel vectors, so the 128-bit loads and stores coalesce.
template <bool LINEAR>
__global__ void __launch_bounds__(256) resize_cl4_kernel(const ResizeParams p) {
    const int C4 = p.C >> 2;
    const long long total = (long long)p.B * p.OH * p.OW * C4;
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
        long long rem = i;
        const int c = (int)(rem % C4) << 2;
        rem /= C4;
        const int ox = (int)(rem % p.OW);
        rem /= p.OW;
        const int oy = (int)(rem % p.OH);
        const int b = (int)(rem / p.OH);
        const float cy = clamped_coord(oy, p.inv_y, p.coord_mode, p.H, p.OH);
        const float cx = clamped_coord(ox, p.inv_x, p.coord_mode, p.W, p.OW);
        const float* xb = p.x + (long long)b * p.xs[0] + c;
        float4 r;
        if (LINEAR) {
            const LinearTap ty = linear_tap(cy, p.H), tx = linear_tap(cx, p.W);
            const float* r1 = xb + (long long)ty.i1 * p.xs[2];
            const float* r2 = xb + (long long)ty.i2 * p.xs[2];
            const float4 tl = __ldg(reinterpret_cast<const float4*>(r1 + (long long)tx.i1 * p.xs[3]));
            const float4 tr = __ldg(reinterpret_cast<const float4*>(r1 + (long long)tx.i2 * p.xs[3]));
            const float4 bl = __ldg(reinterpret_cast<const float4*>(r2 + (long long)tx.i1 * p.xs[3]));
            const float4 br = __ldg(reinterpret_cast<const float4*>(r2 + (long long)tx.i2 * p.xs[3]));
            r.x = bilerp(tl.x, tr.x, bl.x, br.x, tx.w, ty.w);
            r.y = bilerp(tl.y, tr.y, bl.y, br.y, tx.w, ty.w);
            r.z = bilerp(tl.z, tr.z, bl.z, br.z, tx.w, ty.w);
            r.w = bilerp(tl.w, tr.w, bl.w, br.w, tx.w, ty.w);
        } else {
            const int iy = nearest_index(cy, p.nearest_mode), ix = nearest_index(cx, p.nearest_mode);
            r = __ldg(reinterpret_cast<const float4*>(xb + (long long)iy * p.xs[2] + (long long)ix * p.xs[3]));
        }
        *reinterpret_cast<float4*>(p.out + (long long)b * p.os[0] + (long long)oy * p.os[2] + (long long)ox * p.os[3] + c) = r;
    }
}

// Any strides.  ROW: threads along the output row, each producing 4 consecutive ox of one (b, c, oy), stored as one
// float4 when the row allows (`vec`); the source rows are read through L1 (an upsample re-reads each source element
// scale^2 times).  !ROW: one element per thread with the channel fastest, for channel-contiguous outputs whose channel
// count or alignment rules out resize_cl4_kernel.
template <bool LINEAR, bool ROW>
__global__ void __launch_bounds__(256) resize_kernel(const ResizeParams p, const int vec) {
    const int run = ROW ? 4 : 1;
    const int QW = ROW ? (p.OW + 3) / 4 : p.OW;
    const long long total = (long long)p.B * p.C * p.OH * QW;
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
        int b, c, oy, q;
        long long rem = i;
        if (ROW) {
            q = (int)(rem % QW);
            rem /= QW;
            oy = (int)(rem % p.OH);
            rem /= p.OH;
            c = (int)(rem % p.C);
            b = (int)(rem / p.C);
        } else {
            c = (int)(rem % p.C);
            rem /= p.C;
            q = (int)(rem % QW);
            rem /= QW;
            oy = (int)(rem % p.OH);
            b = (int)(rem / p.OH);
        }
        const float cy = clamped_coord(oy, p.inv_y, p.coord_mode, p.H, p.OH);
        const float* xb = p.x + (long long)b * p.xs[0] + (long long)c * p.xs[1];
        const float *r1, *r2 = nullptr;
        LinearTap ty{0, 0, 0.0f};
        if (LINEAR) {
            ty = linear_tap(cy, p.H);
            r1 = xb + (long long)ty.i1 * p.xs[2];
            r2 = xb + (long long)ty.i2 * p.xs[2];
        } else {
            r1 = xb + (long long)nearest_index(cy, p.nearest_mode) * p.xs[2];
        }
        const int ox0 = q * run;
        float v[4] = {0.0f, 0.0f, 0.0f, 0.0f};
#pragma unroll
        for (int k = 0; k < run; k++) {
            const int ox = ox0 + k;
            if (ox >= p.OW) break;
            const float cx = clamped_coord(ox, p.inv_x, p.coord_mode, p.W, p.OW);
            if (LINEAR) {
                const LinearTap tx = linear_tap(cx, p.W);
                const long long o1 = (long long)tx.i1 * p.xs[3], o2 = (long long)tx.i2 * p.xs[3];
                v[k] = bilerp(__ldg(r1 + o1), __ldg(r1 + o2), __ldg(r2 + o1), __ldg(r2 + o2), tx.w, ty.w);
            } else {
                v[k] = __ldg(r1 + (long long)nearest_index(cx, p.nearest_mode) * p.xs[3]);
            }
        }
        float* o = p.out + (long long)b * p.os[0] + (long long)c * p.os[1] + (long long)oy * p.os[2] + (long long)ox0 * p.os[3];
        if (ROW && vec && ox0 + 4 <= p.OW) {
            *reinterpret_cast<float4*>(o) = make_float4(v[0], v[1], v[2], v[3]);
        } else {
#pragma unroll
            for (int k = 0; k < run; k++)
                if (ox0 + k < p.OW) o[(long long)k * p.os[3]] = v[k];
        }
    }
}

// One launch for up to kConcatMaxSources inputs: blockIdx.y picks the source, the x blocks stride over its elements.
template <typename T>
__global__ void __launch_bounds__(256) concat_kernel(const __grid_constant__ ConcatParams p) {
    const ConcatSource& s = p.s[blockIdx.y];
    const T* __restrict__ src = reinterpret_cast<const T*>(s.src);
    T* __restrict__ out = reinterpret_cast<T*>(p.out);
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < s.n; i += stride) {
        long long rem = i, so = 0, dof = s.dst_off;
        for (int d = p.ndim - 1; d >= 0; d--) {
            const long long size = d == p.axis ? s.ext : p.shape[d];
            const long long idx = rem % size;
            rem /= size;
            so += idx * s.strides[d];
            dof += idx * p.out_strides[d];
        }
        out[dof] = src[so];
    }
}

int grid_for(rten_ctx* ctx, long long work_items) {
    long long blocks = (work_items + 255) / 256;
    const long long cap = (long long)ctx->num_sms * 8;
    if (blocks > cap) blocks = cap;
    if (blocks < 1) blocks = 1;
    return (int)blocks;
}

bool aligned4(const long long* s, int a, int b, int c) { return s[a] % 4 == 0 && s[b] % 4 == 0 && s[c] % 4 == 0; }

}  // namespace

rten_status launch_resize(rten_ctx* ctx, const ResizeParams& p) {
    const long long total = (long long)p.B * p.C * p.OH * p.OW;
    if (total == 0) return RTEN_OK;
    const bool linear = p.mode == RTEN_RESIZE_LINEAR;
    const bool out16 = (reinterpret_cast<uintptr_t>(p.out) & 15) == 0;
    const bool cl4 = p.xs[1] == 1 && p.os[1] == 1 && p.C % 4 == 0 && aligned4(p.xs, 0, 2, 3) && aligned4(p.os, 0, 2, 3) &&
                     (reinterpret_cast<uintptr_t>(p.x) & 15) == 0 && out16;
    const char* what = "resize launch";
    if (cl4)
        return launch(ctx, what, linear ? resize_cl4_kernel<true> : resize_cl4_kernel<false>, {grid_for(ctx, total / 4), 256}, p);
    if (p.os[1] == 1 && p.C > 1)
        return launch(ctx, what, linear ? resize_kernel<true, false> : resize_kernel<false, false>, {grid_for(ctx, total), 256}, p, 0);
    const int vec = p.os[3] == 1 && aligned4(p.os, 0, 1, 2) && out16;
    const int grid = grid_for(ctx, (long long)p.B * p.C * p.OH * ((p.OW + 3) / 4));
    return launch(ctx, what, linear ? resize_kernel<true, true> : resize_kernel<false, true>, {grid, 256}, p, vec);
}

rten_status launch_concat(rten_ctx* ctx, const ConcatParams& p) {
    long long most = 0;
    for (int i = 0; i < p.nsrc; i++) most = std::max(most, p.s[i].n);
    if (p.nsrc == 0 || most == 0) return RTEN_OK;
    const dim3 grid((unsigned)grid_for(ctx, most), (unsigned)p.nsrc);
    auto kern = p.esize == 16 ? concat_kernel<uint4> : (p.esize == 4 ? concat_kernel<uint32_t> : concat_kernel<uint8_t>);
    return launch(ctx, "concat launch", kern, {grid, 256}, p);
}

}  // namespace rtb
