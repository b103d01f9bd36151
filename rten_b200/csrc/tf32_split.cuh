// The 3xTF32 operand split done inside the wgmma kernels that stage their own operands (attn_prefill.cu, nbits.cu):
// kind::tf32 reads only the top 10 mantissa bits of an f32, so a tile serves unchanged as its own high part `hi`, and
// the low part lo = x - hi (exact in f32) goes to a second tile; lo*hi + hi*lo + hi*hi then carries f32-grade products.
#pragma once
#include <cstdint>

namespace rtb {

__device__ __forceinline__ float tf32_lo(float x) { return __fsub_rn(x, __uint_as_float(__float_as_uint(x) & 0xffffe000u)); }

// dst = lo(src) elementwise over `bytes` (same swizzled layout), by the NT threads tid = 0 .. NT - 1
template <int NT = 128>
__device__ __forceinline__ void split_lo(uint8_t* dst, const uint8_t* src, uint32_t bytes, int tid) {
    for (uint32_t i = tid; i < bytes / 16; i += NT) {
        const float4 x = reinterpret_cast<const float4*>(src)[i];
        reinterpret_cast<float4*>(dst)[i] = make_float4(tf32_lo(x.x), tf32_lo(x.y), tf32_lo(x.z), tf32_lo(x.w));
    }
}

}  // namespace rtb
