// The one order behind TopK, ArgMax and ArgMin (src/ops/reduce.rs topk, arg_max, arg_min): every element of a lane maps
// to a 64-bit composite key, and each operator takes the largest composite keys.  The high word orders the values, the
// low word breaks ties by index, so no two elements of a lane compare equal.
//
// Value order (order_key): the reference's cmp_nan_greater.  NaN is above every number (all NaNs alike), -0.0 and +0.0
// are equal (the key canonicalises -0 to +0), and the rest is the usual order: for f32 the sign-magnitude bits are
// mapped to an unsigned order, for i32 the sign bit is flipped.  A NaN gets 0xffffffff, which no number reaches.
//
//   mode           high word                        low word               so the largest key is
//   SEL_LARGEST    order_key                        ~index                 the largest value, first index (NaN first)
//   SEL_SMALLEST   NaN ? 0 : ~order_key             ~index                 the smallest value, first index (NaN last)
//   SEL_ARGMAX     order_key                        NaN ? ~index : index   the first NaN, else the last maximum
//   SEL_ARGMIN     NaN ? 0xffffffff : ~order_key    NaN ? ~index : index   the first NaN, else the last minimum
//
// SEL_LARGEST / SEL_SMALLEST are TopK's topk_cmp (ties by ascending index, NaN greater for both directions); ARGMAX /
// ARGMIN are Iterator::max_by over cmp_nan_greater and its reverse, which keeps the last of equal elements but holds on
// to a NaN once reached.  A number's ~order_key is at most 0xff800000 and at least 0x007fffff, so the NaN values above
// stay outside the numbers' range.  Indices are below 2^31.
#pragma once
#include <cstdint>
#include <type_traits>

namespace rtb {

enum SelectMode { SEL_LARGEST = 0, SEL_SMALLEST = 1, SEL_ARGMAX = 2, SEL_ARGMIN = 3 };

__device__ __forceinline__ bool sel_isnan(float v) { return v != v; }
__device__ __forceinline__ bool sel_isnan(int) { return false; }

__device__ __forceinline__ uint32_t order_key(float v) {
    if (v != v) return 0xffffffffu;
    uint32_t u = __float_as_uint(v);
    if (u == 0x80000000u) u = 0;  // -0 ties with +0
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ uint32_t order_key(int v) { return (uint32_t)v ^ 0x80000000u; }

// the high word of the composite key (the radix-select key of TopK)
template <typename T>
__device__ __forceinline__ uint32_t sel_high(T v, int mode) {
    const bool nan = sel_isnan(v);
    const uint32_t k = order_key(v);
    switch (mode) {
        case SEL_SMALLEST: return nan ? 0u : ~k;
        case SEL_ARGMIN: return nan ? 0xffffffffu : ~k;
        default: return k;
    }
}

template <typename T>
__device__ __forceinline__ uint64_t sel_key(T v, uint32_t idx, int mode) {
    const bool later = (mode == SEL_ARGMAX || mode == SEL_ARGMIN) && !sel_isnan(v);
    return ((uint64_t)sel_high(v, mode) << 32) | (later ? idx : ~idx);
}

// the index a composite key was made from (an f32 NaN is the only f32 high word 0xffffffff under ARGMAX / ARGMIN)
template <typename T>
__device__ __forceinline__ uint32_t sel_index(uint64_t key, int mode) {
    const bool nan = std::is_same<T, float>::value && (uint32_t)(key >> 32) == 0xffffffffu;
    const uint32_t lo = (uint32_t)key;
    return ((mode == SEL_ARGMAX || mode == SEL_ARGMIN) && !nan) ? lo : ~lo;
}

__device__ __forceinline__ uint64_t warp_max_u64(uint64_t v) {
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
        const uint64_t o = __shfl_xor_sync(0xffffffffu, v, d);
        v = o > v ? o : v;
    }
    return v;
}

}  // namespace rtb
