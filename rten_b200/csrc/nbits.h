// Launchers of the MatMulNBits kernels (nbits.cu): A [M, K] f32 times a 4-bit block-quantized B (com.microsoft
// MatMulNBits, the reference's src/ops/matmul/contrib.rs:21-195), with B dequantized on chip and never written out:
//   w[k, n] = f32(q[n, k] - 8) * scales[n, k / block]      (q: the nibble of element k of column n, zero point 8)
//   out[m, n] = sum_k A[m, k] * w[k, n]
// M <= NBITS_SKINNY_MAX_ROWS (T): nbits_skinny_kernel streams every column's nibbles and scales from HBM once with 16-byte
//   loads, A staged through shared memory in K chunks; exact f32 FMA arithmetic on the dequantized values.
// M > T: nbits_wgmma_kernel, 128 x 128 output tiles on wgmma tf32: a TMA warp streams 128B-swizzled A tiles and the packed
//   nibbles of the B tile, the consumer warpgroups dequantize them into the swizzled K-major B tile wgmma reads (3xTF32:
//   and the low parts of A and B), overlapped with the products of the previous K step.
#pragma once
#include <cstdint>

#include "common.h"

namespace rtb {

// T: at and below this many rows the streaming kernel runs (tools/nbits_bench.py, H100 SXM at a 400 W power limit; README.md
// "MatMulNBits").  At 16 rows it is as fast as or faster than the wgmma kernel on both benched layer shapes in both f32
// modes; at 32 rows it wins in the default 3xTF32 mode on both (the wgmma kernel has only N / 128 CTAs for one M tile)
// and in single-pass TF32 on the (14336, 4096) layer, and loses only single-pass TF32 on the (4096, 14336) layer.
// RTEN_B200_NBITS_SKINNY_MAX (0-32) overrides T, for the benchmark's crossover measurements.
constexpr int NBITS_SKINNY_MAX_ROWS = 32;

struct NbitsLaunch {
    const float* a = nullptr;  // [M, K], row stride as (elements, multiple of 4), 16-byte aligned base
    long long as = 0;
    const uint8_t* q = nullptr;  // [N, K / 2] packed nibbles, row pitch qs bytes (multiple of 16), 16-byte aligned base
    long long qs = 0;
    const float* scales = nullptr;  // element (n, j) at scales[n * s_n + j * s_k]
    long long s_n = 0, s_k = 0;
    int M = 0, N = 0, K = 0;  // K: a multiple of 16
    int block = 32;           // elements per scale: a power of two >= 16
    int x3 = 1;               // wgmma kernel: 1 = 3xTF32 (lo*hi + hi*lo + hi*hi), 0 = one TF32 pass
    float* out = nullptr;     // [M, N], row stride os
    long long os = 0;
};

// The streaming kernel below T rows, the wgmma kernel above; RTEN_ERR_UNSUPPORTED_VALUE if a tensor map cannot be encoded.
rten_status launch_nbits(rten_ctx* ctx, const NbitsLaunch& L);

}  // namespace rtb
