// MatMulNBits kernels: A [M, K] f32 times B stored as 4-bit blocks (ONNX Runtime's com.microsoft.MatMulNBits layout:
// B [N, K / block, block / 2] bytes, byte j of a block holding element 2j in its low nibble and 2j + 1 in its high
// nibble, zero point 8, one f32 scale per column and block).  Both kernels dequantize on chip exactly as the reference
// does (rten-gemm/src/block_quant.rs:821-852): w = f32(q - 8) * scale, one f32 rounding.  See nbits.h.
//
// nbits_skinny_kernel (few rows, HBM-bound): a warp owns CPW columns; per K chunk of 1024 its lanes load one 16-byte
//   unit (32 elements) of each column and the matching scales, the CTA stages the chunk of A in shared memory, and each
//   lane accumulates its 32 elements of every (row, column) with exact f32 FMAs.  The lanes' partial sums are combined by
//   a butterfly in a fixed order: no atomics, no split over CTAs, repeated runs are bit-identical.
// nbits_wgmma_kernel (many rows): one CTA per 128 x 128 output tile.
//   warp 8, TMA: per K step of 32 the A tile [128 rows x 128 B] into a four-stage ring, and every eighth step the packed
//       nibbles of the next 256 K of the B tile [128 columns x 128 B] into a two-stage ring (both 128B-swizzled)
//   warps 0-7 (two warpgroups, rows 0-63 and 64-127 of the tile): while the tensor core multiplies step j, they
//       dequantize the nibbles of step j + 1 into the swizzled K-major B tile (3xTF32: also the low parts of that B tile
//       and of the A tile) in a second buffer; wgmma tf32 m64n128k8.  3xTF32 runs lo*hi, hi*lo, hi*hi per step from a
//       zero accumulator and adds the step's sum to the output registers in round-to-nearest f32, as attn_prefill.cu
//       does: the tensor core's own accumulation over long K would exceed the f32-grade bound of that mode.
//   The dequantized B exists only in shared memory: nothing but A, the nibbles, the scales and the output touch HBM.
#include <cuda.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>
#include <cstdlib>
#include <cstring>

#include "nbits.h"
#include "ptx.cuh"
#include "tf32_split.cuh"
#include "umma_gemm.h"

namespace rtb {

namespace {

// f32(q - 8) for a nibble q, exactly: 2^23 + q minus 2^23 + 8
__device__ __forceinline__ float nib_value(uint32_t q) { return __fsub_rn(__uint_as_float(0x4B000000u | q), 8388616.0f); }

// =====================================================================================================================
// skinny kernel
// =====================================================================================================================
constexpr int SK_THREADS = 256;
constexpr int KC = 1024;  // K chunk staged in shared memory: one 16-byte unit of every column per lane

struct SkinnyParams {
    NbitsLaunch L;
    int tiles;  // column tiles of 8 * CPW columns
};

template <int MT, int CPW>
__global__ void __launch_bounds__(SK_THREADS, MT <= 8 ? 2 : 1) nbits_skinny_kernel(const SkinnyParams p) {
    // A chunk [MT][KC / 4] float4; float4 f of a row sits at f ^ ((f >> 3) & 7), so that the 32 lanes reading their own
    // 128-byte runs hit distinct banks
    extern __shared__ float4 sa[];
    const NbitsLaunch& L = p.L;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int K = L.K, M = L.M, N = L.N;
    const int lb = __ffs(L.block) - 1;
    constexpr int F = KC / 4;
    pdl_wait();
    pdl_launch_dependents();
    for (int tile = blockIdx.x; tile < p.tiles; tile += gridDim.x) {
        const int n0 = tile * 8 * CPW + warp * CPW;
        float acc[MT * CPW];
#pragma unroll
        for (int i = 0; i < MT * CPW; i++) acc[i] = 0.0f;
        for (int k0 = 0; k0 < K; k0 += KC) {
            const int c = (k0 >> 5) + lane;  // this lane's 16-byte unit of every column: elements 32 c .. 32 c + 31
            const int kc = 32 * c;
            const bool live = n0 < N && kc < K;
            const bool full = kc + 16 < K;  // false: the unit ends K (K % 32 == 16) and holds 16 elements
            uint4 q[CPW];
            float s0[CPW], s1[CPW];
#pragma unroll
            for (int j = 0; j < CPW; j++) {
                const int n = min(n0 + j, N - 1);
                q[j] = make_uint4(0u, 0u, 0u, 0u);
                s0[j] = s1[j] = 0.0f;
                if (live) {
                    q[j] = __ldg(reinterpret_cast<const uint4*>(L.q + (long long)n * L.qs) + c);
                    const float* sr = L.scales + (long long)n * L.s_n;
                    s0[j] = __ldg(sr + (long long)(kc >> lb) * L.s_k);
                    if (full) s1[j] = __ldg(sr + (long long)((kc + 16) >> lb) * L.s_k);
                }
            }
            __syncthreads();  // the previous chunk has been consumed
            // thread tid stages float4 tid of every row (all loads in flight at once)
            static_assert(F == SK_THREADS, "one float4 of each row per thread");
            const bool in_k = tid < (min(KC, K - k0) >> 2);
            float4 v[MT];
#pragma unroll
            for (int r = 0; r < MT; r++) {
                v[r] = make_float4(0.f, 0.f, 0.f, 0.f);
                if (r < M && in_k) v[r] = __ldg(reinterpret_cast<const float4*>(L.a + (long long)r * L.as + k0) + tid);
            }
#pragma unroll
            for (int r = 0; r < MT; r++) sa[r * F + (tid ^ ((tid >> 3) & 7))] = v[r];
            __syncthreads();
            if (live) {
#pragma unroll
                for (int wi = 0; wi < 4; wi++) {  // 8 elements per 32-bit word
                    if (wi >= 2 && !full) break;
                    float w[CPW][8];
#pragma unroll
                    for (int j = 0; j < CPW; j++) {
                        const uint32_t word = wi == 0 ? q[j].x : wi == 1 ? q[j].y : wi == 2 ? q[j].z : q[j].w;
                        const float s = wi < 2 ? s0[j] : s1[j];
#pragma unroll
                        for (int e = 0; e < 8; e++) w[j][e] = __fmul_rn(nib_value((word >> (4 * e)) & 15u), s);
                    }
                    const int f0 = lane * 8 + 2 * wi;
                    const int p0 = f0 ^ (lane & 7), p1 = (f0 + 1) ^ (lane & 7);
#pragma unroll
                    for (int m = 0; m < MT; m++) {
                        const float4 a0 = sa[m * F + p0], a1 = sa[m * F + p1];
#pragma unroll
                        for (int j = 0; j < CPW; j++) {
                            float t = acc[m * CPW + j];
                            t = __fmaf_rn(a0.x, w[j][0], t);
                            t = __fmaf_rn(a0.y, w[j][1], t);
                            t = __fmaf_rn(a0.z, w[j][2], t);
                            t = __fmaf_rn(a0.w, w[j][3], t);
                            t = __fmaf_rn(a1.x, w[j][4], t);
                            t = __fmaf_rn(a1.y, w[j][5], t);
                            t = __fmaf_rn(a1.z, w[j][6], t);
                            t = __fmaf_rn(a1.w, w[j][7], t);
                            acc[m * CPW + j] = t;
                        }
                    }
                }
            }
        }
        // sums over the 32 lanes: an xor butterfly (every lane ends with the same value, the order is fixed)
#pragma unroll
        for (int i = 0; i < MT * CPW; i++) {
#pragma unroll
            for (int o = 16; o >= 1; o >>= 1) acc[i] = __fadd_rn(acc[i], __shfl_xor_sync(0xffffffffu, acc[i], o));
        }
#pragma unroll
        for (int i = 0; i < MT * CPW; i++) {
            const int m = i / CPW, n = n0 + i % CPW;
            if ((i & 31) == lane && m < M && n < N) L.out[(long long)m * L.os + n] = acc[i];
        }
    }
}

rten_status launch_skinny(rten_ctx* ctx, const NbitsLaunch& L) {
    const int mt = L.M <= 8 ? 8 : (L.M <= 16 ? 16 : 32), cpw = mt == 32 ? 2 : 4;
    SkinnyParams p;
    p.L = L;
    p.tiles = (L.N + 8 * cpw - 1) / (8 * cpw);
    const size_t smem = (size_t)mt * KC * sizeof(float);
    auto kern = mt == 8 ? nbits_skinny_kernel<8, 4> : (mt == 16 ? nbits_skinny_kernel<16, 4> : nbits_skinny_kernel<32, 2>);
    return launch(ctx, "MatMulNBits skinny launch", kern, {std::min(p.tiles, 2 * ctx->num_sms), SK_THREADS, smem, (int)smem, true}, p);
}

// =====================================================================================================================
// wgmma kernel
// =====================================================================================================================
constexpr int WG_THREADS = 288;  // warps 0-7: two MMA warpgroups; warp 8: TMA
constexpr int BM = 128, BN = 128, BK = 32;
constexpr int NS = 4;           // A stages
constexpr int QSTEPS = 8;       // K steps per nibble tile (128 bytes of every column: one 128B-swizzled TMA row)
constexpr int NQ = 2;           // nibble stages
constexpr int GROUP_M = 8;      // M tiles per raster group
constexpr uint32_t A_T = BM * 128;  // A tile: 128 rows x 32 f32
constexpr uint32_t Q_T = BN * 128;  // nibble tile: 128 columns x 256 elements
constexpr uint32_t B_T = BN * 128;  // dequantized B tile: 128 columns x 32 f32, K-major

template <bool X3>
struct WCfg {
    static constexpr size_t SMEM = 1024 /* alignment */ + 1024 /* barriers */ + NS * A_T + NQ * Q_T + 2 * B_T + (X3 ? 2 * (B_T + A_T) : 0);
    static_assert(SMEM <= 227 * 1024, "shared memory");
};

struct WgParams {
    int M, N, K, lb, mtiles, ntiles;
    const float* scales;
    long long s_n, s_k;
    float* out;
    long long os;
};

// D[64 x 128] += A[64 x 32] . B[128 x 32]^T from one 128B-swizzled K-major sub-tile each (3xTF32: a_lo*b, a*b_lo, a*b)
template <bool X3>
__device__ __forceinline__ void mma_step(float (&d)[64], const uint8_t* a, const uint8_t* a_lo, const uint8_t* b, const uint8_t* b_lo) {
    wgmma_fence_operand(d);
    wgmma_fence();
#pragma unroll
    for (int pass = X3 ? 0 : 2; pass < 3; pass++) {
        const uint64_t ad = make_kmajor_sw128_desc(smem_u32(pass == 0 ? a_lo : a));
        const uint64_t bd = make_kmajor_sw128_desc(smem_u32(pass == 1 ? b_lo : b));
#pragma unroll
        for (int k = 0; k < 4; k++) wgmma_tf32_n128(d, ad + 2 * k, bd + 2 * k);
    }
    wgmma_commit();
}

template <bool X3>
__global__ void __launch_bounds__(WG_THREADS, 1)
nbits_wgmma_kernel(const __grid_constant__ CUtensorMap tma_a, const __grid_constant__ CUtensorMap tma_q, const __grid_constant__ WgParams p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* full = reinterpret_cast<uint64_t*>(base);  // [NS]: the A tile of the stage landed
    uint64_t* empty = full + NS;                         // [NS]: the 8 MMA warps are done with the stage
    uint64_t* qfull = empty + NS;                        // [NQ]: the nibble tile landed
    uint64_t* qempty = qfull + NQ;                       // [NQ]: the 8 MMA warps have dequantized all of it
    uint8_t* sa = base + 1024;                           // [NS] A tiles
    uint8_t* sq = sa + NS * A_T;                         // [NQ] nibble tiles
    uint8_t* sb = sq + NQ * Q_T;                         // [2] dequantized B tiles
    uint8_t* sb_lo = sb + 2 * B_T;                       // [2] (3xTF32) their low parts
    uint8_t* sa_lo = sb_lo + 2 * B_T;                    // [2] (3xTF32) low parts of the A tiles

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    // raster: groups of GROUP_M tile rows, M fastest inside a group (its A rows and a band of B columns stay in L2)
    const int u = blockIdx.x;
    const int group = u / (GROUP_M * p.ntiles);
    const int first_m = group * GROUP_M;
    const int gm = min(p.mtiles - first_m, GROUP_M);
    const int r = u - group * GROUP_M * p.ntiles;
    const int m0 = (first_m + r % gm) * BM, n0 = (r / gm) * BN;
    const int nk = (p.K + BK - 1) / BK;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tma_a);
        tma_prefetch_desc(&tma_q);
        for (int s = 0; s < NS; s++) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], 8);
        }
        for (int s = 0; s < NQ; s++) {
            mbar_init(&qfull[s], 1);
            mbar_init(&qempty[s], 8);
        }
        fence_mbar_init();
    }
    __syncthreads();
    pdl_wait();
    pdl_launch_dependents();

    if (warp == 8) {
        if (elect_one()) {
            for (int kt = 0; kt < nk; kt++) {
                if (kt % QSTEPS == 0) {
                    const int j = kt / QSTEPS, qs = j % NQ;
                    if (j >= NQ) mbar_wait(&qempty[qs], ((j / NQ) - 1) & 1);
                    mbar_expect_tx(&qfull[qs], Q_T);
                    tma_load_4d(sq + qs * Q_T, &tma_q, &qfull[qs], j * 128, n0, 0, 0);
                }
                const int s = kt % NS;
                if (kt >= NS) mbar_wait(&empty[s], ((kt / NS) - 1) & 1);
                mbar_expect_tx(&full[s], A_T);
                tma_load_4d(sa + s * A_T, &tma_a, &full[s], kt * BK, m0, 0, 0);
            }
        }
        return;
    }

    const int tid = threadIdx.x;  // 0 .. 255
    const int wg = warp >> 2;
    // dequantizing role of this thread in every step: column n0 + dr of the tile, elements 16 dh .. 16 dh + 15 of the step
    const int dr = tid >> 1, dh = tid & 1;
    const int dn = n0 + dr;
    const float* srow = p.scales + (long long)min(dn, p.N - 1) * p.s_n;

    // nibbles of step kt (16-byte unit kt % QSTEPS of the column's 128-byte swizzled row) -> B tile `buf` (3xTF32: + low
    // parts of B and of A)
    auto convert = [&](int kt, int buf) {
        const int s = kt % NS, j = kt / QSTEPS, qs = j % NQ;
        mbar_wait(&full[s], (kt / NS) & 1);
        mbar_wait(&qfull[qs], (j / NQ) & 1);
        const uint2 w2 = *reinterpret_cast<const uint2*>(sq + qs * Q_T + dr * 128 + (((kt % QSTEPS) ^ (dr & 7)) << 4) + 8 * dh);
        if (kt % QSTEPS == QSTEPS - 1) {  // the last step of this nibble tile: its stage may be refilled
            __syncwarp();
            if (lane == 0) mbar_arrive(&qempty[qs]);
        }
        const int k = kt * BK + 16 * dh;  // the 16 elements share one scale (block >= 16)
        const bool ok = dn < p.N && k < p.K;
        const float sc = ok ? __ldg(srow + (long long)(k >> p.lb) * p.s_k) : 0.0f;
#pragma unroll
        for (int i = 0; i < 4; i++) {
            const uint32_t word = i < 2 ? w2.x : w2.y;
            float v[4];
#pragma unroll
            for (int j = 0; j < 4; j++) v[j] = ok ? __fmul_rn(nib_value((word >> (4 * ((4 * i + j) & 7))) & 15u), sc) : 0.0f;
            const uint32_t off = dr * 128 + (((4 * dh + i) ^ (dr & 7)) << 4);
            *reinterpret_cast<float4*>(sb + buf * B_T + off) = make_float4(v[0], v[1], v[2], v[3]);
            if constexpr (X3)
                *reinterpret_cast<float4*>(sb_lo + buf * B_T + off) = make_float4(tf32_lo(v[0]), tf32_lo(v[1]), tf32_lo(v[2]), tf32_lo(v[3]));
        }
        if constexpr (X3) split_lo<256>(sa_lo + buf * A_T, sa + s * A_T, A_T, tid);
        fence_proxy_async();  // the tensor core reads these bytes through the async proxy
    };

    float acc[64];
#pragma unroll
    for (int i = 0; i < 64; i++) acc[i] = 0.0f;
    convert(0, 0);
    asm volatile("bar.sync 1, 256;" ::: "memory");
    for (int kt = 0; kt < nk; kt++) {
        const int s = kt % NS, buf = kt & 1;
        const uint8_t* ta = sa + s * A_T + wg * 64 * 128;
        const uint8_t* ta_lo = sa_lo + buf * A_T + wg * 64 * 128;
        const uint8_t* tb = sb + buf * B_T;
        const uint8_t* tb_lo = sb_lo + buf * B_T;
        if constexpr (X3) {
            float part[64];
#pragma unroll
            for (int i = 0; i < 64; i++) part[i] = 0.0f;
            mma_step<true>(part, ta, ta_lo, tb, tb_lo);
            if (kt + 1 < nk) convert(kt + 1, buf ^ 1);
            wgmma_wait<0>();
            wgmma_fence_operand(part);
#pragma unroll
            for (int i = 0; i < 64; i++) acc[i] = __fadd_rn(acc[i], part[i]);
        } else {
            mma_step<false>(acc, ta, ta_lo, tb, tb_lo);
            if (kt + 1 < nk) convert(kt + 1, buf ^ 1);
            wgmma_wait<0>();
            wgmma_fence_operand(acc);
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[s]);
        // every warp's products of step kt are complete (buffer `buf` is free) and step kt + 1 is converted
        asm volatile("bar.sync 1, 256;" ::: "memory");
    }

    // fragment element i: row 16 (warp % 4) + lane / 4 + 8 ((i >> 1) & 1), column 8 (i >> 2) + 2 (lane % 4) + (i & 1)
    const int row0 = m0 + wg * 64 + 16 * (warp & 3) + (lane >> 2);
    const bool pairs = !(p.os & 1) && !(reinterpret_cast<uintptr_t>(p.out) & 7);  // (col is even) 8-byte stores allowed
#pragma unroll
    for (int i = 0; i < 64; i += 2) {
        const int row = row0 + 8 * ((i >> 1) & 1);
        const int col = n0 + 8 * (i >> 2) + 2 * (lane & 3);
        if (row >= p.M || col >= p.N) continue;
        float* o = p.out + (long long)row * p.os + col;
        if (pairs && col + 1 < p.N) {
            *reinterpret_cast<float2*>(o) = make_float2(acc[i], acc[i + 1]);
        } else {
            o[0] = acc[i];
            if (col + 1 < p.N) o[1] = acc[i + 1];
        }
    }
}

template <bool X3>
rten_status launch_wgmma(rten_ctx* ctx, const NbitsLaunch& L) {
    OperandDesc da, dq;
    da.base = L.a;
    da.dims[0] = L.K;
    da.dims[1] = L.M;
    da.strides[1] = L.as;
    dq.base = L.q;
    dq.dims[0] = L.K / 2;
    dq.dims[1] = L.N;
    dq.strides[1] = L.qs;
    const uint32_t ones[4] = {1, 1, 1, 1};
    const uint32_t abox[4] = {(uint32_t)BK, (uint32_t)BM, 1u, 1u}, qbox[4] = {128u, (uint32_t)BN, 1u, 1u};
    CUtensorMap ma, mq;
    if (!tma_compatible(da, 4, 4) || !tma_compatible(dq, 1, 4) || !encode_map(ctx, &ma, da, 4, true, abox, ones) ||
        !encode_map(ctx, &mq, dq, 1, false, qbox, ones))
        return fail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "MatMulNBits: the tensor maps of A or B could not be encoded");
    WgParams p;
    p.M = L.M;
    p.N = L.N;
    p.K = L.K;
    p.lb = __builtin_ctz((unsigned)L.block);
    p.mtiles = (L.M + BM - 1) / BM;
    p.ntiles = (L.N + BN - 1) / BN;
    p.scales = L.scales;
    p.s_n = L.s_n;
    p.s_k = L.s_k;
    p.out = L.out;
    p.os = L.os;
    if ((long long)p.mtiles * p.ntiles > 0x7fffffffll) return fail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "MatMulNBits: too many output tiles");
    return launch(ctx, "MatMulNBits wgmma launch", nbits_wgmma_kernel<X3>,
                  {(unsigned)(p.mtiles * p.ntiles), WG_THREADS, WCfg<X3>::SMEM, (int)WCfg<X3>::SMEM, true}, ma, mq, p);
}

}  // namespace

rten_status launch_nbits(rten_ctx* ctx, const NbitsLaunch& L) {
    int t = NBITS_SKINNY_MAX_ROWS;
    if (const char* e = getenv("RTEN_B200_NBITS_SKINNY_MAX")) t = std::max(0, std::min(32, atoi(e)));
    if (L.M <= t) return launch_skinny(ctx, L);
    return L.x3 ? launch_wgmma<true>(ctx, L) : launch_wgmma<false>(ctx, L);
}

}  // namespace rtb
