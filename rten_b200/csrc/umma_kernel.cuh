// Device side of the wgmma GEMM / implicit-GEMM convolution: tile decode, the warp-specialised persistent kernel
// (MMA warpgroup / two epilogue groups / TMA producer) and the wide-tile kernel (producer warpgroup / two MMA + epilogue
// warpgroups).  Included ONLY by
// umma_gemm.cu, which holds the host side (launch plans, cost model, autotuner, tensor maps).  See umma_gemm.cu's header
// comment for the design.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>

#include <cstdint>

#include "math.cuh"
#include "ptx.cuh"
#include "umma_gemm.h"

namespace rtb {

constexpr int BM = 128;            // rows per tile: two 64-row wgmma instructions
constexpr int KBYTES = 128;        // bytes of K per stage row = one 128B swizzle atom
constexpr int A_STAGE_BYTES = BM * KBYTES;
constexpr int ACC_STRIDE = 64;     // accumulator columns per stage (two stages, ptx.cuh ACC_COLS); also the widest tile of umma_gemm_kernel
constexpr int PRODUCER_WARP = 12;
constexpr int NUM_THREADS = 416;   // MMA warpgroup (warps 0-3) + 8 epilogue warps (two groups of 4) + TMA producer warp
constexpr int STG_BYTES = 128 * 128;  // one 128-row x 128-byte output staging buffer per epilogue group
constexpr int MAX_STAGES = 8;

// Division by a launch-time constant as multiply-high + shift (exact for 0 <= n < 2^31): the tile decode sits on the
// critical path at the start of every kernel and of every tile, and a hardware-emulated 32-bit division costs ~100
// instructions.
struct FastDiv {
    uint32_t d = 1, mul = 0, shr = 0;
    __host__ void set(int div) {
        d = (uint32_t)(div < 1 ? 1 : div);
        if (d == 1) {
            mul = 0;
            shr = 0;
            return;
        }
        uint32_t lg = 0;
        while ((1ull << lg) < d) lg++;  // ceil(log2(d))
        const uint32_t p = 31 + lg;
        mul = (uint32_t)(((1ull << p) + d - 1) / d);
        shr = p - 32;
    }
    __device__ __forceinline__ int div(int n) const { return d == 1 ? n : (int)(__umulhi((uint32_t)n, mul) >> shr); }
    __device__ __forceinline__ void divmod(int n, int& q, int& r) const {
        q = div(n);
        r = n - q * (int)d;
    }
};

// Epilogue variants of umma_gemm_kernel (umma_epilogue.cuh); the host picks one per launch (pick_epilogue).  The wide
// kernel runs the plain f32 epilogue only.  A "Gelu" variant is the one with the out-of-line activation call (act4):
// it runs every activation code above Relu, not only Gelu.
enum class Epi { Generic, Fast, FastGelu, PlainF32, PlainF32Gelu, PlainI8, PlainI8Gelu };

struct KParams {
    int M, N, K, z0, z1;
    int tiles_m, tiles_n, tiles_total;
    int k_blocks, kelems;
    int bn, stages;
    uint32_t stage_bytes, tx_bytes;  // one 128-byte K block of A and B per pipeline stage
    int sgn;        // integer kind: bit 0 = A signed, bit 1 = B signed
    int conv;
    int tw, th, tb, tiles_x, tiles_y;
    int OH, OW, Bn;
    int sy, sx, dy, dx, pt, pl, kw, c_blocks;
    int a_bcast0, a_bcast1, b_bcast0, b_bcast1;
    int nbuf;       // staging buffers per epilogue group (ring): nbuf-1 (nbuf-2 with res_tma) bulk stores stay in flight
    int res_tma;    // 1: the residual tile is prefetched by TMA into the staging buffer (needs tma_store)
    uint32_t res_tx_bytes;
    int tma_store;  // 1: epilogue stages 128x32 chunks in smem and writes them with TMA (output rows contiguous)
    int splitk;     // > 1: `splitk` CTAs share one output tile, each over `kb_per` K blocks; raw partial accumulators go
                    // to `sk_ws`, the LAST CTA to arrive (per tile and epilogue group, `sk_cnt`) sums them in split order
                    // (deterministic) and runs the epilogue
    int kb_per;
    int units_total;  // tiles_total * splitk
    int x3_cb;      // > 0: 3xTF32 over TWO planes of A -- the K (channel) range is three segments of x3_cb K blocks,
                    //      [lo | hi | hi]: segment 0 reads the low-part plane (tma_a2), segments 1 and 2 read the ORIGINAL f32
                    //      tensor (tf32 wgmma ignores the 13 low mantissa bits, so the raw values ARE the high parts)
    // Projection source (conv only): K blocks [kb_main, k_blocks) are a second 1x1, unpadded convolution of another
    // tensor into the same output pixels -- A from tma_a_proj at (c, ox0 * s_proj, oy0 * s_proj, b0), B from
    // tma_b_proj at (c, n0, 0, 0); x3_cb_proj is its own two-plane 3xTF32 segment length (low parts: tma_a2_proj).
    // Without one, kb_main = k_blocks.
    int kb_main, kb_proj, s_proj, x3_cb_proj;
    // Chained 1x1 convolution (umma_wide_kernel with CHAIN_N2 > 0): a unit is one pixel tile x all N columns, computed
    // in chain_passes passes of bn columns; z = act(y * W2 + chain_bias) over chain_n2 columns, from the staged y chunks
    int chain_n2, chain_passes, chain_act;
    const float* chain_bias;
    FastDiv d_tiles_n, d_tiles_m, d_z0, d_tiles_x, d_tiles_y, d_tiles_total, d_c_blocks, d_kw, d_tw, d_th;
    uint32_t* sk_ws;
    int* sk_cnt;
    EpilogueDesc epi;
};

struct TileCoord {
    int n0;
    int m0;          // plain: first row; conv: unused
    int z0, z1;      // plain batch coords
    int ox0, oy0, b0;  // conv
};

// t indexes output tiles: (n tile, m tile, batch).
__device__ __forceinline__ TileCoord decode_tile(const KParams& p, int t) {
    TileCoord c;
    int n_blk, rest, m_blk, z;
    p.d_tiles_n.divmod(t, rest, n_blk);
    p.d_tiles_m.divmod(rest, z, m_blk);
    c.n0 = n_blk * p.bn;
    c.m0 = m_blk * BM;
    p.d_z0.divmod(z, c.z1, c.z0);
    c.ox0 = c.oy0 = c.b0 = 0;
    if (p.conv) {
        int xt, r2, yt, bt;
        p.d_tiles_x.divmod(m_blk, r2, xt);
        p.d_tiles_y.divmod(r2, bt, yt);
        c.ox0 = xt * p.tw;
        c.oy0 = yt * p.th;
        c.b0 = bt * p.tb;
    }
    return c;
}

// The 4-D output / residual TMA coordinates of column `col` of a tile: (n, x, y, image) for conv, (n, m, z0, z1) else.
__device__ __forceinline__ int4 out_coord(const KParams& p, const TileCoord& tc, int col) {
    return p.conv ? make_int4(tc.n0 + col, tc.ox0, tc.oy0, tc.b0) : make_int4(tc.n0 + col, tc.m0, tc.z0, tc.z1);
}

// Two columns of the plain f32 epilogue, shared by both kernels: x = (acc + residual) + bias, each add rounded to
// nearest, then Relu (Gelu follows on four columns at a time, act4).
__device__ __forceinline__ void plain_f32_pair(uint32_t& v0, uint32_t& v1, bool res, float2 rr, float2 bb, bool relu) {
    if (res) add_f32x2(v0, v1, rr.x, rr.y);
    add_f32x2(v0, v1, bb.x, bb.y);
    if (relu) {
        v0 = __float_as_uint(fmaxf(__uint_as_float(v0), 0.0f));
        v1 = __float_as_uint(fmaxf(__uint_as_float(v1), 0.0f));
    }
}

// The bias of output column n in the plain f32 epilogues: bias[n], or bias[n] + bias2[n] rounded once (the two biases
// of a launch with a projection source)
__device__ __forceinline__ float column_bias(const EpilogueDesc& e, int n) {
    const float b = __ldg(e.bias + n);
    return e.bias2 ? __fadd_rn(b, __ldg(e.bias2 + n)) : b;
}

// cp.async.bulk.wait_group.read takes an immediate: leave at most `n` of this thread's bulk stores un-read
__device__ __forceinline__ void bulk_wait_read(int n) {
    switch (n) {
        case 0: asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); break;
        case 1: asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory"); break;
        case 2: asm volatile("cp.async.bulk.wait_group.read 2;" ::: "memory"); break;
        default: asm volatile("cp.async.bulk.wait_group.read 3;" ::: "memory"); break;
    }
}

__device__ __forceinline__ int f32_to_ordered(float f) {  // same encoding as rowops.cu's min / max kernels
    const int i = __float_as_int(f);
    return i >= 0 ? i : i ^ 0x7fffffff;
}
// fold a warp's running (min, max) into the launch-wide range (EpilogueDesc::range)
__device__ __forceinline__ void range_commit(int* range, float lo, float hi) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        lo = fminf(lo, __shfl_xor_sync(0xffffffffu, lo, o));
        hi = fmaxf(hi, __shfl_xor_sync(0xffffffffu, hi, o));
    }
    if ((threadIdx.x & 31) == 0 && lo <= hi) {
        atomicMin(&range[0], f32_to_ordered(lo));
        atomicMax(&range[1], f32_to_ordered(hi));
    }
}

// Every activation but Relu (Gelu, its tanh form, Sigmoid, Silu, HardSigmoid, HardSwish) of four values as an
// out-of-line call: the specialised epilogue stays short straight-line code (an unrolled polynomial per element would
// multiply its size and thrash the instruction cache), yet these activations do not force a launch into the generic
// epilogue.  The "Gelu" epilogue variants (Epi::*Gelu) are the ones that make this call.
__device__ __noinline__ float4 act4(float4 x, int act, float alpha, float beta) {
    if (act == 2) {  // Gelu: two lanes per packed instruction (bit-identical to gelu_ref, math.cuh)
        gelu_ref_x2(x.x, x.y);
        gelu_ref_x2(x.z, x.w);
        return x;
    }
    x.x = apply_act(x.x, act, alpha, beta);
    x.y = apply_act(x.y, act, alpha, beta);
    x.z = apply_act(x.z, act, alpha, beta);
    x.w = apply_act(x.w, act, alpha, beta);
    return x;
}

// Split-K hand-off of one epilogue group (128 threads): store this CTA's raw accumulator chunks, then count arrivals.
// Returns true for the group of the CTA that arrived last: it owns the epilogue of (tile, group).
// Workspace layout: [tile][split][chunk][column j][row r] so that a warp's 32 rows are contiguous.
__device__ __forceinline__ bool splitk_publish(const KParams& p, int t, int ks, int grp, int q, int lane, uint32_t t_acc,
                                               int* flag, uint32_t acc_smem) {
    const int r = q * 32 + lane;
    const int nchunks = p.bn >> 5;
    for (int c0 = grp * 32; c0 < p.bn; c0 += 64) {
        uint32_t v[32];
        acc_ld(acc_smem, t_acc + c0, v);
        uint32_t* w = p.sk_ws + ((((size_t)t * p.splitk + ks) * nchunks + (c0 >> 5)) << 12) + r;
#pragma unroll
        for (int j = 0; j < 32; j++) __stcg(w + j * 128, v[j]);
    }
    __threadfence();
    asm volatile("bar.sync %0, 128;" ::"r"(1 + grp) : "memory");
    if (q == 0 && lane == 0) {
        int* cnt = p.sk_cnt + t * 2 + grp;
        const int old = atomicAdd(cnt, 1);
        const int last = old == p.splitk - 1;
        if (last) *cnt = 0;  // every split has arrived: re-arm for the next launch
        __threadfence();
        *flag = last;
    }
    asm volatile("bar.sync %0, 128;" ::"r"(1 + grp) : "memory");
    return *reinterpret_cast<volatile int*>(flag) != 0;
}

// Sum of the `splitk` partial chunks in split order (the same order whichever CTA arrived last).
template <int KIND>
__device__ __forceinline__ void splitk_sum(const KParams& p, int t, int c0, int r, uint32_t (&v)[32]) {
    const int nchunks = p.bn >> 5;
    const uint32_t* w = p.sk_ws + ((((size_t)t * p.splitk) * nchunks + (c0 >> 5)) << 12) + r;
    const size_t stride = (size_t)nchunks << 12;
#pragma unroll
    for (int j = 0; j < 32; j++) v[j] = __ldcg(w + j * 128);
#pragma unroll 1
    for (int s = 1; s < p.splitk; s++) {
        w += stride;
#pragma unroll
        for (int j = 0; j < 32; j++) {
            const uint32_t x = __ldcg(w + j * 128);
            if (KIND == 0)
                v[j] = __float_as_uint(__fadd_rn(__uint_as_float(v[j]), __uint_as_float(x)));
            else
                v[j] += x;
        }
    }
}

struct SmemLayout {
    uint8_t* smem;  // operand stages (1024-B aligned), staging buffers behind them
    uint64_t *full_bar, *empty_bar, *acc_full, *acc_empty, *res_bar, *w_bar;
    int* sk_flag;
    float* bias;
    uint32_t acc_smem;  // accumulator tiles (ptx.cuh), between the column vectors and the operand stages
};

}  // namespace rtb

#include "umma_epilogue.cuh"

namespace rtb {

// One 128 x N tile per work unit, accumulated by the warpgroup of warps 0-3 over the unit's K blocks: two 64-row
// wgmma instructions per 32 bytes of K, one wgmma group per pipeline stage.  A stage goes back to the producer once the
// group after it has been issued and it has retired (one arrival per warp); the finished tile is stored to accumulator
// stage (tile count & 1) once the epilogue has released it (8 warp arrivals), then announced (128 arrivals).
template <int KIND, int SGN, int N>
__device__ __forceinline__ void mma_units(const KParams& p, const SmemLayout& L, int worker, int n_workers) {
    const int lane = threadIdx.x & 31;
    const uint32_t smem0 = smem_u32(L.smem);
    uint32_t ring = 0, aphase = 0;  // bit s = uses of operand stage s / accumulator stage s so far, mod 2
    int stage = 0;
    for (int u = worker, it = 0; u < p.units_total; u += n_workers, it++) {
        const int kb0 = p.d_tiles_total.div(u) * p.kb_per, kb1 = min(p.k_blocks, kb0 + p.kb_per);
        const int acc = it & 1;
        acc_t<KIND> d0[N / 2], d1[N / 2];
#pragma unroll
        for (int i = 0; i < N / 2; i++) d0[i] = d1[i] = 0;
        int prev = -1;
        for (int kb = kb0; kb < kb1; kb++) {
            mbar_wait(&L.full_bar[stage], (ring >> stage) & 1);
            wgmma_fence_operand(d0);
            wgmma_fence_operand(d1);
            wgmma_fence();
            const uint32_t sa = smem0 + stage * p.stage_bytes;
            const uint64_t adesc = make_kmajor_sw128_desc(sa);
            const uint64_t bdesc = make_kmajor_sw128_desc(sa + A_STAGE_BYTES);
#pragma unroll
            for (int k = 0; k < 4; k++) {  // +2 in the (addr >> 4) field = 32 B along K in the swizzle atom
                wgmma_k<KIND, SGN, N>(d0, adesc + 2 * k, bdesc + 2 * k);
                wgmma_k<KIND, SGN, N>(d1, adesc + (64 * KBYTES >> 4) + 2 * k, bdesc + 2 * k);  // rows 64-127
            }
            wgmma_commit();
            wgmma_fence_operand(d0);
            wgmma_fence_operand(d1);
            // one group stays in flight across the loop back-edge; the stage before this one has retired and goes back
            wgmma_wait<1>();
            if (prev >= 0 && lane == 0) mbar_arrive(&L.empty_bar[prev]);
            prev = stage;
            ring ^= 1u << stage;
            if (++stage == p.stages) stage = 0;
        }
        wgmma_wait<0>();
        wgmma_fence_operand(d0);
        wgmma_fence_operand(d1);
        if (prev >= 0 && lane == 0) mbar_arrive(&L.empty_bar[prev]);
        mbar_wait(&L.acc_empty[acc], ((aphase >> acc) & 1) ^ 1);
        aphase ^= 1u << acc;
        acc_store_frag<N>(L.acc_smem, d0, 0, acc * ACC_STRIDE);
        acc_store_frag<N>(L.acc_smem, d1, 64, acc * ACC_STRIDE);
        mbar_arrive(&L.acc_full[acc]);
    }
}

template <int KIND, int N>
__device__ __forceinline__ void mma_role(const KParams& p, const SmemLayout& L, int worker, int n_workers) {
    if (KIND == 0) mma_units<KIND, 0, N>(p, L, worker, n_workers);
    else if (p.sgn == 0) mma_units<KIND, 0, N>(p, L, worker, n_workers);
    else if (p.sgn == 1) mma_units<KIND, 1, N>(p, L, worker, n_workers);
    else if (p.sgn == 2) mma_units<KIND, 2, N>(p, L, worker, n_workers);
    else mma_units<KIND, 3, N>(p, L, worker, n_workers);
}

// The tensor maps of one launch: main operands, output, residual, the low-part plane of A (3xTF32) and the projection
// source's A, B and low-part plane (KParams::kb_main); a chained launch's second weights and output (KParams::chain_n2).
struct TmaMaps {
    CUtensorMap a, b, d, r, a2, a_proj, b_proj, a2_proj, w2, z;
};

__device__ __forceinline__ void prefetch_maps(const TmaMaps& m, const KParams& p) {
    tma_prefetch_desc(&m.a);
    tma_prefetch_desc(&m.b);
    if (p.tma_store) tma_prefetch_desc(&m.d);
    if (p.res_tma) tma_prefetch_desc(&m.r);
    if (p.x3_cb) tma_prefetch_desc(&m.a2);
    if (p.kb_proj) {
        tma_prefetch_desc(&m.a_proj);
        tma_prefetch_desc(&m.b_proj);
        if (p.x3_cb_proj) tma_prefetch_desc(&m.a2_proj);
    }
}

// TMA producer of both GEMM kernels: one warp walks this CTA's work units and fills the operand ring -- A (128 rows)
// and B (bn rows) of one 128-byte K block per stage, the conv filter tap / channel walk, the two-plane 3xTF32 segments,
// the projection source and broadcast batch dims.  Runs warp-uniformly, one elected lane issues.
// CHAIN: a unit is one pixel tile in p.chain_passes passes of bn columns, and the chained convolution's weights (N / 32
// K blocks of chain_n2 rows) are loaded once, behind the operand stages, on L.w_bar.
template <bool CHAIN = false>
__device__ __forceinline__ void producer_role(const KParams& p, const TmaMaps& m, const SmemLayout& L, int worker,
                                              int n_workers) {
    uint8_t* smem = L.smem;
    uint64_t* empty_bar = L.empty_bar;
    uint32_t ring = 0;  // bit s = uses of stage s so far, mod 2
    int stage = 0;
    const uint32_t smem0 = smem_u32(smem);
    const uint32_t full0 = smem_u32(L.full_bar);
    for (int u = worker; u < p.units_total; u += n_workers) {
      for (int pass = 0; pass < (CHAIN ? p.chain_passes : 1); pass++) {
        int t, ks;
        p.d_tiles_total.divmod(u, ks, t);
        const int kb0 = ks * p.kb_per, kb1 = min(p.k_blocks, kb0 + p.kb_per);
        TileCoord tc = decode_tile(p, t);
        if (CHAIN) tc.n0 += pass * p.bn;
        // projection source: its blocks follow the main source's, one filter tap, its own channel and segment walk
        bool proj = kb0 >= p.kb_main;
        int x3 = proj ? p.x3_cb_proj : p.x3_cb;
        // conv: K block -> (filter tap, channel block), kept incrementally
        int tap = 0, cb = kb0 - p.kb_main, ky, kx;
        if (!proj) p.d_c_blocks.divmod(kb0, tap, cb);
        p.d_kw.divmod(tap, ky, kx);
        // two-plane 3xTF32: segment of the K / channel range and block inside it (kept incrementally)
        int seg = 0, sblk = p.conv ? cb : kb0;
        if (x3)
            while (sblk >= x3) {
                sblk -= x3;
                seg++;
            }
        // programmatic dependent launch: the producer is the first to touch the predecessor's output; everything
        // above (tile decode) ran while the predecessor grid was still draining
        if (u == worker && pass == 0) {
            pdl_wait();
            if (CHAIN && elect_one()) {
                const int cb2 = p.N / 32;
                const uint32_t wbytes = (uint32_t)(p.chain_n2 * KBYTES);
                uint8_t* w2 = smem + (size_t)p.stages * p.stage_bytes;
                mbar_expect_tx(L.w_bar, cb2 * wbytes);
                for (int c = 0; c < cb2; c++) tma_load_4d(w2 + c * wbytes, &m.w2, L.w_bar, 32 * c, 0, 0, 0);
            }
            if (CHAIN) __syncwarp();
        }
        for (int kb = kb0; kb < kb1; kb++) {
            if (kb == p.kb_main) {  // (never without a projection source: kb_main = k_blocks)
                proj = true;
                x3 = p.x3_cb_proj;
                cb = sblk = seg = 0;
            }
            mbar_wait(&empty_bar[stage], ((ring >> stage) & 1) ^ 1);
            if (elect_one()) {
                const uint32_t fb = full0 + stage * 8;
                mbar_expect_tx_u32(fb, p.tx_bytes);
                const uint32_t sa = smem0 + stage * p.stage_bytes;
                const uint32_t sb = sa + A_STAGE_BYTES;
                const bool lo = x3 && seg == 0;
                if (proj) {
                    const int c0 = cb * p.kelems;
                    tma_load_4d_u32(sa, lo ? &m.a2_proj : &m.a_proj, fb, x3 ? sblk * p.kelems : c0, tc.ox0 * p.s_proj,
                                    tc.oy0 * p.s_proj, tc.b0);
                    tma_load_4d_u32(sb, &m.b_proj, fb, c0, tc.n0, 0, 0);
                } else if (p.conv) {
                    const int c0 = cb * p.kelems;
                    const int ca = x3 ? sblk * p.kelems : c0;
                    tma_load_4d_u32(sa, lo ? &m.a2 : &m.a, fb, ca, tc.ox0 * p.sx - p.pl + kx * p.dx, tc.oy0 * p.sy - p.pt + ky * p.dy, tc.b0);
                    tma_load_4d_u32(sb, &m.b, fb, c0, tc.n0, tap, 0);
                } else {
                    const int k0 = kb * p.kelems;
                    const int ka = x3 ? sblk * p.kelems : k0;
                    tma_load_4d_u32(sa, lo ? &m.a2 : &m.a, fb, ka, tc.m0, p.a_bcast0 ? 0 : tc.z0, p.a_bcast1 ? 0 : tc.z1);
                    tma_load_4d_u32(sb, &m.b, fb, k0, tc.n0, p.b_bcast0 ? 0 : tc.z0, p.b_bcast1 ? 0 : tc.z1);
                }
            }
            if (x3 && ++sblk == x3) {
                sblk = 0;
                seg = seg == 2 ? 0 : seg + 1;  // (conv: the next filter tap starts over at segment 0)
            }
            if (++cb == p.c_blocks && !proj) {
                cb = 0;
                tap++;
                if (++kx == p.kw) {
                    kx = 0;
                    ky++;
                }
            }
            __syncwarp();
            ring ^= 1u << stage;
            if (++stage == p.stages) stage = 0;
        }
      }
    }
}

// Shared-memory carve-up: a fixed 1 KB block of mbarriers first, the column vectors, the accumulator tiles, operand
// stages behind them.
constexpr int SMEM_FIXED_BYTES = 1024 /*align*/ + 4096 /*barriers, column vectors*/ + ACC_SMEM_BYTES;
static_assert(ACC_SMEM_BYTES % 1024 == 0, "operand stages must stay 1024-B aligned");
static_assert(2 * ACC_STRIDE <= ACC_COLS, "two accumulator stages");

__device__ __forceinline__ SmemLayout carve_smem(uint8_t* smem_raw) {
    // 1024-B alignment required by the 128B swizzle atoms / wgmma descriptors (base_offset = 0).
    uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    SmemLayout L;
    L.full_bar = reinterpret_cast<uint64_t*>(base);
    L.empty_bar = L.full_bar + MAX_STAGES;
    L.acc_full = L.empty_bar + MAX_STAGES;
    L.acc_empty = L.acc_full + 2;
    L.res_bar = L.acc_empty + 2;  // [group][buffer], up to 4 buffers per group
    L.sk_flag = reinterpret_cast<int*>(L.res_bar + 8) + 2;  // [group]
    // column vectors of the current unit for the plain epilogues: f32 [group][128] bias (1 KB); integer kind
    // [3][group][128]: za * colsum, scale product, bias (3 KB)
    L.bias = reinterpret_cast<float*>(base + 1024);
    L.acc_smem = smem_u32(base + 4096);
    L.smem = base + 4096 + ACC_SMEM_BYTES;
    return L;
}

__device__ __forceinline__ void kernel_setup(const SmemLayout& L) {
    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    if (warp == PRODUCER_WARP) {
        // the producer initialises its own ring barriers and does NOT wait for the rest of the set-up: it only arrives
        // on a named barrier, so its first TMA is issued that much earlier
        if (lane < MAX_STAGES) {
            mbar_init(&L.full_bar[lane], 1);
            mbar_init(&L.empty_bar[lane], 4);  // one arrival per MMA warp
        }
        fence_mbar_init();
        __syncwarp();
        asm volatile("bar.arrive 15, %0;" ::"r"(NUM_THREADS) : "memory");
        return;
    }
    if (warp == 1) {
        // one barrier per lane: 0-1 accumulator full, 2-3 accumulator empty, 4-11 residual
        if (lane < 2)
            mbar_init(&L.acc_full[lane], 128);  // every thread of the MMA warpgroup stores part of the tile
        else if (lane < 4)
            mbar_init(&L.acc_empty[lane - 2], 8);  // one arrival per epilogue warp
        else if (lane < 12)
            mbar_init(&L.res_bar[lane - 4], 1);
        fence_mbar_init();
    }
    asm volatile("bar.sync 15, %0;" ::"r"(NUM_THREADS) : "memory");  // 12 warps wait, the producer warp only arrives
}

// One CTA per SM walks the work units blockIdx.x, blockIdx.x + gridDim.x, ... in every role.  E selects the epilogue
// variant (umma_epilogue.cuh).
template <int KIND, Epi E>
__global__ void __launch_bounds__(NUM_THREADS, 1)
umma_gemm_kernel(const __grid_constant__ TmaMaps m, const __grid_constant__ KParams p) {
    extern __shared__ uint8_t smem_raw[];
    const SmemLayout L = carve_smem(smem_raw);
    if (threadIdx.x == 0) prefetch_maps(m, p);
    kernel_setup(L);
    // Programmatic dependent launch: everything above (barrier init, descriptor prefetch) overlaps the tail of the
    // previous kernel in the stream; global memory is only touched after this point.
    if (threadIdx.x >> 5 != PRODUCER_WARP) pdl_wait();  // (the producer waits after its tile decode)
    pdl_launch_dependents();
    const int worker = (int)blockIdx.x, n_workers = (int)gridDim.x;
    const int warp = threadIdx.x >> 5;
    // Control warps run their loops WARP-UNIFORMLY (all 32 lanes wait on the barriers, one elected lane issues the
    // TMA / MMA instructions): addresses and descriptors then live in uniform registers instead of being moved
    // there (R2UR) for every instruction, which is what bounds a single issuing thread.
    if (warp == PRODUCER_WARP) {
        producer_role(p, m, L, worker, n_workers);
    } else if (warp < 4) {
        // ===================== MMA warpgroup: accumulators in registers, finished tiles to shared memory
        if (p.bn == 32)
            mma_role<KIND, 32>(p, L, worker, n_workers);
        else
            mma_role<KIND, 64>(p, L, worker, n_workers);
    } else {
        epilogue<KIND, E>(p, L, &m.d, &m.r, worker, n_workers);
    }
}

// ------------------------------------------------------------------------------------------
// Wide tiles: one 128 x 128 or 128 x 256 tile per work unit, for the launches that take the plain f32 epilogue
// (Epi::PlainF32, PlainF32Gelu) without split-K.  A 64-column tile cannot keep the tensor core busy: every m64nNk8 reads
// 2 KB of A from shared memory for N/2 clocks of math, and the fixed cost of a pipeline stage is as large as its
// tensor work.  A wide tile reads A once for up to 256 columns.  Its accumulator (up to 256 f32 registers per
// thread of one warpgroup) does not fit the narrow kernel's role layout, so this kernel has its own:
//   warpgroup 0    : TMA producer (warp 0; producer_role, shared with umma_gemm_kernel), registers released
//   warpgroups 1, 2: rows 0-63 / 64-127 of the tile, m64n{bn}k8 wgmma into bn/2 registers per thread, then the
//                    epilogue straight from those registers in 32-column chunks
// The epilogue is not overlapped with the next main loop; the producer keeps filling the operand ring meanwhile.
// A conv tile's 128 rows form one TMA box (tw x th x tb pixels) that does not split at row 64, so both warpgroups
// write each chunk into one shared 128-row staging buffer (two of them, alternating) stored by one TMA instruction.
// ------------------------------------------------------------------------------------------
constexpr int WIDE_THREADS = 384;
// alignment slack, two 128-row staging buffers, then mbarriers (256 B) and the unit's bias (up to 1 KB)
constexpr int WIDE_SMEM_FIXED_BYTES = 1024 + 2 * STG_BYTES + 2048;

template <int N>
__device__ __forceinline__ void wgmma_wide(float (&d)[N / 2], uint64_t adesc, uint64_t bdesc) {
    if constexpr (N == 128) wgmma_tf32_n128(d, adesc, bdesc);
    else wgmma_tf32_n256(d, adesc, bdesc);
}

// both consumer warpgroups (named barrier 1)
__device__ __forceinline__ void consumers_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

// Bytes of a chained launch's resident second weights: N / 32 K blocks of chain_n2 rows x 128 B.
__device__ __forceinline__ int chain_w_bytes(const KParams& p) { return (p.N / 32) * p.chain_n2 * KBYTES; }

// Operand stages first (1024-B aligned, like the staging buffers behind them), then a chained launch's second weights,
// the staging buffers, the small items last.
template <bool CHAIN>
__device__ __forceinline__ SmemLayout carve_wide_smem(uint8_t* smem_raw, const KParams& p) {
    uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* tail = base + (size_t)p.stages * p.stage_bytes + (CHAIN ? chain_w_bytes(p) : 0) + 2 * STG_BYTES;
    SmemLayout L;
    L.smem = base;
    L.full_bar = reinterpret_cast<uint64_t*>(tail);
    L.empty_bar = L.full_bar + MAX_STAGES;
    L.res_bar = L.empty_bar + MAX_STAGES;  // [staging buffer]
    L.w_bar = L.res_bar + 2;
    L.acc_full = L.acc_empty = nullptr;
    L.sk_flag = nullptr;
    L.bias = reinterpret_cast<float*>(tail + 256);  // up to 1.5 KB: [0, 256) the unit's columns, [256, 384) chained
    L.acc_smem = 0;
    return L;
}

// The K loop of one wide-tile consumer warpgroup into d (see wide_consumer): four k8 wgmma per 128-byte K block, one
// commit group, one group in flight across stages; a stage goes back to the producer once both warpgroups have retired
// it (8 warp arrivals).
template <int N>
__device__ __forceinline__ void wide_main_loop(const KParams& p, const SmemLayout& L, float (&d)[N / 2], int wg, int lane,
                                               int& stage, uint32_t& ring) {
    const uint32_t smem0 = smem_u32(L.smem);
#pragma unroll
    for (int i = 0; i < N / 2; i++) d[i] = 0.0f;
    int prev = -1;
    for (int kb = 0; kb < p.k_blocks; kb++) {
        mbar_wait(&L.full_bar[stage], (ring >> stage) & 1);
        wgmma_fence_operand(d);
        wgmma_fence();
        const uint32_t sa = smem0 + stage * p.stage_bytes;
        const uint64_t adesc = make_kmajor_sw128_desc(sa + wg * (64 * KBYTES));
        const uint64_t bdesc = make_kmajor_sw128_desc(sa + A_STAGE_BYTES);
#pragma unroll
        for (int k = 0; k < 4; k++) wgmma_wide<N>(d, adesc + 2 * k, bdesc + 2 * k);
        wgmma_commit();
        wgmma_fence_operand(d);
        wgmma_wait<1>();
        if (prev >= 0 && lane == 0) mbar_arrive(&L.empty_bar[prev]);
        prev = stage;
        ring ^= 1u << stage;
        if (++stage == p.stages) stage = 0;
    }
    wgmma_wait<0>();
    wgmma_fence_operand(d);
    if (prev >= 0 && lane == 0) mbar_arrive(&L.empty_bar[prev]);
}

// Columns 32k .. 32k + 31 of a wide accumulator (fragment rows row0, row0 + 8; columns 8j + 2cq + {0, 1}) through
// plain_f32_pair -- residual from the staging buffer, bias from `bias` (the chunk's 32 values), Relu -- then act4 for
// the other activations, into the 128-row, 128B-swizzled staging buffer `stg`.  `valid` = false (a chunk past N)
// stores d unchanged.
template <Epi E, int NA>
__device__ __forceinline__ void stage_chunk(float (&d)[NA], int k, uint8_t* stg, const float* bias, bool valid, bool res,
                                            int act, int row0, int sw, int cq, float alpha = 0.0f, float beta = 0.0f) {
#pragma unroll
    for (int j = 0; j < 4; j++) {  // columns 32k + 8j + 2cq + {0, 1}, rows row0 + 8h
        const int i0 = 16 * k + 4 * j;
        float2* px[2];
#pragma unroll
        for (int h = 0; h < 2; h++)
            px[h] = reinterpret_cast<float2*>(stg + (row0 + 8 * h) * 128 + (((2 * j + (cq >> 1)) ^ sw) << 4) + 8 * (cq & 1));
        if (valid) {
            const float2 bb = *reinterpret_cast<const float2*>(bias + 8 * j + 2 * cq);
#pragma unroll
            for (int h = 0; h < 2; h++) {
                uint32_t v0 = __float_as_uint(d[i0 + 2 * h]), v1 = __float_as_uint(d[i0 + 2 * h + 1]);
                float2 rr = make_float2(0.f, 0.f);
                if (res) rr = *px[h];
                plain_f32_pair(v0, v1, res, rr, bb, act == 1);
                d[i0 + 2 * h] = __uint_as_float(v0);
                d[i0 + 2 * h + 1] = __uint_as_float(v1);
            }
            if (E == Epi::PlainF32Gelu) {  // the out-of-line activation, four values per call
                const float4 g = act4(make_float4(d[i0], d[i0 + 1], d[i0 + 2], d[i0 + 3]), act, alpha, beta);
                d[i0] = g.x;
                d[i0 + 1] = g.y;
                d[i0 + 2] = g.z;
                d[i0 + 3] = g.w;
            }
        }
#pragma unroll
        for (int h = 0; h < 2; h++) *px[h] = make_float2(d[i0 + 2 * h], d[i0 + 2 * h + 1]);
    }
}

// Main loop (wide_main_loop) and epilogue of one consumer warpgroup (wg = 0: rows 0-63, 1: rows 64-127).  Epilogue:
// plain_f32_pair, then act4 for Gelu, as in the narrow kernel's PlainF32 variant -- the results equal the narrow
// kernel's.
template <Epi E, int N>
__device__ __forceinline__ void wide_consumer(const KParams& p, const SmemLayout& L, const CUtensorMap* tma_d,
                                              const CUtensorMap* tma_r, int worker, int n_workers) {
    const int t = threadIdx.x - 128;  // 0-255 over both warpgroups
    const int wg = t >> 7;
    const int lane = threadIdx.x & 31;
    const int row0 = 64 * wg + 16 * ((t & 127) >> 5) + (lane >> 2);  // this thread's fragment rows: row0, row0 + 8
    const int sw = lane >> 2;                                          // row0 & 7: 128B swizzle of both rows
    const int cq = lane & 3;                                           // columns 8j + 2cq + {0, 1} of every 8
    const bool issuer = t == 0;
    const EpilogueDesc& e = p.epi;
    uint8_t* const stg0 = L.smem + (size_t)p.stages * p.stage_bytes;
    float* const bias_s = L.bias;
    uint32_t ring = 0, rphase = 0;
    uint32_t ci = 0;  // chunks of this CTA so far: chunk ci uses staging buffer ci & 1
    int stage = 0;
    auto load_residual = [&](const TileCoord& tc, int c0, int buf) {
        uint64_t* rb = &L.res_bar[buf];
        mbar_expect_tx(rb, p.res_tx_bytes);
        const int4 x = out_coord(p, tc, c0);
        tma_load_4d(stg0 + buf * STG_BYTES, tma_r, rb, x.x, x.y, x.z, x.w);
    };
    for (int u = worker; u < p.units_total; u += n_workers) {
        {  // (the tile is decoded again after the main loop: its coordinates would hold registers through it)
            const TileCoord tc = decode_tile(p, u);  // (no split-K: a unit is a tile)
            // The unit's bias (zeros without one: x + 0 keeps the -0 -> +0 of the other epilogues).  Every reader of the
            // previous unit's values has passed the last chunk barrier; the barrier after the main loop publishes these.
            if (t < N) bias_s[t] = (e.bias_kind == 1 && tc.n0 + t < p.N) ? column_bias(e, tc.n0 + t) : 0.0f;
            if (issuer) {
                bulk_wait_read(0);  // staging buffers free
                if (p.res_tma) load_residual(tc, 0, ci & 1);
            }
        }
        float d[N / 2];
        wide_main_loop<N>(p, L, d, wg, lane, stage, ring);
        const TileCoord tc = decode_tile(p, u);
        consumers_sync();
#pragma unroll
        for (int k = 0; k < N / 32; k++, ci++) {
            const int buf = ci & 1;
            uint8_t* stg = stg0 + buf * STG_BYTES;
            const int nbase = tc.n0 + 32 * k;
            if (issuer) {
                // the previous chunk's store has read the other buffer: it takes the next residual chunk, and the
                // writes of the next chunk (after this chunk's barrier) may land in it
                bulk_wait_read(0);
                if (p.res_tma && k + 1 < N / 32) load_residual(tc, 32 * (k + 1), buf ^ 1);
            }
            if (p.res_tma) {
                mbar_wait(&L.res_bar[buf], (rphase >> buf) & 1);
                rphase ^= 1u << buf;
            }
            // (a tile may overhang N by whole chunks: the TMA store clips them)
            stage_chunk<E>(d, k, stg, bias_s + 32 * k, nbase < p.N, p.res_tma, e.act, row0, sw, cq, e.act_alpha, e.act_beta);
            fence_proxy_async();
            consumers_sync();
            if (issuer) {
                const int4 x = out_coord(p, tc, 32 * k);
                tma_store_4d(tma_d, stg, x.x, x.y, x.z, x.w);
                asm volatile("cp.async.bulk.commit_group;" ::: "memory");
            }
        }
    }
    if (issuer) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
}

// A chained unit (umma_wide_kernel with N2 > 0): one conv pixel tile x all N <= 256 columns of y = act(conv + residual
// or projection + bias), computed in 128-column passes (rows of one warpgroup: d[64]), and z = act2(y * W2 + b2) over
// N2 columns (acc2[N2 / 2]).  Each staged 32-column chunk of y is, as the 128B-swizzled 128-row buffer the TMA store
// reads, also the K-major SW128 A operand of one 32-channel K block of z: once it is visible, each warpgroup issues four
// m64nN2k8 wgmma from it (its own 64 rows) against the resident W2 block.  They run behind the next chunk's epilogue and
// retire (wgmma_wait<0> before the chunk barrier) before the buffer they read is reused: the next residual TMA load
// into it, issued after that barrier, and the writes of the chunk after next.  The issuer waits for the previous chunk's
// TMA store before the barrier too, so no chunk writes into a buffer a store still reads.  K order and epilogue equal
// those of the separate 1x1 convolution of y: z is bit-identical to it.
template <int N2>
__device__ __forceinline__ void wide_chain_consumer(const KParams& p, const SmemLayout& L, const TmaMaps& m, int worker,
                                                    int n_workers) {
    constexpr int N = 128;  // columns of a pass
    const int t = threadIdx.x - 128;
    const int wg = t >> 7;
    const int lane = threadIdx.x & 31;
    const int row0 = 64 * wg + 16 * ((t & 127) >> 5) + (lane >> 2);
    const int sw = lane >> 2;
    const int cq = lane & 3;
    const bool issuer = t == 0;
    const EpilogueDesc& e = p.epi;
    const uint32_t w2 = smem_u32(L.smem) + p.stages * p.stage_bytes;
    uint8_t* const stg0 = L.smem + (size_t)p.stages * p.stage_bytes + chain_w_bytes(p);
    float* const bias_s = L.bias;
    uint32_t ring = 0, rphase = 0;
    uint32_t ci = 0;  // chunks of this CTA so far: chunk ci uses staging buffer ci & 1
    int stage = 0;
    auto load_residual = [&](const TileCoord& tc, int c0, int buf) {
        uint64_t* rb = &L.res_bar[buf];
        mbar_expect_tx(rb, p.res_tx_bytes);
        const int4 x = out_coord(p, tc, c0);
        tma_load_4d(stg0 + buf * STG_BYTES, &m.r, rb, x.x, x.y, x.z, x.w);
    };
    // closes chunk ci in buffer stg: the other buffer's wgmma have retired and its store has been read, then the barrier
    auto chunk_barrier = [&](float (&acc2)[N2 / 2]) {
        wgmma_wait<0>();
        wgmma_fence_operand(acc2);
        if (issuer) bulk_wait_read(0);
        fence_proxy_async();
        consumers_sync();
    };
    mbar_wait(L.w_bar, 0);
    for (int u = worker; u < p.units_total; u += n_workers) {
        {
            const TileCoord tc = decode_tile(p, u);
            if (t < p.N) bias_s[t] = e.bias_kind == 1 ? column_bias(e, t) : 0.0f;
            if (t < N2) bias_s[256 + t] = p.chain_bias ? __ldg(p.chain_bias + t) : 0.0f;
            if (issuer && p.res_tma) load_residual(tc, 0, ci & 1);
        }
        float acc2[N2 / 2];
#pragma unroll
        for (int i = 0; i < N2 / 2; i++) acc2[i] = 0.0f;
        for (int pass = 0; pass < p.chain_passes; pass++) {
            float d[N / 2];
            wide_main_loop<N>(p, L, d, wg, lane, stage, ring);
            const TileCoord tc = decode_tile(p, u);
            consumers_sync();
#pragma unroll
            for (int k = 0; k < N / 32; k++) {
                const int c0 = N * pass + 32 * k;
                if (c0 >= p.N) break;  // (N % 32 == 0: whole chunks; uniform over the CTA)
                const int buf = ci & 1;
                uint8_t* stg = stg0 + buf * STG_BYTES;
                if (p.res_tma) {
                    mbar_wait(&L.res_bar[buf], (rphase >> buf) & 1);
                    rphase ^= 1u << buf;
                }
                stage_chunk<Epi::PlainF32>(d, k, stg, bias_s + c0, true, p.res_tma, e.act, row0, sw, cq);
                chunk_barrier(acc2);
                if (issuer) {
                    const int4 x = out_coord(p, tc, c0);
                    tma_store_4d(&m.d, stg, x.x, x.y, x.z, x.w);
                    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
                    if (p.res_tma && c0 + 32 < p.N) load_residual(tc, c0 + 32, buf ^ 1);
                }
                wgmma_fence();
                const uint64_t adesc = make_kmajor_sw128_desc(smem_u32(stg) + wg * (64 * KBYTES));
                const uint64_t bdesc = make_kmajor_sw128_desc(w2 + (c0 / 32) * (N2 * KBYTES));
#pragma unroll
                for (int kk = 0; kk < 4; kk++) {
                    if constexpr (N2 == 64) wgmma_tf32_n64(acc2, adesc + 2 * kk, bdesc + 2 * kk);
                    else wgmma_tf32_n128(acc2, adesc + 2 * kk, bdesc + 2 * kk);
                }
                wgmma_commit();
                wgmma_fence_operand(acc2);
                ci++;
            }
        }
        wgmma_wait<0>();
        wgmma_fence_operand(acc2);
        const TileCoord tc = decode_tile(p, u);
#pragma unroll
        for (int k = 0; k < N2 / 32; k++, ci++) {
            uint8_t* stg = stg0 + (ci & 1) * STG_BYTES;
            stage_chunk<Epi::PlainF32>(acc2, k, stg, bias_s + 256 + 32 * k, true, false, p.chain_act, row0, sw, cq);
            chunk_barrier(acc2);
            if (issuer) {
                tma_store_4d(&m.z, stg, 32 * k, tc.ox0, tc.oy0, tc.b0);
                asm volatile("cp.async.bulk.commit_group;" ::: "memory");
            }
        }
    }
    if (issuer) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
}

// CHAIN_N2 > 0: the chained launches (wide_chain_consumer), plain f32 epilogue only
template <Epi E, int CHAIN_N2 = 0>
__global__ void __launch_bounds__(WIDE_THREADS, 1)
umma_wide_kernel(const __grid_constant__ TmaMaps m, const __grid_constant__ KParams p) {
    extern __shared__ uint8_t smem_raw[];
    const SmemLayout L = carve_wide_smem<(CHAIN_N2 > 0)>(smem_raw, p);
    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
        prefetch_maps(m, p);
        if constexpr (CHAIN_N2 > 0) {
            tma_prefetch_desc(&m.w2);
            tma_prefetch_desc(&m.z);
        }
    }
    if (warp == 1) {
        if (lane < MAX_STAGES) {
            mbar_init(&L.full_bar[lane], 1);
            mbar_init(&L.empty_bar[lane], 8);  // one arrival per consumer warp
        } else if (lane < MAX_STAGES + (CHAIN_N2 > 0 ? 3 : 2)) {
            mbar_init(&L.res_bar[lane - MAX_STAGES], 1);  // (chained: + L.w_bar)
        }
        fence_mbar_init();
    }
    __syncthreads();
    // Programmatic dependent launch: the set-up above overlaps the tail of the previous kernel in the stream; global
    // memory is only touched after this point (the producer waits after its first tile decode).
    if (warp >= 4) pdl_wait();
    pdl_launch_dependents();
    if (warp < 4) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 56;");
        if (warp == 0) producer_role<(CHAIN_N2 > 0)>(p, m, L, (int)blockIdx.x, (int)gridDim.x);
    } else {
        asm volatile("setmaxnreg.inc.sync.aligned.u32 224;");
        if constexpr (CHAIN_N2 > 0) {
            wide_chain_consumer<CHAIN_N2>(p, L, m, (int)blockIdx.x, (int)gridDim.x);
        } else {
            // (Gelu: 128 columns only -- the out-of-line act4 calls would spill around 128 live accumulators per thread)
            if (E == Epi::PlainF32Gelu || p.bn == 128)
                wide_consumer<E, 128>(p, L, &m.d, &m.r, (int)blockIdx.x, (int)gridDim.x);
            else
                wide_consumer<E, 256>(p, L, &m.d, &m.r, (int)blockIdx.x, (int)gridDim.x);
        }
    }
}

}  // namespace rtb
