// Streaming attention for q_seq >= 2 on wgmma (the ONNX Attention operator's prefill: causal, right-padded KV cache,
// grouped-query heads): one CTA per (batch, query head, 64-query tile) computes
//     O = softmax(scale * Q K^T + mask, masked keys -> -inf, NaN -> 0) V
// over key tiles streamed through a two-stage TMA ring, without the scores ever leaving the SM:
//   warp 4, TMA: the Q tile once, then per key tile the K tile and the V tile (transposed value tensor: V^T tiles as
//       they are; natural value tensor: V tiles, transposed below) -> shared memory, 128B-swizzled K-major
//   warps 0-3 (one warpgroup), per key tile:
//       3xTF32: the low parts lo = x - hi (hi = x with the low 13 mantissa bits cleared, what kind::tf32 reads) of the
//           K and V tiles (and once of Q) into shared memory; natural V: the V^T tile written from the V tile
//       wgmma tf32: S = Q K^T (3xTF32: lo*hi, then hi*lo, then hi*hi over the whole head, small terms first)
//       online softmax on the accumulator fragment: scale, + mask, masked keys -> -inf, running row max (from
//           -FLT_MAX, so an all -inf tile gives 0, not NaN) and the rescale of the running sum and output by
//           reduced_range_exp(old max - new max); P = reduced_range_exp(z - max) -> shared memory as the A operand
//       wgmma tf32: O += P V (3xTF32 as above) in registers
//   O / row sum (NaN of a fully masked row flushed to 0) -> global.
// Key tiles wholly above the causal diagonal or past the valid length are neither loaded nor multiplied, and in the tile
// that holds the last valid key the value rows past it are zeroed, so a NaN or inf left in a padded cache never reaches
// the output (as in the decode kernel); the launch
// depends on shapes only (valid lengths are read on the device), so the call can be captured in a CUDA graph.  No
// atomics and no split over CTAs: every output element is written once, and repeated runs are bit-identical.
#include <cuda.h>
#include <cuda_runtime.h>

#include <cfloat>
#include <cstdint>
#include <cstdlib>
#include <cstring>

#include "attn_prefill.h"
#include "math.cuh"
#include "ptx.cuh"
#include "tf32_split.cuh"

namespace rtb {

namespace {

constexpr int AP_THREADS = 160;  // warps 0-3: wgmma warpgroup (rows 16 w + lane / 4 + {0, 8} of the tile); warp 4: TMA
constexpr int BM = 64;           // query rows per CTA (one wgmma M)
constexpr int NS = 2;            // K / V stages

// Shared-memory plan of one (head size, mode).  Head size 128 in 3xTF32 streams 32-key tiles: with 64-key tiles the
// two stages plus the low parts of Q, K, V and P would not fit in 227 KB.
template <int DH, bool X3>
struct Cfg {
    static constexpr int BN = (DH == 128 && X3) ? 32 : 64;  // keys per tile
    static constexpr uint32_t QT = BM * DH * 4;            // Q: DH / 32 sub-tiles [64 rows x 128 B]
    static constexpr uint32_t KT = BN * DH * 4;            // K: DH / 32 sub-tiles [BN rows x 128 B]
    static constexpr uint32_t VT = BN * DH * 4;            // V^T: BN / 32 sub-tiles [DH rows x 128 B] (natural V: as K)
    static constexpr uint32_t PT = BM * BN * 4;            // P: BN / 32 sub-tiles [64 rows x 128 B]
    static constexpr uint32_t LO = X3 ? 1 : 0;
    static constexpr size_t SMEM = 1024 /* alignment */ + 1024 /* barriers */ + QT * (1 + LO) + NS * (KT + VT) +
                                   KT * LO + VT * (1 + LO) + PT * (1 + LO);
    static_assert(SMEM <= 227 * 1024, "shared memory");
};

struct AttnPrefillParams {
    int heads, group, q_seq, kv_seq, q_tiles;
    int v_natural, causal, window;
    const int32_t* len;
    const float* mask;
    long long m_b, m_h, m_s;
    float scale;
    float* out;
    long long o_b, o_h, o_s;
    // MultiHeadAttention (attn_prefill_mha_kernel only; see AttnPrefillMha)
    int c_off;
    float fill;
    const int32_t* kpm;
    long long kpm_b, m_t;
    const float* v_rows;
    long long v_b, v_h, v_t;
};

template <int N>
__device__ __forceinline__ void mma_tf32(float (&d)[N / 2], uint64_t a, uint64_t b) {
    if constexpr (N == 32) wgmma_tf32_n32(d, a, b);
    else if constexpr (N == 64) wgmma_tf32_n64(d, a, b);
    else wgmma_tf32_n128(d, a, b);
}

// D[64 x N] += A[64 x 32 KB] . B[N x 32 KB]^T over KB sub-tiles of 32 K-elements (K-major, 128B-swizzled; A sub-tiles
// a_step bytes apart, B sub-tiles b_step bytes apart).  3xTF32: the three passes a_lo*b, a*b_lo, a*b, each over all K.
template <int N, int KB, bool X3>
__device__ __forceinline__ void mma_block(float (&d)[N / 2], const uint8_t* a, const uint8_t* a_lo, uint32_t a_step, const uint8_t* b,
                                          const uint8_t* b_lo, uint32_t b_step) {
    wgmma_fence_operand(d);
    wgmma_fence();
#pragma unroll
    for (int pass = X3 ? 0 : 2; pass < 3; pass++) {
        const uint8_t* pa = pass == 0 ? a_lo : a;
        const uint8_t* pb = pass == 1 ? b_lo : b;
#pragma unroll
        for (int kb = 0; kb < KB; kb++) {
            const uint64_t ad = make_kmajor_sw128_desc(smem_u32(pa + kb * a_step)), bd = make_kmajor_sw128_desc(smem_u32(pb + kb * b_step));
#pragma unroll
            for (int k = 0; k < 4; k++) mma_tf32<N>(d, ad + 2 * k, bd + 2 * k);
        }
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_operand(d);
}

// byte offset of element (row, col) in a stack of K-major 128B-swizzled sub-tiles of 32 columns and `rows` rows
__device__ __forceinline__ uint32_t sw_off(int row, int col, int rows) {
    return (uint32_t)((col >> 5) * rows * 128 + row * 128 + ((((col & 31) >> 2) ^ (row & 7)) << 4) + ((col & 3) << 2));
}

// MHA: the MultiHeadAttention scores (attn_prefill_mha_kernel).  Masked keys (causal, key_padding_mask) score p.fill
// instead of -inf, the causal diagonal is offset by p.c_off, the mask's key stride is p.m_t, and the key tiles above
// every row's diagonal, skipped as usual, are added back afterwards as n_tail keys of score fill (a row's weight of
// them is e^(fill - m): only when that is non-zero somewhere in the CTA is their value sum read, with plain loads).
// Without MHA this is the Attention / GroupQueryAttention kernel exactly as before.
template <int DH, bool X3, bool MHA>
__device__ __forceinline__ void attn_prefill_body(const CUtensorMap& tma_q, const CUtensorMap& tma_k, const CUtensorMap& tma_v,
                                                  const AttnPrefillParams& p) {
    using C = Cfg<DH, X3>;
    constexpr int BN = C::BN;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* full = reinterpret_cast<uint64_t*>(base);  // [NS]: K and V tiles of the stage landed
    uint64_t* empty = full + NS;                         // [NS]: the 4 MMA warps are done with the stage
    uint64_t* bar_q = empty + NS;
    uint8_t* sq = base + 1024;
    uint8_t* sq_lo = sq + C::QT;
    uint8_t* sk = sq_lo + C::QT * C::LO;  // [NS] K tiles
    uint8_t* sv = sk + NS * C::KT;        // [NS] V^T (or natural V) tiles
    uint8_t* sk_lo = sv + NS * C::VT;
    uint8_t* svt = sk_lo + C::KT * C::LO;  // V^T written from a natural V tile
    uint8_t* sv_lo = svt + C::VT;
    uint8_t* sp = sv_lo + C::VT * C::LO;
    uint8_t* sp_lo = sp + C::PT;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int u = blockIdx.x;
    // the longest causal query tiles first (the grid's tail is then made of short ones)
    const int qt = p.q_tiles - 1 - u % p.q_tiles, h = (u / p.q_tiles) % p.heads, b = u / (p.q_tiles * p.heads);
    const int hk = h / p.group;
    const int q0 = qt * BM;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tma_q);
        tma_prefetch_desc(&tma_k);
        tma_prefetch_desc(&tma_v);
        for (int s = 0; s < NS; s++) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], 4);
        }
        mbar_init(bar_q, 1);
        if constexpr (MHA) *reinterpret_cast<volatile int*>(bar_q + 1) = 0;  // the causal tail's flag
        fence_mbar_init();
    }
    __syncthreads();
    pdl_wait();
    pdl_launch_dependents();

    // keys [0, lim) exist for every row; a causal row s sees keys [0, s + off]
    const int lim = p.len ? min(max(__ldg(p.len + b), 0), p.kv_seq) : p.kv_seq;
    const int off = MHA ? p.c_off : (p.len ? lim - p.q_seq : 0);
    int kend = p.causal ? min(lim, min(q0 + BM, p.q_seq) + off) : lim;
    kend = max(kend, 0);
    const int ntiles = (kend + BN - 1) / BN;
    // sliding window: row s sees no key below s + off + 1 - window; tiles wholly below the first row's window are skipped
    const int jlo = p.window > 0 ? min(max(q0 + off + 1 - p.window, 0) / BN, ntiles) : 0;

    if (warp == 4) {
        if (elect_one()) {
            mbar_expect_tx(bar_q, C::QT);
#pragma unroll
            for (int c = 0; c < DH / 32; c++) tma_load_4d(sq + c * BM * 128, &tma_q, bar_q, c * 32, q0, h, b);
            for (int j = jlo; j < ntiles; j++) {
                const int it = j - jlo, s = it % NS;
                if (it >= NS) mbar_wait(&empty[s], ((it / NS) - 1) & 1);
                mbar_expect_tx(&full[s], C::KT + C::VT);
                uint8_t* dk = sk + s * C::KT;
                uint8_t* dv = sv + s * C::VT;
#pragma unroll
                for (int c = 0; c < DH / 32; c++) tma_load_4d(dk + c * BN * 128, &tma_k, &full[s], c * 32, j * BN, hk, b);
                if (p.v_natural) {
#pragma unroll
                    for (int c = 0; c < DH / 32; c++) tma_load_4d(dv + c * BN * 128, &tma_v, &full[s], c * 32, j * BN, hk, b);
                } else {
#pragma unroll
                    for (int c = 0; c < BN / 32; c++) tma_load_4d(dv + c * DH * 128, &tma_v, &full[s], j * BN + c * 32, 0, hk, b);
                }
            }
        }
        return;
    }

    const int tid = threadIdx.x;
    const int g = lane >> 2, t = lane & 3;
    const int rl0 = 16 * warp + g;  // tile rows of this thread: rl0, rl0 + 8
    const int row0 = q0 + rl0, row1 = row0 + 8;
    const int lim0 = p.causal ? min(lim, row0 + off + 1) : lim;
    const int lim1 = p.causal ? min(lim, row1 + off + 1) : lim;
    const int lo0 = p.window > 0 ? row0 + off + 1 - p.window : 0, lo1 = p.window > 0 ? row1 + off + 1 - p.window : 0;
    const float* mrow0 = nullptr;
    const float* mrow1 = nullptr;
    if (p.mask) {
        const float* mh = p.mask + (long long)b * p.m_b + (long long)h * p.m_h;
        mrow0 = mh + (long long)min(row0, p.q_seq - 1) * p.m_s;
        mrow1 = mh + (long long)min(row1, p.q_seq - 1) * p.m_s;
    }
    const int32_t* krow = MHA && p.kpm ? p.kpm + (long long)b * p.kpm_b : nullptr;

    float o[DH / 2];
#pragma unroll
    for (int i = 0; i < DH / 2; i++) o[i] = 0.0f;
    float m0 = -FLT_MAX, m1 = -FLT_MAX, l0 = 0.0f, l1 = 0.0f;

    mbar_wait(bar_q, 0);
    if constexpr (X3) split_lo(sq_lo, sq, C::QT, tid);

    for (int j = jlo; j < ntiles; j++) {
        const int s = (j - jlo) % NS;
        const uint8_t* tk = sk + s * C::KT;
        const uint8_t* tv = sv + s * C::VT;
        mbar_wait(&full[s], ((j - jlo) / NS) & 1);
        // keys [nv, BN) of the tile lie at or past the valid length (only in the tile of key lim - 1): their value rows
        // are zeroed below, as a decode step never reads them -- P = 0 there, but 0 * NaN or 0 * inf would be NaN
        const int nv = min(lim - j * BN, BN);
        if (X3 || p.v_natural || nv < BN) {
            // every warp's products of the previous tile have completed before its operands are overwritten
            if (j > jlo) asm volatile("bar.sync 1, 128;" ::: "memory");
            if constexpr (X3) split_lo(sk_lo, tk, C::KT, tid);
            if (p.v_natural) {
                // V tile (key row, d column) -> V^T tile (d row, key column); 32 lanes write 32 keys of one row of V^T
                for (int i = tid; i < BN * DH / 4; i += 128) {
                    const int key = i % BN, d = 4 * (i / BN);
                    float4 x = *reinterpret_cast<const float4*>(tv + sw_off(key, d, BN));
                    if (key >= nv) x = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
                    const float e[4] = {x.x, x.y, x.z, x.w};
#pragma unroll
                    for (int q = 0; q < 4; q++) {
                        *reinterpret_cast<float*>(svt + sw_off(d + q, key, DH)) = e[q];
                        if constexpr (X3) *reinterpret_cast<float*>(sv_lo + sw_off(d + q, key, DH)) = tf32_lo(e[q]);
                    }
                }
                tv = svt;
            } else {
                if (nv < BN) {
                    // the V^T tile's columns of keys past the valid length -> 0 (in the stage buffer: TMA rewrites it
                    // only after this tile's products, and the proxy fence below orders these stores before them)
                    for (int i = tid; i < BN * DH; i += 128) {
                        const int key = i % BN, d = i / BN;
                        if (key >= nv) *reinterpret_cast<float*>(sv + s * C::VT + sw_off(d, key, DH)) = 0.0f;
                    }
                    if constexpr (X3) asm volatile("bar.sync 1, 128;" ::: "memory");
                }
                if constexpr (X3) split_lo(sv_lo, tv, C::VT, tid);
            }
        }
        fence_proxy_async();  // the tensor core reads the bytes written above through the async proxy
        asm volatile("bar.sync 1, 128;" ::: "memory");

        // ---- S = Q K^T
        float sc[BN / 2];
#pragma unroll
        for (int i = 0; i < BN / 2; i++) sc[i] = 0.0f;
        mma_block<BN, DH / 32, X3>(sc, sq, sq_lo, BM * 128, tk, sk_lo, BN * 128);

        // ---- online softmax: element i of the fragment is row rl0 + 8 ((i >> 1) & 1), key column 8 (i >> 2) + 2 t + (i & 1)
        const int key0 = j * BN + 2 * t;
        float mx0 = m0, mx1 = m1;
#pragma unroll
        for (int i = 0; i < BN / 2; i++) {
            const bool r1 = (i >> 1) & 1;
            const int key = key0 + 8 * (i >> 2) + (i & 1);
            float z = __fmul_rn(sc[i], p.scale);
            if constexpr (MHA) {
                // absent (beyond the keys: tile padding) -> -inf; masked (causal, padding) -> fill, replacing the bias
                const bool exists = key < lim;
                const bool vis = key < (r1 ? lim1 : lim0) && (!krow || __ldg(krow + min(key, lim - 1)) != 0);
                if (mrow0 && exists) z = __fadd_rn(z, __ldg((r1 ? mrow1 : mrow0) + (long long)key * p.m_t));
                z = !exists ? -INFINITY : vis ? z : p.fill;
            } else {
                const bool ok = key < (r1 ? lim1 : lim0) && key >= (r1 ? lo1 : lo0);
                if (mrow0 && ok) z = __fadd_rn(z, __ldg((r1 ? mrow1 : mrow0) + key));
                z = ok ? z : -INFINITY;
            }
            sc[i] = z;
            if (r1) mx1 = fmaxf(mx1, z);
            else mx0 = fmaxf(mx0, z);
        }
        mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
        mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
        mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
        mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
        const float a0 = reduced_range_exp(__fsub_rn(m0, mx0)), a1 = reduced_range_exp(__fsub_rn(m1, mx1));
        m0 = mx0;
        m1 = mx1;
        l0 = __fmul_rn(l0, a0);
        l1 = __fmul_rn(l1, a1);
#pragma unroll
        for (int i = 0; i < BN / 2; i += 2) {
            const bool r1 = (i >> 1) & 1;
            float e0 = __fsub_rn(sc[i], r1 ? mx1 : mx0), e1 = __fsub_rn(sc[i + 1], r1 ? mx1 : mx0);
            reduced_range_exp_x2(e0, e1);
            if (r1) l1 = __fadd_rn(__fadd_rn(l1, e0), e1);
            else l0 = __fadd_rn(__fadd_rn(l0, e0), e1);
            const int rl = rl0 + (r1 ? 8 : 0), col = 8 * (i >> 2) + 2 * t;
            *reinterpret_cast<float2*>(sp + sw_off(rl, col, BM)) = make_float2(e0, e1);
            if constexpr (X3) *reinterpret_cast<float2*>(sp_lo + sw_off(rl, col, BM)) = make_float2(tf32_lo(e0), tf32_lo(e1));
        }
        fence_proxy_async();
        asm volatile("bar.sync 1, 128;" ::: "memory");  // all of P written

        // ---- O = O * alpha + P V
        if constexpr (X3) {
            // the tile's product from a zero accumulator, added to O in rounded-to-nearest f32: the tensor core's own
            // accumulation does not round to nearest, and over thousands of keys its error alone would exceed the
            // f32-grade bound of this mode
            float pv[DH / 2];
#pragma unroll
            for (int i = 0; i < DH / 2; i++) pv[i] = 0.0f;
            mma_block<DH, BN / 32, X3>(pv, sp, sp_lo, BM * 128, tv, sv_lo, DH * 128);
#pragma unroll
            for (int i = 0; i < DH / 2; i++) o[i] = __fmaf_rn(o[i], ((i >> 1) & 1) ? a1 : a0, pv[i]);
        } else {
#pragma unroll
            for (int i = 0; i < DH / 2; i++) o[i] = __fmul_rn(o[i], ((i >> 1) & 1) ? a1 : a0);
            mma_block<DH, BN / 32, X3>(o, sp, sp_lo, BM * 128, tv, sv_lo, DH * 128);
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[s]);
    }

    // ---- O / row sum (the quad's partial sums, in a fixed order) -> global
    l0 = __fadd_rn(l0, __shfl_xor_sync(0xffffffffu, l0, 1));
    l0 = __fadd_rn(l0, __shfl_xor_sync(0xffffffffu, l0, 2));
    l1 = __fadd_rn(l1, __shfl_xor_sync(0xffffffffu, l1, 1));
    l1 = __fadd_rn(l1, __shfl_xor_sync(0xffffffffu, l1, 2));
    if constexpr (MHA) {
        // the causal tail [kt, kv_seq): keys of score fill for every row of the tile, never loaded
        const int kt = min(ntiles * BN, lim), n_tail = lim - kt;
        if (n_tail > 0) {  // (uniform over the CTA)
            volatile int* flag = reinterpret_cast<volatile int*>(bar_q + 1);
            const float mn0 = fmaxf(m0, p.fill), mn1 = fmaxf(m1, p.fill);
            const float e0 = reduced_range_exp(__fsub_rn(p.fill, mn0)), e1 = reduced_range_exp(__fsub_rn(p.fill, mn1));
            if (e0 != 0.0f || e1 != 0.0f) *flag = 1;
            asm volatile("bar.sync 1, 128;" ::: "memory");  // every product done (P is free) and every row's flag set
            if (*flag) {
                float* vsum = reinterpret_cast<float*>(sp);
                if (tid < DH) {
                    const float* vr = p.v_rows + (long long)b * p.v_b + (long long)hk * p.v_h + tid;
                    float acc = 0.0f;
                    for (int key = kt; key < lim; key++) acc = __fadd_rn(acc, __ldg(vr + (long long)key * p.v_t));
                    vsum[tid] = acc;
                }
                asm volatile("bar.sync 1, 128;" ::: "memory");
                const float a0 = reduced_range_exp(__fsub_rn(m0, mn0)), a1 = reduced_range_exp(__fsub_rn(m1, mn1));
                l0 = __fadd_rn(__fmul_rn(l0, a0), __fmul_rn((float)n_tail, e0));
                l1 = __fadd_rn(__fmul_rn(l1, a1), __fmul_rn((float)n_tail, e1));
#pragma unroll
                for (int i = 0; i < DH / 2; i++) {
                    const bool r1 = (i >> 1) & 1;
                    const float vs = vsum[8 * (i >> 2) + 2 * t + (i & 1)];
                    o[i] = __fadd_rn(__fmul_rn(o[i], r1 ? a1 : a0), __fmul_rn(r1 ? e1 : e0, vs));
                }
            }
        }
    }
    const float inv0 = __fdiv_rn(1.0f, l0), inv1 = __fdiv_rn(1.0f, l1);
    float* ob = p.out + (long long)b * p.o_b + (long long)h * p.o_h;
#pragma unroll
    for (int i = 0; i < DH / 2; i += 2) {
        const bool r1 = (i >> 1) & 1;
        const int row = r1 ? row1 : row0;
        if (row >= p.q_seq) continue;
        float y0 = __fmul_rn(o[i], r1 ? inv1 : inv0), y1 = __fmul_rn(o[i + 1], r1 ? inv1 : inv0);
        y0 = y0 != y0 ? 0.0f : y0;  // a fully masked row: 0 / 0
        y1 = y1 != y1 ? 0.0f : y1;
        *reinterpret_cast<float2*>(ob + (long long)row * p.o_s + 8 * (i >> 2) + 2 * t) = make_float2(y0, y1);
    }
}

template <int DH, bool X3>
__global__ void __launch_bounds__(AP_THREADS, 1)
attn_prefill_kernel(const __grid_constant__ CUtensorMap tma_q, const __grid_constant__ CUtensorMap tma_k,
                    const __grid_constant__ CUtensorMap tma_v, const __grid_constant__ AttnPrefillParams p) {
    attn_prefill_body<DH, X3, false>(tma_q, tma_k, tma_v, p);
}

template <int DH, bool X3>
__global__ void __launch_bounds__(AP_THREADS, 1)
attn_prefill_mha_kernel(const __grid_constant__ CUtensorMap tma_q, const __grid_constant__ CUtensorMap tma_k,
                        const __grid_constant__ CUtensorMap tma_v, const __grid_constant__ AttnPrefillParams p) {
    attn_prefill_body<DH, X3, true>(tma_q, tma_k, tma_v, p);
}

template <int DH, bool X3>
rten_status launch_cfg(rten_ctx* ctx, const AttnPrefillLaunch& L, const AttnPrefillParams& p) {
    using C = Cfg<DH, X3>;
    uint32_t ones[4] = {1, 1, 1, 1};
    const uint32_t qbox[4] = {32u, (uint32_t)BM, 1u, 1u}, kbox[4] = {32u, (uint32_t)C::BN, 1u, 1u};
    const uint32_t vbox[4] = {32u, (uint32_t)(L.v_natural ? C::BN : DH), 1u, 1u};
    CUtensorMap mq, mk, mv;
    if (!encode_map(ctx, &mq, L.q, 4, true, qbox, ones) || !encode_map(ctx, &mk, L.k, 4, true, kbox, ones) ||
        !encode_map(ctx, &mv, L.v, 4, true, vbox, ones))
        return fail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "prefill attention: the tensor maps of query, key or value could not be encoded");
    auto kernel = L.mha ? attn_prefill_mha_kernel<DH, X3> : attn_prefill_kernel<DH, X3>;
    return launch(ctx, "prefill attention launch", kernel,
                  {(unsigned)((long long)L.B * L.q_heads * p.q_tiles), AP_THREADS, C::SMEM, (int)C::SMEM, true}, mq, mk, mv, p);
}

}  // namespace

bool attn_prefill_supported(const AttnPrefillLaunch& L) {
    if (L.dh != 64 && L.dh != 128) return false;
    if (L.window < 0) return false;
    if (L.B < 1 || L.q_heads < 1 || L.kv_heads < 1 || L.q_heads % L.kv_heads || L.q_seq < 1 || L.kv_seq < 1) return false;
    if ((long long)L.B * L.q_heads * ((L.q_seq + BM - 1) / BM) > 0x7fffffffll) return false;
    auto al16 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
    if (!al16(L.out) || (L.o_b & 3) || (L.o_h & 3) || (L.o_s & 3)) return false;
    if (L.mask && (reinterpret_cast<uintptr_t>(L.mask) & 3)) return false;
    if (L.mha && (L.window || L.len || !L.v_natural || !L.mha->v_rows || L.mha->causal_offset < 0)) return false;
    return tma_compatible(L.q, 4, 4) && tma_compatible(L.k, 4, 4) && tma_compatible(L.v, 4, 4);
}

rten_status launch_attn_prefill(rten_ctx* ctx, const AttnPrefillLaunch& L) {
    AttnPrefillParams p;
    memset(&p, 0, sizeof(p));
    p.heads = L.q_heads;
    p.group = L.q_heads / L.kv_heads;
    p.q_seq = L.q_seq;
    p.kv_seq = L.kv_seq;
    p.q_tiles = (L.q_seq + BM - 1) / BM;
    p.v_natural = L.v_natural ? 1 : 0;
    p.causal = L.causal ? 1 : 0;
    p.window = L.window;
    p.len = L.len;
    p.mask = L.mask;
    p.m_b = L.m_b;
    p.m_h = L.m_h;
    p.m_s = L.m_s;
    p.scale = L.scale;
    p.out = L.out;
    p.o_b = L.o_b;
    p.o_h = L.o_h;
    p.o_s = L.o_s;
    if (L.mha) {
        const AttnPrefillMha& M = *L.mha;
        p.c_off = M.causal_offset;
        p.fill = M.fill;
        p.kpm = M.kpm;
        p.kpm_b = M.kpm_b;
        p.m_t = M.m_t;
        p.v_rows = M.v_rows;
        p.v_b = M.v_b;
        p.v_h = M.v_h;
        p.v_t = M.v_t;
    }
    if (L.dh == 64) return L.x3 ? launch_cfg<64, true>(ctx, L, p) : launch_cfg<64, false>(ctx, L, p);
    return L.x3 ? launch_cfg<128, true>(ctx, L, p) : launch_cfg<128, false>(ctx, L, p);
}

}  // namespace rtb
