// Epilogue warps of umma_gemm_kernel (umma_kernel.cuh): one driver owns the protocol -- the unit walk and accumulator
// phases, split-K publish / ownership / sum, the residual ring, staging, TMA store (or the generic variant's direct
// stores) and the final drain -- and each variant supplies only its arithmetic:
//   Generic        every zero-point, scale, range, split-K and edge case of the operator family; rolled slow path
//   Fast(Gelu)     every chunk on the register path (TMA store, N % 32 == 0, vector-addressable column vectors)
//   PlainF32(Gelu) alpha = 1, optional column bias, residual with r_scale = 1, no range: column vector in shared memory
//   PlainI8(Gelu)  the *ToFloat operators with a scalar activation zero point and symmetric weights, no split-K
// Included by umma_kernel.cuh.
#pragma once

namespace rtb {

// Position of accumulator row r of a tile in the output: plain (z0, z1, row m); conv (image b, x, y) in the order of
// EpilogueDesc's strides, and m = the pixel index.  ok = the row lies inside the output.
struct RowPos {
    bool ok;
    int z0, z1, y, m;
};

__device__ __forceinline__ RowPos decode_row(const KParams& p, const TileCoord& tc, int r) {
    RowPos w;
    if (p.conv) {
        int xi, r2, yi, bi;
        p.d_tw.divmod(r, r2, xi);
        p.d_th.divmod(r2, bi, yi);
        w.z0 = tc.b0 + bi;
        w.z1 = tc.ox0 + xi;
        w.y = tc.oy0 + yi;
        w.ok = (bi < p.tb) && (w.z1 < p.OW) && (w.y < p.OH) && (w.z0 < p.Bn);
        w.m = (w.z0 * p.OH + w.y) * p.OW + w.z1;
    } else {
        w.z0 = tc.z0;
        w.z1 = tc.z1;
        w.y = w.m = tc.m0 + r;
        w.ok = w.m < p.M;
    }
    return w;
}

// 16-byte chunk c (columns 4c .. 4c + 3) and word j of a thread's 128-byte staged row (chunks XOR-swizzled by row & 7)
__device__ __forceinline__ uint8_t* staged_chunk(uint8_t* rowp, int sw, int c) { return rowp + ((c ^ sw) << 4); }
__device__ __forceinline__ uint32_t* staged_word(uint8_t* rowp, int sw, int j) {
    return reinterpret_cast<uint32_t*>(staged_chunk(rowp, sw, j >> 2)) + (j & 3);
}

// named barrier of one epilogue group (128 threads)
__device__ __forceinline__ void group_sync(int grp) { asm volatile("bar.sync %0, 128;" ::"r"(1 + grp) : "memory"); }

// The activation (any code above Relu) of four f32 bit patterns in place (the out-of-line act4)
__device__ __forceinline__ void act4_bits(uint32_t& a, uint32_t& b, uint32_t& c, uint32_t& d, const EpilogueDesc& e) {
    const float4 g = act4(make_float4(__uint_as_float(a), __uint_as_float(b), __uint_as_float(c), __uint_as_float(d)),
                          e.act, e.act_alpha, e.act_beta);
    a = __float_as_uint(g.x);
    b = __float_as_uint(g.y);
    c = __float_as_uint(g.z);
    d = __float_as_uint(g.w);
}

// Hooks every variant inherits, doing nothing: unit() runs before the accumulator wait, ready() after it, row() once
// the tile is owned, math() on a chunk's registers, staged() on the staged chunk, finish() after the last unit.
struct EpiBase {
    static constexpr bool kSplitK = true;        // the variant runs split-K launches
    static constexpr bool kDirectStore = false;  // ... and launches whose output TMA cannot store
    bool row_ok = true;
    __device__ __forceinline__ void unit(const KParams&, int) {}
    __device__ __forceinline__ void ready(int) {}
    __device__ __forceinline__ void row(const KParams&, const TileCoord&, int) {}
    __device__ __forceinline__ void staged(const KParams&, int, uint8_t*, int) {}
    __device__ __forceinline__ void finish(const EpilogueDesc&) {}
};

// the warp's running (min, max) of the output (EpilogueDesc::range), folded into the launch-wide range at the end
struct RangedEpi : EpiBase {
    float rg_lo = INFINITY, rg_hi = -INFINITY;
    __device__ __forceinline__ void fold(float x) {
        rg_lo = fminf(rg_lo, x);
        rg_hi = fmaxf(rg_hi, x);
    }
    __device__ __forceinline__ void finish(const EpilogueDesc& e) {
        if (e.range) range_commit(e.range, rg_lo, rg_hi);
    }
};

template <int KIND>
struct GenericEpi : RangedEpi {
    static constexpr bool kDirectStore = true;
    long long d_off = 0, r_off = 0;  // element offsets of this thread's output / residual row
    float row_bias = 0.0f;
    int za_v = 0, rs_v = 0;
    bool fast = false;  // this chunk took the register path
    __device__ GenericEpi(const KParams&, const SmemLayout&, int) {}

    __device__ __forceinline__ void row(const KParams& p, const TileCoord& tc, int r) {
        const EpilogueDesc& e = p.epi;
        const RowPos w = decode_row(p, tc, r);
        row_ok = w.ok;
        d_off = (long long)w.z0 * e.s_z0 + (long long)w.z1 * e.s_z1 + (long long)w.y * e.s_row;
        r_off = (long long)w.z0 * e.r_z0 + (long long)w.z1 * e.r_z1 + (long long)w.y * e.r_row;
        row_bias = 0.0f;
        za_v = rs_v = 0;
        if (row_ok) {
            if (KIND == 0) {
                if (e.bias_kind == 2) row_bias = e.bias[w.m];
            } else {
                if (e.za) za_v = e.za[w.m % e.za_len];
                else if (e.za8) za_v = e.za8_signed ? (int)(int8_t)__ldg(e.za8) : (int)__ldg(e.za8);
                if (e.zb) rs_v = e.rowsum[w.m];
            }
        }
    }

    // Register path (fully unrolled): f32, act in {none, Relu}, residual / bias absent or 128-bit loadable.  Everything
    // else (Gelu, strided residual, N tails, the integer zero-point math) runs in staged() as a ROLLED loop over the
    // staged row: keeps the unrolled code small enough for the instruction cache.
    __device__ __forceinline__ void math(const KParams& p, uint32_t (&v)[32], int, int nbase, uint8_t* rowp, int sw) {
        const EpilogueDesc& e = p.epi;
        const bool full = nbase + 32 <= p.N;
        fast = (KIND == 0) ? (e.act <= 1 && full) : !(e.za || e.za8 || e.zb || e.scale);  // raw i32: nothing to do
        if (fast && e.r && !p.res_tma)
            fast = e.r_col == 1 && ((reinterpret_cast<uintptr_t>(e.r + r_off + nbase) & 15) == 0);
        if (fast && e.bias_kind == 1) fast = (reinterpret_cast<uintptr_t>(e.bias + nbase) & 15) == 0;
        fast = __all_sync(0xffffffffu, fast || !row_ok) || p.res_tma;  // (res_tma launches are fast-path only)
        // (a chunk entirely beyond N is clipped by the TMA store: its bias and residual are not read)
        if (KIND == 0 && fast && row_ok && nbase < p.N) {
            const bool do_relu = e.act == 1;  // (no activation: NaNs must pass through, fmaxf would drop them)
#pragma unroll
            for (int j = 0; j < 32; j += 4) {
                float4 rr = make_float4(0.f, 0.f, 0.f, 0.f), bb = make_float4(0.f, 0.f, 0.f, 0.f);
                if (p.res_tma)
                    rr = *reinterpret_cast<const float4*>(staged_chunk(rowp, sw, j >> 2));
                else if (e.r)
                    rr = __ldcg(reinterpret_cast<const float4*>(e.r + r_off + nbase + j));
                if (e.bias_kind == 1) bb = __ldg(reinterpret_cast<const float4*>(e.bias + nbase + j));
                const float r4[4] = {rr.x, rr.y, rr.z, rr.w}, b4[4] = {bb.x, bb.y, bb.z, bb.w};
#pragma unroll
                for (int u = 0; u < 4; u++) {
                    float x = __uint_as_float(v[j + u]) * e.alpha;
                    x = fmaf(e.r_scale, r4[u], x);
                    x = x + b4[u] + row_bias;
                    v[j + u] = __float_as_uint(do_relu ? fmaxf(x, 0.0f) : x);
                }
            }
        }
    }

    __device__ __forceinline__ void staged(const KParams& p, int nbase, uint8_t* rowp, int sw) {
        const EpilogueDesc& e = p.epi;
        if (!fast && row_ok) {
            // rolled slow path on this thread's own staged row
#pragma unroll 1
            for (int j = 0; j < 32 && nbase + j < p.N; j++) {
                const int n = nbase + j;
                uint32_t* sp = staged_word(rowp, sw, j);
                if (KIND == 0) {
                    float x = __uint_as_float(*sp) * e.alpha;
                    if (e.r) x = fmaf(e.r_scale, __ldcg(e.r + r_off + (long long)n * e.r_col), x);
                    if (e.bias_kind == 1) x += e.bias[n];
                    x += row_bias;
                    *sp = __float_as_uint(apply_act(x, e.act, e.act_alpha, e.act_beta));
                } else {
                    // exact i32 arithmetic with wrap-around (unsigned ops)
                    unsigned c = *sp;
                    if (e.za || e.za8) c -= (unsigned)za_v * (unsigned)e.colsum[n];
                    if (e.zb) {
                        const unsigned zbv = (unsigned)e.zb[n % e.zb_len];
                        c -= zbv * (unsigned)rs_v;
                        if (e.za || e.za8) c += (unsigned)p.K * (unsigned)za_v * zbv;
                    }
                    if (e.scale) {
                        float sv = e.scale[n % e.scale_len];
                        if (e.scale2) sv = __fmul_rn(__ldg(e.scale2), sv);
                        float x = __fmul_rn(__int2float_rn((int)c), sv);
                        if (e.bias_kind == 1) x = __fadd_rn(x, e.bias[n]);
                        if (e.r) x = __fadd_rn(x, __ldcg(e.r + r_off + (long long)n * e.r_col));
                        *sp = __float_as_uint(apply_act(x, e.act, e.act_alpha, e.act_beta));
                    } else {
                        *sp = c;
                    }
                }
            }
        }
        if (e.range && row_ok) {  // (rolled: the generic epilogue trades speed for size)
#pragma unroll 1
            for (int j = 0; j < 32 && nbase + j < p.N; j++) fold(__uint_as_float(*staged_word(rowp, sw, j)));
        }
    }
};

template <int KIND, bool GELU>
struct FastEpi : RangedEpi {
    unsigned za_v = 0, t_m = 0;  // integer zero-point terms of this thread's row
    __device__ FastEpi(const KParams&, const SmemLayout&, int) {}

    // C = acc - za*colsum[n] - zb[n]*(rowsum - K*za)
    __device__ __forceinline__ void row(const KParams& p, const TileCoord& tc, int r) {
        const EpilogueDesc& e = p.epi;
        za_v = t_m = 0;
        row_ok = true;
        if ((KIND == 1 && (e.za || e.za8 || e.zb)) || e.range) {
            const RowPos w = decode_row(p, tc, r);
            row_ok = w.ok;
            if (row_ok) {
                if (e.za) za_v = (unsigned)e.za[w.m % e.za_len];
                else if (e.za8) za_v = (unsigned)(e.za8_signed ? (int)(int8_t)__ldg(e.za8) : (int)__ldg(e.za8));
                if (e.zb) t_m = (unsigned)e.rowsum[w.m] - (unsigned)p.K * za_v;
            }
        }
    }

    __device__ __forceinline__ void math(const KParams& p, uint32_t (&v)[32], int, int nbase, uint8_t* rowp, int sw) {
        const EpilogueDesc& e = p.epi;
        const bool has_bias = e.bias_kind == 1;
        const bool do_relu = e.act == 1;  // (no activation: NaNs must pass through, fmaxf would drop them)
        // a tile may overhang N (N % bn != 0): its last 32-column chunks are then entirely out of range -- the TMA
        // store clips them, and neither the column vectors (bias, sums, scales) nor the range may touch them
        if (nbase >= p.N) return;
        if (KIND == 0) {
#pragma unroll
            for (int j = 0; j < 32; j += 4) {
                float4 rr = make_float4(0.f, 0.f, 0.f, 0.f), bb = make_float4(0.f, 0.f, 0.f, 0.f);
                if (p.res_tma) rr = *reinterpret_cast<const float4*>(staged_chunk(rowp, sw, j >> 2));
                if (has_bias) bb = __ldg(reinterpret_cast<const float4*>(e.bias + nbase + j));
                const float r4[4] = {rr.x, rr.y, rr.z, rr.w}, b4[4] = {bb.x, bb.y, bb.z, bb.w};
#pragma unroll
                for (int u = 0; u < 4; u++) {
                    float x = __uint_as_float(v[j + u]) * e.alpha;
                    x = fmaf(e.r_scale, r4[u], x);
                    x = x + b4[u];
                    v[j + u] = __float_as_uint(do_relu ? fmaxf(x, 0.0f) : x);
                }
                if (GELU && e.act > 1) act4_bits(v[j], v[j + 1], v[j + 2], v[j + 3], e);
            }
        } else if (e.za || e.za8 || e.zb || e.scale) {
            // exact i32 arithmetic with wrap-around (unsigned ops), column vectors fetched 128 bits at a time
#pragma unroll
            for (int j = 0; j < 32; j += 4) {
                uint4 cs = make_uint4(0u, 0u, 0u, 0u), zb4 = make_uint4(0u, 0u, 0u, 0u);
                float4 sc = make_float4(1.f, 1.f, 1.f, 1.f);
                if (e.za || e.za8) cs = __ldg(reinterpret_cast<const uint4*>(e.colsum + nbase + j));
                if (e.zb) {
                    if (e.zb_len == 1) {
                        const unsigned z = (unsigned)__ldg(e.zb);
                        zb4 = make_uint4(z, z, z, z);
                    } else {
                        zb4 = __ldg(reinterpret_cast<const uint4*>(e.zb + nbase + j));
                    }
                }
                if (e.scale) {
                    if (e.scale_len == 1) {
                        const float z = __ldg(e.scale);
                        sc = make_float4(z, z, z, z);
                    } else {
                        sc = __ldg(reinterpret_cast<const float4*>(e.scale + nbase + j));
                    }
                    if (e.scale2) {
                        const float s2 = __ldg(e.scale2);
                        sc = make_float4(__fmul_rn(s2, sc.x), __fmul_rn(s2, sc.y), __fmul_rn(s2, sc.z), __fmul_rn(s2, sc.w));
                    }
                }
                float4 rr = make_float4(0.f, 0.f, 0.f, 0.f), bb = make_float4(0.f, 0.f, 0.f, 0.f);
                if (p.res_tma) rr = *reinterpret_cast<const float4*>(staged_chunk(rowp, sw, j >> 2));
                if (has_bias) bb = __ldg(reinterpret_cast<const float4*>(e.bias + nbase + j));
                const unsigned c4[4] = {cs.x, cs.y, cs.z, cs.w}, z4[4] = {zb4.x, zb4.y, zb4.z, zb4.w};
                const float s4[4] = {sc.x, sc.y, sc.z, sc.w}, r4[4] = {rr.x, rr.y, rr.z, rr.w},
                            b4[4] = {bb.x, bb.y, bb.z, bb.w};
#pragma unroll
                for (int u = 0; u < 4; u++) {
                    const unsigned c = v[j + u] - za_v * c4[u] - z4[u] * t_m;
                    if (e.scale) {
                        // ConvIntegerToFloat / MatMulIntegerToFloat, then the graph's Add(bias), Add(residual), Relu as
                        // separate exactly-rounded f32 operations (no contraction)
                        float x = __fmul_rn(__int2float_rn((int)c), s4[u]);
                        if (has_bias) x = __fadd_rn(x, b4[u]);
                        if (p.res_tma) x = __fadd_rn(x, r4[u]);
                        v[j + u] = __float_as_uint(do_relu ? fmaxf(x, 0.0f) : x);
                    } else {
                        v[j + u] = c;
                    }
                }
                if (GELU && e.scale && e.act > 1) act4_bits(v[j], v[j + 1], v[j + 2], v[j + 3], e);
            }
        }
        if (e.range && row_ok) {
#pragma unroll
            for (int j = 0; j < 32; j++) fold(__uint_as_float(v[j]));
        }
    }
};

// The common float case as the shortest instruction stream its roundings allow: x = act((acc + residual) + bias),
// with the bias of the unit's columns read from shared memory (loaded while the main loop runs) instead of eight
// dependent global loads behind the accumulator wait.
template <bool GELU>
struct PlainF32Epi : EpiBase {
    float* bias_s;  // chunk k of this group (columns grp*32 + 64k ..) -> bias_s[32k .. 32k + 32)
    float bv = 0.0f;
    int col;  // this thread's column of the unit's bias: (i / 32) * 64 + grp * 32 + i % 32 for thread i of the group
    __device__ PlainF32Epi(const KParams&, const SmemLayout& L, int grp)
        : bias_s(L.bias + grp * 128), col(((threadIdx.x & 127) >> 5) * 64 + grp * 32 + (threadIdx.x & 31)) {}

    __device__ __forceinline__ void unit(const KParams& p, int t) {
        const TileCoord tc = decode_tile(p, t);
        bv = 0.0f;
        if (p.epi.bias_kind == 1 && col < p.bn && tc.n0 + col < p.N) bv = column_bias(p.epi, tc.n0 + col);
    }
    // (the previous unit's readers of bias_s are past their last chunk barrier: every thread arrives there after its math)
    __device__ __forceinline__ void ready(int grp) {
        bias_s[threadIdx.x & 127] = bv;
        group_sync(grp);
    }

    __device__ __forceinline__ void math(const KParams& p, uint32_t (&v)[32], int k, int nbase, uint8_t* rowp, int sw) {
        if (nbase >= p.N) return;  // (a tile may overhang N by whole chunks: the TMA store clips them)
        const float4* bq = reinterpret_cast<const float4*>(bias_s + 32 * k);
#pragma unroll
        for (int j = 0; j < 32; j += 4) {
            float4 rr = make_float4(0.f, 0.f, 0.f, 0.f);
            if (p.res_tma) rr = *reinterpret_cast<const float4*>(staged_chunk(rowp, sw, j >> 2));
            const float4 bb = bq[j >> 2];  // (zeros without a bias: x + 0 keeps the generic path's -0 -> +0)
            plain_f32_pair(v[j], v[j + 1], p.res_tma, make_float2(rr.x, rr.y), make_float2(bb.x, bb.y), p.epi.act == 1);
            plain_f32_pair(v[j + 2], v[j + 3], p.res_tma, make_float2(rr.z, rr.w), make_float2(bb.z, bb.w), p.epi.act == 1);
            if (GELU) act4_bits(v[j], v[j + 1], v[j + 2], v[j + 3], p.epi);
        }
    }
};

// ConvIntegerToFloat / MatMulIntegerToFloat with a scalar activation zero point and symmetric weights -- the quantised
// ResNet-50 / GPT-2 layers:  x = act(((f32(acc - za * colsum[n]) * (x_scale * w_scale[n])) + bias[n]) + residual)
// with every operation rounded separately (bit-identical to the operator chain), plus the output's (min, max) for the
// next DynamicQuantizeLinear.  The three column vectors of the unit are computed once into shared memory while the
// main loop runs.
template <bool GELU>
struct PlainI8Epi : RangedEpi {
    static constexpr bool kSplitK = false;
    unsigned* zc_s;  // za * colsum, scale product, bias: same column mapping as PlainF32Epi::bias_s
    float *scl_s, *bias_s;
    unsigned za_v;
    float s2;
    unsigned zc = 0;
    float sc = 0.0f, bv = 0.0f;
    int col;
    __device__ PlainI8Epi(const KParams& p, const SmemLayout& L, int grp)
        : zc_s(reinterpret_cast<unsigned*>(L.bias) + grp * 128), scl_s(L.bias + 256 + grp * 128),
          bias_s(L.bias + 512 + grp * 128),
          za_v(p.epi.za8 ? (unsigned)(p.epi.za8_signed ? (int)(int8_t)__ldg(p.epi.za8) : (int)__ldg(p.epi.za8)) : 0u),
          s2(p.epi.scale2 ? __ldg(p.epi.scale2) : 1.0f),
          col(((threadIdx.x & 127) >> 5) * 64 + grp * 32 + (threadIdx.x & 31)) {}

    __device__ __forceinline__ void unit(const KParams& p, int t) {
        const TileCoord tc = decode_tile(p, t);
        const EpilogueDesc& e = p.epi;
        const int n = tc.n0 + col;
        zc = 0;
        sc = bv = 0.0f;
        if (col < p.bn && n < p.N) {
            if (e.za8) zc = za_v * (unsigned)__ldg(e.colsum + n);
            sc = e.scale_len == 1 ? __ldg(e.scale) : __ldg(e.scale + n);
            if (e.scale2) sc = __fmul_rn(s2, sc);
            if (e.bias_kind == 1) bv = __ldg(e.bias + n);
        }
    }
    __device__ __forceinline__ void ready(int grp) {
        const int i = threadIdx.x & 127;
        zc_s[i] = zc;
        scl_s[i] = sc;
        bias_s[i] = bv;
        group_sync(grp);
    }
    __device__ __forceinline__ void row(const KParams& p, const TileCoord& tc, int r) {
        row_ok = !p.epi.range || decode_row(p, tc, r).ok;  // rows of the tile beyond the tensor must not enter the range
    }

    __device__ __forceinline__ void math(const KParams& p, uint32_t (&v)[32], int k, int nbase, uint8_t* rowp, int sw) {
        const EpilogueDesc& e = p.epi;
        if (nbase >= p.N) return;  // (a tile may overhang N by whole chunks: the TMA store clips them)
        const uint4* zq = reinterpret_cast<const uint4*>(zc_s + 32 * k);
        const float4* sq = reinterpret_cast<const float4*>(scl_s + 32 * k);
        const float4* bq = reinterpret_cast<const float4*>(bias_s + 32 * k);
#pragma unroll
        for (int j = 0; j < 32; j += 4) {
            const uint4 z = zq[j >> 2];
            const float4 s4 = sq[j >> 2];
            // exact i32 arithmetic with wrap-around, then f32(acc) * scale as ONE rounded product per element
            uint32_t f0 = __float_as_uint(__int2float_rn((int)(v[j] - z.x)));
            uint32_t f1 = __float_as_uint(__int2float_rn((int)(v[j + 1] - z.y)));
            uint32_t f2 = __float_as_uint(__int2float_rn((int)(v[j + 2] - z.z)));
            uint32_t f3 = __float_as_uint(__int2float_rn((int)(v[j + 3] - z.w)));
            mul_f32x2(f0, f1, s4.x, s4.y);
            mul_f32x2(f2, f3, s4.z, s4.w);
            if (e.bias_kind == 1) {
                const float4 bb = bq[j >> 2];
                add_f32x2(f0, f1, bb.x, bb.y);
                add_f32x2(f2, f3, bb.z, bb.w);
            }
            if (p.res_tma) {
                const float4 rr = *reinterpret_cast<const float4*>(staged_chunk(rowp, sw, j >> 2));
                add_f32x2(f0, f1, rr.x, rr.y);
                add_f32x2(f2, f3, rr.z, rr.w);
            }
            if (e.act == 1) {
                f0 = __float_as_uint(fmaxf(__uint_as_float(f0), 0.0f));
                f1 = __float_as_uint(fmaxf(__uint_as_float(f1), 0.0f));
                f2 = __float_as_uint(fmaxf(__uint_as_float(f2), 0.0f));
                f3 = __float_as_uint(fmaxf(__uint_as_float(f3), 0.0f));
            }
            if (GELU) act4_bits(f0, f1, f2, f3, e);  // Gelu / ApproxGelu after the integer product
            v[j] = f0;
            v[j + 1] = f1;
            v[j + 2] = f2;
            v[j + 3] = f3;
        }
        if (e.range && row_ok) {
#pragma unroll
            for (int j = 0; j < 32; j += 2) {
                rg_lo = fminf(rg_lo, fminf(__uint_as_float(v[j]), __uint_as_float(v[j + 1])));
                rg_hi = fmaxf(rg_hi, fmaxf(__uint_as_float(v[j]), __uint_as_float(v[j + 1])));
            }
        }
    }
};

template <int KIND, Epi E>
using EpiOps = std::conditional_t<E == Epi::Generic, GenericEpi<KIND>,
               std::conditional_t<E == Epi::Fast || E == Epi::FastGelu, FastEpi<KIND, E == Epi::FastGelu>,
               std::conditional_t<E == Epi::PlainF32 || E == Epi::PlainF32Gelu, PlainF32Epi<E == Epi::PlainF32Gelu>,
                                  PlainI8Epi<E == Epi::PlainI8Gelu>>>>;

// The epilogue warps (4-11) of umma_gemm_kernel: two groups of four warps, group g takes the 32-column chunks g, g + 2,
// ... of every tile this CTA computes; warp q of a group owns accumulator rows [32 q, 32 q + 32), one row per thread.
// A chunk goes accumulator -> registers -> variant arithmetic -> 128B-swizzled staging buffer (a ring of nbuf per
// group) -> TMA store; a TMA-staged residual chunk lands in the staging buffer the chunk will be written to.
template <int KIND, Epi E>
__device__ __forceinline__ void epilogue(const KParams& p, const SmemLayout& L, const CUtensorMap* tma_d,
                                         const CUtensorMap* tma_r, int worker, int n_workers) {
    using Ops = EpiOps<KIND, E>;
    const EpilogueDesc& e = p.epi;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int q = warp & 3;
    const int grp = (warp - 4) >> 2;
    const int r = q * 32 + lane;
    const int sw = r & 7;
    const int nbuf = p.nbuf;
    uint8_t* const stg0 = L.smem + (size_t)p.stages * p.stage_bytes + grp * nbuf * STG_BYTES;
    const bool issuer = (q == 0 && lane == 0);
    const int splitk = Ops::kSplitK ? p.splitk : 1;
    const bool tma_store = Ops::kDirectStore ? p.tma_store != 0 : true;
    Ops ops(p, L, grp);
    uint32_t ci = 0;                  // chunks processed by this group so far (selects the staging buffer)
    uint32_t aphase = 0, rphase = 0;  // bit b = phase of acc_full[b] / res_bar[grp][b]
    for (int u = worker, it = 0; u < p.units_total; u += n_workers, it++) {
        int t = u, ks = 0;
        if (splitk > 1) p.d_tiles_total.divmod(u, ks, t);
        const int acc = it & 1;
        // residual of chunk `c` (column `col` of the tile) into its ring slot, once the store that last used the slot
        // has been read (at most `in_flight` of this group's stores left un-read)
        auto request_residual = [&](const TileCoord& tc, uint32_t c, int col, int in_flight) {
            const int b = c % nbuf;
            bulk_wait_read(in_flight);
            uint64_t* rb = &L.res_bar[grp * 4 + b];
            mbar_expect_tx(rb, p.res_tx_bytes);
            const int4 x = out_coord(p, tc, col);
            tma_load_4d(stg0 + b * STG_BYTES, tma_r, rb, x.x, x.y, x.z, x.w);
        };
        // the first chunk's residual is independent of the accumulator: requested before waiting for it (split-K: only
        // once this CTA knows that it owns the tile's epilogue)
        const bool first_res = p.res_tma && issuer && grp * 32 < p.bn;
        if (first_res && splitk == 1) request_residual(decode_tile(p, t), ci, grp * 32, nbuf - 1);
        const TileCoord tc0 = decode_tile(p, t);  // (Fast keeps it from here; the others decode again below: that
                                                   //  choice gives each variant its lowest register count and no spills)
        ops.unit(p, t);
        mbar_wait(&L.acc_full[acc], (aphase >> acc) & 1);
        aphase ^= 1u << acc;
        ops.ready(grp);
        const uint32_t t_row = ((uint32_t)(q * 32) << 16) + acc * ACC_STRIDE;
        bool owner = true;
        if (splitk > 1) {  // raw partial accumulators to the workspace; the LAST CTA of the tile sums them in split order
            owner = splitk_publish(p, t, ks, grp, q, lane, t_row, &L.sk_flag[grp], L.acc_smem);
            if (owner && first_res) request_residual(decode_tile(p, t), ci, grp * 32, nbuf - 1);
        }
        if (owner) {
            const TileCoord tc = (E == Epi::Fast || E == Epi::FastGelu) ? tc0 : decode_tile(p, t);
            ops.row(p, tc, r);
            // group g owns the tile's 32-column chunk g: a tile of umma_gemm_kernel has at most ACC_STRIDE = 64 columns
            if (const int c0 = grp * 32, k = 0; c0 < p.bn) {
                uint32_t v[32];
                if (splitk > 1)
                    splitk_sum<KIND>(p, t, c0, r, v);
                else
                    acc_ld(L.acc_smem, t_row + c0, v);
                const int nbase = tc.n0 + c0;
                const int bcur = ci % nbuf;
                uint8_t* stg = stg0 + bcur * STG_BYTES;
                uint8_t* rowp = stg + r * 128;
                if (p.res_tma) {
                    mbar_wait(&L.res_bar[grp * 4 + bcur], (rphase >> bcur) & 1);
                    rphase ^= 1u << bcur;
                }
                ops.math(p, v, k, nbase, rowp, sw);
                // Buffer reuse: (no residual) the issuer waited, before the previous chunk's barrier, until the store of
                // chunk ci - nbuf had been read; (res_tma) the residual mbarrier of this buffer orders it.  Direct stores
                // rotate the buffers too: each thread reads back only its own row.
                if (tma_store && nbuf == 1) {  // single staging buffer: the previous store must have been read
                    if (issuer) bulk_wait_read(0);
                    group_sync(grp);
                }
#pragma unroll
                for (int j = 0; j < 8; j++)
                    *reinterpret_cast<uint4*>(staged_chunk(rowp, sw, j)) = make_uint4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
                ops.staged(p, nbase, rowp, sw);
                if (tma_store) {
                    // leave nbuf-1 stores in flight minus the one about to be issued: frees the buffer of chunk ci+1
                    if (issuer && !p.res_tma && nbuf > 1) bulk_wait_read(nbuf - 2);
                    fence_proxy_async();
                    group_sync(grp);
                    if (issuer) {
                        const int4 x = out_coord(p, tc, c0);
                        tma_store_4d(tma_d, stg, x.x, x.y, x.z, x.w);
                        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
                    }
                } else if (ops.row_ok) {
                    // direct stores from the staged row (any output strides); consecutive lanes = consecutive rows
                    if constexpr (Ops::kDirectStore) {
                        uint32_t* dptr = reinterpret_cast<uint32_t*>(e.d) + ops.d_off;
#pragma unroll 1
                        for (int j = 0; j < 32 && nbase + j < p.N; j++)
                            dptr[(long long)(nbase + j) * e.s_col] = *staged_word(rowp, sw, j);
                    }
                }
                ci++;
            }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&L.acc_empty[acc]);
    }
    ops.finish(e);
    // shared memory must stay valid until the last bulk store has READ it; the global writes complete on their own
    // before the grid is considered finished
    if (tma_store && issuer) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
}

}  // namespace rtb
