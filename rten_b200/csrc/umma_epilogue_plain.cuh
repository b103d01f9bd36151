// Plain epilogues of the wgmma GEMM / conv kernel: the common f32 case (FAST = 3, + Gelu: 5) and the integer *ToFloat
// case (FAST = 4, + Gelu: 6) as the shortest instruction streams their roundings allow -- column vectors of the unit in
// shared memory, paired f32 arithmetic, output at the SM's store-port rate.  Included by umma_kernel.cuh.
#pragma once

namespace rtb {

// Everything an epilogue warp needs from umma_gemm_kernel (umma_kernel.cuh): one struct of references / values so that
// the four epilogue variants can live in their own headers.
struct EpiCtx {
    const KParams& p;
    const SmemLayout& L;
    uint8_t* stg_base;  // staging buffers behind the operand ring
    int nbuf;
    uint64_t *acc_full, *acc_empty, *res_bar;
    int* sk_flag;
    const CUtensorMap *tma_d, *tma_r;
    uint32_t acc_smem;  // shared-memory address of the accumulator tiles (ptx.cuh)
    int worker, n_workers;
    int warp, lane;
};

template <int FAST>
__device__ __forceinline__ void epilogue_plain_f32(const EpiCtx& c) {
    constexpr int KIND = 0;
    (void)KIND;
    const KParams& p = c.p;
    const SmemLayout& L = c.L;
    uint8_t* const stg_base = c.stg_base;
    const int nbuf = c.nbuf;
    uint64_t* const acc_full = c.acc_full;
    uint64_t* const acc_empty = c.acc_empty;
    uint64_t* const res_bar = c.res_bar;
    int* const sk_flag = c.sk_flag;
    const CUtensorMap* const tma_d = c.tma_d;
    const CUtensorMap* const tma_r = c.tma_r;
    const uint32_t acc_smem = c.acc_smem;
    const int worker = c.worker, n_workers = c.n_workers;
    const int warp = c.warp, lane = c.lane;
    (void)L; (void)sk_flag; (void)tma_r; (void)res_bar;
    // ===================== epilogue (plain f32) =====================
    // The common float case -- alpha = 1, optional column bias, optional residual (r_scale = 1, TMA-staged), act in
    // {none, Relu}, no range output -- as the shortest instruction stream the result
    // allows: packed adds (add.rn.f32x2: the same IEEE roundings as two scalar adds), the bias of the unit's
    // columns read from shared memory (loaded while the main loop runs) instead of eight dependent global loads
    // behind the accumulator wait.   x = relu((acc + residual) + bias), rounded after each add like the generic path.
    const EpilogueDesc& e = p.epi;
    const int q = warp & 3;
    const int grp = (warp - 4) >> 2;
    const int r = q * 32 + lane;
    const int sw = r & 7;
    uint8_t* stg0 = stg_base + grp * nbuf * STG_BYTES;
    const bool issuer = (q == 0 && lane == 0);
    const bool has_bias = e.bias_kind == 1;
    const bool do_relu = e.act == 1;
    float* bias_s = L.bias + grp * 128;  // chunk k of this group (columns grp*32 + 64k ..) -> bias_s[32k .. 32k + 32)
    uint32_t ci = 0;
    uint32_t aphase = 0, rphase = 0;  // bit b = phase of acc_full[b] / res_bar[grp][b]
    for (int u = worker, it = 0; u < p.units_total; u += n_workers, it++) {
        int t, ks_u;
        p.d_tiles_total.divmod(u, ks_u, t);
        const int acc = it & 1;
        const uint32_t acc_phase = (aphase >> acc) & 1;
        aphase ^= 1u << acc;
        const TileCoord tc = decode_tile(p, t);
        // residual of the first chunk: independent of the accumulator -> requested before waiting for it (split-K: only
        // once this CTA knows that it owns the tile's epilogue)
        auto first_residual = [&]() {
            const int b0 = ci % nbuf;
            bulk_wait_read(nbuf - 1);
            uint64_t* rb = &res_bar[grp * 4 + b0];
            mbar_expect_tx(rb, p.res_tx_bytes);
            if (p.conv)
                tma_load_4d(stg0 + b0 * STG_BYTES, tma_r, rb, tc.n0 + grp * 32, tc.ox0, tc.oy0, tc.b0);
            else
                tma_load_4d(stg0 + b0 * STG_BYTES, tma_r, rb, tc.n0 + grp * 32, tc.m0, tc.z0, tc.z1);
        };
        if (p.res_tma && p.splitk == 1 && issuer && grp * 32 < p.bn) first_residual();
        float bv = 0.0f;
        if (has_bias) {  // thread i of the group: column (i / 32) * 64 + grp * 32 + i % 32 of the tile
            const int c = (r >> 5) * 64 + grp * 32 + (r & 31);
            if (c < p.bn && tc.n0 + c < p.N) bv = __ldg(e.bias + tc.n0 + c);
        }
        mbar_wait(&acc_full[acc], acc_phase);
        // (the previous unit's readers of bias_s are past their last chunk barrier: every thread arrives there after its math)
        bias_s[r] = bv;
        asm volatile("bar.sync %0, 128;" ::"r"(1 + grp) : "memory");
        bool owner = true;
        if (p.splitk > 1) {  // raw partial accumulators to the workspace; the LAST CTA of the tile sums them in split order
            owner = splitk_publish(p, t, ks_u, grp, q, lane,
                                   ((uint32_t)(q * 32) << 16) + acc * ACC_STRIDE, &sk_flag[grp], acc_smem);
            if (owner && p.res_tma && issuer && grp * 32 < p.bn) first_residual();
        }
        if (owner) {
            const uint32_t t_row = ((uint32_t)(q * 32) << 16) + acc * ACC_STRIDE;
            int k = 0;
            for (int c0 = grp * 32; c0 < p.bn; c0 += 64, k++) {
                uint32_t v[32];
                if (p.splitk > 1)
                    splitk_sum<0>(p, t, c0, r, v);
                else
                    acc_ld(acc_smem, t_row + c0, v);
                const int nbase = tc.n0 + c0;
                const int bcur = ci % nbuf;
                uint8_t* stg = stg0 + bcur * STG_BYTES;
                uint8_t* rowp = stg + r * 128;
                if (p.res_tma && issuer && c0 + 64 < p.bn) {  // prefetch the next chunk's residual of this unit into the next ring slot
                    const int bnext = (ci + 1) % nbuf;
                    bulk_wait_read(nbuf - 2);
                    uint64_t* rb = &res_bar[grp * 4 + bnext];
                    mbar_expect_tx(rb, p.res_tx_bytes);
                    if (p.conv)
                        tma_load_4d(stg0 + bnext * STG_BYTES, tma_r, rb, tc.n0 + c0 + 64, tc.ox0, tc.oy0, tc.b0);
                    else
                        tma_load_4d(stg0 + bnext * STG_BYTES, tma_r, rb, tc.n0 + c0 + 64, tc.m0, tc.z0, tc.z1);
                }
                if (p.res_tma) {
                    mbar_wait(&res_bar[grp * 4 + bcur], (rphase >> bcur) & 1);
                    rphase ^= 1u << bcur;
                }
                if (nbase < p.N) {  // (a tile may overhang N by whole chunks: the TMA store clips them)
                    const float4* bq = reinterpret_cast<const float4*>(bias_s + 32 * k);
#pragma unroll
                    for (int j = 0; j < 32; j += 4) {
                        if (p.res_tma) {
                            const float4 rr = *reinterpret_cast<const float4*>(rowp + (((j >> 2) ^ sw) << 4));
                            add_f32x2(v[j], v[j + 1], rr.x, rr.y);
                            add_f32x2(v[j + 2], v[j + 3], rr.z, rr.w);
                        }
                        const float4 bb = bq[j >> 2];  // (zeros without a bias: x + 0 keeps the generic path's -0 -> +0)
                        add_f32x2(v[j], v[j + 1], bb.x, bb.y);
                        add_f32x2(v[j + 2], v[j + 3], bb.z, bb.w);
                        if (do_relu) {
#pragma unroll
                            for (int w = 0; w < 4; w++) v[j + w] = __float_as_uint(fmaxf(__uint_as_float(v[j + w]), 0.0f));
                        }
                        if (FAST == 5) {  // Gelu / ApproxGelu (own instantiation; the polynomial stays an out-of-line call)
                            const float4 g = act4(make_float4(__uint_as_float(v[j]), __uint_as_float(v[j + 1]), __uint_as_float(v[j + 2]),
                                                              __uint_as_float(v[j + 3])), e.act);
                            v[j] = __float_as_uint(g.x);
                            v[j + 1] = __float_as_uint(g.y);
                            v[j + 2] = __float_as_uint(g.z);
                            v[j + 3] = __float_as_uint(g.w);
                        }
                    }
                }
                if (nbuf == 1) {  // single staging buffer: the previous store must have been read before it is rewritten
                    if (issuer) bulk_wait_read(0);
                    asm volatile("bar.sync %0, 128;" ::"r"(1 + grp) : "memory");
                }
#pragma unroll
                for (int j = 0; j < 8; j++)
                    *reinterpret_cast<uint4*>(rowp + ((j ^ sw) << 4)) = make_uint4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
                if (issuer && !p.res_tma && nbuf > 1) bulk_wait_read(nbuf - 2);
                fence_proxy_async();
                asm volatile("bar.sync %0, 128;" ::"r"(1 + grp) : "memory");
                if (issuer) {
                    if (p.conv)
                        tma_store_4d(tma_d, stg, nbase, tc.ox0, tc.oy0, tc.b0);
                    else
                        tma_store_4d(tma_d, stg, nbase, tc.m0, tc.z0, tc.z1);
                    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
                }
                ci++;
            }
        }
        __syncwarp();
        if (lane == 0) {
            mbar_arrive(&acc_empty[acc]);
        }
    }
    if (issuer) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
}

template <int FAST>
__device__ __forceinline__ void epilogue_plain_i8(const EpiCtx& c) {
    constexpr int KIND = 1;
    (void)KIND;
    const KParams& p = c.p;
    const SmemLayout& L = c.L;
    uint8_t* const stg_base = c.stg_base;
    const int nbuf = c.nbuf;
    uint64_t* const acc_full = c.acc_full;
    uint64_t* const acc_empty = c.acc_empty;
    uint64_t* const res_bar = c.res_bar;
    int* const sk_flag = c.sk_flag;
    const CUtensorMap* const tma_d = c.tma_d;
    const CUtensorMap* const tma_r = c.tma_r;
    const uint32_t acc_smem = c.acc_smem;
    const int worker = c.worker, n_workers = c.n_workers;
    const int warp = c.warp, lane = c.lane;
    (void)L; (void)sk_flag; (void)tma_r; (void)res_bar;
    // ===================== epilogue (plain, integer kind) =====================
    // ConvIntegerToFloat / MatMulIntegerToFloat with a scalar activation zero point and symmetric weights -- the
    // quantised ResNet-50 / GPT-2 layers:  x = relu(((f32(acc - za * colsum[n]) * (x_scale * w_scale[n])) + bias[n]) + residual)
    // with every operation rounded separately (bit-identical to the operator chain), plus the output's (min, max)
    // for the next DynamicQuantizeLinear.  The three column vectors of the unit are computed once into shared memory
    // while the main loop runs (the specialised epilogue fetched them with 24 dependent 128-bit global loads per
    // chunk behind the accumulator wait), products / sums are done two lanes at a time.
    const EpilogueDesc& e = p.epi;
    const int q = warp & 3;
    const int grp = (warp - 4) >> 2;
    const int r = q * 32 + lane;
    const int sw = r & 7;
    uint8_t* stg0 = stg_base + grp * nbuf * STG_BYTES;
    const bool issuer = (q == 0 && lane == 0);
    const bool has_bias = e.bias_kind == 1;
    const bool do_relu = e.act == 1;
    unsigned* zc_s = reinterpret_cast<unsigned*>(L.bias) + grp * 128;
    float* scl_s = L.bias + 256 + grp * 128;
    float* bias_s = L.bias + 512 + grp * 128;
    uint32_t ci = 0;
    uint32_t aphase = 0, rphase = 0;  // bit b = phase of acc_full[b] / res_bar[grp][b]
    float rg_lo = __int_as_float(0x7f800000), rg_hi = __int_as_float(0xff800000);  // output range (e.range)
    const unsigned za_v = e.za8 ? (unsigned)(e.za8_signed ? (int)(int8_t)__ldg(e.za8) : (int)__ldg(e.za8)) : 0u;
    const float s2 = e.scale2 ? __ldg(e.scale2) : 1.0f;
    for (int u = worker, it = 0; u < p.units_total; u += n_workers, it++) {
        const int t = u;  // (no split-K on this path)
        const int acc = it & 1;
        const uint32_t acc_phase = (aphase >> acc) & 1;
        aphase ^= 1u << acc;
        const TileCoord tc = decode_tile(p, t);
        if (p.res_tma && issuer && grp * 32 < p.bn) {  // residual of the first chunk: independent of the accumulator
            const int b0 = ci % nbuf;
            bulk_wait_read(nbuf - 1);
            uint64_t* rb = &res_bar[grp * 4 + b0];
            mbar_expect_tx(rb, p.res_tx_bytes);
            if (p.conv)
                tma_load_4d(stg0 + b0 * STG_BYTES, tma_r, rb, tc.n0 + grp * 32, tc.ox0, tc.oy0, tc.b0);
            else
                tma_load_4d(stg0 + b0 * STG_BYTES, tma_r, rb, tc.n0 + grp * 32, tc.m0, tc.z0, tc.z1);
        }
        // thread i of the group: column (i / 32) * 64 + grp * 32 + i % 32 of the tile
        unsigned zc = 0;
        float sc = 0.0f, bv = 0.0f;
        {
            const int c = (r >> 5) * 64 + grp * 32 + (r & 31);
            const int n = tc.n0 + c;
            if (c < p.bn && n < p.N) {
                if (e.za8) zc = za_v * (unsigned)__ldg(e.colsum + n);
                sc = e.scale_len == 1 ? __ldg(e.scale) : __ldg(e.scale + n);
                if (e.scale2) sc = __fmul_rn(s2, sc);
                if (has_bias) bv = __ldg(e.bias + n);
            }
        }
        mbar_wait(&acc_full[acc], acc_phase);
        zc_s[r] = zc;
        scl_s[r] = sc;
        bias_s[r] = bv;
        asm volatile("bar.sync %0, 128;" ::"r"(1 + grp) : "memory");
        const uint32_t t_row = ((uint32_t)(q * 32) << 16) + acc * ACC_STRIDE;
        bool row_ok = true;
        if (e.range) {  // rows of the tile beyond the tensor must not enter the range
            if (p.conv) {
                int xi, r2, yi, bi;
                p.d_tw.divmod(r, r2, xi);
                p.d_th.divmod(r2, bi, yi);
                row_ok = (bi < p.tb) && (tc.ox0 + xi < p.OW) && (tc.oy0 + yi < p.OH) && (tc.b0 + bi < p.Bn);
            } else {
                row_ok = tc.m0 + r < p.M;
            }
        }
        int k = 0;
        for (int c0 = grp * 32; c0 < p.bn; c0 += 64, k++) {
            uint32_t v[32];
            acc_ld(acc_smem, t_row + c0, v);
            const int nbase = tc.n0 + c0;
            const int bcur = ci % nbuf;
            uint8_t* stg = stg0 + bcur * STG_BYTES;
            uint8_t* rowp = stg + r * 128;
            if (p.res_tma && issuer && c0 + 64 < p.bn) {  // prefetch the next chunk's residual of this unit into the next ring slot
                const int bnext = (ci + 1) % nbuf;
                bulk_wait_read(nbuf - 2);
                uint64_t* rb = &res_bar[grp * 4 + bnext];
                mbar_expect_tx(rb, p.res_tx_bytes);
                if (p.conv)
                    tma_load_4d(stg0 + bnext * STG_BYTES, tma_r, rb, tc.n0 + c0 + 64, tc.ox0, tc.oy0, tc.b0);
                else
                    tma_load_4d(stg0 + bnext * STG_BYTES, tma_r, rb, tc.n0 + c0 + 64, tc.m0, tc.z0, tc.z1);
            }
            if (p.res_tma) {
                mbar_wait(&res_bar[grp * 4 + bcur], (rphase >> bcur) & 1);
                rphase ^= 1u << bcur;
            }
            const bool col_ok = nbase < p.N;  // (a tile may overhang N by whole chunks: the TMA store clips them)
            if (col_ok) {
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
                    if (has_bias) {
                        const float4 bb = bq[j >> 2];
                        add_f32x2(f0, f1, bb.x, bb.y);
                        add_f32x2(f2, f3, bb.z, bb.w);
                    }
                    if (p.res_tma) {
                        const float4 rr = *reinterpret_cast<const float4*>(rowp + (((j >> 2) ^ sw) << 4));
                        add_f32x2(f0, f1, rr.x, rr.y);
                        add_f32x2(f2, f3, rr.z, rr.w);
                    }
                    if (do_relu) {
                        f0 = __float_as_uint(fmaxf(__uint_as_float(f0), 0.0f));
                        f1 = __float_as_uint(fmaxf(__uint_as_float(f1), 0.0f));
                        f2 = __float_as_uint(fmaxf(__uint_as_float(f2), 0.0f));
                        f3 = __float_as_uint(fmaxf(__uint_as_float(f3), 0.0f));
                    }
                    if (FAST == 6) {  // Gelu / ApproxGelu after the integer product (own instantiation, out-of-line polynomial)
                        const float4 g = act4(make_float4(__uint_as_float(f0), __uint_as_float(f1), __uint_as_float(f2), __uint_as_float(f3)), e.act);
                        f0 = __float_as_uint(g.x);
                        f1 = __float_as_uint(g.y);
                        f2 = __float_as_uint(g.z);
                        f3 = __float_as_uint(g.w);
                    }
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
            if (nbuf == 1) {  // single staging buffer: the previous store must have been read before it is rewritten
                if (issuer) bulk_wait_read(0);
                asm volatile("bar.sync %0, 128;" ::"r"(1 + grp) : "memory");
            }
#pragma unroll
            for (int j = 0; j < 8; j++)
                *reinterpret_cast<uint4*>(rowp + ((j ^ sw) << 4)) = make_uint4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
            if (issuer && !p.res_tma && nbuf > 1) bulk_wait_read(nbuf - 2);
            fence_proxy_async();
            asm volatile("bar.sync %0, 128;" ::"r"(1 + grp) : "memory");
            if (issuer) {
                if (p.conv)
                    tma_store_4d(tma_d, stg, nbase, tc.ox0, tc.oy0, tc.b0);
                else
                    tma_store_4d(tma_d, stg, nbase, tc.m0, tc.z0, tc.z1);
                asm volatile("cp.async.bulk.commit_group;" ::: "memory");
            }
            ci++;
        }
        __syncwarp();
        if (lane == 0) {
            mbar_arrive(&acc_empty[acc]);
        }
    }
    if (e.range) range_commit(e.range, rg_lo, rg_hi);
    if (issuer) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
}

}  // namespace rtb
