// Operator entry points of the C ABI, MatMul family (Gemm, MatMul / FusedMatMul, MatMulInteger(ToFloat), prepack):
// shape / argument validation with the reference's error strings,
// operand normalisation (K-major, TMA-addressable), kernel dispatch.  Mirrors, per function, the
// reference operator named in include/rten_b200.h.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "api_shared.h"
#include "api_util.h"
#include "nbits.h"
#include "rowops.h"
#include "skinny.h"
#include "umma_gemm.h"

using namespace rtb;
using namespace rtb::api;

namespace rtb {
namespace api {

rten_status to_kmajor(rten_ctx* ctx, int esize, const Mat& m, OperandDesc* od) {
    OperandDesc d;
    d.base = m.base;
    d.dims[0] = m.K;
    d.dims[1] = m.rows;
    // broadcast batch dims (stride 0) become size-1 dims: the kernel then always passes coordinate 0
    d.dims[2] = (m.z0 > 1 && m.zs0 != 0) ? m.z0 : 1;
    d.dims[3] = (m.z1 > 1 && m.zs1 != 0) ? m.z1 : 1;
    d.strides[0] = m.ks;
    d.strides[1] = m.rs;
    d.strides[2] = d.dims[2] > 1 ? m.zs0 : 0;
    d.strides[3] = d.dims[3] > 1 ? m.zs1 : 0;
    if (m.K == 1) d.strides[0] = 1;  // a single k element is trivially contiguous
    if (tma_compatible(d, esize, 4)) {
        *od = d;
        return RTEN_OK;
    }
    // pack: [z1', z0', rows, Kpad]; broadcast batch dims (stride 0) are NOT expanded
    const int64_t kpad = round_up(m.K, 16 / esize);
    const int64_t e0 = (m.z0 > 1 && m.zs0 == 0) ? 1 : m.z0;
    const int64_t e1 = (m.z1 > 1 && m.zs1 == 0) ? 1 : m.z1;
    void* buf = nullptr;
    RTB_TRY(temp_alloc(ctx, (size_t)(e1 * e0 * m.rows * kpad) * esize, &buf));
    long long shape[4] = {e1, e0, m.rows, m.K};
    long long ss[4] = {m.zs1, m.zs0, m.rs, m.ks};
    long long ds[4] = {e0 * m.rows * kpad, m.rows * kpad, kpad, 1};
    RTB_TRY(launch_nd_copy(ctx, esize, m.base, buf, 4, shape, ss, ds));
    d.base = buf;
    d.dims[2] = e0;
    d.dims[3] = e1;
    d.strides[0] = 1;
    d.strides[1] = kpad;
    d.strides[2] = e0 > 1 ? m.rows * kpad : 0;
    d.strides[3] = e1 > 1 ? e0 * m.rows * kpad : 0;
    *od = d;
    return RTEN_OK;
}

}  // namespace api
}  // namespace rtb

namespace {

// Collapse broadcast prefix dims of a matmul into at most 2 batch dims (z0 inner, z1 outer).  Dims are merged
// only when A, B and the output all advance uniformly across them.
struct BatchDims {
    int64_t z0 = 1, z1 = 1;
    int64_t a0 = 0, a1 = 0, b0 = 0, b1 = 0, o0 = 0, o1 = 0;
    bool ok = true;
};

BatchDims collapse_batch(const std::vector<int64_t>& size, const std::vector<int64_t>& as, const std::vector<int64_t>& bs,
                         const std::vector<int64_t>& os) {
    std::vector<int64_t> s, a, b, o;
    for (size_t i = 0; i < size.size(); i++) {
        if (size[i] == 1) continue;
        if (!s.empty() && a.back() == as[i] * size[i] && b.back() == bs[i] * size[i] && o.back() == os[i] * size[i]) {
            s.back() *= size[i];
            a.back() = as[i];
            b.back() = bs[i];
            o.back() = os[i];
            continue;
        }
        s.push_back(size[i]);
        a.push_back(as[i]);
        b.push_back(bs[i]);
        o.push_back(os[i]);
    }
    BatchDims r;
    if (s.size() > 2) {
        r.ok = false;
        return r;
    }
    if (s.size() == 1) {
        r.z0 = s[0];
        r.a0 = a[0];
        r.b0 = b[0];
        r.o0 = o[0];
    } else if (s.size() == 2) {
        r.z1 = s[0];
        r.a1 = a[0];
        r.b1 = b[0];
        r.o1 = o[0];
        r.z0 = s[1];
        r.a0 = a[1];
        r.b0 = b[1];
        r.o0 = o[1];
    }
    return r;
}

struct MatMulArgs {
    int kind;  // 0 f32, 1 int8
    const rten_tensor* a;
    const rten_tensor* b;
    const rten_packed* pb;
    EpilogueDesc epi;  // d / strides filled by matmul_core
    int out_dtype;
    // int8 extras
    const rten_tensor* a_zp = nullptr;
    const rten_tensor* b_zp = nullptr;
    // residual (same shape as out) for matmul_ex
    const rten_tensor* residual = nullptr;
};

// numpy-matmul shape logic of src/ops/matmul.rs:208-385 + kernel dispatch
rten_status matmul_core(OpScope& sc, MatMulArgs& A, rten_tensor* out) {
    rten_ctx* ctx = sc.ctx;
    rten_tensor a = *A.a, b = *A.b;
    if (a.ndim < 1 || b.ndim < 1) return fail(ctx, RTEN_ERR_INVALID_VALUE, "Inputs must have >= 1 dimensions");
    const bool a_vec = a.ndim == 1, b_vec = b.ndim == 1;
    if (a_vec) {  // [K] -> [1, K]
        a.ndim = 2;
        a.shape[1] = a.shape[0];
        a.strides[1] = a.strides[0];
        a.shape[0] = 1;
        a.strides[0] = 0;
    }
    if (b_vec) {  // [K] -> [K, 1]
        b.ndim = 2;
        b.shape[1] = 1;
        b.strides[1] = 0;
    }
    const int64_t M = a.shape[a.ndim - 2], K = a.shape[a.ndim - 1];
    const int64_t Kb = b.shape[b.ndim - 2], N = b.shape[b.ndim - 1];
    if (K != Kb)
        return fail(ctx, RTEN_ERR_INCOMPATIBLE_SHAPES, "Columns of first matrix does not match rows of second matrix");
    // broadcast prefixes
    const int pa = a.ndim - 2, pb = b.ndim - 2, pn = std::max(pa, pb);
    std::vector<int64_t> psize(pn), pas(pn), pbs(pn);
    for (int i = 0; i < pn; i++) {
        const int ia = i - (pn - pa), ib = i - (pn - pb);
        const int64_t sa = ia >= 0 ? a.shape[ia] : 1, sb = ib >= 0 ? b.shape[ib] : 1;
        if (sa != sb && sa != 1 && sb != 1) return fail(ctx, RTEN_ERR_INCOMPATIBLE_SHAPES, "Cannot broadcast shapes");
        psize[i] = std::max(sa, sb);
        if (sa == 0 || sb == 0) psize[i] = 0;
        pas[i] = (ia >= 0 && sa != 1) ? a.strides[ia] : 0;
        pbs[i] = (ib >= 0 && sb != 1) ? b.strides[ib] : 0;
    }
    // output shape
    int64_t oshape[RTEN_MAX_DIMS];
    int on = 0;
    for (int i = 0; i < pn; i++) oshape[on++] = psize[i];
    if (!a_vec) oshape[on++] = M;
    if (!b_vec) oshape[on++] = N;
    if (on > RTEN_MAX_DIMS) return fail(ctx, RTEN_ERR_INVALID_VALUE, "tensor rank out of range");
    rten_tensor ov;
    RTB_TRY(sc.out(out, A.out_dtype, on, oshape, &ov, nullptr));
    int64_t total = 1;
    for (int i = 0; i < on; i++) total *= oshape[i];
    if (total == 0) return RTEN_OK;
    // output strides of the prefix dims / row / col in the (vector-expanded) [prefix.., M, N] view
    std::vector<int64_t> pos(pn, 0);
    int64_t o_rs = 0, o_cs = 0;
    {
        int k = 0;
        for (int i = 0; i < pn; i++) pos[i] = ov.strides[k++];
        if (!a_vec) o_rs = ov.strides[k++];
        if (!b_vec) o_cs = ov.strides[k++];
    }
    rten_tensor dv = ov;
    bool copy_out = false;
    const int esize = A.kind == 0 ? 4 : 1;
    int64_t nbatch = 1;
    for (int i = 0; i < pn; i++) nbatch *= psize[i];
    int64_t nb_mats = 1;
    for (int i = 0; i < pb; i++) nb_mats *= b.shape[i];

    GemmLaunch L;
    L.kind = A.kind;
    L.a_signed = A.a->dtype == RTEN_I8;
    L.b_signed = (A.pb ? A.pb->dtype : A.b->dtype) == RTEN_I8;
    L.N = (int)N;
    L.K = (int)K;
    L.epi = A.epi;
    L.epi.d_is_i32 = A.out_dtype == RTEN_I32;

    if (K == 0) {
        // lib.rs:843-873: product term vanishes; out = bias (f32) / 0 (int).  Reuse Add machinery: fill.
        if (!is_contiguous(&ov)) {
            set_contiguous(&dv);
            void* t = nullptr;
            RTB_TRY(temp_alloc(ctx, (size_t)total * 4, &t));
            dv.data = t;
            copy_out = true;
        }
        RTB_CUDA(ctx, cudaMemsetAsync(dv.data, 0, (size_t)total * 4, ctx->stream));
        if (A.kind == 0 && L.epi.bias) {
            long long shp[2] = {total / N, N}, s0[2] = {N, 1}, sb[2] = {0, 1};
            RTB_TRY(launch_binary(ctx, RTEN_F32, BIN_ADD, 0, dv.data, L.epi.bias, dv.data, 2, shp, s0, sb, s0));
        }
    } else {
        // B operand
        Mat mb;
        if (A.pb) {
            if (A.pb->kind != 0 || A.pb->K != K || A.pb->N != N)
                return fail(ctx, RTEN_ERR_INVALID_VALUE, "prepacked B does not match the matmul shape");
            mb.base = A.pb->data;
            mb.rows = N;
            mb.K = K;
            mb.rs = A.pb->ld;
            mb.ks = 1;
            nb_mats = 1;
        } else {
            mb.base = b.data;
            mb.rows = N;
            mb.K = K;
            mb.rs = b.strides[b.ndim - 1];
            mb.ks = b.strides[b.ndim - 2];
        }
        Mat ma;
        ma.base = a.data;
        ma.K = K;
        ma.ks = a.strides[a.ndim - 1];
        ma.rs = a.strides[a.ndim - 2];
        ma.rows = M;

        // Flatten [A.., M, K] x [K, N] into one [A*M, K] GEMM (matmul.rs:266-297) when A's rows are
        // uniformly strided; otherwise keep (up to two) batch dims.
        bool flat = false;
        BatchDims bd;
        const std::vector<int64_t> b_eff = A.pb ? std::vector<int64_t>(pn, 0) : pbs;
        for (int attempt = 0; attempt < 2; attempt++) {
            // attempt 0: write straight into the caller's (possibly strided) output; attempt 1: contiguous temp
            if (attempt == 1) {
                set_contiguous(&dv);
                void* t = nullptr;
                RTB_TRY(temp_alloc(ctx, (size_t)total * 4, &t));
                dv.data = t;
                copy_out = true;
                int k = 0;
                for (int i = 0; i < pn; i++) pos[i] = dv.strides[k++];
                if (!a_vec) o_rs = dv.strides[k++];
                if (!b_vec) o_cs = dv.strides[k++];
            }
            flat = false;
            if (nb_mats == 1) {
                std::vector<int64_t> sz = psize, as = pas, zs(pn, 0), os = pos;
                sz.push_back(M);
                as.push_back(ma.rs);
                zs.push_back(0);
                os.push_back(o_rs);
                BatchDims c = collapse_batch(sz, as, zs, os);
                if (c.ok && c.z1 == 1) {
                    flat = true;
                    ma.rows = c.z0;
                    if (c.z0 > 1) {
                        ma.rs = c.a0;
                        o_rs = c.o0;
                    }
                    break;
                }
            }
            bd = collapse_batch(psize, pas, b_eff, pos);
            if (bd.ok) break;
            if (attempt == 1)
                return fail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "matmul batch dims do not collapse to 2 strided dims");
        }
        L.epi.d = dv.data;
        L.epi.s_row = o_rs;
        L.epi.s_col = b_vec ? 1 : o_cs;
        if (flat) {
            L.M = (int)ma.rows;
            L.z0 = L.z1 = 1;
        } else {
            L.M = (int)M;
            L.z0 = (int)bd.z0;
            L.z1 = (int)bd.z1;
            ma.z0 = bd.z0;
            ma.z1 = bd.z1;
            ma.zs0 = bd.a0;
            ma.zs1 = bd.a1;
            mb.z0 = bd.z0;
            mb.z1 = bd.z1;
            mb.zs0 = bd.b0;
            mb.zs1 = bd.b1;
            L.epi.s_z0 = bd.o0;
            L.epi.s_z1 = bd.o1;
        }
        if (A.kind == 1 && !flat && (A.a_zp || A.b_zp) && nbatch > 1)
            return fail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "MatMulInteger with a batched RHS and zero points is not supported");
        RTB_TRY(to_kmajor(ctx, esize, ma, &L.a));
        if (mb.z0 > 1 && mb.zs0 == 0) {}  // broadcast handled by stride 0
        RTB_TRY(to_kmajor(ctx, esize, mb, &L.b));
        if (A.pb && A.kind == 0 && L.b.base == A.pb->data) L.b_x3_slot = &const_cast<rten_packed*>(A.pb)->x3;

        // residual (same shape as out, any strides) -> only contiguous or row-strided supported directly
        if (A.residual) {
            rten_tensor rv;
            RTB_TRY(sc.in(A.residual, &rv));
            if (rv.ndim != on) return fail(ctx, RTEN_ERR_INCOMPATIBLE_SHAPES, "residual shape does not match output");
            for (int i = 0; i < on; i++)
                if (rv.shape[i] != oshape[i]) return fail(ctx, RTEN_ERR_INCOMPATIBLE_SHAPES, "residual shape does not match output");
            rten_tensor rc;
            RTB_TRY(sc.contiguous(&rv, &rc));
            L.epi.r = (const float*)rc.data;
            L.epi.r_scale = 1.0f;
            L.epi.r_col = 1;
            L.epi.r_row = N;
            L.epi.r_z0 = flat ? 0 : M * N;
            L.epi.r_z1 = flat ? 0 : bd.z0 * M * N;
        }

        // integer zero points
        if (A.kind == 1) {
            const int64_t rows_total = flat ? ma.rows : M;
            if (A.a_zp) {
                rten_tensor z;
                RTB_TRY(sc.in(A.a_zp, &z));
                const int len = z.ndim == 0 ? 1 : (int)z.shape[0];
                if (len == 1) {  // scalar (DynamicQuantizeLinear's zero point): read in place by the epilogue
                    L.epi.za8 = (const uint8_t*)z.data;
                    L.epi.za8_signed = z.dtype == RTEN_I8;
                } else {
                    int32_t* za = nullptr;
                    RTB_TRY(temp_alloc(ctx, (size_t)len * 4, (void**)&za));
                    RTB_TRY(launch_zp_to_i32(ctx, z.data, z.dtype == RTEN_I8, len, z.ndim == 0 ? 0 : z.strides[0], za));
                    L.epi.za = za;
                    L.epi.za_len = len;
                }
                if (A.pb && A.pb->colsum) {
                    L.epi.colsum = A.pb->colsum;
                } else {
                    int32_t* cs = nullptr;
                    RTB_TRY(temp_alloc(ctx, (size_t)N * 4, (void**)&cs));
                    RTB_TRY(launch_rowsum8(ctx, L.b.base, L.b_signed, N, (int)K, L.b.strides[1], cs));
                    L.epi.colsum = cs;
                }
            }
            if (A.b_zp) {
                rten_tensor z;
                RTB_TRY(sc.in(A.b_zp, &z));
                const int len = z.ndim == 0 ? 1 : (int)z.shape[0];
                int32_t* zb = nullptr;
                RTB_TRY(temp_alloc(ctx, (size_t)len * 4, (void**)&zb));
                RTB_TRY(launch_zp_to_i32(ctx, z.data, z.dtype == RTEN_I8, len, z.ndim == 0 ? 0 : z.strides[0], zb));
                L.epi.zb = zb;
                L.epi.zb_len = len;
                int32_t* rs = nullptr;
                RTB_TRY(temp_alloc(ctx, (size_t)rows_total * 4, (void**)&rs));
                RTB_TRY(launch_rowsum8(ctx, L.a.base, L.a_signed, rows_total, (int)K, L.a.strides[1], rs));
                L.epi.rowsum = rs;
            }
        }
        // M <= 32 f32 rows: the HBM-streaming skinny kernel (exact f32 FMA arithmetic) instead of a 128-row MMA tile
        // (rten-gemm's gemv path, rten-gemm/src/lib.rs:668-747)
        if (A.kind == 0 && L.z0 == 1 && L.z1 == 1 && L.M <= 32 && L.epi.s_col == 1 && L.epi.bias_kind != 2 &&
            (!L.epi.r || L.epi.r_col == 1) && !L.epi.range && L.a.strides[0] == 1 && L.b.strides[0] == 1) {
            SkinnyF32Launch S;
            S.a = (const float*)L.a.base;
            S.as = L.a.strides[1];
            S.b = (const float*)L.b.base;
            S.bs = L.b.strides[1];
            S.M = L.M;
            S.N = L.N;
            S.K = L.K;
            S.alpha = L.epi.alpha;
            S.bias = L.epi.bias_kind == 1 ? L.epi.bias : nullptr;
            S.residual = L.epi.r;
            S.rs = L.epi.r_row;
            S.r_scale = L.epi.r_scale;
            S.act = L.epi.act;
            S.out = (float*)L.epi.d;
            S.os = L.epi.s_row;
            if (skinny_f32_supported(S)) {
                RTB_TRY(launch_skinny_f32(ctx, S));
                goto launched;
            }
        }
        {
        rten_status st = launch_umma_gemm(ctx, L);
        if (st == RTEN_ERR_UNSUPPORTED_VALUE) return fail(ctx, st, "GEMM operands are not addressable by TMA after packing");
        RTB_TRY(st);
        }
    launched:;
    }
    return copy_out ? copy_view(ctx, dv, ov) : RTEN_OK;
}

// The leading ndim - 1 dims of `t` as one row dimension of uniform stride (*rs; any value when there is one row).
bool flat_rows(const rten_tensor& t, int64_t* rs) {
    *rs = 0;
    int64_t next = -1;  // stride the next outer dim must have
    for (int i = t.ndim - 2; i >= 0; i--) {
        if (t.shape[i] == 1) continue;
        if (next >= 0 && t.strides[i] != next) return false;
        if (next < 0) *rs = t.strides[i];
        next = t.strides[i] * t.shape[i];
    }
    return true;
}

// src/ops/matmul/contrib.rs:21-186 (MatMulNBits): validation in the reference's order, then one kernel (nbits.cu)
rten_status matmul_nbits(OpScope& sc, const rten_tensor* a, const rten_tensor* b, const rten_tensor* scales, int bits,
                         int block_size, rten_tensor* out) {
    rten_ctx* ctx = sc.ctx;
    rten_tensor av, bv, sv;
    RTB_TRY(sc.in(a, &av));
    RTB_TRY(sc.in(b, &bv));
    RTB_TRY(sc.in(scales, &sv));
    const int64_t N = bv.shape[0];
    // `scales` [N, k_blocks], or 1-D [N * k_blocks] with k_blocks = K / block_size (older models)
    int64_t s_n, s_k, s_blocks;
    if (sv.ndim == 2) {
        s_n = sv.strides[0];
        s_k = sv.strides[1];
        s_blocks = sv.shape[1];
        if (sv.shape[0] != N) s_blocks = -1;
    } else if (sv.ndim == 1) {
        const int64_t k = av.ndim >= 1 ? av.shape[av.ndim - 1] : 1;
        s_blocks = block_size > 0 ? k / block_size : 0;
        if (sv.shape[0] != N * s_blocks)
            return fail(ctx, RTEN_ERR_INVALID_VALUE, "Expected 1D `scales` size to match columns * block_size");
        s_k = sv.strides[0];
        s_n = s_blocks * s_k;
    } else {
        return fail(ctx, RTEN_ERR_INVALID_VALUE, "Expected `scales` to have one or two dims");
    }
    if (av.ndim < 2) return fail(ctx, RTEN_ERR_INVALID_VALUE, "A input must have at least 2 dims");
    if (bits != 4) return fail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "Unsupported bits-per-element");
    const int64_t kb = bv.shape[1], blob = bv.shape[2], block = 2 * blob;
    if (block < 16 || (block & (block - 1))) return fail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "Unsupported K block size");
    const int64_t K = av.shape[av.ndim - 1];
    int64_t oshape[RTEN_MAX_DIMS];
    int64_t rows = 1;
    for (int i = 0; i < av.ndim - 1; i++) {
        oshape[i] = av.shape[i];
        rows *= av.shape[i];
    }
    oshape[av.ndim - 1] = N;
    if (K != kb * block)
        return fail(ctx, RTEN_ERR_INCOMPATIBLE_SHAPES, "Columns of first matrix does not match rows of second matrix");
    // (the reference does not check this and would read past the scales)
    if (s_blocks != kb) return fail(ctx, RTEN_ERR_INCOMPATIBLE_SHAPES, "MatMulNBits: `scales` must have shape [N, k_blocks]");
    if (rows > 0x7fffffffll || N > 0x7fffffffll || K > 0x7fffffffll)
        return fail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "MatMulNBits: dimension out of range");
    rten_tensor ov;
    RTB_TRY(sc.out(out, RTEN_F32, av.ndim, oshape, &ov, nullptr));
    if (rows == 0 || N == 0) return RTEN_OK;

    // output: [rows, N] with unit column stride, else a contiguous temporary copied back
    int64_t o_rs;
    rten_tensor dv = ov;
    const bool direct = flat_rows(ov, &o_rs) && ov.strides[ov.ndim - 1] == 1;
    if (!direct) {
        set_contiguous(&dv);
        void* t = nullptr;
        RTB_TRY(temp_alloc(ctx, (size_t)(rows * N) * 4, &t));
        dv.data = t;
        o_rs = N;
    }
    if (K == 0) {  // block_quant.rs:80-84
        RTB_CUDA(ctx, cudaMemsetAsync(dv.data, 0, (size_t)(rows * N) * 4, ctx->stream));
    } else {
        // A: [rows, K] with 16-byte aligned rows (K is a multiple of 16), else packed into a workspace
        int64_t a_rs;
        const float* ap = (const float*)av.data;
        if (!flat_rows(av, &a_rs) || av.strides[av.ndim - 1] != 1 || (a_rs & 3) || (reinterpret_cast<uintptr_t>(ap) & 15)) {
            rten_tensor c = av;
            set_contiguous(&c);
            RTB_TRY(temp_alloc(ctx, (size_t)(rows * K) * 4, &c.data));
            RTB_TRY(copy_view(ctx, av, c));
            ap = (const float*)c.data;
            a_rs = K;
        }
        // B: rows of K / 2 contiguous bytes at a pitch of a multiple of 16 bytes (K % 32 == 0), else copied to one
        const uint8_t* qp = (const uint8_t*)bv.data;
        int64_t q_rs = N > 1 ? bv.strides[0] : K / 2;
        const bool dense = bv.strides[2] == 1 && (kb == 1 || bv.strides[1] == blob);
        if (!dense || (q_rs & 15) || (reinterpret_cast<uintptr_t>(qp) & 15)) {
            const int64_t pitch = round_up(K / 2, 16);
            void* t = nullptr;
            RTB_TRY(temp_alloc(ctx, (size_t)(N * pitch), &t));
            long long shape[3] = {N, kb, blob}, ss[3] = {bv.strides[0], bv.strides[1], bv.strides[2]}, ds[3] = {pitch, blob, 1};
            RTB_TRY(launch_nd_copy(ctx, 1, bv.data, t, 3, shape, ss, ds));
            qp = (const uint8_t*)t;
            q_rs = pitch;
        }
        NbitsLaunch L;
        L.a = ap;
        L.as = a_rs;
        L.q = qp;
        L.qs = q_rs;
        L.scales = (const float*)sv.data;
        L.s_n = s_n;
        L.s_k = s_k;
        L.M = (int)rows;
        L.N = (int)N;
        L.K = (int)K;
        L.block = (int)block;
        L.x3 = ctx->f32_mode == RTEN_F32_TF32X3;
        L.out = (float*)dv.data;
        L.os = o_rs;
        RTB_TRY(launch_nbits(ctx, L));
    }
    return direct ? RTEN_OK : copy_view(ctx, dv, ov);
}

// src/ops/matmul.rs:513-533 zero_point_to_vec validation
}  // namespace

extern "C" {

rten_status rten_b200_prepack_b(rten_ctx* ctx, const rten_tensor* b, rten_packed** out) {
    RTB_TRY(check_ctx(ctx));
    if (!b || !out) return RTEN_ERR_INVALID_VALUE;
    *out = nullptr;
    if (b->ndim != 2) return fail(ctx, RTEN_ERR_INVALID_VALUE, "prepack expects a matrix");  // matmul_prepack_b: try_into Matrix
    if (b->dtype == RTEN_I32) return fail(ctx, RTEN_ERR_UNSUPPORTED_TYPE, "unsupported type");
    OpScope sc(ctx);
    rten_tensor bv;
    RTB_TRY(sc.in(b, &bv));
    const int es = dtype_size(b->dtype);
    PackedPtr p(new rten_packed(), PackedFree{ctx});
    p->kind = 0;
    p->dtype = b->dtype;
    p->K = bv.shape[0];
    p->N = bv.shape[1];
    p->ld = round_up(std::max<int64_t>(p->K, 1), 16 / es);
    RTB_TRY(pool_alloc(ctx, (size_t)std::max<int64_t>(p->N * p->ld, 1) * es, &p->data));
    RTB_CUDA(ctx, cudaMemsetAsync(p->data, 0, (size_t)std::max<int64_t>(p->N * p->ld, 1) * es, ctx->stream));
    long long shape[2] = {p->N, p->K}, ss[2] = {bv.strides[1], bv.strides[0]}, ds[2] = {p->ld, 1};
    RTB_TRY(launch_nd_copy(ctx, es, bv.data, p->data, 2, shape, ss, ds));
    if (es == 1 && p->N > 0) {
        RTB_TRY(pool_alloc(ctx, (size_t)p->N * 4, (void**)&p->colsum));
        RTB_TRY(launch_rowsum8(ctx, p->data, p->dtype == RTEN_I8, p->N, (int)p->K, p->ld, p->colsum));
    }
    RTB_TRY(sc.finish(RTEN_OK));
    *out = p.release();
    return RTEN_OK;
}

void rten_b200_packed_free(rten_ctx* ctx, rten_packed* p) {
    if (!p) return;
    for (rten_packed* ph : p->phases) rten_b200_packed_free(ctx, ph);
    if (ctx) {
        pool_free(ctx, p->data);
        pool_free(ctx, p->colsum);
    }
    if (p->x3) cudaFree(p->x3);
    delete p;
}

// ---- Gemm ---------------------------------------------------------------------------------
rten_status rten_b200_gemm(rten_ctx* ctx, const rten_tensor* a, const rten_tensor* b, const rten_tensor* c, float alpha,
                           float beta, int trans_a, int trans_b, rten_tensor* out) {
    RTB_TRY(check_ctx(ctx));
    if (!a || !b || !out) return fail(ctx, RTEN_ERR_MISSING_INPUTS, "missing inputs");
    if (a->dtype != RTEN_F32 || b->dtype != RTEN_F32 || (c && c->dtype != RTEN_F32))
        return fail(ctx, RTEN_ERR_UNSUPPORTED_TYPE, "unsupported type");
    if (a->ndim != 2 || b->ndim != 2) return fail(ctx, RTEN_ERR_INVALID_VALUE, "input must have 2 dims");
    OpScope sc(ctx);
    rten_tensor av, bv, cv;
    RTB_TRY(sc.in(a, &av));
    RTB_TRY(sc.in(b, &bv));
    if (c) RTB_TRY(sc.in(c, &cv));
    auto transpose = [](rten_tensor& t) {
        std::swap(t.shape[0], t.shape[1]);
        std::swap(t.strides[0], t.strides[1]);
    };
    if (trans_a) transpose(av);
    if (trans_b) transpose(bv);
    if (av.shape[1] != bv.shape[0])
        return fail(ctx, RTEN_ERR_INCOMPATIBLE_SHAPES, "Columns of first matrix does not match rows of second matrix");
    MatMulArgs A{};
    A.kind = 0;
    A.a = &av;
    A.b = &bv;
    A.pb = nullptr;
    A.out_dtype = RTEN_F32;
    A.epi.alpha = alpha;
    const int64_t M = av.shape[0], N = bv.shape[1];
    if (c && beta != 0.0f) {
        // broadcast c to [M, N] (matmul.rs:63-67)
        int64_t cs[2] = {0, 0};
        if (cv.ndim > 2) return fail(ctx, RTEN_ERR_INCOMPATIBLE_SHAPES, "Cannot broadcast c to output shape");
        for (int i = 0; i < cv.ndim; i++) {
            const int od = 2 - cv.ndim + i;
            const int64_t want = od == 0 ? M : N;
            if (cv.shape[i] == want)
                cs[od] = cv.strides[i];
            else if (cv.shape[i] == 1)
                cs[od] = 0;
            else
                return fail(ctx, RTEN_ERR_INCOMPATIBLE_SHAPES, "Cannot broadcast c to output shape");
        }
        A.epi.r = (const float*)cv.data;
        A.epi.r_scale = beta;
        A.epi.r_row = cs[0];
        A.epi.r_col = cs[1];
    }
    // matmul_core's residual plumbing is for same-shape tensors; C is already set in epi.
    return sc.finish(matmul_core(sc, A, out));
}

// ---- MatMul / FusedMatMul -----------------------------------------------------------------
rten_status rten_b200_matmul_ex(rten_ctx* ctx, const rten_tensor* a, const rten_tensor* b, const rten_packed* pb,
                                const rten_tensor* bias, float alpha, const rten_tensor* residual, int activation,
                                rten_tensor* out) {
    RTB_TRY(check_ctx(ctx));
    if (!a || !b || !out) return fail(ctx, RTEN_ERR_MISSING_INPUTS, "missing inputs");
    if (a->dtype != RTEN_F32 || b->dtype != RTEN_F32 || (pb && pb->dtype != RTEN_F32))
        return fail(ctx, RTEN_ERR_UNSUPPORTED_TYPE, "unsupported type");
    OpScope sc(ctx);
    rten_tensor av, bv, biasv, biasc;
    RTB_TRY(sc.in(a, &av));
    if (pb) {
        bv = *b;  // only the shape is consulted
        bv.data = nullptr;
    } else {
        RTB_TRY(sc.in(b, &bv));
    }
    MatMulArgs A{};
    A.kind = 0;
    A.a = &av;
    A.b = &bv;
    A.pb = pb;
    A.out_dtype = RTEN_F32;
    A.epi.alpha = alpha;
    A.epi.act = activation;
    A.residual = residual;
    if (bias) {
        if (bias->dtype != RTEN_F32 || bias->ndim != 1) return fail(ctx, RTEN_ERR_CAST_FAILED, "bias must be a float vector");
        RTB_TRY(sc.in(bias, &biasv));
        RTB_TRY(sc.contiguous(&biasv, &biasc));
        const int64_t N = bv.ndim >= 2 ? bv.shape[bv.ndim - 1] : 1;
        if (biasc.shape[0] != N) return fail(ctx, RTEN_ERR_INVALID_VALUE, "WrongBiasSize");
        A.epi.bias = (const float*)biasc.data;
        A.epi.bias_kind = 1;
    }
    return sc.finish(matmul_core(sc, A, out));
}

rten_status rten_b200_matmul(rten_ctx* ctx, const rten_tensor* a, const rten_tensor* b, const rten_packed* pb,
                             const rten_tensor* bias, float alpha, rten_tensor* out) {
    return rten_b200_matmul_ex(ctx, a, b, pb, bias, alpha, nullptr, 0, out);
}

// ---- MatMulNBits ----------------------------------------------------------------------------
rten_status rten_b200_matmul_nbits(rten_ctx* ctx, const rten_tensor* a, const rten_tensor* b, const rten_tensor* scales,
                                   int bits, int block_size, rten_tensor* out) {
    RTB_TRY(check_ctx(ctx));
    if (!a || !b || !scales || !out) return fail(ctx, RTEN_ERR_MISSING_INPUTS, "missing inputs");
    if (a->dtype != RTEN_F32 || scales->dtype != RTEN_F32 || b->dtype != RTEN_U8 || b->ndim != 3)
        return fail(ctx, RTEN_ERR_CAST_FAILED, "MatMulNBits: A and scales must be f32, B u8 [N, k_blocks, blob_bytes]");
    OpScope sc(ctx);
    return sc.finish(matmul_nbits(sc, a, b, scales, bits, block_size, out));
}

// ---- MatMulInteger / MatMulIntegerToFloat ------------------------------------------------------
rten_status rten_b200_matmul_integer(rten_ctx* ctx, const rten_tensor* a, const rten_tensor* b, const rten_packed* pb,
                                     const rten_tensor* a_zp, const rten_tensor* b_zp, const rten_tensor* scale,
                                     rten_tensor* out) {
    return rten_b200_matmul_integer_ex(ctx, a, b, pb, a_zp, b_zp, scale, nullptr, nullptr, nullptr, 0, nullptr, out);
}

rten_status rten_b200_matmul_integer_ex(rten_ctx* ctx, const rten_tensor* a, const rten_tensor* b, const rten_packed* pb,
                                        const rten_tensor* a_zp, const rten_tensor* b_zp, const rten_tensor* scale,
                                        const rten_tensor* scale_b, const rten_tensor* bias, const rten_tensor* residual,
                                        int activation, rten_tensor* out_range, rten_tensor* out) {
    RTB_TRY(check_ctx(ctx));
    if (!a || !b || !out) return fail(ctx, RTEN_ERR_MISSING_INPUTS, "missing inputs");
    if ((bias || residual || activation || scale_b) && !scale)
        return fail(ctx, RTEN_ERR_INVALID_VALUE, "bias / residual / activation follow the float conversion: a scale is required");
    if (activation < 0 || activation > 3) return fail(ctx, RTEN_ERR_INVALID_VALUE, "unknown activation");
    auto is8 = [](int dt) { return dt == RTEN_U8 || dt == RTEN_I8; };
    if (!is8(a->dtype) || !is8(b->dtype)) return fail(ctx, RTEN_ERR_UNSUPPORTED_TYPE, "unsupported type");
    const int64_t a_rows = a->ndim > 1 ? a->shape[a->ndim - 2] : 1;
    const int64_t b_cols = b->ndim > 1 ? b->shape[b->ndim - 1] : 1;
    RTB_TRY(check_zero_point(ctx, a_zp, a_rows, a->dtype));
    RTB_TRY(check_zero_point(ctx, b_zp, b_cols, b->dtype));
    OpScope sc(ctx);
    rten_tensor av, bv, sv, svc;
    RTB_TRY(sc.in(a, &av));
    if (pb && pb->dtype == b->dtype) {
        bv = *b;
        bv.data = nullptr;
    } else {
        pb = nullptr;
        RTB_TRY(sc.in(b, &bv));
    }
    MatMulArgs A{};
    A.kind = 1;
    A.a = &av;
    A.b = &bv;
    A.pb = pb;
    A.a_zp = a_zp;
    A.b_zp = b_zp;
    A.out_dtype = scale ? RTEN_F32 : RTEN_I32;
    if (scale) {
        // OutputScale::from_view (matmul.rs:712-721)
        if (scale->dtype != RTEN_F32) return fail(ctx, RTEN_ERR_CAST_FAILED, "scale must be float");
        if (scale->ndim > 1) return fail(ctx, RTEN_ERR_INVALID_VALUE, "scale should have rank 0 or 1");
        RTB_TRY(sc.in(scale, &sv));
        RTB_TRY(sc.contiguous(&sv, &svc));
        const int64_t len = svc.ndim == 0 ? 1 : svc.shape[0];
        if (len != 1 && len != b_cols) return fail(ctx, RTEN_ERR_INCOMPATIBLE_SHAPES, "Scale length does not match tensor columns");
        A.epi.scale = (const float*)svc.data;
        A.epi.scale_len = (int)len;
    }
    rten_tensor biasv, biasc, s2v;
    if (scale_b) {
        if (scale_b->dtype != RTEN_F32 || numel(scale_b) != 1)
            return fail(ctx, RTEN_ERR_INVALID_VALUE, "the second scale factor must be a float scalar");
        RTB_TRY(sc.in(scale_b, &s2v));
        A.epi.scale2 = (const float*)s2v.data;
    }
    if (bias) {
        if (bias->dtype != RTEN_F32 || bias->ndim != 1) return fail(ctx, RTEN_ERR_CAST_FAILED, "bias must be a float vector");
        RTB_TRY(sc.in(bias, &biasv));
        RTB_TRY(sc.contiguous(&biasv, &biasc));
        if (biasc.shape[0] != b_cols) return fail(ctx, RTEN_ERR_INVALID_VALUE, "WrongBiasSize");
        A.epi.bias = (const float*)biasc.data;
        A.epi.bias_kind = 1;
    }
    A.epi.act = activation;
    A.residual = residual;
    if (out_range) {
        if (!scale || out_range->dtype != RTEN_I32 || numel(out_range) != 2 || out_range->device < 0 || !is_contiguous(out_range))
            return fail(ctx, RTEN_ERR_INVALID_VALUE, "the output range must be a device-resident i32[2] (float outputs only)");
        A.epi.range = (int*)out_range->data;
    }
    return sc.finish(matmul_core(sc, A, out));
}

}  // extern "C"
