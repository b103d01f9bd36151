// Operator entry points of the C ABI, Conv family (Conv, ConvInteger(ToFloat), weight prepack) and pooling:
// shape / argument validation with the reference's error strings,
// operand normalisation (K-major, TMA-addressable), kernel dispatch.  Mirrors, per function, the
// reference operator named in include/rten_b200.h.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <numeric>
#include <vector>

#include "api_shared.h"
#include "api_util.h"
#include "depthwise.h"
#include "resize.h"
#include "rowops.h"
#include "skinny.h"
#include "umma_gemm.h"

using namespace rtb;
using namespace rtb::api;

namespace {

struct ConvArgs {
    int kind;  // 0 f32, 1 int8
    const rten_tensor* x;
    const rten_tensor* w;
    const rten_packed* pw;
    const rten_tensor* bias = nullptr;
    const rten_conv_params* p;
    const rten_tensor* residual = nullptr;
    int act = 0;                              // apply_act code (math.cuh)
    float act_alpha = 0.0f, act_beta = 0.0f;  // HardSigmoid's alpha / beta (act 6)
    const rten_tensor* x_zp = nullptr;
    const rten_tensor* w_zp = nullptr;
    const rten_tensor* scale = nullptr;
    const rten_tensor* scale_b = nullptr;  // optional second scalar factor (x_scale of a DynamicQuantizeLinear)
    const rten_tensor* out_range = nullptr;  // optional i32[2] device tensor: (min, max) of the output, ordered-int encoded
    // 3xTF32: low parts of x computed by the caller, laid out like x (same strides), used when x is read in place
    const void* x_lo = nullptr;
    bool cache_x3 = true;  // pw outlives the call: its 3xTF32 split may be cached with it
};

rten_status pack_conv_weight(rten_ctx* ctx, const rten_tensor* w, int esize, void* dst) {
    // OIHW (any strides) -> [O, kh, kw, C]
    const int64_t O = w->shape[0], Cg = w->shape[1], kh = w->shape[2], kw = w->shape[3];
    long long shape[4] = {O, kh, kw, Cg};
    long long ss[4] = {w->strides[0], w->strides[2], w->strides[3], w->strides[1]};
    long long ds[4] = {kh * kw * Cg, kw * Cg, Cg, 1};
    return launch_nd_copy(ctx, esize, w->data, dst, 4, shape, ss, ds);
}

// t (3-D, the [B, C, W] of a 1-D convolution) as the 4-D [B, C, 1, W]
void expand_1d(rten_tensor& t) {
    t.ndim = 4;
    t.shape[3] = t.shape[2];
    t.strides[3] = t.strides[2];
    t.shape[2] = 1;
    t.strides[2] = 0;
}

// Validated geometry of one convolution (2-D form: a 1-D convolution is a 2-D one over a height-1 image).
struct ConvShape {
    rten_tensor x, w, bias_v;
    bool one_d = false;
    int64_t strides[2], dil[2];
    int64_t B, C, H, W, O, Cg, kh, kw, OH, OW, pt, pb, pl, pr, Og;
    int groups;
};

rten_status conv_shape(OpScope& sc, const ConvArgs& A, ConvShape& S) {
    rten_ctx* ctx = sc.ctx;
    const rten_conv_params* cp = A.p;
    rten_tensor& x = S.x;
    rten_tensor& w = S.w;
    RTB_TRY(sc.in(A.x, &x));
    RTB_TRY(sc.in(A.w, &w));
    // 1-D convolution via 2-D (conv.rs:142-185)
    const bool one_d = S.one_d = x.ndim == 3;
    int64_t pads_in[4] = {cp->pads[0], cp->pads[1], cp->pads[2], cp->pads[3]};
    int64_t* strides = S.strides;
    int64_t* dil = S.dil;
    strides[0] = cp->strides[0];
    strides[1] = cp->strides[1];
    dil[0] = cp->dilations[0];
    dil[1] = cp->dilations[1];
    if (one_d) {
        if (w.ndim != 3) return fail(ctx, RTEN_ERR_INVALID_VALUE, "input must have 3 dims (OCW)");
        if (cp->n_strides != 1) return fail(ctx, RTEN_ERR_INVALID_VALUE, "expected 1 stride value");
        if (cp->n_dilations != 1) return fail(ctx, RTEN_ERR_INVALID_VALUE, "expected 1 dilation value");
        expand_1d(x);
        expand_1d(w);
        strides[1] = strides[0];
        strides[0] = 1;
        dil[1] = dil[0];
        dil[0] = 1;
        pads_in[1] = cp->pads[0];
        pads_in[3] = cp->pads[1];
        pads_in[0] = pads_in[2] = 0;
    } else {
        if (x.ndim != 4) return fail(ctx, RTEN_ERR_INVALID_VALUE, "input must have 4 dims (NCHW)");
        if (w.ndim != 4) return fail(ctx, RTEN_ERR_INVALID_VALUE, "input must have 4 dims (OCHW)");
        if (cp->n_strides != 2) return fail(ctx, RTEN_ERR_INVALID_VALUE, "expected 2 stride values");
        if (cp->n_dilations != 2) return fail(ctx, RTEN_ERR_INVALID_VALUE, "expected 2 dilation values");
    }
    S.B = x.shape[0];
    const int64_t C = S.C = x.shape[1], H = S.H = x.shape[2], W = S.W = x.shape[3];
    const int64_t O = S.O = w.shape[0], Cg = S.Cg = w.shape[1], kh = S.kh = w.shape[2], kw = S.kw = w.shape[3];
    if (A.bias) {
        RTB_TRY(sc.in(A.bias, &S.bias_v));
        if (S.bias_v.ndim != 1 || S.bias_v.shape[0] != O)
            return fail(ctx, RTEN_ERR_INCOMPATIBLE_SHAPES, "bias.size(0) != out_channels");
    }
    RTB_TRY(axis_out(ctx, H, kh, strides[0], cp->auto_pad_same != 0, pads_in[0], pads_in[2], dil[0], &S.OH, &S.pt, &S.pb));
    RTB_TRY(axis_out(ctx, W, kw, strides[1], cp->auto_pad_same != 0, pads_in[1], pads_in[3], dil[1], &S.OW, &S.pl, &S.pr));
    const int groups = S.groups = cp->groups;
    if (groups == 0) return fail(ctx, RTEN_ERR_INVALID_VALUE, "Group count must be > 0");
    if (groups < 0 || C % groups != 0) return fail(ctx, RTEN_ERR_INVALID_VALUE, "Input channel count not divisible by groups");
    if (C / groups != Cg)
        return fail(ctx, RTEN_ERR_INCOMPATIBLE_SHAPES, "Input channels (per group) does not match kernel input channels");
    if (O % groups != 0) return fail(ctx, RTEN_ERR_INVALID_VALUE, "Output channel count not divisible by groups");
    S.Og = O / groups;
    return RTEN_OK;
}

rten_status check_packed(rten_ctx* ctx, const ConvArgs& A, const ConvShape& S) {
    if (A.pw && (A.pw->kind != 1 || A.pw->O != S.O || A.pw->Cg != S.Cg || A.pw->kh != S.kh || A.pw->kw != S.kw))
        return fail(ctx, RTEN_ERR_INVALID_VALUE, "prepacked conv weight does not match the kernel shape");
    return RTEN_OK;
}

// Weights as [O, kh, kw, C]: the prepacked handle, or packed per call (the reference prepacks per call too)
rten_status conv_weight(rten_ctx* ctx, const ConvArgs& A, const ConvShape& S, int esize, const void** wp,
                        const int32_t** colsum) {
    *colsum = nullptr;
    if (A.pw) {
        RTB_TRY(check_packed(ctx, A, S));
        *wp = A.pw->data;
        *colsum = A.pw->colsum;
        return RTEN_OK;
    }
    void* buf = nullptr;
    RTB_TRY(temp_alloc(ctx, (size_t)(S.O * S.kh * S.kw * S.Cg) * esize, &buf));
    RTB_TRY(pack_conv_weight(ctx, &S.w, esize, buf));
    *wp = buf;
    return RTEN_OK;
}

// An output [B, C, OH, OW] ([B, C, OW] when one_d) laid out like the input x: channels-last when x is (channel stride 1,
// more than one channel), else NCHW
struct OutLayout {
    int ndim = 0;
    int64_t shape[4], strides[4];
};

OutLayout layout_like(const rten_tensor& x, bool one_d, int64_t B, int64_t C, int64_t OH, int64_t OW) {
    const bool cl = x.strides[1] == 1 && x.shape[1] > 1;
    const int64_t shape[4] = {B, C, OH, OW};
    const int64_t strides[4] = {C * OH * OW, cl ? 1 : OH * OW, cl ? OW * C : OW, cl ? C : 1};
    OutLayout l;
    for (int i = 0; i < 4; i++)
        if (!one_d || i != 2) {
            l.shape[l.ndim] = shape[i];
            l.strides[l.ndim++] = strides[i];
        }
    return l;
}

// The output of an op on x, allocated here (when out->data is null) in x's layout; *ov is its 4-D view
rten_status out_like(OpScope& sc, rten_tensor* out, int dtype, const rten_tensor& x, bool one_d, int64_t B, int64_t C,
                     int64_t OH, int64_t OW, rten_tensor* ov) {
    const OutLayout l = layout_like(x, one_d, B, C, OH, OW);
    RTB_TRY(sc.out(out, dtype, l.ndim, l.shape, ov, out->data ? nullptr : l.strides));
    if (one_d) expand_1d(*ov);
    return RTEN_OK;
}

// x (4-D) as the implicit-GEMM kernel addresses it: channels-last with a 16-byte aligned base and pixel strides.  That is
// x itself when it qualifies, else a channels-last copy in a temp.  A padded copy (pt, pl, pb, pr) is always made, its
// border filled with `fill` (the reference's pad value of a u8 image).
rten_status nhwc_input(rten_ctx* ctx, const rten_tensor& x, rten_tensor* xs, int64_t pt = 0, int64_t pl = 0, int64_t pb = 0,
                       int64_t pr = 0, uint8_t fill = 0) {
    const int es = dtype_size(x.dtype);
    const bool padded = (pt | pl | pb | pr) != 0;
    *xs = x;
    if (!padded && x.strides[1] == 1 && reinterpret_cast<uintptr_t>(x.data) % 16 == 0 && (x.strides[3] * es) % 16 == 0 &&
        (x.strides[2] * es) % 16 == 0 && (x.strides[0] * es) % 16 == 0)
        return RTEN_OK;
    const int64_t B = x.shape[0], C = x.shape[1], H = x.shape[2], W = x.shape[3], Hp = H + pt + pb, Wp = W + pl + pr;
    void* buf = nullptr;
    RTB_TRY(temp_alloc(ctx, (size_t)(B * Hp * Wp * C) * es, &buf));
    if (padded) RTB_TRY(launch_fill8(ctx, buf, B * Hp * Wp * C, fill));
    long long shape[4] = {B, H, W, C};
    long long ss[4] = {x.strides[0], x.strides[2], x.strides[3], x.strides[1]};
    long long ds[4] = {Hp * Wp * C, Wp * C, C, 1};
    RTB_TRY(launch_nd_copy(ctx, es, x.data, (uint8_t*)buf + ((pt * Wp + pl) * C) * es, 4, shape, ss, ds));
    xs->data = buf;
    xs->shape[2] = Hp;
    xs->shape[3] = Wp;
    xs->strides[0] = Hp * Wp * C;
    xs->strides[1] = 1;
    xs->strides[2] = Wp * C;
    xs->strides[3] = C;
    return RTEN_OK;
}

// (c, x, y, b) of `channels` channels of a 4-D channels-last view, from element offset `off`: an implicit-GEMM A operand
OperandDesc nhwc(const rten_tensor& v, int64_t channels, int64_t off = 0) {
    OperandDesc d;
    d.base = (const uint8_t*)v.data + off * dtype_size(v.dtype);
    d.dims[0] = channels;
    d.dims[1] = v.shape[3];
    d.dims[2] = v.shape[2];
    d.dims[3] = v.shape[0];
    d.strides[1] = v.strides[3];
    d.strides[2] = v.strides[2];
    d.strides[3] = v.strides[0];
    return d;
}

// (c, o, tap) of a packed conv weight [O, taps, C]: an implicit-GEMM B operand
OperandDesc packed_weight(const void* w, int64_t C, int64_t O, int64_t taps) {
    OperandDesc d;
    d.base = w;
    d.dims[0] = C;
    d.dims[1] = O;
    d.dims[2] = taps;
    d.strides[1] = taps * C;
    d.strides[2] = C;
    return d;
}

// Conv-mode launch geometry of one group of S: M output pixels, N = Og, K = kh*kw*Cg
void conv_geom(GemmLaunch& L, const ConvShape& S) {
    L.conv = 1;
    L.M = (int)(S.B * S.OH * S.OW);
    L.N = (int)S.Og;
    L.K = (int)(S.kh * S.kw * S.Cg);
    ConvGeom& g = L.g;
    g.B = (int)S.B;
    g.H = (int)S.H;
    g.W = (int)S.W;
    g.C = (int)S.Cg;
    g.OH = (int)S.OH;
    g.OW = (int)S.OW;
    g.kh = (int)S.kh;
    g.kw = (int)S.kw;
    g.sy = (int)S.strides[0];
    g.sx = (int)S.strides[1];
    g.dy = (int)S.dil[0];
    g.dx = (int)S.dil[1];
    g.pt = (int)S.pt;
    g.pl = (int)S.pl;
}

// Points the epilogue at the 4-D output view v (f32 or i32) from channel c0 on
void epi_out(EpilogueDesc& e, const rten_tensor& v, int64_t c0 = 0) {
    e.d = (uint8_t*)v.data + (size_t)(c0 * v.strides[1]) * 4;
    e.d_is_i32 = v.dtype == RTEN_I32;
    e.s_z0 = v.strides[0];
    e.s_row = v.strides[2];
    e.s_z1 = v.strides[3];
    e.s_col = v.strides[1];
}

// ... and its residual at the 4-D view r
void epi_residual(EpilogueDesc& e, const rten_tensor& r, int64_t c0 = 0) {
    e.r = (const float*)r.data + c0 * r.strides[1];
    e.r_scale = 1.0f;
    e.r_z0 = r.strides[0];
    e.r_row = r.strides[2];
    e.r_z1 = r.strides[3];
    e.r_col = r.strides[1];
}

rten_status conv_core(OpScope& sc, ConvArgs& A, rten_tensor* out) {
    rten_ctx* ctx = sc.ctx;
    ConvShape S;
    RTB_TRY(conv_shape(sc, A, S));
    const rten_tensor& x = S.x;
    const rten_tensor& w = S.w;
    const bool one_d = S.one_d;
    const int64_t* strides = S.strides;
    const int64_t* dil = S.dil;
    const int64_t B = S.B, C = S.C, H = S.H, W = S.W, O = S.O, Cg = S.Cg, kh = S.kh, kw = S.kw;
    const int64_t OH = S.OH, OW = S.OW, pt = S.pt, pb = S.pb, pl = S.pl, pr = S.pr, Og = S.Og;
    const int groups = S.groups;

    // ---- output (layout follows the input: channels-last in -> channels-last out)
    const int out_dtype = (A.kind == 1 && !A.scale) ? RTEN_I32 : RTEN_F32;
    rten_tensor ov;
    RTB_TRY(out_like(sc, out, out_dtype, x, one_d, B, O, OH, OW, &ov));
    if (B * O * OH * OW == 0) return RTEN_OK;

    const int esize = A.kind == 0 ? 4 : 1;
    RTB_TRY(check_packed(ctx, A, S));

    // ---- integer zero points (x_zp scalar, w_zp per output channel), as given
    const bool x_signed = x.dtype == RTEN_I8, w_signed = w.dtype == RTEN_I8;
    rten_tensor xz_v{}, wz_v{};
    if (A.kind == 1) {
        if (A.x_zp) {
            RTB_TRY(sc.in(A.x_zp, &xz_v));
            if (numel(&xz_v) != 1) return fail(ctx, RTEN_ERR_INVALID_VALUE, "input zero point must be a scalar");
            if (xz_v.dtype != x.dtype) return fail(ctx, RTEN_ERR_CAST_FAILED, "zero point type does not match its tensor");
        }
        if (A.w_zp) {
            RTB_TRY(check_zero_point(ctx, A.w_zp, O, w.dtype));
            RTB_TRY(sc.in(A.w_zp, &wz_v));
        }
    }
    const float *scale_p = nullptr, *scale2_p = nullptr;
    if (A.scale) {
        rten_tensor s;
        RTB_TRY(sc.in(A.scale, &s));
        if (numel(&s) != 1 || s.ndim > 1) return fail(ctx, RTEN_ERR_INVALID_VALUE, "scale should be a scalar");
        scale_p = (const float*)s.data;
    }
    if (A.scale_b) {
        rten_tensor s;
        RTB_TRY(sc.in(A.scale_b, &s));
        if (s.dtype != RTEN_F32 || numel(&s) != 1) return fail(ctx, RTEN_ERR_INVALID_VALUE, "scale should be a scalar");
        scale2_p = (const float*)s.data;
    }
    int* range_p = nullptr;
    if (A.out_range) {
        if (A.out_range->dtype != RTEN_I32 || numel(A.out_range) != 2 || A.out_range->device < 0 || !is_contiguous(A.out_range))
            return fail(ctx, RTEN_ERR_INVALID_VALUE, "the output range must be a device-resident i32[2]");
        range_p = (int*)A.out_range->data;
    }
    rten_tensor res_v;
    if (A.residual) {
        RTB_TRY(sc.in(A.residual, &res_v));
        if (res_v.ndim != (one_d ? 3 : 4)) return fail(ctx, RTEN_ERR_INCOMPATIBLE_SHAPES, "residual shape does not match output");
        if (one_d) expand_1d(res_v);
        for (int i = 0; i < 4; i++)
            if (res_v.shape[i] != ov.shape[i]) return fail(ctx, RTEN_ERR_INCOMPATIBLE_SHAPES, "residual shape does not match output");
    }

    // ---- depthwise (the reference's condition, src/ops/conv.rs:248-284: not the pointwise case, then C == O and
    //      groups == C): one direct launch on x, w (or its pack) and the zero points as they are
    const bool pointwise_1x1 = kh == 1 && kw == 1 && (pt | pb | pl | pr) == 0 && groups == 1 && strides[0] == 1 &&
                               strides[1] == 1 && dil[0] == 1 && dil[1] == 1;
    if (C == O && groups == C && !pointwise_1x1) {
        DepthwiseParams d;
        d.x_dtype = x.dtype;
        d.w_dtype = w.dtype;
        d.B = (int)B;
        d.C = (int)C;
        d.H = (int)H;
        d.W = (int)W;
        d.OH = (int)OH;
        d.OW = (int)OW;
        d.kh = (int)kh;
        d.kw = (int)kw;
        d.sy = (int)strides[0];
        d.sx = (int)strides[1];
        d.dy = (int)dil[0];
        d.dx = (int)dil[1];
        d.pt = (int)pt;
        d.pl = (int)pl;
        d.x = x.data;
        d.out = ov.data;
        for (int i = 0; i < 4; i++) {
            d.xs[i] = x.strides[i];
            d.os[i] = ov.strides[i];
        }
        if (A.pw) {  // [C, kh, kw, 1]
            d.w = A.pw->data;
            d.ws_c = kh * kw;
            d.ws_h = kw;
            d.ws_w = 1;
        } else {
            d.w = w.data;
            d.ws_c = w.strides[0];
            d.ws_h = w.strides[2];
            d.ws_w = w.strides[3];
        }
        if (A.bias) {
            d.bias = (const float*)S.bias_v.data;
            d.bias_stride = S.bias_v.strides[0];
        }
        if (A.residual) {
            d.res = (const float*)res_v.data;
            for (int i = 0; i < 4; i++) d.rs[i] = res_v.strides[i];
        }
        d.act = A.act;
        d.act_alpha = A.act_alpha;
        d.act_beta = A.act_beta;
        if (A.kind == 1) {
            d.x_zp = A.x_zp ? xz_v.data : nullptr;
            d.w_zp = A.w_zp ? wz_v.data : nullptr;
            d.w_zp_stride = (A.w_zp && wz_v.ndim == 1) ? wz_v.strides[0] : 0;
            d.scale = scale_p;
            d.scale_b = scale2_p;
            d.range = range_p;
        }
        return launch_depthwise(ctx, d);
    }

    const void* wp = nullptr;
    const int32_t* w_colsum = nullptr;
    RTB_TRY(conv_weight(ctx, A, S, esize, &wp, &w_colsum));
    const uint8_t* za8 = nullptr;  // x zero point (GEMM A operand = activations): the 8-bit scalar as it is
    const int32_t* zb = nullptr;   // w zero points per column
    int zb_len = 0;
    int pad_value = 0;
    if (A.kind == 1) {
        // padded taps: literal 0 in the reference's shifted-i8 domain (rten-gemm/src/im2col.rs:340-358)
        // == 128 for u8 images, 0 for i8 images
        pad_value = x_signed ? 0 : 128;
        if (A.x_zp) {
            za8 = (const uint8_t*)xz_v.data;  // scalar: read in place by the epilogue
            if (!w_colsum) {
                int32_t* cs = nullptr;
                RTB_TRY(temp_alloc(ctx, (size_t)O * 4, (void**)&cs));
                RTB_TRY(launch_rowsum8(ctx, wp, w_signed, O, (int)(kh * kw * Cg), kh * kw * Cg, cs));
                w_colsum = cs;
            }
        }
        if (A.w_zp) {
            zb_len = wz_v.ndim == 0 ? 1 : (int)wz_v.shape[0];
            int32_t* p = nullptr;
            RTB_TRY(temp_alloc(ctx, (size_t)zb_len * 4, (void**)&p));
            RTB_TRY(launch_zp_to_i32(ctx, wz_v.data, w_signed, zb_len, wz_v.ndim == 0 ? 0 : wz_v.strides[0], p));
            zb = p;
        }
    }

    // ---- choose the addressing path
    //  implicit: x channels-last (c stride 1), C_g*esize % 16 == 0, TMA-addressable strides
    //  explicit: materialise the im2col matrix (odd channel counts such as the 3-channel stem)
    const bool need_pad_copy = (A.kind == 1 && !x_signed && (pt | pb | pl | pr) != 0);
    rten_tensor xs = x;  // source tensor for addressing (may be replaced by an NHWC / padded copy)
    bool implicit_ok = (Cg * esize) % 16 == 0 && Cg * esize >= 32;
    if (implicit_ok)  // (u8 images with padding: a copy with the reference's pad value baked in)
        RTB_TRY(need_pad_copy ? nhwc_input(ctx, x, &xs, pt, pl, pb, pr, (uint8_t)pad_value) : nhwc_input(ctx, x, &xs));

    rten_tensor bias_c;
    if (A.bias) RTB_TRY(sc.contiguous(&S.bias_v, &bias_c));
    // the epilogue of output channels [c0, c0 + N)
    auto epilogue = [&](EpilogueDesc& e, int64_t c0) {
        epi_out(e, ov, c0);
        e.act = A.act;
        e.act_alpha = A.act_alpha;
        e.act_beta = A.act_beta;
        if (A.bias) {
            e.bias = (const float*)bias_c.data + c0;
            e.bias_kind = 1;
        }
        if (A.residual) epi_residual(e, res_v, c0);
        if (A.kind == 1) {
            e.za8 = za8;
            e.za8_signed = x_signed;
            e.scale2 = scale2_p;
            e.range = range_p;
            e.colsum = w_colsum ? w_colsum + c0 : nullptr;
            e.zb = zb ? (zb_len == 1 ? zb : zb + c0) : nullptr;
            e.zb_len = zb ? (zb_len == 1 ? 1 : (int)Og) : 0;
            e.scale = scale_p;
            e.scale_len = scale_p ? 1 : 0;
        }
    };

    // ---- small-channel path (the RGB stem: C <= 4 in f32, C <= 16 in 8-bit): a zero-padded copy with `pitch` channels
    //      per pixel, one 128-byte K block per filter row holding kw pixels x pitch channels.  The 8-bit copy also holds
    //      the vertical padding (the reference's pad value); f32 leaves vertical padding / stride to the TMA tile addressing.
    const bool smallc_ok = !implicit_ok && groups == 1 && dil[1] == 1 && (int64_t)B * OH * OW > 0 &&
                           (A.kind == 0 ? Cg <= 4 && kw * 4 <= 32 : Cg <= 16 && kw <= 8 && !zb);
    if (smallc_ok) {
        const bool q8 = A.kind == 1;
        const int64_t pitch = q8 ? 16 : 4, kb = 128 / esize;  // channels per pixel of the copy, elements per K block
        const int64_t Hp = q8 ? H + pt + pb : H;
        // every window of 8 pixels stays inside the padded row
        const int64_t Wp = std::max<int64_t>(q8 ? W + pl + pr : 0, (OW - 1) * strides[1] + 8);
        void *xp = nullptr, *wsm = nullptr;
        RTB_TRY(temp_alloc(ctx, (size_t)(B * Hp * Wp * pitch) * esize, &xp));
        if (q8) {
            RTB_TRY(launch_smallc8_pad(ctx, x.data, xp, (int)B, (int)C, (int)H, (int)W, (int)Hp, (int)Wp, (int)pt, (int)pl,
                                       x.strides[0], x.strides[1], x.strides[2], x.strides[3], pad_value));
        } else {
            RTB_TRY(launch_smallc_pad(ctx, (const float*)x.data, (float*)xp, (int)B, (int)C, (int)H, (int)W, (int)Wp, (int)pl,
                                      x.strides[0], x.strides[1], x.strides[2], x.strides[3]));
        }
        RTB_TRY(temp_alloc(ctx, (size_t)(O * kh * 128), &wsm));
        if (q8) {
            RTB_TRY(launch_smallc8_pack_w(ctx, w.data, wsm, (int)O, (int)C, (int)kh, (int)kw, w.strides[0], w.strides[1],
                                          w.strides[2], w.strides[3]));
        } else {
            RTB_TRY(launch_smallc_pack_w(ctx, (const float*)w.data, (float*)wsm, (int)O, (int)C, (int)kh, (int)kw, w.strides[0],
                                         w.strides[1], w.strides[2], w.strides[3]));
        }
        GemmLaunch L;
        L.kind = A.kind;
        L.a_signed = x_signed;
        L.b_signed = w_signed;
        conv_geom(L, S);
        L.K = (int)(kh * kb);
        L.g.H = (int)Hp;
        L.g.W = (int)OW;  // dim 1 of the A map indexes output columns directly
        L.g.C = (int)kb;
        L.g.kw = 1;
        L.g.sx = 1;
        L.g.pt = q8 ? 0 : (int)pt;
        L.g.pl = 0;
        L.a.base = xp;
        L.a.dims[0] = kb;
        L.a.dims[1] = OW;
        L.a.dims[2] = Hp;
        L.a.dims[3] = B;
        L.a.strides[1] = strides[1] * pitch;
        L.a.strides[2] = Wp * pitch;
        L.a.strides[3] = Hp * Wp * pitch;
        if (!q8 && ctx->f32_mode == RTEN_F32_TF32X3 && !getenv("RTEN_B200_X3_THREE_PLANES")) {
            // 3xTF32: the low parts of the padded copy, once (the window view above overlaps itself 8 / stride times)
            float* xlo = nullptr;
            const long long n = (long long)B * H * Wp * 4;
            RTB_TRY(temp_alloc(ctx, (size_t)n * 4, (void**)&xlo));
            const long long fd[4] = {n, 1, 1, 1}, fs[4] = {1, n, n, n};
            RTB_TRY(launch_tf32x3_split(ctx, (const float*)xp, xlo, fd, fs, n, 2));
            L.a_lo_base = xlo;
        }
        L.b = packed_weight(wsm, kb, O, kh);
        epilogue(L.epi, 0);
        const rten_status st = launch_umma_gemm(ctx, L);
        if (st != RTEN_ERR_UNSUPPORTED_VALUE) return st;
        // otherwise fall through to the generic explicit path
    }

    for (int g = 0; g < groups; g++) {
        GemmLaunch L;
        L.kind = A.kind;
        L.a_signed = x_signed;
        L.b_signed = w_signed;
        L.N = (int)Og;
        L.K = (int)(kh * kw * Cg);
        EpilogueDesc& e = L.epi;
        epilogue(e, g * Og);
        const uint8_t* wg = (const uint8_t*)wp + (size_t)(g * Og * kh * kw * Cg) * esize;

        if (implicit_ok) {
            conv_geom(L, S);
            L.g.H = (int)xs.shape[2];
            L.g.W = (int)xs.shape[3];
            if (need_pad_copy) L.g.pt = L.g.pl = 0;  // (the copy holds the padding)
            L.a = nhwc(xs, Cg, g * Cg);
            L.b = packed_weight(wg, Cg, Og, kh * kw);
            if (A.pw && A.kind == 0 && groups == 1 && wg == A.pw->data && A.cache_x3)
                L.b_x3_slot = &const_cast<rten_packed*>(A.pw)->x3;
            if (A.x_lo && xs.data == x.data) L.a_lo_base = (const float*)A.x_lo + g * Cg;
            if (zb) {
                // per-pixel window sums of the image = N=1 GEMM against an all-ones kernel row
                int32_t* rs = nullptr;
                RTB_TRY(temp_alloc(ctx, (size_t)(B * OH * OW) * 4, (void**)&rs));
                void* ones = nullptr;
                RTB_TRY(temp_alloc(ctx, (size_t)(kh * kw * Cg), &ones));
                RTB_TRY(launch_fill8(ctx, ones, kh * kw * Cg, 1));
                GemmLaunch R = L;
                R.N = 1;
                R.b_signed = 1;
                R.b.base = ones;
                R.b.dims[1] = 1;
                R.epi = EpilogueDesc();
                R.epi.d = rs;
                R.epi.d_is_i32 = 1;
                R.epi.s_z0 = OH * OW;
                R.epi.s_row = OW;
                R.epi.s_z1 = 1;
                R.epi.s_col = B * OH * OW;
                if (const rten_status st = launch_umma_gemm(ctx, R)) return fail(ctx, st, "conv window-sum GEMM could not be launched");
                e.rowsum = rs;
            }
            const rten_status st = launch_umma_gemm(ctx, L);
            if (st != RTEN_ERR_UNSUPPORTED_VALUE) {
                RTB_TRY(st);
                continue;
            }
            // fall through to the explicit path
        }
        // explicit im2col: A = [B*OH*OW, kpad]
        const int64_t Kd = kh * kw * Cg;
        const int64_t kpad = round_up(Kd, 16 / esize);
        void* col = nullptr;
        RTB_TRY(temp_alloc(ctx, (size_t)(B * OH * OW * kpad) * esize, &col));
        Im2ColParams ip;
        ip.B = (int)B;
        ip.C = (int)Cg;
        ip.H = (int)H;
        ip.W = (int)W;
        ip.OH = (int)OH;
        ip.OW = (int)OW;
        ip.kh = (int)kh;
        ip.kw = (int)kw;
        ip.sy = (int)strides[0];
        ip.sx = (int)strides[1];
        ip.dy = (int)dil[0];
        ip.dx = (int)dil[1];
        ip.pt = (int)pt;
        ip.pl = (int)pl;
        ip.c0 = (int)(g * Cg);
        ip.kpad = (int)kpad;
        ip.xs_b = x.strides[0];
        ip.xs_c = x.strides[1];
        ip.xs_h = x.strides[2];
        ip.xs_w = x.strides[3];
        RTB_TRY(launch_im2col(ctx, esize, x.data, col, ip, pad_value));
        L.conv = 0;
        L.M = (int)(B * OH * OW);
        L.z0 = L.z1 = 1;
        L.a = OperandDesc();
        L.a.base = col;
        L.a.dims[0] = Kd;
        L.a.dims[1] = B * OH * OW;
        L.a.strides[1] = kpad;
        L.b = OperandDesc();
        L.b.base = wg;
        L.b.dims[0] = Kd;
        L.b.dims[1] = Og;
        L.b.strides[1] = Kd;
        if (!tma_compatible(L.b, esize, 4)) {
            void* wb = nullptr;
            RTB_TRY(temp_alloc(ctx, (size_t)(Og * kpad) * esize, &wb));
            long long shape[2] = {Og, Kd}, ss[2] = {Kd, 1}, ds[2] = {kpad, 1};
            RTB_TRY(launch_nd_copy(ctx, esize, wg, wb, 2, shape, ss, ds));
            L.b.base = wb;
            L.b.strides[1] = kpad;
        }
        // plain-mode epilogue needs a uniform row stride over (b, oy, ox): use the conv decomposition when the
        // output is not pixel-contiguous by writing through a temp
        const bool uniform = (ov.strides[2] == OW * ov.strides[3]) && (ov.strides[0] == OH * ov.strides[2] || B == 1);
        const bool r_uniform = !A.residual || ((res_v.strides[2] == OW * res_v.strides[3]) &&
                                               (res_v.strides[0] == OH * res_v.strides[2] || B == 1));
        if (zb) {
            int32_t* rs = nullptr;
            RTB_TRY(temp_alloc(ctx, (size_t)(B * OH * OW) * 4, (void**)&rs));
            RTB_TRY(launch_rowsum8(ctx, col, x_signed, B * OH * OW, (int)Kd, kpad, rs));
            e.rowsum = rs;
        }
        if (uniform && r_uniform) {
            e.s_row = ov.strides[3];
            e.s_z0 = e.s_z1 = 0;
            if (A.residual) {
                e.r_row = res_v.strides[3];
                e.r_z0 = e.r_z1 = 0;
            }
            if (const rten_status st = launch_umma_gemm(ctx, L)) return fail(ctx, st, "conv GEMM could not be launched");
        } else {
            // NCHW-style output: GEMM into [pixels, Og] temp (no fusion), then strided copy + residual/act
            void* tmp = nullptr;
            RTB_TRY(temp_alloc(ctx, (size_t)(B * OH * OW * Og) * 4, &tmp));
            EpilogueDesc e2 = e;
            e2.d = tmp;
            e2.s_row = Og;
            e2.s_col = 1;
            e2.s_z0 = e2.s_z1 = 0;
            e2.r = nullptr;
            e2.act = A.residual ? 0 : A.act;
            GemmLaunch L2 = L;
            L2.epi = e2;
            if (const rten_status st = launch_umma_gemm(ctx, L2)) return fail(ctx, st, "conv GEMM could not be launched");
            long long shape[4] = {B, OH, OW, Og};
            long long ss[4] = {OH * OW * Og, OW * Og, Og, 1};
            long long ds[4] = {ov.strides[0], ov.strides[2], ov.strides[3], ov.strides[1]};
            if (A.residual) {
                long long rs4[4] = {res_v.strides[0], res_v.strides[2], res_v.strides[3], res_v.strides[1]};
                RTB_TRY(launch_binary(ctx, RTEN_F32, BIN_ADD, A.act == 1, tmp, e.r, e.d, 4, shape, ss, rs4, ds));
                if (A.act > 1)
                    return fail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "an activation other than Relu after a residual needs a pixel-contiguous output");
            } else {
                RTB_TRY(launch_nd_copy(ctx, 4, tmp, e.d, 4, shape, ss, ds));
            }
        }
    }
    return RTEN_OK;
}

// A 1x1, unpadded convolution over a channels-last, TMA-addressable input whose channels fill whole 128-byte K blocks:
// one side of a folded launch
bool pointwise(const ConvShape& s) {
    return !s.one_d && s.kh == 1 && s.kw == 1 && s.groups == 1 && (s.pt | s.pb | s.pl | s.pr) == 0 && s.dil[0] == 1 &&
           s.dil[1] == 1 && s.x.strides[1] == 1 && s.C % 32 == 0 && tma_compatible(nhwc(s.x, s.C), 4, 4);
}

// The launch of act(Conv(x, w, bias) [+ Conv(x_proj, w_proj, bias_proj)]) into the 4-D view ov: with a projection, ONE
// GEMM over both K ranges (GemmLaunch::proj)
rten_status folded_launch(OpScope& sc, const ConvArgs& M, const ConvShape& sm, const ConvArgs* P, const ConvShape& sp,
                          const rten_tensor& ov, GemmLaunch& L) {
    const void *wm = nullptr, *wpj = nullptr;
    const int32_t* unused = nullptr;
    RTB_TRY(conv_weight(sc.ctx, M, sm, 4, &wm, &unused));
    if (P) RTB_TRY(conv_weight(sc.ctx, *P, sp, 4, &wpj, &unused));
    L.kind = 0;
    conv_geom(L, sm);
    L.a = nhwc(sm.x, sm.C);
    L.b = packed_weight(wm, sm.C, sm.O, 1);
    if (P) {
        L.proj.C = (int)sp.C;
        L.proj.stride = (int)sp.strides[0];
        L.proj.a = nhwc(sp.x, sp.C);
        L.proj.b = packed_weight(wpj, sp.C, sp.O, 1);
    }
    EpilogueDesc& e = L.epi;
    epi_out(e, ov);
    e.act = M.act;
    const bool p_bias = P && P->bias;
    rten_tensor bm, bp;
    if (M.bias) RTB_TRY(sc.contiguous(&sm.bias_v, &bm));
    if (p_bias) RTB_TRY(sc.contiguous(&sp.bias_v, &bp));
    if (M.bias || p_bias) {
        e.bias_kind = 1;
        e.bias = (const float*)(M.bias ? bm.data : bp.data);
        if (M.bias && p_bias) e.bias2 = (const float*)bp.data;
    }
    return RTEN_OK;
}

// act(Conv(x, w, bias) + Conv(x_proj, w_proj, bias_proj)) -- a residual block's last convolution and its projection
// shortcut.  Two 1x1 convolutions over channels-last, TMA-addressable inputs with whole 128-byte channel blocks run as
// ONE GEMM over both K ranges (GemmLaunch::proj): the shortcut tensor is never written.  Anything else computes the
// projection into a temporary and adds it as the residual of the main convolution, exactly as two conv2d_ex calls do.
rten_status conv_projected(OpScope& sc, ConvArgs& M, ConvArgs& P, rten_tensor* out) {
    rten_ctx* ctx = sc.ctx;
    ConvShape sm, sp;
    RTB_TRY(conv_shape(sc, M, sm));
    RTB_TRY(conv_shape(sc, P, sp));
    if (sm.one_d != sp.one_d || sm.B != sp.B || sm.O != sp.O || sm.OH != sp.OH || sm.OW != sp.OW)
        return fail(ctx, RTEN_ERR_INCOMPATIBLE_SHAPES, "projection output shape does not match the convolution's output shape");
    const int64_t B = sm.B, O = sm.O, OH = sm.OH, OW = sm.OW;
    const bool fold = pointwise(sm) && pointwise(sp) && sp.strides[0] == sp.strides[1] && (!out->data || out->device >= 0) &&
                      B * O * OH * OW > 0;
    if (fold) {
        rten_tensor ov;
        RTB_TRY(out_like(sc, out, RTEN_F32, sm.x, false, B, O, OH, OW, &ov));  // (x is channels-last: so is the output)
        GemmLaunch L;
        RTB_TRY(folded_launch(sc, M, sm, &P, sp, ov, L));
        if (M.pw) L.b_x3_slot = &const_cast<rten_packed*>(M.pw)->x3;
        if (P.pw) L.proj.b_x3_slot = &const_cast<rten_packed*>(P.pw)->x3;
        const rten_status st = launch_umma_gemm(ctx, L);
        if (st != RTEN_ERR_UNSUPPORTED_VALUE) return st;
        // (no launch plan takes the plain f32 epilogue for this output: two convolutions)
    }
    // the projection in the layout rten_b200_conv2d_ex would give it, then the main convolution with it as the residual
    const OutLayout l = layout_like(sp.x, sp.one_d, B, O, OH, OW);
    rten_tensor tmp{};
    tmp.dtype = RTEN_F32;
    tmp.device = ctx->device;
    tmp.ndim = l.ndim;
    std::copy(l.shape, l.shape + l.ndim, tmp.shape);
    std::copy(l.strides, l.strides + l.ndim, tmp.strides);
    RTB_TRY(temp_alloc(ctx, (size_t)std::max<int64_t>(B * O * OH * OW, 1) * 4, &tmp.data));
    RTB_TRY(conv_core(sc, P, &tmp));
    M.residual = &tmp;
    return conv_core(sc, M, out);
}

// y = act(Conv(x, w, bias) [+ residual | + Conv(x_proj, ...)]) and z = act_next(Conv1x1(y, w_next, bias_next)): a
// residual block's last convolution and the next block's first.  In single-pass TF32, a 1x1 convolution over a
// channels-last input (with a 1x1 projection, as conv_projected folds it) whose N <= 256 output channels are a multiple
// of 32, followed by a 1x1, stride-1, unpadded convolution to 64 or 128 channels, runs as ONE launch
// (GemmLaunch::chain): z is computed from y's tiles as they are stored, and y is not read back.  Anything else runs as
// the calls it replaces, with the same results.
rten_status conv_chained(OpScope& sc, ConvArgs& M, ConvArgs* P, ConvArgs& Nx, rten_tensor* out, rten_tensor* out_next) {
    rten_ctx* ctx = sc.ctx;
    ConvShape sm, sp, sn;
    RTB_TRY(conv_shape(sc, M, sm));
    if (P) {
        RTB_TRY(conv_shape(sc, *P, sp));
        if (sm.one_d != sp.one_d || sm.B != sp.B || sm.O != sp.O || sm.OH != sp.OH || sm.OW != sp.OW)
            return fail(ctx, RTEN_ERR_INCOMPATIBLE_SHAPES, "projection output shape does not match the convolution's output shape");
    }
    const int64_t B = sm.B, O = sm.O, OH = sm.OH, OW = sm.OW;
    const rten_conv_params* np = Nx.p;
    const bool next_1x1 = Nx.w->ndim == 4 && Nx.w->shape[1] == O && Nx.w->shape[2] == 1 && Nx.w->shape[3] == 1 &&
                          np->groups == 1 && np->n_strides == 2 && np->n_dilations == 2 && np->strides[0] == 1 &&
                          np->strides[1] == 1 && np->dilations[0] == 1 && np->dilations[1] == 1 && !np->auto_pad_same &&
                          (np->pads[0] | np->pads[1] | np->pads[2] | np->pads[3]) == 0;
    const int64_t N2 = Nx.w->ndim == 4 ? Nx.w->shape[0] : 0;
    rten_tensor res_v;
    if (M.residual) RTB_TRY(sc.in(M.residual, &res_v));
    const bool chain = ctx->f32_mode == RTEN_F32_TF32 && next_1x1 && (N2 == 64 || N2 == 128) && O % 32 == 0 && O <= 256 &&
                       pointwise(sm) && (!P || (pointwise(sp) && sp.strides[0] == sp.strides[1])) &&
                       (!M.residual || (res_v.ndim == 4 && res_v.strides[1] == 1)) && (!out->data || out->device >= 0) &&
                       (!out_next->data || out_next->device >= 0) && B * O * OH * OW > 0;
    if (chain) {
        rten_tensor ov, zv;  // (x is channels-last: so are y and z)
        RTB_TRY(out_like(sc, out, RTEN_F32, sm.x, false, B, O, OH, OW, &ov));
        RTB_TRY(out_like(sc, out_next, RTEN_F32, sm.x, false, B, N2, OH, OW, &zv));
        for (int i = 0; M.residual && i < 4; i++)
            if (res_v.shape[i] != ov.shape[i]) return fail(ctx, RTEN_ERR_INCOMPATIBLE_SHAPES, "residual shape does not match output");
        RTB_TRY(conv_shape(sc, Nx, sn));  // (x = y: checks w_next and bias_next against it)
        GemmLaunch L;
        RTB_TRY(folded_launch(sc, M, sm, P, sp, ov, L));
        if (M.residual) epi_residual(L.epi, res_v);
        const void* wn = nullptr;
        const int32_t* unused = nullptr;
        RTB_TRY(conv_weight(ctx, Nx, sn, 4, &wn, &unused));
        GemmLaunch::Chain& c = L.chain;
        c.N2 = (int)N2;
        c.w = packed_weight(wn, O, N2, 1);
        rten_tensor bn;
        if (Nx.bias) {
            RTB_TRY(sc.contiguous(&sn.bias_v, &bn));
            c.bias = (const float*)bn.data;
        }
        c.act = Nx.act;
        c.z = nhwc(zv, N2);
        if (zv.strides[1] == 1) {
            const rten_status st = launch_umma_gemm(ctx, L);
            if (st != RTEN_ERR_UNSUPPORTED_VALUE) return st;
        }
        // (no chained launch for these operands: the separate calls)
    }
    RTB_TRY(P ? conv_projected(sc, M, *P, out) : conv_core(sc, M, out));
    Nx.x = out;
    return conv_core(sc, Nx, out_next);
}

// ---- ConvTranspose as stride-phase convolutions ----------------------------------------------------------------------
// Per spatial axis (input length H, kernel k, stride s, dilation d, top pad pt), output row o receives x[i] * W[k]
// wherever i*s + k*d = o + pt.  The rows o = q + s*j of phase q = o mod s receive exactly the taps k with
// k*d = q + pt (mod s); they step by s / gcd(d, s).  With the taps in decreasing order k_0 > k_1 > ... and
// e_0 = (q + pt - k_0*d) / s, out_q[j] = sum_t x[j + e_0 + t*d/gcd(d, s)] * W[k_t]: a stride-1 convolution with
// dilation d/gcd(d, s), the reversed sub-kernel and top pad -e_0.  The sub-kernel depends only on the residue
// r = (q + pt) mod s, so a prepacked weight holds one per residue.

// Taps of residue r of one axis
struct AxisTaps {
    int64_t T = 0;     // count; 0: a phase with this residue receives only the bias
    int64_t k0 = 0;    // largest tap
    int64_t step = 1;  // s / gcd(d, s)
};

AxisTaps axis_taps(int64_t k, int64_t s, int64_t d, int64_t r) {
    AxisTaps t;
    t.step = s / std::gcd(d, s);
    for (int64_t kk = k - 1; kk >= 0; kk--)
        if ((kk * d) % s == r) {
            if (t.T == 0) t.k0 = kk;
            t.T++;
        }
    return t;
}

// Phase q of one axis as a convolution over rows [row0, row0 + rows) of the input
struct AxisPhase {
    bool live = false;  // has taps that reach the input
    int64_t n = 0;      // output rows q, q + s, ...
    int64_t r = 0;      // residue: which sub-kernel
    AxisTaps taps;
    int64_t dil = 1;
    int64_t row0 = 0, rows = 0, pad0 = 0, pad1 = 0;
};

AxisPhase axis_phase(int64_t H, int64_t OH, int64_t k, int64_t s, int64_t d, int64_t pt, int64_t q) {
    AxisPhase a;
    a.n = q < OH ? (OH - q + s - 1) / s : 0;
    a.r = (q + pt) % s;
    a.taps = axis_taps(k, s, d, a.r);
    a.dil = d / std::gcd(d, s);
    if (a.n == 0 || a.taps.T == 0) return a;
    const int64_t e0 = (q + pt - a.taps.k0 * d) / s;  // exact
    const int64_t last = a.n - 1 + e0 + (a.taps.T - 1) * a.dil;  // last input row any output of the phase reads
    const int64_t r0 = std::max<int64_t>(e0, 0), r1 = std::min<int64_t>(last, H - 1) + 1;
    if (r0 >= r1) return a;  // every window lies in the padding
    a.live = true;
    a.row0 = r0;
    a.rows = r1 - r0;
    a.pad0 = r0 - e0;
    a.pad1 = last - (r1 - 1);
    return a;
}

}  // namespace

// Argument checks in the reference's order (conv_transpose.rs:226-345, conv_transpose_output_size_and_padding
// :144-220) on the kernel `w` (and input `x` when given)
rten_status api::conv_transpose_shape(rten_ctx* ctx, const rten_tensor* xp, const rten_tensor& w0, const rten_tensor* bias,
                                      const rten_conv_transpose_params* cp, ConvTShape& S) {
    const bool one_d = S.one_d = xp ? xp->ndim == 3 : w0.ndim == 3;
    if (xp) S.x = *xp;
    S.w = w0;
    int64_t pads[4] = {cp->pads[0], cp->pads[1], cp->pads[2], cp->pads[3]};
    int64_t st[2] = {cp->strides[0], cp->strides[1]}, dl[2] = {cp->dilations[0], cp->dilations[1]};
    int64_t op[2] = {0, 0};
    const bool same = cp->auto_pad_same != 0;
    if (one_d) {
        if (S.w.ndim != 3) return fail(ctx, RTEN_ERR_INVALID_VALUE, "kernel must have 3 dims (OCW)");
        if (!same && cp->n_pads != 2) return fail(ctx, RTEN_ERR_INVALID_VALUE, "expected 2 pad values");
        if (cp->n_strides != 1) return fail(ctx, RTEN_ERR_INVALID_VALUE, "expected 1 stride value");
        if (cp->n_dilations != 1) return fail(ctx, RTEN_ERR_INVALID_VALUE, "expected 1 dilation value");
        if (cp->n_output_padding != 0 && cp->n_output_padding != 1)
            return fail(ctx, RTEN_ERR_INVALID_VALUE, "expected 1 output_padding value");
        if (xp) expand_1d(S.x);
        expand_1d(S.w);
        pads[0] = pads[2] = 0;
        pads[1] = cp->pads[0];
        pads[3] = cp->pads[1];
        st[1] = st[0];
        st[0] = 1;
        dl[1] = dl[0];
        dl[0] = 1;
        op[1] = cp->n_output_padding ? cp->output_padding[0] : 0;
    } else if (cp->n_output_padding == 2) {
        op[0] = cp->output_padding[0];
        op[1] = cp->output_padding[1];
    }
    const int groups = S.groups = cp->groups;
    if (groups <= 0) return fail(ctx, RTEN_ERR_INVALID_VALUE, "Group count must be > 0");
    if (xp && S.x.ndim != 4) return fail(ctx, RTEN_ERR_INVALID_VALUE, "input must have 4 dims (NCHW)");
    if (S.w.ndim != 4) return fail(ctx, RTEN_ERR_INVALID_VALUE, "kernel must have 4 dims (COHW)");
    const int64_t Cin = S.w.shape[0];
    S.Og = S.w.shape[1];
    S.O = S.Og * groups;
    S.kh = S.w.shape[2];
    S.kw = S.w.shape[3];
    if (bias && (bias->ndim != 1 || bias->shape[0] != S.O))
        return fail(ctx, RTEN_ERR_INCOMPATIBLE_SHAPES, "bias.size(0) != out_channels");
    if (xp && S.x.shape[1] != Cin)
        return fail(ctx, RTEN_ERR_INCOMPATIBLE_SHAPES, "Input channels does not match kernel input channels");
    if (Cin % groups != 0) return fail(ctx, RTEN_ERR_INVALID_VALUE, "Input channel count not divisible by groups");
    S.Cg = Cin / groups;
    if (!one_d) {
        if (cp->n_strides != 2) return fail(ctx, RTEN_ERR_INVALID_VALUE, "expected 2 stride values");
        if (cp->n_dilations != 2) return fail(ctx, RTEN_ERR_INVALID_VALUE, "expected 2 dilation values");
        if (cp->n_output_padding != 0 && cp->n_output_padding != 2)
            return fail(ctx, RTEN_ERR_INVALID_VALUE, "expected 2 output_padding values");
    }
    S.sy = st[0];
    S.sx = st[1];
    S.dy = dl[0];
    S.dx = dl[1];
    if (S.sy <= 0 || S.sx <= 0) return fail(ctx, RTEN_ERR_INVALID_VALUE, "Strides must be > 0");
    if (S.dy <= 0 || S.dx <= 0) return fail(ctx, RTEN_ERR_INVALID_VALUE, "Dilations must be > 0");
    if (S.kh <= 0 || S.kw <= 0) return fail(ctx, RTEN_ERR_INVALID_VALUE, "Kernel size must be > 0");
    if (!xp) return RTEN_OK;  // (prepack: the weight's checks only)
    S.B = S.x.shape[0];
    S.C = S.x.shape[1];
    S.H = S.x.shape[2];
    S.W = S.x.shape[3];
    if (S.H == 0 || S.W == 0) return fail(ctx, RTEN_ERR_INVALID_VALUE, "Input width and height must be > 0");
    if (!same && !one_d && cp->n_pads != 4) return fail(ctx, RTEN_ERR_INVALID_VALUE, "Wrong number of pad values");
    for (int i = 0; i < 4; i++)
        if (!same && pads[i] < 0) return fail(ctx, RTEN_ERR_INVALID_VALUE, "Pads must be >= 0");
    if (op[0] < 0 || op[1] < 0) return fail(ctx, RTEN_ERR_INVALID_VALUE, "Output padding must be >= 0");
    const int64_t keh = (S.kh - 1) * S.dy + 1, kew = (S.kw - 1) * S.dx + 1;
    const int64_t full_h = (S.H - 1) * S.sy + op[0] + keh, full_w = (S.W - 1) * S.sx + op[1] + kew;
    if (same) {
        S.OH = S.H * S.sy;
        S.OW = S.W * S.sx;
        const int64_t ph = full_h - S.OH, pw = full_w - S.OW;
        if (ph < 0 || pw < 0) return fail(ctx, RTEN_ERR_INVALID_VALUE, "Input is too small");
        S.pt = ph / 2;
        S.pb = ph - S.pt;
        S.pl = pw / 2;
        S.pr = pw - S.pl;
    } else {
        S.pt = pads[0];
        S.pl = pads[1];
        S.pb = pads[2];
        S.pr = pads[3];
        S.OH = full_h - S.pt - S.pb;
        S.OW = full_w - S.pl - S.pr;
        if (S.OH < 0 || S.OW < 0) return fail(ctx, RTEN_ERR_INVALID_VALUE, "Input is too small");
    }
    return RTEN_OK;
}

namespace {

// The sub-kernel of residue phase (ty, tx) of W (4-D view) as a conv weight [O, Th, Tw, Cg]
rten_status pack_transpose_phase(rten_ctx* ctx, const ConvTShape& S, const AxisTaps& ty, const AxisTaps& tx, void* dst) {
    ConvTransposePack p;
    p.O = (int)S.O;
    p.Og = (int)S.Og;
    p.Cg = (int)S.Cg;
    p.Th = (int)ty.T;
    p.Tw = (int)tx.T;
    p.ky0 = (int)ty.k0;
    p.kx0 = (int)tx.k0;
    p.step_y = (int)ty.step;
    p.step_x = (int)tx.step;
    p.ws_i = S.w.strides[0];
    p.ws_o = S.w.strides[1];
    p.ws_h = S.w.strides[2];
    p.ws_w = S.w.strides[3];
    return launch_conv_transpose_pack(ctx, (const float*)S.w.data, (float*)dst, p);
}

rten_status conv_transpose_core(OpScope& sc, const rten_tensor* x_in, const rten_tensor* w_in, const rten_packed* pw,
                                const rten_tensor* bias_in, const rten_conv_transpose_params* cp, rten_tensor* out) {
    rten_ctx* ctx = sc.ctx;
    rten_tensor xd, wd, bd;
    RTB_TRY(sc.in(x_in, &xd));
    RTB_TRY(sc.in(w_in, &wd));
    if (bias_in) RTB_TRY(sc.in(bias_in, &bd));
    ConvTShape S;
    RTB_TRY(conv_transpose_shape(ctx, &xd, wd, bias_in ? &bd : nullptr, cp, S));
    const int64_t B = S.B, C = S.C, H = S.H, W = S.W, O = S.O, Cg = S.Cg, OH = S.OH, OW = S.OW;
    const int groups = S.groups;

    // ---- output (layout follows the input: channels-last in -> channels-last out)
    rten_tensor ov;
    RTB_TRY(out_like(sc, out, RTEN_F32, S.x, S.one_d, B, O, OH, OW, &ov));
    if (B * O * OH * OW == 0) return RTEN_OK;
    if (S.sy > 256 || S.sx > 256) return fail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "ConvTranspose strides above 256 are not supported");
    if (pw && (pw->kind != 2 || pw->O != O || pw->Cg != Cg || pw->kh != S.kh || pw->kw != S.kw || pw->groups != groups ||
               pw->sy != S.sy || pw->sx != S.sx || pw->dy != S.dy || pw->dx != S.dx))
        return fail(ctx, RTEN_ERR_INVALID_VALUE, "prepacked conv transpose weight does not match the kernel and parameters");

    std::vector<AxisPhase> py, px;
    for (int64_t q = 0; q < S.sy; q++) py.push_back(axis_phase(H, OH, S.kh, S.sy, S.dy, S.pt, q));
    for (int64_t q = 0; q < S.sx; q++) px.push_back(axis_phase(W, OW, S.kw, S.sx, S.dx, S.pl, q));
    bool any_live = false, any_empty = false;
    for (int64_t qy = 0; qy < std::min(S.sy, OH); qy++)
        for (int64_t qx = 0; qx < std::min(S.sx, OW); qx++) {
            const bool live = py[qy].live && px[qx].live;
            any_live |= live;
            any_empty |= !live;
        }
    rten_tensor bias_c;
    if (bias_in) RTB_TRY(sc.contiguous(&bd, &bias_c));

    // ---- every phase without a convolution: the bias, in one launch
    if (any_empty) {
        ConvTransposeFill f;
        memset(&f, 0, sizeof(f));
        f.B = (int)B;
        f.O = (int)O;
        f.OH = (int)OH;
        f.OW = (int)OW;
        f.sy = (int)S.sy;
        f.sx = (int)S.sx;
        f.s_b = ov.strides[0];
        f.s_o = ov.strides[1];
        f.s_h = ov.strides[2];
        f.s_w = ov.strides[3];
        for (int64_t q = 0; q < S.sy; q++)
            if (py[q].live) f.live_y[q >> 5] |= 1u << (q & 31);
        for (int64_t q = 0; q < S.sx; q++)
            if (px[q].live) f.live_x[q >> 5] |= 1u << (q & 31);
        RTB_TRY(launch_conv_transpose_fill(ctx, (float*)ov.data, bias_in ? (const float*)bias_c.data : nullptr, f));
    }
    if (!any_live) return RTEN_OK;

    // ---- the input, shared by every phase: channels-last and 16-byte addressable for the implicit-GEMM path (one
    //      copy when it is not), and in 3xTF32 its low parts, split once
    const bool implicit = (Cg * 4) % 16 == 0 && Cg * 4 >= 32;
    rten_tensor x = S.x;
    if (implicit) RTB_TRY(nhwc_input(ctx, S.x, &x));
    const float* x_lo = nullptr;
    const bool compact_nhwc = x.strides[1] == 1 && x.strides[3] == C && x.strides[2] == W * C && x.strides[0] == H * W * C;
    if (implicit && ctx->f32_mode == RTEN_F32_TF32X3 && Cg % 32 == 0 && compact_nhwc && !getenv("RTEN_B200_X3_THREE_PLANES")) {
        float* lo = nullptr;
        RTB_TRY(temp_alloc(ctx, (size_t)(B * H * W * C) * 4, (void**)&lo));
        const long long dims[4] = {C, W, H, B}, strides[4] = {1, C, W * C, H * W * C};
        RTB_TRY(launch_tf32x3_split(ctx, (const float*)x.data, lo, dims, strides, C, 2));
        x_lo = lo;
    }

    // ---- the sub-kernels: prepacked, or packed here for the residues this call uses
    std::vector<rten_packed> call_packs;
    std::vector<int> call_index((size_t)(S.sy * S.sx), -1);
    if (!pw) {
        for (int64_t qy = 0; qy < std::min(S.sy, OH); qy++)
            for (int64_t qx = 0; qx < std::min(S.sx, OW); qx++) {
                if (!py[qy].live || !px[qx].live) continue;
                const size_t ri = (size_t)(py[qy].r * S.sx + px[qx].r);
                if (call_index[ri] >= 0) continue;
                rten_packed p;
                p.kind = 1;
                p.O = O;
                p.Cg = Cg;
                p.kh = py[qy].taps.T;
                p.kw = px[qx].taps.T;
                p.groups = groups;
                RTB_TRY(temp_alloc(ctx, (size_t)(O * p.kh * p.kw * Cg) * 4, &p.data));
                RTB_TRY(pack_transpose_phase(ctx, S, py[qy].taps, px[qx].taps, p.data));
                call_index[ri] = (int)call_packs.size();
                call_packs.push_back(p);
            }
    }

    // ---- one stride-1 convolution per phase with taps, into a strided view of the output
    for (int64_t qy = 0; qy < std::min(S.sy, OH); qy++)
        for (int64_t qx = 0; qx < std::min(S.sx, OW); qx++) {
            const AxisPhase &ay = py[qy], &ax = px[qx];
            if (!ay.live || !ax.live) continue;
            const size_t ri = (size_t)(ay.r * S.sx + ax.r);
            const rten_packed* pp = pw ? pw->phases[ri] : &call_packs[(size_t)call_index[ri]];
            const int64_t xoff = ay.row0 * x.strides[2] + ax.row0 * x.strides[3];
            rten_tensor xv = x;
            xv.data = (float*)x.data + xoff;
            xv.shape[2] = ay.rows;
            xv.shape[3] = ax.rows;
            rten_tensor wv{};
            wv.data = pp->data;
            wv.dtype = RTEN_F32;
            wv.device = ctx->device;
            wv.ndim = 4;
            const int64_t wshape[4] = {O, Cg, pp->kh, pp->kw}, wstr[4] = {pp->kh * pp->kw * Cg, 1, pp->kw * Cg, Cg};
            for (int i = 0; i < 4; i++) {
                wv.shape[i] = wshape[i];
                wv.strides[i] = wstr[i];
            }
            rten_tensor oq = ov;
            oq.data = (float*)ov.data + qy * ov.strides[2] + qx * ov.strides[3];
            oq.shape[2] = ay.n;
            oq.shape[3] = ax.n;
            oq.strides[2] = ov.strides[2] * S.sy;
            oq.strides[3] = ov.strides[3] * S.sx;
            rten_conv_params p{};
            p.pads[0] = (int32_t)ay.pad0;
            p.pads[1] = (int32_t)ax.pad0;
            p.pads[2] = (int32_t)ay.pad1;
            p.pads[3] = (int32_t)ax.pad1;
            p.groups = groups;
            p.strides[0] = p.strides[1] = 1;
            p.dilations[0] = (int32_t)ay.dil;
            p.dilations[1] = (int32_t)ax.dil;
            p.n_strides = p.n_dilations = 2;
            ConvArgs A{};
            A.kind = 0;
            A.x = &xv;
            A.w = &wv;
            A.pw = pp;
            A.bias = bias_in ? &bias_c : nullptr;
            A.p = &p;
            A.x_lo = x_lo ? x_lo + xoff : nullptr;
            A.cache_x3 = pw != nullptr;
            RTB_TRY(conv_core(sc, A, &oq));
        }
    return RTEN_OK;
}

// `f32 as i32` (saturating, NaN -> 0)
int64_t f32_as_i32(float v) {
    if (v != v) return 0;
    if (v >= 2147483648.0f) return INT32_MAX;
    if (v <= -2147483648.0f) return INT32_MIN;
    return (int64_t)v;
}

}  // namespace

// calc_output_size of Resize (src/ops/resize.rs:273-308).  Each value is ONE rounded f32 operation (a product, a
// quotient), which no host compiler can contract; everything that chains operations runs on the device.
rten_status api::resize_output_size(rten_ctx* ctx, const rten_tensor& x, const rten_resize_params* p, int64_t osz[4], float inv[4]) {
    const int nd = x.ndim;
    if (p->n != nd) return fail(ctx, RTEN_ERR_INCOMPATIBLE_SHAPES, "scales/sizes length should equal input rank");
    if (nd > 4) return fail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "Only 1D to 4D inputs are supported with up to two resized dimensions");
    for (int i = 0; i < nd; i++) {
        const volatile float in = (float)x.shape[i];
        if (p->use_sizes) {
            const volatile float o = (float)p->sizes[i];
            osz[i] = p->sizes[i];
            inv[i] = in / o;
        } else {
            const volatile float s = p->scales[i];
            const volatile float prod = in * s;
            osz[i] = f32_as_i32(floorf(prod));
            inv[i] = 1.0f / s;
        }
    }
    for (int i = 0; i < nd; i++)
        if (osz[i] < 0) return fail(ctx, RTEN_ERR_INVALID_VALUE, "scales/sizes must be positive");
    return RTEN_OK;
}

extern "C" {

rten_status rten_b200_prepack_conv_weight(rten_ctx* ctx, const rten_tensor* w, int groups, rten_packed** out) {
    RTB_TRY(check_ctx(ctx));
    if (!w || !out) return RTEN_ERR_INVALID_VALUE;
    *out = nullptr;
    if (w->ndim != 4) return fail(ctx, RTEN_ERR_INVALID_VALUE, "input must have 4 dims (OCHW)");
    if (w->dtype == RTEN_I32) return fail(ctx, RTEN_ERR_UNSUPPORTED_TYPE, "unsupported type");
    OpScope sc(ctx);
    rten_tensor wv;
    RTB_TRY(sc.in(w, &wv));
    const int es = dtype_size(w->dtype);
    PackedPtr p(new rten_packed(), PackedFree{ctx});
    p->kind = 1;
    p->dtype = w->dtype;
    p->O = wv.shape[0];
    p->Cg = wv.shape[1];
    p->kh = wv.shape[2];
    p->kw = wv.shape[3];
    p->groups = groups;
    const int64_t n = std::max<int64_t>(p->O * p->Cg * p->kh * p->kw, 1);
    RTB_TRY(pool_alloc(ctx, (size_t)n * es, &p->data));
    RTB_TRY(pack_conv_weight(ctx, &wv, es, p->data));
    if (es == 1 && p->O > 0) {
        RTB_TRY(pool_alloc(ctx, (size_t)p->O * 4, (void**)&p->colsum));
        const int64_t Kd = p->Cg * p->kh * p->kw;
        RTB_TRY(launch_rowsum8(ctx, p->data, p->dtype == RTEN_I8, p->O, (int)Kd, Kd, p->colsum));
    }
    RTB_TRY(sc.finish(RTEN_OK));
    *out = p.release();
    return RTEN_OK;
}

// ---- Conv family ----------------------------------------------------------------------------
rten_status rten_b200_conv2d_act(rten_ctx* ctx, const rten_tensor* x, const rten_tensor* w, const rten_packed* pw,
                                 const rten_tensor* bias, const rten_conv_params* p, const rten_tensor* residual,
                                 const rten_activation* act, rten_tensor* out) {
    RTB_TRY(check_ctx(ctx));
    if (!x || !w || !p || !out) return fail(ctx, RTEN_ERR_MISSING_INPUTS, "missing inputs");
    if (x->dtype != RTEN_F32 || w->dtype != RTEN_F32 || (bias && bias->dtype != RTEN_F32))
        return fail(ctx, RTEN_ERR_UNSUPPORTED_TYPE, "unsupported type");
    if (act && (act->kind < RTEN_ACT_NONE || act->kind > RTEN_ACT_HARD_SWISH))
        return fail(ctx, RTEN_ERR_INVALID_VALUE, "unknown activation");
    OpScope sc(ctx);
    ConvArgs A{};
    A.kind = 0;
    A.x = x;
    A.w = w;
    A.pw = pw;
    A.bias = bias;
    A.p = p;
    A.residual = residual;
    if (act) {
        A.act = act->kind;
        A.act_alpha = act->alpha;
        A.act_beta = act->beta;
    }
    return sc.finish(conv_core(sc, A, out));
}

rten_status rten_b200_conv2d_ex(rten_ctx* ctx, const rten_tensor* x, const rten_tensor* w, const rten_packed* pw,
                                const rten_tensor* bias, const rten_conv_params* p, const rten_tensor* residual,
                                int activation, rten_tensor* out) {
    RTB_TRY(check_ctx(ctx));
    if (activation < RTEN_ACT_NONE || activation > RTEN_ACT_GELU_TANH) return fail(ctx, RTEN_ERR_INVALID_VALUE, "unknown activation");
    const rten_activation a = {activation, 0.0f, 0.0f};
    return rten_b200_conv2d_act(ctx, x, w, pw, bias, p, residual, &a, out);
}

rten_status rten_b200_conv2d_projected(rten_ctx* ctx, const rten_tensor* x, const rten_tensor* w, const rten_packed* pw,
                                       const rten_tensor* bias, const rten_conv_params* p, const rten_tensor* x_proj,
                                       const rten_tensor* w_proj, const rten_packed* pw_proj, const rten_tensor* bias_proj,
                                       const rten_conv_params* p_proj, int activation, rten_tensor* out) {
    RTB_TRY(check_ctx(ctx));
    if (!x || !w || !p || !x_proj || !w_proj || !p_proj || !out) return fail(ctx, RTEN_ERR_MISSING_INPUTS, "missing inputs");
    for (const rten_tensor* t : {x, w, bias, x_proj, w_proj, bias_proj})
        if (t && t->dtype != RTEN_F32) return fail(ctx, RTEN_ERR_UNSUPPORTED_TYPE, "unsupported type");
    if (activation < RTEN_ACT_NONE || activation > RTEN_ACT_GELU_TANH) return fail(ctx, RTEN_ERR_INVALID_VALUE, "unknown activation");
    OpScope sc(ctx);
    ConvArgs M{}, P{};
    M.kind = P.kind = 0;
    M.x = x;
    M.w = w;
    M.pw = pw;
    M.bias = bias;
    M.p = p;
    M.act = activation;
    P.x = x_proj;
    P.w = w_proj;
    P.pw = pw_proj;
    P.bias = bias_proj;
    P.p = p_proj;
    return sc.finish(conv_projected(sc, M, P, out));
}

rten_status rten_b200_conv2d_chained(rten_ctx* ctx, const rten_tensor* x, const rten_tensor* w, const rten_packed* pw,
                                     const rten_tensor* bias, const rten_conv_params* p, const rten_tensor* residual,
                                     const rten_tensor* x_proj, const rten_tensor* w_proj, const rten_packed* pw_proj,
                                     const rten_tensor* bias_proj, const rten_conv_params* p_proj, int activation,
                                     const rten_tensor* w_next, const rten_packed* pw_next, const rten_tensor* bias_next,
                                     const rten_conv_params* p_next, int activation_next, rten_tensor* out,
                                     rten_tensor* out_next) {
    RTB_TRY(check_ctx(ctx));
    if (!x || !w || !p || !w_next || !p_next || !out || !out_next || (x_proj && (!w_proj || !p_proj)))
        return fail(ctx, RTEN_ERR_MISSING_INPUTS, "missing inputs");
    if (residual && x_proj) return fail(ctx, RTEN_ERR_INVALID_VALUE, "a residual and a projection shortcut are exclusive");
    for (const rten_tensor* t : {x, w, bias, residual, x_proj, w_proj, bias_proj, w_next, bias_next})
        if (t && t->dtype != RTEN_F32) return fail(ctx, RTEN_ERR_UNSUPPORTED_TYPE, "unsupported type");
    for (int a : {activation, activation_next})
        if (a < RTEN_ACT_NONE || a > RTEN_ACT_GELU_TANH) return fail(ctx, RTEN_ERR_INVALID_VALUE, "unknown activation");
    OpScope sc(ctx);
    ConvArgs M{}, P{}, Nx{};
    M.kind = P.kind = Nx.kind = 0;
    M.x = x;
    M.w = w;
    M.pw = pw;
    M.bias = bias;
    M.p = p;
    M.residual = residual;
    M.act = activation;
    P.x = x_proj;
    P.w = w_proj;
    P.pw = pw_proj;
    P.bias = bias_proj;
    P.p = p_proj;
    Nx.x = out;
    Nx.w = w_next;
    Nx.pw = pw_next;
    Nx.bias = bias_next;
    Nx.p = p_next;
    Nx.act = activation_next;
    return sc.finish(conv_chained(sc, M, x_proj ? &P : nullptr, Nx, out, out_next));
}

// ---- ConvTranspose ------------------------------------------------------------------------------------------------
rten_status rten_b200_prepack_conv_transpose_weight(rten_ctx* ctx, const rten_tensor* w, const rten_conv_transpose_params* params,
                                                    rten_packed** out) {
    RTB_TRY(check_ctx(ctx));
    if (!w || !params || !out) return fail(ctx, RTEN_ERR_MISSING_INPUTS, "missing inputs");
    *out = nullptr;
    if (w->dtype != RTEN_F32) return fail(ctx, RTEN_ERR_UNSUPPORTED_TYPE, "unsupported type");
    OpScope sc(ctx);
    rten_tensor wv;
    ConvTShape S;
    RTB_TRY(sc.in(w, &wv));
    RTB_TRY(conv_transpose_shape(ctx, nullptr, wv, nullptr, params, S));
    if (S.sy > 256 || S.sx > 256) return fail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "ConvTranspose strides above 256 are not supported");
    PackedPtr p(new rten_packed(), PackedFree{ctx});
    p->kind = 2;
    p->O = S.O;
    p->Cg = S.Cg;
    p->kh = S.kh;
    p->kw = S.kw;
    p->groups = S.groups;
    p->sy = S.sy;
    p->sx = S.sx;
    p->dy = S.dy;
    p->dx = S.dx;
    p->phases.assign((size_t)(S.sy * S.sx), nullptr);
    for (int64_t ry = 0; ry < S.sy; ry++)
        for (int64_t rx = 0; rx < S.sx; rx++) {
            const AxisTaps ty = axis_taps(S.kh, S.sy, S.dy, ry), tx = axis_taps(S.kw, S.sx, S.dx, rx);
            if (ty.T == 0 || tx.T == 0) continue;
            rten_packed* ph = new rten_packed();
            p->phases[(size_t)(ry * S.sx + rx)] = ph;
            ph->kind = 1;
            ph->O = S.O;
            ph->Cg = S.Cg;
            ph->kh = ty.T;
            ph->kw = tx.T;
            ph->groups = S.groups;
            RTB_TRY(pool_alloc(ctx, (size_t)std::max<int64_t>(S.O * ty.T * tx.T * S.Cg, 1) * 4, &ph->data));
            RTB_TRY(pack_transpose_phase(ctx, S, ty, tx, ph->data));
        }
    RTB_TRY(sc.finish(RTEN_OK));
    *out = p.release();
    return RTEN_OK;
}

rten_status rten_b200_conv_transpose(rten_ctx* ctx, const rten_tensor* x, const rten_tensor* w, const rten_packed* pw,
                                     const rten_tensor* bias, const rten_conv_transpose_params* p, rten_tensor* out) {
    RTB_TRY(check_ctx(ctx));
    if (!x || !w || !p || !out) return fail(ctx, RTEN_ERR_MISSING_INPUTS, "missing inputs");
    if (x->dtype != RTEN_F32 || w->dtype != RTEN_F32 || (bias && bias->dtype != RTEN_F32))
        return fail(ctx, RTEN_ERR_UNSUPPORTED_TYPE, "unsupported type");
    OpScope sc(ctx);
    return sc.finish(conv_transpose_core(sc, x, w, pw, bias, p, out));
}

rten_status rten_b200_conv2d(rten_ctx* ctx, const rten_tensor* x, const rten_tensor* w, const rten_packed* pw,
                             const rten_tensor* bias, const rten_conv_params* p, rten_tensor* out) {
    return rten_b200_conv2d_ex(ctx, x, w, pw, bias, p, nullptr, 0, out);
}

rten_status rten_b200_conv_integer(rten_ctx* ctx, const rten_tensor* x, const rten_tensor* w, const rten_packed* pw,
                                   const rten_tensor* x_zp, const rten_tensor* w_zp, const rten_tensor* scale,
                                   const rten_conv_params* p, rten_tensor* out) {
    return rten_b200_conv_integer_ex(ctx, x, w, pw, x_zp, w_zp, scale, nullptr, p, nullptr, nullptr, 0, nullptr, out);
}

rten_status rten_b200_conv_integer_ex(rten_ctx* ctx, const rten_tensor* x, const rten_tensor* w, const rten_packed* pw,
                                      const rten_tensor* x_zp, const rten_tensor* w_zp, const rten_tensor* scale,
                                      const rten_tensor* scale_b, const rten_conv_params* p, const rten_tensor* bias,
                                      const rten_tensor* residual, int activation, rten_tensor* out_range,
                                      rten_tensor* out) {
    RTB_TRY(check_ctx(ctx));
    if (!x || !w || !p || !out) return fail(ctx, RTEN_ERR_MISSING_INPUTS, "missing inputs");
    auto is8 = [](int dt) { return dt == RTEN_U8 || dt == RTEN_I8; };
    if (!is8(x->dtype) || !is8(w->dtype)) return fail(ctx, RTEN_ERR_UNSUPPORTED_TYPE, "unsupported type");
    if (scale && scale->dtype != RTEN_F32) return fail(ctx, RTEN_ERR_CAST_FAILED, "scale must be float");
    if ((bias || residual || activation || scale_b) && !scale)
        return fail(ctx, RTEN_ERR_INVALID_VALUE, "bias / residual / activation follow the float conversion: a scale is required");
    if ((bias && bias->dtype != RTEN_F32) || (residual && residual->dtype != RTEN_F32))
        return fail(ctx, RTEN_ERR_UNSUPPORTED_TYPE, "unsupported type");
    if (activation < 0 || activation > 1) return fail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "only Relu can follow an integer convolution");
    if (out_range && !scale) return fail(ctx, RTEN_ERR_INVALID_VALUE, "the output range is defined for float outputs: a scale is required");
    OpScope sc(ctx);
    ConvArgs A{};
    A.kind = 1;
    A.x = x;
    A.w = w;
    A.pw = (pw && pw->dtype == w->dtype) ? pw : nullptr;
    A.p = p;
    A.x_zp = x_zp;
    A.w_zp = w_zp;
    A.scale = scale;
    A.scale_b = scale_b;
    A.bias = bias;
    A.residual = residual;
    A.act = activation;
    A.out_range = out_range;
    return sc.finish(conv_core(sc, A, out));
}

// ---- pooling / gather ---------------------------------------------------------------------------------
// MaxPool (average = false) and AveragePool over an NCHW tensor in any strides; the output follows the input's layout
static rten_status pool2d(rten_ctx* ctx, const rten_tensor* x, const int32_t kernel[2], const int32_t pads[4],
                          const int32_t strides[2], bool average, int count_include_pad, rten_tensor* out) {
    RTB_TRY(check_ctx(ctx));
    if (!x || !out) return fail(ctx, RTEN_ERR_MISSING_INPUTS, "missing inputs");
    if (x->dtype != RTEN_F32) return fail(ctx, RTEN_ERR_UNSUPPORTED_TYPE, "unsupported type");
    if (x->ndim != 4) return fail(ctx, RTEN_ERR_INVALID_VALUE, "input must have 4 dims (NCHW)");
    OpScope sc(ctx);
    rten_tensor xv, ov;
    RTB_TRY(sc.in(x, &xv));
    int64_t OH = 0, OW = 0, p0, p1;
    RTB_TRY(axis_out(ctx, xv.shape[2], kernel[0], strides[0], false, pads[0], pads[2], 1, &OH, &p0, &p1));
    RTB_TRY(axis_out(ctx, xv.shape[3], kernel[1], strides[1], false, pads[1], pads[3], 1, &OW, &p0, &p1));
    const int64_t B = xv.shape[0], C = xv.shape[1];
    RTB_TRY(out_like(sc, out, RTEN_F32, xv, false, B, C, OH, OW, &ov));
    PoolParams p;
    p.B = (int)B;
    p.C = (int)C;
    p.H = (int)xv.shape[2];
    p.W = (int)xv.shape[3];
    p.OH = (int)OH;
    p.OW = (int)OW;
    p.kh = kernel[0];
    p.kw = kernel[1];
    p.sy = strides[0];
    p.sx = strides[1];
    p.pt = pads[0];
    p.pl = pads[1];
    p.xs_b = xv.strides[0];
    p.xs_c = xv.strides[1];
    p.xs_h = xv.strides[2];
    p.xs_w = xv.strides[3];
    p.ys_b = ov.strides[0];
    p.ys_c = ov.strides[1];
    p.ys_h = ov.strides[2];
    p.ys_w = ov.strides[3];
    p.channels_fastest = ov.strides[1] == 1;
    return sc.finish(average ? launch_avgpool(ctx, (const float*)xv.data, (float*)ov.data, p, count_include_pad)
                             : launch_maxpool(ctx, (const float*)xv.data, (float*)ov.data, p));
}

rten_status rten_b200_max_pool(rten_ctx* ctx, const rten_tensor* x, const int32_t kernel[2], const int32_t pads[4],
                               const int32_t strides[2], rten_tensor* out) {
    return pool2d(ctx, x, kernel, pads, strides, false, 0, out);
}

rten_status rten_b200_average_pool(rten_ctx* ctx, const rten_tensor* x, const int32_t kernel[2], const int32_t pads[4],
                                   const int32_t strides[2], int count_include_pad, rten_tensor* out) {
    return pool2d(ctx, x, kernel, pads, strides, true, count_include_pad, out);
}

// ---- Resize -------------------------------------------------------------------------------------------
rten_status rten_b200_resize(rten_ctx* ctx, const rten_tensor* x, const rten_resize_params* p, rten_tensor* out) {
    RTB_TRY(check_ctx(ctx));
    if (!x || !p || !out) return fail(ctx, RTEN_ERR_MISSING_INPUTS, "missing inputs");
    if (x->dtype != RTEN_F32) return fail(ctx, RTEN_ERR_UNSUPPORTED_TYPE, "unsupported type");
    if (p->mode < RTEN_RESIZE_NEAREST || p->mode > RTEN_RESIZE_LINEAR || p->coord_mode < RTEN_RESIZE_HALF_PIXEL ||
        p->coord_mode > RTEN_RESIZE_PYTORCH_HALF_PIXEL || p->nearest_mode < RTEN_RESIZE_FLOOR ||
        p->nearest_mode > RTEN_RESIZE_ROUND_PREFER_CEIL)
        return fail(ctx, RTEN_ERR_INVALID_VALUE, "unknown resize mode");
    OpScope sc(ctx);
    rten_tensor xv;
    RTB_TRY(sc.in(x, &xv));
    const int nd = xv.ndim;
    int64_t osz[4] = {0, 0, 0, 0};
    float inv[4] = {1.0f, 1.0f, 1.0f, 1.0f};
    RTB_TRY(resize_output_size(ctx, xv, p, osz, inv));
    // resize_impl (resize.rs:350-407): which input axis plays (n, c, h, w); -1 = an added axis of size 1
    bool same = true;
    for (int i = 0; i < nd; i++) same = same && osz[i] == xv.shape[i];
    auto eq = [&](int i) { return osz[i] == xv.shape[i]; };
    int map[4] = {-1, -1, -1, -1};
    if (same) {
    } else if (nd == 4 && eq(0) && eq(1)) {
        map[0] = 0, map[1] = 1, map[2] = 2, map[3] = 3;
    } else if (nd == 3 && eq(0) && eq(1)) {  // NCW
        map[0] = 0, map[1] = 1, map[3] = 2;
    } else if (nd == 3 && eq(0)) {  // NHW
        map[0] = 0, map[2] = 1, map[3] = 2;
    } else if (nd == 2) {
        map[2] = 0, map[3] = 1;
    } else if (nd == 1) {
        map[3] = 0;
    } else {
        return fail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "Only 1D to 4D inputs are supported with up to two resized dimensions");
    }
    // output: a 4-D result follows the input's layout, like MaxPool and the convolutions
    rten_tensor ov;
    RTB_TRY(nd == 4 ? out_like(sc, out, RTEN_F32, xv, false, osz[0], osz[1], osz[2], osz[3], &ov)
                    : sc.out(out, RTEN_F32, nd, osz, &ov, nullptr));
    if (same) return sc.finish(numel(&xv) ? copy_view(ctx, xv, ov) : RTEN_OK);
    ResizeParams r;
    r.mode = p->mode;
    r.coord_mode = p->coord_mode;
    r.nearest_mode = p->nearest_mode;
    int64_t in4[4], out4[4];
    for (int i = 0; i < 4; i++) {
        const int a = map[i];
        in4[i] = a >= 0 ? xv.shape[a] : 1;
        out4[i] = a >= 0 ? osz[a] : 1;
        r.xs[i] = a >= 0 ? xv.strides[a] : 0;
        r.os[i] = a >= 0 ? ov.strides[a] : 0;
    }
    if (out4[0] * out4[1] * out4[2] * out4[3] != 0 && in4[2] * in4[3] == 0)
        return fail(ctx, RTEN_ERR_INVALID_VALUE, "cannot resize an empty input");
    for (int i = 0; i < 4; i++)
        if (in4[i] > INT32_MAX || out4[i] > INT32_MAX) return fail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "dimension too large");
    r.B = (int)out4[0];
    r.C = (int)out4[1];
    r.H = (int)in4[2];
    r.W = (int)in4[3];
    r.OH = (int)out4[2];
    r.OW = (int)out4[3];
    r.inv_y = map[2] >= 0 ? inv[map[2]] : 1.0f;
    r.inv_x = inv[map[3]];
    r.x = (const float*)xv.data;
    r.out = (float*)ov.data;
    return sc.finish(launch_resize(ctx, r));
}

// ---- Concat -------------------------------------------------------------------------------------------
rten_status rten_b200_concat(rten_ctx* ctx, const rten_tensor* const* inputs, int n, int axis, rten_tensor* out) {
    RTB_TRY(check_ctx(ctx));
    if (!inputs || n < 1 || !out) return fail(ctx, RTEN_ERR_MISSING_INPUTS, "missing inputs");
    for (int i = 0; i < n; i++)
        if (!inputs[i]) return fail(ctx, RTEN_ERR_MISSING_INPUTS, "missing inputs");
    const rten_tensor& first = *inputs[0];
    const int nd = first.ndim, dt = first.dtype;
    if (dt != RTEN_F32 && dt != RTEN_I32 && dt != RTEN_I8 && dt != RTEN_U8) return fail(ctx, RTEN_ERR_UNSUPPORTED_TYPE, "unsupported type");
    for (int i = 1; i < n; i++)
        if (inputs[i]->dtype != dt) return fail(ctx, RTEN_ERR_CAST_FAILED, "inputs must have the same type");
    if (nd < 1 || nd > RTEN_MAX_DIMS || axis < -nd || axis >= nd) return fail(ctx, RTEN_ERR_INVALID_VALUE, "Axis is invalid");
    if (axis < 0) axis += nd;
    // concatenated_shape (src/ops/concat.rs:20-47)
    int64_t oshape[RTEN_MAX_DIMS];
    for (int d = 0; d < nd; d++) oshape[d] = first.shape[d];
    for (int i = 1; i < n; i++) {
        if (inputs[i]->ndim != nd) return fail(ctx, RTEN_ERR_INCOMPATIBLE_SHAPES, "Tensors must have the same number of dimensions");
        for (int d = 0; d < nd; d++) {
            if (d != axis && inputs[i]->shape[d] != first.shape[d])
                return fail(ctx, RTEN_ERR_INCOMPATIBLE_SHAPES, "Dimensions must be the same except for concat axis");
            if (d == axis) oshape[d] += inputs[i]->shape[d];
        }
    }
    OpScope sc(ctx);
    std::vector<rten_tensor> iv((size_t)n);
    for (int i = 0; i < n; i++) RTB_TRY(sc.in(inputs[i], &iv[(size_t)i]));
    rten_tensor ov;
    // an allocated 4-D output follows input 0's layout
    OutLayout l;
    if (nd == 4) l = layout_like(iv[0], false, oshape[0], oshape[1], oshape[2], oshape[3]);
    RTB_TRY(sc.out(out, dt, nd, oshape, &ov, (nd == 4 && !out->data) ? l.strides : nullptr));
    const int es = dtype_size(dt);
    // dimensions of extent 1 dropped, the rest put in the output's memory order, then adjacent dimensions merged where the
    // output and every copied input allow it (the concat axis merges with the dimensions inside it only)
    struct Src {
        const uint8_t* p;
        long long ext, start;
        long long st[RTEN_MAX_DIMS];
    };
    std::vector<Src> srcs;
    long long shape[RTEN_MAX_DIMS], ost[RTEN_MAX_DIMS];
    int dims[RTEN_MAX_DIMS], k = 0, ax = 0;
    for (int d = 0; d < nd; d++)
        if (d == axis || oshape[d] != 1) dims[k++] = d;
    // in the output's memory order, outermost first: a channels-last output iterates (b, h, w, c)
    std::stable_sort(dims, dims + k, [&](int a, int b) { return ov.strides[a] > ov.strides[b]; });
    for (int j = 0; j < k; j++)
        if (dims[j] == axis) ax = j;
    for (int j = 0; j < k; j++) shape[j] = oshape[dims[j]], ost[j] = ov.strides[dims[j]];
    long long start = 0;
    for (int i = 0; i < n; i++) {
        const rten_tensor& t = iv[(size_t)i];
        Src s;
        s.p = (const uint8_t*)t.data;
        s.ext = t.shape[axis];
        s.start = start;
        start += s.ext;
        for (int j = 0; j < k; j++) s.st[j] = t.strides[dims[j]];
        if (numel(&t) == 0) continue;
        // already its slice of the output: nothing to copy
        bool in_place = s.p == (const uint8_t*)ov.data + s.start * ost[ax] * es;
        for (int j = 0; j < k && in_place; j++) in_place = (j == ax ? s.ext : shape[j]) == 1 || s.st[j] == ost[j];
        if (!in_place) srcs.push_back(s);
    }
    for (int j = k - 2; j >= 0; j--) {
        if (j + 1 == ax) continue;
        bool ok = ost[j] == ost[j + 1] * shape[j + 1];
        for (const Src& s : srcs) ok = ok && s.st[j] == s.st[j + 1] * shape[j + 1];
        if (!ok) continue;
        const long long inner = shape[j + 1];
        shape[j] *= inner;
        ost[j] = ost[j + 1];
        for (Src& s : srcs) {
            s.st[j] = s.st[j + 1];
            if (j == ax) s.ext *= inner, s.start *= inner;
        }
        for (int m = j + 1; m + 1 < k; m++) {
            shape[m] = shape[m + 1];
            ost[m] = ost[m + 1];
            for (Src& s : srcs) s.st[m] = s.st[m + 1];
        }
        if (ax > j) ax--;
        k--;
    }
    // 16-byte units when every slice is 16-byte addressable and the innermost dimension is contiguous on both sides
    const long long v = 16 / es;
    bool vec = ost[k - 1] == 1 && reinterpret_cast<uintptr_t>(ov.data) % 16 == 0 && (ax == k - 1 || shape[k - 1] % v == 0);
    for (int j = 0; j + 1 < k && vec; j++) vec = ost[j] % v == 0;
    for (const Src& s : srcs) {
        vec = vec && s.st[k - 1] == 1 && reinterpret_cast<uintptr_t>(s.p) % 16 == 0;
        if (ax == k - 1) vec = vec && s.ext % v == 0 && s.start % v == 0;
        for (int j = 0; j + 1 < k && vec; j++) vec = s.st[j] % v == 0;
    }
    // strides and innermost extents in units of the copied element
    auto stride_of = [&](int j, long long st) { return vec ? (j == k - 1 ? 1 : st / v) : st; };
    const long long unit = vec ? v : 1;
    ConcatParams cp;
    memset(&cp, 0, sizeof(cp));
    cp.esize = vec ? 16 : es;
    cp.ndim = k;
    cp.axis = ax;
    cp.out = ov.data;
    for (int j = 0; j < k; j++) {
        cp.shape[j] = j == k - 1 ? shape[j] / unit : shape[j];
        cp.out_strides[j] = stride_of(j, ost[j]);
    }
    for (size_t base = 0; base < srcs.size(); base += kConcatMaxSources) {
        cp.nsrc = (int)std::min<size_t>(kConcatMaxSources, srcs.size() - base);
        for (int i = 0; i < cp.nsrc; i++) {
            const Src& s = srcs[base + (size_t)i];
            ConcatSource& c = cp.s[i];
            c.src = s.p;
            c.ext = ax == k - 1 ? s.ext / unit : s.ext;
            c.dst_off = s.start * ost[ax] / unit;
            c.n = 1;
            for (int j = 0; j < k; j++) {
                c.strides[j] = stride_of(j, s.st[j]);
                c.n *= j == ax ? c.ext : cp.shape[j];
            }
        }
        RTB_TRY(launch_concat(ctx, cp));
    }
    return sc.finish(RTEN_OK);
}

rten_status rten_b200_global_average_pool(rten_ctx* ctx, const rten_tensor* x, rten_tensor* out) {
    RTB_TRY(check_ctx(ctx));
    if (!x || !out) return fail(ctx, RTEN_ERR_MISSING_INPUTS, "missing inputs");
    if (x->dtype != RTEN_F32) return fail(ctx, RTEN_ERR_UNSUPPORTED_TYPE, "unsupported type");
    if (x->ndim != 4) return fail(ctx, RTEN_ERR_INVALID_VALUE, "input must have 4 dims (NCHW)");
    OpScope sc(ctx);
    rten_tensor xv, ov;
    RTB_TRY(sc.in(x, &xv));
    const int64_t B = xv.shape[0], C = xv.shape[1], H = xv.shape[2], W = xv.shape[3];
    int64_t oshape[4] = {B, C, 1, 1};
    RTB_TRY(sc.out(out, RTEN_F32, 4, oshape, &ov, nullptr));
    if (!is_contiguous(&ov)) return fail(ctx, RTEN_ERR_UNSUPPORTED_OUTPUT, "pooled output must be contiguous");
    if (B * C == 0) return sc.finish(RTEN_OK);
    rten_tensor src = xv;
    if (!(xv.strides[2] == W * xv.strides[3])) RTB_TRY(sc.contiguous(&xv, &src));  // need a uniform stride over (h, w)
    return sc.finish(launch_row_mean(ctx, (const float*)src.data, (float*)ov.data, B * C, (int)(H * W), C, src.strides[0],
                                     src.strides[1], src.strides[3]));
}

}  // extern "C"
