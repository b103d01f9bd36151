// Operator entry points of the C ABI, row / elementwise operators (Softmax, LayerNormalization, Erf / Gelu / Relu / Sqrt / Exp
// / Tanh ..., Add / Mul / Div / Pow, ReduceSum / ReduceMean,
// DynamicQuantizeLinear, Gather / Scatter rows): shape / argument validation with the reference's error strings,
// operand normalisation (K-major, TMA-addressable), kernel dispatch.  Mirrors, per function, the
// reference operator named in include/rten_b200.h.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "api_shared.h"
#include "comm_device.cuh"
#include "api_util.h"
#include "groupnorm.h"
#include "reduce.h"
#include "rowops.h"
#include "skinny.h"
#include "umma_gemm.h"

using namespace rtb;
using namespace rtb::api;

extern "C" {

// ---- Softmax / AddSoftmax -------------------------------------------------------------------
rten_status rten_b200_softmax(rten_ctx* ctx, const rten_tensor* x, const rten_tensor* mask, int axis, int flush_nans,
                              rten_tensor* out) {
    RTB_TRY(check_ctx(ctx));
    if (!x || !out) return fail(ctx, RTEN_ERR_MISSING_INPUTS, "missing inputs");
    if (x->dtype != RTEN_F32 || (mask && mask->dtype != RTEN_F32)) return fail(ctx, RTEN_ERR_UNSUPPORTED_TYPE, "unsupported type");
    const int nd = x->ndim;
    if (nd == 0 || axis < -nd || axis >= nd) return fail(ctx, RTEN_ERR_INVALID_VALUE, "Axis is invalid");
    const int ax = axis < 0 ? axis + nd : axis;
    OpScope sc(ctx);
    rten_tensor xv, mv, ov;
    RTB_TRY(sc.in(x, &xv));
    if (mask) RTB_TRY(sc.in(mask, &mv));
    RTB_TRY(sc.out(out, RTEN_F32, nd, xv.shape, &ov, nullptr));
    if (numel(&xv) == 0) return sc.finish(RTEN_OK);
    // view with `ax` moved last
    int perm[RTEN_MAX_DIMS], k = 0;
    for (int i = 0; i < nd; i++)
        if (i != ax) perm[k++] = i;
    perm[nd - 1] = ax;
    rten_tensor xp = xv, op = ov;
    for (int i = 0; i < nd; i++) {
        xp.shape[i] = xv.shape[perm[i]];
        xp.strides[i] = xv.strides[perm[i]];
        op.shape[i] = ov.shape[perm[i]];
        op.strides[i] = ov.strides[perm[i]];
    }
    rten_tensor xc;
    RTB_TRY(sc.contiguous(&xp, &xc));
    // run in place on the output when it is lane-contiguous in the permuted view, else via temp
    rten_tensor yc = op;
    const bool out_direct = is_contiguous(&op);
    if (!out_direct) {
        set_contiguous(&yc);
        RTB_TRY(temp_alloc(ctx, (size_t)numel(&xv) * 4, &yc.data));
    }
    const int n = (int)xp.shape[nd - 1];
    const long long rows = numel(&xv) / n;
    const float* mp = nullptr;
    long long lead[4] = {1, 1, 1, 1}, ms[4] = {0, 0, 0, 0}, ms_last = 0;
    int nlead = 0;
    if (mask) {
        // broadcast mask to x's shape (numpy rules), in the permuted dim order
        if (mv.ndim > nd) return fail(ctx, RTEN_ERR_INCOMPATIBLE_SHAPES, "Cannot broadcast inputs");
        long long mstr[RTEN_MAX_DIMS];
        for (int i = 0; i < nd; i++) {
            const int mi = i - (nd - mv.ndim);
            if (mi < 0 || mv.shape[mi] == 1)
                mstr[i] = 0;
            else if (mv.shape[mi] == xv.shape[i])
                mstr[i] = mv.strides[mi];
            else
                return fail(ctx, RTEN_ERR_INCOMPATIBLE_SHAPES, "Cannot broadcast inputs");
        }
        // leading dims in permuted order, collapsed where the mask advances uniformly
        std::vector<long long> ls, lst;
        for (int i = 0; i < nd - 1; i++) {
            const long long s = xp.shape[i], stv = mstr[perm[i]];
            if (s == 1) continue;
            if (!ls.empty() && lst.back() == stv * s) {
                ls.back() *= s;
                lst.back() = stv;
            } else {
                ls.push_back(s);
                lst.push_back(stv);
            }
        }
        if (ls.size() > 4) return fail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "mask broadcast pattern needs more than 4 strided dims");
        nlead = (int)ls.size();
        for (int i = 0; i < nlead; i++) {
            lead[i] = ls[i];
            ms[i] = lst[i];
        }
        ms_last = mstr[ax];
        mp = (const float*)mv.data;
    }
    RTB_TRY(launch_softmax(ctx, (const float*)xc.data, (float*)yc.data, rows, n, flush_nans, mp, nlead, lead, ms, ms_last));
    return sc.finish(out_direct ? RTEN_OK : copy_view(ctx, yc, op));
}

// ---- LayerNormalization -------------------------------------------------------------------------
// A scale / bias of the normalization over x's dims [ax, ndim) (src/ops/norm.rs layer_normalization_impl): one element
// stays a scalar (`item()`), read on the device later; anything else is broadcast to the normalized shape and
// materialised contiguous, or fails with `err`.
static rten_status norm_param(OpScope& sc, const rten_tensor& pv, const rten_tensor& xv, int ax, const char* err,
                              const float** ptr, bool* is_scalar) {
    if (numel(&pv) == 1) {
        *is_scalar = true;
        *ptr = (const float*)pv.data;
        return RTEN_OK;
    }
    *is_scalar = false;
    const int nn = xv.ndim - ax;  // normalized dims
    if (pv.ndim > nn) return fail(sc.ctx, RTEN_ERR_INVALID_VALUE, err);
    rten_tensor b = pv;
    b.ndim = nn;
    for (int i = 0; i < nn; i++) {
        const int pi = i - (nn - pv.ndim);
        const int64_t want = xv.shape[ax + i];
        b.shape[i] = want;
        if (pi < 0 || pv.shape[pi] == 1)
            b.strides[i] = 0;
        else if (pv.shape[pi] == want)
            b.strides[i] = pv.strides[pi];
        else
            return fail(sc.ctx, RTEN_ERR_INVALID_VALUE, err);
    }
    rten_tensor c;
    RTB_TRY(sc.contiguous(&b, &c));
    *ptr = (const float*)c.data;
    return RTEN_OK;
}

rten_status rten_b200_layer_norm(rten_ctx* ctx, const rten_tensor* x, const rten_tensor* scale, const rten_tensor* bias,
                                 int axis, float epsilon, rten_tensor* out) {
    RTB_TRY(check_ctx(ctx));
    if (!x || !scale || !out) return fail(ctx, RTEN_ERR_MISSING_INPUTS, "missing inputs");
    if (x->dtype != RTEN_F32 || scale->dtype != RTEN_F32 || (bias && bias->dtype != RTEN_F32))
        return fail(ctx, RTEN_ERR_UNSUPPORTED_TYPE, "unsupported type");
    const int nd = x->ndim;
    if (axis < -nd || axis >= std::max(nd, 1)) return fail(ctx, RTEN_ERR_INVALID_VALUE, "Axis is invalid");
    const int ax = axis < 0 ? axis + nd : axis;
    OpScope sc(ctx);
    rten_tensor xv, xc, sv, bv, ov;
    NormParams p;
    p.eps = epsilon < 0.0f ? 1e-5f : epsilon;
    RTB_TRY(sc.in(x, &xv));
    RTB_TRY(sc.in(scale, &sv));
    if (bias) RTB_TRY(sc.in(bias, &bv));
    bool g_scalar = false, b_scalar = false;
    RTB_TRY(norm_param(sc, sv, xv, ax, "`scale` is not broadcastable to normalized axes of input", &p.gamma, &g_scalar));
    if (bias) RTB_TRY(norm_param(sc, bv, xv, ax, "`bias` is not broadcastable to normalized axes of input", &p.beta, &b_scalar));
    RTB_TRY(sc.contiguous(&xv, &xc));
    RTB_TRY(sc.out(out, RTEN_F32, nd, xv.shape, &ov, nullptr));
    if (numel(&xv) == 0) return sc.finish(RTEN_OK);
    long long n = 1;
    for (int i = ax; i < nd; i++) n *= xv.shape[i];
    // scalar gamma / beta stay on the device and are read by the kernel (the reference's scalar-scale arm computes
    // rstd = scale / sqrt(var + eps), src/ops/norm.rs:456-529): no host read, no synchronisation, capturable
    if (g_scalar) std::swap(p.gamma, p.gamma_sp);
    if (b_scalar) std::swap(p.beta, p.beta_sp);
    rten_tensor yc = ov;
    const bool direct = is_contiguous(&ov);
    if (!direct) {
        set_contiguous(&yc);
        RTB_TRY(temp_alloc(ctx, (size_t)numel(&xv) * 4, &yc.data));
    }
    p.x = (const float*)xc.data;
    p.xs = n;
    p.y = (float*)yc.data;
    p.n = (int)n;
    p.rows = numel(&xv) / n;
    RTB_TRY(launch_norm(ctx, p));
    return sc.finish(direct ? RTEN_OK : copy_view(ctx, yc, ov));
}

// ---- RMSNormalization and the skip layer norms ------------------------------------------------------
// Row stride of x viewed as rows over its dims [ax, ndim), when those are packed (element stride 1) and the leading
// dims step uniformly; false for any other layout.
static bool row_stride(const rten_tensor& t, int ax, long long* rs) {
    long long s = 1;
    for (int i = t.ndim - 1; i >= ax; i--) {
        if (t.shape[i] != 1 && t.strides[i] != s) return false;
        s *= t.shape[i];
    }
    long long step = -1, span = 1;  // stride of the row index; rows spanned by the dims after i
    for (int i = ax - 1; i >= 0; i--) {
        if (t.shape[i] == 1) continue;
        if (step < 0) {
            step = t.strides[i];
        } else if (t.strides[i] != step * span) {
            return false;
        }
        span *= t.shape[i];
    }
    *rs = step < 0 ? s : step;
    return true;
}

// x as rows for the kernels: a device view, a contiguous copy when the layout has no single row stride
static rten_status norm_rows(OpScope& sc, const rten_tensor& xv, int ax, rten_tensor* xr, long long* rs) {
    if (row_stride(xv, ax, rs)) {
        *xr = xv;
        return RTEN_OK;
    }
    RTB_TRY(sc.contiguous(&xv, xr));
    return row_stride(*xr, ax, rs) ? RTEN_OK : fail(sc.ctx, RTEN_ERR_INVALID_VALUE, "row view");
}

static rten_status norm_out(OpScope& sc, rten_tensor* o, const rten_tensor& xv, rten_tensor* ov) {
    RTB_TRY(sc.out(o, RTEN_F32, xv.ndim, xv.shape, ov, nullptr));
    return is_contiguous(ov) ? RTEN_OK : fail(sc.ctx, RTEN_ERR_UNSUPPORTED_OUTPUT, "normalization outputs must be contiguous");
}

rten_status rten_b200_rms_norm(rten_ctx* ctx, const rten_tensor* x, const rten_tensor* scale, int axis, float epsilon,
                               rten_tensor* out) {
    RTB_TRY(check_ctx(ctx));
    if (!x || !scale || !out) return fail(ctx, RTEN_ERR_MISSING_INPUTS, "missing inputs");
    if (x->dtype != RTEN_F32 || scale->dtype != RTEN_F32) return fail(ctx, RTEN_ERR_UNSUPPORTED_TYPE, "unsupported type");
    const int nd = x->ndim;
    if (axis < -nd || axis >= std::max(nd, 1)) return fail(ctx, RTEN_ERR_INVALID_VALUE, "Axis is invalid");
    const int ax = axis < 0 ? axis + nd : axis;
    OpScope sc(ctx);
    rten_tensor xv, sv, xr, ov;
    NormParams p;
    p.eps = epsilon < 0.0f ? 1e-5f : epsilon;
    p.rms = 1;
    bool g_scalar = false;
    RTB_TRY(sc.in(x, &xv));
    RTB_TRY(sc.in(scale, &sv));
    RTB_TRY(norm_param(sc, sv, xv, ax, "`scale` is not broadcastable to normalized axes of input", &p.gamma, &g_scalar));
    RTB_TRY(norm_out(sc, out, xv, &ov));
    if (numel(&xv) == 0) return sc.finish(RTEN_OK);
    RTB_TRY(norm_rows(sc, xv, ax, &xr, &p.xs));
    if (g_scalar) std::swap(p.gamma, p.gamma_sp);
    long long n = 1;
    for (int i = ax; i < nd; i++) n *= xv.shape[i];
    p.x = (const float*)xr.data;
    p.y = (float*)ov.data;
    p.n = (int)n;
    p.rows = numel(&xv) / n;
    return sc.finish(launch_norm(ctx, p));
}

rten_status rten_b200_skip_layer_norm(rten_ctx* ctx, const rten_tensor* x, const rten_tensor* skip, const rten_tensor* gamma,
                                      const rten_tensor* beta, const rten_tensor* bias, float epsilon, int rms,
                                      rten_tensor* out, rten_tensor* sum_out) {
    RTB_TRY(check_ctx(ctx));
    if (!x || !skip || !gamma || !out) return fail(ctx, RTEN_ERR_MISSING_INPUTS, "missing inputs");
    for (const rten_tensor* t : {x, skip, gamma, beta, bias})
        if (t && t->dtype != RTEN_F32) return fail(ctx, RTEN_ERR_UNSUPPORTED_TYPE, "unsupported type");
    for (const rten_tensor* t : {gamma, beta, bias})
        if (t && t->ndim != 1) return fail(ctx, RTEN_ERR_CAST_FAILED, "gamma, beta and bias must be 1-D tensors");
    if (rms && beta) return fail(ctx, RTEN_ERR_INVALID_VALUE, "SkipSimplifiedLayerNormalization has no beta input");
    // src/ops/norm/contrib.rs skip_layer_normalization
    const int nd = x->ndim, sd = skip->ndim;
    if (nd != 2 && nd != 3) return fail(ctx, RTEN_ERR_INVALID_VALUE, "input must be 2 or 3 dimensioned");
    if (sd != 2 && sd != 3) return fail(ctx, RTEN_ERR_INVALID_VALUE, "skip must be 2 or 3 dimensioned");
    bool bcast = skip->shape[sd - 1] == x->shape[nd - 1] && skip->shape[sd - 2] == x->shape[nd - 2] && sd <= nd;
    if (bcast && sd == 3) bcast = skip->shape[0] == x->shape[0] || skip->shape[0] == 1;
    if (!bcast) return fail(ctx, RTEN_ERR_INCOMPATIBLE_SHAPES, "skip must broadcast to input over the batch dimension");
    const int64_t H = x->shape[nd - 1];
    // (the reference panics in add_in_place on any other length)
    if (bias && bias->shape[0] != H && bias->shape[0] != 1)
        return fail(ctx, RTEN_ERR_INVALID_VALUE, "bias length must equal the hidden size");
    OpScope sc(ctx);
    rten_tensor xv, kv, gv, bev, biv, xr, kr, ov, smv;
    NormParams p;
    p.eps = epsilon;
    p.rms = rms ? 1 : 0;
    bool g_scalar = false, b_scalar = false;
    RTB_TRY(sc.in(x, &xv));
    RTB_TRY(sc.in(skip, &kv));
    RTB_TRY(sc.in(gamma, &gv));
    if (beta) RTB_TRY(sc.in(beta, &bev));
    if (bias) RTB_TRY(sc.in(bias, &biv));
    const int ax = nd - 1;
    RTB_TRY(norm_param(sc, gv, xv, ax, "`scale` is not broadcastable to normalized axes of input", &p.gamma, &g_scalar));
    if (beta) RTB_TRY(norm_param(sc, bev, xv, ax, "`bias` is not broadcastable to normalized axes of input", &p.beta, &b_scalar));
    RTB_TRY(norm_out(sc, out, xv, &ov));
    if (sum_out) RTB_TRY(norm_out(sc, sum_out, xv, &smv));
    if (numel(&xv) == 0) return sc.finish(RTEN_OK);
    RTB_TRY(norm_rows(sc, xv, ax, &xr, &p.xs));
    RTB_TRY(norm_rows(sc, kv, sd - 1, &kr, &p.ss));
    if (g_scalar) std::swap(p.gamma, p.gamma_sp);
    if (b_scalar) std::swap(p.beta, p.beta_sp);
    if (bias) {
        p.bias = (const float*)biv.data;
        p.bias_inc = biv.shape[0] == 1 ? 0 : (int)biv.strides[0];
    }
    p.x = (const float*)xr.data;
    p.skip = (const float*)kr.data;
    p.skip_rows = numel(&kv) / H;
    p.y = (float*)ov.data;
    p.sum = sum_out ? (float*)smv.data : nullptr;
    p.n = (int)H;
    p.rows = numel(&xv) / H;
    return sc.finish(launch_norm(ctx, p));
}

// ---- InstanceNormalization, the GroupNorm chain and BatchNormalization ------------------------------------
// The kernels' view of x: 0 for [N, C, P] contiguous, 1 for a dense channels-last 4-D tensor, -1 for anything else
static int gn_layout(const rten_tensor& t) {
    if (is_contiguous(&t)) return 0;
    if (t.ndim != 4) return -1;
    const int64_t C = t.shape[1], H = t.shape[2], W = t.shape[3];
    return t.strides[1] == 1 && t.strides[3] == C && (t.strides[2] == W * C || H == 1) && (t.strides[0] == H * W * C || t.shape[0] == 1)
               ? 1 : -1;
}

// One [n] vector of an operator as a contiguous device array (checked by the caller)
static rten_status gn_vector(OpScope& sc, const rten_tensor* t, const float** ptr) {
    rten_tensor v, c;
    RTB_TRY(sc.in(t, &v));
    RTB_TRY(sc.contiguous(&v, &c));
    *ptr = (const float*)c.data;
    return RTEN_OK;
}

// Rows of `groups` per image, checked by the entry points.  With bn_mean (and bn_var): BatchNormalization, groups = C,
// inst_scale / inst_bias its scale and bias; a rank-1 x is one channel.
static rten_status group_norm_run(rten_ctx* ctx, const rten_tensor* x, int groups, const rten_tensor* inst_scale,
                                  const rten_tensor* inst_bias, const rten_tensor* gamma, const rten_tensor* beta, float epsilon,
                                  const rten_activation* act, rten_tensor* out, const rten_tensor* bn_mean = nullptr,
                                  const rten_tensor* bn_var = nullptr) {
    OpScope sc(ctx);
    rten_tensor xv, xc, ov;
    GroupNormParams p;
    RTB_TRY(sc.in(x, &xv));
    int layout = gn_layout(xv);
    if (layout < 0) {  // any other strides: a contiguous copy, and the [N, C, P] path
        RTB_TRY(sc.contiguous(&xv, &xc));
        layout = 0;
    } else {
        xc = xv;
    }
    RTB_TRY(sc.out(out, RTEN_F32, xv.ndim, xv.shape, &ov, (out->data == nullptr && layout == 1) ? xc.strides : nullptr));
    if (numel(&xv) == 0) return sc.finish(RTEN_OK);
    RTB_TRY(gn_vector(sc, inst_scale, &p.inst_scale));
    RTB_TRY(gn_vector(sc, inst_bias, &p.inst_bias));
    if (gamma) RTB_TRY(gn_vector(sc, gamma, &p.gamma));
    if (beta) RTB_TRY(gn_vector(sc, beta, &p.beta));
    const float *mean = nullptr, *var = nullptr;
    if (bn_mean) RTB_TRY(gn_vector(sc, bn_mean, &mean));
    if (bn_var) RTB_TRY(gn_vector(sc, bn_var, &var));
    // the output in the layout the kernels write: `out` itself when it has it, else a temporary copied into `out`
    bool direct = gn_layout(ov) == layout;
    for (int i = 0; i < ov.ndim && direct; i++)
        if (ov.shape[i] != 1 && ov.strides[i] != xc.strides[i]) direct = false;
    rten_tensor yc = xc;
    if (direct) yc.data = ov.data;
    else RTB_TRY(temp_alloc(ctx, (size_t)numel(&xv) * 4, &yc.data));
    p.x = (const float*)xc.data;
    p.y = (float*)yc.data;
    p.N = xv.shape[0];
    p.C = xv.ndim >= 2 ? (int)xv.shape[1] : 1;
    p.G = groups;
    p.P = numel(&xv) / (p.N * p.C);
    p.channels_last = layout;
    if (bn_mean && p.P == 1) {  // [N, C], [N, C, 1, ..] and rank 1: the memory of one channels-last image of N pixels
        p.P = p.N;
        p.N = 1;
        p.channels_last = 1;
    }
    p.eps = epsilon < 0.0f ? 1e-5f : epsilon;
    if (act) {
        p.act = act->kind;
        p.act_alpha = act->alpha;
        p.act_beta = act->beta;
    }
    RTB_TRY(mean ? launch_batch_norm(ctx, p, mean, var) : launch_group_norm(ctx, p));
    return sc.finish(direct ? RTEN_OK : copy_view(ctx, yc, ov));
}

rten_status rten_b200_instance_norm(rten_ctx* ctx, const rten_tensor* x, const rten_tensor* scale, const rten_tensor* bias,
                                    float epsilon, rten_tensor* out) {
    RTB_TRY(check_ctx(ctx));
    if (!x || !scale || !bias || !out) return fail(ctx, RTEN_ERR_MISSING_INPUTS, "missing inputs");
    for (const rten_tensor* t : {x, scale, bias})
        if (t->dtype != RTEN_F32) return fail(ctx, RTEN_ERR_UNSUPPORTED_TYPE, "unsupported type");
    if (scale->ndim != 1 || bias->ndim != 1) return fail(ctx, RTEN_ERR_CAST_FAILED, "scale and bias must be 1-D tensors");
    // src/ops/norm.rs instance_normalization_in_place
    if (x->ndim < 2) return fail(ctx, RTEN_ERR_INVALID_VALUE, "expected input with >= 2 dims");
    if (scale->shape[0] != x->shape[1]) return fail(ctx, RTEN_ERR_INVALID_VALUE, "scale length should match channel count");
    if (bias->shape[0] != x->shape[1]) return fail(ctx, RTEN_ERR_INVALID_VALUE, "bias length should match channel count");
    if (x->shape[1] > INT32_MAX) return fail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "channel count out of range");
    return group_norm_run(ctx, x, (int)x->shape[1], scale, bias, nullptr, nullptr, epsilon, nullptr, out);
}

rten_status rten_b200_group_norm(rten_ctx* ctx, const rten_tensor* x, int groups, const rten_tensor* inst_scale,
                                 const rten_tensor* inst_bias, const rten_tensor* gamma, const rten_tensor* beta, float epsilon,
                                 const rten_activation* act, rten_tensor* out) {
    RTB_TRY(check_ctx(ctx));
    if (!x || !inst_scale || !inst_bias || !out) return fail(ctx, RTEN_ERR_MISSING_INPUTS, "missing inputs");
    for (const rten_tensor* t : {x, inst_scale, inst_bias, gamma, beta})
        if (t && t->dtype != RTEN_F32) return fail(ctx, RTEN_ERR_UNSUPPORTED_TYPE, "unsupported type");
    if (inst_scale->ndim != 1 || inst_bias->ndim != 1) return fail(ctx, RTEN_ERR_CAST_FAILED, "scale and bias must be 1-D tensors");
    if (x->ndim < 2) return fail(ctx, RTEN_ERR_INVALID_VALUE, "expected input with >= 2 dims");
    if (groups <= 0 || x->shape[1] % groups != 0 || x->shape[1] > INT32_MAX)  // Reshape [N, G, -1]
        return fail(ctx, RTEN_ERR_INVALID_VALUE, "Input length must be a multiple of specified dimensions");
    if (inst_scale->shape[0] != groups) return fail(ctx, RTEN_ERR_INVALID_VALUE, "scale length should match channel count");
    if (inst_bias->shape[0] != groups) return fail(ctx, RTEN_ERR_INVALID_VALUE, "bias length should match channel count");
    for (const rten_tensor* t : {gamma, beta})  // Mul / Add of a per-channel [C, 1, ..] constant
        if (t && numel(t) != x->shape[1]) return fail(ctx, RTEN_ERR_INCOMPATIBLE_SHAPES, "Cannot broadcast inputs");
    if (act && (act->kind < RTEN_ACT_NONE || act->kind > RTEN_ACT_HARD_SWISH))
        return fail(ctx, RTEN_ERR_INVALID_VALUE, "unknown activation kind");
    return group_norm_run(ctx, x, groups, inst_scale, inst_bias, gamma, beta, epsilon, act, out);
}

rten_status rten_b200_batch_norm(rten_ctx* ctx, const rten_tensor* x, const rten_tensor* scale, const rten_tensor* bias,
                                 const rten_tensor* mean, const rten_tensor* var, float epsilon, const rten_activation* act,
                                 rten_tensor* out) {
    RTB_TRY(check_ctx(ctx));
    if (!x || !scale || !bias || !mean || !var || !out) return fail(ctx, RTEN_ERR_MISSING_INPUTS, "missing inputs");
    for (const rten_tensor* t : {x, scale, bias, mean, var})
        if (t->dtype != RTEN_F32) return fail(ctx, RTEN_ERR_UNSUPPORTED_TYPE, "unsupported type");
    if (scale->ndim != 1 || bias->ndim != 1 || mean->ndim != 1 || var->ndim != 1)
        return fail(ctx, RTEN_ERR_CAST_FAILED, "scale, bias, mean and var must be 1-D tensors");
    // src/ops/norm.rs batch_norm_in_place
    if (x->ndim < 1) return fail(ctx, RTEN_ERR_INVALID_VALUE, "Input must have at least 1 dim");
    const int64_t C = x->ndim >= 2 ? x->shape[1] : 1;
    if (scale->shape[0] != C) return fail(ctx, RTEN_ERR_INCOMPATIBLE_SHAPES, "scale.size(0) != channels");
    if (bias->shape[0] != C) return fail(ctx, RTEN_ERR_INCOMPATIBLE_SHAPES, "bias.size(0) != channels");
    if (mean->shape[0] != C) return fail(ctx, RTEN_ERR_INCOMPATIBLE_SHAPES, "mean.size(0) != channels");
    if (var->shape[0] != C) return fail(ctx, RTEN_ERR_INCOMPATIBLE_SHAPES, "var.size(0) != channels");
    if (C > INT32_MAX) return fail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "channel count out of range");
    if (act && (act->kind < RTEN_ACT_NONE || act->kind > RTEN_ACT_HARD_SWISH))
        return fail(ctx, RTEN_ERR_INVALID_VALUE, "unknown activation kind");
    return group_norm_run(ctx, x, (int)C, scale, bias, nullptr, nullptr, epsilon, act, out, mean, var);
}

// ---- unary elementwise ----------------------------------------------------------------------------
// out = f(x) elementwise for a 4-byte element type, `flat(in, out, n)` launching f over n contiguous elements.  Dense
// (any dim order) tensors are processed in memory order: the output takes the input's strides.
extern "C++" {
template <class Flat>
rten_status elementwise_op(OpScope& sc, const rten_tensor* x, rten_tensor* out, Flat flat) {
    rten_ctx* ctx = sc.ctx;
    rten_tensor xv, ov;
    RTB_TRY(sc.in(x, &xv));
    const bool dense = span_elems(&xv) == numel(&xv);
    RTB_TRY(sc.out(out, xv.dtype, xv.ndim, xv.shape, &ov, (out->data == nullptr && dense) ? xv.strides : nullptr));
    if (numel(&xv) == 0) return RTEN_OK;
    bool same_layout = dense;
    for (int i = 0; i < xv.ndim && same_layout; i++)
        if (xv.shape[i] != 1 && xv.strides[i] != ov.strides[i]) same_layout = false;
    if (same_layout) return flat(xv.data, ov.data, numel(&xv));
    rten_tensor xc;
    RTB_TRY(sc.contiguous(&xv, &xc));
    if (is_contiguous(&ov)) return flat(xc.data, ov.data, numel(&xv));
    rten_tensor t = xc;
    RTB_TRY(temp_alloc(ctx, (size_t)numel(&xv) * 4, &t.data));
    RTB_TRY(flat(xc.data, t.data, numel(&xv)));
    return copy_view(ctx, t, ov);
}
}  // extern "C++"

static rten_status unary_op(rten_ctx* ctx, int op, const rten_tensor* x, rten_tensor* out, float alpha = 0.0f,
                            float beta = 0.0f) {
    RTB_TRY(check_ctx(ctx));
    if (!x || !out) return fail(ctx, RTEN_ERR_MISSING_INPUTS, "missing inputs");
    if (x->dtype != RTEN_F32) return fail(ctx, RTEN_ERR_UNSUPPORTED_TYPE, "unsupported type");
    OpScope sc(ctx);
    return sc.finish(elementwise_op(sc, x, out, [&](const void* a, void* y, long long n) {
        return launch_unary(ctx, op, (const float*)a, (float*)y, n, alpha, beta);
    }));
}

rten_status rten_b200_clip(rten_ctx* ctx, const rten_tensor* x, const rten_tensor* min, const rten_tensor* max, rten_tensor* out) {
    RTB_TRY(check_ctx(ctx));
    if (!x || !out) return fail(ctx, RTEN_ERR_MISSING_INPUTS, "missing inputs");
    if (x->dtype != RTEN_F32 && x->dtype != RTEN_I32) return fail(ctx, RTEN_ERR_UNSUPPORTED_TYPE, "unsupported type");
    for (const rten_tensor* b : {min, max})
        if (b && (b->dtype != x->dtype || numel(b) != 1))
            return fail(ctx, RTEN_ERR_INVALID_VALUE, "min and max must be scalars of the input's type");
    OpScope sc(ctx);
    rten_tensor mn, mx;  // (read on the device by the kernel: no host synchronisation)
    if (min) RTB_TRY(sc.in(min, &mn));
    if (max) RTB_TRY(sc.in(max, &mx));
    return sc.finish(elementwise_op(sc, x, out, [&](const void* a, void* y, long long n) {
        return launch_clip(ctx, x->dtype == RTEN_I32, a, y, n, min ? mn.data : nullptr, max ? mx.data : nullptr);
    }));
}

rten_status rten_b200_erf(rten_ctx* ctx, const rten_tensor* x, rten_tensor* out) { return unary_op(ctx, UNARY_ERF, x, out); }
rten_status rten_b200_gelu(rten_ctx* ctx, const rten_tensor* x, int approximate, rten_tensor* out) {
    return unary_op(ctx, approximate ? UNARY_APPROX_GELU : UNARY_GELU, x, out);
}
rten_status rten_b200_relu(rten_ctx* ctx, const rten_tensor* x, rten_tensor* out) { return unary_op(ctx, UNARY_RELU, x, out); }
rten_status rten_b200_sigmoid(rten_ctx* ctx, const rten_tensor* x, rten_tensor* out) { return unary_op(ctx, UNARY_SIGMOID, x, out); }
rten_status rten_b200_silu(rten_ctx* ctx, const rten_tensor* x, rten_tensor* out) { return unary_op(ctx, UNARY_SILU, x, out); }
rten_status rten_b200_hard_sigmoid(rten_ctx* ctx, const rten_tensor* x, float alpha, float beta, rten_tensor* out) {
    return unary_op(ctx, UNARY_HARD_SIGMOID, x, out, alpha, beta);
}
rten_status rten_b200_hard_swish(rten_ctx* ctx, const rten_tensor* x, rten_tensor* out) {
    return unary_op(ctx, UNARY_HARD_SWISH, x, out);
}
rten_status rten_b200_sqrt(rten_ctx* ctx, const rten_tensor* x, rten_tensor* out) { return unary_op(ctx, UNARY_SQRT, x, out); }
rten_status rten_b200_reciprocal(rten_ctx* ctx, const rten_tensor* x, rten_tensor* out) {
    return unary_op(ctx, UNARY_RECIPROCAL, x, out);
}
rten_status rten_b200_exp(rten_ctx* ctx, const rten_tensor* x, rten_tensor* out) { return unary_op(ctx, UNARY_EXP, x, out); }
rten_status rten_b200_tanh(rten_ctx* ctx, const rten_tensor* x, rten_tensor* out) { return unary_op(ctx, UNARY_TANH, x, out); }
rten_status rten_b200_neg(rten_ctx* ctx, const rten_tensor* x, rten_tensor* out) { return unary_op(ctx, UNARY_NEG, x, out); }
rten_status rten_b200_abs(rten_ctx* ctx, const rten_tensor* x, rten_tensor* out) { return unary_op(ctx, UNARY_ABS, x, out); }

// ---- Add / Sub / Mul / Div / Pow ----------------------------------------------------------------------------
// Add / Sub / Mul / Div / Pow with numpy broadcasting (src/ops/binary_elementwise.rs), f32 or i32.  `scalar_b`: a
// one-element b is the 0-D scalar the reference maps a with (Div's multiplication by the reciprocal, Pow's map_in), so
// the output takes a's shape.
static rten_status binary_op(rten_ctx* ctx, const rten_tensor* a, const rten_tensor* b, rten_tensor* out, int op,
                             bool scalar_b = false) {
    RTB_TRY(check_ctx(ctx));
    if (!a || !b || !out) return fail(ctx, RTEN_ERR_MISSING_INPUTS, "missing inputs");
    if ((a->dtype != RTEN_F32 && a->dtype != RTEN_I32) || b->dtype != a->dtype) return fail(ctx, RTEN_ERR_UNSUPPORTED_TYPE, "unsupported type");
    const int dt = a->dtype;
    OpScope sc(ctx);
    rten_tensor av, bv, ov;
    RTB_TRY(sc.in(a, &av));
    RTB_TRY(sc.in(b, &bv));
    scalar_b = scalar_b && numel(&bv) == 1;
    if (scalar_b) bv.ndim = 0;
    if (scalar_b && dt == RTEN_F32 && op == BIN_DIV) op = BIN_RCP_MUL;
    int nd = std::max(av.ndim, bv.ndim);
    int64_t shape[RTEN_MAX_DIMS];
    long long sa[RTEN_MAX_DIMS], sb[RTEN_MAX_DIMS];
    for (int i = 0; i < nd; i++) {
        const int ia = i - (nd - av.ndim), ib = i - (nd - bv.ndim);
        const int64_t da = ia >= 0 ? av.shape[ia] : 1, db = ib >= 0 ? bv.shape[ib] : 1;
        if (da != db && da != 1 && db != 1) return fail(ctx, RTEN_ERR_INCOMPATIBLE_SHAPES, "Cannot broadcast inputs");
        shape[i] = (da == 0 || db == 0) ? 0 : std::max(da, db);
        sa[i] = (ia >= 0 && da != 1) ? av.strides[ia] : 0;
        sb[i] = (ib >= 0 && db != 1) ? bv.strides[ib] : 0;
    }
    // same-shape dense operands, or a dense a and a scalar b: keep a's layout for the output
    const bool a_dense = span_elems(&av) == numel(&av);
    bool same = av.ndim == bv.ndim && a_dense;
    for (int i = 0; i < nd && same; i++)
        if (av.shape[i] != bv.shape[i] || (av.shape[i] != 1 && av.strides[i] != bv.strides[i])) same = false;
    RTB_TRY(sc.out(out, dt, nd, shape, &ov, (out->data == nullptr && (same || (scalar_b && a_dense))) ? av.strides : nullptr));
    // i32 Div checks every divisor, also when nothing is divided: the reference's check_nonzero runs over all of b
    // before the broadcast (binary_elementwise.rs:627-629)
    const bool check_b_only = numel(&ov) == 0 && dt == RTEN_I32 && op == BIN_DIV && numel(&bv) > 0;
    if (numel(&ov) == 0 && !check_b_only) return sc.finish(RTEN_OK);
    // i32 Div: the kernels flag a zero divisor or INT_MIN / -1, read back below
    int* err = nullptr;
    if (dt == RTEN_I32 && op == BIN_DIV) {
        RTB_TRY(temp_alloc(ctx, sizeof(int), (void**)&err));
        RTB_CUDA(ctx, cudaMemsetAsync(err, 0, sizeof(int), ctx->stream));
    }
    bool flat = same || (scalar_b && a_dense);
    for (int i = 0; i < nd && flat; i++)
        if (ov.shape[i] != 1 && ov.strides[i] != av.strides[i]) flat = false;
    const long long n = numel(&ov), one = 1, zero = 0;
    if (check_b_only) {  // b / b over b's own elements flags exactly its zeros
        long long shp[RTEN_MAX_DIMS], bs[RTEN_MAX_DIMS], sd[RTEN_MAX_DIMS];
        long long st = 1;
        for (int i = bv.ndim - 1; i >= 0; i--) {
            shp[i] = bv.shape[i];
            bs[i] = bv.strides[i];
            sd[i] = st;
            st *= bv.shape[i];
        }
        void* tmp = nullptr;
        RTB_TRY(temp_alloc(ctx, (size_t)numel(&bv) * sizeof(int), &tmp));
        RTB_TRY(launch_binary(ctx, dt, op, 0, bv.data, bv.data, tmp, bv.ndim, shp, bs, bs, sd, err));
    } else if (flat) {  // dense operands of one layout: one flat pass over the n elements from the lowest address
        RTB_TRY(launch_binary(ctx, dt, op, 0, av.data, bv.data, ov.data, 1, &n, &one, same ? &one : &zero, &one, err));
    } else {
        long long shp[RTEN_MAX_DIMS], sd[RTEN_MAX_DIMS];
        for (int i = 0; i < nd; i++) {
            shp[i] = shape[i];
            sd[i] = ov.strides[i];
        }
        RTB_TRY(launch_binary(ctx, dt, op, 0, av.data, bv.data, ov.data, nd, shp, sa, sb, sd, err));
    }
    if (err) {
        int h = 0;
        RTB_CUDA(ctx, cudaMemcpyAsync(&h, err, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
        RTB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        if (h) return fail(ctx, RTEN_ERR_INVALID_VALUE, "Divisor contains zero");
    }
    return sc.finish(RTEN_OK);
}

rten_status rten_b200_add(rten_ctx* ctx, const rten_tensor* a, const rten_tensor* b, rten_tensor* out) {
    return binary_op(ctx, a, b, out, BIN_ADD);
}
rten_status rten_b200_sub(rten_ctx* ctx, const rten_tensor* a, const rten_tensor* b, rten_tensor* out) {
    return binary_op(ctx, a, b, out, BIN_SUB);
}
rten_status rten_b200_mul(rten_ctx* ctx, const rten_tensor* a, const rten_tensor* b, rten_tensor* out) {
    return binary_op(ctx, a, b, out, BIN_MUL);
}
rten_status rten_b200_div(rten_ctx* ctx, const rten_tensor* a, const rten_tensor* b, rten_tensor* out) {
    return binary_op(ctx, a, b, out, BIN_DIV, b && b->dtype == RTEN_F32);
}
rten_status rten_b200_pow(rten_ctx* ctx, const rten_tensor* a, const rten_tensor* b, rten_tensor* out) {
    return binary_op(ctx, a, b, out, BIN_POW, true);
}

// ---- ReduceSum, ReduceMean ----------------------------------------------------------------------------------
// src/ops/reduce.rs reduce_sum / reduce_mean: the axes resolved (negative from the end), sorted and de-duplicated; none
// reduces every axis.  A 0-D input is its own one-element lane.  `mean`: f32 only, each sum divided by the lane length.
static rten_status reduce_run(rten_ctx* ctx, const rten_tensor* x, const int32_t* axes, int n_axes, int keep_dims, rten_tensor* out,
                              int mean) {
    RTB_TRY(check_ctx(ctx));
    if (!x || !out) return fail(ctx, RTEN_ERR_MISSING_INPUTS, "missing inputs");
    if (x->dtype != RTEN_F32 && (mean || x->dtype != RTEN_I32)) return fail(ctx, RTEN_ERR_UNSUPPORTED_TYPE, "unsupported type");
    if (n_axes < 0 || (n_axes > 0 && !axes)) return fail(ctx, RTEN_ERR_INVALID_VALUE, "axes must be a list of n_axes values");
    const int nd = x->ndim;
    bool red[RTEN_MAX_DIMS] = {};
    for (int i = 0; i < n_axes; i++) {
        const int64_t a = axes[i] < 0 ? (int64_t)axes[i] + nd : axes[i];
        if (a < 0 || a >= nd) return fail(ctx, RTEN_ERR_INVALID_VALUE, "Axis is invalid");
        red[a] = true;
    }
    if (n_axes == 0)
        for (int i = 0; i < nd; i++) red[i] = true;
    int ond = 0;
    int64_t oshape[RTEN_MAX_DIMS];
    for (int i = 0; i < nd; i++)
        if (!red[i] || keep_dims) oshape[ond++] = red[i] ? 1 : x->shape[i];
    OpScope sc(ctx);
    rten_tensor xv, ov;
    RTB_TRY(sc.in(x, &xv));
    RTB_TRY(sc.out(out, x->dtype, ond, oshape, &ov, nullptr));
    ReduceParams p;
    p.x = xv.data;
    p.y = ov.data;
    p.nout = numel(&ov);
    p.L = 1;
    // kept dims of size > 1 (with the output stride of each), reduced dims of size != 1, adjacent dense reduced dims merged
    for (int i = 0, k = 0; i < nd; i++) {
        const int oi = (!red[i] || keep_dims) ? k++ : -1;
        if (!red[i]) {
            if (xv.shape[i] == 1) continue;
            p.os[p.no] = xv.shape[i], p.ox[p.no] = xv.strides[i], p.oy[p.no] = ov.strides[oi];
            p.no++;
        } else {
            p.L *= xv.shape[i];
            if (xv.shape[i] == 1) continue;
            if (p.nr > 0 && p.rx[p.nr - 1] == xv.strides[i] * xv.shape[i]) {
                p.rs[p.nr - 1] *= xv.shape[i];
                p.rx[p.nr - 1] = xv.strides[i];
            } else {
                p.rs[p.nr] = xv.shape[i], p.rx[p.nr] = xv.strides[i];
                p.nr++;
            }
        }
    }
    bool vec = (p.nr == 0 || (p.nr == 1 && p.rx[0] == 1)) && (reinterpret_cast<uintptr_t>(xv.data) & 15) == 0;
    for (int k = 0; k < p.no && vec; k++) vec = p.ox[k] % 4 == 0;
    p.vec = vec;
    p.mean = mean;
    return sc.finish(launch_reduce_sum(ctx, x->dtype, p));
}

rten_status rten_b200_reduce_sum(rten_ctx* ctx, const rten_tensor* x, const int32_t* axes, int n_axes, int keep_dims, rten_tensor* out) {
    return reduce_run(ctx, x, axes, n_axes, keep_dims, out, 0);
}
rten_status rten_b200_reduce_mean(rten_ctx* ctx, const rten_tensor* x, const int32_t* axes, int n_axes, int keep_dims,
                                  rten_tensor* out) {
    return reduce_run(ctx, x, axes, n_axes, keep_dims, out, 1);
}

// ---- TopK, ArgMax, ArgMin --------------------------------------------------------------------------------
// One lane per output row along axis `a` of x (any strides); ys[i] is the output stride of input dim i != a, and
// ys[a] the output stride along the axis (TopK).  p.r.y / p.vals are the caller's.
static void select_lanes(const rten_tensor& xv, int a, const int64_t* ys, SelectParams& p) {
    p.r.x = xv.data;
    p.r.L = xv.shape[a];
    p.r.nr = 1, p.r.rs[0] = xv.shape[a], p.r.rx[0] = xv.strides[a];
    p.r.nout = 1;
    for (int i = 0; i < xv.ndim; i++) {
        if (i == a) continue;
        p.r.nout *= xv.shape[i];
        if (xv.shape[i] == 1) continue;
        p.r.os[p.r.no] = xv.shape[i], p.r.ox[p.r.no] = xv.strides[i], p.r.oy[p.r.no] = ys[i];
        p.r.no++;
    }
    p.ys = ys[a];
}

static bool same_layout(const rten_tensor& a, const rten_tensor& b) {
    for (int i = 0; i < a.ndim; i++)
        if (a.shape[i] != 1 && a.strides[i] != b.strides[i]) return false;
    return true;
}

// src/ops/reduce.rs topk (reduce.rs:1236-1306), with the checks in the reference's order
rten_status rten_b200_topk(rten_ctx* ctx, const rten_tensor* x, int64_t k, int axis, int largest, int sorted,
                           rten_tensor* values, rten_tensor* indices) {
    (void)sorted;  // the output is always sorted, which the reference's unspecified unsorted order allows
    RTB_TRY(check_ctx(ctx));
    if (!x || !values || !indices) return fail(ctx, RTEN_ERR_MISSING_INPUTS, "missing inputs");
    if (x->dtype != RTEN_F32 && x->dtype != RTEN_I32) return fail(ctx, RTEN_ERR_UNSUPPORTED_TYPE, "unsupported type");
    if (k < 0) return fail(ctx, RTEN_ERR_INVALID_VALUE, "k must be positive");
    const int nd = x->ndim;
    const int a = axis < 0 ? axis + nd : axis;
    if (a < 0 || a >= nd) return fail(ctx, RTEN_ERR_INVALID_VALUE, "Axis is invalid");
    if (k > 0 && k > x->shape[a]) return fail(ctx, RTEN_ERR_INVALID_VALUE, "k > dimension size");
    if (k > TOPK_MAX_K) return fail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "TopK: k > 2048 is not supported");
    if (x->shape[a] > INT32_MAX)
        return fail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "TopK: an axis of 2^31 or more elements is not supported (i32 indices)");
    int64_t oshape[RTEN_MAX_DIMS];
    for (int i = 0; i < nd; i++) oshape[i] = i == a ? k : x->shape[i];
    OpScope sc(ctx);
    rten_tensor xv, vv, iv;
    RTB_TRY(sc.in(x, &xv));
    RTB_TRY(sc.out(values, x->dtype, nd, oshape, &vv, nullptr));
    RTB_TRY(sc.out(indices, RTEN_I32, nd, oshape, &iv, vv.strides));
    if (numel(&vv) == 0) return sc.finish(RTEN_OK);
    // the kernels write both outputs at the same offsets: indices laid out otherwise go through a copy
    rten_tensor ik = iv;
    if (!same_layout(vv, iv)) {
        ik = vv;
        ik.dtype = RTEN_I32;
        RTB_TRY(temp_alloc(ctx, (size_t)span_elems(&vv) * 4, &ik.data));
    }
    SelectParams p;
    select_lanes(xv, a, vv.strides, p);
    p.r.y = ik.data;
    p.vals = vv.data;
    p.k = (int)k;
    p.mode = largest ? SEL_LARGEST : SEL_SMALLEST;
    RTB_TRY(launch_topk(ctx, x->dtype, p));
    if (ik.data != iv.data) RTB_TRY(copy_view(ctx, ik, iv));
    return sc.finish(RTEN_OK);
}

// src/ops/reduce.rs select_max_index (reduce.rs:62-177)
static rten_status arg_select(rten_ctx* ctx, const rten_tensor* x, int axis, int keep_dims, rten_tensor* out, int mode) {
    RTB_TRY(check_ctx(ctx));
    if (!x || !out) return fail(ctx, RTEN_ERR_MISSING_INPUTS, "missing inputs");
    if (x->dtype != RTEN_F32 && x->dtype != RTEN_I32) return fail(ctx, RTEN_ERR_UNSUPPORTED_TYPE, "unsupported type");
    const int nd = x->ndim;
    const int a = axis < 0 ? axis + nd : axis;
    if (a < 0 || a >= nd) return fail(ctx, RTEN_ERR_INVALID_VALUE, "Axis is invalid");
    if (x->shape[a] == 0) return fail(ctx, RTEN_ERR_INVALID_VALUE, "Cannot select index from empty sequence");
    if (x->shape[a] > INT32_MAX)
        return fail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "ArgMax / ArgMin: an axis of 2^31 or more elements is not supported (i32 indices)");
    int ond = 0;
    int64_t oshape[RTEN_MAX_DIMS];
    for (int i = 0; i < nd; i++)
        if (i != a || keep_dims) oshape[ond++] = i == a ? 1 : x->shape[i];
    OpScope sc(ctx);
    rten_tensor xv, ov;
    RTB_TRY(sc.in(x, &xv));
    RTB_TRY(sc.out(out, RTEN_I32, ond, oshape, &ov, nullptr));
    if (numel(&ov) == 0) return sc.finish(RTEN_OK);
    int64_t ys[RTEN_MAX_DIMS];
    for (int i = 0, o = 0; i < nd; i++) ys[i] = (i != a || keep_dims) ? ov.strides[o++] : 0;
    SelectParams p;
    select_lanes(xv, a, ys, p);
    p.r.y = ov.data;
    p.mode = mode;
    return sc.finish(launch_arg_reduce(ctx, x->dtype, p));
}

rten_status rten_b200_arg_max(rten_ctx* ctx, const rten_tensor* x, int axis, int keep_dims, rten_tensor* out) {
    return arg_select(ctx, x, axis, keep_dims, out, SEL_ARGMAX);
}
rten_status rten_b200_arg_min(rten_ctx* ctx, const rten_tensor* x, int axis, int keep_dims, rten_tensor* out) {
    return arg_select(ctx, x, axis, keep_dims, out, SEL_ARGMIN);
}

// ---- DynamicQuantizeLinear ---------------------------------------------------------------------------
rten_status rten_b200_range_reset(rten_ctx* ctx, rten_tensor* ranges) {
    RTB_TRY(check_ctx(ctx));
    if (!ranges) return fail(ctx, RTEN_ERR_MISSING_INPUTS, "missing inputs");
    if (ranges->dtype != RTEN_I32 || ranges->device < 0 || !is_contiguous(ranges) || numel(ranges) % 2)
        return fail(ctx, RTEN_ERR_INVALID_VALUE, "ranges must be a contiguous device-resident i32[n, 2]");
    cudaSetDevice(ctx->device);
    return launch_range_reset(ctx, (int*)ranges->data, (int)(numel(ranges) / 2));
}

rten_status rten_b200_dynamic_quantize_linear(rten_ctx* ctx, const rten_tensor* x, rten_tensor* y, rten_tensor* scale,
                                              rten_tensor* zero_point, void* nccl_comm) {
    return rten_b200_dynamic_quantize_linear_ranged(ctx, x, nullptr, y, scale, zero_point, nccl_comm);
}

rten_status rten_b200_dynamic_quantize_linear_ranged(rten_ctx* ctx, const rten_tensor* x, const rten_tensor* range,
                                                     rten_tensor* y, rten_tensor* scale, rten_tensor* zero_point,
                                                     void* nccl_comm) {
    RTB_TRY(check_ctx(ctx));
    if (!x || !y || !scale || !zero_point) return fail(ctx, RTEN_ERR_MISSING_INPUTS, "missing inputs");
    if (x->dtype != RTEN_F32) return fail(ctx, RTEN_ERR_UNSUPPORTED_TYPE, "unsupported type");
    if (range && (range->dtype != RTEN_I32 || numel(range) != 2 || range->device < 0 || !is_contiguous(range)))
        return fail(ctx, RTEN_ERR_INVALID_VALUE, "the range must be a device-resident i32[2]");
    OpScope sc(ctx);
    rten_tensor xv, xc, yv, sv, zv;
    RTB_TRY(sc.in(x, &xv));
    // The op is elementwise plus an order-independent min / max: a DENSE input in any dim order (e.g. channels-last
    // activations) is processed in memory order and the quantised output keeps the input's strides.
    bool dense = span_elems(&xv) == numel(&xv) && y->data == nullptr;
    for (int i = 0; i < xv.ndim && dense; i++)
        if (xv.strides[i] <= 0 && xv.shape[i] > 1) dense = false;
    const bool x_cl_dense = xv.ndim == 4 && xv.strides[1] == 1 && xv.strides[3] == xv.shape[1] &&
                            xv.strides[2] == xv.shape[3] * xv.shape[1] && xv.strides[0] == xv.shape[2] * xv.shape[3] * xv.shape[1];
    if (dense || (x_cl_dense && y->data && y->ndim == 4 && y->strides[1] == 1))
        xc = xv;
    else
        RTB_TRY(sc.contiguous(&xv, &xc));
    // A caller-provided channels-last output whose rows (b, h) sit at arbitrary pitches -- the interior of a spatially
    // pre-padded buffer, so that the consuming ConvInteger needs no padded copy -- is written row by row.
    bool rows_out = false;
    if (y->data && xv.ndim == 4 && y->ndim == 4 && y->device >= 0) {
        const int64_t Cc = xv.shape[1], Hh = xv.shape[2], Ww = xv.shape[3];
        rows_out = xv.strides[1] == 1 && xv.strides[3] == Cc && xv.strides[2] == Ww * Cc && xv.strides[0] == Hh * Ww * Cc &&
                   y->strides[1] == 1 && y->strides[3] == Cc && !is_contiguous(y) &&
                   !(y->strides[2] == Ww * Cc && y->strides[0] == Hh * Ww * Cc);
        if (rows_out) xc = xv;
    }
    RTB_TRY(sc.out(y, RTEN_U8, xv.ndim, xv.shape, &yv, dense ? xv.strides : nullptr));
    RTB_TRY(sc.out(scale, RTEN_F32, 0, nullptr, &sv, nullptr));
    RTB_TRY(sc.out(zero_point, RTEN_U8, 0, nullptr, &zv, nullptr));
    if (!dense && !rows_out && !is_contiguous(&yv)) return fail(ctx, RTEN_ERR_UNSUPPORTED_OUTPUT, "quantized output must be contiguous");
    const long long n = numel(&xv);
    if (n == 0) {
        // quantize.rs:378-386: scale 1, zero point 0
        const float one = 1.0f;
        RTB_CUDA(ctx, cudaMemcpyAsync(sv.data, &one, 4, cudaMemcpyHostToDevice, ctx->stream));
        RTB_CUDA(ctx, cudaMemsetAsync(zv.data, 0, 1, ctx->stream));
        return sc.finish(RTEN_OK);
    }
    if (!nccl_comm && !range && !rows_out && n <= 16384)
        return sc.finish(launch_dql_small(ctx, (const float*)xc.data, (uint8_t*)yv.data, (int)n, (float*)sv.data, (uint8_t*)zv.data));
    // `range`: the producer of x already accumulated (min, max) in its epilogue -- no pass over x for it
    int* mm = range ? (int*)range->data : nullptr;
    if (!mm) {
        RTB_TRY(temp_alloc(ctx, 8, (void**)&mm));
        RTB_TRY(launch_minmax(ctx, (const float*)xc.data, n, mm));
    }
    // batch-sharded run: the range is the range of the whole (unsharded) tensor -- exchanged over NVLink peer
    // mailboxes by the quantise kernel's own prologue, or by two ncclAllReduce calls in front of it
    RangeExchange xch;
    const bool fused_xch = nccl_comm && comm_range_exchange(reinterpret_cast<rten_comm*>(nccl_comm), &xch);
    if (nccl_comm && !fused_xch) RTB_TRY(comm_allreduce_minmax(ctx, reinterpret_cast<rten_comm*>(nccl_comm), mm));
    if (rows_out)
        return sc.finish(launch_dql_quantize_rows(ctx, (const float*)xc.data, (uint8_t*)yv.data, xv.shape[0] * xv.shape[2],
                                                  (int)(xv.shape[3] * xv.shape[1]), (int)xv.shape[2], yv.strides[2], yv.strides[0],
                                                  mm, (float*)sv.data, (uint8_t*)zv.data, fused_xch ? &xch : nullptr));
    return sc.finish(launch_dql_quantize(ctx, (const float*)xc.data, (uint8_t*)yv.data, n, mm, (float*)sv.data, (uint8_t*)zv.data,
                                         fused_xch ? &xch : nullptr));
}

// ---- gather / scatter ------------------------------------------------------------------------------
rten_status rten_b200_gather_rows(rten_ctx* ctx, const rten_tensor* table, const rten_tensor* idx, rten_tensor* out) {
    RTB_TRY(check_ctx(ctx));
    if (!table || !idx || !out) return fail(ctx, RTEN_ERR_MISSING_INPUTS, "missing inputs");
    if (table->dtype != RTEN_F32 || idx->dtype != RTEN_I32) return fail(ctx, RTEN_ERR_UNSUPPORTED_TYPE, "unsupported type");
    if (table->ndim != 2) return fail(ctx, RTEN_ERR_INVALID_VALUE, "gather_rows expects a 2-D table");
    OpScope sc(ctx);
    rten_tensor tv, iv, ic, ov;
    RTB_TRY(sc.in(table, &tv));
    RTB_TRY(sc.in(idx, &iv));
    RTB_TRY(sc.contiguous(&iv, &ic));
    int64_t oshape[RTEN_MAX_DIMS];
    if (iv.ndim + 1 > RTEN_MAX_DIMS) return fail(ctx, RTEN_ERR_INVALID_VALUE, "tensor rank out of range");
    for (int i = 0; i < iv.ndim; i++) oshape[i] = iv.shape[i];
    oshape[iv.ndim] = tv.shape[1];
    RTB_TRY(sc.out(out, RTEN_F32, iv.ndim + 1, oshape, &ov, nullptr));
    if (!is_contiguous(&ov)) return fail(ctx, RTEN_ERR_UNSUPPORTED_OUTPUT, "gather output must be contiguous");
    return sc.finish(launch_gather_rows(ctx, (const float*)tv.data, (const int*)ic.data, (float*)ov.data, numel(&iv),
                                        (int)tv.shape[1], tv.strides[0], tv.strides[1], tv.shape[0]));
}

rten_status rten_b200_scatter_rows(rten_ctx* ctx, rten_tensor* table, const rten_tensor* idx, const rten_tensor* src) {
    RTB_TRY(check_ctx(ctx));
    if (!table || !idx || !src) return fail(ctx, RTEN_ERR_MISSING_INPUTS, "missing inputs");
    if (table->dtype != RTEN_F32 || src->dtype != RTEN_F32 || idx->dtype != RTEN_I32)
        return fail(ctx, RTEN_ERR_UNSUPPORTED_TYPE, "unsupported type");
    if (table->ndim != 2 || src->ndim != 2 || idx->ndim != 1) return fail(ctx, RTEN_ERR_INVALID_VALUE, "scatter_rows expects 2-D table / updates and 1-D indices");
    if (src->shape[0] != idx->shape[0] || src->shape[1] != table->shape[1])
        return fail(ctx, RTEN_ERR_INCOMPATIBLE_SHAPES, "updates do not match the indices / table width");
    if (table->device < 0) return fail(ctx, RTEN_ERR_UNSUPPORTED_OUTPUT, "the table must be device resident (updated in place)");
    OpScope sc(ctx);
    rten_tensor iv, ic, sv;
    RTB_TRY(sc.in(idx, &iv));
    RTB_TRY(sc.contiguous(&iv, &ic));
    RTB_TRY(sc.in(src, &sv));
    return sc.finish(launch_scatter_rows(ctx, (float*)table->data, (const int*)ic.data, (const float*)sv.data, iv.shape[0],
                                         (int)table->shape[1], table->strides[0], table->strides[1], sv.strides[0], sv.strides[1],
                                         table->shape[0]));
}

}  // extern "C"
