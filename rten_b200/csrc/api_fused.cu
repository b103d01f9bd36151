// Fused operator entry point of the C ABI for the autoregressive decode path (include/rten_b200.h):
//   rten_b200_quantized_linear : [LayerNormalization] -> DynamicQuantizeLinear -> MatMulIntegerToFloat -> Add -> Add -> act
// It has a hand-written skinny-M kernel (skinny.cu) for the decode shapes and otherwise composes the public operators of
// this library, so every shape the operator chain accepts is served with identical results.
#include <cuda_runtime.h>

#include "api_util.h"
#include "rowops.h"
#include "skinny.h"

using namespace rtb;

extern "C" {

rten_status rten_b200_quantized_linear(rten_ctx* ctx, const rten_tensor* x, const rten_tensor* ln_scale, const rten_tensor* ln_bias,
                                       float ln_epsilon, const rten_tensor* w, const rten_packed* pw, const rten_tensor* w_zp,
                                       const rten_tensor* w_scale, const rten_tensor* bias, const rten_tensor* residual,
                                       int activation, rten_tensor* out) {
    RTB_TRY(check_ctx(ctx));
    if (!x || !w || !w_scale || !out) return fail(ctx, RTEN_ERR_MISSING_INPUTS, "missing inputs");
    if (x->dtype != RTEN_F32 || w_scale->dtype != RTEN_F32) return fail(ctx, RTEN_ERR_UNSUPPORTED_TYPE, "unsupported type");
    if (w->dtype != RTEN_I8 && w->dtype != RTEN_U8) return fail(ctx, RTEN_ERR_UNSUPPORTED_TYPE, "unsupported type");
    if (w->ndim != 2) return fail(ctx, RTEN_ERR_INVALID_VALUE, "the weight must be a matrix");
    if (activation < 0 || activation > 3) return fail(ctx, RTEN_ERR_INVALID_VALUE, "unknown activation");
    if (ln_bias && !ln_scale) return fail(ctx, RTEN_ERR_MISSING_INPUTS, "missing inputs");
    if (x->ndim < 1) return fail(ctx, RTEN_ERR_INVALID_VALUE, "Inputs must have >= 1 dimensions");
    const int64_t K = x->shape[x->ndim - 1], N = w->shape[1];
    if (K != w->shape[0])
        return fail(ctx, RTEN_ERR_INCOMPATIBLE_SHAPES, "Columns of first matrix does not match rows of second matrix");
    int64_t M = 1;
    for (int i = 0; i + 1 < x->ndim; i++) M *= x->shape[i];

    // ---- fast path: every operand resident, rows uniformly strided, M <= 16
    bool fast = x->device >= 0 && pw && pw->kind == 0 && pw->dtype == w->dtype && pw->K == K && pw->N == N && pw->colsum &&
                w_scale->device >= 0 && (!bias || bias->device >= 0) && (!residual || residual->device >= 0) &&
                (!w_zp || w_zp->device >= 0) && (!ln_scale || ln_scale->device >= 0) && (!ln_bias || ln_bias->device >= 0) &&
                (out->data == nullptr || out->device >= 0) && M >= 1 && N >= 1;
    // x rows: [.., K] with unit inner stride and one uniform row stride
    int64_t xs = K;
    if (fast) {
        if (x->strides[x->ndim - 1] != 1 && K > 1) fast = false;
        if (x->ndim >= 2) {
            xs = x->strides[x->ndim - 2];
            int64_t expect = xs * x->shape[x->ndim - 2];
            for (int i = x->ndim - 3; i >= 0 && fast; i--) {
                if (x->shape[i] != 1 && x->strides[i] != expect) fast = false;
                expect *= x->shape[i];
            }
        }
    }
    auto vec_ok = [&](const rten_tensor* t, int64_t n) {
        return t->dtype == RTEN_F32 && ((t->ndim == 1 && t->shape[0] == n && (t->strides[0] == 1 || n == 1)) || (numel(t) == 1 && n == 1));
    };
    if (fast && ln_scale && !vec_ok(ln_scale, K)) fast = false;
    if (fast && ln_bias && !vec_ok(ln_bias, K)) fast = false;
    if (fast && bias && !vec_ok(bias, N)) fast = false;
    if (fast && !(numel(w_scale) == 1 || vec_ok(w_scale, N))) fast = false;
    if (fast && w_zp && !((w_zp->dtype == w->dtype) && (numel(w_zp) == 1 || (w_zp->ndim == 1 && w_zp->shape[0] == N)))) fast = false;
    if (fast && residual) {
        if (residual->dtype != RTEN_F32 || numel(residual) != M * N || !is_contiguous(residual)) fast = false;
    }
    if (fast) {
        QLinearLaunch L;
        L.x = (const float*)x->data;
        L.xs = xs;
        L.M = (int)M;
        L.K = (int)K;
        L.N = (int)N;
        L.has_ln = ln_scale ? 1 : 0;
        L.ln_gamma = ln_scale ? (const float*)ln_scale->data : nullptr;
        L.ln_beta = ln_bias ? (const float*)ln_bias->data : nullptr;
        L.ln_eps = ln_epsilon < 0.0f ? 1e-5f : ln_epsilon;
        L.w = pw->data;
        L.ldw = pw->ld;
        L.w_signed = pw->dtype == RTEN_I8;
        L.colsum = pw->colsum;
        L.w_scale = (const float*)w_scale->data;
        L.w_scale_len = (int)numel(w_scale);
        L.bias = bias ? (const float*)bias->data : nullptr;
        L.residual = residual ? (const float*)residual->data : nullptr;
        L.rs = N;
        L.act = activation;
        if (qlinear_supported(L)) {
            OpScope sc(ctx);
            rten_tensor ov;
            int64_t oshape[RTEN_MAX_DIMS];
            for (int i = 0; i + 1 < x->ndim; i++) oshape[i] = x->shape[i];
            oshape[x->ndim - 1] = N;
            RTB_TRY(sc.out(out, RTEN_F32, x->ndim, oshape, &ov, nullptr));
            if (!is_contiguous(&ov)) return fail(ctx, RTEN_ERR_UNSUPPORTED_OUTPUT, "output tensor must be contiguous");
            if (w_zp) {
                int32_t* zb = nullptr;
                const int len = (int)numel(w_zp);
                RTB_TRY(temp_alloc(ctx, (size_t)len * 4, (void**)&zb));
                RTB_TRY(launch_zp_to_i32(ctx, w_zp->data, w_zp->dtype == RTEN_I8, len, w_zp->ndim == 0 ? 0 : w_zp->strides[0], zb));
                L.zb = zb;
                L.zb_len = len;
            }
            L.out = (float*)ov.data;
            L.os = N;
            return sc.finish(launch_qlinear(ctx, L));
        }
    }

    // ---- general path: the operator chain, through this library's own entry points
    Intermediate h(ctx), q(ctx), qs(ctx), qz(ctx);
    const rten_tensor* cur = x;
    if (ln_scale) {
        RTB_TRY(rten_b200_layer_norm(ctx, x, ln_scale, ln_bias, -1, ln_epsilon, &h));
        cur = &h;
    }
    RTB_TRY(rten_b200_dynamic_quantize_linear(ctx, cur, &q, &qs, &qz, nullptr));
    return rten_b200_matmul_integer_ex(ctx, &q, w, pw, &qz, w_zp, w_scale, &qs, bias, residual, activation, nullptr, out);
}

}  // extern "C"
