// Entry points of the C ABI for the recurrent operators (include/rten_b200.h):
//   rten_b200_gru  : GRU  (src/ops/rnn.rs gru)
//   rten_b200_lstm : LSTM (src/ops/rnn.rs lstm)
// Validation restates the reference's checks and messages and adds the dimension checks it leaves out.  The input
// projection x . W^T of all steps and directions is one wgmma GEMM in the context's f32 mode; the recurrence runs on
// rnn.cu's cluster kernel (one launch) or, when R does not fit a cluster, one recurrent product and one gate launch
// per step.
#include <cuda_runtime.h>

#include <climits>
#include <cstdlib>

#include "api_shared.h"
#include "api_util.h"
#include "rnn.h"
#include "rowops.h"
#include "skinny.h"
#include "umma_gemm.h"

using namespace rtb;
using namespace rtb::api;

namespace {

bool same_shape(const rten_tensor* t, int64_t a, int64_t b, int64_t c) {
    return t->shape[0] == a && t->shape[1] == b && t->shape[2] == c;
}

rten_status rnn_run(rten_ctx* ctx, bool gru, const rten_tensor* x, const rten_tensor* w, const rten_packed* pw,
                    const rten_tensor* r, const rten_tensor* bias, const rten_tensor* seq_lens, const rten_tensor* h0,
                    const rten_tensor* c0, const rten_tensor* peephole, const rten_rnn_params* p, rten_tensor* y,
                    rten_tensor* yh, rten_tensor* yc) {
    RTB_TRY(check_ctx(ctx));
    if (!x || !w || !r || !p) return fail(ctx, RTEN_ERR_MISSING_INPUTS, "missing inputs");
    for (const rten_tensor* t : {x, w, r, bias, h0, c0})
        if (t && t->dtype != RTEN_F32) return fail(ctx, RTEN_ERR_CAST_FAILED, "GRU / LSTM inputs must be f32");
    if (seq_lens && seq_lens->dtype != RTEN_I32) return fail(ctx, RTEN_ERR_CAST_FAILED, "sequence_lens must be i32");
    if (p->direction < 0 || p->direction > 2)
        return fail(ctx, RTEN_ERR_INVALID_VALUE, "direction must be forward (0), reverse (1) or bidirectional (2)");
    if (peephole) return fail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "LSTM peephole weights are not supported");
    const int G = gru ? 3 : 4;
    const int dirs = p->direction == 2 ? 2 : 1;
    // src/ops/rnn.rs: the reference's checks, in its order and with its messages
    if (gru) {
        if (!p->linear_before_reset) return fail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "`linear_before_reset=0` is not supported");
        if (x->ndim != 3) return fail(ctx, RTEN_ERR_INVALID_VALUE, "input must have 3 dims (seq, batch, input)");
        if (w->ndim != 3) return fail(ctx, RTEN_ERR_INVALID_VALUE, "weights must have 3 dims (dir, hidden x 3, input)");
        if (r->ndim != 3) return fail(ctx, RTEN_ERR_INVALID_VALUE, "recurrent_weights must have 3 dims");
        if (bias && bias->ndim != 2) return fail(ctx, RTEN_ERR_INVALID_VALUE, "bias must have 2 dims (dir, hidden x 6)");
        if (h0 && h0->ndim != 3) return fail(ctx, RTEN_ERR_INVALID_VALUE, "initial_hidden must have 3 dims");
        if (w->shape[1] % 3 != 0) return fail(ctx, RTEN_ERR_INVALID_VALUE, "weights dim 1 must be 3 * hidden_size");
    } else {
        if (x->ndim != 3) return fail(ctx, RTEN_ERR_INVALID_VALUE, "input must have 3 dims (seq, batch, input)");
        if (w->ndim != 3) return fail(ctx, RTEN_ERR_INVALID_VALUE, "weights must have 3 dims (dir, hidden x 4, input)");
        if (r->ndim != 3) return fail(ctx, RTEN_ERR_INVALID_VALUE, "recurrent_weights must have 3 dims (dir, hidden x 4, hidden)");
        if (w->shape[1] % 4 != 0) return fail(ctx, RTEN_ERR_INVALID_VALUE, "weights dim 1 must be 4 * hidden_size");
        if (bias && bias->ndim != 2) return fail(ctx, RTEN_ERR_INVALID_VALUE, "bias must have 2 dims");
        if (bias && bias->shape[1] % 8 != 0) return fail(ctx, RTEN_ERR_INVALID_VALUE, "bias dim 1 must be 8 * hidden_size");
        if (h0 && h0->ndim != 3) return fail(ctx, RTEN_ERR_INVALID_VALUE, "initial_hidden must have 3 dims");
        if (c0 && c0->ndim != 3) return fail(ctx, RTEN_ERR_INVALID_VALUE, "initial_cell must have 3 dims");
    }
    const int64_t T = x->shape[0], B = x->shape[1], I = x->shape[2], H = w->shape[1] / G, GH = G * H;
    // the dimensions the reference leaves unchecked (it would index out of bounds or silently misread them)
    if (w->shape[0] != dirs) return fail(ctx, RTEN_ERR_INVALID_VALUE, "weights dim 0 must be the number of directions");
    if (w->shape[2] != I) return fail(ctx, RTEN_ERR_INVALID_VALUE, "weights dim 2 must be the input size");
    if (!same_shape(r, dirs, GH, H))
        return fail(ctx, RTEN_ERR_INVALID_VALUE, "recurrent_weights must have shape [directions, gates * hidden_size, hidden_size]");
    if (bias && (bias->shape[0] != dirs || bias->shape[1] != 2 * GH))
        return fail(ctx, RTEN_ERR_INVALID_VALUE, "bias must have shape [directions, 2 * gates * hidden_size]");
    if (h0 && !same_shape(h0, dirs, B, H))
        return fail(ctx, RTEN_ERR_INVALID_VALUE, "initial_hidden must have shape [directions, batch, hidden_size]");
    if (c0 && !gru && !same_shape(c0, dirs, B, H))
        return fail(ctx, RTEN_ERR_INVALID_VALUE, "initial_cell must have shape [directions, batch, hidden_size]");
    if (pw && (pw->kind != 0 || pw->dtype != RTEN_F32 || pw->K != I || pw->N != dirs * GH))
        return fail(ctx, RTEN_ERR_INVALID_VALUE, "packed weights do not match W [directions, gates * hidden_size, input]");
    if (T * B > INT_MAX || dirs * GH > INT_MAX || I > INT_MAX)
        return fail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "GRU / LSTM dimensions exceed the kernels' 32-bit indexing");

    OpScope sc(ctx);
    rten_tensor xv, wv, rv, bv, h0v, c0v, yv, yhv, ycv;
    RTB_TRY(sc.in(x, &xv));
    if (!pw) RTB_TRY(sc.in(w, &wv));
    RTB_TRY(sc.in(r, &rv));
    if (bias) RTB_TRY(sc.in(bias, &bv));
    if (h0) RTB_TRY(sc.in(h0, &h0v));
    if (c0 && !gru) RTB_TRY(sc.in(c0, &c0v));
    const int64_t yshape[4] = {T, dirs, B, H}, hshape[3] = {dirs, B, H};
    if (y) RTB_TRY(sc.out(y, RTEN_F32, 4, yshape, &yv, nullptr));
    if (yh) RTB_TRY(sc.out(yh, RTEN_F32, 3, hshape, &yhv, nullptr));
    if (yc && !gru) RTB_TRY(sc.out(yc, RTEN_F32, 3, hshape, &ycv, nullptr));

    RnnLaunch L;
    L.gru = gru;
    L.T = (int)T;
    L.B = (int)B;
    L.H = (int)H;
    L.dirs = dirs;
    L.reverse = p->direction == 1;
    L.r = (const float*)rv.data;
    L.r_d = rv.strides[0];
    L.r_row = rv.strides[1];
    L.r_k = rv.strides[2];
    if (bias) {
        L.bias = (const float*)bv.data;
        L.b_d = bv.strides[0];
        L.b_k = bv.strides[1];
    }
    if (h0) {
        L.h0 = (const float*)h0v.data;
        L.h0_d = h0v.strides[0];
        L.h0_b = h0v.strides[1];
        L.h0_k = h0v.strides[2];
    }
    if (c0 && !gru) {
        L.c0 = (const float*)c0v.data;
        L.c0_d = c0v.strides[0];
        L.c0_b = c0v.strides[1];
        L.c0_k = c0v.strides[2];
    }
    if (y) {
        L.y = (float*)yv.data;
        L.y_t = yv.strides[0];
        L.y_d = yv.strides[1];
        L.y_b = yv.strides[2];
        L.y_k = yv.strides[3];
    }
    if (yh) {
        L.yh = (float*)yhv.data;
        L.yh_d = yhv.strides[0];
        L.yh_b = yhv.strides[1];
        L.yh_k = yhv.strides[2];
    }
    if (yc && !gru) {
        L.yc = (float*)ycv.data;
        L.yc_d = ycv.strides[0];
        L.yc_b = ycv.strides[1];
        L.yc_k = ycv.strides[2];
    }
    if (B == 0 || H == 0) return sc.finish(RTEN_OK);
    if (T == 0) return sc.finish(launch_rnn_state_init(ctx, L, nullptr, nullptr, (int)H));

    // ---- input projection: xp [T * B, dirs * G * H] = x . W^T, one GEMM over every step and direction
    const int64_t N = dirs * GH;
    float* xp = nullptr;
    RTB_TRY(temp_alloc(ctx, (size_t)(T * B * N) * 4, (void**)&xp));
    if (I == 0) {
        RTB_CUDA(ctx, cudaMemsetAsync(xp, 0, (size_t)(T * B * N) * 4, ctx->stream));
    } else {
        rten_tensor xc;
        RTB_TRY(sc.contiguous(&xv, &xc));
        Mat ma{xc.data, T * B, I, I, 1};
        Mat mb;
        if (pw) {
            mb = Mat{pw->data, N, I, pw->ld, 1};
        } else {
            rten_tensor wc;
            RTB_TRY(sc.contiguous(&wv, &wc));
            mb = Mat{wc.data, N, I, I, 1};
        }
        GemmLaunch G;
        G.kind = 0;
        G.M = (int)(T * B);
        G.N = (int)N;
        G.K = (int)I;
        RTB_TRY(to_kmajor(ctx, 4, ma, &G.a));
        RTB_TRY(to_kmajor(ctx, 4, mb, &G.b));
        if (pw && G.b.base == pw->data) G.b_x3_slot = &const_cast<rten_packed*>(pw)->x3;
        G.epi.d = xp;
        G.epi.s_row = N;
        G.epi.s_col = 1;
        const rten_status st = launch_umma_gemm(ctx, G);
        if (st == RTEN_ERR_UNSUPPORTED_VALUE) return fail(ctx, st, "GEMM operands are not addressable by TMA after packing");
        RTB_TRY(st);
    }
    L.xp = xp;

    // ---- the recurrence: one cluster launch when R fits on chip
    if (!getenv("RTEN_B200_NO_RNN_CLUSTER")) {
        const rten_status st = launch_rnn_cluster(ctx, L);
        if (st != RTEN_ERR_UNSUPPORTED_VALUE) return sc.finish(st);
    }

    // ---- per-step path: rec = h . R^T (skinny kernel in exact f32, or the wgmma GEMM), then the gate kernel
    const int64_t ld = round_up(H, 4);  // 16-byte rows for the products; the padding stays 0
    float *hs = nullptr, *cs = nullptr, *rec = nullptr;
    RTB_TRY(temp_alloc(ctx, (size_t)(dirs * B * ld) * 4, (void**)&hs));
    RTB_CUDA(ctx, cudaMemsetAsync(hs, 0, (size_t)(dirs * B * ld) * 4, ctx->stream));
    // R with K-contiguous, 16-byte rows: as given when it has them, else one zero-padded copy [dirs, G * H, ld]
    const float* Rb = (const float*)rv.data;
    int64_t r_d = rv.strides[0], r_row = rv.strides[1];
    if (rv.strides[2] != 1 || ld != H || (r_row & 3) || (r_d & 3) || (reinterpret_cast<uintptr_t>(Rb) & 15)) {
        float* Rp = nullptr;
        RTB_TRY(temp_alloc(ctx, (size_t)(dirs * GH * ld) * 4, (void**)&Rp));
        RTB_CUDA(ctx, cudaMemsetAsync(Rp, 0, (size_t)(dirs * GH * ld) * 4, ctx->stream));
        long long shape[3] = {dirs, GH, H}, ss[3] = {rv.strides[0], rv.strides[1], rv.strides[2]}, ds[3] = {GH * ld, ld, 1};
        RTB_TRY(launch_nd_copy(ctx, 4, Rb, Rp, 3, shape, ss, ds));
        Rb = Rp;
        r_d = GH * ld;
        r_row = ld;
    }
    if (!gru) RTB_TRY(temp_alloc(ctx, (size_t)(dirs * B * ld) * 4, (void**)&cs));
    RTB_TRY(temp_alloc(ctx, (size_t)(dirs * B * GH) * 4, (void**)&rec));
    RTB_TRY(launch_rnn_state_init(ctx, L, hs, cs, (int)ld));
    SkinnyF32Launch S[2];
    GemmLaunch Gd[2];
    void* x3[2] = {nullptr, nullptr};
    bool skinny = true;
    for (int d = 0; d < dirs; d++) {
        S[d].a = hs + d * B * ld;
        S[d].as = ld;
        S[d].b = Rb + d * r_d;
        S[d].bs = r_row;
        S[d].M = (int)B;
        S[d].N = (int)GH;
        S[d].K = (int)ld;
        S[d].out = rec + d * B * GH;
        S[d].os = GH;
        skinny = skinny && skinny_f32_supported(S[d]);
    }
    if (!skinny) {
        for (int d = 0; d < dirs; d++) {
            GemmLaunch& Q = Gd[d];
            Q.kind = 0;
            Q.M = (int)B;
            Q.N = (int)GH;
            Q.K = (int)H;
            Q.a.base = hs + d * B * ld;
            Q.a.dims[0] = H;
            Q.a.dims[1] = B;
            Q.a.strides[1] = ld;
            RTB_TRY(to_kmajor(ctx, 4, Mat{S[d].b, GH, H, r_row, 1}, &Q.b));
            Q.epi.d = rec + d * B * GH;
            Q.epi.s_row = GH;
            Q.epi.s_col = 1;
            {
                // R is constant for the whole sequence: split it for 3xTF32 once, not once per step
                const long long d0p = round_up(H, 4);
                const long long dims[4] = {H, GH, 1, 1}, strides[4] = {1, Q.b.strides[1], 0, 0};
                RTB_TRY(temp_alloc(ctx, (size_t)(3 * d0p * GH) * 4, &x3[d]));
                RTB_TRY(launch_tf32x3_split(ctx, (const float*)Q.b.base, (float*)x3[d], dims, strides, d0p, 1));
                Q.b_x3_slot = &x3[d];
            }
        }
    }
    for (int s = 0; s < T; s++) {
        for (int d = 0; d < dirs; d++) {
            if (skinny) {
                RTB_TRY(launch_skinny_f32(ctx, S[d]));
            } else {
                // the recurrent product runs in 3xTF32 in both f32 modes: a single TF32 pass would round h and R
                // at every step, which the cluster path and the skinny kernel never do
                const int saved = ctx->f32_mode;
                ctx->f32_mode = RTEN_F32_TF32X3;
                const rten_status st = launch_umma_gemm(ctx, Gd[d]);
                ctx->f32_mode = saved;
                if (st == RTEN_ERR_UNSUPPORTED_VALUE) return fail(ctx, st, "GEMM operands are not addressable by TMA after packing");
                RTB_TRY(st);
            }
        }
        RTB_TRY(launch_rnn_step_gates(ctx, L, s, rec, hs, cs, (int)ld));
    }
    return sc.finish(RTEN_OK);
}

}  // namespace

extern "C" {

rten_status rten_b200_gru(rten_ctx* ctx, const rten_tensor* x, const rten_tensor* w, const rten_packed* packed_w,
                          const rten_tensor* r, const rten_tensor* bias, const rten_tensor* sequence_lens,
                          const rten_tensor* initial_h, const rten_rnn_params* params, rten_tensor* y, rten_tensor* y_h) {
    return rnn_run(ctx, true, x, w, packed_w, r, bias, sequence_lens, initial_h, nullptr, nullptr, params, y, y_h, nullptr);
}

rten_status rten_b200_lstm(rten_ctx* ctx, const rten_tensor* x, const rten_tensor* w, const rten_packed* packed_w,
                           const rten_tensor* r, const rten_tensor* bias, const rten_tensor* sequence_lens,
                           const rten_tensor* initial_h, const rten_tensor* initial_c, const rten_tensor* peephole,
                           const rten_rnn_params* params, rten_tensor* y, rten_tensor* y_h, rten_tensor* y_c) {
    return rnn_run(ctx, false, x, w, packed_w, r, bias, sequence_lens, initial_h, initial_c, peephole, params, y, y_h, y_c);
}

}  // extern "C"
