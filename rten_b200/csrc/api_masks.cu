// C-ABI entry points of the mask and layout operators (masks.cu): Where, the comparisons, the logical operators, Trilu,
// Expand, Slice and Split.
#include <algorithm>
#include <vector>

#include "api_util.h"
#include "masks.h"

using namespace rtb;

namespace {

// numpy broadcasting of `n` operands: the output dims and each operand's strides over them (0 on broadcast dims)
rten_status broadcast(rten_ctx* ctx, const rten_tensor* const* v, int n, int* nd, int64_t* shape, long long st[][RTEN_MAX_DIMS],
                      const char* msg = "Cannot broadcast inputs") {
    *nd = 0;
    for (int o = 0; o < n; o++) *nd = std::max(*nd, v[o]->ndim);
    for (int i = 0; i < *nd; i++) {
        int64_t d = 1;
        for (int o = 0; o < n; o++) {
            const int k = i - (*nd - v[o]->ndim);
            const int64_t s = k >= 0 ? v[o]->shape[k] : 1;
            if (s != 1) {
                if (d != 1 && d != s) return fail(ctx, RTEN_ERR_INCOMPATIBLE_SHAPES, msg);
                d = s;
            }
        }
        shape[i] = d;
        for (int o = 0; o < n; o++) {
            const int k = i - (*nd - v[o]->ndim);
            st[o][i] = (k >= 0 && v[o]->shape[k] != 1) ? v[o]->strides[k] : 0;
        }
    }
    return RTEN_OK;
}

// a, b -> i32 0 / 1 with broadcasting (b null: Not)
rten_status compare_op(rten_ctx* ctx, const rten_tensor* a, const rten_tensor* b, rten_tensor* out, int op) {
    RTB_TRY(check_ctx(ctx));
    const bool unary = op == LOG_NOT;
    if (!a || (!b && !unary) || !out) return fail(ctx, RTEN_ERR_MISSING_INPUTS, "missing inputs");
    const bool logical = op >= LOG_AND;
    if (logical ? a->dtype != RTEN_I32 : (a->dtype != RTEN_F32 && a->dtype != RTEN_I32)) return fail(ctx, RTEN_ERR_UNSUPPORTED_TYPE, "unsupported type");
    if (!unary && b->dtype != a->dtype) return fail(ctx, RTEN_ERR_UNSUPPORTED_TYPE, "unsupported type");
    OpScope sc(ctx);
    rten_tensor av, bv, ov;
    RTB_TRY(sc.in(a, &av));
    if (unary) bv = av;
    else RTB_TRY(sc.in(b, &bv));
    const rten_tensor* v[2] = {&av, &bv};
    int nd;
    int64_t shape[RTEN_MAX_DIMS];
    long long st[4][RTEN_MAX_DIMS];
    RTB_TRY(broadcast(ctx, v, 2, &nd, shape, st));
    RTB_TRY(sc.out(out, RTEN_I32, nd, shape, &ov, nullptr));
    long long shp[RTEN_MAX_DIMS];
    for (int i = 0; i < nd; i++) {
        shp[i] = shape[i];
        st[3][i] = ov.strides[i];
    }
    const long long* const s[4] = {st[0], st[1], st[2], st[3]};
    return sc.finish(launch_compare(ctx, av.dtype, op, av.data, bv.data, (int*)ov.data, nd, shp, s));
}

}  // namespace

extern "C" {

rten_status rten_b200_where(rten_ctx* ctx, const rten_tensor* cond, const rten_tensor* x, const rten_tensor* y, rten_tensor* out) {
    RTB_TRY(check_ctx(ctx));
    if (!cond || !x || !y || !out) return fail(ctx, RTEN_ERR_MISSING_INPUTS, "missing inputs");
    if (cond->dtype != RTEN_I32 || (x->dtype != RTEN_F32 && x->dtype != RTEN_I32) || y->dtype != x->dtype)
        return fail(ctx, RTEN_ERR_UNSUPPORTED_TYPE, "unsupported type");
    OpScope sc(ctx);
    rten_tensor cv, xv, yv, ov;
    RTB_TRY(sc.in(cond, &cv));
    RTB_TRY(sc.in(x, &xv));
    RTB_TRY(sc.in(y, &yv));
    const rten_tensor* v[3] = {&cv, &xv, &yv};
    int nd;
    int64_t shape[RTEN_MAX_DIMS];
    long long st[4][RTEN_MAX_DIMS];
    RTB_TRY(broadcast(ctx, v, 3, &nd, shape, st));
    RTB_TRY(sc.out(out, x->dtype, nd, shape, &ov, nullptr));
    long long shp[RTEN_MAX_DIMS];
    for (int i = 0; i < nd; i++) {
        shp[i] = shape[i];
        st[3][i] = ov.strides[i];
    }
    const long long* const s[4] = {st[0], st[1], st[2], st[3]};
    return sc.finish(launch_where(ctx, (const int*)cv.data, xv.data, yv.data, ov.data, nd, shp, s));
}

rten_status rten_b200_equal(rten_ctx* ctx, const rten_tensor* a, const rten_tensor* b, rten_tensor* out) {
    return compare_op(ctx, a, b, out, CMP_EQ);
}
rten_status rten_b200_less(rten_ctx* ctx, const rten_tensor* a, const rten_tensor* b, rten_tensor* out) {
    return compare_op(ctx, a, b, out, CMP_LT);
}
rten_status rten_b200_less_or_equal(rten_ctx* ctx, const rten_tensor* a, const rten_tensor* b, rten_tensor* out) {
    return compare_op(ctx, a, b, out, CMP_LE);
}
rten_status rten_b200_greater(rten_ctx* ctx, const rten_tensor* a, const rten_tensor* b, rten_tensor* out) {
    return compare_op(ctx, a, b, out, CMP_GT);
}
rten_status rten_b200_greater_or_equal(rten_ctx* ctx, const rten_tensor* a, const rten_tensor* b, rten_tensor* out) {
    return compare_op(ctx, a, b, out, CMP_GE);
}
rten_status rten_b200_and(rten_ctx* ctx, const rten_tensor* a, const rten_tensor* b, rten_tensor* out) {
    return compare_op(ctx, a, b, out, LOG_AND);
}
rten_status rten_b200_or(rten_ctx* ctx, const rten_tensor* a, const rten_tensor* b, rten_tensor* out) {
    return compare_op(ctx, a, b, out, LOG_OR);
}
rten_status rten_b200_xor(rten_ctx* ctx, const rten_tensor* a, const rten_tensor* b, rten_tensor* out) {
    return compare_op(ctx, a, b, out, LOG_XOR);
}
rten_status rten_b200_not(rten_ctx* ctx, const rten_tensor* x, rten_tensor* out) { return compare_op(ctx, x, nullptr, out, LOG_NOT); }

rten_status rten_b200_trilu(rten_ctx* ctx, const rten_tensor* x, int64_t k, int upper, rten_tensor* out) {
    RTB_TRY(check_ctx(ctx));
    if (!x || !out) return fail(ctx, RTEN_ERR_MISSING_INPUTS, "missing inputs");
    if (x->dtype != RTEN_F32 && x->dtype != RTEN_I32) return fail(ctx, RTEN_ERR_UNSUPPORTED_TYPE, "unsupported type");
    if (x->ndim < 2) return fail(ctx, RTEN_ERR_INVALID_VALUE, "Input must have >= 2 dims");
    OpScope sc(ctx);
    rten_tensor xv, ov;
    RTB_TRY(sc.in(x, &xv));
    RTB_TRY(sc.out(out, x->dtype, xv.ndim, xv.shape, &ov, nullptr));
    long long shp[RTEN_MAX_DIMS], sx[RTEN_MAX_DIMS], sd[RTEN_MAX_DIMS];
    for (int i = 0; i < xv.ndim; i++) {
        shp[i] = xv.shape[i];
        sx[i] = xv.strides[i];
        sd[i] = ov.strides[i];
    }
    return sc.finish(launch_trilu(ctx, xv.data, ov.data, xv.ndim, shp, sx, sd, k, upper != 0));
}

rten_status rten_b200_expand(rten_ctx* ctx, const rten_tensor* x, const int64_t* shape, int n, rten_tensor* out) {
    RTB_TRY(check_ctx(ctx));
    if (!x || !out || (n > 0 && !shape)) return fail(ctx, RTEN_ERR_MISSING_INPUTS, "missing inputs");
    if (x->dtype != RTEN_F32 && x->dtype != RTEN_I32) return fail(ctx, RTEN_ERR_UNSUPPORTED_TYPE, "unsupported type");
    if (n < 0 || n > RTEN_MAX_DIMS) return fail(ctx, RTEN_ERR_INVALID_VALUE, "tensor rank out of range");
    for (int i = 0; i < n; i++)
        if (shape[i] < 0) return fail(ctx, RTEN_ERR_INVALID_VALUE, "Target shape contains negative values");
    rten_tensor target{};
    target.ndim = n;
    for (int i = 0; i < n; i++) target.shape[i] = shape[i];
    const rten_tensor* v[2] = {x, &target};
    int nd;
    int64_t oshape[RTEN_MAX_DIMS];
    long long st[4][RTEN_MAX_DIMS];
    RTB_TRY(broadcast(ctx, v, 2, &nd, oshape, st, "Cannot broadcast input with target shape"));
    OpScope sc(ctx);
    rten_tensor xv, ov;
    RTB_TRY(sc.in(x, &xv));
    RTB_TRY(sc.out(out, x->dtype, nd, oshape, &ov, nullptr));
    if (numel(&ov) == 0) return sc.finish(RTEN_OK);
    // the dims x is broadcast over (size 1 or absent in x, larger in the output)
    int first = -1, last = -1;
    for (int i = 0; i < nd; i++) {
        const int k = i - (nd - xv.ndim);
        if ((k < 0 || xv.shape[k] == 1) && oshape[i] != 1) {
            if (first < 0) first = i;
            last = i;
        }
    }
    bool block = first >= 0;  // one run of broadcast dims, x dense
    for (int i = first; block && i <= last; i++) {
        const int k = i - (nd - xv.ndim);
        if (k >= 0 && xv.shape[k] != 1) block = false;
    }
    long long outer = 1, reps = 1, inner = 1;
    for (int i = 0; i < nd; i++) (i < first ? outer : i <= last ? reps : inner) *= oshape[i];
    // rows of fewer than 128 elements would leave most of a repeat unit's threads idle: those take the strided copy
    if (block && inner >= 128 && is_contiguous(&xv) && is_contiguous(&ov))
        return sc.finish(launch_expand_repeat(ctx, xv.data, ov.data, outer, reps, inner));
    rten_tensor src = ov;  // x as a zero-stride view of the output's shape
    src.data = xv.data;
    for (int i = 0; i < nd; i++) src.strides[i] = st[0][i];
    return sc.finish(copy_view(ctx, src, ov));
}

rten_status rten_b200_slice(rten_ctx* ctx, const rten_tensor* x, const int32_t* starts, const int32_t* ends, const int32_t* axes,
                            const int32_t* steps, int n, rten_tensor* out) {
    RTB_TRY(check_ctx(ctx));
    if (!x || !out || (n > 0 && (!starts || !ends))) return fail(ctx, RTEN_ERR_MISSING_INPUTS, "missing inputs");
    if (dtype_size(x->dtype) != 4) return fail(ctx, RTEN_ERR_UNSUPPORTED_TYPE, "unsupported type");
    int64_t b[RTEN_MAX_DIMS], len[RTEN_MAX_DIMS], step[RTEN_MAX_DIMS];
    RTB_TRY(slice_ranges(ctx, x->ndim, x->shape, starts, n, ends, n, axes, n, steps, n, b, len, step));
    OpScope sc(ctx);
    rten_tensor xv, ov;
    RTB_TRY(sc.in(x, &xv));
    rten_tensor view = xv;
    for (int i = 0; i < xv.ndim; i++) {
        if (len[i] > 0) view.data = (char*)view.data + b[i] * xv.strides[i] * 4;
        view.shape[i] = len[i];
        view.strides[i] = xv.strides[i] * step[i];
    }
    RTB_TRY(sc.out(out, x->dtype, view.ndim, view.shape, &ov, nullptr));
    if (numel(&ov) == 0) return sc.finish(RTEN_OK);
    return sc.finish(copy_view(ctx, view, ov));
}

rten_status rten_b200_split(rten_ctx* ctx, const rten_tensor* x, int axis, const int32_t* split, int n_split, int num_outputs,
                            rten_tensor* outs, int n_outs, int32_t* n_pieces) {
    RTB_TRY(check_ctx(ctx));
    if (!x || !outs || !n_pieces) return fail(ctx, RTEN_ERR_MISSING_INPUTS, "missing inputs");
    if (dtype_size(x->dtype) != 4) return fail(ctx, RTEN_ERR_UNSUPPORTED_TYPE, "unsupported type");
    const int a = axis < 0 ? axis + x->ndim : axis;
    if (a < 0 || a >= x->ndim) return fail(ctx, RTEN_ERR_INVALID_VALUE, "Axis is invalid");
    std::vector<int64_t> pieces;
    RTB_TRY(split_pieces(ctx, x->shape[a], split, n_split, num_outputs, &pieces));
    const int np = (int)pieces.size() / 2;
    if (np > n_outs) return fail(ctx, RTEN_ERR_INVALID_VALUE, "Split gives more pieces than there are outputs");
    OpScope sc(ctx);
    rten_tensor xv;
    RTB_TRY(sc.in(x, &xv));
    for (int i = 0; i < np; i++) {
        rten_tensor view = xv, ov;
        view.shape[a] = pieces[(size_t)(2 * i + 1)];
        if (view.shape[a] > 0) view.data = (char*)view.data + pieces[(size_t)(2 * i)] * xv.strides[a] * 4;
        RTB_TRY(sc.out(&outs[i], x->dtype, view.ndim, view.shape, &ov, nullptr));
        if (numel(&ov) > 0) RTB_TRY(copy_view(ctx, view, ov));
    }
    *n_pieces = np;
    return sc.finish(RTEN_OK);
}

}  // extern "C"
