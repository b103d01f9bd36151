// Mask and layout kernels: Where (src/ops/binary_elementwise.rs where_op), Equal / Less / LessOrEqual / Greater /
// GreaterOrEqual (boolean_op), And / Or / Xor (logical_boolean_op), Not (src/ops/unary_elementwise.rs not), Trilu
// (src/ops/trilu.rs), Expand's cycle-and-repeat path (src/ops/layout.rs expand_to) and ConstantOfShape's fill
// (src/ops/generate.rs).  The layouts are described in masks.h.
#include <algorithm>
#include <cstdint>
#include <type_traits>
#include <vector>

#include "masks.h"

namespace rtb {

constexpr int MB = 128;         // threads of the rows / expand kernels
constexpr int CHUNK = 4 * MB;   // row elements one CTA covers per unit

// The rows layout: `nd` leading dims decomposed per unit, rows of `inner` elements.  Operands 0..2 are inputs, 3 the
// output.
struct MaskRows {
    int nd;
    int vec;            // every row start 16-byte aligned, each operand's row dense (ist 1) or one element (ist 0)
    long long inner;
    long long chunks;   // CHUNK-element pieces of a row
    long long units;    // rows * chunks
    long long shape[RTEN_MAX_DIMS];
    long long st[4][RTEN_MAX_DIMS];
    long long ist[4];
};

__device__ __forceinline__ void row_start(const MaskRows& p, long long row, long long off[4]) {
    off[0] = off[1] = off[2] = off[3] = 0;
#pragma unroll 1
    for (int k = p.nd - 1; k >= 0; k--) {
        const long long i = row % p.shape[k];
        row /= p.shape[k];
#pragma unroll
        for (int o = 0; o < 4; o++) off[o] += i * p.st[o][k];
    }
}

// f(off, j, row) on the element j of each row; f4(off, j, row) on elements j .. j + 3 when p.vec
template <typename F, typename F4>
__device__ __forceinline__ void rows_loop(const MaskRows& p, F f, F4 f4) {
    for (long long u = blockIdx.x; u < p.units; u += gridDim.x) {
        const long long row = u / p.chunks, j0 = (u - row * p.chunks) * CHUNK;
        long long off[4];
        row_start(p, row, off);
        if (p.vec) {
            const long long j = j0 + 4 * threadIdx.x;
            if (j < p.inner) f4(off, j, row);
        } else {
#pragma unroll
            for (int q = 0; q < 4; q++) {
                const long long j = j0 + q * MB + threadIdx.x;
                if (j < p.inner) f(off, j, row);
            }
        }
    }
}

__device__ __forceinline__ unsigned sel(int c, unsigned x, unsigned y) { return c != 0 ? x : y; }

// 16 bytes at p + j, or one element splatted when the operand's row is one element (stride 0)
template <typename V, typename T>
__device__ __forceinline__ V ld4(const T* p, long long j, long long s) {
    if (s == 0) {
        const T v = p[0];
        return V{v, v, v, v};
    }
    return *reinterpret_cast<const V*>(p + j);
}

// ---- Where ------------------------------------------------------------------------------------------------------
// one: bit 0 / 1 / 2 when c / x / y is one element
__global__ void where_flat_kernel(const int* __restrict__ c, const unsigned* __restrict__ x,
                                  const unsigned* __restrict__ y, unsigned* __restrict__ d, long long n,
                                  int one, int vec) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    const int c0 = (one & 1) ? c[0] : 0;
    const unsigned x0 = (one & 2) ? x[0] : 0u, y0 = (one & 4) ? y[0] : 0u;
    const long long n4 = vec ? (n >> 2) : 0;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
        int4 cv = make_int4(c0, c0, c0, c0);
        uint4 xv = make_uint4(x0, x0, x0, x0), yv = make_uint4(y0, y0, y0, y0);
        if (!(one & 1)) cv = reinterpret_cast<const int4*>(c)[i];
        if (!(one & 2)) xv = reinterpret_cast<const uint4*>(x)[i];
        if (!(one & 4)) yv = reinterpret_cast<const uint4*>(y)[i];
        reinterpret_cast<uint4*>(d)[i] = uint4{sel(cv.x, xv.x, yv.x), sel(cv.y, xv.y, yv.y), sel(cv.z, xv.z, yv.z), sel(cv.w, xv.w, yv.w)};
    }
    for (long long j = (n4 << 2) + (long long)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += stride) {
        const int cj = (one & 1) ? c0 : c[j];
        d[j] = cj != 0 ? ((one & 2) ? x0 : x[j]) : ((one & 4) ? y0 : y[j]);  // (only the chosen operand is read)
    }
}

__global__ void __launch_bounds__(MB) where_rows_kernel(const int* __restrict__ c, const unsigned* __restrict__ x,
                                                        const unsigned* __restrict__ y, unsigned* __restrict__ d, const MaskRows p) {
    rows_loop(
        p,
        [&](const long long* o, long long j, long long) {
            d[o[3] + j * p.ist[3]] = sel(c[o[0] + j * p.ist[0]], x[o[1] + j * p.ist[1]], y[o[2] + j * p.ist[2]]);
        },
        [&](const long long* o, long long j, long long) {
            const int4 cv = ld4<int4>(c + o[0], j, p.ist[0]);
            const uint4 xv = ld4<uint4>(x + o[1], j, p.ist[1]), yv = ld4<uint4>(y + o[2], j, p.ist[2]);
            *reinterpret_cast<uint4*>(d + o[3] + j) =
                uint4{sel(cv.x, xv.x, yv.x), sel(cv.y, xv.y, yv.y), sel(cv.z, xv.z, yv.z), sel(cv.w, xv.w, yv.w)};
        });
}

// ---- comparisons and logical operators ----------------------------------------------------------------------------
// IEEE comparisons (no flush to zero: the library is built without --use_fast_math), so NaN compares false and -0 == +0.
// The logical operators take nonzero as true (rten-base AsBool for i32).
template <typename T>
__device__ __forceinline__ int compare(int op, T a, T b) {
    switch (op) {
        case CMP_EQ: return a == b;
        case CMP_LT: return a < b;
        case CMP_LE: return a <= b;
        case CMP_GT: return a > b;
        case CMP_GE: return a >= b;
        default: break;
    }
    if constexpr (std::is_same<T, int>::value) {
        switch (op) {
            case LOG_AND: return a != 0 && b != 0;
            case LOG_OR: return a != 0 || b != 0;
            case LOG_XOR: return (a != 0) != (b != 0);
            default: return a == 0;  // LOG_NOT
        }
    }
    return 0;
}

template <typename T>
using Vec4T = typename std::conditional<std::is_same<T, float>::value, float4, int4>::type;

template <typename T>
__device__ __forceinline__ int4 compare4(int op, Vec4T<T> a, Vec4T<T> b) {
    return int4{compare(op, a.x, b.x), compare(op, a.y, b.y), compare(op, a.z, b.z), compare(op, a.w, b.w)};
}

// one: bit 0 / 1 when a / b is one element
template <typename T>
__global__ void __launch_bounds__(256) compare_flat_kernel(const T* __restrict__ a, const T* __restrict__ b, int* __restrict__ d,
                                                           long long n, int one, int vec, int op) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    const T a0 = (one & 1) ? a[0] : T(0), b0 = (one & 2) ? b[0] : T(0);
    const long long n4 = vec ? (n >> 2) : 0;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
        Vec4T<T> av{a0, a0, a0, a0}, bv{b0, b0, b0, b0};
        if (!(one & 1)) av = reinterpret_cast<const Vec4T<T>*>(a)[i];
        if (!(one & 2)) bv = reinterpret_cast<const Vec4T<T>*>(b)[i];
        reinterpret_cast<int4*>(d)[i] = compare4<T>(op, av, bv);
    }
    for (long long j = (n4 << 2) + (long long)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += stride)
        d[j] = compare(op, (one & 1) ? a0 : a[j], (one & 2) ? b0 : b[j]);
}

template <typename T>
__global__ void __launch_bounds__(MB) compare_rows_kernel(const T* __restrict__ a, const T* __restrict__ b, int* __restrict__ d,
                                                          const MaskRows p, int op) {
    rows_loop(
        p, [&](const long long* o, long long j, long long) { d[o[3] + j * p.ist[3]] = compare(op, a[o[0] + j * p.ist[0]], b[o[1] + j * p.ist[1]]); },
        [&](const long long* o, long long j, long long) {
            *reinterpret_cast<int4*>(d + o[3] + j) = compare4<T>(op, ld4<Vec4T<T>>(a + o[0], j, p.ist[0]), ld4<Vec4T<T>>(b + o[1], j, p.ist[1]));
        });
}

// ---- Trilu ------------------------------------------------------------------------------------------------------
// rows of the matrices over the last two dims (`rows` per matrix, the last leading dim); (i, j) kept when
// i + k - j <= 0 (upper) or >= 0 (lower), as trilu_kernel computes it
__global__ void __launch_bounds__(MB) trilu_kernel(const unsigned* __restrict__ x, unsigned* __restrict__ d, const MaskRows p,
                                                   long long rows, long long k, int upper) {
    auto keep = [&](long long row, long long j) {
        const long long delta = row % rows + k - j;
        return upper ? delta <= 0 : delta >= 0;
    };
    rows_loop(
        p, [&](const long long* o, long long j, long long row) { d[o[3] + j * p.ist[3]] = keep(row, j) ? x[o[0] + j * p.ist[0]] : 0u; },
        [&](const long long* o, long long j, long long row) {
            const uint4 v = ld4<uint4>(x + o[0], j, p.ist[0]);
            *reinterpret_cast<uint4*>(d + o[3] + j) =
                uint4{keep(row, j) ? v.x : 0u, keep(row, j + 1) ? v.y : 0u, keep(row, j + 2) ? v.z : 0u, keep(row, j + 3) ? v.w : 0u};
        });
}

// ---- Expand, fill -----------------------------------------------------------------------------------------------
// d [outer, reps, inner] = s [outer, inner]: one unit is a CHUNK-element piece of one output row (vec: 16 bytes per
// thread, both bases 16-byte aligned and inner % 4 == 0)
__global__ void __launch_bounds__(MB) expand_repeat_kernel(const unsigned* __restrict__ s, unsigned* __restrict__ d, long long inner,
                                                           long long chunks, long long units, long long reps, int vec) {
    for (long long u = blockIdx.x; u < units; u += gridDim.x) {
        const long long row = u / chunks, j0 = (u - row * chunks) * CHUNK;
        const unsigned* src = s + (row / reps) * inner;
        unsigned* dst = d + row * inner;
        if (vec) {
            const long long j = j0 + 4 * threadIdx.x;
            if (j < inner) *reinterpret_cast<uint4*>(dst + j) = *reinterpret_cast<const uint4*>(src + j);
        } else {
#pragma unroll
            for (int q = 0; q < 4; q++) {
                const long long j = j0 + q * MB + threadIdx.x;
                if (j < inner) dst[j] = src[j];
            }
        }
    }
}

__global__ void __launch_bounds__(256) fill_kernel(unsigned* __restrict__ d, unsigned bits, long long n, int vec) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    const long long n4 = vec ? (n >> 2) : 0;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride)
        reinterpret_cast<uint4*>(d)[i] = uint4{bits, bits, bits, bits};
    for (long long j = (n4 << 2) + (long long)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += stride) d[j] = bits;
}

// ---- host side --------------------------------------------------------------------------------------------------
namespace {

int grid_of(rten_ctx* ctx, long long blocks) {
    return (int)std::max(1LL, std::min(blocks, (long long)ctx->num_sms * 16));
}

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// Operands over the output's dims, size-1 dims dropped and adjacent dims merged where every operand allows it
struct Layout {
    int nd = 0;
    long long shape[RTEN_MAX_DIMS];
    long long st[4][RTEN_MAX_DIMS];
    long long n = 1;

    Layout(int nd0, const long long* shape0, const long long* const st0[4], int nops) {
        for (int i = 0; i < nd0; i++) {
            n *= shape0[i];
            if (shape0[i] == 1) continue;
            if (nd > 0) {
                bool merge = true;
                for (int o = 0; o < 4; o++)
                    if ((o < nops || o == 3) && st[o][nd - 1] != st0[o][i] * shape0[i]) merge = false;
                if (merge) {
                    shape[nd - 1] *= shape0[i];
                    for (int o = 0; o < 4; o++) st[o][nd - 1] = (o < nops || o == 3) ? st0[o][i] : 0;
                    continue;
                }
            }
            shape[nd] = shape0[i];
            for (int o = 0; o < 4; o++) st[o][nd] = (o < nops || o == 3) ? st0[o][i] : 0;
            nd++;
        }
        if (nd == 0) {  // one element
            shape[0] = 1;
            for (int o = 0; o < 4; o++) st[o][0] = 1;
            nd = 1;
        }
    }
    // flat: one dim, the output dense, each input dense (stride 1) or one element (stride 0); `one` gets the latter
    bool flat(int nops, int* one) const {
        if (nd != 1 || st[3][0] != 1) return false;
        *one = 0;
        for (int o = 0; o < nops; o++) {
            if (st[o][0] == 0 || shape[0] == 1) *one |= 1 << o;
            else if (st[o][0] != 1) return false;
        }
        return true;
    }
    MaskRows rows(const void* const ptr[4], int nops) const {
        MaskRows p{};
        p.nd = nd - 1;
        p.inner = shape[nd - 1];
        p.chunks = (p.inner + CHUNK - 1) / CHUNK;
        p.units = p.chunks * (n / std::max(1LL, p.inner));
        for (int i = 0; i < nd - 1; i++) p.shape[i] = shape[i];
        bool vec = p.inner % 4 == 0;
        for (int o = 0; o < 4; o++) {
            if (o >= nops && o != 3) continue;
            p.ist[o] = st[o][nd - 1];
            for (int i = 0; i < nd - 1; i++) {
                p.st[o][i] = st[o][i];
                if (p.ist[o] == 1 && st[o][i] % 4) vec = false;
            }
            if (p.ist[o] > 1 || (o == 3 && p.ist[o] != 1) || (p.ist[o] == 1 && !aligned16(ptr[o]))) vec = false;
        }
        p.vec = vec;
        return p;
    }
};

bool flat_vec(const void* const ptr[4], int nops, int one) {
    bool v = aligned16(ptr[3]);
    for (int o = 0; o < nops; o++)
        if (!(one >> o & 1)) v = v && aligned16(ptr[o]);
    return v;
}

}  // namespace

rten_status launch_where(rten_ctx* ctx, const int* c, const void* x, const void* y, void* d, int nd, const long long* shape,
                         const long long* const st[4]) {
    const Layout l(nd, shape, st, 3);
    if (l.n == 0) return RTEN_OK;
    const void* const ptr[4] = {c, x, y, d};
    int one = 0;
    if (l.flat(3, &one)) {
        const bool vec = flat_vec(ptr, 3, one);
        return launch(ctx, "where launch", where_flat_kernel, {dim3(grid_of(ctx, ((vec ? l.n / 4 : l.n) + 255) / 256)), dim3(256)}, c,
                      (const unsigned*)x, (const unsigned*)y, (unsigned*)d, l.n, one, vec ? 1 : 0);
    }
    const MaskRows p = l.rows(ptr, 3);
    return launch(ctx, "where launch", where_rows_kernel, {dim3(grid_of(ctx, p.units)), dim3(MB)}, c, (const unsigned*)x,
                  (const unsigned*)y, (unsigned*)d, p);
}

template <typename T>
static rten_status compare_typed(rten_ctx* ctx, int op, const T* a, const T* b, int* d, const Layout& l) {
    const void* const ptr[4] = {a, b, nullptr, d};
    int one = 0;
    if (l.flat(2, &one)) {
        const bool vec = flat_vec(ptr, 2, one);
        return launch(ctx, "compare launch", compare_flat_kernel<T>, {dim3(grid_of(ctx, ((vec ? l.n / 4 : l.n) + 255) / 256)), dim3(256)},
                      a, b, d, l.n, one, vec ? 1 : 0, op);
    }
    const MaskRows p = l.rows(ptr, 2);
    return launch(ctx, "compare launch", compare_rows_kernel<T>, {dim3(grid_of(ctx, p.units)), dim3(MB)}, a, b, d, p, op);
}

rten_status launch_compare(rten_ctx* ctx, int dtype, int op, const void* a, const void* b, int* d, int nd, const long long* shape,
                           const long long* const st[4]) {
    if (op < CMP_EQ || op > LOG_NOT || (op >= LOG_AND && dtype != RTEN_I32)) return fail(ctx, RTEN_ERR_INVALID_VALUE, "unknown comparison");
    const Layout l(nd, shape, st, 2);
    if (l.n == 0) return RTEN_OK;
    if (dtype == RTEN_F32) return compare_typed(ctx, op, (const float*)a, (const float*)b, d, l);
    return compare_typed(ctx, op, (const int*)a, (const int*)b, d, l);
}

rten_status launch_trilu(rten_ctx* ctx, const void* x, void* d, int nd, const long long* shape, const long long* sx,
                         const long long* sd, long long k, bool upper) {
    long long n = 1;
    for (int i = 0; i < nd; i++) n *= shape[i];
    if (n == 0) return RTEN_OK;
    // no merging: the last two dims are the matrix, the leading ones decomposed per unit
    MaskRows p{};
    p.nd = nd - 1;
    p.inner = shape[nd - 1];
    p.chunks = (p.inner + CHUNK - 1) / CHUNK;
    p.units = p.chunks * (n / p.inner);
    p.ist[0] = sx[nd - 1];
    p.ist[3] = sd[nd - 1];
    bool vec = p.inner % 4 == 0 && p.ist[0] == 1 && p.ist[3] == 1 && aligned16(x) && aligned16(d);
    for (int i = 0; i < nd - 1; i++) {
        p.shape[i] = shape[i];
        p.st[0][i] = sx[i];
        p.st[3][i] = sd[i];
        if (sx[i] % 4 || sd[i] % 4) vec = false;
    }
    p.vec = vec;
    return launch(ctx, "trilu launch", trilu_kernel, {dim3(grid_of(ctx, p.units)), dim3(MB)}, (const unsigned*)x, (unsigned*)d, p,
                  (long long)shape[nd - 2], k, upper ? 1 : 0);
}

rten_status launch_expand_repeat(rten_ctx* ctx, const void* s, void* d, long long outer, long long reps, long long inner) {
    const long long chunks = (inner + CHUNK - 1) / CHUNK, units = outer * reps * chunks;
    if (units == 0) return RTEN_OK;
    const int vec = inner % 4 == 0 && aligned16(s) && aligned16(d);
    return launch(ctx, "expand launch", expand_repeat_kernel, {dim3(grid_of(ctx, units)), dim3(MB)}, (const unsigned*)s, (unsigned*)d,
                  inner, chunks, units, reps, vec);
}

rten_status launch_fill(rten_ctx* ctx, void* d, uint32_t bits, long long n) {
    if (n == 0) return RTEN_OK;
    const int vec = aligned16(d) ? 1 : 0;
    return launch(ctx, "fill launch", fill_kernel, {dim3(grid_of(ctx, ((vec ? n / 4 : n) + 255) / 256)), dim3(256)}, (unsigned*)d, bits, n,
                  vec);
}

// ---- Slice, Split geometry --------------------------------------------------------------------------------------
rten_status slice_ranges(rten_ctx* ctx, int ndim, const int64_t* shape, const int32_t* starts, int n_starts, const int32_t* ends,
                         int n_ends, const int32_t* axes, int n_axes, const int32_t* steps, int n_steps, int64_t* start,
                         int64_t* len, int64_t* step) {
    if (axes && n_axes > ndim) return fail(ctx, RTEN_ERR_INVALID_VALUE, "`axes` length must be <= input rank");
    const int n = axes ? n_axes : ndim;
    if (n_starts != n) return fail(ctx, RTEN_ERR_INVALID_VALUE, "`starts` length must match axis count");
    if (n_ends != n) return fail(ctx, RTEN_ERR_INVALID_VALUE, "`ends` length must match axis count");
    if (steps) {
        if (n_steps != n) return fail(ctx, RTEN_ERR_INVALID_VALUE, "`steps` length must match axis count");
        for (int i = 0; i < n; i++)
            if (steps[i] == 0) return fail(ctx, RTEN_ERR_INVALID_VALUE, "steps must be non-zero");
        for (int i = 0; i < n; i++)
            if (steps[i] < 0) return fail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "Slice with a negative step is not supported");
    }
    for (int i = 0; i < ndim; i++) {
        start[i] = 0;
        len[i] = shape[i];
        step[i] = 1;
    }
    for (int i = 0; i < n; i++) {
        int64_t axis = i;
        if (axes) {
            axis = axes[i] < 0 ? axes[i] + ndim : axes[i];
            if (axis < 0 || axis >= ndim) return fail(ctx, RTEN_ERR_INVALID_VALUE, "Axis is invalid");
        }
        const int64_t d = shape[axis], s = steps ? steps[i] : 1;
        // SliceRange::clamp for a positive step, then resolve: [-d, d], negative from the end, empty when end <= start
        int64_t b = std::min(d, std::max(-d, (int64_t)starts[i])), e = std::min(d, std::max(-d, (int64_t)ends[i]));
        if (b < 0) b += d;
        if (e < 0) e += d;
        start[axis] = b;
        len[axis] = e > b ? (e - b + s - 1) / s : 0;
        step[axis] = s;
    }
    return RTEN_OK;
}

rten_status split_pieces(rten_ctx* ctx, int64_t dim, const int32_t* sizes, int n_sizes, int64_t num_outputs,
                         std::vector<int64_t>* pieces) {
    pieces->clear();
    if (sizes) {
        int64_t sum = 0;
        for (int i = 0; i < n_sizes; i++) {
            if (sizes[i] < 0) return fail(ctx, RTEN_ERR_INVALID_VALUE, "Split sizes must be >= 0");
            sum += sizes[i];
        }
        if (sum != dim) return fail(ctx, RTEN_ERR_INVALID_VALUE, "Split sizes do not sum to dimension size");
        int64_t at = 0;
        for (int i = 0; i < n_sizes; i++) {
            pieces->push_back(at);
            pieces->push_back(sizes[i]);
            at += sizes[i];
        }
        return RTEN_OK;
    }
    if (num_outputs <= 0) return fail(ctx, RTEN_ERR_INVALID_VALUE, "num_outputs must be > 0");
    if (num_outputs > dim) return fail(ctx, RTEN_ERR_INVALID_VALUE, "num_outputs exceeds dim size");
    const int64_t chunk = (dim + num_outputs - 1) / num_outputs;
    for (int64_t at = 0; at < dim; at += chunk) {
        pieces->push_back(at);
        pieces->push_back(std::min(chunk, dim - at));
    }
    return RTEN_OK;
}

}  // namespace rtb
