// Mask and layout kernels (masks.cu): Where, the comparisons and logical operators, Trilu, Expand's repeat path and the
// fill of ConstantOfShape.  Where, Trilu, Expand and the fill move 32-bit words, so one instance serves f32 and i32.
//
// Broadcast operands are described over the output's dims: `shape` (nd dims) and, per operand, its element strides
// (0 on a broadcast dim).  The launchers collapse the dims first; what is left runs either
//   flat: every operand dense in one layout with the output, or one element (read once per thread), 16 bytes per
//         thread when the dense bases are 16-byte aligned, else one element per thread;
//   rows: the last dim is a row, the ones before it are decomposed once per 512-element piece of a row (one CTA's
//         unit), so the per-element index arithmetic is one multiply-add per operand; 16 bytes per thread when every
//         row start is 16-byte aligned and each operand's row is dense or one element.
#pragma once
#include "common.h"

namespace rtb {

enum CompareOp { CMP_EQ = 0, CMP_LT = 1, CMP_LE = 2, CMP_GT = 3, CMP_GE = 4, LOG_AND = 5, LOG_OR = 6, LOG_XOR = 7, LOG_NOT = 8 };

// d = c != 0 ? x : y (i32 c; x, y, d 32-bit words).  st[0..2]: the strides of c, x, y; st[3]: d's.
rten_status launch_where(rten_ctx* ctx, const int* c, const void* x, const void* y, void* d, int nd, const long long* shape,
                         const long long* const st[4]);
// d = a (op) b as i32 0 / 1 (f32 or i32 a and b; LOG_* only on i32; LOG_NOT reads a only).  st[0], st[1]: a, b; st[3]: d.
rten_status launch_compare(rten_ctx* ctx, int dtype, int op, const void* a, const void* b, int* d, int nd, const long long* shape,
                           const long long* const st[4]);
// d = x where the element (i, j) of each matrix over the last two dims is kept (upper: j - i >= k; else j - i <= k), else 0
rten_status launch_trilu(rten_ctx* ctx, const void* x, void* d, int nd, const long long* shape, const long long* sx,
                         const long long* sd, long long k, bool upper);
// dense d [outer, reps, inner] = dense s [outer, inner] repeated over the middle dim
rten_status launch_expand_repeat(rten_ctx* ctx, const void* s, void* d, long long outer, long long reps, long long inner);
// n words of d set to `bits`
rten_status launch_fill(rten_ctx* ctx, void* d, uint32_t bits, long long n);

// Slice's ranges (src/ops/slice.rs slice_ranges) over a tensor of `ndim` dims `shape`: `axes` / `steps` may be null
// (n_axes / n_steps ignored then).  Each range is clamped as SliceRange::clamp does and resolved to (start, len, step).
// A negative step is refused with RTEN_ERR_UNSUPPORTED_VALUE: a strided view cannot have negative strides.
rten_status slice_ranges(rten_ctx* ctx, int ndim, const int64_t* shape, const int32_t* starts, int n_starts, const int32_t* ends,
                         int n_ends, const int32_t* axes, int n_axes, const int32_t* steps, int n_steps, int64_t* start,
                         int64_t* len, int64_t* step);
// Split's pieces (src/ops/split.rs split) of a dim of `dim` elements: `sizes` (n_sizes of them) when not null, else
// num_outputs chunks of ceil(dim / num_outputs).  `pieces` gets (start, length) pairs.
rten_status split_pieces(rten_ctx* ctx, int64_t dim, const int32_t* sizes, int n_sizes, int64_t num_outputs,
                         std::vector<int64_t>* pieces);

}  // namespace rtb
