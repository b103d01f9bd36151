// wgmma GEMM / implicit-GEMM convolution for sm_90a.
//
// Replaces rten-gemm's packed BLIS-style GEMM (rten-gemm/src/lib.rs:794-1093, micro-kernels
// rten-gemm/src/kernels/simd_generic.rs:285,576) and the im2col packing
// (rten-gemm/src/im2col.rs:110-389) on the MatMul / MatMulInteger / Conv / ConvInteger path.
//
// Persistent, warp-specialised kernel, one CTA of 416 threads per SM:
//   warp 12  : TMA producer   -- cp.async.bulk.tensor tiles of A (128 rows x 128 B) and B (bn rows x 128 B) into a
//                                ring of 128B-swizzled shared-memory stages; starts before the rest of the CTA has
//                                finished its set-up
//   warps 0-3: MMA warpgroup  -- wgmma (tf32 -> f32 or 8-bit -> s32), 8 instructions per 128-byte K block (two 64-row
//                                halves), accumulating in registers; a finished tile goes to one of two accumulator
//                                stages of 64 columns in shared memory
//   warps 4-11: epilogue      -- two groups of 4 warps, each taking every other 32-column chunk of the tile:
//                                accumulator rows -> registers -> fused epilogue (alpha, residual /
//                                beta*C, bias, activation; or the integer zero-point correction, cast*scale, bias,
//                                residual, activation; optionally the output's min / max) -> 128B-swizzled smem
//                                staging -> cp.async.bulk.tensor store (full-line writes; TMA clips rows/columns
//                                outside the output).  Outputs whose rows are not contiguous fall back to direct
//                                register->global stores.  Runs concurrently with the next tile's main loop thanks
//                                to the second accumulator stage.
// Launches that take the plain f32 epilogue (alpha = 1, optional column bias, TMA-staged residual, none / Relu / Gelu)
// can also run on umma_wide_kernel (umma_kernel.cuh), which computes 128 x 128 or 128 x 256 tiles with 384 threads:
//   warpgroup 0    : the same TMA producer (one warp issues, registers released with setmaxnreg)
//   warpgroups 1, 2: 64 rows each, m64n128k8 / m64n256k8 wgmma into registers, then the epilogue from those registers
//                    through 128-row staging buffers and TMA stores; not overlapped with the next main loop.
// A wide tile reads each A tile from shared memory once for up to 256 columns and amortises the fixed cost of a
// pipeline stage over 2-4x the tensor work; the plans of both kernels compete in the cost model and the autotuner.
// Work decomposition (tile width, split-K, staging buffers) is a launch `Plan` (see "Launch plans" below), ranked by
// a cost model and, optionally, measured on the device per problem.
// For Conv the A tile is a TMA box over the NHWC activation tensor at (c0, ox0*sx - pad + kx*dx,
// oy0*sy - pad + ky*dy, b0): padding comes from TMA out-of-bounds zero fill, the stride from the
// tensor map's element strides; the im2col matrix is never materialised.
#include <cuda.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <array>
#include <cmath>
#include <vector>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>

#include "math.cuh"
#include "ptx.cuh"
#include "rowops.h"
#include "umma_gemm.h"
#include "umma_kernel.cuh"  // device side: KParams, the kernels

namespace rtb {

// ------------------------------------------------------------------------------------------
// Host side
// ------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode(rten_ctx* ctx) {
    if (!ctx->encode_tiled) {
        void* fn = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) != cudaSuccess ||
            qres != cudaDriverEntryPointSuccess)
            return nullptr;
        ctx->encode_tiled = fn;
    }
    return reinterpret_cast<EncodeTiledFn>(ctx->encode_tiled);
}

bool tma_compatible(const OperandDesc& od, int esize, int rank) {
    if (reinterpret_cast<uintptr_t>(od.base) & 15) return false;
    if (od.strides[0] != 1) return false;
    for (int i = 1; i < rank; i++) {
        if (od.dims[i] > 1) {
            if ((od.strides[i] * esize) % 16 != 0) return false;
            if (od.strides[i] * esize >= (1ll << 40)) return false;
        }
    }
    for (int i = 0; i < rank; i++)
        if (od.dims[i] < 1 || od.dims[i] > 0xFFFFFFFFll) return false;
    return true;
}

bool encode_map(rten_ctx* ctx, CUtensorMap* map, const OperandDesc& od, int esize, bool is_f32,
                const uint32_t box[4], const uint32_t estr[4]) {
    EncodeTiledFn enc = get_encode(ctx);
    if (!enc) return false;
    cuuint64_t dims[4];
    cuuint64_t strides[3];
    cuuint32_t b[4], es[4];
    for (int i = 0; i < 4; i++) {
        dims[i] = (cuuint64_t)od.dims[i];
        b[i] = box[i];
        es[i] = estr[i];
    }
    for (int i = 1; i < 4; i++) {
        long long s = od.strides[i] * esize;
        // size-1 / broadcast dims: any legal multiple of 16 works, the coordinate is always 0
        if (s == 0 || od.dims[i] == 1) s = 16;
        strides[i - 1] = (cuuint64_t)s;
    }
    CUresult r = enc(map, is_f32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_UINT8, 4,
                     const_cast<void*>(od.base), dims, strides, b, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS;
}

// Pick the output-pixel box (tw x th x tb <= 128 rows) that wastes the fewest MMA rows.
static void pick_conv_tile(const ConvGeom& g, int& tw, int& th, int& tb) {
    double best = -1.0;
    tw = th = tb = 1;
    for (int w = 1; w <= std::min(g.OW, 128); w++) {
        if (w * g.sx > 256) break;
        for (int h = 1; h <= std::min(g.OH, 128 / w); h++) {
            if (h * g.sy > 256) break;
            int b = std::min(g.B, 128 / (w * h));
            if (b < 1) continue;
            long long tiles = (long long)((g.OW + w - 1) / w) * ((g.OH + h - 1) / h) * ((g.B + b - 1) / b);
            double eff = (double)g.B * g.OH * g.OW / ((double)tiles * 128.0);
            // prefer wider boxes on ties (longer contiguous runs for TMA and the epilogue)
            if (eff > best + 1e-9 || (eff > best - 1e-9 && w > tw)) {
                best = eff;
                tw = w;
                th = h;
                tb = b;
            }
        }
    }
}

// ------------------------------------------------------------------------------------------
// Launch plans
// ------------------------------------------------------------------------------------------
// A plan fixes the kernel, tile shape and work decomposition of one launch: bn, splitk, nbuf on the implicit-GEMM
// kernels, or units of bn channels x T 128-slot tiles on the halo-reuse kernel (umma_halo.cu).  Plans come from (a) the
// cost models or (b) the per-context autotune cache: with rten_b200_set_autotune(ctx, 1) the first launch of every
// distinct problem times the best candidates on the device (CUDA events on the context stream) and remembers the winner.
struct Plan {
    int bn = 32, splitk = 1, nbuf = 1;
    bool halo = false;
    int T = 0;  // (halo)
};

static Plan halo_plan(int bn, int T) {
    Plan pl;
    pl.halo = true;
    pl.bn = bn;
    pl.T = T;
    return pl;
}

// Everything about a launch that does not depend on the plan.
struct Prepared {
    KParams p;  // geometry filled in; plan-dependent fields zero
    uint32_t abox[4], aes[4], bbox_k;
    uint32_t pbox[4], pes[4];  // A box / element strides of the projection source
    uint32_t a_rows;
    long long batch;
    OperandDesc od, ord;
    uint32_t dbox[4];
    int tma_store, res_tma;  // eligibility
    int wide;                // the wide-tile kernel may run this launch (plain f32 epilogue, see pick_epilogue)
    int chain_bytes;         // > 0: a chained launch (GemmLaunch::chain) and the bytes of its resident second weights
    int step;
    int esize, kelems;
};

constexpr int SK_CNT_INTS = 1 << 16;
// 227 KB of shared memory per block; SMEM_FIXED_BYTES: alignment slack, barriers, column vectors, accumulators
static int smem_budget_for(int n_stg) { return 227 * 1024 - SMEM_FIXED_BYTES - n_stg * STG_BYTES; }
// operand stages of the wide-tile kernel: 6 at bn = 128, 4 at bn = 256; chained at bn = 128, 4 with 64 KB of second
// weights (N2 = 64), 2 with 128 KB (N2 = 128)
static int wide_stages(int stage_bytes, int chain_bytes) {
    return std::min(MAX_STAGES, (227 * 1024 - WIDE_SMEM_FIXED_BYTES - chain_bytes) / stage_bytes);
}
static bool is_wide(int bn) { return bn > ACC_STRIDE; }

// The epilogue variant (umma_epilogue.cuh) of a launch with the given output path and split.  RTEN_B200_NO_FAST=1 sends every launch to Generic, RTEN_B200_NO_PLAIN=1 keeps launches off the plain variants
// (comparisons between variants).
static Epi pick_epilogue(const GemmLaunch& L, int tma_store, int res_tma, int splitk) {
    const EpilogueDesc& e = L.epi;
    auto aligned = [](const void* ptr) { return (reinterpret_cast<uintptr_t>(ptr) & 15) == 0; };
    // Fast: every chunk qualifies for the register path -- TMA store, whole 32-column chunks, column vectors 128-bit
    // loadable (integer: zero-point / scale vectors per column or scalar), residual TMA-staged
    bool fast = tma_store && (L.N % 32) == 0 && !getenv("RTEN_B200_NO_FAST") && e.bias_kind != 2 &&
                (e.r == nullptr || res_tma) && (e.bias_kind != 1 || aligned(e.bias));
    if (L.kind == 1)
        fast = fast && (!(e.za || e.za8) || aligned(e.colsum)) && (!e.zb || e.zb_len == 1 || (e.zb_len == L.N && aligned(e.zb))) &&
               (!e.scale || e.scale_len == 1 || (e.scale_len == L.N && aligned(e.scale)));
    if (!fast) return Epi::Generic;
    const bool gelu = e.act > 1;  // every activation but Relu: the out-of-line act4 of the *Gelu variants
    if (!getenv("RTEN_B200_NO_PLAIN") && e.act <= 7) {
        // f32: alpha = 1, optional column bias, residual with r_scale = 1, no range output
        if (L.kind == 0 && e.alpha == 1.0f && !e.range && (e.r == nullptr || e.r_scale == 1.0f))
            return gelu ? Epi::PlainF32Gelu : Epi::PlainF32;
        // integer: the *ToFloat operators with a scalar (or no) activation zero point and symmetric weights
        if (L.kind == 1 && e.scale && !e.za && !e.zb && (e.scale_len == 1 || e.scale_len == L.N) && splitk == 1 &&
            (!e.za8 || e.colsum))
            return gelu ? Epi::PlainI8Gelu : Epi::PlainI8;
    }
    return gelu ? Epi::FastGelu : Epi::Fast;
}

static const char* epi_name(Epi v) {
    static const char* const names[] = {"Generic", "Fast", "FastGelu", "PlainF32", "PlainF32Gelu", "PlainI8", "PlainI8Gelu"};
    return names[(int)v];
}

static bool is_plain_f32(Epi v) { return v == Epi::PlainF32 || v == Epi::PlainF32Gelu; }

struct PlanShape {
    long long tiles_n, units_m, tiles, units;
    int kb_per, stage_bytes, stages, n_stg;
};

// Derived sizes of a plan; false if the plan cannot run (accumulator columns, shared memory, counters).  The kernels
// compute one 128 x bn tile per unit: bn in {32, 64} (umma_gemm_kernel), or bn in {128, 256} without split-K for the
// launches that take the plain f32 epilogue (umma_wide_kernel).  One 128-byte K block per pipeline stage.
static bool plan_shape(const Prepared& q, const Plan& pl, PlanShape& ps) {
    const KParams& p = q.p;
    if (pl.splitk < 1) return false;  // (recorded plans are read from a text file: no division by zero, no negative units)
    if (is_wide(pl.bn)) {
        if ((pl.bn != 128 && pl.bn != 256) || !q.wide || pl.splitk != 1) return false;
        if (pl.bn == 256 && q.p.epi.act > 1) return false;  // act4 (Gelu and up): 128-column tiles only (umma_wide_kernel)
    } else if (pl.bn < 16 || pl.bn % 32 || pl.bn % q.step) {
        return false;
    }
    if (pl.nbuf < (q.res_tma ? 2 : 1) || pl.nbuf > 4) return false;  // staging buffers per group: res_bar has 4; a
                                                                     // TMA-staged residual needs two
    ps.tiles_n = q.chain_bytes ? 1 : (p.N + pl.bn - 1) / pl.bn;  // (chained: all N columns in one unit, by passes)
    ps.units_m = p.tiles_m;
    ps.tiles = ps.units_m * ps.tiles_n * q.batch;
    ps.units = ps.tiles * pl.splitk;
    if (ps.units > 0x7FFFFFFFll) return false;
    ps.kb_per = (p.k_blocks + pl.splitk - 1) / pl.splitk;
    if (pl.splitk > 1) {
        if (pl.bn % 32 || (long long)(pl.splitk - 1) * ps.kb_per >= p.k_blocks) return false;  // no empty split
        if (ps.tiles * 2 > SK_CNT_INTS) return false;
    }
    ps.n_stg = 2 * pl.nbuf;
    ps.stage_bytes = A_STAGE_BYTES + pl.bn * KBYTES;
    ps.stages = is_wide(pl.bn) ? wide_stages(ps.stage_bytes, q.chain_bytes) : std::min(MAX_STAGES, smem_budget_for(ps.n_stg) / ps.stage_bytes);
    if (ps.stages < 2) return false;
    return true;
}

// Cost model in SM clocks.  Its constants are unmeasured estimates that only rank candidate plans:
//   * the operand stream L2 -> shared memory (~7400 B/clk for the whole chip, at most ~64 B/clk for one SM) bounds a K block;
//   * the tensor pipe needs bn clk per 128 x bn x 32-byte step at the data-sheet TF32 rate (~1024 MAC / clk / SM),
//     issuing it ~42 clk;
//   * every pipeline stage costs a fixed ~320 clk (barrier wait, fence, descriptors, commit);
//   * a stage cannot complete faster than the TMA latency (~2300 clk under load) / stages in flight;
//   * the narrow kernel's epilogue (~350 clk per 32-column chunk, two warp groups) overlaps the next main loop; the
//     wide kernel's (~400 clk per chunk, both warpgroups on every chunk) follows its main loop.
static double plan_cost(const Prepared& q, const Plan& pl, const PlanShape& ps, int num_sms) {
    const double active = (double)std::min<long long>(ps.units, num_sms);
    const double waves = std::ceil((double)ps.units / num_sms);
    const double bw = std::min(64.0, 7400.0 / active);
    const double mmas = 4.0;
    const double t_kb = std::max(mmas * std::max(42.0, (double)pl.bn), ps.stage_bytes / bw);
    double t_stage = std::max(t_kb, 320.0 + mmas * 42.0);
    t_stage = std::max(t_stage, 2300.0 / ps.stages);
    const double mainloop = ps.kb_per * t_stage;
    const double epi = is_wide(pl.bn) ? (pl.bn / 32.0) * 400.0 + 600.0 : (pl.bn / 32.0) * 350.0 / 2.0 + 600.0;
    double unit = (is_wide(pl.bn) ? mainloop + epi : std::max(mainloop, epi)) + 1500.0;
    double cost = waves * unit + 2500.0;
    if (pl.splitk > 1) cost += epi * (1.0 + 0.25 * pl.splitk) + 1500.0;  // publish + the owner's reduction

    return cost;
}

static void enumerate_plans(const Prepared& q, int num_sms, std::vector<std::pair<double, Plan>>& out) {
    const KParams& p = q.p;
    const int nmax = (p.N + q.step - 1) / q.step * q.step;
    static const int splits[] = {1, 2, 3, 4, 5, 6, 8, 10, 12, 16};
    for (int bn : {32, 64, 128, 256}) {
        if (bn > nmax && bn != 32) break;
        for (int sk : splits) {
            Plan pl;
            pl.bn = bn;
            pl.splitk = sk;
            if (sk > 1 && p.k_blocks / sk < 4) continue;
            const int kb_per = (p.k_blocks + sk - 1) / sk;
            pl.nbuf = (q.res_tma || kb_per < 24) ? 2 : 1;
            PlanShape ps;
            if (is_wide(bn)) {
                pl.nbuf = 2;  // (the wide kernel has two fixed staging buffers)
            } else if (pl.nbuf == 2 && !getenv("RTEN_B200_NO_NBUF3")) {
                // A third staging buffer per group takes the wait for the previous store's shared-memory read and, with a
                // residual, the late request of the next residual tile off the chunk's critical path -- as long as the
                // operand ring keeps three stages (or loses none)
                PlanShape ps2;
                const bool ok2 = plan_shape(q, pl, ps2);
                pl.nbuf = 3;
                if (!plan_shape(q, pl, ps) || (ps.stages < 3 && !(ok2 && ps.stages == ps2.stages))) pl.nbuf = 2;
            }
            if (!plan_shape(q, pl, ps)) continue;
            if (sk > 1 && ps.tiles >= 2 * num_sms) continue;  // enough parallelism without splitting K
            if (ps.stages < 2) continue;
            out.emplace_back(plan_cost(q, pl, ps, num_sms), pl);
        }
    }
    std::sort(out.begin(), out.end(), [](const std::pair<double, Plan>& x, const std::pair<double, Plan>& y) {
        return x.first < y.first;
    });
}

static rten_status prepare_launch(rten_ctx* ctx, const GemmLaunch& L, Prepared& q) {
    const int esize = L.kind == 0 ? 4 : 1;
    const int kelems = KBYTES / esize;
    if (!tma_compatible(L.a, esize, 4) || !tma_compatible(L.b, esize, 4)) return RTEN_ERR_UNSUPPORTED_VALUE;
    if (L.M <= 0 || L.N <= 0 || L.K <= 0) return RTEN_ERR_UNSUPPORTED_VALUE;
    q.esize = esize;
    q.kelems = kelems;
    KParams& p = q.p;
    memset(&p, 0, sizeof(p));
    p.M = L.M;
    p.N = L.N;
    p.K = L.K;
    p.z0 = L.z0;
    p.z1 = L.z1;
    p.kelems = kelems;
    p.conv = L.conv;
    p.epi = L.epi;
    p.c_blocks = 1;
    p.kw = 1;
    for (int i = 0; i < 4; i++) q.aes[i] = 1;
    if (L.conv) {
        const ConvGeom& g = L.g;
        pick_conv_tile(g, p.tw, p.th, p.tb);
        p.tiles_x = (g.OW + p.tw - 1) / p.tw;
        p.tiles_y = (g.OH + p.th - 1) / p.th;
        int tiles_b = (g.B + p.tb - 1) / p.tb;
        p.tiles_m = p.tiles_x * p.tiles_y * tiles_b;
        p.OH = g.OH;
        p.OW = g.OW;
        p.Bn = g.B;
        p.sy = g.sy;
        p.sx = g.sx;
        p.dy = g.dy;
        p.dx = g.dx;
        p.pt = g.pt;
        p.pl = g.pl;
        p.kw = g.kw;
        p.c_blocks = (g.C + kelems - 1) / kelems;
        p.k_blocks = g.kh * g.kw * p.c_blocks;
        p.z0 = p.z1 = 1;
        q.abox[0] = kelems;
        q.abox[1] = p.tw * g.sx;
        q.abox[2] = p.th * g.sy;
        q.abox[3] = p.tb;
        q.aes[1] = g.sx;
        q.aes[2] = g.sy;
        q.a_rows = p.tw * p.th * p.tb;
        q.batch = 1;
    } else {
        p.tiles_m = (L.M + BM - 1) / BM;
        p.k_blocks = (L.K + kelems - 1) / kelems;
        q.abox[0] = kelems;
        q.abox[1] = BM;
        q.abox[2] = 1;
        q.abox[3] = 1;
        q.a_rows = BM;
        q.batch = (long long)L.z0 * L.z1;
        p.a_bcast0 = (L.a.dims[2] == 1 && L.z0 > 1) ? 1 : 0;
        p.a_bcast1 = (L.a.dims[3] == 1 && L.z1 > 1) ? 1 : 0;
        p.b_bcast0 = (L.b.dims[2] == 1 && L.z0 > 1) ? 1 : 0;
        p.b_bcast1 = (L.b.dims[3] == 1 && L.z1 > 1) ? 1 : 0;
    }
    // ---- output path: TMA store needs contiguous 4-byte rows at 16-byte aligned pitches
    OperandDesc& od = q.od;
    OperandDesc& ord = q.ord;
    q.dbox[0] = 32;
    q.dbox[1] = q.dbox[2] = q.dbox[3] = 1;
    const EpilogueDesc& e = L.epi;
    od.base = e.d;
    od.dims[0] = L.N;
    od.strides[0] = 1;
    if (L.conv) {
        od.dims[1] = L.g.OW;
        od.dims[2] = L.g.OH;
        od.dims[3] = L.g.B;
        od.strides[1] = e.s_z1;
        od.strides[2] = e.s_row;
        od.strides[3] = e.s_z0;
        q.dbox[1] = p.tw;
        q.dbox[2] = p.th;
        q.dbox[3] = p.tb;
    } else {
        od.dims[1] = L.M;
        od.dims[2] = L.z0;
        od.dims[3] = L.z1;
        od.strides[1] = e.s_row;
        od.strides[2] = e.s_z0;
        od.strides[3] = e.s_z1;
        q.dbox[1] = BM;
    }
    q.tma_store = (e.s_col == 1 && L.N >= 4 && tma_compatible(od, 4, 4)) ? 1 : 0;
    if (getenv("RTEN_B200_NO_TMA_STORE")) q.tma_store = 0;
    // residual prefetched by TMA: same geometry as the output, own strides (fast-path epilogue only)
    ord = od;
    ord.base = e.r;
    if (L.conv) {
        ord.strides[1] = e.r_z1;
        ord.strides[2] = e.r_row;
        ord.strides[3] = e.r_z0;
    } else {
        ord.strides[1] = e.r_row;
        ord.strides[2] = e.r_z0;
        ord.strides[3] = e.r_z1;
    }
    q.res_tma = (q.tma_store && (L.kind == 0 || e.scale) && e.r && e.r_col == 1 && (L.N % 32) == 0 &&
                 (e.bias_kind != 1 || (reinterpret_cast<uintptr_t>(e.bias) & 15) == 0) && tma_compatible(ord, 4, 4))
                    ? 1
                    : 0;
    // a broadcast residual (Gemm's C) has zero strides on real dims: keep the register path for it
    for (int i = 1; i < 4; i++)
        if (ord.dims[i] > 1 && ord.strides[i] == 0) q.res_tma = 0;
    if (getenv("RTEN_B200_NO_RES_TMA")) q.res_tma = 0;
    p.res_tx_bytes = q.a_rows * KBYTES;
    q.step = q.tma_store ? 32 : 16;
    const bool plain = is_plain_f32(pick_epilogue(L, q.tma_store, q.res_tma, 1));
    // RTEN_B200_NO_WIDE=1: no wide-tile plans (measures what they gain; recorded wide plans are re-planned)
    q.wide = plain && !getenv("RTEN_B200_NO_WIDE");
    // ---- projection source: whole 128-byte channel blocks after the main K range; its A box covers the same 128 output
    //      pixels as the main one, read at `stride` (element strides), so a stage's byte count does not change
    p.kb_main = p.k_blocks;
    if (L.proj.C > 0) {
        const GemmLaunch::Projection& pr = L.proj;
        const int s = pr.stride;
        if (!L.conv || L.kind != 0 || pr.C % kelems || s < 1 || s > 8 || p.tw * s > 256 || p.th * s > 256 || !plain ||
            pr.a.dims[0] * (pr.x3_cb ? 3 : 1) != pr.C || pr.b.dims[0] != pr.C || !tma_compatible(pr.a, 4, 4) || !tma_compatible(pr.b, 4, 4))
            return RTEN_ERR_UNSUPPORTED_VALUE;
        p.kb_proj = pr.C / kelems;
        p.s_proj = s;
        p.k_blocks += p.kb_proj;
        const uint32_t box[4] = {(uint32_t)kelems, (uint32_t)(p.tw * s), (uint32_t)(p.th * s), (uint32_t)p.tb};
        const uint32_t es[4] = {1, (uint32_t)s, (uint32_t)s, 1};
        for (int i = 0; i < 4; i++) {
            q.pbox[i] = box[i];
            q.pes[i] = es[i];
        }
    }
    // ---- chained 1x1 convolution of the output: the wide kernel's plain f32 epilogue, whole 32-column chunks, a unit
    //      holds all N columns
    q.chain_bytes = 0;
    if (L.chain.N2 > 0) {
        const GemmLaunch::Chain& c = L.chain;
        if (!L.conv || L.kind != 0 || ctx->f32_mode != RTEN_F32_TF32 || !q.wide || !q.tma_store || L.epi.act > 1 ||
            L.N % 32 || L.N > 256 || (c.N2 != 64 && c.N2 != 128) || c.act < 0 || c.act > 1 || c.w.dims[0] != L.N ||
            c.w.dims[1] != c.N2 || c.z.dims[0] != c.N2 || !tma_compatible(c.w, 4, 4) || !tma_compatible(c.z, 4, 4) ||
            (L.epi.r && !q.res_tma))
            return RTEN_ERR_UNSUPPORTED_VALUE;
        q.chain_bytes = L.N / 32 * c.N2 * KBYTES;
    }
    return RTEN_OK;
}

static size_t splitk_ws_bytes(const PlanShape& ps, const Plan& pl) {
    return pl.splitk > 1 ? (size_t)ps.tiles * pl.splitk * (pl.bn / 32) * 4096 * 4 : 0;
}

static rten_status ensure_splitk_counters(rten_ctx* ctx) {
    if (!ctx->sk_counters) {
        cudaError_t ce = cudaMalloc(&ctx->sk_counters, SK_CNT_INTS * sizeof(int));
        if (ce != cudaSuccess) return fail_cuda(ctx, ce, "split-K counters");
        ce = cudaMemset(ctx->sk_counters, 0, SK_CNT_INTS * sizeof(int));
        if (ce != cudaSuccess) return fail_cuda(ctx, ce, "split-K counters");
    }
    return RTEN_OK;
}

// `ws`: split-K workspace of at least splitk_ws_bytes() (null: taken from the op's temporaries)
static rten_status launch_plan(rten_ctx* ctx, const GemmLaunch& L, const Prepared& q, const Plan& pl, bool verbose,
                               void* ws = nullptr) {
    PlanShape ps;
    if (!plan_shape(q, pl, ps)) return RTEN_ERR_UNSUPPORTED_VALUE;
    KParams p = q.p;
    p.bn = pl.bn;
    p.splitk = pl.splitk;
    p.nbuf = pl.nbuf;
    p.tma_store = q.tma_store;
    p.res_tma = q.res_tma ? 1 : 0;
    p.kb_per = ps.kb_per;
    p.tiles_n = (int)ps.tiles_n;
    p.tiles_total = (int)ps.tiles;
    p.units_total = (int)ps.units;
    p.d_tiles_n.set(p.tiles_n);
    p.d_tiles_m.set(p.tiles_m);
    p.d_z0.set(p.z0);
    p.d_tiles_x.set(p.conv ? p.tiles_x : 1);
    p.d_tiles_y.set(p.conv ? p.tiles_y : 1);
    p.d_tiles_total.set(p.tiles_total);
    p.d_c_blocks.set(p.c_blocks);
    p.d_kw.set(p.kw);
    p.d_tw.set(p.conv ? p.tw : 1);
    p.d_th.set(p.conv ? p.th : 1);
    p.stage_bytes = ps.stage_bytes;
    p.tx_bytes = q.a_rows * KBYTES + p.bn * KBYTES;  // per 128-byte K block
    p.stages = ps.stages;
    p.sgn = L.kind == 0 ? 0 : (L.a_signed ? 1 : 0) | (L.b_signed ? 2 : 0);
    if (p.splitk > 1) {
        RTB_TRY(ensure_splitk_counters(ctx));
        if (!ws) RTB_TRY(temp_alloc(ctx, splitk_ws_bytes(ps, pl), &ws));
        p.sk_ws = reinterpret_cast<uint32_t*>(ws);
        p.sk_cnt = reinterpret_cast<int*>(ctx->sk_counters);
    }

    uint32_t bbox[4] = {(uint32_t)q.kelems, (uint32_t)p.bn, 1, 1}, bes[4] = {1, 1, 1, 1}, des[4] = {1, 1, 1, 1};
    TmaMaps m;
    if (!encode_map(ctx, &m.a, L.a, q.esize, L.kind == 0, q.abox, q.aes)) return RTEN_ERR_UNSUPPORTED_VALUE;
    if (!encode_map(ctx, &m.b, L.b, q.esize, L.kind == 0, bbox, bes)) return RTEN_ERR_UNSUPPORTED_VALUE;
    m.d = m.r = m.a2 = m.a_proj = m.b_proj = m.a2_proj = m.w2 = m.z = m.a;  // (maps the launch does not use)
    p.x3_cb = L.x3_cb;
    if (L.x3_cb && !encode_map(ctx, &m.a2, L.a_lo, q.esize, true, q.abox, q.aes)) return RTEN_ERR_UNSUPPORTED_VALUE;
    if (p.kb_proj) {
        p.x3_cb_proj = L.proj.x3_cb;
        if (!encode_map(ctx, &m.a_proj, L.proj.a, 4, true, q.pbox, q.pes) ||
            !encode_map(ctx, &m.b_proj, L.proj.b, 4, true, bbox, bes) ||
            (L.proj.x3_cb && !encode_map(ctx, &m.a2_proj, L.proj.a_lo, 4, true, q.pbox, q.pes)))
            return RTEN_ERR_UNSUPPORTED_VALUE;
    }
    if (p.tma_store && !encode_map(ctx, &m.d, q.od, 4, true, q.dbox, des)) {
        p.tma_store = 0;  // the generic epilogue stores directly
        p.res_tma = 0;
        m.d = m.a;
    }
    if (p.res_tma && !encode_map(ctx, &m.r, q.ord, 4, true, q.dbox, des)) {
        p.res_tma = 0;
        m.r = m.a;
    }
    const Epi epi = pick_epilogue(L, p.tma_store, p.res_tma, p.splitk);
    // the generic epilogue takes a TMA-staged residual only on its register path (f32, act <= Relu)
    if (epi == Epi::Generic && (L.kind == 1 || L.epi.act > 1)) p.res_tma = 0;
    if (q.chain_bytes) {
        const GemmLaunch::Chain& c = L.chain;
        const uint32_t wbox[4] = {32, (uint32_t)c.N2, 1, 1}, zbox[4] = {32, q.dbox[1], q.dbox[2], q.dbox[3]};
        if (epi != Epi::PlainF32 || (L.epi.r && !p.res_tma) || !encode_map(ctx, &m.w2, c.w, 4, true, wbox, des) ||
            !encode_map(ctx, &m.z, c.z, 4, true, zbox, des))
            return RTEN_ERR_UNSUPPORTED_VALUE;
        p.chain_n2 = c.N2;
        p.chain_passes = (L.N + p.bn - 1) / p.bn;
        p.chain_act = c.act;
        p.chain_bias = c.bias;
    }

    if (verbose)
        fprintf(stderr, "[umma_gemm] kind=%d conv=%d M=%d N=%d K=%d kb=%d kb_proj=%d tiles_m=%d bn=%d splitk=%d units=%d stages=%d tma_store=%d res_tma=%d nbuf=%d box=%dx%dx%d epi=%s%s\n",
                L.kind, L.conv, L.M, L.N, L.K, p.k_blocks, p.kb_proj, p.tiles_m, p.bn, p.splitk, p.units_total, p.stages,
                p.tma_store, p.res_tma, p.nbuf, p.tw, p.th, p.tb, epi_name(epi),
                p.chain_n2 == 64 ? " chain=64" : p.chain_n2 == 128 ? " chain=128" : "");
    // (an output / residual map failed to encode; a projection source and a second bias need the plain f32 epilogue)
    if ((is_wide(p.bn) || p.kb_proj || L.epi.bias2) && !is_plain_f32(epi)) return RTEN_ERR_UNSUPPORTED_VALUE;
    const size_t smem_bytes = (size_t)p.stages * p.stage_bytes + q.chain_bytes +
                              (is_wide(p.bn) ? WIDE_SMEM_FIXED_BYTES : ps.n_stg * STG_BYTES + SMEM_FIXED_BYTES);
    using Kernel = void (*)(TmaMaps, KParams);
    // [kind][variant]: the integer kind has no plain f32 kernels, the f32 kind no plain integer ones
    static const Kernel narrow[2][7] = {
        {umma_gemm_kernel<0, Epi::Generic>, umma_gemm_kernel<0, Epi::Fast>, umma_gemm_kernel<0, Epi::FastGelu>,
         umma_gemm_kernel<0, Epi::PlainF32>, umma_gemm_kernel<0, Epi::PlainF32Gelu>, nullptr, nullptr},
        {umma_gemm_kernel<1, Epi::Generic>, umma_gemm_kernel<1, Epi::Fast>, umma_gemm_kernel<1, Epi::FastGelu>, nullptr,
         nullptr, umma_gemm_kernel<1, Epi::PlainI8>, umma_gemm_kernel<1, Epi::PlainI8Gelu>}};
    const Kernel kern = !is_wide(p.bn)              ? narrow[L.kind][(int)epi]
                        : p.chain_n2 == 64         ? umma_wide_kernel<Epi::PlainF32, 64>
                        : p.chain_n2 == 128        ? umma_wide_kernel<Epi::PlainF32, 128>
                        : epi == Epi::PlainF32Gelu ? umma_wide_kernel<Epi::PlainF32Gelu>
                                                   : umma_wide_kernel<Epi::PlainF32>;

    const int threads = is_wide(p.bn) ? WIDE_THREADS : NUM_THREADS;
    return launch(ctx, "umma_gemm launch", kern, {std::min(p.units_total, ctx->num_sms), threads, smem_bytes, 227 * 1024, true}, m, p);
}

// Problem signature for the autotune cache: everything that changes which plan is fastest.
static std::vector<long long> tune_key(const GemmLaunch& L, const Prepared& q) {
    const EpilogueDesc& e = L.epi;
    std::vector<long long> k = {L.kind, L.conv, L.M, L.N, L.K, L.z0, L.z1, q.tma_store, q.res_tma, e.act, e.bias_kind,
                                e.r != nullptr, (e.za != nullptr || e.za8 != nullptr), e.zb != nullptr, e.scale != nullptr,
                                L.a.strides[1], L.b.strides[1], L.x3_cb};
    if (L.conv) {
        const ConvGeom& g = L.g;
        for (long long v : {g.B, g.H, g.W, g.C, g.OH, g.OW, g.kh, g.kw, g.sy, g.sx, g.dy, g.dx, g.pt, g.pl}) k.push_back(v);
    }
    if (L.proj.C > 0) {  // (absent from keys without one: recorded plans of unfolded launches stay valid)
        const GemmLaunch::Projection& pr = L.proj;
        for (int64_t v : {(int64_t)-1, (int64_t)pr.C, (int64_t)pr.stride, (int64_t)pr.x3_cb, pr.a.dims[1], pr.a.dims[2],
                          pr.a.strides[1], pr.a.strides[2], pr.a.strides[3], pr.b.strides[1]})
            k.push_back(v);
    }
    return k;
}

// A plan as the three integers of its tune_cache entry and plans-file line: `bn splitk nbuf`, or `-1 bn T` for the
// halo-reuse kernel.
static std::array<int, 3> plan_record(const Plan& pl) {
    return pl.halo ? std::array<int, 3>{-1, pl.bn, pl.T} : std::array<int, 3>{pl.bn, pl.splitk, pl.nbuf};
}

static Plan plan_from_record(const std::array<int, 3>& r) {
    if (r[0] < 0) return halo_plan(r[1], r[2]);
    Plan pl;
    pl.bn = r[0];
    pl.splitk = r[1];
    pl.nbuf = r[2];
    return pl;
}

// Measured launch plans can be kept across processes: RTEN_B200_TUNE_FILE names a text file that is read when a
// context is created and rewritten when a context that measured new plans is destroyed (one line per problem:
// tune_key's integers, '|', the three integers of plan_record).  Lines with any other number of plan integers (files
// written by older builds) are skipped: those problems are planned afresh.  A recorded plan that no longer fits its
// problem is dropped when it is used.
void tune_cache_load(rten_ctx* ctx, const char* path) {
    FILE* f = fopen(path, "r");
    if (!f) return;
    char line[2048];
    while (fgets(line, sizeof(line), f)) {
        std::vector<long long> key;
        std::array<int, 3> plan{};
        char* p = line;
        bool in_plan = false;
        int np = 0;
        while (*p) {
            while (*p == ' ') p++;
            if (*p == '|') {
                in_plan = true;
                p++;
                continue;
            }
            if (*p == '\n' || *p == 0) break;
            char* end = nullptr;
            const long long v = strtoll(p, &end, 10);
            if (end == p) break;
            if (in_plan) {
                if (np < 3) plan[np] = (int)v;
                np++;
            } else {
                key.push_back(v);
            }
            p = end;
        }
        if (np == 3 && !key.empty()) ctx->tune_cache[key] = plan;
    }
    fclose(f);
}

void tune_cache_save(rten_ctx* ctx, const char* path) {
    FILE* f = fopen(path, "w");
    if (!f) return;
    for (const auto& kv : ctx->tune_cache) {
        for (long long v : kv.first) fprintf(f, "%lld ", v);
        fprintf(f, "|");
        for (int v : kv.second) fprintf(f, " %d", v);
        fprintf(f, "\n");
    }
    fclose(f);
}

// RTEN_F32_TF32X3: run the same kernel over split operands -- K (plain) or C (conv; K order is (ky, kx, c)) tripled:
// A' = [lo | hi | hi], B' = [hi | lo | hi]  =>  lo*hi + hi*lo + hi*hi, small terms first.
//  * B: a constant operand (prepacked weights, `b_x3_slot`) is split ONCE and cached with its owner.
//  * A: kind::tf32 ignores the 13 low mantissa bits, so the ORIGINAL tensor serves as both `hi` segments; only the low
//    parts are written (4 B / element instead of 12) and the kernel's producer switches tensor maps per segment
//    (KParams::x3_cb).  Needs K (C) % 32 == 0 and a TMA-addressable A; otherwise the three-segment copy is built.
static rten_status launch_tf32x3(rten_ctx* ctx, const GemmLaunch& L0) {
    GemmLaunch L = L0;
    long long d0 = 0, d0p = 0;  // K or channels per group of the source being split; thirds stay 16-byte aligned for TMA
    auto split = [&](const OperandDesc& src, OperandDesc& dst, int role, void* into) -> rten_status {
        const long long planes = role == 2 ? 1 : 3;
        long long dims[4], strides[4], n = planes * d0p;
        for (int i = 0; i < 4; i++) {
            // broadcast dims (stride 0) are split once and stay broadcast
            dims[i] = (i > 0 && src.strides[i] == 0) ? 1 : src.dims[i];
            strides[i] = src.strides[i];
        }
        for (int i = 1; i < 4; i++) n *= dims[i];
        void* buf = into;
        if (!buf) RTB_TRY(temp_alloc(ctx, (size_t)n * 4, &buf));
        RTB_TRY(launch_tf32x3_split(ctx, (const float*)src.base, (float*)buf, dims, strides, d0p, role));
        dst = src;
        dst.base = buf;
        dst.dims[0] = planes * d0p;
        long long st = planes * d0p;
        for (int i = 1; i < 4; i++) {
            dst.strides[i] = (src.strides[i] == 0 && src.dims[i] > 1) ? 0 : st;
            st *= dims[i];
        }
        return RTEN_OK;
    };
    // One (A, B) source -- the main one, or the projection source (GemmLaunch::proj) with its own B copy and A planes
    auto split_source = [&](const OperandDesc& a0, const OperandDesc& b0, void** slot, const void* a_lo_base,
                            OperandDesc& a, OperandDesc& b, OperandDesc& a_lo, int& x3_cb) -> rten_status {
        d0 = a0.dims[0];
        d0p = (d0 + 3) / 4 * 4;
        if (b0.dims[0] != d0) return RTEN_ERR_UNSUPPORTED_VALUE;
        // ---- B
        if (slot && !getenv("RTEN_B200_X3_NO_CACHE")) {
            if (!*slot && !ctx->capturing) {
                long long n = 3 * d0p;
                for (int i = 1; i < 4; i++) n *= (b0.strides[i] == 0 ? 1 : b0.dims[i]);
                void* buf = nullptr;
                if (cudaMalloc(&buf, (size_t)n * 4) != cudaSuccess) return fail(ctx, RTEN_ERR_CUDA, "cudaMalloc failed for the 3xTF32 copy of a prepacked operand");
                OperandDesc tmp;
                const rten_status st = split(b0, tmp, 1, buf);
                if (st != RTEN_OK) {
                    cudaFree(buf);
                    return st;
                }
                *slot = buf;
            }
        }
        if (slot && *slot && !getenv("RTEN_B200_X3_NO_CACHE")) {
            b = b0;
            b.base = *slot;
            b.dims[0] = 3 * d0p;
            long long st = 3 * d0p;
            for (int i = 1; i < 4; i++) {
                const long long di = b0.strides[i] == 0 ? 1 : b0.dims[i];
                b.strides[i] = (b0.strides[i] == 0 && b0.dims[i] > 1) ? 0 : st;
                st *= di;
            }
        } else {
            RTB_TRY(split(b0, b, 1, nullptr));
        }
        // ---- A
        const bool two_plane = d0 % 32 == 0 && tma_compatible(a0, 4, 4) && !getenv("RTEN_B200_X3_THREE_PLANES");
        if (two_plane && a_lo_base) {
            a_lo = a0;
            a_lo.base = a_lo_base;
            x3_cb = (int)(d0 / 32);
        } else if (two_plane) {
            RTB_TRY(split(a0, a_lo, 2, nullptr));
            x3_cb = (int)(d0 / 32);
        } else {
            RTB_TRY(split(a0, a, 0, nullptr));
        }
        return RTEN_OK;
    };
    RTB_TRY(split_source(L0.a, L0.b, L0.b_x3_slot, L0.a_lo_base, L.a, L.b, L.a_lo, L.x3_cb));
    if (L.conv)
        L.g.C = (int)(3 * d0p);
    L.K = L.conv ? (int)(L0.K / d0 * 3 * d0p) : (int)(3 * d0p);
    L.b_x3_slot = nullptr;
    L.a_lo_base = nullptr;
    if (L0.proj.C > 0) {
        RTB_TRY(split_source(L0.proj.a, L0.proj.b, L0.proj.b_x3_slot, nullptr, L.proj.a, L.proj.b, L.proj.a_lo, L.proj.x3_cb));
        L.proj.C = (int)(3 * d0p);
        L.proj.b_x3_slot = nullptr;
    }
    const int saved = ctx->f32_mode;
    ctx->f32_mode = RTEN_F32_TF32;
    const rten_status st = launch_umma_gemm(ctx, L);
    ctx->f32_mode = saved;
    return st;
}

static rten_status run_plan(rten_ctx* ctx, const GemmLaunch& L, const Prepared& q, const Plan& pl, bool verbose,
                            void* ws = nullptr) {
    return pl.halo ? launch_umma_halo_conv(ctx, L, pl.bn, pl.T, verbose) : launch_plan(ctx, L, q, pl, verbose, ws);
}

// With the stream idle and the launch safe to repeat: times up to 24 of the model's candidates and, where `halo`, the
// halo kernel's unit shapes, records the fastest and leaves it in `plan`.  Otherwise leaves `plan` as it is.
static rten_status autotune(rten_ctx* ctx, const GemmLaunch& L, const Prepared& q,
                            const std::vector<std::pair<double, Plan>>& cands, bool halo, bool verbose, Plan& plan) {
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    cudaStreamIsCapturing(ctx->stream, &cs);
    // re-running the launch must be idempotent: the output may not alias the residual
    if (ctx->capturing || cs != cudaStreamCaptureStatusNone || (L.epi.r && (const void*)L.epi.r == (const void*)L.epi.d))
        return RTEN_OK;
    const size_t ncand = std::min<size_t>(cands.size(), 24);
    // one split-K workspace for every candidate (allocating inside the timed launches would time cudaMalloc)
    size_t ws_max = 0;
    for (size_t i = 0; i < ncand; i++) {
        PlanShape ps;
        if (plan_shape(q, cands[i].second, ps)) ws_max = std::max(ws_max, splitk_ws_bytes(ps, cands[i].second));
    }
    void* ws = nullptr;
    if (ws_max) {
        RTB_TRY(ensure_splitk_counters(ctx));
        RTB_TRY(temp_alloc(ctx, ws_max, &ws));
        cudaStreamSynchronize(ctx->stream);
    }
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0);
    cudaEventCreate(&e1);
    // ms per launch over n launches after a warm-up launch (which also validates the plan); < 0: the plan did not run
    auto time_plan = [&](const Plan& x, int n) -> double {
        if (run_plan(ctx, L, q, x, false, ws) != RTEN_OK) return -1.0;
        cudaEventRecord(e0, ctx->stream);
        bool ok = true;
        for (int r = 0; r < n && ok; r++) ok = run_plan(ctx, L, q, x, false, ws) == RTEN_OK;
        cudaEventRecord(e1, ctx->stream);
        if (cudaEventSynchronize(e1) != cudaSuccess || !ok) return -1.0;
        float t = 0.f;
        cudaEventElapsedTime(&t, e0, e1);
        return (double)t / n;
    };
    double best_ms = 1e30;
    int reps = 4;  // raised after the first candidate so that every timed window is >= ~150 us (event resolution)
    std::vector<std::pair<double, size_t>> timed;
    for (size_t i = 0; i < ncand; i++) {
        const Plan& x = cands[i].second;
        double ms = time_plan(x, reps);
        if (ms < 0) continue;
        timed.emplace_back(ms, i);
        if (verbose)
            fprintf(stderr, "[autotune] bn=%d splitk=%d nbuf=%d model=%.0f -> %.2f us\n", x.bn, x.splitk, x.nbuf,
                    cands[i].first, ms * 1e3);
        if (ms < best_ms) {
            best_ms = ms;
            plan = x;
        }
        reps = std::max(4, std::min(32, (int)(0.15 / std::max(best_ms, 1e-3))));
    }
    // second look at the three fastest with longer windows: single measurements of 20-40 us kernels are noisy enough
    // to flip the choice between near-equal plans from run to run
    std::sort(timed.begin(), timed.end());
    best_ms = 1e30;
    for (size_t k = 0; k < std::min<size_t>(3, timed.size()); k++) {
        const Plan& x = cands[timed[k].second].second;
        const double again = time_plan(x, 2 * reps);
        const double ms = again < 0 ? timed[k].first : again;  // the longer window decides
        if (ms < best_ms) {
            best_ms = ms;
            plan = x;
        }
    }
    for (const auto& s : HALO_SHAPES) {
        const Plan x = halo_plan(s[0], s[1]);
        if (!halo || x.bn > L.N) continue;
        double ms = time_plan(x, reps);
        if (ms > 0 && ms < best_ms * 1.05) ms = time_plan(x, 2 * reps);  // a second, longer look at contenders
        if (verbose && ms > 0) fprintf(stderr, "[autotune] halo bn=%d T=%d -> %.2f us\n", x.bn, x.T, ms * 1e3);
        if (ms > 0 && ms < best_ms * 0.97) {  // must win clearly: the generic kernel is the better-trodden path
            best_ms = ms;
            plan = x;
        }
    }
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    ctx->tune_cache[tune_key(L, q)] = plan_record(plan);
    return RTEN_OK;
}

rten_status launch_umma_gemm(rten_ctx* ctx, const GemmLaunch& L) {
    const bool verbose = getenv("RTEN_B200_VERBOSE") != nullptr;
    const char* force_bn = getenv("RTEN_B200_FORCE_BN");
    const char* force_sk = getenv("RTEN_B200_FORCE_SPLITK");
    const char* halo_on = getenv("RTEN_B200_HALO");
    // stride-1 windows (the 3x3 layers) may run on the halo-reuse kernel, which moves the activations into shared
    // memory once per channel block instead of once per filter tap (umma_halo.cu)
    const bool halo = L.conv && L.kind == 0 && L.g.kh * L.g.kw > 1 && !L.x3_cb && !L.proj.C && !getenv("RTEN_B200_NO_HALO");
    Prepared q;
    if (L.chain.N2 > 0) {
        // chained: a fixed plan (128-column passes of one pixel tile), not autotuned; single-pass TF32 only (a 3xTF32
        // chain would not equal the separate launches)
        if (L.kind != 0 || ctx->f32_mode != RTEN_F32_TF32 || L.x3_cb || getenv("RTEN_B200_NO_CHAIN"))
            return RTEN_ERR_UNSUPPORTED_VALUE;
        RTB_TRY(prepare_launch(ctx, L, q));
        Plan pl;
        pl.bn = 128;
        pl.nbuf = 2;
        return launch_plan(ctx, L, q, pl, verbose);
    }
    if (L.kind == 0 && ctx->f32_mode == RTEN_F32_TF32X3) return launch_tf32x3(ctx, L);
    // RTEN_B200_HALO=1: the halo kernel's model shape without measurements.  Otherwise only a measurement picks the halo
    // kernel: which of the two kernels is faster depends on the layer.
    int hbn, hT;
    if (halo && halo_on && atoi(halo_on) != 0 && halo_model_shape(ctx, L, hbn, hT)) {
        const rten_status hs = run_plan(ctx, L, q, halo_plan(hbn, hT), verbose);
        if (hs != RTEN_ERR_UNSUPPORTED_VALUE) return hs;
    }
    RTB_TRY(prepare_launch(ctx, L, q));
    const bool forced = force_bn || force_sk;
    if (!forced && !ctx->tune_cache.empty()) {  // measured plan on record: no need to enumerate and rank candidates
        auto hit = ctx->tune_cache.find(tune_key(L, q));
        if (hit != ctx->tune_cache.end()) {
            const Plan pl = plan_from_record(hit->second);
            PlanShape ps;
            if (pl.halo ? halo && halo_shape_fits(L, pl.bn, pl.T) : plan_shape(q, pl, ps)) return run_plan(ctx, L, q, pl, verbose);
            // a stale entry (plans file written by another build / geometry): drop it and plan afresh
            if (verbose) fprintf(stderr, "[umma_gemm] recorded plan no longer valid for this problem: re-planning\n");
            ctx->tune_cache.erase(hit);
        }
    }
    std::vector<std::pair<double, Plan>> cands;
    enumerate_plans(q, ctx->num_sms, cands);
    if (cands.empty()) return RTEN_ERR_UNSUPPORTED_VALUE;
    Plan plan = cands[0].second;
    if (forced) {
        // debugging / sweeps: the best-ranked candidate that matches every forced field
        bool found = false;
        for (const auto& c : cands) {
            const Plan& x = c.second;
            if (force_bn && x.bn != atoi(force_bn)) continue;
            if (force_sk && x.splitk != atoi(force_sk)) continue;
            plan = x;
            found = true;
            break;
        }
        // RTEN_B200_FORCE_STRICT=1 (tests): a forced combination that no valid plan satisfies is an error instead of a
        // silent fall-back to the model's choice -- a sweep must exercise what it names
        if (!found) {
            ctx->forced_misses++;
            if (verbose) fprintf(stderr, "[umma_gemm] no valid plan matches the forced fields: using the model's choice\n");
            if (getenv("RTEN_B200_FORCE_STRICT"))
                return fail(ctx, RTEN_ERR_INVALID_VALUE, "no launch plan matches the forced RTEN_B200_FORCE_* fields");
        } else {
            ctx->forced_hits++;
        }
    } else if (ctx->autotune) {
        RTB_TRY(autotune(ctx, L, q, cands, halo, verbose, plan));
    }
    return run_plan(ctx, L, q, plan, verbose);
}

}  // namespace rtb
