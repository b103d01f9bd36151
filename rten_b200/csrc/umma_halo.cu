// Halo-reuse convolution on wgmma: stride-1 convolutions with a kh x kw window (the 3x3 layers of ResNet-50).
//
// The generic implicit-GEMM kernel (umma_gemm.cu) streams one activation box per filter tap from L2: a 3x3 layer moves
// its input nine times into shared memory, and at 4 bytes per TF32 operand the L2 -> SM stream, not the tensor pipe, sets
// its pace.  Here a CTA loads ONE zero-padded activation patch per 32-channel block
//     patch[b][y][x][32 ch]   y in [oy0 - pt, oy0 + R + kh - 1 - pt),  x in [-pl, -pl + P),  P = OW + kw - 1
// with a single TMA box (out-of-bounds -> 0 = the padding) and treats it as a LINEAR array of P-pitched pixel slots of
// 128 bytes: output slot s = y P + x reads, for tap (ky, kx), input slot s + ky P + kx.  Every tap is therefore the same
// patch seen through a shared-memory matrix descriptor whose start address is shifted by (ky P + kx) x 128 bytes -- the
// 128B swizzle is a function of the absolute shared-memory address, so TMA's layout and the shifted descriptor agree
// (base offset 0; checked against float64 by the halo parity test).  Slots with x >= OW (and the rows past the strip) are
// computed and thrown away: 2 / P of the MMA rows for a 3x3 window.  The weights stream through a ring of stages of one
// tap x (bn x 32 channel) tile.
//
// A unit is T x 128 slots x bn output channels.  Roles (384 threads):
//   warpgroup 0    : TMA producer (warp 0), registers released
//   warpgroups 1, 2: slots [64 T w, 64 T (w + 1)) of the unit, w = 0, 1: T m64nbnk8 wgmma per k8 step, then the
//                    epilogue straight from those registers
// Both consumers read the same weight stage, so a stage carries 2 T x 64 slots of MMA work (T = 2, bn = 128: 16 KB of
// weights per 2.1 MFLOP).  One wgmma group stays in flight across stages; a stage goes back to the producer once both
// consumers have retired it (8 warp arrivals), and the producer keeps loading the next unit while the consumers run the
// epilogue.  Every unit shape accumulates in the same order -- channel block outer, tap inner, four k8 steps -- so every
// shape gives the same bits.
//
// Replaces rten-gemm/src/im2col.rs:110-212 (the A-operand gather of the packed GEMM) for these layers.
#include <cuda.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>

#include "math.cuh"
#include "ptx.cuh"
#include "umma_gemm.h"

namespace rtb {

namespace {

constexpr int HALO_THREADS = 384;      // warpgroup 0: TMA producer; warpgroups 1, 2: MMA + epilogue
constexpr int HB_MAX = 8;              // weight ring stages
constexpr int HALO_STG_BYTES = 128 * 128;  // one consumer's output staging: up to 128 slots x 32 columns
// alignment, barriers + bias, the two consumers' staging buffers: everything but the patches and the weight ring
constexpr int HALO_FIXED_BYTES = 1024 + 2048 + 2 * HALO_STG_BYTES;
constexpr int HALO_SMEM_MAX = 227 * 1024;

struct HaloParams {
    // geometry
    int B, OH, OW, N, C;
    int kh, kw, pt, pl;
    int P;         // slot pitch of a patch row = OW + kw - 1
    int R;         // output rows per unit
    int tb;        // images per unit
    int nr;        // patch rows per image = R + kh - 1
    int T;         // 128-slot tiles per unit (1 or 2)
    int bn;        // output channels per unit
    int c_blocks;  // 32-channel blocks
    int taps;
    int strips, units_n, units_total;
    int b_stages;  // weight ring depth
    uint32_t patch_bytes, patch_tx, b_bytes;
    uint32_t tap_off[32];  // (ky P + kx) * 128: byte offset of filter tap ky * kw + kx inside the patch
    uint32_t m_img, m_P;  // floor(2^32 / d) + 1 for d = nr * P and d = P: n / d == __umulhi(n, m) for the slot numbers of a unit
    EpilogueDesc epi;
};

__device__ __forceinline__ void halo_unit(const HaloParams& p, int u, int& n0, int& oy0, int& b0) {
    const int nt = u % p.units_n;
    const int rest = u / p.units_n;
    const int st = rest % p.strips;
    n0 = nt * p.bn;
    oy0 = st * p.R;
    b0 = (rest / p.strips) * p.tb;
}

template <int N>
__device__ __forceinline__ void halo_wgmma(float (&d)[N / 2], uint64_t adesc, uint64_t bdesc) {
    if constexpr (N == 128) wgmma_tf32_n128(d, adesc, bdesc);
    else wgmma_k<0, 0, N>(d, adesc, bdesc);
}

// One consumer warpgroup (w = 0, 1): H = T m64 halves of 64 slots x N columns per unit, accumulated over every
// (channel block, tap) stage, then + bias, Relu, staged in 32-column chunks (128B-swizzled slot rows) and written out as
// whole 128-byte slot rows, skipping the slots that are padding (x >= OW, rows past the strip / image, tail images).
template <int N, int H>
__device__ __forceinline__ void halo_consumer(const HaloParams& p, uint64_t* patch_full, uint64_t* patch_empty,
                                              uint64_t* b_full, uint64_t* b_empty, const uint8_t* patch0,
                                              const uint8_t* bring, uint8_t* stg, float* bias_s) {
    const int w = (threadIdx.x >> 7) - 1;
    const int t = threadIdx.x & 127;
    const int q = t >> 5, lane = threadIdx.x & 31;
    const int slot0 = 64 * H * w;                  // this warpgroup's first slot of a unit
    const int row0 = 16 * q + (lane >> 2);         // fragment rows row0, row0 + 8 of each half
    const int sw = lane >> 2;                      // row0 & 7: 128B swizzle of both rows
    const int cq = lane & 3;                       // columns 8j + 2cq + {0, 1} of every 8
    const int piece = lane & 7;                    // 16-byte piece of a slot row on the way out
    const EpilogueDesc& e = p.epi;
    const bool do_relu = e.act == 1;
    const uint32_t img_slots = (uint32_t)(p.nr * p.P);
    const uint32_t bar_id = 1 + w;
    float* outp = reinterpret_cast<float*>(e.d);
    uint32_t pphase = 0, bphase = 0;  // bit s = uses of stage s so far, mod 2
    int ps = 0, bs = 0;
    for (int u = blockIdx.x; u < p.units_total; u += gridDim.x) {
        int n0, oy0, b0;
        halo_unit(p, u, n0, oy0, b0);
        // the unit's bias (zeros without one: x + 0 keeps the -0 -> +0 of the other epilogues); every reader of the
        // previous unit's values is past that unit's last chunk barrier, the first chunk barrier publishes these
        if (t < N) bias_s[t] = (e.bias_kind == 1 && n0 + t < p.N) ? __ldg(e.bias + n0 + t) : 0.0f;
        float d[H][N / 2];
#pragma unroll
        for (int h = 0; h < H; h++)
#pragma unroll
            for (int i = 0; i < N / 2; i++) d[h][i] = 0.0f;
        // (channel block, tap) pairs as one flat loop: the wgmma issue stays in straight-line code.  One group stays in
        // flight across stages: the previous stage's weights (and, after a channel block's last tap, its patch) go back
        // once the group after it has been issued and it has retired.
        const int steps = p.c_blocks * p.taps;
        int prev_b = -1, prev_p = -1;
        for (int i = 0, tap = 0; i < steps; i++) {
            if (tap == 0) mbar_wait(&patch_full[ps], (pphase >> ps) & 1);
            mbar_wait(&b_full[bs], (bphase >> bs) & 1);
#pragma unroll
            for (int h = 0; h < H; h++) wgmma_fence_operand(d[h]);
            wgmma_fence();
            // the tap is the SAME patch seen (ky P + kx) pixel slots of 128 bytes further on
            const uint32_t sa = smem_u32(patch0 + (size_t)ps * p.patch_bytes) + p.tap_off[tap] + slot0 * 128;
            const uint64_t bdesc = make_kmajor_sw128_desc(smem_u32(bring + (size_t)bs * p.b_bytes));
#pragma unroll
            for (int k = 0; k < 4; k++)
#pragma unroll
                for (int h = 0; h < H; h++) halo_wgmma<N>(d[h], make_kmajor_sw128_desc(sa + h * 64 * 128) + 2 * k, bdesc + 2 * k);
            wgmma_commit();
#pragma unroll
            for (int h = 0; h < H; h++) wgmma_fence_operand(d[h]);
            wgmma_wait<1>();
            if (lane == 0) {
                if (prev_b >= 0) mbar_arrive(&b_empty[prev_b]);
                if (prev_p >= 0) mbar_arrive(&patch_empty[prev_p]);
            }
            prev_b = bs;
            prev_p = -1;
            bphase ^= 1u << bs;
            if (++bs == p.b_stages) bs = 0;
            if (++tap == p.taps) {
                tap = 0;
                prev_p = ps;
                pphase ^= 1u << ps;
                ps ^= 1;
            }
        }
        wgmma_wait<0>();
#pragma unroll
        for (int h = 0; h < H; h++) wgmma_fence_operand(d[h]);
        if (lane == 0) {
            mbar_arrive(&b_empty[prev_b]);
            mbar_arrive(&patch_empty[prev_p]);  // (the last stage of a unit closes a channel block)
        }
        // the slot rows this thread writes out per chunk: row i * 16 + q * 4 + lane / 8 of this warpgroup's 64 H
        long long off[4 * H];
        unsigned valid = 0;
#pragma unroll
        for (int i = 0; i < 4 * H; i++) {
            const uint32_t slot = (uint32_t)(slot0 + i * 16 + q * 4 + (lane >> 3));
            const uint32_t img = __umulhi(slot, p.m_img);
            const uint32_t rem = slot - img * img_slots;
            const uint32_t yy = __umulhi(rem, p.m_P);
            const uint32_t ox = rem - yy * (uint32_t)p.P;
            const int oy = oy0 + (int)yy, b = b0 + (int)img;
            if ((int)img < p.tb && b < p.B && (int)yy < p.R && oy < p.OH && (int)ox < p.OW) valid |= 1u << i;
            off[i] = (long long)b * e.s_z0 + (long long)oy * e.s_row + (long long)ox * e.s_z1 + n0 + piece * 4;
        }
#pragma unroll
        for (int k = 0; k < N / 32; k++) {
            // every thread of the warpgroup has read the previous chunk out of the staging buffer (for the first chunk of
            // a unit: the bias values are in place)
            asm volatile("bar.sync %0, 128;" ::"r"(bar_id) : "memory");
#pragma unroll
            for (int h = 0; h < H; h++)
#pragma unroll
                for (int j = 0; j < 4; j++) {  // columns 32k + 8j + 2cq + {0, 1}, rows 64h + row0 + 8r
                    const float2 bb = *reinterpret_cast<const float2*>(bias_s + 32 * k + 8 * j + 2 * cq);
#pragma unroll
                    for (int r = 0; r < 2; r++) {
                        const int i0 = 16 * k + 4 * j + 2 * r;
                        uint32_t v0 = __float_as_uint(d[h][i0]), v1 = __float_as_uint(d[h][i0 + 1]);
                        add_f32x2(v0, v1, bb.x, bb.y);
                        if (do_relu) {
                            v0 = __float_as_uint(fmaxf(__uint_as_float(v0), 0.0f));
                            v1 = __float_as_uint(fmaxf(__uint_as_float(v1), 0.0f));
                        }
                        uint8_t* px = stg + (64 * h + row0 + 8 * r) * 128 + (((2 * j + (cq >> 1)) ^ sw) << 4) + 8 * (cq & 1);
                        *reinterpret_cast<uint2*>(px) = make_uint2(v0, v1);
                    }
                }
            asm volatile("bar.sync %0, 128;" ::"r"(bar_id) : "memory");
#pragma unroll
            for (int i = 0; i < 4 * H; i++) {
                const int sl = i * 16 + q * 4 + (lane >> 3);  // staging row
                const uint4 v = *reinterpret_cast<const uint4*>(stg + sl * 128 + ((piece ^ (sl & 7)) << 4));
                if (valid & (1u << i)) *reinterpret_cast<uint4*>(outp + off[i] + 32 * k) = v;
            }
        }
    }
}

template <int N, int H>
__global__ void __launch_bounds__(HALO_THREADS, 1)
umma_halo_kernel(const __grid_constant__ CUtensorMap tma_a, const __grid_constant__ CUtensorMap tma_b, const __grid_constant__ HaloParams p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* patch_full = reinterpret_cast<uint64_t*>(base);  // [2]
    uint64_t* patch_empty = patch_full + 2;
    uint64_t* b_full = patch_empty + 2;                         // [HB_MAX]
    uint64_t* b_empty = b_full + HB_MAX;
    float* bias_s = reinterpret_cast<float*>(base + 1024);  // [consumer][128]: column bias of the current unit
    uint8_t* stage0 = base + 2048;                          // [consumer] 128 slots x 128 B output staging (128B-swizzled)
    uint8_t* patch0 = stage0 + 2 * HALO_STG_BYTES;
    uint8_t* bring = patch0 + 2 * (size_t)p.patch_bytes;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tma_a);
        tma_prefetch_desc(&tma_b);
    }
    if (warp == 1) {
        if (lane < 2) {
            mbar_init(&patch_full[lane], 1);
            mbar_init(&patch_empty[lane], 8);  // one arrival per consumer warp
        }
        if (lane < HB_MAX) {
            mbar_init(&b_full[lane], 1);
            mbar_init(&b_empty[lane], 8);
        }
        fence_mbar_init();
    }
    __syncthreads();
    pdl_wait();
    pdl_launch_dependents();

    if (warp < 4) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 56;");
        if (warp != 0) return;
        // ===================== TMA producer: runs warp-uniformly, one elected lane issues =====================
        uint32_t pphase = 0, bphase = 0;  // bit s = uses of stage s so far, mod 2
        int ps = 0, bs = 0;
        for (int u = blockIdx.x; u < p.units_total; u += gridDim.x) {
            int n0, oy0, b0;
            halo_unit(p, u, n0, oy0, b0);
            for (int cb = 0; cb < p.c_blocks; cb++) {
                mbar_wait(&patch_empty[ps], ((pphase >> ps) & 1) ^ 1);
                if (elect_one()) {
                    mbar_expect_tx(&patch_full[ps], p.patch_tx);
                    tma_load_4d(patch0 + (size_t)ps * p.patch_bytes, &tma_a, &patch_full[ps], cb * 32, -p.pl, oy0 - p.pt, b0);
                }
                __syncwarp();
                pphase ^= 1u << ps;
                ps ^= 1;
                for (int tap = 0; tap < p.taps; tap++) {
                    mbar_wait(&b_empty[bs], ((bphase >> bs) & 1) ^ 1);
                    if (elect_one()) {
                        mbar_expect_tx(&b_full[bs], p.b_bytes);
                        tma_load_4d(bring + (size_t)bs * p.b_bytes, &tma_b, &b_full[bs], cb * 32, n0, tap, 0);
                    }
                    __syncwarp();
                    bphase ^= 1u << bs;
                    if (++bs == p.b_stages) bs = 0;
                }
            }
        }
    } else {
        asm volatile("setmaxnreg.inc.sync.aligned.u32 224;");
        const int w = (warp >> 2) - 1;
        halo_consumer<N, H>(p, patch_full, patch_empty, b_full, b_empty, patch0, bring, stage0 + w * HALO_STG_BYTES,
                            bias_s + w * 128);
    }
}

}  // namespace

// force_bn / force_T > 0: that unit shape or RTEN_ERR_UNSUPPORTED_VALUE (the autotuner times a few of them against the
// generic kernel's plans and records the winner); 0: the cost model's choice, and only with RTEN_B200_HALO=1 -- without
// measurements the generic kernel stays the default (which of the two is faster depends on the layer).
rten_status launch_umma_halo_conv(rten_ctx* ctx, const GemmLaunch& L, int force_bn, int force_T) {
    if (getenv("RTEN_B200_NO_HALO")) return RTEN_ERR_UNSUPPORTED_VALUE;
    if (!force_bn) {
        const char* on = getenv("RTEN_B200_HALO");
        if (!on || atoi(on) == 0) return RTEN_ERR_UNSUPPORTED_VALUE;
    }
    if (!L.conv || L.kind != 0) return RTEN_ERR_UNSUPPORTED_VALUE;
    const ConvGeom& g = L.g;
    const EpilogueDesc& e = L.epi;
    if (g.sy != 1 || g.sx != 1 || g.dy != 1 || g.dx != 1 || g.kh * g.kw < 2 || g.kh * g.kw > 32) return RTEN_ERR_UNSUPPORTED_VALUE;
    if (g.C % 32 || g.C < 32) return RTEN_ERR_UNSUPPORTED_VALUE;
    if (L.N % 32 || L.N < 32) return RTEN_ERR_UNSUPPORTED_VALUE;
    if (e.r || e.range || e.bias_kind == 2 || e.act > 1 || e.s_col != 1 || e.d_is_i32 || e.alpha != 1.0f) return RTEN_ERR_UNSUPPORTED_VALUE;
    auto al16 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
    if (!al16(e.d) || (e.s_z0 & 3) || (e.s_row & 3) || (e.s_z1 & 3) || (e.bias_kind == 1 && !al16(e.bias))) return RTEN_ERR_UNSUPPORTED_VALUE;
    if (!tma_compatible(L.a, 4, 4) || !tma_compatible(L.b, 4, 4)) return RTEN_ERR_UNSUPPORTED_VALUE;
    HaloParams p;
    memset(&p, 0, sizeof(p));
    p.B = g.B;
    p.OH = g.OH;
    p.OW = g.OW;
    p.N = L.N;
    p.C = g.C;
    p.kh = g.kh;
    p.kw = g.kw;
    p.pt = g.pt;
    p.pl = g.pl;
    p.P = g.OW + g.kw - 1;
    p.c_blocks = g.C / 32;
    p.taps = g.kh * g.kw;
    p.epi = e;
    if (p.P > 256) return RTEN_ERR_UNSUPPORTED_VALUE;
    // ---- unit shape.  Candidates: output-channel tile bn, 128-slot tiles T per unit (T = 1: one m64 half per consumer,
    // bn <= 64; T = 2: two halves per consumer), whole images (tb >= 1 images of OH + kh - 1 patch rows) or row strips
    // (R rows of one image).  Ranked by waves x (clocks of a unit), with the slots that are thrown away counted in.
    const int num_sms = ctx->num_sms;
    double best = 1e30;
    int bbn = 0, bT = 0, bR = 0, btb = 0;
    const char* fbn = getenv("RTEN_B200_HALO_BN");
    const char* fT = getenv("RTEN_B200_HALO_T");
    const int want_bn = force_bn ? force_bn : (fbn ? atoi(fbn) : 0), want_T = force_T ? force_T : (fT ? atoi(fT) : 0);
    for (int bn = 32; bn <= std::min(L.N, 128); bn *= 2) {
        if (L.N % bn) continue;
        if (want_bn && bn != want_bn) continue;
        for (int T = 1; T <= 2; T++) {
            if (want_T && T != want_T) continue;
            if (T == 1 && bn > 64) continue;  // (a 64-slot half per consumer: the wide columns go to T = 2)
            // whole-image mode when tb >= 1 padded images fit T tiles, else strips of R rows
            const int img_slots = (g.OH + g.kh - 1) * p.P;
            int tb = 1, R = 0;
            if (g.OH * p.P <= T * 128) {
                R = g.OH;
                tb = 1 + (T * 128 - g.OH * p.P) / img_slots;
                tb = std::min(tb, g.B);
            } else {
                R = (T * 128) / p.P;
                if (R < 1) continue;
            }
            const int nr = R + g.kh - 1;
            if (nr > 256 || tb > 256) continue;
            const long long alloc_slots = (long long)T * 128 + (g.kh - 1) * p.P + g.kw - 1;
            const long long loaded_slots = (long long)tb * nr * p.P;
            const long long patch_bytes = (std::max(alloc_slots, loaded_slots) * 128 + 1023) / 1024 * 1024;
            // a weight stage must be requested ~1500 clk (TMA latency + its own transfer) before its MMAs start: at least
            // three stages in flight beside the two patches
            const long long budget = HALO_SMEM_MAX - HALO_FIXED_BYTES - 2 * patch_bytes;
            if ((long long)bn * 128 * 3 > budget) continue;
            const long long strips = (g.OH + R - 1) / R;
            const long long units = strips * ((g.B + tb - 1) / tb) * (L.N / bn);
            const double waves = std::ceil((double)units / num_sms);
            // per unit: MMA clocks (c_blocks x taps stages of 2 T m64 instructions x 4 k8 steps, bn / 2 clocks each, plus a
            // fixed cost per stage) vs the operand bytes entering the SM, then the epilogue (bn columns of 128 T slots
            // through the staging buffers).  The clock and bandwidth constants are unmeasured estimates that only rank the
            // candidate shapes.
            const double mma = (double)p.c_blocks * p.taps * (8.0 * T * std::max(16.0, bn / 2.0) + 60.0);
            const double bytes = (double)p.c_blocks * (loaded_slots * 128.0 + (double)p.taps * bn * 128.0);
            const double ingest = bytes / 55.0;
            const double epi = (double)T * 128 * bn * 4 / 16.0;
            const double unit = std::max(mma, ingest) + epi + 800.0;
            const double cost = waves * unit + 4000.0;
            if (cost < best) {
                best = cost;
                bbn = bn;
                bT = T;
                bR = R;
                btb = tb;
            }
        }
    }
    if (!bbn) return RTEN_ERR_UNSUPPORTED_VALUE;
    p.bn = bbn;
    p.T = bT;
    p.R = bR;
    p.tb = btb;
    p.nr = p.R + g.kh - 1;
    p.strips = (g.OH + p.R - 1) / p.R;
    p.units_n = L.N / p.bn;
    p.units_total = p.strips * ((g.B + p.tb - 1) / p.tb) * p.units_n;
    const long long alloc_slots = (long long)p.T * 128 + (g.kh - 1) * p.P + g.kw - 1;
    const long long loaded_slots = (long long)p.tb * p.nr * p.P;
    p.patch_bytes = (uint32_t)((std::max(alloc_slots, loaded_slots) * 128 + 1023) / 1024 * 1024);
    p.patch_tx = (uint32_t)(loaded_slots * 128);
    p.b_bytes = (uint32_t)p.bn * 128u;
    p.b_stages = (int)std::min<long long>(HB_MAX, (HALO_SMEM_MAX - HALO_FIXED_BYTES - 2LL * p.patch_bytes) / p.b_bytes);
    for (int ky = 0; ky < g.kh; ky++)
        for (int kx = 0; kx < g.kw; kx++) p.tap_off[ky * g.kw + kx] = (uint32_t)((ky * p.P + kx) * 128);
    p.m_img = (uint32_t)(0x100000000ull / (unsigned long long)(p.nr * p.P)) + 1u;
    p.m_P = (uint32_t)(0x100000000ull / (unsigned long long)p.P) + 1u;

    uint32_t abox[4] = {32u, (uint32_t)p.P, (uint32_t)p.nr, (uint32_t)p.tb}, ones[4] = {1, 1, 1, 1};
    uint32_t bbox[4] = {32u, (uint32_t)p.bn, 1u, 1u};
    CUtensorMap map_a, map_b;
    if (!encode_map(ctx, &map_a, L.a, 4, true, abox, ones)) return RTEN_ERR_UNSUPPORTED_VALUE;
    if (!encode_map(ctx, &map_b, L.b, 4, true, bbox, ones)) return RTEN_ERR_UNSUPPORTED_VALUE;
    if (getenv("RTEN_B200_VERBOSE"))
        fprintf(stderr, "[umma_halo] B=%d %dx%d C=%d N=%d k=%dx%d: bn=%d T=%d R=%d tb=%d P=%d units=%d b_stages=%d patch=%u B\n", g.B,
                g.OH, g.OW, g.C, L.N, g.kh, g.kw, p.bn, p.T, p.R, p.tb, p.P, p.units_total, p.b_stages, p.patch_bytes);
    const size_t smem = HALO_FIXED_BYTES + 2 * (size_t)p.patch_bytes + (size_t)p.b_stages * p.b_bytes;
    auto kern = p.T == 1 ? (p.bn == 32 ? umma_halo_kernel<32, 1> : umma_halo_kernel<64, 1>)
                         : (p.bn == 32 ? umma_halo_kernel<32, 2> : p.bn == 64 ? umma_halo_kernel<64, 2> : umma_halo_kernel<128, 2>);
    return launch(ctx, "umma_halo launch", kern, {std::min(p.units_total, num_sms), HALO_THREADS, smem, HALO_SMEM_MAX, true},
                  map_a, map_b, p);
}

}  // namespace rtb
