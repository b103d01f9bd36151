// Recurrent kernels of GRU and LSTM (src/ops/rnn.rs gru / lstm); see rnn.h.
//
// Gate arithmetic, per element and in the reference's order (every operation rounded on its own, no contraction):
//   GRU : gx = xW (+ Wb), s = hR (+ Rb); z = sig(gx_z + s_z), r = sig(gx_r + s_r); h~ = tanh(gx_h + s_h * r);
//         h = (1 - z) * h~ + z * h
//   LSTM: g = ((xW (+ Wb)) + hR) (+ Rb); i, o, f = sig(g); c~ = tanh(g_c); c = f * c + i * c~; h = o * tanhf(c)
// sig(x) = 1 / (1 + exp(0 - x)) and tanh are rten-vecmath's recipes (math.cuh); the LSTM's last tanh is CUDA's tanhf
// where the reference calls f32::tanh.  tanhf is not correctly rounded: CUDA documents 2 ulp, and over 10^7 float32
// inputs in [-10, 10] about 3.5% of its results differ from the correctly rounded tanh, by at most 1.79 ulp (measured
// by tests/test_gpu_rnn_kernels.py on an H100).  The recurrent product hR is f32 FMA arithmetic in both f32 modes on
// the cluster kernel (one chain per output over k in ascending order) and on the per-step path's skinny kernel
// (B <= 32); the per-step path's wgmma GEMM (B > 32) computes it in 3xTF32 in both modes (api_rnn.cu).
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>
#include <cstdlib>

#include "math.cuh"
#include "rnn.h"

namespace rtb {

namespace {

constexpr int RNN_THREADS = 256;
constexpr int RNN_MAX_SMEM = 227 * 1024;  // sm_90 opt-in shared memory per block

// Inputs of one (direction, batch row, hidden unit) update.  xg: x . W^T of the G gates; rec: h . R^T of the G gates.
template <bool GRU>
__device__ __forceinline__ void gate_update(const RnnLaunch& L, int d, int j, const float* xg, const float* rec, float& h,
                                           float& c) {
    constexpr int G = GRU ? 3 : 4;
    const int GH = G * L.H;
    const float* wb = L.bias ? L.bias + d * L.b_d : nullptr;
    if (GRU) {
        float gx[3], s[3];
#pragma unroll
        for (int g = 0; g < 3; g++) {
            gx[g] = wb ? __fadd_rn(xg[g], wb[(long long)(g * L.H + j) * L.b_k]) : xg[g];
            s[g] = wb ? __fadd_rn(rec[g], wb[(long long)(GH + g * L.H + j) * L.b_k]) : rec[g];
        }
        const float z = sigmoid_ref(__fadd_rn(gx[0], s[0]));
        const float r = sigmoid_ref(__fadd_rn(gx[1], s[1]));
        const float ht = tanh_ref(__fadd_rn(gx[2], __fmul_rn(s[2], r)));
        h = __fadd_rn(__fmul_rn(__fsub_rn(1.0f, z), ht), __fmul_rn(z, h));
    } else {
        float g4[4];
#pragma unroll
        for (int g = 0; g < 4; g++) {
            float v = wb ? __fadd_rn(xg[g], wb[(long long)(g * L.H + j) * L.b_k]) : xg[g];
            v = __fadd_rn(v, rec[g]);
            g4[g] = wb ? __fadd_rn(v, wb[(long long)(GH + g * L.H + j) * L.b_k]) : v;
        }
        const float i = sigmoid_ref(g4[0]), o = sigmoid_ref(g4[1]), f = sigmoid_ref(g4[2]);
        const float cc = tanh_ref(g4[3]);
        c = __fadd_rn(__fmul_rn(f, c), __fmul_rn(i, cc));
        h = __fmul_rn(o, tanhf(c));
    }
}

__device__ __forceinline__ int step_time(const RnnLaunch& L, int d, int s) {
    const bool rev = (d == 0 && L.reverse) || d == 1;
    return rev ? L.T - 1 - s : s;
}

// ---------------------------------------------------------------------------------------------------------------------
// Cluster kernel
// ---------------------------------------------------------------------------------------------------------------------
// Grid: dirs * slices clusters of C CTAs (cluster id = blockIdx.x / C).  CTA `rank` owns hidden units
// [rank * Hc, (rank + 1) * Hc) of its direction, i.e. the G * Hc rows g * H + j of R, and the batch rows
// [slice * Bs, slice * Bs + bn).  Shared memory:
//   Rs  [G * Hc][RS]      its rows of R, zero-padded to Hp = round_up(H, 4) columns; RS = Hp (+ 4) with RS / 4 odd, so
//                         the float4 loads of 8 consecutive rows hit distinct bank groups
//   hb  [2][Bsp][Hp]      h_{t-1} of every unit (double-buffered: step t reads hb[t & 1], peers write hb[(t + 1) & 1])
//   pre [G * Hc][Bsp]     h . R^T of its rows for the current step
// One step: (1) each thread owning a (unit, batch row) pair loads its G input projections; (2) the products, each a
// serial f32 FMA chain; (3) the owning threads apply the gate arithmetic, write Y and store h_t into hb of every CTA
// of the cluster (st.shared::cluster); (4) one barrier.cluster arrive.release / wait.acquire.  c_t stays in the owning
// thread's register.  Clusters never wait on each other.
struct ClusterPlan {
    int C = 0, Hc = 0, Bs = 0, BT = 0, Bsp = 0, Hp = 0, RS = 0, slices = 0;
    size_t smem = 0;
};

struct ClusterParams {
    RnnLaunch L;
    int C, Hc, Bs, Bsp, Hp, RS, slices;
};

__device__ __forceinline__ uint32_t smem_addr(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void st_cluster(uint32_t local, uint32_t rank, float v) {
    uint32_t remote;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(local), "r"(rank));
    asm volatile("st.shared::cluster.f32 [%0], %1;" ::"r"(remote), "f"(v) : "memory");
}

__device__ __forceinline__ void cluster_sync() {
    asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
    asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}

template <bool GRU, int BT>
__global__ void __launch_bounds__(RNN_THREADS, 1) rnn_cluster_kernel(const __grid_constant__ ClusterParams p) {
    constexpr int G = GRU ? 3 : 4;
    const RnnLaunch& L = p.L;
    extern __shared__ __align__(16) float sm[];
    const int rows = G * p.Hc;
    float* Rs = sm;
    float* hb = Rs + (size_t)rows * p.RS;
    float* pre = hb + (size_t)2 * p.Bsp * p.Hp;

    uint32_t rank;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(rank));
    const int cid = blockIdx.x / p.C;
    const int d = cid / p.slices;
    const int b0 = (cid % p.slices) * p.Bs;
    const int bn = min(p.Bs, L.B - b0);
    const int j0 = (int)rank * p.Hc;
    const int tid = threadIdx.x;

    // ---- R rows, h_0, zero padding
    const float* Rd = L.r + d * L.r_d;
    for (int e = tid; e < rows * p.RS; e += RNN_THREADS) {
        const int row = e / p.RS, k = e % p.RS;
        const int g = row / p.Hc, j = j0 + row % p.Hc;
        Rs[e] = (k < L.H && j < L.H) ? Rd[(long long)(g * L.H + j) * L.r_row + (long long)k * L.r_k] : 0.0f;
    }
    for (int e = tid; e < 2 * p.Bsp * p.Hp; e += RNN_THREADS) {
        const int buf = e / (p.Bsp * p.Hp), b = e / p.Hp % p.Bsp, k = e % p.Hp;
        float v = 0.0f;
        if (buf == 0 && b < bn && k < L.H && L.h0) v = L.h0[d * L.h0_d + (long long)(b0 + b) * L.h0_b + (long long)k * L.h0_k];
        hb[e] = v;
    }
    // the (unit, batch row) pair this thread updates, if any
    const int jl = tid % p.Hc, bb = tid / p.Hc;
    const int j = j0 + jl;
    const bool owner = bb < bn && j < L.H;
    float h = 0.0f, c = 0.0f;
    if (owner) {
        if (L.h0) h = L.h0[d * L.h0_d + (long long)(b0 + bb) * L.h0_b + (long long)j * L.h0_k];
        if (!GRU && L.c0) c = L.c0[d * L.c0_d + (long long)(b0 + bb) * L.c0_b + (long long)j * L.c0_k];
    }
    const long long xrow = (long long)L.dirs * G * L.H;
    const float* xcol = L.xp + (long long)d * G * L.H + j;
    const uint32_t hb_own = smem_addr(hb + bb * p.Hp + j);
    // every CTA of the cluster has initialised its buffers before any peer writes into them
    cluster_sync();

    const int Hp4 = p.Hp / 4, RS4 = p.RS / 4;
    const int items = rows * (p.Bsp / BT);
    for (int s = 0; s < L.T; s++) {
        const int t = step_time(L, d, s);
        const int cur = s & 1;
        float xg[G];
        if (owner) {
            const float* xr = xcol + ((long long)t * L.B + b0 + bb) * xrow;
#pragma unroll
            for (int g = 0; g < G; g++) xg[g] = xr[(long long)g * L.H];
        }
        // ---- h_{t-1} . R^T of this CTA's rows
        const float4* R4 = reinterpret_cast<const float4*>(Rs);
        const float4* h4 = reinterpret_cast<const float4*>(hb + (size_t)cur * p.Bsp * p.Hp);
        for (int it = tid; it < items; it += RNN_THREADS) {
            const int row = it % rows, bg = it / rows;
            float acc[BT];
#pragma unroll
            for (int q = 0; q < BT; q++) acc[q] = 0.0f;
            const float4* rp = R4 + (size_t)row * RS4;
            const float4* hp = h4 + (size_t)bg * BT * Hp4;
            for (int k4 = 0; k4 < Hp4; k4++) {
                const float4 rv = rp[k4];
#pragma unroll
                for (int q = 0; q < BT; q++) {
                    const float4 hv = hp[q * Hp4 + k4];
                    acc[q] = __fmaf_rn(rv.x, hv.x, acc[q]);
                    acc[q] = __fmaf_rn(rv.y, hv.y, acc[q]);
                    acc[q] = __fmaf_rn(rv.z, hv.z, acc[q]);
                    acc[q] = __fmaf_rn(rv.w, hv.w, acc[q]);
                }
            }
#pragma unroll
            for (int q = 0; q < BT; q++) pre[row * p.Bsp + bg * BT + q] = acc[q];
        }
        __syncthreads();
        // ---- gates, outputs, h_t to every CTA of the cluster
        if (owner) {
            float rec[G];
#pragma unroll
            for (int g = 0; g < G; g++) rec[g] = pre[(g * p.Hc + jl) * p.Bsp + bb];
            gate_update<GRU>(L, d, j, xg, rec, h, c);
            if (L.y) L.y[t * L.y_t + d * L.y_d + (long long)(b0 + bb) * L.y_b + (long long)j * L.y_k] = h;
            const uint32_t dst = hb_own + (uint32_t)((cur ^ 1) * p.Bsp * p.Hp * 4);
            for (int q = 0; q < p.C; q++) st_cluster(dst, (uint32_t)q, h);
        }
        cluster_sync();
    }
    if (owner) {
        if (L.yh) L.yh[d * L.yh_d + (long long)(b0 + bb) * L.yh_b + (long long)j * L.yh_k] = h;
        if (!GRU && L.yc) L.yc[d * L.yc_d + (long long)(b0 + bb) * L.yc_b + (long long)j * L.yc_k] = c;
    }
}

size_t cluster_smem(int G, int C, int H, int Bsp, int* Hc, int* Hp, int* RS) {
    *Hc = (H + C - 1) / C;
    *Hp = (H + 3) / 4 * 4;
    int rs4 = *Hp / 4;
    if (rs4 % 2 == 0) rs4++;
    *RS = rs4 * 4;
    return 4 * ((size_t)G * *Hc * *RS + (size_t)2 * Bsp * *Hp + (size_t)G * *Hc * Bsp);
}

int batch_tile(int Bs) { return Bs >= 8 ? 8 : Bs >= 4 ? 4 : Bs >= 2 ? 2 : 1; }

// The smallest cluster whose shared memory holds its rows of R (with one batch row), then the batch slice: enough
// slices to give every SM a CTA, no more rows than shared memory or the gate threads (Hc * Bs <= threads) allow.
bool plan_cluster(int num_sms, int gru, int H, int B, int dirs, int min_C, ClusterPlan* out) {
    const int G = gru ? 3 : 4;
    if (H < 1 || B < 1) return false;
    for (int C = min_C; C <= 16; C *= 2) {
        ClusterPlan P;
        P.C = C;
        if (cluster_smem(G, C, H, 1, &P.Hc, &P.Hp, &P.RS) > (size_t)RNN_MAX_SMEM || P.Hc > RNN_THREADS) continue;
        const int want_slices = std::max(1, num_sms / C / dirs);
        int Bs = std::max(1, (B + want_slices - 1) / want_slices);
        Bs = std::min(Bs, RNN_THREADS / P.Hc);
        for (; Bs > 1; Bs--) {
            const int bt = batch_tile(Bs), bsp = (Bs + bt - 1) / bt * bt;
            if (cluster_smem(G, C, H, bsp, &P.Hc, &P.Hp, &P.RS) <= (size_t)RNN_MAX_SMEM) break;
        }
        P.Bs = Bs;
        P.BT = batch_tile(Bs);
        P.Bsp = (Bs + P.BT - 1) / P.BT * P.BT;
        P.slices = (B + Bs - 1) / Bs;
        P.smem = cluster_smem(G, C, H, P.Bsp, &P.Hc, &P.Hp, &P.RS);
        *out = P;
        return true;
    }
    return false;
}

template <bool GRU, int BT>
rten_status launch_cluster_t(rten_ctx* ctx, const ClusterPlan& P, const ClusterParams& p, bool* unschedulable) {
    auto kern = rnn_cluster_kernel<GRU, BT>;
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)P.smem);
    if (e == cudaSuccess && P.C > 8) e = cudaFuncSetAttribute(kern, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
    if (e != cudaSuccess) return fail_cuda(ctx, e, "rnn_cluster_kernel attributes");
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)(P.C * p.L.dirs * P.slices), 1, 1);
    cfg.blockDim = dim3(RNN_THREADS, 1, 1);
    cfg.dynamicSmemBytes = P.smem;
    cfg.stream = ctx->stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = (unsigned)P.C;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    // not launch(): the occupancy query must see this exact cluster config, and its failure means "use the per-step path"
    int active = 0;
    e = cudaOccupancyMaxActiveClusters(&active, kern, &cfg);
    if (e != cudaSuccess || active < 1) {
        cudaGetLastError();
        *unschedulable = true;
        return RTEN_ERR_UNSUPPORTED_VALUE;
    }
    e = cudaLaunchKernelEx(&cfg, kern, p);
    if (e != cudaSuccess) return fail_cuda(ctx, e, "rnn_cluster_kernel launch");
    count_launch(ctx);
    return RTEN_OK;
}

template <bool GRU>
rten_status launch_cluster_g(rten_ctx* ctx, const ClusterPlan& P, const ClusterParams& p, bool* unschedulable) {
    switch (P.BT) {
        case 8: return launch_cluster_t<GRU, 8>(ctx, P, p, unschedulable);
        case 4: return launch_cluster_t<GRU, 4>(ctx, P, p, unschedulable);
        case 2: return launch_cluster_t<GRU, 2>(ctx, P, p, unschedulable);
        default: return launch_cluster_t<GRU, 1>(ctx, P, p, unschedulable);
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// Per-step path
// ---------------------------------------------------------------------------------------------------------------------
__global__ void rnn_state_init_kernel(const __grid_constant__ RnnLaunch L, float* h, float* c, int ld) {
    const long long n = (long long)L.dirs * L.B * L.H;
    for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
        const int k = (int)(e % L.H), b = (int)(e / L.H % L.B), d = (int)(e / ((long long)L.H * L.B));
        const float hv = L.h0 ? L.h0[d * L.h0_d + b * L.h0_b + k * L.h0_k] : 0.0f;
        const float cv = L.c0 ? L.c0[d * L.c0_d + b * L.c0_b + k * L.c0_k] : 0.0f;
        const long long o = ((long long)d * L.B + b) * ld + k;
        if (h) h[o] = hv;
        if (c) c[o] = cv;
        if (L.T == 0) {
            if (L.yh) L.yh[d * L.yh_d + b * L.yh_b + k * L.yh_k] = hv;
            if (!L.gru && L.yc) L.yc[d * L.yc_d + b * L.yc_b + k * L.yc_k] = cv;
        }
    }
}

template <bool GRU>
__global__ void rnn_step_gates_kernel(const __grid_constant__ RnnLaunch L, int s, const float* rec, float* hs, float* cs,
                                      int ld) {
    constexpr int G = GRU ? 3 : 4;
    const long long n = (long long)L.dirs * L.B * L.H;
    const long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (e >= n) return;
    const int j = (int)(e % L.H), b = (int)(e / L.H % L.B), d = (int)(e / ((long long)L.H * L.B));
    const int t = step_time(L, d, s);
    const float* xr = L.xp + ((long long)t * L.B + b) * L.dirs * G * L.H + (long long)d * G * L.H + j;
    const float* rr = rec + ((long long)d * L.B + b) * G * L.H + j;
    float xg[G], rv[G];
#pragma unroll
    for (int g = 0; g < G; g++) {
        xg[g] = xr[(long long)g * L.H];
        rv[g] = rr[(long long)g * L.H];
    }
    const long long o = ((long long)d * L.B + b) * ld + j;
    float h = hs[o], c = GRU ? 0.0f : cs[o];
    gate_update<GRU>(L, d, j, xg, rv, h, c);
    hs[o] = h;
    if (!GRU) cs[o] = c;
    if (L.y) L.y[t * L.y_t + d * L.y_d + b * L.y_b + j * L.y_k] = h;
    if (s == L.T - 1) {
        if (L.yh) L.yh[d * L.yh_d + b * L.yh_b + j * L.yh_k] = h;
        if (!GRU && L.yc) L.yc[d * L.yc_d + b * L.yc_b + j * L.yc_k] = c;
    }
}

}  // namespace

rten_status launch_rnn_cluster(rten_ctx* ctx, const RnnLaunch& L) {
    ClusterPlan P;
    int min_C = 1;
    while (plan_cluster(ctx->num_sms, L.gru, L.H, L.B, L.dirs, min_C, &P)) {
        ClusterParams p;
        p.L = L;
        p.C = P.C;
        p.Hc = P.Hc;
        p.Bs = P.Bs;
        p.Bsp = P.Bsp;
        p.Hp = P.Hp;
        p.RS = P.RS;
        p.slices = P.slices;
        bool unschedulable = false;
        const rten_status st = L.gru ? launch_cluster_g<true>(ctx, P, p, &unschedulable)
                                     : launch_cluster_g<false>(ctx, P, p, &unschedulable);
        if (!unschedulable) return st;
        // 16-CTA clusters need the non-portable size and may not fit the device's partitioning: no smaller cluster
        // holds these weights, so the per-step path takes over
        if (P.C >= 16) break;
        min_C = P.C * 2;
    }
    return RTEN_ERR_UNSUPPORTED_VALUE;
}

rten_status launch_rnn_state_init(rten_ctx* ctx, const RnnLaunch& L, float* h, float* c, int ld) {
    const long long n = (long long)L.dirs * L.B * L.H;
    if (n == 0) return RTEN_OK;
    const int grid = (int)std::min<long long>((n + 255) / 256, 4LL * ctx->num_sms);
    return launch(ctx, "rnn_state_init_kernel launch", rnn_state_init_kernel, {grid, 256}, L, h, c, ld);
}

rten_status launch_rnn_step_gates(rten_ctx* ctx, const RnnLaunch& L, int s, const float* rec, float* h, float* c, int ld) {
    const long long n = (long long)L.dirs * L.B * L.H;
    if (n == 0) return RTEN_OK;
    const long long grid = (n + 255) / 256;
    return launch(ctx, "rnn_step_gates_kernel launch", L.gru ? rnn_step_gates_kernel<true> : rnn_step_gates_kernel<false>,
                  {(unsigned)grid, 256}, L, s, rec, h, c, ld);
}

}  // namespace rtb
