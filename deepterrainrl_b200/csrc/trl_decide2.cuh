// deepterrainrl_b200 -- batched policy decision path (included by trl_step.cu after trl_decide.cuh; same translation unit).
//
// All decisions that became due in one env-step are served by ONE pass over the MACE network
// (data/policies/dog/nets/dog_mace3_deploy.prototxt; cNeuralNet::Eval, learning/NeuralNet.cpp:352-375,977-986,1027-1036), split where
// the arithmetic changes character:
//
//   trl_decide_conv_kernel   the three terrain convolutions: 2.4 of the net's 3.5 MFLOP per decision on 6 K weights.  Parallel over
//                            decisions (one 4-CTA cluster each, activations in shared memory / DSMEM, trl_decide.cuh's conv
//                            stage); the flattened conv2 output [32 x 187] of decision idx goes to row idx of a scratch matrix.
//   trl_decide_fc_kernel     everything behind it as GEMMs over the batch: rows = decisions (chunks of 32), weights streamed ONCE
//                            per launch instead of once per decision (4.5 MB instead of 16 x 4.5 MB from L2).  One 8-CTA cluster:
//                              terr_ip0  [32 x 5984] x [5984 x 64]   K split over the CTAs; weight and activation tiles come in
//                                        through TMA (cp.async.bulk.tensor.2d, 128-byte swizzle, mbarrier ring), partial sums
//                                        reduced over DSMEM in rank order
//                              ip0       [32 x 147]  x [147 x 256]   32 output columns per CTA (weights resident in shared memory)
//                              heads     [32 x 256]  x [256 x 512],  [32 x 128] x [128 x {3,29,29,29}]
//                            every product on mma.sync.m8n8k4.f64 (DMMA), f64 throughout like the reference's Caffe Net<double>;
//                            then the scalar decision logic of cDogControllerMACE::UpdateAction / cBaseControllerMACE::
//                            DecideActionBoltzmann for up to 32 decisions at once, one lane each.
//
// Results differ from trl_decide.cuh's single-decision pass only in summation order (<= 1e-13 relative on the net outputs;
// tests/test_gpu_decide_batches.py checks this and the batch shapes the FC stage branches on).
#pragma once
#include <cooperative_groups.h>

#include "trl_types.h"
#include "trl_fcmaps.h"

namespace trl {

constexpr int kFcCluster = 8;            // CTAs of the FC-stage cluster
constexpr int kFcThreads = 512;
constexpr int kFcRows = 32;              // decisions per chunk (GEMM rows)
constexpr int kTipIn = kConv2Out * kW2;   // 5984 = terr_ip0 fan-in
constexpr int kKT = 16;                  // k extent of a TMA tile: 16 doubles = the 128-byte swizzle span
constexpr int kNumKTiles = kTipIn / kKT;  // 374
static_assert(kNumKTiles * kKT == kTipIn, "terr_ip0 fan-in must be a whole number of TMA tiles");
// A pipeline stage carries kTilesPerStage k-tiles: the per-stage cost of the ring (full / empty barrier round trip of the whole CTA,
// tools/microbench/tma_stream.cu measures it) is paid half as often as with one tile per stage
constexpr int kTilesPerStage = 2;
constexpr int kFcStages = 4;
constexpr int kWTileBytes = kTip0Out * kKT * 8;          // 8 KB  [64 n][16 k]
constexpr int kATileBytes = kFcRows * kKT * 8;           // 4 KB  [32 m][16 k]
constexpr int kTileBytes = kWTileBytes + kATileBytes;    // 12 KB, a multiple of 1024 (swizzle atom alignment)
constexpr int kStageBytes = kTilesPerStage * kTileBytes;
constexpr int kCatStride = 148;          // doubles per row of concat0 (64 + n_char <= 147, +1 zero pad): 1184 B = 32 mod 128 -> conflict-free fragments
constexpr int kHStride = 260;            // doubles per row of the ip0 output (256 + 4): 2080 B = 32 mod 128
constexpr int kHHStride = 132;           // doubles per row of one head's hidden layer (128 + 4)
constexpr int kYStride = 96;
// shared memory map of the FC kernel (bytes)
constexpr int kFcOffPipe = 0;                                              // kFcStages x {W tile, A tile}; later H and HH
constexpr int kFcOffH = 0;                                                 //   H   [32][260]  (after terr_ip0)
constexpr int kFcOffHH = kFcOffH + kFcRows * kHStride * 8;                 //   HH  [32][132]  (one head's 128 hidden units)
constexpr int kFcPipeBytes = (kFcStages * kStageBytes > kFcOffHH + kFcRows * kHHStride * 8) ? kFcStages * kStageBytes
                                                                                           : kFcOffHH + kFcRows * kHHStride * 8;
constexpr int kFcOffPart = (kFcPipeBytes + 1023) / 1024 * 1024;           // P   [32][64] partial terr_ip0 sums of this CTA
constexpr int kFcOffCat = kFcOffPart + kFcRows * kTip0Out * 8;             // CAT [32][148]
constexpr int kFcOffWip = kFcOffCat + kFcRows * kCatStride * 8;            // ip0 weight slice [32 n][148]
constexpr int kFcOffY = kFcOffWip + 32 * kCatStride * 8;                   // Y   [32][96] (rank 0)
constexpr int kFcOffBar = kFcOffY + kFcRows * kYStride * 8;                // mbarriers: full[kFcStages], empty[kFcStages]
constexpr int kFcSmemBytes = kFcOffBar + 2 * kFcStages * 8 + 64 + 1024;    // + slack for the 1024-byte alignment of the window

// ---- the pieces of PTX the FC kernel needs; the test-only emulator build (g++) gets plain-C++ stand-ins with the same data layout
__device__ __forceinline__ void dmma_8x8x4(double& c0, double& c1, double a, double b) {
#ifndef TRL_SIMT_EMU
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
#else
    // lane (g = lane / 4, t = lane % 4) holds A[g][t], B[t][g] and C[g][2t], C[g][2t + 1]
    const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    double s0 = c0, s1 = c1;
    for (int k = 0; k < 4; ++k) {
        const double ak = __shfl_sync(0xffffffffu, a, g * 4 + k);
        const double b0 = __shfl_sync(0xffffffffu, b, (2 * t) * 4 + k), b1 = __shfl_sync(0xffffffffu, b, (2 * t + 1) * 4 + k);
        s0 += ak * b0; s1 += ak * b1;
    }
    c0 = s0; c1 = s1;
#endif
}
// element (row, k) of a [rows][16] f64 tile written by TMA with CU_TENSOR_MAP_SWIZZLE_128B: 16-byte chunk j of row r sits at chunk j ^ (r % 8)
__device__ __forceinline__ int swz(int row, int k) { return row * kKT + ((((k >> 1) ^ (row & 7)) << 1) | (k & 1)); }

#ifndef TRL_SIMT_EMU
__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(void* bar, unsigned count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count)); }
__device__ __forceinline__ void mbar_expect_tx(void* bar, unsigned bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(void* bar) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory"); }
__device__ __forceinline__ void mbar_wait(void* bar, unsigned parity) {
    asm volatile(
        "{\n .reg .pred p;\n WAIT_%=:\n mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n @p bra DONE_%=;\n bra WAIT_%=;\n DONE_%=:\n}\n" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, void* bar, int c0, int c1) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(smem_u32(dst)),
                 "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
                 : "memory");
}
#endif

// ------------------------------------------------------------------------------------------------ conv stage
// The three terrain convolutions of ONE decision on a 4-CTA cluster, every layer as an implicit-im2col GEMM on DMMA:
//   C[t][o] = sum over (c, k) of act[c][t + k] * w[o][c][k]      rows = output positions, columns = output channels
// A fragments come straight from the activation rows in shared memory (lane (g, t4) reads act[c][t0 + g + t4]: neighbouring lanes
// read neighbouring or identical words), B fragments from a padded copy of the weights (row stride = 32 B mod 128 B).  conv1 / conv2
// have 4 taps = exactly one k-step per input channel.  Each CTA computes conv0 in full and its own 8 output channels of conv1 /
// conv2; the conv1 slices are exchanged through DSMEM, the conv2 slice goes to row idx of the FC stage's input matrix.
constexpr int kCvX = 0;                                    // 283 (+pad) normalised input
constexpr int kCvA0 = 288;                                 // conv0 output [16][193]
constexpr int kCvA1 = kCvA0 + kConv0Out * kW0 + 8;         // conv1 output [32][190] (own slice computed, rest gathered)
constexpr int kCvW0 = kCvA1 + kConv1Out * kW1 + 8;         // conv0 weights [16][12]  (8 taps + pad)
constexpr int kCvW1 = kCvW0 + kConv0Out * 12;              // conv1 weight slice [8][68]   (16 x 4 + pad)
constexpr int kCvW2 = kCvW1 + kC1Slice * 68;               // conv2 weight slice [8][132]  (32 x 4 + pad)
constexpr int kConvSmemDoubles = kCvW2 + kC2Slice * 132;
static_assert(kC1Slice == 8 && kC2Slice == 8, "the DMMA conv stage assumes 8 output channels (one n tile) per CTA");

// 4-tap convolution layer slice: out[o][t] = relu(b[o] + sum_c sum_k act[c][t + k] w[o][c][k]) for this CTA's 8 channels
template <int CIN, int WIN, int WOUT, int WSTRIDE>
__device__ __forceinline__ void conv4_dmma(const double* __restrict__ act, const double* __restrict__ ws, const double* __restrict__ bias8,
                                           double* __restrict__ out, int out_stride) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, g = lane >> 2, t4 = lane & 3;
    constexpr int nmt = (WOUT + 7) / 8, nwarp = kDecideThreads / 32;
    const double b0 = bias8[2 * t4], b1 = bias8[2 * t4 + 1];
    const double* brow = ws + g * WSTRIDE + t4;
    for (int mt = warp; mt < nmt; mt += 2 * nwarp) {
        // two row tiles per pass share the B fragment
        const int mt2 = mt + nwarp;
        const bool two = mt2 < nmt;
        const double* a0p = act + min(mt * 8 + g, WOUT - 1) + t4;
        const double* a1p = act + min((two ? mt2 : mt) * 8 + g, WOUT - 1) + t4;
        double c00 = b0, c01 = b1, c10 = b0, c11 = b1;
#pragma unroll 4
        for (int c = 0; c < CIN; ++c) {
            const double b = brow[4 * c];
            dmma_8x8x4(c00, c01, a0p[c * WIN], b);
            dmma_8x8x4(c10, c11, a1p[c * WIN], b);
        }
        const int ta = mt * 8 + g, tb = mt2 * 8 + g;
        if (ta < WOUT) {
            out[(2 * t4) * out_stride + ta] = c00 > 0.0 ? c00 : 0.0;
            out[(2 * t4 + 1) * out_stride + ta] = c01 > 0.0 ? c01 : 0.0;
        }
        if (two && tb < WOUT) {
            out[(2 * t4) * out_stride + tb] = c10 > 0.0 ? c10 : 0.0;
            out[(2 * t4 + 1) * out_stride + tb] = c11 > 0.0 ? c11 : 0.0;
        }
    }
}

__device__ void conv_stage_cluster(cg::cluster_group& cluster, const NetWeights& W, const double* __restrict__ x_in, double* sh, int n_char,
                                   double* __restrict__ out_row, bool normalised = false, double* __restrict__ a0_out = nullptr,
                                   double* __restrict__ a1_out = nullptr) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = lane >> 2, t4 = lane & 3;
    const int rank = (int)cluster.block_rank();
    const int n_in = 200 + n_char;
    double* X = sh + kCvX;
    double* A0 = sh + kCvA0;
    double* A1 = sh + kCvA1;
    double* W0s = sh + kCvW0;
    double* W1s = sh + kCvW1;
    double* W2s = sh + kCvW2;
    for (int i = tid; i < n_in; i += kDecideThreads) X[i] = normalised ? x_in[i] : (x_in[i] + W.in_off[i]) * W.in_scale[i];
    for (int i = tid; i < kConv0Out * kConv0K; i += kDecideThreads) W0s[(i >> 3) * 12 + (i & 7)] = W.conv0_w[i];
    for (int i = tid; i < kC1Slice * 64; i += kDecideThreads) W1s[(i >> 6) * 68 + (i & 63)] = W.conv1_w[rank * kC1Slice * 64 + i];
    for (int i = tid; i < kC2Slice * 128; i += kDecideThreads) W2s[(i >> 7) * 132 + (i & 127)] = W.conv2_w[rank * kC2Slice * 128 + i];
    __syncthreads();
    // conv0: 1 -> 16 channels, 8 taps (two k-steps), 25 x 2 C tiles
    for (int item = warp; item < ((kW0 + 7) / 8) * 2; item += kDecideThreads / 32) {
        const int mt = item >> 1, nt = item & 1;
        const double* ap = X + min(mt * 8 + g, kW0 - 1) + t4;
        const double* bp = W0s + (nt * 8 + g) * 12 + t4;
        double c0 = W.conv0_b[nt * 8 + 2 * t4], c1 = W.conv0_b[nt * 8 + 2 * t4 + 1];
        dmma_8x8x4(c0, c1, ap[0], bp[0]);
        dmma_8x8x4(c0, c1, ap[4], bp[4]);
        const int t = mt * 8 + g;
        if (t < kW0) {
            A0[(nt * 8 + 2 * t4) * kW0 + t] = c0 > 0.0 ? c0 : 0.0;
            A0[(nt * 8 + 2 * t4 + 1) * kW0 + t] = c1 > 0.0 ? c1 : 0.0;
        }
    }
    __syncthreads();
    if (a0_out && rank == 0) for (int i = tid; i < kConv0Out * kW0; i += kDecideThreads) a0_out[i] = A0[i];
    conv4_dmma<kConv0Out, kW0, kW1, 68>(A0, W1s, W.conv1_b + rank * kC1Slice, A1 + rank * kC1Slice * kW1, kW1);
    cluster.sync();
    if (a1_out) for (int i = tid; i < kC1Slice * kW1; i += kDecideThreads) a1_out[rank * kC1Slice * kW1 + i] = A1[rank * kC1Slice * kW1 + i];
    for (int r = 1; r < kClusterSize; ++r) {
        int src = (rank + r) % kClusterSize;
        const double* remote = cluster.map_shared_rank(A1, src);
        for (int i = tid; i < kC1Slice * kW1; i += kDecideThreads) {
            int off = src * kC1Slice * kW1 + i;
            A1[off] = remote[off];
        }
    }
    __syncthreads();
    conv4_dmma<kConv1Out, kW1, kW2, 132>(A1, W2s, W.conv2_b + rank * kC2Slice, out_row + (size_t)rank * kC2Slice * kW2, kW2);
    cluster.sync();   // peers read this CTA's A1 slice until here; the next decision overwrites it
}

// 64 registers: two of these CTAs fit one SM, and one fits beside two resident env-step CTAs (a whole-SM CTA waits for all four to drain)
__global__ void __cluster_dims__(kClusterSize, 1, 1) __launch_bounds__(kDecideThreads, 2)
trl_decide_conv_kernel(Buffers B, NetWeights W, double* __restrict__ act2, int list) {
    TRL_DYN_SHARED(double, sh);
    cg::cluster_group cluster = cg::this_cluster();
    const ModelConst& m = c_model;
    if (!m.has_net) return;
    const int cid = blockIdx.x / kClusterSize, ncl = gridDim.x / kClusterSize;
    const int count = B.pending_count[list];
    for (int idx = cid; idx < count; idx += ncl) {
        const int env = B.pending_list[list * B.n + idx];
        conv_stage_cluster(cluster, W, B.poli_state + (size_t)env * B.S, sh, m.n_char, act2 + (size_t)idx * kTipIn);
    }
}

// slot build: the same stage with the weights and input offset / scale of the env's policy slot
__global__ void __cluster_dims__(kClusterSize, 1, 1) __launch_bounds__(kDecideThreads, 2)
trl_decide_conv_slots_kernel(Buffers B, PolicySlots P, double* __restrict__ act2, int list) {
    TRL_DYN_SHARED(double, sh);
    cg::cluster_group cluster = cg::this_cluster();
    const ModelConst& m = c_model;
    if (!m.has_net) return;
    const int cid = blockIdx.x / kClusterSize, ncl = gridDim.x / kClusterSize;
    const int count = B.pending_count[list];
    for (int idx = cid; idx < count; idx += ncl) {
        const int env = B.pending_list[list * B.n + idx];
        conv_stage_cluster(cluster, P.W[P.env_slot[env]], B.poli_state + (size_t)env * B.S, sh, m.n_char, act2 + (size_t)idx * kTipIn);
    }
}

// Slot build, ahead of the conv stage: regroups pending list `list` by policy slot (a counting sort in one CTA; the order within a
// slot is whatever the atomics give -- every row of the pass is independent of the others, and so is the catch-up launch that
// reads the list afterwards) and writes the FC stage's chunk table: each 32-row chunk belongs to one slot, a slot's last chunk
// may be ragged.
__global__ void __launch_bounds__(1024) trl_slot_sort_kernel(Buffers B, PolicySlots P, int* __restrict__ tmp, int* __restrict__ tab, int list) {
    __shared__ int cnt[kMaxPolicySlots], next[kMaxPolicySlots];
    const int count = B.pending_count[list];
    int* L = B.pending_list + (size_t)list * B.n;
    if (threadIdx.x < kMaxPolicySlots) cnt[threadIdx.x] = 0;
    __syncthreads();
    for (int i = threadIdx.x; i < count; i += blockDim.x) {
        const int env = L[i];
        tmp[i] = env;
        atomicAdd(&cnt[P.env_slot[env]], 1);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        int row = 0, nc = 0;
        for (int p = 0; p < kMaxPolicySlots; ++p) {
            next[p] = row;
            for (int r = 0; r < cnt[p]; r += kFcRows, ++nc) {
                tab[1 + 3 * nc] = p; tab[2 + 3 * nc] = row + r; tab[3 + 3 * nc] = min(kFcRows, cnt[p] - r);
            }
            row += cnt[p];
        }
        tab[0] = nc;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < count; i += blockDim.x) {
        const int env = tmp[i];
        L[atomicAdd(&next[P.env_slot[env]], 1)] = env;
    }
}

// cycles / episodes / env-steps / episode-weighted distance of the envs in one (policy slot, terrain slot) cell into
// out[kMaxPolicySlots + 1][kMaxTerrainSlots + 1][4]; index kMaxPolicySlots / kMaxTerrainSlots = any slot.  One CTA per cell, each
// with trl_stats_kernel's traversal and reduction order, so a cell's figures do not depend on the others (env_slot null: every env is
// on policy slot 0; the terrain slot is the one the env's present ground came from)
__global__ void __launch_bounds__(1024) trl_cell_stats_kernel(Buffers B, const int* __restrict__ env_slot, double* __restrict__ out) {
    __shared__ double red[4][32];
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31, nw = blockDim.x >> 5;
    const int p = blockIdx.x / (kMaxTerrainSlots + 1), t = blockIdx.x % (kMaxTerrainSlots + 1);
    const int* terrain_slot = B.i + (size_t)I_TERRAIN_SLOT * B.n;
    double c = 0, e = 0, st = 0, ds = 0;
    for (int env = threadIdx.x; env < B.n; env += blockDim.x) {
        if (p < kMaxPolicySlots && (env_slot ? env_slot[env] : 0) != p) continue;
        if (t < kMaxTerrainSlots && terrain_slot[env] != t) continue;
        const int ec = B.i[(size_t)I_EPISODE_COUNT * B.n + env];
        c += B.i[(size_t)I_CYCLE_COUNT * B.n + env];
        e += ec;
        st += (double)(((uint64_t)(uint32_t)B.i[(size_t)I_STEPS_HI * B.n + env] << 32) | (uint32_t)B.i[(size_t)I_STEPS_LO * B.n + env]);
        ds += B.d[(size_t)D_AVG_DIST * B.n + env] * ec;
    }
    c = warp_sum_all(c); e = warp_sum_all(e); st = warp_sum_all(st); ds = warp_sum_all(ds);
    if (l == 0) { red[0][w] = c; red[1][w] = e; red[2][w] = st; red[3][w] = ds; }
    __syncthreads();
    if (w == 0)
        for (int k = 0; k < 4; ++k) {
            const double v = warp_sum_all(l < nw ? red[k][l] : 0.0);
            if (l == 0) out[4 * blockIdx.x + k] = v;
        }
}

// the same four figures over the envs of one (policy slot, terrain slot, physics slot) cell into out[4], -1 = any slot; one CTA with
// trl_stats_kernel's traversal and reduction order.  The physics slot is the one of the env's present episode (env_phys row 0).
// env_eval (optional, null: any mode): only the envs whose present episode's mode (row 0 of trl_set_env_eval's array) is `eval`;
// env_body (optional, null: any body) likewise only the envs whose present episode runs on body slot `b` (row 0 of env_body)
__global__ void __launch_bounds__(1024) trl_phys_stats_kernel(Buffers B, const int* __restrict__ env_slot, const int* __restrict__ env_phys, int p,
                                                              int t, int q, const int* __restrict__ env_eval, int eval,
                                                              const int* __restrict__ env_body, int b, double* __restrict__ out) {
    __shared__ double red[4][32];
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31, nw = blockDim.x >> 5;
    const int* terrain_slot = B.i + (size_t)I_TERRAIN_SLOT * B.n;
    double c = 0, e = 0, st = 0, ds = 0;
    for (int env = threadIdx.x; env < B.n; env += blockDim.x) {
        if (p >= 0 && (env_slot ? env_slot[env] : 0) != p) continue;
        if (t >= 0 && terrain_slot[env] != t) continue;
        if (q >= 0 && env_phys[env] != q) continue;
        if (env_eval && env_eval[env] != eval) continue;
        if (env_body && env_body[env] != b) continue;
        const int ec = B.i[(size_t)I_EPISODE_COUNT * B.n + env];
        c += B.i[(size_t)I_CYCLE_COUNT * B.n + env];
        e += ec;
        st += (double)(((uint64_t)(uint32_t)B.i[(size_t)I_STEPS_HI * B.n + env] << 32) | (uint32_t)B.i[(size_t)I_STEPS_LO * B.n + env]);
        ds += B.d[(size_t)D_AVG_DIST * B.n + env] * ec;
    }
    c = warp_sum_all(c); e = warp_sum_all(e); st = warp_sum_all(st); ds = warp_sum_all(ds);
    if (l == 0) { red[0][w] = c; red[1][w] = e; red[2][w] = st; red[3][w] = ds; }
    __syncthreads();
    if (w == 0)
        for (int k = 0; k < 4; ++k) {
            const double v = warp_sum_all(l < nw ? red[k][l] : 0.0);
            if (l == 0) out[k] = v;
        }
}

// the conv stage over the rows of a trainer minibatch (one cluster per row)
__global__ void __cluster_dims__(kClusterSize, 1, 1) __launch_bounds__(kDecideThreads, 2)
trl_fwd_conv_train_kernel(NetWeights W, FwdTrain f, double* __restrict__ act2) {
    TRL_DYN_SHARED(double, sh);
    cg::cluster_group cluster = cg::this_cluster();
    if (f.gate && *f.gate == 0) return;
    const int cid = blockIdx.x / kClusterSize, ncl = gridDim.x / kClusterSize;
    for (int r = cid; r < f.rows; r += ncl)
        conv_stage_cluster(cluster, W, f.xn + (size_t)r * f.S, sh, f.S - 200, act2 + (size_t)r * kTipIn, true,
                           f.a0 ? f.a0 + (size_t)r * kConv0Out * kW0 : nullptr, f.a1 ? f.a1 + (size_t)r * kConv1Out * kW1 : nullptr);
}

// ------------------------------------------------------------------------------------------------ FC stage
// the scalar decision of one env (cDogControllerMACE::UpdateAction, cBaseControllerMACE::DecideActionBoltzmann, BuildActorAction,
// ApplyExpNoiseAction: sim/DogController.cpp:847-868, sim/BaseControllerMACE.cpp:254-318,339-396,437-518); Y = this decision's
// unnormalised net output (unused when the scene has no net).  kSlots: the exploration noise is scaled by the deciding slot's own actor
// output scale `noise_scale` (the net of a training slot sets it); otherwise by the scene's, c_model.out_scale_actor0.  An evaluating
// env (kSlots only: trl_set_env_eval) decides with exploration off, whatever the settings `ex` of its slot say
template <bool kSlots = false>
__device__ void decide_one(const Buffers& B, const ExpSettings& ex, int env, const double* Y, const double* noise_scale = nullptr,
                           bool evaluates = false) {
    const ModelConst& m = c_model;
    const bool slot_explores = kSlots && ex.enable && !evaluates;     // read where the single-policy build reads ex.enable
    Lane L{nullptr, env, B.n, B.d, B.i};
    double params[kNumParams];
    int id, eflags = 4;
    CounterRng rng = load_rng(L);
    for (int k = 0; k < m.n_params; ++k) params[k] = L.d(D_PARAMS + k);
    id = L.i(I_ACTION_ID);
    const int cmd = L.i(I_CMD);
    if (cmd >= 0) {
        if (m.is_mace) eflags |= 3;
        id = build_base_action(L, rng, cmd, params);
        L.i(I_CMD) = -1;
    } else if (m.has_net) {
        const double base_rand = rng.uniform();
        if ((kSlots ? slot_explores : ex.enable) && base_rand < ex.base_rate) {
            const int a = rng.rand_int(0, m.n_actions);
            id = build_base_action(L, rng, a, params);
            eflags = 4 | 3;
        } else {
            for (int i = 0; i < m.n_out; ++i) B.net_out[(size_t)env * kMaxNetOut + i] = Y[i];
            eflags = 0;
            const int nf = m.n_frags, fs = m.frag;
            int a_max = 0;
            for (int i = 1; i < nf; ++i) if (Y[i] > Y[a_max]) a_max = i;
            int a = a_max;
            if ((kSlots ? slot_explores : ex.enable) && ex.temp != 0.0) {   // BoltzmannSelectActor
                double vals[8], sum = 0.0;
                for (int i = 0; i < nf; ++i) { vals[i] = exp((Y[i] - Y[a_max]) / ex.temp); sum += vals[i]; }
                double r = rng.uniform() * sum;
                for (int i = 0; i < nf; ++i) { r -= vals[i]; if (r <= 0.0) { a = i; break; } }
            }
            id = a;
            for (int k = 0; k < fs; ++k) params[m.opt_idx[k]] = Y[nf + a * fs + k];
            params[mTransTime] = fabs(params[mTransTime]); params[mCv] = fabs(params[mCv]);
            if (m.char_type == 2) params[rmCd] = fabs(params[rmCd]);
            if (kSlots ? slot_explores : ex.enable) {
                const double rn = rng.uniform();
                if (rn < ex.rate) {              // ApplyExpNoiseAction
                    for (int k = 0; k < fs; ++k) params[m.opt_idx[k]] += (ex.noise * rng.normal()) * (1.0 / (kSlots ? noise_scale[k] : m.out_scale_actor0[k]));
                    eflags |= 2;
                }
                if (a != a_max) eflags |= 1;
                if (eflags & 3) eflags |= 4;
            }
        }
    } else {
        const bool cyclic = m.is_mace ? false : (m.act_cyclic[id] != 0);
        if (!cyclic) id = build_base_action(L, rng, m.default_action, params);
    }
    L.i(I_EXP_FLAGS) = eflags;
    apply_action(L, id, params, B.com_stash[env], B.com_stash[B.n + env]);
    store_rng(L, rng);
}

// kSlots: the slot build (trl_decide_fc_slots_kernel).  The chunks come from the table trl_slot_sort_kernel wrote, each with its slot's
// weights (W0 = the slot table), terr_ip0 descriptor (smaps) and output offset / scale; the ip0 weight slice is restaged when a
// cluster moves on to a chunk of another slot.  Without it, the single-policy kernel: chunk k = rows 32 k .., W0 = the one net.
template <bool kTrain, bool kSlots = false>
__device__ __forceinline__ void fc_stage(const Buffers& B, const NetWeights& W0, const ExpSettings* __restrict__ ex_dev, const FcMaps& maps, const FwdTrain& ft,
                                         int* done_count, int list, int rearm, const FcSlotMaps* smaps = nullptr, const int* __restrict__ tab = nullptr,
                                         const int* __restrict__ env_eval = nullptr) {
    TRL_DYN_SHARED(unsigned char, fc_smem_raw);
    // the swizzled TMA tiles need 1024-byte alignment; the dynamic window starts at the same offset in every CTA of the cluster, so
    // the rounded address is a valid DSMEM offset as well
#ifndef TRL_SIMT_EMU
    unsigned char* fc_smem = fc_smem_raw + ((1024u - (smem_u32(fc_smem_raw) & 1023u)) & 1023u);
#else
    unsigned char* fc_smem = fc_smem_raw;      // no hardware swizzle to satisfy; per-CTA host allocations are not equally aligned
#endif
    cg::cluster_group cluster = cg::this_cluster();
    const ModelConst& m = c_model;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = lane >> 2, t4 = lane & 3;
    const int rank = (int)cluster.block_rank();
    const int cid = blockIdx.x / kFcCluster, ncl = gridDim.x / kFcCluster;
    if (kTrain && ft.gate && *ft.gate == 0) return;
    const int count = kTrain ? ft.rows : B.pending_count[list];
    // the slot build reads the settings of each chunk's slot where it decides (ex_dev is the handle's table of kMaxPolicySlots
    // entries); the single-policy kernel reads entry 0 once
    ExpSettings ex{};
    if (!kTrain && !kSlots) ex = *ex_dev;
    const int n_char = kTrain ? ft.S - 200 : m.n_char, ncat = kTip0Out + n_char;
    const bool has_net = kTrain || m.has_net;
    const int n_frags = kTrain ? ft.n_frags : m.n_frags, frag = kTrain ? ft.frag : m.frag;
    double* P = (double*)(fc_smem + kFcOffPart);
    double* CAT = (double*)(fc_smem + kFcOffCat);
    double* WIP = (double*)(fc_smem + kFcOffWip);
    double* H = (double*)(fc_smem + kFcOffH);
    double* HH = (double*)(fc_smem + kFcOffHH);
    double* Y = (double*)(fc_smem + kFcOffY);
    unsigned long long* bar_full = (unsigned long long*)(fc_smem + kFcOffBar);
    unsigned long long* bar_empty = bar_full + kFcStages;
    const int nchunks = kSlots ? tab[0] : (count + kFcRows - 1) / kFcRows;
    int prof_n = 0;
    auto stamp = [&]() {
#ifndef TRL_SIMT_EMU
        if (maps.prof && blockIdx.x == 0 && tid == 0 && prof_n < 16) {
            unsigned long long t;
            asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
            maps.prof[prof_n++] = t;
        }
#endif
    };
    stamp();     // 0: kernel entry

    if (has_net && cid < nchunks) {
        // ip0 weight slice of this CTA (32 output columns x ncat, zero-padded to kCatStride): resident for the whole launch
        if (!kSlots)
            for (int i = tid; i < 32 * kCatStride; i += kFcThreads) {
                const int n = i / kCatStride, k = i - n * kCatStride;
                WIP[i] = k < ncat ? W0.ip0_w[(size_t)(rank * 32 + n) * ncat + k] : 0.0;
            }
#ifndef TRL_SIMT_EMU
        if (tid == 0) {
            for (int s = 0; s < kFcStages; ++s) { mbar_init(&bar_full[s], 1); mbar_init(&bar_empty[s], kFcThreads / 32); }
            asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        }
#endif
        __syncthreads();
    }
    stamp();     // 1: ip0 weights staged, barriers initialised
    // k tiles of terr_ip0 this CTA multiplies
    const int kt0 = (kNumKTiles * rank) / kFcCluster, kt1 = (kNumKTiles * (rank + 1)) / kFcCluster;
    unsigned pipe_iter = 0;      // tiles issued / consumed so far over all chunks (stage = iter % kFcStages, parity from iter / kFcStages)
    int staged = -1;             // slot build: the slot whose ip0 slice WIP holds

    for (int chunk = cid; chunk < nchunks; chunk += ncl) {
        const int slot = kSlots ? tab[1 + 3 * chunk] : 0;
        const int row0 = kSlots ? tab[2 + 3 * chunk] : chunk * kFcRows;
        const int rows = kSlots ? tab[3 + 3 * chunk] : min(kFcRows, count - row0);
        const NetWeights& W = kSlots ? (&W0)[slot] : W0;
        if (kSlots && has_net && slot != staged) {
            // WIP was last read by the previous chunk's ip0, before its closing cluster.sync; the cluster.sync behind terr_ip0 below
            // orders these writes before this chunk's reads
            for (int i = tid; i < 32 * kCatStride; i += kFcThreads) {
                const int n = i / kCatStride, k = i - n * kCatStride;
                WIP[i] = k < ncat ? W.ip0_w[(size_t)(rank * 32 + n) * ncat + k] : 0.0;
            }
            staged = slot;
        }
        if (has_net) {
            // ---------------- terr_ip0: P[32][64] = A[32][k slice] * Wt[k slice][64]; warp w owns C tiles (m tile w / 4, n tiles 2 (w % 4) + {0, 1})
            const int mt = warp >> 2, nt0 = (warp & 3) * 2;
            double c00 = 0, c01 = 0, c10 = 0, c11 = 0;
            const int ntile = kt1 - kt0, nload = (ntile + kTilesPerStage - 1) / kTilesPerStage;
#ifndef TRL_SIMT_EMU
            // producer: thread 0 keeps up to kFcStages tiles in flight
            int issued = 0;
            auto issue = [&](int j) {          // stage-load j: k-tiles kt0 + 2 j, kt0 + 2 j + 1 (the last one may hold a single tile)
                const unsigned it = pipe_iter + (unsigned)j;
                const int s = (int)(it % kFcStages);
                const unsigned round = it / kFcStages;
                if (round > 0) mbar_wait(&bar_empty[s], (round - 1) & 1);
                unsigned char* st = fc_smem + kFcOffPipe + (size_t)s * kStageBytes;
                const int nt = min(kTilesPerStage, ntile - j * kTilesPerStage);
                mbar_expect_tx(&bar_full[s], nt * kTileBytes);
                for (int q = 0; q < nt; ++q) {
                    const int kt = kt0 + j * kTilesPerStage + q;
                    tma_load_2d(st + q * kTileBytes, kSlots ? &smaps->w[slot] : &maps.w, &bar_full[s], kt * kKT, 0);
                    tma_load_2d(st + q * kTileBytes + kWTileBytes, &maps.a, &bar_full[s], kt * kKT, row0);
                }
            };
            if (tid == 0) {
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");     // H / HH of the previous chunk live in the same bytes
                for (; issued < min(kFcStages, nload); ++issued) issue(issued);
            }
#endif
            for (int j = 0; j < nload; ++j) {
                const unsigned it = pipe_iter + (unsigned)j;
                const int s = (int)(it % kFcStages);
                const int nt = min(kTilesPerStage, ntile - j * kTilesPerStage);
#ifndef TRL_SIMT_EMU
                mbar_wait(&bar_full[s], (it / kFcStages) & 1);
#else
                // emulator: the tile copies TMA would perform, same swizzled layout
                __syncthreads();
                for (int q = 0; q < nt; ++q) {
                    double* Wq = (double*)(fc_smem + kFcOffPipe + (size_t)s * kStageBytes + (size_t)q * kTileBytes);
                    double* Aq = (double*)(fc_smem + kFcOffPipe + (size_t)s * kStageBytes + (size_t)q * kTileBytes + kWTileBytes);
                    const int kt = kt0 + j * kTilesPerStage + q;
                    for (int i = tid; i < kTip0Out * kKT; i += kFcThreads) {
                        const int n = i / kKT, k = i - n * kKT;
                        Wq[swz(n, k)] = (kSlots ? smaps->w_ptr[slot] : maps.w_ptr)[(size_t)n * kTipIn + kt * kKT + k];
                    }
                    for (int i = tid; i < kFcRows * kKT; i += kFcThreads) {
                        const int r = i / kKT, k = i - r * kKT;
                        Aq[swz(r, k)] = (row0 + r) < maps.a_rows ? maps.a_ptr[(size_t)(row0 + r) * kTipIn + kt * kKT + k] : 0.0;
                    }
                }
                __syncthreads();
#endif
                for (int q = 0; q < nt; ++q) {
                    const double* Wt = (const double*)(fc_smem + kFcOffPipe + (size_t)s * kStageBytes + (size_t)q * kTileBytes);
                    const double* At = (const double*)(fc_smem + kFcOffPipe + (size_t)s * kStageBytes + (size_t)q * kTileBytes + kWTileBytes);
#pragma unroll
                    for (int ks = 0; ks < kKT / 4; ++ks) {
                        const double a = At[swz(mt * 8 + g, ks * 4 + t4)];
                        const double b0 = Wt[swz(nt0 * 8 + g, ks * 4 + t4)];
                        const double b1 = Wt[swz(nt0 * 8 + 8 + g, ks * 4 + t4)];
                        dmma_8x8x4(c00, c01, a, b0);
                        dmma_8x8x4(c10, c11, a, b1);
                    }
                }
#ifndef TRL_SIMT_EMU
                __syncwarp();
                if (lane == 0) mbar_arrive(&bar_empty[s]);
                if (tid == 0 && issued < nload) { issue(issued); ++issued; }
#endif
            }
            pipe_iter += (unsigned)nload;
            P[(mt * 8 + g) * kTip0Out + nt0 * 8 + 2 * t4] = c00;
            P[(mt * 8 + g) * kTip0Out + nt0 * 8 + 2 * t4 + 1] = c01;
            P[(mt * 8 + g) * kTip0Out + nt0 * 8 + 8 + 2 * t4] = c10;
            P[(mt * 8 + g) * kTip0Out + nt0 * 8 + 8 + 2 * t4 + 1] = c11;
            stamp();     // 2: terr_ip0 tiles consumed
            cluster.sync();
            stamp();     // 3
            // ---------------- concat0 = [relu(sum of the partials in rank order + bias) | normalised character features]
            for (int i = tid; i < kFcRows * kTip0Out; i += kFcThreads) {
                const int r = i / kTip0Out, o = i - r * kTip0Out;
                double acc = W.tip0_b[o];
#pragma unroll
                for (int q = 0; q < kFcCluster; ++q) acc += cluster.map_shared_rank(P, q)[i];
                CAT[r * kCatStride + o] = acc > 0.0 ? acc : 0.0;
            }
            for (int i = tid; i < kFcRows * (kCatStride - kTip0Out); i += kFcThreads) {
                const int r = i / (kCatStride - kTip0Out), c = i - r * (kCatStride - kTip0Out);
                double v = 0.0;
                if (r < rows && c < n_char) {
                    if (kTrain) v = ft.xn[(size_t)(row0 + r) * ft.S + 200 + c];
                    else {
                        const int env = B.pending_list[list * B.n + row0 + r];
                        v = (B.poli_state[(size_t)env * B.S + 200 + c] + W.in_off[200 + c]) * W.in_scale[200 + c];
                    }
                }
                CAT[r * kCatStride + kTip0Out + c] = v;
            }
            stamp();     // 4: concat0 built
            cluster.sync();      // CAT complete here; every peer has finished reading this CTA's P
            if (kTrain && rank == 0) {
                for (int i = tid; i < rows * ncat; i += kFcThreads) { const int r = i / ncat, c = i - r * ncat; ft.catb[(size_t)(row0 + r) * ft.cat + c] = CAT[r * kCatStride + c]; }
                for (int i = tid; i < rows * kTip0Out; i += kFcThreads) { const int r = i / kTip0Out, c = i - r * kTip0Out; ft.t[(size_t)(row0 + r) * kTip0Out + c] = CAT[r * kCatStride + c]; }
            }
            stamp();     // 5
            // ---------------- ip0: H[:, 32 rank .. 32 rank + 32) = relu(CAT * Wip^T + b); 16 C tiles, one per warp
            {
                const int mt2 = warp >> 2, nt2 = warp & 3;
                double c0 = 0, c1 = 0;
                const double* arow = CAT + (mt2 * 8 + g) * kCatStride + t4;
                const double* brow = WIP + (nt2 * 8 + g) * kCatStride + t4;
#pragma unroll 4
                for (int ks = 0; ks < kCatStride / 4; ++ks) dmma_8x8x4(c0, c1, arow[ks * 4], brow[ks * 4]);
                const int col = rank * 32 + nt2 * 8 + 2 * t4;
                const double v0 = c0 + W.ip0_b[col], v1 = c1 + W.ip0_b[col + 1];
                // every CTA needs the whole H: write the two values into all eight copies
#pragma unroll
                for (int q = 0; q < kFcCluster; ++q) {
                    double* Hq = cluster.map_shared_rank(H, q);
                    Hq[(mt2 * 8 + g) * kHStride + col] = v0 > 0.0 ? v0 : 0.0;
                    Hq[(mt2 * 8 + g) * kHStride + col + 1] = v1 > 0.0 ? v1 : 0.0;
                }
            }
            stamp();     // 6: ip0 done, H scattered
            cluster.sync();
            if (kTrain && rank == 1)
                for (int i = tid; i < rows * kIp0Out; i += kFcThreads) { const int r = i / kIp0Out, c = i - r * kIp0Out; ft.h[(size_t)(row0 + r) * kIp0Out + c] = H[r * kHStride + c]; }
            stamp();     // 7
            // ---------------- head hidden layers: CTA pair (2 hd, 2 hd + 1) owns head hd; this CTA computes 64 of its 128 hidden units.
            // warp w: n tile w % 8 (of 8), m tiles 2 (w / 8) + {0, 1}; B fragments straight from L2 (each weight is used once per chunk)
            const int hd = rank >> 1, half = rank & 1;
            {
                const int ntl = warp & 7, mt3 = (warp >> 3) * 2;
                const double* wrow = W.h0_w[hd] + (size_t)(half * 64 + ntl * 8 + g) * kIp0Out + t4;
                const double* a0 = H + (mt3 * 8 + g) * kHStride + t4;
                const double* a1 = a0 + 8 * kHStride;
                double c00h = 0, c01h = 0, c10h = 0, c11h = 0;
#pragma unroll 8
                for (int ks = 0; ks < kIp0Out / 4; ++ks) {
                    const double b = wrow[ks * 4];
                    dmma_8x8x4(c00h, c01h, a0[ks * 4], b);
                    dmma_8x8x4(c10h, c11h, a1[ks * 4], b);
                }
                const int col = half * 64 + ntl * 8 + 2 * t4;
                const double b0 = W.h0_b[hd][col], b1 = W.h0_b[hd][col + 1];
                double* HHo = cluster.map_shared_rank(HH, rank & ~1);      // both halves land in the even CTA of the pair
                double v;
                v = c00h + b0; HHo[(mt3 * 8 + g) * kHHStride + col] = v > 0.0 ? v : 0.0;
                v = c01h + b1; HHo[(mt3 * 8 + g) * kHHStride + col + 1] = v > 0.0 ? v : 0.0;
                v = c10h + b0; HHo[(mt3 * 8 + 8 + g) * kHHStride + col] = v > 0.0 ? v : 0.0;
                v = c11h + b1; HHo[(mt3 * 8 + 8 + g) * kHHStride + col + 1] = v > 0.0 ? v : 0.0;
            }
            stamp();     // 8: head hidden layers done
            cluster.sync();
            if (kTrain && half == 0 && ft.hh)
                for (int i = tid; i < rows * kHeadHidden; i += kFcThreads) {
                    const int r = i / kHeadHidden, c = i - r * kHeadHidden;
                    ft.hh[((size_t)hd * ft.rows + row0 + r) * kHeadHidden + c] = HH[r * kHHStride + c];
                }
            stamp();     // 9
            // ---------------- output layers: the even CTA of a pair multiplies its head's [32 x 128] by [128 x nout] (n padded to 32) and
            // un-normalises into rank 0's Y
            if (half == 0) {
                const int nout = hd == 0 ? n_frags : frag;
                const int obase = hd == 0 ? 0 : n_frags + (hd - 1) * frag;
                const int mt4 = warp >> 2, nt4 = warp & 3;
                const int nrow = nt4 * 8 + g;                              // output unit this lane's B fragment belongs to
                const double* wrow = W.h1_w[hd] + (size_t)min(nrow, nout - 1) * kHeadHidden + t4;
                const double* arow = HH + (mt4 * 8 + g) * kHHStride + t4;
                double c0 = 0, c1 = 0;
#pragma unroll 8
                for (int ks = 0; ks < kHeadHidden / 4; ++ks) {
                    const double b = nrow < nout ? wrow[ks * 4] : 0.0;
                    dmma_8x8x4(c0, c1, arow[ks * 4], b);
                }
                const int o = nt4 * 8 + 2 * t4, yrow = mt4 * 8 + g;
                if (kTrain) {
                    // the trainer works on the net's own (normalised) outputs
                    if (yrow < rows && o < nout) ft.y[(size_t)(row0 + yrow) * ft.n_out + obase + o] = c0 + W.h1_b[hd][o];
                    if (yrow < rows && o + 1 < nout) ft.y[(size_t)(row0 + yrow) * ft.n_out + obase + o + 1] = c1 + W.h1_b[hd][o + 1];
                } else {
                    double* Y0 = cluster.map_shared_rank(Y, 0);
                    if (o < nout) Y0[yrow * kYStride + obase + o] = (c0 + W.h1_b[hd][o]) / W.out_scale[obase + o] - W.out_off[obase + o];
                    if (o + 1 < nout) Y0[yrow * kYStride + obase + o + 1] = (c1 + W.h1_b[hd][o + 1]) / W.out_scale[obase + o + 1] - W.out_off[obase + o + 1];
                }
            }
            stamp();     // 10: output layers done
            cluster.sync();
            stamp();     // 11
        }
        // ---------------- the scalar decisions of this chunk, one lane each
        if (!kTrain && rank == 0 && tid < rows) {
            if (kSlots) {
                const int env = B.pending_list[list * B.n + row0 + tid];
                decide_one<true>(B, ex_dev[slot], env, Y + tid * kYStride, W.out_scale + n_frags, env_eval && env_eval[env]);
            }
            else decide_one(B, ex, B.pending_list[list * B.n + row0 + tid], Y + tid * kYStride);
        }
        stamp();         // 12: decisions applied
        cluster.sync();      // Y / H / HH / the pipeline buffers are reused by the next chunk
        stamp();         // 13
    }
    // serial schedule: the last CTA to finish re-arms the list (in the overlapped schedule the catch-up launch, which still needs
    // the count, does it)
    if (!kTrain && rearm && threadIdx.x == 0) {
        __threadfence();
        int done = atomicAdd(done_count, 1);
        if (done == (int)gridDim.x - 1) { B.pending_count[list] = 0; *done_count = 0; __threadfence(); }
    }
}

__global__ void __cluster_dims__(kFcCluster, 1, 1) __launch_bounds__(kFcThreads, 1)
trl_decide_fc_kernel(Buffers B, NetWeights W, const ExpSettings* __restrict__ ex_dev, const TRL_GRID_CONSTANT FcMaps maps, int* done_count, int list,
                     int rearm) {
    const FwdTrain none{};
    fc_stage<false>(B, W, ex_dev, maps, none, done_count, list, rearm);
}
// slot build: chunks from the table of trl_slot_sort_kernel, weights and exploration settings (ex_dev[slot]) of each chunk's slot
__global__ void __cluster_dims__(kFcCluster, 1, 1) __launch_bounds__(kFcThreads, 1)
trl_decide_fc_slots_kernel(Buffers B, PolicySlots P, const ExpSettings* __restrict__ ex_dev, const TRL_GRID_CONSTANT FcMaps maps,
                           const TRL_GRID_CONSTANT FcSlotMaps smaps, const int* __restrict__ tab, int* done_count, int list, int rearm) {
    const FwdTrain none{};
    fc_stage<false, true>(B, *P.W, ex_dev, maps, none, done_count, list, rearm, &smaps, tab, P.env_eval);
}
// the FC stage over a trainer minibatch: activations and raw outputs to global memory, no decisions
__global__ void __cluster_dims__(kFcCluster, 1, 1) __launch_bounds__(kFcThreads, 1)
trl_fwd_fc_train_kernel(NetWeights W, const TRL_GRID_CONSTANT FcMaps maps, FwdTrain f) {
    Buffers none{};
    fc_stage<true>(none, W, nullptr, maps, f, nullptr, 0, 0);
}


size_t decide_fc_smem_bytes() { return (size_t)kFcSmemBytes; }
cudaError_t configure_decide2_kernels() {
    cudaError_t e = cudaFuncSetAttribute(trl_decide_conv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kConvSmemDoubles * 8);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(trl_fwd_conv_train_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kConvSmemDoubles * 8);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(trl_fwd_fc_train_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)decide_fc_smem_bytes());
    if (e == cudaSuccess) e = cudaFuncSetAttribute(trl_decide_conv_slots_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kConvSmemDoubles * 8);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(trl_decide_fc_slots_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)decide_fc_smem_bytes());
    if (e != cudaSuccess) return e;
    return cudaFuncSetAttribute(trl_decide_fc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)decide_fc_smem_bytes());
}
// conv stage for every pending decision (grid of 4-CTA clusters), then the batched FC stage + decisions (fc_clusters 8-CTA clusters)
void launch_decide2(const Buffers& B, const NetWeights& W, const ExpSettings* ex, const FcMaps& maps, double* act2, int* done_count, int grid,
                    int fc_clusters, int list, int rearm, cudaStream_t st, int part = 3) {
    if (part & 1) TRL_LAUNCH_CLUSTER(kClusterSize, trl_decide_conv_kernel, grid, kDecideThreads, (size_t)kConvSmemDoubles * 8, st, B, W, act2, list);
    if (part & 2)
        TRL_LAUNCH_CLUSTER(kFcCluster, trl_decide_fc_kernel, fc_clusters * kFcCluster, kFcThreads, decide_fc_smem_bytes(), st, B, W, ex, maps, done_count,
                           list, rearm);
}

// slot build of the same pass: regroup the list by slot (part 1, before the conv stage), conv stage, FC stage over the chunk table
// tab (one per side stream, like act2)
void launch_decide2_slots(const Buffers& B, const PolicySlots& P, const ExpSettings* ex, const FcMaps& maps, const FcSlotMaps& smaps, double* act2,
                          int* tmp, int* tab, int* done_count, int grid, int fc_clusters, int list, int rearm, cudaStream_t st, int part) {
    if (part & 1) {
        TRL_LAUNCH(trl_slot_sort_kernel, 1, 1024, 0, st, B, P, tmp, tab, list);
        TRL_LAUNCH_CLUSTER(kClusterSize, trl_decide_conv_slots_kernel, grid, kDecideThreads, (size_t)kConvSmemDoubles * 8, st, B, P, act2, list);
    }
    if (part & 2)
        TRL_LAUNCH_CLUSTER(kFcCluster, trl_decide_fc_slots_kernel, fc_clusters * kFcCluster, kFcThreads, decide_fc_smem_bytes(), st, B, P, ex, maps, smaps,
                           (const int*)tab, done_count, list, rearm);
}
void launch_cell_stats(const Buffers& B, const int* env_slot, double* out, cudaStream_t st) {
    TRL_LAUNCH(trl_cell_stats_kernel, (kMaxPolicySlots + 1) * (kMaxTerrainSlots + 1), 1024, 0, st, B, env_slot, out);
}
void launch_phys_stats(const Buffers& B, const int* env_slot, const int* env_phys, int policy_slot, int terrain_slot, int phys_slot,
                       const int* env_eval, int eval, const int* env_body, int body_slot, double* out, cudaStream_t st) {
    TRL_LAUNCH(trl_phys_stats_kernel, 1, 1024, 0, st, B, env_slot, env_phys, policy_slot, terrain_slot, phys_slot, env_eval, eval, env_body,
               body_slot, out);
}

// the forward pass of a trainer minibatch through the same two kernels (trl_train.cu: enqueue_forward); act2 = [rows][5984] scratch the
// FC stage's TMA descriptor `maps.a` covers
void launch_forward_train(const NetWeights& W, const FcMaps& maps, const FwdTrain& f, double* act2, cudaStream_t st) {
    TRL_LAUNCH_CLUSTER(kClusterSize, trl_fwd_conv_train_kernel, kClusterSize * f.rows, kDecideThreads, (size_t)kConvSmemDoubles * 8, st, W, f, act2);
    TRL_LAUNCH_CLUSTER(kFcCluster, trl_fwd_fc_train_kernel, kFcCluster * ((f.rows + kFcRows - 1) / kFcRows), kFcThreads, decide_fc_smem_bytes(), st, W, maps, f);   // one cluster per chunk of 32 rows
}

}  // namespace trl
