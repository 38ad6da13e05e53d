// deepterrainrl_b200 -- MACE trainer on the GPU (SURVEY.md §8 f1): the consumer of the experience tuples.
//
// cMACETrainer (learning/MACETrainer.cpp) + cNeuralNetTrainer (learning/NeuralNetTrainer.cpp) in synchronous mode, pool size 1,
// with the pieces of Caffe they drive written as CUDA kernels: batch-32 forward / backward of the MACE topology
// (data/policies/dog/nets/dog_mace3_train.prototxt) in f64 like Caffe's Net<double>, the EuclideanLoss over the normalised outputs
// and the SGD step of dog_mace3_solver.prototxt (lr 1e-3 fixed, momentum 0.9, L2 weight decay 5e-4, per-blob lr_mult / decay_mult).
// The replay memory (float rows [r | s | a | s'], learning/MACETrainer.cpp:515-539), the critic / actor index buffers
// (UpdateBuffers, :730-800), the positive-temporal-difference actor batch (:575-626) and the target net (:844-856) all live in
// HBM; tuples arrive device-to-device from the rollout engine's tuple block, and the engine evaluates the trainer's weights in
// place (cNeuralNetLearner::SyncNet becomes a pointer binding), so a training iteration involves no host copy.
//
// Control flow that depends on buffer sizes (critic batch available? actor batch full? target refresh due?) is decided on the
// device: every kernel of a step starts by reading its predicate from the counter block and returns if it is off.  That
// makes one cNeuralNetTrainer::Train() a fixed launch sequence, captured once as a CUDA graph.
//
// CPU restatement used by the tests: oracle/trainer.h.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <random>
#include <string>
#include <vector>

#include "../../include/terrainrl_b200.h"
#include "trl_handle.h"
#include "trl_comm.h"
#include "trl_mix64.h"

namespace trl {
void launch_forward_train(const NetWeights& W, const FcMaps& maps, const FwdTrain& f, double* act2, cudaStream_t st);
}
namespace trl_train {
using namespace trl;

constexpr int kB = 32;                               // MemoryData batch_size
constexpr int C0 = 16, K0 = 8, W0 = 193, C1 = 32, K1 = 4, W1 = 190, C2 = 32, K2 = 4, W2 = 187, T = 64, H = 256, HH = 128;
constexpr int kTerr = 200;                           // terrain samples at the head of the policy state

enum Pred { P_ALWAYS = 0, P_CRITIC, P_CAND, P_ACTOR, P_INIT };

struct Counters {
    int head, num, iter, actor_iter, stage, critic_count, actor_count, actor_batch_count;
    long long total;
    unsigned long long rng_ctr;
    int critic_ok, cand_count, actor_ok, succ, init_now, add_count;
    double critic_loss, actor_loss;
};

struct Dev {
    int S, A, Wd, n_char, n_out, n_frags, frag, cap, P, cat;
    int off[27];
    double *theta, *target, *history, *grad;
    double *in_off, *in_scale, *out_off, *out_scale;             // current net
    double *t_in_off, *t_in_scale, *t_out_off, *t_out_scale;     // target net
    float* mem;
    int *flags, *pos_critic, *pos_actor, *critic_list, *actor_list, *actor_batch;
    Counters* c;
    int *valid, *slot, *order, *ids, *ids2, *cand;      // ids: the critic's / the actor's batch; ids2: the actor candidates (padded)
    double *xn, *a0, *a1, *a2, *t, *catb, *h, *hh, *y;           // activations of the most recent forward pass (kB rows)
    double *v0, *v1;
    double *dy, *dhh, *dh, *dt, *da2, *da1, *da0;
    double* mean;
    double discount, base_lr, momentum, weight_decay;
    int freeze, nis, init_offset_scale, steps_per_iter;
    unsigned long long rng_key;
};

// Programmatic dependent launch: every trainer kernel is launched with programmatic stream serialization and starts with
// pdl_sync(): wait until the preceding kernel has completed (and its writes are visible), then let the next kernel of the
// stream be scheduled right away -- it parks at its own wait.  The dependency chain stays strictly serial; what disappears is
// the launch latency between the small dependent kernels of a training iteration (40 at one step per iteration).
__device__ __forceinline__ void pdl_sync() {
#ifndef TRL_SIMT_EMU   // the test-only emulator runs launches strictly in order
    asm volatile("griddepcontrol.wait;" ::: "memory");
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
#endif
}
template <typename... KArgs, typename... Args>
void launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr; cfg.numAttrs = 1;
    cudaLaunchKernelEx(&cfg, kern, KArgs(args)...);
}

__device__ __forceinline__ bool pred_on(const Dev& d, int pred) {
    switch (pred) {
        case P_CRITIC: return d.c->critic_ok != 0;
        case P_CAND: return d.c->cand_count > 0;
        case P_ACTOR: return d.c->actor_ok != 0;
        case P_INIT: return d.c->init_now != 0;
        default: return true;
    }
}
__device__ __forceinline__ int rand_int(const Dev& d, int mn, int mx) {      // cMathUtil::RandInt(min, max), counter RNG
    if (mn == mx) return mn;
    unsigned long long v = mix64(d.rng_key + (d.c->rng_ctr++) * 0xD1342543DE82EF95ull);
    int r = (int)(v >> 33);
    return mn + r % (mx - mn);
}
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// ================================================================================================ replay memory
// cNeuralNetTrainer::CheckTuple (learning/NeuralNetTrainer.cpp:541-576): one block per incoming tuple
__global__ void k_add_check(Dev d, const double* rows, const int* count_ptr, int count_val) {
    pdl_sync();
    const int count = count_ptr ? min(*count_ptr, (int)gridDim.x) : count_val;     // the scenario's cursor may run past its capacity
    const int i = blockIdx.x;
    if (i >= count) return;
    const double* r = rows + (size_t)i * d.Wd;
    int bad = 0;
    for (int k = threadIdx.x; k < d.Wd; k += blockDim.x) bad |= !isfinite(r[k]);
    bad = __syncthreads_or(bad);
    if (threadIdx.x == 0) d.valid[i] = !bad;
}
// Canonical arrival order for tuples that come from the scenario's block: its slots are filled through an atomic cursor, so
// their order is timing dependent; ranking them by env id (an env finishes at most one cycle per outer update) makes the
// replay memory -- and with it the whole training run -- reproducible.  One block per tuple: rank = #tuples with a smaller key.
__global__ void k_add_order(Dev d, const int* env_ids, const int* count_ptr) {
    pdl_sync();
    const int count = min(*count_ptr, (int)gridDim.x), i = blockIdx.x;
    if (i >= count) return;
    const int key = env_ids[i];
    int r = 0;
    for (int j = threadIdx.x; j < count; j += blockDim.x) {
        const int kj = env_ids[j];
        r += (kj < key) || (kj == key && j < i);
    }
    __shared__ int red[32];
    for (int o = 16; o > 0; o >>= 1) r += __shfl_xor_sync(0xffffffffu, r, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = r;
    __syncthreads();
    if (threadIdx.x == 0) {
        int tot = 0;
        for (int w = 0; w < (int)(blockDim.x >> 5); ++w) tot += red[w];
        d.order[tot] = i;
    }
}
__device__ void list_remove(int* list, int* pos, int& count, int t) {
    const int p = pos[t];
    if (p < 0) return;
    const int last = list[count - 1];
    list[p] = last; pos[last] = p;
    pos[t] = -1;
    --count;
}
// one incoming tuple: replay slot (cNeuralNetTrainer::AddTuple) + cMACETrainer::UpdateBuffers; returns the slot
__device__ int assign_slot(const Dev& d, Counters& c, uint32_t flags) {
    const int t = c.head;
    c.head = (c.head + 1) % d.cap;
    c.num = min(d.cap, c.num + 1);
    ++c.total;
    const bool ea = (flags & 4u) != 0;          // eFlagExpActor
    if (ea) {
        if (d.pos_actor[t] < 0) { d.pos_actor[t] = c.actor_count; d.actor_list[c.actor_count++] = t; }
        list_remove(d.critic_list, d.pos_critic, c.critic_count, t);
    } else {
        if (d.pos_critic[t] < 0) { d.pos_critic[t] = c.critic_count; d.critic_list[c.critic_count++] = t; }
        list_remove(d.actor_list, d.pos_actor, c.actor_count, t);
    }
    for (int k = 0; k < c.actor_batch_count;) {        // the overwritten slot leaves the pending actor batch
        if (d.actor_batch[k] == t) d.actor_batch[k] = d.actor_batch[--c.actor_batch_count];
        else ++k;
    }
    return t;
}
// One batch of up to 32 incoming tuples in arrival order, one per lane (lane order = arrival order): `take` = the lane's tuple gets a
// replay slot, `flags` its tuple flags.  Returns the lane's slot (-1 if not taken).  Counters live in lane 0's `c` (a register copy of
// *d.c); every lane's copy is refreshed at the end.  Fast path -- every slot of the batch is fresh (never written: the ring has not
// wrapped onto it): head / list positions are prefix sums over the batch, all stores in parallel, the result is what the sequential
// loop produces.  Otherwise lane 0 runs the sequential cNeuralNetTrainer::AddTuple + cMACETrainer::UpdateBuffers (assign_slot) tuple
// by tuple.  The loads a tuple needs (its slot's list positions) are issued for the whole batch at once instead of one dependent
// L2 round trip after the other (a dependent L2 round trip per tuple made the single-thread loop the bottleneck of the intake).
__device__ int assign_batch(const Dev& d, Counters& c, bool take, uint32_t flags) {
    const unsigned lane = threadIdx.x & 31;
    const unsigned tmask = __ballot_sync(0xffffffffu, take);
    if (tmask == 0) return -1;
    const int pre = __popc(tmask & ((1u << lane) - 1u));
    const int nt = __popc(tmask);
    const int t = (int)(((long long)c.head + pre) % d.cap);
    const int pa = take ? d.pos_actor[t] : -1, pc = take ? d.pos_critic[t] : -1;
    const bool fresh = __all_sync(0xffffffffu, !take || (pa < 0 && pc < 0)) && nt <= d.cap;
    int slot = -1;
    if (fresh) {
        const bool ea = take && (flags & 4u) != 0, ec = take && !ea;       // eFlagExpActor -> actor buffer, else critic buffer
        const unsigned am = __ballot_sync(0xffffffffu, ea), cm = __ballot_sync(0xffffffffu, ec);
        if (ea) { const int q = c.actor_count + __popc(am & ((1u << lane) - 1u)); d.pos_actor[t] = q; d.actor_list[q] = t; }
        if (ec) { const int q = c.critic_count + __popc(cm & ((1u << lane) - 1u)); d.pos_critic[t] = q; d.critic_list[q] = t; }
        c.actor_count += __popc(am); c.critic_count += __popc(cm);
        c.head = (int)(((long long)c.head + nt) % d.cap);
        c.num = min(d.cap, c.num + nt);
        c.total += nt;
        if (take) slot = t;
    } else if (d.cap >= 64) {
        // The ring has wrapped onto used slots (the steady state of a long run): the reference's sequential order matters -- a slot
        // moves between the critic and the actor list by swap-remove + append, and leaves the pending actor batch.  Lane 0 walks the
        // batch in arrival order on shared-memory copies of everything the walk can touch: the list positions of the batch's own
        // slots, a 64-entry window around either list's tail (all reads are tail reads), the pending actor batch.  Stores that fall
        // outside go to memory directly (nothing in the batch reads them back); the copies are written back at the end.
        __shared__ int w_list[2][64], w_pos[2][32], w_ab[4 * kB], w_slot[32], w_hit[32];
        __shared__ uint32_t w_flags[32];
        const int head0 = c.head;
        const int base0 = max(0, c.critic_count - 32), base1 = max(0, c.actor_count - 32);
        for (int k = lane; k < 64; k += 32) {
            w_list[0][k] = base0 + k < d.cap ? d.critic_list[base0 + k] : -1;
            w_list[1][k] = base1 + k < d.cap ? d.actor_list[base1 + k] : -1;
        }
        w_hit[lane] = 0;
        __syncwarp();
        for (int k = lane; k < 4 * kB; k += 32) {
            const int v = k < c.actor_batch_count ? d.actor_batch[k] : -1;
            w_ab[k] = v;
            if (v >= 0) {                                  // which of the batch's slots sit in the pending actor batch (rare): only those scan it
                int bl = v - head0;
                if (bl < 0) bl += d.cap;
                if (bl < nt) w_hit[bl] = 1;
            }
        }
        if (take) { w_pos[0][pre] = pc; w_pos[1][pre] = pa; w_flags[pre] = flags; }
        __syncwarp();
        if (lane == 0) {
            int cnt[2] = {c.critic_count, c.actor_count};
            const int wbase[2] = {base0, base1};
            int* lists[2] = {d.critic_list, d.actor_list};
            int* poss[2] = {d.pos_critic, d.pos_actor};
            int abc = c.actor_batch_count;
            for (int bi = 0; bi < nt; ++bi) {
                int tq = head0 + bi;                                           // head0 < cap, bi < 32 <= cap
                if (tq >= d.cap) tq -= d.cap;
                const int nl = (w_flags[bi] & 4u) ? 1 : 0, ol = 1 - nl;       // eFlagExpActor -> actor list (1), else critic list (0)
                if (w_pos[nl][bi] < 0) {                                       // append to the list it belongs to now
                    const int k = cnt[nl] - wbase[nl];
                    w_pos[nl][bi] = cnt[nl];
                    if (k >= 0 && k < 64) w_list[nl][k] = tq; else lists[nl][cnt[nl]] = tq;
                    ++cnt[nl];
                }
                const int pq = w_pos[ol][bi];
                if (pq >= 0) {                                                 // list_remove from the other one (swap with its tail)
                    const int kl = cnt[ol] - 1 - wbase[ol];
                    const int last = (kl >= 0 && kl < 64) ? w_list[ol][kl] : lists[ol][cnt[ol] - 1];
                    const int kp = pq - wbase[ol];
                    if (kp >= 0 && kp < 64) w_list[ol][kp] = last; else lists[ol][pq] = last;
                    int bl = last - head0;
                    if (bl < 0) bl += d.cap;
                    if (bl < nt) w_pos[ol][bl] = pq; else poss[ol][last] = pq;
                    w_pos[ol][bi] = -1;
                    --cnt[ol];
                }
                if (w_hit[bi]) {
                    for (int k = 0; k < abc;) {                                // the overwritten slot leaves the pending actor batch
                        if (w_ab[k] == tq) w_ab[k] = w_ab[--abc];
                        else ++k;
                    }
                }
                w_slot[bi] = tq;
            }
            c.critic_count = cnt[0]; c.actor_count = cnt[1]; c.actor_batch_count = abc;
            c.head = head0 + nt >= d.cap ? head0 + nt - d.cap : head0 + nt;
            c.num = min(d.cap, c.num + nt);
            c.total += nt;
        }
        __syncwarp();
        for (int k = lane; k < 64; k += 32) {
            if (base0 + k < d.cap) d.critic_list[base0 + k] = w_list[0][k];
            if (base1 + k < d.cap) d.actor_list[base1 + k] = w_list[1][k];
        }
        for (int k = lane; k < 4 * kB; k += 32) if (w_ab[k] >= 0 || k < 4 * kB) d.actor_batch[k] = w_ab[k];
        if (take) { d.pos_critic[t] = w_pos[0][pre]; d.pos_actor[t] = w_pos[1][pre]; slot = w_slot[pre]; }
        c.head = __shfl_sync(0xffffffffu, c.head, 0); c.num = __shfl_sync(0xffffffffu, c.num, 0);
        c.total = __shfl_sync(0xffffffffu, c.total, 0);
        c.actor_count = __shfl_sync(0xffffffffu, c.actor_count, 0); c.critic_count = __shfl_sync(0xffffffffu, c.critic_count, 0);
        c.actor_batch_count = __shfl_sync(0xffffffffu, c.actor_batch_count, 0);
        __syncwarp();
    } else {
        // tiny replay memories (tests): the sequential loop against memory
        __syncwarp();
        for (int q = 0; q < 32; ++q) {
            if (!((tmask >> q) & 1u)) continue;
            const uint32_t fq = __shfl_sync(0xffffffffu, flags, q);
            int tq = 0;
            if (lane == 0) tq = assign_slot(d, c, fq);
            tq = __shfl_sync(0xffffffffu, tq, 0);
            if ((int)lane == q) slot = tq;
        }
        c.head = __shfl_sync(0xffffffffu, c.head, 0); c.num = __shfl_sync(0xffffffffu, c.num, 0);
        c.total = __shfl_sync(0xffffffffu, c.total, 0);
        c.actor_count = __shfl_sync(0xffffffffu, c.actor_count, 0); c.critic_count = __shfl_sync(0xffffffffu, c.critic_count, 0);
        c.actor_batch_count = __shfl_sync(0xffffffffu, c.actor_batch_count, 0);
        __syncwarp();
    }
    return slot;
}
// cNeuralNetTrainer::AddTuple slot assignment + cMACETrainer::UpdateBuffers, in arrival order (one thread: O(1) per tuple)
__global__ void k_add_assign(Dev d, const uint32_t* src_flags, const int* count_ptr, int count_val, int max_count, int* reset_count, int use_order) {
    pdl_sync();
    if (blockIdx.x != 0 || threadIdx.x >= 32) return;
    const int lane = threadIdx.x;
    const int count = count_ptr ? min(*count_ptr, max_count) : count_val;
    Counters c = *d.c;                                     // register copy, written back once
    for (int base = 0; base < count; base += 32) {
        const int r = base + lane;
        const bool in = r < count;
        const int i = in ? (use_order ? d.order[r] : r) : 0;
        const bool take = in && d.valid[i] != 0;
        const uint32_t f = take ? src_flags[i] : 0u;
        const int t = assign_batch(d, c, take, f);
        if (in) d.slot[i] = t;
    }
    if (lane == 0) {
        Counters& g = *d.c;
        g.head = c.head; g.num = c.num; g.total = c.total; g.actor_count = c.actor_count; g.critic_count = c.critic_count;
        g.actor_batch_count = c.actor_batch_count;
        g.add_count = count;                               // k_add_copy must not re-read a counter that is reset here
        if (reset_count) *reset_count = 0;                 // cScenarioExp::ResetTupleBuffer
    }
}
__global__ void k_add_copy(Dev d, const double* rows, const uint32_t* src_flags) {
    pdl_sync();
    const int count = d.c->add_count;
    const int i = blockIdx.x;
    if (i >= count) return;
    const int t = d.slot[i];
    if (t < 0) return;
    const double* r = rows + (size_t)i * d.Wd;
    float* dst = d.mem + (size_t)t * d.Wd;
    for (int k = threadIdx.x; k < d.Wd; k += blockDim.x) dst[k] = (float)r[k];     // SetTuple stores floats
    if (threadIdx.x == 0) d.flags[t] = (int)src_flags[i];
}

// ---- the slot-filtered hand-over of a handle with training slots (trl_train_run_slots): trainer p takes the rows whose env is on
// policy slot p, in the order of its envs' ids, and leaves the rest of the block to the other trainers.  k_add_assign / k_add_copy
// serve it unchanged: the slot's rows come first in d.order, every other row is invalid and takes no replay slot, so the replay memory
// sees exactly the batches of 32 a single trainer fed only this slot's rows (in env order) sees.
struct SlotRows { const int* env_ids; const int* env_slot; int slot; };
__device__ __forceinline__ bool slot_row(const SlotRows& s, int i) { return s.env_slot[s.env_ids[i]] == s.slot; }
__global__ void k_add_check_slot(Dev d, const double* rows, const int* count_ptr, SlotRows s) {
    pdl_sync();
    const int count = min(*count_ptr, (int)gridDim.x), i = blockIdx.x;
    if (i >= count) return;
    const double* r = rows + (size_t)i * d.Wd;
    const bool mine = slot_row(s, i);
    int bad = !mine;
    if (mine)
        for (int k = threadIdx.x; k < d.Wd; k += blockDim.x) bad |= !isfinite(r[k]);
    bad = __syncthreads_or(bad);
    if (threadIdx.x == 0) d.valid[i] = !bad;
}
// rank = #rows of the same slot with a smaller env id; the other rows are ranked after all of them (key bit 30)
__global__ void k_add_order_slot(Dev d, const int* count_ptr, SlotRows s) {
    pdl_sync();
    const int count = min(*count_ptr, (int)gridDim.x), i = blockIdx.x;
    if (i >= count) return;
    const int key = s.env_ids[i] | (slot_row(s, i) ? 0 : 0x40000000);
    int r = 0;
    for (int j = threadIdx.x; j < count; j += blockDim.x) {
        const int kj = s.env_ids[j] | (slot_row(s, j) ? 0 : 0x40000000);
        r += (kj < key) || (kj == key && j < i);
    }
    __shared__ int red[32];
    for (int o = 16; o > 0; o >>= 1) r += __shfl_xor_sync(0xffffffffu, r, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = r;
    __syncthreads();
    if (threadIdx.x == 0) {
        int tot = 0;
        for (int w = 0; w < (int)(blockDim.x >> 5); ++w) tot += red[w];
        d.order[tot] = i;
    }
}

// ---- tuples from the all-gathered blocks of every rank (trl_comm.cu: {i32 count, i32 queued, i32 rank, i32 R, u32 flags[R],
// i32 env[R], f32 rows[R][Wd]} per rank).  Arrival order = rank order, env order inside a rank: the same on every rank, so
// replicated trainers stay bit-identical.  The validity bit (cNeuralNetTrainer::CheckTuple on the f64 values) was set by the
// pack kernel; rows are already the floats SetTuple would store.  Flat index i = rank * R + j for valid/slot/order.
struct GBlocks { const unsigned char* recv; size_t block_bytes; int R, world; };
__device__ __forceinline__ const int* gb_hdr(const GBlocks& g, int r) { return (const int*)(g.recv + (size_t)r * g.block_bytes); }
__device__ __forceinline__ const uint32_t* gb_flags(const GBlocks& g, int r) { return (const uint32_t*)(g.recv + (size_t)r * g.block_bytes + 16); }
__device__ __forceinline__ const int* gb_env(const GBlocks& g, int r) { return (const int*)(g.recv + (size_t)r * g.block_bytes + 16 + (size_t)4 * g.R); }
__device__ __forceinline__ const float* gb_rows(const GBlocks& g, int r) { return (const float*)(g.recv + (size_t)r * g.block_bytes + 16 + (size_t)8 * g.R); }
// In a handle with training slots the gathered intake of trainer `slot` takes only the rows whose flag bits 24..26 name its slot
// (kSlot): they are ranked first inside each block, by env id, the other rows after them; those are invalid and take no replay slot,
// so the replay memory sees what a single trainer fed only this slot's rows (rank order, env order inside a rank) sees.  The plain
// order and copy kernels are the kSlot = false instances (their SASS is the one they had as plain kernels).
__device__ __forceinline__ bool gb_mine(uint32_t f, int slot) { return (int)((f >> 24) & 7u) == slot; }
// grid (R, world): rank of tuple j inside its block by env id -> d.order[r * R + rank_in_block] = j
template <bool kSlot>
__device__ __forceinline__ void addg_order(const Dev& d, const GBlocks& g, int slot) {
    pdl_sync();
    const int r = blockIdx.y, i = blockIdx.x;
    const int count = min(max(gb_hdr(g, r)[0], 0), g.R);
    if (i >= count) return;
    const int* env = gb_env(g, r);
    const uint32_t* fl = gb_flags(g, r);
    const int key = kSlot ? env[i] | (gb_mine(fl[i], slot) ? 0 : 0x40000000) : env[i];
    int rk = 0;
    for (int j = threadIdx.x; j < count; j += blockDim.x) {
        const int kj = kSlot ? env[j] | (gb_mine(fl[j], slot) ? 0 : 0x40000000) : env[j];
        rk += (kj < key) || (kj == key && j < i);
    }
    __shared__ int red[32];
    for (int o = 16; o > 0; o >>= 1) rk += __shfl_xor_sync(0xffffffffu, rk, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = rk;
    __syncthreads();
    if (threadIdx.x == 0) {
        int tot = 0;
        for (int w = 0; w < (int)(blockDim.x >> 5); ++w) tot += red[w];
        d.order[r * g.R + tot] = i;
    }
}
__global__ void k_addg_assign(Dev d, GBlocks g) {
    pdl_sync();
    if (blockIdx.x != 0 || threadIdx.x >= 32) return;
    const int lane = threadIdx.x;
    Counters c = *d.c;
    int total = 0;
    for (int r = 0; r < g.world; ++r) {
        const int count = min(max(gb_hdr(g, r)[0], 0), g.R);
        const uint32_t* flags = gb_flags(g, r);
        for (int base = 0; base < count; base += 32) {
            const int k = base + lane;
            const bool in = k < count;
            const int j = in ? d.order[r * g.R + k] : 0;
            const uint32_t f = in ? flags[j] : 0x80000000u;
            const bool take = in && !(f & 0x80000000u);
            const int t = assign_batch(d, c, take, f);
            if (in) d.slot[r * g.R + j] = t;
        }
        total += count;
    }
    if (lane == 0) {
        Counters& gc = *d.c;
        gc.head = c.head; gc.num = c.num; gc.total = c.total; gc.actor_count = c.actor_count; gc.critic_count = c.critic_count;
        gc.actor_batch_count = c.actor_batch_count;
        gc.add_count = total;
    }
}
// k_addg_assign with the slot filter, written out rather than shared: as one template the plain instance compiled to other SASS
__global__ void k_addg_assign_slot(Dev d, GBlocks g, int slot) {
    pdl_sync();
    if (blockIdx.x != 0 || threadIdx.x >= 32) return;
    const int lane = threadIdx.x;
    Counters c = *d.c;
    int total = 0;
    for (int r = 0; r < g.world; ++r) {
        const int count = min(max(gb_hdr(g, r)[0], 0), g.R);
        const uint32_t* flags = gb_flags(g, r);
        for (int base = 0; base < count; base += 32) {
            const int k = base + lane;
            const bool in = k < count;
            const int j = in ? d.order[r * g.R + k] : 0;
            const uint32_t f = in ? flags[j] : 0x80000000u;
            const bool take = in && !(f & 0x80000000u) && gb_mine(f, slot);
            const int t = assign_batch(d, c, take, f);
            if (in) d.slot[r * g.R + j] = t;
        }
        total += count;
    }
    if (lane == 0) {
        Counters& gc = *d.c;
        gc.head = c.head; gc.num = c.num; gc.total = c.total; gc.actor_count = c.actor_count; gc.critic_count = c.critic_count;
        gc.actor_batch_count = c.actor_batch_count;
        gc.add_count = total;
    }
}
template <bool kSlot>
__device__ __forceinline__ void addg_copy(const Dev& d, const GBlocks& g) {
    pdl_sync();
    const int r = blockIdx.y, j = blockIdx.x;
    const int count = min(max(gb_hdr(g, r)[0], 0), g.R);
    if (j >= count) return;
    const int t = d.slot[r * g.R + j];
    if (t < 0) return;
    const float* src = gb_rows(g, r) + (size_t)j * d.Wd;
    float* dst = d.mem + (size_t)t * d.Wd;
    for (int k = threadIdx.x; k < d.Wd; k += blockDim.x) dst[k] = src[k];
    if (threadIdx.x == 0) d.flags[t] = (int)(gb_flags(g, r)[j] & (kSlot ? 0x00ffffffu : 0x7fffffffu));
}
__global__ void k_addg_order(Dev d, GBlocks g) { addg_order<false>(d, g, 0); }
__global__ void k_addg_copy(Dev d, GBlocks g) { addg_copy<false>(d, g); }
__global__ void k_addg_order_slot(Dev d, GBlocks g, int slot) { addg_order<true>(d, g, slot); }
__global__ void k_addg_copy_slot(Dev d, GBlocks g) { addg_copy<true>(d, g); }

// ================================================================================================ stage switch
__global__ void k_stage_check(Dev d) {
    pdl_sync();
    Counters& c = *d.c;
    c.init_now = 0;
    c.succ = 0;
    if (c.stage == 0) {
        const int nis = min(d.nis, d.cap);
        if (c.num >= nis && c.num > 0) c.init_now = (nis > 1 && d.init_offset_scale) ? 1 : 2;   // 2: switch without refit
    }
}
// cNeuralNet::CalcOffsetScale (learning/NeuralNet.cpp:280-313) over the state-begin columns of the replay memory
__global__ void k_col_mean(Dev d) {
    pdl_sync();
    if (d.c->init_now != 1) return;
    const int j = blockIdx.x, num = d.c->num;
    double s = 0;
    for (int t = threadIdx.x; t < num; t += blockDim.x) s += (double)d.mem[(size_t)t * d.Wd + 1 + j];
    __shared__ double red[32];
    s = warp_sum(s);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        double tot = 0;
        for (int w = 0; w < (int)(blockDim.x >> 5); ++w) tot += red[w];
        d.mean[j] = tot / num;
    }
}
__global__ void k_col_scale(Dev d) {
    pdl_sync();
    if (d.c->init_now != 1) return;
    const int j = blockIdx.x, num = d.c->num;
    const double m = d.mean[j];
    double s = 0;
    for (int t = threadIdx.x; t < num; t += blockDim.x) { double x = (double)d.mem[(size_t)t * d.Wd + 1 + j] - m; s += x * x; }
    __shared__ double red[32];
    s = warp_sum(s);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        double tot = 0;
        for (int w = 0; w < (int)(blockDim.x >> 5); ++w) tot += red[w];
        const double sd = sqrt(tot / num);
        d.in_off[j] = -m; d.in_scale[j] = sd == 0 ? 0 : 1.0 / sd;
        d.t_in_off[j] = d.in_off[j]; d.t_in_scale[j] = d.in_scale[j];       // SetInputOffsetScale reaches every net of the pool
    }
}
__global__ void k_stage_commit(Dev d) {
    pdl_sync();
    if (d.c->init_now) d.c->stage = 1;
}

// ================================================================================================ sampling
// cMACETrainer::FetchMinibatch (learning/MACETrainer.cpp:164-188)
__global__ void k_sample_critic(Dev d) {
    pdl_sync();
    if (threadIdx.x != 0) return;
    Counters& c = *d.c;
    const bool ok = c.stage == 1 && c.critic_count >= kB;
    c.critic_ok = ok;
    c.succ = ok;
    if (!ok) return;
    for (int i = 0; i < kB; ++i) d.ids[i] = d.critic_list[rand_int(d, 0, c.critic_count)];
}
// cMACETrainer::FetchActorMinibatch (learning/MACETrainer.cpp:190-214)
__global__ void k_sample_actor(Dev d) {
    pdl_sync();
    if (threadIdx.x != 0) return;
    Counters& c = *d.c;
    c.cand_count = 0;
    c.actor_ok = 0;
    if (c.stage != 1) return;
    const int n_exp = c.actor_count, ns = min(kB, n_exp);
    int nc = 0;
    for (int i = 0; i < ns; ++i) {
        const int t = d.actor_list[rand_int(d, 0, n_exp)];
        bool contains = false;
        for (int k = 0; k < c.actor_batch_count && !contains; ++k) contains = d.actor_batch[k] == t;
        for (int k = 0; k < nc && !contains; ++k) contains = d.cand[k] == t;
        if (!contains) d.cand[nc++] = t;
    }
    c.cand_count = nc;
    for (int i = 0; i < kB; ++i) d.ids2[i] = nc > 0 ? d.cand[i < nc ? i : 0] : 0;   // pad the batch with the first candidate
}
// UpdateActorBatchBuffer's test (learning/MACETrainer.cpp:556-573) + the batch for cMACETrainer::StepActor
__global__ void k_actor_select(Dev d) {
    pdl_sync();
    if (threadIdx.x != 0) return;
    Counters& c = *d.c;
    if (c.stage != 1) return;
    for (int i = 0; i < c.cand_count; ++i)
        if (d.v1[i] > d.v0[i]) d.actor_batch[c.actor_batch_count++] = d.cand[i];
    c.actor_ok = c.actor_batch_count >= kB;
    if (c.actor_ok)
        for (int i = 0; i < kB; ++i) d.ids[i] = d.actor_batch[i];
}
__global__ void k_actor_pop(Dev d) {
    pdl_sync();
    if (threadIdx.x != 0) return;
    Counters& c = *d.c;
    if (!c.actor_ok) return;
    for (int i = kB; i < c.actor_batch_count; ++i) d.actor_batch[i - kB] = d.actor_batch[i];
    c.actor_batch_count -= kB;
    ++c.actor_iter;
}
__global__ void k_end_iter(Dev d) {
    pdl_sync();
    if (threadIdx.x == 0 && d.c->succ) ++d.c->iter;       // cNeuralNetTrainer::ApplySteps / IncIter
}
// cMACETrainer::Step's target refresh (learning/MACETrainer.cpp:350-358): uses the iteration count before IncIter
__global__ void k_target_update(Dev d) {
    pdl_sync();
    const Counters& c = *d.c;
    if (!(c.stage == 1 && d.freeze > 0 && c.iter > 0 && c.iter % d.freeze == 0)) return;
    const int stride = gridDim.x * blockDim.x, tid = blockIdx.x * blockDim.x + threadIdx.x;
    for (int i = tid; i < d.P; i += stride) d.target[i] = d.theta[i];
    for (int i = tid; i < d.S; i += stride) { d.t_in_off[i] = d.in_off[i]; d.t_in_scale[i] = d.in_scale[i]; }
    for (int i = tid; i < d.n_out; i += stride) { d.t_out_off[i] = d.out_off[i]; d.t_out_scale[i] = d.out_scale[i]; }
}

// ================================================================================================ forward
// rows ids[0..kB) of the replay memory, columns [col0, col0 + S), normalised like cNeuralNet::NormalizeInput
// (a launch of 2 kB or 3 kB blocks stacks further blocks of kB rows under the first: block b takes the columns starting at
// col0 / col1 / col2 and, where bit b of ids2_mask is set, the candidate ids d.ids2 instead of d.ids)
__global__ void k_gather_norm(Dev d, int pred, int col0, int col1, int col2, int ids2_mask, const double* in_off, const double* in_scale) {
    pdl_sync();
    if (!pred_on(d, pred)) return;
    const int n = blockIdx.x, b = n / kB;
    const int* ids = ((ids2_mask >> b) & 1) ? d.ids2 : d.ids;
    const float* r = d.mem + (size_t)ids[n % kB] * d.Wd + (b == 0 ? col0 : (b == 1 ? col1 : col2));
    for (int i = threadIdx.x; i < d.S; i += blockDim.x) d.xn[(size_t)n * d.S + i] = ((double)r[i] + in_off[i]) * in_scale[i];
}

// ================================================================================================ labels + loss
// max over the critic outputs of the un-normalised target-net output (GetMaxFragValAux) -> v0 (state begin) or the Bellman
// value r (1 - gamma) + gamma max V'(s') -> v1 (CalcNewCumulativeRewardBatch, learning/MACETrainer.cpp:472-513)
__global__ void k_vals(Dev d, int pred, int with_reward, double* out, int row0, int use_ids2) {
    pdl_sync();
    if (!pred_on(d, pred)) return;
    const int n = threadIdx.x;
    if (n >= kB) return;
    double m = -INFINITY;
    for (int f = 0; f < d.n_frags; ++f) m = fmax(m, d.y[(size_t)(row0 + n) * d.n_out + f] / d.t_out_scale[f] - d.t_out_off[f]);
    if (with_reward) {
        const int t = use_ids2 ? d.ids2[n] : d.ids[n];
        const double r = (double)d.mem[(size_t)t * d.Wd] * (1.0 - d.discount);
        m = (d.flags[t] & 1) ? r : r + d.discount * m;       // eFlagFail
    }
    out[n] = m;
}
// BuildProblemY / BuildActorProblemY + LoadTrainData's label normalisation + EuclideanLoss gradient.
// mode 0: critic (value of the taken actor <- v1), mode 1: actor (fragment of the taken actor <- the action taken)
__global__ void k_labels(Dev d, int pred, int mode) {
    pdl_sync();
    if (!pred_on(d, pred)) return;
    const int no = d.n_out;
    double part = 0;
    for (int idx = threadIdx.x; idx < kB * no; idx += blockDim.x) {
        const int n = idx / no, j = idx - n * no;
        const float* r = d.mem + (size_t)d.ids[n] * d.Wd;
        const int a = (int)r[1 + d.S];
        const double yraw = d.y[idx];
        double Y = yraw / d.out_scale[j] - d.out_off[j];                         // cNeuralNet::EvalBatch un-normalises
        if (mode == 0) { if (j == a) Y = d.v1[n]; }
        else if (j >= d.n_frags + a * d.frag && j < d.n_frags + (a + 1) * d.frag) Y = (double)r[1 + d.S + 1 + (j - d.n_frags - a * d.frag)];
        const double lab = (Y + d.out_off[j]) * d.out_scale[j];                  // LoadTrainData normalises again
        const double df = yraw - lab;
        part += df * df;
        d.dy[idx] = df / kB;
    }
    __shared__ double red[32];
    part = warp_sum(part);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = part;
    __syncthreads();
    if (threadIdx.x == 0) {
        double tot = 0;
        for (int w = 0; w < (int)(blockDim.x >> 5); ++w) tot += red[w];
        (mode == 0 ? d.c->critic_loss : d.c->actor_loss) = tot / (2.0 * kB);
    }
}

// ================================================================================================ backward
// The four backward operations are written as bodies over explicit block / thread coordinates, so that k_bwd_multi (further down)
// can run several independent bodies in ONE launch (blocks of 256 threads).
// dw[o][i] = sum_n dy[n][o] x[n][i], db[o] = sum_n dy[n][o].  grid (nout, ceil(nin / nthreads))
__device__ __forceinline__ void fc_bwd_w_body(int bx, int by, int tid, int nthreads, const double* dy, int ldy, const double* x, int ldx, int nin,
                                              double* dw, double* db) {
    __shared__ double dys[kB];
    const int o = bx;
    if (tid < kB) dys[tid] = dy[(size_t)tid * ldy + o];
    __syncthreads();
    const int i = by * nthreads + tid;
    if (i < nin) {
        double s = 0;
#pragma unroll
        for (int n = 0; n < kB; ++n) s += dys[n] * x[(size_t)n * ldx + i];
        dw[(size_t)o * nin + i] = s;
    }
    if (by == 0 && tid == 0) {
        double s = 0;
        for (int n = 0; n < kB; ++n) s += dys[n];
        db[o] = s;
    }
}
// dx[n][i] (=|+=) mask(act[n][i]) * sum_o dy[n][o] w[o][i] for i < ncols.  grid (ceil(ncols / 32), kB), block (32, 8): the
// output neurons are split over ty and reduced through shared memory in a fixed order.  `heads` > 1: the sum over several
// (dy, w) pairs (dy at stride dy_stride, w from w_heads), accumulated head after head in head order.
__device__ __forceinline__ void fc_bwd_x_body(int bx, int by, int tx, int ty, const double* dy, int ldy, int nout, const double* w, int nin, int ncols,
                                              const double* act, int lda, double* dx, int ldx, int accumulate, int heads, size_t dy_stride,
                                              const double* const* w_heads) {
    __shared__ double dys[H];
    __shared__ double part[8][33];
    const int n = by;
    const int i = bx * 32 + tx;
    double acc = 0;
    for (int hd = 0; hd < heads; ++hd) {
        const double* dyh = dy + (size_t)hd * dy_stride;
        const double* wh = w_heads ? w_heads[hd] : w;
        if (hd > 0) __syncthreads();                       // dys / part of the previous head have been consumed
        for (int o = ty * 32 + tx; o < nout; o += 256) dys[o] = dyh[(size_t)n * ldy + o];
        __syncthreads();
        double s = 0;
        if (i < ncols)
            for (int o = ty; o < nout; o += 8) s += dys[o] * wh[(size_t)o * nin + i];
        part[ty][tx] = s;
        __syncthreads();
        if (ty == 0 && i < ncols) {
            double tot = 0;
#pragma unroll
            for (int q = 0; q < 8; ++q) tot += part[q][tx];
            if (act && !(act[(size_t)n * lda + i] > 0)) tot = 0;
            if (hd == 0) acc = tot; else acc += tot;
        }
    }
    if (ty == 0 && i < ncols) {
        if (accumulate) dx[(size_t)n * ldx + i] += acc; else dx[(size_t)n * ldx + i] = acc;
    }
}
// dw[o][c][kk] = sum_{n,t} dy[n][o][t] x[n][c][t + kk]; db[o] = sum dy[n][o][t].  grid (cin, cout)
__device__ __forceinline__ void conv_bwd_w_body(int bx, int by, int tid, int nthreads, const double* dy, int cout, int k, const double* x, int ldn,
                                                int cin, int win, double* dw, double* db) {
    const int c = bx, o = by, wout = win - k + 1;
    double acc[K0 + 1];
#pragma unroll
    for (int kk = 0; kk <= K0; ++kk) acc[kk] = 0.0;
    for (int idx = tid; idx < kB * wout; idx += nthreads) {
        const int n = idx / wout, t = idx - n * wout;
        const double g = dy[((size_t)n * cout + o) * wout + t];
        const double* xr = x + (size_t)n * ldn + (size_t)c * win + t;
#pragma unroll
        for (int kk = 0; kk < K0; ++kk)
            if (kk < k) acc[kk] += g * xr[kk];
        acc[K0] += g;
    }
    __shared__ double red[8][K0 + 1];
#pragma unroll
    for (int kk = 0; kk <= K0; ++kk) {
        double v = warp_sum(acc[kk]);
        if ((tid & 31) == 0) red[tid >> 5][kk] = v;
    }
    __syncthreads();
    if (tid <= K0) {
        double s = 0;
        for (int wq = 0; wq < (nthreads >> 5); ++wq) s += red[wq][tid];
        if (tid < k) dw[((size_t)o * cin + c) * k + tid] = s;
        else if (tid == K0 && c == 0) db[o] = s;
    }
}
// dx[n][c][s] = mask * sum_{o,kk} dy[n][o][s - kk] w[o][c][kk].  grid (cin, kB), one thread per input position
__device__ __forceinline__ void conv_bwd_x_body(int bx, int by, int tid, int nthreads, const double* dy, int cout, int k, const double* w, int cin,
                                                int win, const double* act, double* dx) {
    __shared__ double ws[C2 * K2];            // cout * k <= 128
    const int c = bx, n = by, wout = win - k + 1;
    for (int i = tid; i < cout * k; i += nthreads) { int o = i / k, kk = i - o * k; ws[i] = w[((size_t)o * cin + c) * k + kk]; }
    __syncthreads();
    const int s = tid;
    if (s >= win) return;
    double acc = 0;
    for (int o = 0; o < cout; ++o) {
        const double* g = dy + ((size_t)n * cout + o) * wout;
        for (int kk = 0; kk < k; ++kk) {
            const int t = s - kk;
            if (t >= 0 && t < wout) acc += g[t] * ws[o * k + kk];
        }
    }
    const size_t idx = ((size_t)n * cin + c) * win + s;
    dx[idx] = (act[idx] > 0) ? acc : 0;
}
// Several independent backward bodies in one launch (fewer, fatter launches: one launch per body and layer of a batch-32 step
// would be bound by launch latency).  Blocks of 256 threads; job q owns `blocks` consecutive blocks, laid out as a gx x gy grid of
// that body.  Each body's per-element arithmetic and summation order do not depend on which jobs share its launch.
enum JobKind { J_FC_BWD_W = 0, J_FC_BWD_X, J_FC_BWD_X_HEADS, J_CONV_BWD_W, J_CONV_BWD_X };
struct Job {
    int kind, blocks, gx;
    const double *dy, *a, *act;          // a: x (bwd_w) or w (bwd_x)
    double *o0, *o1;                     // dw / dx, db
    int i0, i1, i2, i3, i4, i5, i6;
    const double* wh[4];                 // J_FC_BWD_X_HEADS: the four heads' weights
};
constexpr int kMaxJobs = 8;
struct JobList { int n; Job j[kMaxJobs]; };
__global__ void __launch_bounds__(256) k_bwd_multi(Dev d, int pred, JobList jl) {
    pdl_sync();
    if (!pred_on(d, pred)) return;
    int b = blockIdx.x, q = 0;
    while (q < jl.n - 1 && b >= jl.j[q].blocks) { b -= jl.j[q].blocks; ++q; }
    const Job& J = jl.j[q];
    const int bx = b % J.gx, by = b / J.gx, tid = threadIdx.x;
    switch (J.kind) {
        case J_FC_BWD_W: fc_bwd_w_body(bx, by, tid, 256, J.dy, J.i0, J.a, J.i1, J.i2, J.o0, J.o1); break;                       // ldy, ldx, nin
        case J_FC_BWD_X: fc_bwd_x_body(bx, by, tid & 31, tid >> 5, J.dy, J.i0, J.i1, J.a, J.i2, J.i3, J.act, J.i4, J.o0, J.i5, J.i6, 1, 0, nullptr); break;
        case J_FC_BWD_X_HEADS: fc_bwd_x_body(bx, by, tid & 31, tid >> 5, J.dy, J.i0, J.i1, nullptr, J.i2, J.i3, J.act, J.i4, J.o0, J.i5, 0, 4, (size_t)J.i6, J.wh); break;
        case J_CONV_BWD_W: conv_bwd_w_body(bx, by, tid, 256, J.dy, J.i0, J.i1, J.a, J.i2, J.i3, J.i4, J.o0, J.o1); break;      // cout, k, ldn, cin, win
        default: conv_bwd_x_body(bx, by, tid, 256, J.dy, J.i0, J.i1, J.a, J.i2, J.i3, J.act, J.o0); break;                      // cout, k, cin, win
    }
}
// Caffe SGDSolver: Regularize (L2) + ComputeUpdateValue + Net::Update, one pass over all 26 blobs
__global__ void k_sgd(Dev d, int pred) {
    pdl_sync();
    if (!pred_on(d, pred)) return;
    const int stride = gridDim.x * blockDim.x;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < d.P; i += stride) {
        int b = 0;
        while (i >= d.off[b + 1]) ++b;
        const double rate = d.base_lr * ((b & 1) ? 2.0 : 1.0);
        const double decay = d.weight_decay * ((b & 1) ? (b < 6 ? 1.0 : 0.0) : 1.0);
        const double g = d.grad[i] + decay * d.theta[i];
        const double hst = rate * g + d.momentum * d.history[i];
        d.history[i] = hst;
        d.theta[i] -= hst;
    }
}

}  // namespace trl_train

// ==================================================================================================== host side
using trl_train::Dev;
using trl_train::Counters;

struct trl_trainer {
    trl_handle* h = nullptr;
    Dev d;
    std::vector<void*> allocs;
    cudaGraphExec_t train_graph = nullptr;
    int64_t graph_launches = 0;        // kernels in train_graph (one training iteration)
    // forward passes run through the batched decision kernels (trl_decide2.cuh): per net the weight views and TMA descriptors
    trl::NetWeights nw[2];             // 0 current net, 1 target net
    trl::FcMaps fmaps[2];
    double* stage_rows = nullptr;      // device staging for tuples handed in from the host
    uint32_t* stage_flags = nullptr;
    int stage_cap = 0;
    long long gather_cap = 0;          // entries of valid / slot / order (>= stage_cap; grown by trl_trainer_add_gathered)
    // asynchronous mode (trl_trainer_set_async; the reference's cAsyncMACETrainer): hand-over and training run on their own stream
    // beside the next update; the scenario evaluates a snapshot of the net that is refreshed between updates
    cudaStream_t async_stream = nullptr;
    cudaEvent_t ev_snap = nullptr, ev_trained = nullptr;
    bool async = false, trained_pending = false, job_pending = false;
    double* snap = nullptr;            // [P + 2 S + 2 n_out]: theta, in_off, in_scale, out_off, out_scale as the decision kernels see them
    cudaStream_t work() const { return async ? async_stream : h->stream; }
    int64_t launches = 0;
    int slot = 0;                      // policy slot whose net this trainer is (0: the handle's own, h->trainer)
    cudaStream_t own_stream = nullptr; // trl_train_run_slots: hand-over + iterations of this trainer beside the other trainers'
    cudaEvent_t ev_own = nullptr;
    double params[10] = {};            // the creation parameters (trl_trainer_create's p[10])
};

#define TCK(call)                                                                                       \
    do {                                                                                                \
        cudaError_t e__ = (call);                                                                       \
        if (e__ != cudaSuccess) return trl_fail(std::string(#call) + ": " + cudaGetErrorString(e__));   \
    } while (0)

namespace {
using namespace trl_train;

template <typename Tp>
cudaError_t talloc(trl_trainer* t, Tp** p, size_t count) {
    cudaError_t e = cudaMalloc((void**)p, std::max<size_t>(count, 1) * sizeof(Tp));
    if (e == cudaSuccess) { t->allocs.push_back(*p); e = cudaMemset(*p, 0, std::max<size_t>(count, 1) * sizeof(Tp)); }
    return e;
}

struct NetRef { const double* theta; const double *in_off, *in_scale; };

// forward pass of the kB rows named by d.ids (replay columns starting at col0) through `net`; activations stay in d.*
// (col1 / col2 >= 0: further blocks of kB rows with the columns starting there ride along; bit b of ids2_mask: block b is taken
// from the candidate ids)
int enqueue_forward(trl_trainer* t, int pred, int col0, const NetRef& net, cudaStream_t st, bool keep_act = true, int col1 = -1, int col2 = -1,
                    int ids2_mask = 0) {
    const Dev& d = t->d;
    const int rows = kB * (1 + (col1 >= 0 ? 1 : 0) + (col2 >= 0 ? 1 : 0));
    launch_pdl(k_gather_norm, dim3(rows), dim3(128), 0, st, d, pred, col0, col1, col2, ids2_mask, net.in_off, net.in_scale);
    // conv stage (one 4-CTA cluster per row, DMMA) + FC stage (one 8-CTA cluster, TMA-fed terr_ip0, DMMA).  Plain stream order on
    // both sides (no programmatic attribute): the pass starts after k_gather_norm has finished and the next kernel's
    // griddepcontrol.wait covers it.
    const int which = net.theta == d.target ? 1 : 0;
    FwdTrain f{};
    f.xn = d.xn; f.rows = rows; f.S = d.S; f.cat = d.cat; f.n_out = d.n_out; f.n_frags = d.n_frags; f.frag = d.frag;
    f.gate = pred == P_CRITIC ? &d.c->critic_ok : pred == P_CAND ? &d.c->cand_count : pred == P_ACTOR ? &d.c->actor_ok : nullptr;
    f.a0 = keep_act ? d.a0 : nullptr; f.a1 = keep_act ? d.a1 : nullptr; f.hh = keep_act ? d.hh : nullptr;
    f.t = d.t; f.catb = d.catb; f.h = d.h; f.y = d.y;
    launch_forward_train(t->nw[which], t->fmaps[which], f, d.a2, st);
    t->launches += 3;
    return 0;
}
// backward of the current net from d.dy (activations of the last forward) into d.grad, then the SGD step
static JobList job_list(std::initializer_list<Job> jobs) {
    JobList jl{};
    for (const Job& j : jobs) jl.j[jl.n++] = j;
    return jl;
}
static int job_blocks(const JobList& jl) { int b = 0; for (int q = 0; q < jl.n; ++q) b += jl.j[q].blocks; return b; }
static Job job_fc_w(const double* dy, int ldy, const double* x, int ldx, int nin, int nout, double* dw, double* db) {
    Job j{}; j.kind = J_FC_BWD_W; j.gx = nout; j.blocks = nout * ((nin + 255) / 256);
    j.dy = dy; j.a = x; j.o0 = dw; j.o1 = db; j.i0 = ldy; j.i1 = ldx; j.i2 = nin;
    return j;
}
static Job job_fc_x(const double* dy, int ldy, int nout, const double* w, int nin, int ncols, const double* act, int lda, double* dx, int ldx, int accumulate) {
    Job j{}; j.kind = J_FC_BWD_X; j.gx = (ncols + 31) / 32; j.blocks = j.gx * kB;
    j.dy = dy; j.a = w; j.act = act; j.o0 = dx; j.i0 = ldy; j.i1 = nout; j.i2 = nin; j.i3 = ncols; j.i4 = lda; j.i5 = ldx; j.i6 = accumulate;
    return j;
}
static Job job_conv_w(const double* dy, int cout, int k, const double* x, int ldn, int cin, int win, double* dw, double* db) {
    Job j{}; j.kind = J_CONV_BWD_W; j.gx = cin; j.blocks = cin * cout;
    j.dy = dy; j.a = x; j.o0 = dw; j.o1 = db; j.i0 = cout; j.i1 = k; j.i2 = ldn; j.i3 = cin; j.i4 = win;
    return j;
}
static Job job_conv_x(const double* dy, int cout, int k, const double* w, int cin, int win, const double* act, double* dx) {
    Job j{}; j.kind = J_CONV_BWD_X; j.gx = cin; j.blocks = cin * kB;
    j.dy = dy; j.a = w; j.act = act; j.o0 = dx; j.i0 = cout; j.i1 = k; j.i2 = cin; j.i3 = win;
    return j;
}
int enqueue_backward_update(trl_trainer* t, int pred, cudaStream_t st) {
    const Dev& d = t->d;
    auto W = [&](int b) { return d.theta + d.off[b]; };
    auto G = [&](int b) { return d.grad + d.off[b]; };
    const int nflat = C2 * W2;
    // 8 launches: independent bodies of one level share a launch; the four heads run side by side (dhh holds one block per head)
    auto multi = [&](const JobList& jl) { launch_pdl(k_bwd_multi, dim3(job_blocks(jl)), dim3(256), 0, st, d, pred, jl); };
    JobList l1{}, l2{};
    int col = 0;
    Job hx{}; hx.kind = J_FC_BWD_X_HEADS; hx.gx = H / 32; hx.blocks = hx.gx * kB;
    hx.dy = d.dhh; hx.act = d.h; hx.o0 = d.dh; hx.i0 = HH; hx.i1 = HH; hx.i2 = H; hx.i3 = H; hx.i4 = H; hx.i5 = H; hx.i6 = kB * HH;
    for (int hd = 0; hd < 4; ++hd) {
        const int nout = hd == 0 ? d.n_frags : d.frag;
        double* hh = d.hh + (size_t)hd * kB * HH;
        double* dhh = d.dhh + (size_t)hd * kB * HH;
        l1.j[l1.n++] = job_fc_w(d.dy + col, d.n_out, hh, HH, HH, nout, G(12 + 4 * hd), G(13 + 4 * hd));
        l1.j[l1.n++] = job_fc_x(d.dy + col, d.n_out, nout, W(12 + 4 * hd), HH, HH, hh, HH, dhh, HH, 0);
        l2.j[l2.n++] = job_fc_w(dhh, HH, d.h, H, H, HH, G(10 + 4 * hd), G(11 + 4 * hd));
        hx.wh[hd] = W(10 + 4 * hd);
        col += nout;
    }
    l2.j[l2.n++] = hx;
    multi(l1);
    multi(l2);
    multi(job_list({job_fc_w(d.dh, H, d.catb, d.cat, d.cat, H, G(8), G(9)), job_fc_x(d.dh, H, H, W(8), d.cat, T, d.t, T, d.dt, T, 0)}));
    multi(job_list({job_fc_w(d.dt, T, d.a2, nflat, nflat, T, G(6), G(7)), job_fc_x(d.dt, T, T, W(6), nflat, nflat, d.a2, nflat, d.da2, nflat, 0)}));
    multi(job_list({job_conv_w(d.da2, C2, K2, d.a1, C1 * W1, C1, W1, G(4), G(5)), job_conv_x(d.da2, C2, K2, W(4), C1, W1, d.a1, d.da1)}));
    multi(job_list({job_conv_w(d.da1, C1, K1, d.a0, C0 * W0, C0, W0, G(2), G(3)), job_conv_x(d.da1, C1, K1, W(2), C0, W0, d.a0, d.da0)}));
    multi(job_list({job_conv_w(d.da0, C0, K0, d.xn, d.S, 1, kTerr, G(0), G(1))}));
    launch_pdl(k_sgd, dim3(296), dim3(256), 0, st, d, pred);
    t->launches += 8;
    return 0;
}
// cNeuralNetTrainer::Train: UpdateStage, then num_steps_per_iter x cMACETrainer::Step, then IncIter
int enqueue_train(trl_trainer* t, cudaStream_t st) {
    const Dev& d = t->d;
    const NetRef cur{d.theta, d.in_off, d.in_scale}, tar{d.target, d.t_in_off, d.t_in_scale};
    const int col_beg = 1, col_end = 1 + d.S + d.A;
    launch_pdl(k_stage_check, dim3(1), dim3(1), 0, st, d);
    launch_pdl(k_col_mean, dim3(d.S), dim3(256), 0, st, d);
    launch_pdl(k_col_scale, dim3(d.S), dim3(256), 0, st, d);
    launch_pdl(k_stage_commit, dim3(1), dim3(1), 0, st, d);
    t->launches += 4;
    for (int s = 0; s < d.steps_per_iter; ++s) {
        // ---- both batches are drawn up front (the draws of k_sample_actor follow those of k_sample_critic in the RNG stream as before;
        // nothing between them consumes a draw or touches what they read), so that everything the frozen TARGET net has to evaluate
        // -- the critic's s', the actor candidates' s and s' -- goes through it in ONE pass of 3 kB rows (three FC clusters side by side)
        launch_pdl(k_sample_critic, dim3(1), dim3(32), 0, st, d);
        launch_pdl(k_sample_actor, dim3(1), dim3(32), 0, st, d);
        enqueue_forward(t, P_ALWAYS, col_end, tar, st, false, col_beg, col_end, 0x6);
        // ---- critic: BuildProblem + UpdateNet (learning/NeuralNetTrainer.cpp:414-456, MACETrainer.cpp:222-247)
        launch_pdl(k_vals, dim3(1), dim3(32), 0, st, d, P_CRITIC, 1, d.v1, 0, 0);
        enqueue_forward(t, P_CRITIC, col_beg, cur, st);
        launch_pdl(k_labels, dim3(1), dim3(256), 0, st, d, P_CRITIC, 0);
        enqueue_backward_update(t, P_CRITIC, st);
        // ---- actor: UpdateActorBatchBuffer + UpdateActor (learning/MACETrainer.cpp:541-626)
        launch_pdl(k_vals, dim3(1), dim3(32), 0, st, d, P_CAND, 0, d.v0, kB, 1);
        launch_pdl(k_vals, dim3(1), dim3(32), 0, st, d, P_CAND, 1, d.v1, 2 * kB, 1);
        launch_pdl(k_actor_select, dim3(1), dim3(32), 0, st, d);
        enqueue_forward(t, P_ACTOR, col_beg, cur, st);
        launch_pdl(k_labels, dim3(1), dim3(256), 0, st, d, P_ACTOR, 1);
        enqueue_backward_update(t, P_ACTOR, st);
        launch_pdl(k_actor_pop, dim3(1), dim3(32), 0, st, d);
        launch_pdl(k_target_update, dim3(132), dim3(256), 0, st, d);
        t->launches += 10;
    }
    launch_pdl(k_end_iter, dim3(1), dim3(32), 0, st, d);
    t->launches += 1;
    return 0;
}

int enqueue_add(trl_trainer* t, const double* rows, const uint32_t* flags, const int* count_ptr, int count_val, int max_count, int* reset,
                cudaStream_t st, const int* env_ids = nullptr) {
    const Dev& d = t->d;
    if (max_count <= 0) return 0;
    launch_pdl(k_add_check, dim3(max_count), dim3(128), 0, st, d, rows, count_ptr, count_val);
    if (env_ids) { launch_pdl(k_add_order, dim3(max_count), dim3(128), 0, st, d, env_ids, count_ptr); t->launches += 1; }
    launch_pdl(k_add_assign, dim3(1), dim3(32), 0, st, d, flags, count_ptr, count_val, max_count, reset, env_ids ? 1 : 0);
    launch_pdl(k_add_copy, dim3(max_count), dim3(128), 0, st, d, rows, flags);
    t->launches += 3;
    return 0;
}
// the hand-over of a handle with training slots: this trainer's slot's rows of the scene's block; the block stays for the others
void enqueue_add_slot(trl_trainer* t, cudaStream_t st) {
    const Dev& d = t->d;
    const trl_handle* h = t->h;
    const int max_count = h->B.tuple_cap;
    const SlotRows s{h->B.tuple_env, h->P.env_slot, t->slot};
    launch_pdl(k_add_check_slot, dim3(max_count), dim3(128), 0, st, d, (const double*)h->B.tuples, (const int*)h->B.tuple_count, s);
    launch_pdl(k_add_order_slot, dim3(max_count), dim3(128), 0, st, d, (const int*)h->B.tuple_count, s);
    launch_pdl(k_add_assign, dim3(1), dim3(32), 0, st, d, (const uint32_t*)h->B.tuple_flags, (const int*)h->B.tuple_count, 0, max_count, (int*)nullptr, 1);
    launch_pdl(k_add_copy, dim3(max_count), dim3(128), 0, st, d, (const double*)h->B.tuples, (const uint32_t*)h->B.tuple_flags);
    t->launches += 4;
}

void trainer_free(trl_trainer* t) {
    for (void* q : t->allocs) cudaFree(q);
    delete t;
}
}  // namespace

extern "C" {

// p[10]: replay_cap, num_init_samples, num_steps_per_iter, freeze_target_iters, init_input_offset_scale, discount, base_lr,
//        momentum, weight_decay, seed   (cTrainerInterface::tParams + the solver prototxt)
// the trainer's dimensions and device buffers; the handle is not touched (nullptr, with the reason recorded, on failure)
static trl_trainer* trainer_new(trl_handle* h, const double* p) {
    auto* t = new trl_trainer();
    t->h = h;
    Dev& d = t->d;
    std::memset(&d, 0, sizeof(d));
    const ModelConst& m = h->mc;
    d.S = m.n_in; d.n_char = m.n_char; d.n_out = m.n_out; d.n_frags = m.n_frags; d.frag = m.frag;
    d.A = 1 + m.frag; d.Wd = 1 + d.S + d.A + d.S; d.cat = T + m.n_char;
    d.cap = (int)p[0]; d.nis = (int)p[1]; d.steps_per_iter = std::max(1, (int)p[2]); d.freeze = (int)p[3];
    d.init_offset_scale = (int)p[4]; d.discount = p[5]; d.base_lr = p[6]; d.momentum = p[7]; d.weight_decay = p[8];
    std::memcpy(t->params, p, sizeof(t->params));
    d.rng_key = trl::mix64((unsigned long long)p[9] ^ trl::mix64(0x7472616eull));     // CounterRng::seed(seed, stream) of the engine, stream tag "tran"
    if (d.S != kTerr + d.n_char || d.cat > 160 || d.n_out != d.n_frags * (1 + d.frag) || d.cap < 2 * kB) {
        trl_fail("trl_trainer_create: unsupported net dimensions / replay capacity");
        delete t;
        return nullptr;
    }
    const int sizes[10] = {C0 * K0, C0, C1 * C0 * K1, C1, C2 * C1 * K2, C2, T * C2 * W2, T, H * d.cat, H};
    d.off[0] = 0;
    for (int b = 0; b < 26; ++b) {
        int sz;
        if (b < 10) sz = sizes[b];
        else {
            const int hd = (b - 10) / 4, r = (b - 10) % 4, nout = hd == 0 ? d.n_frags : d.frag;
            sz = r == 0 ? HH * H : (r == 1 ? HH : (r == 2 ? nout * HH : nout));
        }
        if (sz != (int)h->net_counts[b]) { trl_fail("trl_trainer_create: weight blob sizes do not match the MACE topology"); delete t; return nullptr; }
        d.off[b + 1] = d.off[b] + sz;
    }
    d.P = d.off[26];
    bool ok = true;
    auto A = [&](cudaError_t e) { if (e != cudaSuccess) { if (ok) trl_fail(std::string("trainer alloc: ") + cudaGetErrorString(e)); ok = false; } };
    A(talloc(t, &d.theta, d.P)); A(talloc(t, &d.target, d.P)); A(talloc(t, &d.history, d.P)); A(talloc(t, &d.grad, d.P));
    A(talloc(t, &d.in_off, d.S)); A(talloc(t, &d.in_scale, d.S)); A(talloc(t, &d.out_off, d.n_out)); A(talloc(t, &d.out_scale, d.n_out));
    A(talloc(t, &d.t_in_off, d.S)); A(talloc(t, &d.t_in_scale, d.S)); A(talloc(t, &d.t_out_off, d.n_out)); A(talloc(t, &d.t_out_scale, d.n_out));
    A(talloc(t, &d.mem, (size_t)d.cap * d.Wd)); A(talloc(t, &d.flags, d.cap));
    A(talloc(t, &d.pos_critic, d.cap)); A(talloc(t, &d.pos_actor, d.cap)); A(talloc(t, &d.critic_list, d.cap)); A(talloc(t, &d.actor_list, d.cap));
    A(talloc(t, &d.actor_batch, 4 * kB)); A(talloc(t, &d.c, 1));
    const int add_cap = std::max(h->B.tuple_cap, 4096);
    A(talloc(t, &d.valid, add_cap)); A(talloc(t, &d.slot, add_cap)); A(talloc(t, &d.order, add_cap)); A(talloc(t, &d.ids, kB)); A(talloc(t, &d.ids2, kB)); A(talloc(t, &d.cand, kB));
    // xn, a2, t, catb, h, y hold 3 kB rows: the target net's triple pass (critic s', candidates' s and s' in one launch)
    A(talloc(t, &d.xn, (size_t)3 * kB * d.S)); A(talloc(t, &d.a0, (size_t)kB * C0 * W0)); A(talloc(t, &d.a1, (size_t)kB * C1 * W1));
    A(talloc(t, &d.a2, (size_t)3 * kB * C2 * W2)); A(talloc(t, &d.t, (size_t)3 * kB * T)); A(talloc(t, &d.catb, (size_t)3 * kB * d.cat));
    A(talloc(t, &d.h, (size_t)3 * kB * H)); A(talloc(t, &d.hh, (size_t)4 * kB * HH)); A(talloc(t, &d.y, (size_t)3 * kB * d.n_out));
    A(talloc(t, &d.v0, kB)); A(talloc(t, &d.v1, kB)); A(talloc(t, &d.dy, (size_t)kB * d.n_out)); A(talloc(t, &d.dhh, (size_t)4 * kB * HH));
    A(talloc(t, &d.dh, (size_t)kB * H)); A(talloc(t, &d.dt, (size_t)kB * T)); A(talloc(t, &d.da2, (size_t)kB * C2 * W2));
    A(talloc(t, &d.da1, (size_t)kB * C1 * W1)); A(talloc(t, &d.da0, (size_t)kB * C0 * W0)); A(talloc(t, &d.mean, d.S));
    t->stage_cap = add_cap;
    t->gather_cap = add_cap;
    A(talloc(t, &t->stage_rows, (size_t)add_cap * d.Wd)); A(talloc(t, &t->stage_flags, add_cap));
    if (ok) {
        A(cudaMemset(d.pos_critic, 0xff, (size_t)d.cap * 4));
        A(cudaMemset(d.pos_actor, 0xff, (size_t)d.cap * 4));
    }
    if (!ok) {
        trainer_free(t);
        return nullptr;
    }
    return t;
}
// LoadModel: start from the 26 blobs + 4 offset / scale vectors of `src` (the engine's copy of the slot's policy); the target net is a
// copy.  Then the descriptors of the trainer's own forward passes
static int trainer_start(trl_trainer* t, const std::vector<double*>& src) {
    trl_handle* h = t->h;
    Dev& d = t->d;
    bool ok = true;
    auto A = [&](cudaError_t e) { if (e != cudaSuccess) { if (ok) trl_fail(std::string("trainer load: ") + cudaGetErrorString(e)); ok = false; } };
    cudaStreamSynchronize(h->stream);
    for (int b = 0; b < 26 && ok; ++b) A(cudaMemcpy(d.theta + d.off[b], src[b], (size_t)h->net_counts[b] * 8, cudaMemcpyDeviceToDevice));
    A(cudaMemcpy(d.target, d.theta, (size_t)d.P * 8, cudaMemcpyDeviceToDevice));
    double* dst[8] = {d.in_off, d.in_scale, d.out_off, d.out_scale, d.t_in_off, d.t_in_scale, d.t_out_off, d.t_out_scale};
    for (int k = 0; k < 8 && ok; ++k) A(cudaMemcpy(dst[k], src[26 + (k & 3)], (size_t)h->net_counts[26 + (k & 3)] * 8, cudaMemcpyDeviceToDevice));
    if (!ok) return 1;
    const double* blobs[2][26];            // the blobs of the current net (in theta) and of the target net (in target)
    for (int b = 0; b < 26; ++b) { blobs[0][b] = d.theta + d.off[b]; blobs[1][b] = d.target + d.off[b]; }
    for (int k = 0; k < 2; ++k) {
        t->nw[k] = net_weights(blobs[k], nullptr, nullptr, nullptr, nullptr);     // the minibatch arrives normalised; outputs stay normalised
        if (trl_make_fc_maps(&t->fmaps[k], t->nw[k].tip0_w, d.a2, 3 * kB)) return 1;
    }
    return 0;
}

trl_trainer* trl_trainer_create(trl_handle* h, const double* p) { return trl_trainer_create_slot(h, 0, p, nullptr, nullptr); }

// A trainer for policy slot `slot`: slot 0 is the handle's own policy (trl_trainer_create); slots 1..7 are training slots of an
// exploration handle, whose envs (trl_set_env_policy) explore with the slot trainer's net and feed it their tuples
trl_trainer* trl_trainer_create_slot(trl_handle* h, int slot, const double* p, const char* h5_path, const char* scale_path) {
    auto refuse = [](const std::string& why) -> trl_trainer* { trl_fail(why); return nullptr; };
    if (!h || !h->mc.has_net) return refuse("trl_trainer_create: the scene has no policy net");
    if (slot < 0 || slot >= kMaxPolicySlots) return refuse("trl_trainer_create_slot: slot " + std::to_string(slot) + " out of range (0.." + std::to_string(kMaxPolicySlots - 1) + ")");
    if (slot == 0) {
        if (h->trainer) return refuse("trl_trainer_create: a trainer is already attached");
        if (h->slots_active && !h->train_slots && h->mode == TRL_MODE_POLI_EVAL)
            return refuse("trl_trainer_create: the handle evaluates several policy slots (trl_load_policy); a trainer needs a single-policy handle");
    } else {
        if (h->mode != TRL_MODE_EXPLORE) return refuse("trl_trainer_create_slot: training slots are for exploration handles (TRL_MODE_EXPLORE)");
        if (h->slot_trainer[slot]) return refuse("trl_trainer_create_slot: slot " + std::to_string(slot) + " already has a trainer");
        if (!h->decide_v2) return refuse("trl_trainer_create_slot: the TRL_DECIDE_V1 decision kernel has no policy slots");
    }
    trl_trainer* t = trainer_new(h, p);
    if (!t) return nullptr;
    t->slot = slot;
    const bool files = h5_path && scale_path;
    const int rc = slot == 0 ? (files ? trl_load_model(h, h5_path, scale_path) : 0) : trl_stage_slot_model(h, slot, h5_path, scale_path);
    if (rc || trainer_start(t, slot == 0 ? h->net_blobs : h->slot_blobs[slot])) {
        trainer_free(t);
        return nullptr;
    }
    // cNeuralNetLearner::SyncNet as a binding: the decision kernels read the trainer's weights from now on (a slot's through the slot
    // table and its terr_ip0 descriptor, rewritten by ensure_slot_tables before the next decision)
    const Dev& d = t->d;
    const double* blobs[26];
    for (int b = 0; b < 26; ++b) blobs[b] = d.theta + d.off[b];
    if (slot == 0) {
        h->W = net_weights(blobs, d.in_off, d.in_scale, d.out_off, d.out_scale);
        h->trainer = t;
    } else {
        h->slot_W[slot] = net_weights(blobs, d.in_off, d.in_scale, d.out_off, d.out_scale);
        h->slot_trainer[slot] = t;
        h->slots_active = h->train_slots = true;
        h->slot_dirty = true;
    }
    trl_drop_graphs(h);
    return t;
}

// trl_destroy of the scenario a trainer is still attached to: the trainer's device state goes with it; the (host) object stays
// valid so that a later trl_trainer_destroy is harmless and every other call on it fails with a message instead of
// touching freed memory.
void trl_trainer_orphan(trl_trainer* t) {
    if (!t || !t->h) return;
    cudaStreamSynchronize(t->h->stream);
    if (t->async_stream) {
        cudaStreamSynchronize(t->async_stream); cudaStreamDestroy(t->async_stream); cudaEventDestroy(t->ev_snap); cudaEventDestroy(t->ev_trained);
        t->async_stream = nullptr; t->async = false;
    }
    if (t->own_stream) { cudaStreamSynchronize(t->own_stream); cudaStreamDestroy(t->own_stream); cudaEventDestroy(t->ev_own); t->own_stream = nullptr; }
    if (t->train_graph) { cudaGraphExecDestroy(t->train_graph); t->train_graph = nullptr; }
    for (void* q : t->allocs) cudaFree(q);
    t->allocs.clear();
    (t->slot == 0 ? t->h->trainer : t->h->slot_trainer[t->slot]) = nullptr;
    t->h = nullptr;
}
#define TRL_TRAINER_LIVE(t) do { if (!(t) || !(t)->h) return trl_fail("trainer: the scenario it was attached to has been destroyed"); } while (0)
static cudaError_t trainer_sync(trl_trainer* t) {
    cudaError_t e = cudaStreamSynchronize(t->h->stream);
    if (e == cudaSuccess && t->async_stream) e = cudaStreamSynchronize(t->async_stream);
    if (e == cudaSuccess && t->own_stream) e = cudaStreamSynchronize(t->own_stream);
    return e;
}

int trl_trainer_destroy(trl_trainer* t) {
    if (!t) return 0;
    trl_handle* h = t->h;
    if (!h) { delete t; return 0; }
    cudaStreamSynchronize(h->stream);
    if (t->own_stream) { cudaStreamSynchronize(t->own_stream); cudaStreamDestroy(t->own_stream); cudaEventDestroy(t->ev_own); }
    if (t->slot == 0) {
        // hand the weights back to the engine's own buffers so the scenario stays usable
        for (int b = 0; b < 26; ++b) cudaMemcpy(h->net_blobs[b], t->d.theta + t->d.off[b], (size_t)h->net_counts[b] * 8, cudaMemcpyDeviceToDevice);
        cudaMemcpy(h->net_blobs[26], t->d.in_off, (size_t)h->net_counts[26] * 8, cudaMemcpyDeviceToDevice);
        cudaMemcpy(h->net_blobs[27], t->d.in_scale, (size_t)h->net_counts[27] * 8, cudaMemcpyDeviceToDevice);
        double** b = h->net_blobs.data();
        h->W = net_weights(b, b[26], b[27], b[28], b[29]);
        h->trainer = nullptr;
    } else {
        // into the slot's own blobs, offset / scale vectors included (the slot's exploration noise is scaled by its output scale): the
        // slot stays loaded with the trained net
        std::vector<double*>& sb = h->slot_blobs[t->slot];
        const double* vec[4] = {t->d.in_off, t->d.in_scale, t->d.out_off, t->d.out_scale};
        for (int b = 0; b < 30; ++b)
            cudaMemcpy(sb[b], b < 26 ? t->d.theta + t->d.off[b] : vec[b - 26], (size_t)h->net_counts[b] * 8, cudaMemcpyDeviceToDevice);
        double** b = sb.data();
        h->slot_W[t->slot] = net_weights(b, b[26], b[27], b[28], b[29]);
        h->slot_dirty = true;
        h->slot_trainer[t->slot] = nullptr;
    }
    trl_drop_graphs(h);
    if (t->train_graph) cudaGraphExecDestroy(t->train_graph);
    if (t->async_stream) { cudaStreamSynchronize(t->async_stream); cudaStreamDestroy(t->async_stream); cudaEventDestroy(t->ev_snap); cudaEventDestroy(t->ev_trained); }
    for (void* q : t->allocs) cudaFree(q);
    delete t;
    return 0;
}

// cNeuralNetLearner::Train's AddTuples(exp->GetTuples()) + ResetTupleBuffer, device to device
int trl_trainer_add_from_scene(trl_trainer* t) {
    TRL_TRAINER_LIVE(t);
    trl_handle* h = t->h;
    if (h->train_slots) enqueue_add_slot(t, h->stream);      // this slot's rows; the block stays for the other trainers
    else enqueue_add(t, h->B.tuples, h->B.tuple_flags, h->B.tuple_count, 0, h->B.tuple_cap, h->B.tuple_count, h->stream, h->B.tuple_env);
    TCK(cudaGetLastError());
    return 0;
}
// tuples handed in from host memory (the adapter path of INTEGRATION.md, and the tests)
int trl_trainer_add_tuples(trl_trainer* t, const double* rows, const uint32_t* flags, int n) {
    TRL_TRAINER_LIVE(t);
    trl_handle* h = t->h;
    for (int base = 0; base < n; base += t->stage_cap) {
        const int cnt = std::min(t->stage_cap, n - base);
        TCK(cudaMemcpyAsync(t->stage_rows, rows + (size_t)base * t->d.Wd, (size_t)cnt * t->d.Wd * 8, cudaMemcpyHostToDevice, h->stream));
        TCK(cudaMemcpyAsync(t->stage_flags, flags + base, (size_t)cnt * 4, cudaMemcpyHostToDevice, h->stream));
        enqueue_add(t, t->stage_rows, t->stage_flags, nullptr, cnt, cnt, nullptr, h->stream);
        TCK(cudaStreamSynchronize(h->stream));
    }
    TCK(cudaGetLastError());
    return 0;
}

// tuples already on the device (e.g. the NCCL all-gather of every rank's tuple block, parallel.gather_tuple_blocks*): rows f64
// [n][1 + S + A + S], flags u32 [n]; enqueued on the scenario's stream, which the caller must have ordered after the producer
int trl_trainer_add_device(trl_trainer* t, const double* rows_dev, const uint32_t* flags_dev, int n) {
    TRL_TRAINER_LIVE(t);
    if (n > t->stage_cap) return trl_fail("trl_trainer_add_device: more tuples than the staging capacity (split the call)");
    enqueue_add(t, rows_dev, flags_dev, nullptr, n, n, nullptr, t->h->stream);
    TCK(cudaGetLastError());
    return 0;
}

// AddTuples of the blocks every rank contributed to the last trl_gather_tuples (rank order, env order inside a rank), on stream `ws`
// behind the all-gather; identical input on every rank keeps replicated trainers bit-identical.  In a handle with training slots the
// trainer takes only its slot's rows (the pack kernel stamped each row with its env's slot)
static int add_gathered_on(trl_trainer* t, cudaStream_t ws) {
    trl_handle* h = t->h;
    trl_comm_blocks v;
    if (ws == h->stream ? trl_comm_view(h, &v) : trl_comm_view_on(h, &v, ws)) return 1;
    if (v.width != t->d.Wd) return trl_fail("trl_trainer_add_gathered: tuple width mismatch");
    if ((long long)v.world * v.block_rows > t->gather_cap) {
        // valid / slot / order are indexed by rank * block_rows + j
        const size_t need = (size_t)v.world * v.block_rows;
        int *nv = nullptr, *ns = nullptr, *no = nullptr;
        TCK(cudaStreamSynchronize(h->stream));
        TCK(cudaStreamSynchronize(ws));
        TCK(talloc(t, &nv, need)); TCK(talloc(t, &ns, need)); TCK(talloc(t, &no, need));
        TCK(cudaDeviceSynchronize());      // talloc's memsets run on the legacy stream: done before the intake kernels on `ws` write
        t->d.valid = nv; t->d.slot = ns; t->d.order = no;
        t->gather_cap = (long long)need;
    }
    const Dev& d = t->d;
    const GBlocks g{v.recv, v.block_bytes, v.block_rows, v.world};
    if (h->train_slots) {
        launch_pdl(k_addg_order_slot, dim3(v.block_rows, v.world), dim3(128), 0, ws, d, g, t->slot);
        launch_pdl(k_addg_assign_slot, dim3(1), dim3(32), 0, ws, d, g, t->slot);
        launch_pdl(k_addg_copy_slot, dim3(v.block_rows, v.world), dim3(128), 0, ws, d, g);
    } else {
        launch_pdl(k_addg_order, dim3(v.block_rows, v.world), dim3(128), 0, ws, d, g);
        launch_pdl(k_addg_assign, dim3(1), dim3(32), 0, ws, d, g);
        launch_pdl(k_addg_copy, dim3(v.block_rows, v.world), dim3(128), 0, ws, d, g);
    }
    t->launches += 3;
    TCK(cudaGetLastError());
    return 0;
}
int trl_trainer_add_gathered(trl_trainer* t) {
    TRL_TRAINER_LIVE(t);
    cudaStream_t ws = t->work();
    if (add_gathered_on(t, ws)) return 1;
    if (t->async && trl_comm_mark_consumed(t->h, ws)) return 1;      // the next all-gather may overwrite the blocks only after this
    return 0;
}

// cNeuralNetLearner::SyncNet across ranks (learning/NeuralNetLearner.cpp:85-89): the complete net state of `root`'s trainer --
// weights, target net, momentum history, the eight offset / scale vectors -- reaches every rank's trainer, and with it the
// policy each rank's decision kernel evaluates (pointer binding)
int trl_trainer_broadcast(trl_trainer* t, int root) {
    TRL_TRAINER_LIVE(t);
    const Dev& d = t->d;
    double* arrays[11] = {d.theta, d.target, d.history, d.in_off, d.in_scale, d.out_off, d.out_scale, d.t_in_off, d.t_in_scale, d.t_out_off, d.t_out_scale};
    const size_t counts[11] = {(size_t)d.P, (size_t)d.P, (size_t)d.P, (size_t)d.S, (size_t)d.S, (size_t)d.n_out, (size_t)d.n_out,
                               (size_t)d.S, (size_t)d.S, (size_t)d.n_out, (size_t)d.n_out};
    return trl_comm_broadcast_list(t->h, arrays, counts, 11, root);
}

int trl_trainer_replica_spread(trl_trainer* t, double* max_abs_diff) {
    TRL_TRAINER_LIVE(t);
    return trl_comm_replica_spread(t->h, t->d.theta, (size_t)t->d.P, max_abs_diff);
}

// `iters` replays of the captured training iteration on stream `st`
static int train_on(trl_trainer* t, int iters, cudaStream_t st) {
    if (!t->train_graph) {
        cudaGraph_t graph;
        const int64_t before = t->launches;
        TCK(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
        enqueue_train(t, st);
        TCK(cudaStreamEndCapture(st, &graph));
        TCK(cudaGraphInstantiate(&t->train_graph, graph, 0));
        cudaGraphDestroy(graph);
        t->graph_launches = t->launches - before;      // capturing ran no kernel; each replay runs the kernels it recorded
        t->launches = before;
    }
    for (int i = 0; i < iters; ++i) {
        TCK(cudaGraphLaunch(t->train_graph, st));
        t->launches += t->graph_launches;
    }
    return 0;
}
// `iters` x cNeuralNetTrainer::Train() on the engine's stream (ordered after the update that produced the tuples and before
// the next one, which then evaluates the updated weights)
int trl_trainer_train(trl_trainer* t, int iters) {
    TRL_TRAINER_LIVE(t);
    return train_on(t, iters, t->work());
}

// Training from scratch: the net the reference builds when no -policy_model is given.
//  * weights: Caffe `xavier` fillers of the train prototxt (uniform(-s, s), s = sqrt(3 / fan_in), fan_in = count / num_output),
//    biases 0 (`constant` filler); the filler RNG is Caffe's own, so only the distribution is defined -- std::mt19937_64(seed) here;
//  * output offset / scale: cScenarioTrain::SetupTrainerOutputOffsetScale -> cBaseControllerMACE::BuildNNOutputOffsetScale
//    (scenarios/ScenarioTrain.cpp:322-336, sim/BaseControllerMACE.cpp:75-113,131-167): critic outputs offset -0.5 scale 2; actor f is
//    centred on the optimised parameters of control-parameter set f % n_ctrl (cDogControllerMACE::BuildActorBias,
//    sim/DogControllerMACE.cpp:93-99) and scaled by 1 / max_a |opt(a) - opt(default action)| over the action library;
//  * input offset 0 / scale 1 until the init stage refits them from the replay memory; momentum history cleared; target = copy.
int trl_trainer_init_fresh(trl_trainer* t, uint64_t seed) {
    TRL_TRAINER_LIVE(t);
    trl_handle* h = t->h;
    const Dev& d = t->d;
    ModelConst& m = h->mc;
    TCK(cudaStreamSynchronize(h->stream));
    const int fs = d.frag, nf = d.n_frags;
    std::vector<double> out_off(d.n_out, 0.0), out_scale(d.n_out, 1.0);
    if (trl_get_output_offset_scale(h, out_off.data(), out_scale.data(), d.n_out)) return 1;
    std::vector<double> theta(d.P, 0.0);
    std::mt19937_64 gen(seed);
    const int num_out[13] = {C0, C1, C2, T, H, HH, nf, HH, fs, HH, fs, HH, fs};
    for (int l = 0; l < 13; ++l) {
        const int b = 2 * l, count = d.off[b + 1] - d.off[b];
        const double sc = std::sqrt(3.0 / ((double)count / num_out[l]));
        std::uniform_real_distribution<double> U(-sc, sc);
        for (int i = d.off[b]; i < d.off[b + 1]; ++i) theta[i] = U(gen);
    }
    std::vector<double> zeros(d.S, 0.0), ones(d.S, 1.0);
    TCK(cudaMemcpy(d.theta, theta.data(), (size_t)d.P * 8, cudaMemcpyHostToDevice));
    TCK(cudaMemcpy(d.target, d.theta, (size_t)d.P * 8, cudaMemcpyDeviceToDevice));
    TCK(cudaMemset(d.history, 0, (size_t)d.P * 8));
    double* offs[2] = {d.in_off, d.t_in_off};
    double* scls[2] = {d.in_scale, d.t_in_scale};
    for (int k = 0; k < 2; ++k) {
        TCK(cudaMemcpy(offs[k], zeros.data(), (size_t)d.S * 8, cudaMemcpyHostToDevice));
        TCK(cudaMemcpy(scls[k], ones.data(), (size_t)d.S * 8, cudaMemcpyHostToDevice));
    }
    double* oo[2] = {d.out_off, d.t_out_off};
    double* os[2] = {d.out_scale, d.t_out_scale};
    for (int k = 0; k < 2; ++k) {
        TCK(cudaMemcpy(oo[k], out_off.data(), (size_t)d.n_out * 8, cudaMemcpyHostToDevice));
        TCK(cudaMemcpy(os[k], out_scale.data(), (size_t)d.n_out * 8, cudaMemcpyHostToDevice));
    }
    if (t->slot != 0) return 0;      // a training slot's exploration noise is scaled by the slot's own out_scale, just written
    for (int k = 0; k < fs; ++k) m.out_scale_actor0[k] = out_scale[nf + k];       // exploration noise scale of the decision kernel
    return trl_reupload_model(h);
}

// cScenarioTrain::Run for one batch (scenarios/ScenarioTrain.cpp:100-115,376-410): `num_updates` x { Update(time_step); hand the
// tuples to the trainer; `iters_per_update` trainer iterations (0: one per `tuple_buffer_size` new tuples, which costs one small
// read-back per update); anneal the exploration settings and the curriculum phase from the iteration count }.  sp[9] as in
// trl_train_schedule.  Everything is enqueued on the scenario's stream; the call returns after the last update is queued
// (iters_per_update > 0) -- synchronise with trl_sync / trl_trainer_counters.
// Asynchronous training (the reference's cAsyncMACETrainer / `-trainer_... async` path: exploration keeps running on the net it has
// while the trainer works, scenarios/ScenarioTrain.cpp:388-408 + learning/AsyncTrainer): the hand-over of gathered tuples and the
// trainer iterations move to their own low-priority stream and overlap the NEXT outer update; the decision kernels evaluate a snapshot
// of the net that trl_train_run* refreshes between two updates, once the trainer job enqueued before the previous update is done.
// Tuples of update u therefore shape the policy from update u + 2 on.  Needs a communicator (trl_comm_init*; a single rank will
// do): the tuples leave the scenario through the pack kernel of trl_gather_tuples.
int trl_trainer_set_async(trl_trainer* t, int enable) {
    TRL_TRAINER_LIVE(t);
    trl_handle* h = t->h;
    if ((enable != 0) == t->async) return 0;
    if (h->train_slots && !h->comm)
        return trl_fail("trl_trainer_set_async: the handle has training slots and no communicator (asynchronous slot trainers run through trl_train_run_slots_comm)");
    TCK(trainer_sync(t));
    const Dev& d = t->d;
    if (t->train_graph) { cudaGraphExecDestroy(t->train_graph); t->train_graph = nullptr; }      // it was captured on the other stream
    if (enable) {
        if (!h->comm) return trl_fail("trl_trainer_set_async: asynchronous training needs a communicator (trl_comm_init first)");
        if (!t->async_stream) {
            int lo = 0, hi = 0;
            cudaDeviceGetStreamPriorityRange(&lo, &hi);
            // highest priority: the trainer's launches are a few CTAs each; behind the step launch's CTAs every one of them would
            // wait for a free slot
            TCK(cudaStreamCreateWithPriority(&t->async_stream, cudaStreamNonBlocking, hi));
            TCK(cudaEventCreateWithFlags(&t->ev_snap, cudaEventDisableTiming));
            TCK(cudaEventCreateWithFlags(&t->ev_trained, cudaEventDisableTiming));
            TCK(talloc(t, &t->snap, (size_t)d.P + 2 * (size_t)d.S + 2 * (size_t)d.n_out));
        }
        double* sn = t->snap;
        TCK(cudaMemcpy(sn, d.theta, (size_t)d.P * 8, cudaMemcpyDeviceToDevice));
        TCK(cudaMemcpy(sn + d.P, d.in_off, (size_t)d.S * 8, cudaMemcpyDeviceToDevice));
        TCK(cudaMemcpy(sn + d.P + d.S, d.in_scale, (size_t)d.S * 8, cudaMemcpyDeviceToDevice));
        TCK(cudaMemcpy(sn + d.P + 2 * d.S, d.out_off, (size_t)d.n_out * 8, cudaMemcpyDeviceToDevice));
        TCK(cudaMemcpy(sn + d.P + 2 * d.S + d.n_out, d.out_scale, (size_t)d.n_out * 8, cudaMemcpyDeviceToDevice));
    }
    // bind the decision kernels to the snapshot (async) or straight to the trainer's arrays (synchronous: SyncNet as a pointer binding);
    // a training slot's net through its entry of the slot table (and its terr_ip0 descriptor), rewritten before the next decision
    const double* th = enable ? t->snap : d.theta;
    const double* blobs[26];
    for (int b = 0; b < 26; ++b) blobs[b] = th + d.off[b];
    const NetWeights nw = net_weights(blobs, enable ? t->snap + d.P : d.in_off, enable ? t->snap + d.P + d.S : d.in_scale,
                                      enable ? t->snap + d.P + 2 * d.S : d.out_off, enable ? t->snap + d.P + 2 * d.S + d.n_out : d.out_scale);
    if (t->slot == 0) {
        h->W = nw;
    } else {
        h->slot_W[t->slot] = nw;
        h->slot_dirty = true;
    }
    trl_drop_graphs(h);
    t->async = enable != 0;
    t->trained_pending = t->job_pending = false;
    return 0;
}
// between two updates, on the scenario's stream: wait for the trainer job that was enqueued before the previous update, refresh the
// snapshot the decision kernels read, then hand the trainer its next job (the tuples gathered after the previous update)
static int async_turnover(trl_trainer* t, int iters) {
    trl_handle* h = t->h;
    const Dev& d = t->d;
    cudaStream_t A = h->stream, T = t->async_stream;
    if (t->trained_pending) { TCK(cudaStreamWaitEvent(A, t->ev_trained, 0)); t->trained_pending = false; }
    double* sn = t->snap;
    TCK(cudaMemcpyAsync(sn, d.theta, (size_t)d.P * 8, cudaMemcpyDeviceToDevice, A));
    TCK(cudaMemcpyAsync(sn + d.P, d.in_off, (size_t)d.S * 8, cudaMemcpyDeviceToDevice, A));
    TCK(cudaMemcpyAsync(sn + d.P + d.S, d.in_scale, (size_t)d.S * 8, cudaMemcpyDeviceToDevice, A));
    TCK(cudaEventRecord(t->ev_snap, A));
    if (t->job_pending) {
        TCK(cudaStreamWaitEvent(T, t->ev_snap, 0));           // the trainer must not move theta under the copy
        if (trl_trainer_add_gathered(t)) return 1;            // (on T, behind the all-gather)
        if (iters > 0 && trl_trainer_train(t, iters)) return 1;
        TCK(cudaEventRecord(t->ev_trained, T));
        t->trained_pending = true;
        t->job_pending = false;
    }
    return 0;
}

static int train_run_impl(trl_trainer* t, const double* sp, int num_updates, int iters_per_update, int tuple_buffer_size, double time_step,
                          int block_rows, long long* iters_state, void* flush_buf = nullptr, size_t flush_bytes = 0) {
    trl_handle* h = t->h;
    long long last_total = -1, carry = 0;
    long long iters_req = iters_state ? *iters_state : 0;
    double last_phase = -1.0;
    for (int u = 0; u < num_updates; ++u) {
        double s[4];
        long long it = iters_req;
        if (iters_per_update <= 0) {
            int64_t c[9];
            if (trl_trainer_counters(t, c, nullptr)) return 1;
            it = c[0];
            if (last_total < 0) last_total = c[5];
        }
        trl_train_schedule(sp, (int)std::min<long long>(it, 2000000000LL), s);
        if (trl_set_explore(h, 1, s[0], s[1], s[2])) return 1;
        if (s[3] != last_phase) { if (trl_set_terrain_lerp(h, s[3])) return 1; last_phase = s[3]; }
        if (flush_buf) TCK(cudaMemsetAsync(flush_buf, u & 0xff, flush_bytes, h->stream));     // measurement: evict L2 between updates
        if (t->async) {
            if (iters_per_update <= 0) return trl_fail("asynchronous training needs a fixed number of trainer iterations per update");
            if (async_turnover(t, iters_per_update)) return 1;
            if (trl_update(h, time_step)) return 1;
            if (trl_gather_tuples(h, block_rows)) return 1;
            t->job_pending = true;
            iters_req += iters_per_update;
            continue;
        }
        if (trl_update(h, time_step)) return 1;
        if (h->comm) {
            // N GPUs: the tuples of every rank reach every rank's trainer (one all-gather), scenarios/ScenarioTrain.cpp:388-395
            if (trl_gather_tuples(h, block_rows)) return 1;
            if (trl_trainer_add_gathered(t)) return 1;
        } else if (trl_trainer_add_from_scene(t)) return 1;
        int k = iters_per_update;
        if (iters_per_update <= 0) {
            int64_t c[9];
            if (trl_trainer_counters(t, c, nullptr)) return 1;
            const long long fresh = c[5] - last_total + carry;
            last_total = c[5];
            k = (int)(fresh / std::max(1, tuple_buffer_size));
            carry = fresh % std::max(1, tuple_buffer_size);
        }
        if (k > 0 && trl_trainer_train(t, k)) return 1;
        iters_req += k;
    }
    if (t->async) {
        // the trainer job of the last update, and the end of the stream of work: the caller's trl_sync must cover the trainer too
        if (async_turnover(t, iters_per_update)) return 1;
        if (t->trained_pending) { TCK(cudaStreamWaitEvent(h->stream, t->ev_trained, 0)); t->trained_pending = false; }
    }
    if (iters_state) *iters_state = iters_req;
    return 0;
}
int trl_train_run(trl_trainer* t, const double* sp, int num_updates, int iters_per_update, int tuple_buffer_size, double time_step) {
    TRL_TRAINER_LIVE(t);
    if (t->h->train_slots) return trl_fail("trl_train_run: the handle has training slots, whose trainers share its tuple block (trl_train_run_slots)");
    return train_run_impl(t, sp, num_updates, iters_per_update, tuple_buffer_size, time_step, 0, nullptr);
}
// the same loop, device-timed: CUDA events on the scenario's stream around `num_updates` iterations of {update, tuple exchange,
// hand-over, trainer iterations} (bench.py's config-4 figure).  *iters_state carries the annealing position from call to call.
int trl_train_run_timed(trl_trainer* t, const double* sp, int num_updates, int iters_per_update, int block_rows, double time_step,
                        int flush_l2, int64_t* iters_state, double* ms) {
    TRL_TRAINER_LIVE(t);
    if (iters_per_update <= 0) return trl_fail("trl_train_run_timed: iters_per_update must be positive (no read-backs inside a timed region)");
    trl_handle* h = t->h;
    if (h->train_slots) return trl_fail("trl_train_run_timed: the handle has training slots, whose trainers share its tuple block (trl_train_run_slots)");
    const size_t flush_bytes = (size_t)256 << 20;
    if (flush_l2 && !h->flush_buf) { TCK(cudaMalloc(&h->flush_buf, flush_bytes)); h->allocs.push_back(h->flush_buf); }
    cudaEvent_t e0, e1;
    TCK(cudaEventCreate(&e0)); TCK(cudaEventCreate(&e1));
    TCK(cudaStreamSynchronize(h->stream));
    TCK(cudaEventRecord(e0, h->stream));
    long long st = iters_state ? (long long)*iters_state : 0;
    const int rc = train_run_impl(t, sp, num_updates, iters_per_update, 32, time_step, block_rows, &st, flush_l2 ? h->flush_buf : nullptr, flush_bytes);
    if (iters_state) *iters_state = (int64_t)st;
    if (rc == 0) {
        TCK(cudaEventRecord(e1, h->stream));
        TCK(cudaEventSynchronize(e1));
        float f = 0;
        TCK(cudaEventElapsedTime(&f, e0, e1));
        if (ms) *ms = f;
    }
    cudaEventDestroy(e0); cudaEventDestroy(e1);
    return rc;
}

// The trl_train_run loop for k trainers of one handle (slot 0's and / or training slots'), shared by trl_train_run_slots and
// trl_train_run_slots_sched.  Per update: the exploration settings and curriculum blend of the schedule, the update, then one branch
// per trainer on its own stream -- its hand-over (its slot's rows of the block, in env order) and its replays of the training
// iteration --, the join, and the block's cursor back to zero.  Each trainer computes what a single-trainer handle fed only its
// slot's rows computes.
//   per_slot = false: ONE schedule `sp` applied handle-wide (trl_set_explore); iters_per_update > 0.
//   per_slot = true:  trainer i follows sp + 9 i on its own slot's entry (trl_set_explore_slot).
//   iters_per_update > 0: lock-step, every trainer's schedule position counts the iterations requested in this call (from 0).
//   iters_per_update == 0: train_run_impl's pacing per trainer: the schedule at the trainer's iteration counter at the start of the
//   update, then k_i = (fresh tuples + carry) / tuple_buffer_size iterations.  The counters of all k trainers come back in one round
//   trip at the start of the update and one after the hand-overs, so the iterations need a second fork behind the first join.
//   comm = true (trl_train_run_slots_comm): the update is followed by ONE trl_gather_tuples(h, block_rows) and each branch takes its
//   slot's rows of the gathered blocks instead (rank order, env order inside a rank); the pack kernel clears the block, keeping the
//   rows beyond block_rows queued.  Every rank sees the same blocks, so counters, pacing and replicas agree across ranks.
//   Asynchronous trainers (comm only, all or none, lock-step): per update each trainer's async_turnover -- wait for its previous
//   job, refresh its snapshot, enqueue its intake of the last gathered blocks and its iterations on its own async stream --, then the
//   update and the gather.  The next all-gather waits for every trainer's intake (trl_comm_mark_consumed joins the consumers).
// The caller has checked the curricula: every trainer sees the same phase at every update, so the blend is trainer 0's.
static int run_slots_impl(const char* who, trl_trainer* const* ts, int k, const double* sp, bool per_slot, int num_updates,
                          int iters_per_update, int tuple_buffer_size, double time_step, bool comm = false, int block_rows = 0) {
    trl_handle* h = ts[0]->h;
    const bool async = ts[0]->async;
    for (int i = 0; i < k; ++i) {
        trl_trainer* t = ts[i];
        if (!t->own_stream) {
            TCK(cudaStreamCreateWithFlags(&t->own_stream, cudaStreamNonBlocking));
            TCK(cudaEventCreateWithFlags(&t->ev_own, cudaEventDisableTiming));
        }
    }
    const bool paced = iters_per_update == 0;
    Counters* hc = nullptr;            // pinned: the k trainers' counters, one synchronisation per read-back
    if (paced) TCK(cudaMallocHost(&hc, (size_t)k * sizeof(Counters)));
    auto read_counters = [&]() -> int {
        for (int i = 0; i < k; ++i) TCK(cudaMemcpyAsync(hc + i, ts[i]->d.c, sizeof(Counters), cudaMemcpyDeviceToHost, h->stream));
        TCK(cudaStreamSynchronize(h->stream));      // every trainer's stream was joined into the handle's
        return 0;
    };
    cudaEvent_t fork;
    TCK(cudaEventCreateWithFlags(&fork, cudaEventDisableTiming));
    auto branch = [&](auto&& body) {
        cudaEventRecord(fork, h->stream);
        int rc = 0;
        for (int i = 0; i < k && rc == 0; ++i) {
            trl_trainer* t = ts[i];
            cudaStreamWaitEvent(t->own_stream, fork, 0);
            rc = body(i, t);
            cudaEventRecord(t->ev_own, t->own_stream);
        }
        for (int i = 0; i < k; ++i) cudaStreamWaitEvent(h->stream, ts[i]->ev_own, 0);
        return rc;
    };
    auto hand_over = [&](int, trl_trainer* t) {
        if (comm) return add_gathered_on(t, t->own_stream);
        if (h->train_slots) enqueue_add_slot(t, t->own_stream);
        else enqueue_add(t, h->B.tuples, h->B.tuple_flags, h->B.tuple_count, 0, h->B.tuple_cap, nullptr, t->own_stream, h->B.tuple_env);
        return 0;
    };
    std::vector<long long> pos(k, 0), last_total(k, -1), carry(k, 0);
    std::vector<int> iters(k, iters_per_update);
    int rc = 0;
    double last_phase = -1.0;
    for (int u = 0; u < num_updates && rc == 0; ++u) {
        if (paced) {
            if ((rc = read_counters())) break;
            for (int i = 0; i < k; ++i) {
                pos[i] = hc[i].iter;
                if (last_total[i] < 0) last_total[i] = hc[i].total;
            }
        }
        double s[4], phase = 0.0;
        for (int i = 0; i < k && rc == 0; ++i) {
            trl_train_schedule(per_slot ? sp + 9 * i : sp, (int)std::min<long long>(pos[i], 2000000000LL), s);
            if (i == 0) phase = s[3];
            if (!per_slot) { rc = trl_set_explore(h, 1, s[0], s[1], s[2]); break; }
            rc = trl_set_explore_slot(h, ts[i]->slot, 1, s[0], s[1], s[2]);
        }
        if (rc) break;
        if (phase != last_phase) { if ((rc = trl_set_terrain_lerp(h, phase))) break; last_phase = phase; }
        if (async) {
            for (int i = 0; i < k && rc == 0; ++i) rc = async_turnover(ts[i], iters_per_update);
            if (rc || (rc = trl_update(h, time_step)) || (rc = trl_gather_tuples(h, block_rows))) break;
            for (int i = 0; i < k; ++i) { ts[i]->job_pending = true; pos[i] += iters[i]; }
            continue;
        }
        if ((rc = trl_update(h, time_step))) break;
        if (comm && (rc = trl_gather_tuples(h, block_rows))) break;
        if (!paced) {
            rc = branch([&](int i, trl_trainer* t) {
                const int r = hand_over(i, t);
                return r ? r : train_on(t, iters_per_update, t->own_stream);
            });
        } else {
            rc = branch(hand_over);
            if (rc == 0 && (rc = read_counters()) == 0) {
                for (int i = 0; i < k; ++i) {
                    const long long fresh = hc[i].total - last_total[i] + carry[i];
                    last_total[i] = hc[i].total;
                    iters[i] = (int)(fresh / tuple_buffer_size);
                    carry[i] = fresh % tuple_buffer_size;
                }
                rc = branch([&](int i, trl_trainer* t) { return iters[i] > 0 ? train_on(t, iters[i], t->own_stream) : 0; });
            }
        }
        if (!comm) cudaMemsetAsync(h->B.tuple_count, 0, 4, h->stream);      // cScenarioExp::ResetTupleBuffer, once every trainer has taken its rows
        for (int i = 0; i < k; ++i) pos[i] += iters[i];
        const cudaError_t e = cudaGetLastError();
        if (rc == 0 && e != cudaSuccess) rc = trl_fail(std::string(who) + ": " + cudaGetErrorString(e));
    }
    if (async && rc == 0) {
        // the trainer jobs of the last update, and the end of the stream of work: the caller's trl_sync must cover the trainers too
        for (int i = 0; i < k && rc == 0; ++i) {
            trl_trainer* t = ts[i];
            if ((rc = async_turnover(t, iters_per_update))) break;
            if (t->trained_pending) { cudaStreamWaitEvent(h->stream, t->ev_trained, 0); t->trained_pending = false; }
        }
    }
    cudaEventDestroy(fork);
    if (hc) cudaFreeHost(hc);
    return rc;
}

// what both entries refuse, with the handle unchanged
static int check_slot_trainers(const char* who, trl_trainer* const* ts, int k, bool allow_async = false) {
    const std::string w(who);
    if (!ts || k < 1) return trl_fail(w + ": need at least one trainer");
    for (int i = 0; i < k; ++i) {
        TRL_TRAINER_LIVE(ts[i]);
        if (ts[i]->h != ts[0]->h) return trl_fail(w + ": the trainers belong to different handles");
        for (int j = 0; j < i; ++j)
            if (ts[j] == ts[i]) return trl_fail(w + ": trainer " + std::to_string(i) + " is listed twice");
        if (ts[i]->async && !allow_async) return trl_fail(w + ": asynchronous trainers are not run in lock-step");
    }
    return 0;
}

// the per-trainer schedules' arguments (trl_train_run_slots_sched and trl_train_run_slots_comm)
static int check_sched_args(const char* who, int k, const double* sp, int iters_per_update, int tuple_buffer_size) {
    if (iters_per_update < 0) return trl_fail(std::string(who) + ": iters_per_update must be positive, or 0 for one iteration per tuple_buffer_size tuples");
    if (iters_per_update == 0 && tuple_buffer_size < 1) return trl_fail(std::string(who) + ": tuple_buffer_size must be positive when the trainers are paced by tuples");
    // one terrain blend per update for the whole handle: every trainer must be at the same curriculum phase at every update
    bool all_off = true, same = true;
    for (int i = 0; i < k; ++i) {
        all_off = all_off && sp[9 * i + 8] < 1;
        same = same && sp[9 * i + 8] == sp[8];
    }
    if (iters_per_update == 0 && !all_off)
        return trl_fail(std::string(who) + ": trainers paced by tuples reach different curriculum phases (the handle has one terrain blend): "
                        "every trainer_curriculum_iters must be < 1");
    if (!all_off && !same)
        return trl_fail(std::string(who) + ": the schedules differ in trainer_curriculum_iters (the handle has one terrain blend per update)");
    return 0;
}

// k trainers in lock-step under ONE schedule, applied handle-wide
int trl_train_run_slots(trl_trainer* const* ts, int k, const double* sp, int num_updates, int iters_per_update, double time_step) {
    if (check_slot_trainers("trl_train_run_slots", ts, k)) return 1;
    if (iters_per_update <= 0) return trl_fail("trl_train_run_slots: iters_per_update must be positive (the trainers advance in lock-step)");
    if (ts[0]->h->comm) return trl_fail("trl_train_run_slots: the handle has a communicator (multi-GPU training runs through trl_train_run)");
    return run_slots_impl("trl_train_run_slots", ts, k, sp, false, num_updates, iters_per_update, 32, time_step);
}

// k trainers, each under its own schedule sp + 9 i on its own slot's exploration entry; lock-step (iters_per_update > 0) or each paced
// by its own fresh tuples (iters_per_update == 0, one iteration per tuple_buffer_size)
int trl_train_run_slots_sched(trl_trainer* const* ts, int k, const double* sp, int num_updates, int iters_per_update, int tuple_buffer_size,
                              double time_step) {
    const char* who = "trl_train_run_slots_sched";
    if (check_slot_trainers(who, ts, k)) return 1;
    if (!sp) return trl_fail(std::string(who) + ": no schedules");
    if (ts[0]->h->comm) return trl_fail(std::string(who) + ": the handle has a communicator (multi-GPU training runs through trl_train_run)");
    if (check_sched_args(who, k, sp, iters_per_update, tuple_buffer_size)) return 1;
    return run_slots_impl(who, ts, k, sp, true, num_updates, iters_per_update, tuple_buffer_size, time_step);
}

// trl_train_run_slots_sched over the tuple exchange of a communicator: every rank's slot-p rows reach every rank's trainer p
int trl_train_run_slots_comm(trl_trainer* const* ts, int k, const double* sp, int num_updates, int iters_per_update, int tuple_buffer_size,
                             int block_rows, double time_step) {
    const char* who = "trl_train_run_slots_comm";
    const std::string w(who);
    // the only refusals made alone: without a live first trainer and its handle's communicator there is no rank to agree with
    if (!ts || k < 1) return trl_fail(w + ": need at least one trainer");
    TRL_TRAINER_LIVE(ts[0]);
    trl_handle* h = ts[0]->h;
    if (!h->comm) return trl_fail(w + ": the handle has no communicator (trl_comm_init first; trl_train_run_slots_sched trains without one)");
    // every other check is made here and then shared: all ranks take part in the one reduction below and refuse together
    auto local_check = [&]() -> int {
        if (check_slot_trainers(who, ts, k, true)) return 1;
        if (!sp) return trl_fail(w + ": no schedules");
        if (check_sched_args(who, k, sp, iters_per_update, tuple_buffer_size)) return 1;
        int n_async = 0;
        for (int i = 0; i < k; ++i) n_async += ts[i]->async ? 1 : 0;
        if (n_async != 0 && n_async != k)
            return trl_fail(w + ": " + std::to_string(n_async) + " of " + std::to_string(k) + " trainers are asynchronous (all or none)");
        if (n_async && iters_per_update == 0)
            return trl_fail(w + ": asynchronous training needs a fixed number of trainer iterations per update");
        return 0;
    };
    const bool ok = local_check() == 0;
    const std::string why = ok ? std::string() : std::string(trl_last_error());
    // every rank must run the same call: the same slots in the same order under the same schedules, counts and modes
    unsigned long long sig = trl::mix64((unsigned long long)k);
    auto mix = [&](unsigned long long v) { sig = trl::mix64(sig + v); };
    if (ok) {
        for (int i = 0; i < k; ++i) {
            mix((unsigned long long)ts[i]->slot);
            mix(ts[i]->async ? 1ull : 0ull);
            for (int j = 0; j < 9; ++j) { unsigned long long b; std::memcpy(&b, sp + 9 * i + j, 8); mix(b); }
        }
        mix((unsigned long long)(long long)iters_per_update);
        mix((unsigned long long)(long long)(iters_per_update == 0 ? tuple_buffer_size : 0));
        mix((unsigned long long)(long long)block_rows);
    }
    bool same = false, all_ok = false;
    if (trl_comm_agree(h, sig, ok, &same, &all_ok)) return 1;
    if (!ok) return trl_fail(why);
    if (!all_ok) return trl_fail(w + ": another rank refused the call; every rank refuses it");
    if (!same)
        return trl_fail(w + ": the ranks differ in the call (listed slots, schedules, iters_per_update, tuple_buffer_size, block_rows or "
                        "asynchronous trainers); every rank must train the same slots the same way");
    return run_slots_impl(who, ts, k, sp, true, num_updates, iters_per_update, tuple_buffer_size, time_step, true, block_rows);
}

// c[9]: iter, actor_iter, stage, num, head, total, critic buffer, actor buffer, pending actor batch; l[2]: last losses
int trl_trainer_counters(trl_trainer* t, int64_t* c, double* l) {
    TRL_TRAINER_LIVE(t);
    Counters hc;
    TCK(trainer_sync(t));
    TCK(cudaMemcpy(&hc, t->d.c, sizeof(hc), cudaMemcpyDeviceToHost));
    if (c) {
        c[0] = hc.iter; c[1] = hc.actor_iter; c[2] = hc.stage; c[3] = hc.num; c[4] = hc.head; c[5] = hc.total;
        c[6] = hc.critic_count; c[7] = hc.actor_count; c[8] = hc.actor_batch_count;
    }
    if (l) { l[0] = hc.critic_loss; l[1] = hc.actor_loss; }
    return 0;
}
int trl_trainer_num_params(trl_trainer* t) { return t->d.P; }
int64_t trl_trainer_launches(trl_trainer* t) { return t->launches; }

// what: 0 theta, 1 target theta, 2 history, 3 in_off, 4 in_scale, 5 out_off, 6 out_scale, 7 last gradient
int trl_trainer_get(trl_trainer* t, int what, double* out) {
    TRL_TRAINER_LIVE(t);
    const Dev& d = t->d;
    const double* src[8] = {d.theta, d.target, d.history, d.in_off, d.in_scale, d.out_off, d.out_scale, d.grad};
    const size_t cnt[8] = {(size_t)d.P, (size_t)d.P, (size_t)d.P, (size_t)d.S, (size_t)d.S, (size_t)d.n_out, (size_t)d.n_out, (size_t)d.P};
    if (what < 0 || what > 7) return trl_fail("trl_trainer_get: bad selector");
    TCK(trainer_sync(t));
    TCK(cudaMemcpy(out, src[what], cnt[what] * 8, cudaMemcpyDeviceToHost));
    return 0;
}
// cNeuralNetTrainer::LoadModel: weights (26 blobs concatenated in layer order) into the current AND the target net
int trl_trainer_set_theta(trl_trainer* t, const double* theta) {
    TRL_TRAINER_LIVE(t);
    TCK(cudaStreamSynchronize(t->h->stream));
    TCK(cudaMemcpy(t->d.theta, theta, (size_t)t->d.P * 8, cudaMemcpyHostToDevice));
    TCK(cudaMemcpy(t->d.target, t->d.theta, (size_t)t->d.P * 8, cudaMemcpyDeviceToDevice));
    return 0;
}
// replay rows (float, [n][1 + S + A + S]) and flags of the given slots
int trl_trainer_rows(trl_trainer* t, const int32_t* ids, int n, float* rows, int32_t* flags) {
    TRL_TRAINER_LIVE(t);
    TCK(trainer_sync(t));
    for (int i = 0; i < n; ++i) {
        if (ids[i] < 0 || ids[i] >= t->d.cap) return trl_fail("trl_trainer_rows: slot out of range");
        TCK(cudaMemcpy(rows + (size_t)i * t->d.Wd, t->d.mem + (size_t)ids[i] * t->d.Wd, (size_t)t->d.Wd * 4, cudaMemcpyDeviceToHost));
        TCK(cudaMemcpy(flags + i, t->d.flags + ids[i], 4, cudaMemcpyDeviceToHost));
    }
    return 0;
}
// which: 0 critic buffer, 1 actor buffer, 2 pending actor batch, 3 ids of the last sampled batch; returns the length
int trl_trainer_list(trl_trainer* t, int which, int32_t* out, int cap, int* len) {
    TRL_TRAINER_LIVE(t);
    Counters hc;
    TCK(trainer_sync(t));
    TCK(cudaMemcpy(&hc, t->d.c, sizeof(hc), cudaMemcpyDeviceToHost));
    const int* src = which == 0 ? t->d.critic_list : (which == 1 ? t->d.actor_list : (which == 2 ? t->d.actor_batch : t->d.ids));
    const int n = which == 0 ? hc.critic_count : (which == 1 ? hc.actor_count : (which == 2 ? hc.actor_batch_count : trl_train::kB));
    if (len) *len = n;
    TCK(cudaMemcpy(out, src, (size_t)std::min(n, cap) * 4, cudaMemcpyDeviceToHost));
    return 0;
}

// the creation parameters p[10] of trl_trainer_create and the policy slot the trainer trains
int trl_trainer_params(trl_trainer* t, double* params10, int* slot) {
    TRL_TRAINER_LIVE(t);
    if (params10) std::memcpy(params10, t->params, sizeof(t->params));
    if (slot) *slot = t->slot;
    return 0;
}

}  // extern "C"

// A new field of Dev or Counters is either state a checkpoint carries (list it below) or scratch one Train() rewrites before reading it:
// these sizes make the decision explicit
static_assert(sizeof(Counters) == 88, "Counters changed: update trl_trainer_state");
static_assert(sizeof(Dev) == 568, "Dev changed: update trl_trainer_state");

// What carries from one call on the trainer to the next (trl_checkpoint.cu), after its streams have drained: the current and target nets
// with their offset / scale vectors, the momentum history, replay rows [0, num) and their flags, the critic / actor buffers with their
// position tables, the pending actor batch, the ids of the last sampled batch (trl_trainer_list 3), the counter block and the RNG key.
// Not carried: the gradient, activations, candidates, labels, column means (each Train() writes them before it reads them) and the
// hand-over scratch.  An asynchronous trainer has a job in flight across updates and is refused.
int trl_trainer_state(trl_trainer* t, const std::string& prefix, std::vector<CkptSection>* out) {
    TRL_TRAINER_LIVE(t);
    if (t->async) return trl_fail("trl_checkpoint_save: the trainer of slot " + std::to_string(t->slot) + " is asynchronous");
    TCK(trainer_sync(t));
    Dev& d = t->d;
    Counters c;
    TCK(cudaMemcpy(&c, d.c, sizeof(c), cudaMemcpyDeviceToHost));
    const size_t P = (size_t)d.P * 8, S = (size_t)d.S * 8, O = (size_t)d.n_out * 8, cap = (size_t)d.cap, num = (size_t)c.num;
    auto fixed = [&](const char* name, int dtype, void* p, size_t bytes) { out->push_back(CkptSection{prefix + name, dtype, p, nullptr, bytes, bytes}); };
    fixed("theta", 3, d.theta, P); fixed("target", 3, d.target, P); fixed("history", 3, d.history, P);
    fixed("in_off", 3, d.in_off, S); fixed("in_scale", 3, d.in_scale, S); fixed("out_off", 3, d.out_off, O); fixed("out_scale", 3, d.out_scale, O);
    fixed("t_in_off", 3, d.t_in_off, S); fixed("t_in_scale", 3, d.t_in_scale, S); fixed("t_out_off", 3, d.t_out_off, O); fixed("t_out_scale", 3, d.t_out_scale, O);
    out->push_back(CkptSection{prefix + "mem", 2, d.mem, nullptr, num * d.Wd * 4, cap * d.Wd * 4});
    out->push_back(CkptSection{prefix + "flags", 1, d.flags, nullptr, num * 4, cap * 4});
    fixed("pos_critic", 1, d.pos_critic, cap * 4); fixed("pos_actor", 1, d.pos_actor, cap * 4);
    fixed("critic_list", 1, d.critic_list, cap * 4); fixed("actor_list", 1, d.actor_list, cap * 4);
    fixed("actor_batch", 1, d.actor_batch, 4 * trl_train::kB * 4); fixed("ids", 1, d.ids, trl_train::kB * 4);
    fixed("counters", 0, d.c, sizeof(Counters));
    out->push_back(CkptSection{prefix + "rng_key", 0, nullptr, &d.rng_key, 8, 8});
    return 0;
}
