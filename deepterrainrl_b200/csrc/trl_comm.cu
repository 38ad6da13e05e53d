// deepterrainrl_b200 -- multi-GPU exchange behind the C ABI (SURVEY.md §8e): one process per GPU, environments sharded by rank.
//
// The reference couples its exploration threads to the trainer in two places, both under the trainer mutex
// (scenarios/ScenarioTrain.cpp:388-395): tuples flow in (`learner->Train(exp->GetTuples())`, learning/NeuralNetLearner.cpp:33-46) and
// weights flow back (`SyncNet`, :85-89).  Across GPUs these become
//   * ONE all-gather of a fixed-capacity tuple block per rank and outer update -- packed on the device (f32 rows as
//     cMACETrainer stores them, flags, global env ids, a count header), issued on a side stream of the handle, no host
//     synchronisation anywhere: the next trl_update() can be enqueued right behind it;
//   * a broadcast of the policy (weights + the four offset / scale vectors; with a trainer also target net and momentum).
// Evaluation needs one all-reduce of the batch counters (cOptScenarioPoliEval::OutputResults' merge).
//
// Backends: NCCL, opened with dlopen at trl_comm_init (the library itself has no NCCL dependency; inside a PyTorch process the
// soname resolves to the libnccl torch already loaded), or caller-supplied collectives (trl_comm_init_external).
#include <cuda_runtime.h>
#include <dlfcn.h>

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/terrainrl_b200.h"
#include "trl_handle.h"
#include "trl_comm.h"

namespace trl {
void launch_stats(const Buffers& B, double* out, cudaStream_t st);
}

using namespace trl;

#define CCK(call)                                                                                       \
    do {                                                                                                \
        cudaError_t e__ = (call);                                                                       \
        if (e__ != cudaSuccess) return trl_fail(std::string(#call) + ": " + cudaGetErrorString(e__));   \
    } while (0)

// ---------------------------------------------------------------------------------------------------- NCCL, resolved at run time
namespace {
// the handful of NCCL entry points used, with the ABI-stable scalar types of nccl.h spelled out (ncclInt8 = 0, ncclFloat64 = 8,
// ncclSum = 0, ncclUniqueId = 128 bytes passed by value)
struct NcclId { char internal[TRL_COMM_ID_BYTES]; };
struct NcclApi {
    void* lib = nullptr;
    int (*GetUniqueId)(NcclId*) = nullptr;
    int (*CommInitRank)(void**, int, NcclId, int) = nullptr;
    int (*CommDestroy)(void*) = nullptr;
    const char* (*GetErrorString)(int) = nullptr;
    int (*AllGather)(const void*, void*, size_t, int, void*, cudaStream_t) = nullptr;
    int (*Broadcast)(const void*, void*, size_t, int, int, void*, cudaStream_t) = nullptr;
    int (*AllReduce)(const void*, void*, size_t, int, int, void*, cudaStream_t) = nullptr;
    int (*GroupStart)() = nullptr;
    int (*GroupEnd)() = nullptr;
};
NcclApi g_nccl;
constexpr int kNcclInt8 = 0, kNcclFloat64 = 8, kNcclSum = 0;

int load_nccl() {
    if (g_nccl.lib) return 0;
    const char* names[] = {std::getenv("TRL_NCCL_LIB"), "libnccl.so.2", "libnccl.so"};
    void* lib = nullptr;
    for (const char* n : names) {
        if (!n || !*n) continue;
        lib = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
        if (lib) break;
    }
    if (!lib) return trl_fail(std::string("trl_comm: cannot open libnccl.so.2 (") + (dlerror() ? dlerror() : "?") + "); set TRL_NCCL_LIB");
    NcclApi a;
    a.lib = lib;
    auto sym = [&](const char* s) { return dlsym(lib, s); };
    a.GetUniqueId = (decltype(a.GetUniqueId))sym("ncclGetUniqueId");
    a.CommInitRank = (decltype(a.CommInitRank))sym("ncclCommInitRank");
    a.CommDestroy = (decltype(a.CommDestroy))sym("ncclCommDestroy");
    a.GetErrorString = (decltype(a.GetErrorString))sym("ncclGetErrorString");
    a.AllGather = (decltype(a.AllGather))sym("ncclAllGather");
    a.Broadcast = (decltype(a.Broadcast))sym("ncclBroadcast");
    a.AllReduce = (decltype(a.AllReduce))sym("ncclAllReduce");
    a.GroupStart = (decltype(a.GroupStart))sym("ncclGroupStart");
    a.GroupEnd = (decltype(a.GroupEnd))sym("ncclGroupEnd");
    if (!a.GetUniqueId || !a.CommInitRank || !a.CommDestroy || !a.GetErrorString || !a.AllGather || !a.Broadcast || !a.AllReduce ||
        !a.GroupStart || !a.GroupEnd)
        return trl_fail("trl_comm: libnccl lacks a required entry point");
    g_nccl = a;
    return 0;
}
int nccl_fail(const char* what, int rc) {
    return trl_fail(std::string(what) + ": " + (g_nccl.GetErrorString ? g_nccl.GetErrorString(rc) : "NCCL error"));
}
}  // namespace

// ---------------------------------------------------------------------------------------------------- device side
namespace trl_comm_k {

// Pack the rank's tuple block for the exchange.  One CTA per tuple slot; slots [0, m) go to the send block as
// {flags (bit 31 = failed cNeuralNetTrainer::CheckTuple, evaluated on the f64 values; bits 24..26 = the env's policy slot when
// env_slot is given, i.e. in a handle with training slots), env_offset + env, f32 row}; slots [m, count) -- more tuples than one
// block carries -- go to the scratch block and are moved to the front by k_pack_finish.
__global__ void k_pack_tuples(Buffers B, unsigned char* send, int R, int W, int rank, long long env_offset, double* scr_rows,
                              uint32_t* scr_flags, int* scr_env, int* dropped, const int* env_slot) {
    const int raw = *B.tuple_count;
    const int count = min(raw, B.tuple_cap);
    const int m = min(count, R);
    int* hdr = (int*)send;
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        hdr[0] = m; hdr[1] = count - m; hdr[2] = rank; hdr[3] = R;
        if (raw > B.tuple_cap) *dropped += raw - B.tuple_cap;       // the step kernel refused these (trl_step.cu: exp_new_cycle_update)
    }
    const int i = blockIdx.x;
    if (i >= count) return;
    const double* src = B.tuples + (size_t)i * W;
    if (i < m) {
        uint32_t* flags = (uint32_t*)(send + 16);
        int* env = (int*)(send + 16 + (size_t)4 * R);
        float* rows = (float*)(send + 16 + (size_t)8 * R) + (size_t)i * W;
        int bad = 0;
        for (int k = threadIdx.x; k < W; k += blockDim.x) { const double v = src[k]; bad |= !isfinite(v); rows[k] = (float)v; }
        bad = __syncthreads_or(bad);
        if (threadIdx.x == 0) {
            const int e = B.tuple_env[i];
            const uint32_t slot = env_slot ? (uint32_t)env_slot[e] << 24 : 0u;
            flags[i] = (B.tuple_flags[i] & 0x7fffffffu) | slot | (bad ? 0x80000000u : 0u);
            env[i] = (int)(env_offset + e);
        }
    } else {
        double* dst = scr_rows + (size_t)(i - m) * W;
        for (int k = threadIdx.x; k < W; k += blockDim.x) dst[k] = src[k];
        if (threadIdx.x == 0) { scr_flags[i - m] = B.tuple_flags[i]; scr_env[i - m] = B.tuple_env[i]; }
    }
}
// the queued remainder moves to the front of the tuple block; the block's count becomes the remainder (cScenarioExp::ResetTupleBuffer
// for what was shipped)
__global__ void k_pack_finish(Buffers B, const unsigned char* send, int W, const double* scr_rows, const uint32_t* scr_flags,
                              const int* scr_env) {
    const int left = ((const int*)send)[1];
    if (blockIdx.x == 0 && threadIdx.x == 0) *B.tuple_count = left;
    const int i = blockIdx.x;
    if (i >= left) return;
    double* dst = B.tuples + (size_t)i * W;
    const double* src = scr_rows + (size_t)i * W;
    for (int k = threadIdx.x; k < W; k += blockDim.x) dst[k] = src[k];
    if (threadIdx.x == 0) { B.tuple_flags[i] = scr_flags[i]; B.tuple_env[i] = scr_env[i]; }
}
// max |a - b| over n doubles -> out[0] (one CTA)
__global__ void k_max_abs_diff(const double* a, const double* b, int n, double* out) {
    __shared__ double red[32];
    double v = 0;
    for (int i = threadIdx.x; i < n; i += blockDim.x) v = fmax(v, fabs(a[i] - b[i]));
    for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0;
        for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t = fmax(t, red[w]);
        out[0] = t;
    }
}
}  // namespace trl_comm_k

// ---------------------------------------------------------------------------------------------------- host side
struct trl_comm {
    int rank = 0, world = 1;
    void* nccl = nullptr;                 // ncclComm_t
    bool external = false;
    trl_collectives coll{};
    cudaStream_t stream = nullptr;        // collectives run here; ordered against the handle's stream with events
    cudaEvent_t ev_packed = nullptr, ev_gathered = nullptr, ev_misc = nullptr, ev_consumed = nullptr;
    int block_rows = 0, width = 0;
    size_t block_bytes = 0;
    unsigned char *send = nullptr, *recv = nullptr;
    double* scr_rows = nullptr;
    uint32_t* scr_flags = nullptr;
    int* scr_env = nullptr;
    int* dropped = nullptr;               // device counter
    double* small = nullptr;              // [9] device scratch for the small reductions
    double* wscratch = nullptr;           // parameter-sized scratch (replica check)
    size_t wscratch_n = 0;
    long long env_offset = 0;
    bool gathered = false;
    std::vector<void*> allocs;
};

static int coll_all_gather(trl_comm* c, const void* send, void* recv, size_t bytes) {
    if (c->external) {
        if (c->coll.all_gather(c->coll.ctx, send, recv, bytes, (void*)c->stream)) return trl_fail("trl_comm: external all_gather failed");
        return 0;
    }
    const int rc = g_nccl.AllGather(send, recv, bytes, kNcclInt8, c->nccl, c->stream);
    return rc ? nccl_fail("ncclAllGather", rc) : 0;
}
static int coll_broadcast(trl_comm* c, void* buf, size_t bytes, int root) {
    if (c->external) {
        if (c->coll.broadcast(c->coll.ctx, buf, bytes, root, (void*)c->stream)) return trl_fail("trl_comm: external broadcast failed");
        return 0;
    }
    const int rc = g_nccl.Broadcast(buf, buf, bytes, kNcclInt8, root, c->nccl, c->stream);
    return rc ? nccl_fail("ncclBroadcast", rc) : 0;
}
static int coll_all_reduce_sum(trl_comm* c, double* buf, size_t count) {
    if (c->external) {
        if (c->coll.all_reduce_sum_f64(c->coll.ctx, buf, count, (void*)c->stream)) return trl_fail("trl_comm: external all_reduce failed");
        return 0;
    }
    const int rc = g_nccl.AllReduce(buf, buf, count, kNcclFloat64, kNcclSum, c->nccl, c->stream);
    return rc ? nccl_fail("ncclAllReduce", rc) : 0;
}
static void group_start(trl_comm* c) { if (!c->external) g_nccl.GroupStart(); }
static int group_end(trl_comm* c) {
    if (c->external) return 0;
    const int rc = g_nccl.GroupEnd();
    return rc ? nccl_fail("ncclGroupEnd", rc) : 0;
}

// cudaMemset of device memory runs on the legacy default stream, which does not order against the handle's non-blocking streams:
// without the synchronisation a late memset could clear what the first kernel or copy on those streams wrote (the replica check's
// scratch, a first send block)
template <typename T>
static cudaError_t calloc_dev(trl_comm* c, T** p, size_t count) {
    cudaError_t e = cudaMalloc((void**)p, std::max<size_t>(count, 1) * sizeof(T));
    if (e == cudaSuccess) { c->allocs.push_back(*p); e = cudaMemset(*p, 0, std::max<size_t>(count, 1) * sizeof(T)); }
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    return e;
}

static int comm_common(trl_handle* h, trl_comm* c) {
    CCK(cudaSetDevice(h->device));
    CCK(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
    CCK(cudaEventCreate(&c->ev_packed));
    CCK(cudaEventCreate(&c->ev_gathered));
    CCK(cudaEventCreateWithFlags(&c->ev_misc, cudaEventDisableTiming));
    CCK(cudaEventCreateWithFlags(&c->ev_consumed, cudaEventDisableTiming));
    c->width = 1 + h->B.S + h->B.A + h->B.S;
    c->env_offset = (long long)c->rank * h->n;
    CCK(calloc_dev(c, &c->dropped, 1));
    CCK(calloc_dev(c, &c->small, 9));
    CCK(calloc_dev(c, &c->scr_rows, (size_t)h->B.tuple_cap * c->width));
    CCK(calloc_dev(c, &c->scr_flags, (size_t)h->B.tuple_cap));
    CCK(calloc_dev(c, &c->scr_env, (size_t)h->B.tuple_cap));
    h->comm = c;
    return 0;
}

static int ensure_blocks(trl_handle* h, int block_rows) {
    trl_comm* c = h->comm;
    if (block_rows <= 0) block_rows = 1024;
    block_rows = std::min((block_rows + 3) & ~3, (h->B.tuple_cap + 3) & ~3);
    if (c->block_rows == block_rows) return 0;
    if (c->block_rows != 0) {
        // a different capacity: the old blocks may still be in flight
        CCK(cudaStreamSynchronize(c->stream));
        CCK(cudaStreamSynchronize(h->stream));
        cudaFree(c->send); cudaFree(c->recv);
        c->allocs.erase(std::remove(c->allocs.begin(), c->allocs.end(), (void*)c->send), c->allocs.end());
        c->allocs.erase(std::remove(c->allocs.begin(), c->allocs.end(), (void*)c->recv), c->allocs.end());
        c->gathered = false;
    }
    c->block_rows = block_rows;
    c->block_bytes = 16 + (size_t)8 * block_rows + (size_t)4 * block_rows * c->width;
    CCK(calloc_dev(c, &c->send, c->block_bytes));
    CCK(calloc_dev(c, &c->recv, c->block_bytes * c->world));
    return 0;
}

extern "C" {

int trl_comm_unique_id(void* id128) {
    if (!id128) return trl_fail("trl_comm_unique_id: null buffer");
    if (load_nccl()) return 1;
    NcclId id;
    const int rc = g_nccl.GetUniqueId(&id);
    if (rc) return nccl_fail("ncclGetUniqueId", rc);
    std::memcpy(id128, &id, TRL_COMM_ID_BYTES);
    return 0;
}

int trl_comm_init(trl_handle* h, const void* id128, int rank, int world) {
    if (!h) return trl_fail("trl_comm_init: null handle");
    if (h->comm) return trl_fail("trl_comm_init: the handle already has a communicator");
    if (h->env_eval) return trl_fail("trl_comm_init: the handle has evaluation envs (trl_set_env_eval)");
    if (h->ranges.body_ranged || h->ranges.phys_ranged) return trl_fail("trl_comm_init: the handle has ranged slots (trl_load_body_range / trl_load_physics_range)");
    if (!id128 || world < 1 || rank < 0 || rank >= world) return trl_fail("trl_comm_init: bad rank / world / id");
    if (load_nccl()) return 1;
    CCK(cudaSetDevice(h->device));
    auto* c = new trl_comm();
    c->rank = rank; c->world = world;
    NcclId id;
    std::memcpy(&id, id128, TRL_COMM_ID_BYTES);
    const int rc = g_nccl.CommInitRank(&c->nccl, world, id, rank);
    if (rc) { delete c; return nccl_fail("ncclCommInitRank", rc); }
    if (comm_common(h, c)) { h->comm = c; trl_comm_destroy(h); return 1; }
    return 0;
}

int trl_comm_init_external(trl_handle* h, const trl_collectives* coll, int rank, int world) {
    if (!h) return trl_fail("trl_comm_init_external: null handle");
    if (h->comm) return trl_fail("trl_comm_init_external: the handle already has a communicator");
    if (h->env_eval) return trl_fail("trl_comm_init_external: the handle has evaluation envs (trl_set_env_eval)");
    if (h->ranges.body_ranged || h->ranges.phys_ranged) return trl_fail("trl_comm_init_external: the handle has ranged slots (trl_load_body_range / trl_load_physics_range)");
    if (!coll || !coll->all_gather || !coll->broadcast || !coll->all_reduce_sum_f64 || world < 1 || rank < 0 || rank >= world)
        return trl_fail("trl_comm_init_external: bad rank / world / callbacks");
    auto* c = new trl_comm();
    c->rank = rank; c->world = world; c->external = true; c->coll = *coll;
    if (comm_common(h, c)) { h->comm = c; trl_comm_destroy(h); return 1; }
    return 0;
}

int trl_comm_destroy(trl_handle* h) {
    if (!h || !h->comm) return 0;
    trl_comm* c = h->comm;
    if (c->stream) cudaStreamSynchronize(c->stream);
    if (h->stream) cudaStreamSynchronize(h->stream);
    if (c->nccl) g_nccl.CommDestroy(c->nccl);
    for (void* p : c->allocs) cudaFree(p);
    if (c->ev_packed) cudaEventDestroy(c->ev_packed);
    if (c->ev_gathered) cudaEventDestroy(c->ev_gathered);
    if (c->ev_misc) cudaEventDestroy(c->ev_misc);
    if (c->ev_consumed) cudaEventDestroy(c->ev_consumed);
    if (c->stream) cudaStreamDestroy(c->stream);
    delete c;
    h->comm = nullptr;
    return 0;
}

int trl_comm_info(trl_handle* h, int* rank, int* world, int* block_rows) {
    if (!h || !h->comm) return trl_fail("trl_comm_info: no communicator (trl_comm_init first)");
    if (rank) *rank = h->comm->rank;
    if (world) *world = h->comm->world;
    if (block_rows) *block_rows = h->comm->block_rows;
    return 0;
}

int trl_comm_set_env_offset(trl_handle* h, int64_t env_offset) {
    if (!h || !h->comm) return trl_fail("trl_comm_set_env_offset: no communicator (trl_comm_init first)");
    h->comm->env_offset = env_offset;
    return 0;
}

// pack on the handle's stream (behind the update that produced the tuples), all-gather on the comm stream
int trl_gather_tuples(trl_handle* h, int block_rows) {
    if (!h || !h->comm) return trl_fail("trl_gather_tuples: no communicator (trl_comm_init first)");
    trl_comm* c = h->comm;
    if (ensure_blocks(h, block_rows)) return 1;
    // the previous all-gather must have finished reading the send block (it has, whenever its result was consumed)
    if (c->gathered) CCK(cudaStreamWaitEvent(h->stream, c->ev_gathered, 0));
    const Buffers& B = h->B;
    TRL_LAUNCH(trl_comm_k::k_pack_tuples, B.tuple_cap, 128, 0, h->stream, B, c->send, c->block_rows, c->width, c->rank, c->env_offset,
               c->scr_rows, c->scr_flags, c->scr_env, c->dropped, h->train_slots ? h->P.env_slot : (const int*)nullptr);
    TRL_LAUNCH(trl_comm_k::k_pack_finish, B.tuple_cap, 128, 0, h->stream, B, (const unsigned char*)c->send, c->width,
               (const double*)c->scr_rows, (const uint32_t*)c->scr_flags, (const int*)c->scr_env);
    h->launches += 2;
    CCK(cudaGetLastError());
    CCK(cudaEventRecord(c->ev_packed, h->stream));
    CCK(cudaStreamWaitEvent(c->stream, c->ev_packed, 0));
    if (coll_all_gather(c, c->send, c->recv, c->block_bytes)) return 1;
    CCK(cudaEventRecord(c->ev_gathered, c->stream));
    c->gathered = true;
    return 0;
}

int trl_gathered_blocks(trl_handle* h, const void** dev_blocks, size_t* block_bytes, int* block_rows, int* row_width) {
    if (!h || !h->comm) return trl_fail("trl_gathered_blocks: no communicator (trl_comm_init first)");
    trl_comm* c = h->comm;
    if (!c->gathered) return trl_fail("trl_gathered_blocks: nothing gathered yet (trl_gather_tuples first)");
    CCK(cudaStreamWaitEvent(h->stream, c->ev_gathered, 0));
    if (dev_blocks) *dev_blocks = c->recv;
    if (block_bytes) *block_bytes = c->block_bytes;
    if (block_rows) *block_rows = c->block_rows;
    if (row_width) *row_width = c->width;
    return 0;
}

int trl_gathered_fetch(trl_handle* h, int32_t* counts, float* rows, uint32_t* flags, int32_t* env, int cap, int* n_total) {
    if (!h || !h->comm) return trl_fail("trl_gathered_fetch: no communicator (trl_comm_init first)");
    trl_comm* c = h->comm;
    if (!c->gathered) return trl_fail("trl_gathered_fetch: nothing gathered yet (trl_gather_tuples first)");
    CCK(cudaEventSynchronize(c->ev_gathered));
    const int R = c->block_rows, W = c->width;
    int total = 0;
    for (int r = 0; r < c->world; ++r) {
        const unsigned char* blk = c->recv + (size_t)r * c->block_bytes;
        int hdr[4];
        CCK(cudaMemcpy(hdr, blk, 16, cudaMemcpyDeviceToHost));
        if (hdr[0] < 0 || hdr[0] > R || hdr[3] != R) return trl_fail("trl_gathered_fetch: corrupt block header");
        if (counts) counts[r] = hdr[0];
        const int take = std::max(0, std::min(hdr[0], cap - total));
        if (take > 0) {
            if (flags) CCK(cudaMemcpy(flags + total, blk + 16, (size_t)take * 4, cudaMemcpyDeviceToHost));
            if (env) CCK(cudaMemcpy(env + total, blk + 16 + (size_t)4 * R, (size_t)take * 4, cudaMemcpyDeviceToHost));
            if (rows) CCK(cudaMemcpy(rows + (size_t)total * W, blk + 16 + (size_t)8 * R, (size_t)take * W * 4, cudaMemcpyDeviceToHost));
        }
        total += hdr[0];
    }
    if (n_total) *n_total = total;
    return 0;
}

int trl_gather_last_ms(trl_handle* h, double* ms) {
    if (!h || !h->comm) return trl_fail("trl_gather_last_ms: no communicator (trl_comm_init first)");
    trl_comm* c = h->comm;
    if (!c->gathered) return trl_fail("trl_gather_last_ms: nothing gathered yet");
    CCK(cudaEventSynchronize(c->ev_gathered));
    float f = 0;
    CCK(cudaEventElapsedTime(&f, c->ev_packed, c->ev_gathered));
    if (ms) *ms = f;
    return 0;
}

int trl_tuples_dropped(trl_handle* h, int64_t* out) {
    if (!h) return trl_fail("trl_tuples_dropped: null handle");
    int64_t total = h->tuples_dropped;
    if (h->comm) {
        int d = 0;
        CCK(cudaStreamSynchronize(h->stream));
        CCK(cudaMemcpy(&d, h->comm->dropped, 4, cudaMemcpyDeviceToHost));
        total += d;
    }
    if (out) *out = total;
    return 0;
}

// every array that defines the policy the decision kernel evaluates, from `root` to all ranks (cNeuralNetLearner::SyncNet)
static int broadcast_arrays(trl_handle* h, double* const* arrays, const size_t* counts, int n, int root) {
    trl_comm* c = h->comm;
    CCK(cudaEventRecord(c->ev_misc, h->stream));
    CCK(cudaStreamWaitEvent(c->stream, c->ev_misc, 0));
    group_start(c);
    for (int i = 0; i < n; ++i)
        if (coll_broadcast(c, arrays[i], counts[i] * 8, root)) { group_end(c); return 1; }
    if (group_end(c)) return 1;
    CCK(cudaEventRecord(c->ev_misc, c->stream));
    CCK(cudaStreamWaitEvent(h->stream, c->ev_misc, 0));
    return 0;
}

int trl_comm_broadcast_weights(trl_handle* h, int root) {
    if (!h || !h->comm) return trl_fail("trl_comm_broadcast_weights: no communicator (trl_comm_init first)");
    if (!h->mc.has_net) return trl_fail("trl_comm_broadcast_weights: scene has no policy net");
    if (h->trainer) return trl_fail("trl_comm_broadcast_weights: a trainer owns the weights (use trl_trainer_broadcast)");
    if (root < 0 || root >= h->comm->world) return trl_fail("trl_comm_broadcast_weights: bad root");
    std::vector<size_t> counts(30);
    for (int i = 0; i < 30; ++i) counts[i] = (size_t)h->net_counts[i];
    if (broadcast_arrays(h, h->net_blobs.data(), counts.data(), 30, root)) return 1;
    // OutputScale of actor 0 scales the exploration noise from constant memory (trl_set_weights does the same)
    std::vector<double> os((size_t)h->net_counts[29]);
    CCK(cudaStreamSynchronize(h->stream));
    CCK(cudaMemcpy(os.data(), h->net_blobs[29], os.size() * 8, cudaMemcpyDeviceToHost));
    for (int k = 0; k < h->mc.frag; ++k) h->mc.out_scale_actor0[k] = os[h->mc.n_frags + k];
    return trl_reupload_model(h);
}

int trl_comm_eval_stats(trl_handle* h, int64_t* cycles, int64_t* episodes, double* avg_dist, int64_t* env_steps) {
    if (!h || !h->comm) return trl_fail("trl_comm_eval_stats: no communicator (trl_comm_init first)");
    trl_comm* c = h->comm;
    launch_stats(h->B, c->small, h->stream);
    h->launches += 1;
    CCK(cudaEventRecord(c->ev_misc, h->stream));
    CCK(cudaStreamWaitEvent(c->stream, c->ev_misc, 0));
    if (coll_all_reduce_sum(c, c->small, 4)) return 1;
    CCK(cudaStreamSynchronize(c->stream));
    double st[4];
    CCK(cudaMemcpy(st, c->small, 32, cudaMemcpyDeviceToHost));
    if (cycles) *cycles = (int64_t)st[0];
    if (episodes) *episodes = (int64_t)st[1];
    if (env_steps) *env_steps = (int64_t)st[2];
    if (avg_dist) *avg_dist = st[1] > 0 ? st[3] / st[1] : 0.0;
    return 0;
}

// trl_comm_eval_stats over the envs of one policy slot: trl_eval_stats_slot of every rank, summed
int trl_comm_eval_stats_slot(trl_handle* h, int slot, int64_t* cycles, int64_t* episodes, double* avg_dist, int64_t* env_steps) {
    if (!h || !h->comm) return trl_fail("trl_comm_eval_stats_slot: no communicator (trl_comm_init first)");
    trl_comm* c = h->comm;
    if (trl_slot_stats_dev(h, "trl_comm_eval_stats_slot", slot, c->small)) return 1;
    CCK(cudaEventRecord(c->ev_misc, h->stream));
    CCK(cudaStreamWaitEvent(c->stream, c->ev_misc, 0));
    if (coll_all_reduce_sum(c, c->small, 4)) return 1;
    CCK(cudaStreamSynchronize(c->stream));
    double st[4];
    CCK(cudaMemcpy(st, c->small, 32, cudaMemcpyDeviceToHost));
    if (cycles) *cycles = (int64_t)st[0];
    if (episodes) *episodes = (int64_t)st[1];
    if (env_steps) *env_steps = (int64_t)st[2];
    if (avg_dist) *avg_dist = st[1] > 0 ? st[3] / st[1] : 0.0;
    return 0;
}

}  // extern "C"

// ---------------------------------------------------------------------------------------------------- used by trl_train.cu
int trl_comm_view(trl_handle* h, trl_comm_blocks* out) {
    if (!h || !h->comm) return trl_fail("trainer: the scenario has no communicator (trl_comm_init first)");
    trl_comm* c = h->comm;
    if (!c->gathered) return trl_fail("trainer: nothing gathered yet (trl_gather_tuples first)");
    CCK(cudaStreamWaitEvent(h->stream, c->ev_gathered, 0));
    out->recv = c->recv; out->block_bytes = c->block_bytes; out->block_rows = c->block_rows; out->width = c->width;
    out->world = c->world; out->rank = c->rank;
    return 0;
}
int trl_comm_view_on(trl_handle* h, trl_comm_blocks* out, cudaStream_t consumer) {
    if (!h || !h->comm) return trl_fail("trainer: the scenario has no communicator (trl_comm_init first)");
    trl_comm* c = h->comm;
    if (!c->gathered) return trl_fail("trainer: nothing gathered yet (trl_gather_tuples first)");
    CCK(cudaStreamWaitEvent(consumer, c->ev_gathered, 0));
    out->recv = c->recv; out->block_bytes = c->block_bytes; out->block_rows = c->block_rows; out->width = c->width;
    out->world = c->world; out->rank = c->rank;
    return 0;
}
// the comm stream waits for every consumer as it is marked (a join): any number of trainers, each on its own stream, may read one
// gathered set of blocks, and the next all-gather overwrites them only after the last of them
int trl_comm_mark_consumed(trl_handle* h, cudaStream_t consumer) {
    if (!h || !h->comm) return 0;
    CCK(cudaEventRecord(h->comm->ev_consumed, consumer));
    CCK(cudaStreamWaitEvent(h->comm->stream, h->comm->ev_consumed, 0));
    return 0;
}
int trl_comm_broadcast_list(trl_handle* h, double* const* arrays, const size_t* counts, int n, int root) {
    if (!h || !h->comm) return trl_fail("trainer: the scenario has no communicator (trl_comm_init first)");
    if (root < 0 || root >= h->comm->world) return trl_fail("trainer: bad broadcast root");
    return broadcast_arrays(h, arrays, counts, n, root);
}
// max over ranks of max_i |theta_i - theta_i(root 0)|: 0 iff every replica holds rank 0's parameters bit for bit
int trl_comm_replica_spread(trl_handle* h, const double* theta, size_t n, double* out) {
    if (!h || !h->comm) return trl_fail("trainer: the scenario has no communicator (trl_comm_init first)");
    trl_comm* c = h->comm;
    if (c->wscratch_n < n) {
        CCK(calloc_dev(c, &c->wscratch, n));
        c->wscratch_n = n;
    }
    CCK(cudaMemcpyAsync(c->wscratch, theta, n * 8, cudaMemcpyDeviceToDevice, h->stream));
    CCK(cudaEventRecord(c->ev_misc, h->stream));
    CCK(cudaStreamWaitEvent(c->stream, c->ev_misc, 0));
    if (coll_broadcast(c, c->wscratch, n * 8, 0)) return 1;
    TRL_LAUNCH(trl_comm_k::k_max_abs_diff, 1, 1024, 0, c->stream, theta, (const double*)c->wscratch, (int)n, c->small + 4);
    if (coll_all_reduce_sum(c, c->small + 4, 1)) return 1;
    CCK(cudaStreamSynchronize(c->stream));
    CCK(cudaMemcpy(out, c->small + 4, 8, cudaMemcpyDeviceToHost));
    return 0;
}
// Do all ranks hold the same 64-bit signature, and did every rank accept the call (`ok`)?  Four 16-bit pieces v, their squares and a
// refusal count go through one all-reduce; the pieces agree on every rank iff (sum v)^2 == world * sum v^2 (Cauchy-Schwarz), and every
// rank evaluates that on the same reduced numbers, so all ranks reach the same answers.  The sums stay below 2^53, exact in f64, up to
// 1024 ranks.  Synchronises.
int trl_comm_agree(trl_handle* h, uint64_t sig, bool ok, bool* same, bool* all_ok) {
    if (!h || !h->comm) return trl_fail("trainer: the scenario has no communicator (trl_comm_init first)");
    trl_comm* c = h->comm;
    double v[9];
    for (int k = 0; k < 4; ++k) {
        v[k] = (double)((sig >> (16 * k)) & 0xffffu);
        v[4 + k] = v[k] * v[k];
    }
    v[8] = ok ? 0.0 : 1.0;
    CCK(cudaStreamSynchronize(h->stream));
    CCK(cudaMemcpyAsync(c->small, v, sizeof(v), cudaMemcpyHostToDevice, c->stream));
    if (coll_all_reduce_sum(c, c->small, 9)) return 1;
    CCK(cudaMemcpyAsync(v, c->small, sizeof(v), cudaMemcpyDeviceToHost, c->stream));
    CCK(cudaStreamSynchronize(c->stream));
    *same = true;
    for (int k = 0; k < 4; ++k) *same = *same && v[k] * v[k] == (double)c->world * v[4 + k];
    *all_ok = v[8] == 0.0;
    return 0;
}
