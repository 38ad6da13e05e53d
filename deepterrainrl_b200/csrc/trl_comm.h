// deepterrainrl_b200 -- what the trainer (trl_train.cu) needs from the multi-GPU exchange (trl_comm.cu); private to csrc/
#pragma once
#include <cuda_runtime.h>

#include <cstddef>
#include <cstdint>

struct trl_handle;

// the all-gathered tuple blocks as device memory: `world` blocks of block_bytes, each
// {i32 count, i32 queued, i32 rank, i32 block_rows, u32 flags[block_rows], i32 env[block_rows], f32 rows[block_rows][width]}
struct trl_comm_blocks {
    const unsigned char* recv;
    size_t block_bytes;
    int block_rows, width, world, rank;
};
// orders the handle's stream behind the last all-gather and returns the view
int trl_comm_view(trl_handle* h, trl_comm_blocks* out);
int trl_comm_broadcast_list(trl_handle* h, double* const* arrays, const size_t* counts, int n, int root);
int trl_comm_replica_spread(trl_handle* h, const double* theta, size_t n, double* out);
// the consumer of the gathered blocks runs on `consumer` (not the handle's stream): orders it behind the last all-gather, and makes
// the next all-gather wait until `mark_consumed` has been recorded on that stream
int trl_comm_view_on(trl_handle* h, trl_comm_blocks* out, cudaStream_t consumer);
int trl_comm_mark_consumed(trl_handle* h, cudaStream_t consumer);
// whether every rank passed the same signature, and whether every rank passed ok (one small all-reduce; synchronises).  Every rank
// gets the same answers.
int trl_comm_agree(trl_handle* h, uint64_t sig, bool ok, bool* same, bool* all_ok);
// policy slot `slot`'s {cycles, episodes, env-steps, distance sum} into device memory out4 on the handle's stream (trl_host.cu)
extern "C" int trl_slot_stats_dev(trl_handle* h, const char* who, int slot, double* out4);
