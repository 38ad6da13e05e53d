// deepterrainrl_b200 -- the batch handle behind the C ABI (private to csrc/: trl_host.cu, trl_train.cu)
#pragma once
#include <cuda_runtime.h>

#include <cstdint>
#include <map>
#include <string>
#include <vector>

#include "scene_pack.h"
#include "trl_types.h"
#include "trl_fcmaps.h"

struct trl_trainer;
struct trl_comm;

struct trl_handle {
    trl_trainer* trainer = nullptr;      // attached MACE trainer (trl_train.cu), owns the policy weights when present
    trl_comm* comm = nullptr;            // multi-GPU exchange (trl_comm.cu), present after trl_comm_init*
    int64_t tuples_dropped = 0;          // tuples the full tuple block refused, as observed by the host-side readers
    int device = 0, n = 0, mode = 0;
    trl::ScenePack scene;
    trl::ModelConst mc;
    // exploration settings per policy slot (trl_set_explore writes every entry, trl_set_explore_slot one).  Host copy; the kernels read
    // the device table d_ex: the single-policy kernels entry 0, the slot build the entry of each chunk's slot.  `noise` is the same in
    // every entry (the scene's exploration noise std)
    trl::ExpSettings ex[trl::kMaxPolicySlots];
    trl::ExpSettings* d_ex = nullptr;
    trl::Buffers B;
    trl::NetWeights W{};
    std::vector<double*> net_blobs;      // 26 + 4 device arrays
    std::vector<int64_t> net_counts;
    int* done_count = nullptr;
    cudaStream_t stream = nullptr;
    cudaStream_t aux_stream = nullptr;           // = side[0]
    cudaStream_t side[8] = {nullptr};            // high-priority side streams: decisions + catch-up launches of env-step l run on side[l % lag]
    int groups = 2;                              // env groups of the main step launches (TRL_GROUPS, 1..kMaxGroups; reduced when a group would be empty): see enqueue_update
    cudaStream_t group_stream[7] = {nullptr};    // streams of groups 1 .. groups-1 (group 0 runs on `stream`)
    int lag = 6;                                 // overlap depth: env-steps a pending env may trail the main launches (TRL_LAG, 1..7)
    std::vector<cudaEvent_t> fork_events;        // dependencies between the two streams inside one update
    bool overlap = true;                         // TRL_SERIAL_SCHEDULE=1 turns the overlapped schedule off
    int decide_grid = 288;   // CTAs of the decision launch: a multiple of its cluster size (create_common sizes it from the SM count)
    int num_update_steps = 20;
    // batched decision path (trl_decide2.cuh): conv2 outputs of the pending decisions, the TMA descriptors over them and over the
    // terr_ip0 weights (re-encoded whenever the weight pointer changes), number of FC-stage clusters
    bool decide_v2 = true;                       // TRL_DECIDE_V1=1 selects the one-cluster-per-decision kernel (trl_decide.cuh)
    double* act2[8] = {nullptr};                 // one scratch matrix per side stream (the decisions of several env-steps can overlap)
    trl::FcMaps fc_maps[8];
    const double* fc_maps_w = nullptr;
    int fc_clusters = 2;
    // policy slots (trl_load_policy, evaluation handles only): slot 0 is W / net_blobs above, slots 1.. own their blobs.  While any
    // slot >= 1 is loaded (slots_active) every decision goes through the slot build of the decision kernels; before that nothing below
    // is allocated and the single-policy kernels run
    bool slots_active = false;
    bool slot_dirty = false;                                 // a slot was (re)loaded: device table and descriptors to be rewritten
    std::vector<double*> slot_blobs[trl::kMaxPolicySlots];   // [0] unused
    trl::NetWeights slot_W[trl::kMaxPolicySlots] = {};       // [0] mirrors W when the device table was last written
    std::vector<int> env_slot_host;
    trl::PolicySlots P{};                                    // device views (env_slot, weight table, sort scratch, chunk tables)
    trl::FcSlotMaps slot_maps{};
    // training slots (trl_trainer_create_slot, exploration handles only): slot p >= 1 trains with slot_trainer[p], whose current net is
    // slot_W[p]; slot 0's trainer stays `trainer`.  train_slots stays set once a slot trainer was created: the tuple block is then
    // shared by slot, and its hand-over no longer clears it (trl_train_run_slots does, once every trainer has taken its rows)
    bool train_slots = false;
    trl_trainer* slot_trainer[trl::kMaxPolicySlots] = {};    // [0] unused
    // terrain slots (trl_load_terrain, any mode): slot 0 is mc.terrain_type / terrain_params, slots 1.. keep a terrain file's parameter
    // sets, blended at terrain_lerp into terrain[] (the __constant__ table, uploaded with the model).  Until a slot >= 1 is loaded
    // env_terrain_host is empty and every env is on slot 0 (the planes I_TERRAIN_SLOT / I_TERRAIN_SLOT_NEXT stay zero)
    double terrain_lerp = 0.0;                                 // the handle's blend: -terrain_blend, then trl_set_terrain_lerp
    trl::TerrainSlot terrain[trl::kMaxTerrainSlots] = {};
    std::vector<double> terrain_sets[trl::kMaxTerrainSlots];   // [n_sets][40] of each loaded slot ([0] unused)
    bool terrain_loaded[trl::kMaxTerrainSlots] = {};           // [0] unused
    std::vector<int> env_terrain_host;                         // the assignment of every env (I_TERRAIN_SLOT_NEXT)
    double* cell_stats = nullptr;                              // [kMaxPolicySlots + 1][kMaxTerrainSlots + 1][4] (trl_eval_stats_cell)
    // physics slots (trl_load_physics, any mode): slot 0 is mc.phys (trl_set_phys_params), copied into phys[0] at every upload; slots 1..
    // hold loaded values.  phys[] is the __constant__ table of the physics-slot build.  Until a slot >= 1 is loaded env_phys is null,
    // env_phys_host empty, every env on slot 0, and the step launches run the other builds
    trl::PhysParams phys[trl::kMaxPhysSlots] = {};
    bool phys_loaded[trl::kMaxPhysSlots] = {};                 // [0] unused
    std::vector<int> env_phys_host;                            // the assignment of every env (row 1 of env_phys)
    int* env_phys = nullptr;                                   // device [2][n]: slot of the present episode, slot from the next reset on
    double* phys_stats = nullptr;                              // [4] (trl_eval_stats_phys)
    // evaluation envs (trl_set_env_eval, exploration handles only): until the first call env_eval is null, env_eval_host empty and
    // every env explores.  From then on the decisions run the slot build (slots_active) and the step launches the physics-slot build
    std::vector<int> env_eval_host;                            // the assignment of every env (row 1 of env_eval)
    int* env_eval = nullptr;                                   // device [2][n]: mode of the present episode, mode from the next reset on
    // body slots (trl_load_body, any mode): slot 0 is the scene's body (the per-link numbers of mc), copied into body[0] at every upload;
    // slots 1.. hold bodies loaded from character files of the scene's topology.  body[] is the table of the body-slot build.  Until a
    // slot >= 1 is loaded env_body is null, env_body_host empty, every env on slot 0, and the step launches run the other builds
    trl::BodyConst body[trl::kMaxBodySlots] = {};
    bool body_loaded[trl::kMaxBodySlots] = {};                 // [0] unused
    std::vector<int> env_body_host;                            // the assignment of every env (row 1 of env_body)
    int* env_body = nullptr;                                   // device [2][n]: slot of the present episode, slot from the next reset on
    // ranged slots (trl_load_body_range, trl_load_physics_range): body[s] / phys[s] hold a ranged slot's lo numbers, ranges its hi
    // numbers, its bit in ranges.body_ranged / phys_ranged, and the per-env draw tables (allocated at the first ranged slot, with
    // the body-slot build; null before)
    trl::RangeTables ranges = {};
    std::string data_root;                                     // trl_create's: the directory relative character and controller paths refer to
    int64_t launches = 0;
    std::map<long long, cudaGraphExec_t> graphs;   // keyed by the bit pattern of dt
    bool use_graph = true;
    // host staging
    std::vector<double> h_tuples;
    std::vector<float> h_tuples_f32;
    std::vector<uint32_t> h_tuple_flags;
    std::vector<int32_t> h_tuple_env;
    std::vector<double> h_dist;
    std::vector<int32_t> h_dist_env;
    std::vector<void*> allocs;
    void* flush_buf = nullptr;
    double bench_span_ms = 0.0;          // trl_bench_updates: first update's start to last update's end, flushes included
    double* probe_dump = nullptr;        // every blob of one forward pass (trl_probe.cu: trl_get_layer_state)
    // pipelined read-back (trl_snapshot / trl_snapshot_wait)
    cudaStream_t copy_stream = nullptr;
    cudaEvent_t snap_ready = nullptr, snap_copied = nullptr;
    double* snap_dev = nullptr;      // [2 * ndof * n + 4] device staging (pose planes, vel planes, stats)
    double* snap_host = nullptr;     // pinned mirror
    bool snap_pending = false;
};

// the weights the decisions of `env` use
inline const trl::NetWeights& env_policy(const trl_handle* h, int env) {
    const int p = h->slots_active ? h->env_slot_host[env] : 0;
    return p == 0 ? h->W : h->slot_W[p];
}

// shared by the translation units behind the C ABI
int trl_fail(const std::string& msg);                 // records the message for trl_last_error(), returns 1
void trl_drop_graphs(trl_handle* h);
extern "C" void trl_trainer_orphan(trl_trainer* t);              // trl_destroy with a trainer still attached (trl_train.cu)
int trl_make_fc_maps(trl::FcMaps* out, const double* tip0_w, const double* act2, int rows);   // trl_host.cu
int trl_reupload_model(trl_handle* h);                // after editing h->mc: refresh the __constant__ copies                  // captured graphs bake kernel arguments (weight pointers) in
// policy slot `slot` >= 1 gets its own blobs holding the Caffe-HDF5 model + `_scale.txt` (both paths given) or a copy of slot 0's
// current net, and the handle gets its slot machinery; refused, with nothing changed, for a model of another topology
extern "C" int trl_stage_slot_model(trl_handle* h, int slot, const char* h5_path, const char* scale_path);
// the rest of trl_create_from_pack once h->scene is loaded (nullptr, with h deleted and the reason recorded, on failure)
extern "C" trl_handle* trl_create_common(trl_handle* h, int num_envs, int device, int mode, const uint64_t* terrain_seeds, uint64_t rng_seed);
int trl_drain(trl_handle* h);                         // every stream of the handle idle
// terrain slot `slot` >= 1 holds parameter sets [n][40] of generator `type` (trl_load_terrain once the file is read)
int trl_set_terrain_slot(trl_handle* h, int slot, int type, std::vector<double> sets);
// the per-env modes of trl_set_env_eval, every env exploring, and the decision / step builds that read them (trl_host.cu)
extern "C" int trl_enable_env_eval(trl_handle* h);
// body slot `slot` >= 1 holds `b` (trl_load_body once the file is read and checked), and the handle moves onto the body-slot build
extern "C" int trl_set_body_slot(trl_handle* h, int slot, const trl::BodyConst& b);
// ranged slots: the per-env draw tables and the body-slot build (trl_load_body_range / trl_load_physics_range, a checkpoint's restore);
// body / physics slot `slot` >= 1 drawn in [lo, hi] at every episode reset, after the loaders' checks of the two ends
extern "C" int trl_enable_ranges(trl_handle* h);
extern "C" int trl_set_body_range(trl_handle* h, int slot, const trl::BodyConst& lo, const trl::BodyConst& hi);
extern "C" int trl_set_phys_range(trl_handle* h, int slot, const trl::PhysParams& lo, const trl::PhysParams& hi);

// One array of a checkpoint (trl_checkpoint.cu): `bytes` of device memory at `dev`, or of host memory at `host` when dev is null.
// `cap` is the room there is: a restore accepts up to cap bytes (the replay rows, the tuple block and the distance log are saved up
// to their fill level)
struct CkptSection {
    std::string name;
    int dtype;             // 0 raw bytes, 1 i32, 2 f32, 3 f64 (informative)
    void* dev;
    void* host;
    size_t bytes, cap;
};
// the sections of a trainer's carried state, named prefix + field (trl_train.cu); drains the trainer, refuses an asynchronous one
int trl_trainer_state(trl_trainer* t, const std::string& prefix, std::vector<CkptSection>* out);
