// deepterrainrl_b200 -- batched locomotion rollout engine for H100 (sm_90a).
// Shared host/device types: model constants (constant memory), SoA state layout in HBM, launch parameters.
//
// HBM layout (DESIGN.md §2): every per-env scalar lives in a struct-of-arrays plane `plane[field][env]`, so a warp
// (32 consecutive envs, one env per lane) reads/writes each field as one coalesced 256-byte (f64) or 128-byte (i32)
// transaction.  Bulk per-env records that are touched by one env at a time (terrain strips, policy state, tuple
// staging) are env-major rows instead.
#pragma once
#include <cstdint>

// Kernel launches and dynamic shared memory are spelled through two macros so that the same sources also compile for the
// test-only SIMT emulator (tests/simt/, -DTRL_SIMT_EMU: g++, one fiber per CUDA thread).  In the product build they expand to
// exactly the CUDA syntax they name.
#ifdef TRL_SIMT_EMU
#define TRL_LAUNCH(kern, grid, block, smem, st, ...) SIMT_LAUNCH(1, kern, grid, block, smem, st, __VA_ARGS__)
#define TRL_LAUNCH_CLUSTER(csize, kern, grid, block, smem, st, ...) SIMT_LAUNCH(csize, kern, grid, block, smem, st, __VA_ARGS__)
#define TRL_DYN_SHARED(type, name) type* name = reinterpret_cast<type*>(simt::dyn_smem())
#else
#define TRL_LAUNCH(kern, grid, block, smem, st, ...) kern<<<grid, block, smem, st>>>(__VA_ARGS__)
#define TRL_LAUNCH_CLUSTER(csize, kern, grid, block, smem, st, ...) kern<<<grid, block, smem, st>>>(__VA_ARGS__)   // cluster size: __cluster_dims__ of the kernel
#define TRL_DYN_SHARED(type, name) extern __shared__ type name[]
#endif

#if defined(__CUDACC__) && !defined(TRL_SIMT_EMU)
#define TRL_HD __host__ __device__
#else
#define TRL_HD
#endif

namespace trl {

constexpr int kMaxJoints = 21;      // dog / goat: 21 joints, raptor: 19
constexpr int kMaxDof = 23;
constexpr int kNumParams = 37;      // max gait controller parameter vector: dog 30 (sim/DogController.h:14-46), raptor 37 (sim/RaptorController.h:14-47)
constexpr int kNumGroundSamples = 200;
constexpr int kTerrainCap = 512;    // floats per terrain segment (20 m nominal + overshoot + 2 m pad at 0.1 m)
constexpr int kTerrainParams = 40;
constexpr int kMaxActions = 16;
constexpr int kMaxCtrlSets = 8;
constexpr int kMaxNetOut = 96;
constexpr int kWarp = 32;
constexpr int kMaxGroups = 8;      // env groups a main step launch can be split into (one stream each)
// envs per group when a main launch is split into n_groups launches: a multiple of 16 envs (= one 128-byte line of an f64 plane)
TRL_HD inline int group_chunk(int n, int n_groups) { return ((n + 16 * n_groups - 1) / (16 * n_groups)) * 16; }
constexpr int kMaxLists = 8;       // pending-decision lists (overlap depth + 1 <= 8)

// ---- f64 SoA planes -------------------------------------------------------------------------------------------
enum DField : int {
    D_Q = 0,                               // 23 generalised positions [x, y, th_root, th_1..]
    D_QD = D_Q + kMaxDof,                  // 23 generalised velocities
    D_TAU = D_QD + kMaxDof,                // 23 held (clamped) joint torques, applied by the next env-step
    D_PARAMS = D_TAU + kMaxDof,            // 30 current action parameters
    D_PD_TARGET = D_PARAMS + kNumParams,   // 21 PD target angles
    D_PHASE = D_PD_TARGET + kMaxJoints,
    D_CUR_CYCLE_T, D_PREV_CYCLE_T, D_CUR_STUMBLE, D_PREV_STUMBLE,
    D_PREV_COM_X, D_PREV_COM_Y, D_PREV_DIST_X, D_PREV_DIST_Y,
    D_FALL_DIST_CNT, D_FALL_CONTACT_CNT, D_SUM_FALL, D_PREV_CHECK_X, D_PREV_CHECK_Y,
    D_AVG_DIST, D_POS_START_X,
    D_SEG_MINX0, D_SEG_MINX1,              // terrain segment origins
    D_NUM_FIELDS
};

// ---- i32 SoA planes -------------------------------------------------------------------------------------------
enum IField : int {
    I_STATE = 0, I_FIRST_CYCLE, I_ACTION_ID, I_CONTACT, I_FAIL_FALL_DIST,
    I_EXP_FLAGS,        // bit0 exp_critic, bit1 exp_actor, bit2 off_policy
    I_CYCLE_COUNT, I_EPISODE_COUNT, I_PENDING, I_CMD,
    I_SEG_N0, I_SEG_N1, I_SEG_FLIP, I_TERRAIN_RNG,   // minstd_rand0 state of the env's terrain generator
    I_TUPLE_FLAGS, I_RNG_CTR_LO, I_RNG_CTR_HI, I_STEPS_LO, I_STEPS_HI,
    I_STANCE,           // raptor: 0 = right leg is the stance leg, 1 = left
    I_NUM_FIELDS,
    // terrain slots (trl_load_terrain): planes past the fields the env-step kernel stages, read and written only where the ground is
    // generated.  reset_env copies the assignment into the current slot before ResetGround
    I_TERRAIN_SLOT = I_NUM_FIELDS,   // slot the env's present terrain was generated from
    I_TERRAIN_SLOT_NEXT,             // slot assigned by the host (trl_set_env_terrain), used from the env's next reset on
    I_NUM_PLANES
};

struct PhysParams {
    double kn, dn, mu, v_eps, contact_tol, k_lim, d_lim;
    int vertex_contacts;      // terrain vertices inside body boxes produce contacts too (opt-in: TRL_VERTEX_CONTACTS=1; DESIGN §3)
};

// Model / scene constants, uploaded once into __constant__ memory (uniform across lanes -> constant-cache broadcast).
struct ModelConst {
    int nj, ndof;
    int parent[kMaxJoints];
    int dof[kMaxJoints];                   // parameter offset of each joint
    double attach_x[kMaxJoints], attach_y[kMaxJoints];
    double lim_lo[kMaxJoints], lim_hi[kMaxJoints];
    int has_limit[kMaxJoints];
    // bodies
    double mass[kMaxJoints], body_ax[kMaxJoints], body_ay[kMaxJoints], body_theta[kMaxJoints];
    double body_cos[kMaxJoints], body_sin[kMaxJoints];
    double half_x[kMaxJoints], half_y[kMaxJoints];
    double izz_o[kMaxJoints];              // planar rotational inertia about the joint origin
    double izz_c[kMaxJoints];              // planar rotational inertia about the body COM
    int collidable[kMaxJoints];
    double total_mass;
    // tree topology helpers for the level-synchronous warp passes
    int depth[kMaxJoints], max_depth;
    int child[kMaxJoints][4];              // up to 4 children per link (-1 = none)
    int anc_pow[kMaxJoints][4];            // 2^k-th ancestor of each link (k = 0..3), -1 if it does not exist
    // chain schedule of the tree recursions (inward sums / eliminations, outward accelerations): the tree is split into chains,
    // maximal runs of single-child links from a leaf or a branch point up to the child of the next branch point.  Lane c walks
    // chain c (chain 0 holds the root); chains of level l only merge chains of lower levels into their bottom link, so a pass is
    // chain_levels steps of at most chain_level_len[l] links each, with one warp barrier per level.
    int n_chains, chain_levels;
    int chain_level_len[kMaxJoints];
    unsigned long long chain_links[kMaxJoints];   // 5 bits per link, bottom link first
    int chain_len[kMaxJoints], chain_level[kMaxJoints];
    int chain_merge[kMaxJoints];           // 5 bits per child chain summed into the bottom link, in summation order (31 = none)
    int chain_up[kMaxJoints];              // parent link of the chain's top link (-1 for the root's chain)
    int n_corners;                         // 4 * number of collidable bodies
    double corner_lx[4 * kMaxJoints], corner_ly[4 * kMaxJoints];   // corner position in the link (joint) frame
    int corner_base[kMaxJoints];           // first corner index of a body (-1 if not collidable)
    double reach;                          // upper bound of |box corner - root joint| over all poses
    unsigned anc_mask_toe, anc_mask_finger;   // links on the chain effector -> root (inclusive)
    unsigned vf_mask_toe, vf_mask_finger;     // links that receive the virtual force (chain up to root / torso, exclusive)
    // PD
    double kp[kMaxJoints], kd[kMaxJoints], torque_lim[kMaxJoints], target_theta0[kMaxJoints], target_vel[kMaxJoints];
    int world_pd[kMaxJoints];
    // gait controller
    int char_type;                         // 1 dog / goat, 2 raptor
    int n_params, n_opt, misc_max, sp_max;  // parameter vector layout (30/29/6/6 dog, 37/28/5/8 raptor)
    int opt_idx[kNumParams];               // indices of the optimised parameters (= actor outputs)
    unsigned stumble_mask, fall_mask;      // parts whose ground contact counts as a stumble / towards a fall
    double exp_noise;                      // exploration noise std (sim/DogControllerMACE.cpp:3-9, RaptorControllerMACE.cpp:7)
    int n_ctrl, n_actions, default_action, grav_comp, virt_forces, is_mace;
    double ctrl_params[kMaxCtrlSets][kNumParams];
    int act_idx0[kMaxActions], act_idx1[kMaxActions], act_cyclic[kMaxActions];
    double act_blend[kMaxActions];
    double target_vel_x;
    // initial state
    double pose0[kMaxDof], vel0[kMaxDof];
    int has_init_x;
    double init_x;
    // terrain
    int terrain_type;
    double terrain_params[kTerrainParams];
    // scenario
    int num_sim_substeps, exp_mode, has_net;
    double gx, gy;
    // net dims
    int n_in, n_char, n_out, n_frags, frag;
    double out_scale_actor0[32];           // OutputScale of actor 0 (exploration noise scale)
    PhysParams phys;
    uint64_t rng_seed;
};

// Terrain slots: slot 0 is the scene's own terrain (ModelConst::terrain_type / terrain_params), slots 1 .. kMaxTerrainSlots - 1 are
// loaded from terrain files; every slot holds its parameter sets blended with the handle's blend.  The table sits in __constant__
// memory beside the model and is uploaded with it.
constexpr int kMaxTerrainSlots = 8;
struct TerrainSlot {
    int type;
    double params[kTerrainParams];
};

// Physics slots: slot 0 is the scene's own PhysParams (ModelConst::phys), slots 1 .. kMaxPhysSlots - 1 are loaded by
// trl_load_physics.  The table sits in __constant__ memory of the physics-slot build beside the model and is uploaded with it; the
// per-env slots ([2][n]: current, assigned) are an allocation of their own, so ModelConst, Buffers and the planes keep their layout.
constexpr int kMaxPhysSlots = 8;
// Broad phase of the env-step: a box corner more than kClearMargin above the terrain maximum under the character is no contact
// candidate.  That holds while contact_tol * sqrt(1 + slope^2) <= kClearMargin for every slope the corner can meet.  The steepest
// slope of the generators with the shipped terrain files and defaults is a 2 m gap wall between two vertices 0.1 m apart, plus the
// slope overlay and bumps: below kMaxSlope.  trl_load_physics refuses a contact tolerance above kClearMargin / sqrt(1 + kMaxSlope^2)
// (0.001998 m; the scenes' own is 0.00025 m).
constexpr double kClearMargin = 0.05;
constexpr double kMaxSlope = 25.0;

// Body slots: slot 0 is the scene's own body (the per-link numbers of ModelConst), slots 1 .. kMaxBodySlots - 1 are loaded from
// character files of the scene's topology and controllers by trl_load_body.  A slot holds every per-link number fill_model reads from a
// character file, and what it derives from them; the topology, masks, corner layout, controller tables and net dimensions stay
// ModelConst's.  The body-slot build of the env-step kernels reads the table from a global-memory mirror (lane-indexed reads) and
// total_mass / reach from a __constant__ copy (warp-uniform reads); the per-env slots ([2][n]: current, assigned) are an allocation of
// their own, so ModelConst, Buffers and the planes keep their layout.
constexpr int kMaxBodySlots = 8;
struct BodyConst {
    double attach_x[kMaxJoints], attach_y[kMaxJoints], lim_lo[kMaxJoints], lim_hi[kMaxJoints];
    int has_limit[kMaxJoints];
    double mass[kMaxJoints], body_ax[kMaxJoints], body_ay[kMaxJoints], body_theta[kMaxJoints], body_cos[kMaxJoints], body_sin[kMaxJoints];
    double half_x[kMaxJoints], half_y[kMaxJoints], izz_o[kMaxJoints], izz_c[kMaxJoints];
    double corner_lx[4 * kMaxJoints], corner_ly[4 * kMaxJoints];
    double kp[kMaxJoints], kd[kMaxJoints], torque_lim[kMaxJoints], target_theta0[kMaxJoints], target_vel[kMaxJoints];
    int world_pd[kMaxJoints];
    double total_mass, reach;
};
// The broad phase of the env-step reads the terrain maximum over [x - reach - 0.25, x + reach + 0.25] around the root joint
// (trl_step.cu: window_max).  That window has to lie inside the ground the env holds: UpdateGround keeps [x - 2, x + 11] generated,
// so the body of a slot may reach at most kMaxReach = 2 - 0.25 m behind the root (the front side has 11 m).  The shipped characters
// reach about 1.1 m (dog, goat) and 1.0 m (raptor); trl_load_body refuses a reach above kMaxReach.
constexpr double kMaxReach = 1.75;

// Ranged slots (trl_load_body_range, trl_load_physics_range): a body or physics slot whose randomizable numbers are drawn again at
// every episode reset of every env on it, each independently and uniformly in [lo, hi]:
//   key = mix64(mix64(mix64(rng_seed ^ tag) + env) + draw)       tag: kBodyDrawTag or kPhysDrawTag; draw: the env's earlier draws of
//                                                                that kind (from 0; carried by checkpoints, not reset by trl_reset)
//   u_i = (mix64(key + i) >> 11) * 2^-53                         body: i = field * nj + link, fields Mass, Kp, Kd, TorqueLim;
//                                                                physics: i = 0..6 in the order of PhysParams
//   v_i = min(hi_i, lo_i + u_i * (hi_i - lo_i))                  every operation rounded on its own (no FMA); lo == hi gives lo
// A body draw then derives izz_o, izz_c per link and total_mass (summed over the links from 0) with fill_model's expressions.  The
// slot's table holds the lo numbers; everything but the drawn fields is the lo file's and equals the hi file's.
constexpr unsigned long long kBodyDrawTag = 0x626f64792d726e67ull;   // "body-rng"
constexpr unsigned long long kPhysDrawTag = 0x706879732d726e67ull;   // "phys-rng"
constexpr int kBodyDrawFields = 4;
// what the body-slot build holds of the ranged slots: their hi tables (the slot tables hold lo), which slots are ranged (bit s), and
// the handle's per-env tables (trl_handle.h; null until its first ranged slot)
struct RangeTables {
    BodyConst body_hi[kMaxBodySlots];
    PhysParams phys_hi[kMaxPhysSlots];
    unsigned body_ranged, phys_ranged;
    BodyConst* env_bdraw;        // [n] the drawn body of every env's present episode on a ranged body slot
    PhysParams* env_pdraw;       // [n] likewise its drawn physics
    long long* env_draws;        // [2][n] every env's draws so far: body, physics
};

// Exploration settings can change between updates (cScenarioExp::SetExpRate/Temp/BaseActionRate).
struct ExpSettings {
    int enable;
    double rate, temp, base_rate, noise;
};

// Policy network weights (device pointers, f64, Caffe blob order).
struct NetWeights {
    const double *conv0_w, *conv0_b, *conv1_w, *conv1_b, *conv2_w, *conv2_b, *tip0_w, *tip0_b, *ip0_w, *ip0_b;
    const double *h0_w[4], *h0_b[4], *h1_w[4], *h1_b[4];
    const double *in_off, *in_scale, *out_off, *out_scale;
};
// Binds the 26 weight blobs (w, b per layer: terr_conv0..2, terr_ip0, ip0, then h0 w, h0 b, h1 w, h1 b of each of the four heads)
// and the input / output offset and scale vectors.  The vectors may be null for a net that is fed normalised inputs.
inline NetWeights net_weights(const double* const* b, const double* in_off, const double* in_scale, const double* out_off,
                              const double* out_scale) {
    NetWeights W;
    W.conv0_w = b[0]; W.conv0_b = b[1]; W.conv1_w = b[2]; W.conv1_b = b[3]; W.conv2_w = b[4]; W.conv2_b = b[5];
    W.tip0_w = b[6]; W.tip0_b = b[7]; W.ip0_w = b[8]; W.ip0_b = b[9];
    for (int k = 0; k < 4; ++k) { W.h0_w[k] = b[10 + 4 * k]; W.h0_b[k] = b[11 + 4 * k]; W.h1_w[k] = b[12 + 4 * k]; W.h1_b[k] = b[13 + 4 * k]; }
    W.in_off = in_off; W.in_scale = in_scale; W.out_off = out_off; W.out_scale = out_scale;
    return W;
}

// Policy slots of an evaluation handle (trl_load_policy): slot 0 is the handle's own net, slots 1 .. kMaxPolicySlots - 1 hold further
// models of the same topology, each env is evaluated by the slot it is assigned to.  Only the slot build of the decision kernels
// (trl_decide2.cuh) reads this; a handle with one policy never allocates it.
constexpr int kMaxPolicySlots = 8;
struct PolicySlots {
    const int* env_slot;     // [n]  slot of each env
    const NetWeights* W;     // [kMaxPolicySlots]  device table of the slots' weights (entries of empty slots are null)
    int* sort_tmp;           // [lag][n]  copy of a pending list while it is regrouped by slot
    int* chunks;             // [lag][1 + 3 * chunk_cap]  {number of chunks, then {slot, row0, rows} per 32-row FC chunk}
    int chunk_cap;           // n / 32 + kMaxPolicySlots: every slot's ragged last chunk included
    const int* env_eval;     // [2][n]  mode of each env's present episode (row 0; 1 evaluates) and next one (trl_set_env_eval), or null
};

// Device buffers of one batch of environments.
struct Buffers {
    int n;                 // number of envs
    double* d;             // [D_NUM_FIELDS][n]
    int* i;                // [I_NUM_PLANES][n]
    float* terrain;        // [n][2][kTerrainCap]
    double* poli_state;    // [n][S]   policy state built at the last decision
    double* net_out;       // [n][kMaxNetOut]
    double* tuple_sbeg;    // [n][S]
    double* tuple_action;  // [n][kNumParams]
    double* com_stash;     // [2][n]   COM at decision time
    int* pending_list;     // [lists][n]  used round robin by successive env-steps (see trl_host.cu: enqueue_update)
    int* pending_count;    // [kMaxLists]
    int* catchup_done;     // [kMaxLists + 1]  [l] CTA completion counter of the catch-up launch of list l (re-arms the list it consumed), [kMaxLists] fault flag
    // outputs
    double* tuples;        // [tuple_cap][1 + S + A + S]
    uint32_t* tuple_flags; // [tuple_cap]
    int* tuple_env;        // [tuple_cap]
    int* tuple_count;      // [1]
    int tuple_cap;
    double* dist_log;      // [dist_cap] episode distances
    int* dist_env;         // [dist_cap]
    int* dist_count;       // [1]
    int dist_cap;
    int S;                 // policy state size
    int A;                 // action record size (1 + number of optimised parameters)
};

}  // namespace trl
