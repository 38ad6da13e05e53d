// deepterrainrl_b200 -- the env-step kernel (sm_90a), warp-per-environment formulation.
//
// One environment per WARP: lane j owns link j of the kinematic tree (21 links) for the kinematics, contacts and integration.
// The tree recursions (composite sums, articulated-body eliminations, outward accelerations) run one lane per CHAIN -- a maximal run
// of single-child links -- through a per-warp, link-indexed block in shared memory: a chain lane eliminates its links one after the
// other in registers, and chains meet only at branch points, one warp barrier per level of the chain tree.  All spatial
// quantities are planar 3-vectors expressed in WORLD axes about the root joint's
// current position O (an inertial frame that instantaneously coincides with the root), which removes every
// per-link coordinate transform from the recursions: motion (w, vOx, vOy), force (nO, fx, fy), joint axis of a
// revolute joint at r (relative to O): S = (1, r_y, -r_x).
//
// One launch = the *controller half* of env-step k followed by the *physics half* of env-step k+1:
//
//   ctrl half  (reference: cSimCharacter::Update -> cDogController::Update, sim/DogController.cpp:229-268)
//     RNEA bias force with the reference's Cj and composite inertias (restates sim/RBDUtil.cpp:4-176 in planar algebra)
//     ApplyFeedback, stable-PD solve (M + h Kd) acc = rhs by the articulated-body recursion (h Kd as joint armature), gravity compensation,
//     virtual forces, torque clamp (sim/Joint.cpp:257-264), fall counters (sim/SimCharSoftFall.cpp:74-125),
//     cycle bookkeeping: reward, tuple record, episode statistics (scenarios/ScenarioExp.cpp:209-243)
//   [end of outer update: fall -> episode reset, scenarios/ScenarioPoliEval.cpp:110-125, ScenarioExp.cpp:83-98]
//   phys half  (reference: cWorld::Update + cGroundVar2D::Update + the head of the controller update)
//     num_sim_substeps x articulated-body forward dynamics with implicit contact / joint-limit terms (this project's
//     own physics model -- Bullet is not restatable, DESIGN.md §3); box corners are evaluated one per lane
//     contact bits, streaming terrain update, cycle timers, gait FSM (sim/DogController.cpp:805-845)
//     warps whose FSM reaches a cycle boundary build the 283-float policy state cooperatively and enqueue a decision
//
// The decision itself (MACE forward pass + action decode) runs in trl_decide.cuh between two launches of this kernel.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>

#include "trl_rcp.cuh"
#include "trl_terrain.cuh"
#include "trl_types.h"
#include "trl_mix64.h"

// The file is compiled twice: as is (namespace trl), and through trl_step_cg.cu with -Xptxas -dlcm=cg (namespace trl_cg), where
// every global load bypasses L1.  The cg build serves the catch-up launches of the overlapped schedule: they read env state the
// decision kernel has just written, while step CTAs running on the same SM may already have pulled the neighbouring envs'
// words of the same 32-byte sectors into that SM's L1.
// Terrain slots (trl_load_terrain) are served by two more builds, trl_step_ts.cu (namespace trl_ts) and trl_step_ts_cg.cu (trl_ts_cg),
// compiled with TRL_TERRAIN_SLOTS_VARIANT: their envs generate their ground from their own slot of c_terrain.  The builds without it
// generate from c_model's terrain, so a handle without terrain slots runs the same kernels as before slots existed.  The emulator
// (tests/simt) compiles only trl_step.cu / trl_step_cg.cu and always with slots, which computes the same for a handle without any.
// Physics slots (trl_load_physics) are served by a third pair, trl_step_ps.cu (namespace trl_ps) and trl_step_ps_cg.cu (trl_ps_cg),
// compiled with TRL_PHYS_SLOTS_VARIANT as well as TRL_TERRAIN_SLOTS_VARIANT: their physics sub-steps read the env's own slot of
// c_phys.  The emulator's "always with slots" includes physics slots; a handle without any has no per-env array and reads slot 0.
// Body slots (trl_load_body) are served by a fourth pair, trl_step_bs.cu (namespace trl_bs) and trl_step_bs_cg.cu (trl_bs_cg), compiled
// with TRL_BODY_SLOTS_VARIANT as well as the terrain- and physics-slot flags: every warp stages the link and box tables of its own
// env's body, and the per-link reads of the controller take the env's slot of g_body.  The emulator includes body slots too.
#if defined(TRL_BODY_SLOTS_VARIANT) && defined(TRL_CG_VARIANT)
#define TRL_IMPL_NS trl_bs_cg
#elif defined(TRL_BODY_SLOTS_VARIANT)
#define TRL_IMPL_NS trl_bs
#elif defined(TRL_PHYS_SLOTS_VARIANT) && defined(TRL_CG_VARIANT)
#define TRL_IMPL_NS trl_ps_cg
#elif defined(TRL_PHYS_SLOTS_VARIANT)
#define TRL_IMPL_NS trl_ps
#elif defined(TRL_TERRAIN_SLOTS_VARIANT) && defined(TRL_CG_VARIANT)
#define TRL_IMPL_NS trl_ts_cg
#elif defined(TRL_TERRAIN_SLOTS_VARIANT)
#define TRL_IMPL_NS trl_ts
#elif defined(TRL_CG_VARIANT)
#define TRL_IMPL_NS trl_cg
#else
#define TRL_IMPL_NS trl
#endif

namespace TRL_IMPL_NS {
using namespace trl;
#if defined(TRL_TERRAIN_SLOTS_VARIANT) || defined(TRL_SIMT_EMU)
constexpr bool kTerrainSlots = true;
#else
constexpr bool kTerrainSlots = false;
#endif

__constant__ ModelConst c_model;
__constant__ TerrainSlot c_terrain[kMaxTerrainSlots];    // slot 0 = c_model's terrain_type / terrain_params (trl_types.h: TerrainSlot)
#if defined(TRL_PHYS_SLOTS_VARIANT) || defined(TRL_SIMT_EMU)
#define TRL_PHYS_TABLE 1
__constant__ PhysParams c_phys[kMaxPhysSlots];   // slot 0 = c_model.phys (trl_types.h: kMaxPhysSlots)
__constant__ int* c_env_phys;                    // [2][n] of the owning handle: the physics slot of every env's present episode, then
                                                 // the slot it gets at its next reset; null while the handle has no physics slot
__constant__ int* c_env_eval;                    // [2][n] likewise the mode (1 evaluates, 0 explores) of the envs of an exploration
                                                 // handle (trl_set_env_eval); null while no env has been given one
// whether the present episode of `env` explores: every env of an exploration handle does, unless it has been set to evaluate
__device__ __forceinline__ bool env_explores(int env) { return c_model.exp_mode && !(c_env_eval && c_env_eval[env]); }
#else
#define TRL_PHYS_TABLE 0
__device__ __forceinline__ bool env_explores(int) { return c_model.exp_mode; }
#endif
// character-type branches: a run-time constant of the scene (the raptor's controller differs from the dog's / goat's); an experiment
// build can fix it at compile time (-DTRL_FIXED_CHAR=0 dog / goat, 2 raptor) to see what the unused branches cost
#ifdef TRL_FIXED_CHAR
#define TRL_IS_RAPTOR(mc) (TRL_FIXED_CHAR == 2)
#else
#define TRL_IS_RAPTOR(mc) ((mc).char_type == 2)
#endif
// Lane-indexed tables (one entry per link / corner) are read from a global-memory mirror of the same struct: the constant cache
// serves one address per access, so `c_model.kp[lane]` costs one replay per distinct lane, while the mirror is one coalesced,
// L1-cached read-only load.  Warp-uniform reads stay in constant memory.
#ifndef TRL_TABLE_MIRROR
#define TRL_TABLE_MIRROR 1      // 0 = the round-1 reads from constant memory
#endif
#if TRL_TABLE_MIRROR
__device__ ModelConst g_model;
#define LT(field, idx) __ldg(&g_model.field[(idx)])
#define LT2(field, i, j) __ldg(&g_model.field[(i)][(j)])
#else
#define LT(field, idx) c_model.field[(idx)]
#define LT2(field, i, j) c_model.field[(i)][(j)]
#endif
#ifndef TRL_LINK_SMEM
#define TRL_LINK_SMEM 1     // 1: the per-lane link constants live in shared memory (one table per CTA) instead of ~28 registers per thread
                            //    (the register build spills them and reloads them inside the ABA rounds)
#endif
// Body slots: the per-link numbers of the env's body.  `bb` (the env's body: its slot's entry of g_body, or on a ranged slot its own
// drawn entry of c_env_bdraw; warp-uniform, one env per warp) must be in scope.  BL: lane-indexed reads; BU: warp-uniform reads of a
// per-link number; BM: total_mass / reach.  They are coherent loads: a reset rewrites the drawn entry inside the launch that reads it.
// The other builds read the scene's body from the model, as before slots.  The body build needs the link tables in shared memory
// (restaged per warp when its env changes body); the emulator's TRL_LINK_SMEM=0 experiment build runs without body slots.
#if (defined(TRL_BODY_SLOTS_VARIANT) || defined(TRL_SIMT_EMU)) && TRL_LINK_SMEM
#define TRL_BODY_TABLE 1
__device__ BodyConst g_body[kMaxBodySlots];      // slot 0 = the scene's body; a ranged slot holds its lo numbers (trl_types.h: BodyConst)
__device__ BodyConst g_body_hi[kMaxBodySlots];   // a ranged slot's hi numbers
__constant__ int* c_env_body;                    // [2][n] of the owning handle: the body slot of every env's present episode, then the slot
                                                 // it gets at its next reset; null while the handle has no body slot
// Ranged slots (trl_types.h: kBodyDrawTag): bit s of c_body_ranged / c_phys_ranged marks body / physics slot s as ranged.  The
// per-env tables exist from the handle's first ranged slot on (null before): the drawn body and physics of every env's present
// episode on a ranged slot, and every env's count of draws of either kind ([2][n]: body, physics)
__constant__ unsigned c_body_ranged, c_phys_ranged;
__constant__ PhysParams c_phys_hi[kMaxPhysSlots];
__constant__ BodyConst* c_env_bdraw;
__constant__ PhysParams* c_env_pdraw;
__constant__ long long* c_env_draws;
#define BL(field, idx) bb->field[(idx)]
#define BU(field, idx) BL(field, idx)
#define BM(field) bb->field
#define TRL_BS_DECL , const BodyConst* bb
#define TRL_BS_ARG , bb
#else
#if defined(TRL_BODY_SLOTS_VARIANT)
#error "the body-slot build stages its link tables in shared memory (TRL_LINK_SMEM=1)"
#endif
#define TRL_BODY_TABLE 0
#define BL(field, idx) LT(field, idx)
#define BU(field, idx) c_model.field[(idx)]
#define BM(field) c_model.field
#define TRL_BS_DECL
#define TRL_BS_ARG
#endif

#ifndef TRL_WARPS_PER_BLOCK
#define TRL_WARPS_PER_BLOCK 4
#endif
constexpr int kWarpsPerBlock = TRL_WARPS_PER_BLOCK;   // one env per warp; 16 resident warps per SM at 128 registers whatever the CTA size
constexpr int kBlockThreads = kWarpsPerBlock * kWarp;
constexpr unsigned kFull = 0xffffffffu;
#ifndef TRL_STEP_MIN_BLOCKS
#define TRL_STEP_MIN_BLOCKS 4   // CTAs of 4 warps per SM the register budget is sized for
#endif
constexpr int kStepSkipPending = 8, kStepCatchUp = 16;   // flag bits of trl_step_kernel beyond ctrl (1) / phys (2) / end (4)
// `lists` packs: bits 0-2 the list new boundary envs are appended to, bits 3-5 the list a catch-up launch serves, bits 6-9 the number
// of env-steps a catch-up launch advances its envs by
constexpr int kZeroLane = 31;   // always idle (nj <= 23): its per-link registers are zero, used as the "no source" lane
// per-warp shared scratch (doubles; every block starts 16-byte aligned)
// Link block: one slot per link, written by the link lanes and walked by the chain lanes (chain_inward / chain_outward).  A slot is
// 9 double2, an odd number of 16-byte units, so the 128-bit accesses of 8 lanes to 8 different links fall in distinct banks.
constexpr int kLinkStride = 18;
enum {
    LK_IA = 0,     // [0, 9): articulated inertia (a, bx, by, cxx, cxy, cyy) + bias force (n, fx, fy) of the link alone; composite sums
    LK_TAU = 9,    // joint force of the elimination
    LK_CV = 10,    // (cvx, cvy): velocity-product acceleration c_j
    LK_S = 12,     // (s1, s2): joint axis S_j = (1, s1, s2)
    LK_LIM = 14,   // (lim_f, cl): implicit joint term, u_j -= lim_f, D_j += dt * cl
    // written by the elimination over [0, 5) and by the outward pass
    LK_U = 0, LK_DINV = 3, LK_UU = 4, LK_QDD = 5, LK_ACC = 6 /* (aw, ax, ay) */
};
constexpr int kChainStride = 10;                            // per chain: the 9 values its top link hands to its parent link
constexpr int X_LNK = 0;
constexpr int X_CHO = X_LNK + kMaxJoints * kLinkStride;
constexpr int X_CHO_END = X_CHO + kMaxJoints * kChainStride;
// Experiments (shuffles are a large share of the kernel's instructions).  Each knob moves one
// family of lane-to-lane exchanges from warp shuffles (2 SHFL + register moves per double) to per-warp shared memory (128-bit
// stores / loads); values and operation order are untouched, so every variant is bit-identical to the default build
// (tests/test_simt_cpu.py checks that on the CPU emulator).  Default build: all off.  -DTRL_SMEM_XCHG=1: all on.
// TRL_ACCUM_SMEM and TRL_LDLT_SMEM name exchanges the chain passes removed (the round-by-round child -> parent hand-off, the
// LDL^T pivot column), TRL_CONTACT_SMEM the corner -> body-lane exchanges the per-body contact pass removed; they are accepted and
// change nothing.
#ifndef TRL_SMEM_XCHG
#define TRL_SMEM_XCHG 0
#endif
#ifndef TRL_KIN_SMEM
#define TRL_KIN_SMEM TRL_SMEM_XCHG       // pointer-jumping prefix sums of the kinematics (26 doubles x 6 per env-step)
#endif
#ifndef TRL_OUTWARD_SMEM
#define TRL_OUTWARD_SMEM TRL_SMEM_XCHG   // floating-base broadcast of the root's articulated inertia (9 doubles x 6 per env-step)
#endif
#if TRL_KIN_SMEM
constexpr int X_PFX = (X_CHO_END + 1) & ~1;                 // three buffers of 32 double2: prefix rounds alternate 0 / 1, buffer 2 = (cos, sin) exchange
constexpr int X_PFX_END = X_PFX + 3 * 2 * kWarp;
#else
constexpr int X_PFX_END = X_CHO_END;
#endif
#if TRL_OUTWARD_SMEM
constexpr int X_BASE = (X_PFX_END + 1) & ~1;                // the 9 floating-base values of lane 0
constexpr int X_OUT_END = X_BASE + 10;
#else
constexpr int X_OUT_END = X_PFX_END;
#endif
constexpr int X_END = (X_OUT_END + 1) & ~1;
// Measurement build (-DTRL_PHASE_CLOCKS=1, TRL_VARIANT=phase_clocks): lane 0 of every warp adds the clock64() delta of each
// phase of the launch to g_phase_clocks[phase]; slot kNumPhases counts the physics halves (env-steps).  Read out by
// trl_debug_step_phases (trl_probe.cu), printed by tools/step_phase_probe.py.  The product build compiles none of it.
#ifndef TRL_PHASE_CLOCKS
#define TRL_PHASE_CLOCKS 0
#endif
enum StepPhase { PH_LOAD, PH_RNEA, PH_SOLVE, PH_CTRL_REST, PH_KIN, PH_CONTACT, PH_INWARD, PH_OUTWARD, PH_TAIL, kNumPhases };
#if TRL_PHASE_CLOCKS
__device__ unsigned long long g_phase_clocks[kNumPhases + 1];
#define TRL_CLK_DECL(a, b) , int a, int b      // phases a helper's parts are counted under
#define TRL_CLK_ARG(a, b) , a, b
#define TRL_CLK_BEGIN(t) long long t = clock64()
#define TRL_CLK_RESET(t) (t) = clock64()
#define TRL_CLK_END(p, t)                                                                                              \
    do {                                                                                                               \
        const long long n_ = clock64();                                                                                \
        if ((threadIdx.x & 31) == 0) atomicAdd(&g_phase_clocks[(p)], (unsigned long long)(n_ - (t)));                  \
        (t) = n_;                                                                                                      \
    } while (0)
#else
#define TRL_CLK_DECL(a, b)
#define TRL_CLK_ARG(a, b)
#define TRL_CLK_BEGIN(t)
#define TRL_CLK_RESET(t)
#define TRL_CLK_END(p, t)
#endif
// the scratch pointer is only threaded through the helpers that need it, so the default build's code is untouched
#if TRL_KIN_SMEM
#define TRL_KIN_XS_DECL , double* xs, int lane
#define TRL_KIN_XS_ARG , xs, lane
#define TRL_RESET_XS_DECL , double* xs
#define TRL_RESET_XS_ARG , xs
#else
#define TRL_KIN_XS_DECL
#define TRL_KIN_XS_ARG
#define TRL_RESET_XS_DECL
#define TRL_RESET_XS_ARG
#endif
#ifndef TRL_REUSE_KIN
#define TRL_REUSE_KIN 0    // 1 (experiment): the first physics sub-step of a launch reuses the kinematics the controller half of the same
#endif                     // launch computed for the same state (one of six kinematics() per env-step); same inputs, bit-identical
#if TRL_REUSE_KIN
#define TRL_REUSE_KIN_DECL , const Kin* k0
#else
#define TRL_REUSE_KIN_DECL
#endif
// the physics slot of the env a sub-step serves (physics-slot builds only: the other builds keep the parent's signature); the body build
// hands it the env's physics itself, staged per warp (a ranged slot's envs each have their own)
#if TRL_BODY_TABLE
#define TRL_PS_DECL , const PhysParams& pp
#define TRL_PS_ARG , s_pp_w[warp]
#elif TRL_PHYS_TABLE
#define TRL_PS_DECL , int ps
#define TRL_PS_ARG , ps
#else
#define TRL_PS_DECL
#define TRL_PS_ARG
#endif

// 128-bit shared-memory accesses of the experiment builds need 16-byte aligned addresses (a misaligned one faults on the GPU);
// the emulator build checks every such cast, the CUDA build compiles to the plain cast
#ifdef TRL_SIMT_EMU
template <typename T2, typename T>
inline T2* trl_as2(T* p) {
    if (reinterpret_cast<uintptr_t>(p) & 15u) { std::fprintf(stderr, "simt: misaligned 128-bit shared-memory access\n"); std::abort(); }
    return reinterpret_cast<T2*>(p);
}
#else
template <typename T2, typename T>
__device__ __forceinline__ T2* trl_as2(T* p) { return reinterpret_cast<T2*>(p); }
#endif

__device__ __forceinline__ int tri(int a, int b) { return a * (a + 1) / 2 + b; }  // a >= b
__device__ __forceinline__ double shf(double v, int src) { return __shfl_sync(kFull, v, src); }
__device__ __forceinline__ int shfi(int v, int src) { return __shfl_sync(kFull, v, src); }
__device__ __forceinline__ double warp_sum_all(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(kFull, v, o);
    return v;
}

__device__ __forceinline__ double wrap_pi(double a) {
    double s, c;
    sincos(a, &s, &c);
    double th = acos(fmin(1.0, fmax(-1.0, c)));
    return (s >= 0) ? th : -th;
}

// dog / goat joint indices (sim/SimDog.h:11-36)
enum DogJoint {
    jRoot, jSpine0, jSpine1, jSpine2, jSpine3, jTorso, jNeck0, jNeck1, jHead, jTail0, jTail1, jTail2, jTail3,
    jShoulder, jElbow, jWrist, jFinger, jHip, jKnee, jAnkle, jToe
};
// raptor joint indices (sim/SimRaptor.h:11-33) and controller layout (sim/RaptorController.h:14-47)
enum RaptorJoint {
    rRoot, rSpine0, rSpine1, rSpine2, rSpine3, rHead, rTail0, rTail1, rTail2, rTail3, rTail4,
    rRightHip, rRightKnee, rRightAnkle, rRightToe, rLeftHip, rLeftKnee, rLeftAnkle, rLeftToe
};
enum { rsContact, rsDown, rsPassing, rsUp };
enum { rmTransTime, rmCv, rmCd, rmForceX, rmForceY };
enum { rpRootPitch, rpSpineCurve, rpStanceHip, rpStanceKnee, rpStanceAnkle, rpSwingHip, rpSwingKnee, rpSwingAnkle };
enum { sBackStance, sExtend, sFrontStance, sGather };
enum { mTransTime, mCv, mBackForceX, mBackForceY, mFrontForceX, mFrontForceY, mMiscMax };
enum { spSpineCurve, spShoulder, spElbow, spHip, spKnee, spAnkle, spMax };

// ------------------------------------------------------------------------------------------------ counter RNG
struct CounterRng {
    uint64_t key, ctr;
    __device__ static uint64_t mix(uint64_t z) {
        z += 0x9E3779B97F4A7C15ull;
        z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
        z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
        return z ^ (z >> 31);
    }
    __device__ void init(uint64_t seed, uint64_t stream, uint64_t c) { key = mix(seed ^ mix(stream)); ctr = c; }
    __device__ uint64_t next() { return mix(key + (ctr++) * 0xD1342543DE82EF95ull); }
    __device__ double uniform() { return (double)(next() >> 11) * (1.0 / 9007199254740992.0); }
    __device__ int rand_int(int mn, int mx) {
        if (mn == mx) return mn;
        int r = (int)(next() >> 33);
        return mn + r % (mx - mn);
    }
    __device__ bool flip_coin() { return uniform() < 0.5; }
    __device__ double normal() {
        double u1 = 1.0 - uniform(), u2 = uniform();
        return sqrt(-2.0 * log(u1)) * cos(6.283185307179586476925 * u2);
    }
};

// ------------------------------------------------------------------------------------------------ global accessors
#ifndef TRL_FIELD_SMEM
#define TRL_FIELD_SMEM 0    // 1: the step kernel stages every per-env field of its env in shared memory (one batch of independent loads at
#endif                      //    the start, one batch of stores at the end) instead of ~50 dependent L2 round trips spread over the launch
struct Lane {
    double* sm;          // unused by the warp kernel (kept for the decision kernel's scalar helpers)
    int env, n;
    double* D;
    int* I;
#if TRL_FIELD_SMEM
    double* sd;          // staged copy of the env's f64 fields [D_NUM_FIELDS] (null: read / write the planes directly)
    int* si;             // staged copy of the env's i32 fields [I_NUM_FIELDS]
    __device__ __forceinline__ double& d(int f) { return sd ? sd[f] : D[(size_t)f * n + env]; }
    __device__ __forceinline__ int& i(int f) { return si ? si[f] : I[(size_t)f * n + env]; }
#else
    __device__ __forceinline__ double& d(int f) { return D[(size_t)f * n + env]; }
    __device__ __forceinline__ int& i(int f) { return I[(size_t)f * n + env]; }
#endif
};

__device__ __forceinline__ bool has_fallen(Lane& L, double root_theta) {
    return L.d(D_SUM_FALL) > 0.25 || L.i(I_FAIL_FALL_DIST) != 0 || fabs(wrap_pi(root_theta)) > 3.14159265358979323846 * 0.8;
}

// cDogController::SetStateParams (sim/DogController.cpp:1042-1054) / cRaptorController::SetStateParams
// (sim/RaptorController.cpp:1108-1125) for the given state
__device__ void set_state_params(Lane& L, int state) {
    const ModelConst& m = c_model;
    int base = D_PARAMS + m.misc_max + state * m.sp_max;
    if (TRL_IS_RAPTOR(m)) {
        const int st = L.i(I_STANCE) == 0 ? rRightHip : rLeftHip, sw = L.i(I_STANCE) == 0 ? rLeftHip : rRightHip;
        L.d(D_PD_TARGET + st) = L.d(base + rpStanceHip); L.d(D_PD_TARGET + st + 1) = L.d(base + rpStanceKnee);
        L.d(D_PD_TARGET + st + 2) = L.d(base + rpStanceAnkle);
        L.d(D_PD_TARGET + sw) = L.d(base + rpSwingHip); L.d(D_PD_TARGET + sw + 1) = L.d(base + rpSwingKnee);
        L.d(D_PD_TARGET + sw + 2) = L.d(base + rpSwingAnkle);
        return;
    }
    double sc = L.d(base + spSpineCurve);
    L.d(D_PD_TARGET + jSpine0) = sc; L.d(D_PD_TARGET + jSpine1) = sc; L.d(D_PD_TARGET + jSpine2) = sc;
    L.d(D_PD_TARGET + jSpine3) = sc; L.d(D_PD_TARGET + jTorso) = sc;
    L.d(D_PD_TARGET + jShoulder) = L.d(base + spShoulder);
    L.d(D_PD_TARGET + jElbow) = L.d(base + spElbow);
    L.d(D_PD_TARGET + jHip) = L.d(base + spHip);
    L.d(D_PD_TARGET + jKnee) = L.d(base + spKnee);
    L.d(D_PD_TARGET + jAnkle) = L.d(base + spAnkle);
}

// cDogController::CalcReward (sim/DogController.cpp:594-623)
__device__ double calc_reward(Lane& L, bool fallen) {
    double vel_r = 0.0, stum_r = 0.0;
    if (!fallen) {
        double ct = L.d(D_PREV_CYCLE_T);
        double avg_vel = L.d(D_PREV_DIST_X) / ct;
        double err = c_model.target_vel_x - avg_vel;
        vel_r = exp(-0.5 * err * err);
        double avg_st = L.d(D_PREV_STUMBLE) / ct;
        stum_r = 1.0 / (1.0 + 10.0 * avg_st);
        if (TRL_IS_RAPTOR(c_model) && avg_vel < 0.0) { vel_r = 0.0; stum_r = 0.0; }   // sim/RaptorController.cpp:583-587
    }
    return 0.8 * vel_r + 0.2 * stum_r;
}

// cScenarioExp::NewCycleUpdate (scenarios/ScenarioExp.cpp:209-243): finish the previous tuple, start the next.
// Cooperative: the row copies are spread over the warp, the scalar bookkeeping is done by lane 0.
__device__ void exp_new_cycle_update(Lane& L, const Buffers& B, bool fallen, int lane) {
    const int S = B.S, A = B.A;
    const double* s_end = B.poli_state + (size_t)L.env * S;
    double* s_beg = B.tuple_sbeg + (size_t)L.env * S;
    double* act = B.tuple_action + (size_t)L.env * kNumParams;
    int slot = -1;
    if (lane == 0 && L.i(I_CYCLE_COUNT) > 1) slot = atomicAdd(B.tuple_count, 1);
    slot = shfi(slot, 0);
    if (slot >= 0 && slot < B.tuple_cap) {
        double* row = B.tuples + (size_t)slot * (1 + S + A + S);
        for (int k = lane; k < S; k += kWarp) { row[1 + k] = s_beg[k]; row[1 + S + A + k] = s_end[k]; }
        for (int k = lane; k < A; k += kWarp) row[1 + S + k] = act[k];
        if (lane == 0) {
            unsigned flags = (unsigned)L.i(I_TUPLE_FLAGS);
            flags = fallen ? (flags | 1u) : (flags & ~1u);
            row[0] = calc_reward(L, fallen);
            B.tuple_flags[slot] = flags;
            B.tuple_env[slot] = L.env;
        }
    }
    __syncwarp();
    for (int k = lane; k < S; k += kWarp) s_beg[k] = s_end[k];
    for (int k = lane; k < A; k += kWarp) act[k] = (k == 0) ? (double)L.i(I_ACTION_ID) : L.d(D_PARAMS + c_model.opt_idx[k - 1]);
    if (lane == 0) {
        int ef = L.i(I_EXP_FLAGS);
        unsigned nf = 0;
        if (ef & 1) nf |= 2u;   // exp critic -> eFlagExpCritic (bit 1)
        if (ef & 2) nf |= 4u;   // exp actor  -> eFlagExpActor  (bit 2)
        L.i(I_TUPLE_FLAGS) = (int)nf;
        L.i(I_CYCLE_COUNT) += 1;
    }
    __syncwarp();
}

// cDogController::BlendCtrlParams / BuildBaseAction (+ cDogControllerMACE::AssignFragID); writes params, returns id
__device__ int build_base_action(Lane& L, CounterRng& rng, int a, double* params /*local[30]*/) {
    const ModelConst& m = c_model;
    int i0 = m.act_idx0[a], i1 = m.act_idx1[a];
    double blend = m.act_blend[a];
    for (int k = 0; k < m.n_params; ++k) {
        double p0 = m.ctrl_params[i0][k], p1 = m.ctrl_params[i1][k];
        if (k == mTransTime || k == mCv || (TRL_IS_RAPTOR(m) && k == rmCd)) { p0 = fabs(p0); p1 = fabs(p1); }
        params[k] = (1.0 - blend) * p0 + blend * p1;
    }
    int id = a;
    if (m.is_mace) {
        int nf = m.has_net ? m.n_frags : 0, frag = 0;
        if (nf > 0) {
            if (i0 >= nf && i1 >= nf) frag = rng.rand_int(0, nf);
            else if (i0 >= nf) frag = i1;
            else if (i1 >= nf) frag = i0;
            else {
                frag = rng.flip_coin() ? i0 : i1;
                int ncp = m.n_ctrl, copies = nf / ncp, rem = nf % ncp;
                if (frag < rem) ++copies;
                frag += rng.rand_int(0, copies) * ncp;
            }
        }
        id = frag;
    }
    return id;
}

// cTerrainRLCharController::ApplyAction + cDogController::{NewCycleUpdate, ApplyAction}: commit an action
__device__ void apply_action(Lane& L, int id, const double* params, double comx, double comy) {
    for (int k = 0; k < c_model.n_params; ++k) L.d(D_PARAMS + k) = params[k];
    L.d(D_PARAMS + mTransTime) = fabs(params[mTransTime]);
    L.d(D_PARAMS + mCv) = fabs(params[mCv]);
    if (TRL_IS_RAPTOR(c_model)) L.d(D_PARAMS + rmCd) = fabs(params[rmCd]);
    L.i(I_ACTION_ID) = id;
    L.d(D_PREV_CYCLE_T) = L.d(D_CUR_CYCLE_T); L.d(D_CUR_CYCLE_T) = 0.0;
    L.d(D_PREV_STUMBLE) = L.d(D_CUR_STUMBLE); L.d(D_CUR_STUMBLE) = 0.0;
    L.d(D_PREV_DIST_X) = comx - L.d(D_PREV_COM_X); L.d(D_PREV_DIST_Y) = comy - L.d(D_PREV_COM_Y);
    L.d(D_PREV_COM_X) = comx; L.d(D_PREV_COM_Y) = comy;
    L.i(I_STATE) = sBackStance;
    L.d(D_PHASE) = 0.0;
    set_state_params(L, sBackStance);
}

__device__ GroundView load_ground(Lane& L, const Buffers& B) {
    GroundView g;
    g.data = B.terrain + (size_t)L.env * 2 * kTerrainCap;
    g.n[0] = L.i(I_SEG_N0); g.n[1] = L.i(I_SEG_N1);
    g.min_x[0] = L.d(D_SEG_MINX0); g.min_x[1] = L.d(D_SEG_MINX1);
    g.flip = L.i(I_SEG_FLIP);
    g.rng_state = (uint32_t)L.i(I_TERRAIN_RNG);
    return g;
}
__device__ void store_ground(Lane& L, const GroundView& g) {
    L.i(I_SEG_N0) = g.n[0]; L.i(I_SEG_N1) = g.n[1];
    L.d(D_SEG_MINX0) = g.min_x[0]; L.d(D_SEG_MINX1) = g.min_x[1];
    L.i(I_SEG_FLIP) = g.flip;
    L.i(I_TERRAIN_RNG) = (int)g.rng_state;
}

// the terrain slot the env's present ground comes from; I_TERRAIN_SLOT is not a staged field, so this reads the plane itself
__device__ __forceinline__ const TerrainSlot& env_terrain(const Lane& L) { return c_terrain[L.I[(size_t)I_TERRAIN_SLOT * L.n + L.env]]; }

__device__ CounterRng load_rng(Lane& L) {
    CounterRng r;
    uint64_t c = ((uint64_t)(uint32_t)L.i(I_RNG_CTR_HI) << 32) | (uint32_t)L.i(I_RNG_CTR_LO);
    r.init(c_model.rng_seed, (uint64_t)L.env, c);
    return r;
}
__device__ void store_rng(Lane& L, const CounterRng& r) {
    L.i(I_RNG_CTR_LO) = (int)(uint32_t)(r.ctr & 0xffffffffull);
    L.i(I_RNG_CTR_HI) = (int)(uint32_t)(r.ctr >> 32);
}

// ================================================================================================ warp context
// Per-lane constants of link `lane` and the env state held in registers (TRL_LINK_SMEM: above).
#if TRL_LINK_SMEM
enum { LF_AX, LF_AY, LF_MASS, LF_BAX, LF_BAY, LF_IZZ, LF_LIM_LO, LF_LIM_HI, LF_NUM };
enum { LI_PARENT, LI_DEPTH, LI_ANC1, LI_ANC2, LI_ANC4, LI_ANC8, LI_CH_LEN, LI_CH_LEVEL, LI_CH_MERGE, LI_CH_UP, LI_NUM };
// a field of the table as a value: every read is one conflict-free LDS (tables are [field][lane])
template <int F> struct LkD { const double* p; __device__ __forceinline__ operator double() const { return p[F * kWarp]; } };
template <int F> struct LkI { const int* p; __device__ __forceinline__ operator int() const { return p[F * kWarp]; } };
struct LkU { const unsigned long long* p; __device__ __forceinline__ operator unsigned long long() const { return *p; } };
struct LinkTables {
    double d[LF_NUM * kWarp];
    unsigned long long u[kWarp];
    int i[LI_NUM * kWarp];
};
struct LinkC {
    int act;            // lane < nj
    LkI<LI_PARENT> parent; LkI<LI_DEPTH> depth;
    LkU ch_links; LkI<LI_CH_LEN> ch_len; LkI<LI_CH_LEVEL> ch_level; LkI<LI_CH_MERGE> ch_merge; LkI<LI_CH_UP> ch_up;
    LkI<LI_ANC1> anc1; LkI<LI_ANC2> anc2; LkI<LI_ANC4> anc4; LkI<LI_ANC8> anc8;
    LkD<LF_AX> ax; LkD<LF_AY> ay;
    LkD<LF_MASS> mass; LkD<LF_BAX> bax; LkD<LF_BAY> bay; LkD<LF_IZZ> izz_c;
    LkD<LF_LIM_LO> lim_lo; LkD<LF_LIM_HI> lim_hi;
};
#define TRL_LINK_TABLES_DECL __shared__ LinkTables s_link; LinkTables* const link_tabs = &s_link;
#else
struct LinkTables;
struct LinkC {
    int act;            // lane < nj
    int parent, depth;
    unsigned long long ch_links;  // chain `lane` of the schedule (ModelConst::chain_*; level -1: no chain)
    int ch_len, ch_level, ch_merge, ch_up;
    int anc1, anc2, anc4, anc8;   // 2^k-th ancestors (31 = none: the idle zero lane) for the pointer-jumping prefix sums
    double ax, ay;      // attach point in the parent's joint frame
    double mass, bax, bay, izz_c;
    double lim_lo, lim_hi;
};
#define TRL_LINK_TABLES_DECL LinkTables* const link_tabs = nullptr;
#endif
struct Kin {            // world-axes kinematics of link `lane` about O (the root joint position)
    double phi, cw, sw, rx, ry, w, vx, vy;   // joint frame rotation, joint origin, spatial velocity (w, vO)
    double cx, cy;                           // body COM
};
struct EnvRegs {
    double q, qd;            // lane j: joint angle / rate of link j (lane 0: root angle)
    double ox, oy, oxd, oyd; // root translation and its rate (same value in every lane)
    double tau;              // held joint torque of link j
};

// the link constants of lane `lane` as plain values (constant memory -> registers)
struct LinkVals {
    int act, parent, depth, anc1, anc2, anc4, anc8, ch_len, ch_level, ch_merge, ch_up;
    unsigned long long ch_links;
    double ax, ay, mass, bax, bay, izz_c, lim_lo, lim_hi;
};
__device__ __forceinline__ LinkVals link_values(int lane TRL_BS_DECL) {
    const ModelConst& m = c_model;
    LinkVals c;
    c.act = lane < m.nj;
    int j = c.act ? lane : 0;
    c.parent = (c.act && j > 0) ? LT(parent, j) : 0;
    c.depth = c.act ? LT(depth, j) : -1;
    const bool has_chain = lane < m.n_chains;
    const int ci = has_chain ? lane : 0;
    c.ch_links = has_chain ? LT(chain_links, ci) : 0ull;
    c.ch_len = has_chain ? LT(chain_len, ci) : 0;
    c.ch_level = has_chain ? LT(chain_level, ci) : -1;
    c.ch_merge = has_chain ? LT(chain_merge, ci) : ~0;
    c.ch_up = has_chain ? LT(chain_up, ci) : -1;
    c.anc1 = c.act ? LT2(anc_pow, j, 0) : -1; c.anc2 = c.act ? LT2(anc_pow, j, 1) : -1;
    c.anc4 = c.act ? LT2(anc_pow, j, 2) : -1; c.anc8 = c.act ? LT2(anc_pow, j, 3) : -1;
    if (c.anc1 < 0) c.anc1 = kZeroLane;
    if (c.anc2 < 0) c.anc2 = kZeroLane;
    if (c.anc4 < 0) c.anc4 = kZeroLane;
    if (c.anc8 < 0) c.anc8 = kZeroLane;
    c.ax = BL(attach_x, j); c.ay = BL(attach_y, j);
    c.mass = c.act ? BL(mass, j) : 0.0;
    c.bax = BL(body_ax, j); c.bay = BL(body_ay, j);
    c.izz_c = c.act ? BL(izz_c, j) : 0.0;
    const int has_lim = c.act ? BL(has_limit, j) : 0;
    c.lim_lo = has_lim ? BL(lim_lo, j) : -INFINITY;    // no limit: never violated, so the limit force needs no branch
    c.lim_hi = has_lim ? BL(lim_hi, j) : INFINITY;
    return c;
}
// TRL_LINK_SMEM: the first warp of the CTA fills the table (the caller's __syncthreads() publishes it); in the body build every warp
// fills its own table with the links of body slot bs (the caller's __syncwarp() publishes it)
__device__ __forceinline__ void stage_link_tables(LinkTables* t TRL_BS_DECL) {
#if TRL_LINK_SMEM
#if TRL_BODY_TABLE
    {
        const int lane = threadIdx.x & 31;
        const LinkVals v = link_values(lane, bb);
#else
    if (threadIdx.x < kWarp) {
        const int lane = threadIdx.x;
        const LinkVals v = link_values(lane);
#endif
        t->d[LF_AX * kWarp + lane] = v.ax; t->d[LF_AY * kWarp + lane] = v.ay; t->d[LF_MASS * kWarp + lane] = v.mass;
        t->d[LF_BAX * kWarp + lane] = v.bax; t->d[LF_BAY * kWarp + lane] = v.bay; t->d[LF_IZZ * kWarp + lane] = v.izz_c;
        t->d[LF_LIM_LO * kWarp + lane] = v.lim_lo; t->d[LF_LIM_HI * kWarp + lane] = v.lim_hi;
        t->u[lane] = v.ch_links;
        t->i[LI_PARENT * kWarp + lane] = v.parent; t->i[LI_DEPTH * kWarp + lane] = v.depth;
        t->i[LI_CH_LEN * kWarp + lane] = v.ch_len; t->i[LI_CH_LEVEL * kWarp + lane] = v.ch_level;
        t->i[LI_CH_MERGE * kWarp + lane] = v.ch_merge; t->i[LI_CH_UP * kWarp + lane] = v.ch_up;
        t->i[LI_ANC1 * kWarp + lane] = v.anc1; t->i[LI_ANC2 * kWarp + lane] = v.anc2; t->i[LI_ANC4 * kWarp + lane] = v.anc4;
        t->i[LI_ANC8 * kWarp + lane] = v.anc8;
    }
#else
    (void)t;
#endif
}
__device__ __forceinline__ LinkC load_link(int lane, const LinkTables* t) {
    LinkC c;
#if TRL_LINK_SMEM
    c.act = lane < c_model.nj;
    const double* d = t->d + lane;
    const int* i = t->i + lane;
    c.parent.p = i; c.depth.p = i; c.anc1.p = i; c.anc2.p = i; c.anc4.p = i; c.anc8.p = i;
    c.ch_len.p = i; c.ch_level.p = i; c.ch_merge.p = i; c.ch_up.p = i;
    c.ch_links.p = t->u + lane;
    c.ax.p = d; c.ay.p = d; c.mass.p = d; c.bax.p = d; c.bay.p = d; c.izz_c.p = d; c.lim_lo.p = d; c.lim_hi.p = d;
#else
    (void)t;
    const LinkVals v = link_values(lane);
    c.act = v.act; c.parent = v.parent; c.depth = v.depth;
    c.ch_links = v.ch_links; c.ch_len = v.ch_len; c.ch_level = v.ch_level; c.ch_merge = v.ch_merge; c.ch_up = v.ch_up;
    c.anc1 = v.anc1; c.anc2 = v.anc2; c.anc4 = v.anc4; c.anc8 = v.anc8;
    c.ax = v.ax; c.ay = v.ay; c.mass = v.mass; c.bax = v.bax; c.bay = v.bay; c.izz_c = v.izz_c; c.lim_lo = v.lim_lo; c.lim_hi = v.lim_hi;
#endif
    return c;
}
#if TRL_BODY_TABLE
// The warp's own tables for body bb: the link table, and (s_clx non-null) the corner tables with the six per-body box tables behind
// them (the layout the other builds stage once per CTA in trl_step_kernel).  The leading barrier lets every lane finish reading the tables
// of the env's previous body; the trailing one publishes the new ones.
__device__ __forceinline__ void stage_body(LinkTables* lt, double* s_clx, double* s_cly, int lane, const BodyConst* bb) {
    const ModelConst& m = c_model;
    __syncwarp();
    stage_link_tables(lt, bb);
    if (s_clx) {
        for (int t = lane; t < m.n_corners; t += kWarp) { s_clx[t] = BL(corner_lx, t); s_cly[t] = BL(corner_ly, t); }
        if (lane < m.nj) {
            double* tb = s_clx + 4 * kMaxJoints;
            const int t = lane;
            tb[t] = BL(body_ax, t); tb[kMaxJoints + t] = BL(body_ay, t); tb[2 * kMaxJoints + t] = BL(body_cos, t); tb[3 * kMaxJoints + t] = BL(body_sin, t);
            tb[4 * kMaxJoints + t] = BL(half_x, t); tb[5 * kMaxJoints + t] = BL(half_y, t);
        }
    }
    __syncwarp();
}
// the draws run once per episode: out of line, they leave the step kernel's registers to its hot loop (inlined, its spill stores / loads
// grow from 260 / 824 B to 324 / 1,276 B)
#ifdef TRL_SIMT_EMU
#define TRL_NOINLINE
#else
#define TRL_NOINLINE __noinline__
#endif
// one number of a ranged slot's draw (trl_types.h: kBodyDrawTag): lo + u (hi - lo), each operation rounded on its own, at most hi
__device__ __forceinline__ double draw_in(double lo, double hi, double u) { return fmin(hi, __dadd_rn(lo, __dmul_rn(u, __dsub_rn(hi, lo)))); }
// The env's body on ranged body slot bs for the episode a reset begins: the slot's table with Mass, Kp, Kd and TorqueLim drawn per link
// (lane j draws link j), and izz_c, izz_o and total_mass derived from the drawn masses with fill_model's expressions (trl_host.cu), in
// its association and each operation rounded on its own, so the entry equals what trl_load_body makes of a file holding the drawn
// numbers.  Lane 0 sums total_mass over the links in index order, as fill_model does.  Writes the env's entry of c_env_bdraw.
__device__ TRL_NOINLINE const BodyConst* draw_body(const Lane& L, int bs, int lane) {
    const ModelConst& m = c_model;
    BodyConst* d = c_env_bdraw + L.env;
    const BodyConst& lo = g_body[bs];
    const BodyConst& hi = g_body_hi[bs];
    const unsigned long long* src = reinterpret_cast<const unsigned long long*>(&lo);
    unsigned long long* dst = reinterpret_cast<unsigned long long*>(d);
    static_assert(sizeof(BodyConst) % 8 == 0, "the body table is copied in 8-byte words");
    for (int w = lane; w < (int)(sizeof(BodyConst) / 8); w += kWarp) dst[w] = src[w];
    const long long draw = c_env_draws[L.env];
    __syncwarp();
    if (lane < m.nj) {
        const int nj = m.nj;
        const unsigned long long key = draw_key(m.rng_seed, kBodyDrawTag, L.env, draw);
        const double mass = draw_in(lo.mass[lane], hi.mass[lane], draw_unit(key, lane));
        d->mass[lane] = mass;
        d->kp[lane] = draw_in(lo.kp[lane], hi.kp[lane], draw_unit(key, nj + lane));
        d->kd[lane] = draw_in(lo.kd[lane], hi.kd[lane], draw_unit(key, 2 * nj + lane));
        d->torque_lim[lane] = draw_in(lo.torque_lim[lane], hi.torque_lim[lane], draw_unit(key, 3 * nj + lane));
        // the box sizes are twice the half sizes (exact), the centre offsets the BodyDefs AttachX / AttachY
        const double sx = 2.0 * lo.half_x[lane], sy = 2.0 * lo.half_y[lane], ax = lo.body_ax[lane], ay = lo.body_ay[lane];
        const double izz_c = __dmul_rn(__ddiv_rn(mass, 12.0), __dadd_rn(__dmul_rn(sx, sx), __dmul_rn(sy, sy)));
        d->izz_c[lane] = izz_c;
        d->izz_o[lane] = __dadd_rn(izz_c, __dmul_rn(mass, __dadd_rn(__dmul_rn(ax, ax), __dmul_rn(ay, ay))));
    }
    __syncwarp();
    if (lane == 0) {
        double total = 0.0;
        for (int j = 0; j < m.nj; ++j) total = __dadd_rn(total, d->mass[j]);
        d->total_mass = total;
        c_env_draws[L.env] = draw + 1;
    }
    __syncwarp();
    return d;
}
// The env's physics on ranged physics slot q for the episode a reset begins (lane 0): the seven constants drawn, vertex_contacts the slot's.
// Writes the env's entry of c_env_pdraw
__device__ TRL_NOINLINE void draw_phys(const Lane& L, int q) {
    const long long draw = c_env_draws[(size_t)L.n + L.env];
    const unsigned long long key = draw_key(c_model.rng_seed, kPhysDrawTag, L.env, draw);
    const PhysParams& lo = c_phys[q];
    const PhysParams& hi = c_phys_hi[q];
    PhysParams* d = c_env_pdraw + L.env;
    d->kn = draw_in(lo.kn, hi.kn, draw_unit(key, 0));
    d->dn = draw_in(lo.dn, hi.dn, draw_unit(key, 1));
    d->mu = draw_in(lo.mu, hi.mu, draw_unit(key, 2));
    d->v_eps = draw_in(lo.v_eps, hi.v_eps, draw_unit(key, 3));
    d->contact_tol = draw_in(lo.contact_tol, hi.contact_tol, draw_unit(key, 4));
    d->k_lim = draw_in(lo.k_lim, hi.k_lim, draw_unit(key, 5));
    d->d_lim = draw_in(lo.d_lim, hi.d_lim, draw_unit(key, 6));
    d->vertex_contacts = lo.vertex_contacts;
    c_env_draws[(size_t)L.n + L.env] = draw + 1;
}
// the body of the env's present episode: its slot's entry, or on a ranged slot its own drawn one
__device__ __forceinline__ const BodyConst* env_body(int bs, int env) {
    return ((c_body_ranged >> bs) & 1u) ? c_env_bdraw + env : &g_body[bs];
}
// at an episode reset: the body slot assigned to the env (trl_set_env_body) becomes its current one, a ranged slot draws the episode's
// body, and the warp restages its tables for it.  Returns the body
__device__ __forceinline__ const BodyConst* begin_body(const Lane& L, LinkTables* lt, double* s_clx, double* s_cly, int lane) {
    int bs = 0;
    if (c_env_body) {
        bs = c_env_body[(size_t)L.n + L.env];
        if (lane == 0) c_env_body[L.env] = bs;
    }
    const BodyConst* bb = ((c_body_ranged >> bs) & 1u) ? draw_body(L, bs, lane) : &g_body[bs];
    stage_body(lt, s_clx, s_cly, lane, bb);
    return bb;
}
#endif

// root-ward prefix sums over the kinematic tree by pointer jumping: after 4 rounds every link holds the sum of its own
// value and those of all its ancestors (depth <= 15), using the static 2^k-th ancestor table.  A missing ancestor points
// at lane 31, which is idle and holds zeros, so the adds need no predicate.
#if TRL_KIN_SMEM
// the same rounds through shared memory: every lane stores its pair, the receiver loads the pair of its 2^r-th ancestor.
// Rounds alternate between two buffers, so one __syncwarp per round suffices (a buffer is rewritten two rounds later, and
// the barrier of the round in between orders that write after every read).  `xs`, `lane` must be in scope.
#define TRL_TREE_PREFIX2(a, b)                                                                  \
    do {                                                                                        \
        _Pragma("unroll") for (int r_ = 0; r_ < 4; ++r_) {                                      \
            const int an_ = (r_ == 0) ? kin_anc1 : ((r_ == 1) ? kin_anc2 : ((r_ == 2) ? kin_anc4 : kin_anc8));                 \
            double2* buf_ = trl_as2<double2>(xs + X_PFX + (r_ & 1) * 2 * kWarp);      \
            buf_[lane] = make_double2((a), (b));                                                \
            __syncwarp();                                                                       \
            const double2 t_ = buf_[an_];                                                       \
            (a) += t_.x; (b) += t_.y;                                                           \
        }                                                                                       \
    } while (0)
#else
#define TRL_TREE_PREFIX2(a, b)                                                                  \
    do {                                                                                        \
        _Pragma("unroll") for (int r_ = 0; r_ < 4; ++r_) {                                      \
            const int an_ = (r_ == 0) ? kin_anc1 : ((r_ == 1) ? kin_anc2 : ((r_ == 2) ? kin_anc4 : kin_anc8));                 \
            double ta_ = shf((a), an_), tb_ = shf((b), an_);                                    \
            (a) += ta_; (b) += tb_;                                                             \
        }                                                                                       \
    } while (0)

#endif

// outward kinematics: world rotation, joint origin (rel. O) and spatial velocity of every link
__device__ __forceinline__ Kin kinematics(const LinkC& c, const EnvRegs& e TRL_KIN_XS_DECL) {
    Kin k;
    // the link's table entries are read once per call (they live in shared memory; a read cannot move across the shuffles below)
    const int kin_anc1 = c.anc1, kin_anc2 = c.anc2, kin_anc4 = c.anc4, kin_anc8 = c.anc8, kin_parent = c.parent, kin_depth = c.depth;
    double phi = e.q, w = e.qd;
    TRL_TREE_PREFIX2(phi, w);
    k.phi = phi; k.w = w;
    sincos(phi, &k.sw, &k.cw);
    // offset of this joint from its parent's joint, in world axes
#if TRL_KIN_SMEM
    double pcw, psw;
    {
        double2* buf = trl_as2<double2>(xs + X_PFX + 2 * 2 * kWarp);
        buf[lane] = make_double2(k.cw, k.sw);
        __syncwarp();
        const double2 t = buf[kin_parent];
        pcw = t.x; psw = t.y;
    }
#else
    double pcw = shf(k.cw, kin_parent), psw = shf(k.sw, kin_parent);
#endif
    double rx = 0.0, ry = 0.0;
    if (kin_depth > 0) { const double ax = c.ax, ay = c.ay; rx = pcw * ax - psw * ay; ry = psw * ax + pcw * ay; }
    TRL_TREE_PREFIX2(rx, ry);
    // v_j = v_root + sum over the chain of S_a qd_a,  S_a = (1, r_ay, -r_ax)
    double vx = (kin_depth > 0) ? e.qd * ry : e.oxd, vy = (kin_depth > 0) ? -e.qd * rx : e.oyd;
    if (kin_depth < 0) { vx = 0.0; vy = 0.0; }
    TRL_TREE_PREFIX2(vx, vy);
    k.rx = rx; k.ry = ry; k.vx = vx; k.vy = vy;
    const double bax = c.bax, bay = c.bay;
    k.cx = rx + k.cw * bax - k.sw * bay;
    k.cy = ry + k.sw * bax + k.cw * bay;
    return k;
}

// ================================================================================================ chain passes
// The tree recursions run one lane per chain (ModelConst::chain_*): the link lanes fill their slots of the link block, then lane c
// walks chain c through it, carrying the running values in registers from link to link -- in world axes the hand-off to the
// parent is a plain addition -- and other chains' results are added only at branch points, in the schedule's fixed order.
// Per-link values live in the link block, never in dynamically indexed register arrays (those would be local memory).
struct ChainC {
    unsigned long long links;   // 5 bits per link, bottom first
    int len, level, merge, up;  // level -1: this lane walks no chain
};
__device__ __forceinline__ ChainC chain_of(const LinkC& lc) {
    return ChainC{lc.ch_links, lc.ch_len, lc.ch_level, lc.ch_merge, lc.ch_up};
}
template <int NV>
__device__ __forceinline__ void load_vals(const double* p, double (&v)[NV]) {
#pragma unroll
    for (int k = 0; k + 1 < NV; k += 2) { const double2 t = *trl_as2<const double2>(p + k); v[k] = t.x; v[k + 1] = t.y; }
    if (NV & 1) v[NV - 1] = p[NV - 1];
}
template <int NV>
__device__ __forceinline__ void store_vals(double* p, const double (&v)[NV]) {
#pragma unroll
    for (int k = 0; k + 1 < NV; k += 2) *trl_as2<double2>(p + k) = make_double2(v[k], v[k + 1]);
    if (NV & 1) p[NV - 1] = v[NV - 1];
}

// Inward pass, leaf chains first.  Every link's slot value is summed with what its child hands up (own + child; at a branch point
// own + the child chains in merge order).  kElim: articulated-body elimination of every link but the root -- U_j, 1/D_j and u_j go
// back to the slot, the reduced inertia and bias force go up; the root's chain lane (lane 0) ends with the root's articulated
// inertia and bias force in `a`.  !kElim: plain subtree sums (composite inertias), written back to every slot.
template <int NV, bool kElim>
__device__ __forceinline__ void chain_inward(double* xs, const ChainC& ch, int lane, double dt, double (&a)[NV]) {
    const ModelConst& m = c_model;
#pragma unroll
    for (int k = 0; k < NV; ++k) a[k] = 0.0;
    for (int lev = 0; lev < m.chain_levels; ++lev) {
        const int n = ch.level == lev ? ch.len : 0;     // links this lane walks in this level
        for (int i = 0; i < n; ++i) {
            const int j = (int)(ch.links >> (5 * i)) & 31;
            double* sl = xs + X_LNK + j * kLinkStride;
            double v[NV];
            load_vals(sl, v);
            if (i == 0) {
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const int src = (ch.merge >> (5 * q)) & 31;
                    if (src == 31) continue;
                    const double* o = xs + X_CHO + src * kChainStride;
#pragma unroll
                    for (int k = 0; k < NV; ++k) v[k] += o[k];
                }
            } else {
#pragma unroll
                for (int k = 0; k < NV; ++k) v[k] += a[k];
            }
            if (kElim && j != 0) {
                const double2 cv = *trl_as2<const double2>(sl + LK_CV), sv = *trl_as2<const double2>(sl + LK_S),
                              lm = *trl_as2<const double2>(sl + LK_LIM);
                const double s1 = sv.x, s2 = sv.y;
                const double U0 = v[0] + v[1] * s1 + v[2] * s2;
                const double U1 = v[1] + v[3] * s1 + v[4] * s2;
                const double U2 = v[2] + v[4] * s1 + v[5] * s2;
                double Dj = U0 + s1 * U1 + s2 * U2;
                double uu = sl[LK_TAU] - (v[6] + s1 * v[7] + s2 * v[8]);
                uu -= lm.x;
                Dj += dt * lm.y;
                const double dinv = rcp_pivot(Dj);
                // Ia = IA - U U^T / D ;  pa = pA + Ia c + U u / D
                const double n0 = v[0] - U0 * U0 * dinv, n1 = v[1] - U0 * U1 * dinv, n2 = v[2] - U0 * U2 * dinv;
                const double n3 = v[3] - U1 * U1 * dinv, n4 = v[4] - U1 * U2 * dinv, n5 = v[5] - U2 * U2 * dinv;
                const double ud = uu * dinv;
                a[6] = v[6] + (n1 * cv.x + n2 * cv.y + U0 * ud);
                a[7] = v[7] + (n3 * cv.x + n4 * cv.y + U1 * ud);
                a[8] = v[8] + (n4 * cv.x + n5 * cv.y + U2 * ud);
                a[0] = n0; a[1] = n1; a[2] = n2; a[3] = n3; a[4] = n4; a[5] = n5;
                *trl_as2<double2>(sl + LK_U) = make_double2(U0, U1);
                *trl_as2<double2>(sl + LK_U + 2) = make_double2(U2, dinv);
                sl[LK_UU] = uu;
            } else {
#pragma unroll
                for (int k = 0; k < NV; ++k) a[k] = v[k];
                if (!kElim) store_vals(sl, v);
            }
        }
        if (n > 0) store_vals(xs + X_CHO + lane * kChainStride, a);
        __syncwarp();
    }
}

// Outward pass, root chain first: qdd_j = (u_j - U_j . (a_parent + c_j)) / D_j, a_j = a_parent + c_j + S_j qdd_j; the root's
// spatial acceleration is (a0, a1, a2).  qdd and a go to every link's slot.
__device__ __forceinline__ void chain_outward(double* xs, const ChainC& ch, double a0, double a1, double a2) {
    const ModelConst& m = c_model;
    for (int lev = m.chain_levels - 1; lev >= 0; --lev) {
        const int n = ch.level == lev ? ch.len : 0;     // links this lane walks in this level, top link first
        double aw = 0.0, alx = 0.0, aly = 0.0;
        for (int i = 0; i < n; ++i) {
            const int j = (int)(ch.links >> (5 * (n - 1 - i))) & 31;
            double* sl = xs + X_LNK + j * kLinkStride;
            if (j == 0) {
                aw = a0; alx = a1; aly = a2;
            } else {
                double paw = aw, pax = alx, pay = aly;
                if (i == 0) {
                    const double* ps = xs + X_LNK + ch.up * kLinkStride;
                    const double2 t = *trl_as2<const double2>(ps + LK_ACC);
                    paw = t.x; pax = t.y; pay = ps[LK_ACC + 2];
                }
                const double2 u01 = *trl_as2<const double2>(sl + LK_U), u2d = *trl_as2<const double2>(sl + LK_U + 2);
                const double2 cv = *trl_as2<const double2>(sl + LK_CV), sv = *trl_as2<const double2>(sl + LK_S);
                const double bx = pax + cv.x, by = pay + cv.y;
                const double qdd = (sl[LK_UU] - (u01.x * paw + u01.y * bx + u2d.x * by)) * u2d.y;
                aw = paw + qdd; alx = bx + sv.x * qdd; aly = by + sv.y * qdd;
                sl[LK_QDD] = qdd;
            }
            *trl_as2<double2>(sl + LK_ACC) = make_double2(aw, alx);
            sl[LK_ACC + 2] = aly;
        }
        __syncwarp();
    }
}

// Articulated-body forward dynamics of the tree over the link block: inward eliminations, floating base IA_0 a_0 = -pA_0 (symmetric
// 3x3 LDL^T, every lane computes it from lane 0's values), outward accelerations.  The caller has filled every link's slot and
// synchronised the warp; afterwards slot LK_QDD holds each joint's acceleration, (a0, a1, a2) the root's.
__device__ __forceinline__ void chain_aba(double* xs, const ChainC& ch, int lane, double dt, double& a0, double& a1, double& a2
                                          TRL_CLK_DECL(ph_in, ph_out)) {
    TRL_CLK_BEGIN(clk);
    double ia[9];
    chain_inward<9, true>(xs, ch, lane, dt, ia);
    TRL_CLK_END(ph_in, clk);
    {
#if TRL_OUTWARD_SMEM
        double* bs = xs + X_BASE;
        if (lane == 0) store_vals(bs, ia);
        __syncwarp();
        double q[9];
        load_vals(bs, q);
        const double a = q[0], bx = q[1], by = q[2], cxx = q[3], cxy = q[4], cyy = q[5];
        const double r0 = -q[6], r1 = -q[7], r2 = -q[8];
#else
        const double a = shf(ia[0], 0), bx = shf(ia[1], 0), by = shf(ia[2], 0), cxx = shf(ia[3], 0), cxy = shf(ia[4], 0), cyy = shf(ia[5], 0);
        const double r0 = -shf(ia[6], 0), r1 = -shf(ia[7], 0), r2 = -shf(ia[8], 0);
#endif
        const double i0 = rcp_pivot(a), l10 = bx * i0, l20 = by * i0;
        const double d1 = cxx - l10 * bx, i1 = rcp_pivot(d1), t21 = cxy - l20 * bx, l21 = t21 * i1;
        const double d2 = cyy - l20 * by - l21 * t21, i2 = rcp_pivot(d2);
        const double y0 = r0, y1 = r1 - l10 * y0, y2 = r2 - l20 * y0 - l21 * y1;
        a2 = y2 * i2; a1 = y1 * i1 - l21 * a2; a0 = y0 * i0 - l10 * a1 - l20 * a2;
    }
    chain_outward(xs, ch, a0, a1, a2);
    TRL_CLK_END(ph_out, clk);
}

// ================================================================================================ controller half
// Returns the clamped joint torque of link `lane` (0 for the root and idle lanes).
__device__ double controller_torque(Lane& L, const LinkC& lc, const EnvRegs& e, const Kin& k, double* xs, int lane,
                                    double h, int contact TRL_BS_DECL) {
    const double lk_mass = lc.mass;      // read once (shared-memory table; a read cannot move across the shuffles below)
    const ModelConst& m = c_model;
    const int md = m.max_depth;
    const ChainC ch = chain_of(lc);
    double* slot = xs + X_LNK + lane * kLinkStride;     // this link's slot of the link block (written by active link lanes only)
    TRL_CLK_BEGIN(clk);

    // ---- body inertia about O in world axes, RNEA accelerations with qdd = 0 and the reference's Cj
    const double hx = lk_mass * k.cx, hy = lk_mass * k.cy, Io = lc.izz_c + lk_mass * (k.cx * k.cx + k.cy * k.cy);
    double alx, aly;
    {
        // root: a0 = -g + R0 * cj, cj from cRBDUtil::BuildCjPlanar with c = s = cos(theta_dot) (sim/RBDUtil.cpp:821-822)
        double thd = shf(e.qd, 0), c0 = shf(k.cw, 0), s0 = shf(k.sw, 0);
        double cb = cos(thd);
        double cjx = (-cb * e.oxd + cb * e.oyd) * thd, cjy = (-cb * e.oxd - cb * e.oyd) * thd;
        alx = -m.gx + c0 * cjx - s0 * cjy;
        aly = -m.gy + s0 * cjx + c0 * cjy;
    }
    const int ctl_parent = lc.parent, ctl_depth = lc.depth;
    for (int l = 1; l <= md; ++l) {
        double pax = shf(alx, ctl_parent), pay = shf(aly, ctl_parent);
        if (ctl_depth == l) {
            alx = pax + e.qd * (k.w * k.rx + k.vy);   // a_j = a_parent + v_j x (S_j qd_j)
            aly = pay + e.qd * (k.w * k.ry - k.vx);
        }
    }
    // vals: composite inertia (Io, hx, hy, m) and subtree force (n, fx, fy)
    double vals[7];
    {
        double hlx = -hy * k.w + lk_mass * k.vx, hly = hx * k.w + lk_mass * k.vy;
        vals[0] = Io; vals[1] = hx; vals[2] = hy; vals[3] = lk_mass;
        vals[4] = (-hy * alx + hx * aly) + (k.vx * hly - k.vy * hlx);
        vals[5] = lk_mass * alx - k.w * hly;
        vals[6] = lk_mass * aly + k.w * hlx;
        if (!lc.act) { vals[4] = vals[5] = vals[6] = 0.0; }
    }
    {
        if (lc.act) store_vals(slot, vals);
        __syncwarp();
        double sum[7];
        chain_inward<7, false>(xs, ch, lane, 0.0, sum);
        if (lc.act) load_vals(slot, vals);
    }
    TRL_CLK_END(PH_RNEA, clk);
    const double s1 = k.ry, s2 = -k.rx;                       // S_j = (1, s1, s2)
    // bias force C (per link lane; the root's three entries live in lane 0)
    const double Cj = vals[4] + s1 * vals[5] + s2 * vals[6];
    const double C0 = shf(vals[5], 0), C1 = shf(vals[6], 0), C2 = shf(vals[4], 0);

    // ---- ApplyFeedback (sim/DogController.cpp:903-945) / ApplySwingFeedback (sim/RaptorController.cpp:907-931)
    const int state = L.i(I_STATE);
    const bool raptor = TRL_IS_RAPTOR(m);
    const int stance = raptor ? L.i(I_STANCE) : 0;
    const int st_hip = stance == 0 ? rRightHip : rLeftHip, sw_hip = stance == 0 ? rLeftHip : rRightHip, st_toe = st_hip + 3;
    // cRaptorController::IsActiveVFEffector(stance toe): stance foot on the ground during Contact / Down
    const bool active_vf = raptor && (state == rsContact || state == rsDown) && ((contact >> st_toe) & 1);
    {
        double bvx = lk_mass * (k.vx - k.w * k.cy);
        double comvx = warp_sum_all(bvx) / BM(total_mass);
        if (raptor) {
            double comx = warp_sum_all(lk_mass * k.cx) / BM(total_mass);
            double toe_x = shf(k.cx, st_toe);
            if (lane == 0) {
                bool first_half = state == rsContact || state == rsDown;
                double cd = first_half ? 0.0 : L.d(D_PARAMS + rmCd), cv = first_half ? L.d(D_PARAMS + rmCv) : 0.0;
                int base = D_PARAMS + m.misc_max + state * m.sp_max;
                L.d(D_PD_TARGET + sw_hip) = L.d(base + rpSwingHip) + (cd * (comx - toe_x) + cv * comvx);
            }
        } else if (lane == 0) {
            double cv = L.d(D_PARAMS + mCv);
            int base = D_PARAMS + mMiscMax + state * spMax;
            if (!((contact >> jToe) & 1)) L.d(D_PD_TARGET + jHip) = L.d(base + spHip) + comvx * cv;
            if (!((contact >> jFinger) & 1)) L.d(D_PD_TARGET + jShoulder) = L.d(base + spShoulder) + comvx * cv;
        }
        __syncwarp();
    }

    // ---- cImpPDController::CalcControlForces (sim/ImpPDController.cpp:234-278); the raptor's stance hip PD is
    // switched off while its foot is an active virtual-force effector (UpdateStanceHip, sim/RaptorController.cpp:899-905):
    // zero gains in the torque law, but its Kd stays on the diagonal of the solved system
    double tau0 = 0.0, rhs_link = 0.0, kd_link = 0.0, kd_eff = 0.0;
    if (lc.act && lane > 0) {
        double theta = e.q;
        if (BL(world_pd, lane)) {
            // child body's world rotation, wrapped (cPDController::CalcTheta, sim/PDController.cpp:181-198)
            double c = k.cw * BL(body_cos, lane) - k.sw * BL(body_sin, lane);
            double s = k.sw * BL(body_cos, lane) + k.cw * BL(body_sin, lane);
            double a = acos(fmin(1.0, fmax(-1.0, c)));
            theta = (s >= 0) ? a : -a;
        }
        const bool pd_on = !(active_vf && lane == st_hip);
        kd_link = BL(kd, lane);
        kd_eff = pd_on ? kd_link : 0.0;
        double perr = L.d(D_PD_TARGET + lane) - theta, verr = BL(target_vel, lane) - e.qd;
        tau0 = pd_on ? (BL(kp, lane) * (perr - h * e.qd) + kd_link * verr) : 0.0;
        rhs_link = tau0 - Cj;
    }
    // (M + h Kd) acc = rhs is the articulated-body problem of the same tree at rest: no velocity products, no gravity, joint
    // forces rhs_j, the root's generalised force (-C0, -C1, -C2) as the spatial force (n, fx, fy) = (-C2, -C0, -C1) (a bias
    // force is its negative), and h kd_j as a joint armature added to D_j -- O(n) instead of the dense 23x23 factorisation
    if (lc.act) {
        const double own[9] = {Io, -hy, hx, lk_mass, 0.0, lk_mass, lane == 0 ? C2 : 0.0, lane == 0 ? C0 : 0.0, lane == 0 ? C1 : 0.0};
        store_vals(slot, own);
        slot[LK_TAU] = rhs_link;
        *trl_as2<double2>(slot + LK_CV) = make_double2(0.0, 0.0);
        *trl_as2<double2>(slot + LK_S) = make_double2(s1, s2);
        *trl_as2<double2>(slot + LK_LIM) = make_double2(0.0, kd_link);
    }
    __syncwarp();
    TRL_CLK_END(PH_SOLVE, clk);          // feedback laws + the link block; chain_aba counts its own parts, once
    double tau = 0.0;
    {
        double b0, b1, b2;
        chain_aba(xs, ch, lane, h, b0, b1, b2 TRL_CLK_ARG(PH_SOLVE, PH_SOLVE));
        TRL_CLK_RESET(clk);
        if (lc.act && lane > 0) tau = tau0 - kd_eff * h * slot[LK_QDD];
    }
    TRL_CLK_END(PH_SOLVE, clk);

    // ---- ApplyGravityCompensation (sim/DogController.cpp:947-995, 1120-1175; sim/RaptorController.cpp:983-1026)
    // effector 0 / 1: dog back foot (toe) / front foot (finger); raptor right / left toe.  A dog foot supports when
    // it touches the ground, a raptor foot only while it is the active virtual-force effector.
    const int eff0 = raptor ? (int)rRightToe : (int)jToe, eff1 = raptor ? (int)rLeftToe : (int)jFinger;
    const bool toe_c = raptor ? (active_vf && stance == 0) : (((contact >> jToe) & 1) != 0);
    const bool fin_c = raptor ? (active_vf && stance == 1) : (((contact >> jFinger) & 1) != 0);
    // foot bottom-centre positions (GetEndEffectorContactPos), relative to O
    double ex[2], ey[2];
    {
        double bc = k.cw * BL(body_cos, lc.act ? lane : 0) - k.sw * BL(body_sin, lc.act ? lane : 0);
        double bsn = k.sw * BL(body_cos, lc.act ? lane : 0) + k.cw * BL(body_sin, lc.act ? lane : 0);
        double ly = -BL(half_y, lc.act ? lane : 0);
        double px = k.cx - bsn * ly, py = k.cy + bc * ly;
        ex[0] = shf(px, eff0); ey[0] = shf(py, eff0);
        ex[1] = shf(px, eff1); ey[1] = shf(py, eff1);
    }
    if (m.grav_comp && (toe_c || fin_c)) {
        // tau_g = -G,  G_k = (sum_subtree m (c - r_k)) x g   (generalised gravity force, sim/RBDUtil.cpp:850-895)
        const double ms = vals[3], mhx = vals[1], mhy = vals[2];
        double tg;
        if (lane == 0) tg = 0.0;
        else tg = -((mhx - ms * k.rx) * m.gy - (mhy - ms * k.ry) * m.gx);
        const double ms0 = shf(ms, 0), mhx0 = shf(mhx, 0), mhy0 = shf(mhy, 0);
        const double b0 = -(ms0 * m.gx), b1 = -(ms0 * m.gy), b2 = -(mhx0 * m.gy - mhy0 * m.gx);
        // root-row weights of the ridge least squares: identity for the dog, (1e-4, 1e-4, 1) for the raptor
        const double W0 = raptor ? 0.0001 : 1.0, W1 = raptor ? 0.0001 : 1.0, W2 = 1.0;
        // basis columns [eff0 +y, eff0 +x, eff1 +y, eff1 +x]; root rows = (Fx, Fy, r x F)
        double Ar[3][4];
#pragma unroll
        for (int e2 = 0; e2 < 2; ++e2) {
            bool on = e2 == 0 ? toe_c : fin_c;
            Ar[0][2 * e2] = 0.0;            Ar[0][2 * e2 + 1] = on ? 1.0 : 0.0;
            Ar[1][2 * e2] = on ? 1.0 : 0.0; Ar[1][2 * e2 + 1] = 0.0;
            Ar[2][2 * e2] = on ? ex[e2] : 0.0; Ar[2][2 * e2 + 1] = on ? -ey[e2] : 0.0;
        }
        double A[4][5];
#pragma unroll
        for (int a = 0; a < 4; ++a) {
#pragma unroll
            for (int b = 0; b < 4; ++b) A[a][b] = Ar[0][a] * W0 * Ar[0][b] + Ar[1][a] * W1 * Ar[1][b] + Ar[2][a] * W2 * Ar[2][b];
            A[a][a] += 0.0001;
            A[a][4] = Ar[0][a] * W0 * b0 + Ar[1][a] * W1 * b1 + Ar[2][a] * W2 * b2;
        }
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            int piv = c;
#pragma unroll
            for (int r = c + 1; r < 4; ++r) if (fabs(A[r][c]) > fabs(A[piv][c])) piv = r;
#pragma unroll
            for (int r = 0; r < 4; ++r) {
                if (r == piv && piv != c) {
#pragma unroll
                    for (int kk = 0; kk < 5; ++kk) { double t = A[c][kk]; A[c][kk] = A[r][kk]; A[r][kk] = t; }
                }
            }
#pragma unroll
            for (int r = c + 1; r < 4; ++r) {
                double f = A[r][c] / A[c][c];
#pragma unroll
                for (int kk = c; kk < 5; ++kk) A[r][kk] -= f * A[c][kk];
            }
        }
        double x[4];
#pragma unroll
        for (int r = 3; r >= 0; --r) {
            double v = A[r][4];
#pragma unroll
            for (int kk = r + 1; kk < 4; ++kk) v -= A[r][kk] * x[kk];
            x[r] = v / A[r][r];
        }
        if (lc.act && lane > 0) {
            double tc = 0.0;
            if (toe_c && ((m.anc_mask_toe >> lane) & 1)) { double rx = ex[0] - k.rx, ry = ey[0] - k.ry; tc += rx * x[0] - ry * x[1]; }
            if (fin_c && ((m.anc_mask_finger >> lane) & 1)) { double rx = ex[1] - k.rx, ry = ey[1] - k.ry; tc += rx * x[2] - ry * x[3]; }
            tau += tg - tc;
        }
    }

    // ---- ApplyStanceFeedback (sim/RaptorController.cpp:933-981): the stance hip balances the swing hip's torque and
    // a PD on the root pitch while its foot pushes
    if (raptor) {
        const double sw_tau = shf(tau, sw_hip), th0 = shf(e.q, 0), thd0 = shf(e.qd, 0);
        if (active_vf && lane == st_hip) {
            int base = D_PARAMS + m.misc_max + state * m.sp_max;
            double root_tau = BU(kp, st_hip) * (L.d(base + rpRootPitch) - wrap_pi(th0)) + BU(kd, st_hip) * (-thd0);
            tau += -sw_tau - root_tau;
        }
    }

    // ---- ApplyVirtualForces (sim/DogController.cpp:997-1029; sim/RaptorController.cpp:1028-1075)
    if (m.virt_forces && raptor) {
        // only the stance toe can be active; the chain runs up to (excluding) the root and the stance hip's share is
        // mirrored onto the swing hip
        const bool on = active_vf;
        const int e2 = stance;
        double fx = -L.d(D_PARAMS + rmForceX), fy = -L.d(D_PARAMS + rmForceY);
        unsigned mask = e2 == 0 ? m.vf_mask_toe : m.vf_mask_finger;
        double t = 0.0;
        if (on && lc.act && ((mask >> lane) & 1)) t = (ex[e2] - k.rx) * fy - (ey[e2] - k.ry) * fx;
        double t_hip = shf(t, st_hip);
        tau += t;
        if (on && lane == sw_hip) tau -= t_hip;
    } else if (m.virt_forces && lc.act && lane > 0) {
        if ((state == sBackStance || state == sExtend) && toe_c && ((m.vf_mask_toe >> lane) & 1)) {
            double fx = -L.d(D_PARAMS + mBackForceX), fy = -L.d(D_PARAMS + mBackForceY);
            tau += (ex[0] - k.rx) * fy - (ey[0] - k.ry) * fx;
        }
        if ((state == sFrontStance || state == sGather) && fin_c && ((m.vf_mask_finger >> lane) & 1)) {
            double fx = -L.d(D_PARAMS + mFrontForceX), fy = -L.d(D_PARAMS + mFrontForceY);
            tau += (ex[1] - k.rx) * fy - (ey[1] - k.ry) * fx;
        }
    }

    // ---- cJoint::ApplyTorque clamp (sim/Joint.cpp:171-201,257-264)
    if (lc.act && lane > 0) {
        double lim = BL(torque_lim, lane);
        if (fabs(tau) > lim) tau *= lim / fabs(tau);
    } else tau = 0.0;
    TRL_CLK_END(PH_CTRL_REST, clk);
    return tau;
}

// ================================================================================================ physics half
// One sub-step of articulated-body forward dynamics with linearly-implicit contact / joint-limit terms.
// Updates e (q, qd, root translation) in place and returns the contact bitmask (same value in every lane).
__device__ int physics_substep(const LinkC& lc, EnvRegs& e, const GroundView& g, const double* s_clx, const double* s_cly,
                               int lane, double dt, double clear_y, double* xs TRL_REUSE_KIN_DECL TRL_PS_DECL) {
    const double lk_mass = lc.mass;      // read once (shared-memory table; a read cannot move across the shuffles below)
    // per-body box tables (link frame): centre offset, axis rotation, half sizes -- staged by the kernel next to the corner tables
    const double *s_bax = s_clx + 4 * kMaxJoints, *s_bay = s_bax + kMaxJoints, *s_bc = s_bay + kMaxJoints, *s_bs = s_bc + kMaxJoints,
                 *s_hx = s_bs + kMaxJoints, *s_hy = s_hx + kMaxJoints;
    const ModelConst& m = c_model;
#if TRL_BODY_TABLE
    // pp: the env's physics in the warp's shared-memory copy (the same in every lane: one broadcast per read)
#elif TRL_PHYS_TABLE
    // the env's slot: ps is the same in every lane (one env per warp), so each read is one broadcast from the constant cache
    const PhysParams& pp = c_phys[ps];
#else
    const PhysParams& pp = m.phys;
#endif
    TRL_CLK_BEGIN(clk);
#if TRL_REUSE_KIN
    Kin k;
    if (k0) k = *k0; else k = kinematics(lc, e TRL_KIN_XS_ARG);
#else
    Kin k = kinematics(lc, e TRL_KIN_XS_ARG);
#endif

    // rigid inertia about O, bias force incl. gravity as an external force
    const double hx = lk_mass * k.cx, hy = lk_mass * k.cy, Io = lc.izz_c + lk_mass * (k.cx * k.cx + k.cy * k.cy);
    double ia[9];   // articulated inertia (a, bx, by, cxx, cxy, cyy) and bias force (n, fx, fy)
    {
        double hlx = -hy * k.w + lk_mass * k.vx, hly = hx * k.w + lk_mass * k.vy;
        ia[0] = Io; ia[1] = -hy; ia[2] = hx; ia[3] = lk_mass; ia[4] = 0.0; ia[5] = lk_mass;
        ia[6] = (k.vx * hly - k.vy * hlx) - (hx * m.gy - hy * m.gx);
        ia[7] = -k.w * hly - lk_mass * m.gx;
        ia[8] = k.w * hlx - lk_mass * m.gy;
        if (!lc.act) { ia[6] = ia[7] = ia[8] = 0.0; }
    }
    const double cvx = e.qd * (k.w * k.rx + k.vy), cvy = e.qd * (k.w * k.ry - k.vx);   // c_j = v_j x (S_j qd_j)
    TRL_CLK_END(PH_KIN, clk);

    // ---- contacts: the lane of each collidable body tests its own box against the height field, with the body's kinematics in its
    // registers, and adds the forces straight into its articulated inertia: its 4 corners in corner order, then its vertex slots
    // one compliant contact at the point (rpx, rpy) rel. O of the body: penetration `pen` along the unit direction (nx, ny) the force
    // pushes the body in; implicit in the point velocity (adds dt X^T D X to the articulated inertia and X^T w to the bias force,
    // D = cnn n n^T + ctt t t^T).  The sums are __dadd_rn so that no add is merged with the multiply that produced a term or the
    // value it adds to: each contribution is rounded on its own, then added.
    auto contact_force = [&](double rpx, double rpy, double pen, double nx, double ny) {
        const double tx = ny, ty = -nx;
        const double pvx = k.vx - k.w * rpy, pvy = k.vy + k.w * rpx;
        const double vn = pvx * nx + pvy * ny, vt = pvx * tx + pvy * ty;
        const double fn0 = pp.kn * pen - pp.dn * vn;
        if (fn0 > 0.0) {
            const double cnn = pp.dn + dt * pp.kn;
            const double ctt = pp.mu * fn0 / fmax(fabs(vt), pp.v_eps);
            const double fwx = pp.kn * pen * nx - cnn * vn * nx - ctt * vt * tx;
            const double fwy = pp.kn * pen * ny - cnn * vn * ny - ctt * vt * ty;
            const double dxx = dt * (cnn * nx * nx + ctt * tx * tx), dxy = dt * (cnn * nx * ny + ctt * tx * ty),
                         dyy = dt * (cnn * ny * ny + ctt * ty * ty);
            const double kx = -rpy, ky = rpx;
            const double dkx = dxx * kx + dxy * ky, dky = dxy * kx + dyy * ky;
            if (dxx != 0.0 || dyy != 0.0) {
                // kx * dkx + ky * dky, spelled as the difference it is (kx = -rpy): written as a sum, the compiler fuses it into an FMA
                // of its own choosing, which rounds differently
                ia[0] = __dadd_rn(ia[0], ky * dky - dkx * rpy); ia[1] = __dadd_rn(ia[1], dkx); ia[2] = __dadd_rn(ia[2], dky);
                ia[3] = __dadd_rn(ia[3], dxx); ia[4] = __dadd_rn(ia[4], dxy); ia[5] = __dadd_rn(ia[5], dyy);
                ia[6] = __dadd_rn(ia[6], -(rpx * fwy - rpy * fwx)); ia[7] = __dadd_rn(ia[7], -fwx); ia[8] = __dadd_rn(ia[8], -fwy);
            }
        }
    };
    const int cb = lc.act ? LT(corner_base, lane) : -1;   // the body's 4 corners are cb .. cb + 3 of the corner tables
    bool touching = false;
    {
        // box corners.  Broad phase: a corner above clear_y (terrain maximum under the character + margin) cannot be within the
        // contact tolerance; a body with no candidate corner skips the height samples, a warp with none skips the pass.  The corner
        // loop is unrolled by two, so two height samples are in flight at a time (unrolled by four, the kernel spills more)
        const int c0 = cb >= 0 ? cb : 0;
        unsigned cand = 0;
#pragma unroll
        for (int cn = 0; cn < 4; ++cn) {
            const double ly = s_cly[c0 + cn], rpy = k.ry + k.sw * s_clx[c0 + cn] + k.cw * ly;
            if (cb >= 0 && (e.oy + rpy <= clear_y)) cand |= 1u << cn;
        }
        if (__any_sync(kFull, cand != 0) && cand) {
#pragma unroll 2
            for (int cn = 0; cn < 4; ++cn) {
                if (!((cand >> cn) & 1u)) continue;
                const double lx = s_clx[c0 + cn], ly = s_cly[c0 + cn];
                const double rpx = k.rx + k.cw * lx - k.sw * ly, rpy = k.ry + k.sw * lx + k.cw * ly;   // corner rel. O
                double slope;
                const double hgt = g.sample_fast(e.ox + rpx, &slope);
                const double inv = rsqrt(1.0 + slope * slope);
                const double pen = (hgt - (e.oy + rpy)) * inv;
                if (pen > -pp.contact_tol) {
                    touching = true;
                    if (pen > 0.0) contact_force(rpx, rpy, pen, -slope * inv, inv);
                }
            }
        }
    }
    if (pp.vertex_contacts) {
        // the terrain vertices inside the box (opt-in), after the corners: slot s is the s-th vertex under the body's x extent (a
        // box spans at most 4 vertices); where the surface is convex and the vertex lies inside, it is pushed out through the nearest
        // face (sim/GroundVar2D.cpp:440-448 hands Bullet a height field: an edge of the terrain can enter a box between two of its
        // corners)
        const int j = cb >= 0 ? lane : 0;
        const double bax = s_bax[j], bay = s_bay[j], bc = s_bc[j], bs = s_bs[j], hxb = s_hx[j], hyb = s_hy[j];
        const double C = k.cw * bc - k.sw * bs, S = k.sw * bc + k.cw * bs;                        // box axes in the world
        const double cxr = k.rx + k.cw * bax - k.sw * bay, cyr = k.ry + k.sw * bax + k.cw * bay;   // box centre rel. O
        const bool cand = cb >= 0 && (e.oy + cyr - (fabs(S) * hxb + fabs(C) * hyb) <= clear_y);
        if (__any_sync(kFull, cand) && cand) {
            const double extx = fabs(C) * hxb + fabs(S) * hyb, cxw = e.ox + cxr;
#pragma unroll 1
            for (int slot = 0; slot < 4; ++slot) {
                double xv, hv, hp, hn;
                if (!g.vertex_slot(cxw - extx - pp.contact_tol, cxw + extx + pp.contact_tol, slot, &xv, &hv, &hp, &hn) ||
                    !(hv - 0.5 * (hp + hn) > 1e-9))
                    continue;
                const double rx = xv - cxw, ry = hv - (e.oy + cyr);
                const double lx = C * rx + S * ry, ly = -S * rx + C * ry;
                const double dx = hxb - fabs(lx), dy = hyb - fabs(ly);
                if (dx > -pp.contact_tol && dy > -pp.contact_tol) {
                    touching = true;
                    if (dx > 0.0 && dy > 0.0) {
                        double nlx = 0.0, nly = 0.0, pen;
                        if (dx < dy) { nlx = lx > 0.0 ? -1.0 : 1.0; pen = dx; } else { nly = ly > 0.0 ? -1.0 : 1.0; pen = dy; }
                        contact_force(xv - e.ox, hv - e.oy, pen, C * nlx - S * nly, S * nlx + C * nly);
                    }
                }
            }
        }
    }
    const int contact = (int)__ballot_sync(kFull, touching);   // lane index == link index
    TRL_CLK_END(PH_CONTACT, clk);

    // ---- articulated-body forward dynamics over the chain schedule
    // one-sided implicit spring-damper at the joint limits (branch-free: the range of a free joint is infinite)
    const double viol = fmax(e.q - lc.lim_hi, 0.0) + fmin(e.q - lc.lim_lo, 0.0);
    const double cl = (viol != 0.0) ? pp.d_lim + dt * pp.k_lim : 0.0;
#if TRL_PHYS_TABLE
    // the FMA the builds reading c_model.phys make of k_lim * viol + cl * qd, spelled out: with the parameters in a register-indexed
    // table the compiler fuses the other product, which rounds differently
    const double lim_f = __fma_rn(viol, pp.k_lim, cl * e.qd);
#else
    const double lim_f = pp.k_lim * viol + cl * e.qd;
#endif
    double* slot = xs + X_LNK + lane * kLinkStride;
    if (lc.act) {
        store_vals(slot, ia);
        slot[LK_TAU] = e.tau;
        *trl_as2<double2>(slot + LK_CV) = make_double2(cvx, cvy);
        *trl_as2<double2>(slot + LK_S) = make_double2(k.ry, -k.rx);
        *trl_as2<double2>(slot + LK_LIM) = make_double2(lim_f, cl);
    }
    const double thd0 = shf(e.qd, 0);
    __syncwarp();
    TRL_CLK_END(PH_INWARD, clk);
    double a0, a1, a2;
    chain_aba(xs, chain_of(lc), lane, dt, a0, a1, a2 TRL_CLK_ARG(PH_INWARD, PH_OUTWARD));
    // each link lane integrates its own joint (semi-implicit Euler)
    if (lc.act && lane > 0) {
        e.qd += dt * slot[LK_QDD];
        e.q += dt * e.qd;
    }
    {
        // root: classical acceleration of the origin = spatial acceleration + w x v
        double xdd = a1 - thd0 * e.oyd, ydd = a2 + thd0 * e.oxd;
        e.oxd += dt * xdd; e.oyd += dt * ydd;
        e.ox += dt * e.oxd; e.oy += dt * e.oyd;
        if (lane == 0) { e.qd += dt * a0; e.q += dt * e.qd; }
    }
    TRL_CLK_RESET(clk);
    return contact;
}

// cTerrainRLCharController::ParseGround + BuildPoliState (sim/TerrainRLCharController.cpp:168-285), cooperative
__device__ void build_poli_state(const LinkC& lc, const EnvRegs& e, const Kin& k, const Buffers& B, const GroundView& g, int env,
                                 int lane, int stance) {
    const ModelConst& m = c_model;
    double* out = B.poli_state + (size_t)env * B.S;
    const double oy = g.sample(e.ox);
    for (int i = lane; i < kNumGroundSamples; i += kWarp) {
        double dist = ((10.0 - (-0.5)) * i) / (kNumGroundSamples - 1) + (-0.5);
        out[i] = g.sample(dist + e.ox) - oy;
    }
    if (lane == 0) out[kNumGroundSamples] = e.oy - oy;
    if (lc.act) {
        // raptor: when the left leg is the stance leg the two legs' entries are swapped
        // (cRaptorController::FlipPoliPoseStance, sim/RaptorController.cpp:1414-1432,1469-1487)
        int slot = lane;
        if (TRL_IS_RAPTOR(m) && stance != 0 && lane >= rRightHip) slot = lane < rLeftHip ? lane + 4 : lane - 4;
        if (lane > 0) {
            out[kNumGroundSamples + 1 + 2 * (slot - 1)] = k.cx;       // body COM relative to the root joint position
            out[kNumGroundSamples + 1 + 2 * (slot - 1) + 1] = k.cy;
        }
        int vo = kNumGroundSamples + 2 * m.nj - 1;
        out[vo + 2 * slot] = k.vx - k.w * k.cy;                       // body COM velocity
        out[vo + 2 * slot + 1] = k.vy + k.w * k.cx;
    }
}

// cScenarioSimChar::Reset (+ PoliEval / Exp specifics): scenarios/ScenarioSimChar.cpp:121-132.  Cooperative kinematics,
// scalar bookkeeping + terrain generation on lane 0.
__device__ void reset_env(Lane& L, const LinkC& lc, EnvRegs& e, const Buffers& B, int lane TRL_RESET_XS_DECL TRL_BS_DECL) {
    const ModelConst& m = c_model;
#if TRL_BODY_TABLE
    // the PD targets no gait state sets keep the TargetTheta of the episode's body (the others are set by apply_action below)
    if (lc.act) L.d(D_PD_TARGET + lane) = BL(target_theta0, lane);
    __syncwarp();
#endif
    e.q = lc.act ? m.pose0[lane == 0 ? 2 : lane + 2] : 0.0;
    e.qd = lc.act ? m.vel0[lane == 0 ? 2 : lane + 2] : 0.0;
    e.ox = m.pose0[0]; e.oy = m.pose0[1]; e.oxd = m.vel0[0]; e.oyd = m.vel0[1];
    e.tau = 0.0;
    Kin k = kinematics(lc, e TRL_KIN_XS_ARG);
    double comx = e.ox + warp_sum_all(lc.mass * k.cx) / BM(total_mass);
    double comy = e.oy + warp_sum_all(lc.mass * k.cy) / BM(total_mass);
    double newx = e.ox, newy = e.oy;
    if (lane == 0) {
        L.i(I_CONTACT) = 0;
        CounterRng rng = load_rng(L);
        // controller reset: default action, FSM state 0, counters zeroed (sim/TerrainRLCharController.cpp:47-58,
        // sim/DogController.cpp:210-216,640-650)
        double params[kNumParams];
        L.i(I_STANCE) = 0;   // cRaptorController::Reset -> SetStance(gDefaultStance)
        int id = build_base_action(L, rng, m.default_action, params);
        apply_action(L, id, params, comx, comy);
        L.i(I_EXP_FLAGS) = 0;
        L.i(I_FIRST_CYCLE) = 1;
        L.d(D_PREV_CYCLE_T) = 0.0; L.d(D_CUR_CYCLE_T) = 0.0; L.d(D_PREV_STUMBLE) = 0.0; L.d(D_CUR_STUMBLE) = 0.0;
        L.d(D_PREV_DIST_X) = 0.0; L.d(D_PREV_DIST_Y) = 0.0;
        L.d(D_PREV_COM_X) = comx; L.d(D_PREV_COM_Y) = comy;
        L.i(I_CMD) = -1;
        L.i(I_PENDING) = 0;
        // cSimCharSoftFall::Reset
        L.d(D_FALL_DIST_CNT) = 5.0; L.d(D_PREV_CHECK_X) = e.ox; L.d(D_PREV_CHECK_Y) = e.oy;
        L.i(I_FAIL_FALL_DIST) = 0; L.d(D_FALL_CONTACT_CNT) = 0.1; L.d(D_SUM_FALL) = 0.0;
        // ResetGround + InitCharacterPos
        int slot = 0;
        if constexpr (kTerrainSlots) {      // the terrain slot assigned to the env (trl_set_env_terrain) becomes its current one
            slot = L.I[(size_t)I_TERRAIN_SLOT_NEXT * L.n + L.env];
            L.I[(size_t)I_TERRAIN_SLOT * L.n + L.env] = slot;
        }
#if TRL_PHYS_TABLE
        if (c_env_phys) c_env_phys[L.env] = c_env_phys[(size_t)L.n + L.env];   // likewise the physics slot (trl_set_env_physics)
#if TRL_BODY_TABLE
        if (c_env_phys && ((c_phys_ranged >> c_env_phys[L.env]) & 1u)) draw_phys(L, c_env_phys[L.env]);   // a ranged one draws
#endif
        if (c_env_eval) {       // and the mode (trl_set_env_eval): evaluation counts cycles over episodes, from 0 when it begins
            const int next = c_env_eval[(size_t)L.n + L.env];
            if (next && !c_env_eval[L.env]) L.i(I_CYCLE_COUNT) = 0;
            c_env_eval[L.env] = next;
        }
#endif
        GroundView g = load_ground(L, B);
        g.n[0] = g.n[1] = 0; g.flip = 0;
        if constexpr (kTerrainSlots) g.update(-11.0, 9.0, c_terrain[slot].type, c_terrain[slot].params, 20.0);
        else g.update(-11.0, 9.0, m.terrain_type, m.terrain_params, 20.0);
        if (m.has_init_x) newx = m.init_x;
        newy = e.oy + g.sample(newx);
        store_ground(L, g);
        if (env_explores(L.env)) {
            L.i(I_CYCLE_COUNT) = 0;
            L.i(I_CMD) = rng.rand_int(0, m.n_actions);   // cScenarioExp::CommandRandAction
        } else {
            L.d(D_POS_START_X) = newx;
        }
        store_rng(L, rng);
    }
    __syncwarp();
    e.ox = shf(newx, 0); e.oy = shf(newy, 0);
}

__device__ __forceinline__ void load_env(Lane& L, const LinkC& lc, EnvRegs& e, int lane) {
    const int dq = (lane == 0) ? 2 : lane + 2;
    e.q = lc.act ? L.d(D_Q + dq) : 0.0;
    e.qd = lc.act ? L.d(D_QD + dq) : 0.0;
    e.tau = (lc.act && lane > 0) ? L.d(D_TAU + dq) : 0.0;
    e.ox = L.d(D_Q); e.oy = L.d(D_Q + 1); e.oxd = L.d(D_QD); e.oyd = L.d(D_QD + 1);
}
__device__ __forceinline__ void store_env(Lane& L, const LinkC& lc, const EnvRegs& e, int lane) {
    const int dq = (lane == 0) ? 2 : lane + 2;
    if (lc.act) { L.d(D_Q + dq) = e.q; L.d(D_QD + dq) = e.qd; L.d(D_TAU + dq) = (lane > 0) ? e.tau : 0.0; }
    if (lane == 0) {
        L.d(D_Q) = e.ox; L.d(D_Q + 1) = e.oy; L.d(D_QD) = e.oxd; L.d(D_QD + 1) = e.oyd;
        L.d(D_TAU) = 0.0; L.d(D_TAU + 1) = 0.0;
    }
}

// ================================================================================================ the kernel
// flags: bit0 do_ctrl (finish env-step k), bit1 do_phys (start env-step k+1), bit2 end of outer update
// Catch-up launch bookkeeping: every warp calls this once when it is done; the last one of the grid re-arms the consumed list.
__device__ __forceinline__ void catchup_leave(const Buffers& B, int prev) {
    __syncwarp();
    if ((threadIdx.x & 31) == 0) {
        __threadfence();
        const int total = (int)gridDim.x * kWarpsPerBlock;
        // one counter per list: the catch-up launches of two consecutive env-steps can be in flight at the same time
        if (atomicAdd(&B.catchup_done[prev], 1) == total - 1) { B.pending_count[prev] = 0; B.catchup_done[prev] = 0; __threadfence(); }
    }
}

__global__ void __launch_bounds__(kBlockThreads, TRL_STEP_MIN_BLOCKS)
trl_step_kernel(Buffers B, double h, int flags, int lists) {
#if TRL_BODY_TABLE
    // one copy of the link, corner and box tables per warp, staged below with its env's body, and of the env's physics
    __shared__ double s_clx_w[kWarpsPerBlock][4 * kMaxJoints + 6 * kMaxJoints], s_cly_w[kWarpsPerBlock][4 * kMaxJoints];
    __shared__ LinkTables s_link_w[kWarpsPerBlock];
    __shared__ PhysParams s_pp_w[kWarpsPerBlock];
#else
    __shared__ double s_clx[4 * kMaxJoints + 6 * kMaxJoints], s_cly[4 * kMaxJoints];     // s_clx also carries the six per-body box tables
#endif
    __shared__ __align__(16) double s_x[kWarpsPerBlock * X_END];
    TRL_CLK_BEGIN(clk);
    const ModelConst& m = c_model;
#if !TRL_BODY_TABLE
    for (int t = threadIdx.x; t < m.n_corners; t += kBlockThreads) {
        s_clx[t] = LT(corner_lx, t); s_cly[t] = LT(corner_ly, t);
    }
    for (int t = threadIdx.x; t < m.nj; t += kBlockThreads) {
        double* tb = s_clx + 4 * kMaxJoints;
        tb[t] = LT(body_ax, t); tb[kMaxJoints + t] = LT(body_ay, t); tb[2 * kMaxJoints + t] = LT(body_cos, t); tb[3 * kMaxJoints + t] = LT(body_sin, t);
        tb[4 * kMaxJoints + t] = LT(half_x, t); tb[5 * kMaxJoints + t] = LT(half_y, t);
    }
    TRL_LINK_TABLES_DECL
#endif
#if TRL_FIELD_SMEM
    static_assert(I_NUM_FIELDS <= kWarp, "one lane per i32 field");
    __shared__ double s_fd[kWarpsPerBlock * D_NUM_FIELDS];
    __shared__ int s_fi[kWarpsPerBlock * I_NUM_FIELDS];
#endif
#if !TRL_BODY_TABLE
    stage_link_tables(link_tabs);
    __syncthreads();
#endif
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#if TRL_BODY_TABLE
    double* const s_clx = s_clx_w[warp];
    double* const s_cly = s_cly_w[warp];
    LinkTables* const link_tabs = &s_link_w[warp];
#endif
    // pending-decision lists (lag + 1 of them, used round robin by successive env-steps): envs that reach a cycle boundary in this
    // launch are appended to list `app`; an env's I_PENDING tag is 1 + the list it was last appended to.  The decision of a list is
    // made on a side stream and its envs are then caught up over `lag` env-steps by a side launch (trl_host.cu: enqueue_update), so
    // the main launch of step j skips every tagged env except those of list j % (lag + 1), whose tag is lag + 1 steps old.
    const int app = lists & 7, prev = (lists >> 3) & 7;

    int env = blockIdx.x * kWarpsPerBlock + warp;
    int env_end = B.n;
    {
        // env groups (trl_host.cu: enqueue_update): a main launch covers group g of G contiguous env ranges, each on its own stream,
        // so that the tail of one group's launch is filled by the next group's CTAs instead of leaving SM slots idle
        const int G = (lists >> 14) & 15;
        if (G > 1) {
            const int chunk = group_chunk(B.n, G);
            env += ((lists >> 10) & 15) * chunk;
            env_end = min(B.n, (((lists >> 10) & 15) + 1) * chunk);
        }
    }
    if (flags & kStepCatchUp) {
        // catch-up launch: one warp per entry of list `prev`, after the decision kernel has served it.
        // The last CTA to leave re-arms that list (the main launch three steps later appends to it again).
        const int count = B.pending_count[prev];
        if (env >= count) { catchup_leave(B, prev); return; }
        env = B.pending_list[prev * B.n + env];
    } else if (env >= env_end) {
        return;
    }
    Lane L{nullptr, env, B.n, B.d, B.i};
    int tag = 0;
    if (flags & kStepSkipPending) {
        // overlapped main launch: envs waiting for a decision or being caught up are not touched
        tag = L.i(I_PENDING);
        if (tag != 0 && tag != 1 + app) return;
    }
#if TRL_FIELD_SMEM
    // every field of this env in one batch of independent loads (the planes are B.n apart: a field costs an L2 round trip wherever it
    // is first touched); the env is private to this warp for the whole launch, so the copy is written back in one batch at the end
    {
        double* sd = s_fd + warp * D_NUM_FIELDS;
        int* si = s_fi + warp * I_NUM_FIELDS;
        for (int f = lane; f < D_NUM_FIELDS; f += kWarp) sd[f] = L.D[(size_t)f * L.n + env];
        if (lane < I_NUM_FIELDS) si[lane] = L.I[(size_t)lane * L.n + env];
        __syncwarp();
        L.sd = sd; L.si = si;
    }
#endif
    if (flags & kStepSkipPending) {
        if (tag == 1 + app && lane == 0) L.i(I_PENDING) = 0;   // stale tag of lag + 1 steps ago (already caught up)
    } else if (!(flags & kStepCatchUp) && (flags & 1) && lane == 0) {
        L.i(I_PENDING) = 0;    // serial schedule / end of the update: every decision has been served before this launch
    }
    double* xs = s_x + warp * X_END;
#if TRL_BODY_TABLE
    const BodyConst* bb = env_body(c_env_body ? c_env_body[env] : 0, env);   // the env's present body; an episode reset below may change it
    stage_body(link_tabs, s_clx, s_cly, lane, bb);
#endif
    const LinkC lc = load_link(lane, link_tabs);
    EnvRegs e;
    load_env(L, lc, e, lane);
    int contact = L.i(I_CONTACT);
    TRL_CLK_END(PH_LOAD, clk);

#if TRL_REUSE_KIN
    Kin k_ctrl;
    bool have_k = false;       // warp-uniform: the controller half ran and nothing has moved the state since
#endif
#ifdef TRL_CG_VARIANT
    const int reps = max(1, (lists >> 6) & 15);        // a catch-up launch advances its envs by several env-steps (registers stay live)
#else
    constexpr int reps = 1;                            // catch-up launches are the other build of this file (trl_step_cg.cu)
#endif
    for (int rep = 0; rep < reps; ++rep) {
    if (flags & 1) {
        // ---------------- controller half of env-step k
        Kin k = kinematics(lc, e TRL_KIN_XS_ARG);
#if TRL_REUSE_KIN
        k_ctrl = k; have_k = true;
#endif
        TRL_CLK_END(PH_KIN, clk);
        e.tau = controller_torque(L, lc, e, k, xs, lane, h, contact TRL_BS_ARG);
        TRL_CLK_RESET(clk);
        if (lane == 0) {
            // fall checks (sim/SimCharSoftFall.cpp:74-125)
            double cnt = L.d(D_FALL_DIST_CNT) - h;
            if (cnt <= 0.0) {
                double dx = e.ox - L.d(D_PREV_CHECK_X), dy = e.oy - L.d(D_PREV_CHECK_Y);
                if (dx * dx + dy * dy < 0.25) L.i(I_FAIL_FALL_DIST) = 1;
                L.d(D_PREV_CHECK_X) = e.ox; L.d(D_PREV_CHECK_Y) = e.oy;
                cnt = 5.0;
            }
            L.d(D_FALL_DIST_CNT) = cnt;
            double cc = L.d(D_FALL_CONTACT_CNT) - h;
            if (cc <= 0.0) {
                double val = ((unsigned)contact & m.fall_mask) ? 1.0 : 0.0;
                const double norm = (1.0 + 1.0 / (1.0 - 0.9));
                L.d(D_SUM_FALL) = val / norm + 0.9 * L.d(D_SUM_FALL);
                cc = 0.1;
            }
            L.d(D_FALL_CONTACT_CNT) = cc;
            unsigned lo = (unsigned)L.i(I_STEPS_LO) + 1u;
            L.i(I_STEPS_LO) = (int)lo;
            if (lo == 0u) L.i(I_STEPS_HI) += 1;
        }
        __syncwarp();
        // PostSubstepUpdate: cycle boundary bookkeeping
        int nc = 0, fl = 0;
        if (lane == 0) { nc = (L.i(I_STATE) == 0 && L.d(D_PHASE) == 0.0) ? 1 : 0; fl = has_fallen(L, e.q) ? 1 : 0; }
        nc = shfi(nc, 0); fl = shfi(fl, 0);
        if (nc) {
            if (env_explores(env)) exp_new_cycle_update(L, B, fl != 0, lane);
            else if (lane == 0) L.i(I_CYCLE_COUNT) += 1;
        }
        TRL_CLK_END(PH_CTRL_REST, clk);
    }

    if (flags & 4) {
        // ---------------- end of the outer update: fall -> episode bookkeeping + reset
        int fallen = 0, new_cycle = 0;
        if (lane == 0) { fallen = has_fallen(L, e.q) ? 1 : 0; new_cycle = (L.i(I_STATE) == 0 && L.d(D_PHASE) == 0.0) ? 1 : 0; }
        fallen = shfi(fallen, 0); new_cycle = shfi(new_cycle, 0);
        bool do_reset = false;
        if (env_explores(env)) {     // the ending episode's own mode: reset_env then gives the next one its assigned mode
            if (!new_cycle && fallen) { exp_new_cycle_update(L, B, true, lane); do_reset = true; }
        } else if (fallen) {
            if (lane == 0 && L.i(I_CYCLE_COUNT) >= 1) {
                double dist = e.ox - L.d(D_POS_START_X);
                int ec = L.i(I_EPISODE_COUNT);
                L.d(D_AVG_DIST) = (ec * L.d(D_AVG_DIST) + dist) / (ec + 1.0);
                L.i(I_EPISODE_COUNT) = ec + 1;
                int slot = atomicAdd(B.dist_count, 1);
                if (slot < B.dist_cap) { B.dist_log[slot] = dist; B.dist_env[slot] = env; }
            }
            do_reset = true;
        }
        if (do_reset) {
#if TRL_BODY_TABLE
            bb = begin_body(L, link_tabs, s_clx, s_cly, lane);   // lc reads the warp's tables, which now hold the new episode's body
#endif
            reset_env(L, lc, e, B, lane TRL_RESET_XS_ARG TRL_BS_ARG); contact = 0;
#if TRL_REUSE_KIN
            have_k = false;
#endif
        }
    }

    if (flags & 2) {
        // ---------------- physics half of env-step k+1
#if TRL_PHASE_CLOCKS
        if (lane == 0) atomicAdd(&g_phase_clocks[kNumPhases], 1ull);
#endif
        TRL_CLK_END(PH_TAIL, clk);
        GroundView g = load_ground(L, B);
        const int ns = m.num_sim_substeps;
        const double dt = h / ns;
        // terrain maximum over the window the character's corners can reach during this env-step; kClearMargin covers the
        // contact tolerance measured along the surface normal on (near-)vertical cliff faces and the root's travel
        const double clear_y = g.window_max(e.ox - BM(reach) - 0.25, e.ox + BM(reach) + 0.25, lane) + kClearMargin;
#if TRL_PHYS_TABLE
        // the slot of the env's present episode (a reset above has already made its assignment current)
        const int ps = c_env_phys ? c_env_phys[env] : 0;
#endif
#if TRL_BODY_TABLE
        if (lane == 0) s_pp_w[warp] = ((c_phys_ranged >> ps) & 1u) ? c_env_pdraw[env] : c_phys[ps];
        __syncwarp();
#endif
#if TRL_REUSE_KIN
        for (int s = 0; s < ns; ++s)
            contact = physics_substep(lc, e, g, s_clx, s_cly, lane, dt, clear_y, xs, (s == 0 && have_k) ? &k_ctrl : nullptr TRL_PS_ARG);
#else
        for (int s = 0; s < ns; ++s) contact = physics_substep(lc, e, g, s_clx, s_cly, lane, dt, clear_y, xs TRL_PS_ARG);
#endif
        TRL_CLK_RESET(clk);
        // UpdateGround (scenarios/ScenarioSimChar.cpp:564-572): regenerate a segment when the view window crosses it
        {
            int smin = g.seg_id(0), smax = g.seg_id(1);
            double bmin = e.ox - 2.0, bmax = e.ox + 10.0 + 1.0;
            bool need = !(bmax < g.seg_max_x(smax) && bmin > g.seg_min_x(smin));
            if (need) {
                if (lane == 0) {
                    if constexpr (kTerrainSlots) { const TerrainSlot& ts = env_terrain(L); g.update(bmin, bmax, ts.type, ts.params, 20.0); }
                    else g.update(bmin, bmax, m.terrain_type, m.terrain_params, 20.0);
                    store_ground(L, g);
                }
                __syncwarp();
                g = load_ground(L, B);
            }
        }
        // head of cDogController::Update: cycle timers, stumble counter, gait FSM (lane 0)
        int end_step = 0;
        if (lane == 0) {
            L.i(I_CONTACT) = contact;
            L.d(D_CUR_CYCLE_T) += h;
            if ((unsigned)contact & m.stumble_mask) L.d(D_CUR_STUMBLE) += h;
            int state = L.i(I_STATE);
            int first = L.i(I_FIRST_CYCLE);
            double phase = L.d(D_PHASE) + h / L.d(D_PARAMS + mTransTime);
            bool advance = first != 0;
            int ns2;
            if (TRL_IS_RAPTOR(m)) {
                // cRaptorController::UpdateState (sim/RaptorController.cpp:804-849): Contact, Down, Passing are timed,
                // Up ends when the swing toe touches down; the stance flips at the end of every cycle but the first
                const int sw_toe = (L.i(I_STANCE) == 0 ? rLeftHip : rRightHip) + 3;
                if (state != rsUp && phase >= 1.0) advance = true;
                if (state == rsUp && ((contact >> sw_toe) & 1)) advance = true;
                ns2 = first ? rsContact : (state == rsUp ? -1 : state + 1);
            } else {
                if ((state == sBackStance || state == sFrontStance) && phase >= 1.0) advance = true;
                if (state == sExtend && ((contact >> jFinger) & 1)) advance = true;
                if (state == sGather && ((contact >> jToe) & 1)) advance = true;
                ns2 = first ? sBackStance : (state == sGather ? -1 : state + 1);
            }
            L.d(D_PHASE) = phase;
            if (advance) {
                if ((ns2 < 0) || first) {
                    end_step = 1;
                    if (TRL_IS_RAPTOR(m) && !first) L.i(I_STANCE) = 1 - L.i(I_STANCE);   // FlipStance
                } else { L.i(I_STATE) = ns2; L.d(D_PHASE) = 0.0; set_state_params(L, ns2); }
            }
        }
        end_step = shfi(end_step, 0);
        __syncwarp();
        if (end_step) {
            // cycle boundary: build the policy state and hand the env to the decision kernel
            Kin k = kinematics(lc, e TRL_KIN_XS_ARG);
            build_poli_state(lc, e, k, B, g, env, lane, TRL_IS_RAPTOR(m) ? L.i(I_STANCE) : 0);
            double comx = e.ox + warp_sum_all(lc.mass * k.cx) / BM(total_mass);
            double comy = e.oy + warp_sum_all(lc.mass * k.cy) / BM(total_mass);
            if (lane == 0) {
                B.com_stash[env] = comx; B.com_stash[B.n + env] = comy;
                L.i(I_FIRST_CYCLE) = 0;
                if (flags & kStepCatchUp) {
                    // a gait cycle shorter than the catch-up depth (the shipped controllers' timed states alone last 150 env-steps): the side
                    // launch cannot hand the env to a decision in time -- flag it (trl_sync reports; TRL_SERIAL_SCHEDULE=1 runs it)
                    B.catchup_done[kMaxLists] = 1;
                }
                L.i(I_PENDING) = 1 + app;
                int slot = atomicAdd(&B.pending_count[app], 1);
                B.pending_list[app * B.n + slot] = env;
            }
        }
        TRL_CLK_END(PH_TAIL, clk);
    }
    }   // rep
    store_env(L, lc, e, lane);
#if TRL_FIELD_SMEM
    __syncwarp();
    for (int f = lane; f < D_NUM_FIELDS; f += kWarp) L.D[(size_t)f * L.n + env] = L.sd[f];
    if (lane < I_NUM_FIELDS) L.I[(size_t)lane * L.n + env] = L.si[lane];
#endif
    TRL_CLK_END(PH_LOAD, clk);
    if (flags & kStepCatchUp) catchup_leave(B, prev);
}

// Initial reset of every env (trl_create / trl_reset): seeds the terrain RNG and runs the episode reset.
__global__ void __launch_bounds__(kBlockThreads)
trl_reset_kernel(Buffers B, const uint64_t* terrain_seeds, const int* env_ids, int count, int reseed) {
#if TRL_BODY_TABLE
    __shared__ LinkTables s_link_w[kWarpsPerBlock];     // staged per warp with the body of the episode the reset starts (below)
    LinkTables* const link_tabs = &s_link_w[threadIdx.x >> 5];
#else
    TRL_LINK_TABLES_DECL
#if TRL_LINK_SMEM
    stage_link_tables(link_tabs);
    __syncthreads();
#endif
#endif
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int idx = blockIdx.x * kWarpsPerBlock + warp;
    if (idx >= count) return;
    const int env = env_ids ? env_ids[idx] : idx;
    Lane L{nullptr, env, B.n, B.d, B.i};
    const ModelConst& m = c_model;
    if (reseed && lane == 0) {
        uint64_t seed = terrain_seeds ? terrain_seeds[idx] : (uint64_t)(1 + env);
        L.i(I_TERRAIN_RNG) = (int)TerrainRng::seed_state(seed);
        L.i(I_RNG_CTR_LO) = 0; L.i(I_RNG_CTR_HI) = 0;
        L.i(I_CYCLE_COUNT) = 0; L.i(I_EPISODE_COUNT) = 0; L.d(D_AVG_DIST) = 0.0; L.d(D_POS_START_X) = 0.0;
        L.i(I_STEPS_LO) = 0; L.i(I_STEPS_HI) = 0; L.i(I_TUPLE_FLAGS) = 0;
        L.i(I_SEG_N0) = 0; L.i(I_SEG_N1) = 0; L.i(I_SEG_FLIP) = 0; L.d(D_SEG_MINX0) = 0.0; L.d(D_SEG_MINX1) = 0.0;
        for (int j = 0; j < m.nj; ++j) L.d(D_PD_TARGET + j) = m.target_theta0[j];
        for (int k = 0; k < kNumParams; ++k) L.d(D_PARAMS + k) = 0.0;
        L.d(D_CUR_CYCLE_T) = 0.0; L.d(D_CUR_STUMBLE) = 0.0; L.d(D_PREV_COM_X) = 0.0; L.d(D_PREV_COM_Y) = 0.0;
    }
    __syncwarp();
#if TRL_BODY_TABLE
    const BodyConst* const bb = begin_body(L, link_tabs, nullptr, nullptr, lane);
#endif
    const LinkC lc = load_link(lane, link_tabs);
    EnvRegs e;
#if TRL_KIN_SMEM
    __shared__ __align__(16) double s_pfx[kWarpsPerBlock * 3 * 2 * kWarp];
    double* xs = s_pfx + warp * 3 * 2 * kWarp - X_PFX;    // kinematics() only touches [X_PFX, X_PFX_END)
#endif
    reset_env(L, lc, e, B, lane TRL_RESET_XS_ARG TRL_BS_ARG);
    store_env(L, lc, e, lane);
}

// Terrain look-ahead: regenerates, ahead of the step kernels of the coming outer update, the segment of every env
// whose view window [x-2, x+11] will cross the end of its terrain during that update (look-ahead 0.5 m >> the distance
// covered in 1/30 s).  cGroundVar2D::Update's result does not depend on *when* it runs (segment bounds, joint height
// and the generator stream are functions of the previous segment only, sim/GroundVar2D.cpp:43-91), so the terrain is
// bit-identical to generating it at the exact step; doing it here keeps the serial generator off the critical path
// of the 21 step launches (it used to stall one warp for each regeneration).
__global__ void trl_terrain_kernel(Buffers B, double lookahead) {
    const int env = blockIdx.x * blockDim.x + threadIdx.x;
    if (env >= B.n) return;
    Lane L{nullptr, env, B.n, B.d, B.i};
    const double x = L.d(D_Q);
    GroundView g = load_ground(L, B);
    const int smin = g.seg_id(0), smax = g.seg_id(1);
    const double bmin = x - 2.0, bmax = x + 10.0 + 1.0 + lookahead;
    if (bmax < g.seg_max_x(smax) && bmin > g.seg_min_x(smin)) return;
    if constexpr (kTerrainSlots) {
        const TerrainSlot& ts = env_terrain(L);
        g.update(bmin, bmax, ts.type, ts.params, 20.0);
    } else {
        g.update(bmin, bmax, c_model.terrain_type, c_model.terrain_params, 20.0);
    }
    store_ground(L, g);
}
void launch_terrain(const Buffers& B, double lookahead, cudaStream_t st) {
    TRL_LAUNCH(trl_terrain_kernel, (B.n + 127) / 128, 128, 0, st, B, lookahead);
}

// Batch statistics (cOptScenarioPoliEval::OutputResults merges the same counters under a mutex): one block reduces
// cycles / episodes / env-steps / episode-weighted distance into out[4] (doubles).
__global__ void trl_stats_kernel(Buffers B, double* out) {
    __shared__ double red[4][32];
    double c = 0, e = 0, st = 0, ds = 0;
    for (int env = threadIdx.x; env < B.n; env += blockDim.x) {
        int ec = B.i[(size_t)I_EPISODE_COUNT * B.n + env];
        c += B.i[(size_t)I_CYCLE_COUNT * B.n + env];
        e += ec;
        st += (double)(((uint64_t)(uint32_t)B.i[(size_t)I_STEPS_HI * B.n + env] << 32) | (uint32_t)B.i[(size_t)I_STEPS_LO * B.n + env]);
        ds += B.d[(size_t)D_AVG_DIST * B.n + env] * ec;
    }
    c = warp_sum_all(c); e = warp_sum_all(e); st = warp_sum_all(st); ds = warp_sum_all(ds);
    int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    if (l == 0) { red[0][w] = c; red[1][w] = e; red[2][w] = st; red[3][w] = ds; }
    __syncthreads();
    if (w == 0) {
        int nw = blockDim.x >> 5;
        for (int k = 0; k < 4; ++k) {
            double v = l < nw ? red[k][l] : 0.0;
            v = warp_sum_all(v);
            if (l == 0) out[k] = v;
        }
    }
}
void launch_stats(const Buffers& B, double* out, cudaStream_t st) { TRL_LAUNCH(trl_stats_kernel, 1, 1024, 0, st, B, out); }

// ---- host-side launch helpers (called from trl_host.cu)
cudaError_t upload_model(const ModelConst& mc, const TerrainSlot* terrain) {
    cudaError_t e = cudaMemcpyToSymbol(c_model, &mc, sizeof(ModelConst));
    if (e == cudaSuccess) e = cudaMemcpyToSymbol(c_terrain, terrain, sizeof(TerrainSlot) * kMaxTerrainSlots);
#if TRL_TABLE_MIRROR
    if (e == cudaSuccess) e = cudaMemcpyToSymbol(g_model, &mc, sizeof(ModelConst));
#endif
    return e;
}
#if TRL_PHYS_TABLE
// the physics table (slot 0 = mc.phys), the handle's per-env slot array (null: every env on slot 0) and per-env mode array (null: every
// env in the handle's mode), uploaded with the model
cudaError_t upload_phys(const PhysParams* phys, int* env_phys, int* env_eval) {
    cudaError_t e = cudaMemcpyToSymbol(c_phys, phys, sizeof(PhysParams) * kMaxPhysSlots);
    if (e == cudaSuccess) e = cudaMemcpyToSymbol(c_env_phys, &env_phys, sizeof(env_phys));
    if (e == cudaSuccess) e = cudaMemcpyToSymbol(c_env_eval, &env_eval, sizeof(env_eval));
    return e;
}
#endif
#if TRL_BODY_TABLE
// the body table (slot 0 = the scene's body) and the handle's per-env slot array (null: every env on slot 0), uploaded with the model
cudaError_t upload_body(const BodyConst* body, int* env_body) {
    cudaError_t e = cudaMemcpyToSymbol(g_body, body, sizeof(BodyConst) * kMaxBodySlots);
    if (e == cudaSuccess) e = cudaMemcpyToSymbol(c_env_body, &env_body, sizeof(env_body));
    return e;
}
// the ranged slots (masks, hi tables) and the handle's per-env draw tables (null: the handle has no ranged slot), uploaded with the model
cudaError_t upload_ranges(const RangeTables& r) {
    cudaError_t e = cudaMemcpyToSymbol(g_body_hi, r.body_hi, sizeof(BodyConst) * kMaxBodySlots);
    if (e == cudaSuccess) e = cudaMemcpyToSymbol(c_phys_hi, r.phys_hi, sizeof(PhysParams) * kMaxPhysSlots);
    if (e == cudaSuccess) e = cudaMemcpyToSymbol(c_body_ranged, &r.body_ranged, sizeof(unsigned));
    if (e == cudaSuccess) e = cudaMemcpyToSymbol(c_phys_ranged, &r.phys_ranged, sizeof(unsigned));
    if (e == cudaSuccess) e = cudaMemcpyToSymbol(c_env_bdraw, &r.env_bdraw, sizeof(r.env_bdraw));
    if (e == cudaSuccess) e = cudaMemcpyToSymbol(c_env_pdraw, &r.env_pdraw, sizeof(r.env_pdraw));
    if (e == cudaSuccess) e = cudaMemcpyToSymbol(c_env_draws, &r.env_draws, sizeof(r.env_draws));
    return e;
}
#elif defined(TRL_SIMT_EMU)
// the emulator's TRL_LINK_SMEM=0 experiment build has no body slots: a handle with one is refused
cudaError_t upload_body(const BodyConst*, int* env_body) { return env_body ? static_cast<cudaError_t>(1) : cudaSuccess; }
cudaError_t upload_ranges(const RangeTables& r) { return r.env_draws ? static_cast<cudaError_t>(1) : cudaSuccess; }
#endif
size_t step_smem_bytes() { return 0; }
// TRL_PHASE_CLOCKS builds: copy the accumulated phase clocks (kNumPhases + the env-step count) into out[], optionally zero them
cudaError_t step_phase_clocks(unsigned long long* out, int reset) {
#if TRL_PHASE_CLOCKS
    cudaError_t e = cudaMemcpyFromSymbol(out, g_phase_clocks, sizeof(g_phase_clocks));
    if (e == cudaSuccess && reset) {
        const unsigned long long zero[kNumPhases + 1] = {};
        e = cudaMemcpyToSymbol(g_phase_clocks, zero, sizeof(zero));
    }
    return e;
#else
    (void)out; (void)reset;
    return static_cast<cudaError_t>(1);   // not a measurement build
#endif
}
cudaError_t configure_step_kernels() {
#if !defined(TRL_SIMT_EMU)
    // the per-warp link blocks take the CTA's static shared memory to ~25 KB: ask for a carve-out that holds the
    // TRL_STEP_MIN_BLOCKS CTAs per SM the register budget is sized for (+1 KB the system reserves per CTA), and no more (L1)
    cudaFuncAttributes fa;
    cudaError_t e = cudaFuncGetAttributes(&fa, trl_step_kernel);
    if (e != cudaSuccess) return e;
    const double need = (double)TRL_STEP_MIN_BLOCKS * (double)(fa.sharedSizeBytes + 1024);
    const int pct = std::min(100, (int)std::ceil(100.0 * need / (228.0 * 1024.0)));
    return cudaFuncSetAttribute(trl_step_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, pct);
#else
    return cudaSuccess;
#endif
}
void launch_step(const Buffers& B, double h, int flags, int lists, cudaStream_t st, int group, int n_groups) {
    int envs = B.n;
    if (n_groups > 1) {
        const int chunk = group_chunk(B.n, n_groups);
        envs = std::max(0, std::min(B.n, (group + 1) * chunk) - group * chunk);
        lists |= (group << 10) | (n_groups << 14);
        if (envs == 0) return;
    }
    int blocks = (envs + kWarpsPerBlock - 1) / kWarpsPerBlock;
    TRL_LAUNCH(trl_step_kernel, blocks, kBlockThreads, 0, st, B, h, flags, lists);
}
void launch_reset(const Buffers& B, const uint64_t* seeds, const int* env_ids, int count, int reseed, cudaStream_t st) {
    int blocks = (count + kWarpsPerBlock - 1) / kWarpsPerBlock;
    TRL_LAUNCH(trl_reset_kernel, blocks, kBlockThreads, 0, st, B, seeds, env_ids, count, reseed);
}

}  // namespace TRL_IMPL_NS

#if !defined(TRL_CG_VARIANT) && !defined(TRL_TERRAIN_SLOTS_VARIANT) && !defined(TRL_PHYS_SLOTS_VARIANT) && !defined(TRL_BODY_SLOTS_VARIANT)
#include "trl_decide.cuh"
#include "trl_decide2.cuh"
#endif
