// deepterrainrl_b200 -- host runtime behind the C ABI (include/terrainrl_b200.h).
// Owns device memory (plain cudaMalloc; no torch in the boundary), the CUDA stream, the captured CUDA graph of one
// outer update (21 step launches + 20 decision launches) and the pinned staging buffers for tuple / statistics reads.
#include <cuda_runtime.h>

#include <cmath>
#include <cstddef>
#include <type_traits>
#include <cstdio>
#include <cstring>
#include <map>
#include <string>
#include <algorithm>
#include <vector>

#include "../../include/terrainrl_b200.h"
#include "ref_loader.h"
#include "scene_pack.h"
#include "model_io.h"
#include "trl_types.h"
#include "trl_fcmaps.h"

namespace trl {
cudaError_t upload_model(const ModelConst& mc, const TerrainSlot* terrain);
size_t step_smem_bytes();
cudaError_t configure_step_kernels();
void launch_step(const Buffers& B, double h, int flags, int lists, cudaStream_t st, int group = 0, int n_groups = 1);
void launch_reset(const Buffers& B, const uint64_t* seeds, const int* env_ids, int count, int reseed, cudaStream_t st);
size_t decide_smem_bytes();
cudaError_t configure_decide_kernel();
void launch_decide(const Buffers& B, const NetWeights& W, const ExpSettings* ex, int* done_count, int grid, int list, int rearm,
                   cudaStream_t st);
void launch_stats(const Buffers& B, double* out, cudaStream_t st);
size_t decide_fc_smem_bytes();
cudaError_t configure_decide2_kernels();
void launch_decide2(const Buffers& B, const NetWeights& W, const ExpSettings* ex, const FcMaps& maps, double* act2, int* done_count, int grid,
                    int fc_clusters, int list, int rearm, cudaStream_t st, int part);
void launch_decide2_slots(const Buffers& B, const PolicySlots& P, const ExpSettings* ex, const FcMaps& maps, const FcSlotMaps& smaps, double* act2,
                          int* tmp, int* tab, int* done_count, int grid, int fc_clusters, int list, int rearm, cudaStream_t st, int part);
void launch_cell_stats(const Buffers& B, const int* env_slot, double* out, cudaStream_t st);
void launch_phys_stats(const Buffers& B, const int* env_slot, const int* env_phys, int policy_slot, int terrain_slot, int phys_slot,
                       const int* env_eval, int eval, const int* env_body, int body_slot, double* out, cudaStream_t st);
void launch_terrain(const Buffers& B, double lookahead, cudaStream_t st);
}  // namespace trl
namespace trl_cg {
cudaError_t upload_model(const trl::ModelConst& mc, const trl::TerrainSlot* terrain);
cudaError_t configure_step_kernels();
void launch_step(const trl::Buffers& B, double h, int flags, int lists, cudaStream_t st, int group = 0, int n_groups = 1);
}  // namespace trl_cg
// the terrain-slot builds of the env-step kernels (trl_step_ts.cu, trl_step_ts_cg.cu), the physics-slot builds (trl_step_ps.cu,
// trl_step_ps_cg.cu) and the body-slot builds (trl_step_bs.cu, trl_step_bs_cg.cu); the emulator's trl / trl_cg builds are all of those
#ifdef TRL_SIMT_EMU
namespace trl {
cudaError_t upload_phys(const PhysParams* phys, int* env_phys, int* env_eval);
cudaError_t upload_body(const BodyConst* body, int* env_body);
cudaError_t upload_ranges(const RangeTables& r);
}
namespace trl_cg {
cudaError_t upload_phys(const trl::PhysParams* phys, int* env_phys, int* env_eval);
cudaError_t upload_body(const trl::BodyConst* body, int* env_body);
cudaError_t upload_ranges(const trl::RangeTables& r);
}
namespace trl_ts = trl;
namespace trl_ts_cg = trl_cg;
namespace trl_ps = trl;
namespace trl_ps_cg = trl_cg;
namespace trl_bs = trl;
namespace trl_bs_cg = trl_cg;
#else
namespace trl_ts {
cudaError_t upload_model(const trl::ModelConst& mc, const trl::TerrainSlot* terrain);
cudaError_t configure_step_kernels();
void launch_step(const trl::Buffers& B, double h, int flags, int lists, cudaStream_t st, int group = 0, int n_groups = 1);
void launch_reset(const trl::Buffers& B, const uint64_t* seeds, const int* env_ids, int count, int reseed, cudaStream_t st);
void launch_terrain(const trl::Buffers& B, double lookahead, cudaStream_t st);
}  // namespace trl_ts
namespace trl_ts_cg {
cudaError_t upload_model(const trl::ModelConst& mc, const trl::TerrainSlot* terrain);
cudaError_t configure_step_kernels();
void launch_step(const trl::Buffers& B, double h, int flags, int lists, cudaStream_t st, int group = 0, int n_groups = 1);
}  // namespace trl_ts_cg
namespace trl_ps {
cudaError_t upload_model(const trl::ModelConst& mc, const trl::TerrainSlot* terrain);
cudaError_t upload_phys(const trl::PhysParams* phys, int* env_phys, int* env_eval);
cudaError_t configure_step_kernels();
void launch_step(const trl::Buffers& B, double h, int flags, int lists, cudaStream_t st, int group = 0, int n_groups = 1);
void launch_reset(const trl::Buffers& B, const uint64_t* seeds, const int* env_ids, int count, int reseed, cudaStream_t st);
void launch_terrain(const trl::Buffers& B, double lookahead, cudaStream_t st);
}  // namespace trl_ps
namespace trl_ps_cg {
cudaError_t upload_model(const trl::ModelConst& mc, const trl::TerrainSlot* terrain);
cudaError_t upload_phys(const trl::PhysParams* phys, int* env_phys, int* env_eval);
cudaError_t configure_step_kernels();
void launch_step(const trl::Buffers& B, double h, int flags, int lists, cudaStream_t st, int group = 0, int n_groups = 1);
}  // namespace trl_ps_cg
namespace trl_bs {
cudaError_t upload_model(const trl::ModelConst& mc, const trl::TerrainSlot* terrain);
cudaError_t upload_phys(const trl::PhysParams* phys, int* env_phys, int* env_eval);
cudaError_t upload_body(const trl::BodyConst* body, int* env_body);
cudaError_t upload_ranges(const trl::RangeTables& r);
cudaError_t configure_step_kernels();
void launch_step(const trl::Buffers& B, double h, int flags, int lists, cudaStream_t st, int group = 0, int n_groups = 1);
void launch_reset(const trl::Buffers& B, const uint64_t* seeds, const int* env_ids, int count, int reseed, cudaStream_t st);
void launch_terrain(const trl::Buffers& B, double lookahead, cudaStream_t st);
}  // namespace trl_bs
namespace trl_bs_cg {
cudaError_t upload_model(const trl::ModelConst& mc, const trl::TerrainSlot* terrain);
cudaError_t upload_phys(const trl::PhysParams* phys, int* env_phys, int* env_eval);
cudaError_t upload_body(const trl::BodyConst* body, int* env_body);
cudaError_t upload_ranges(const trl::RangeTables& r);
cudaError_t configure_step_kernels();
void launch_step(const trl::Buffers& B, double h, int flags, int lists, cudaStream_t st, int group = 0, int n_groups = 1);
}  // namespace trl_bs_cg
#endif


using namespace trl;

// both builds of the step kernels keep their own copy of the model constants
struct trl_handle;
static const trl_handle* g_model_owner = nullptr;    // whose ModelConst currently sits in the __constant__ copies
static int g_device = -1;                             // the one device this process drives (set by the first handle)
static cudaError_t upload_model_all(const ModelConst& mc, const TerrainSlot* terrain, const PhysParams* phys, int* env_phys, int* env_eval,
                                    const BodyConst* body, int* env_body, const RangeTables& ranges) {
    cudaError_t e = trl::upload_model(mc, terrain);
    if (e == cudaSuccess) e = trl_cg::upload_model(mc, terrain);
    if (e == cudaSuccess) e = trl_ts::upload_model(mc, terrain);
    if (e == cudaSuccess) e = trl_ts_cg::upload_model(mc, terrain);
    if (e == cudaSuccess) e = trl_ps::upload_model(mc, terrain);
    if (e == cudaSuccess) e = trl_ps_cg::upload_model(mc, terrain);
    if (e == cudaSuccess) e = trl_ps::upload_phys(phys, env_phys, env_eval);
    if (e == cudaSuccess) e = trl_ps_cg::upload_phys(phys, env_phys, env_eval);
#ifndef TRL_SIMT_EMU
    if (e == cudaSuccess) e = trl_bs::upload_model(mc, terrain);
    if (e == cudaSuccess) e = trl_bs_cg::upload_model(mc, terrain);
    if (e == cudaSuccess) e = trl_bs::upload_phys(phys, env_phys, env_eval);
    if (e == cudaSuccess) e = trl_bs_cg::upload_phys(phys, env_phys, env_eval);
#endif
    if (e == cudaSuccess) e = trl_bs::upload_body(body, env_body);
    if (e == cudaSuccess) e = trl_bs_cg::upload_body(body, env_body);
    if (e == cudaSuccess) e = trl_bs::upload_ranges(ranges);
    return e != cudaSuccess ? e : trl_bs_cg::upload_ranges(ranges);
}

// the per-link numbers of the scene's body (slot 0 of the body table), as fill_model derived them from the character file
static BodyConst body_of(const ModelConst& m) {
    BodyConst b;
    std::memset(&b, 0, sizeof(b));
#define TRL_BODY_COPY(f) std::memcpy(&b.f, &m.f, sizeof(b.f))
    TRL_BODY_COPY(attach_x); TRL_BODY_COPY(attach_y); TRL_BODY_COPY(lim_lo); TRL_BODY_COPY(lim_hi); TRL_BODY_COPY(has_limit);
    TRL_BODY_COPY(mass); TRL_BODY_COPY(body_ax); TRL_BODY_COPY(body_ay); TRL_BODY_COPY(body_theta); TRL_BODY_COPY(body_cos);
    TRL_BODY_COPY(body_sin); TRL_BODY_COPY(half_x); TRL_BODY_COPY(half_y); TRL_BODY_COPY(izz_o); TRL_BODY_COPY(izz_c);
    TRL_BODY_COPY(corner_lx); TRL_BODY_COPY(corner_ly); TRL_BODY_COPY(kp); TRL_BODY_COPY(kd); TRL_BODY_COPY(torque_lim);
    TRL_BODY_COPY(target_theta0); TRL_BODY_COPY(target_vel); TRL_BODY_COPY(world_pd); TRL_BODY_COPY(total_mass); TRL_BODY_COPY(reach);
#undef TRL_BODY_COPY
    return b;
}

static thread_local std::string g_err;
static int fail(const std::string& msg) { g_err = msg; return 1; }
int trl_fail(const std::string& msg) { return fail(msg); }
#define CK(call)                                                                                   \
    do {                                                                                           \
        cudaError_t e__ = (call);                                                                  \
        if (e__ != cudaSuccess) return fail(std::string(#call) + ": " + cudaGetErrorString(e__)); \
    } while (0)

static const char* kNetLayers[13] = {"terr_conv0", "terr_conv1", "terr_conv2", "terr_ip0", "ip0", "val_ip0", "val_ip1",
                                     "a0_ip0", "a0_ip1", "a1_ip0", "a1_ip1", "a2_ip0", "a2_ip1"};

#include "trl_handle.h"

// The kernels read the scene from __constant__ memory, of which there is one copy per process: a handle that is not the
// current owner re-uploads its model (after draining the owner's work) before it launches anything.
static int ensure_fc_maps(trl_handle* h);
static int ensure_slot_tables(trl_handle* h);
static int ensure_model_only(trl_handle* h);
static int ensure_model(trl_handle* h) {
    if (ensure_model_only(h)) return 1;
    if (ensure_fc_maps(h)) return 1;
    return ensure_slot_tables(h);
}
static int ensure_model_only(trl_handle* h) {
    // one process drives one GPU (DESIGN.md §7): __constant__ scene memory and the streams belong to the device of the handle
    // that was created first; a handle on another device is refused at creation (create_common)
    if (g_model_owner == h) return 0;
    if (cudaDeviceSynchronize() != cudaSuccess) return 1;
    h->terrain[0].type = h->mc.terrain_type;      // slot 0 of the terrain table is the scene's own terrain
    std::memcpy(h->terrain[0].params, h->mc.terrain_params, sizeof(h->mc.terrain_params));
    h->phys[0] = h->mc.phys;                      // and slot 0 of the physics table its own physics
    h->body[0] = body_of(h->mc);                  // and slot 0 of the body table its own body
    if (upload_model_all(h->mc, h->terrain, h->phys, h->env_phys, h->env_eval, h->body, h->env_body, h->ranges) != cudaSuccess) return 1;
    g_model_owner = h;
    return 0;
}

int trl_reupload_model(trl_handle* h) {
    if (!h) return fail("trl_reupload_model: null handle");
    g_model_owner = nullptr;
    return ensure_model(h) ? fail("model upload failed") : 0;
}

// cScenarioSimChar::SetTerrainParamsLerp (scenarios/ScenarioSimChar.cpp:255-272): n_sets parameter sets [n_sets][40] blended at
// `lerp` (clamped to the sets there are); no set = the generator's defaults
static void blend_terrain(const double* sets, int n_sets, const double* dflt, double lerp, double* out) {
    if (n_sets <= 0) {
        for (int i = 0; i < kTerrainParams; ++i) out[i] = dflt[i];
        return;
    }
    lerp = std::min(std::max(lerp, 0.0), n_sets - 1.0);
    const int i0 = (int)lerp, i1 = std::min(i0 + 1, n_sets - 1);
    lerp -= i0;
    for (int i = 0; i < kTerrainParams; ++i) out[i] = (1 - lerp) * sets[i0 * kTerrainParams + i] + lerp * sets[i1 * kTerrainParams + i];
}

template <typename T>
static cudaError_t dalloc(trl_handle* h, T** p, size_t count) {
    cudaError_t e = cudaMalloc((void**)p, count * sizeof(T));
    if (e == cudaSuccess) { h->allocs.push_back(*p); e = cudaMemset(*p, 0, count * sizeof(T)); }
    return e;
}

static int fill_model(trl_handle* h, uint64_t rng_seed) {
    const ScenePack& s = h->scene;
    ModelConst& m = h->mc;
    std::memset(&m, 0, sizeof(m));
    const auto& mi = s.i32("meta_i32");
    const auto& mf = s.f64("meta_f64");
    if (mi.size() < 15 || mf.size() < 7) return fail("scene pack: meta records missing or too short");
    int char_type = mi[0], ctrl = mi[1];
    m.nj = mi[8]; m.ndof = mi[9];
    const bool raptor = char_type == 2;
    if (!((char_type == 1 && m.nj == 21 && m.ndof == 23) || (raptor && m.nj == 19 && m.ndof == 21)))
        return fail("unsupported character: expected the dog / goat (21 joints) or raptor (19 joints) skeleton");
    m.char_type = char_type;
    {
        // parameter layout and optimised-parameter mask (sim/DogController.cpp:81-121, sim/RaptorController.cpp:78-122)
        static const bool raptor_mask[37] = {false, true, true, false, false,
                                             true, false, true, true, true, true, true, true,
                                             true, false, true, true, true, true, true, true,
                                             false, false, true, true, true, true, true, true,
                                             false, false, true, true, true, true, true, true};
        m.n_params = raptor ? 37 : 30; m.misc_max = raptor ? 5 : 6; m.sp_max = raptor ? 8 : 6;
        m.n_opt = 0;
        for (int i = 0; i < m.n_params; ++i)
            if (raptor ? raptor_mask[i] : (i != 0)) m.opt_idx[m.n_opt++] = i;
        m.exp_noise = raptor ? 0.15 : 0.2;
        m.stumble_mask = 0; m.fall_mask = 0;
        if (raptor) {
            for (int j = 0; j < m.nj; ++j) if (j != 14 && j != 18 && j != 13 && j != 17) m.stumble_mask |= 1u << j;
            for (int j : {0, 1, 2, 3, 4, 5}) m.fall_mask |= 1u << j;
        } else {
            for (int j = 0; j < m.nj; ++j) if (j != 20 && j != 16 && j != 19 && j != 15) m.stumble_mask |= 1u << j;
            for (int j : {0, 1, 2, 3, 4, 5, 6, 7, 8}) m.fall_mask |= 1u << j;
        }
    }
    h->num_update_steps = mi[2];
    m.num_sim_substeps = mi[3];
    m.has_init_x = mi[4]; m.init_x = mf[2];
    m.terrain_type = mi[5];
    int n_sets = mi[6];
    m.has_net = mi[7];
    m.n_ctrl = mi[10]; m.n_actions = mi[11]; m.default_action = mi[12]; m.grav_comp = mi[13]; m.virt_forces = mi[14];
    if (m.n_ctrl > kMaxCtrlSets || m.n_actions > kMaxActions) return fail("too many controller sets / actions");
    m.is_mace = (ctrl == 3 || ctrl == 4 || ctrl == 7) ? 1 : 0;
    m.target_vel_x = (ctrl == 4) ? 2.0 : 4.0;   // sim/GoatControllerMACE.cpp:11-14, sim/DogController.cpp:625-628
    m.gx = mf[0]; m.gy = mf[1];
    m.exp_mode = h->mode == TRL_MODE_EXPLORE;
    m.rng_seed = rng_seed;
    const auto& J = s.f64("joints");
    const auto& Bd = s.f64("bodies");
    const auto& P = s.f64("pd");
    {
        // every table the loops below index, against the sizes they assume
        const size_t nj = (size_t)m.nj, np = (size_t)m.n_params;
        const int n_ctrl = mi[10], n_act = mi[11];
        if (n_ctrl < 1 || n_ctrl > kMaxCtrlSets || n_act < 0 || n_act > kMaxActions) return fail("too many controller sets / actions");
        if (J.size() < 7 * nj || Bd.size() < 9 * nj || P.size() < 6 * nj) return fail("scene pack: joints / bodies / pd tables too short");
        if (s.f64("ctrl_params").size() < (size_t)n_ctrl * np || s.f64("actions").size() < (size_t)4 * n_act)
            return fail("scene pack: controller parameter / action tables too short");
        if (s.f64("pose0").size() < (size_t)m.ndof || s.f64("vel0").size() < (size_t)m.ndof) return fail("scene pack: initial state too short");
        if (s.f64("terrain_default_params").size() < (size_t)kTerrainParams || mi[6] < 0 ||
            s.f64("terrain_params").size() < (size_t)mi[6] * kTerrainParams)
            return fail("scene pack: terrain parameter sets too short");
        for (size_t j = 0; j < nj; ++j) {
            const int par = (int)J[7 * j + 1];
            if (par >= (int)j || par < -1) return fail("scene pack: a joint's parent must precede it");
        }
    }
    int off = 0;
    m.total_mass = 0;
    for (int j = 0; j < m.nj; ++j) {
        const double* r = &J[7 * j];
        int type = (int)r[0];
        m.parent[j] = (int)r[1];
        if ((j == 0) != (m.parent[j] < 0) || (j == 0 && type != 1) || (j > 0 && type != 0)) return fail("unsupported joint layout");
        m.attach_x[j] = r[2]; m.attach_y[j] = r[3];
        m.lim_lo[j] = r[5]; m.lim_hi[j] = r[6];
        m.has_limit[j] = (j > 0 && r[5] <= r[6]) ? 1 : 0;
        m.dof[j] = off;
        off += (j == 0) ? 3 : 1;
        const double* b = &Bd[9 * j];
        if ((int)b[0] != 0) return fail("only box bodies are supported");
        m.mass[j] = b[1]; m.body_ax[j] = b[2]; m.body_ay[j] = b[3]; m.body_theta[j] = b[5];
        m.body_cos[j] = std::cos(b[5]); m.body_sin[j] = std::sin(b[5]);
        m.half_x[j] = 0.5 * b[6]; m.half_y[j] = 0.5 * b[7];
        // planar inertia about the joint origin: box about its COM + parallel-axis shift (sim/RBDUtil.cpp:562-583,614-623)
        m.izz_o[j] = b[1] / 12.0 * (b[6] * b[6] + b[7] * b[7]) + b[1] * (b[2] * b[2] + b[3] * b[3]);
        m.izz_c[j] = b[1] / 12.0 * (b[6] * b[6] + b[7] * b[7]);
        m.total_mass += b[1];
        // tail parts carry collision group "none" (sim/SimDog.cpp:7,21-24)
        m.collidable[j] = (!raptor && j >= 9 && j <= 12) ? 0 : 1;   // every raptor part collides (sim/SimRaptor.cpp:4-27)
        const double* p = &P[6 * j];
        m.kp[j] = (j == 0) ? 0.0 : p[0]; m.kd[j] = (j == 0) ? 0.0 : p[1];
        m.torque_lim[j] = p[2]; m.target_theta0[j] = p[3]; m.target_vel[j] = p[4]; m.world_pd[j] = p[5] != 0;
    }
    // topology helpers
    m.max_depth = 0;
    for (int j = 0; j < m.nj; ++j) {
        m.depth[j] = (j == 0) ? 0 : m.depth[m.parent[j]] + 1;
        m.max_depth = std::max(m.max_depth, m.depth[j]);
        for (int c = 0; c < 4; ++c) m.child[j][c] = -1;
    }
    if (m.max_depth >= 12) return fail("kinematic tree too deep");
    for (int j = 1; j < m.nj; ++j) {
        int p = m.parent[j], slot = 0;
        while (slot < 4 && m.child[p][slot] >= 0) ++slot;
        if (slot == 4) return fail("a link has more than 4 children");
        m.child[p][slot] = j;
    }
    if (m.max_depth >= 16) return fail("kinematic tree too deep for the 4-round ancestor jumps");
    if (m.nj > 31) return fail("lane 31 must stay idle (zero source of the warp passes)");
    {
        // chain schedule.  Summation order at a branch point: children by the earliest step their subtree is complete in (ties by
        // index) -- the order of the level-synchronous schedule this one replaced, so the sums are the same to the bit
        std::vector<int> earliest(m.nj, 0), nch(m.nj, 0);
        std::vector<std::vector<int>> merge_order(m.nj);
        for (int j = 1; j < m.nj; ++j) ++nch[m.parent[j]];
        for (int p = m.nj - 1; p >= 0; --p) {     // parents precede children in index order
            std::vector<std::pair<int, int>> ch;
            for (int c = 0; c < 4; ++c) if (m.child[p][c] >= 0) ch.push_back({earliest[m.child[p][c]], m.child[p][c]});
            std::sort(ch.begin(), ch.end());
            int last = -1;
            for (auto& ec : ch) { merge_order[p].push_back(ec.second); last = std::max(ec.first, last + 1); }
            earliest[p] = last + 1;
        }
        // chain tops: the root and every child of a link with more than one child; chain 0 is the root's
        std::vector<int> tops, chain_of(m.nj, -1);
        for (int j = 0; j < m.nj; ++j) if (j == 0 || nch[m.parent[j]] != 1) tops.push_back(j);
        m.n_chains = (int)tops.size();
        if (m.n_chains > kWarp) return fail("more chains than lanes");
        std::vector<int> bottom(m.n_chains);
        for (int c = 0; c < m.n_chains; ++c) {
            std::vector<int> links{tops[c]};
            while (nch[links.back()] == 1) links.push_back(m.child[links.back()][0]);
            if ((int)links.size() > 12) return fail("kinematic chain longer than 12 links");
            m.chain_len[c] = (int)links.size();
            m.chain_links[c] = 0;
            for (int i = 0; i < m.chain_len[c]; ++i) {
                m.chain_links[c] |= (unsigned long long)links[m.chain_len[c] - 1 - i] << (5 * i);
                chain_of[links[i]] = c;
            }
            bottom[c] = links.back();
            m.chain_up[c] = tops[c] == 0 ? -1 : m.parent[tops[c]];
        }
        m.chain_levels = 0;
        for (int c = m.n_chains - 1; c >= 0; --c) {    // a child chain's top has a larger index than its parent chain's bottom
            m.chain_merge[c] = 0;
            int lev = 0;
            for (int q = 0; q < 4; ++q) {
                const int ch = (nch[bottom[c]] > 1 && q < nch[bottom[c]]) ? merge_order[bottom[c]][q] : -1;
                const int cc = ch >= 0 ? chain_of[ch] : 31;
                if (ch >= 0) lev = std::max(lev, m.chain_level[cc] + 1);
                m.chain_merge[c] |= cc << (5 * q);
            }
            m.chain_level[c] = lev;
            m.chain_levels = std::max(m.chain_levels, lev + 1);
        }
        for (int l = 0; l < m.chain_levels; ++l) {
            m.chain_level_len[l] = 0;
            for (int c = 0; c < m.n_chains; ++c) if (m.chain_level[c] == l) m.chain_level_len[l] = std::max(m.chain_level_len[l], m.chain_len[c]);
        }
    }
    for (int j = 0; j < m.nj; ++j) {
        m.anc_pow[j][0] = m.parent[j];
        for (int k = 1; k < 4; ++k) m.anc_pow[j][k] = m.anc_pow[j][k - 1] >= 0 ? m.anc_pow[m.anc_pow[j][k - 1]][k - 1] : -1;
    }
    {
        // box corners in the link frame, the 4 of a collidable body from corner_base[j] on (the body's lane tests them in this order).
        // reach = upper bound of |corner - root joint| over all poses (bounds the terrain window the contacts can see)
        std::vector<double> jr(m.nj, 0.0);
        m.reach = 0.0;
        m.n_corners = 0;
        for (int j = 0; j < m.nj; ++j) {
            if (j > 0) jr[j] = jr[m.parent[j]] + std::hypot(m.attach_x[j], m.attach_y[j]);
            m.corner_base[j] = -1;
            if (!m.collidable[j]) continue;
            m.corner_base[j] = m.n_corners;
            for (int cn = 0; cn < 4; ++cn) {
                double bx = (cn & 1) ? m.half_x[j] : -m.half_x[j], by = (cn & 2) ? m.half_y[j] : -m.half_y[j];
                double lx = m.body_ax[j] + m.body_cos[j] * bx - m.body_sin[j] * by;
                double ly = m.body_ay[j] + m.body_sin[j] * bx + m.body_cos[j] * by;
                m.corner_lx[m.n_corners] = lx;
                m.corner_ly[m.n_corners] = ly;
                ++m.n_corners;
                m.reach = std::max(m.reach, jr[j] + std::hypot(lx, ly));
            }
        }
    }
    {
        // effector 0 / 1: dog toe (back foot) / finger (front foot); raptor right toe / left toe.
        // dog virtual forces stop at the root / torso (sim/DogController.cpp:1014-1016), raptor's at the root (:1053)
        const int toe = raptor ? 14 : 20, finger = raptor ? 18 : 16, torso = raptor ? 0 : 5;
        m.anc_mask_toe = m.anc_mask_finger = m.vf_mask_toe = m.vf_mask_finger = 0;
        for (int c = toe; c >= 0; c = m.parent[c]) m.anc_mask_toe |= 1u << c;
        for (int c = finger; c >= 0; c = m.parent[c]) m.anc_mask_finger |= 1u << c;
        for (int c = toe; c != 0 && c != torso; c = m.parent[c]) m.vf_mask_toe |= 1u << c;
        for (int c = finger; c != 0 && c != torso; c = m.parent[c]) m.vf_mask_finger |= 1u << c;
    }
    const auto& C = s.f64("ctrl_params");
    for (int c = 0; c < m.n_ctrl; ++c)
        for (int k = 0; k < m.n_params; ++k) m.ctrl_params[c][k] = C[c * m.n_params + k];
    const auto& A = s.f64("actions");
    for (int a = 0; a < m.n_actions; ++a) {
        m.act_idx0[a] = (int)A[4 * a]; m.act_idx1[a] = (int)A[4 * a + 1]; m.act_blend[a] = A[4 * a + 2]; m.act_cyclic[a] = A[4 * a + 3] != 0;
    }
    const auto& p0 = s.f64("pose0");
    const auto& v0 = s.f64("vel0");
    for (int k = 0; k < m.ndof; ++k) { m.pose0[k] = p0[k]; m.vel0[k] = v0[k]; }
    // cScenarioSimChar::SetTerrainParamsLerp (scenarios/ScenarioSimChar.cpp:255-272)
    blend_terrain(s.f64("terrain_params").data(), n_sets, s.f64("terrain_default_params").data(), mf[3], m.terrain_params);
    h->terrain_lerp = mf[3];
    {
        const char* vc = std::getenv("TRL_VERTEX_CONTACTS");
        m.phys = PhysParams{2.0e5, 2.0e3, 0.81, 0.01, 0.00025, 2.0e4, 20.0, (vc && vc[0] == '1') ? 1 : 0};
    }
    for (ExpSettings& e : h->ex) e = ExpSettings{h->mode == TRL_MODE_EXPLORE ? 1 : 0, mf[4], mf[5], mf[6], m.exp_noise};   // uploaded by create_common
    if (m.has_net) {
        const auto& nd = s.i32("net_dims");
        if (nd.size() < 5) return fail("scene pack: net_dims missing");
        m.n_in = nd[0]; m.n_char = nd[1]; m.n_out = nd[2]; m.n_frags = nd[3]; m.frag = nd[4];
        if (m.n_out > kMaxNetOut || m.frag > 32 || m.n_frags > 8 || m.n_char > 96) return fail("unsupported net dimensions");
        const auto& os = s.f64("net_out_scale");
        if (m.n_frags < 1 || m.frag < 1 || os.size() < (size_t)(m.n_frags + m.frag)) return fail("scene pack: net_out_scale too short");
        for (int k = 0; k < m.frag; ++k) m.out_scale_actor0[k] = os[m.n_frags + k];
    }
    return 0;
}

// into policy slot `slot` (0: the handle's own net, W); every slot has the topology of the first upload
static int upload_net(trl_handle* h, const double* const* blobs, const int64_t* counts, const double* const* vecs4, const int64_t* vcounts,
                      int slot = 0) {
    // blobs: 26 (w, b per layer), vecs4: in_off, in_scale, out_off, out_scale
    std::vector<double*>& dst = slot == 0 ? h->net_blobs : h->slot_blobs[slot];
    if (h->net_counts.empty()) {
        h->net_counts.assign(30, 0);
        for (int i = 0; i < 30; ++i) h->net_counts[i] = i < 26 ? counts[i] : vcounts[i - 26];
    }
    if (dst.empty()) {
        dst.assign(30, nullptr);
        for (int i = 0; i < 30; ++i) CK(dalloc(h, &dst[i], (size_t)h->net_counts[i]));
    }
    for (int i = 0; i < 30; ++i) {
        int64_t c = i < 26 ? counts[i] : vcounts[i - 26];
        if (c != h->net_counts[i]) return fail("trl_set_weights: blob size mismatch");
        const double* src = i < 26 ? blobs[i] : vecs4[i - 26];
        CK(cudaMemcpyAsync(dst[i], src, (size_t)c * 8, cudaMemcpyHostToDevice, h->stream));
    }
    CK(cudaStreamSynchronize(h->stream));
    double** b = dst.data();
    (slot == 0 ? h->W : h->slot_W[slot]) = net_weights(b, b[26], b[27], b[28], b[29]);
    return 0;
}

// the decision kernel indexes the 26 blobs with the MACE topology's strides (data/policies/dog/nets/dog_mace3_deploy.prototxt):
// anything else must be refused before it reaches the device
static int check_net_counts(const ModelConst& m, const int64_t* counts, const int64_t* vcounts) {
    const int64_t want[10] = {16 * 8, 16, 32 * 16 * 4, 32, 32 * 32 * 4, 32, 64 * 32 * 187, 64, 256 * (int64_t)(64 + m.n_char), 256};
    for (int b = 0; b < 26; ++b) {
        int64_t w;
        if (b < 10) w = want[b];
        else {
            const int hd = (b - 10) / 4, r = (b - 10) % 4, nout = hd == 0 ? m.n_frags : m.frag;
            w = r == 0 ? 128 * 256 : (r == 1 ? 128 : (r == 2 ? (int64_t)nout * 128 : nout));
        }
        if (counts[b] != w) return fail("policy net: blob " + std::to_string(b) + " has " + std::to_string(counts[b]) + " values, the MACE topology needs " + std::to_string(w));
    }
    if (vcounts) {
        const int64_t vw[4] = {m.n_in, m.n_in, m.n_out, m.n_out};
        for (int k = 0; k < 4; ++k)
            if (vcounts[k] != vw[k]) return fail("policy net: offset / scale vector " + std::to_string(k) + " has the wrong length");
    }
    if (m.n_in != 200 + m.n_char || m.n_out != m.n_frags * (1 + m.frag)) return fail("policy net: input / output sizes do not match the MACE topology");
    return 0;
}

// ---- batched decision path: TMA descriptors over the terr_ip0 weights and the conv2-output scratch (trl_decide2.cuh)
#ifndef TRL_SIMT_EMU
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn tensor_map_encoder() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
            fn = (EncodeTiledFn)p;
    }
    return fn;
}
// [rows][5984] f64 row-major, box [box_rows][16 doubles = 128 B], 128-byte swizzle, rows past the end read as zero
static int encode_rows_map(CUtensorMap* map, const double* base, uint64_t rows, uint32_t box_rows) {
    EncodeTiledFn enc = tensor_map_encoder();
    if (!enc) return fail("cuTensorMapEncodeTiled is not available from this driver");
    if (((uintptr_t)base & 15u) != 0) return fail("TMA needs 16-byte aligned weights");
    const cuuint64_t dims[2] = {5984, rows};
    const cuuint64_t strides[1] = {5984 * 8};
    const cuuint32_t box[2] = {16, box_rows};
    const cuuint32_t estr[2] = {1, 1};
    const CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT64, 2, (void*)base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                           CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return fail("cuTensorMapEncodeTiled failed (" + std::to_string((int)r) + ")");
    return 0;
}
#endif
// TMA descriptors for a forward pass through the batched kernels outside the decision path (the trainer's minibatch)
int trl_make_fc_maps(trl::FcMaps* out, const double* tip0_w, const double* act2, int rows) {
    std::memset(out, 0, sizeof(*out));
    out->w_ptr = tip0_w; out->a_ptr = act2; out->a_rows = rows; out->prof = nullptr;
#ifndef TRL_SIMT_EMU
    if (encode_rows_map(&out->w, tip0_w, 64, 64)) return 1;
    if (encode_rows_map(&out->a, act2, (uint64_t)rows, 32)) return 1;
#endif
    return 0;
}
static int ensure_fc_maps(trl_handle* h) {
    if (!h->decide_v2 || !h->mc.has_net || !h->act2[0] || !h->W.tip0_w) return 0;
    if (h->fc_maps_w == h->W.tip0_w) return 0;
    for (int k = 0; k < h->lag; ++k) {
        h->fc_maps[k].w_ptr = h->W.tip0_w;
        h->fc_maps[k].a_ptr = h->act2[k];
        h->fc_maps[k].a_rows = h->n;
        h->fc_maps[k].prof = nullptr;
#ifndef TRL_SIMT_EMU
        if (encode_rows_map(&h->fc_maps[k].w, h->W.tip0_w, 64, 64)) return 1;
        if (encode_rows_map(&h->fc_maps[k].a, h->act2[k], (uint64_t)h->n, 32)) return 1;
#endif
    }
    h->fc_maps_w = h->W.tip0_w;
    return 0;
}
static void destroy_graphs(trl_handle* h);
// slot build: the device table of the slots' weights and each slot's terr_ip0 descriptor, rewritten after a slot was loaded or slot 0's
// weights moved.  Captured graphs bake the descriptors in and are dropped.  Called with the handle drained.
static int ensure_slot_tables(trl_handle* h) {
    if (!h->slots_active) return 0;
    if (!h->slot_dirty && std::memcmp(&h->slot_W[0], &h->W, sizeof(NetWeights)) == 0) return 0;
    h->slot_W[0] = h->W;
    CK(cudaMemcpy((void*)h->P.W, h->slot_W, sizeof(h->slot_W), cudaMemcpyHostToDevice));
    for (int p = 0; p < kMaxPolicySlots; ++p) {
        const double* w = h->slot_W[p].tip0_w;
        if (!w || h->slot_maps.w_ptr[p] == w) continue;
#ifndef TRL_SIMT_EMU
        if (encode_rows_map(&h->slot_maps.w[p], w, 64, 64)) return 1;
#endif
        h->slot_maps.w_ptr[p] = w;
    }
    destroy_graphs(h);
    h->slot_dirty = false;
    return 0;
}
// the decision launch(es) of one env-step; `side` = the side stream's index (its act2 scratch, descriptors and chunk table)
static void enqueue_decide(trl_handle* h, int list, int rearm, cudaStream_t st, int part = 3, int side = 0) {
    if (h->decide_v2 && h->slots_active)
        launch_decide2_slots(h->B, h->P, h->d_ex, h->fc_maps[side], h->slot_maps, h->act2[side], h->P.sort_tmp + (size_t)side * h->n,
                             h->P.chunks + (size_t)side * (1 + 3 * h->P.chunk_cap), h->done_count, h->decide_grid, h->fc_clusters, list, rearm, st,
                             part);
    else if (h->decide_v2)
        launch_decide2(h->B, h->W, h->d_ex, h->fc_maps[side], h->act2[side], h->done_count, h->decide_grid, h->fc_clusters, list, rearm, st, part);
    else if (part & 1)
        launch_decide(h->B, h->W, h->d_ex, h->done_count, h->decide_grid, list, rearm, st);
}
// the env-step launches of a handle: the body-slot builds once a body slot is loaded (trl_load_body; they serve terrain and physics
// slots and evaluation envs too), else the physics-slot builds once a physics slot is loaded (trl_load_physics) or an env was given a
// mode (trl_set_env_eval; they serve terrain slots too), else the terrain-slot builds once a terrain slot is loaded
// (trl_load_terrain), else the plain ones
static bool terrain_slots(const trl_handle* h) { return !h->env_terrain_host.empty(); }
static bool phys_slots(const trl_handle* h) { return h->env_phys != nullptr || h->env_eval != nullptr; }
static bool body_slots(const trl_handle* h) { return h->env_body != nullptr; }
static void step_launch(const trl_handle* h, double step, int flags, int lists, cudaStream_t st, int group = 0, int n_groups = 1) {
    if (body_slots(h)) trl_bs::launch_step(h->B, step, flags, lists, st, group, n_groups);
    else if (phys_slots(h)) trl_ps::launch_step(h->B, step, flags, lists, st, group, n_groups);
    else if (terrain_slots(h)) trl_ts::launch_step(h->B, step, flags, lists, st, group, n_groups);
    else launch_step(h->B, step, flags, lists, st, group, n_groups);
}
static void catchup_launch(const trl_handle* h, double step, int flags, int lists, cudaStream_t st) {
    if (body_slots(h)) trl_bs_cg::launch_step(h->B, step, flags, lists, st);
    else if (phys_slots(h)) trl_ps_cg::launch_step(h->B, step, flags, lists, st);
    else if (terrain_slots(h)) trl_ts_cg::launch_step(h->B, step, flags, lists, st);
    else trl_cg::launch_step(h->B, step, flags, lists, st);
}
static void terrain_launch(const trl_handle* h, cudaStream_t st) {
    if (body_slots(h)) trl_bs::launch_terrain(h->B, 0.5, st);
    else if (phys_slots(h)) trl_ps::launch_terrain(h->B, 0.5, st);
    else if (terrain_slots(h)) trl_ts::launch_terrain(h->B, 0.5, st);
    else launch_terrain(h->B, 0.5, st);
}
static void reset_launch(const trl_handle* h, const uint64_t* seeds, const int* env_ids, int count, int reseed) {
    if (body_slots(h)) trl_bs::launch_reset(h->B, seeds, env_ids, count, reseed, h->stream);
    else if (phys_slots(h)) trl_ps::launch_reset(h->B, seeds, env_ids, count, reseed, h->stream);
    else if (terrain_slots(h)) trl_ts::launch_reset(h->B, seeds, env_ids, count, reseed, h->stream);
    else launch_reset(h->B, seeds, env_ids, count, reseed, h->stream);
}
static int num_decide_launches(const trl_handle* h) { return h->decide_v2 ? (h->slots_active ? 3 : 2) : 1; }

void trl_drop_graphs(trl_handle* h) { destroy_graphs(h); }
static void destroy_graphs(trl_handle* h) {
    for (auto& kv : h->graphs) cudaGraphExecDestroy(kv.second);
    h->graphs.clear();
}

// One outer update = num_update_steps env-steps.  An env-step is split at the policy decision: launch S_i runs the
// controller half of env-step i-1 and the physics half of env-step i for every env, then the decision kernel D_i serves the
// (few) envs that reached a cycle boundary in S_i.
//
//   serial schedule      T  S_0  D_0  S_1  D_1 ... S_{ns-1}  D_{ns-1}  S_end
//   overlapped schedule  main stream    T  S_0  S_1  S_2  S_3  S_4 ...  S_{ns-1}  S_end          (back to back)
//   (lag = 2 shown)      side stream 0        D_0 -> C_0 [steps 1, 2]     D_2 -> C_2 [steps 3, 4] ...
//                        side stream 1             D_1 -> C_1 [steps 2, 3]     D_3 -> C_3 ...
//
// In the overlapped schedule the envs that reach a cycle boundary in S_l wait for D_l and are then advanced by the catch-up
// launch C_l (same kernel, one warp per list entry, registers live across its `lag` env-steps) while S_{l+1} .. S_{l+lag} skip
// them; S_{l+lag+1} needs C_l.  lag + 1 pending lists rotate (S_l appends to list l % (lag + 1), which C_{l-lag-1} re-armed); side
// stream l % lag carries D_l and C_l.  Every env still advances by exactly one env-step per launch equivalent, so results are
// the same as in the serial schedule up to the rounding of the catch-up build (a second instantiation of the kernel source with the
// env-step loop: ~1e-12 after 45 updates; tests/test_gpu_scenarios.py::test_overlap_matches_serial).  Why several steps of slack
// (trl_update_timeline): a lone warp needs a fixed latency per env-step whatever else runs, and the decision kernels wait for SM
// resources the step launch holds, so the chain D_l -> C_l is more than two step launches long; with one step of slack it bounded the update.
// optional recorder of a timeline (trl_update_timeline): an event pair around every launch, on the stream it is launched on
struct Timeline {
    std::vector<cudaEvent_t> beg, end, fork;
    std::vector<int> kind, idx;      // kind: 0 terrain, 1 step S_i, 2 decision D_i (conv stage of the batched path), 3 catch-up C_i, 4 FC stage of D_i
    std::string err;                 // first CUDA error seen while enqueueing, with the launch it followed
    void check(const char* where) {
        const cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess && err.empty())
            err = std::string(where) + " of launch kind " + std::to_string(kind.empty() ? -1 : kind.back()) + " #" + std::to_string(idx.empty() ? -1 : idx.back()) + ": " + cudaGetErrorString(e);
    }
    void open(cudaStream_t st, int k, int i) {
        check("before");
        cudaEvent_t b, e;
        cudaEventCreate(&b); cudaEventCreate(&e);
        beg.push_back(b); end.push_back(e); kind.push_back(k); idx.push_back(i);
        cudaEventRecord(b, st);
        check("open");
    }
    void close(cudaStream_t st) { check("launch"); cudaEventRecord(end.back(), st); check("close"); }
};
static void enqueue_update(trl_handle* h, double dt, bool overlap, Timeline* tl = nullptr) {
    const int ns = h->num_update_steps;
    const double step = dt / ns;
    cudaStream_t A = h->stream;
#define TL_OPEN(st, k, i) do { if (tl) tl->open(st, k, i); } while (0)
#define TL_CLOSE(st) do { if (tl) tl->close(st); } while (0)
    TL_OPEN(A, 0, 0); terrain_launch(h, A); TL_CLOSE(A);
    if (!overlap) {
        for (int i = 0; i < ns; ++i) {
            TL_OPEN(A, 1, i); step_launch(h, step, i == 0 ? 2 : 3, 0, A); TL_CLOSE(A);
            TL_OPEN(A, 2, i); enqueue_decide(h, 0, 1, A, 1); TL_CLOSE(A); TL_OPEN(A, 4, i); enqueue_decide(h, 0, 1, A, 2); TL_CLOSE(A);
        }
        TL_OPEN(A, 1, ns); step_launch(h, step, 1 | 4, 0, A); TL_CLOSE(A);
        return;
    }
    // Overlapped schedule, `lag` env-steps deep.  Main stream: T S_0 S_1 S_2 ... S_{ns-1} S_end back to back.  The envs that reach a
    // cycle boundary in S_l (list l % (lag + 1)) are served on side stream l % lag: D_l decides them, the catch-up launch C_l then
    // advances exactly those envs by `lag` env-steps (fewer if the update ends first) while S_{l+1} .. S_{l+lag} skip them.
    // S_{l+lag+1} needs C_l.  The chain D_l -> C_l therefore has `lag` step launches of slack.
    const int lag = h->lag, nl = lag + 1;
    // Env groups: the main launch of an env-step is split into G launches over contiguous env ranges, group g on its own stream
    // (group 0 on the engine stream).  The groups only meet where the side work does (D_l needs S_l of every group, S_{l+lag+1} of every
    // group needs C_l), so group g's S_{i+1} starts as soon as ITS S_i has drained and its CTAs fill the SM slots the tail of the other
    // groups' launches would leave idle (4096 warps over 2368 resident-warp slots = 1.73 waves per monolithic launch).
    const int G = std::max(1, std::min(h->groups, kMaxGroups));
    std::vector<cudaEvent_t>& fe = tl ? tl->fork : h->fork_events;
    const size_t need = (size_t)(ns + 1) * G + ns + 2;
    if (fe.size() < need) {
        size_t old = fe.size();
        fe.resize(need);
        for (size_t i = old; i < fe.size(); ++i) cudaEventCreateWithFlags(&fe[i], cudaEventDisableTiming);
    }
    cudaEvent_t* ev_s = fe.data();                    // ev_s[i * G + g]: S_i of group g done
    cudaEvent_t* ev_c = fe.data() + (ns + 1) * G;     // ev_c[l]: C_l (l < ns - 1) / D_{ns-1} done
    cudaEvent_t ev_t = fe[need - 1];                  // terrain look-ahead done
    auto lists_of = [&](int app, int prev, int reps) { return (app % nl) | ((prev % nl) << 3) | (reps << 6); };
    auto stream_of = [&](int g) { return g == 0 ? A : h->group_stream[g - 1]; };
    if (G > 1) { cudaEventRecord(ev_t, A); for (int g = 1; g < G; ++g) cudaStreamWaitEvent(stream_of(g), ev_t, 0); }
    for (int g = 0; g < G; ++g) {
        cudaStream_t M = stream_of(g);
        TL_OPEN(M, 1, 0); step_launch(h, step, 2, lists_of(0, 0, 0), M, g, G); TL_CLOSE(M);
        cudaEventRecord(ev_s[g], M);
    }
    for (int i = 1; i < ns; ++i) {
        // side work for the envs that became due in S_{i-1}
        const int l = i - 1, slot = l % lag;
        cudaStream_t X = h->side[slot];
        for (int g = 0; g < G; ++g) cudaStreamWaitEvent(X, ev_s[l * G + g], 0);
        TL_OPEN(X, 2, l); enqueue_decide(h, l % nl, 0, X, 1, slot); TL_CLOSE(X); TL_OPEN(X, 4, l); enqueue_decide(h, l % nl, 0, X, 2, slot); TL_CLOSE(X);
        const int reps = std::min(lag, ns - 1 - l);     // equivalents l + 1 .. l + reps of the main launches; S_end is never caught up
        TL_OPEN(X, 3, l); catchup_launch(h, step, 1 | 2 | 16, lists_of(l + 1, l, reps), X); TL_CLOSE(X);
        cudaEventRecord(ev_c[l], X);
        for (int g = 0; g < G; ++g) {
            cudaStream_t M = stream_of(g);
            if (i >= nl) cudaStreamWaitEvent(M, ev_c[i - nl], 0);
            TL_OPEN(M, 1, i); step_launch(h, step, 1 | 2 | 8, lists_of(i, i, 0), M, g, G); TL_CLOSE(M);
            cudaEventRecord(ev_s[i * G + g], M);
        }
    }
    {
        const int l = ns - 1, slot = l % lag;
        cudaStream_t X = h->side[slot];
        for (int g = 0; g < G; ++g) cudaStreamWaitEvent(X, ev_s[l * G + g], 0);
        TL_OPEN(X, 2, l); enqueue_decide(h, l % nl, 1, X, 1, slot); TL_CLOSE(X); TL_OPEN(X, 4, l); enqueue_decide(h, l % nl, 1, X, 2, slot); TL_CLOSE(X);
        cudaEventRecord(ev_c[l], X);
    }
    for (int l = std::max(0, ns - nl); l < ns; ++l) cudaStreamWaitEvent(A, ev_c[l], 0);     // every side stream joins here
    for (int g = 1; g < G; ++g) cudaStreamWaitEvent(A, ev_s[(ns - 1) * G + g], 0);          // and every group stream
    TL_OPEN(A, 1, ns); step_launch(h, step, 1 | 4, 0, A); TL_CLOSE(A);
#undef TL_OPEN
#undef TL_CLOSE
}
static int update_launches(const trl_handle* h, bool overlap) {
    const int ns = h->num_update_steps, d = num_decide_launches(h);
    const int G = std::max(1, std::min(h->groups, kMaxGroups));
    return overlap ? (1 + G + d) * ns : (1 + d) * ns + 2;    // G x S_0..S_{ns-1} + D_0..D_{ns-1} + S_end + C_0..C_{ns-2} (the terrain look-ahead is not counted)
}

extern "C" {

const char* trl_last_error(void) { return g_err.c_str(); }


trl_handle* trl_create_from_pack(const char* pack_path, int num_envs, int device, int mode, const uint64_t* terrain_seeds,
                                 uint64_t rng_seed) {
    auto* h = new trl_handle();
    try {
        std::string err;
        if (!h->scene.load(pack_path, &err)) { g_err = err; delete h; return nullptr; }
        return trl_create_common(h, num_envs, device, mode, terrain_seeds, rng_seed);
    } catch (const std::exception& e) {       // bad_alloc / out_of_range from a damaged pack must not cross the C ABI
        g_err = std::string("trl_create_from_pack: ") + e.what();
        delete h;
        return nullptr;
    }
}

trl_handle* trl_create(int argc, const char* const* argv, const char* data_root, int num_envs, int device, int mode,
                       const uint64_t* terrain_seeds, uint64_t rng_seed) {
    auto* h = new trl_handle();
    try {
        build_scene_from_args(argc, argv, data_root ? data_root : "", &h->scene);
    } catch (const std::exception& e) {
        g_err = e.what();
        delete h;
        return nullptr;
    }
    h->data_root = data_root ? data_root : "";
    return trl_create_common(h, num_envs, device, mode, terrain_seeds, rng_seed);
}

int trl_pack_from_args(int argc, const char* const* argv, const char* data_root, const char* out_path) {
    ScenePack pack;
    try {
        build_scene_from_args(argc, argv, data_root ? data_root : "", &pack);
    } catch (const std::exception& e) {
        return fail(e.what());
    }
    std::string err;
    if (!pack.save(out_path, &err)) return fail(err);
    return 0;
}

trl_handle* trl_create_common(trl_handle* h, int num_envs, int device, int mode, const uint64_t* terrain_seeds, uint64_t rng_seed) {
    auto bail = [&](const std::string& why) -> trl_handle* {
        if (!why.empty()) g_err = why;
        trl_destroy(h);
        return nullptr;
    };
    h->device = device; h->n = num_envs; h->mode = mode;
    if (num_envs <= 0) return bail("num_envs must be positive");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
        return bail("terrainrl_b200 needs a CUDA device: no GPU visible (the product path has no CPU fallback)");
    if (g_device >= 0 && g_device != device)
        return bail("terrainrl_b200 drives one GPU per process (device " + std::to_string(g_device) + " is in use): start one process per GPU");
    if (cudaSetDevice(device) != cudaSuccess) return bail("cudaSetDevice failed");
    g_device = device;
    if (fill_model(h, rng_seed)) return bail("");
    if (cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking) != cudaSuccess) return bail("cudaStreamCreate failed");
    {
        int lo = 0, hi = 0;
        cudaDeviceGetStreamPriorityRange(&lo, &hi);   // hi = numerically lowest = greatest priority
        const char* lg = std::getenv("TRL_LAG");
        if (lg && lg[0]) h->lag = std::min(kMaxLists - 1, std::max(1, std::atoi(lg)));
        for (int k = 0; k < h->lag; ++k)
            if (cudaStreamCreateWithPriority(&h->side[k], cudaStreamNonBlocking, hi) != cudaSuccess) return bail("cudaStreamCreate (side) failed");
        h->aux_stream = h->side[0];
        const char* gr = std::getenv("TRL_GROUPS");
        if (gr && gr[0]) h->groups = std::min(kMaxGroups, std::max(1, std::atoi(gr)));     // default 2
        while (h->groups > 1 && group_chunk(num_envs, h->groups) * (h->groups - 1) >= num_envs) --h->groups;   // no empty group
        for (int g = 1; g < h->groups; ++g)
            if (cudaStreamCreateWithFlags(&h->group_stream[g - 1], cudaStreamNonBlocking) != cudaSuccess) return bail("cudaStreamCreate (group) failed");
        const char* serial = std::getenv("TRL_SERIAL_SCHEDULE");
        h->overlap = !(serial && serial[0] == '1');
    }
    auto ck = [&](cudaError_t e, const char* what) -> bool {
        if (e != cudaSuccess) { g_err = std::string(what) + ": " + cudaGetErrorString(e); return false; }
        return true;
    };
    g_model_owner = nullptr;
    if (ensure_model(h)) return bail("upload_model failed");
    if (!ck(configure_step_kernels(), "configure_step_kernels") || !ck(trl_cg::configure_step_kernels(), "configure_step_kernels") ||
        !ck(trl_ts::configure_step_kernels(), "configure_step_kernels") || !ck(trl_ts_cg::configure_step_kernels(), "configure_step_kernels") ||
        !ck(trl_ps::configure_step_kernels(), "configure_step_kernels") || !ck(trl_ps_cg::configure_step_kernels(), "configure_step_kernels") ||
        !ck(trl_bs::configure_step_kernels(), "configure_step_kernels") || !ck(trl_bs_cg::configure_step_kernels(), "configure_step_kernels"))
        return bail("");
    if (!ck(configure_decide_kernel(), "configure_decide_kernel")) return bail("");
    if (!ck(configure_decide2_kernels(), "configure_decide2_kernels")) return bail("");
    {
        const char* v1 = std::getenv("TRL_DECIDE_V1");
        h->decide_v2 = !(v1 && v1[0] == '1');
    }
    Buffers& B = h->B;
    std::memset(&B, 0, sizeof(B));
    const size_t n = (size_t)num_envs;
    B.n = num_envs;
    B.S = kNumGroundSamples + 4 * h->mc.nj - 1;
    B.A = 1 + h->mc.n_opt;
    const int A = 1 + h->mc.n_opt;
    // an env finishes at most one cycle per outer update; twice that leaves room for the bursts of a synchronised start while a
    // fixed-size exchange block (trl_gather_tuples) drains the queue
    B.tuple_cap = std::max(4096, 2 * num_envs);
    B.dist_cap = std::max(65536, 16 * num_envs);
    bool ok = ck(dalloc(h, &B.d, (size_t)D_NUM_FIELDS * n), "alloc d") && ck(dalloc(h, &B.i, (size_t)I_NUM_PLANES * n), "alloc i") &&
              ck(dalloc(h, &B.terrain, n * 2 * kTerrainCap), "alloc terrain") && ck(dalloc(h, &B.poli_state, n * B.S), "alloc poli") &&
              ck(dalloc(h, &B.net_out, n * kMaxNetOut), "alloc net_out") && ck(dalloc(h, &B.tuple_sbeg, n * B.S), "alloc sbeg") &&
              ck(dalloc(h, &B.tuple_action, n * kNumParams), "alloc action") && ck(dalloc(h, &B.com_stash, 2 * n), "alloc com") &&
              ck(dalloc(h, &B.pending_list, (size_t)(h->lag + 1) * n), "alloc pending") && ck(dalloc(h, &B.pending_count, kMaxLists), "alloc pc") &&
              ck(dalloc(h, &B.catchup_done, kMaxLists + 1), "alloc cd") &&
              ck(dalloc(h, &B.tuples, (size_t)B.tuple_cap * (1 + B.S + A + B.S)), "alloc tuples") &&
              ck(dalloc(h, &B.tuple_flags, (size_t)B.tuple_cap), "alloc tf") && ck(dalloc(h, &B.tuple_env, (size_t)B.tuple_cap), "alloc te") &&
              ck(dalloc(h, &B.tuple_count, 1), "alloc tc") && ck(dalloc(h, &B.dist_log, (size_t)B.dist_cap), "alloc dl") &&
              ck(dalloc(h, &B.dist_env, (size_t)B.dist_cap), "alloc de") && ck(dalloc(h, &B.dist_count, 1), "alloc dc") &&
              ck(dalloc(h, &h->done_count, 1), "alloc done") && ck(dalloc(h, &h->d_ex, (size_t)kMaxPolicySlots), "alloc ex");
    for (int k = 0; ok && h->mc.has_net && k < h->lag; ++k) ok = ck(dalloc(h, &h->act2[k], n * (size_t)5984), "alloc act2");
    if (ok) ok = ck(cudaMemcpy(h->d_ex, h->ex, sizeof(h->ex), cudaMemcpyHostToDevice), "upload ex");
    if (!ok) return bail("");
    if (h->mc.has_net) {
        const double* blobs[26];
        int64_t counts[26];
        for (int l = 0; l < 13; ++l) {
            const auto& w = h->scene.f64(std::string("net_") + kNetLayers[l] + "_w");
            const auto& b = h->scene.f64(std::string("net_") + kNetLayers[l] + "_b");
            blobs[2 * l] = w.data(); counts[2 * l] = (int64_t)w.size();
            blobs[2 * l + 1] = b.data(); counts[2 * l + 1] = (int64_t)b.size();
        }
        const char* vn[4] = {"net_in_offset", "net_in_scale", "net_out_offset", "net_out_scale"};
        const double* vecs[4];
        int64_t vcounts[4];
        for (int k = 0; k < 4; ++k) { const auto& v = h->scene.f64(vn[k]); vecs[k] = v.data(); vcounts[k] = (int64_t)v.size(); }
        if (check_net_counts(h->mc, counts, vcounts)) return bail("");
        if (upload_net(h, blobs, counts, vecs, vcounts)) return bail("");
    } else {
        std::memset(&h->W, 0, sizeof(h->W));
    }
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) == cudaSuccess) h->decide_grid = 8 * std::max(1, (2 * prop.multiProcessorCount) / 8);
    if (trl_seed_terrain(h, terrain_seeds, terrain_seeds ? num_envs : 0)) return bail("");
    return h;
}

int trl_destroy(trl_handle* h) {
    if (!h) return 0;
    if (h->comm) trl_comm_destroy(h);
    if (h->trainer) trl_trainer_orphan(h->trainer);   // the trainer object outlives its scenario as an inert shell
    for (int p = 1; p < kMaxPolicySlots; ++p)
        if (h->slot_trainer[p]) trl_trainer_orphan(h->slot_trainer[p]);
    if (g_model_owner == h) g_model_owner = nullptr;
    if (h->stream) cudaStreamSynchronize(h->stream);
    destroy_graphs(h);
    if (h->copy_stream) { cudaStreamSynchronize(h->copy_stream); cudaStreamDestroy(h->copy_stream); }
    if (h->snap_ready) cudaEventDestroy(h->snap_ready);
    if (h->snap_copied) cudaEventDestroy(h->snap_copied);
    if (h->snap_host) cudaFreeHost(h->snap_host);
    for (void* p : h->allocs) cudaFree(p);
    for (int k = 0; k < 8; ++k)
        if (h->side[k]) { cudaStreamSynchronize(h->side[k]); cudaStreamDestroy(h->side[k]); }
    for (int g = 0; g < kMaxGroups - 1; ++g)
        if (h->group_stream[g]) { cudaStreamSynchronize(h->group_stream[g]); cudaStreamDestroy(h->group_stream[g]); }
    for (auto e : h->fork_events) cudaEventDestroy(e);
    if (h->stream) cudaStreamDestroy(h->stream);
    delete h;
    return 0;
}

int trl_seed_terrain(trl_handle* h, const uint64_t* seeds, int n) {
    if (!h) return fail("trl_seed_terrain: null handle");
    if (ensure_model(h)) return fail("model upload failed");
    uint64_t* d_seeds = nullptr;
    if (seeds) {
        if (n != h->n) return fail("trl_seed_terrain: need one seed per env");
        CK(cudaMalloc((void**)&d_seeds, (size_t)n * 8));
        cudaError_t e = cudaMemcpyAsync(d_seeds, seeds, (size_t)n * 8, cudaMemcpyHostToDevice, h->stream);
        if (e != cudaSuccess) { cudaFree(d_seeds); return fail(std::string("trl_seed_terrain: ") + cudaGetErrorString(e)); }
    }
    cudaError_t e = cudaMemsetAsync(h->B.pending_count, 0, kMaxLists * 4, h->stream);
    if (e == cudaSuccess) {
        reset_launch(h, d_seeds, nullptr, h->n, 1);
        h->launches += 1;
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaStreamSynchronize(h->stream);
    if (d_seeds) cudaFree(d_seeds);
    if (e != cudaSuccess) return fail(std::string("trl_seed_terrain: ") + cudaGetErrorString(e));
    return 0;
}

int trl_reset(trl_handle* h, const int32_t* env_ids, int n) {
    if (!h) return fail("trl_reset: null handle");
    if (ensure_model(h)) return fail("model upload failed");
    int* d_ids = nullptr;
    int count = h->n;
    if (env_ids) {
        if (n < 0 || n > h->n) return fail("trl_reset: env count out of range");
        for (int k = 0; k < n; ++k)
            if (env_ids[k] < 0 || env_ids[k] >= h->n) return fail("trl_reset: env id out of range");
        if (n == 0) return 0;
        count = n;
        CK(cudaMalloc((void**)&d_ids, (size_t)n * 4));
        cudaError_t e = cudaMemcpyAsync(d_ids, env_ids, (size_t)n * 4, cudaMemcpyHostToDevice, h->stream);
        if (e != cudaSuccess) { cudaFree(d_ids); return fail(std::string("trl_reset: ") + cudaGetErrorString(e)); }
    }
    reset_launch(h, nullptr, d_ids, count, 0);
    h->launches += 1;
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaStreamSynchronize(h->stream);
    if (d_ids) cudaFree(d_ids);
    if (e != cudaSuccess) return fail(std::string("trl_reset: ") + cudaGetErrorString(e));
    return 0;
}

int trl_update(trl_handle* h, double dt) {
    if (!h) return fail("trl_update: null handle");
    if (ensure_model(h)) return fail("model upload failed");
    if (!(dt > 0)) return 0;
    const int nlaunch = update_launches(h, h->overlap);
    if (h->use_graph) {
        long long key;
        std::memcpy(&key, &dt, 8);
        auto it = h->graphs.find(key);
        if (it == h->graphs.end()) {
            cudaGraph_t graph;
            CK(cudaStreamBeginCapture(h->stream, cudaStreamCaptureModeThreadLocal));
            enqueue_update(h, dt, h->overlap);
            CK(cudaStreamEndCapture(h->stream, &graph));
            cudaGraphExec_t exec;
            CK(cudaGraphInstantiate(&exec, graph, 0));
            cudaGraphDestroy(graph);
            it = h->graphs.emplace(key, exec).first;
        }
        CK(cudaGraphLaunch(it->second, h->stream));
    } else {
        enqueue_update(h, dt, h->overlap);
        CK(cudaGetLastError());
    }
    h->launches += nlaunch;
    return 0;
}

int trl_env_step(trl_handle* h, double step) {
    if (!h) return fail("trl_env_step: null handle");
    if (ensure_model(h)) return fail("model upload failed");
    step_launch(h, step, 2, 0, h->stream);
    enqueue_decide(h, 0, 1, h->stream);
    step_launch(h, step, 1, 0, h->stream);
    h->launches += 2 + num_decide_launches(h);
    CK(cudaGetLastError());
    return 0;
}

int trl_sync(trl_handle* h) {
    if (!h) return fail("trl_sync: null handle");
    CK(cudaStreamSynchronize(h->stream));
    int fault = 0;
    CK(cudaMemcpy(&fault, h->B.catchup_done + kMaxLists, 4, cudaMemcpyDeviceToHost));
    if (fault)
        return fail("an env finished a gait cycle inside a catch-up launch (cycle shorter than three env-steps): the overlapped schedule "
                    "cannot serve it; run with TRL_SERIAL_SCHEDULE=1");
    return 0;
}

int trl_set_explore(trl_handle* h, int enable, double rate, double temp, double base_rate) {
    if (!h) return fail("trl_set_explore: null handle");
    // the decision kernel reads the settings from device memory, so annealing them every update (cScenarioTrain::CalcExpRate
    // ...) neither re-captures the update graph nor drains the stream: the copy is ordered behind the work already queued
    for (ExpSettings& e : h->ex) { e.enable = enable; e.rate = rate; e.temp = temp; e.base_rate = base_rate; }
    CK(cudaMemcpyAsync(h->d_ex, h->ex, sizeof(h->ex), cudaMemcpyHostToDevice, h->stream));
    return 0;
}
// the settings of the envs on policy slot `slot` only (slot 0: also those of every single-policy decision); the same ordering as
// trl_set_explore.  An entry of a slot that holds no policy yet is kept for the policy it will hold
int trl_set_explore_slot(trl_handle* h, int slot, int enable, double rate, double temp, double base_rate) {
    if (!h) return fail("trl_set_explore_slot: null handle");
    if (slot < 0 || slot >= kMaxPolicySlots)
        return fail("trl_set_explore_slot: slot " + std::to_string(slot) + " out of range (0.." + std::to_string(kMaxPolicySlots - 1) + ")");
    ExpSettings& e = h->ex[slot];
    e.enable = enable; e.rate = rate; e.temp = temp; e.base_rate = base_rate;
    CK(cudaMemcpyAsync(h->d_ex + slot, &e, sizeof(ExpSettings), cudaMemcpyHostToDevice, h->stream));
    return 0;
}

// ---------------------------------------------------------------------------------------------- model files
static const char* kDeployLayers[27] = {"slice0", "terr_conv0", "terr_relu0", "terr_conv1", "terr_relu1", "terr_conv2", "terr_relu2",
                                        "terr_ip0", "terr_relu3", "char_flatten0", "concat0", "ip0", "relu0", "relu0_relu0_0_split",
                                        "val_ip0", "val_relu0", "val_ip1", "a0_ip0", "a0_relu0", "a0_ip1", "a1_ip0", "a1_relu0", "a1_ip1",
                                        "a2_ip0", "a2_relu0", "a2_ip1", "output"};
// Caffe blob shapes of the 13 parameter layers (weights; the bias of each is [num_output])
static std::vector<std::vector<uint64_t>> mace_weight_dims(int n_char, int n_frags, int frag) {
    std::vector<std::vector<uint64_t>> d = {{16, 1, 1, 8}, {32, 16, 1, 4}, {32, 32, 1, 4}, {64, 32 * 187}, {256, (uint64_t)(64 + n_char)}};
    for (int hd = 0; hd < 4; ++hd) { d.push_back({128, 256}); d.push_back({(uint64_t)(hd == 0 ? n_frags : frag), 128}); }
    return d;
}
// cNeuralNet::OutputModel for host-side weights: blobs[26] in layer order (w, b per layer)
int trl_write_model(const char* path, const double* const* blobs, int n_char, int n_frags, int frag, const double* in_off,
                    const double* in_scale, const double* out_off, const double* out_scale, uint32_t mtime) {
    try {
        auto dims = mace_weight_dims(n_char, n_frags, frag);
        std::map<std::string, std::vector<H5Writer::Blob>> named;
        for (int l = 0; l < 13; ++l)
            named[kNetLayers[l]] = {H5Writer::Blob{dims[l], blobs[2 * l]}, H5Writer::Blob{{dims[l][0]}, blobs[2 * l + 1]}};
        std::vector<std::string> layers(kDeployLayers, kDeployLayers + 27);
        std::vector<uint8_t> img = H5Writer::build(layers, named, mtime);
        const std::string p = path;
        write_file(p, img.data(), img.size());
        const size_t dot = p.find_last_of('.');
        const int n_in = 200 + n_char, n_out = n_frags * (1 + frag);
        write_scale_file((dot == std::string::npos ? p : p.substr(0, dot)) + "_scale.txt", in_off, in_scale, n_in, out_off, out_scale, n_out);
    } catch (const std::exception& e) {
        return fail(e.what());
    }
    return 0;
}
static int drain(trl_handle* h);
// the policy the scenario currently evaluates (the attached trainer's net if there is one)
int trl_output_model(trl_handle* h, const char* path, uint32_t mtime) {
    if (!h) return fail("trl_output_model: null handle");
    return trl_output_model_slot(h, 0, path, mtime);
}
// the policy of slot `slot` (its trainer's net if it has one)
int trl_output_model_slot(trl_handle* h, int slot, const char* path, uint32_t mtime) {
    if (!h) return fail("trl_output_model_slot: null handle");
    if (!h->mc.has_net) return fail("trl_output_model: scene has no policy net");
    if (slot < 0 || slot >= kMaxPolicySlots) return fail("trl_output_model_slot: slot " + std::to_string(slot) + " out of range");
    if (slot > 0 && h->slot_blobs[slot].empty()) return fail("trl_output_model_slot: slot " + std::to_string(slot) + " is empty");
    if (drain(h)) return 1;
    const NetWeights& W = slot == 0 ? h->W : h->slot_W[slot];
    const double* dev[30] = {W.conv0_w, W.conv0_b, W.conv1_w, W.conv1_b, W.conv2_w, W.conv2_b, W.tip0_w, W.tip0_b, W.ip0_w, W.ip0_b};
    for (int k = 0; k < 4; ++k) { dev[10 + 4 * k] = W.h0_w[k]; dev[11 + 4 * k] = W.h0_b[k]; dev[12 + 4 * k] = W.h1_w[k]; dev[13 + 4 * k] = W.h1_b[k]; }
    dev[26] = W.in_off; dev[27] = W.in_scale; dev[28] = W.out_off; dev[29] = W.out_scale;
    std::vector<std::vector<double>> host(30);
    const double* ptr[30];
    for (int i = 0; i < 30; ++i) {
        host[i].resize((size_t)h->net_counts[i]);
        CK(cudaMemcpy(host[i].data(), dev[i], host[i].size() * 8, cudaMemcpyDeviceToHost));
        ptr[i] = host[i].data();
    }
    return trl_write_model(path, ptr, h->mc.n_char, h->mc.n_frags, h->mc.frag, ptr[26], ptr[27], ptr[28], ptr[29], mtime);
}
int trl_trainer_set_theta(trl_trainer* t, const double* theta);
// cNeuralNet::LoadModel + LoadScale (learning/NeuralNet.cpp:157-186): reads Caffe HDF5 weights + `_scale.txt` and hands the 26 blobs and
// the four offset / scale vectors (lengths checked against the scene's net) to use(blobs, counts, vec)
extern "C++" {
template <typename Use>
static int read_model_files(trl_handle* h, const std::string& who, const char* h5_path, const char* scale_path, Use&& use) {
    try {
        H5Reader h5(h5_path);
        const auto& ds = h5.datasets();
        const double* blobs[26];
        int64_t counts[26];
        for (int l = 0; l < 13; ++l)
            for (int k = 0; k < 2; ++k) {
                auto it = ds.find(std::string("/data/") + kNetLayers[l] + "/" + std::to_string(k));
                if (it == ds.end()) return fail(who + ": missing dataset for layer " + kNetLayers[l]);
                blobs[2 * l + k] = it->second.data(); counts[2 * l + k] = (int64_t)it->second.size();
            }
        JValue sc = load_json(scale_path);
        const char* keys[4] = {"InputOffset", "InputScale", "OutputOffset", "OutputScale"};
        std::vector<double> vec[4];
        for (int k = 0; k < 4; ++k) {
            const JValue* v = sc.get(keys[k]);
            if (!v || v->type != JValue::Arr) return fail(who + ": scale file lacks " + keys[k]);
            for (auto& e : v->arr) vec[k].push_back(e.num);
            const size_t want = (size_t)(k < 2 ? h->mc.n_in : h->mc.n_out);
            if (vec[k].size() != want)
                return fail(who + ": " + keys[k] + " has " + std::to_string(vec[k].size()) + " entries, the net needs " + std::to_string(want));
        }
        return use((const double* const*)blobs, (const int64_t*)counts, vec);
    } catch (const std::exception& e) {
        return fail(e.what());
    }
}
}  // extern "C++"
int trl_load_model(trl_handle* h, const char* h5_path, const char* scale_path) {
    if (!h) return fail("trl_load_model: null handle");
    if (!h->mc.has_net) return fail("trl_load_model: scene has no policy net");
    if (h->trainer) return fail("trl_load_model: a trainer owns the policy weights (load before trl_trainer_create)");
    return read_model_files(h, "trl_load_model", h5_path, scale_path, [&](const double* const* blobs, const int64_t* counts, std::vector<double>* vec) {
        return trl_set_weights(h, blobs, counts, 26, vec[0].data(), vec[1].data(), vec[2].data(), vec[3].data());
    });
}

// every stream of the handle idle (the overlapped schedule leaves decisions and catch-up launches on the side streams, env groups on theirs)
static int drain(trl_handle* h) {
    CK(cudaStreamSynchronize(h->stream));
    for (int k = 0; k < h->lag; ++k) CK(cudaStreamSynchronize(h->side[k]));
    for (int g = 0; g < kMaxGroups - 1; ++g)
        if (h->group_stream[g]) CK(cudaStreamSynchronize(h->group_stream[g]));
    return 0;
}

// the slot machinery, allocated with a handle's first slot >= 1: per-env slots (all 0), weight table, sort scratch and chunk tables
static int ensure_policy_slots(trl_handle* h) {
    if (h->P.W) return 0;
    PolicySlots& P = h->P;
    int* env_slot = nullptr;
    NetWeights* table = nullptr;
    const size_t n = (size_t)h->n;
    P.chunk_cap = h->n / 32 + kMaxPolicySlots;
    CK(dalloc(h, &env_slot, n));
    CK(dalloc(h, &table, (size_t)kMaxPolicySlots));
    CK(dalloc(h, &P.sort_tmp, (size_t)h->lag * n));
    CK(dalloc(h, &P.chunks, (size_t)h->lag * (1 + 3 * P.chunk_cap)));
    P.env_slot = env_slot; P.W = table;
    h->env_slot_host.assign(n, 0);
    return 0;
}

int trl_stage_slot_model(trl_handle* h, int slot, const char* h5_path, const char* scale_path) {
    const int64_t vcounts[4] = {h->mc.n_in, h->mc.n_in, h->mc.n_out, h->mc.n_out};
    if (h5_path && scale_path)
        return read_model_files(h, "trl_trainer_create_slot", h5_path, scale_path, [&](const double* const* blobs, const int64_t* counts, std::vector<double>* vec) {
            if (check_net_counts(h->mc, counts, vcounts)) return 1;
            if (drain(h) || ensure_policy_slots(h)) return 1;
            const double* vecs[4] = {vec[0].data(), vec[1].data(), vec[2].data(), vec[3].data()};
            return upload_net(h, blobs, counts, vecs, vcounts, slot);
        });
    // a copy of the net slot 0 evaluates now (its trainer's, if it has one)
    if (drain(h) || ensure_policy_slots(h)) return 1;
    std::vector<double*>& dst = h->slot_blobs[slot];
    if (dst.empty()) {
        dst.assign(30, nullptr);
        for (int i = 0; i < 30; ++i) CK(dalloc(h, &dst[i], (size_t)h->net_counts[i]));
    }
    const NetWeights& W = h->W;
    const double* src[30] = {W.conv0_w, W.conv0_b, W.conv1_w, W.conv1_b, W.conv2_w, W.conv2_b, W.tip0_w, W.tip0_b, W.ip0_w, W.ip0_b};
    for (int k = 0; k < 4; ++k) { src[10 + 4 * k] = W.h0_w[k]; src[11 + 4 * k] = W.h0_b[k]; src[12 + 4 * k] = W.h1_w[k]; src[13 + 4 * k] = W.h1_b[k]; }
    src[26] = W.in_off; src[27] = W.in_scale; src[28] = W.out_off; src[29] = W.out_scale;
    for (int i = 0; i < 30; ++i) CK(cudaMemcpy(dst[i], src[i], (size_t)h->net_counts[i] * 8, cudaMemcpyDeviceToDevice));
    double** b = dst.data();
    h->slot_W[slot] = net_weights(b, b[26], b[27], b[28], b[29]);
    return 0;
}

static bool slot_loaded(const trl_handle* h, int slot) { return slot == 0 || (slot > 0 && slot < kMaxPolicySlots && !h->slot_blobs[slot].empty()); }

int trl_load_policy(trl_handle* h, int slot, const char* h5_path, const char* scale_path) {
    if (!h) return fail("trl_load_policy: null handle");
    if (slot < 1 || slot >= kMaxPolicySlots)
        return fail("trl_load_policy: slot " + std::to_string(slot) + " out of range (1.." + std::to_string(kMaxPolicySlots - 1) + "; slot 0 is trl_load_model's)");
    if (!h->mc.has_net) return fail("trl_load_policy: scene has no policy net");
    if (h->mode != TRL_MODE_POLI_EVAL) return fail("trl_load_policy: policy slots are for evaluation handles (TRL_MODE_POLI_EVAL)");
    if (h->trainer) return fail("trl_load_policy: a trainer is attached (it trains slot 0 in place; slots are for evaluation)");
    if (!h->decide_v2) return fail("trl_load_policy: the TRL_DECIDE_V1 decision kernel has no policy slots");
    if (!h5_path || !scale_path) return fail("trl_load_policy: null path");
    return read_model_files(h, "trl_load_policy", h5_path, scale_path, [&](const double* const* blobs, const int64_t* counts, std::vector<double>* vec) {
        const int64_t vcounts[4] = {h->mc.n_in, h->mc.n_in, h->mc.n_out, h->mc.n_out};
        if (check_net_counts(h->mc, counts, vcounts)) return 1;
        if (drain(h)) return 1;
        if (ensure_policy_slots(h)) return 1;
        const double* vecs[4] = {vec[0].data(), vec[1].data(), vec[2].data(), vec[3].data()};
        if (upload_net(h, blobs, counts, vecs, vcounts, slot)) return 1;
        h->slots_active = true;
        h->slot_dirty = true;
        return ensure_model(h) ? fail("trl_load_policy: slot table upload failed") : 0;
    });
}

int trl_set_env_policy(trl_handle* h, const int32_t* env_ids, const int32_t* slots, int n) {
    if (!h) return fail("trl_set_env_policy: null handle");
    if (n < 0 || n > h->n) return fail("trl_set_env_policy: env count out of range");
    if (n > 0 && !slots) return fail("trl_set_env_policy: null slot list");
    for (int k = 0; k < n; ++k) {
        const int e = env_ids ? env_ids[k] : k;
        if (e < 0 || e >= h->n) return fail("trl_set_env_policy: env id " + std::to_string(e) + " out of range");
        if (slots[k] < 0 || slots[k] >= kMaxPolicySlots) return fail("trl_set_env_policy: slot " + std::to_string(slots[k]) + " out of range");
        if (!slot_loaded(h, slots[k])) return fail("trl_set_env_policy: slot " + std::to_string(slots[k]) + " is empty (trl_load_policy first)");
    }
    if (!h->slots_active) return 0;      // only slot 0 exists, and every env is on it
    std::vector<int> next = h->env_slot_host;
    for (int k = 0; k < n; ++k) next[env_ids ? env_ids[k] : k] = slots[k];
    if (drain(h)) return 1;
    std::vector<int32_t> moved;
    if (h->train_slots) {
        // every tuple belongs to the slot that chose its action: no move while the block holds tuples, and a moved env starts over
        // (cScenarioExp::Reset zeroes its cycle count, so its unfinished cycle records no tuple)
        int held = 0;
        CK(cudaMemcpy(&held, h->B.tuple_count, 4, cudaMemcpyDeviceToHost));
        if (held != 0)
            return fail("trl_set_env_policy: the tuple block holds " + std::to_string(held) + " tuples of the present assignment (hand them over or trl_reset_tuples first)");
        for (int e = 0; e < h->n; ++e)
            if (next[e] != h->env_slot_host[e]) moved.push_back(e);
    }
    CK(cudaMemcpy((void*)h->P.env_slot, next.data(), next.size() * 4, cudaMemcpyHostToDevice));
    h->env_slot_host.swap(next);
    return moved.empty() ? 0 : trl_reset(h, moved.data(), (int)moved.size());
}

static bool terrain_loaded(const trl_handle* h, int slot) { return slot == 0 || (slot > 0 && slot < kMaxTerrainSlots && h->terrain_loaded[slot]); }

int trl_load_terrain(trl_handle* h, int slot, const char* terrain_json_path) {
    if (!h) return fail("trl_load_terrain: null handle");
    if (slot < 1 || slot >= kMaxTerrainSlots)
        return fail("trl_load_terrain: slot " + std::to_string(slot) + " out of range (1.." + std::to_string(kMaxTerrainSlots - 1) + "; slot 0 is the scene's terrain)");
    if (!terrain_json_path) return fail("trl_load_terrain: null path");
    TerrainFile tf;
    try {
        tf = read_terrain_file(terrain_json_path);
    } catch (const std::exception& e) {
        return fail(std::string("trl_load_terrain: ") + e.what());
    }
    return trl_set_terrain_slot(h, slot, tf.type, std::move(tf.params));
}

int trl_set_env_terrain(trl_handle* h, const int32_t* env_ids, const int32_t* slots, int n) {
    if (!h) return fail("trl_set_env_terrain: null handle");
    if (n < 0 || n > h->n) return fail("trl_set_env_terrain: env count out of range");
    if (n > 0 && !slots) return fail("trl_set_env_terrain: null slot list");
    for (int k = 0; k < n; ++k) {
        const int e = env_ids ? env_ids[k] : k;
        if (e < 0 || e >= h->n) return fail("trl_set_env_terrain: env id " + std::to_string(e) + " out of range");
        if (slots[k] < 0 || slots[k] >= kMaxTerrainSlots) return fail("trl_set_env_terrain: slot " + std::to_string(slots[k]) + " out of range");
        if (!terrain_loaded(h, slots[k])) return fail("trl_set_env_terrain: slot " + std::to_string(slots[k]) + " is empty (trl_load_terrain first)");
    }
    if (h->env_terrain_host.empty()) return 0;      // only slot 0 exists, and every env is on it
    std::vector<int> next = h->env_terrain_host;
    for (int k = 0; k < n; ++k) next[env_ids ? env_ids[k] : k] = slots[k];
    if (drain(h)) return 1;
    CK(cudaMemcpy(h->B.i + (size_t)I_TERRAIN_SLOT_NEXT * h->n, next.data(), next.size() * 4, cudaMemcpyHostToDevice));
    h->env_terrain_host.swap(next);
    return 0;
}

int trl_env_terrain(trl_handle* h, int32_t* current, int32_t* assigned, int n) {
    if (!h) return fail("trl_env_terrain: null handle");
    if (n < 0 || n > h->n) return fail("trl_env_terrain: env count out of range");
    if (drain(h)) return 1;
    const size_t N = (size_t)h->n;
    if (current && n > 0) CK(cudaMemcpy(current, h->B.i + (size_t)I_TERRAIN_SLOT * N, (size_t)n * 4, cudaMemcpyDeviceToHost));
    if (assigned && n > 0) CK(cudaMemcpy(assigned, h->B.i + (size_t)I_TERRAIN_SLOT_NEXT * N, (size_t)n * 4, cudaMemcpyDeviceToHost));
    return 0;
}
// the policy slot of envs 0 .. n-1 (all 0 while only slot 0 exists)
int trl_env_policy(trl_handle* h, int32_t* slots, int n) {
    if (!h) return fail("trl_env_policy: null handle");
    if (n < 0 || n > h->n) return fail("trl_env_policy: env count out of range");
    for (int k = 0; k < n; ++k) slots[k] = h->slots_active ? h->env_slot_host[k] : 0;
    return 0;
}
int trl_get_output_offset_scale(trl_handle* h, double* off, double* scale, int n);
// the same for a scene pack, without a device (host-only: parses the pack and the controller tables); used to check the
// restatement against the reference's own compiled BuildNNOutputOffsetScale (tests/test_ref_pinning_cpu.py)
int trl_pack_output_offset_scale(const char* pack_path, double* off, double* scale, int n) {
    trl_handle h;
    std::string err;
    if (!h.scene.load(pack_path, &err)) return fail(err);
    if (fill_model(&h, 0)) return 1;
    return trl_get_output_offset_scale(&h, off, scale, n);
}

// cBaseControllerMACE::BuildNNOutputOffsetScale (sim/BaseControllerMACE.cpp:75-113,131-167): critic outputs offset -0.5 scale 2;
// actor f centred on the optimised parameters of control set f % n_ctrl (cDogControllerMACE::BuildActorBias) and scaled by
// 1 / max_a |opt(a) - opt(default action)| over the action library
int trl_get_output_offset_scale(trl_handle* h, double* off, double* scale, int n) {
    if (!h) return fail("trl_get_output_offset_scale: null handle");
    const ModelConst& m = h->mc;
    const int fs = m.n_opt, nf = m.has_net ? m.n_frags : 0;
    if (n != nf * (1 + fs)) return fail("trl_get_output_offset_scale: size mismatch");
    auto ctrl_opt = [&](int set, int k) {
        const int idx = m.opt_idx[k];
        double v = m.ctrl_params[set][idx];
        if (idx == 0 || idx == 1 || (m.char_type == 2 && idx == 2)) v = std::fabs(v);     // PostProcessParams (TransTime, Cv, raptor Cd)
        return v;
    };
    auto action_opt = [&](int a, int k) {
        const double b = m.act_blend[a];
        return (1.0 - b) * ctrl_opt(m.act_idx0[a], k) + b * ctrl_opt(m.act_idx1[a], k);   // BlendCtrlParams + GetOptParams
    };
    std::vector<double> frag_scale(fs, 1.0);
    if (m.n_actions > 1) {
        const int d0 = m.default_action >= 0 ? m.default_action : 0;
        for (int k = 0; k < fs; ++k) {
            double mx = 0;
            for (int a = 0; a < m.n_actions; ++a)
                if (a != d0) mx = std::max(mx, std::fabs(action_opt(a, k) - action_opt(d0, k)));
            frag_scale[k] = mx > 0 ? 1.0 / mx : 1.0;
        }
    }
    for (int f = 0; f < nf; ++f) {
        off[f] = -0.5; scale[f] = 2.0;
        for (int k = 0; k < fs; ++k) { off[nf + f * fs + k] = -ctrl_opt(f % m.n_ctrl, k); scale[nf + f * fs + k] = frag_scale[k]; }
    }
    return 0;
}

// cScenarioSimChar::SetTerrainParamsLerp (scenarios/ScenarioSimChar.cpp:255-272), as cScenarioTrain::UpdateSceneCurriculum calls it
// (scenarios/ScenarioTrain.cpp:412-416): blends the scene's terrain parameter sets; segments generated from now on use the
// blend (cGroundVar2D::SetTerrainParams), existing terrain stays.  Every loaded terrain slot is re-blended at the same `lerp`.
int trl_set_terrain_lerp(trl_handle* h, double lerp) {
    if (!h) return fail("trl_set_terrain_lerp: null handle");
    h->terrain_lerp = lerp;
    const auto& tp = h->scene.f64("terrain_params");
    const auto& td = h->scene.f64("terrain_default_params");
    const int n_sets = (int)(tp.size() / kTerrainParams);
    double blended[kMaxTerrainSlots][kTerrainParams];
    bool same = true;
    if (n_sets > 0) {       // a scene without parameter sets keeps its defaults whatever the blend
        blend_terrain(tp.data(), n_sets, td.data(), lerp, blended[0]);
        same = std::equal(blended[0], blended[0] + kTerrainParams, h->mc.terrain_params);
    }
    for (int s = 1; s < kMaxTerrainSlots; ++s) {
        if (!h->terrain_loaded[s]) continue;
        blend_terrain(h->terrain_sets[s].data(), (int)(h->terrain_sets[s].size() / kTerrainParams), td.data(), lerp, blended[s]);
        same = same && std::equal(blended[s], blended[s] + kTerrainParams, h->terrain[s].params);
    }
    if (same) return 0;      // cScenarioTrain calls this after every trainer step; an unchanged blend must not drain the device
    if (drain(h)) return 1;
    if (n_sets > 0) std::memcpy(h->mc.terrain_params, blended[0], sizeof(blended[0]));
    for (int s = 1; s < kMaxTerrainSlots; ++s)
        if (h->terrain_loaded[s]) std::memcpy(h->terrain[s].params, blended[s], sizeof(blended[s]));
    g_model_owner = nullptr;
    if (ensure_model(h)) return fail("model upload failed");
    return 0;
}

// cScenarioTrain::CalcExpRate / CalcExpTemp / CalcExpBaseRate / CalcCurriculumPhase (scenarios/ScenarioTrain.cpp:418-460).
// sp[9] = {init_exp_rate, exp_rate, init_exp_temp, exp_temp, init_exp_base_rate, exp_base_rate, trainer_num_anneal_iters,
// exp_base_anneal_iters, trainer_curriculum_iters}; out[4] = {exp_rate, exp_temp, exp_base_rate, curriculum_phase}
int trl_train_schedule(const double* sp, int iters, double* out) {
    auto clamp01 = [](double v) { return std::min(std::max(v, 0.0), 1.0); };
    double lerp = clamp01((double)iters / sp[6]);
    out[0] = (1 - lerp) * sp[0] + lerp * sp[1];
    out[1] = (1 - lerp) * sp[2] + lerp * sp[3];
    lerp = clamp01((double)iters / sp[7]);
    out[2] = (1 - lerp) * sp[4] + lerp * sp[5];
    const bool enable = sp[8] >= 1;
    out[3] = clamp01(enable ? (double)iters / sp[8] : 1.0);
    if (iters == 0) out[3] = 1.0;      // gInitCurriculumPhase
    return 0;
}

int trl_set_phys_params(trl_handle* h, const double* p) {
    if (!h) return fail("trl_set_phys_params: null handle");
    CK(cudaStreamSynchronize(h->stream));
    h->mc.phys = PhysParams{p[0], p[1], p[2], p[3], p[4], p[5], p[6], h->mc.phys.vertex_contacts};
    g_model_owner = nullptr;
    if (ensure_model(h)) return fail("model upload failed");
    return 0;
}

int trl_set_weights(trl_handle* h, const double* const* blobs, const int64_t* counts, int nblobs, const double* in_off,
                    const double* in_scale, const double* out_off, const double* out_scale) {
    if (!h) return fail("trl_set_weights: null handle");
    if (nblobs != 26) return fail("trl_set_weights: expected 26 blobs");
    if (!h->mc.has_net) return fail("trl_set_weights: scene has no policy net");
    if (h->trainer) return fail("trl_set_weights: a trainer owns the policy weights (use trl_trainer_set_theta)");
    if (!blobs || !counts || !in_off || !in_scale || !out_off || !out_scale) return fail("trl_set_weights: null argument");
    if (check_net_counts(h->mc, counts, nullptr)) return 1;
    CK(cudaStreamSynchronize(h->stream));
    const double* vecs[4] = {in_off, in_scale, out_off, out_scale};
    int64_t vcounts[4] = {h->mc.n_in, h->mc.n_in, h->mc.n_out, h->mc.n_out};
    if (upload_net(h, blobs, counts, vecs, vcounts)) return 1;
    for (int k = 0; k < h->mc.frag; ++k) h->mc.out_scale_actor0[k] = out_scale[h->mc.n_frags + k];
    g_model_owner = nullptr;
    if (ensure_model(h)) return fail("model upload failed");
    return 0;
}

int trl_sizes(trl_handle* h, int* num_envs, int* state, int* action, int* num_frags, int* frag_size, int* num_dof, int* num_joints) {
    if (!h) return fail("trl_sizes: null handle");
    if (num_envs) *num_envs = h->n;
    if (state) *state = h->B.S;
    if (action) *action = h->B.A;
    if (num_frags) *num_frags = h->mc.n_frags;
    if (frag_size) *frag_size = h->mc.n_opt;
    if (num_dof) *num_dof = h->mc.ndof;
    if (num_joints) *num_joints = h->mc.nj;
    return 0;
}

// The step kernel takes tuple slots from an atomic cursor and refuses rows past tuple_cap (trl_step.cu: exp_new_cycle_update), so the
// cursor itself says how many were refused.  The readers deliver what fits, count the rest in h->tuples_dropped when the block is
// reset, and answer TRL_E_TUPLE_OVERFLOW so that the loss cannot go unnoticed.
static int overflow_error(trl_handle* h, int overflow) {
    g_err = "tuple block overflow: " + std::to_string(overflow) + " tuples were refused (capacity " + std::to_string(h->B.tuple_cap) +
            "); hand the tuples over more often";
    return TRL_E_TUPLE_OVERFLOW;
}
static int fetch_tuples(trl_handle* h, int* n_out, int* overflow) {
    int n = 0;
    CK(cudaMemcpyAsync(&n, h->B.tuple_count, 4, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    *overflow = n > h->B.tuple_cap ? n - h->B.tuple_cap : 0;
    if (n > h->B.tuple_cap) n = h->B.tuple_cap;
    const size_t W = 1 + h->B.S + h->B.A + h->B.S;
    h->h_tuples.resize((size_t)std::max(n, 1) * W);
    h->h_tuple_flags.resize(std::max(n, 1));
    h->h_tuple_env.resize(std::max(n, 1));
    if (n > 0) {
        CK(cudaMemcpyAsync(h->h_tuples.data(), h->B.tuples, (size_t)n * W * 8, cudaMemcpyDeviceToHost, h->stream));
        CK(cudaMemcpyAsync(h->h_tuple_flags.data(), h->B.tuple_flags, (size_t)n * 4, cudaMemcpyDeviceToHost, h->stream));
        CK(cudaMemcpyAsync(h->h_tuple_env.data(), h->B.tuple_env, (size_t)n * 4, cudaMemcpyDeviceToHost, h->stream));
        CK(cudaStreamSynchronize(h->stream));
    }
    *n_out = n;
    return 0;
}

int trl_num_tuples(trl_handle* h, int* out) {
    if (!h) return fail("trl_num_tuples: null handle");
    int n = 0;
    CK(cudaMemcpyAsync(&n, h->B.tuple_count, 4, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    *out = std::min(n, h->B.tuple_cap);
    return n > h->B.tuple_cap ? overflow_error(h, n - h->B.tuple_cap) : 0;
}

int trl_get_tuples_f64(trl_handle* h, const double** rows, const uint32_t** flags, const int32_t** env_id, int* n) {
    if (!h) return fail("trl_get_tuples_f64: null handle");
    int overflow = 0;
    if (fetch_tuples(h, n, &overflow)) return 1;
    *rows = h->h_tuples.data(); *flags = h->h_tuple_flags.data(); *env_id = h->h_tuple_env.data();
    return overflow ? overflow_error(h, overflow) : 0;
}

int trl_get_tuples(trl_handle* h, const float** rows, const uint32_t** flags, const int32_t** env_id, int* n) {
    if (!h) return fail("trl_get_tuples: null handle");
    int overflow = 0;
    if (fetch_tuples(h, n, &overflow)) return 1;
    const size_t W = 1 + h->B.S + h->B.A + h->B.S;
    h->h_tuples_f32.resize((size_t)std::max(*n, 1) * W);
    for (size_t k = 0; k < (size_t)*n * W; ++k) h->h_tuples_f32[k] = (float)h->h_tuples[k];
    *rows = h->h_tuples_f32.data(); *flags = h->h_tuple_flags.data(); *env_id = h->h_tuple_env.data();
    return overflow ? overflow_error(h, overflow) : 0;
}

int trl_reset_tuples(trl_handle* h) {
    if (!h) return fail("trl_reset_tuples: null handle");
    int n = 0;
    CK(cudaMemcpyAsync(&n, h->B.tuple_count, 4, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    if (n > h->B.tuple_cap) h->tuples_dropped += n - h->B.tuple_cap;
    CK(cudaMemsetAsync(h->B.tuple_count, 0, 4, h->stream));
    return 0;
}

// cScenarioPoliEval::ResetAvgDist (scenarios/ScenarioPoliEval.cpp:132-136) for every env: mean distance and episode count back to
// zero, cycle count and distance log kept -- cOptScenarioPoliEval::EvalHelper calls it after each UpdateRecord
// (optimizer/scenarios/OptScenarioPoliEval.cpp:189-195)
int trl_reset_avg_dist(trl_handle* h) {
    if (!h) return fail("trl_reset_avg_dist: null handle");
    const size_t n = (size_t)h->n;
    CK(cudaMemsetAsync(h->B.d + (size_t)D_AVG_DIST * n, 0, n * 8, h->stream));
    CK(cudaMemsetAsync(h->B.i + (size_t)I_EPISODE_COUNT * n, 0, n * 4, h->stream));
    return 0;
}

int trl_eval_stats(trl_handle* h, int64_t* cycles, int64_t* episodes, double* avg_dist, int64_t* env_steps) {
    if (!h) return fail("trl_eval_stats: null handle");
    const size_t n = (size_t)h->n;
    std::vector<int> cyc(n), eps(n), lo(n), hi(n);
    std::vector<double> avg(n);
    CK(cudaStreamSynchronize(h->stream));
    CK(cudaMemcpy(cyc.data(), h->B.i + (size_t)I_CYCLE_COUNT * n, n * 4, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(eps.data(), h->B.i + (size_t)I_EPISODE_COUNT * n, n * 4, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(lo.data(), h->B.i + (size_t)I_STEPS_LO * n, n * 4, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(hi.data(), h->B.i + (size_t)I_STEPS_HI * n, n * 4, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(avg.data(), h->B.d + (size_t)D_AVG_DIST * n, n * 8, cudaMemcpyDeviceToHost));
    int64_t c = 0, e = 0, st = 0;
    double sum = 0;
    for (size_t k = 0; k < n; ++k) {
        c += cyc[k]; e += eps[k]; sum += avg[k] * eps[k];
        st += ((int64_t)hi[k] << 32) | (uint32_t)lo[k];
    }
    if (cycles) *cycles = c;
    if (episodes) *episodes = e;
    if (avg_dist) *avg_dist = e ? sum / e : 0.0;
    if (env_steps) *env_steps = st;
    return 0;
}

// trl_eval_stats over the envs of one (policy slot, terrain slot) cell, -1 = any slot.  A cell that holds every env is trl_eval_stats
// itself; the others come from trl_cell_stats_kernel
static int eval_stats_cell(trl_handle* h, const char* who, int policy_slot, int terrain_slot, int64_t* cycles, int64_t* episodes,
                           double* avg_dist, int64_t* env_steps) {
    if (!h) return fail(std::string(who) + ": null handle");
    if (policy_slot < -1 || policy_slot >= kMaxPolicySlots) return fail(std::string(who) + ": policy slot " + std::to_string(policy_slot) + " out of range");
    if (policy_slot >= 0 && !slot_loaded(h, policy_slot)) return fail(std::string(who) + ": policy slot " + std::to_string(policy_slot) + " is empty");
    if (terrain_slot < -1 || terrain_slot >= kMaxTerrainSlots) return fail(std::string(who) + ": terrain slot " + std::to_string(terrain_slot) + " out of range");
    if (terrain_slot >= 0 && !terrain_loaded(h, terrain_slot)) return fail(std::string(who) + ": terrain slot " + std::to_string(terrain_slot) + " is empty");
    const bool any_p = policy_slot < 0 || !h->slots_active, any_t = terrain_slot < 0 || h->env_terrain_host.empty();
    if (any_p && any_t) return trl_eval_stats(h, cycles, episodes, avg_dist, env_steps);
    if (!h->cell_stats) CK(dalloc(h, &h->cell_stats, (size_t)(kMaxPolicySlots + 1) * (kMaxTerrainSlots + 1) * 4));
    const int cell = (any_p ? kMaxPolicySlots : policy_slot) * (kMaxTerrainSlots + 1) + (any_t ? kMaxTerrainSlots : terrain_slot);
    double st[4];
    launch_cell_stats(h->B, h->slots_active ? h->P.env_slot : nullptr, h->cell_stats, h->stream);
    h->launches += 1;
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(st, h->cell_stats + 4 * cell, sizeof(st), cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    if (cycles) *cycles = (int64_t)st[0];
    if (episodes) *episodes = (int64_t)st[1];
    if (env_steps) *env_steps = (int64_t)st[2];
    if (avg_dist) *avg_dist = st[1] > 0 ? st[3] / st[1] : 0.0;
    return 0;
}

int trl_eval_stats_cell(trl_handle* h, int policy_slot, int terrain_slot, int64_t* cycles, int64_t* episodes, double* avg_dist, int64_t* env_steps) {
    return eval_stats_cell(h, "trl_eval_stats_cell", policy_slot, terrain_slot, cycles, episodes, avg_dist, env_steps);
}

int trl_eval_stats_slot(trl_handle* h, int slot, int64_t* cycles, int64_t* episodes, double* avg_dist, int64_t* env_steps) {
    if (!h) return fail("trl_eval_stats_slot: null handle");
    if (slot < 0 || slot >= kMaxPolicySlots) return fail("trl_eval_stats_slot: slot " + std::to_string(slot) + " out of range");
    return eval_stats_cell(h, "trl_eval_stats_slot", slot, -1, cycles, episodes, avg_dist, env_steps);
}

// policy slot `slot`'s statistics as trl_eval_stats_slot counts them, {cycles, episodes, env-steps, distance sum}, into device memory
// out4 on the handle's stream: the operand of the all-reduce of trl_comm_eval_stats_slot
int trl_slot_stats_dev(trl_handle* h, const char* who, int slot, double* out4) {
    if (slot < 0 || slot >= kMaxPolicySlots) return fail(std::string(who) + ": slot " + std::to_string(slot) + " out of range");
    if (!slot_loaded(h, slot)) return fail(std::string(who) + ": policy slot " + std::to_string(slot) + " is empty");
    if (!h->slots_active) {
        launch_stats(h->B, out4, h->stream);
    } else {
        if (!h->cell_stats) CK(dalloc(h, &h->cell_stats, (size_t)(kMaxPolicySlots + 1) * (kMaxTerrainSlots + 1) * 4));
        launch_cell_stats(h->B, h->P.env_slot, h->cell_stats, h->stream);
        CK(cudaMemcpyAsync(out4, h->cell_stats + 4 * (slot * (kMaxTerrainSlots + 1) + kMaxTerrainSlots), 32, cudaMemcpyDeviceToDevice, h->stream));
    }
    h->launches += 1;
    CK(cudaGetLastError());
    return 0;
}

static bool phys_loaded(const trl_handle* h, int slot) { return slot == 0 || (slot > 0 && slot < kMaxPhysSlots && h->phys_loaded[slot]); }

// physics slot `slot` >= 1 holds `q` (its numbers checked), fixed or (hi non-null) ranged up to *hi, and the handle moves onto the
// physics-slot build
static int set_phys_slot(trl_handle* h, const std::string& who, int slot, const PhysParams& q, const PhysParams* hi = nullptr) {
    if (drain(h)) return 1;
    if (!h->env_phys) {     // first slot: from now on the step launches run the physics-slot build
        int* d = nullptr;
        CK(dalloc(h, &d, 2 * (size_t)h->n));
        h->env_phys = d;
        h->env_phys_host.assign((size_t)h->n, 0);
        destroy_graphs(h);
    }
    h->phys[slot] = q;
    h->phys_loaded[slot] = true;
    if (hi) {
        h->ranges.phys_hi[slot] = *hi;
        h->ranges.phys_ranged |= 1u << slot;
    } else {
        h->ranges.phys_ranged &= ~(1u << slot);
    }
    g_model_owner = nullptr;
    return ensure_model(h) ? fail(who + ": physics table upload failed") : 0;
}

static const char* kPhysNames[7] = {"kn", "dn", "mu", "v_eps", "contact_tol", "k_lim", "d_lim"};

// the checks trl_load_physics makes of a slot's seven constants (`what`: "" or the name of a range's end, for the messages)
static int check_p7(const std::string& who, const double* p, const std::string& what) {
    const char* const* names = kPhysNames;
    for (int k = 0; k < 7; ++k)
        if (!std::isfinite(p[k])) return fail(who + ": " + what + names[k] + " is not finite");
    for (int k : {0, 1, 2, 5, 6})
        if (p[k] < 0.0) return fail(who + ": " + what + names[k] + " = " + std::to_string(p[k]) + " is negative");
    if (!(p[3] > 0.0)) return fail(who + ": " + what + "v_eps = " + std::to_string(p[3]) + " must be positive");
    if (p[4] * std::sqrt(1.0 + kMaxSlope * kMaxSlope) > kClearMargin)
        return fail(who + ": " + what + "contact_tol = " + std::to_string(p[4]) + " exceeds what the broad phase covers (contact_tol * sqrt(1 + 25^2) <= 0.05)");
    return 0;
}

int trl_load_physics(trl_handle* h, int slot, const double* p, int vertex_contacts) {
    const std::string who = "trl_load_physics";
    if (!h) return fail(who + ": null handle");
    if (slot < 1 || slot >= kMaxPhysSlots)
        return fail(who + ": slot " + std::to_string(slot) + " out of range (1.." + std::to_string(kMaxPhysSlots - 1) + "; slot 0 is the scene's physics, set by trl_set_phys_params)");
    if (!p) return fail(who + ": null parameter array");
    if (check_p7(who, p, "")) return 1;
    return set_phys_slot(h, who, slot, PhysParams{p[0], p[1], p[2], p[3], p[4], p[5], p[6], vertex_contacts ? 1 : 0});
}

int trl_set_env_physics(trl_handle* h, const int32_t* env_ids, const int32_t* slots, int n) {
    const std::string who = "trl_set_env_physics";
    if (!h) return fail(who + ": null handle");
    if (n < 0 || n > h->n) return fail(who + ": env count out of range");
    if (n > 0 && !slots) return fail(who + ": null slot list");
    for (int k = 0; k < n; ++k) {
        const int e = env_ids ? env_ids[k] : k;
        if (e < 0 || e >= h->n) return fail(who + ": env id " + std::to_string(e) + " out of range");
        if (slots[k] < 0 || slots[k] >= kMaxPhysSlots) return fail(who + ": slot " + std::to_string(slots[k]) + " out of range");
        if (!phys_loaded(h, slots[k])) return fail(who + ": slot " + std::to_string(slots[k]) + " is empty (trl_load_physics first)");
    }
    if (!h->env_phys) return 0;      // only slot 0 exists, and every env is on it
    std::vector<int> next = h->env_phys_host;
    for (int k = 0; k < n; ++k) next[env_ids ? env_ids[k] : k] = slots[k];
    if (drain(h)) return 1;
    CK(cudaMemcpy(h->env_phys + h->n, next.data(), next.size() * 4, cudaMemcpyHostToDevice));
    h->env_phys_host.swap(next);
    return 0;
}

int trl_env_physics(trl_handle* h, int32_t* current, int32_t* assigned, int n) {
    if (!h) return fail("trl_env_physics: null handle");
    if (n < 0 || n > h->n) return fail("trl_env_physics: env count out of range");
    if (!h->env_phys) {
        for (int k = 0; k < n; ++k) {
            if (current) current[k] = 0;
            if (assigned) assigned[k] = 0;
        }
        return 0;
    }
    if (drain(h)) return 1;
    if (current && n > 0) CK(cudaMemcpy(current, h->env_phys, (size_t)n * 4, cudaMemcpyDeviceToHost));
    if (assigned && n > 0) CK(cudaMemcpy(assigned, h->env_phys + h->n, (size_t)n * 4, cudaMemcpyDeviceToHost));
    return 0;
}

// a cell with any physics slot, or any cell of a handle whose envs are all on physics slot 0, is trl_eval_stats_cell's; the others come
// from trl_phys_stats_kernel.  env_eval (trl_eval_stats_mode): only the envs whose present episode has mode `eval` (1 evaluates)
static int eval_stats_phys(trl_handle* h, const std::string& who, int policy_slot, int terrain_slot, int phys_slot, const int* env_eval, int eval,
                           int64_t* cycles, int64_t* episodes, double* avg_dist, int64_t* env_steps, const int* env_body = nullptr,
                           int body_slot = -1) {
    if (!h) return fail(who + ": null handle");
    if (phys_slot < -1 || phys_slot >= kMaxPhysSlots) return fail(who + ": physics slot " + std::to_string(phys_slot) + " out of range");
    if (phys_slot >= 0 && !phys_loaded(h, phys_slot)) return fail(who + ": physics slot " + std::to_string(phys_slot) + " is empty");
    if (!env_eval && !env_body && (phys_slot < 0 || !h->env_phys))
        return eval_stats_cell(h, who.c_str(), policy_slot, terrain_slot, cycles, episodes, avg_dist, env_steps);
    if (policy_slot < -1 || policy_slot >= kMaxPolicySlots) return fail(who + ": policy slot " + std::to_string(policy_slot) + " out of range");
    if (policy_slot >= 0 && !slot_loaded(h, policy_slot)) return fail(who + ": policy slot " + std::to_string(policy_slot) + " is empty");
    if (terrain_slot < -1 || terrain_slot >= kMaxTerrainSlots) return fail(who + ": terrain slot " + std::to_string(terrain_slot) + " out of range");
    if (terrain_slot >= 0 && !terrain_loaded(h, terrain_slot)) return fail(who + ": terrain slot " + std::to_string(terrain_slot) + " is empty");
    if (!h->phys_stats) CK(dalloc(h, &h->phys_stats, 4));
    double st[4];
    launch_phys_stats(h->B, h->slots_active ? h->P.env_slot : nullptr, h->env_phys, h->slots_active ? policy_slot : -1,
                      h->env_terrain_host.empty() ? -1 : terrain_slot, h->env_phys ? phys_slot : -1, env_eval, eval, env_body, body_slot,
                      h->phys_stats, h->stream);
    h->launches += 1;
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(st, h->phys_stats, sizeof(st), cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    if (cycles) *cycles = (int64_t)st[0];
    if (episodes) *episodes = (int64_t)st[1];
    if (env_steps) *env_steps = (int64_t)st[2];
    if (avg_dist) *avg_dist = st[1] > 0 ? st[3] / st[1] : 0.0;
    return 0;
}

int trl_eval_stats_phys(trl_handle* h, int policy_slot, int terrain_slot, int phys_slot, int64_t* cycles, int64_t* episodes, double* avg_dist,
                        int64_t* env_steps) {
    return eval_stats_phys(h, "trl_eval_stats_phys", policy_slot, terrain_slot, phys_slot, nullptr, 0, cycles, episodes, avg_dist, env_steps);
}

// evaluation envs of an exploration handle: the per-env modes ([2][n]: present episode, next one), the slot build of the decision
// kernels (which turns exploration off for an evaluating env) and the physics-slot build of the step kernels (which keeps an
// evaluating env's episode statistics instead of its tuples).  Called with the handle drained; once made, they stay
int trl_enable_env_eval(trl_handle* h) {
    if (h->env_eval) return 0;
    if (ensure_policy_slots(h)) return 1;
    int* d = nullptr;
    CK(dalloc(h, &d, 2 * (size_t)h->n));
    h->env_eval = d;
    h->env_eval_host.assign((size_t)h->n, 0);
    h->P.env_eval = d;
    h->slots_active = true;      // slot 0 alone: its table entry is bound to h->W (its trainer's net) by ensure_slot_tables
    h->slot_dirty = true;
    destroy_graphs(h);
    g_model_owner = nullptr;
    return ensure_model(h) ? fail("trl_set_env_eval: model upload failed") : 0;
}

int trl_set_env_eval(trl_handle* h, const int32_t* env_ids, const int32_t* flags, int n) {
    const std::string who = "trl_set_env_eval";
    if (!h) return fail(who + ": null handle");
    if (h->mode != TRL_MODE_EXPLORE) return fail(who + ": every env of an evaluation handle evaluates (evaluation envs are for exploration handles)");
    if (!h->mc.has_net) return fail(who + ": the scene has no policy net");
    if (!h->decide_v2) return fail(who + ": the TRL_DECIDE_V1 decision kernel has no evaluation envs");
    if (h->comm) return fail(who + ": evaluation envs do not run with a communicator");
    if (n < 0 || n > h->n) return fail(who + ": env count out of range");
    if (n > 0 && !flags) return fail(who + ": null flag list");
    for (int k = 0; k < n; ++k) {
        const int e = env_ids ? env_ids[k] : k;
        if (e < 0 || e >= h->n) return fail(who + ": env id " + std::to_string(e) + " out of range");
    }
    if (drain(h) || trl_enable_env_eval(h)) return 1;
    std::vector<int> next = h->env_eval_host;
    for (int k = 0; k < n; ++k) next[env_ids ? env_ids[k] : k] = flags[k] ? 1 : 0;
    CK(cudaMemcpy(h->env_eval + h->n, next.data(), next.size() * 4, cudaMemcpyHostToDevice));
    h->env_eval_host.swap(next);
    return 0;
}

int trl_env_eval(trl_handle* h, int32_t* current, int32_t* assigned, int n) {
    if (!h) return fail("trl_env_eval: null handle");
    if (n < 0 || n > h->n) return fail("trl_env_eval: env count out of range");
    if (!h->env_eval) {
        const int all = h->mode == TRL_MODE_POLI_EVAL ? 1 : 0;
        for (int k = 0; k < n; ++k) {
            if (current) current[k] = all;
            if (assigned) assigned[k] = all;
        }
        return 0;
    }
    if (drain(h)) return 1;
    if (current && n > 0) CK(cudaMemcpy(current, h->env_eval, (size_t)n * 4, cudaMemcpyDeviceToHost));
    if (assigned && n > 0) CK(cudaMemcpy(assigned, h->env_eval + h->n, (size_t)n * 4, cudaMemcpyDeviceToHost));
    return 0;
}

// trl_eval_stats_phys over the envs whose present episode runs in `mode`; a handle whose envs all run in one mode gives that mode
// every env and the other none
// env_body (trl_eval_stats_body): only the envs whose present episode runs on body slot body_slot
static int eval_stats_mode(trl_handle* h, const std::string& who, int mode, int policy_slot, int terrain_slot, int phys_slot, int64_t* cycles,
                           int64_t* episodes, double* avg_dist, int64_t* env_steps, const int* env_body, int body_slot) {
    if (!h) return fail(who + ": null handle");
    if (mode != -1 && mode != TRL_MODE_POLI_EVAL && mode != TRL_MODE_EXPLORE)
        return fail(who + ": mode " + std::to_string(mode) + " is none of TRL_MODE_POLI_EVAL, TRL_MODE_EXPLORE or -1 (any)");
    if (mode == -1 || (!h->env_eval && mode == h->mode))
        return eval_stats_phys(h, who, policy_slot, terrain_slot, phys_slot, nullptr, 0, cycles, episodes, avg_dist, env_steps, env_body, body_slot);
    if (!h->env_eval) {     // no env runs in the other mode: the slots are checked, the figures are zero
        if (eval_stats_phys(h, who, policy_slot, terrain_slot, phys_slot, nullptr, 0, nullptr, nullptr, nullptr, nullptr, env_body, body_slot)) return 1;
        if (cycles) *cycles = 0;
        if (episodes) *episodes = 0;
        if (avg_dist) *avg_dist = 0.0;
        if (env_steps) *env_steps = 0;
        return 0;
    }
    return eval_stats_phys(h, who, policy_slot, terrain_slot, phys_slot, h->env_eval, mode == TRL_MODE_POLI_EVAL ? 1 : 0, cycles, episodes,
                           avg_dist, env_steps, env_body, body_slot);
}
int trl_eval_stats_mode(trl_handle* h, int mode, int policy_slot, int terrain_slot, int phys_slot, int64_t* cycles, int64_t* episodes,
                        double* avg_dist, int64_t* env_steps) {
    return eval_stats_mode(h, "trl_eval_stats_mode", mode, policy_slot, terrain_slot, phys_slot, cycles, episodes, avg_dist, env_steps, nullptr, -1);
}

static bool body_loaded(const trl_handle* h, int slot) { return slot == 0 || (slot > 0 && slot < kMaxBodySlots && h->body_loaded[slot]); }

// what every body of the table must satisfy (trl_load_body checks the file's numbers with its own messages; a checkpoint's table comes
// through here only): finite numbers, positive masses and box sizes, gains and torque limits >= 0, reach within kMaxReach
static bool body_ok(const BodyConst& b, int nj, std::string* why) {
    auto finite = [&](const double* p, int k) { for (int i = 0; i < k; ++i) if (!std::isfinite(p[i])) return false; return true; };
    for (const double* p : {b.attach_x, b.attach_y, b.mass, b.body_ax, b.body_ay, b.body_theta, b.body_cos, b.body_sin, b.half_x, b.half_y,
                            b.izz_o, b.izz_c, b.kp, b.kd, b.torque_lim, b.target_theta0, b.target_vel})
        if (!finite(p, nj)) { *why = "a per-link number is not finite"; return false; }
    for (int j = 0; j < nj; ++j) {
        if (b.has_limit[j] && !(std::isfinite(b.lim_lo[j]) && std::isfinite(b.lim_hi[j]))) { *why = "a joint limit is not finite"; return false; }
        if (!(b.mass[j] > 0.0) || !(b.half_x[j] > 0.0) || !(b.half_y[j] > 0.0)) { *why = "a mass or box size is not positive"; return false; }
        if (b.kp[j] < 0.0 || b.kd[j] < 0.0 || b.torque_lim[j] < 0.0) { *why = "Kp, Kd or TorqueLim is negative"; return false; }
    }
    if (!finite(b.corner_lx, 4 * nj) || !finite(b.corner_ly, 4 * nj) || !(b.total_mass > 0.0) || !(b.reach >= 0.0 && b.reach <= kMaxReach)) {
        *why = "the corners, total mass or reach are out of range";
        return false;
    }
    return true;
}

// the per-env body slots, every env on slot 0: from now on the step launches run the body-slot build (drained by the caller)
static int enable_body_slots(trl_handle* h) {
    if (h->env_body) return 0;
    int* d = nullptr;
    CK(dalloc(h, &d, 2 * (size_t)h->n));
    h->env_body = d;
    h->env_body_host.assign((size_t)h->n, 0);
    destroy_graphs(h);
    return 0;
}

int trl_set_body_slot(trl_handle* h, int slot, const BodyConst& b) {
    std::string why;
    if (slot < 1 || slot >= kMaxBodySlots) return fail("body slot " + std::to_string(slot) + " out of range");
    if (!body_ok(b, h->mc.nj, &why)) return fail("body slot " + std::to_string(slot) + ": " + why);
    if (drain(h)) return 1;
    if (enable_body_slots(h)) return 1;
    h->body[slot] = b;
    h->body_loaded[slot] = true;
    h->ranges.body_ranged &= ~(1u << slot);
    g_model_owner = nullptr;
    return ensure_model(h) ? fail("trl_load_body: body table upload failed") : 0;
}

// the body a character file describes, checked as trl_load_body checks it (topology, controllers, numbers, reach)
static int read_body(trl_handle* h, const std::string& who, const char* character_json_path, BodyConst* out) {
    if (!character_json_path) return fail(who + ": null path");
    const ModelConst& sm = h->mc;
    // the scene with this file's character records: fill_model derives from it what it derives for a handle created with
    // -character_file=<this file>, and everything but the per-link numbers has to come out as the scene's
    trl_handle t;
    t.mode = h->mode;
    try {
        const CharacterRecords cr = read_character_file(join_path(h->data_root, character_json_path), h->data_root, sm.char_type == 2, sm.nj);
        for (const char* rec : {"meta_f64", "pose0", "vel0", "terrain_params", "terrain_default_params", "net_out_scale"})
            if (h->scene.has(rec)) t.scene.set_f64(rec, h->scene.f64(rec));
        if (h->scene.has("net_dims")) t.scene.set_i32("net_dims", h->scene.i32("net_dims"));
        std::vector<int32_t> mi = h->scene.i32("meta_i32");
        if (mi.size() < 15) return fail(who + ": the scene's meta record is too short");
        mi[8] = cr.nj; mi[9] = cr.ndof; mi[10] = cr.n_ctrl; mi[11] = cr.n_actions; mi[12] = cr.default_action; mi[13] = cr.grav_comp;
        mi[14] = cr.virt_forces;
        t.scene.set_i32("meta_i32", mi);
        t.scene.set_f64("joints", cr.joints); t.scene.set_f64("bodies", cr.bodies); t.scene.set_f64("pd", cr.pd);
        t.scene.set_f64("ctrl_params", cr.ctrl_params); t.scene.set_f64("actions", cr.actions);
        const int nj = cr.nj;
        for (int j = 0; j < nj; ++j) {
            const double* r = &cr.joints[7 * j];
            const double* b = &cr.bodies[9 * j];
            const double* p = &cr.pd[6 * j];
            const std::string at = " of link " + std::to_string(j);
            for (int k : {2, 3, 5, 6})
                if (!std::isfinite(r[k])) return fail(who + ": a Skeleton number" + at + " is not finite");
            for (int k : {1, 2, 3, 5, 6, 7})
                if (!std::isfinite(b[k])) return fail(who + ": a BodyDefs number" + at + " is not finite");
            for (int k = 0; k < 5; ++k)
                if (!std::isfinite(p[k])) return fail(who + ": a PDControllers number" + at + " is not finite");
            if (!(b[1] > 0.0)) return fail(who + ": Mass" + at + " = " + std::to_string(b[1]) + " must be positive");
            if (!(b[6] > 0.0) || !(b[7] > 0.0)) return fail(who + ": a box size" + at + " is not positive");
            if (p[0] < 0.0 || p[1] < 0.0 || p[2] < 0.0) return fail(who + ": Kp, Kd or TorqueLim" + at + " is negative");
        }
    } catch (const std::exception& e) {
        return fail(who + ": " + e.what());
    }
    if (fill_model(&t, sm.rng_seed)) return fail(who + ": the character's topology differs from the scene's: " + g_err);
    const ModelConst& bm = t.mc;
    // the topology, masks, corner layout, controller tables and net dimensions stay the scene's
#define TRL_SAME(f) (std::memcmp(&bm.f, &sm.f, sizeof(sm.f)) == 0)
    if (!(TRL_SAME(nj) && TRL_SAME(ndof) && TRL_SAME(parent) && TRL_SAME(dof) && TRL_SAME(collidable) && TRL_SAME(depth) &&
          TRL_SAME(max_depth) && TRL_SAME(child) && TRL_SAME(anc_pow) && TRL_SAME(n_chains) && TRL_SAME(chain_levels) &&
          TRL_SAME(chain_level_len) && TRL_SAME(chain_links) && TRL_SAME(chain_len) && TRL_SAME(chain_level) && TRL_SAME(chain_merge) &&
          TRL_SAME(chain_up) && TRL_SAME(n_corners) && TRL_SAME(corner_base) && TRL_SAME(anc_mask_toe) && TRL_SAME(anc_mask_finger) &&
          TRL_SAME(vf_mask_toe) && TRL_SAME(vf_mask_finger)))
        return fail(who + ": the character's topology (joint types, parents or body shapes) differs from the scene's");
    if (!(TRL_SAME(n_ctrl) && TRL_SAME(n_actions) && TRL_SAME(default_action) && TRL_SAME(grav_comp) && TRL_SAME(virt_forces) &&
          TRL_SAME(ctrl_params) && TRL_SAME(act_idx0) && TRL_SAME(act_idx1) && TRL_SAME(act_cyclic) && TRL_SAME(act_blend)))
        return fail(who + ": the character's Controllers section (controller files, actions, default action or flags) differs from the scene's");
#undef TRL_SAME
    if (bm.reach > kMaxReach)
        return fail(who + ": the body reaches " + std::to_string(bm.reach) + " m from its root joint, more than the " + std::to_string(kMaxReach) +
                    " m the ground window covers (UpdateGround keeps 2 m behind the root; the broad phase reads reach + 0.25 m)");
    *out = body_of(bm);
    return 0;
}

// refused while `slot` is some env's present or assigned slot (`cur_dev`: the device [2][n] array, null when there is none)
static int slot_unused(trl_handle* h, const std::string& who, int slot, const int* cur_dev, const std::vector<int>& assigned, const char* what) {
    if (!cur_dev) return 0;
    if (drain(h)) return 1;
    std::vector<int> cur((size_t)h->n);
    CK(cudaMemcpy(cur.data(), cur_dev, cur.size() * 4, cudaMemcpyDeviceToHost));
    for (int e = 0; e < h->n; ++e)
        if (cur[e] == slot || assigned[e] == slot)
            return fail(who + ": slot " + std::to_string(slot) + " is in use (env " + std::to_string(e) + "'s present or assigned " + what + ")");
    return 0;
}

int trl_load_body(trl_handle* h, int slot, const char* character_json_path) {
    const std::string who = "trl_load_body";
    if (!h) return fail(who + ": null handle");
    if (slot < 1 || slot >= kMaxBodySlots)
        return fail(who + ": slot " + std::to_string(slot) + " out of range (1.." + std::to_string(kMaxBodySlots - 1) + "; slot 0 is the scene's body)");
    BodyConst b;
    if (read_body(h, who, character_json_path, &b)) return 1;
    if (slot_unused(h, who, slot, h->env_body, h->env_body_host, "body")) return 1;
    return trl_set_body_slot(h, slot, b);
}

int trl_set_env_body(trl_handle* h, const int32_t* env_ids, const int32_t* slots, int n) {
    const std::string who = "trl_set_env_body";
    if (!h) return fail(who + ": null handle");
    if (n < 0 || n > h->n) return fail(who + ": env count out of range");
    if (n > 0 && !slots) return fail(who + ": null slot list");
    for (int k = 0; k < n; ++k) {
        const int e = env_ids ? env_ids[k] : k;
        if (e < 0 || e >= h->n) return fail(who + ": env id " + std::to_string(e) + " out of range");
        if (slots[k] < 0 || slots[k] >= kMaxBodySlots) return fail(who + ": slot " + std::to_string(slots[k]) + " out of range");
        if (!body_loaded(h, slots[k])) return fail(who + ": slot " + std::to_string(slots[k]) + " is empty (trl_load_body first)");
    }
    if (!h->env_body) return 0;      // only slot 0 exists, and every env is on it
    std::vector<int> next = h->env_body_host;
    for (int k = 0; k < n; ++k) next[env_ids ? env_ids[k] : k] = slots[k];
    if (drain(h)) return 1;
    CK(cudaMemcpy(h->env_body + h->n, next.data(), next.size() * 4, cudaMemcpyHostToDevice));
    h->env_body_host.swap(next);
    return 0;
}

int trl_env_body(trl_handle* h, int32_t* current, int32_t* assigned, int n) {
    if (!h) return fail("trl_env_body: null handle");
    if (n < 0 || n > h->n) return fail("trl_env_body: env count out of range");
    if (!h->env_body) {
        for (int k = 0; k < n; ++k) {
            if (current) current[k] = 0;
            if (assigned) assigned[k] = 0;
        }
        return 0;
    }
    if (drain(h)) return 1;
    if (current && n > 0) CK(cudaMemcpy(current, h->env_body, (size_t)n * 4, cudaMemcpyDeviceToHost));
    if (assigned && n > 0) CK(cudaMemcpy(assigned, h->env_body + h->n, (size_t)n * 4, cudaMemcpyDeviceToHost));
    return 0;
}

// trl_eval_stats_mode over the envs whose present episode runs on body slot body_slot (-1: any); a handle whose envs are all on body
// slot 0 needs no filter
int trl_eval_stats_body(trl_handle* h, int mode, int policy_slot, int terrain_slot, int phys_slot, int body_slot, int64_t* cycles,
                        int64_t* episodes, double* avg_dist, int64_t* env_steps) {
    const std::string who = "trl_eval_stats_body";
    if (!h) return fail(who + ": null handle");
    if (body_slot < -1 || body_slot >= kMaxBodySlots) return fail(who + ": body slot " + std::to_string(body_slot) + " out of range");
    if (body_slot >= 0 && !body_loaded(h, body_slot)) return fail(who + ": body slot " + std::to_string(body_slot) + " is empty");
    const bool filter = body_slot >= 0 && h->env_body;
    return eval_stats_mode(h, who, mode, policy_slot, terrain_slot, phys_slot, cycles, episodes, avg_dist, env_steps, filter ? h->env_body : nullptr,
                           filter ? body_slot : -1);
}

// ---- ranged slots (trl_types.h: kBodyDrawTag)
// the per-env draw tables, at the handle's first ranged slot; a ranged slot is drawn where the body-slot build restages bodies, so the
// handle moves onto that build (drained by the caller)
int trl_enable_ranges(trl_handle* h) {
    if (h->ranges.env_draws) return 0;
    if (enable_body_slots(h)) return 1;
    const size_t n = (size_t)h->n;
    CK(dalloc(h, &h->ranges.env_bdraw, n));
    CK(dalloc(h, &h->ranges.env_pdraw, n));
    CK(dalloc(h, &h->ranges.env_draws, 2 * n));
    return 0;
}

// what a ranged body slot's two ends must satisfy: each a body trl_set_body_slot accepts, the same numbers but for the four drawn
// fields (and what fill_model derives from them), lo <= hi in those
static int check_body_range(const std::string& who, const BodyConst& lo, const BodyConst& hi, int nj) {
    std::string why;
    if (!body_ok(lo, nj, &why)) return fail(who + ": lo: " + why);
    if (!body_ok(hi, nj, &why)) return fail(who + ": hi: " + why);
    struct F { const char* name; size_t off; int per_link; bool is_int; };
#define TRL_F(f, name, k) F{name, offsetof(BodyConst, f), k, std::is_same<decltype(+lo.f[0]), int>::value}
    static const F fixed[] = {TRL_F(attach_x, "Skeleton AttachX", 1), TRL_F(attach_y, "Skeleton AttachY", 1), TRL_F(lim_lo, "LimLow", 1),
                              TRL_F(lim_hi, "LimHigh", 1), TRL_F(has_limit, "joint limit", 1), TRL_F(body_ax, "BodyDefs AttachX", 1),
                              TRL_F(body_ay, "BodyDefs AttachY", 1), TRL_F(body_theta, "Theta", 1), TRL_F(body_cos, "Theta", 1),
                              TRL_F(body_sin, "Theta", 1), TRL_F(half_x, "Param0 (box size)", 1), TRL_F(half_y, "Param1 (box size)", 1),
                              TRL_F(corner_lx, "box corner", 4), TRL_F(corner_ly, "box corner", 4), TRL_F(target_theta0, "TargetTheta", 1),
                              TRL_F(target_vel, "TargetVel", 1), TRL_F(world_pd, "UseWorldCoord", 1)};
#undef TRL_F
    for (const F& f : fixed) {
        const size_t w = f.is_int ? 4 : 8;
        const unsigned char* a = reinterpret_cast<const unsigned char*>(&lo) + f.off;
        const unsigned char* b = reinterpret_cast<const unsigned char*>(&hi) + f.off;
        for (int i = 0; i < f.per_link * nj; ++i)
            if (std::memcmp(a + i * w, b + i * w, w) != 0)
                return fail(who + ": the lo and hi bodies differ in " + f.name + " of link " + std::to_string(i / f.per_link) +
                            " (only Mass, Kp, Kd and TorqueLim are drawn)");
    }
    if (std::memcmp(&lo.reach, &hi.reach, sizeof(lo.reach)) != 0) return fail(who + ": the lo and hi bodies differ in their reach");
    const double* l[kBodyDrawFields] = {lo.mass, lo.kp, lo.kd, lo.torque_lim};
    const double* u[kBodyDrawFields] = {hi.mass, hi.kp, hi.kd, hi.torque_lim};
    static const char* names[kBodyDrawFields] = {"Mass", "Kp", "Kd", "TorqueLim"};
    for (int f = 0; f < kBodyDrawFields; ++f)
        for (int j = 0; j < nj; ++j)
            if (!(l[f][j] <= u[f][j]))
                return fail(who + ": " + names[f] + " of link " + std::to_string(j) + ": lo " + std::to_string(l[f][j]) + " > hi " + std::to_string(u[f][j]));
    return 0;
}

int trl_set_body_range(trl_handle* h, int slot, const BodyConst& lo, const BodyConst& hi) {
    const std::string who = "trl_load_body_range";
    if (slot < 1 || slot >= kMaxBodySlots) return fail(who + ": slot " + std::to_string(slot) + " out of range");
    if (check_body_range(who, lo, hi, h->mc.nj)) return 1;
    if (drain(h)) return 1;
    if (trl_enable_ranges(h)) return 1;
    h->body[slot] = lo;
    h->body_loaded[slot] = true;
    h->ranges.body_hi[slot] = hi;
    h->ranges.body_ranged |= 1u << slot;
    g_model_owner = nullptr;
    return ensure_model(h) ? fail("trl_load_body_range: body table upload failed") : 0;
}

int trl_load_body_range(trl_handle* h, int slot, const char* lo_path, const char* hi_path) {
    const std::string who = "trl_load_body_range";
    if (!h) return fail(who + ": null handle");
    if (h->comm) return fail(who + ": ranged slots do not run with a communicator");
    if (slot < 1 || slot >= kMaxBodySlots)
        return fail(who + ": slot " + std::to_string(slot) + " out of range (1.." + std::to_string(kMaxBodySlots - 1) + "; slot 0 is the scene's body)");
    BodyConst lo, hi;
    if (read_body(h, who + ": lo", lo_path, &lo) || read_body(h, who + ": hi", hi_path, &hi)) return 1;
    if (slot_unused(h, who, slot, h->env_body, h->env_body_host, "body")) return 1;
    return trl_set_body_range(h, slot, lo, hi);
}

int trl_set_phys_range(trl_handle* h, int slot, const PhysParams& lo, const PhysParams& hi) {
    const std::string who = "trl_load_physics_range";
    if (slot < 1 || slot >= kMaxPhysSlots) return fail(who + ": slot " + std::to_string(slot) + " out of range");
    const double l[7] = {lo.kn, lo.dn, lo.mu, lo.v_eps, lo.contact_tol, lo.k_lim, lo.d_lim};
    const double u[7] = {hi.kn, hi.dn, hi.mu, hi.v_eps, hi.contact_tol, hi.k_lim, hi.d_lim};
    if (check_p7(who, l, "lo ") || check_p7(who, u, "hi ")) return 1;
    for (int k = 0; k < 7; ++k)
        if (!(l[k] <= u[k])) return fail(who + ": " + kPhysNames[k] + ": lo " + std::to_string(l[k]) + " > hi " + std::to_string(u[k]));
    if (lo.vertex_contacts != hi.vertex_contacts || (lo.vertex_contacts & ~1)) return fail(who + ": vertex_contacts malformed");
    if (drain(h)) return 1;
    if (trl_enable_ranges(h)) return 1;
    return set_phys_slot(h, who, slot, lo, &hi);
}

int trl_load_physics_range(trl_handle* h, int slot, const double* lo7, const double* hi7, int vertex_contacts) {
    const std::string who = "trl_load_physics_range";
    if (!h) return fail(who + ": null handle");
    if (h->comm) return fail(who + ": ranged slots do not run with a communicator");
    if (slot < 1 || slot >= kMaxPhysSlots)
        return fail(who + ": slot " + std::to_string(slot) + " out of range (1.." + std::to_string(kMaxPhysSlots - 1) + "; slot 0 is the scene's physics, set by trl_set_phys_params)");
    if (!lo7 || !hi7) return fail(who + ": null parameter array");
    if (slot_unused(h, who, slot, h->env_phys, h->env_phys_host, "physics")) return 1;
    const int vc = vertex_contacts ? 1 : 0;
    return trl_set_phys_range(h, slot, PhysParams{lo7[0], lo7[1], lo7[2], lo7[3], lo7[4], lo7[5], lo7[6], vc},
                              PhysParams{hi7[0], hi7[1], hi7[2], hi7[3], hi7[4], hi7[5], hi7[6], vc});
}

// every env's present slot (row 0 of a device [2][n] array; null: every env on slot 0) and draw count of one kind (0 body, 1 physics)
static int present_slots(trl_handle* h, const int* dev, int kind, std::vector<int>* cur, std::vector<long long>* draws) {
    const size_t n = (size_t)h->n;
    cur->assign(n, 0);
    draws->assign(n, 0);
    if (drain(h)) return 1;
    if (dev) CK(cudaMemcpy(cur->data(), dev, n * 4, cudaMemcpyDeviceToHost));
    if (h->ranges.env_draws) CK(cudaMemcpy(draws->data(), h->ranges.env_draws + kind * n, n * 8, cudaMemcpyDeviceToHost));
    return 0;
}

int trl_env_body_draws(trl_handle* h, double* out, int64_t* draws) {
    if (!h) return fail("trl_env_body_draws: null handle");
    std::vector<int> cur;
    std::vector<long long> cnt;
    if (present_slots(h, h->env_body, 0, &cur, &cnt)) return 1;
    const int n = h->n, nj = h->mc.nj;
    std::vector<BodyConst> drawn;
    if (h->ranges.body_ranged) {
        drawn.resize((size_t)n);
        CK(cudaMemcpy(drawn.data(), h->ranges.env_bdraw, (size_t)n * sizeof(BodyConst), cudaMemcpyDeviceToHost));
    }
    const BodyConst scene = body_of(h->mc);
    for (int e = 0; e < n; ++e) {
        const int b = cur[e];
        const BodyConst& x = ((h->ranges.body_ranged >> b) & 1u) ? drawn[e] : (b == 0 ? scene : h->body[b]);
        if (out) {
            double* o = out + (size_t)e * kBodyDrawFields * nj;
            for (int j = 0; j < nj; ++j) { o[j] = x.mass[j]; o[nj + j] = x.kp[j]; o[2 * nj + j] = x.kd[j]; o[3 * nj + j] = x.torque_lim[j]; }
        }
        if (draws) draws[e] = cnt[e];
    }
    return 0;
}

int trl_env_physics_draws(trl_handle* h, double* out, int64_t* draws) {
    if (!h) return fail("trl_env_physics_draws: null handle");
    std::vector<int> cur;
    std::vector<long long> cnt;
    if (present_slots(h, h->env_phys, 1, &cur, &cnt)) return 1;
    const int n = h->n;
    std::vector<PhysParams> drawn;
    if (h->ranges.phys_ranged) {
        drawn.resize((size_t)n);
        CK(cudaMemcpy(drawn.data(), h->ranges.env_pdraw, (size_t)n * sizeof(PhysParams), cudaMemcpyDeviceToHost));
    }
    for (int e = 0; e < n; ++e) {
        const int q = cur[e];
        const PhysParams& x = ((h->ranges.phys_ranged >> q) & 1u) ? drawn[e] : (q == 0 ? h->mc.phys : h->phys[q]);
        if (out) {
            double* o = out + (size_t)e * 7;
            o[0] = x.kn; o[1] = x.dn; o[2] = x.mu; o[3] = x.v_eps; o[4] = x.contact_tol; o[5] = x.k_lim; o[6] = x.d_lim;
        }
        if (draws) draws[e] = cnt[e];
    }
    return 0;
}

int trl_dist_log(trl_handle* h, const double** dist, const int32_t** env_id, int* n) {
    if (!h) return fail("trl_dist_log: null handle");
    int cnt = 0;
    CK(cudaStreamSynchronize(h->stream));
    CK(cudaMemcpy(&cnt, h->B.dist_count, 4, cudaMemcpyDeviceToHost));
    cnt = std::min(cnt, h->B.dist_cap);
    h->h_dist.resize(std::max(cnt, 1));
    h->h_dist_env.resize(std::max(cnt, 1));
    if (cnt > 0) {
        CK(cudaMemcpy(h->h_dist.data(), h->B.dist_log, (size_t)cnt * 8, cudaMemcpyDeviceToHost));
        CK(cudaMemcpy(h->h_dist_env.data(), h->B.dist_env, (size_t)cnt * 4, cudaMemcpyDeviceToHost));
    }
    *dist = h->h_dist.data(); *env_id = h->h_dist_env.data(); *n = cnt;
    return 0;
}

static int copy_plane_d(trl_handle* h, int field, int count, int env, double* out) {
    // strided gather of `count` consecutive planes for one env
    return cudaMemcpy2D(out, 8, h->B.d + (size_t)field * h->n + env, (size_t)h->n * 8, 8, count, cudaMemcpyDeviceToHost) != cudaSuccess;
}
static int copy_plane_i(trl_handle* h, int field, int count, int env, int* out) {
    return cudaMemcpy2D(out, 4, h->B.i + (size_t)field * h->n + env, (size_t)h->n * 4, 4, count, cudaMemcpyDeviceToHost) != cudaSuccess;
}

int trl_get_state(trl_handle* h, int env, double* pose, double* vel, double* held_torque, uint8_t* contact) {
    if (!h) return fail("trl_get_state: null handle");
    if (env < 0 || env >= h->n) return fail("env out of range");
    CK(cudaStreamSynchronize(h->stream));
    int nd = h->mc.ndof;
    if (pose && copy_plane_d(h, D_Q, nd, env, pose)) return fail("copy failed");
    if (vel && copy_plane_d(h, D_QD, nd, env, vel)) return fail("copy failed");
    if (held_torque && copy_plane_d(h, D_TAU, nd, env, held_torque)) return fail("copy failed");
    if (contact) {
        int mask = 0;
        if (copy_plane_i(h, I_CONTACT, 1, env, &mask)) return fail("copy failed");
        for (int j = 0; j < h->mc.nj; ++j) contact[j] = (mask >> j) & 1;
    }
    return 0;
}

int trl_set_state(trl_handle* h, int env, const double* pose, const double* vel, const double* held_torque, const uint8_t* contact) {
    if (!h) return fail("trl_set_state: null handle");
    if (env < 0 || env >= h->n) return fail("env out of range");
    CK(cudaStreamSynchronize(h->stream));
    int nd = h->mc.ndof;
    auto put = [&](int field, const double* src) {
        return cudaMemcpy2D(h->B.d + (size_t)field * h->n + env, (size_t)h->n * 8, src, 8, 8, nd, cudaMemcpyHostToDevice);
    };
    if (pose) CK(put(D_Q, pose));
    if (vel) CK(put(D_QD, vel));
    if (held_torque) CK(put(D_TAU, held_torque));
    if (contact) {
        int mask = 0;
        for (int j = 0; j < h->mc.nj; ++j) if (contact[j]) mask |= 1 << j;
        CK(cudaMemcpy(h->B.i + (size_t)I_CONTACT * h->n + env, &mask, 4, cudaMemcpyHostToDevice));
    }
    return 0;
}

int trl_get_state_all(trl_handle* h, double* pose, double* vel) {
    if (!h) return fail("trl_get_state_all: null handle");
    CK(cudaStreamSynchronize(h->stream));
    size_t bytes = (size_t)h->mc.ndof * h->n * 8;
    if (pose) CK(cudaMemcpy(pose, h->B.d + (size_t)D_Q * h->n, bytes, cudaMemcpyDeviceToHost));
    if (vel) CK(cudaMemcpy(vel, h->B.d + (size_t)D_QD * h->n, bytes, cudaMemcpyDeviceToHost));
    return 0;
}

int trl_get_ctrl(trl_handle* h, int env, double* out, int cap, int* n_out) {
    if (!h) return fail("trl_get_ctrl: null handle");
    if (env < 0 || env >= h->n) return fail("env out of range");
    CK(cudaStreamSynchronize(h->stream));
    std::vector<double> d(D_NUM_FIELDS);
    std::vector<int> iv(I_NUM_FIELDS);
    if (copy_plane_d(h, 0, D_NUM_FIELDS, env, d.data()) || copy_plane_i(h, 0, I_NUM_FIELDS, env, iv.data())) return fail("copy failed");
    std::vector<double> o;
    o.push_back(iv[I_STATE]); o.push_back(d[D_PHASE]); o.push_back(iv[I_FIRST_CYCLE]); o.push_back(d[D_CUR_CYCLE_T]);
    o.push_back(d[D_PREV_CYCLE_T]); o.push_back(d[D_CUR_STUMBLE]); o.push_back(d[D_PREV_STUMBLE]); o.push_back(d[D_PREV_COM_X]);
    o.push_back(d[D_PREV_COM_Y]); o.push_back(d[D_PREV_DIST_X]); o.push_back(d[D_PREV_DIST_Y]); o.push_back(iv[I_ACTION_ID]);
    for (int k = 0; k < h->mc.n_params; ++k) o.push_back(d[D_PARAMS + k]);
    for (int j = 0; j < h->mc.nj; ++j) o.push_back(d[D_PD_TARGET + j]);
    o.push_back(d[D_FALL_DIST_CNT]); o.push_back(d[D_FALL_CONTACT_CNT]); o.push_back(d[D_SUM_FALL]); o.push_back(d[D_PREV_CHECK_X]);
    o.push_back(d[D_PREV_CHECK_Y]); o.push_back(iv[I_FAIL_FALL_DIST]); o.push_back(iv[I_EXP_FLAGS] & 1); o.push_back((iv[I_EXP_FLAGS] >> 1) & 1);
    o.push_back(iv[I_CYCLE_COUNT]); o.push_back(iv[I_STANCE]);
    int n = (int)std::min<size_t>(o.size(), (size_t)cap);
    std::memcpy(out, o.data(), (size_t)n * 8);
    if (n_out) *n_out = n;
    return 0;
}

int trl_get_poli_state(trl_handle* h, int env, double* out) {
    if (!h) return fail("trl_get_poli_state: null handle");
    if (env < 0 || env >= h->n) return fail("env out of range");
    CK(cudaStreamSynchronize(h->stream));
    CK(cudaMemcpy(out, h->B.poli_state + (size_t)env * h->B.S, (size_t)h->B.S * 8, cudaMemcpyDeviceToHost));
    return 0;
}
int trl_get_net_out(trl_handle* h, int env, double* out) {
    if (!h) return fail("trl_get_net_out: null handle");
    if (env < 0 || env >= h->n) return fail("env out of range");
    CK(cudaStreamSynchronize(h->stream));
    CK(cudaMemcpy(out, h->B.net_out + (size_t)env * kMaxNetOut, (size_t)h->mc.n_out * 8, cudaMemcpyDeviceToHost));
    return 0;
}
int trl_get_terrain(trl_handle* h, int env, int seg, float* data, int cap, int* n, double* min_x, int* flip) {
    if (!h) return fail("trl_get_terrain: null handle");
    if (env < 0 || env >= h->n) return fail("env out of range");
    if (seg < 0 || seg > 1) return fail("terrain segment out of range (0 or 1)");
    CK(cudaStreamSynchronize(h->stream));
    int sn = 0, fl = 0;
    double mx = 0;
    if (copy_plane_i(h, seg == 0 ? I_SEG_N0 : I_SEG_N1, 1, env, &sn) || copy_plane_i(h, I_SEG_FLIP, 1, env, &fl) ||
        copy_plane_d(h, seg == 0 ? D_SEG_MINX0 : D_SEG_MINX1, 1, env, &mx))
        return fail("copy failed");
    int cnt = std::min(sn, cap);
    if (cnt > 0) CK(cudaMemcpy(data, h->B.terrain + ((size_t)env * 2 + seg) * kTerrainCap, (size_t)cnt * 4, cudaMemcpyDeviceToHost));
    *n = sn; *min_x = mx; *flip = fl;
    return 0;
}

int64_t trl_kernel_launches(trl_handle* h) { return h ? h->launches : -1; }

// Stage pending list 0 for the debug entry points below: `env_ids` (NULL = envs 0 .. n-1) with count n, on the handle's stream.
// The decision launch that consumes the list with rearm = 1 resets the count, so this runs before every launch.
static int stage_pending_list(trl_handle* h, const int32_t* env_ids, int n) {
    std::vector<int32_t> ids;
    if (!env_ids) {
        ids.resize(n);
        for (int i = 0; i < n; ++i) ids[i] = i;
        env_ids = ids.data();
    }
    if (n > 0) CK(cudaMemcpyAsync(h->B.pending_list, env_ids, (size_t)n * 4, cudaMemcpyHostToDevice, h->stream));
    CK(cudaMemcpyAsync(h->B.pending_count, &n, 4, cudaMemcpyHostToDevice, h->stream));
    return 0;
}

// One decision pass over a chosen batch (tests): the listed envs, in list order (row k of the pass = env_ids[k]), optionally with
// new policy states, through the same launch(es) one env-step's decisions take.  Returns after the pass has finished.
int trl_debug_decide(trl_handle* h, const int32_t* env_ids, int n, const double* poli_states) {
    if (!h) return fail("trl_debug_decide: null handle");
    if (n < 0 || n > h->n) return fail("trl_debug_decide: env count out of range");
    if (n > 0 && !env_ids) return fail("trl_debug_decide: no env list");
    {
        std::vector<char> seen(h->n, 0);
        for (int k = 0; k < n; ++k) {
            const int e = env_ids[k];
            if (e < 0 || e >= h->n) return fail("trl_debug_decide: env id out of range");
            if (seen[e]) return fail("trl_debug_decide: env " + std::to_string(e) + " listed twice");
            seen[e] = 1;
        }
    }
    if (ensure_model(h)) return fail("model upload failed");
    if (drain(h)) return 1;
    if (poli_states) {
        const size_t S = (size_t)h->B.S;
        for (int k = 0; k < n;) {      // one copy per run of consecutive env ids
            int r = 1;
            while (k + r < n && env_ids[k + r] == env_ids[k] + r) ++r;
            CK(cudaMemcpyAsync(h->B.poli_state + (size_t)env_ids[k] * S, poli_states + (size_t)k * S, (size_t)r * S * 8, cudaMemcpyHostToDevice,
                               h->stream));
            k += r;
        }
    }
    if (stage_pending_list(h, env_ids, n)) return 1;
    enqueue_decide(h, 0, 1, h->stream);
    h->launches += num_decide_launches(h);
    CK(cudaGetLastError());
    CK(cudaStreamSynchronize(h->stream));
    return 0;
}

// Micro-benchmark of the decision kernel: marks the first `n_pending` envs as pending (their policy state is whatever the
// last real decision left) and times `iters` launches.  Perturbs those envs' actions: measurement use only.
int trl_debug_time_decide(trl_handle* h, int n_pending, int iters, double* ms_avg) {
    if (!h) return fail("trl_debug_time_decide: null handle");
    if (ensure_model(h)) return fail("model upload failed");
    if (n_pending > h->n) n_pending = h->n;
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
    double total = 0;
    for (int it = 0; it < iters; ++it) {
        if (stage_pending_list(h, nullptr, n_pending)) return 1;
        CK(cudaEventRecord(e0, h->stream));
        enqueue_decide(h, 0, 1, h->stream);
        CK(cudaEventRecord(e1, h->stream));
        CK(cudaEventSynchronize(e1));
        float ms = 0;
        CK(cudaEventElapsedTime(&ms, e0, e1));
        total += ms;
    }
    cudaEventDestroy(e0); cudaEventDestroy(e1);
    if (ms_avg) *ms_avg = total / iters;
    return 0;
}

// Phase stamps of the batched decision path's FC kernel for `n_pending` decisions (measurement only): out[k] = nanoseconds from
// kernel entry to stamp k (see trl_decide2.cuh: stamp()); conv_us / fc_us = event-timed durations of the two launches
int trl_debug_fc_phases(trl_handle* h, int n_pending, double* out_ns16, double* conv_us, double* fc_us) {
    if (!h) return fail("trl_debug_fc_phases: null handle");
    if (!h->decide_v2 || !h->mc.has_net || h->slots_active) return fail("trl_debug_fc_phases: the single-policy batched decision path is not active");
    if (ensure_model(h)) return fail("model upload failed");
    n_pending = std::max(1, std::min(n_pending, h->n));
    unsigned long long* prof = nullptr;
    CK(cudaMalloc((void**)&prof, 16 * 8));
    CK(cudaMemset(prof, 0, 16 * 8));
    FcMaps maps = h->fc_maps[0];
    maps.prof = prof;
    cudaEvent_t e0, e1, e2;
    CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1)); CK(cudaEventCreate(&e2));
    for (int it = 0; it < 3; ++it) {      // the last of three runs is reported (weights L2-resident, clocks up)
        if (stage_pending_list(h, nullptr, n_pending)) return 1;
        CK(cudaEventRecord(e0, h->stream));
        launch_decide2(h->B, h->W, h->d_ex, maps, h->act2[0], h->done_count, h->decide_grid, h->fc_clusters, 0, 1, h->stream, 1);
        CK(cudaEventRecord(e1, h->stream));
        launch_decide2(h->B, h->W, h->d_ex, maps, h->act2[0], h->done_count, h->decide_grid, h->fc_clusters, 0, 1, h->stream, 2);
        CK(cudaEventRecord(e2, h->stream));
        CK(cudaEventSynchronize(e2));
    }
    h->launches += 6;
    float a = 0, b = 0;
    CK(cudaEventElapsedTime(&a, e0, e1)); CK(cudaEventElapsedTime(&b, e1, e2));
    if (conv_us) *conv_us = a * 1e3;
    if (fc_us) *fc_us = b * 1e3;
    unsigned long long st[16];
    CK(cudaMemcpy(st, prof, sizeof(st), cudaMemcpyDeviceToHost));
    for (int k = 0; k < 16; ++k) out_ns16[k] = st[k] ? (double)(st[k] - st[0]) : -1.0;
    cudaFree(prof);
    cudaEventDestroy(e0); cudaEventDestroy(e1); cudaEventDestroy(e2);
    return 0;
}

// Pipelined read-back: trl_snapshot() enqueues, behind the work already on the handle's stream, a device-side copy
// of all pose / velocity planes plus the reduced batch statistics, then moves them to pinned host memory on a second
// stream; trl_snapshot_wait() blocks on that copy only, so the caller can enqueue the next trl_update() first and
// read update k's results while update k+1 runs.
int trl_snapshot(trl_handle* h) {
    if (!h) return fail("trl_snapshot: null handle");
    const size_t plane = (size_t)h->mc.ndof * h->n;
    const size_t total = 2 * plane + 4;
    if (!h->snap_dev) {
        CK(cudaMalloc((void**)&h->snap_dev, total * 8)); h->allocs.push_back(h->snap_dev);
        CK(cudaMallocHost((void**)&h->snap_host, total * 8));
        CK(cudaStreamCreateWithFlags(&h->copy_stream, cudaStreamNonBlocking));
        CK(cudaEventCreateWithFlags(&h->snap_ready, cudaEventDisableTiming));
        CK(cudaEventCreateWithFlags(&h->snap_copied, cudaEventDisableTiming));
    }
    if (h->snap_pending) CK(cudaEventSynchronize(h->snap_copied));   // previous snapshot must have left the staging area
    CK(cudaMemcpyAsync(h->snap_dev, h->B.d + (size_t)D_Q * h->n, plane * 8, cudaMemcpyDeviceToDevice, h->stream));
    CK(cudaMemcpyAsync(h->snap_dev + plane, h->B.d + (size_t)D_QD * h->n, plane * 8, cudaMemcpyDeviceToDevice, h->stream));
    launch_stats(h->B, h->snap_dev + 2 * plane, h->stream);
    h->launches += 1;
    CK(cudaEventRecord(h->snap_ready, h->stream));
    CK(cudaStreamWaitEvent(h->copy_stream, h->snap_ready, 0));
    CK(cudaMemcpyAsync(h->snap_host, h->snap_dev, total * 8, cudaMemcpyDeviceToHost, h->copy_stream));
    CK(cudaEventRecord(h->snap_copied, h->copy_stream));
    h->snap_pending = true;
    return 0;
}

int trl_snapshot_wait(trl_handle* h, double* pose, double* vel, int64_t* cycles, int64_t* episodes, double* avg_dist, int64_t* env_steps) {
    if (!h) return fail("trl_snapshot_wait: null handle");
    if (!h->snap_pending) return fail("trl_snapshot_wait: no snapshot in flight");
    CK(cudaEventSynchronize(h->snap_copied));
    h->snap_pending = false;
    const size_t plane = (size_t)h->mc.ndof * h->n;
    if (pose) std::memcpy(pose, h->snap_host, plane * 8);
    if (vel) std::memcpy(vel, h->snap_host + plane, plane * 8);
    const double* st = h->snap_host + 2 * plane;
    if (cycles) *cycles = (int64_t)st[0];
    if (episodes) *episodes = (int64_t)st[1];
    if (env_steps) *env_steps = (int64_t)st[2];
    if (avg_dist) *avg_dist = st[1] > 0 ? st[3] / st[1] : 0.0;
    return 0;
}

// Raw device views of the tuple block for zero-copy hand-off to a collective (NCCL all-gather of ExpTuple blocks,
// SURVEY §8e).  Pointers are device addresses on the handle's GPU; the caller must trl_sync() before using them on
// another stream.
int trl_device_tuple_block(trl_handle* h, void** rows_f64, void** flags_u32, void** env_i32, void** count_i32, int* cap, int* width) {
    if (!h) return fail("trl_device_tuple_block: null handle");
    if (rows_f64) *rows_f64 = h->B.tuples;
    if (flags_u32) *flags_u32 = h->B.tuple_flags;
    if (env_i32) *env_i32 = h->B.tuple_env;
    if (count_i32) *count_i32 = h->B.tuple_count;
    if (cap) *cap = h->B.tuple_cap;
    if (width) *width = 1 + h->B.S + h->B.A + h->B.S;
    return 0;
}

// K outer updates timed with CUDA events on the handle's own stream (the stream the kernels are launched on);
// optionally evicts L2 between updates by writing a 256 MiB scratch buffer.
int trl_bench_updates(trl_handle* h, double dt, int k, int flush_l2, double* ms_total) {
    if (!h) return fail("trl_bench_updates: null handle");
    if (ensure_model(h)) return fail("model upload failed");
    const size_t flush_bytes = (size_t)256 << 20;
    if (flush_l2 && !h->flush_buf) { CK(cudaMalloc(&h->flush_buf, flush_bytes)); h->allocs.push_back(h->flush_buf); }
    // One event pair per update; the L2 flush (a measurement device, not part of the path) sits BETWEEN the pairs, so the reported
    // time is the sum of the K updates' own device time, every one of them starting from a cold L2.
    std::vector<cudaEvent_t> ev(2 * (size_t)std::max(k, 0));
    for (auto& e : ev) CK(cudaEventCreate(&e));
    CK(cudaStreamSynchronize(h->stream));
    for (int i = 0; i < k; ++i) {
        if (flush_l2) CK(cudaMemsetAsync(h->flush_buf, i & 0xff, flush_bytes, h->stream));
        CK(cudaEventRecord(ev[2 * i], h->stream));
        if (trl_update(h, dt)) return 1;
        CK(cudaEventRecord(ev[2 * i + 1], h->stream));
    }
    CK(cudaStreamSynchronize(h->stream));
    double ms = 0.0;
    for (int i = 0; i < k; ++i) {
        float t = 0.f;
        CK(cudaEventElapsedTime(&t, ev[2 * i], ev[2 * i + 1]));
        ms += t;
    }
    if (k > 0) {
        float t = 0.f;
        CK(cudaEventElapsedTime(&t, ev[0], ev[2 * k - 1]));      // first update's start to last update's end, flushes included
        h->bench_span_ms = t;
    }
    for (auto& e : ev) cudaEventDestroy(e);
    if (ms_total) *ms_total = ms;
    return 0;
}

// the span of the last trl_bench_updates call from the first update's start to the last update's end, L2 flushes included
int trl_bench_last_span(trl_handle* h, double* ms) {
    if (!h || !ms) return fail("trl_bench_last_span: null argument");
    *ms = h->bench_span_ms;
    return 0;
}

// One outer update launched kernel by kernel with an event pair around every launch: returns the summed device time
// of the step kernel launches and of the decision kernel launches (roofline numerator's denominator).
// One outer update in the schedule trl_update uses (overlapped unless TRL_SERIAL_SCHEDULE=1), launched eagerly with an event pair
// around every launch on its own stream: out[4 * k + {0,1,2,3}] = {kind (0 terrain, 1 step, 2 decision, 3 catch-up), index, start
// ms, end ms} relative to the first launch.  Shows what bounds the update: the step launches or the decision -> catch-up chain.
int trl_update_timeline(trl_handle* h, double dt, double* out, int cap, int* n_out) {
    if (!h) return fail("trl_update_timeline: null handle");
    if (ensure_model(h)) return fail("model upload failed");
    Timeline tl;
    CK(cudaStreamSynchronize(h->stream));
    for (int k = 0; k < h->lag; ++k) CK(cudaStreamSynchronize(h->side[k]));
    (void)cudaGetLastError();        // a stale, already reported status of an earlier call must not be charged to this run
    enqueue_update(h, dt, h->overlap, &tl);
    {
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess && tl.err.empty()) tl.err = std::string("after enqueue: ") + cudaGetErrorString(e);
        if (!tl.err.empty()) return fail("trl_update_timeline: " + tl.err);
    }
    CK(cudaStreamSynchronize(h->stream));
    for (int k = 0; k < h->lag; ++k) CK(cudaStreamSynchronize(h->side[k]));
    h->launches += update_launches(h, h->overlap);
    const int n = (int)tl.beg.size();
    for (int k = 0; k < n; ++k) {
        float a = 0, b = 0;
        cudaEventElapsedTime(&a, tl.beg[0], tl.beg[k]);
        cudaEventElapsedTime(&b, tl.beg[0], tl.end[k]);
        if (k < cap) { out[4 * k] = tl.kind[k]; out[4 * k + 1] = tl.idx[k]; out[4 * k + 2] = a; out[4 * k + 3] = b; }
    }
    for (int k = 0; k < n; ++k) { cudaEventDestroy(tl.beg[k]); cudaEventDestroy(tl.end[k]); }
    for (auto e : tl.fork) cudaEventDestroy(e);
    if (n_out) *n_out = std::min(n, cap);
    return 0;
}

static int update_timed_impl(trl_handle* h, double dt, double* step_ms, int* step_launches, double* decide_ms, int* decide_launches,
                             double* per_step, double* per_decide);
int trl_update_timed(trl_handle* h, double dt, double* step_ms, int* step_launches, double* decide_ms, int* decide_launches) {
    if (!h) return fail("trl_update_timed: null handle");
    return update_timed_impl(h, dt, step_ms, step_launches, decide_ms, decide_launches, nullptr, nullptr);
}
// same, also returning every launch's duration: per_step[num_update_steps + 1], per_decide[num_update_steps]
int trl_update_timed_detail(trl_handle* h, double dt, double* per_step, double* per_decide) {
    if (!h) return fail("trl_update_timed_detail: null handle");
    return update_timed_impl(h, dt, nullptr, nullptr, nullptr, nullptr, per_step, per_decide);
}
static int update_timed_impl(trl_handle* h, double dt, double* step_ms, int* step_launches, double* decide_ms, int* decide_launches,
                             double* per_step, double* per_decide) {
    if (ensure_model(h)) return fail("model upload failed");
    const int ns = h->num_update_steps;
    const double step = dt / ns;
    std::vector<cudaEvent_t> ev(2 * (2 * ns + 1));
    for (auto& e : ev) CK(cudaEventCreate(&e));
    int k = 0;
    terrain_launch(h, h->stream);
    for (int i = 0; i < ns; ++i) {
        CK(cudaEventRecord(ev[k++], h->stream));
        step_launch(h, step, i == 0 ? 2 : 3, 0, h->stream);
        CK(cudaEventRecord(ev[k++], h->stream));
        CK(cudaEventRecord(ev[k++], h->stream));
        enqueue_decide(h, 0, 1, h->stream);
        CK(cudaEventRecord(ev[k++], h->stream));
    }
    CK(cudaEventRecord(ev[k++], h->stream));
    step_launch(h, step, 1 | 4, 0, h->stream);
    CK(cudaEventRecord(ev[k++], h->stream));
    CK(cudaStreamSynchronize(h->stream));
    CK(cudaGetLastError());
    double sm = 0, dm = 0;
    int idx = 0;
    for (int i = 0; i < ns; ++i) {
        float a = 0, b = 0;
        CK(cudaEventElapsedTime(&a, ev[idx], ev[idx + 1])); idx += 2;
        CK(cudaEventElapsedTime(&b, ev[idx], ev[idx + 1])); idx += 2;
        sm += a; dm += b;
        if (per_step) per_step[i] = a;
        if (per_decide) per_decide[i] = b;
    }
    float a = 0;
    CK(cudaEventElapsedTime(&a, ev[idx], ev[idx + 1]));
    sm += a;
    if (per_step) per_step[ns] = a;
    for (auto& e : ev) cudaEventDestroy(e);
    h->launches += (1 + num_decide_launches(h)) * ns + 2;
    if (step_ms) *step_ms = sm;
    if (step_launches) *step_launches = ns + 1;
    if (decide_ms) *decide_ms = dm;
    if (decide_launches) *decide_launches = ns;
    return 0;
}

}  // extern "C"

int trl_drain(trl_handle* h) { return drain(h); }

int trl_set_terrain_slot(trl_handle* h, int slot, int type, std::vector<double> sets) {
    TerrainSlot ts{};
    ts.type = type;
    blend_terrain(sets.data(), (int)(sets.size() / kTerrainParams), h->scene.f64("terrain_default_params").data(), h->terrain_lerp, ts.params);
    if (drain(h)) return 1;
    if (h->env_terrain_host.empty()) {     // first slot: from now on the step launches run the terrain-slot build
        h->env_terrain_host.assign((size_t)h->n, 0);
        destroy_graphs(h);
    }
    h->terrain_sets[slot] = std::move(sets);
    h->terrain_loaded[slot] = true;
    h->terrain[slot] = ts;
    g_model_owner = nullptr;
    return ensure_model(h) ? fail("trl_load_terrain: terrain table upload failed") : 0;
}
