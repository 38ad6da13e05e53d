/* terrainrl_b200 -- C ABI of the H100-native batched rollout engine.
 *
 * One handle = one batch of N independent environments stepped in lock-step on one GPU.  Each entry point names
 * the reference interface it replaces (file:line under the DeepTerrainRL tree); the reference has no FFI layer,
 * its seam is the C++ virtual scenario API that cScenarioTrain / cOptScenarioPoliEval call on every pooled env
 * (scenarios/ScenarioTrain.cpp:197-222,376-410; optimizer/scenarios/OptScenarioPoliEval.cpp:135-237).
 *
 * Conventions: all functions return 0 on success, non-zero on error (trl_last_error() gives the message; the
 * reference's printf+assert convention cannot cross an ABI).  A handle is single-writer.  Pointers returned by
 * the library stay valid until the next call that mutates the same data (documented per function).
 * Plain C types only: no torch / CUDA types in any signature.
 */
#ifndef TERRAINRL_B200_H
#define TERRAINRL_B200_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct trl_handle trl_handle;

enum { TRL_MODE_POLI_EVAL = 0, TRL_MODE_EXPLORE = 1 };

/* cScenario{PoliEval,ExpMACE}::ParseArgs + Init + SetRandSeed + Reset for N envs
 * (scenarios/ScenarioSimChar.cpp:80-119, ScenarioPoliEval.cpp:60-108,153-160, ScenarioExp.cpp:29-73).
 * `pack_path` is a scene pack produced by tools/pack_scene.py from a reference arg file.  terrain_seeds may be NULL
 * (env i gets seed 1+i).  Returns NULL on failure. */
trl_handle* trl_create_from_pack(const char* pack_path, int num_envs, int device, int mode,
                                 const uint64_t* terrain_seeds, uint64_t rng_seed);
/* Same, straight from the reference's own inputs: argv holds cArgParser-style tokens (e.g. "-arg_file=",
 * "args/dog_slopes_mixed_args.txt", plus overrides, CLI first = CLI wins, optimizer/Main.cpp:19-32); relative paths
 * inside are resolved against data_root (a DeepTerrainRL checkout).  Native readers for the arg file, the JSON assets
 * and the Caffe HDF5 weights (util/ArgParser.cpp:42-140, anim/KinTree.cpp:9-60, learning/NeuralNet.cpp:81-215). */
trl_handle* trl_create(int argc, const char* const* argv, const char* data_root, int num_envs, int device, int mode,
                       const uint64_t* terrain_seeds, uint64_t rng_seed);
/* Scene files -> .trlpack without touching the GPU (what tools/pack_scene.py does in Python) */
int trl_pack_from_args(int argc, const char* const* argv, const char* data_root, const char* out_path);
int trl_destroy(trl_handle* h);

/* cScenario::Reset for the listed envs (NULL = all)            scenarios/ScenarioSimChar.cpp:121-132 */
int trl_reset(trl_handle* h, const int32_t* env_ids, int n);
/* cScenarioPoliEval::SetRandSeed + Reset for every env         scenarios/ScenarioPoliEval.cpp:153-160 */
int trl_seed_terrain(trl_handle* h, const uint64_t* seeds, int n);

/* cScenario::Update(dt) for all envs in lock-step: num_update_steps env-steps, then the fall -> reset handling
 * (scenarios/ScenarioSimChar.cpp:141-182, ScenarioPoliEval.cpp:110-125, ScenarioExp.cpp:83-98).
 * Asynchronous: enqueued on the handle's stream; trl_sync() or any getter waits. */
int trl_update(trl_handle* h, double dt);
/* one iteration of the loop at scenarios/ScenarioSimChar.cpp:162-173 (parity probe; no fall handling) */
int trl_env_step(trl_handle* h, double step);
int trl_sync(trl_handle* h);

/* cScenarioExp::{EnableExplore,SetExpRate,SetExpTemp,SetExpBaseActionRate}   scenarios/ScenarioExp.cpp:156-185
 *   trl_set_explore       the settings of every env (every policy slot's entry)
 *   trl_set_explore_slot  the settings of the envs on policy slot `slot` (0..7) only; slot 0's entry is also the one a handle
 *                         without policy slots uses.  A slot that holds no policy yet keeps its entry until it does.  Refused for a
 *                         slot out of range.  The exploration noise std stays the scene's, for every slot.
 * Both are ordered on the handle's stream behind the work already queued; neither drains it. */
int trl_set_explore(trl_handle* h, int enable, double rate, double temp, double base_rate);
int trl_set_explore_slot(trl_handle* h, int slot, int enable, double rate, double temp, double base_rate);
/* engine contact / joint-limit parameters (7 doubles: kn, dn, mu, v_eps, contact_tol, k_lim, d_lim) */
int trl_set_phys_params(trl_handle* h, const double* p7);

/* cNeuralNet::CopyModel into every env's controller net (learning/NeuralNetLearner.cpp:85-89): 26 blobs in Caffe
 * order (w, b of terr_conv0..2, terr_ip0, ip0, val_ip0, val_ip1, a{0,1,2}_ip{0,1}) + the four offset/scale vectors. */
int trl_set_weights(trl_handle* h, const double* const* blobs, const int64_t* counts, int nblobs,
                    const double* in_off, const double* in_scale, const double* out_off, const double* out_scale);

/* sizes: policy state, action record, MACE fragments           sim/NNController.cpp:49-78, BaseControllerMACE.cpp:36-56 */
int trl_sizes(trl_handle* h, int* num_envs, int* state, int* action, int* num_frags, int* frag_size, int* num_dof,
              int* num_joints);

/* cScenarioExp::{IsTupleBufferFull,GetTuples,ResetTupleBuffer} for the whole batch: rows are
 * [reward | s(S) | a(A) | s'(S)] exactly like cMACETrainer's replay rows (learning/MACETrainer.cpp:515-539);
 * flags bit0 fail, bit1 expCritic, bit2 expActor (learning/MACETrainer.h:11-17).  The f32 view is what the
 * trainer stores; the f64 view is what tExpTuple holds.  Pointers valid until trl_reset_tuples / trl_update. */
int trl_num_tuples(trl_handle* h, int* out);
int trl_get_tuples(trl_handle* h, const float** rows, const uint32_t** flags, const int32_t** env_id, int* n);
int trl_get_tuples_f64(trl_handle* h, const double** rows, const uint32_t** flags, const int32_t** env_id, int* n);
int trl_reset_tuples(trl_handle* h);

/* cScenarioPoliEval::{GetNumCycles,GetNumEpisodes,GetAvgDist,GetDistLog}   scenarios/ScenarioPoliEval.cpp:127-151 */
int trl_eval_stats(trl_handle* h, int64_t* cycles, int64_t* episodes, double* avg_dist, int64_t* env_steps);
int trl_dist_log(trl_handle* h, const double** dist, const int32_t** env_id, int* n);
/* cScenarioPoliEval::ResetAvgDist for every env                scenarios/ScenarioPoliEval.cpp:132-136 */
int trl_reset_avg_dist(trl_handle* h);

/* cSimCharacter::{BuildPose,BuildVel} / SetPose+SetVel and contact bits for one env (sim/SimCharacter.cpp:166-315) */
int trl_get_state(trl_handle* h, int env, double* pose, double* vel, double* held_torque, uint8_t* contact);
int trl_set_state(trl_handle* h, int env, const double* pose, const double* vel, const double* held_torque,
                  const uint8_t* contact);
/* bulk SoA views: pose/vel as [num_dof][num_envs] doubles */
int trl_get_state_all(trl_handle* h, double* pose, double* vel);

/* parity probes (same layouts as the oracle's probes) */
int trl_get_ctrl(trl_handle* h, int env, double* out, int cap, int* n);
int trl_get_poli_state(trl_handle* h, int env, double* out);
int trl_get_net_out(trl_handle* h, int env, double* out);
/* cNeuralNet::GetLayerState (learning/NeuralNet.cpp:814-833) for the policy state of env's last decision: the blob `layer_name` of the
 * deploy net (any top name of data/policies/<char>/nets/<char>_mace3_deploy.prototxt, e.g. "terr_conv1", "relu0", "a1_ip0", "output");
 * what cScenarioPoliEval::RecordNNActivation writes per cycle (scenarios/ScenarioPoliEval.cpp:271-296).  *n = the blob's size. */
int trl_get_layer_state(trl_handle* h, int env, const char* layer_name, double* out, int cap, int* n);
int trl_get_terrain(trl_handle* h, int env, int seg, float* data, int cap, int* n, double* min_x, int* flip);

/* number of engine kernels launched since creation (bench.py's gpu_launches claim) */
int64_t trl_kernel_launches(trl_handle* h);

/* pipelined read-back of what cOptScenarioPoliEval::EvalHelper reads after every Update (counters; optionally every
 * env's pose/vel as [num_dof][num_envs] planes): trl_snapshot() enqueues the capture behind the updates already
 * submitted, trl_snapshot_wait() returns it from pinned host memory -- call trl_update() for the next step in between. */
int trl_snapshot(trl_handle* h);
int trl_snapshot_wait(trl_handle* h, double* pose, double* vel, int64_t* cycles, int64_t* episodes, double* avg_dist,
                      int64_t* env_steps);

/* device-resident view of the tuple block (rows f64 [cap][width], flags, env ids, count) for zero-copy hand-off to
 * NCCL; replaces the per-thread `learner->Train(exp->GetTuples())` hand-off (scenarios/ScenarioTrain.cpp:388-395) */
int trl_device_tuple_block(trl_handle* h, void** rows_f64, void** flags_u32, void** env_i32, void** count_i32,
                           int* cap, int* width);

/* measurement helpers: K outer updates timed with CUDA events on the handle's stream, one event pair per update, *ms_total = the sum
 * (flush_l2: a 256 MiB memset between the pairs evicts L2 before every update; it is a measurement device and is not timed --
 * trl_bench_last_span returns the span from the first update's start to the last update's end with the flushes in it);
 * one update with an event pair around every kernel launch (per-kernel device time for the roofline). */
int trl_bench_updates(trl_handle* h, double dt, int k, int flush_l2, double* ms_total);
int trl_bench_last_span(trl_handle* h, double* ms);
int trl_update_timed(trl_handle* h, double dt, double* step_ms, int* step_launches, double* decide_ms, int* decide_launches);
int trl_update_timed_detail(trl_handle* h, double dt, double* per_step_ms, double* per_decide_ms);
/* one update in trl_update's own (overlapped) schedule with an event pair around every launch: out[4k..4k+3] = {kind (0 terrain, 1 step,
 * 2 decision, 3 catch-up), index, start ms, end ms} */
int trl_update_timeline(trl_handle* h, double dt, double* out4, int cap, int* n);

int trl_debug_time_decide(trl_handle* h, int n_pending, int iters, double* ms_avg);
/* tests: one policy decision pass over the listed envs, row k = env_ids[k] (distinct ids, 0 <= n <= num_envs; n = 0 changes nothing).
 * poli_states: NULL, or [n][state] rows written into those envs' policy states first.  Waits for the handle's queued work, runs the
 * decision launch(es) of one env-step on that list and returns when they have finished. */
int trl_debug_decide(trl_handle* h, const int32_t* env_ids, int n, const double* poli_states);
/* measurement only: in-kernel phase stamps (ns from entry, 16 slots) of the batched decision path's FC kernel + event-timed conv / FC launches */
int trl_debug_fc_phases(trl_handle* h, int n_pending, double* out_ns16, double* conv_us, double* fc_us);
/* measurement only, TRL_PHASE_CLOCKS=1 builds: clock64() cycles of the env-step kernel summed over warps per phase (9 slots: state
 * load/store, controller RNEA, mass-matrix solve, rest of the controller, kinematics, contacts, inward pass, base + outward pass,
 * terrain / FSM / policy state) + out[9] = env-steps counted; n must be 10 */
int trl_debug_step_phases(trl_handle* h, unsigned long long* out, int n, int reset);

/* ---------------------------------------------------------------------------------------------------------------------
 * MACE trainer on the GPU (SURVEY.md §8 f1) -- replaces cMACETrainer / cNeuralNetLearner behind cScenarioTrainMACE:
 *   trl_trainer_create        cTrainerInterface::Init + LoadModel (learning/NeuralNetTrainer.cpp:26-49, MACETrainer.cpp:78-90);
 *                             p[10] = {replay_mem_size, num_init_samples, num_steps_per_iter, freeze_target_iters,
 *                             init_input_offset_scale, discount, base_lr, momentum, weight_decay, seed}.  From this call on the
 *                             scenario's decision kernel evaluates the trainer's current net (cNeuralNetLearner::SyncNet,
 *                             learning/NeuralNetLearner.cpp:83-87, becomes a pointer binding).
 *   trl_trainer_add_from_scene  AddTuples(exp.GetTuples()) + ResetTupleBuffer (learning/NeuralNetLearner.cpp:33-45,
 *                             scenarios/ScenarioTrain.cpp:388-408), device to device
 *   trl_trainer_add_tuples    cNeuralNetTrainer::AddTuples from host rows [n][1 + S + A + S] (learning/NeuralNetTrainer.cpp:145-173)
 *   trl_trainer_train         iters x cNeuralNetTrainer::Train (learning/NeuralNetTrainer.cpp:175-183 -> cMACETrainer::Step,
 *                             learning/MACETrainer.cpp:335-361), asynchronous on the scenario's stream
 *   trl_trainer_counters      GetIter / GetNumTuples / buffer sizes / last losses
 *   trl_trainer_get, _set_theta, _list   model read-back (OutputModel), LoadModel, buffer inspection for the tests */
/* model files in the reference's formats, natively (no Python, no libhdf5):
 *   trl_load_model     cNeuralNet::LoadModel + LoadScale (learning/NeuralNet.cpp:157-186): Caffe ToHDF5 weights + `_scale.txt`
 *   trl_output_model   cNeuralNet::OutputModel + WriteOffsetScale (learning/NeuralNet.cpp:571-587,1182-1205) of the policy the
 *                      scenario currently evaluates (the attached trainer's net if there is one); mtime = HDF5 modification stamp
 *   trl_write_model    the same for host-side weights: blobs[26] = (weights, bias) of the 13 parameter layers in net order
 *   trl_get_output_offset_scale   cBaseControllerMACE::BuildNNOutputOffsetScale (sim/BaseControllerMACE.cpp:75-113) */
int trl_load_model(trl_handle* h, const char* h5_path, const char* scale_json_path);
int trl_output_model(trl_handle* h, const char* path, uint32_t mtime);
/* trl_output_model for the net policy slot `slot` evaluates (its trainer's, if it has one); slot 0 is trl_output_model */
int trl_output_model_slot(trl_handle* h, int slot, const char* path, uint32_t mtime);
int trl_write_model(const char* path, const double* const* blobs26, int n_char, int n_frags, int frag_size, const double* in_off,
                    const double* in_scale, const double* out_off, const double* out_scale, uint32_t mtime);
int trl_get_output_offset_scale(trl_handle* h, double* offset, double* scale, int n_out);

/* policy slots: one evaluation handle (TRL_MODE_POLI_EVAL) evaluates up to 8 models of the scene's net topology side by side, each env
 * with the model of its slot.  Slot 0 is the handle's own policy (trl_create*, trl_load_model, trl_set_weights, trl_output_model);
 * slots 1..7 start empty.  Results of an env do not depend on what else is in the batch: a mixed batch computes exactly what the
 * single-policy handles would, env for env.
 *   trl_load_policy      Caffe-HDF5 model + `_scale.txt` into slot 1..7; refused (handle unchanged) for another topology, an
 *                        exploration handle, a handle with a trainer, and the TRL_DECIDE_V1 build.  trl_trainer_create refuses a
 *                        handle with a loaded slot >= 1.  (Slots that carry trainers: trl_trainer_create_slot below.)
 *   trl_set_env_policy   env_ids[k] (NULL: env k) -> slots[k] for k < n; every env starts on slot 0.  Refused, with nothing changed,
 *                        for an env id or slot out of range or an empty slot.  Takes effect at the env's next decision, no reset.
 *   trl_eval_stats_slot  trl_eval_stats over the envs now on `slot`.  trl_get_net_out / trl_get_layer_state / trl_debug_decide follow
 *                        each env's slot; trl_dist_log entries carry env ids, so a caller splits them by slot itself. */
int trl_load_policy(trl_handle* h, int slot, const char* h5_path, const char* scale_json_path);
int trl_set_env_policy(trl_handle* h, const int32_t* env_ids, const int32_t* slots, int n);
int trl_eval_stats_slot(trl_handle* h, int slot, int64_t* cycles, int64_t* episodes, double* avg_dist, int64_t* env_steps);

/* terrain slots: one handle (any mode, trainer or not) generates the ground of each env from one of up to 8 terrains.  Slot 0 is the
 * scene's own terrain (the pack's, or -terrain_file); slots 1..7 start empty.  Every slot blends its parameter sets with the handle's
 * blend (-terrain_blend, then trl_set_terrain_lerp, which re-blends every loaded slot).  Env i computes exactly what env i of a handle
 * created with its slot's file as -terrain_file computes, with the same seeds.
 *   trl_load_terrain     a terrain file of the reference's format ({"Type": ..., "Params": [...]}, read as -terrain_file is) into slot
 *                        1..7; refused (handle unchanged) for slot 0 or >= 8, a null path, an unknown type or malformed JSON.
 *   trl_set_env_terrain  env_ids[k] (NULL: env k) -> slots[k] for k < n; every env starts on slot 0.  Refused, with nothing changed,
 *                        for an env id or slot out of range, n > num_envs or an empty slot.  Takes effect at the env's next episode
 *                        reset (a fall inside trl_update, trl_reset, trl_seed_terrain): the ground already generated stays until then.
 *   trl_env_terrain      per env (first n), the slot its present ground came from and the slot it will use after its next reset.
 *   trl_eval_stats_cell  trl_eval_stats over the envs now on policy slot `policy_slot` and whose present ground comes from terrain slot
 *                        `terrain_slot`; -1 = any slot.  trl_eval_stats_slot(h, p) is the cell (p, -1). */
int trl_load_terrain(trl_handle* h, int slot, const char* terrain_json_path);
int trl_set_env_terrain(trl_handle* h, const int32_t* env_ids, const int32_t* slots, int n);
int trl_env_terrain(trl_handle* h, int32_t* current, int32_t* assigned, int n);
int trl_eval_stats_cell(trl_handle* h, int policy_slot, int terrain_slot, int64_t* cycles, int64_t* episodes, double* avg_dist,
                        int64_t* env_steps);
/* Physics slots (any mode, with or without trainers, policy or terrain slots): up to 8 contact / joint-limit settings per handle.
 * Slot 0 is the handle's own, which trl_set_phys_params edits; slots 1..7 start empty.  With the same seeds, env i on physics slot q
 * computes bit for bit what env i computes in a handle whose trl_set_phys_params holds slot q's values (created with
 * TRL_VERTEX_CONTACTS=1 when the slot has vertex contacts).
 *   trl_load_physics      p7 (trl_set_phys_params order: kn, dn, mu, v_eps, contact_tol, k_lim, d_lim) and the vertex contact model
 *                         (0 off, else on) into slot 1..7.  Refused, handle unchanged, for slot 0 or >= 8, a null p7, a non-finite
 *                         value, kn, dn, mu, k_lim or d_lim < 0, v_eps <= 0, or contact_tol * sqrt(1 + 25^2) > 0.05, i.e.
 *                         contact_tol > 0.001998: the broad phase keeps corners within 0.05 m of the terrain maximum, and 25 bounds
 *                         the steepest slope the generators produce with the shipped terrain files (a 2 m gap wall over one 0.1 m
 *                         vertex spacing, plus slopes and bumps).  Reloading a slot applies from the next env-step to every env on it,
 *                         as trl_set_phys_params does for slot 0.
 *   trl_set_env_physics   env_ids[k] (NULL: env k) -> slots[k] for k < n; every env starts on slot 0.  Refused, with nothing changed,
 *                         for an env id or slot out of range, n > num_envs or an empty slot.  Takes effect at the env's next episode
 *                         reset (a fall inside trl_update, trl_reset, trl_seed_terrain): an episode never mixes two settings.
 *   trl_env_physics       per env (first n), the slot of its present episode and the slot it gets at its next reset.
 *   trl_eval_stats_phys   trl_eval_stats_cell over the envs of one (policy, terrain, physics) cell, -1 = any slot; an env counts
 *                         toward the physics slot of its present episode.  (p, t, -1) is trl_eval_stats_cell(p, t). */
int trl_load_physics(trl_handle* h, int slot, const double* p7, int vertex_contacts);
int trl_set_env_physics(trl_handle* h, const int32_t* env_ids, const int32_t* slots, int n);
int trl_env_physics(trl_handle* h, int32_t* current, int32_t* assigned, int n);
int trl_eval_stats_phys(trl_handle* h, int policy_slot, int terrain_slot, int phys_slot, int64_t* cycles, int64_t* episodes,
                        double* avg_dist, int64_t* env_steps);
/* Evaluation envs (exploration handles, with or without trainers, training, terrain or physics slots): an env set to evaluate runs its
 * policy slot's current net (its trainer's, if the slot has one) with exploration off, records no tuples, and keeps the episode and
 * distance statistics of an evaluation handle.  Its slot's trainer goes on training from the slot's exploring envs.  With the same
 * seeds, an evaluating env j on policy slot p computes bit for bit what env j computes in a TRL_MODE_POLI_EVAL handle on the same
 * terrain / physics slot whose net is, before every update, the one slot p holds then -- except the counter-RNG position
 * (I_RNG_CTR_LO/HI): evaluation decisions draw a number they do not use, and earlier exploring episodes moved the counter.  An exploring
 * env computes what it computes in the same handle without evaluation envs; each trainer is fed only its slot's exploring envs' tuples.
 *   trl_set_env_eval    env_ids[k] (NULL: env k) evaluates from its next episode if flags[k] != 0, explores otherwise; every env starts
 *                       exploring.  Takes effect at the env's next episode reset (a fall inside trl_update, trl_reset,
 *                       trl_seed_terrain): the ending episode's bookkeeping follows its own mode, and an episode never mixes two.  Entering
 *                       evaluation restarts the env's cycle count at 0; episodes and mean distance accumulate over its evaluating
 *                       episodes until trl_reset_avg_dist.  Refused, handle unchanged, for an evaluation handle, a scene without a policy
 *                       net, the TRL_DECIDE_V1 build, a handle with a communicator (trl_comm_init* refuses a handle with evaluation
 *                       envs), an env id out of range or n > num_envs.
 *   trl_env_eval        per env (first n), 1 if its present episode evaluates, and the same for the mode it gets at its next reset.
 *   trl_eval_stats_mode trl_eval_stats_phys(policy_slot, terrain_slot, phys_slot) over the envs whose present episode runs in `mode`
 *                       (TRL_MODE_POLI_EVAL, TRL_MODE_EXPLORE, -1 = any); (-1, p, t, q) is trl_eval_stats_phys(p, t, q).  The other
 *                       statistics entries keep counting every env. */
int trl_set_env_eval(trl_handle* h, const int32_t* env_ids, const int32_t* flags, int n);
int trl_env_eval(trl_handle* h, int32_t* current, int32_t* assigned, int n);
int trl_eval_stats_mode(trl_handle* h, int mode, int policy_slot, int terrain_slot, int phys_slot, int64_t* cycles, int64_t* episodes,
                        double* avg_dist, int64_t* env_steps);
/* Body slots (any mode; with or without trainers, policy, terrain or physics slots, or evaluation envs): up to 8 bodies of the scene's
 * character per handle.  Slot 0 is the scene's own body; slots 1..7 start empty.  With the same seeds, env i on body slot b computes
 * bit for bit what env i computes in a handle created from the same arguments plus -character_file=<slot b's file>.
 *   trl_load_body        a character file of the reference's format into slot 1..7: per link its Skeleton AttachX/Y and LimLow/LimHigh,
 *                        BodyDefs Mass, AttachX/Y, Theta, Param0/1, PDControllers Kp, Kd, TorqueLim, TargetTheta, TargetVel and
 *                        UseWorldCoord.  A relative path (and the controller files the file names) refers to trl_create's data_root;
 *                        a handle made by trl_create_from_pack or trl_create_from_checkpoint has none, and resolves relative paths
 *                        against the process's working directory (give absolute paths there).
 *                        Refused, handle unchanged, for slot 0 or >= 8, a null path, malformed JSON, a joint count, joint Type or
 *                        Parent, or body Shape other than the scene's, a Controllers section whose files resolve to other parameter
 *                        sets or whose Actions, DefaultAction or gravity-compensation / virtual-force flags differ, a non-finite number,
 *                        Mass <= 0, a box size <= 0, Kp, Kd or TorqueLim < 0, a body that reaches more than 1.75 m from its root joint
 *                        (UpdateGround keeps the ground from 2 m behind the root on, and the broad phase reads 0.25 m beyond the
 *                        reach), or a slot that is some env's present or assigned body.
 *   trl_set_env_body     env_ids[k] (NULL: env k) -> slots[k] for k < n; every env starts on slot 0.  Refused, with nothing changed, for
 *                        an env id or slot out of range, n > num_envs or an empty slot.  Takes effect at the env's next episode reset
 *                        (a fall inside trl_update, trl_reset, trl_seed_terrain): an episode never mixes two bodies.
 *   trl_env_body         per env (first n), the slot of its present episode and the slot it gets at its next reset.
 *   trl_eval_stats_body  trl_eval_stats_mode(mode, policy_slot, terrain_slot, phys_slot) over the envs whose present episode runs on
 *                        body slot body_slot (-1 = any: then it is trl_eval_stats_mode's).  The other statistics entries keep counting
 *                        every env. */
int trl_load_body(trl_handle* h, int slot, const char* character_json_path);
int trl_set_env_body(trl_handle* h, const int32_t* env_ids, const int32_t* slots, int n);
int trl_env_body(trl_handle* h, int32_t* current, int32_t* assigned, int n);
int trl_eval_stats_body(trl_handle* h, int mode, int policy_slot, int terrain_slot, int phys_slot, int body_slot, int64_t* cycles,
                        int64_t* episodes, double* avg_dist, int64_t* env_steps);
/* Ranged slots (domain randomization; any mode): a body or physics slot whose randomizable numbers are drawn again at every episode
 * reset of every env on it (a fall inside trl_update, trl_reset, trl_seed_terrain).  With the same seeds, an episode of env i on a
 * ranged slot computes bit for bit what env i computes on a fixed slot loaded with that episode's drawn numbers (a character file
 * holding them for trl_load_body, the drawn p7 for trl_load_physics), and so what a handle created with that file / those constants
 * computes.  The draws have keys of their own and never move an env's counter RNG.  Each number is drawn independently:
 *   key  = mix64(mix64(mix64(rng_seed ^ TAG) + env) + draw)   mix64: the splitmix64 finaliser; rng_seed: the handle's seed; env: the
 *                                                             env's index; draw: the env's earlier draws of that kind (from 0; kept
 *                                                             by checkpoints, not reset by trl_reset or trl_seed_terrain);
 *                                                             TAG = 0x626f64792d726e67 for bodies, 0x706879732d726e67 for physics
 *   u_i  = (mix64(key + i) >> 11) * 2^-53                     body: i = field * nj + link, fields Mass, Kp, Kd, TorqueLim;
 *                                                             physics: i = 0..6 in p7 order
 *   v_i  = min(hi_i, lo_i + u_i * (hi_i - lo_i))              each operation rounded on its own; lo == hi gives lo exactly
 * A body draw derives izz (per link) and the total mass from the drawn masses as trl_load_body does.  The root's Kp and Kd stay 0.
 *   trl_load_body_range      lo and hi character files into slot 1..7: per link Mass, Kp, Kd and TorqueLim are drawn; everything else is
 *                            the files' and must be the same in both.  Refused, handle unchanged, for whatever trl_load_body refuses
 *                            in either file, two files that differ in anything but the four drawn fields (the message names the
 *                            field and link), lo > hi in any of them, and a handle with a communicator.
 *   trl_load_physics_range   lo7 and hi7 (kn, dn, mu, v_eps, contact_tol, k_lim, d_lim) into slot 1..7, vertex_contacts fixed.
 *                            Refused, handle unchanged, when either end fails trl_load_physics's checks, lo > hi in any constant, the
 *                            slot is some env's present or assigned physics, or the handle has a communicator.
 * Envs move onto ranged slots with trl_set_env_body / trl_set_env_physics; to trl_env_body, the statistics entries and the Python
 * filters a ranged slot is a slot.  trl_load_body / trl_load_physics make a slot fixed again.  The first ranged slot allocates the
 * per-env tables (about 4.7 KB per env) and moves the handle onto the body-slot build.
 *   trl_env_body_draws       the numbers of every env's present episode: out[n][4][nj] (Mass, Kp, Kd, TorqueLim), draws[n] its body
 *                            draws so far; an env on a fixed slot reports its slot's numbers.  Either pointer may be NULL.
 *   trl_env_physics_draws    likewise out[n][7] (p7 order) and draws[n] of physics. */
int trl_load_body_range(trl_handle* h, int slot, const char* lo_path, const char* hi_path);
int trl_load_physics_range(trl_handle* h, int slot, const double* lo7, const double* hi7, int vertex_contacts);
int trl_env_body_draws(trl_handle* h, double* out, int64_t* draws);
int trl_env_physics_draws(trl_handle* h, double* out, int64_t* draws);
int trl_pack_output_offset_scale(const char* pack_path, double* offset, double* scale, int n_out);   /* host only, no device */

/* cScenarioSimChar::SetTerrainParamsLerp (scenarios/ScenarioSimChar.cpp:255-272) and cScenarioTrain's annealing schedule
 * (scenarios/ScenarioTrain.cpp:412-460): sp[9] = {init_exp_rate, exp_rate, init_exp_temp, exp_temp, init_exp_base_rate,
 * exp_base_rate, trainer_num_anneal_iters, exp_base_anneal_iters, trainer_curriculum_iters};
 * out[4] = {exp_rate, exp_temp, exp_base_rate, curriculum_phase} */
int trl_set_terrain_lerp(trl_handle* h, double lerp);
int trl_train_schedule(const double* sp9, int iters, double* out4);

typedef struct trl_trainer trl_trainer;
trl_trainer* trl_trainer_create(trl_handle* h, const double* params10);
int trl_trainer_destroy(trl_trainer* t);
/* training from scratch: xavier-filled weights + cBaseControllerMACE::BuildNNOutputOffsetScale (sim/BaseControllerMACE.cpp:75-113),
 * what cScenarioTrain::InitTrainer leaves when no -policy_model is given (scenarios/ScenarioTrain.cpp:253-259,322-336) */
int trl_trainer_init_fresh(trl_trainer* t, uint64_t seed);
int trl_trainer_add_from_scene(trl_trainer* t);
int trl_trainer_add_tuples(trl_trainer* t, const double* rows, const uint32_t* flags, int n);
/* same from device memory (the all-gathered tuple blocks of every rank, SURVEY.md §8e); ordered on the scenario's stream */
int trl_trainer_add_device(trl_trainer* t, const double* rows_dev, const uint32_t* flags_dev, int n);
int trl_trainer_train(trl_trainer* t, int iters);
/* cScenarioTrain::Run for one batch (scenarios/ScenarioTrain.cpp:100-115,376-410): num_updates x {update, tuple hand-over,
 * trainer iterations (iters_per_update, or 0 = one per tuple_buffer_size new tuples), annealed exploration + curriculum} */
int trl_train_run(trl_trainer* t, const double* sp9, int num_updates, int iters_per_update, int tuple_buffer_size, double time_step);
/* the same loop with the tuple exchange of a multi-GPU run (when the scenario has a communicator: trl_gather_tuples(block_rows) +
 * trl_trainer_add_gathered instead of the local hand-over), timed with CUDA events on the scenario's stream (flush_l2: a 256 MiB
 * memset before every update, as trl_bench_updates does); *iters_state carries the annealing position across calls (start at 0) */
int trl_train_run_timed(trl_trainer* t, const double* sp9, int num_updates, int iters_per_update, int block_rows, double time_step,
                        int flush_l2, int64_t* iters_state, double* ms);
/* asynchronous training (the reference's asynchronous trainer: exploration keeps running on the net it has while the trainer works):
 * hand-over + trainer iterations run on their own stream beside the NEXT update inside trl_train_run / trl_train_run_timed; the
 * decision kernels read a snapshot of the net refreshed between updates (tuples of update u shape the policy from update u + 2 on).
 * Needs a communicator (a single rank will do) and a fixed iters_per_update.  A trainer of a handle with training slots may be made
 * asynchronous only on a handle with a communicator (trl_train_run_slots_comm runs it): slot 0 then evaluates its snapshot through the
 * handle's own net, a slot p >= 1 through its entry of the slot table; disabling binds the trainer's arrays again. */
int trl_trainer_set_async(trl_trainer* t, int enable);
int trl_trainer_counters(trl_trainer* t, int64_t* counters9, double* losses2);
int trl_trainer_num_params(trl_trainer* t);
int64_t trl_trainer_launches(trl_trainer* t);
int trl_trainer_get(trl_trainer* t, int what, double* out);
int trl_trainer_set_theta(trl_trainer* t, const double* theta);
int trl_trainer_list(trl_trainer* t, int which, int32_t* out, int cap, int* len);
int trl_trainer_rows(trl_trainer* t, const int32_t* slots, int n, float* rows, int32_t* flags);
/* the creation parameters params10 of trl_trainer_create and the policy slot the trainer trains (either may be NULL) */
int trl_trainer_params(trl_trainer* t, double* params10, int* slot);

/* checkpoints: a run stopped between two calls and resumed in another process is the same run.
 *   trl_checkpoint_save         drains the handle and its trainers' streams, then writes everything a later call reads to `path`
 *                               (TRLCKPT1: a section table of name, dtype, byte count and device-computed 64-bit digest, then the raw
 *                               bytes): the scene pack, the env state, the tuple block, the distance log, the exploration settings,
 *                               the physics parameters, every policy and terrain slot, every trainer with its replay memory, and
 *                               `user_bytes` of `user` stored verbatim.  Saving changes nothing in the handle.  Refused, with nothing
 *                               written, for a handle with a communicator, an asynchronous trainer or a pending trl_snapshot.
 *   trl_create_from_checkpoint  a handle on `device` from such a file with its trainers: trainers[p] (an array of 8, or NULL) is the
 *                               trainer of policy slot p or NULL; destroy them with trl_trainer_destroy as usual.  The user blob is
 *                               copied into `user` (up to user_cap bytes; *user_bytes = its full length).  Every later call on the
 *                               new handle and its trainers returns, bit for bit, what it returns on the handle that saved, under any
 *                               of the overlapped schedule, the serial schedule or env groups.  NULL on failure (a damaged,
 *                               truncated or foreign file, a digest mismatch: trl_last_error names the section), with nothing left
 *                               allocated.
 *   trl_env_policy              the policy slot of envs 0 .. n-1. */
int trl_checkpoint_save(trl_handle* h, const char* path, const void* user, size_t user_bytes);
trl_handle* trl_create_from_checkpoint(const char* path, int device, trl_trainer** trainers, void* user, size_t user_cap, size_t* user_bytes);
int trl_env_policy(trl_handle* h, int32_t* slots, int n);

/* training slots: one exploration handle (TRL_MODE_EXPLORE) trains up to 8 policies side by side, one trainer per policy slot, each
 * env exploring with the net of its slot (trl_set_env_policy) and feeding that slot's trainer.  Env i on slot p computes exactly what
 * env i computes in a single-trainer handle of the same pack, seeds and size whose trainer is fed only the tuples of slot p's envs,
 * and trainer p ends with that trainer's weights, buffers and counters.
 *   trl_trainer_create_slot  a trainer for slot 0 (the handle's own policy; trl_trainer_create(h, p) is the call with slot 0 and no
 *                        paths) or a training slot 1..7.  The starting net is the Caffe-HDF5 model + `_scale.txt` if both paths are
 *                        given, else a copy of the net slot 0 evaluates now.  Refused, with the handle unchanged, for a slot out of
 *                        range or with a trainer, a slot >= 1 on an evaluation handle or in the TRL_DECIDE_V1 build, slot 0 on a
 *                        handle with trl_load_policy slots, and a model of another topology.  On a handle with a communicator the
 *                        trainers run through trl_train_run_slots_comm.
 *                        trl_trainer_destroy of a slot trainer leaves its trained net in the slot.
 *   trl_train_run_slots  the trl_train_run loop for k trainers of one handle in lock-step (iters_per_update > 0 each per update,
 *                        one exploration setting and curriculum blend per update, annealed from 0 in every call).  Refused for
 *                        trainers of different handles, a trainer listed twice, k < 1 and iters_per_update <= 0.
 *   trl_train_run_slots_sched  the same loop with a schedule per trainer: trainer i anneals by sp9[9 i .. 9 i + 9) and applies the
 *                        result to its own slot (trl_set_explore_slot); slots of unlisted trainers keep their entries.
 *                        iters_per_update > 0: lock-step, annealed from 0 in every call.  iters_per_update == 0: each trainer paced
 *                        as trl_train_run(t, sp, U, 0, tuple_buffer_size, dt) paces it: the schedule at its iteration counter at the
 *                        start of the update, one iteration per tuple_buffer_size fresh tuples of its slot, the remainder carried.
 *                        The handle keeps one terrain blend per update: refused unless every schedule has the same
 *                        trainer_curriculum_iters or all have it < 1 (paced: all < 1).  Also refused for whatever
 *                        trl_train_run_slots refuses, iters_per_update < 0 and, paced, tuple_buffer_size < 1.  Both entries
 *                        refuse a handle with a communicator and asynchronous trainers.
 *   trl_train_run_slots_comm  the trl_train_run_slots_sched loop over N GPUs: per update the schedules, trl_update, ONE
 *                        trl_gather_tuples(h, block_rows), then each trainer's slot-filtered trl_trainer_add_gathered and its
 *                        iterations on its own stream, and the join.  Every rank sees the same blocks, so the counters and the
 *                        replicas agree without a further collective, lock-step or paced (iters_per_update == 0, as
 *                        trl_train_run_slots_sched paces); rows beyond block_rows stay queued.  With a single-rank
 *                        communicator and block_rows >= the tuples of an update it computes, bit for bit, what
 *                        trl_train_run_slots_sched computes on a handle without one.  If every listed trainer is
 *                        asynchronous (trl_trainer_set_async), each one's intake and iterations overlap the next update as in
 *                        trl_train_run: tuples of update u shape slot p's policy from update u + 2 on.  Every rank must make the same
 *                        call: at its start the ranks compare the listed slots in order, the schedules, iters_per_update,
 *                        tuple_buffer_size, block_rows and the asynchronous flags (one small all-reduce), and on a mismatch every
 *                        rank refuses with nothing run.  Also refused: a mix of asynchronous and synchronous trainers,
 *                        asynchronous trainers paced by tuples, and whatever trl_train_run_slots_sched refuses (its curriculum rule
 *                        included); a rank that refuses one of these takes part in the same reduction, so every rank refuses
 *                        together.  Refused by the calling rank alone: no trainer, a destroyed first trainer, no communicator.
 * Once a handle has a training slot: trl_trainer_add_from_scene hands a trainer only its slot's tuples and leaves the block to the
 * others (trl_reset_tuples clears it); trl_set_env_policy is refused while the block holds tuples and resets the envs it moves, so
 * every tuple belongs to the slot that chose its action; trl_train_run / trl_train_run_timed are refused, and trl_trainer_set_async
 * without a communicator. */
trl_trainer* trl_trainer_create_slot(trl_handle* h, int slot, const double* params10, const char* h5_path, const char* scale_json_path);
int trl_train_run_slots(trl_trainer* const* ts, int k, const double* sp9, int num_updates, int iters_per_update, double time_step);
int trl_train_run_slots_sched(trl_trainer* const* ts, int k, const double* sp9k, int num_updates, int iters_per_update, int tuple_buffer_size,
                              double time_step);
int trl_train_run_slots_comm(trl_trainer* const* ts, int k, const double* sp9k, int num_updates, int iters_per_update, int tuple_buffer_size,
                             int block_rows, double time_step);

/* number of tuples the engine could not record because the tuple block was full (cScenarioExp's ring overwrites, scenarios/
 * ScenarioExp.cpp:296-301; a batch block refuses instead and counts).  trl_num_tuples / trl_get_tuples* return
 * TRL_E_TUPLE_OVERFLOW (rows up to the capacity are still delivered) once this is non-zero since the last trl_reset_tuples. */
enum { TRL_E_TUPLE_OVERFLOW = 2 };
int trl_tuples_dropped(trl_handle* h, int64_t* out);

/* ---------------------------------------------------------------------------------------------------------------------
 * Multi-GPU exchange (SURVEY.md §8e): one process per GPU, environments sharded by rank, no collective in the rollout.
 * The two couplings of the reference's training loop become two collectives on a side stream of the handle:
 *   trl_gather_tuples      every rank's finished tuples of this update -> every rank; replaces `learner->Train(exp->GetTuples())`
 *                          under the trainer mutex (scenarios/ScenarioTrain.cpp:388-395, learning/NeuralNetLearner.cpp:33-46):
 *                          a device pack kernel (f32 rows like cMACETrainer's replay memory, learning/MACETrainer.cpp:515-539, flags,
 *                          global env ids, count header) + ONE all-gather of a fixed-capacity block per rank.  No host
 *                          synchronisation; rows beyond block_rows stay queued in the tuple block for the next call.
 *   trl_trainer_add_gathered   AddTuples of all gathered blocks (rank order, env order inside a rank) into the attached trainer;
 *                          in a handle with training slots, only the rows of the trainer's slot (flag bits 24..26), the others
 *                          taking no replay slot
 *   trl_trainer_broadcast  cNeuralNetLearner::SyncNet across ranks (learning/NeuralNetLearner.cpp:85-89): weights + offset/scale
 *                          (and the trainer's target net / momentum history) from `root` to every rank
 *   trl_comm_eval_stats    cOptScenarioPoliEval::OutputResults' merge of the per-thread results
 *                          (optimizer/scenarios/OptScenarioPoliEval.cpp:213-237) as one all-reduce
 * Backends: NCCL (libnccl.so.2 is opened at run time by trl_comm_init; the library does not link against it), or caller-supplied
 * collectives (trl_comm_init_external: MPI, gloo, a test double) that receive device pointers and the CUDA stream to enqueue on. */
enum { TRL_COMM_ID_BYTES = 128 };
int trl_comm_unique_id(void* id128);                                           /* ncclGetUniqueId; call on one rank, ship to all */
int trl_comm_init(trl_handle* h, const void* id128, int rank, int world);     /* ncclCommInitRank on the handle's device */
typedef struct trl_collectives {
    void* ctx;
    int (*all_gather)(void* ctx, const void* send, void* recv, size_t bytes_per_rank, void* cuda_stream);
    int (*broadcast)(void* ctx, void* buf, size_t bytes, int root, void* cuda_stream);
    int (*all_reduce_sum_f64)(void* ctx, void* buf, size_t count, void* cuda_stream);
} trl_collectives;
int trl_comm_init_external(trl_handle* h, const trl_collectives* coll, int rank, int world);
int trl_comm_destroy(trl_handle* h);
int trl_comm_info(trl_handle* h, int* rank, int* world, int* block_rows);
/* env i of this rank is reported as env_offset + i in gathered blocks (default rank * num_envs) */
int trl_comm_set_env_offset(trl_handle* h, int64_t env_offset);
int trl_gather_tuples(trl_handle* h, int block_rows);
/* gathered blocks as device memory: world blocks of block_bytes; block = {i32 count, i32 queued, i32 rank, i32 block_rows,
 * u32 flags[block_rows], i32 env[block_rows], f32 rows[block_rows][1+S+A+S]}.  Ordered on the handle's stream.  A row's flags are
 * the tuple's flags (low bits) with bit 31 set if it fails cNeuralNetTrainer::CheckTuple and, in a handle with training slots,
 * bits 24..26 holding the policy slot of the env that recorded it (zero in a handle without training slots).  Every trainer
 * intake clears bits 24..31: a replay memory stores the tuple's own flags. */
int trl_gathered_blocks(trl_handle* h, const void** dev_blocks, size_t* block_bytes, int* block_rows, int* row_width);
/* host copy for tests / a CPU-side trainer: counts[world]; rows/flags/env may be NULL; cap in rows; synchronises */
int trl_gathered_fetch(trl_handle* h, int32_t* counts, float* rows, uint32_t* flags, int32_t* env, int cap, int* n_total);
/* exposed device time of the last gather (pack end -> all-gather end on the comm stream), ms; synchronises */
int trl_gather_last_ms(trl_handle* h, double* ms);
int trl_trainer_add_gathered(trl_trainer* t);
int trl_trainer_broadcast(trl_trainer* t, int root);
int trl_comm_broadcast_weights(trl_handle* h, int root);                       /* same for a handle without a trainer (eval ranks) */
int trl_comm_eval_stats(trl_handle* h, int64_t* cycles, int64_t* episodes, double* avg_dist, int64_t* env_steps);
/* the same over the envs of one policy slot: trl_eval_stats_slot of every rank, summed (a learning curve per policy over all ranks) */
int trl_comm_eval_stats_slot(trl_handle* h, int slot, int64_t* cycles, int64_t* episodes, double* avg_dist, int64_t* env_steps);
/* max - min over ranks of every trainer parameter (replica drift check), via two all-reduces of +/-theta maxima; synchronises */
int trl_trainer_replica_spread(trl_trainer* t, double* max_abs_diff);

const char* trl_last_error(void);

/* ---- EXPERIMENT (not on the decision path, which stays f64): the policy's wide inner product terr_ip0 (5984 -> 64; cNeuralNet::Eval,
 * learning/NeuralNet.cpp:352-375) as a TMA-fed wgmma GEMM over a batch of decisions in split precision (csrc/trl_tc_policy.cu);
 * tools/tc_policy_probe.py measures what the narrow arithmetic does to real decisions.  kind: 0 = bf16 parts, 1 = tf32 parts.
 * trl_tc_split: x[rows][K] f64 -> planes[parts][rows][K]; trl_tc_fc: out[M][64] (FP32) = sum over the part pairs in `pairs` (bit 3 i + j)
 * of A_i[M][K] B_j[64][K]^T; all pointers are device pointers, stream is a cudaStream_t, *err_flag is set if a barrier wait gave up. */
int trl_tc_split(const double* x, long long rows, int K, int kind, int parts, void* planes, void* stream);
int trl_tc_fc(const void* a_planes, const void* b_planes, int M, int K, int kind, int parts, int pairs, int ksplit, float* out, int* err_flag,
              void* stream);
const char* trl_tc_last_error(void);

#ifdef __cplusplus
}
#endif
#endif
