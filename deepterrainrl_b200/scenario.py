"""Host-side mirror of the reference's per-env scenario API over a *batch* of environments.

Method names follow scenarios/ScenarioExp.h:16-40, ScenarioPoliEval.h:13-28 and ScenarioSimChar.h:49-82 so the
parity tests read like the reference's own call sites (scenarios/ScenarioTrain.cpp:376-410,
optimizer/scenarios/OptScenarioPoliEval.cpp:170-237).  Everything forwards to the C ABI (include/terrainrl_b200.h).
"""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

_PKG = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_PKG)
_LIB = None

ARCH_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a"]      # H100 (Hopper); the kernels use wgmma, TMA and clusters
NVCC_FLAGS = ARCH_FLAGS + ["-lineinfo", "-O3", "-std=c++17", "-Xcompiler", "-fPIC"]


# Experimental builds of the env-step kernel.  Selected with TRL_VARIANT=<name> in
# the environment of a measurement run; every variant is the same CUDA path compiled with one more -D flag and lives beside
# the product library (lib/variants/<name>/).  Unset = the product build.  There is still no CPU path behind any of them.
VARIANTS = {
    "kin_smem": ["-DTRL_KIN_SMEM=1"],
    "outward_smem": ["-DTRL_OUTWARD_SMEM=1"],    # since the chain passes: only the floating-base broadcast (parent -> child accelerations always use the link block)
    "smem_xchg": ["-DTRL_SMEM_XCHG=1"],
    "smem_xchg_3cta": ["-DTRL_SMEM_XCHG=1", "-DTRL_STEP_MIN_BLOCKS=3"],
    "noinline_cold": ["-DTRL_NOINLINE_COLD=1"],
    "regs96": ["-DTRL_STEP_MIN_BLOCKS=5"],       # 5 CTAs (20 warps) per SM at 96 registers, more spills; only makes sense with env groups
    "regs80": ["-DTRL_STEP_MIN_BLOCKS=6"],
    "phase_clocks": ["-DTRL_PHASE_CLOCKS=1"],    # per-phase clock64() sums of the step kernel (tools/step_phase_probe.py)
    "field_smem": ["-DTRL_FIELD_SMEM=1"],        # every per-env field staged in shared memory for the launch (one load batch, one store batch): not adopted
    "cta1": ["-DTRL_WARPS_PER_BLOCK=1", "-DTRL_STEP_MIN_BLOCKS=16"],     # CTA size of the step kernel: 1 / 2 / 8 warps (default 4), 16 warps per SM in all
    "cta2": ["-DTRL_WARPS_PER_BLOCK=2", "-DTRL_STEP_MIN_BLOCKS=8"],
    "cta8": ["-DTRL_WARPS_PER_BLOCK=8", "-DTRL_STEP_MIN_BLOCKS=2"],
    "table_const": ["-DTRL_TABLE_MIRROR=0"],     # lane-indexed model tables from constant memory (divergent LDC, the round-1 reads); the default reads a global-memory mirror
    "link_regs": ["-DTRL_LINK_SMEM=0"],          # the round-1 layout: per-lane link constants in registers (the default keeps them in shared memory)          # per-lane link constants in shared memory instead of ~28 registers (180 B instead of 216 B spilled)
    "reuse_kin": ["-DTRL_REUSE_KIN=1"],
    "smem_xchg_reuse_kin": ["-DTRL_SMEM_XCHG=1", "-DTRL_REUSE_KIN=1"],
    # decision kernel: register-tiled conv1 / conv2 (the untiled loops are shared-memory-bandwidth bound)
    "decide_tile2": ["-DTRL_DECIDE_TILE=1", "-DTRL_CONV_TILE=2"],
    "decide_tile4": ["-DTRL_DECIDE_TILE=1", "-DTRL_CONV_TILE=4"],
    "decide_tile4_128r": ["-DTRL_DECIDE_TILE=1", "-DTRL_CONV_TILE=4", "-DTRL_DECIDE_MIN_BLOCKS=1"],
    "smem_xchg_decide_tile4": ["-DTRL_SMEM_XCHG=1", "-DTRL_DECIDE_TILE=1", "-DTRL_CONV_TILE=4"],
    "all": ["-DTRL_SMEM_XCHG=1", "-DTRL_REUSE_KIN=1", "-DTRL_DECIDE_TILE=1", "-DTRL_CONV_TILE=4"],
}
# The body-slot units (trl_step_bs.cu, trl_step_bs_cg.cu) are not among them: a variant library links the product's body-slot objects,
# since their per-warp tables need TRL_LINK_SMEM=1 and fit the 48 KB of static shared memory only at the product's 4 warps per CTA.
STEP_UNITS = ("trl_step.cu", "trl_step_cg.cu", "trl_step_ts.cu", "trl_step_ts_cg.cu", "trl_step_ps.cu", "trl_step_ps_cg.cu")      # the only translation units the variant flags reach


def _variant():
    v = os.environ.get("TRL_VARIANT", "")
    if v and v not in VARIANTS:
        raise RuntimeError(f"TRL_VARIANT={v!r}: unknown variant (known: {sorted(VARIANTS)})")
    return v


def build_dir():
    """scratch directory of the native builds (TRL_BUILD_DIR, else one per user under the system's temporary directory)"""
    return os.environ.get("TRL_BUILD_DIR") or os.path.join(tempfile.gettempdir(), f"terrainrl_b200_build_{os.getuid()}")


def library_path():
    v = _variant()
    if v:
        return os.path.join(_PKG, "lib", "variants", v, "libterrainrl_b200.so")
    return os.path.join(_PKG, "lib", "libterrainrl_b200.so")


def build_library(force=False, verbose=False):
    """Compile csrc/*.cu for sm_90a into lib/libterrainrl_b200.so (nvcc cross-compiles without a GPU).
    trl_step_cg.cu is the env-step translation unit again with -Xptxas -dlcm=cg (L1-bypassing loads, see trl_step.cu);
    trl_step_ts.cu / trl_step_ts_cg.cu are both again with terrain slots, trl_step_ps.cu / trl_step_ps_cg.cu with terrain and
    physics slots, trl_step_bs.cu / trl_step_bs_cg.cu with terrain, physics and body slots.
    With TRL_VARIANT set, the env-step units of STEP_UNITS are compiled with the variant's flags and linked with the product's other
    objects (the body-slot build included) into lib/variants/<name>/."""
    variant = _variant()
    if variant:
        prev = os.environ.pop("TRL_VARIANT")
        try:
            build_library(force=False)          # the shared objects (host, trainer, loaders) come from the product build
        finally:
            os.environ["TRL_VARIANT"] = prev
    out = library_path()
    csrc = os.path.join(_PKG, "csrc")
    units = [("trl_step.cu", []), ("trl_step_cg.cu", ["-Xptxas", "-dlcm=cg"]), ("trl_step_ts.cu", []), ("trl_step_ts_cg.cu", ["-Xptxas", "-dlcm=cg"]),
             ("trl_step_ps.cu", []), ("trl_step_ps_cg.cu", ["-Xptxas", "-dlcm=cg"]),
             ("trl_step_bs.cu", []), ("trl_step_bs_cg.cu", ["-Xptxas", "-dlcm=cg"]),
             ("trl_host.cu", []), ("trl_train.cu", []), ("trl_checkpoint.cu", []),
             ("trl_comm.cu", []), ("trl_probe.cu", []), ("trl_tc_policy.cu", []), ("ref_loader.cpp", [])]
    deps = [os.path.join(csrc, f) for f in os.listdir(csrc)]
    deps.append(os.path.join(_ROOT, "include", "terrainrl_b200.h"))
    if not force and os.path.exists(out) and all(os.path.getmtime(out) >= os.path.getmtime(d) for d in deps):
        return out
    # objects live outside the tree, in a directory of this user (they are rebuilt from the sources where they are missing)
    base_objdir = os.path.join(build_dir(), "obj")
    objdir = os.path.join(base_objdir, "variants", variant) if variant else base_objdir
    os.makedirs(objdir, exist_ok=True)
    os.makedirs(os.path.dirname(out), exist_ok=True)
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    extra = os.environ.get("TRL_NVCC_EXTRA", "").split()     # developer knob (e.g. -DTRL_STEP_MIN_BLOCKS=7)
    extra += VARIANTS.get(variant, [])

    def compile_unit(unit):
        name, flags = unit
        if variant and name not in STEP_UNITS:
            return os.path.join(base_objdir, os.path.splitext(name)[0] + ".o")
        obj = os.path.join(objdir, os.path.splitext(name)[0] + ".o")
        cmd = [nvcc] + NVCC_FLAGS + extra + flags + (["-Xptxas", "-v"] if verbose else []) + ["-c", "-o", obj,
                                                                                              os.path.join(csrc, name)]
        subprocess.run(cmd, check=True)
        return obj

    from concurrent.futures import ThreadPoolExecutor
    with ThreadPoolExecutor(len(units)) as ex:
        objs = list(ex.map(compile_unit, units))
    subprocess.run([nvcc] + ARCH_FLAGS + ["-shared", "-o", out] + objs + ["-ldl"], check=True)
    return out


EXPORTS = [
    "trl_create_from_pack", "trl_create", "trl_pack_from_args", "trl_destroy", "trl_reset", "trl_seed_terrain", "trl_update", "trl_env_step", "trl_sync",
    "trl_set_explore", "trl_set_phys_params", "trl_set_weights", "trl_sizes", "trl_num_tuples", "trl_get_tuples",
    "trl_get_tuples_f64", "trl_reset_tuples", "trl_eval_stats", "trl_dist_log", "trl_reset_avg_dist", "trl_get_state", "trl_set_state",
    "trl_get_state_all", "trl_get_ctrl", "trl_get_poli_state", "trl_get_net_out", "trl_get_layer_state", "trl_get_terrain",
    "trl_kernel_launches", "trl_last_error", "trl_bench_updates", "trl_update_timed", "trl_device_tuple_block", "trl_snapshot", "trl_snapshot_wait", "trl_update_timed_detail", "trl_update_timeline", "trl_debug_time_decide", "trl_debug_decide", "trl_debug_fc_phases", "trl_debug_step_phases",
    "trl_load_model", "trl_output_model", "trl_write_model", "trl_get_output_offset_scale", "trl_pack_output_offset_scale",
    "trl_set_terrain_lerp", "trl_train_schedule", "trl_trainer_create", "trl_trainer_destroy", "trl_trainer_init_fresh", "trl_trainer_add_from_scene", "trl_trainer_add_tuples", "trl_trainer_add_device", "trl_trainer_train", "trl_train_run", "trl_train_run_timed",
    "trl_trainer_counters", "trl_trainer_num_params", "trl_trainer_launches", "trl_trainer_get", "trl_trainer_set_theta", "trl_trainer_list", "trl_trainer_rows",
    "trl_tuples_dropped", "trl_comm_unique_id", "trl_comm_init", "trl_comm_init_external", "trl_comm_destroy", "trl_comm_info", "trl_comm_set_env_offset",
    "trl_gather_tuples", "trl_gathered_blocks", "trl_gathered_fetch", "trl_gather_last_ms", "trl_trainer_add_gathered", "trl_trainer_broadcast",
    "trl_comm_broadcast_weights", "trl_comm_eval_stats", "trl_trainer_replica_spread", "trl_trainer_set_async",
    "trl_tc_split", "trl_tc_fc", "trl_tc_last_error", "trl_bench_last_span",
    "trl_load_policy", "trl_set_env_policy", "trl_eval_stats_slot",
    "trl_load_terrain", "trl_set_env_terrain", "trl_env_terrain", "trl_eval_stats_cell",
    "trl_trainer_create_slot", "trl_train_run_slots", "trl_output_model_slot",
    "trl_set_explore_slot", "trl_train_run_slots_sched",
    "trl_checkpoint_save", "trl_create_from_checkpoint", "trl_trainer_params", "trl_env_policy",
    "trl_load_physics", "trl_set_env_physics", "trl_env_physics", "trl_eval_stats_phys",
    "trl_set_env_eval", "trl_env_eval", "trl_eval_stats_mode",
    "trl_load_body", "trl_set_env_body", "trl_env_body", "trl_eval_stats_body",
    "trl_load_body_range", "trl_load_physics_range", "trl_env_body_draws", "trl_env_physics_draws",
    "trl_train_run_slots_comm", "trl_comm_eval_stats_slot",
]


def load_library():
    """dlopen the CUDA library; raises if it has not been built (no silent fallback)."""
    global _LIB
    if _LIB is None:
        path = library_path()
        if not os.path.exists(path):
            raise RuntimeError(f"{path} is missing: run __graft_entry__.build() (nvcc) first; there is no CPU fallback")
        L = C.CDLL(path)
        L.trl_create_from_pack.restype = C.c_void_p
        L.trl_create_from_pack.argtypes = [C.c_char_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_uint64]
        L.trl_last_error.restype = C.c_char_p
        L.trl_kernel_launches.restype = C.c_int64
        L.trl_kernel_launches.argtypes = [C.c_void_p]
        _LIB = L
    return _LIB


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def pack_from_args(args, data_root, out_path):
    """Native (C++) scene packer: reference arg tokens + checkout directory -> .trlpack (no GPU needed)."""
    L = load_library()
    argv = (C.c_char_p * len(args))(*[a.encode() for a in args])
    if L.trl_pack_from_args(len(args), argv, os.fspath(data_root).encode(), os.fspath(out_path).encode()) != 0:
        raise RuntimeError(L.trl_last_error().decode())
    return out_path


class BatchedScenario:
    """N environments of one scene stepped in lock-step on one GPU (one handle of the C ABI)."""

    MODE = 0

    def __init__(self, pack, num_envs, device=0, terrain_seeds=None, rng_seed=1234, args=None, data_root=None):
        """pack: path of a .trlpack; or pass args=[...] (cArgParser tokens) + data_root (a DeepTerrainRL checkout)."""
        self.L = load_library()
        seeds = None if terrain_seeds is None else np.ascontiguousarray(terrain_seeds, dtype=np.uint64)
        if args is not None:
            self.L.trl_create.restype = C.c_void_p
            argv = (C.c_char_p * len(args))(*[a.encode() for a in args])
            h = self.L.trl_create(len(args), argv, os.fspath(data_root or "").encode(), int(num_envs), int(device), self.MODE,
                                  _p(seeds), C.c_uint64(rng_seed))
        else:
            h = self.L.trl_create_from_pack(os.fspath(pack).encode(), int(num_envs), int(device), self.MODE, _p(seeds),
                                            C.c_uint64(rng_seed))
        if not h:
            raise RuntimeError("trl_create: " + self.L.trl_last_error().decode())
        self._attach(h)

    @classmethod
    def _wrap(cls, L, h):
        """a scenario object over a handle the library has already created (load_checkpoint)"""
        obj = cls.__new__(cls)
        obj.L = L
        obj._attach(h)
        return obj

    def _attach(self, h):
        self.h = C.c_void_p(h)
        v = [C.c_int(0) for _ in range(7)]
        self._ck(self.L.trl_sizes(self.h, *[C.byref(x) for x in v]))
        self.num_envs, self.state_size, self.action_size, self.num_frags, self.frag_size, self.num_dof, self.num_joints = \
            [x.value for x in v]
        self.tuple_width = 1 + self.state_size + self.action_size + self.state_size

    def _ck(self, rc):
        if rc != 0:
            raise RuntimeError(self.L.trl_last_error().decode())

    def close(self):
        if getattr(self, "h", None):
            self.L.trl_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- cScenario interface
    def Update(self, dt=1.0 / 30.0):
        self._ck(self.L.trl_update(self.h, C.c_double(dt)))

    def Reset(self, env_ids=None):
        ids = None if env_ids is None else np.ascontiguousarray(env_ids, dtype=np.int32)
        self._ck(self.L.trl_reset(self.h, _p(ids), 0 if ids is None else ids.size))

    def OutputModel(self, path, mtime=0, slot=0):
        """cNeuralNet::OutputModel of the policy the scenario evaluates (of policy slot `slot`: its trainer's net if it has one):
        Caffe-layout HDF5 + `<stem>_scale.txt`, written natively."""
        if slot == 0:
            self._ck(self.L.trl_output_model(self.h, path.encode(), C.c_uint32(mtime)))
        else:
            self._ck(self.L.trl_output_model_slot(self.h, int(slot), path.encode(), C.c_uint32(mtime)))

    def SaveCheckpoint(self, path, user=b""):
        """everything a later call on this scenario and its trainers reads, to `path` (trl_checkpoint_save), with the bytes `user`
        stored verbatim; deepterrainrl_b200.load_checkpoint resumes it bit for bit in another process.  The scenario is unchanged."""
        user = bytes(user)
        self._ck(self.L.trl_checkpoint_save(self.h, os.fspath(path).encode(), user, C.c_size_t(len(user))))

    def LoadModel(self, h5_path, scale_path=None):
        """cNeuralNet::LoadModel + LoadScale from the reference's file formats."""
        scale_path = scale_path or (os.path.splitext(h5_path)[0] + "_scale.txt")
        self._ck(self.L.trl_load_model(self.h, h5_path.encode(), scale_path.encode()))

    def LoadPolicy(self, slot, h5_path, scale_path=None):
        """a further model (same net topology) into policy slot 1..7 of an evaluation scenario; envs move to it with SetEnvPolicy"""
        scale_path = scale_path or (os.path.splitext(h5_path)[0] + "_scale.txt")
        self._ck(self.L.trl_load_policy(self.h, int(slot), h5_path.encode(), scale_path.encode()))

    def SetEnvPolicy(self, slots, env_ids=None):
        """env_ids[k] (default: env k) is evaluated by the model in slots[k] from its next decision on"""
        s = np.ascontiguousarray(slots, dtype=np.int32).ravel()
        ids = None if env_ids is None else np.ascontiguousarray(env_ids, dtype=np.int32).ravel()
        if ids is not None and ids.size != s.size:
            raise ValueError("SetEnvPolicy: one slot per env id")
        self._ck(self.L.trl_set_env_policy(self.h, _p(ids), _p(s), int(s.size)))
        if not hasattr(self, "_env_slot"):
            self._env_slot = np.zeros(self.num_envs, np.int32)
        self._env_slot[np.arange(s.size) if ids is None else ids] = s

    def EnvPolicy(self):
        """the slot of every env"""
        return getattr(self, "_env_slot", np.zeros(self.num_envs, np.int32)).copy()

    def LoadTerrain(self, slot, path):
        """a terrain file of the reference's format (as -terrain_file) into terrain slot 1..7; envs move to it with SetEnvTerrain"""
        self._ck(self.L.trl_load_terrain(self.h, int(slot), os.fspath(path).encode()))

    def SetEnvTerrain(self, slots, env_ids=None):
        """env_ids[k] (default: env k) generates its ground from terrain slot slots[k] from its next episode reset on"""
        s = np.ascontiguousarray(slots, dtype=np.int32).ravel()
        ids = None if env_ids is None else np.ascontiguousarray(env_ids, dtype=np.int32).ravel()
        if ids is not None and ids.size != s.size:
            raise ValueError("SetEnvTerrain: one slot per env id")
        self._ck(self.L.trl_set_env_terrain(self.h, _p(ids), _p(s), int(s.size)))

    def EnvTerrain(self):
        """(current, assigned): per env, the terrain slot its present ground came from and the one it uses after its next reset"""
        cur = np.zeros(self.num_envs, np.int32)
        nxt = np.zeros(self.num_envs, np.int32)
        self._ck(self.L.trl_env_terrain(self.h, _p(cur), _p(nxt), self.num_envs))
        return cur, nxt

    def LoadPhysics(self, slot, p7, vertex_contacts=False):
        """contact / joint-limit parameters (SetPhysParams order: kn, dn, mu, v_eps, contact_tol, k_lim, d_lim) and the vertex contact
        model into physics slot 1..7; envs move to it with SetEnvPhysics.  Reloading a slot acts from the next env-step."""
        a = np.ascontiguousarray(p7, dtype=np.float64).ravel()
        if a.size != 7:
            raise ValueError("LoadPhysics: 7 parameters")
        self._ck(self.L.trl_load_physics(self.h, int(slot), _p(a), int(bool(vertex_contacts))))

    def SetEnvPhysics(self, slots, env_ids=None):
        """env_ids[k] (default: env k) runs on physics slot slots[k] from its next episode reset on"""
        s = np.ascontiguousarray(slots, dtype=np.int32).ravel()
        ids = None if env_ids is None else np.ascontiguousarray(env_ids, dtype=np.int32).ravel()
        if ids is not None and ids.size != s.size:
            raise ValueError("SetEnvPhysics: one slot per env id")
        self._ck(self.L.trl_set_env_physics(self.h, _p(ids), _p(s), int(s.size)))

    def EnvPhysics(self):
        """(current, assigned): per env, the physics slot of its present episode and the one it gets at its next reset"""
        cur = np.zeros(self.num_envs, np.int32)
        nxt = np.zeros(self.num_envs, np.int32)
        self._ck(self.L.trl_env_physics(self.h, _p(cur), _p(nxt), self.num_envs))
        return cur, nxt

    def LoadBody(self, slot, path):
        """a character file of the reference's format (as -character_file) into body slot 1..7; envs move to it with SetEnvBody.  The
        file must have the scene's topology and controllers; its masses, dimensions, joint limits and PD gains may differ.  A relative
        path (and the controller files it names) refers to the scenario's data_root."""
        self._ck(self.L.trl_load_body(self.h, int(slot), os.fspath(path).encode()))

    def SetEnvBody(self, slots, env_ids=None):
        """env_ids[k] (default: env k) runs on body slot slots[k] from its next episode reset on"""
        s = np.ascontiguousarray(slots, dtype=np.int32).ravel()
        ids = None if env_ids is None else np.ascontiguousarray(env_ids, dtype=np.int32).ravel()
        if ids is not None and ids.size != s.size:
            raise ValueError("SetEnvBody: one slot per env id")
        self._ck(self.L.trl_set_env_body(self.h, _p(ids), _p(s), int(s.size)))

    def EnvBody(self):
        """(current, assigned): per env, the body slot of its present episode and the one it gets at its next reset"""
        cur = np.zeros(self.num_envs, np.int32)
        nxt = np.zeros(self.num_envs, np.int32)
        self._ck(self.L.trl_env_body(self.h, _p(cur), _p(nxt), self.num_envs))
        return cur, nxt

    def LoadBodyRange(self, slot, lo_path, hi_path):
        """a ranged body slot 1..7 (domain randomization): at every episode reset of an env on it, each link's Mass, Kp, Kd and
        TorqueLim are drawn uniformly between the lo and hi character files' values (include/terrainrl_b200.h gives the recipe).
        Both files must pass LoadBody's checks and agree in everything else.  Envs move to it with SetEnvBody."""
        self._ck(self.L.trl_load_body_range(self.h, int(slot), os.fspath(lo_path).encode(), os.fspath(hi_path).encode()))

    def LoadPhysicsRange(self, slot, lo7, hi7, vertex_contacts=False):
        """a ranged physics slot 1..7: at every episode reset of an env on it, each of the seven constants (LoadPhysics order) is drawn
        uniformly in [lo7[k], hi7[k]].  Envs move to it with SetEnvPhysics."""
        lo = np.ascontiguousarray(lo7, dtype=np.float64).ravel()
        hi = np.ascontiguousarray(hi7, dtype=np.float64).ravel()
        if lo.size != 7 or hi.size != 7:
            raise ValueError("LoadPhysicsRange: 7 parameters at each end")
        self._ck(self.L.trl_load_physics_range(self.h, int(slot), _p(lo), _p(hi), int(bool(vertex_contacts))))

    def EnvBodyDraws(self):
        """(numbers [n][4][nj]: Mass, Kp, Kd, TorqueLim of every env's present episode; draws [n]: its body draws so far).  An env on a
        fixed body slot reports its slot's numbers."""
        out = np.zeros((self.num_envs, 4, self.num_joints), np.float64)
        draws = np.zeros(self.num_envs, np.int64)
        self._ck(self.L.trl_env_body_draws(self.h, _p(out), _p(draws)))
        return out, draws

    def EnvPhysicsDraws(self):
        """(numbers [n][7] of every env's present episode in LoadPhysics order; draws [n]: its physics draws so far)"""
        out = np.zeros((self.num_envs, 7), np.float64)
        draws = np.zeros(self.num_envs, np.int64)
        self._ck(self.L.trl_env_physics_draws(self.h, _p(out), _p(draws)))
        return out, draws

    def SetEnvEval(self, flags, env_ids=None):
        """env_ids[k] (default: env k) of an exploration scenario evaluates its policy slot's current net, exploration off and no
        tuples recorded, from its next episode reset on if flags[k] is true; it explores again from its next reset if false"""
        f = np.ascontiguousarray(flags, dtype=np.int32).ravel()
        ids = None if env_ids is None else np.ascontiguousarray(env_ids, dtype=np.int32).ravel()
        if ids is not None and ids.size != f.size:
            raise ValueError("SetEnvEval: one flag per env id")
        self._ck(self.L.trl_set_env_eval(self.h, _p(ids), _p(f), int(f.size)))

    def EnvEval(self):
        """(current, assigned): per env, whether its present episode evaluates and whether the one after its next reset will"""
        cur = np.zeros(self.num_envs, np.int32)
        nxt = np.zeros(self.num_envs, np.int32)
        self._ck(self.L.trl_env_eval(self.h, _p(cur), _p(nxt), self.num_envs))
        return cur.astype(bool), nxt.astype(bool)

    def GetOutputOffsetScale(self):
        """cBaseControllerMACE::BuildNNOutputOffsetScale."""
        n = self.num_frags * (1 + self.frag_size)
        off = np.zeros(n); scale = np.zeros(n)
        self._ck(self.L.trl_get_output_offset_scale(self.h, _p(off), _p(scale), n))
        return off, scale

    def SetTerrainParamsLerp(self, lerp):
        """cScenarioSimChar::SetTerrainParamsLerp (scenarios/ScenarioSimChar.cpp:255-272)."""
        self._ck(self.L.trl_set_terrain_lerp(self.h, C.c_double(lerp)))

    def SetRandSeed(self, seeds):
        s = np.ascontiguousarray(seeds, dtype=np.uint64)
        self._ck(self.L.trl_seed_terrain(self.h, _p(s), s.size))

    def Sync(self):
        self._ck(self.L.trl_sync(self.h))

    def EnvStep(self, h=1.0 / 600.0):
        self._ck(self.L.trl_env_step(self.h, C.c_double(h)))

    def SetPhysParams(self, p7):
        a = np.ascontiguousarray(p7, dtype=np.float64)
        self._ck(self.L.trl_set_phys_params(self.h, _p(a)))

    def SetWeights(self, blobs, in_off, in_scale, out_off, out_scale):
        blobs = [np.ascontiguousarray(b, dtype=np.float64).ravel() for b in blobs]
        ptrs = (C.c_void_p * len(blobs))(*[b.ctypes.data for b in blobs])
        counts = np.array([b.size for b in blobs], dtype=np.int64)
        vs = [np.ascontiguousarray(v, dtype=np.float64) for v in (in_off, in_scale, out_off, out_scale)]
        self._ck(self.L.trl_set_weights(self.h, ptrs, _p(counts), len(blobs), *[_p(v) for v in vs]))

    # ---- state probes
    def GetState(self, env=0):
        q = np.zeros(self.num_dof); qd = np.zeros(self.num_dof); tau = np.zeros(self.num_dof)
        c = np.zeros(self.num_joints, np.uint8)
        self._ck(self.L.trl_get_state(self.h, env, _p(q), _p(qd), _p(tau), _p(c)))
        return q, qd, tau, c

    def SetState(self, env=0, q=None, qd=None, tau=None, contact=None):
        f = lambda a, t: None if a is None else np.ascontiguousarray(a, dtype=t)
        q, qd, tau, contact = f(q, np.float64), f(qd, np.float64), f(tau, np.float64), f(contact, np.uint8)
        self._ck(self.L.trl_set_state(self.h, env, _p(q), _p(qd), _p(tau), _p(contact)))

    def GetStateAll(self):
        q = np.zeros((self.num_dof, self.num_envs)); qd = np.zeros((self.num_dof, self.num_envs))
        self._ck(self.L.trl_get_state_all(self.h, _p(q), _p(qd)))
        return q, qd

    def GetCtrl(self, env=0):
        out = np.zeros(160)
        n = C.c_int(0)
        self._ck(self.L.trl_get_ctrl(self.h, env, _p(out), 160, C.byref(n)))
        return out[:n.value]

    def GetPoliState(self, env=0):
        s = np.zeros(self.state_size)
        self._ck(self.L.trl_get_poli_state(self.h, env, _p(s)))
        return s

    def GetNetOut(self, env=0, n=90):
        y = np.zeros(96)
        self._ck(self.L.trl_get_net_out(self.h, env, _p(y)))
        return y[:n]

    def DebugDecide(self, env_ids, poli_states=None):
        """tests: one decision pass over exactly these envs (row k = env_ids[k]), after writing poli_states ([n, state_size]) into
        their policy states if given"""
        ids = np.ascontiguousarray(env_ids, dtype=np.int32).ravel()
        x = None if poli_states is None else np.ascontiguousarray(poli_states, dtype=np.float64).reshape(ids.size, self.state_size)
        self._ck(self.L.trl_debug_decide(self.h, _p(ids), int(ids.size), _p(x)))

    def GetLayerState(self, layer_name, env=0):
        """cNeuralNet::GetLayerState: the named blob of the deploy net for the policy state of env's last decision"""
        out = np.zeros(8192)
        n = C.c_int(0)
        self._ck(self.L.trl_get_layer_state(self.h, int(env), layer_name.encode(), _p(out), out.size, C.byref(n)))
        return out[:n.value].copy()

    def GetTerrain(self, env=0, seg=0, cap=512):
        d = np.zeros(cap, np.float32)
        n = C.c_int(0); mx = C.c_double(0); fl = C.c_int(0)
        self._ck(self.L.trl_get_terrain(self.h, env, seg, _p(d), cap, C.byref(n), C.byref(mx), C.byref(fl)))
        return d[:min(n.value, cap)].copy(), mx.value, fl.value

    def Snapshot(self):
        """enqueue a capture of all poses / velocities + batch counters behind the submitted updates"""
        self._ck(self.L.trl_snapshot(self.h))

    def SnapshotWait(self, pose=None, vel=None):
        """wait for the last Snapshot(); fills pose / vel ([num_dof, num_envs] float64 arrays) and returns the counters"""
        c = C.c_int64(0); e = C.c_int64(0); a = C.c_double(0); s = C.c_int64(0)
        self._ck(self.L.trl_snapshot_wait(self.h, _p(pose), _p(vel), C.byref(c), C.byref(e), C.byref(a), C.byref(s)))
        return dict(cycles=c.value, episodes=e.value, avg_dist=a.value, steps=s.value)

    def KernelLaunches(self):
        return int(self.L.trl_kernel_launches(self.h))

    def BenchUpdates(self, k, dt=1.0 / 30.0, flush_l2=True):
        """k outer updates, device-timed on the library's stream with one event pair per update (the optional L2 flush sits between the
        pairs); returns the summed milliseconds.  BenchLastSpan() = first start to last end, flushes included."""
        ms = C.c_double(0)
        self._ck(self.L.trl_bench_updates(self.h, C.c_double(dt), int(k), int(bool(flush_l2)), C.byref(ms)))
        return ms.value

    def BenchLastSpan(self):
        ms = C.c_double(0)
        self._ck(self.L.trl_bench_last_span(self.h, C.byref(ms)))
        return ms.value

    def UpdateTimedDetail(self, dt=1.0 / 30.0, num_update_steps=20):
        ps = np.zeros(num_update_steps + 1); pd = np.zeros(num_update_steps)
        self._ck(self.L.trl_update_timed_detail(self.h, C.c_double(dt), _p(ps), _p(pd)))
        return ps, pd

    def UpdateTimeline(self, dt=1.0 / 30.0):
        """one update in Update()'s own schedule, every launch timed on its stream: list of (kind, index, start_ms, end_ms);
        kind 0 terrain, 1 step, 2 decision, 3 catch-up"""
        out = np.zeros(4 * 128)
        n = C.c_int(0)
        self._ck(self.L.trl_update_timeline(self.h, C.c_double(dt), _p(out), 128, C.byref(n)))
        return [(int(out[4 * k]), int(out[4 * k + 1]), float(out[4 * k + 2]), float(out[4 * k + 3])) for k in range(n.value)]

    def UpdateTimed(self, dt=1.0 / 30.0):
        """one outer update with per-launch events: (step_ms, step_launches, decide_ms, decide_launches)."""
        sm = C.c_double(0); dm = C.c_double(0); sl = C.c_int(0); dl = C.c_int(0)
        self._ck(self.L.trl_update_timed(self.h, C.c_double(dt), C.byref(sm), C.byref(sl), C.byref(dm), C.byref(dl)))
        return sm.value, sl.value, dm.value, dl.value

    # ---- cScenarioPoliEval statistics
    def _stats(self):
        c = C.c_int64(0); e = C.c_int64(0); a = C.c_double(0); s = C.c_int64(0)
        self._ck(self.L.trl_eval_stats(self.h, C.byref(c), C.byref(e), C.byref(a), C.byref(s)))
        return dict(cycles=c.value, episodes=e.value, avg_dist=a.value, steps=s.value)

    def GetNumCycles(self):
        return self._stats()["cycles"]

    def GetNumEpisodes(self):
        return self._stats()["episodes"]

    def GetAvgDist(self):
        return self._stats()["avg_dist"]

    def ResetAvgDist(self):
        self._ck(self.L.trl_reset_avg_dist(self.h))

    def GetNumEnvSteps(self):
        return self._stats()["steps"]

    def GetEvalStats(self, slot=0, terrain=None, physics=None, mode=None, body=None):
        """cycles / episodes / avg_dist / env-steps of the envs now on policy slot `slot` (None: any) whose present ground comes from
        terrain slot `terrain` (None: any), whose present episode runs on physics slot `physics` (None: any), in mode `mode`
        (TRL_MODE_POLI_EVAL = 0 evaluates, TRL_MODE_EXPLORE = 1 explores; None: any) and on body slot `body` (None: any)"""
        c = C.c_int64(0); e = C.c_int64(0); a = C.c_double(0); s = C.c_int64(0)
        if body is not None:
            rc = self.L.trl_eval_stats_body(self.h, -1 if mode is None else int(mode), -1 if slot is None else int(slot),
                                            -1 if terrain is None else int(terrain), -1 if physics is None else int(physics), int(body),
                                            C.byref(c), C.byref(e), C.byref(a), C.byref(s))
        elif mode is not None:
            rc = self.L.trl_eval_stats_mode(self.h, int(mode), -1 if slot is None else int(slot), -1 if terrain is None else int(terrain),
                                            -1 if physics is None else int(physics), C.byref(c), C.byref(e), C.byref(a), C.byref(s))
        elif physics is not None:
            rc = self.L.trl_eval_stats_phys(self.h, -1 if slot is None else int(slot), -1 if terrain is None else int(terrain), int(physics),
                                            C.byref(c), C.byref(e), C.byref(a), C.byref(s))
        elif terrain is None and slot is not None:
            rc = self.L.trl_eval_stats_slot(self.h, int(slot), C.byref(c), C.byref(e), C.byref(a), C.byref(s))
        else:
            rc = self.L.trl_eval_stats_cell(self.h, -1 if slot is None else int(slot), -1 if terrain is None else int(terrain),
                                            C.byref(c), C.byref(e), C.byref(a), C.byref(s))
        self._ck(rc)
        return dict(cycles=c.value, episodes=e.value, avg_dist=a.value, steps=s.value)

    def GetDistLog(self, slot=None, terrain=None, physics=None, mode=None, body=None):
        """(distances, env ids) of the episodes logged so far; slot / terrain / physics / mode / body: only the entries of envs now on
        that policy slot / whose present ground comes from that terrain slot / whose present episode runs on that physics slot / whose
        present episode runs in that mode (0 evaluates, 1 explores) / whose present episode runs on that body slot.  Every filter reads the env's present assignment, not the one of
        the logged episode: only evaluating episodes log a distance, but an env that has gone back to exploring keeps its entries,
        which mode=1 then returns and mode=0 drops."""
        d = C.c_void_p(); e = C.c_void_p(); n = C.c_int(0)
        self._ck(self.L.trl_dist_log(self.h, C.byref(d), C.byref(e), C.byref(n)))
        if n.value == 0:
            return np.zeros(0), np.zeros(0, np.int32)
        dist = np.ctypeslib.as_array(C.cast(d, C.POINTER(C.c_double)), (n.value,)).copy()
        env = np.ctypeslib.as_array(C.cast(e, C.POINTER(C.c_int32)), (n.value,)).copy()
        if slot is not None:
            keep = self.EnvPolicy()[env] == slot
            dist, env = dist[keep], env[keep]
        if terrain is not None:
            keep = self.EnvTerrain()[0][env] == terrain
            dist, env = dist[keep], env[keep]
        if physics is not None:
            keep = self.EnvPhysics()[0][env] == physics
            dist, env = dist[keep], env[keep]
        if mode is not None:
            keep = self.EnvEval()[0][env] == (int(mode) == 0)
            dist, env = dist[keep], env[keep]
        if body is not None:
            keep = self.EnvBody()[0][env] == body
            dist, env = dist[keep], env[keep]
        return dist, env


class ScenarioPoliEval(BatchedScenario):
    """cScenarioPoliEval over a batch (scenarios/ScenarioPoliEval.h:13-28)."""
    MODE = 0


class ScenarioExpMACE(BatchedScenario):
    """cScenarioExpMACE over a batch (scenarios/ScenarioExp.h:16-40, ScenarioExpMACE.h)."""
    MODE = 1

    def EnableExplore(self, enable, rate, temp, base_rate, slot=None):
        """the exploration settings of every env, or (slot = p) only of the envs on policy slot p"""
        if slot is None:
            self._ck(self.L.trl_set_explore(self.h, int(enable), C.c_double(rate), C.c_double(temp), C.c_double(base_rate)))
        else:
            self._ck(self.L.trl_set_explore_slot(self.h, int(slot), int(enable), C.c_double(rate), C.c_double(temp),
                                                 C.c_double(base_rate)))

    def GetNumTuples(self):
        n = C.c_int(0)
        self._ck(self.L.trl_num_tuples(self.h, C.byref(n)))
        return n.value

    def IsTupleBufferFull(self, tuple_buffer_size=32):
        return self.GetNumTuples() >= tuple_buffer_size

    def GetTuples(self, f64=False):
        rows = C.c_void_p(); fl = C.c_void_p(); ev = C.c_void_p(); n = C.c_int(0)
        fn = self.L.trl_get_tuples_f64 if f64 else self.L.trl_get_tuples
        self._ck(fn(self.h, C.byref(rows), C.byref(fl), C.byref(ev), C.byref(n)))
        W = self.tuple_width
        if n.value == 0:
            return (np.zeros((0, W), np.float64 if f64 else np.float32), np.zeros(0, np.uint32), np.zeros(0, np.int32))
        ct = C.c_double if f64 else C.c_float
        r = np.ctypeslib.as_array(C.cast(rows, C.POINTER(ct)), (n.value, W)).copy()
        f = np.ctypeslib.as_array(C.cast(fl, C.POINTER(C.c_uint32)), (n.value,)).copy()
        e = np.ctypeslib.as_array(C.cast(ev, C.POINTER(C.c_int32)), (n.value,)).copy()
        return r, f, e

    def ResetTupleBuffer(self):
        self._ck(self.L.trl_reset_tuples(self.h))

    def DeviceTupleBlock(self):
        """torch views (zero-copy) of the device tuple block: rows f64 [cap, W], flags i32 [cap], env i32 [cap], count i32 [1]."""
        import torch
        ptrs = [C.c_void_p() for _ in range(4)]
        cap = C.c_int(0); width = C.c_int(0)
        self._ck(self.L.trl_device_tuple_block(self.h, *[C.byref(p) for p in ptrs], C.byref(cap), C.byref(width)))

        class _Arr:
            def __init__(self, ptr, shape, typestr):
                self.__cuda_array_interface__ = {"shape": shape, "typestr": typestr, "data": (ptr, False), "version": 2}

        dev = torch.device("cuda", torch.cuda.current_device())
        rows = torch.as_tensor(_Arr(ptrs[0].value, (cap.value, width.value), "<f8"), device=dev)
        flags = torch.as_tensor(_Arr(ptrs[1].value, (cap.value,), "<i4"), device=dev)
        env = torch.as_tensor(_Arr(ptrs[2].value, (cap.value,), "<i4"), device=dev)
        count = torch.as_tensor(_Arr(ptrs[3].value, (1,), "<i4"), device=dev)
        return rows, flags, env, count
