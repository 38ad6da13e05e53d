"""Python mirror of cMACETrainer / cNeuralNetLearner over the C ABI (trl_trainer_*).  The trainer lives on the GPU next to the
scenario it was created from: tuples move device to device, and the scenario's decision kernel evaluates the trainer's weights
in place (learning/NeuralNetLearner.cpp:33-45,83-87)."""
import ctypes as C
import os

import numpy as np

from .scenario import load_library

NET_LAYERS = ["terr_conv0", "terr_conv1", "terr_conv2", "terr_ip0", "ip0", "val_ip0", "val_ip1",
              "a0_ip0", "a0_ip1", "a1_ip0", "a1_ip1", "a2_ip0", "a2_ip1"]


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


class MACETrainer:
    """cTrainerInterface::tParams defaults as set by cScenarioTrainMACE for the shipped training runs
    (scenarios/ScenarioTrain.cpp:8-35, args/opt_args_train_mace.txt) and data/policies/dog/nets/dog_mace3_solver.prototxt."""

    DEFAULTS = dict(replay_mem_size=500000, num_init_samples=50000, num_steps_per_iter=1, freeze_target_iters=500,
                    init_input_offset_scale=1, discount=0.9, base_lr=1e-3, momentum=0.9, weight_decay=5e-4, seed=1)

    def __init__(self, scenario, slot=0, model=None, **kw):
        """slot: the policy slot this trainer trains (0: the scenario's own policy; 1..7: a training slot of an exploration
        scenario, whose envs are moved to it with SetEnvPolicy).  model: (h5_path, scale_path) of the starting net; None = the net
        slot 0 evaluates now."""
        self.L = load_library()
        L = self.L
        L.trl_trainer_create_slot.restype = C.c_void_p
        L.trl_trainer_create_slot.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_char_p, C.c_char_p]
        L.trl_trainer_launches.restype = C.c_int64
        for name in ("trl_trainer_destroy", "trl_trainer_add_from_scene", "trl_trainer_add_tuples", "trl_trainer_train",
                     "trl_trainer_add_device", "trl_trainer_counters", "trl_trainer_get", "trl_trainer_set_theta", "trl_trainer_list"):
            getattr(L, name).restype = C.c_int
        p = dict(self.DEFAULTS)
        p.update(kw)
        self.params = p
        arr = np.array([p[k] for k in self.PARAM_KEYS], float)
        self.slot = int(slot)
        h5, scale = (None, None) if model is None else (os.fspath(model[0]).encode(), os.fspath(model[1]).encode())
        h = L.trl_trainer_create_slot(scenario.h, self.slot, _p(arr), h5, scale)
        if not h:
            raise RuntimeError(L.trl_last_error().decode())
        self._attach(scenario, h)

    PARAM_KEYS = ("replay_mem_size", "num_init_samples", "num_steps_per_iter", "freeze_target_iters", "init_input_offset_scale",
                  "discount", "base_lr", "momentum", "weight_decay", "seed")

    @classmethod
    def _wrap(cls, scenario, h):
        """a trainer object over a trainer the library has already created (load_checkpoint): parameters and slot as created"""
        obj = cls.__new__(cls)
        obj.L = scenario.L
        p = np.zeros(10)
        slot = C.c_int(0)
        if obj.L.trl_trainer_params(C.c_void_p(h), _p(p), C.byref(slot)) != 0:
            raise RuntimeError(obj.L.trl_last_error().decode())
        obj.params = {k: (float(v) if k in ("discount", "base_lr", "momentum", "weight_decay") else int(v)) for k, v in zip(cls.PARAM_KEYS, p)}
        obj.slot = slot.value
        obj._attach(scenario, h)
        return obj

    def _attach(self, scenario, h):
        self.scenario = scenario
        self.h = C.c_void_p(h)
        self.num_params = self.L.trl_trainer_num_params(self.h)
        self.S, self.A = scenario.state_size, scenario.action_size
        self.n_out = scenario.num_frags * (1 + scenario.frag_size)
        self.W = 1 + 2 * self.S + self.A

    def close(self):
        if getattr(self, "h", None):
            self.L.trl_trainer_destroy(self.h)
            self.h = None

    def __del__(self):
        self.close()

    def _ck(self, rc):
        if rc != 0:
            raise RuntimeError(self.L.trl_last_error().decode())

    def InitFresh(self, seed=1):
        """Start from a freshly initialised net (no -policy_model): xavier weights, controller-derived output offset / scale."""
        self._ck(self.L.trl_trainer_init_fresh(self.h, C.c_uint64(seed)))

    # ---- cNeuralNetLearner::Train = AddTuples + Train + SyncNet
    def AddTuplesFromScene(self):
        self._ck(self.L.trl_trainer_add_from_scene(self.h))

    def AddTuples(self, rows, flags):
        rows = np.ascontiguousarray(rows, np.float64)
        flags = np.ascontiguousarray(flags, np.uint32)
        assert rows.ndim == 2 and rows.shape[1] == self.W
        self._ck(self.L.trl_trainer_add_tuples(self.h, _p(rows), _p(flags), rows.shape[0]))

    def AddTuplesDevice(self, rows, flags):
        """rows: CUDA tensor [n, W] (any float dtype), flags: CUDA int tensor [n] -- e.g. the output of
        parallel.unpack_tuple_blocks.  The scenario's stream waits for the current torch stream first."""
        import torch
        n = int(rows.shape[0])
        if n == 0:
            return
        r64 = rows.to(torch.float64).contiguous()
        f32 = flags.to(torch.int32).contiguous()
        torch.cuda.current_stream().synchronize()          # producer (NCCL / torch kernels) done before the engine stream reads
        cap = self.params["replay_mem_size"]
        step = 4096
        for b in range(0, n, step):
            e = min(n, b + step)
            self._ck(self.L.trl_trainer_add_device(self.h, C.c_void_p(r64[b:e].data_ptr()), C.c_void_p(f32[b:e].data_ptr()), e - b))
        self.scenario.Sync()                               # the tensors may be freed once the copies have run

    def SetAsync(self, enable=True):
        """Asynchronous training (trl_trainer_set_async): the intake and iterations run on their own stream beside the next update,
        and the envs explore with a snapshot of the net refreshed between updates.  Needs a communicator on the scenario."""
        self._ck(self.L.trl_trainer_set_async(self.h, 1 if enable else 0))

    def Train(self, iters=1):
        self._ck(self.L.trl_trainer_train(self.h, int(iters)))

    def counters(self):
        c = np.zeros(9, np.int64)
        l = np.zeros(2)
        self._ck(self.L.trl_trainer_counters(self.h, _p(c), _p(l)))
        out = dict(zip(("iter", "actor_iter", "stage", "num", "head", "total", "critic", "actor", "actor_batch"), c.tolist()))
        out["critic_loss"], out["actor_loss"] = float(l[0]), float(l[1])
        return out

    def GetIter(self):
        return self.counters()["iter"]

    def GetNumTuples(self):
        return self.counters()["num"]

    def get(self, what):
        idx = {"theta": 0, "target": 1, "history": 2, "in_off": 3, "in_scale": 4, "out_off": 5, "out_scale": 6, "grad": 7}[what]
        n = self.num_params if idx in (0, 1, 2, 7) else (self.S if idx in (3, 4) else self.n_out)
        out = np.zeros(n)
        self._ck(self.L.trl_trainer_get(self.h, idx, _p(out)))
        return out

    def set_theta(self, theta):
        theta = np.ascontiguousarray(theta, np.float64)
        assert theta.size == self.num_params
        self._ck(self.L.trl_trainer_set_theta(self.h, _p(theta)))

    def lists(self, which):
        cap = max(self.params["replay_mem_size"], 64)
        out = np.zeros(cap, np.int32)
        n = C.c_int(0)
        self._ck(self.L.trl_trainer_list(self.h, {"critic": 0, "actor": 1, "actor_batch": 2, "last_ids": 3}[which], _p(out), cap, C.byref(n)))
        return out[:n.value].copy()

    def rows(self, slots):
        slots = np.ascontiguousarray(slots, np.int32)
        rows = np.zeros((slots.size, self.W), np.float32)
        flags = np.zeros(slots.size, np.int32)
        self._ck(self.L.trl_trainer_rows(self.h, _p(slots), slots.size, _p(rows), _p(flags)))
        return rows, flags

    def KernelLaunches(self):
        return int(self.L.trl_trainer_launches(self.h))

    def blobs(self, theta=None):
        """Split a flat parameter vector into the 26 Caffe blobs {layer: (w, b)} in NET_LAYERS order."""
        theta = self.get("theta") if theta is None else theta
        n_char = self.S - 200
        frag, nf = self.scenario.frag_size, self.scenario.num_frags
        shapes = [(16, 1, 1, 8), (32, 16, 1, 4), (32, 32, 1, 4), (64, 32 * 187), (256, 64 + n_char)]
        for hd in range(4):
            shapes += [(128, 256), ((nf if hd == 0 else frag), 128)]
        out, o = {}, 0
        for name, shp in zip(NET_LAYERS, shapes):
            nw = int(np.prod(shp))
            w = theta[o:o + nw].reshape(shp); o += nw
            b = theta[o:o + shp[0]].copy(); o += shp[0]
            out[name] = (w.copy(), b)
        assert o == theta.size
        return out
