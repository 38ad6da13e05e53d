"""Multi-GPU plumbing: environments shard across ranks (one process per GPU), no collective in the rollout data path.

The exchange itself is native (csrc/trl_comm.cu, include/terrainrl_b200.h `trl_comm_*`, `trl_gather_tuples`,
`trl_trainer_add_gathered`, `trl_trainer_broadcast`): a device pack kernel + ONE all-gather of a fixed-capacity tuple block per
rank and outer update on a side stream, replacing the reference's in-process `learner->Train(exp->GetTuples())` under the
trainer mutex (scenarios/ScenarioTrain.cpp:388-395, learning/NeuralNetLearner.cpp:33-46), and a broadcast for `SyncNet`
(learning/NeuralNetLearner.cpp:85-89).  This module is only the ctypes mirror of those entry points plus the rendezvous glue a
Python launcher needs (shipping the NCCL unique id through torch.distributed, or wrapping a torch.distributed group as the
external-collectives backend for CPU tests over gloo).
"""
import ctypes as C

import numpy as np


def shard_seeds(rank, envs_per_rank, base=1):
    """Terrain seed of env i on rank r: base + r * envs_per_rank + i (SURVEY.md §8d, config 4)."""
    return np.arange(base + rank * envs_per_rank, base + (rank + 1) * envs_per_rank, dtype=np.uint64)


class _Collectives(C.Structure):
    AG = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p)
    BC = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.c_void_p)
    AR = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p)
    _fields_ = [("ctx", C.c_void_p), ("all_gather", AG), ("broadcast", BC), ("all_reduce_sum_f64", AR)]


class Comm:
    """The communicator of one BatchedScenario (one rank).  backend="nccl": the library opens libnccl itself; the 128-byte
    unique id is created on rank 0 and shipped through `torch.distributed` (any backend) or given as `unique_id`.
    backend="external": the collectives are the given torch.distributed group's (host memory: the emulator build / gloo)."""

    def __init__(self, scenario, rank, world, backend="nccl", unique_id=None, group=None):
        self.sc, self.rank, self.world = scenario, int(rank), int(world)
        self.L = scenario.L
        L = self.L
        L.trl_comm_init.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int]
        L.trl_gather_tuples.argtypes = [C.c_void_p, C.c_int]
        L.trl_comm_set_env_offset.argtypes = [C.c_void_p, C.c_int64]
        self._keep = None
        if backend == "nccl":
            if unique_id is None:
                unique_id = self.exchange_unique_id(L, self.rank, group)
            buf = (C.c_ubyte * 128).from_buffer_copy(bytes(unique_id))
            self._ck(L.trl_comm_init(scenario.h, buf, self.rank, self.world))
        elif backend == "external":
            self._keep = self._torch_collectives(group)
            self._ck(L.trl_comm_init_external(scenario.h, C.byref(self._keep[0]), self.rank, self.world))
        else:
            raise ValueError(backend)

    def _ck(self, rc):
        if rc != 0:
            raise RuntimeError(self.L.trl_last_error().decode())

    @staticmethod
    def exchange_unique_id(L, rank, group=None):
        """rank 0 asks the library (ncclGetUniqueId) and broadcasts the 128 bytes over torch.distributed"""
        import torch
        import torch.distributed as dist
        buf = (C.c_ubyte * 128)()
        if rank == 0 and L.trl_comm_unique_id(buf) != 0:
            raise RuntimeError(L.trl_last_error().decode())
        dev = "cuda" if dist.get_backend(group) == "nccl" else "cpu"
        t = torch.tensor(list(bytes(buf)), dtype=torch.uint8, device=dev)
        dist.broadcast(t, src=0, group=group)
        return bytes(t.cpu().tolist())

    @staticmethod
    def _torch_collectives(group):
        """trl_collectives over a torch.distributed group, for buffers in host memory (the library hands over raw pointers)"""
        import torch
        import torch.distributed as dist
        world = dist.get_world_size(group)

        def view(ptr, nbytes, dtype=torch.uint8):
            arr = np.ctypeslib.as_array(C.cast(ptr, C.POINTER(C.c_ubyte)), (nbytes,))
            return torch.from_numpy(arr).view(dtype)

        def all_gather(ctx, send, recv, nbytes, stream):
            out = view(recv, nbytes * world)
            dist.all_gather(list(out.view(world, nbytes).unbind(0)), view(send, nbytes).clone(), group=group)
            return 0

        def broadcast(ctx, buf, nbytes, root, stream):
            dist.broadcast(view(buf, nbytes), src=root, group=group)
            return 0

        def all_reduce(ctx, buf, count, stream):
            dist.all_reduce(view(buf, 8 * count, torch.float64), group=group)
            return 0

        fns = (_Collectives.AG(all_gather), _Collectives.BC(broadcast), _Collectives.AR(all_reduce))
        return _Collectives(None, *fns), fns

    def close(self):
        if self.sc is not None and getattr(self.sc, "h", None):
            self.L.trl_comm_destroy(self.sc.h)
        self.sc = None

    # ---- the exchange
    def SetEnvOffset(self, offset):
        self._ck(self.L.trl_comm_set_env_offset(self.sc.h, int(offset)))

    def GatherTuples(self, block_rows=1024):
        """pack + all-gather of this update's tuples (asynchronous; shipped tuples leave the scenario's tuple block)"""
        self._ck(self.L.trl_gather_tuples(self.sc.h, int(block_rows)))

    def Fetch(self, cap=None):
        """host copy of what the last GatherTuples delivered: (counts[world], rows f32 [n, W], flags u32 [n], env i32 [n])"""
        W = self.sc.tuple_width
        br = C.c_int(0)
        self._ck(self.L.trl_comm_info(self.sc.h, None, None, C.byref(br)))
        cap = int(cap or br.value * self.world)
        counts = np.zeros(self.world, np.int32)
        rows = np.zeros((cap, W), np.float32); flags = np.zeros(cap, np.uint32); env = np.zeros(cap, np.int32)
        n = C.c_int(0)
        self._ck(self.L.trl_gathered_fetch(self.sc.h, counts.ctypes.data_as(C.c_void_p), rows.ctypes.data_as(C.c_void_p),
                                           flags.ctypes.data_as(C.c_void_p), env.ctypes.data_as(C.c_void_p), cap, C.byref(n)))
        k = min(n.value, cap)
        return counts, rows[:k], flags[:k], env[:k]

    def LastGatherMs(self):
        ms = C.c_double(0)
        self._ck(self.L.trl_gather_last_ms(self.sc.h, C.byref(ms)))
        return ms.value

    def AddGathered(self, trainer):
        self._ck(self.L.trl_trainer_add_gathered(trainer.h))

    def BroadcastTrainer(self, trainer, root=0):
        self._ck(self.L.trl_trainer_broadcast(trainer.h, int(root)))

    def BroadcastWeights(self, root=0):
        self._ck(self.L.trl_comm_broadcast_weights(self.sc.h, int(root)))

    def ReplicaSpread(self, trainer):
        """sum over ranks of max |theta - theta(rank 0)|: 0.0 iff all replicas are bit-identical"""
        d = C.c_double(0)
        self._ck(self.L.trl_trainer_replica_spread(trainer.h, C.byref(d)))
        return d.value

    def EvalStats(self, slot=None):
        """cOptScenarioPoliEval::OutputResults' merge over all ranks (optimizer/scenarios/OptScenarioPoliEval.cpp:213-237);
        slot: only the envs of that policy slot (trl_comm_eval_stats_slot, a learning curve per policy over all ranks)"""
        c = C.c_int64(0); e = C.c_int64(0); a = C.c_double(0); s = C.c_int64(0)
        if slot is None:
            self._ck(self.L.trl_comm_eval_stats(self.sc.h, C.byref(c), C.byref(e), C.byref(a), C.byref(s)))
        else:
            self._ck(self.L.trl_comm_eval_stats_slot(self.sc.h, int(slot), C.byref(c), C.byref(e), C.byref(a), C.byref(s)))
        return dict(cycles=c.value, episodes=e.value, avg_dist=a.value, steps=s.value)

    def TuplesDropped(self):
        n = C.c_int64(0)
        self._ck(self.L.trl_tuples_dropped(self.sc.h, C.byref(n)))
        return n.value
