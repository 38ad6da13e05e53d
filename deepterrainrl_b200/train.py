"""cScenarioTrainMACE over one batched scenario per GPU (scenarios/ScenarioTrain.cpp, ScenarioTrainMACE.cpp): the loop that the
reference runs once per exploration thread

    exp.Update(dt); if exp.IsTupleBufferFull(): learner.Train(exp.GetTuples()); anneal exploration; exp.ResetTupleBuffer()

(ScenarioTrain.cpp:376-410) becomes: one outer update of the whole batch, a device-to-device hand-over of the tuples, K trainer
iterations on the GPU, and the annealed exploration settings for the next update.  The reference trains once per
`tuple_buffer_size` (32) tuples of one thread; a batch produces hundreds of tuples per update, so the number of trainer
iterations per update is a parameter here (`iters_per_update`; None = one iteration per tuple_buffer_size new tuples, read back
from the device once per update)."""
import ctypes as C
import json
import os

import numpy as np

from .scenario import ScenarioExpMACE, load_library
from .trainer import MACETrainer


class TrainSchedule:
    """CalcExpRate / CalcExpTemp / CalcExpBaseRate / CalcCurriculumPhase (scenarios/ScenarioTrain.cpp:418-460); defaults of
    cScenarioTrain's constructor (:8-35), values of args/opt_args_train_mace.txt via from_args()."""

    KEYS = ("init_exp_rate", "exp_rate", "init_exp_temp", "exp_temp", "init_exp_base_rate", "exp_base_rate",
            "trainer_num_anneal_iters", "exp_base_anneal_iters", "trainer_curriculum_iters")
    DEFAULTS = dict(init_exp_rate=1.0, exp_rate=0.1, init_exp_temp=1.0, exp_temp=0.1, init_exp_base_rate=1.0, exp_base_rate=0.1,
                    trainer_num_anneal_iters=1, exp_base_anneal_iters=1, trainer_curriculum_iters=0)

    def __init__(self, **kw):
        self.p = dict(self.DEFAULTS)
        self.p.update({k: v for k, v in kw.items() if k in self.DEFAULTS})
        self.L = load_library()
        self.L.trl_train_schedule.argtypes = [C.c_void_p, C.c_int, C.c_void_p]

    @classmethod
    def from_args(cls, args):
        """args: {key: string} parsed from a reference arg file (util/ArgParser.cpp semantics: `-key= value`)."""
        return cls(**{k: float(args[k]) for k in cls.DEFAULTS if k in args})

    def __call__(self, iters):
        sp = np.array([self.p[k] for k in self.KEYS], float)
        out = np.zeros(4)
        self.L.trl_train_schedule(sp.ctypes.data_as(C.c_void_p), int(iters), out.ctypes.data_as(C.c_void_p))
        return dict(exp_rate=out[0], exp_temp=out[1], exp_base_rate=out[2], curriculum_phase=out[3])


def parse_arg_file(path):
    """cArgParser::AppendArgs(file) (util/ArgParser.cpp:42-140): whitespace-separated tokens, `-key=` introduces a key."""
    args, key = {}, None
    with open(path) as f:
        for line in f:
            line = line.split("//")[0]
            for tok in line.split():
                if tok.startswith("-") and tok.endswith("="):
                    key = tok[1:-1]
                    args[key] = ""
                elif key is not None:
                    args[key] = (args[key] + " " + tok).strip()
    return args


class ScenarioTrainMACE:
    def __init__(self, pack, num_envs, device=0, terrain_seeds=None, rng_seed=1234, schedule=None, trainer_params=None,
                 iters_per_update=None, tuple_buffer_size=32, iters_per_output=200, output_path=None, max_iter=10 ** 9):
        self.schedule = schedule or TrainSchedule()
        self.exp = ScenarioExpMACE(pack, num_envs, device=device, terrain_seeds=terrain_seeds, rng_seed=rng_seed)
        self.trainer = MACETrainer(self.exp, **(trainer_params or {}))
        self.iters_per_update = iters_per_update
        self.tuple_buffer_size = tuple_buffer_size
        self.iters_per_output = iters_per_output
        self.output_path = output_path
        self.max_iter = max_iter
        self.time_step = 1.0 / 30.0                       # cScenarioTrain::mTimeStep
        self._iters = 0
        self._last_total = 0
        self._carry = 0
        # BuildScenePool: start from the initial exploration settings, curriculum phase gInitCurriculumPhase, then rebuild the ground
        self._apply_schedule(0)
        self.exp.Reset()

    def _apply_schedule(self, iters):
        s = self.schedule(iters)
        self.exp.EnableExplore(True, s["exp_rate"], s["exp_temp"], s["exp_base_rate"])
        self.exp.SetTerrainParamsLerp(s["curriculum_phase"])
        return s

    def Update(self, time_elapsed=None):
        """UpdateExpScene for the batch (scenarios/ScenarioTrain.cpp:376-410)."""
        self.exp.Update(self.time_step if time_elapsed is None else time_elapsed)
        self.trainer.AddTuplesFromScene()
        if self.iters_per_update is None:
            c = self.trainer.counters()                   # one small read-back per update
            new = c["total"] - self._last_total + self._carry
            self._last_total = c["total"]
            k, self._carry = divmod(new, self.tuple_buffer_size)
        else:
            k = self.iters_per_update
        if k > 0:
            self.trainer.Train(k)
        self._iters += k
        # exploration annealing follows the trainer's iteration count; between read-backs the host-side count of requested
        # iterations is its upper bound (equal once the trainer has left the init stage)
        return self._apply_schedule(self._iters if self.iters_per_update is not None else self.trainer.GetIter())

    def RunNative(self, num_updates):
        """The same loop entirely behind the C ABI (trl_train_run): no Python between the updates."""
        sp = np.array([self.schedule.p[k] for k in TrainSchedule.KEYS], float)
        L = self.trainer.L
        rc = L.trl_train_run(self.trainer.h, sp.ctypes.data_as(C.c_void_p), int(num_updates), int(self.iters_per_update or 0),
                             int(self.tuple_buffer_size), C.c_double(self.time_step))
        if rc != 0:
            raise RuntimeError(L.trl_last_error().decode())
        self._iters = self.trainer.GetIter()

    def Run(self, num_updates, log_every=0):
        for u in range(num_updates):
            s = self.Update()
            if log_every and (u + 1) % log_every == 0:
                c = self.trainer.counters()
                print(f"update {u + 1}: iter {c['iter']} tuples {c['num']} critic {c['critic']} actor {c['actor']} "
                      f"loss {c['critic_loss']:.5f} exp_rate {s['exp_rate']:.4f} exp_temp {s['exp_temp']:.4f}", flush=True)
            if self.output_path and self.iters_per_output and (u + 1) % self.iters_per_output == 0:
                self.OutputModel(self.output_path)
            if self.trainer.params and self._iters >= self.max_iter:
                break

    # the loop's own state, stored in a checkpoint's user blob
    _LOOP_STATE = ("iters_per_update", "tuple_buffer_size", "iters_per_output", "output_path", "max_iter", "time_step", "_iters",
                   "_last_total", "_carry")

    def Checkpoint(self, path):
        """the scenario, its trainer and this loop's state to `path`: resume(path) continues the run as if it had never stopped"""
        state = {k: getattr(self, k) for k in self._LOOP_STATE}
        state["schedule"] = self.schedule.p
        self.exp.SaveCheckpoint(path, json.dumps(state).encode())

    @classmethod
    def resume(cls, path, device=0):
        """the loop a Checkpoint() wrote, on `device`: Run(N + M) == Run(N); Checkpoint(path); resume(path).Run(M)"""
        from .checkpoint import load_checkpoint
        exp, trainers, user = load_checkpoint(path, device)
        if set(trainers) != {0}:
            raise RuntimeError(f"{path}: not a checkpoint of ScenarioTrainMACE (trainers on slots {sorted(trainers)})")
        state = json.loads(user.decode())
        obj = cls.__new__(cls)
        obj.schedule = TrainSchedule(**state.pop("schedule"))
        for k in cls._LOOP_STATE:
            setattr(obj, k, state[k])
        obj.exp, obj.trainer = exp, trainers[0]
        return obj

    def OutputModel(self, path):
        """cNeuralNet::OutputModel (learning/NeuralNet.cpp:571-587, 1182-1205): Caffe-layout HDF5 + `<stem>_scale.txt`."""
        import time
        os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
        self.exp.OutputModel(path, mtime=int(time.time()))            # native writer behind the C ABI (csrc/model_io.h)


def train_run_slots(trainers, schedule, num_updates, iters_per_update, time_step=1.0 / 30.0, tuple_buffer_size=32, comm=None,
                    block_rows=1024):
    """cScenarioTrain::Run for several trainers of one exploration scenario: `num_updates` updates of the whole batch, each followed
    by every trainer's hand-over of its slot's tuples and its iterations, the trainers side by side on their own streams.

    schedule: one TrainSchedule for all trainers, or a list with one per trainer (each applied to its own slot's envs).
    iters_per_update: the iterations of every trainer per update (lock-step; the schedules are read at the iterations done in this
    call); None = each trainer paced as in ScenarioTrainMACE: one iteration per `tuple_buffer_size` fresh tuples of its slot, its
    schedule read at its own iteration count.  One schedule with a fixed count is trl_train_run_slots (applied handle-wide); every
    other call is trl_train_run_slots_sched.

    comm: the scenario's parallel.Comm (multi-GPU, one process per GPU): trl_train_run_slots_comm, where every update's tuples of
    all ranks go through ONE all-gather of up to `block_rows` rows per rank (the rest stays queued) and trainer p takes slot p's
    rows of every rank.  Every rank must make the same call (same slots in the same order, schedules, counts; checked at the
    start).  If every trainer is asynchronous (MACETrainer.SetAsync), each one's intake and iterations overlap the next update.

    A learning curve per slot, from evaluation envs of the same scenario (they run their slot's current net, exploration off, and
    feed no trainer)::

        ex.SetEnvEval(np.arange(ex.num_envs) % 8 == 0)     # every 8th env evaluates from its next episode on
        ex.Reset()
        curve = []
        for _ in range(blocks):
            train_run_slots(trainers, schedules, 10, None)
            curve.append([ex.GetEvalStats(slot=t.slot, mode=0)["avg_dist"] for t in trainers])
            ex.ResetAvgDist()"""
    trainers = list(trainers)
    if not trainers:
        raise ValueError("train_run_slots: no trainer")
    L = trainers[0].L
    arr = (C.c_void_p * len(trainers))(*[t.h.value if t.h is not None else None for t in trainers])
    per_trainer = isinstance(schedule, (list, tuple))
    if comm is None and not per_trainer and iters_per_update is not None:
        sp = np.array([schedule.p[k] for k in TrainSchedule.KEYS], float)
        rc = L.trl_train_run_slots(arr, len(trainers), sp.ctypes.data_as(C.c_void_p), int(num_updates), int(iters_per_update),
                                   C.c_double(time_step))
    else:
        scheds = list(schedule) if per_trainer else [schedule] * len(trainers)
        if len(scheds) != len(trainers):
            raise ValueError("train_run_slots: %d schedules for %d trainers" % (len(scheds), len(trainers)))
        if iters_per_update is not None and int(iters_per_update) <= 0:
            raise ValueError("train_run_slots: iters_per_update must be positive, or None for tuple pacing")
        sp = np.array([[s.p[k] for k in TrainSchedule.KEYS] for s in scheds], float)
        ipu = 0 if iters_per_update is None else int(iters_per_update)
        if comm is None:
            rc = L.trl_train_run_slots_sched(arr, len(trainers), sp.ctypes.data_as(C.c_void_p), int(num_updates), ipu,
                                             int(tuple_buffer_size), C.c_double(time_step))
        else:
            rc = L.trl_train_run_slots_comm(arr, len(trainers), sp.ctypes.data_as(C.c_void_p), int(num_updates), ipu,
                                            int(tuple_buffer_size), int(block_rows), C.c_double(time_step))
    if rc != 0:
        raise RuntimeError(L.trl_last_error().decode())
