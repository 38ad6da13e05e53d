"""Per-slot exploration schedules on the SIMT emulator (tests/simt/): a miniature of tests/test_gpu_train_schedules.py run without a
GPU.  2 training slots, 16 envs, 3 tuple-paced updates (trl_train_run_slots_sched with iters_per_update = 0), the two schedules far
apart: slot 0 puts exploration noise on every decision at a high Boltzmann temperature, slot 1 hardly explores.  The slot build of the
FC stage reads each chunk's own settings; under a permuted lane schedule (the race check of tests/test_simt_cpu.py) every env and
both trainers must be bit-identical to single-trainer emulator runs on their own schedules."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "simt"))
from loader import simt_library  # noqa: E402
from test_gpu_train_schedules import ref_loop_paced  # noqa: E402
from test_gpu_train_slots import assert_envs, assert_trainer, close, make_group, make_ref, start_models  # noqa: E402

pytestmark = pytest.mark.skipif(__import__("platform").machine() != "x86_64",
                                reason="the emulator's fiber switch is written for x86-64")
N = 16
UPDATES = 3
TRAINER = dict(replay_mem_size=160, num_init_samples=160, freeze_target_iters=2)
LOUD = dict(init_exp_rate=1.0, exp_rate=1.0, init_exp_temp=5.0, exp_temp=5.0, init_exp_base_rate=0.0, exp_base_rate=0.0)
QUIET = dict(init_exp_rate=1e-3, exp_rate=1e-3, init_exp_temp=1e-3, exp_temp=1e-3, init_exp_base_rate=1e-3, exp_base_rate=1e-3)


def test_two_schedules_equal_single_trainer_runs(assets, tmp_path):
    import deepterrainrl_b200 as trl
    from deepterrainrl_b200.train import TrainSchedule, train_run_slots
    with simt_library() as L:
        pack = os.path.join(assets, "dog_slopes_mixed.trlpack")
        models = start_models(pack, str(tmp_path))[:2]
        slots = np.random.default_rng(6).integers(0, 2, N)
        scheds = [TrainSchedule(**LOUD), TrainSchedule(**QUIET)]
        refs = []
        for p in range(2):
            sc, tr = make_ref(trl, pack, N, models, p, slots, trainer_kw=TRAINER)
            ref_loop_paced(sc, tr, p, slots, scheds[p], UPDATES)
            refs.append((sc, tr))
        L.simt_set_sched_seed(C.c_ulonglong(2025))
        try:
            group, trs = make_group(trl, pack, N, models, slots, trainer_kw=TRAINER)
            train_run_slots(trs, scheds, UPDATES, None)
            group.Sync()
        finally:
            L.simt_set_sched_seed(C.c_ulonglong(0))
        for p in range(2):
            assert_trainer(trs[p], refs[p][1], "slot %d" % p)
        assert_envs(group, [r[0] for r in refs], slots, 90)
        close(*trs, group, *[o for r in refs for o in r])
