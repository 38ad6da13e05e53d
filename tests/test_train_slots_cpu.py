"""Training slots on the SIMT emulator (tests/simt/): a miniature of tests/test_gpu_train_slots.py run without a GPU.  2 slots (the
pack's model and a perturbed model file), 16 envs, 3 updates with exploration on: the slot build's per-slot noise scale on every
env's first decisions, and the fork / join of trl_train_run_slots (each trainer's slot-filtered hand-over and iteration on its own
stream) under a permuted lane schedule (the race check of tests/test_simt_cpu.py), bit-identical to single-trainer emulator runs.
The first tuples of a synchronised start arrive later than an emulator run can afford to wait; the hand-over of real tuples and
the training it drives are compared on the GPU."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "simt"))
from loader import simt_library  # noqa: E402
from test_gpu_train_slots import SCHEDULE, assert_envs, assert_trainer, close, make_group, make_ref, ref_loop, start_models  # noqa: E402

pytestmark = pytest.mark.skipif(__import__("platform").machine() != "x86_64",
                                reason="the emulator's fiber switch is written for x86-64")
N = 16
UPDATES = 3
TRAINER = dict(replay_mem_size=160, num_init_samples=160, freeze_target_iters=2)


def test_training_slots_equal_single_trainer_runs(assets, tmp_path):
    import deepterrainrl_b200 as trl
    from deepterrainrl_b200.train import TrainSchedule, train_run_slots
    with simt_library() as L:
        pack = os.path.join(assets, "dog_slopes_mixed.trlpack")
        models = start_models(pack, str(tmp_path))[:2]
        slots = np.random.default_rng(4).integers(0, 2, N)
        sched = TrainSchedule(**SCHEDULE)
        refs = []
        for p in range(2):
            sc, tr = make_ref(trl, pack, N, models, p, slots, trainer_kw=TRAINER)
            ref_loop(sc, tr, p, slots, sched, UPDATES, 1)
            refs.append((sc, tr))
        L.simt_set_sched_seed(C.c_ulonglong(2024))
        try:
            group, trs = make_group(trl, pack, N, models, slots, trainer_kw=TRAINER)
            train_run_slots(trs, sched, UPDATES, 1)
            group.Sync()
        finally:
            L.simt_set_sched_seed(C.c_ulonglong(0))
        for p in range(2):
            assert_trainer(trs[p], refs[p][1], "slot %d" % p)
        assert_envs(group, [r[0] for r in refs], slots, 90)
        close(*trs, group, *[o for r in refs for o in r])
