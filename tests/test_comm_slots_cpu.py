"""Training slots over the tuple exchange on the SIMT emulator (tests/simt/): a miniature of the world-2 check of
tests/test_gpu_comm_slots.py without a GPU.  Two gloo ranks with host-memory collectives, 2 slots (the pack's model and a fresh net),
8 envs per rank with a different slot assignment on each, 48 updates, each followed by one gather into blocks small enough to queue
rows and every slot trainer's slot-filtered intake (trl_trainer_add_gathered; an emulated trainer iteration costs seconds, so none is
run): the replicas of every slot stay bit-identical and equal to the host-filtered reference trainers, under two permuted lane
schedules (the race check of tests/test_simt_cpu.py on the slot-filtered intake kernels); calls of trl_train_run_slots_comm
that differ between the ranks, or that one rank refuses by itself, are refused on both ranks, and the run that follows them equals
the run without them."""
import os
import platform

import pytest
import torch.multiprocessing as mp

from test_gpu_comm_slots import check_world2, world2_worker

pytestmark = pytest.mark.skipif(platform.machine() != "x86_64", reason="the emulator's fiber switch is written for x86-64")


def test_gloo_world2_slot_trainers_on_the_emulator(assets, tmp_path):
    pack = os.path.join(assets, "dog_slopes_mixed.trlpack")
    port = 29500 + ((os.getpid() + 733) % 1000)
    mp.spawn(world2_worker, args=(2, port, pack, str(tmp_path), True, 8, 48, "intake", [2024, 7]), nprocs=2, join=True)
    check_world2(str(tmp_path), 2)
