"""Policy slots on the SIMT emulator (tests/simt/): the slot build of the decision kernels (regrouping by slot, per-slot weights and
terr_ip0 tiles, ip0 restaging, slot-ragged chunks) run without a GPU.  A miniature of tests/test_gpu_policy_slots.py: 3 slots,
40 envs, whole updates under a permuted lane schedule (the race check of tests/test_simt_cpu.py), bit-identical to single-slot
emulator runs, and the decision pass at slot-ragged batch shapes against torch f64 and single-policy passes."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "simt"))
from loader import simt_library  # noqa: E402
from test_gpu_policy_slots import (_decide_sweep, assert_union, env_ids, exported_model, pack_net, perturbed, run_handle,  # noqa: E402
                                   write_net)

pytestmark = pytest.mark.skipif(__import__("platform").machine() != "x86_64",
                                reason="the emulator's fiber switch is written for x86-64")
N = 40
UPDATES = 10        # 200 env-steps


def _models(trl, assets, tmp_path):
    pack = os.path.join(assets, "dog_slopes_mixed.trlpack")
    goat = exported_model(trl, os.path.join(assets, "goat_cliffs.trlpack"), str(tmp_path / "goat.h5"))
    pert = write_net(str(tmp_path / "dog_perturbed.h5"), perturbed(pack_net(pack), 5))
    return pack, [None] + [(m, os.path.splitext(m)[0] + "_scale.txt") for m in (goat, pert)]


def test_mixed_batch_is_the_union_of_single_slot_runs(assets, tmp_path):
    import deepterrainrl_b200 as trl
    with simt_library() as L:
        pack, models = _models(trl, assets, tmp_path)
        slots = np.random.default_rng(4).integers(0, 3, N)
        slots[:3] = [0, 1, 2]
        refs = [run_handle(trl, pack, N, [m], None, UPDATES) for m in models]
        L.simt_set_sched_seed(C.c_ulonglong(2024))
        try:
            mixed = run_handle(trl, pack, N, models, slots, UPDATES)
        finally:
            L.simt_set_sched_seed(C.c_ulonglong(0))
        assert mixed.KernelLaunches() > refs[0].KernelLaunches()     # the slot build ran (one regrouping launch per env-step more)
        assert_union(mixed, refs, slots, 90)
        for sc in refs + [mixed]:
            sc.close()


def test_decision_pass_with_mixed_slots(assets, tmp_path):
    """70 envs (2 FC clusters, act2 zero fill past row 70): slot-ragged chunks, an empty slot, all rows in the last slot, more chunks
    than clusters"""
    import deepterrainrl_b200 as trl
    with simt_library():
        pack = os.path.join(assets, "dog_slopes_mixed.trlpack")
        base = pack_net(pack)
        nets = [base, perturbed(base, 1), perturbed(base, 2)]
        paths = [None] + [(write_net(str(tmp_path / ("p%d.h5" % p)), nets[p]), str(tmp_path / ("p%d_scale.txt" % p))) for p in (1, 2)]
        n = 70
        rng = np.random.default_rng(0)
        cases = [(env_ids("permuted", 67, n, 1), rng.integers(0, 3, 67))]
        ids = env_ids("identity", 45, n)
        cases.append((ids, np.where(np.arange(45) < 33, 1, 2)))                  # 33 rows in slot 1 (ragged second chunk), none in slot 0
        ids = env_ids("last", 20, n)
        cases.append((ids, np.full(20, 2)))                                        # every row in the last slot
        worst = _decide_sweep(trl, pack, n, nets, paths, 90, cases)
        assert worst <= 1e-10
