"""Evaluation envs on the SIMT emulator (tests/simt/), without a GPU: a miniature of tests/test_gpu_eval_envs.py.

  * 12 dog envs, one trainer (trl_train_run), every 4th env evaluating, 3 updates under a permuted lane schedule (the race check of
    tests/test_simt_cpu.py): the exploring envs and the trainer equal a pure exploration handle whose trainer is fed only the exploring
    envs' tuples, the evaluating envs equal an evaluation handle given the trainer's net before every update;
  * the refusals of trl_set_env_eval / trl_eval_stats_mode;
  * a checkpoint with evaluation envs (csrc/trl_checkpoint.cu linked in, as tests/test_checkpoint_cpu.py does) restores the modes, and
    a byte flipped in each new section is refused with the section named."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "simt"))
from test_checkpoint_cpu import simt_library  # noqa: E402
from test_gpu_checkpoint import assert_refused, damaged_copies  # noqa: E402
from test_gpu_eval_envs import Run, eval_mask  # noqa: E402

pytestmark = pytest.mark.skipif(__import__("platform").machine() != "x86_64",
                                reason="the emulator's fiber switch is written for x86-64")
N = 12
TRAINER = dict(replay_mem_size=160, num_init_samples=40, freeze_target_iters=2)


def test_mixed_handle_equals_references(assets):
    import deepterrainrl_b200 as trl
    pack = os.path.join(assets, "dog_slopes_mixed.trlpack")
    with simt_library() as L:
        L.simt_set_sched_seed(C.c_ulonglong(2026))
        try:
            run = Run(trl, pack, N, [None], np.zeros(N, np.int32), eval_mask("every4", N), single_trainer_run=True, trainer_kw=TRAINER)
            for _ in range(3):
                run.step()
        finally:
            L.simt_set_sched_seed(C.c_ulonglong(0))
        run.check(90, falls=False)      # 3 updates: too short for a fall (tests/test_gpu_eval_envs.py tips envs over)
        run.close()


def test_refusals_and_checkpoint_round_trip(assets, tmp_path):
    import deepterrainrl_b200 as trl
    pack = os.path.join(assets, "dog_slopes_mixed.trlpack")
    with simt_library() as L:
        ev = trl.ScenarioPoliEval(pack, N)
        with pytest.raises(RuntimeError, match="evaluation handle"):
            ev.SetEnvEval([1])
        g = trl.ScenarioExpMACE(pack, N)
        for call, msg in [(lambda: g.SetEnvEval([1], env_ids=[N]), "env id"), (lambda: g.SetEnvEval(np.ones(N + 1, np.int32)), "env count"),
                          (lambda: g.GetEvalStats(None, mode=3), "mode")]:
            with pytest.raises(RuntimeError, match=msg):
                call()
        flags = eval_mask("block", N)
        g.SetEnvEval(flags.astype(np.int32))
        g.Reset()
        g.Update(1.0 / 30.0)
        path = str(tmp_path / "eval.ckpt")
        g.SaveCheckpoint(path)
        b, trs, _ = trl.load_checkpoint(path)
        assert trs == {}
        assert all(np.array_equal(x, y) for x, y in zip(g.EnvEval(), b.EnvEval()))
        assert np.array_equal(b.EnvEval()[0], flags)
        for sc in (g, b):
            sc.Update(1.0 / 30.0)
        for e in range(N):
            assert all(np.array_equal(x, y) for x, y in zip(g.GetState(e), b.GetState(e))), e
        d = tmp_path / "bad"
        d.mkdir()
        flipped = [(p, msg) for p, msg in damaged_copies(path, str(d)) if "eval" in msg]
        assert len(flipped) == 3
        for p, msg in flipped:
            assert_refused(L, p, msg)
        g.close(); b.close(); ev.close()
