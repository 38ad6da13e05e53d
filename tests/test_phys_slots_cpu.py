"""Physics slots on the SIMT emulator (tests/simt/), without a GPU: a miniature of tests/test_gpu_phys_slots.py.

  * 6 dog envs on 3 physics slots (one with vertex contacts), 40 free-running env-steps under a permuted lane schedule (the race check
    of tests/test_simt_cpu.py), against one oracle batch per setting;
  * every refusal of trl_load_physics / trl_set_env_physics / trl_eval_stats_phys;
  * a checkpoint of that handle (with csrc/trl_checkpoint.cu linked in, as tests/test_checkpoint_cpu.py does) restores its physics
    slots and assignment, and a byte flipped in each physics section is refused with the section named."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "simt"))
from test_checkpoint_cpu import simt_library  # noqa: E402
from test_gpu_checkpoint import assert_refused, damaged_copies  # noqa: E402
from test_gpu_phys_slots import DEFAULT, setting  # noqa: E402

pytestmark = pytest.mark.skipif(__import__("platform").machine() != "x86_64",
                                reason="the emulator's fiber switch is written for x86-64")
N = 6
H = 1.0 / 600.0
SETTINGS = [setting(), setting(mu=0.3, kn=5e4, dn=5e2), setting(vertex=True, mu=0.5)]
SLOTS = np.array([2, 0, 1, 1, 2, 0], np.int32)


def _mixed(trl, pack, seeds):
    g = trl.ScenarioPoliEval(pack, N, terrain_seeds=seeds)
    for q, (p, vertex) in enumerate(SETTINGS[1:], 1):
        g.LoadPhysics(q, p, vertex)
    g.SetEnvPhysics(SLOTS)
    g.SetRandSeed(seeds)
    return g


def test_mixed_settings_against_the_oracle(assets, monkeypatch):
    import deepterrainrl_b200 as trl
    from pyoracle import Oracle
    pack = os.path.join(assets, "dog_slopes_mixed.trlpack")
    seeds = np.arange(11, 11 + N, dtype=np.uint64)
    orc = []
    for p, vertex in SETTINGS:
        if vertex:
            monkeypatch.setenv("ORC_VTX", "1")
        o = Oracle(pack, N, 0, terrain_seeds=seeds)
        monkeypatch.delenv("ORC_VTX", raising=False)
        o.set_phys(p)
        orc.append(o)
    with simt_library() as L:
        L.simt_set_sched_seed(C.c_ulonglong(2024))
        try:
            g = _mixed(trl, pack, seeds)
            assert np.array_equal(g.EnvPhysics()[0], SLOTS)
            for k in range(40):
                g.EnvStep(H)
                for e in range(N):
                    orc[SLOTS[e]].env_step(e, H)
        finally:
            L.simt_set_sched_seed(C.c_ulonglong(0))
        for e in range(N):
            gq, gqd, _, gc = g.GetState(e)
            oq, oqd, _, oc = orc[SLOTS[e]].get_state(e)
            assert np.max(np.abs(gq - oq) / (1 + np.abs(oq))) < 1e-6, e
            assert np.max(np.abs(gqd - oqd) / (1 + np.abs(oqd))) < 1e-6, e
            assert np.array_equal(gc, oc), e
        g.close()


def test_refusals_and_checkpoint_round_trip(assets, tmp_path):
    import deepterrainrl_b200 as trl
    pack = os.path.join(assets, "dog_slopes_mixed.trlpack")
    seeds = np.arange(1, N + 1, dtype=np.uint64)
    with simt_library() as L:
        g = _mixed(trl, pack, seeds)
        tol = list(DEFAULT)
        tol[4] = 0.0021
        neg = list(DEFAULT)
        neg[2] = -0.1
        for call, msg in [(lambda: g.LoadPhysics(0, DEFAULT), "out of range"), (lambda: g.LoadPhysics(3, tol), "contact_tol"),
                          (lambda: g.LoadPhysics(3, neg), "negative"), (lambda: g.SetEnvPhysics([3]), "empty"),
                          (lambda: g.SetEnvPhysics([1], env_ids=[N]), "env id"), (lambda: g.GetEvalStats(None, physics=4), "empty")]:
            with pytest.raises(RuntimeError, match=msg):
                call()
        assert np.array_equal(g.EnvPhysics()[1], SLOTS)
        for _ in range(3):
            g.EnvStep(H)
        path = str(tmp_path / "phys.ckpt")
        g.SaveCheckpoint(path)
        b, trs, _ = trl.load_checkpoint(path)
        assert trs == {}
        assert all(np.array_equal(x, y) for x, y in zip(g.EnvPhysics(), b.EnvPhysics()))
        for _ in range(5):
            g.EnvStep(H)
            b.EnvStep(H)
        for e in range(N):
            assert all(np.array_equal(x, y) for x, y in zip(g.GetState(e), b.GetState(e))), e
        d = tmp_path / "bad"
        d.mkdir()
        flipped = [(p, msg) for p, msg in damaged_copies(path, str(d)) if "phys" in msg]
        assert len(flipped) == 4
        for p, msg in flipped:
            assert_refused(L, p, msg)
        g.close(); b.close()
