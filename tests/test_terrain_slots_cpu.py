"""Terrain slots on the SIMT emulator (tests/simt/), without a GPU: a miniature of tests/test_gpu_terrain_slots.py.

  * 6 dog envs on 3 terrain slots, whole updates under a permuted lane schedule (the race check of tests/test_simt_cpu.py), through a
    forced fall and a trl_reset, bit-identical env for env to three single-terrain emulator handles;
  * the loader: every committed terrain file loaded into a slot generates the strips a handle created with it as -terrain_file does,
    and both match the CPU oracle's strips and reset state for that file."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "simt"))
from loader import simt_library  # noqa: E402
from test_gpu_terrain_slots import REF, assert_same_env, data_root, make_handle, scene_args  # noqa: E402

pytestmark = pytest.mark.skipif(__import__("platform").machine() != "x86_64",
                                reason="the emulator's fiber switch is written for x86-64")
N = 6
TERRAINS = ["tight_gaps", "slopes_mixed", "cliffs_rugged"]


def _fall(sc, e):
    """tip env e over (root angle past 0.8 pi): it falls at the end of the next update and resets"""
    q, qd, tau, c = sc.GetState(e)
    q[2] = 3.0
    sc.SetState(e, q=q)


def _run(handles, updates):
    for _ in range(updates):
        for sc in handles:
            sc.Update(1.0 / 30.0)
    for sc in handles:
        sc.Sync()


def test_mixed_batch_is_the_union_of_single_terrain_runs(assets, tmp_path):
    import deepterrainrl_b200 as trl
    with simt_library() as L:
        root, models = data_root(trl, assets, str(tmp_path))
        slots = np.array([2, 0, 1, 1, 2, 0])
        refs = [make_handle(trl, "dog", root, models["dog"], [t], N, None) for t in TERRAINS]
        L.simt_set_sched_seed(C.c_ulonglong(2024))
        try:
            mixed = make_handle(trl, "dog", root, models["dog"], TERRAINS, N, slots)
            handles = refs + [mixed]
            _run(handles, 4)
            for sc in handles:
                _fall(sc, 0); _fall(sc, 3)
            _run(handles, 2)
            for sc in handles:
                sc.Reset([4])
            _run(handles, 2)
        finally:
            L.simt_set_sched_seed(C.c_ulonglong(0))
        assert all(r.GetNumEpisodes() >= 1 for r in refs[1:])       # the forced falls were logged
        cur, nxt = mixed.EnvTerrain()
        assert np.array_equal(cur, slots) and np.array_equal(nxt, slots)
        for e in range(N):
            assert_same_env(mixed, e, refs[slots[e]], e, 90, "terrain %d" % slots[e])
        dist, denv = mixed.GetDistLog()
        for e in range(N):
            rd, re = refs[slots[e]].GetDistLog()
            assert np.array_equal(dist[denv == e], rd[re == e]), e
        for t in range(3):
            st = mixed.GetEvalStats(None, terrain=t)
            rd, re = refs[t].GetDistLog()
            assert st["episodes"] == int(np.isin(re, np.flatnonzero(slots == t)).sum())
        for sc in handles:
            sc.close()


def test_loaded_terrain_generates_what_terrain_file_does(assets, tmp_path):
    import deepterrainrl_b200 as trl
    from pyoracle import Oracle
    names = sorted(os.path.splitext(f)[0] for f in os.listdir(os.path.join(REF, "data", "terrain")))
    assert len(names) == 7
    n = 3
    with simt_library():
        root, models = data_root(trl, assets, str(tmp_path))
        for name in names:
            slotted = make_handle(trl, "dog", root, models["dog"], ["flat", name], n, np.ones(n, np.int32))
            direct = make_handle(trl, "dog", root, models["dog"], [name], n, None)
            pack = str(tmp_path / (name + ".trlpack"))
            trl.pack_from_args(scene_args("dog", name, models["dog"]), root, pack)
            o = Oracle(pack, n, 0, terrain_seeds=np.arange(1, n + 1, dtype=np.uint64))
            for e in range(n):
                for seg in (0, 1):
                    a, b, od = slotted.GetTerrain(e, seg), direct.GetTerrain(e, seg), o.terrain(e, seg)
                    assert np.array_equal(a[0], b[0]) and a[1:] == b[1:], (name, e, seg)
                    assert np.array_equal(a[0], od[0]) and a[1:] == od[1:], (name, e, seg, "oracle")
                np.testing.assert_array_equal(slotted.GetState(e)[0], o.get_state(e)[0])
            assert np.array_equal(slotted.EnvTerrain()[0], np.ones(n, np.int32))
            slotted.close(); direct.close()
