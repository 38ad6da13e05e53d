"""Body slots on the SIMT emulator (tests/simt/), without a GPU: a miniature of tests/test_gpu_body_slots.py.

  * 6 dog envs on 3 body slots, whole updates under a permuted lane schedule (the race check of tests/test_simt_cpu.py), through a
    forced fall and a trl_reset, bit-identical env for env to three single-body emulator handles, and free-running env-steps against one
    oracle batch per character file (its pack made by trl_pack_from_args with that -character_file);
  * the loader: the table trl_load_body stores for a file is the body a handle created with that -character_file derives, for the three
    committed characters and their generated variants;
  * the refusals, and a checkpoint round trip with the body sections named when damaged (csrc/trl_checkpoint.cu linked in, as
    tests/test_checkpoint_cpu.py does)."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "simt"))
from test_checkpoint_cpu import simt_library  # noqa: E402
from test_gpu_body_slots import VARIANTS, body_files, make_body_handle, write_variants  # noqa: E402
from test_gpu_checkpoint import assert_refused, damaged_copies  # noqa: E402
from test_gpu_terrain_slots import assert_same_env, data_root, scene_args  # noqa: E402

pytestmark = pytest.mark.skipif(__import__("platform").machine() != "x86_64",
                                reason="the emulator's fiber switch is written for x86-64")
N = 6
SLOTS = np.array([2, 0, 1, 1, 2, 0])


def _fall(sc, e):
    q = sc.GetState(e)[0]
    q[2] = 3.0
    sc.SetState(e, q=q)


def _run(handles, updates):
    for _ in range(updates):
        for sc in handles:
            sc.Update(1.0 / 30.0)
    for sc in handles:
        sc.Sync()


def test_mixed_batch_is_the_union_of_single_body_runs(assets, tmp_path):
    import deepterrainrl_b200 as trl
    with simt_library() as L:
        root, models = data_root(trl, assets, str(tmp_path))
        var = write_variants(root, str(tmp_path))
        files = body_files(root, var, "dog")[:3]
        refs = [make_body_handle(trl, "dog", root, models["dog"], [f], N, None) for f in files]
        L.simt_set_sched_seed(C.c_ulonglong(2024))
        try:
            mixed = make_body_handle(trl, "dog", root, models["dog"], files, N, SLOTS)
            handles = refs + [mixed]
            _run(handles, 3)
            for sc in handles:
                _fall(sc, 0); _fall(sc, 3)
            _run(handles, 1)
            for sc in handles:
                sc.Reset([4])
            _run(handles, 1)
        finally:
            L.simt_set_sched_seed(C.c_ulonglong(0))
        assert all(r.GetNumEpisodes() >= 1 for r in refs[1:])
        assert all(np.array_equal(x, SLOTS) for x in mixed.EnvBody())
        for e in range(N):
            assert_same_env(mixed, e, refs[SLOTS[e]], e, 90, "body %d" % SLOTS[e])
        for sc in handles:
            sc.close()


def test_free_running_against_the_oracle(assets, tmp_path):
    import deepterrainrl_b200 as trl
    from pyoracle import Oracle
    h = 1.0 / 600.0
    seeds = np.arange(11, 11 + N, dtype=np.uint64)
    with simt_library() as L:
        root, models = data_root(trl, assets, str(tmp_path))
        var = write_variants(root, str(tmp_path))
        files = body_files(root, var, "dog")[:3]
        orc = []
        for b, f in enumerate(files):
            pack = str(tmp_path / ("body%d.trlpack" % b))
            trl.pack_from_args(scene_args("dog", "slopes_mixed", models["dog"], ["-character_file=", f]), root, pack)
            orc.append(Oracle(pack, N, 0, terrain_seeds=seeds))
        g = make_body_handle(trl, "dog", root, models["dog"], files, N, SLOTS, seeds=seeds)
        L.simt_set_sched_seed(C.c_ulonglong(7))
        try:
            for _ in range(60):
                g.EnvStep(h)
                for e in range(N):
                    orc[SLOTS[e]].env_step(e, h)
        finally:
            L.simt_set_sched_seed(C.c_ulonglong(0))
        for e in range(N):
            gq, gqd, _, gc = g.GetState(e)
            oq, oqd, _, oc = orc[SLOTS[e]].get_state(e)
            assert np.max(np.abs(gq - oq) / (1 + np.abs(oq))) < 1e-6, e
            assert np.max(np.abs(gqd - oqd) / (1 + np.abs(oqd))) < 1e-6, e
            assert np.array_equal(gc, oc), e
        g.close()


def _body_table(path):
    """the body table ([8] raw BodyConst records) a checkpoint stores"""
    from deepterrainrl_b200.checkpoint import sections
    data = open(path, "rb").read()
    for name, _, _, off, nbytes, _ in sections(path):
        if name == "body_table":
            rec = data[off:off + nbytes]
            size = nbytes // 8
            return [rec[k * size:(k + 1) * size] for k in range(8)]
    raise AssertionError("no body_table section")


def test_loader_stores_what_a_handle_of_that_file_derives(assets, tmp_path):
    import deepterrainrl_b200 as trl
    with simt_library():
        root, models = data_root(trl, assets, str(tmp_path))
        var = write_variants(root, str(tmp_path))
        for ch in ("dog", "goat", "raptor"):
            own = os.path.join(root, "data", "characters", ch + ".txt")
            kinds = ["copy"] + [k for k in VARIANTS if k != "copy"]
            mixed = make_body_handle(trl, ch, root, models[ch], [own] + [var[ch, k] for k in kinds], 1, None)
            path = str(tmp_path / ("%s_mixed.ckpt" % ch))
            mixed.SaveCheckpoint(path)
            table = _body_table(path)
            assert table[1] == table[0], ch                  # an unmodified copy is the scene's body
            for b, k in enumerate(kinds, 1):
                single = make_body_handle(trl, ch, root, models[ch], [var[ch, k], var[ch, "copy"]], 1, None)
                p = str(tmp_path / ("%s_%s.ckpt" % (ch, k)))
                single.SaveCheckpoint(p)
                assert _body_table(p)[0] == table[b], (ch, k)
                assert k == "copy" or table[b] != table[0], (ch, k)
                single.close()
            mixed.close()


def test_refusals_and_checkpoint_round_trip(assets, tmp_path):
    import deepterrainrl_b200 as trl
    with simt_library() as L:
        root, models = data_root(trl, assets, str(tmp_path))
        var = write_variants(root, str(tmp_path))
        files = body_files(root, var, "dog")[:3]
        g = make_body_handle(trl, "dog", root, models["dog"], files, N, SLOTS)
        for call, msg in [(lambda: g.LoadBody(0, files[1]), "out of range"), (lambda: g.LoadBody(3, var["raptor", "copy"]), "topology"),
                          (lambda: g.LoadBody(3, var["goat", "copy"]), "Controllers"), (lambda: g.LoadBody(1, files[2]), "in use"),
                          (lambda: g.SetEnvBody([3]), "empty"), (lambda: g.SetEnvBody([1], env_ids=[N]), "env id"),
                          (lambda: g.GetEvalStats(None, body=4), "empty")]:
            with pytest.raises(RuntimeError, match=msg):
                call()
        assert np.array_equal(g.EnvBody()[1], SLOTS)
        _run([g], 1)
        path = str(tmp_path / "body.ckpt")
        g.SaveCheckpoint(path)
        b, trs, _ = trl.load_checkpoint(path)
        assert trs == {}
        assert all(np.array_equal(x, y) for x, y in zip(g.EnvBody(), b.EnvBody()))
        _run([g, b], 1)
        for e in range(N):
            assert_same_env(g, e, b, e, 90, "resumed")
        d = tmp_path / "bad"
        d.mkdir()
        flipped = [(p, msg) for p, msg in damaged_copies(path, str(d)) if "body" in msg]
        assert len(flipped) == 4
        for p, msg in flipped:
            assert_refused(L, p, msg)
        g.close(); b.close()
