"""Ranged slots on the SIMT emulator (tests/simt/), without a GPU: a miniature of tests/test_gpu_body_ranges.py under the permuted lane
schedule (the race check of tests/test_simt_cpu.py).

  * the read-backs against the numpy restatement of the recipe, over episodes begun by trl_seed_terrain, a fall and trl_reset;
  * lo == hi against the fixed slot, and one episode of a ranged body and physics against fixed slots holding its drawn numbers;
  * a checkpoint round trip with the new sections named when damaged, and the refusals;
  * a handle with body and physics slots but no ranged slot writes the checkpoint the format before ranged slots wrote."""
import ctypes as C
import hashlib
import json
import os
import struct
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "simt"))
from test_checkpoint_cpu import simt_library  # noqa: E402
from test_gpu_body_ranges import (PHYS_HI, PHYS_LO, body_draw, ends_files, make, phys_draw, reseed, with_numbers,  # noqa: E402
                                  write_char)
from test_gpu_checkpoint import assert_refused, damaged_copies  # noqa: E402
from test_gpu_terrain_slots import assert_same_env, data_root, tip_over  # noqa: E402

pytestmark = pytest.mark.skipif(__import__("platform").machine() != "x86_64",
                                reason="the emulator's fiber switch is written for x86-64")
N = 4
SEED = 77
# the checkpoint of fixed_slot_checkpoint() as the format before ranged slots writes it (the emulator build of that format), digested by
# layout_digest()
PRE_RANGES_DIGEST = "696cc81daf90779feb09ceb805ddfa51aed52ba58ad57c6d43a8256d48ad7c74"


def _run(handles, updates):
    for _ in range(updates):
        for sc in handles:
            sc.Update(1.0 / 30.0)
    for sc in handles:
        sc.Sync()


def test_draws_and_episodes_on_the_emulator(assets, tmp_path):
    import deepterrainrl_b200 as trl
    with simt_library() as L:
        root, models = data_root(trl, assets, str(tmp_path))
        d = str(tmp_path)
        base, lo_f, hi_f, lo, hi = ends_files(root, d, "dog", "emu")
        _, pt_f, _, pt, _ = ends_files(root, d, "dog", "emu_point", scale=0.9)
        L.simt_set_sched_seed(C.c_ulonglong(2024))
        try:
            sc = make(trl, "dog", root, models["dog"], N, rng_seed=SEED)
            sc.LoadBodyRange(1, lo_f, hi_f)
            sc.LoadBodyRange(2, pt_f, pt_f)
            sc.LoadPhysicsRange(1, PHYS_LO, PHYS_HI)
            body = np.array([1, 1, 2, 0])
            sc.SetEnvBody(body)
            sc.SetEnvPhysics(np.array([1, 0, 1, 0]))
            # the reference: env 0 and 1 on fixed slots holding their first draws, env 2 on the fixed point body
            ref = make(trl, "dog", root, models["dog"], N, rng_seed=SEED)
            for e in (0, 1):
                ref.LoadBody(1 + e, write_char(with_numbers(base, body_draw(SEED, e, 0, lo, hi)), os.path.join(d, "emu_e%d.txt" % e)))
            ref.LoadBody(3, pt_f)
            ref.LoadPhysics(1, phys_draw(SEED, 0, 0, PHYS_LO, PHYS_HI))
            ref.LoadPhysics(2, phys_draw(SEED, 2, 0, PHYS_LO, PHYS_HI))
            ref.SetEnvBody(np.array([1, 2, 3, 0]))
            ref.SetEnvPhysics(np.array([1, 0, 2, 0]))
            for h in (sc, ref):
                reseed(h, N)
            _run([sc, ref], 2)
        finally:
            L.simt_set_sched_seed(C.c_ulonglong(0))
        for e in range(N):
            assert_same_env(sc, e, ref, e, 90, "first ranged episode")
        out, draws = sc.EnvBodyDraws()
        pout, pdraws = sc.EnvPhysicsDraws()
        assert np.array_equal(draws, [1, 1, 1, 0]) and np.array_equal(pdraws, [1, 0, 1, 0])
        assert np.array_equal(out[1], body_draw(SEED, 1, 0, lo, hi)) and np.array_equal(out[2], pt)
        tip_over(sc, [0])
        _run([sc], 1)
        sc.Reset([1])
        out, draws = sc.EnvBodyDraws()
        pout, pdraws = sc.EnvPhysicsDraws()
        assert np.array_equal(draws, [2, 2, 1, 0]) and np.array_equal(pdraws, [2, 0, 1, 0])
        for e in (0, 1):
            assert np.array_equal(out[e], body_draw(SEED, e, 1, lo, hi))
        assert np.array_equal(pout[0], phys_draw(SEED, 0, 1, PHYS_LO, PHYS_HI))
        # refusals leave the handle as it is
        for call, msg in [(lambda: sc.LoadBodyRange(3, hi_f, lo_f), "lo"), (lambda: sc.LoadBodyRange(1, lo_f, hi_f), "in use"),
                          (lambda: sc.LoadPhysicsRange(2, PHYS_HI, PHYS_LO), "kn: lo"), (lambda: sc.LoadPhysicsRange(1, PHYS_LO, PHYS_HI), "in use")]:
            with pytest.raises(RuntimeError, match=msg):
                call()
        assert np.array_equal(sc.EnvBodyDraws()[1], draws)
        # a checkpoint resumes the draws; every new section is named when damaged
        path = str(tmp_path / "ranged.ckpt")
        sc.SaveCheckpoint(path)
        b, _, _ = trl.load_checkpoint(path)
        for h in (sc, b):
            tip_over(h, [2])
        _run([sc, b], 1)
        for x, y in zip(sc.EnvBodyDraws() + sc.EnvPhysicsDraws(), b.EnvBodyDraws() + b.EnvPhysicsDraws()):
            assert np.array_equal(x, y)
        for e in range(N):
            assert_same_env(sc, e, b, e, 90, "resumed")
        dd = tmp_path / "bad"
        dd.mkdir()
        new = ("env_bdraw", "env_pdraw", "env_draws", "ranges", "range_body_hi", "range_phys_hi")
        flipped = [(p, msg) for p, msg in damaged_copies(path, str(dd)) if any("'%s'" % s in msg for s in new)]
        assert len(flipped) == len(new)
        for p, msg in flipped:
            assert_refused(L, p, msg)
        for h in (sc, ref, b):
            h.close()


def fixed_slot_checkpoint(trl, tree, d, path):
    """a handle with a body slot and a physics slot but no ranged slot, after one update, saved to path"""
    ref = os.path.join(tree, "tests", "golden", "reference")
    with open(os.path.join(ref, "data", "characters", "dog.txt")) as f:
        c = json.load(f)
    c["Controllers"]["Files"] = [os.path.join(ref, x) for x in c["Controllers"]["Files"]]
    c["BodyDefs"][5]["Mass"] *= 1.25
    c["PDControllers"][13]["Kp"] *= 0.8
    body = os.path.join(d, "dog_heavy.txt")
    with open(body, "w") as f:
        json.dump(c, f)
    sc = trl.ScenarioPoliEval(os.path.join(tree, "assets", "dog_slopes_mixed.trlpack"), 2, rng_seed=9)
    sc.LoadBody(1, body)
    sc.LoadPhysics(1, [1.6e5, 2.0e3, 0.6, 0.01, 0.00025, 2.0e4, 20.0])
    sc.SetEnvBody([1, 0])
    sc.SetEnvPhysics([0, 1])
    sc.SetRandSeed(np.array([1, 2], np.uint64))
    sc.Update(1.0 / 30.0)
    sc.Sync()
    sc.SaveCheckpoint(path, b"golden")
    sc.close()


def layout_digest(path):
    """SHA-256 over every section's name, dtype, kind, size and bytes.  The 4 padding bytes behind each PhysParams of phys_table are
    zeroed: the writer copies them from whatever the struct held, so no two runs of either format need agree on them (the section
    digests in the table cover them and are left out for that reason)"""
    from deepterrainrl_b200.checkpoint import sections
    data = open(path, "rb").read()
    h = hashlib.sha256()
    for name, dtype, kind, off, nb, _ in sections(path):
        b = bytearray(data[off:off + nb])
        if name == "phys_table":
            for s in range(0, nb, 64):
                b[s + 60:s + 64] = bytes(4)
        h.update(struct.pack("<48sIIQ", name.encode(), dtype, kind, nb))
        h.update(bytes(b))
    return h.hexdigest()


def test_a_handle_without_ranged_slots_writes_the_earlier_format(tmp_path):
    import deepterrainrl_b200 as trl
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    with simt_library():
        path = str(tmp_path / "fixed.ckpt")
        fixed_slot_checkpoint(trl, root, str(tmp_path), path)
    assert layout_digest(path) == PRE_RANGES_DIGEST
