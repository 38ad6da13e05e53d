"""Terrain slots (trl_load_terrain / trl_set_env_terrain / trl_env_terrain / trl_eval_stats_cell): one handle generates the ground of
each env from one of up to 8 terrains.  The contract is exact: env i of a handle with terrain slots computes, bit for bit, what env i of
a handle created with `-terrain_file=<its slot's file>` computes from the same seeds, because the generator, the env-step and the
decision are per env.

  1. whole updates of dog, raptor and goat scenes (overlapped schedule, serial schedule, env groups; evaluation and exploration)
     against one single-terrain handle per file;
  2. a policy x terrain matrix against the nine single handles, and the cell statistics against sums over them;
  3. 600 free-running env-steps of a 4-terrain dog handle against the CPU oracle, one oracle batch per terrain file;
  4. the "next reset" rule across a fall, trl_reset and a reseed, and the blend of a two-set terrain file;
  5. a training run on a terrain-slot exploration handle, twice;
  6. every refusal.
tests/test_terrain_slots_cpu.py runs a miniature of (1) on the emulator and the loader check without a GPU."""
import ctypes as C
import json
import os
import shutil

import numpy as np
import pytest

import torch_net  # noqa: F401  (torch before the library: see tests/test_gpu_decide_batches.py)
from test_gpu_policy_slots import assignment, exported_model, pack_net, perturbed, raptor_mixed_model, write_net

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "tests", "golden", "reference")
UPDATES = 30
H = 1.0 / 600.0

DOG_TERRAINS = ["slopes_mixed", "mixed", "narrow_gaps", "tight_gaps", "flat", "cliffs_rugged"]
SCENES = {
    # arg file, terrains (the first is slot 0), the pack whose policy the args' model path gets
    "dog": ("args/dog_mixed_args.txt", DOG_TERRAINS, "dog_slopes_mixed.trlpack"),
    "raptor": ("args/raptor_mixed_args.txt", ["mixed_raptor", "narrow_gaps", "slopes_mixed", "flat"], None),
    "goat": ("args/goat_cliffs_args.txt", ["cliffs_rugged", "flat"], "goat_cliffs.trlpack"),
}


# ------------------------------------------------------------------------------------------------ shared helpers (also the CPU test's)
def data_root(trl, assets, dst):
    """a copy of tests/golden/reference (args + data) with the models the arg files name: dog and goat written by trl_output_model from
    the packs, raptor put back together from its committed parts.  Returns (root, {scene: model path})"""
    root = os.path.join(dst, "ref")
    if not os.path.isdir(root):
        shutil.copytree(REF, root)
    models = {}
    for scene, (_, _, pack) in SCENES.items():
        if pack is None:      # where the raptor args expect it, beside its committed _scale.txt
            models[scene] = os.path.join(root, "data", "policies", "raptor", "models", "raptor_mace3_mixed_model.h5")
            if not os.path.exists(models[scene]):
                raptor_mixed_model(os.path.dirname(models[scene]))
        else:
            models[scene] = os.path.join(root, "%s_model.h5" % scene)
            if not os.path.exists(models[scene]):
                exported_model(trl, os.path.join(assets, pack), models[scene])
    return root, models


def terrain_path(root, name):
    return os.path.join(root, "data", "terrain", name + ".txt")


def scene_args(scene, terrain, model, extra=()):
    return ["-arg_file=", SCENES[scene][0], "-terrain_file=", "data/terrain/%s.txt" % terrain, "-policy_model=", model] + list(extra)


def make_handle(trl, scene, root, model, terrains, n, slots, explore=False, extra=(), seeds=None, rng_seed=77):
    """a handle of `scene` created with terrains[0]; terrains[1:] loaded into slots 1.., envs assigned by `slots` and then reseeded (so
    that every env starts on its own terrain, exactly as a fresh handle of that terrain does)"""
    cls = trl.ScenarioExpMACE if explore else trl.ScenarioPoliEval
    sc = cls(None, n, args=scene_args(scene, terrains[0], model, extra), data_root=root, rng_seed=rng_seed, terrain_seeds=seeds)
    for t, name in enumerate(terrains[1:], 1):
        sc.LoadTerrain(t, terrain_path(root, name))
    if slots is not None:
        sc.SetEnvTerrain(slots)
        sc.SetRandSeed(np.arange(1, n + 1, dtype=np.uint64) if seeds is None else seeds)
    if explore:
        sc.EnableExplore(1, 0.3, 0.5, 0.05)
    return sc


def env_record(sc, e, n_out):
    q, qd, tau, c = sc.GetState(e)
    rec = [q, qd, tau, c, sc.GetCtrl(e), sc.GetNetOut(e, n_out), sc.GetPoliState(e)]
    for seg in (0, 1):
        d, mx, fl = sc.GetTerrain(e, seg)
        rec += [d, np.array([mx, fl])]
    return rec


def assert_same_env(a, ea, b, eb, n_out, what):
    for k, (x, y) in enumerate(zip(env_record(a, ea, n_out), env_record(b, eb, n_out))):
        assert np.array_equal(x, y), (what, ea, eb, "field", k)


def assert_union(mixed, refs, slots, n_out, stride=1):
    """env e of `mixed` == env e of refs[slots[e]]: state, controller, decision, policy state, counters, both terrain segments and its
    own distance-log sequence"""
    dist, denv = mixed.GetDistLog()
    logs = [r.GetDistLog() for r in refs]
    cur, nxt = mixed.EnvTerrain()
    for e in range(0, mixed.num_envs, stride):
        t = int(slots[e])
        assert nxt[e] == t
        assert_same_env(mixed, e, refs[t], e, n_out, "terrain %d" % t)
        rd, re = logs[t]
        assert np.array_equal(dist[denv == e], rd[re == e]), ("distance log", e, t)
    assert np.array_equal(cur, np.asarray(slots)), "every env is on its assigned terrain after the reseed"


def tuples_by_env(sc):
    r, f, e = sc.GetTuples(f64=True)
    order = np.lexsort((np.arange(len(e)), e))
    return r[order], f[order], e[order]


def cell_stats(sc, p, t):
    c = C.c_int64(0); e = C.c_int64(0); a = C.c_double(0); s = C.c_int64(0)
    sc._ck(sc.L.trl_eval_stats_cell(sc.h, int(p), int(t), C.byref(c), C.byref(e), C.byref(a), C.byref(s)))
    return dict(cycles=c.value, episodes=e.value, avg_dist=a.value, steps=s.value)


@pytest.fixture(scope="module")
def ref_root(tmp_path_factory, assets):
    import deepterrainrl_b200 as trl
    return data_root(trl, assets, str(tmp_path_factory.mktemp("terrain_slots")))


def _schedule(monkeypatch, schedule):
    monkeypatch.delenv("TRL_SERIAL_SCHEDULE", raising=False)
    monkeypatch.delenv("TRL_GROUPS", raising=False)
    if schedule == "serial":
        monkeypatch.setenv("TRL_SERIAL_SCHEDULE", "1")
    elif schedule == "groups3":
        monkeypatch.setenv("TRL_GROUPS", "3")


def _run(sc, updates):
    for _ in range(updates):
        sc.Update(1.0 / 30.0)
    sc.Sync()
    return sc


def tip_over(sc, envs):
    """root angle past 0.8 pi: these envs fall at the end of the next update and reset"""
    for e in envs:
        q = sc.GetState(int(e))[0]
        q[2] = 3.0
        sc.SetState(int(e), q=q)


def _run_with_falls(sc, updates, n):
    """`updates` updates; a tenth of the way in, every 16th env is tipped over, so that every scene resets envs inside the window"""
    _run(sc, updates // 10)
    tip_over(sc, range(0, n, 16))
    return _run(sc, updates - updates // 10)


# ------------------------------------------------------------------------------------------------ (1) union of single-terrain handles
CASES = [("dog", p, 1536, "overlap") for p in ("round_robin", "blocks", "random", "no_slot0")]
CASES += [("dog", "random", 1536, "serial"), ("dog", "blocks", 1536, "groups3")]
CASES += [("raptor", "random", 1024, "overlap"), ("raptor", "no_slot0", 1024, "serial"), ("goat", "round_robin", 512, "overlap"),
          ("goat", "random", 512, "groups3")]


@pytest.mark.parametrize("scene,pattern,n,schedule", CASES)
def test_mixed_batch_is_the_union_of_single_terrain_runs(ref_root, monkeypatch, scene, pattern, n, schedule):
    import deepterrainrl_b200 as trl
    root, models = ref_root
    _schedule(monkeypatch, schedule)
    terrains = SCENES[scene][1]
    n_out = 87 if scene == "raptor" else 90
    slots = assignment(pattern, n, len(terrains), seed=n)
    refs = [_run_with_falls(make_handle(trl, scene, root, models[scene], [t], n, None), UPDATES, n) for t in terrains]
    mixed = _run_with_falls(make_handle(trl, scene, root, models[scene], terrains, n, slots), UPDATES, n)
    assert all(r.GetNumEpisodes() > 0 for r in refs)          # falls and resets happen inside the window compared
    assert_union(mixed, refs, slots, n_out)
    for t in range(len(terrains)):                             # per-terrain statistics against the single handles' envs
        on = np.flatnonzero(slots == t)
        st = mixed.GetEvalStats(None, terrain=t)
        rd, re = refs[t].GetDistLog()
        keep = np.isin(re, on)
        assert st["episodes"] == int(keep.sum())
        assert st["cycles"] == int(sum(refs[t].GetCtrl(int(e))[-2] for e in on))
        if keep.any():
            assert abs(st["avg_dist"] - float(np.mean(rd[keep]))) <= 1e-12 * max(1.0, abs(float(np.mean(rd[keep]))))
    for sc in refs + [mixed]:
        sc.close()


@pytest.mark.parametrize("schedule", ["overlap", "serial"])
def test_exploration_tuples_are_the_union(ref_root, monkeypatch, schedule):
    import deepterrainrl_b200 as trl
    root, models = ref_root
    _schedule(monkeypatch, schedule)
    terrains = DOG_TERRAINS[:4]
    n = 512
    slots = assignment("random", n, len(terrains), seed=9)
    refs = [_run(make_handle(trl, "dog", root, models["dog"], [t], n, None, explore=True), UPDATES) for t in terrains]
    mixed = _run(make_handle(trl, "dog", root, models["dog"], terrains, n, slots, explore=True), UPDATES)
    assert_union(mixed, refs, slots, 90, stride=3)
    r, f, e = tuples_by_env(mixed)
    assert r.shape[0] > 0
    for t, ref in enumerate(refs):
        rr, rf, re = tuples_by_env(ref)
        keep = np.isin(re, np.flatnonzero(slots == t))
        mine = slots[e] == t
        assert np.array_equal(e[mine], re[keep]) and np.array_equal(f[mine], rf[keep]), t
        assert np.array_equal(r[mine], rr[keep]), t
    for sc in refs + [mixed]:
        sc.close()


# ------------------------------------------------------------------------------------------------ (2) policy x terrain
def test_policy_by_terrain_matrix(ref_root, tmp_path):
    import deepterrainrl_b200 as trl
    root, models = ref_root
    base = pack_net(os.path.join(ROOT, "assets", "dog_slopes_mixed.trlpack"))
    nets = [write_net(str(tmp_path / ("p%d.h5" % p)), perturbed(base, p)) for p in (1, 2)]
    pol = [None] + [(m, os.path.splitext(m)[0] + "_scale.txt") for m in nets]
    terrains = ["slopes_mixed", "tight_gaps", "flat"]
    n = 1800
    rng = np.random.default_rng(5)
    pslots, tslots = rng.integers(0, 3, n), rng.integers(0, 3, n)
    mixed = make_handle(trl, "dog", root, models["dog"], terrains, n, tslots)
    for p in (1, 2):
        mixed.LoadPolicy(p, *pol[p])
    mixed.SetEnvPolicy(pslots)
    _run_with_falls(mixed, UPDATES, n)
    singles = {}
    for p in range(3):
        for t in range(3):
            sc = make_handle(trl, "dog", root, models["dog"], [terrains[t]], n, None)
            if pol[p] is not None:
                sc.LoadModel(*pol[p])
            singles[p, t] = _run_with_falls(sc, UPDATES, n)
    for e in range(n):
        assert_same_env(mixed, e, singles[int(pslots[e]), int(tslots[e])], e, 90, ("cell", int(pslots[e]), int(tslots[e])))
    logs = {k: s.GetDistLog() for k, s in singles.items()}
    steps = mixed.GetNumEnvSteps() // n
    for p in (-1, 0, 1, 2):
        for t in (-1, 0, 1, 2):
            on = np.flatnonzero(((pslots == p) | (p < 0)) & ((tslots == t) | (t < 0)))
            d = np.concatenate([logs[int(pslots[e]), int(tslots[e])][0][logs[int(pslots[e]), int(tslots[e])][1] == e] for e in on] + [np.zeros(0)])
            st = cell_stats(mixed, p, t)
            assert st["episodes"] == d.size, (p, t)
            assert st["cycles"] == int(sum(singles[int(pslots[e]), int(tslots[e])].GetCtrl(int(e))[-2] for e in on)), (p, t)
            assert st["steps"] == on.size * steps, (p, t)
            if d.size:
                assert abs(st["avg_dist"] - float(np.mean(d))) <= 1e-12 * max(1.0, abs(float(np.mean(d)))), (p, t)
    assert sum(cell_stats(mixed, 0, t)["episodes"] for t in range(3)) > 0
    for p in range(3):
        assert mixed.GetEvalStats(p) == cell_stats(mixed, p, -1), p     # trl_eval_stats_slot is the cell (p, any), bit for bit
    for sc in list(singles.values()) + [mixed]:
        sc.close()


# ------------------------------------------------------------------------------------------------ (3) against the oracle
def test_free_running_against_oracle(ref_root, tmp_path):
    import deepterrainrl_b200 as trl
    from pyoracle import Oracle
    root, models = ref_root
    terrains = ["mixed", "tight_gaps", "slopes_mixed", "narrow_gaps"]
    n = 64
    seeds = np.arange(101, 101 + n, dtype=np.uint64)
    slots = np.arange(n) % 4
    packs = []
    for t in terrains:
        packs.append(str(tmp_path / (t + ".trlpack")))
        trl.pack_from_args(scene_args("dog", t, models["dog"]), root, packs[-1])
    g = trl.ScenarioPoliEval(packs[0], n, terrain_seeds=seeds)
    for t, name in enumerate(terrains[1:], 1):
        g.LoadTerrain(t, terrain_path(root, name))
    g.SetEnvTerrain(slots)
    g.SetRandSeed(seeds)
    orc = [Oracle(p, n, 0, terrain_seeds=seeds) for p in packs]

    def check_terrain():
        for e in range(n):
            o = orc[slots[e]]
            for seg in (0, 1):
                gd, gmx, gfl = g.GetTerrain(e, seg)
                od, omx, ofl = o.terrain(e, seg)
                assert gd.size == od.size and gfl == ofl and gmx == omx, (e, seg)
                assert np.array_equal(gd, od), (e, seg)

    check_terrain()
    worst = 0.0
    for k in range(600):
        g.EnvStep(H)
        for e in range(n):
            orc[slots[e]].env_step(e, H)
        if k % 50 == 49:
            for e in range(n):
                gq, gqd, _, _ = g.GetState(e)
                oq, oqd, _, _ = orc[slots[e]].get_state(e)
                err = max(np.max(np.abs(gq - oq) / (1 + np.abs(oq))), np.max(np.abs(gqd - oqd) / (1 + np.abs(oqd))))
                worst = max(worst, err)
                assert err < 1e-4, (k, e, terrains[slots[e]])
    check_terrain()
    print("terrain slots vs oracle, 600 env-steps: worst rel err %.3e" % worst)


# ------------------------------------------------------------------------------------------------ (4) next reset, blend
def test_assignment_takes_effect_at_the_next_reset(ref_root):
    import deepterrainrl_b200 as trl
    root, models = ref_root
    n = 2048
    terrains = ["slopes_mixed", "tight_gaps"]
    a = _run(make_handle(trl, "dog", root, models["dog"], terrains, n, None), 10)
    b = _run(make_handle(trl, "dog", root, models["dog"], terrains, n, None), 10)
    before = [a.GetTerrain(e, s)[0] for e in range(n) for s in (0, 1)]
    moved = np.arange(0, n, 2)
    a.SetEnvTerrain(np.ones(moved.size, np.int32), env_ids=moved)
    cur, nxt = a.EnvTerrain()
    assert np.all(cur == 0) and np.array_equal(np.flatnonzero(nxt), moved)
    assert all(np.array_equal(x, a.GetTerrain(e, s)[0]) for x, (e, s) in zip(before, [(e, s) for e in range(n) for s in (0, 1)]))
    _run(a, 5); _run(b, 5)
    tipped = moved[::4]
    tip_over(a, tipped); tip_over(b, tipped)
    _run(a, 35); _run(b, 35)
    cur, nxt = a.EnvTerrain()
    # a moved env switches at its first fall and not before: until then (and every unmoved env throughout) it is the env of the handle
    # without the assignment; after it, its ground comes from slot 1
    switched = cur == 1
    assert switched[tipped].all() and not switched[moved].all()
    assert not switched[1::2].any()
    for e in np.flatnonzero(~switched)[::3]:
        assert_same_env(a, int(e), b, int(e), 90, "no reset yet / not moved")
    for e in np.flatnonzero(switched):
        assert not np.array_equal(a.GetTerrain(int(e), 0)[0], b.GetTerrain(int(e), 0)[0]), e
    # trl_reset switches the rest; an assignment survives a reseed, which then reproduces a fresh handle of that terrain
    a.Reset(moved)
    assert np.array_equal(a.EnvTerrain()[0], nxt)
    a.SetRandSeed(np.arange(1, n + 1, dtype=np.uint64))
    fresh = make_handle(trl, "dog", root, models["dog"], ["tight_gaps"], n, None)
    base = make_handle(trl, "dog", root, models["dog"], ["slopes_mixed"], n, None)
    assert np.array_equal(a.EnvTerrain()[1], nxt)
    for e in range(0, n, 13):
        for s in (0, 1):
            want = (fresh if nxt[e] else base).GetTerrain(e, s)
            got = a.GetTerrain(e, s)
            assert np.array_equal(got[0], want[0]) and got[1:] == want[1:], (e, s)
    for sc in (a, b, fresh, base):
        sc.close()


def test_slot_follows_the_handle_blend(ref_root, tmp_path):
    import deepterrainrl_b200 as trl
    root, models = ref_root
    two = str(tmp_path / "two_sets.txt")
    sets = [dict(SlopeDeltaRange=0.05, SlopeDeltaMin=-0.1, SlopeDeltaMax=0.1, GapSpacingMin=6, GapWMin=0.2, GapWMax=0.6),
            dict(SlopeDeltaRange=0.3, SlopeDeltaMin=-0.4, SlopeDeltaMax=0.4, GapSpacingMin=3, GapWMin=0.5, GapWMax=1.4)]
    with open(two, "w") as f:
        json.dump({"Type": "slopes_gaps", "Params": sets}, f)
    n = 256
    shutil.copy(two, terrain_path(root, "two_sets"))
    ref = make_handle(trl, "dog", root, models["dog"], ["two_sets"], n, None, extra=["-terrain_blend=", "0.5"])
    ref.SetRandSeed(np.arange(1, n + 1, dtype=np.uint64))
    sc = make_handle(trl, "dog", root, models["dog"], ["flat"], n, None)
    sc.LoadTerrain(1, two)
    sc.SetTerrainParamsLerp(0.5)
    sc.SetTerrainParamsLerp(0.5)                      # unchanged blend: nothing to do
    sc.SetEnvTerrain(np.ones(n, np.int32))
    sc.SetRandSeed(np.arange(1, n + 1, dtype=np.uint64))
    unblended = make_handle(trl, "dog", root, models["dog"], ["two_sets"], n, None)
    _run(ref, 20); _run(sc, 20); _run(unblended, 20)
    for e in range(0, n, 3):
        assert_same_env(sc, e, ref, e, 90, "blend 0.5")
    assert any(not np.array_equal(sc.GetTerrain(e, 0)[0], unblended.GetTerrain(e, 0)[0]) for e in range(n))
    for h in (ref, sc, unblended):
        h.close()


# ------------------------------------------------------------------------------------------------ (5) beside a trainer
def test_training_on_a_terrain_slot_exploration_handle_is_reproducible(ref_root, assets):
    from deepterrainrl_b200.train import ScenarioTrainMACE, TrainSchedule
    root, _ = ref_root
    pack = os.path.join(assets, "dog_slopes_mixed.trlpack")
    n = 512
    slots = np.arange(n) % 3

    def run():
        st = ScenarioTrainMACE(pack, n, rng_seed=11, iters_per_update=2,
                               schedule=TrainSchedule(init_exp_rate=0.5, exp_rate=0.2, init_exp_temp=5, exp_temp=0.025,
                                                      init_exp_base_rate=0.2, exp_base_rate=0.002, trainer_num_anneal_iters=60,
                                                      exp_base_anneal_iters=60),
                               trainer_params=dict(replay_mem_size=20000, num_init_samples=300, freeze_target_iters=7, seed=2))
        st.exp.LoadTerrain(1, terrain_path(root, "mixed"))
        st.exp.LoadTerrain(2, terrain_path(root, "narrow_gaps"))
        st.exp.SetEnvTerrain(slots)
        st.exp.SetRandSeed(np.arange(1, n + 1, dtype=np.uint64))
        st.RunNative(40)
        return st

    a, b = run(), run()
    ca, cb = a.trainer.counters(), b.trainer.counters()
    assert ca == cb and ca["iter"] > 5
    np.testing.assert_array_equal(a.trainer.get("theta"), b.trainer.get("theta"))
    np.testing.assert_array_equal(a.exp.GetStateAll()[0], b.exp.GetStateAll()[0])
    assert np.array_equal(a.exp.EnvTerrain()[0], slots)


# ------------------------------------------------------------------------------------------------ (6) refusals
def test_refusals_leave_the_handle_unchanged(ref_root, tmp_path):
    import deepterrainrl_b200 as trl
    root, models = ref_root
    n = 128
    terrains = ["slopes_mixed", "tight_gaps"]
    slots = np.arange(n) % 2
    sc = make_handle(trl, "dog", root, models["dog"], terrains, n, slots)
    bad_type = str(tmp_path / "bad_type.txt")
    with open(bad_type, "w") as f:
        f.write('{"Type": "lava", "Params": []}')
    bad_json = str(tmp_path / "bad_json.txt")
    with open(bad_json, "w") as f:
        f.write('{"Type": "flat", "Params": [ {"GapWMin": 1,, } ]')
    L = sc.L
    for call, msg in [(lambda: sc.LoadTerrain(0, terrain_path(root, "flat")), "out of range"),
                      (lambda: sc.LoadTerrain(8, terrain_path(root, "flat")), "out of range"),
                      (lambda: sc.LoadTerrain(3, bad_type), "unknown terrain type"),
                      (lambda: sc.LoadTerrain(3, bad_json), "json"),
                      (lambda: sc.LoadTerrain(3, str(tmp_path / "missing.txt")), "trl_load_terrain"),
                      (lambda: sc._ck(L.trl_load_terrain(sc.h, 3, None)), "null path"),
                      (lambda: sc.SetEnvTerrain([2]), "empty"),
                      (lambda: sc.SetEnvTerrain([8]), "out of range"),
                      (lambda: sc.SetEnvTerrain([1], env_ids=[n]), "env id"),
                      (lambda: sc.SetEnvTerrain([1], env_ids=[-1]), "env id"),
                      (lambda: sc.SetEnvTerrain(np.zeros(n + 1, np.int32)), "env count"),
                      (lambda: sc.GetEvalStats(None, terrain=2), "empty"),
                      (lambda: sc.GetEvalStats(None, terrain=9), "out of range")]:
        with pytest.raises(RuntimeError, match=msg):
            call()
    null = C.c_void_p(0)
    i32 = C.c_void_p(np.zeros(1, np.int32).ctypes.data)
    keep = i32
    for fn, args in [("trl_load_terrain", (1, terrain_path(root, "flat").encode())), ("trl_set_env_terrain", (None, keep, 1)),
                     ("trl_env_terrain", (keep, keep, 1)),
                     ("trl_eval_stats_cell", (-1, -1, None, None, None, None))]:
        assert getattr(L, fn)(null, *args) != 0
        assert b"null handle" in L.trl_last_error()
    assert np.array_equal(sc.EnvTerrain()[1], slots)
    _run(sc, UPDATES)
    clean = _run(make_handle(trl, "dog", root, models["dog"], terrains, n, slots), UPDATES)
    for e in range(0, n, 5):
        assert_same_env(sc, e, clean, e, 90, "after refusals")
    sc.close(); clean.close()
