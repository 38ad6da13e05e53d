"""Physics slots (trl_load_physics / trl_set_env_physics / trl_env_physics / trl_eval_stats_phys): one handle runs the contact and
joint-limit model of each env with one of up to 8 settings.  The contract is exact: with the same seeds, env i on physics slot q computes,
bit for bit, what env i computes in a handle of the same pack, size and seeds whose trl_set_phys_params holds slot q's values (created
with TRL_VERTEX_CONTACTS=1 when the slot has vertex contacts).

  1. whole updates of dog (4 settings), raptor (3) and goat (2) under the overlapped schedule, the serial schedule and 3 env groups, in
     evaluation and in exploration (tuples by env), against one single-physics handle per setting;
  2. policy x terrain x physics (2 x 2 x 2) against the 8 single handles, every trl_eval_stats_phys cell and its marginals;
  3. 600 free-running env-steps against one oracle batch per setting;
  4. the assignment rule (next reset; a reseed keeps it), reloading a slot and trl_set_phys_params on slot 0, two handles alternated;
  5. three training slots on three physics slots, lock-step and paced, against single-trainer handles; one trainer over 4 settings;
  6. checkpoints with physics, terrain and training slots; 7. every refusal.
tests/test_phys_slots_cpu.py runs a miniature on the emulator."""
import ctypes as C
import os

import numpy as np
import pytest

import torch_net  # noqa: F401  (torch before the library: see tests/test_gpu_decide_batches.py)
from test_gpu_checkpoint import assert_refused, assert_same, damaged_copies, save_and_load
from test_gpu_policy_slots import assignment, pack_net, perturbed, write_net
from test_gpu_terrain_slots import assert_same_env, tuples_by_env
from test_gpu_train_schedules import ref_loop_paced
from test_gpu_train_slots import (DT, SCHEDULE, TERRAIN, TRAINER, _schedule_env, assert_envs, assert_trainer, close, make_group, make_ref,
                                  ref_loop, start_models)

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ASSETS = os.path.join(ROOT, "assets")
UPDATES = 30
H = 1.0 / 600.0
DEFAULT = [2.0e5, 2.0e3, 0.81, 0.01, 0.00025, 2.0e4, 20.0]


def setting(vertex=False, **kw):
    p = list(DEFAULT)
    for k, v in kw.items():
        p[["kn", "dn", "mu", "v_eps", "tol", "k_lim", "d_lim"].index(k)] = v
    return p, vertex


# slot 0 is the scene's own setting (DEFAULT, no vertex contacts)
SCENES = {
    "dog": ("dog_slopes_mixed.trlpack", [setting(), setting(mu=0.3), setting(kn=5e4, dn=5e2), setting(vertex=True)], 90),
    "raptor": ("raptor_narrow_gaps.trlpack", [setting(), setting(vertex=True, mu=1.0), setting(tol=0.001, k_lim=5e4, d_lim=50.0)], 87),
    "goat": ("goat_cliffs.trlpack", [setting(), setting(vertex=True, mu=0.5, kn=1e5)], 90),
}


# ------------------------------------------------------------------------------------------------ shared helpers (also the CPU test's)
def single(trl, pack, n, s, monkeypatch, explore=False, rng_seed=77):
    """the reference handle of setting s: trl_set_phys_params holds its values, created with TRL_VERTEX_CONTACTS=1 if it has vertex
    contacts"""
    p, vertex = s
    if vertex:
        monkeypatch.setenv("TRL_VERTEX_CONTACTS", "1")
    try:
        sc = (trl.ScenarioExpMACE if explore else trl.ScenarioPoliEval)(pack, n, rng_seed=rng_seed)
    finally:
        monkeypatch.delenv("TRL_VERTEX_CONTACTS", raising=False)
    sc.SetPhysParams(p)
    sc.SetRandSeed(np.arange(1, n + 1, dtype=np.uint64))
    if explore:
        sc.EnableExplore(1, 0.3, 0.5, 0.05)
    return sc


def mixed(trl, pack, n, settings, slots, explore=False, rng_seed=77):
    """one handle with settings[1:] in physics slots 1.., envs assigned by `slots`, then reseeded (every env starts on its own
    setting, as the single handle's envs do)"""
    sc = (trl.ScenarioExpMACE if explore else trl.ScenarioPoliEval)(pack, n, rng_seed=rng_seed)
    for q, (p, vertex) in enumerate(settings[1:], 1):
        sc.LoadPhysics(q, p, vertex)
    sc.SetEnvPhysics(slots)
    sc.SetRandSeed(np.arange(1, n + 1, dtype=np.uint64))
    if explore:
        sc.EnableExplore(1, 0.3, 0.5, 0.05)
    return sc


def run(sc, updates):
    for _ in range(updates):
        sc.Update(DT)
    sc.Sync()
    return sc


def tip_over(sc, envs):
    for e in envs:
        q = sc.GetState(int(e))[0]
        q[2] = 3.0
        sc.SetState(int(e), q=q)


def run_with_falls(sc, updates, n):
    run(sc, updates // 10)
    tip_over(sc, range(0, n, 16))
    return run(sc, updates - updates // 10)


def assert_union(mix, refs, slots, n_out, stride=1):
    """env e of `mix` == env e of refs[slots[e]], its distance log included; every env is on its assigned slot"""
    dist, denv = mix.GetDistLog()
    logs = [r.GetDistLog() for r in refs]
    cur, nxt = mix.EnvPhysics()
    assert np.array_equal(cur, slots) and np.array_equal(nxt, slots)
    for e in range(0, mix.num_envs, stride):
        q = int(slots[e])
        assert_same_env(mix, e, refs[q], e, n_out, "physics %d" % q)
        rd, re = logs[q]
        assert np.array_equal(dist[denv == e], rd[re == e]), ("distance log", e, q)


def phys_stats(sc, p, t, q):
    c = C.c_int64(0); e = C.c_int64(0); a = C.c_double(0); s = C.c_int64(0)
    sc._ck(sc.L.trl_eval_stats_phys(sc.h, int(p), int(t), int(q), C.byref(c), C.byref(e), C.byref(a), C.byref(s)))
    return dict(cycles=c.value, episodes=e.value, avg_dist=a.value, steps=s.value)


def cell_stats(sc, p, t):
    c = C.c_int64(0); e = C.c_int64(0); a = C.c_double(0); s = C.c_int64(0)
    sc._ck(sc.L.trl_eval_stats_cell(sc.h, int(p), int(t), C.byref(c), C.byref(e), C.byref(a), C.byref(s)))
    return dict(cycles=c.value, episodes=e.value, avg_dist=a.value, steps=s.value)


# ------------------------------------------------------------------------------------------------ (1) union of single-physics handles
CASES = [("dog", p, 1024, "overlap") for p in ("round_robin", "blocks", "random", "no_slot0")]
CASES += [("dog", "random", 1024, "serial"), ("dog", "blocks", 1024, "groups3")]
CASES += [("raptor", "random", 768, "overlap"), ("raptor", "no_slot0", 768, "serial"), ("raptor", "blocks", 768, "groups3"),
          ("goat", "round_robin", 512, "overlap"), ("goat", "random", 512, "groups3"), ("goat", "no_slot0", 512, "serial")]


@pytest.mark.parametrize("scene,pattern,n,schedule", CASES)
def test_mixed_batch_is_the_union_of_single_physics_runs(monkeypatch, scene, pattern, n, schedule):
    import deepterrainrl_b200 as trl
    _schedule_env(monkeypatch, schedule)
    pack, settings, n_out = SCENES[scene]
    pack = os.path.join(ASSETS, pack)
    slots = assignment(pattern, n, len(settings), seed=n)
    refs = [run_with_falls(single(trl, pack, n, s, monkeypatch), UPDATES, n) for s in settings]
    mix = run_with_falls(mixed(trl, pack, n, settings, slots), UPDATES, n)
    assert all(r.GetNumEpisodes() > 0 for r in refs)
    assert_union(mix, refs, slots, n_out, stride=2)
    for q in range(len(settings)):                   # a physics-only cell against the single handle's envs of that slot
        on = np.flatnonzero(slots == q)
        st = mix.GetEvalStats(None, physics=q)
        rd, re = refs[q].GetDistLog()
        keep = np.isin(re, on)
        assert st["episodes"] == int(keep.sum()), q
        assert st["cycles"] == int(sum(refs[q].GetCtrl(int(e))[-2] for e in on)), q
        if keep.any():
            assert abs(st["avg_dist"] - float(np.mean(rd[keep]))) <= 1e-12 * max(1.0, abs(float(np.mean(rd[keep])))), q
    # the settings really differ: some env of each slot leaves the slot-0 trajectory
    for q in range(1, len(settings)):
        assert any(not np.array_equal(mix.GetState(int(e))[0], refs[0].GetState(int(e))[0]) for e in np.flatnonzero(slots == q)), q
    close(*refs, mix)


@pytest.mark.parametrize("schedule", ["overlap", "serial", "groups3"])
def test_exploration_tuples_are_the_union(monkeypatch, schedule):
    import deepterrainrl_b200 as trl
    _schedule_env(monkeypatch, schedule)
    pack, settings, _ = SCENES["dog"]
    pack = os.path.join(ASSETS, pack)
    n = 512
    slots = assignment("random", n, len(settings), seed=9)
    refs = [run(single(trl, pack, n, s, monkeypatch, explore=True), UPDATES) for s in settings]
    mix = run(mixed(trl, pack, n, settings, slots, explore=True), UPDATES)
    assert_union(mix, refs, slots, 90, stride=3)
    r, f, e = tuples_by_env(mix)
    assert r.shape[0] > 0
    for q, ref in enumerate(refs):
        rr, rf, re = tuples_by_env(ref)
        keep = np.isin(re, np.flatnonzero(slots == q))
        mine = slots[e] == q
        assert np.array_equal(e[mine], re[keep]) and np.array_equal(f[mine], rf[keep]), q
        assert np.array_equal(r[mine], rr[keep]), q
    close(*refs, mix)


# ------------------------------------------------------------------------------------------------ (2) policy x terrain x physics
def test_policy_terrain_physics_cube(monkeypatch, tmp_path):
    import deepterrainrl_b200 as trl
    pack = os.path.join(ASSETS, "dog_slopes_mixed.trlpack")
    net = write_net(str(tmp_path / "p1.h5"), perturbed(pack_net(pack), 1))
    model = (net, os.path.splitext(net)[0] + "_scale.txt")
    tfile = os.path.join(TERRAIN, "tight_gaps.txt")
    settings = [setting(), setting(mu=0.3)]
    n = 1600
    rng = np.random.default_rng(5)
    ps, ts, qs = rng.integers(0, 2, n), rng.integers(0, 2, n), rng.integers(0, 2, n)

    def make(pol, terr, phys_slots, s=None):
        sc = trl.ScenarioPoliEval(pack, n, rng_seed=77)
        sc.LoadTerrain(1, tfile)
        sc.SetEnvTerrain(terr)
        if phys_slots is None:
            sc.SetPhysParams(s[0])
        else:
            sc.LoadPhysics(1, *settings[1])
            sc.SetEnvPhysics(phys_slots)
        if isinstance(pol, np.ndarray):
            sc.LoadPolicy(1, *model)
            sc.SetEnvPolicy(pol)
        elif pol:
            sc.LoadModel(*model)
        sc.SetRandSeed(np.arange(1, n + 1, dtype=np.uint64))
        return run_with_falls(sc, UPDATES, n)

    mix = make(ps, ts, qs)
    singles = {}
    for p in range(2):
        for t in range(2):
            for q in range(2):
                singles[p, t, q] = make(p == 1, np.full(n, t), None, settings[q])
    key = lambda e: (int(ps[e]), int(ts[e]), int(qs[e]))
    for e in range(0, n, 3):
        assert_same_env(mix, e, singles[key(e)], e, 90, ("cell",) + key(e))
    logs = {k: s.GetDistLog() for k, s in singles.items()}
    steps = mix.GetNumEnvSteps() // n
    for p in (-1, 0, 1):
        for t in (-1, 0, 1):
            for q in (-1, 0, 1):
                on = np.flatnonzero(((ps == p) | (p < 0)) & ((ts == t) | (t < 0)) & ((qs == q) | (q < 0)))
                d = np.concatenate([logs[key(e)][0][logs[key(e)][1] == e] for e in on] + [np.zeros(0)])
                st = phys_stats(mix, p, t, q)
                assert st["episodes"] == d.size, (p, t, q)
                assert st["cycles"] == int(sum(singles[key(e)].GetCtrl(int(e))[-2] for e in on)), (p, t, q)
                assert st["steps"] == on.size * steps, (p, t, q)
                if d.size:
                    assert abs(st["avg_dist"] - float(np.mean(d))) <= 1e-12 * max(1.0, abs(float(np.mean(d)))), (p, t, q)
            assert phys_stats(mix, p, t, -1) == cell_stats(mix, p, t), (p, t)      # bit for bit
    assert mix.GetEvalStats(None, None, physics=-1) == mix._stats()
    close(mix, *singles.values())


# ------------------------------------------------------------------------------------------------ (3) against the oracle
def test_free_running_against_oracle(monkeypatch):
    import deepterrainrl_b200 as trl
    from pyoracle import Oracle
    pack, settings, _ = SCENES["dog"]
    pack = os.path.join(ASSETS, pack)
    n = 64
    seeds = np.arange(101, 101 + n, dtype=np.uint64)
    slots = np.arange(n) % len(settings)
    g = trl.ScenarioPoliEval(pack, n, terrain_seeds=seeds)
    for q, (p, vertex) in enumerate(settings[1:], 1):
        g.LoadPhysics(q, p, vertex)
    g.SetEnvPhysics(slots)
    g.SetRandSeed(seeds)
    orc = []
    for p, vertex in settings:
        if vertex:
            monkeypatch.setenv("ORC_VTX", "1")
        o = Oracle(pack, n, 0, terrain_seeds=seeds)
        monkeypatch.delenv("ORC_VTX", raising=False)
        o.set_phys(p)
        orc.append(o)
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
                assert err < 1e-4, (k, e, slots[e])
    print("physics slots vs oracle, 600 env-steps: worst rel err %.3e" % worst)


# ------------------------------------------------------------------------------------------------ (4) assignment rule, values, two handles
def test_assignment_takes_effect_at_the_next_reset(monkeypatch):
    import deepterrainrl_b200 as trl
    pack = os.path.join(ASSETS, "dog_slopes_mixed.trlpack")
    n = 1024
    soft = setting(kn=5e4, dn=5e2)
    a = trl.ScenarioPoliEval(pack, n, rng_seed=77)
    a.LoadPhysics(1, *soft)
    b = trl.ScenarioPoliEval(pack, n, rng_seed=77)
    run(a, 10); run(b, 10)
    moved = np.arange(0, n, 2)
    a.SetEnvPhysics(np.ones(moved.size, np.int32), env_ids=moved)
    cur, nxt = a.EnvPhysics()
    assert np.all(cur == 0) and np.array_equal(np.flatnonzero(nxt), moved)
    run(a, 5); run(b, 5)
    tipped = moved[::4]
    tip_over(a, tipped); tip_over(b, tipped)
    run(a, 35); run(b, 35)
    cur, nxt = a.EnvPhysics()
    switched = cur == 1
    assert switched[tipped].all() and not switched[moved].all() and not switched[1::2].any()
    for e in np.flatnonzero(~switched)[::3]:        # the ongoing episode is untouched until the env's next reset
        assert_same_env(a, int(e), b, int(e), 90, "no reset yet / not moved")
    # trl_reset applies the rest; a reseed keeps the assignment and then reproduces a fresh handle of each setting
    a.Reset(moved)
    assert np.array_equal(a.EnvPhysics()[0], nxt)
    a.SetRandSeed(np.arange(1, n + 1, dtype=np.uint64))
    assert np.array_equal(a.EnvPhysics()[0], nxt) and np.array_equal(a.EnvPhysics()[1], nxt)
    refs = [single(trl, pack, n, s, monkeypatch) for s in (setting(), soft)]
    run(a, 20)
    for r in refs:
        run(r, 20)
    for e in range(0, n, 5):
        assert_same_env(a, e, refs[int(nxt[e])], e, 90, "after the reseed")
    close(a, b, *refs)


def test_slot_values_apply_from_the_next_env_step(monkeypatch):
    import deepterrainrl_b200 as trl
    pack = os.path.join(ASSETS, "dog_slopes_mixed.trlpack")
    n = 512
    slots = np.arange(n) % 2
    s1, s1b, s0b = setting(mu=0.3), setting(mu=0.5), setting(mu=0.6)
    mix = mixed(trl, pack, n, [setting(), s1], slots)
    r0, r1 = single(trl, pack, n, setting(), monkeypatch), single(trl, pack, n, s1, monkeypatch)
    for sc in (mix, r0, r1):
        run(sc, 8)
    mix.LoadPhysics(1, *s1b)                 # reload: slot 1's envs only
    r1.SetPhysParams(s1b[0])
    for sc in (mix, r0, r1):
        run(sc, 8)
    mix.SetPhysParams(s0b[0])                # slot 0: its envs only
    r0.SetPhysParams(s0b[0])
    for sc in (mix, r0, r1):
        run(sc, 8)
    for e in range(n):
        assert_same_env(mix, e, (r0, r1)[slots[e]], e, 90, "slot %d" % slots[e])
    close(mix, r0, r1)


def test_two_handles_alternated(monkeypatch):
    import deepterrainrl_b200 as trl
    pack = os.path.join(ASSETS, "dog_slopes_mixed.trlpack")
    n = 256
    tabs = [[setting(), setting(mu=0.3), setting(vertex=True)], [setting(), setting(kn=5e4, dn=5e2)]]
    slots = [np.arange(n) % 3, (np.arange(n) // 7) % 2]
    alone = [run(mixed(trl, pack, n, t, s), 20) for t, s in zip(tabs, slots)]
    pair = [mixed(trl, pack, n, t, s) for t, s in zip(tabs, slots)]
    for _ in range(20):
        for sc in pair:
            sc.Update(DT)
    for x, y in zip(pair, alone):
        x.Sync()
        for e in range(0, n, 3):
            assert_same_env(x, e, y, e, 90, "alternated")
    close(*alone, *pair)


# ------------------------------------------------------------------------------------------------ (5) training
TRAIN_PHYS = [setting(), setting(mu=0.3), setting(kn=5e4, dn=5e2)]


@pytest.mark.parametrize("paced", [False, True])
def test_training_slots_on_their_own_physics(tmp_path, paced):
    import deepterrainrl_b200 as trl
    from deepterrainrl_b200.train import TrainSchedule, train_run_slots
    pack = os.path.join(ASSETS, "dog_slopes_mixed.trlpack")
    n = 2048
    models = start_models(pack, str(tmp_path))
    slots = assignment("random", n, 3, seed=1)

    def group_setup(sc):
        for q in (1, 2):
            sc.LoadPhysics(q, *TRAIN_PHYS[q])
        sc.SetEnvPhysics(slots)       # the resets of trl_set_env_policy make them current

    sched = TrainSchedule(**dict(SCHEDULE, trainer_curriculum_iters=0))
    updates = 60 if paced else 30
    group, trs = make_group(trl, pack, n, models, slots, setup=group_setup)
    train_run_slots(trs, sched, updates, None if paced else 2)
    refs = []
    for p in range(3):
        sc, tr = make_ref(trl, pack, n, models, p, slots, setup=lambda sc, p=p: sc.SetPhysParams(TRAIN_PHYS[p][0]))
        if paced:
            ref_loop_paced(sc, tr, p, slots, sched, updates)
        else:
            ref_loop(sc, tr, p, slots, sched, updates, 2)
        refs.append((sc, tr))
    assert np.array_equal(group.EnvPhysics()[0], slots)
    for p in range(3):
        assert trs[p].counters()["iter"] > 0
        assert_trainer(trs[p], refs[p][1], "slot %d" % p)
    assert_envs(group, [r[0] for r in refs], slots, 90, stride=2)
    close(*trs, group, *[o for r in refs for o in r])


def test_one_trainer_over_four_settings_is_reproducible(monkeypatch):
    import deepterrainrl_b200 as trl
    from deepterrainrl_b200.train import TrainSchedule
    from test_gpu_checkpoint import sp_of, train_run
    pack = os.path.join(ASSETS, "dog_slopes_mixed.trlpack")
    n = 1024
    settings = SCENES["dog"][1]
    slots = np.arange(n) % 4
    sp = sp_of(TrainSchedule(**SCHEDULE))
    out = []
    for schedule in ("overlap", "overlap", "serial", "groups3"):
        _schedule_env(monkeypatch, schedule)
        sc = mixed(trl, pack, n, settings, slots, explore=True, rng_seed=5)
        tr = trl.MACETrainer(sc, seed=3, **TRAINER)
        train_run(tr, sp, 30, 2)
        out.append((sc, tr))
    a, ta = out[0]
    assert ta.counters()["iter"] > 0
    for b, tb in out[1:]:
        assert_trainer(ta, tb, "reproducible")
        for e in range(0, n, 7):
            assert_same_env(a, e, b, e, 90, "reproducible")
    close(*[o for r in out for o in r[::-1]])


# ------------------------------------------------------------------------------------------------ (6) checkpoints
def test_checkpoint_with_physics_terrain_and_training_slots(tmp_path):
    import deepterrainrl_b200 as trl
    from deepterrainrl_b200.checkpoint import sections
    from deepterrainrl_b200.train import TrainSchedule, train_run_slots
    pack = os.path.join(ASSETS, "dog_slopes_mixed.trlpack")
    n = 1024
    models = start_models(pack, str(tmp_path))
    slots = np.arange(n) % 3
    phys = (np.arange(n) // 5) % 3

    def setup(sc):
        sc.LoadTerrain(1, os.path.join(TERRAIN, "narrow_gaps.txt"))
        sc.SetEnvTerrain((np.arange(n) // 3) % 2)
        sc.LoadPhysics(1, *TRAIN_PHYS[1])
        sc.LoadPhysics(2, DEFAULT, True)
        sc.SetEnvPhysics(phys)
    sched = TrainSchedule(**SCHEDULE)
    a, ta = make_group(trl, pack, n, models, slots, trainer_kw=TRAINER, setup=setup)
    b, tb = make_group(trl, pack, n, models, slots, trainer_kw=TRAINER, setup=setup)
    for trs in (ta, tb):
        train_run_slots(trs, sched, 20, 2)
    path = str(tmp_path / "phys.ckpt")
    b, tb = save_and_load(b, tb, path, user=b"phys")
    tb = [tb[p] for p in range(3)]
    names = [s[0] for s in sections(path)]
    assert all(k in names for k in ("phys_loaded", "phys_table", "env_phys_host", "env_phys"))
    for trs in (ta, tb):
        train_run_slots(trs, sched, 10, 2)
    assert all(np.array_equal(x, y) for x, y in zip(a.EnvPhysics(), b.EnvPhysics()))
    for q in range(3):
        assert a.GetEvalStats(None, physics=q) == b.GetEvalStats(None, physics=q), q
    assert_same(a, b, ta, tb, stride=3)
    d = tmp_path / "bad"
    d.mkdir()
    for p, msg in damaged_copies(path, str(d)):
        if any(k in msg for k in ("phys", "version", "truncated")):
            assert_refused(a.L, p, msg)
    # a handle without physics slots writes no physics section
    c = trl.ScenarioPoliEval(pack, 64)
    c.SaveCheckpoint(str(tmp_path / "plain.ckpt"))
    assert not any("phys" in s[0] for s in sections(str(tmp_path / "plain.ckpt")))
    c2, _, _ = trl.load_checkpoint(str(tmp_path / "plain.ckpt"))
    assert not any(x.any() for x in c2.EnvPhysics())
    close(*ta, *tb, a, b, c, c2)


# ------------------------------------------------------------------------------------------------ (7) refusals
def test_refusals_leave_the_handle_unchanged():
    import deepterrainrl_b200 as trl
    pack = os.path.join(ASSETS, "dog_slopes_mixed.trlpack")
    n = 128
    settings = [setting(), setting(mu=0.3)]
    slots = np.arange(n) % 2
    sc = mixed(trl, pack, n, settings, slots)
    L = sc.L
    bad = []
    for k, v in [(0, -1.0), (1, -1.0), (2, -0.1), (5, -1.0), (6, -1.0), (3, 0.0), (3, -1e-3), (4, 0.0021), (0, np.nan), (4, np.inf)]:
        p = list(DEFAULT)
        p[k] = v
        bad.append(p)
    cases = [(lambda: sc.LoadPhysics(0, DEFAULT), "out of range"), (lambda: sc.LoadPhysics(8, DEFAULT), "out of range"),
             (lambda: sc._ck(L.trl_load_physics(sc.h, 2, None, 0)), "null")]
    cases += [(lambda p=p: sc.LoadPhysics(2, p), "trl_load_physics") for p in bad]
    cases += [(lambda: sc.SetEnvPhysics([2]), "empty"), (lambda: sc.SetEnvPhysics([8]), "out of range"),
              (lambda: sc.SetEnvPhysics([-1]), "out of range"),
              (lambda: sc.SetEnvPhysics([1], env_ids=[n]), "env id"), (lambda: sc.SetEnvPhysics([1], env_ids=[-1]), "env id"),
              (lambda: sc.SetEnvPhysics(np.zeros(n + 1, np.int32)), "env count"),
              (lambda: sc.GetEvalStats(None, physics=2), "empty"), (lambda: sc.GetEvalStats(None, physics=9), "out of range"),
              (lambda: sc.GetEvalStats(None, terrain=3, physics=1), "terrain slot 3")]
    for call, msg in cases:
        with pytest.raises(RuntimeError, match=msg):
            call()
    sc.LoadPhysics(2, [2.0e5, 2.0e3, 0.81, 0.01, 0.0019, 2.0e4, 20.0])      # the largest tolerance the broad phase covers is accepted
    keep = C.c_void_p(np.zeros(1, np.int32).ctypes.data)
    null = C.c_void_p(0)
    for fn, args in [("trl_load_physics", (1, C.c_void_p(np.array(DEFAULT).ctypes.data), 0)), ("trl_set_env_physics", (None, keep, 1)),
                     ("trl_env_physics", (keep, keep, 1)), ("trl_eval_stats_phys", (-1, -1, 0, None, None, None, None))]:
        assert getattr(L, fn)(null, *args) != 0
        assert b"null handle" in L.trl_last_error()
    assert np.array_equal(sc.EnvPhysics()[1], slots)
    run(sc, UPDATES)
    clean = run(mixed(trl, pack, n, settings, slots), UPDATES)
    for e in range(0, n, 5):
        assert_same_env(sc, e, clean, e, 90, "after refusals")
    close(sc, clean)
