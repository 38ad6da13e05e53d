"""Evaluation envs (trl_set_env_eval): some envs of an exploration handle evaluate their policy slot's current net while the slot's trainer
goes on training from the other envs.  The contract is exact, and the references below use no new code:

  (1) an exploring env i computes what env i of a single-trainer exploration handle computes when that handle's trainer is fed only the
      tuples of slot p's exploring envs (in env order), and trainer p ends with that trainer's state;
  (2) an evaluating env j on slot p computes what env j of an evaluation handle computes whose net is set, before every update, to the
      net trainer p holds then -- every state plane but the counter-RNG position, the distance log and the episode statistics.

The group handle is driven one update per call, so (2) can read each trainer's net between updates.

  * dog with one trainer (trl_train_run) and with 3 training slots, raptor with 2 slots; evaluation envs every 4th env, in a block,
    at random and a single env; the overlapped schedule, the serial schedule and 3 env groups;
  * evaluation envs beside terrain and physics slots, with every trl_eval_stats_mode cell;
  * the next-reset rule across trl_update (no unassigned env switches), trl_reset and trl_seed_terrain; explore -> evaluate ->
    explore; I_EXP_FLAGS;
  * a checkpoint with evaluation envs resumed bit for bit; every refusal.
tests/test_eval_envs_cpu.py runs a miniature on the emulator."""
import ctypes as C
import os

import numpy as np
import pytest

import torch_net  # noqa: F401  (torch before the library: see tests/test_gpu_decide_batches.py)
from test_gpu_phys_slots import setting
from test_gpu_policy_slots import assignment, raptor_mixed_model
from test_gpu_terrain_slots import tip_over
from test_gpu_train_schedules import schedules as own_schedules
from test_gpu_train_slots import TRAINER, _schedule_env, assert_trainer, close, env_record, make_trainer, start_models

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TERRAIN = os.path.join(ROOT, "tests", "golden", "reference", "data", "terrain")
DT = 1.0 / 30.0
ITERS = 2
SCHEDULE = dict(init_exp_rate=0.5, exp_rate=0.2, init_exp_temp=5, exp_temp=0.025, init_exp_base_rate=0.2, exp_base_rate=0.002,
                trainer_num_anneal_iters=40, exp_base_anneal_iters=40, trainer_curriculum_iters=30)
POLI_EVAL, EXPLORE = 0, 1


def eval_mask(pattern, n, seed=0):
    """which envs evaluate: every 4th, a contiguous block, random, a single env"""
    if pattern == "every4":
        return np.arange(n) % 4 == 1
    if pattern == "block":
        return (np.arange(n) >= n // 3) & (np.arange(n) < n // 3 + n // 5)
    if pattern == "random":
        return np.random.default_rng(seed).uniform(size=n) < 0.3
    if pattern == "single":
        return np.arange(n) == n // 2 + 1
    raise ValueError(pattern)


def net_of(tr):
    blobs = tr.blobs()
    return [x for k in blobs for x in blobs[k]], *[tr.get(v) for v in ("in_off", "in_scale", "out_off", "out_scale")]


class Run:
    """the group handle (trainers on slots, evaluation envs `ev`), and for every slot p the single-trainer exploration reference and
    the evaluation reference; step() advances all of them by one update.

    schedules: one TrainSchedule per slot.  paced: trainers paced by their own tuples (one iteration per 32, the remainder carried
    inside a call), else ITERS iterations per update in lock-step.  single_trainer_run: the one trainer through trl_train_run, else
    every trainer through train_run_slots.  Before the updates in `tips`, the envs in `tip` (every evaluating env and every 8th env)
    are tipped over in the group and in their references, so that evaluating and exploring episodes end in falls inside the window."""

    def __init__(self, trl, pack, n, models, slots, ev, setup=None, rng_seed=5, single_trainer_run=False, trainer_kw=TRAINER,
                 schedules=None, paced=False, tips=()):
        from deepterrainrl_b200.train import TrainSchedule
        self.trl, self.slots, self.ev, self.K = trl, np.asarray(slots), np.asarray(ev, bool), len(models)
        self.scheds = schedules or [TrainSchedule(**SCHEDULE)] * self.K
        self.paced, self.single, self.tips, self.u = paced, single_trainer_run, set(tips), 0
        self.shared = schedules is None        # one schedule object: trl_train_run_slots (or trl_train_run)
        self.tip = (np.arange(n) % 8 == 0) | self.ev
        moved = np.flatnonzero(self.slots != 0)
        g = trl.ScenarioExpMACE(pack, n, rng_seed=rng_seed)
        if setup:
            setup(g)
        self.trs = [make_trainer(trl, g, p, m, p, trainer_kw) for p, m in enumerate(models)]
        if self.K > 1:
            g.SetEnvPolicy(self.slots)
        g.SetEnvEval(self.ev.astype(np.int32))
        g.Reset()
        self.g = g
        self.refs, self.evs = [], []
        for p in range(self.K):
            sc = trl.ScenarioExpMACE(pack, n, rng_seed=rng_seed)
            if setup:
                setup(sc)
            tr = make_trainer(trl, sc, 0, models[p], p, trainer_kw)
            if moved.size:
                sc.Reset(moved)
            sc.Reset()
            self.refs.append((sc, tr))
            e = trl.ScenarioPoliEval(pack, n, rng_seed=rng_seed)
            if setup:
                setup(e)
            if moved.size:
                e.Reset(moved)
            e.Reset()
            self.evs.append(e)

    def step(self):
        from deepterrainrl_b200.train import train_run_slots
        if self.u in self.tips:
            tip_over(self.g, np.flatnonzero(self.tip))
            for p in range(self.K):
                mine = self.tip & (self.slots == p)
                tip_over(self.refs[p][0], np.flatnonzero(mine & ~self.ev))
                tip_over(self.evs[p], np.flatnonzero(mine & self.ev))
        self.u += 1
        # the evaluation references get the net each trainer holds before this update, and the terrain blend of its schedule
        for p in range(self.K):
            it = self.trs[p].counters()["iter"] if self.paced else 0
            self.evs[p].SetWeights(*net_of(self.trs[p]))
            self.evs[p].SetTerrainParamsLerp(self.scheds[p](it)["curriculum_phase"])
        if self.single:
            sp = np.array([self.scheds[0].p[k] for k in type(self.scheds[0]).KEYS], float)
            tr = self.trs[0]
            rc = tr.L.trl_train_run(tr.h, sp.ctypes.data_as(C.c_void_p), 1, 0 if self.paced else ITERS, 32, C.c_double(DT))
            assert rc == 0, tr.L.trl_last_error()
        else:
            train_run_slots(self.trs, self.scheds[0] if self.shared else self.scheds, 1, None if self.paced else ITERS)
        for p, (sc, tr) in enumerate(self.refs):
            c = tr.counters()
            s = self.scheds[p](c["iter"] if self.paced else 0)
            sc.EnableExplore(True, s["exp_rate"], s["exp_temp"], s["exp_base_rate"])
            sc.SetTerrainParamsLerp(s["curriculum_phase"])
            sc.Update(DT)
            rows, flags, env = sc.GetTuples(f64=True)
            mine = (self.slots == p) & ~self.ev
            keep = np.flatnonzero(mine[env])
            keep = keep[np.argsort(env[keep], kind="stable")]
            tr.AddTuples(rows[keep], flags[keep])
            sc.ResetTupleBuffer()
            k = (tr.counters()["total"] - c["total"]) // 32 if self.paced else ITERS      # pacing counts recorded tuples only
            if k > 0:
                tr.Train(k)
            self.evs[p].Update(DT)

    def check(self, n_out, stride=1, falls=True):
        g = self.g
        for p in range(self.K):
            assert_trainer(self.trs[p], self.refs[p][1], "slot %d" % p)
        dist, denv = g.GetDistLog()
        logs = [e.GetDistLog() for e in self.evs]
        assert set(denv.tolist()) <= set(np.flatnonzero(self.ev).tolist()), "only evaluating envs log distances"
        for e in range(0, g.num_envs, stride):
            p = int(self.slots[e])
            ref = self.evs[p] if self.ev[e] else self.refs[p][0]
            for k, (a, b) in enumerate(zip(env_record(g, e, n_out), env_record(ref, e, n_out))):
                assert np.array_equal(a, b), ("env", e, "slot", p, "evaluates", bool(self.ev[e]), "field", k)
            if self.ev[e]:
                rd, re = logs[p]
                assert np.array_equal(dist[denv == e], rd[re == e]), ("distance log", e, p)
        assert np.array_equal(g.EnvEval()[0], self.ev)
        if not falls:
            return
        # the evaluating episodes ended in falls inside the window: every slot with evaluating envs logged distances, and the per-slot
        # statistics (cycles, episodes, mean distance over the logged distances) are the references'
        for p in range(self.K):
            if not (self.ev & (self.slots == p)).any():
                continue
            st = g.GetEvalStats(p, mode=POLI_EVAL)
            c, e, ds = expected_cell(self, POLI_EVAL, p)
            assert e > 0 and np.isin(denv, np.flatnonzero(self.slots == p)).any(), ("no evaluating episode ended", p)
            assert (st["cycles"], st["episodes"]) == (c, e), p
            assert abs(st["avg_dist"] - ds / e) <= 1e-12 * (1 + abs(ds / e)), p
        # the exploring envs fell too, and recorded their fail tuples instead of distances
        assert g.GetEvalStats(None, mode=EXPLORE)["episodes"] == 0

    def close(self):
        close(*self.trs, self.g, *[o for r in self.refs for o in r], *self.evs)


def expected_cell(run, mode, p, t_of=None, t=-1, q_of=None, q=-1):
    """trl_eval_stats_mode(mode, p, t, q) from the references' own envs: cycles, episodes and the sum of logged distances"""
    c = e = 0
    ds = 0.0
    for env in range(run.g.num_envs):
        if (mode == POLI_EVAL) != bool(run.ev[env]) or (p >= 0 and run.slots[env] != p):
            continue
        if t >= 0 and t_of[env] != t or q >= 0 and q_of[env] != q:
            continue
        ref = run.evs[run.slots[env]] if run.ev[env] else run.refs[run.slots[env]][0]
        ctrl = ref.GetCtrl(env)
        dist, denv = ref.GetDistLog()
        mine = dist[denv == env]
        c += int(ctrl[-2]); e += mine.size; ds += float(mine.sum())
    return c, e, ds


# ------------------------------------------------------------------------------------------------ (1) + (2) whole runs
CASES = [("every4", "overlap"), ("block", "overlap"), ("random", "serial"), ("single", "groups3"), ("random", "groups3")]
UPDATES = 36
TIPS = (14, 26)          # an evaluating env has finished a cycle by then, so its fall logs a distance


@pytest.mark.parametrize("pattern,schedule", CASES)
@pytest.mark.parametrize("paced", [False, True], ids=["fixed", "paced"])
def test_one_trainer_train_run(assets, monkeypatch, pattern, schedule, paced):
    import deepterrainrl_b200 as trl
    _schedule_env(monkeypatch, schedule)
    pack = os.path.join(assets, "dog_slopes_mixed.trlpack")
    n = 1024
    run = Run(trl, pack, n, [None], np.zeros(n, np.int32), eval_mask(pattern, n, seed=2), single_trainer_run=True, paced=paced, tips=TIPS)
    for _ in range(UPDATES):
        run.step()
    run.check(90)
    st = run.g.GetEvalStats(None, mode=POLI_EVAL)
    ex = run.g.GetEvalStats(None, mode=EXPLORE)
    assert ex["steps"] + st["steps"] == run.g.GetEvalStats(None)["steps"]
    run.close()


@pytest.mark.parametrize("pattern,schedule", CASES)
@pytest.mark.parametrize("mode", ["shared", "own", "paced"])
def test_three_training_slots(assets, tmp_path, monkeypatch, pattern, schedule, mode):
    """one schedule for all slots, each slot on its own schedule in lock-step (trl_train_run_slots_sched), and each paced by its own
    tuples on its own schedule"""
    import deepterrainrl_b200 as trl
    _schedule_env(monkeypatch, schedule)
    pack = os.path.join(assets, "dog_slopes_mixed.trlpack")
    n = 1536
    scheds = None if mode == "shared" else own_schedules(curriculum=0 if mode == "paced" else None)
    run = Run(trl, pack, n, start_models(pack, str(tmp_path)), assignment("random", n, 3, seed=4), eval_mask(pattern, n, seed=5),
              schedules=scheds, paced=mode == "paced", tips=TIPS)
    for _ in range(UPDATES):
        run.step()
    run.check(90)
    run.close()


def test_raptor_two_slots(assets, tmp_path):
    import deepterrainrl_b200 as trl
    pack = os.path.join(assets, "raptor_narrow_gaps.trlpack")
    n = 800
    run = Run(trl, pack, n, [None, raptor_mixed_model(str(tmp_path))], assignment("random", n, 2, seed=3), eval_mask("every4", n),
              tips=TIPS)
    for _ in range(UPDATES):
        run.step()
    run.check(87, stride=3)
    run.close()


def test_beside_terrain_and_physics_slots(assets, tmp_path):
    import deepterrainrl_b200 as trl
    pack = os.path.join(assets, "dog_slopes_mixed.trlpack")
    n = 768
    terr = np.arange(n) % 2
    phys = (np.arange(n) // 2) % 2
    p1, _ = setting(mu=0.3, kn=5e4, dn=5e2)

    def ev_setup(sc):
        sc.LoadTerrain(1, os.path.join(TERRAIN, "mixed.txt"))
        sc.SetEnvTerrain(terr)
        sc.LoadPhysics(1, p1)
        sc.SetEnvPhysics(phys)
        sc.Reset()

    models = start_models(pack, str(tmp_path))[:2]
    run = Run(trl, pack, n, models, assignment("blocks", n, 2), eval_mask("random", n, seed=9), setup=ev_setup, tips=TIPS)
    for _ in range(UPDATES):
        run.step()
    run.check(90, stride=2)
    g = run.g
    for mode in (POLI_EVAL, EXPLORE):
        for p in (-1, 0, 1):
            for t in (-1, 0, 1):
                for q in (-1, 0, 1):
                    st = g.GetEvalStats(None if p < 0 else p, terrain=None if t < 0 else t, physics=None if q < 0 else q, mode=mode)
                    c, e, ds = expected_cell(run, mode, p, terr, t, phys, q)
                    assert (st["cycles"], st["episodes"]) == (c, e), (mode, p, t, q)
                    if mode == POLI_EVAL:       # every cell holds evaluating envs, and some of their episodes ended
                        assert e > 0, (p, t, q)
                        assert abs(st["avg_dist"] - ds / e) <= 1e-12 * (1 + abs(ds / e)), (mode, p, t, q)
                    else:
                        assert e == 0 and st["avg_dist"] == 0.0, (p, t, q)
    # mode -1 is trl_eval_stats_phys
    for p, t, q in [(-1, -1, -1), (0, 1, 0), (1, 0, 1)]:
        a = C.c_int64(0), C.c_int64(0), C.c_double(0), C.c_int64(0)
        b = C.c_int64(0), C.c_int64(0), C.c_double(0), C.c_int64(0)
        assert g.L.trl_eval_stats_mode(g.h, -1, p, t, q, *[C.byref(x) for x in a]) == 0
        assert g.L.trl_eval_stats_phys(g.h, p, t, q, *[C.byref(x) for x in b]) == 0
        assert [x.value for x in a] == [x.value for x in b]
    run.close()


# ------------------------------------------------------------------------------------------------ the mode rule
def test_next_reset_rule_and_round_trip(assets):
    import deepterrainrl_b200 as trl
    pack = os.path.join(assets, "dog_slopes_mixed.trlpack")
    n = 512
    idx = np.arange(n)
    g = trl.ScenarioExpMACE(pack, n, rng_seed=3)
    g.EnableExplore(True, 0.2, 0.025, 0.01)
    for _ in range(30):                                          # exploring episodes with a few cycles each
        g.Update(DT)
    cur, nxt = g.EnvEval()
    assert not cur.any() and not nxt.any()
    flags = idx % 2 == 0
    g.SetEnvEval(flags.astype(np.int32))
    cur, nxt = g.EnvEval()
    assert not cur.any() and np.array_equal(nxt, flags)         # nothing happens before a reset
    # a fall inside trl_update: the tipped envs fall at the end of the next update, and only the flagged ones switch.  An exploring
    # env whose fall meets a cycle boundary resets at a later end of update (cScenarioExp), and a few tipped bodies roll back under
    # the root-angle bound and fall later by contact, so most (not all) tipped flagged envs have switched a few updates on
    tipped = idx % 4 < 2
    cycles_before = np.array([g.GetCtrl(int(e))[-2] for e in idx])
    tip_over(g, idx[tipped])
    g.Update(DT)
    cur, nxt = g.EnvEval()
    assert np.array_equal(nxt, flags)
    assert cur.any() and not (cur & ~flags).any() and not (cur & ~tipped).any()
    # entering evaluation restarts the cycle count the exploring episode kept
    assert (cycles_before[cur] > 0).any()
    assert all(g.GetCtrl(int(e))[-2] == 0 for e in idx[cur])
    for _ in range(3):
        g.Update(DT)
    cur, _ = g.EnvEval()
    assert cur[tipped & flags].mean() > 0.9 and not (cur & ~flags).any()
    switched = cur.copy()
    g.Reset(idx[idx % 8 == 2].astype(np.int32))                   # trl_reset switches the flagged envs it resets
    cur, _ = g.EnvEval()
    assert np.array_equal(cur, switched | ((idx % 8 == 2) & flags))
    g.SetRandSeed(np.arange(n, dtype=np.uint64) + 1)             # trl_seed_terrain resets every env
    assert np.array_equal(g.EnvEval()[0], flags)
    # evaluating envs: exploration off, no tuples, distances logged at their falls
    g.ResetTupleBuffer()
    g.ResetAvgDist()
    for u in range(40):
        if u in (14, 28):
            tip_over(g, idx[flags & (idx % 4 == 0)])
        g.Update(DT)
    _, _, env = g.GetTuples(f64=True)
    assert env.size and not flags[env].any()
    for e in idx[flags][:64]:
        ctrl = g.GetCtrl(int(e))
        assert ctrl[-4] == 0 and ctrl[-3] == 0, e                 # I_EXP_FLAGS critic / actor bits
    dist, denv = g.GetDistLog()
    assert denv.size > 0 and flags[denv].all()
    st = g.GetEvalStats(None, mode=POLI_EVAL)
    assert st["episodes"] == denv.size and st["cycles"] > 0
    assert abs(st["avg_dist"] - dist.mean()) <= 1e-12 * (1 + abs(dist.mean()))
    assert g.GetEvalStats(None, mode=EXPLORE)["episodes"] == 0
    d0, e0 = g.GetDistLog(mode=POLI_EVAL)
    assert np.array_equal(d0, dist) and np.array_equal(e0, denv)
    # back to exploring: tuples again, the distance log keeps only the evaluating episodes (filtered by the present mode, none now)
    g.SetEnvEval(np.zeros(n, np.int32))
    g.Reset()
    assert not g.EnvEval()[0].any()
    g.ResetTupleBuffer()
    for _ in range(30):
        g.Update(DT)
    _, _, env = g.GetTuples(f64=True)
    assert flags[env].any()
    d2, e2 = g.GetDistLog()
    assert d2.size and np.array_equal(d2, dist) and np.array_equal(e2, denv)
    assert g.GetDistLog(mode=POLI_EVAL)[0].size == 0 and np.array_equal(g.GetDistLog(mode=EXPLORE)[0], dist)
    assert g.GetEvalStats(None, mode=POLI_EVAL)["steps"] == 0
    g.close()


def test_checkpoint_resumes_bit_for_bit(assets, tmp_path):
    import deepterrainrl_b200 as trl
    from deepterrainrl_b200.train import TrainSchedule, train_run_slots
    pack = os.path.join(assets, "dog_slopes_mixed.trlpack")
    n = 768
    models = start_models(pack, str(tmp_path))
    g = trl.ScenarioExpMACE(pack, n, rng_seed=5)
    trs = [make_trainer(trl, g, p, m, p, TRAINER) for p, m in enumerate(models)]
    g.SetEnvPolicy(assignment("round_robin", n, 3))
    g.SetEnvEval((np.arange(n) % 5 == 0).astype(np.int32))
    sched = TrainSchedule(**SCHEDULE)
    train_run_slots(trs, sched, 6, ITERS)
    g.SetEnvEval((np.arange(n) % 7 == 0).astype(np.int32))      # a pending assignment is saved too
    path = str(tmp_path / "eval.ckpt")
    g.SaveCheckpoint(path)
    b, btrs, _ = trl.load_checkpoint(path)
    btrs = [btrs[p] for p in range(3)]
    assert all(np.array_equal(x, y) for x, y in zip(g.EnvEval(), b.EnvEval()))
    train_run_slots(trs, sched, 6, ITERS)
    train_run_slots(btrs, sched, 6, ITERS)
    for p in range(3):
        assert_trainer(trs[p], btrs[p], "slot %d" % p)
    for e in range(0, n, 3):
        assert all(np.array_equal(x, y) for x, y in zip(env_record(g, e, 90), env_record(b, e, 90))), e
    assert all(np.array_equal(x, y) for x, y in zip(g.GetDistLog(), b.GetDistLog()))
    assert g.GetEvalStats(None, mode=POLI_EVAL) == b.GetEvalStats(None, mode=POLI_EVAL)
    close(*trs, *btrs, g, b)


def test_refusals(assets, monkeypatch):
    import deepterrainrl_b200 as trl
    from deepterrainrl_b200.parallel import _Collectives
    pack = os.path.join(assets, "dog_slopes_mixed.trlpack")
    n = 64

    def unchanged(sc, cur, nxt):
        a, b = sc.EnvEval()
        return np.array_equal(a, cur) and np.array_equal(b, nxt)

    zero = np.zeros(n, bool)
    ev = trl.ScenarioPoliEval(pack, n)
    with pytest.raises(RuntimeError, match="evaluation handle"):
        ev.SetEnvEval([1])
    assert ev.EnvEval()[0].all() and ev.EnvEval()[1].all()
    # a scene without a policy net
    flat = trl.ScenarioExpMACE(os.path.join(assets, "dog_flat.trlpack"), n)
    with pytest.raises(RuntimeError, match="policy net"):
        flat.SetEnvEval([1])
    assert unchanged(flat, zero, zero)
    # the TRL_DECIDE_V1 build
    monkeypatch.setenv("TRL_DECIDE_V1", "1")
    v1 = trl.ScenarioExpMACE(pack, n)
    monkeypatch.delenv("TRL_DECIDE_V1")
    with pytest.raises(RuntimeError, match="TRL_DECIDE_V1"):
        v1.SetEnvEval([1])
    assert unchanged(v1, zero, zero)
    # a handle with a communicator (a single-rank one whose collectives are memory copies)
    cm = trl.ScenarioExpMACE(pack, n)

    def all_gather(ctx, send, recv, nbytes, stream):
        C.memmove(recv, send, nbytes)
        return 0
    coll = _Collectives(None, _Collectives.AG(all_gather), _Collectives.BC(lambda ctx, buf, nbytes, root, stream: 0),
                        _Collectives.AR(lambda ctx, buf, count, stream: 0))
    assert cm.L.trl_comm_init_external(cm.h, C.byref(coll), 0, 1) == 0, cm.L.trl_last_error()
    with pytest.raises(RuntimeError, match="communicator"):
        cm.SetEnvEval([1])
    assert unchanged(cm, zero, zero)
    # bad ids and counts, with and without evaluation envs already set
    g = trl.ScenarioExpMACE(pack, n)
    for state in ("none", "set"):
        cur, nxt = g.EnvEval()
        for call, msg in [(lambda: g.SetEnvEval([1], env_ids=[n]), "env id"), (lambda: g.SetEnvEval([1, 1], env_ids=[0, -1]), "env id"),
                          (lambda: g.SetEnvEval(np.ones(n + 1, np.int32)), "env count"), (lambda: g.GetEvalStats(None, mode=2), "mode")]:
            with pytest.raises(RuntimeError, match=msg):
                call()
            assert unchanged(g, cur, nxt), (state, msg)
        if state == "none":
            assert g.GetEvalStats(None, mode=POLI_EVAL)["steps"] == 0        # no evaluation env yet: an empty cell
            g.SetEnvEval([1, 0, 1])
            assert np.array_equal(g.EnvEval()[1][:4], [True, False, True, False])
    # trl_comm_init* refuses a handle with evaluation envs
    assert g.L.trl_comm_init_external(g.h, C.byref(coll), 0, 1) != 0 and b"evaluation envs" in g.L.trl_last_error()
    idb = (C.c_char * 128)()
    if g.L.trl_comm_unique_id(idb) == 0:
        assert g.L.trl_comm_init(g.h, idb, 0, 1) != 0 and b"evaluation envs" in g.L.trl_last_error()
    close(ev, flat, v1, cm, g)
