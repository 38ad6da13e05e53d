"""Training slots (trl_trainer_create_slot / trl_train_run_slots): one exploration handle trains several policies, one on-device MACE
trainer per policy slot.  The contract is exact: env i on slot p computes what env i of a single-trainer handle of the same pack, seeds
and size computes when that handle's trainer is fed only the tuples of slot p's envs (in env order), and trainer p ends with that
trainer's weights, buffers and counters.  The references below use no new code: a plain exploration handle, Update, GetTuples,
the rows of slot p's envs sorted by env id, AddTuples, ResetTupleBuffer, Train.

  * whole training runs (3 slots: the pack's model, a perturbed model file, a fresh net) under three assignments and the overlapped
    schedule, the serial schedule and 3 env groups; the raptor with 2 slots; training slots beside terrain slots;
  * one trainer without slots == trl_train_run;
  * the moved-env rule of trl_set_env_policy, trl_output_model_slot, destruction orders and every refusal.
tests/test_train_slots_cpu.py runs a miniature of the first on the emulator."""
import ctypes as C
import os

import numpy as np
import pytest

import torch_net  # noqa: F401  (torch before the library: see tests/test_gpu_decide_batches.py)
from test_gpu_policy_slots import assignment, pack_net, perturbed, raptor_mixed_model, write_net

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TERRAIN = os.path.join(ROOT, "tests", "golden", "reference", "data", "terrain")
DT = 1.0 / 30.0
UPDATES = 30
ITERS = 2
# small replay memory / init stage: every trainer leaves the init stage after a few updates and then changes the rollout
TRAINER = dict(replay_mem_size=2000, num_init_samples=300, freeze_target_iters=7)
SCHEDULE = dict(init_exp_rate=0.5, exp_rate=0.2, init_exp_temp=5, exp_temp=0.025, init_exp_base_rate=0.2, exp_base_rate=0.002,
                trainer_num_anneal_iters=40, exp_base_anneal_iters=40, trainer_curriculum_iters=30)


# ------------------------------------------------------------------------------------------------ shared helpers (also the CPU test's)
def start_models(pack, d):
    """slot 0: the pack's model; slot 1: a perturbed copy written to a model file; slot 2: a fresh net (InitFresh)"""
    pert = write_net(os.path.join(d, "dog_perturbed.h5"), perturbed(pack_net(pack), 7))
    return [None, (pert, os.path.splitext(pert)[0] + "_scale.txt"), "fresh"]


def make_trainer(trl, sc, slot, model, p, trainer_kw):
    kw = dict(trainer_kw, seed=10 + p)
    tr = trl.MACETrainer(sc, slot=slot, model=None if model in (None, "fresh") else model, **kw)
    if model == "fresh":
        tr.InitFresh(seed=100 + p)
    return tr


def make_group(trl, pack, n, models, slots, trainer_kw=TRAINER, rng_seed=5, setup=None):
    """one exploration handle with a trainer per slot (models[p] as in start_models), envs assigned by `slots`"""
    sc = trl.ScenarioExpMACE(pack, n, rng_seed=rng_seed)
    if setup:
        setup(sc)
    trs = [make_trainer(trl, sc, p, m, p, trainer_kw) for p, m in enumerate(models)]
    sc.SetEnvPolicy(slots)
    return sc, trs


def make_ref(trl, pack, n, models, p, slots, trainer_kw=TRAINER, rng_seed=5, setup=None):
    """the single-trainer handle of slot p: same pack, size and seeds, slot p's starting model and trainer seed, the envs the group
    handle moved reset"""
    sc = trl.ScenarioExpMACE(pack, n, rng_seed=rng_seed)
    if setup:
        setup(sc)
    tr = make_trainer(trl, sc, 0, models[p], p, trainer_kw)
    moved = np.flatnonzero(np.asarray(slots) != 0)
    if moved.size:
        sc.Reset(moved)
    return sc, tr


def ref_loop(sc, tr, p, slots, schedule, updates, iters):
    """the trl_train_run_slots loop of slot p without new code (annealing from 0, as each trl_train_run_slots call does)"""
    mine = np.asarray(slots) == p
    done = 0
    for _ in range(updates):
        s = schedule(done)
        sc.EnableExplore(True, s["exp_rate"], s["exp_temp"], s["exp_base_rate"])
        sc.SetTerrainParamsLerp(s["curriculum_phase"])
        sc.Update(DT)
        rows, flags, env = sc.GetTuples(f64=True)
        keep = np.flatnonzero(mine[env])
        keep = keep[np.argsort(env[keep], kind="stable")]
        tr.AddTuples(rows[keep], flags[keep])
        sc.ResetTupleBuffer()
        tr.Train(iters)
        done += iters


def env_record(sc, e, n_out):
    q, qd, tau, c = sc.GetState(e)
    return [q, qd, tau, c, sc.GetCtrl(e), sc.GetNetOut(e, n_out), sc.GetPoliState(e)]


def assert_envs(group, refs, slots, n_out, stride=1, moved=()):
    """env e of `group` == env e of refs[slots[e]].  An env in `moved` changed slots mid-run: its state and controller must match,
    while its last net output, policy state and distance log may still hold what it did on its old slot before the reset"""
    dist, denv = group.GetDistLog()
    logs = [r.GetDistLog() for r in refs]
    for e in range(0, group.num_envs, stride):
        p = int(slots[e])
        fields = list(zip(env_record(group, e, n_out), env_record(refs[p], e, n_out)))
        for k, (a, b) in enumerate(fields[:5] if e in moved else fields):
            assert np.array_equal(a, b), ("env", e, "slot", p, "field", k)
        if e in moved:
            continue
        rd, re = logs[p]
        assert np.array_equal(dist[denv == e], rd[re == e]), ("distance log", e, p)


def assert_trainer(a, b, what):
    ca, cb = a.counters(), b.counters()
    assert ca == cb, (what, ca, cb)
    for name in ("theta", "target", "history", "in_off", "in_scale", "out_off", "out_scale"):
        assert np.array_equal(a.get(name), b.get(name)), (what, name)
    for which in ("critic", "actor", "actor_batch", "last_ids"):
        assert np.array_equal(a.lists(which), b.lists(which)), (what, which)
    ids = np.arange(ca["num"], dtype=np.int32)
    ra, rb = a.rows(ids), b.rows(ids)
    assert np.array_equal(ra[0], rb[0]) and np.array_equal(ra[1], rb[1]), (what, "replay rows")


def close(*objs):
    for o in objs:
        o.close()


# ------------------------------------------------------------------------------------------------ (1) whole training runs
def _schedule_env(monkeypatch, schedule):
    monkeypatch.delenv("TRL_SERIAL_SCHEDULE", raising=False)
    monkeypatch.delenv("TRL_GROUPS", raising=False)
    if schedule == "serial":
        monkeypatch.setenv("TRL_SERIAL_SCHEDULE", "1")
    elif schedule == "groups3":
        monkeypatch.setenv("TRL_GROUPS", "3")


CASES = [("blocks", "overlap"), ("round_robin", "overlap"), ("random", "overlap"), ("random", "serial"), ("round_robin", "groups3")]


@pytest.mark.parametrize("pattern,schedule", CASES)
def test_training_slots_equal_single_trainer_runs(assets, tmp_path, monkeypatch, pattern, schedule):
    import deepterrainrl_b200 as trl
    from deepterrainrl_b200.train import TrainSchedule, train_run_slots
    _schedule_env(monkeypatch, schedule)
    pack = os.path.join(assets, "dog_slopes_mixed.trlpack")
    n = 2048
    models = start_models(pack, str(tmp_path))
    slots = assignment(pattern, n, 3, seed=1)
    sched = TrainSchedule(**SCHEDULE)
    group, trs = make_group(trl, pack, n, models, slots)
    train_run_slots(trs, sched, UPDATES, ITERS)
    refs = []
    for p in range(3):
        sc, tr = make_ref(trl, pack, n, models, p, slots)
        ref_loop(sc, tr, p, slots, sched, UPDATES, ITERS)
        refs.append((sc, tr))
    for p in range(3):
        c = trs[p].counters()
        assert c["stage"] == 1 and c["iter"] > 0, ("slot", p, "left the init stage", c)
        assert_trainer(trs[p], refs[p][1], "slot %d" % p)
    assert_envs(group, [r[0] for r in refs], slots, 90)
    assert group.GetEvalStats(1)["cycles"] == sum(int(refs[1][0].GetCtrl(int(e))[-2]) for e in np.flatnonzero(slots == 1))
    close(*trs, group, *[o for r in refs for o in r])


def test_raptor_two_training_slots(assets, tmp_path):
    import deepterrainrl_b200 as trl
    from deepterrainrl_b200.train import TrainSchedule, train_run_slots
    pack = os.path.join(assets, "raptor_narrow_gaps.trlpack")
    n = 1000
    models = [None, raptor_mixed_model(str(tmp_path))]
    slots = assignment("random", n, 2, seed=3)
    sched = TrainSchedule(**SCHEDULE)
    group, trs = make_group(trl, pack, n, models, slots)
    train_run_slots(trs, sched, 20, ITERS)
    refs = []
    for p in range(2):
        sc, tr = make_ref(trl, pack, n, models, p, slots)
        ref_loop(sc, tr, p, slots, sched, 20, ITERS)
        refs.append((sc, tr))
    for p in range(2):
        assert_trainer(trs[p], refs[p][1], "raptor slot %d" % p)
    assert_envs(group, [r[0] for r in refs], slots, 87, stride=3)
    close(*trs, group, *[o for r in refs for o in r])


def test_one_trainer_without_slots_is_train_run(assets):
    import deepterrainrl_b200 as trl
    from deepterrainrl_b200.train import TrainSchedule, train_run_slots
    pack = os.path.join(assets, "dog_slopes_mixed.trlpack")
    n = 2048
    sched = TrainSchedule(**SCHEDULE)
    sp = np.array([sched.p[k] for k in TrainSchedule.KEYS], float)
    a = trl.ScenarioExpMACE(pack, n, rng_seed=9)
    ta = trl.MACETrainer(a, seed=3, **TRAINER)
    assert ta.L.trl_train_run(ta.h, sp.ctypes.data_as(C.c_void_p), UPDATES, ITERS, 32, C.c_double(DT)) == 0
    b = trl.ScenarioExpMACE(pack, n, rng_seed=9)
    tb = trl.MACETrainer(b, seed=3, **TRAINER)
    train_run_slots([tb], sched, UPDATES, ITERS)
    assert ta.counters()["stage"] == 1
    assert_trainer(ta, tb, "k = 1")
    assert np.array_equal(np.stack(a.GetStateAll()), np.stack(b.GetStateAll()))
    assert_envs(b, [a], np.zeros(n, int), 90, stride=7)
    close(ta, tb, a, b)


def test_training_slots_with_terrain_slots(assets, tmp_path):
    """2 policies x 2 terrains in one handle against the two single-trainer handles of the same terrain assignment"""
    import deepterrainrl_b200 as trl
    from deepterrainrl_b200.train import TrainSchedule, train_run_slots
    pack = os.path.join(assets, "dog_slopes_mixed.trlpack")
    n = 1024
    models = start_models(pack, str(tmp_path))[:2]
    slots = assignment("round_robin", n, 2)
    terr = (np.arange(n) // 2) % 2          # every (policy, terrain) cell is a quarter of the envs

    def setup(sc):
        sc.LoadTerrain(1, os.path.join(TERRAIN, "narrow_gaps.txt"))
        sc.SetEnvTerrain(terr)
        sc.SetRandSeed(np.arange(1, n + 1, dtype=np.uint64))

    sched = TrainSchedule(**SCHEDULE)
    group, trs = make_group(trl, pack, n, models, slots, setup=setup)
    train_run_slots(trs, sched, UPDATES, ITERS)
    refs = []
    for p in range(2):
        sc, tr = make_ref(trl, pack, n, models, p, slots, setup=setup)
        ref_loop(sc, tr, p, slots, sched, UPDATES, ITERS)
        refs.append((sc, tr))
    for p in range(2):
        assert_trainer(trs[p], refs[p][1], "slot %d" % p)
        for t in range(2):
            on = np.flatnonzero((slots == p) & (terr == t))
            assert group.GetEvalStats(p, terrain=t)["cycles"] == sum(int(refs[p][0].GetCtrl(int(e))[-2]) for e in on)
    assert_envs(group, [r[0] for r in refs], slots, 90, stride=3)
    assert np.array_equal(group.EnvTerrain()[0], terr)
    close(*trs, group, *[o for r in refs for o in r])


# ------------------------------------------------------------------------------------------------ (2) moving envs between slots
def test_moved_envs_restart_and_match_references(assets, tmp_path):
    import deepterrainrl_b200 as trl
    from deepterrainrl_b200.train import TrainSchedule, train_run_slots
    pack = os.path.join(assets, "dog_slopes_mixed.trlpack")
    n = 1024
    models = start_models(pack, str(tmp_path))[:2]
    slots = assignment("blocks", n, 2)
    sched = TrainSchedule(**SCHEDULE)
    group, trs = make_group(trl, pack, n, models, slots)
    refs = [make_ref(trl, pack, n, models, p, slots) for p in range(2)]
    train_run_slots(trs, sched, 15, ITERS)
    for p, (sc, tr) in enumerate(refs):
        ref_loop(sc, tr, p, slots, sched, 15, ITERS)
    # further updates without a hand-over leave tuples in the block (the envs' cycles end in bursts, so it may take a few): moving
    # envs now would attribute them to the wrong trainer
    for _ in range(20):
        group.Update(DT)
        for sc, _ in refs:
            sc.Update(DT)
        if group.GetNumTuples() > 0:
            break
    assert group.GetNumTuples() > 0
    moved = np.arange(0, n, 5)
    new = slots.copy()
    new[moved] = 1 - new[moved]
    with pytest.raises(RuntimeError, match="tuple block holds"):
        group.SetEnvPolicy(new)
    group.ResetTupleBuffer()
    group.SetEnvPolicy(new)
    assert np.array_equal(group.EnvPolicy(), new)
    for sc, _ in refs:
        sc.ResetTupleBuffer()
        sc.Reset(moved)
    train_run_slots(trs, sched, 15, ITERS)
    for p, (sc, tr) in enumerate(refs):
        ref_loop(sc, tr, p, new, sched, 15, ITERS)
    for p in range(2):
        assert_trainer(trs[p], refs[p][1], "slot %d after the move" % p)
    assert_envs(group, [r[0] for r in refs], new, 90, stride=3, moved=set(moved.tolist()))
    close(*trs, group, *[o for r in refs for o in r])


# ------------------------------------------------------------------------------------------------ (3) output, destruction, refusals
def test_output_model_slot_round_trips(assets, tmp_path):
    import deepterrainrl_b200 as trl
    from deepterrainrl_b200.train import TrainSchedule, train_run_slots
    pack = os.path.join(assets, "dog_slopes_mixed.trlpack")
    n = 512
    models = start_models(pack, str(tmp_path))
    group, trs = make_group(trl, pack, n, models, assignment("round_robin", n, 3))
    train_run_slots(trs, TrainSchedule(**SCHEDULE), 20, ITERS)
    for p in (1, 2):
        path = str(tmp_path / ("slot%d.h5" % p))
        group.OutputModel(path, mtime=7, slot=p)
        a = trl.ScenarioPoliEval(pack, 64, rng_seed=3)
        a.LoadModel(path)
        b = trl.ScenarioPoliEval(pack, 64, rng_seed=3)
        blobs = trs[p].blobs()
        b.SetWeights([x for k in blobs for x in blobs[k]], *[trs[p].get(v) for v in ("in_off", "in_scale", "out_off", "out_scale")])
        for sc in (a, b):
            for _ in range(3):
                sc.Update(DT)
        for e in range(64):
            assert np.array_equal(a.GetNetOut(e, 90), b.GetNetOut(e, 90)), (p, e)
        close(a, b)
    # an evaluation slot writes its model too
    ev = trl.ScenarioPoliEval(pack, 8)
    ev.LoadPolicy(1, *models[1])
    ev.OutputModel(str(tmp_path / "eval1.h5"), slot=1)
    with pytest.raises(RuntimeError, match="empty"):
        ev.OutputModel(str(tmp_path / "eval2.h5"), slot=2)
    close(ev, *trs, group)


def test_destruction_in_either_order(assets, tmp_path):
    import deepterrainrl_b200 as trl
    from deepterrainrl_b200.train import TrainSchedule, train_run_slots
    pack = os.path.join(assets, "dog_slopes_mixed.trlpack")
    n = 256
    models = start_models(pack, str(tmp_path))[:2]
    slots = assignment("round_robin", n, 2)
    # trainers first: slot 1 keeps the trained net, and the scenario goes on evaluating it
    group, trs = make_group(trl, pack, n, models, slots)
    train_run_slots(trs, TrainSchedule(**SCHEDULE), 10, ITERS)
    theta1 = trs[1].get("theta")
    out = str(tmp_path / "kept.h5")
    trs[1].close()
    group.OutputModel(out, slot=1)
    from deepterrainrl_b200.model_io import read_model
    from deepterrainrl_b200.trainer import NET_LAYERS
    net = read_model(out)
    flat = np.concatenate([np.asarray(x).ravel() for k in NET_LAYERS for x in net[0][k]])
    assert np.array_equal(flat, theta1)
    trs[0].close()
    group.Update(DT)
    group.Sync()
    group.close()
    # scenario first: the trainers become inert shells
    group, trs = make_group(trl, pack, n, models, slots)
    group.close()
    for tr in trs:
        with pytest.raises(RuntimeError, match="destroyed"):
            tr.Train(1)
        tr.close()


def test_refusals(assets, tmp_path):
    import deepterrainrl_b200 as trl
    from deepterrainrl_b200.train import TrainSchedule, train_run_slots
    pack = os.path.join(assets, "dog_slopes_mixed.trlpack")
    n = 256
    models = start_models(pack, str(tmp_path))[:2]
    sched = TrainSchedule(**SCHEDULE)
    raptor_model = raptor_mixed_model(str(tmp_path))      # another character: another net topology
    # evaluation handles: no training slot; slot 0 refused beside trl_load_policy slots
    ev = trl.ScenarioPoliEval(pack, n)
    with pytest.raises(RuntimeError, match="exploration handles"):
        trl.MACETrainer(ev, slot=1, **TRAINER)
    ev.LoadPolicy(1, *models[1])
    with pytest.raises(RuntimeError, match="policy slots"):
        trl.MACETrainer(ev, **TRAINER)
    ev.close()
    sc, trs = make_group(trl, pack, n, models, assignment("blocks", n, 2))
    before = sc.EnvPolicy().copy()
    for call, msg in [(lambda: trl.MACETrainer(sc, slot=1, **TRAINER), "already has a trainer"),
                      (lambda: trl.MACETrainer(sc, slot=0, **TRAINER), "already attached"),
                      (lambda: trl.MACETrainer(sc, slot=8, **TRAINER), "out of range"),
                      (lambda: trl.MACETrainer(sc, slot=-1, **TRAINER), "out of range"),
                      (lambda: trl.MACETrainer(sc, slot=2, model=raptor_model, **TRAINER), "MACE topology|entries"),
                      (lambda: train_run_slots(trs, sched, 1, 0), "iters_per_update"),
                      (lambda: train_run_slots([trs[0], trs[0]], sched, 1, 1), "twice"),
                      (lambda: trs[1]._ck(trs[1].L.trl_trainer_set_async(trs[1].h, 1)), "training slots"),
                      (lambda: trs[0]._ck(trs[0].L.trl_train_run(trs[0].h, np.zeros(9).ctypes.data_as(C.c_void_p), 1, 1, 32,
                                                                  C.c_double(DT))), "training slots")]:
        with pytest.raises(RuntimeError, match=msg):
            call()
    L = trs[0].L
    arr = (C.c_void_p * 2)(trs[0].h.value, trs[1].h.value)
    assert L.trl_train_run_slots(arr, 0, np.zeros(9).ctypes.data_as(C.c_void_p), 1, 1, C.c_double(DT)) != 0
    other, otr = make_group(trl, pack, 64, models[:1], np.zeros(64, int))
    arr = (C.c_void_p * 2)(trs[0].h.value, otr[0].h.value)
    assert L.trl_train_run_slots(arr, 2, np.zeros(9).ctypes.data_as(C.c_void_p), 1, 1, C.c_double(DT)) != 0
    assert b"different handles" in L.trl_last_error()
    with pytest.raises(ValueError, match="no trainer"):
        train_run_slots([], sched, 1, 1)
    assert np.array_equal(sc.EnvPolicy(), before)
    # the handle is unchanged: it still trains exactly as a fresh one
    clean, ctrs = make_group(trl, pack, n, models, assignment("blocks", n, 2))
    train_run_slots(trs, sched, 8, ITERS)
    train_run_slots(ctrs, sched, 8, ITERS)
    for p in range(2):
        assert_trainer(trs[p], ctrs[p], "after refusals, slot %d" % p)
    close(*otr, other, *trs, *ctrs, sc, clean)
    # the TRL_DECIDE_V1 build has no slots
    os.environ["TRL_DECIDE_V1"] = "1"
    try:
        v1 = trl.ScenarioExpMACE(pack, 64)
        with pytest.raises(RuntimeError, match="TRL_DECIDE_V1"):
            trl.MACETrainer(v1, slot=1, **TRAINER)
        v1.close()
    finally:
        del os.environ["TRL_DECIDE_V1"]
