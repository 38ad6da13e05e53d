"""Per-slot exploration schedules and tuple pacing for training slots (trl_set_explore_slot / trl_train_run_slots_sched).  The
contract extends the one of tests/test_gpu_train_slots.py: env i on slot p computes what env i of a single-trainer handle of the same
pack, seeds and size computes when that handle's trainer is fed only the tuples of slot p's envs, follows slot p's schedule and is paced
as trl_train_run paces its trainer (a fixed count, or one iteration per tuple_buffer_size fresh tuples with the remainder carried).
The references use existing calls only: the helpers of tests/test_gpu_train_slots.py and, for pacing, a host-side mirror of
train_run_impl's arithmetic (ref_loop_paced).

  * three different schedules in lock-step (overlapped schedule, serial schedule, 3 env groups); tuple pacing on slots of 1/2, 1/3
    and 1/6 of the envs, one schedule read from the reference's arg file; the raptor with 2 paced slots;
  * one trainer without slots, paced == trl_train_run(t, sp, U, 0, 32, dt); k identical schedules in lock-step == trl_train_run_slots;
  * trl_set_explore_slot: an unlisted slot keeps its setting, trl_set_explore overwrites every slot, evaluation slots explore as
    single-policy handles; every refusal.
tests/test_train_schedules_cpu.py runs a miniature of the first on the emulator."""
import ctypes as C
import os

import numpy as np
import pytest

import torch_net  # noqa: F401  (torch before the library: see tests/test_gpu_decide_batches.py)
from test_gpu_policy_slots import assignment, raptor_mixed_model
from test_gpu_train_slots import (DT, TRAINER, _schedule_env, assert_envs, assert_trainer, close, make_group, make_ref, ref_loop,
                                  start_models)

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ARGS = os.path.join(ROOT, "tests", "golden", "reference", "args")
UPDATES = 30
ITERS = 2
# three schedules that differ in every exploration entry and anneal length, with one curriculum
SCHEDULES = [dict(init_exp_rate=0.5, exp_rate=0.2, init_exp_temp=5, exp_temp=0.025, init_exp_base_rate=0.2, exp_base_rate=0.002,
                  trainer_num_anneal_iters=40, exp_base_anneal_iters=40, trainer_curriculum_iters=30),
             dict(init_exp_rate=0.9, exp_rate=0.05, init_exp_temp=20, exp_temp=0.5, init_exp_base_rate=0.6, exp_base_rate=0.05,
                  trainer_num_anneal_iters=12, exp_base_anneal_iters=25, trainer_curriculum_iters=30),
             dict(init_exp_rate=0.1, exp_rate=0.4, init_exp_temp=0.5, exp_temp=2.0, init_exp_base_rate=0.01, exp_base_rate=0.3,
                  trainer_num_anneal_iters=70, exp_base_anneal_iters=6, trainer_curriculum_iters=30)]


def schedules(curriculum=None):
    from deepterrainrl_b200.train import TrainSchedule
    out = []
    for s in SCHEDULES:
        s = dict(s)
        if curriculum is not None:
            s["trainer_curriculum_iters"] = curriculum
        out.append(TrainSchedule(**s))
    return out


def ref_loop_paced(sc, tr, p, slots, schedule, updates, tuple_buffer_size=32):
    """train_run_impl's pacing from the host (trl_train_run(t, sp, U, 0, tuple_buffer_size, dt)) on slot p's tuples: the schedule at
    the trainer's iteration counter at the start of each update, last_total before the first one, then (fresh + carry) / size"""
    mine = np.asarray(slots) == p
    last_total, carry = None, 0
    for _ in range(updates):
        c = tr.counters()
        if last_total is None:
            last_total = c["total"]
        s = schedule(c["iter"])
        sc.EnableExplore(True, s["exp_rate"], s["exp_temp"], s["exp_base_rate"])
        sc.SetTerrainParamsLerp(s["curriculum_phase"])
        sc.Update(DT)
        rows, flags, env = sc.GetTuples(f64=True)
        keep = np.flatnonzero(mine[env])
        keep = keep[np.argsort(env[keep], kind="stable")]
        tr.AddTuples(rows[keep], flags[keep])
        sc.ResetTupleBuffer()
        total = tr.counters()["total"]
        k, carry = divmod(total - last_total + carry, tuple_buffer_size)
        last_total = total
        if k > 0:
            tr.Train(k)


def sp_array(scheds):
    from deepterrainrl_b200.train import TrainSchedule
    return np.array([[s.p[k] for k in TrainSchedule.KEYS] for s in scheds], float)


def run_refs(trl, pack, n, models, slots, scheds, loop, updates, trainer_kw=TRAINER, **kw):
    refs = []
    for p in range(len(models)):
        sc, tr = make_ref(trl, pack, n, models, p, slots, trainer_kw=trainer_kw)
        loop(sc, tr, p, slots, scheds[p], updates, **kw)
        refs.append((sc, tr))
    return refs


# ------------------------------------------------------------------------------------------------ (1) lock-step, three schedules
@pytest.mark.parametrize("schedule", ["overlap", "serial", "groups3"])
def test_three_schedules_lock_step(assets, tmp_path, monkeypatch, schedule):
    import deepterrainrl_b200 as trl
    from deepterrainrl_b200.train import train_run_slots
    _schedule_env(monkeypatch, schedule)
    pack = os.path.join(assets, "dog_slopes_mixed.trlpack")
    n = 2048
    models = start_models(pack, str(tmp_path))
    slots = assignment("random", n, 3, seed=11)
    scheds = schedules()
    group, trs = make_group(trl, pack, n, models, slots)
    train_run_slots(trs, scheds, UPDATES, ITERS)
    refs = run_refs(trl, pack, n, models, slots, scheds, lambda sc, tr, p, sl, s, u: ref_loop(sc, tr, p, sl, s, u, ITERS), UPDATES)
    for p in range(3):
        assert trs[p].counters()["stage"] == 1, ("slot", p, "left the init stage")
        assert_trainer(trs[p], refs[p][1], "slot %d" % p)
    assert_envs(group, [r[0] for r in refs], slots, 90)
    close(*trs, group, *[o for r in refs for o in r])


# ------------------------------------------------------------------------------------------------ (2) tuple pacing
def uneven_slots(n, seed):
    """slot 0: half of the envs, slot 1: a third, slot 2: a sixth, scattered"""
    s = np.repeat([0, 1, 2], [n // 2, n // 3, n - n // 2 - n // 3])
    return np.random.default_rng(seed).permutation(s)


def test_tuple_paced_uneven_slots(assets, tmp_path):
    import deepterrainrl_b200 as trl
    from deepterrainrl_b200.train import TrainSchedule, parse_arg_file, train_run_slots
    pack = os.path.join(assets, "dog_slopes_mixed.trlpack")
    n = 1536
    models = start_models(pack, str(tmp_path))
    slots = uneven_slots(n, 3)
    args = parse_arg_file(os.path.join(ARGS, "opt_args_train_mace.txt"))
    # the arg file's trainer, its replay memory and init stage scaled down 500x so that every trainer trains within the run
    kw = dict(TRAINER, replay_mem_size=int(args["trainer_replay_mem_size"]) // 500,
              num_init_samples=int(args["trainer_num_init_samples"]) // 500)
    scheds = schedules(curriculum=0)[:2] + [TrainSchedule.from_args(args)]
    updates = 90
    group, trs = make_group(trl, pack, n, models, slots, trainer_kw=kw)
    train_run_slots(trs, scheds, updates, None, tuple_buffer_size=32)
    refs = run_refs(trl, pack, n, models, slots, scheds, ref_loop_paced, updates, trainer_kw=kw)
    for p in range(3):
        assert_trainer(trs[p], refs[p][1], "paced slot %d" % p)
    counters = [t.counters() for t in trs]
    assert all(c["stage"] == 1 for c in counters), counters
    assert len({c["iter"] for c in counters}) == 3, counters       # the trainers' schedule positions really diverge
    assert_envs(group, [r[0] for r in refs], slots, 90)
    close(*trs, group, *[o for r in refs for o in r])


def test_raptor_two_paced_slots(assets, tmp_path):
    import deepterrainrl_b200 as trl
    from deepterrainrl_b200.train import train_run_slots
    pack = os.path.join(assets, "raptor_narrow_gaps.trlpack")
    n = 1000
    models = [None, raptor_mixed_model(str(tmp_path))]
    slots = assignment("random", n, 2, seed=3)
    scheds = schedules(curriculum=0)[1:]
    group, trs = make_group(trl, pack, n, models, slots)
    train_run_slots(trs, scheds, 80, None)
    refs = run_refs(trl, pack, n, models, slots, scheds, ref_loop_paced, 80)
    for p in range(2):
        assert trs[p].counters()["iter"] > 0
        assert_trainer(trs[p], refs[p][1], "raptor paced slot %d" % p)
    assert_envs(group, [r[0] for r in refs], slots, 87, stride=3)
    close(*trs, group, *[o for r in refs for o in r])


# ------------------------------------------------------------------------------------------------ (3) equivalences
def test_one_paced_trainer_without_slots_is_train_run(assets):
    import deepterrainrl_b200 as trl
    from deepterrainrl_b200.train import train_run_slots
    pack = os.path.join(assets, "dog_slopes_mixed.trlpack")
    n = 2048
    sched = schedules(curriculum=0)[0]
    sp = sp_array([sched])
    a = trl.ScenarioExpMACE(pack, n, rng_seed=9)
    ta = trl.MACETrainer(a, seed=3, **TRAINER)
    assert ta.L.trl_train_run(ta.h, sp.ctypes.data_as(C.c_void_p), UPDATES, 0, 32, C.c_double(DT)) == 0
    b = trl.ScenarioExpMACE(pack, n, rng_seed=9)
    tb = trl.MACETrainer(b, seed=3, **TRAINER)
    train_run_slots([tb], sched, UPDATES, None)
    assert ta.counters()["stage"] == 1
    assert_trainer(ta, tb, "k = 1, paced")
    assert np.array_equal(np.stack(a.GetStateAll()), np.stack(b.GetStateAll()))
    assert_envs(b, [a], np.zeros(n, int), 90, stride=7)
    close(ta, tb, a, b)


def test_identical_schedules_lock_step_is_train_run_slots(assets, tmp_path):
    import deepterrainrl_b200 as trl
    from deepterrainrl_b200.train import train_run_slots
    pack = os.path.join(assets, "dog_slopes_mixed.trlpack")
    n = 1024
    models = start_models(pack, str(tmp_path))
    slots = assignment("round_robin", n, 3)
    sched = schedules()[1]
    a, tas = make_group(trl, pack, n, models, slots)
    train_run_slots(tas, sched, UPDATES, ITERS)                     # one schedule, handle-wide: trl_train_run_slots
    b, tbs = make_group(trl, pack, n, models, slots)
    train_run_slots(tbs, [sched] * 3, UPDATES, ITERS)               # the same schedule per slot: trl_train_run_slots_sched
    for p in range(3):
        assert_trainer(tas[p], tbs[p], "slot %d" % p)
    assert_envs(b, [a] * 3, slots, 90, stride=3)
    close(*tas, *tbs, a, b)


# ------------------------------------------------------------------------------------------------ (4) trl_set_explore_slot
def test_unlisted_slot_keeps_its_setting_until_set_explore(assets, tmp_path):
    """slots 0 and 1 train under their own paced schedules; slot 2 has a trainer that is not listed, so its envs explore with its
    starting net under the fixed setting given to slot 2 alone.  Then trl_set_explore gives every slot one setting."""
    import deepterrainrl_b200 as trl
    from deepterrainrl_b200.train import train_run_slots
    pack = os.path.join(assets, "dog_slopes_mixed.trlpack")
    n = 1536
    models = start_models(pack, str(tmp_path))
    slots = assignment("random", n, 3, seed=8)
    scheds = schedules(curriculum=0)[:2]
    fixed = (0.7, 3.0, 0.25)
    group, trs = make_group(trl, pack, n, models, slots)
    group.EnableExplore(True, *fixed, slot=2)
    train_run_slots(trs[:2], scheds, 20, None)
    refs = run_refs(trl, pack, n, models[:2], slots, scheds, ref_loop_paced, 20)
    fsc, ftr = make_ref(trl, pack, n, models, 2, slots)
    fsc.EnableExplore(True, *fixed)
    for _ in range(20):
        fsc.SetTerrainParamsLerp(1.0)           # the blend of a schedule without curriculum
        fsc.Update(DT)
        fsc.ResetTupleBuffer()
    refs.append((fsc, ftr))
    for p in range(2):
        assert_trainer(trs[p], refs[p][1], "slot %d" % p)
    assert trs[2].counters()["total"] == 0
    assert_envs(group, [r[0] for r in refs], slots, 90, stride=2)
    # one setting for every slot, fixed slot included
    for sc in [group] + [r[0] for r in refs]:
        sc.EnableExplore(True, 0.3, 0.2, 0.05)
        for _ in range(10):
            sc.Update(DT)
            sc.ResetTupleBuffer()
    assert_envs(group, [r[0] for r in refs], slots, 90, stride=2)
    close(*trs, group, *[o for r in refs for o in r])


def test_evaluation_slots_explore_as_single_policy_handles(assets, tmp_path):
    import deepterrainrl_b200 as trl
    pack = os.path.join(assets, "dog_slopes_mixed.trlpack")
    n = 512
    models = start_models(pack, str(tmp_path))
    slots = assignment("random", n, 2, seed=2)
    settings = [(1, 0.6, 2.0, 0.1), (1, 0.05, 0.3, 0.4)]
    ev = trl.ScenarioPoliEval(pack, n, rng_seed=4)
    L = ev.L
    ev.LoadPolicy(1, *models[1])
    ev.SetEnvPolicy(slots)
    for p, (en, r, t, b) in enumerate(settings):
        assert L.trl_set_explore_slot(ev.h, p, en, C.c_double(r), C.c_double(t), C.c_double(b)) == 0
    refs = []
    for p, (en, r, t, b) in enumerate(settings):
        sc = trl.ScenarioPoliEval(pack, n, rng_seed=4)
        if models[p] is not None:
            sc.LoadModel(*models[p])
        assert L.trl_set_explore(sc.h, en, C.c_double(r), C.c_double(t), C.c_double(b)) == 0
        refs.append(sc)
    for sc in [ev] + refs:
        for _ in range(15):
            sc.Update(DT)
    for e in range(n):
        ref = refs[slots[e]]
        assert np.array_equal(ev.GetState(e)[0], ref.GetState(e)[0]), e
        assert np.array_equal(ev.GetCtrl(e), ref.GetCtrl(e)), e
        assert np.array_equal(ev.GetNetOut(e, 90), ref.GetNetOut(e, 90)), e
    close(ev, *refs)


# ------------------------------------------------------------------------------------------------ (5) refusals
def test_refusals(assets, tmp_path):
    import deepterrainrl_b200 as trl
    from deepterrainrl_b200.parallel import _Collectives
    from deepterrainrl_b200.train import train_run_slots
    pack = os.path.join(assets, "dog_slopes_mixed.trlpack")
    n = 256
    models = start_models(pack, str(tmp_path))[:2]
    scheds = schedules(curriculum=0)[:2]
    sc, trs = make_group(trl, pack, n, models, assignment("blocks", n, 2))
    L = sc.L
    arr = lambda ts: (C.c_void_p * len(ts))(*[t.h.value for t in ts])      # noqa: E731
    sp = sp_array(scheds)
    run = lambda ts, spx, ipu, tbs=32: L.trl_train_run_slots_sched(arr(ts), len(ts), spx.ctypes.data_as(C.c_void_p), 1, ipu, tbs,  # noqa: E731
                                                                   C.c_double(DT))
    # trl_set_explore_slot
    assert L.trl_set_explore_slot(None, 0, 1, C.c_double(0.1), C.c_double(0.1), C.c_double(0.1)) != 0
    assert b"null handle" in L.trl_last_error()
    for slot in (-1, 8):
        assert L.trl_set_explore_slot(sc.h, slot, 1, C.c_double(0.1), C.c_double(0.1), C.c_double(0.1)) != 0
        assert b"out of range" in L.trl_last_error()
    # trl_train_run_slots_sched
    on = sp.copy()
    on[:, 8] = 30
    mixed = on.copy()
    mixed[1, 8] = 40
    other, otr = make_group(trl, pack, 64, models[:1], np.zeros(64, int))
    for call, msg in [(lambda: run(trs, sp, -1), b"iters_per_update"),
                      (lambda: run(trs, sp, 0, 0), b"tuple_buffer_size"),
                      (lambda: run(trs, on, 0), b"curriculum"),
                      (lambda: run(trs, mixed, 2), b"trainer_curriculum_iters"),
                      (lambda: run([trs[0], trs[0]], sp, 2), b"twice"),
                      (lambda: run([trs[0], otr[0]], sp, 2), b"different handles"),
                      (lambda: L.trl_train_run_slots_sched(arr(trs), 0, sp.ctypes.data_as(C.c_void_p), 1, 2, 32, C.c_double(DT)),
                       b"at least one")]:
        assert call() != 0 and msg in L.trl_last_error(), (msg, L.trl_last_error())
    with pytest.raises(ValueError, match="schedules for"):
        train_run_slots(trs, scheds[:1], 1, None)
    with pytest.raises(ValueError, match="iters_per_update"):
        train_run_slots(trs, scheds, 1, 0)
    # an asynchronous trainer and a handle with a communicator (a plain single-trainer handle; asynchronous training needs one)
    c = trl.ScenarioExpMACE(pack, 64)
    tc = trl.MACETrainer(c, **TRAINER)

    def all_gather(ctx, send, recv, nbytes, stream):
        C.memmove(recv, send, nbytes)
        return 0
    fns = (_Collectives.AG(all_gather), _Collectives.BC(lambda ctx, buf, nbytes, root, stream: 0), _Collectives.AR(lambda ctx, buf, count, stream: 0))
    coll = _Collectives(None, *fns)
    assert L.trl_comm_init_external(c.h, C.byref(coll), 0, 1) == 0, L.trl_last_error()
    tc._ck(L.trl_trainer_set_async(tc.h, 1))
    assert run([tc], sp[:1], 0) != 0 and b"asynchronous" in L.trl_last_error()
    tc._ck(L.trl_trainer_set_async(tc.h, 0))
    assert run([tc], sp[:1], 0) != 0 and b"communicator" in L.trl_last_error()
    close(tc, c, *otr, other)
    # the handle is unchanged: it still trains exactly as a fresh one
    clean, ctrs = make_group(trl, pack, n, models, assignment("blocks", n, 2))
    train_run_slots(trs, scheds, 8, None)
    train_run_slots(ctrs, scheds, 8, None)
    for p in range(2):
        assert_trainer(trs[p], ctrs[p], "after refusals, slot %d" % p)
    assert_envs(sc, [clean] * 2, assignment("blocks", n, 2), 90, stride=3)
    close(*trs, *ctrs, sc, clean)
