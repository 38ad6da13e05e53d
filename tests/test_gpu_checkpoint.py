"""Checkpoints (trl_checkpoint_save / trl_create_from_checkpoint): a run stopped between two calls and resumed from the file in a fresh
handle is the same run.  In every case run A makes two calls on one handle (U1 updates, then U2); run B makes the first call, saves,
destroys everything, loads the file and makes the second.  Then every env, every trainer array and list, the replay rows, the
counters, the tuple block, the evaluation statistics (per slot and per cell) and the distance log must be equal to the bit.

  (1) one trainer, trl_train_run with a fixed count and paced by tuples: the ring of the replay memory has wrapped and the trainer
      has left its init stage at the save, a target refresh falls after it; saved under the overlapped schedule, resumed under the
      overlapped schedule, the serial schedule and 3 env groups;
  (2) ScenarioTrainMACE paced: Run(U1 + U2) == Run(U1), Checkpoint, resume, Run(U2);
  (3) three training slots on their own schedules beside a terrain slot, lock-step and paced; the raptor with 2 slots;
  (4) an evaluation handle with 3 policy slots, 2 terrain slots and edited physics parameters (the goat on cliffs: falls and resets);
  (5) an exploration handle without a trainer: the tuples left in the block;
  (6) saving changes nothing; (7) the digests of a file against a numpy restatement; (8) refusals and damaged files.
tests/test_checkpoint_cpu.py runs a miniature of (3), (7) and (8) on the emulator."""
import ctypes as C
import os
import shutil
import struct

import numpy as np
import pytest

import torch_net  # noqa: F401  (torch before the library: see tests/test_gpu_decide_batches.py)
from test_gpu_policy_slots import pack_net, perturbed, raptor_mixed_model, write_net
from test_gpu_train_slots import DT, SCHEDULE, TERRAIN, assert_envs, assert_trainer, close, make_group, start_models

pytestmark = pytest.mark.gpu

# the ring of 600 rows has wrapped after the first call, the init stage (300 tuples) is over, a target refresh every 7 iterations
TRAINER = dict(replay_mem_size=600, num_init_samples=300, freeze_target_iters=7)
PACED = dict(SCHEDULE, trainer_curriculum_iters=0)      # trainers paced by tuples share the handle's one terrain blend


# ------------------------------------------------------------------------------------------------ shared helpers (also the CPU test's)
def mix64(z):
    z = z + np.uint64(0x9E3779B97F4A7C15)
    z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def digest(buf):
    """sum over the little-endian 64-bit words w_i (tail zero-padded) of mix64(w_i + (i + 1) K), mod 2^64"""
    b = np.frombuffer(bytes(buf) + b"\0" * (-len(buf) % 8), dtype="<u8")
    i = np.arange(1, b.size + 1, dtype=np.uint64)
    with np.errstate(over="ignore"):
        return int(np.sum(mix64(b + i * np.uint64(0xD1342543DE82EF95)), dtype=np.uint64))


def check_digests(path):
    from deepterrainrl_b200.checkpoint import sections
    data = open(path, "rb").read()
    secs = sections(path)
    assert secs[-1][3] + secs[-1][4] == len(data)
    for name, _, _, off, nbytes, dig in secs:
        assert digest(data[off:off + nbytes]) == dig, name
    return secs


def save_and_load(sc, trainers, path, user=b"", env=None, monkeypatch=None):
    """SaveCheckpoint, destroy everything, load_checkpoint (with the environment `env` set while the handle is created)"""
    import deepterrainrl_b200 as trl
    sc.SaveCheckpoint(path, user)
    close(*trainers, sc)
    for k, v in (env or {}).items():
        monkeypatch.setenv(k, v)
    sc2, trs, blob = trl.load_checkpoint(path)
    assert blob == user
    return sc2, trs


def by_env(key, *arrays):
    """the entries of the tuple block / distance log grouped by env (their slots come from an atomic cursor, so the order of different
    envs' entries is timing dependent; an env's own entries stay in the order it made them)"""
    order = np.argsort(key, kind="stable")
    return [key[order]] + [x[order] for x in arrays]


def assert_same(a, b, trs_a=(), trs_b=(), n_out=90, stride=1):
    """handle b == handle a: every env (state, controller, net output, policy state, distance log), the batch statistics of every slot
    and cell, the tuple block, the trainers"""
    n = a.num_envs
    assert np.array_equal(a.EnvPolicy(), b.EnvPolicy())
    assert all(np.array_equal(x, y) for x, y in zip(a.EnvTerrain(), b.EnvTerrain()))
    assert_envs(b, [a], np.zeros(n, int), n_out, stride=stride)
    assert all(np.array_equal(x, y) for x, y in zip(by_env(*a.GetDistLog()), by_env(*b.GetDistLog())))
    assert all(np.array_equal(x, y) for x, y in zip(a.GetStateAll(), b.GetStateAll()))
    assert a._stats() == b._stats()
    for p in sorted(set(a.EnvPolicy().tolist())):
        for t in [None] + sorted(set(a.EnvTerrain()[0].tolist())):
            assert a.GetEvalStats(p, terrain=t) == b.GetEvalStats(p, terrain=t), (p, t)
    if hasattr(a, "GetTuples"):
        ra, fa, ea = a.GetTuples(f64=True)
        rb, fb, eb = b.GetTuples(f64=True)
        assert all(np.array_equal(x, y) for x, y in zip(by_env(ea, ra, fa), by_env(eb, rb, fb)))
    assert len(trs_a) == len(trs_b)
    for k, (x, y) in enumerate(zip(trs_a, trs_b)):
        assert x.params == y.params and x.slot == y.slot and (x.S, x.A, x.W) == (y.S, y.A, y.W)
        assert_trainer(x, y, "trainer %d" % k)


def sp_of(schedule):
    from deepterrainrl_b200.train import TrainSchedule
    return np.array([schedule.p[k] for k in TrainSchedule.KEYS], float)


def train_run(tr, sp, updates, iters):
    L = tr.L
    assert L.trl_train_run(tr.h, sp.ctypes.data_as(C.c_void_p), int(updates), int(iters), 32, C.c_double(DT)) == 0, L.trl_last_error().decode()


# ------------------------------------------------------------------------------------------------ (1) one trainer, trl_train_run
@pytest.mark.parametrize("iters", [2, 0])
def test_train_run_resumes_under_every_schedule(assets, tmp_path, monkeypatch, iters):
    import deepterrainrl_b200 as trl
    from deepterrainrl_b200.train import TrainSchedule
    for k in ("TRL_SERIAL_SCHEDULE", "TRL_GROUPS"):
        monkeypatch.delenv(k, raising=False)
    pack = os.path.join(assets, "dog_slopes_mixed.trlpack")
    n, u1, u2 = 2048, 40, 20
    sp = sp_of(TrainSchedule(**SCHEDULE))
    a = trl.ScenarioExpMACE(pack, n, rng_seed=5)
    ta = trl.MACETrainer(a, seed=3, **TRAINER)
    train_run(ta, sp, u1, iters)
    c = ta.counters()
    assert c["total"] > TRAINER["replay_mem_size"] and c["stage"] == 1, c
    path = str(tmp_path / "a.ckpt")
    a.SaveCheckpoint(path)
    it0 = c["iter"]
    train_run(ta, sp, u2, iters)
    assert ta.counters()["iter"] // TRAINER["freeze_target_iters"] > it0 // TRAINER["freeze_target_iters"], "no target refresh in U2"
    for env in ({}, {"TRL_SERIAL_SCHEDULE": "1"}, {"TRL_GROUPS": "3"}):
        with monkeypatch.context() as m:
            for k, v in env.items():
                m.setenv(k, v)
            b, trs, _ = trl.load_checkpoint(path)
        assert set(trs) == {0}
        train_run(trs[0], sp, u2, iters)
        assert_same(a, b, [ta], [trs[0]], stride=5)
        close(trs[0], b)
    close(ta, a)


# ------------------------------------------------------------------------------------------------ (2) ScenarioTrainMACE
def test_scenario_train_mace_resumes(assets, tmp_path):
    from deepterrainrl_b200.train import ScenarioTrainMACE, TrainSchedule
    pack = os.path.join(assets, "dog_slopes_mixed.trlpack")
    kw = dict(rng_seed=7, schedule=TrainSchedule(**SCHEDULE), trainer_params=dict(TRAINER, seed=4), iters_per_update=None)
    u1, u2 = 30, 15
    a = ScenarioTrainMACE(pack, 1024, **kw)
    a.Run(u1 + u2)
    b = ScenarioTrainMACE(pack, 1024, **kw)
    b.Run(u1)
    path = str(tmp_path / "train.ckpt")
    b.Checkpoint(path)
    close(b.trainer, b.exp)
    b = ScenarioTrainMACE.resume(path)
    b.Run(u2)
    assert (a._iters, a._last_total, a._carry) == (b._iters, b._last_total, b._carry)
    assert a.schedule.p == b.schedule.p
    assert_same(a.exp, b.exp, [a.trainer], [b.trainer], stride=3)
    close(a.trainer, a.exp, b.trainer, b.exp)


# ------------------------------------------------------------------------------------------------ (3) training slots
def _slots_setup(n):
    terr = (np.arange(n) // 3) % 2

    def setup(sc):
        sc.LoadTerrain(1, os.path.join(TERRAIN, "narrow_gaps.txt"))
        sc.SetEnvTerrain(terr)
    return setup


@pytest.mark.parametrize("paced", [False, True])
def test_training_slots_resume(assets, tmp_path, paced):
    import deepterrainrl_b200 as trl
    from deepterrainrl_b200.train import TrainSchedule, train_run_slots
    pack = os.path.join(assets, "dog_slopes_mixed.trlpack")
    n, u1, u2 = 2048, 30, 15
    models = start_models(pack, str(tmp_path))
    slots = np.random.default_rng(2).integers(0, 3, n)
    base = PACED if paced else SCHEDULE
    scheds = [TrainSchedule(**dict(base, init_exp_rate=r)) for r in (0.5, 0.35, 0.8)]
    iters = None if paced else 2

    def group():
        return make_group(trl, pack, n, models, slots, trainer_kw=TRAINER, setup=_slots_setup(n))
    a, ta = group()
    b, tb = group()
    for sc, trs in ((a, ta), (b, tb)):
        train_run_slots(trs, scheds, u1, iters)
    assert all(t.counters()["stage"] == 1 for t in ta)
    b, tb = save_and_load(b, tb, str(tmp_path / "slots.ckpt"), user=b"slots")
    tb = [tb[p] for p in range(3)]
    for sc, trs in ((a, ta), (b, tb)):
        train_run_slots(trs, scheds, u2, iters)
    assert_same(a, b, ta, tb, stride=3)
    close(*ta, *tb, a, b)


def test_raptor_two_training_slots_resume(assets, tmp_path):
    import deepterrainrl_b200 as trl
    from deepterrainrl_b200.train import TrainSchedule, train_run_slots
    pack = os.path.join(assets, "raptor_narrow_gaps.trlpack")
    n = 1000
    models = [None, raptor_mixed_model(str(tmp_path))]
    slots = np.arange(n) % 2
    sched = TrainSchedule(**SCHEDULE)
    a, ta = make_group(trl, pack, n, models, slots, trainer_kw=TRAINER)
    b, tb = make_group(trl, pack, n, models, slots, trainer_kw=TRAINER)
    for trs in (ta, tb):
        train_run_slots(trs, sched, 25, 2)
    b, tb = save_and_load(b, tb, str(tmp_path / "raptor.ckpt"))
    tb = [tb[0], tb[1]]
    for trs in (ta, tb):
        train_run_slots(trs, sched, 12, 2)
    assert_same(a, b, ta, tb, n_out=87, stride=3)
    close(*ta, *tb, a, b)


# ------------------------------------------------------------------------------------------------ (4) evaluation handle
def test_evaluation_slots_resume(assets, tmp_path):
    import deepterrainrl_b200 as trl
    pack = os.path.join(assets, "goat_cliffs.trlpack")
    n = 1024
    net = pack_net(pack)
    files = [write_net(str(tmp_path / ("goat%d.h5" % k)), perturbed(net, k)) for k in (1, 2)]

    def make():
        sc = trl.ScenarioPoliEval(pack, n, rng_seed=11)
        for k, f in enumerate(files):
            sc.LoadPolicy(k + 1, f)
        sc.LoadTerrain(1, os.path.join(TERRAIN, "cliffs_rugged.txt"))
        sc.SetEnvPolicy(np.arange(n) % 3)
        sc.SetEnvTerrain((np.arange(n) // 2) % 2)
        sc.SetPhysParams([2.0e5, 2.0e3, 0.7, 0.01, 0.00025, 2.0e4, 20.0])
        return sc
    a, b = make(), make()
    for sc in (a, b):
        for _ in range(6):
            sc.Update(DT)
    eps = a.GetNumEpisodes()
    b, _ = save_and_load(b, [], str(tmp_path / "eval.ckpt"))
    assert isinstance(b, trl.ScenarioPoliEval)
    for sc in (a, b):
        for _ in range(30):
            sc.Update(DT)
    assert a.GetNumEpisodes() > eps, "no fall in U2"
    assert_same(a, b, stride=3)
    close(a, b)


# ------------------------------------------------------------------------------------------------ (5) tuples left in the block
def test_tuple_block_resumes(assets, tmp_path):
    import deepterrainrl_b200 as trl
    pack = os.path.join(assets, "dog_slopes_mixed.trlpack")
    a = trl.ScenarioExpMACE(pack, 512, rng_seed=3)
    a.EnableExplore(True, 0.3, 0.5, 0.1, slot=0)
    for _ in range(40):
        a.Update(DT)
    before = a.GetTuples(f64=True)
    assert before[0].shape[0] > 0
    path = str(tmp_path / "tuples.ckpt")
    a.SaveCheckpoint(path)
    b, trs, _ = trl.load_checkpoint(path)
    assert trs == {} and isinstance(b, trl.ScenarioExpMACE)
    assert all(np.array_equal(x, y) for x, y in zip(before, b.GetTuples(f64=True)))
    for sc in (a, b):
        for _ in range(10):
            sc.Update(DT)
    assert_same(a, b, stride=3)
    close(a, b)


# ------------------------------------------------------------------------------------------------ (6) saving changes nothing, (7) digests
def test_saving_changes_nothing_and_digests_match(assets, tmp_path):
    import deepterrainrl_b200 as trl
    from deepterrainrl_b200.train import TrainSchedule
    pack = os.path.join(assets, "dog_slopes_mixed.trlpack")
    sp = sp_of(TrainSchedule(**SCHEDULE))
    pair = []
    for save in (False, True):
        sc = trl.ScenarioExpMACE(pack, 1024, rng_seed=8)
        tr = trl.MACETrainer(sc, seed=2, **TRAINER)
        train_run(tr, sp, 30, 2)
        if save:
            path = str(tmp_path / "twin.ckpt")
            sc.SaveCheckpoint(path, b"\x01\x02\x03")
            names = [s[0] for s in check_digests(path)]
            assert names[:2] == ["scene", "meta"] and "t0.mem" in names and names.count("user") == 1
        train_run(tr, sp, 15, 2)
        pair.append((sc, tr))
    assert_same(pair[0][0], pair[1][0], [pair[0][1]], [pair[1][1]], stride=3)
    close(pair[0][1], pair[1][1], pair[0][0], pair[1][0])


# ------------------------------------------------------------------------------------------------ (8) refusals and damaged files
def _uid(L):
    buf = (C.c_ubyte * 128)()
    assert L.trl_comm_unique_id(buf) == 0, L.trl_last_error().decode()
    return bytes(buf)


def damaged_copies(path, out_dir):
    """(file, expected message) for a byte flipped in every non-empty section, a truncated copy and a wrong version"""
    from deepterrainrl_b200.checkpoint import sections
    data = open(path, "rb").read()
    out = []
    for name, _, _, off, nbytes, _ in sections(path):
        if nbytes == 0:
            continue
        d = bytearray(data)
        d[off + nbytes // 2] ^= 0x10
        p = os.path.join(out_dir, "flip_%s" % name)
        open(p, "wb").write(d)
        out.append((p, "section '%s'" % name))
    p = os.path.join(out_dir, "truncated")
    open(p, "wb").write(data[:len(data) - 5])
    out.append((p, "truncated"))
    d = bytearray(data)
    d[8:12] = struct.pack("<I", 2)
    p = os.path.join(out_dir, "version")
    open(p, "wb").write(d)
    out.append((p, "version"))
    return out


def assert_refused(L, path, msg):
    tr = (C.c_void_p * 8)()
    L.trl_create_from_checkpoint.restype = C.c_void_p
    h = L.trl_create_from_checkpoint(path.encode(), 0, tr, None, 0, None)
    assert not h and not any(tr), path
    assert msg in L.trl_last_error().decode(), (path, L.trl_last_error().decode())


def test_refusals_and_damaged_files(assets, tmp_path):
    import torch
    import deepterrainrl_b200 as trl
    from deepterrainrl_b200 import parallel
    pack = os.path.join(assets, "dog_slopes_mixed.trlpack")
    sc = trl.ScenarioExpMACE(pack, 128, rng_seed=4)
    L = sc.L
    tr = trl.MACETrainer(sc, replay_mem_size=128, num_init_samples=64, seed=1)
    for _ in range(8):
        sc.Update(DT)
    tr.AddTuplesFromScene()
    tr.Train(2)
    path = str(tmp_path / "ok.ckpt")
    sc.Snapshot()
    with pytest.raises(RuntimeError, match="snapshot"):
        sc.SaveCheckpoint(path)
    sc.SnapshotWait()
    comm = parallel.Comm(sc, 0, 1, backend="nccl", unique_id=_uid(L))
    assert L.trl_trainer_set_async(tr.h, 1) == 0, L.trl_last_error().decode()
    with pytest.raises(RuntimeError, match="communicator"):
        sc.SaveCheckpoint(path)
    assert not os.path.exists(path)
    comm.close()
    with pytest.raises(RuntimeError, match="asynchronous"):
        sc.SaveCheckpoint(path)
    assert L.trl_trainer_set_async(tr.h, 0) == 0
    assert not os.path.exists(path)
    sc.SaveCheckpoint(path)
    close(tr, sc)
    d = tmp_path / "bad"
    d.mkdir()
    cases = damaged_copies(path, str(d))
    assert len(cases) > 40
    ok, trs, _ = trl.load_checkpoint(path)      # every kernel a restore launches is loaded before the memory is counted
    close(*trs.values(), ok)
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    for p, msg in cases:
        assert_refused(L, p, msg)
    assert torch.cuda.mem_get_info()[0] == free0
    shutil.rmtree(str(d))
