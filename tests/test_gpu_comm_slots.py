"""Training slots over the tuple exchange (trl_train_run_slots_comm): several policies of one exploration handle trained from every
rank's experience, synchronously or asynchronously.  The contract is the one of both features: replicas stay bit-identical, and trainer
p ends where a single trainer fed only slot p's rows (rank order, env order inside a rank) ends.

  * world 1 == the local loop: with a single-rank communicator and blocks that hold every tuple of an update, the new entry computes
    bit for bit what trl_train_run_slots_sched computes on a twin handle without one (dog, 3 slots, three assignments, lock-step and
    paced, the three schedules; the raptor with 2 slots);
  * queued rows: with small blocks each trainer equals a host-filtered reference trainer fed, after every update, its slot's rows of
    the blocks the update gathered (trl_gathered_fetch, bit 31 clear, slot bits = p, sorted by global env id);
  * the block format: zero slot bits in a handle without training slots, the env's slot in one with them;
  * world 2 on one GPU (two processes, gloo collectives staged through host memory), lock-step: zero replica spread per slot, the
    host-filtered reference, the per-slot statistics all-reduce, a mismatched call and a paced call refused on both ranks;
  * asynchronous slot trainers: trainer p and slot p's envs of an all-async run == a twin in which p's trainer is the only one listed;
    slot 0 alone == trl_train_run async; every env on slot 1 with its async trainer == trl_train_run async on a plain handle;
  * refusals, each leaving the handle as a fresh one.
tests/test_comm_slots_cpu.py runs the world-2 check on the emulator."""
import ctypes as C
import os

import numpy as np
import pytest

import torch_net  # noqa: F401  (torch before the library: see tests/test_gpu_decide_batches.py)
from test_gpu_policy_slots import assignment, raptor_mixed_model
from test_gpu_train_schedules import schedules, sp_array
from test_gpu_train_slots import (DT, TRAINER, _schedule_env, assert_envs, assert_trainer, close, make_group, make_trainer, start_models)

pytestmark = pytest.mark.gpu

UPDATES = 30
ITERS = 2


def uid(L):
    buf = (C.c_ubyte * 128)()
    assert L.trl_comm_unique_id(buf) == 0, L.trl_last_error().decode()
    return bytes(buf)


def comm1(sc):
    from deepterrainrl_b200 import parallel
    return parallel.Comm(sc, 0, 1, backend="nccl", unique_id=uid(sc.L))


# ------------------------------------------------------------------------------------------------ host-filtered references
def feed_reference(refs, comm, iters, tbs=32):
    """one update's intake for every reference trainer: slot p's rows of the blocks the last gather delivered, in gathered order
    (rank order, env order inside a rank), then the iterations the loop ran (paced: one per tbs fresh rows)"""
    counts, rows, flags, env = comm.Fetch()
    for p, tr in refs.items():
        keep = np.flatnonzero(((flags >> 31) == 0) & (((flags >> 24) & 7) == p))
        keep = keep[np.argsort(env[keep], kind="stable")]
        before = tr.counters()["total"]
        if keep.size:
            tr.AddTuples(rows[keep].astype(np.float64), flags[keep] & 0x00FFFFFF)
        k = iters if iters else (tr.counters()["total"] - before) // tbs
        if k > 0:
            tr.Train(k)
    return flags, env


def reference_trainers(trl, pack, models, trainer_kw):
    """one trainer per slot on a handle of its own that never steps: it is only fed rows"""
    out = {}
    for p, m in enumerate(models):
        sc = trl.ScenarioExpMACE(pack, 32)
        out[p] = (sc, make_trainer(trl, sc, 0, m, p, trainer_kw))
    return out


# ------------------------------------------------------------------------------------------------ (1) world 1 == the local loop
CASES = [("blocks", "overlap", ITERS), ("round_robin", "serial", ITERS), ("random", "groups3", ITERS), ("random", "overlap", None)]


@pytest.mark.parametrize("pattern,schedule,iters", CASES)
def test_world1_equals_local_loop(assets, tmp_path, monkeypatch, pattern, schedule, iters):
    import deepterrainrl_b200 as trl
    from deepterrainrl_b200.train import train_run_slots
    _schedule_env(monkeypatch, schedule)
    pack = os.path.join(assets, "dog_slopes_mixed.trlpack")
    n = 2048
    models = start_models(pack, str(tmp_path))
    slots = assignment(pattern, n, 3, seed=2)
    scheds = schedules(curriculum=None if iters else 0)
    a, tas = make_group(trl, pack, n, models, slots)
    train_run_slots(tas, scheds, UPDATES, iters)
    b, tbs = make_group(trl, pack, n, models, slots)
    comm = comm1(b)
    train_run_slots(tbs, scheds, UPDATES, iters, comm=comm, block_rows=n)
    for p in range(3):
        assert tas[p].counters()["total"] > 0
        assert_trainer(tbs[p], tas[p], "slot %d" % p)
        assert comm.ReplicaSpread(tbs[p]) == 0.0
    assert_envs(b, [a] * 3, slots, 90)
    assert b.GetNumTuples() == 0 and comm.TuplesDropped() == 0
    comm.close()
    close(*tas, *tbs, a, b)


def test_raptor_world1_equals_local_loop(assets, tmp_path):
    import deepterrainrl_b200 as trl
    from deepterrainrl_b200.train import train_run_slots
    pack = os.path.join(assets, "raptor_narrow_gaps.trlpack")
    n = 1000
    models = [None, raptor_mixed_model(str(tmp_path))]
    slots = assignment("random", n, 2, seed=3)
    scheds = schedules(curriculum=0)[1:]
    a, tas = make_group(trl, pack, n, models, slots)
    train_run_slots(tas, scheds, 40, None)
    b, tbs = make_group(trl, pack, n, models, slots)
    comm = comm1(b)
    train_run_slots(tbs, scheds, 40, None, comm=comm, block_rows=n)
    for p in range(2):
        assert_trainer(tbs[p], tas[p], "raptor slot %d" % p)
    assert_envs(b, [a] * 2, slots, 87, stride=3)
    comm.close()
    close(*tas, *tbs, a, b)


# ------------------------------------------------------------------------------------------------ (2) queued rows, (3) block format
def test_queued_rows_match_host_filtered_reference(assets, tmp_path):
    import deepterrainrl_b200 as trl
    from deepterrainrl_b200.train import train_run_slots
    pack = os.path.join(assets, "dog_slopes_mixed.trlpack")
    n = 1024
    models = start_models(pack, str(tmp_path))
    slots = assignment("random", n, 3, seed=5)
    scheds = schedules(curriculum=0)
    g, trs = make_group(trl, pack, n, models, slots)
    comm = comm1(g)
    refs = reference_trainers(trl, pack, models, TRAINER)
    queued = 0
    for u in range(40):
        train_run_slots(trs, scheds, 1, ITERS, comm=comm, block_rows=64)
        queued += g.GetNumTuples()
        flags, env = feed_reference({p: r[1] for p, r in refs.items()}, comm, ITERS)
        assert np.array_equal((flags >> 24) & 0x7F, slots[env]), "slot bits"            # the env's policy slot, nothing else
    assert queued > 0, "no update left rows queued"
    for p in range(3):
        assert trs[p].counters()["total"] > 0
        assert_trainer(trs[p], refs[p][1], "queued, slot %d" % p)
        ids = np.arange(trs[p].counters()["num"], dtype=np.int32)
        assert np.all((trs[p].rows(ids)[1] >> 24) == 0), "replay flags carry slot bits"
    comm.close()
    close(*trs, g, *[o for r in refs.values() for o in r[::-1]])


def test_plain_handle_blocks_have_zero_slot_bits(assets):
    import deepterrainrl_b200 as trl
    pack = os.path.join(assets, "dog_slopes_mixed.trlpack")
    sc = trl.ScenarioExpMACE(pack, 256, rng_seed=3)
    comm = comm1(sc)
    sc.EnableExplore(True, 0.3, 0.025, 0.02)
    seen = 0
    for _ in range(40):
        sc.Update()
        loc, lf, le = sc.GetTuples()
        comm.GatherTuples(block_rows=256)
        counts, rows, flags, env = comm.Fetch()
        np.testing.assert_array_equal(rows, loc); np.testing.assert_array_equal(env, le)
        np.testing.assert_array_equal(flags & 0x7FFFFFFF, lf)               # bits 24..30 zero: the parent's block, byte for byte
        seen += len(loc)
    assert seen > 50
    comm.close(); sc.close()


# ------------------------------------------------------------------------------------------------ (4) world 2 on one GPU
def _device_collectives(group):
    """trl_collectives for device buffers over a gloo group: the library's stream is drained, the bytes staged through host memory"""
    import torch
    import torch.distributed as dist
    from deepterrainrl_b200.parallel import _Collectives
    world = dist.get_world_size(group)

    class _Dev:
        def __init__(self, ptr, nbytes):
            self.__cuda_array_interface__ = dict(shape=(nbytes,), typestr="|u1", data=(ptr, False), version=3)

    def dev(ptr, nbytes):
        return torch.as_tensor(_Dev(ptr, nbytes), device="cuda")

    def drain(stream):
        torch.cuda.ExternalStream(stream).synchronize() if stream else torch.cuda.synchronize()

    def all_gather(ctx, send, recv, nbytes, stream):
        drain(stream)
        out = torch.empty(world * nbytes, dtype=torch.uint8)
        dist.all_gather(list(out.view(world, nbytes).unbind(0)), dev(send, nbytes).cpu(), group=group)
        dev(recv, world * nbytes).copy_(out); torch.cuda.synchronize()
        return 0

    def broadcast(ctx, buf, nbytes, root, stream):
        drain(stream)
        h = dev(buf, nbytes).cpu()
        dist.broadcast(h, src=root, group=group)
        dev(buf, nbytes).copy_(h); torch.cuda.synchronize()
        return 0

    def all_reduce(ctx, buf, count, stream):
        drain(stream)
        h = dev(buf, 8 * count).cpu().view(torch.float64)
        dist.all_reduce(h, group=group)
        dev(buf, 8 * count).copy_(h.view(torch.uint8)); torch.cuda.synchronize()
        return 0

    fns = (_Collectives.AG(all_gather), _Collectives.BC(broadcast), _Collectives.AR(all_reduce))
    return _Collectives(None, *fns), fns


def world2_slots(rank, n):
    """a different assignment on every rank"""
    return np.random.default_rng(40 + rank).integers(0, 2, n)


def world2_refusals(rank, sc, trs, scheds):
    """calls that differ between the ranks, or that one rank refuses by itself: every one must be refused on both ranks (no rank may be
    left waiting in the agreement all-reduce), with nothing run; returns one flag per call"""
    L = sc.L
    sp = sp_array(scheds)

    def call(ts, spx, ipu):
        arr = (C.c_void_p * len(ts))(*[t.h.value for t in ts])
        rc = L.trl_train_run_slots_comm(arr, len(ts), spx.ctypes.data_as(C.c_void_p), 1, ipu, 32, 64, C.c_double(DT))
        return rc, L.trl_last_error().decode()

    other = "another rank refused"
    differ = "ranks differ"
    got = []
    # rank 1 lists the slots the other way round
    rc, e = call(trs if rank == 0 else trs[::-1], sp, 1)
    got.append(rc != 0 and differ in e)
    # rank 1 with another exploration rate in one schedule
    sp2 = sp.copy()
    if rank == 1:
        sp2[0, 1] = 0.3
    rc, e = call(trs, sp2, 1)
    got.append(rc != 0 and differ in e)
    # rank 1 paced by tuples, rank 0 lock-step
    rc, e = call(trs, sp, 0 if rank == 1 else 2)
    got.append(rc != 0 and differ in e)
    # a curriculum on rank 1 only
    sp3 = sp.copy()
    if rank == 1:
        sp3[:, 8] = 30
    rc, e = call(trs, sp3, 1)
    got.append(rc != 0 and differ in e)
    # rank 1's own schedules disagree on the curriculum: rank 1 refuses by itself, rank 0 with it
    sp4 = sp.copy()
    if rank == 1:
        sp4[:, 8] = 30
        sp4[1, 8] = 40
    rc, e = call(trs, sp4, 1)
    got.append(rc != 0 and (("trainer_curriculum_iters" in e) if rank == 1 else (other in e)))
    # one asynchronous trainer on rank 1: the same
    if rank == 1:
        trs[0].SetAsync(True)
    rc, e = call(trs, sp, 1)
    got.append(rc != 0 and (("all or none" in e) if rank == 1 else (other in e)))
    if rank == 1:
        trs[0].SetAsync(False)
    return np.array(got)


def world2_worker(rank, world, port, pack, out_dir, emulated, n, updates, mode, seeds, per_call=1):
    """one rank of a world-2 run of 2 slots (the pack's model, a fresh net), `per_call` updates per call of the native loop; mode: a
    positive count (lock-step), "paced" (one iteration per 32 fresh tuples) or "intake" (the update, the gather and each trainer's
    slot-filtered intake, no iteration: an emulated trainer iteration costs seconds).  With one update per call the gathered blocks of
    each update also feed host-filtered reference trainers.  Then the per-slot statistics and the refused calls"""
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, root)
    sys.path.insert(0, os.path.join(root, "tests"))
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    import torch.distributed as dist
    dist.init_process_group("gloo", rank=rank, world_size=world)
    if emulated:
        sys.path.insert(0, os.path.join(root, "tests", "simt"))
        from loader import open_simt
        from deepterrainrl_b200 import scenario
        scenario._LIB = open_simt()
    import deepterrainrl_b200 as trl
    from deepterrainrl_b200 import parallel
    from deepterrainrl_b200.train import train_run_slots
    trainer_kw = dict(replay_mem_size=160, num_init_samples=64, freeze_target_iters=2) if emulated else TRAINER
    models = [None, "fresh"]
    scheds = schedules(curriculum=0)[:2]
    slots = world2_slots(rank, n)
    out = {}
    for s_i, seed in enumerate(seeds):
        sc = trl.ScenarioExpMACE(pack, n, terrain_seeds=parallel.shard_seeds(rank, n), rng_seed=100 + rank)
        trs = [make_trainer(trl, sc, p, m, p, trainer_kw) for p, m in enumerate(models)]
        sc.SetEnvPolicy(slots)
        if emulated:
            comm = parallel.Comm(sc, rank, world, backend="external")
        else:
            keep = _device_collectives(None)
            comm = parallel.Comm.__new__(parallel.Comm)
            comm.sc, comm.rank, comm.world, comm.L, comm._keep = sc, rank, world, sc.L, keep
            comm._ck(sc.L.trl_comm_init_external(sc.h, C.byref(keep[0]), rank, world))
        refs = reference_trainers(trl, pack, models, trainer_kw)
        if s_i == 0:
            out["refused"] = world2_refusals(rank, sc, trs, scheds)
        if emulated:
            sc.L.simt_set_sched_seed(C.c_ulonglong(seed))
        try:
            if mode == "intake":
                sc.EnableExplore(True, 0.3, 0.025, 0.02)
            for u in range(0, updates, per_call):
                if mode == "intake":
                    sc.Update(DT)
                    comm.GatherTuples(block_rows=8 if emulated else 128)
                    for t in trs:
                        comm.AddGathered(t)
                else:
                    train_run_slots(trs, scheds, per_call, None if mode == "paced" else mode, comm=comm, block_rows=8 if emulated else 128)
                if per_call == 1:
                    feed_reference({p: r[1] for p, r in refs.items()}, comm, mode if isinstance(mode, int) else 0,
                                   tbs=32 if mode == "paced" else 1 << 30)
        finally:
            if emulated:
                sc.L.simt_set_sched_seed(C.c_ulonglong(0))
        for p in range(2):
            c = trs[p].counters()
            out[f"s{s_i}_theta{p}"] = trs[p].get("theta")
            out[f"s{s_i}_ref_theta{p}"] = refs[p][1].get("theta")
            out[f"s{s_i}_counters{p}"] = np.array([c[k] for k in ("iter", "num", "total", "critic", "actor", "stage")])
            out[f"s{s_i}_ref_counters{p}"] = np.array([refs[p][1].counters()[k] for k in ("iter", "num", "total", "critic", "actor", "stage")])
            out[f"s{s_i}_spread{p}"] = comm.ReplicaSpread(trs[p])
            ids = np.arange(c["num"], dtype=np.int32)
            r_a, f_a = trs[p].rows(ids)
            r_b, f_b = refs[p][1].rows(ids)
            out[f"s{s_i}_rows_equal{p}"] = bool(np.array_equal(r_a, r_b) and np.array_equal(f_a, f_b))
            st = sc.GetEvalStats(p)
            g = comm.EvalStats(slot=p)
            out[f"s{s_i}_stats{p}"] = np.array([st["cycles"], st["episodes"], st["steps"], st["avg_dist"] * st["episodes"]], float)
            out[f"s{s_i}_comm_stats{p}"] = np.array([g["cycles"], g["episodes"], g["steps"], g["avg_dist"] * g["episodes"]], float)
        out[f"s{s_i}_state"] = np.stack(sc.GetStateAll())
        comm.close()
        close(*trs, sc, *[o for r in refs.values() for o in r[::-1]])
    np.savez(os.path.join(out_dir, f"w{rank}.npz"), **out)
    dist.destroy_process_group()


def check_world2(out_dir, n_seeds, reference=True, trained=False):
    """both ranks' results of world2_worker: zero replica spread and identical replicas per slot, the host-filtered references (one
    update per call), the per-slot statistics all-reduce, the refused calls; runs after the first (which began with the refused
    calls, or ran under another lane schedule) equal to the first, envs included"""
    w = [np.load(os.path.join(out_dir, f"w{r}.npz")) for r in range(2)]
    for s in range(n_seeds):
        for p in range(2):
            a, b = w[0], w[1]
            np.testing.assert_array_equal(a[f"s{s}_theta{p}"], b[f"s{s}_theta{p}"])
            np.testing.assert_array_equal(a[f"s{s}_counters{p}"], b[f"s{s}_counters{p}"])
            assert float(a[f"s{s}_spread{p}"]) == 0.0 and float(b[f"s{s}_spread{p}"]) == 0.0, ("replica spread", s, p)
            if reference:
                for r in range(2):
                    np.testing.assert_array_equal(w[r][f"s{s}_theta{p}"], w[r][f"s{s}_ref_theta{p}"])
                    np.testing.assert_array_equal(w[r][f"s{s}_counters{p}"], w[r][f"s{s}_ref_counters{p}"])
                    assert bool(w[r][f"s{s}_rows_equal{p}"]), ("replay rows", s, p, r)
            assert int(a[f"s{s}_counters{p}"][2]) > 0, ("slot", p, "received no tuple")
            if trained:
                assert int(a[f"s{s}_counters{p}"][0]) > 0, ("slot", p, "ran no iteration")
            tot = a[f"s{s}_stats{p}"] + b[f"s{s}_stats{p}"]
            for r in range(2):
                np.testing.assert_array_equal(w[r][f"s{s}_comm_stats{p}"][:3], tot[:3])
                np.testing.assert_allclose(w[r][f"s{s}_comm_stats{p}"][3], tot[3], rtol=1e-9)
        if s:
            for r in range(2):
                for p in range(2):
                    np.testing.assert_array_equal(w[r][f"s{s}_theta{p}"], w[r][f"s0_theta{p}"])
                    np.testing.assert_array_equal(w[r][f"s{s}_counters{p}"], w[r][f"s0_counters{p}"])
                np.testing.assert_array_equal(w[r][f"s{s}_state"], w[r]["s0_state"])
    for r in range(2):
        assert w[r]["refused"].all(), (r, w[r]["refused"])


@pytest.mark.parametrize("mode,per_call", [(ITERS, 1), ("paced", 1), ("paced", 3)])
def test_world2_on_one_gpu(assets, tmp_path, mode, per_call):
    """lock-step: two runs, the first after the refused calls, must be equal; paced with one update per call against the
    host-filtered references, with three per call (the pacing carry inside a call) replicas only"""
    import torch.multiprocessing as mp
    pack = os.path.join(assets, "dog_slopes_mixed.trlpack")
    port = 29500 + ((os.getpid() + 11 + 7 * per_call + (3 if mode == "paced" else 0)) % 1000)
    n, updates, seeds = (512, 30, [0, 0]) if mode != "paced" else (1024, 45, [0])
    mp.spawn(world2_worker, args=(2, port, pack, str(tmp_path), False, n, updates, mode, seeds, per_call), nprocs=2, join=True)
    check_world2(str(tmp_path), len(seeds), reference=per_call == 1, trained=mode == "paced")


# ------------------------------------------------------------------------------------------------ (5) asynchronous slot trainers
@pytest.mark.parametrize("schedule", ["overlap", "serial", "groups3"])
def test_async_slots_equal_single_async_trainer(assets, tmp_path, monkeypatch, schedule):
    import deepterrainrl_b200 as trl
    from deepterrainrl_b200.train import train_run_slots
    _schedule_env(monkeypatch, schedule)
    pack = os.path.join(assets, "dog_slopes_mixed.trlpack")
    n = 1024
    models = start_models(pack, str(tmp_path))
    slots = assignment("random", n, 3, seed=8)
    scheds = schedules()
    g, trs = make_group(trl, pack, n, models, slots)
    comm = comm1(g)
    for t in trs:
        t.SetAsync(True)
    train_run_slots(trs, scheds, UPDATES, ITERS, comm=comm, block_rows=n)
    for p in range(3):
        # the twin: the same handle, every slot with its starting net, p's trainer the only one listed and asynchronous
        tw, ttrs = make_group(trl, pack, n, models, slots)
        tc = comm1(tw)
        ttrs[p].SetAsync(True)
        train_run_slots([ttrs[p]], [scheds[p]], UPDATES, ITERS, comm=tc, block_rows=n)
        assert_trainer(trs[p], ttrs[p], "async slot %d" % p)
        for e in np.flatnonzero(slots == p)[::5]:
            for a_, b_ in zip(g.GetState(int(e)), tw.GetState(int(e))):
                assert np.array_equal(a_, b_), ("async env", int(e), "slot", p)
            assert np.array_equal(g.GetCtrl(int(e)), tw.GetCtrl(int(e)))
        tc.close()
        close(*ttrs, tw)
    comm.close()
    close(*trs, g)


def test_async_training_slot_is_train_run(assets, tmp_path):
    """the slot-table binding of an asynchronous slot trainer, against code without slots: every env on slot 1 of a slot handle, its
    trainer the only one and asynchronous == a plain handle started from the same net, trained by trl_train_run asynchronously"""
    import deepterrainrl_b200 as trl
    from deepterrainrl_b200.train import train_run_slots
    from test_gpu_train_slots import make_ref
    pack = os.path.join(assets, "dog_slopes_mixed.trlpack")
    n = 1024
    models = start_models(pack, str(tmp_path))[:2]
    slots = np.ones(n, int)
    sched = schedules()[1]
    g = trl.ScenarioExpMACE(pack, n, rng_seed=5)
    t1 = make_trainer(trl, g, 1, models[1], 1, TRAINER)
    g.SetEnvPolicy(slots)                                    # every env moves to slot 1 and restarts
    cg = comm1(g)
    t1.SetAsync(True)
    train_run_slots([t1], [sched], UPDATES, ITERS, comm=cg, block_rows=n)
    a, ta = make_ref(trl, pack, n, models, 1, slots)        # slot 1's model and trainer seed as slot 0, the same envs restarted
    ca = comm1(a)
    ta.SetAsync(True)
    sp = sp_array([sched])
    assert ta.L.trl_train_run(ta.h, sp.ctypes.data_as(C.c_void_p), UPDATES, ITERS, 32, C.c_double(DT)) == 0, ta.L.trl_last_error()
    assert ta.counters()["stage"] == 1
    assert_trainer(t1, ta, "async slot 1")
    assert_envs(g, [a, a], slots, 90, stride=3)
    cg.close(); ca.close()
    close(t1, ta, g, a)


def test_async_slot0_alone_is_train_run(assets):
    import deepterrainrl_b200 as trl
    from deepterrainrl_b200.train import train_run_slots
    pack = os.path.join(assets, "dog_slopes_mixed.trlpack")
    n = 1024
    sched = schedules()[0]
    sp = sp_array([sched])
    a = trl.ScenarioExpMACE(pack, n, rng_seed=9)
    ta = trl.MACETrainer(a, seed=3, **TRAINER)
    ca = comm1(a)
    ta.SetAsync(True)
    assert ta.L.trl_train_run(ta.h, sp.ctypes.data_as(C.c_void_p), UPDATES, ITERS, 32, C.c_double(DT)) == 0, ta.L.trl_last_error()
    b = trl.ScenarioExpMACE(pack, n, rng_seed=9)
    tb = trl.MACETrainer(b, seed=3, **TRAINER)
    cb = comm1(b)
    tb.SetAsync(True)
    train_run_slots([tb], [sched], UPDATES, ITERS, comm=cb, block_rows=1024)
    assert_trainer(ta, tb, "async slot 0")
    assert np.array_equal(np.stack(a.GetStateAll()), np.stack(b.GetStateAll()))
    ca.close(); cb.close()
    close(ta, tb, a, b)


# ------------------------------------------------------------------------------------------------ (6) refusals
def test_refusals_leave_the_handle_unchanged(assets, tmp_path):
    import deepterrainrl_b200 as trl
    from deepterrainrl_b200.train import train_run_slots
    pack = os.path.join(assets, "dog_slopes_mixed.trlpack")
    n = 256
    models = start_models(pack, str(tmp_path))[:2]
    scheds = schedules(curriculum=0)[:2]
    slots = assignment("blocks", n, 2)
    sc, trs = make_group(trl, pack, n, models, slots)
    L = sc.L
    sp = sp_array(scheds)
    arr = lambda ts: (C.c_void_p * len(ts))(*[t.h.value for t in ts])      # noqa: E731
    run = lambda ts, spx, ipu: L.trl_train_run_slots_comm(arr(ts), len(ts), spx.ctypes.data_as(C.c_void_p), 1, ipu, 32, 256,  # noqa: E731
                                                          C.c_double(DT))
    # without a communicator; asynchronous slot trainers need one
    assert run(trs, sp, 2) != 0 and b"no communicator" in L.trl_last_error()
    with pytest.raises(RuntimeError, match="training slots"):
        trs[1].SetAsync(True)
    comm = comm1(sc)
    on = sp.copy()
    on[:, 8] = 30
    on[1, 8] = 40
    trs[0].SetAsync(True)
    assert run(trs, sp, 2) != 0 and b"all or none" in L.trl_last_error()
    trs[1].SetAsync(True)
    assert run(trs, sp, 0) != 0 and b"fixed number" in L.trl_last_error()
    for t in trs:
        t.SetAsync(False)
    assert run(trs, on, 2) != 0 and b"trainer_curriculum_iters" in L.trl_last_error()
    with pytest.raises(RuntimeError, match="communicator"):
        sc.SaveCheckpoint(str(tmp_path / "ck.trl"))
    # the existing entries keep refusing a communicator
    assert L.trl_train_run_slots_sched(arr(trs), 2, sp.ctypes.data_as(C.c_void_p), 1, 2, 32, C.c_double(DT)) != 0
    assert b"communicator" in L.trl_last_error()
    assert not os.path.exists(tmp_path / "ck.trl")
    # the handle is unchanged: it trains as a fresh one
    clean, ctrs = make_group(trl, pack, n, models, slots)
    cc = comm1(clean)
    train_run_slots(trs, scheds, 8, ITERS, comm=comm, block_rows=n)
    train_run_slots(ctrs, scheds, 8, ITERS, comm=cc, block_rows=n)
    for p in range(2):
        assert_trainer(trs[p], ctrs[p], "after refusals, slot %d" % p)
    assert_envs(sc, [clean] * 2, slots, 90, stride=3)
    comm.close(); cc.close()
    close(*trs, *ctrs, sc, clean)
