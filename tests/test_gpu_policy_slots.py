"""Policy slots (trl_load_policy / trl_set_env_policy / trl_eval_stats_slot): one evaluation handle runs several models, each env
with the model of its slot.  The contract is exact: a mixed batch is the union of single-policy runs, env for env and bit for bit,
because no row of the decision pass depends on the other rows (tests/test_gpu_decide_batches.py) and the env-step is per env.

  * whole updates (falls, resets, overlapped / serial schedule, env groups) against one single-policy handle per model;
  * the decision pass at the batch shapes the slot build branches on (slot-ragged chunks, empty slots, more chunks than FC clusters)
    against torch f64 on each slot's own weights and against the same env decided in a single-policy pass;
  * per-slot statistics, the layer probe, reassignment between updates, and every refusal.
tests/test_policy_slots_cpu.py runs a miniature of the first two on the emulator."""
import os

import numpy as np
import pytest

import torch_net  # noqa: F401  (torch before the library: see tests/test_gpu_decide_batches.py)
from test_gpu_decide_batches import COUNTS, StatePool, _relerr, check_decision, edge_states, env_ids, opt_index

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "reference", "data", "policies", "raptor", "models")
UPDATES = 30                  # 600 env-steps: every env falls and resets at least once on these scenes
TOL = 1e-10


# ------------------------------------------------------------------------------------------------ shared helpers (also the CPU test's)
def pack_net(pack):
    from pack_scene import read_pack
    return torch_net.blobs_from_pack(read_pack(pack))


def write_net(path, net):
    """net = (blobs {layer: (w, b)} flat, in_off, in_scale, out_off, out_scale) -> Caffe-HDF5 + _scale.txt through the native writer"""
    from deepterrainrl_b200.model_io import write_model_native
    blobs, io, isc, oo, osc = net
    shaped = {k: (np.asarray(w).reshape(np.asarray(b).size, -1), np.asarray(b)) for k, (w, b) in blobs.items()}
    write_model_native(path, shaped, io, isc, oo, osc)
    return path


def perturbed(net, seed, rel=0.05):
    """the same topology with every weight and bias scaled by 1 + rel * N(0, 1): a different policy"""
    blobs, io, isc, oo, osc = net
    rng = np.random.default_rng(seed)
    out = {k: (w * (1 + rel * rng.standard_normal(w.shape)), b * (1 + rel * rng.standard_normal(b.shape))) for k, (w, b) in blobs.items()}
    return out, io, isc, oo, osc


def exported_model(trl, pack, path):
    """the policy of a handle of `pack`, written by trl_output_model"""
    sc = trl.ScenarioPoliEval(pack, 1)
    sc.OutputModel(path)
    sc.close()
    return path


def raptor_mixed_model(tmp_path):
    """raptor_mace3_mixed_model.h5, put back together from the parts committed under tests/golden/reference/"""
    path = os.path.join(tmp_path, "raptor_mace3_mixed_model.h5")
    with open(path, "wb") as f:
        for k in range(6):
            with open(os.path.join(GOLDEN, "raptor_mace3_mixed_model.h5.part%d" % k), "rb") as p:
                f.write(p.read())
    return path, os.path.join(GOLDEN, "raptor_mace3_mixed_model_scale.txt")


def assignment(pattern, n, n_slots, seed=0):
    """slot of every env: round robin, contiguous blocks, random, slot 0 left empty, the last loaded slot left unused"""
    if pattern == "round_robin":
        return np.arange(n) % n_slots
    if pattern == "blocks":
        return (np.arange(n) * n_slots) // n
    if pattern == "random":
        return np.random.default_rng(seed).integers(0, n_slots, n)
    if pattern == "no_slot0":
        return 1 + np.arange(n) % (n_slots - 1)
    if pattern == "unused_last":
        return np.arange(n) % (n_slots - 1)
    raise ValueError(pattern)


def env_record(sc, e, n_out):
    q, qd, tau, c = sc.GetState(e)
    return [q, qd, tau, c, sc.GetCtrl(e), sc.GetNetOut(e, n_out), sc.GetPoliState(e)]


def run_handle(trl, pack, n, models, slots, updates, rng_seed=77):
    """an evaluation handle of `pack`: models[0] (None = the pack's) in slot 0 via trl_load_model, models[p] in slot p, envs assigned by
    `slots` (None = no slot machinery: a single-policy handle); returns the handle after `updates` updates"""
    sc = trl.ScenarioPoliEval(pack, n, rng_seed=rng_seed)
    if models[0] is not None:
        sc.LoadModel(*models[0])
    for p, m in enumerate(models[1:], 1):
        if m is not None:
            sc.LoadPolicy(p, *m)
    if slots is not None:
        sc.SetEnvPolicy(slots)
    for _ in range(updates):
        sc.Update(1.0 / 30.0)
    sc.Sync()
    return sc


def assert_union(mixed, refs, slots, n_out):
    """env e of the mixed handle == env e of the single-policy handle of its slot: state, controller, decision, counters, distance log"""
    dist, denv = mixed.GetDistLog()
    ref_logs = [r.GetDistLog() if r is not None else None for r in refs]
    for e in range(mixed.num_envs):
        p = int(slots[e])
        got, want = env_record(mixed, e, n_out), env_record(refs[p], e, n_out)
        for k, (a, b) in enumerate(zip(got, want)):
            assert np.array_equal(a, b), ("env", e, "slot", p, "field", k)
    for p, ref in enumerate(refs):
        if ref is None:
            continue
        on = np.flatnonzero(slots == p)
        rd, re = ref_logs[p]
        for e in on[:: max(1, on.size // 256)]:      # the log is append-only in completion order: compare each env's own sequence
            assert np.array_equal(dist[denv == e], rd[re == e]), ("distance log", e, p)
        # per-slot statistics against the reference restricted to the same envs (episodes = its log entries, avg = their mean)
        st = mixed.GetEvalStats(p)
        keep = np.isin(re, on)
        assert st["episodes"] == int(keep.sum())
        assert st["cycles"] == int(sum(ref.GetCtrl(int(e))[-2] for e in on))
        assert st["steps"] == int(on.size) * (mixed.GetNumEnvSteps() // mixed.num_envs)
        if keep.any():
            want = float(np.mean(rd[keep]))
            assert abs(st["avg_dist"] - want) <= 1e-12 * max(1.0, abs(want))


# ------------------------------------------------------------------------------------------------ (1) whole updates
@pytest.fixture(scope="module")
def dog_models(tmp_path_factory, assets):
    import deepterrainrl_b200 as trl
    d = str(tmp_path_factory.mktemp("slots"))
    pack = os.path.join(assets, "dog_slopes_mixed.trlpack")
    goat = exported_model(trl, os.path.join(assets, "goat_cliffs.trlpack"), os.path.join(d, "goat.h5"))
    pert = write_net(os.path.join(d, "dog_perturbed.h5"), perturbed(pack_net(pack), 5))
    sc = os.path.splitext
    return pack, [None, (goat, sc(goat)[0] + "_scale.txt"), (pert, sc(pert)[0] + "_scale.txt")]


_REFS = {}


def refs_for(trl, pack, models, n, schedule):
    key = (pack, n, schedule)
    if key not in _REFS:
        _REFS.clear()
        _REFS[key] = [run_handle(trl, pack, n, [m], None, UPDATES) for m in models]
    return _REFS[key]


def _schedule(monkeypatch, schedule):
    monkeypatch.delenv("TRL_SERIAL_SCHEDULE", raising=False)
    monkeypatch.delenv("TRL_GROUPS", raising=False)
    if schedule == "serial":
        monkeypatch.setenv("TRL_SERIAL_SCHEDULE", "1")
    elif schedule == "groups3":
        monkeypatch.setenv("TRL_GROUPS", "3")


CASES = [(p, n, "overlap") for n in (4096, 1000) for p in ("round_robin", "blocks", "random", "no_slot0", "unused_last")]
CASES += [("random", 1000, "serial"), ("blocks", 1000, "groups3")]


@pytest.mark.parametrize("pattern,n,schedule", CASES)
def test_mixed_batch_is_the_union_of_single_policy_runs(dog_models, monkeypatch, pattern, n, schedule):
    import deepterrainrl_b200 as trl
    pack, models = dog_models
    _schedule(monkeypatch, schedule)
    refs = refs_for(trl, pack, models, n, schedule)
    slots = assignment(pattern, n, 3, seed=n)
    mixed = run_handle(trl, pack, n, models, slots, UPDATES)
    if n == 4096:
        assert sum(r.GetNumEpisodes() for r in refs) > 0      # some of the 4096 envs fall and reset inside the window compared
    assert_union(mixed, refs, slots, 90)
    mixed.close()


def test_raptor_two_slots(assets, tmp_path):
    import deepterrainrl_b200 as trl
    pack = os.path.join(assets, "raptor_narrow_gaps.trlpack")
    models = [None, raptor_mixed_model(str(tmp_path))]
    slots = assignment("random", 1000, 2, seed=3)
    refs = [run_handle(trl, pack, 1000, [m], None, UPDATES) for m in models]
    mixed = run_handle(trl, pack, 1000, models, slots, UPDATES)
    assert_union(mixed, refs, slots, 87)
    for e in (int(np.flatnonzero(slots == 0)[0]), int(np.flatnonzero(slots == 1)[0])):     # the layer probe follows the env's slot
        for name in ("terr_conv1", "concat0", "a1_ip0", "output"):
            assert np.array_equal(mixed.GetLayerState(name, e), refs[slots[e]].GetLayerState(name, e)), (name, e)


# ------------------------------------------------------------------------------------------------ (2) the decision pass
def _decide_sweep(trl, pack, n, nets, paths, n_out, cases):
    """cases: (ids, slots of those ids).  Mixed pass vs torch on each slot's weights and vs a single-policy pass of the same env"""
    special = edge_states(nets[0][1], nets[0][2], 2, 3)
    pool = StatePool(nets[0], n, special, seed=11)
    mixed = trl.ScenarioPoliEval(pack, n)
    for p, m in enumerate(paths[1:], 1):
        mixed.LoadPolicy(p, *m)
    singles = [trl.ScenarioPoliEval(pack, n) for _ in nets]
    for s, m in zip(singles, paths):
        if m is not None:
            s.LoadModel(*m)
    worst = 0.0
    for ids, sl in cases:
        ids = np.asarray(ids, np.int32)
        slots = np.zeros(n, np.int32)
        slots[ids] = sl
        mixed.SetEnvPolicy(slots)
        X = pool.X[pool.rows(ids)]
        mixed.DebugDecide(ids, X)
        for p, s in enumerate(singles):
            mine = ids[sl == p]
            s.DebugDecide(mine, X[sl == p])
        Ys = {p: torch_net.forward(*nets[p], X[sl == p]) for p in set(sl.tolist())}
        for k, e in enumerate(ids):
            p = int(sl[k])
            g = mixed.GetNetOut(int(e), n_out)
            t = Ys[p][int(np.flatnonzero(ids[sl == p] == e)[0])]
            worst = max(worst, _relerr(g, t))
            assert _relerr(g, t) <= TOL, ("torch", int(e), p, len(ids))
            assert np.array_equal(g, singles[p].GetNetOut(int(e), n_out)), ("single-policy pass", int(e), p)
            # the committed action: id and actor parameters (the rest of the controller block carries each handle's own history)
            got, want = mixed.GetCtrl(int(e)), singles[p].GetCtrl(int(e))
            sel = np.concatenate([[11], 12 + opt_index(mixed)])
            assert np.array_equal(got[sel], want[sel]), ("decision", int(e), p)
            check_decision(mixed, int(e), t, got)
    for s in singles + [mixed]:
        s.close()
    return worst


def slot_cases(n, n_slots, seed=0):
    rng = np.random.default_rng(seed)
    cases = []
    for c in sorted({min(c, n) for c in COUNTS if c > 0} | {n}):
        for order in ("identity", "permuted", "last"):
            ids = env_ids(order, c, n, seed)
            cases.append((ids, rng.integers(0, n_slots, c)))
    for k in (31, 32, 33, 63, 64, 65):                     # k rows in slot 1, a few around it in the others
        ids = env_ids("permuted", min(n, k + 20), n, k)
        sl = np.zeros(ids.size, np.int64)
        sl[:k] = 1
        sl[k:] = rng.choice([0, n_slots - 1], ids.size - k)
        cases.append((ids, sl))
    ids = env_ids("strided", min(n, 70), n, 1)
    cases.append((ids, np.full(ids.size, n_slots - 1)))       # every decision in the last slot, the others without one
    ids = env_ids("permuted", min(n, 7 * 33), n, 2)
    cases.append((ids, np.arange(ids.size) % n_slots))          # 7+ slot-chunks, more than the FC clusters
    return cases


def test_decision_pass_with_mixed_slots(assets, tmp_path):
    import deepterrainrl_b200 as trl
    pack = os.path.join(assets, "dog_slopes_mixed.trlpack")
    base = pack_net(pack)
    nets = [base] + [perturbed(base, s) for s in (1, 2, 3)]
    paths = [None] + [write_net(str(tmp_path / ("p%d.h5" % p)), nets[p]) for p in (1, 2, 3)]
    paths = [None] + [(p, os.path.splitext(p)[0] + "_scale.txt") for p in paths[1:]]
    worst = _decide_sweep(trl, pack, 1000, nets, paths, 90, slot_cases(1000, 4))
    assert worst <= TOL


# ------------------------------------------------------------------------------------------------ (4) reassignment, (5) refusals
def test_reassignment_takes_effect_at_the_next_decision(dog_models):
    """envs moved from slot 0 to slot 2 after 10 updates == a handle that had them on slot 2 from update 10 on; unmoved envs == slot 0"""
    import deepterrainrl_b200 as trl
    pack, models = dog_models
    n = 512
    a = run_handle(trl, pack, n, models, np.zeros(n, np.int32), 10)
    b = run_handle(trl, pack, n, models, np.zeros(n, np.int32), 10)
    moved = np.arange(0, n, 3)
    a.SetEnvPolicy(np.full(moved.size, 2), env_ids=moved)
    slots = np.zeros(n, np.int32)
    slots[moved] = 2
    b.SetEnvPolicy(slots)
    ref0 = run_handle(trl, pack, n, [None], None, 20)
    for _ in range(10):
        a.Update(1.0 / 30.0); b.Update(1.0 / 30.0)
    for e in range(n):
        assert all(np.array_equal(x, y) for x, y in zip(env_record(a, e, 90), env_record(b, e, 90))), e
    unmoved = np.setdiff1d(np.arange(n), moved)
    for e in unmoved[::7]:
        assert all(np.array_equal(x, y) for x, y in zip(env_record(a, int(e), 90), env_record(ref0, int(e), 90))), e
    # a moved env's next decision used slot 2's weights: its output differs from what slot 0 gives it
    assert any(not np.array_equal(a.GetNetOut(int(e), 90), ref0.GetNetOut(int(e), 90)) for e in moved)
    for s in (a, b, ref0):
        s.close()


def test_refusals_leave_the_handle_unchanged(dog_models, assets, tmp_path):
    import deepterrainrl_b200 as trl
    pack, models = dog_models
    n = 256
    raptor = raptor_mixed_model(str(tmp_path))
    sc = trl.ScenarioPoliEval(pack, n)
    sc.LoadPolicy(1, *models[2])
    slots = np.arange(n) % 2
    sc.SetEnvPolicy(slots)
    for call, msg in [(lambda: sc.LoadPolicy(0, *models[2]), "out of range"), (lambda: sc.LoadPolicy(8, *models[2]), "out of range"),
                      (lambda: sc.LoadPolicy(2, *raptor), "entries"), (lambda: sc.SetEnvPolicy([1], env_ids=[n]), "env id"),
                      (lambda: sc.SetEnvPolicy([0, 3]), "empty"), (lambda: sc.SetEnvPolicy([9]), "out of range")]:
        with pytest.raises(RuntimeError, match=msg):
            call()
    with pytest.raises(RuntimeError, match="policy slots"):
        trl.MACETrainer(sc, replay_mem_size=128, num_init_samples=64)
    ex = trl.ScenarioExpMACE(pack, 32)
    with pytest.raises(RuntimeError, match="evaluation handles"):
        ex.LoadPolicy(1, *models[2])
    ev = trl.ScenarioPoliEval(pack, 32)
    tr = trl.MACETrainer(ev, replay_mem_size=128, num_init_samples=64)
    with pytest.raises(RuntimeError, match="trainer"):
        ev.LoadPolicy(1, *models[2])
    del tr
    for _ in range(UPDATES):
        sc.Update(1.0 / 30.0)
    clean = run_handle(trl, pack, n, models[:3:2], slots, UPDATES)
    for e in range(0, n, 5):
        assert all(np.array_equal(x, y) for x, y in zip(env_record(sc, e, 90), env_record(clean, e, 90))), e
    for s in (sc, clean, ex, ev):
        s.close()
