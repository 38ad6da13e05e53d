"""Body slots (trl_load_body / trl_set_env_body / trl_env_body / trl_eval_stats_body): one handle runs each env on one of up to 8 bodies
of the scene's character.  The contract is exact: env i on body slot b computes, bit for bit, what env i computes in a handle created
from the same arguments plus `-character_file=<slot b's file>`.

The body variants are written from the committed dog, goat and raptor files into a temporary directory (`variants`): heavier torso,
longer legs (attach points and box lengths together), weaker motors, narrower joint limits, other PD targets and damping, and an
unmodified copy.  Together they change every per-link number a body slot holds.

  1. whole updates of dog (6 bodies), raptor (3) and goat (2) scenes under several assignments and schedules, in evaluation and in
     exploration, against one single-body handle per file; the per-body statistics; the unmodified copy equals slot 0;
  2. a policy x terrain x body cube (with a physics slot beside it) against the eight single handles, with every statistics cell;
  3. the "next reset" rule across a fall, trl_reset and a reseed; reloading a slot in use is refused, a free one is not;
  4. two handles alternated, each equal to its own run alone;
  5. a checkpoint with body, physics and terrain slots resumes bit for bit; a handle without body slots writes the same file as before;
  6. every refusal leaves the handle unchanged.
tests/test_body_slots_cpu.py runs a miniature on the emulator, and the loader checks without a GPU."""
import copy
import json
import os

import numpy as np
import pytest

import torch_net  # noqa: F401  (torch before the library: see tests/test_gpu_decide_batches.py)
from test_gpu_policy_slots import assignment, pack_net, perturbed, write_net
from test_gpu_terrain_slots import (_run, _run_with_falls, _schedule, assert_same_env, data_root, scene_args, terrain_path,
                                    tuples_by_env)

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
UPDATES = 30
TERRAIN = {"dog": "slopes_mixed", "raptor": "mixed_raptor", "goat": "cliffs_rugged"}
# thigh and shin of every leg (their bodies and the joints below them grow together in the "long" variant)
LEGS = {"dog": (13, 14, 17, 18), "goat": (13, 14, 17, 18), "raptor": (11, 12, 15, 16)}
VARIANTS = ["heavy", "long", "weak", "narrow", "targets", "copy"]
BODIES = {"dog": ["heavy", "long", "weak", "narrow", "targets"], "raptor": ["narrow", "targets"], "goat": ["long"]}   # slots 1..; slot 0 is the scene's file


# ------------------------------------------------------------------------------------------------ body variants (also the CPU test's)
def variant(char, kind):
    """the character file of `char` (a parsed dog / goat / raptor file) changed as `kind` says"""
    c = copy.deepcopy(char)
    J, B, P = c["Skeleton"]["Joints"], c["BodyDefs"], c["PDControllers"]
    name = "raptor" if len(J) == 19 else "dog"
    if kind == "heavy":
        heaviest = max(range(len(B)), key=lambda j: B[j]["Mass"])
        B[heaviest]["Mass"] *= 1.3
        B[heaviest]["Theta"] = B[heaviest].get("Theta", 0.0) + 0.03     # body_cos / body_sin and the corners
    elif kind == "long":
        legs = LEGS[name]
        for j in legs:
            for k in ("AttachX", "AttachY", "Param0", "Param1"):
                B[j][k] *= 1.1
        for j, jt in enumerate(J):
            if jt["Parent"] in legs:
                jt["AttachX"] *= 1.1
                jt["AttachY"] *= 1.1
    elif kind == "weak":
        for p in P:
            p["TorqueLim"] *= 0.7
            p["Kp"] *= 0.8
    elif kind == "narrow":
        for jt in J[1:]:
            lo, hi = jt.get("LimLow", 1), jt.get("LimHigh", 0)
            if lo <= hi:
                mid, half = 0.5 * (lo + hi), 0.5 * (hi - lo)
                jt["LimLow"], jt["LimHigh"] = mid - 0.8 * half, mid + 0.8 * half
    elif kind == "targets":
        for p in P[1:]:
            p["TargetTheta"] = p.get("TargetTheta", 0.0) + 0.05
            p["TargetVel"] = p.get("TargetVel", 0.0) + 0.1
            p["Kd"] *= 1.2
        P[-1]["UseWorldCoord"] = 0 if P[-1].get("UseWorldCoord", 0) else 1
    elif kind != "copy":
        raise ValueError(kind)
    return c


def write_variants(root, dst):
    """{(character, kind): path} of every variant of the committed dog, goat and raptor files, written under dst"""
    out = {}
    for ch in ("dog", "goat", "raptor"):
        with open(os.path.join(root, "data", "characters", ch + ".txt")) as f:
            base = json.load(f)
        # controller files by absolute path: the variants load into handles made from packs too, which have no data root
        base["Controllers"]["Files"] = [os.path.join(root, x) for x in base["Controllers"]["Files"]]
        for kind in VARIANTS:
            p = os.path.join(dst, "%s_%s.txt" % (ch, kind))
            with open(p, "w") as f:
                json.dump(variant(base, kind), f)
            out[ch, kind] = p
    return out


def body_files(root, var, scene):
    """the files of the slots of `scene`: its own character file, then its variants"""
    return [os.path.join(root, "data", "characters", scene + ".txt")] + [var[scene, k] for k in BODIES[scene]]


def make_body_handle(trl, scene, root, model, files, n, slots, explore=False, extra=(), seeds=None, rng_seed=77, terrain=None):
    """a handle of `scene` created with files[0]; files[1:] loaded into body slots 1.., envs assigned by `slots` and then reseeded (so
    that every env starts on its own body, as a fresh handle of that file does)"""
    cls = trl.ScenarioExpMACE if explore else trl.ScenarioPoliEval
    args = scene_args(scene, terrain or TERRAIN[scene], model, ["-character_file=", files[0]] + list(extra))
    sc = cls(None, n, args=args, data_root=root, rng_seed=rng_seed, terrain_seeds=seeds)
    for b, f in enumerate(files[1:], 1):
        sc.LoadBody(b, f)
    if slots is not None:
        sc.SetEnvBody(slots)
        sc.SetRandSeed(np.arange(1, n + 1, dtype=np.uint64) if seeds is None else seeds)
    if explore:
        sc.EnableExplore(1, 0.3, 0.5, 0.05)
    return sc


def assert_body_union(mixed, refs, slots, n_out, stride=1):
    """env e of `mixed` == env e of refs[slots[e]], its distance-log entries included"""
    dist, denv = mixed.GetDistLog()
    logs = [r.GetDistLog() for r in refs]
    cur, nxt = mixed.EnvBody()
    assert np.array_equal(nxt, np.asarray(slots))
    for e in range(0, mixed.num_envs, stride):
        b = int(slots[e])
        assert_same_env(mixed, e, refs[b], e, n_out, "body %d" % b)
        rd, re = logs[b]
        assert np.array_equal(dist[denv == e], rd[re == e]), ("distance log", e, b)
    assert np.array_equal(cur, np.asarray(slots)), "every env is on its assigned body after the reseed"


@pytest.fixture(scope="module")
def ref_root(tmp_path_factory, assets):
    import deepterrainrl_b200 as trl
    d = str(tmp_path_factory.mktemp("body_slots"))
    root, models = data_root(trl, assets, d)
    return root, models, write_variants(root, d)


def body_stats(sc, mode, p, t, q, b):
    import ctypes as C
    c = C.c_int64(0); e = C.c_int64(0); a = C.c_double(0); s = C.c_int64(0)
    sc._ck(sc.L.trl_eval_stats_body(sc.h, int(mode), int(p), int(t), int(q), int(b), C.byref(c), C.byref(e), C.byref(a), C.byref(s)))
    return dict(cycles=c.value, episodes=e.value, avg_dist=a.value, steps=s.value)


def n_out_of(scene):
    return 87 if scene == "raptor" else 90


# ------------------------------------------------------------------------------------------------ (1) union of single-body handles
CASES = [("dog", p, 1024, "overlap") for p in ("round_robin", "blocks", "random", "no_slot0")]
CASES += [("dog", "random", 1024, "serial"), ("dog", "blocks", 1024, "groups3")]
CASES += [("raptor", "random", 768, "overlap"), ("raptor", "no_slot0", 768, "serial"), ("goat", "round_robin", 512, "overlap"),
          ("goat", "random", 512, "groups3")]


@pytest.mark.parametrize("scene,pattern,n,schedule", CASES)
def test_mixed_batch_is_the_union_of_single_body_runs(ref_root, monkeypatch, scene, pattern, n, schedule):
    import deepterrainrl_b200 as trl
    root, models, var = ref_root
    _schedule(monkeypatch, schedule)
    files = body_files(root, var, scene)
    slots = assignment(pattern, n, len(files), seed=n)
    refs = [_run_with_falls(make_body_handle(trl, scene, root, models[scene], [f], n, None), UPDATES, n) for f in files]
    mixed = _run_with_falls(make_body_handle(trl, scene, root, models[scene], files, n, slots), UPDATES, n)
    assert all(r.GetNumEpisodes() > 0 for r in refs)
    assert_body_union(mixed, refs, slots, n_out_of(scene))
    for b in range(len(files)):                                # per-body statistics against the single handles' envs
        on = np.flatnonzero(slots == b)
        st = mixed.GetEvalStats(None, body=b)
        rd, re = refs[b].GetDistLog()
        keep = np.isin(re, on)
        assert st["episodes"] == int(keep.sum())
        assert st["cycles"] == int(sum(refs[b].GetCtrl(int(e))[-2] for e in on))
        if keep.any():
            assert abs(st["avg_dist"] - float(np.mean(rd[keep]))) <= 1e-12 * max(1.0, abs(float(np.mean(rd[keep]))))
        d, de = mixed.GetDistLog(body=b)
        assert np.array_equal(np.sort(de), np.sort(re[keep]))
    assert mixed.GetEvalStats(None, body=None) == mixed.GetEvalStats(None)
    for sc in refs + [mixed]:
        sc.close()


@pytest.mark.parametrize("schedule", ["overlap", "serial", "groups3"])
def test_exploration_tuples_are_the_union(ref_root, monkeypatch, schedule):
    import deepterrainrl_b200 as trl
    root, models, var = ref_root
    _schedule(monkeypatch, schedule)
    files = body_files(root, var, "dog")
    n = 512
    slots = assignment("random", n, len(files), seed=9)
    refs = [_run(make_body_handle(trl, "dog", root, models["dog"], [f], n, None, explore=True), UPDATES) for f in files]
    mixed = _run(make_body_handle(trl, "dog", root, models["dog"], files, n, slots, explore=True), UPDATES)
    assert_body_union(mixed, refs, slots, 90, stride=3)
    r, f, e = tuples_by_env(mixed)
    assert r.shape[0] > 0
    for b, ref in enumerate(refs):
        rr, rf, re = tuples_by_env(ref)
        keep = np.isin(re, np.flatnonzero(slots == b))
        mine = slots[e] == b
        assert np.array_equal(e[mine], re[keep]) and np.array_equal(f[mine], rf[keep]), b
        assert np.array_equal(r[mine], rr[keep]), b
    for sc in refs + [mixed]:
        sc.close()


def test_unmodified_copy_is_slot_zero(ref_root):
    import deepterrainrl_b200 as trl
    root, models, var = ref_root
    n = 256
    slots = np.arange(n) % 2
    files = body_files(root, var, "dog")[:1] + [var["dog", "copy"]]
    mixed = _run_with_falls(make_body_handle(trl, "dog", root, models["dog"], files, n, slots), UPDATES, n)
    ref = _run_with_falls(make_body_handle(trl, "dog", root, models["dog"], files[:1], n, None), UPDATES, n)
    for e in range(n):
        assert_same_env(mixed, e, ref, e, 90, "copy")
    assert mixed.GetEvalStats(None) == ref.GetEvalStats(None)
    for sc in (mixed, ref):
        sc.close()


# ------------------------------------------------------------------------------------------------ (2) policy x terrain x body
@pytest.mark.parametrize("with_physics", [False, True])
def test_policy_by_terrain_by_body_cube(ref_root, tmp_path, with_physics):
    import deepterrainrl_b200 as trl
    root, models, var = ref_root
    base = pack_net(os.path.join(ROOT, "assets", "dog_slopes_mixed.trlpack"))
    net = write_net(str(tmp_path / "p1.h5"), perturbed(base, 1))
    pol = [None, (net, os.path.splitext(net)[0] + "_scale.txt")]
    terrains = ["slopes_mixed", "tight_gaps"]
    files = [body_files(root, var, "dog")[0], var["dog", "long"]]
    phys = [2.0e5, 2.0e3, 0.5, 0.01, 0.00025, 2.0e4, 20.0]
    n = 1024
    rng = np.random.default_rng(11)
    ps, ts, bs = rng.integers(0, 2, n), rng.integers(0, 2, n), rng.integers(0, 2, n)
    qs = bs if with_physics else np.zeros(n, np.int64)        # physics slot 1 rides with body slot 1
    mixed = make_body_handle(trl, "dog", root, models["dog"], files, n, None)
    mixed.LoadTerrain(1, terrain_path(root, terrains[1]))
    mixed.LoadPolicy(1, *pol[1])
    if with_physics:
        mixed.LoadPhysics(1, phys)
        mixed.SetEnvPhysics(qs)
    mixed.SetEnvPolicy(ps); mixed.SetEnvTerrain(ts); mixed.SetEnvBody(bs)
    mixed.SetRandSeed(np.arange(1, n + 1, dtype=np.uint64))
    _run_with_falls(mixed, UPDATES, n)
    singles = {}
    for p in range(2):
        for t in range(2):
            for b in range(2):
                sc = make_body_handle(trl, "dog", root, models["dog"], [files[b]], n, None, terrain=terrains[t])
                if pol[p] is not None:
                    sc.LoadModel(*pol[p])
                if with_physics and b == 1:
                    sc.SetPhysParams(phys)
                singles[p, t, b] = _run_with_falls(sc, UPDATES, n)
    for e in range(n):
        assert_same_env(mixed, e, singles[int(ps[e]), int(ts[e]), int(bs[e])], e, 90, ("cell", int(ps[e]), int(ts[e]), int(bs[e])))
    logs = {k: s.GetDistLog() for k, s in singles.items()}
    steps = mixed.GetNumEnvSteps() // n
    for p in (-1, 0, 1):
        for t in (-1, 0, 1):
            for q in ((-1, 0, 1) if with_physics else (-1,)):
                for b in (-1, 0, 1):
                    on = np.flatnonzero(((ps == p) | (p < 0)) & ((ts == t) | (t < 0)) & ((qs == q) | (q < 0)) & ((bs == b) | (b < 0)))
                    d = np.concatenate([logs[int(ps[e]), int(ts[e]), int(bs[e])][0][logs[int(ps[e]), int(ts[e]), int(bs[e])][1] == e]
                                        for e in on] + [np.zeros(0)])
                    st = body_stats(mixed, -1, p, t, q, b)
                    assert st["episodes"] == d.size, (p, t, q, b)
                    assert st["cycles"] == int(sum(singles[int(ps[e]), int(ts[e]), int(bs[e])].GetCtrl(int(e))[-2] for e in on)), (p, t, q, b)
                    assert st["steps"] == on.size * steps, (p, t, q, b)
                    if d.size:
                        assert abs(st["avg_dist"] - float(np.mean(d))) <= 1e-12 * max(1.0, abs(float(np.mean(d)))), (p, t, q, b)
                    if b >= 0 and q < 0:     # the Python filter takes the same route
                        assert st == mixed.GetEvalStats(None if p < 0 else p, terrain=None if t < 0 else t, body=b), (p, t, b)
    for sc in list(singles.values()) + [mixed]:
        sc.close()


# ------------------------------------------------------------------------------------------------ (3) the next-reset rule
def test_assignment_takes_effect_at_the_next_reset(ref_root):
    import deepterrainrl_b200 as trl
    from test_gpu_terrain_slots import tip_over
    root, models, var = ref_root
    n = 64
    files = body_files(root, var, "dog")
    sc = make_body_handle(trl, "dog", root, models["dog"], files, n, None)
    assert all(np.array_equal(x, np.zeros(n)) for x in sc.EnvBody())
    sc.SetEnvBody(np.full(n, 2, np.int32))
    cur, nxt = sc.EnvBody()
    assert np.array_equal(cur, np.zeros(n)) and np.array_equal(nxt, np.full(n, 2))
    _run(sc, 2)
    assert np.array_equal(sc.EnvBody()[0], np.zeros(n)), "no reset: the present episode keeps its body"
    tip_over(sc, [3, 9])                                     # a fall inside the update
    _run(sc, 1)
    cur = sc.EnvBody()[0]
    assert cur[3] == 2 and cur[9] == 2 and np.count_nonzero(cur) == 2
    with pytest.raises(RuntimeError, match="in use"):
        sc.LoadBody(2, var["dog", "narrow"])                 # present body of envs 3 and 9, assigned body of every env
    sc.Reset([5])                                            # trl_reset
    assert sc.EnvBody()[0][5] == 2
    sc.SetEnvBody(np.ones(n, np.int32))
    with pytest.raises(RuntimeError, match="in use"):
        sc.LoadBody(2, var["dog", "narrow"])                 # still the present body of envs 3, 5, 9
    sc.SetRandSeed(np.arange(1, n + 1, dtype=np.uint64))     # trl_seed_terrain resets every env
    assert all(np.array_equal(x, np.ones(n)) for x in sc.EnvBody())
    sc.LoadBody(2, var["dog", "narrow"])                     # free again: reloaded, then assigned
    sc.SetEnvBody(np.full(n, 2, np.int32))
    sc.SetRandSeed(np.arange(1, n + 1, dtype=np.uint64))
    _run(sc, 3)
    ref = _run(make_body_handle(trl, "dog", root, models["dog"], [var["dog", "narrow"]], n, None), 3)
    for e in range(n):
        assert_same_env(sc, e, ref, e, 90, "reloaded slot")
    sc.close(); ref.close()


# ------------------------------------------------------------------------------------------------ (4) two handles alternated
def test_two_handles_alternated(ref_root):
    import deepterrainrl_b200 as trl
    root, models, var = ref_root
    n = 256
    a_files = body_files(root, var, "dog")
    b_files = body_files(root, var, "raptor")
    sa, sb = assignment("random", n, len(a_files), 3), assignment("random", n, len(b_files), 4)
    alone_a = _run_with_falls(make_body_handle(trl, "dog", root, models["dog"], a_files, n, sa), UPDATES, n)
    alone_b = _run_with_falls(make_body_handle(trl, "raptor", root, models["raptor"], b_files, n, sb), UPDATES, n)
    a = make_body_handle(trl, "dog", root, models["dog"], a_files, n, sa)
    b = make_body_handle(trl, "raptor", root, models["raptor"], b_files, n, sb)
    for k in range(UPDATES):
        if k == UPDATES // 10:
            from test_gpu_terrain_slots import tip_over
            tip_over(a, range(0, n, 16)); tip_over(b, range(0, n, 16))
        a.Update(1.0 / 30.0)
        b.Update(1.0 / 30.0)
    a.Sync(); b.Sync()
    for e in range(n):
        assert_same_env(a, e, alone_a, e, 90, "dog alternated")
        assert_same_env(b, e, alone_b, e, 87, "raptor alternated")
    for sc in (a, b, alone_a, alone_b):
        sc.close()


# ------------------------------------------------------------------------------------------------ (5) checkpoints
def test_checkpoint_round_trip(ref_root, tmp_path):
    import deepterrainrl_b200 as trl
    from test_gpu_checkpoint import assert_refused, damaged_copies
    root, models, var = ref_root
    n = 256
    files = body_files(root, var, "dog")
    slots = assignment("random", n, len(files), 5)

    def build():
        sc = make_body_handle(trl, "dog", root, models["dog"], files, n, slots, explore=True)
        sc.LoadTerrain(1, terrain_path(root, "flat"))
        sc.LoadPhysics(1, [2.0e5, 2.0e3, 0.5, 0.01, 0.00025, 2.0e4, 20.0])
        sc.SetEnvTerrain(np.arange(n) % 2)
        sc.SetEnvPhysics((np.arange(n) // 2) % 2)
        sc.SetEnvBody(assignment("random", n, len(files), 6))     # assignments that differ from the present bodies
        return sc
    a = build()
    _run(a, 4)
    _run(a, 4)
    b = build()
    _run(b, 4)
    path = str(tmp_path / "body.ckpt")
    b.SaveCheckpoint(path)
    b.close()
    c, _, _ = trl.load_checkpoint(path)
    assert all(np.array_equal(x, y) for x, y in zip(c.EnvBody(), a.EnvBody()))
    _run(c, 4)
    for e in range(n):
        assert_same_env(a, e, c, e, 90, "resumed")
    ra, fa, ea = tuples_by_env(a)
    rc, fc, ec = tuples_by_env(c)
    assert np.array_equal(ra, rc) and np.array_equal(fa, fc) and np.array_equal(ea, ec)
    d = tmp_path / "bad"
    d.mkdir()
    flipped = [(p, msg) for p, msg in damaged_copies(path, str(d)) if "body" in msg]
    assert len(flipped) == 4                                  # body_loaded, body_table, env_body_host, env_body
    for p, msg in flipped:
        assert_refused(trl.load_library(), p, msg)
    a.close(); c.close()


def test_checkpoint_without_body_slots_is_unchanged(ref_root, tmp_path):
    """the body-slot sections are written only once a body slot is loaded: a handle without one writes the sections it wrote before"""
    import deepterrainrl_b200 as trl
    from deepterrainrl_b200.checkpoint import sections
    root, models, var = ref_root
    sc = make_body_handle(trl, "dog", root, models["dog"], body_files(root, var, "dog")[:1], 64, None)
    _run(sc, 2)
    path = str(tmp_path / "plain.ckpt")
    sc.SaveCheckpoint(path)
    assert not [s for s in sections(path) if "body" in s[0]]
    sc.close()


# ------------------------------------------------------------------------------------------------ (6) refusals
def test_refusals_leave_the_handle_unchanged(ref_root, tmp_path):
    import deepterrainrl_b200 as trl
    root, models, var = ref_root
    n = 128
    files = body_files(root, var, "dog")[:2]
    slots = np.arange(n) % 2
    ref = _run(make_body_handle(trl, "dog", root, models["dog"], files, n, slots), 3)
    sc = make_body_handle(trl, "dog", root, models["dog"], files, n, slots)
    with open(files[0]) as f:
        dog = json.load(f)
    malformed = str(tmp_path / "malformed.txt")
    with open(malformed, "w") as f:
        f.write(json.dumps(dog)[:-40])

    def bad(name, edit):
        c = copy.deepcopy(dog)
        edit(c)
        p = str(tmp_path / (name + ".txt"))
        with open(p, "w") as f:
            f.write(json.dumps(c).replace('"__inf__"', "1e999"))
        return p
    cases = [
        (lambda: sc.LoadBody(0, files[1]), "out of range"),
        (lambda: sc.LoadBody(8, files[1]), "out of range"),
        (lambda: sc.LoadBody(3, str(tmp_path / "missing.txt")), "trl_load_body"),
        (lambda: sc.LoadBody(3, var["dog", "copy"].replace("copy", "none")), "trl_load_body"),
        (lambda: sc.LoadBody(3, malformed), "trl_load_body"),
        (lambda: sc.LoadBody(3, var["goat", "copy"]), "Controllers"),
        (lambda: sc.LoadBody(3, var["raptor", "copy"]), "topology"),
        (lambda: sc.LoadBody(3, bad("parent", lambda c: c["Skeleton"]["Joints"][20].update(Parent=17))), "topology"),
        (lambda: sc.LoadBody(3, bad("shape", lambda c: c["BodyDefs"][4].update(Shape="capsule"))), "topology"),
        (lambda: sc.LoadBody(3, bad("actions", lambda c: c["Controllers"]["Actions"].pop())), "Controllers"),
        (lambda: sc.LoadBody(3, bad("gravity", lambda c: c["Controllers"].update(EnableGravityCompensation=False))), "Controllers"),
        (lambda: sc.LoadBody(3, bad("inf", lambda c: c["BodyDefs"][3].update(Mass="__inf__"))), "not finite"),
        (lambda: sc.LoadBody(3, bad("mass", lambda c: c["BodyDefs"][3].update(Mass=0.0))), "Mass"),
        (lambda: sc.LoadBody(3, bad("box", lambda c: c["BodyDefs"][3].update(Param1=-0.1))), "box size"),
        (lambda: sc.LoadBody(3, bad("kp", lambda c: c["PDControllers"][3].update(Kp=-1.0))), "negative"),
        (lambda: sc.LoadBody(3, bad("kd", lambda c: c["PDControllers"][3].update(Kd=-1.0))), "negative"),
        (lambda: sc.LoadBody(3, bad("tlim", lambda c: c["PDControllers"][3].update(TorqueLim=-1.0))), "negative"),
        (lambda: sc.LoadBody(3, bad("reach", lambda c: c["BodyDefs"][20].update(Param0=3.0))), "reaches"),
        (lambda: sc.LoadBody(1, var["dog", "weak"]), "in use"),
        (lambda: sc.SetEnvBody([3]), "empty"),
        (lambda: sc.SetEnvBody([8]), "out of range"),
        (lambda: sc.SetEnvBody([1], env_ids=[n]), "env id"),
        (lambda: sc.SetEnvBody(np.zeros(n + 1, np.int32)), "env count"),
        (lambda: sc.GetEvalStats(None, body=3), "empty"),
        (lambda: sc.GetEvalStats(None, body=8), "out of range"),
    ]
    for call, msg in cases:
        with pytest.raises(RuntimeError, match=msg):
            call()
    assert np.array_equal(sc.EnvBody()[1], slots)
    _run(sc, 3)
    for e in range(n):
        assert_same_env(sc, e, ref, e, 90, "after the refusals")
    sc.close(); ref.close()


# ------------------------------------------------------------------------------------------------ a body change at a fall inside an update
def test_body_changes_at_a_fall_inside_an_update(ref_root):
    """envs tipped over right after a reseed fall at the end of the first update; those assigned another body restage their tables
    inside the step kernel and start the next episode on it.  Their ground and random streams have not moved yet, so from that reset on
    they must run as the same envs of a handle created with the new body's file, tipped over the same way"""
    import deepterrainrl_b200 as trl
    from test_gpu_terrain_slots import tip_over
    root, models, var = ref_root
    n = 256
    files = [body_files(root, var, "dog")[0], var["dog", "long"]]
    nxt = (np.arange(n) % 2).astype(np.int32)
    mixed = make_body_handle(trl, "dog", root, models["dog"], files, n, None)
    mixed.SetEnvBody(nxt)
    refs = [make_body_handle(trl, "dog", root, models["dog"], [f], n, None) for f in files]
    for sc in [mixed] + refs:
        tip_over(sc, range(n))
        _run(sc, 1)
    cur = mixed.EnvBody()[0]
    switched = np.flatnonzero(cur == 1)
    assert switched.size > n // 4 and np.array_equal(cur[switched], nxt[switched])
    for sc in [mixed] + refs:
        _run(sc, 8)
    for e in range(n):
        b = int(cur[e])
        ra, rb = env_state(mixed, e), env_state(refs[b], e)
        for k, (x, y) in enumerate(zip(ra, rb)):
            assert np.array_equal(x, y), ("env", e, "body", b, "field", k)
    for sc in [mixed] + refs:
        sc.close()


def env_state(sc, e):
    """state, held torques, contacts, policy state and both terrain segments (no episode statistics: the episodes before the fall ran
    on different bodies)"""
    q, qd, tau, c = sc.GetState(e)
    rec = [q, qd, tau, c, sc.GetNetOut(e, 90), sc.GetPoliState(e)]
    for seg in (0, 1):
        d, mx, fl = sc.GetTerrain(e, seg)
        rec += [d, np.array([mx, fl])]
    return rec


# ------------------------------------------------------------------------------------------------ against the oracle
def body_pack(trl, root, model, f, dst):
    """the pack trl_pack_from_args makes of the dog / slopes_mixed arguments with -character_file=f"""
    p = os.path.join(dst, os.path.basename(f) + ".trlpack")
    if not os.path.exists(p):
        trl.pack_from_args(scene_args("dog", "slopes_mixed", model, ["-character_file=", f]), root, p)
    return p


def test_free_running_against_oracle(ref_root, tmp_path):
    import deepterrainrl_b200 as trl
    from pyoracle import Oracle
    root, models, var = ref_root
    files = body_files(root, var, "dog")
    packs = [body_pack(trl, root, models["dog"], f, str(tmp_path)) for f in files]
    n = 60
    h = 1.0 / 600.0
    seeds = np.arange(101, 101 + n, dtype=np.uint64)
    slots = np.arange(n) % len(files)
    g = trl.ScenarioPoliEval(packs[0], n, terrain_seeds=seeds)
    for b, f in enumerate(files[1:], 1):
        g.LoadBody(b, f)
    g.SetEnvBody(slots)
    g.SetRandSeed(seeds)
    orc = [Oracle(p, n, 0, terrain_seeds=seeds) for p in packs]
    worst = 0.0
    for k in range(600):
        g.EnvStep(h)
        for e in range(n):
            orc[slots[e]].env_step(e, h)
        if k % 50 == 49:
            for e in range(n):
                gq, gqd, _, _ = g.GetState(e)
                oq, oqd, _, _ = orc[slots[e]].get_state(e)
                err = max(np.max(np.abs(gq - oq) / (1 + np.abs(oq))), np.max(np.abs(gqd - oqd) / (1 + np.abs(oqd))))
                worst = max(worst, err)
                assert err < 1e-4, (k, e, slots[e])
    print("body slots vs oracle, 600 env-steps: worst rel err %.3e" % worst)
    g.close()


# ------------------------------------------------------------------------------------------------ training
TRAIN_BODIES = ["heavy", "weak"]          # slots 1, 2; slot 0 is dog.txt


@pytest.mark.parametrize("paced", [False, True])
def test_training_slots_on_their_own_bodies(ref_root, tmp_path, paced):
    """three training slots whose envs run on three bodies (body slot = policy slot) against single-trainer handles created from each
    body's file and fed only their slot's tuples"""
    import deepterrainrl_b200 as trl
    from deepterrainrl_b200.train import TrainSchedule, train_run_slots
    from test_gpu_train_schedules import ref_loop_paced
    from test_gpu_train_slots import SCHEDULE, assert_envs, assert_trainer, close, make_group, make_ref, ref_loop, start_models
    root, models, var = ref_root
    files = body_files(root, var, "dog")[:1] + [var["dog", k] for k in TRAIN_BODIES]
    packs = [body_pack(trl, root, models["dog"], f, str(tmp_path)) for f in files]
    n = 2048
    tm = start_models(packs[0], str(tmp_path))
    slots = assignment("random", n, 3, seed=1)

    def group_setup(sc):
        for b in (1, 2):
            sc.LoadBody(b, files[b])
        sc.SetEnvBody(slots)          # the resets of trl_set_env_policy make them current

    sched = TrainSchedule(**dict(SCHEDULE, trainer_curriculum_iters=0))
    updates = 60          # every slot's replay memory fills past num_init_samples, so each trainer iterates
    group, trs = make_group(trl, packs[0], n, tm, slots, setup=group_setup)
    train_run_slots(trs, sched, updates, None if paced else 2)
    refs = []
    for p in range(3):
        sc, tr = make_ref(trl, packs[p], n, tm, p, slots)
        if paced:
            ref_loop_paced(sc, tr, p, slots, sched, updates)
        else:
            ref_loop(sc, tr, p, slots, sched, updates, 2)
        refs.append((sc, tr))
    assert np.array_equal(group.EnvBody()[0], slots)
    for p in range(3):
        assert trs[p].counters()["iter"] > 0
        assert_trainer(trs[p], refs[p][1], "slot %d" % p)
    assert_envs(group, [r[0] for r in refs], slots, 90, stride=2)
    close(*trs, group, *[o for r in refs for o in r])


def test_one_trainer_over_four_bodies_is_reproducible(ref_root, monkeypatch):
    import deepterrainrl_b200 as trl
    from deepterrainrl_b200.train import TrainSchedule
    from test_gpu_checkpoint import sp_of, train_run
    from test_gpu_train_slots import SCHEDULE, TRAINER, assert_trainer, close
    root, models, var = ref_root
    files = body_files(root, var, "dog")[:4]
    n = 1024
    slots = np.arange(n) % 4
    sp = sp_of(TrainSchedule(**SCHEDULE))
    out = []
    for schedule in ("overlap", "overlap", "serial", "groups3"):
        _schedule(monkeypatch, schedule)
        sc = make_body_handle(trl, "dog", root, models["dog"], files, n, slots, explore=True, rng_seed=5)
        tr = trl.MACETrainer(sc, seed=3, **TRAINER)
        train_run(tr, sp, 30, 2)
        out.append((sc, tr))
    a, ta = out[0]
    assert ta.counters()["iter"] > 0
    assert np.array_equal(a.EnvBody()[0], slots)
    for b, tb in out[1:]:
        assert_trainer(ta, tb, "reproducible")
        for e in range(0, n, 7):
            assert_same_env(a, e, b, e, 90, "reproducible")
    close(*[o for r in out for o in r[::-1]])


def test_evaluation_envs_beside_body_slots(ref_root, assets, tmp_path):
    """evaluation envs of a body-slot exploration handle against the single-trainer and evaluation references (with the same bodies), and
    every (mode, policy, body) statistics cell: the mode and body filters of the statistics kernel together"""
    import deepterrainrl_b200 as trl
    from test_gpu_eval_envs import EXPLORE, POLI_EVAL, TIPS, UPDATES as EV_UPDATES, Run, eval_mask, expected_cell
    from test_gpu_train_slots import start_models
    root, models, var = ref_root
    pack = os.path.join(assets, "dog_slopes_mixed.trlpack")
    n = 768
    body = (np.arange(n) // 2) % 3

    def ev_setup(sc):
        sc.LoadBody(1, var["dog", "heavy"])
        sc.LoadBody(2, var["dog", "targets"])
        sc.SetEnvBody(body)
        sc.Reset()

    tm = start_models(pack, str(tmp_path))[:2]
    run = Run(trl, pack, n, tm, assignment("blocks", n, 2), eval_mask("random", n, seed=9), setup=ev_setup, tips=TIPS)
    for _ in range(EV_UPDATES):
        run.step()
    run.check(90, stride=2)
    g = run.g
    assert np.array_equal(g.EnvBody()[0], body)
    for mode in (POLI_EVAL, EXPLORE):
        for p in (-1, 0, 1):
            for b in (-1, 0, 1, 2):
                st = g.GetEvalStats(None if p < 0 else p, body=None if b < 0 else b, mode=mode)
                c, e, ds = expected_cell(run, mode, p, q_of=body, q=b)
                assert (st["cycles"], st["episodes"]) == (c, e), (mode, p, b)
                if mode == POLI_EVAL:
                    assert e > 0, (p, b)
                    assert abs(st["avg_dist"] - ds / e) <= 1e-12 * (1 + abs(ds / e)), (mode, p, b)
                else:
                    assert e == 0 and st["avg_dist"] == 0.0, (p, b)
    run.close()


# ------------------------------------------------------------------------------------------------ checkpoint with training slots
def test_checkpoint_with_body_physics_terrain_and_training_slots(ref_root, assets, tmp_path):
    import deepterrainrl_b200 as trl
    from deepterrainrl_b200.checkpoint import sections
    from deepterrainrl_b200.train import TrainSchedule, train_run_slots
    from test_gpu_checkpoint import assert_refused, assert_same, damaged_copies, save_and_load
    from test_gpu_train_slots import SCHEDULE, TRAINER, close, make_group, start_models
    root, models, var = ref_root
    pack = os.path.join(assets, "dog_slopes_mixed.trlpack")
    n = 1024
    tm = start_models(pack, str(tmp_path))
    slots = np.arange(n) % 3

    def setup(sc):
        sc.LoadTerrain(1, terrain_path(root, "narrow_gaps"))
        sc.SetEnvTerrain((np.arange(n) // 3) % 2)
        sc.LoadPhysics(1, [2.0e5, 2.0e3, 0.5, 0.01, 0.00025, 2.0e4, 20.0])
        sc.SetEnvPhysics((np.arange(n) // 5) % 2)
        sc.LoadBody(1, var["dog", "long"])
        sc.LoadBody(2, var["dog", "narrow"])
        sc.SetEnvBody((np.arange(n) // 7) % 3)
    sched = TrainSchedule(**SCHEDULE)
    a, ta = make_group(trl, pack, n, tm, slots, trainer_kw=TRAINER, setup=setup)
    b, tb = make_group(trl, pack, n, tm, slots, trainer_kw=TRAINER, setup=setup)
    for trs in (ta, tb):
        train_run_slots(trs, sched, 20, 2)
    path = str(tmp_path / "body.ckpt")
    b, tb = save_and_load(b, tb, path, user=b"body")
    tb = [tb[p] for p in range(3)]
    names = [s[0] for s in sections(path)]
    assert all(k in names for k in ("body_loaded", "body_table", "env_body_host", "env_body"))
    for trs in (ta, tb):
        train_run_slots(trs, sched, 10, 2)
    assert all(np.array_equal(x, y) for x, y in zip(a.EnvBody(), b.EnvBody()))
    for q in range(3):
        assert a.GetEvalStats(None, body=q) == b.GetEvalStats(None, body=q), q
    assert_same(a, b, ta, tb, stride=3)
    d = tmp_path / "bad"
    d.mkdir()
    for p, msg in damaged_copies(path, str(d)):
        if "body" in msg:
            assert_refused(a.L, p, msg)
    close(*ta, *tb, a, b)
