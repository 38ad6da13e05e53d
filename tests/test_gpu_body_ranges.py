"""Ranged slots (trl_load_body_range / trl_load_physics_range / trl_env_body_draws / trl_env_physics_draws): at every episode reset of an
env on a ranged body or physics slot, its link masses, PD gains and torque limits, or its seven contact constants, are drawn afresh
between a lo and a hi end.  The contract is exact: an episode of env i on a ranged slot computes, bit for bit, what env i computes on a
fixed slot loaded with that episode's drawn numbers (a character file holding them, written with %.17g; trl_load_physics with the drawn
p7).

  1. the recipe: the read-backs equal a numpy restatement of the draw (include/terrainrl_b200.h) for every env over three episodes
     begun by a forced fall, trl_reset and trl_seed_terrain, with the draw counters, lo == hi numbers and the [lo, hi] bounds;
  2. degenerate ranges: lo == hi == F computes what the fixed slot F computes, under three schedules, evaluating and exploring;
  3. per episode: dog, raptor and goat on ranged bodies and physics against a reference handle whose fixed slots hold the numbers the
     recipe draws, assigned to take effect at the same resets: the first ranged episode and one begun by a fall inside an update;
  4. beside policy, terrain and training slots and evaluation envs: every statistics cell, and a trainer fed by ranged envs is the
     same under the three schedules;
  5. a checkpoint resumes the draws bit for bit, a damaged new section is refused by name, a handle without ranged slots writes no
     new section;
  6. 600 free-running env-steps of drawn bodies against the CPU oracle on the drawn files;
  7. every refusal leaves the handle unchanged, the communicator ones included;
  8. three training slots on ranged body and physics slots against single-trainer handles whose envs sit on fixed slots holding
     each episode's drawn numbers, with every (policy, physics, body) statistics cell.
tests/test_body_ranges_cpu.py runs a miniature on the emulator."""
import copy
import json
import os

import numpy as np
import pytest

import torch_net  # noqa: F401  (torch before the library: see tests/test_gpu_decide_batches.py)
from test_gpu_terrain_slots import _run, _schedule, assert_same_env, data_root, scene_args, terrain_path, tip_over, tuples_by_env

pytestmark = pytest.mark.gpu

TERRAIN = {"dog": "slopes_mixed", "raptor": "mixed_raptor", "goat": "cliffs_rugged"}
N_OUT = {"dog": 90, "goat": 90, "raptor": 87}
PHYS0 = np.array([5.0e4, 1.0e3, 0.9, 1e-3, 2.5e-4, 1.0e4, 1.0e2])    # LoadPhysics order; the ends below scale it
PHYS_LO = PHYS0 * np.array([0.8, 1.0, 0.5 / 0.9, 1.0, 1.0, 1.0, 1.0])
PHYS_HI = PHYS0 * np.array([1.2, 1.0, 1.1 / 0.9, 1.0, 1.0, 1.0, 1.0])

# ------------------------------------------------------------------------------------------------ the recipe, restated
BODY_TAG = 0x626f64792d726e67
PHYS_TAG = 0x706879732d726e67
M64 = (1 << 64) - 1


def mix64(z):
    z = (z + 0x9E3779B97F4A7C15) & M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
    return z ^ (z >> 31)


def draw_key(seed, tag, env, draw):
    seed, env, draw = int(seed), int(env), int(draw)
    return mix64((mix64((mix64((seed ^ tag) & M64) + env) & M64) + draw) & M64)


def draw_numbers(seed, tag, env, draw, lo, hi):
    """the draw `draw` of env `env`: lo / hi flat arrays of the same length, number i drawn with u_i (Python floats: each operation
    rounded once, as the kernels' __dadd_rn / __dmul_rn / __dsub_rn)"""
    k = draw_key(seed, tag, env, draw)
    out = np.empty(len(lo))
    for i, (a, b) in enumerate(zip(lo, hi)):
        u = float(mix64((k + i) & M64) >> 11) * 2.0 ** -53
        out[i] = min(float(b), float(a) + u * (float(b) - float(a)))
    return out


def body_numbers(char):
    """[4][nj] Mass, Kp, Kd, TorqueLim of a parsed character file as a body slot holds them (the root's Kp and Kd are 0)"""
    B, P = char["BodyDefs"], char["PDControllers"]
    nj = len(char["Skeleton"]["Joints"])
    out = np.zeros((4, nj))
    for j in range(nj):
        out[0, j] = B[j]["Mass"]
        out[1, j] = 0.0 if j == 0 else P[j].get("Kp", 0.0)
        out[2, j] = 0.0 if j == 0 else P[j].get("Kd", 0.0)
        out[3, j] = P[j].get("TorqueLim", 0.0)
    return out


def body_draw(seed, env, draw, lo, hi):
    """[4][nj] of a body draw, lo / hi as body_numbers gives them"""
    return draw_numbers(seed, BODY_TAG, env, draw, lo.ravel(), hi.ravel()).reshape(lo.shape)


def phys_draw(seed, env, draw, lo7, hi7):
    return draw_numbers(seed, PHYS_TAG, env, draw, lo7, hi7)


def with_numbers(char, nums):
    """the character file holding the body numbers nums [4][nj] (the root's Kp / Kd are not read)"""
    c = copy.deepcopy(char)
    for j in range(nums.shape[1]):
        c["BodyDefs"][j]["Mass"] = float(nums[0, j])
        c["PDControllers"][j]["Kp"] = float(nums[1, j])
        c["PDControllers"][j]["Kd"] = float(nums[2, j])
        c["PDControllers"][j]["TorqueLim"] = float(nums[3, j])
    return c


def write_char(c, path):
    """JSON with every number at %.17g (round trips every double)"""
    def enc(x):
        if isinstance(x, float):
            return "%.17g" % x
        if isinstance(x, dict):
            return "{" + ", ".join('"%s": %s' % (k, enc(v)) for k, v in x.items()) + "}"
        if isinstance(x, list):
            return "[" + ", ".join(enc(v) for v in x) + "]"
        return json.dumps(x)
    with open(path, "w") as f:
        f.write(enc(c))
    return path


def base_char(root, ch):
    with open(os.path.join(root, "data", "characters", ch + ".txt")) as f:
        c = json.load(f)
    # controller files by absolute path: the files load into handles made from packs too, which have no data root
    c["Controllers"]["Files"] = [os.path.join(root, x) for x in c["Controllers"]["Files"]]
    return c


WIDE = {"Mass": (0.8, 1.25), "Kp": (0.8, 1.2), "Kd": (0.8, 1.2), "TorqueLim": (0.7, 1.0)}


def range_ends(char, scale=None, f=WIDE):
    """lo / hi files of a ranged body: by default masses x0.8-1.25, Kp / Kd x0.8-1.2, TorqueLim x0.7-1.0 (scale: one factor for all
    four)"""
    lo, hi = copy.deepcopy(char), copy.deepcopy(char)
    for name, (a, b) in f.items():
        a, b = (a, b) if scale is None else (scale, scale)
        for j, x in enumerate(char["BodyDefs"] if name == "Mass" else char["PDControllers"]):
            tgt_lo = lo["BodyDefs"][j] if name == "Mass" else lo["PDControllers"][j]
            tgt_hi = hi["BodyDefs"][j] if name == "Mass" else hi["PDControllers"][j]
            v = float(x.get(name, 0.0))
            tgt_lo[name], tgt_hi[name] = v * a, v * b
    return lo, hi


@pytest.fixture(scope="module")
def ref_root(tmp_path_factory, assets):
    import deepterrainrl_b200 as trl
    d = str(tmp_path_factory.mktemp("body_ranges"))
    root, models = data_root(trl, assets, d)
    return root, models, d


def same_dist_logs(a, b):
    """every env's own sequence of distance-log entries (the log interleaves envs in completion order)"""
    (da, ea), (db, eb) = a.GetDistLog(), b.GetDistLog()
    return all(np.array_equal(da[ea == e], db[eb == e]) for e in range(a.num_envs))


def make(trl, scene, root, model, n, explore=False, rng_seed=77, seeds=None, extra=()):
    cls = trl.ScenarioExpMACE if explore else trl.ScenarioPoliEval
    sc = cls(None, n, args=scene_args(scene, TERRAIN[scene], model, list(extra)), data_root=root, rng_seed=rng_seed, terrain_seeds=seeds)
    if explore:
        sc.EnableExplore(1, 0.3, 0.5, 0.05)
    return sc


def reseed(sc, n, seeds=None):
    sc.SetRandSeed(np.arange(1, n + 1, dtype=np.uint64) if seeds is None else seeds)


def ends_files(root, d, ch, tag, scale=None, f=WIDE):
    base = base_char(root, ch)
    lo, hi = range_ends(base, scale, f)
    return base, write_char(lo, os.path.join(d, "%s_%s_lo.txt" % (ch, tag))), write_char(hi, os.path.join(d, "%s_%s_hi.txt" % (ch, tag))), \
        body_numbers(lo), body_numbers(hi)


# ------------------------------------------------------------------------------------------------ (1) the recipe
def test_readbacks_follow_the_recipe(ref_root):
    import deepterrainrl_b200 as trl
    root, models, d = ref_root
    n, seed = 96, 77
    base, lo_f, hi_f, lo, hi = ends_files(root, d, "dog", "recipe")
    hi[3, 5] = lo[3, 5]          # lo == hi numbers come out exactly lo
    hi_c = with_numbers(base, hi)
    hi_f = write_char(hi_c, os.path.join(d, "dog_recipe_hi2.txt"))
    sc = make(trl, "dog", root, models["dog"], n, rng_seed=seed)
    sc.LoadBodyRange(1, lo_f, hi_f)
    plo, phi = PHYS_LO.copy(), PHYS_HI.copy()
    sc.LoadPhysicsRange(2, plo, phi)
    body = np.arange(n) % 3 != 0           # envs 1, 2 mod 3 on the ranged body, 0, 1 mod 3 on the ranged physics
    phys = np.arange(n) % 3 != 2
    sc.SetEnvBody(np.where(body, 1, 0))
    sc.SetEnvPhysics(np.where(phys, 2, 0))
    nb = np.zeros(n, np.int64)
    npd = np.zeros(n, np.int64)
    scene_body = sc.EnvBodyDraws()[0][0]

    def check():
        out, draws = sc.EnvBodyDraws()
        pout, pdraws = sc.EnvPhysicsDraws()
        assert np.array_equal(draws, nb) and np.array_equal(pdraws, npd)
        for e in range(n):
            if body[e]:
                want = body_draw(seed, e, nb[e] - 1, lo, hi)
                assert np.array_equal(out[e], want), e
                assert np.all(out[e] >= lo) and np.all(out[e] <= hi) and out[e][3, 5] == lo[3, 5]
            else:
                assert np.array_equal(out[e], scene_body), e
            if phys[e]:
                assert np.array_equal(pout[e], phys_draw(seed, e, npd[e] - 1, plo, phi)), e
                assert np.all(pout[e] >= plo) and np.all(pout[e] <= phi)
        return out

    reseed(sc, n)                          # trl_seed_terrain: episode 1 of every env
    nb += body; npd += phys
    check()
    _run(sc, 2)
    falls = np.arange(0, n, 5)
    tip_over(sc, falls)                    # a fall inside the next update: episode 2 of those envs
    _run(sc, 1)
    nb[falls] += body[falls]; npd[falls] += phys[falls]
    check()
    sc.Reset(np.arange(1, n, 2))           # trl_reset: a further episode of the odd envs
    nb[1::2] += body[1::2]; npd[1::2] += phys[1::2]
    check()
    reseed(sc, n)                          # and every env again; the counters go on
    nb += body; npd += phys
    out = check()
    assert nb[body].min() >= 2 and nb.max() == 4 and not nb[~body].any()
    assert len({out[e].tobytes() for e in range(n) if body[e]}) == int(body.sum())   # every env its own body
    sc.close()


# ------------------------------------------------------------------------------------------------ (2) lo == hi == F is the fixed slot F
@pytest.mark.parametrize("schedule", ["overlap", "serial", "groups3"])
@pytest.mark.parametrize("explore", [False, True])
def test_degenerate_range_is_the_fixed_slot(ref_root, monkeypatch, schedule, explore):
    import deepterrainrl_b200 as trl
    root, models, d = ref_root
    _schedule(monkeypatch, schedule)
    n = 256
    base, lo_f, hi_f, lo, hi = ends_files(root, d, "dog", "point", scale=0.9)
    assert np.array_equal(lo, hi)
    handles = []
    for ranged in (True, False):
        sc = make(trl, "dog", root, models["dog"], n, explore=explore)
        if ranged:
            sc.LoadBodyRange(1, lo_f, lo_f)
            sc.LoadPhysicsRange(1, PHYS_LO, PHYS_LO)
        else:
            sc.LoadBody(1, lo_f)
            sc.LoadPhysics(1, PHYS_LO)
        sc.SetEnvBody(np.arange(n) % 2)
        sc.SetEnvPhysics((np.arange(n) // 2) % 2)
        reseed(sc, n)
        _run(sc, 3)
        tip_over(sc, range(0, n, 16))
        _run(sc, 12)
        handles.append(sc)
    a, b = handles
    assert a.GetNumEpisodes() == b.GetNumEpisodes() and (explore or a.GetNumEpisodes() > 0)
    assert np.all(a.EnvBodyDraws()[1][1::2] >= 1) and not b.EnvBodyDraws()[1].any()
    for e in range(n):
        assert_same_env(a, e, b, e, 90, "ranged point")
    assert same_dist_logs(a, b)
    if explore:
        assert all(np.array_equal(x, y) for x, y in zip(tuples_by_env(a), tuples_by_env(b)))
    assert np.array_equal(a.EnvBodyDraws()[0], b.EnvBodyDraws()[0])
    assert np.array_equal(a.EnvPhysicsDraws()[0], b.EnvPhysicsDraws()[0])
    for sc in handles:
        sc.close()


# ------------------------------------------------------------------------------------------------ (3) every episode is a fixed slot
@pytest.mark.parametrize("scene", ["dog", "raptor", "goat"])
def test_each_episode_is_the_fixed_slot_of_its_draw(ref_root, scene):
    """3 envs on a ranged body and physics (envs 3..5 on slot 0): a reference handle's env e holds the numbers of its first ranged
    episode in slot 1 + e and those of its second in slot 4 + e, assigned during the first so that the fall switches it"""
    import deepterrainrl_b200 as trl
    root, models, d = ref_root
    n, seed, k = 6, 91, 3
    base, lo_f, hi_f, lo, hi = ends_files(root, d, scene, "episodes")
    sc = make(trl, scene, root, models[scene], n, rng_seed=seed)
    sc.LoadBodyRange(1, lo_f, hi_f)
    sc.LoadPhysicsRange(1, PHYS_LO, PHYS_HI)
    ref = make(trl, scene, root, models[scene], n, rng_seed=seed)
    for ep in range(2):
        for e in range(k):
            nums = body_draw(seed, e, ep, lo, hi)
            slot = 1 + e + ep * k
            ref.LoadBody(slot, write_char(with_numbers(base, nums), os.path.join(d, "%s_e%d_ep%d.txt" % (scene, e, ep))))
            ref.LoadPhysics(slot, phys_draw(seed, e, ep, PHYS_LO, PHYS_HI))
    first = np.array([1 + e if e < k else 0 for e in range(n)])
    second = np.array([1 + e + k if e < k else 0 for e in range(n)])
    sc.SetEnvBody(np.where(np.arange(n) < k, 1, 0)); sc.SetEnvPhysics(np.where(np.arange(n) < k, 1, 0))
    ref.SetEnvBody(first); ref.SetEnvPhysics(first)
    for h in (sc, ref):
        reseed(h, n)
    ref.SetEnvBody(second); ref.SetEnvPhysics(second)          # takes effect at the fall below
    assert np.array_equal(sc.EnvBodyDraws()[0][:k], np.stack([body_draw(seed, e, 0, lo, hi) for e in range(k)]))
    for h in (sc, ref):
        _run(h, 4)
    for e in range(n):
        assert_same_env(sc, e, ref, e, N_OUT[scene], "first ranged episode")
    for h in (sc, ref):
        tip_over(h, range(n))
        _run(h, 6)
    assert np.array_equal(sc.EnvBodyDraws()[1], [2, 2, 2, 0, 0, 0])
    assert np.array_equal(ref.EnvBody()[0], second)
    for e in range(n):
        assert_same_env(sc, e, ref, e, N_OUT[scene], "episode begun by a fall")
    assert same_dist_logs(sc, ref)
    sc.close(); ref.close()


# ------------------------------------------------------------------------------------------------ (4) beside the other slot kinds
def _stats(sc, mode, p, t, q, b):
    import ctypes as C
    c = C.c_int64(0); e = C.c_int64(0); a = C.c_double(0); s = C.c_int64(0)
    sc._ck(sc.L.trl_eval_stats_body(sc.h, int(mode), int(p), int(t), int(q), int(b), C.byref(c), C.byref(e), C.byref(a), C.byref(s)))
    return c.value, e.value, a.value, s.value


def test_beside_terrain_slots_evaluation_envs_and_training(ref_root, monkeypatch):
    import deepterrainrl_b200 as trl
    root, models, d = ref_root
    n = 192
    base, lo_f, hi_f, lo, hi = ends_files(root, d, "dog", "mixed")
    runs = []
    for schedule in ("overlap", "serial", "groups3"):
        _schedule(monkeypatch, schedule)
        sc = make(trl, "dog", root, models["dog"], n, explore=True)
        sc.LoadTerrain(1, terrain_path(root, "flat"))
        sc.LoadBodyRange(2, lo_f, hi_f)
        sc.LoadPhysicsRange(3, PHYS_LO, PHYS_HI)
        sc.SetEnvTerrain(np.arange(n) % 2)
        sc.SetEnvBody(np.where(np.arange(n) % 3 == 0, 2, 0))
        sc.SetEnvPhysics(np.where(np.arange(n) % 4 == 0, 3, 0))
        sc.SetEnvEval((np.arange(n) % 5 == 0).astype(np.int32))
        reseed(sc, n)
        tr = trl.MACETrainer(sc, replay_mem_size=4096, num_init_samples=64, seed=3)
        for _ in range(3):
            _run(sc, 4)
            tip_over(sc, range(0, n, 9))
            tr.AddTuplesFromScene()
            tr.Train(2)
        _run(sc, 4)
        cells = {(m, t, q, b): _stats(sc, m, -1, t, q, b) for m in (-1, 0, 1) for t in (-1, 0, 1) for q in (-1, 0, 3) for b in (-1, 0, 2)}
        total = _stats(sc, -1, -1, -1, -1, -1)
        assert sum(cells[-1, t, -1, -1][1] for t in (0, 1)) == total[1]
        assert sum(cells[-1, -1, -1, b][1] for b in (0, 2)) == total[1]
        assert cells[-1, -1, -1, 2][1] > 0 and cells[-1, -1, 3, -1][1] > 0
        runs.append((cells, tr.get("theta"), sc.GetStateAll(), sc.EnvBodyDraws(), sc.EnvPhysicsDraws()))
        tr.close()
        sc.close()
    for r in runs[1:]:
        assert r[0] == runs[0][0]
        assert np.array_equal(r[1], runs[0][1])
        for x, y in zip(r[2] + r[3] + r[4], runs[0][2] + runs[0][3] + runs[0][4]):
            assert np.array_equal(x, y)


# ------------------------------------------------------------------------------------------------ (5) checkpoints
def test_checkpoint_resumes_the_draws(ref_root, tmp_path):
    import deepterrainrl_b200 as trl
    from deepterrainrl_b200.checkpoint import sections
    from test_gpu_checkpoint import damaged_copies
    root, models, d = ref_root
    n = 128
    base, lo_f, hi_f, lo, hi = ends_files(root, d, "dog", "ckpt")
    plain = make(trl, "dog", root, models["dog"], n)
    plain.LoadBody(1, lo_f)
    p0 = str(tmp_path / "plain.ckpt")
    plain.SaveCheckpoint(p0)
    new = {"env_bdraw", "env_pdraw", "env_draws", "ranges", "range_body_hi", "range_phys_hi"}
    assert not new & {s[0] for s in sections(p0)}
    plain.close()
    a = make(trl, "dog", root, models["dog"], n)
    a.LoadBodyRange(1, lo_f, hi_f)
    a.LoadPhysicsRange(1, PHYS_LO, PHYS_HI)
    a.SetEnvBody(np.arange(n) % 2); a.SetEnvPhysics((np.arange(n) // 2) % 2)
    reseed(a, n)
    _run(a, 3)
    tip_over(a, range(0, n, 7))
    _run(a, 2)
    path = str(tmp_path / "ranged.ckpt")
    a.SaveCheckpoint(path)
    assert new <= {s[0] for s in sections(path)}
    b, _, _ = trl.load_checkpoint(path)
    for h in (a, b):
        _run(h, 3)
        tip_over(h, range(3, n, 7))
        _run(h, 4)
        h.Reset([5, 6])
    for x, y in zip(a.EnvBodyDraws() + a.EnvPhysicsDraws(), b.EnvBodyDraws() + b.EnvPhysicsDraws()):
        assert np.array_equal(x, y)
    assert a.EnvBodyDraws()[1].max() == 2
    for e in range(n):
        assert_same_env(a, e, b, e, 90, "resumed")
    dd = tmp_path / "bad"
    dd.mkdir()
    named = set()
    for p, msg in damaged_copies(path, str(dd)):
        if any("'%s'" % s in msg for s in new):
            with pytest.raises(RuntimeError) as ei:
                trl.load_checkpoint(p)
            assert msg in str(ei.value), (msg, str(ei.value))
            named |= {s for s in new if "'%s'" % s in msg}
    assert named == new
    a.close(); b.close()


# ------------------------------------------------------------------------------------------------ (6) the CPU oracle on drawn files
def test_drawn_bodies_against_the_oracle(ref_root, tmp_path):
    """600 free-running env-steps of 8 envs on a ranged body, each against the CPU oracle on a pack of its drawn file, at the body-slot
    test's tolerance, checked every 50 env-steps"""
    import deepterrainrl_b200 as trl
    from pyoracle import Oracle
    root, models, d = ref_root
    n, seed, h = 8, 77, 1.0 / 600.0
    seeds = np.arange(11, 11 + n, dtype=np.uint64)
    base, lo_f, hi_f, lo, hi = ends_files(root, d, "dog", "oracle")
    g = make(trl, "dog", root, models["dog"], n, rng_seed=seed, seeds=seeds)
    g.LoadBodyRange(1, lo_f, hi_f)
    g.SetEnvBody(np.ones(n, np.int32))
    g.SetRandSeed(seeds)
    orc = []
    for e in range(n):
        f = write_char(with_numbers(base, body_draw(seed, e, 0, lo, hi)), str(tmp_path / ("drawn%d.txt" % e)))
        pack = str(tmp_path / ("drawn%d.trlpack" % e))
        trl.pack_from_args(scene_args("dog", "slopes_mixed", models["dog"], ["-character_file=", f]), root, pack)
        orc.append(Oracle(pack, n, 0, terrain_seeds=seeds))
    worst = 0.0
    for k in range(600):
        g.EnvStep(h)
        for e in range(n):
            orc[e].env_step(e, h)
        if k % 50 == 49:
            for e in range(n):
                gq, gqd, _, _ = g.GetState(e)
                oq, oqd, _, _ = orc[e].get_state(e)
                err = max(np.max(np.abs(gq - oq) / (1 + np.abs(oq))), np.max(np.abs(gqd - oqd) / (1 + np.abs(oqd))))
                worst = max(worst, err)
                assert err < 1e-4, (k, e)
    assert np.array_equal(g.EnvBodyDraws()[1], np.ones(n))      # no env fell: every env ran its first draw throughout
    print("ranged bodies vs oracle, 600 env-steps: worst rel err %.3e" % worst)
    g.close()


# ------------------------------------------------------------------------------------------------ (7) refusals
def test_refusals_leave_the_handle_unchanged(ref_root):
    import deepterrainrl_b200 as trl
    root, models, d = ref_root
    n = 32
    base, lo_f, hi_f, lo, hi = ends_files(root, d, "dog", "refuse")
    sc = make(trl, "dog", root, models["dog"], n)
    sc.LoadBodyRange(1, lo_f, hi_f)
    sc.LoadPhysicsRange(1, PHYS_LO, PHYS_HI)
    sc.SetEnvBody(np.ones(n, np.int32)); sc.SetEnvPhysics(np.ones(n, np.int32))
    reseed(sc, n)
    longer = copy.deepcopy(base)
    longer["BodyDefs"][13]["Param0"] *= 1.1
    bad_geom = write_char(longer, os.path.join(d, "dog_refuse_geom.txt"))
    swapped = os.path.join(d, "dog_refuse_swapped")
    before = (sc.EnvBodyDraws(), sc.EnvPhysicsDraws(), sc.EnvBody(), sc.EnvPhysics())
    bad_p = PHYS_HI.copy(); bad_p[4] = 0.01
    for call, msg in [(lambda: sc.LoadBodyRange(0, lo_f, hi_f), "out of range"), (lambda: sc.LoadBodyRange(8, lo_f, hi_f), "out of range"),
                      (lambda: sc.LoadBodyRange(2, lo_f, bad_geom), "Param0 \\(box size\\) of link 13"),
                      (lambda: sc.LoadBodyRange(2, hi_f, lo_f), "Mass of link 0: lo"),
                      (lambda: sc.LoadBodyRange(2, lo_f, swapped + "_missing.txt"), "hi"),
                      (lambda: sc.LoadBodyRange(1, lo_f, hi_f), "in use"),
                      (lambda: sc.LoadPhysicsRange(2, PHYS_HI, PHYS_LO), "kn: lo"),
                      (lambda: sc.LoadPhysicsRange(2, PHYS_LO, bad_p), "hi contact_tol"),
                      (lambda: sc.LoadPhysicsRange(0, PHYS_LO, PHYS_HI), "out of range"),
                      (lambda: sc.LoadPhysicsRange(1, PHYS_LO, PHYS_HI), "in use")]:
        with pytest.raises(RuntimeError, match=msg):
            call()
    after = (sc.EnvBodyDraws(), sc.EnvPhysicsDraws(), sc.EnvBody(), sc.EnvPhysics())
    for x, y in zip(before, after):
        assert all(np.array_equal(u, v) for u, v in zip(x, y))
    sc.close()


def test_communicator_refusals(ref_root):
    """ranged slots do not run with a communicator: the range loaders refuse a handle with one, trl_comm_init* a handle with a ranged
    slot (a single-rank communicator whose collectives are memory copies)"""
    import ctypes as C
    import deepterrainrl_b200 as trl
    from deepterrainrl_b200.parallel import _Collectives
    root, models, d = ref_root
    n = 16
    base, lo_f, hi_f, lo, hi = ends_files(root, d, "dog", "comm")

    def all_gather(ctx, send, recv, nbytes, stream):
        C.memmove(recv, send, nbytes)
        return 0
    coll = _Collectives(None, _Collectives.AG(all_gather), _Collectives.BC(lambda ctx, buf, nbytes, root, stream: 0),
                        _Collectives.AR(lambda ctx, buf, count, stream: 0))
    cm = make(trl, "dog", root, models["dog"], n, explore=True)
    assert cm.L.trl_comm_init_external(cm.h, C.byref(coll), 0, 1) == 0, cm.L.trl_last_error()
    for call in (lambda: cm.LoadBodyRange(1, lo_f, hi_f), lambda: cm.LoadPhysicsRange(1, PHYS_LO, PHYS_HI)):
        with pytest.raises(RuntimeError, match="communicator"):
            call()
    assert not cm.EnvBodyDraws()[1].any() and np.array_equal(cm.EnvBody()[0], np.zeros(n))
    for kind in ("body", "physics"):
        g = make(trl, "dog", root, models["dog"], n, explore=True)
        if kind == "body":
            g.LoadBodyRange(1, lo_f, hi_f)
        else:
            g.LoadPhysicsRange(1, PHYS_LO, PHYS_HI)
        assert g.L.trl_comm_init_external(g.h, C.byref(coll), 0, 1) != 0 and b"ranged slots" in g.L.trl_last_error()
        idb = (C.c_char * 128)()
        if g.L.trl_comm_unique_id(idb) == 0:
            assert g.L.trl_comm_init(g.h, idb, 0, 1) != 0 and b"ranged slots" in g.L.trl_last_error()
        g.LoadBodyRange(2, lo_f, hi_f)          # still a handle without a communicator
        g.close()
    cm.close()


# ------------------------------------------------------------------------------------------------ (8) training slots on ranged slots
def test_training_slots_on_ranged_slots(ref_root, assets, tmp_path):
    """three training slots whose envs all run on a ranged body and a ranged physics slot, against single-trainer handles (fed only
    their slot's tuples) whose envs of that slot sit on fixed slots holding the numbers each episode draws: two fixed slots per env, the
    one of its present episode and the one its next reset moves it to, refilled with the following draw after every reset.  Every
    trainer array, every env and every (policy, physics, body) statistics cell against the references' own envs."""
    import deepterrainrl_b200 as trl
    from deepterrainrl_b200.train import TrainSchedule, train_run_slots
    from test_gpu_train_slots import DT, SCHEDULE, assert_envs, assert_trainer, close, make_group, make_ref, start_models
    root, models, d = ref_root
    pack = os.path.join(assets, "dog_slopes_mixed.trlpack")
    n, seed, k = 9, 5, 3
    slots = np.arange(n) % 3
    trainer_kw = dict(replay_mem_size=400, num_init_samples=32, freeze_target_iters=7)
    # ranges around the scene's own body and physics, narrow enough that the policies walk and every slot gathers tuples
    base, lo_f, hi_f, lo, hi = ends_files(root, d, "dog", "train", f={"Mass": (0.95, 1.05), "Kp": (0.95, 1.05), "Kd": (0.95, 1.05),
                                                                      "TorqueLim": (0.95, 1.0)})
    scene_phys = np.array([2.0e5, 2.0e3, 0.81, 0.01, 0.00025, 2.0e4, 20.0])
    plo, phi = scene_phys * np.array([0.9, 1.0, 0.9, 1.0, 1.0, 1.0, 1.0]), scene_phys * np.array([1.1, 1.0, 1.1, 1.0, 1.0, 1.0, 1.0])
    tm = start_models(pack, str(tmp_path))

    def group_setup(sc):
        sc.LoadBodyRange(1, lo_f, hi_f)
        sc.LoadPhysicsRange(1, plo, phi)
        sc.SetEnvBody(np.ones(n, np.int32))
        sc.SetEnvPhysics(np.ones(n, np.int32))     # the resets of trl_set_env_policy make them current

    class Tracker:
        """the fixed slots of slot p's envs in a reference handle: env j of the slot alternates between slots 1 + 2j and 2 + 2j"""
        def __init__(self, p):
            self.envs = np.flatnonzero(slots == p)
            self.draw = {e: 0 for e in self.envs}          # the draw the env's assigned slot holds
            self.nxt = {}

        def load(self, sc, e, slot):
            nums = body_draw(seed, e, self.draw[e], lo, hi)
            sc.LoadBody(slot, write_char(with_numbers(base, nums), os.path.join(d, "train_e%d_k%d.txt" % (e, self.draw[e]))))
            sc.LoadPhysics(slot, phys_draw(seed, e, self.draw[e], plo, phi))
            sc.SetEnvBody([slot], env_ids=[e])
            sc.SetEnvPhysics([slot], env_ids=[e])
            self.nxt[e] = slot

        def setup(self, sc):
            for j, e in enumerate(self.envs):
                self.load(sc, e, 1 + 2 * j)

        def follow(self, sc):
            cur = sc.EnvBody()[0]
            for j, e in enumerate(self.envs):
                if cur[e] == self.nxt[e]:                  # a reset made the assigned slot current: prepare the next draw
                    self.draw[e] += 1
                    self.load(sc, e, (1 + 2 * j) if self.nxt[e] == 2 + 2 * j else (2 + 2 * j))

    sched = TrainSchedule(**dict(SCHEDULE, trainer_curriculum_iters=0))
    updates = 200                         # twice (3 envs per slot gather a tuple per gait cycle), with envs tipped over between the two
                                          # runs: their next episodes begin inside a run
    tipped = [0, 3, 6, 4, 8]               # slot 0's envs are not reset by trl_set_env_policy: their falls put them on the ranged slots
    group, trs = make_group(trl, pack, n, tm, slots, trainer_kw=trainer_kw, setup=group_setup)
    train_run_slots(trs, sched, updates, 2)
    tip_over(group, tipped)
    train_run_slots(trs, sched, updates, 2)
    refs, trackers = [], []
    for p in range(3):
        t = Tracker(p)
        sc, tr = make_ref(trl, pack, n, tm, p, slots, trainer_kw=trainer_kw, setup=t.setup)
        t.follow(sc)
        mine = slots == p
        for u in range(2 * updates):      # test_gpu_train_slots.ref_loop, the fixed slots followed after every update
            if u % updates == 0:
                done = 0                  # each trl_train_run_slots call anneals from 0
                if u:
                    tip_over(sc, tipped)
            s = sched(done)
            sc.EnableExplore(True, s["exp_rate"], s["exp_temp"], s["exp_base_rate"])
            sc.SetTerrainParamsLerp(s["curriculum_phase"])
            sc.Update(DT)
            t.follow(sc)
            rows, flags, env = sc.GetTuples(f64=True)
            keep = np.flatnonzero(mine[env])
            keep = keep[np.argsort(env[keep], kind="stable")]
            tr.AddTuples(rows[keep], flags[keep])
            sc.ResetTupleBuffer()
            tr.Train(2)
            done += 2
        refs.append((sc, tr))
        trackers.append(t)
    bdraws, pdraws = group.EnvBodyDraws()[1], group.EnvPhysicsDraws()[1]
    for t in trackers:
        for e in t.envs:
            assert bdraws[e] == pdraws[e] == t.draw[e], ("draws", e, bdraws[e], t.draw[e])
    assert bdraws.min() >= 1 and bdraws.max() >= 2          # every env drew, and some episodes began inside the run
    for p in range(3):
        assert trs[p].counters()["iter"] > 0, [t.counters() for t in trs]
        assert_trainer(trs[p], refs[p][1], "slot %d" % p)
    assert_envs(group, [r[0] for r in refs], slots, 90)
    # the statistics cube with policy slots: every (policy, physics, body) cell against the references' own envs
    qcur, bcur = group.EnvPhysics()[0], group.EnvBody()[0]
    for p in (-1, 0, 1, 2):
        for q in (-1, 0, 1):
            for b in (-1, 0, 1):
                cyc = eps = 0
                for e in range(n):
                    if (p >= 0 and slots[e] != p) or (q >= 0 and qcur[e] != q) or (b >= 0 and bcur[e] != b):
                        continue
                    ref = refs[slots[e]][0]
                    cyc += int(ref.GetCtrl(e)[-2])
                    dist, denv = ref.GetDistLog()
                    eps += int((denv == e).sum())
                got = _stats(group, -1, p, -1, q, b)
                assert (got[0], got[1]) == (cyc, eps), ((p, q, b), got, cyc, eps)
    close(*trs, group, *[o for r in refs for o in r])
