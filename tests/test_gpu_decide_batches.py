"""The batched policy decision pass (csrc/trl_decide2.cuh: trl_decide_conv_kernel + trl_decide_fc_kernel) at the batch shapes where
it branches, driven through trl_debug_decide on chosen env lists, against torch's own f64 conv1d / linear (tools/torch_net.py).

What the shapes reach (fc_clusters = 2 clusters of 8 CTAs, 32 rows per chunk, decide_grid = 264 CTAs = 66 conv clusters on 132 SMs):
  * more than 64 pending decisions: a cluster runs a second chunk with its TMA ring mid-way (46 / 47 k-tiles per rank = 23 / 24
    stage loads per chunk, so the ranks start chunk 2 at different stages and parities);
  * ragged last chunks, and the TMA zero fill when a chunk runs past row num_envs of the act2 matrix (1000 envs, count >= 993);
  * more than 66 decisions: the conv stage's persistent loop;
  * row k of the pass belongs to env ids[k]: reversed, permuted, strided and tail lists make a row / env mix-up visible.
Every call writes fresh policy states (rows of a pool, rotated per call), so a row the kernel skipped keeps an output that cannot
match.  tests/test_simt_cpu.py runs a small version of the same sweep on the emulator."""
import os

import numpy as np
import pytest

# torch before anything opens NCCL: the library's multi-GPU exchange dlopens libnccl.so.2 (tests/test_gpu_comm.py), which has to
# resolve to the NCCL torch loads, not the other way round
import torch_net

pytestmark = pytest.mark.gpu

SCENES = {"dog_slopes_mixed": 90, "goat_cliffs": 90, "raptor_narrow_gaps": 87}
COUNTS = [0, 1, 2, 31, 32, 33, 63, 64, 65, 66, 67, 96, 127, 128, 129, 132, 133, 255, 256, 257]
ORDERS = ["identity", "reversed", "permuted", "strided", "last"]
TOL = 1e-10                 # max |g - t| / (1 + |t|), the bar of tests/test_gpu_net_torch.py
RAPTOR_OPT = np.array([0, 1, 1, 0, 0] + [1, 0, 1, 1, 1, 1, 1, 1] * 2 + [0, 0, 1, 1, 1, 1, 1, 1] * 2, bool)


def _relerr(g, t):
    return float(np.max(np.abs(g - t) / (1.0 + np.abs(t)))) if np.size(t) else 0.0


def env_ids(order, count, n, seed=0):
    """the list of `count` distinct env ids of one pass; row k of the pass decides env ids[k]"""
    if order == "identity":
        ids = np.arange(count)
    elif order == "reversed":
        ids = np.arange(count)[::-1]
    elif order == "permuted":
        ids = np.random.default_rng(1000 * seed + count).permutation(n)[:count]
    elif order == "strided":            # every s-th env, ending at the last one
        s = max(1, n // max(count, 1))
        ids = (n - 1) - s * np.arange(count)[::-1]
    elif order == "last":               # the last `count` envs: row k holds env n - count + k
        ids = np.arange(n - count, n)
    else:
        raise ValueError(order)
    return np.ascontiguousarray(ids, dtype=np.int32)


def counts_for(n, counts=COUNTS):
    """the sweep's pending counts clipped to the batch, largest first: the entries past `count` of the pending list then hold the
    envs of the previous, longer list -- envs that a row bound past `count` would decide by mistake"""
    return sorted({min(c, n) for c in counts} | {n - 1, n}, reverse=True)


def _next_prime(k):
    while any(k % d == 0 for d in range(2, int(k ** 0.5) + 1)):
        k += 1
    return k


def edge_states(in_off, in_scale, per_kind, seed):
    """policy states at the edges of the input range, each kind with different character features (distinct outputs):
    normalised terrain 0 (the conv outputs are their biases), the whole input normalised to 0, terrain far below / above its
    normalisation, terrain alternating +-3 per sample, character features at +-8"""
    sc = np.where(in_scale == 0, 1.0, in_scale)
    X = torch_net.typical_inputs(in_off, in_scale, 6 * per_kind, seed)
    k = per_kind
    X[0:k, :200] = -in_off[:200]
    X[k] = -in_off
    X[2 * k:3 * k, :200] = -in_off[:200] - 25.0 / sc[:200]
    X[3 * k:4 * k, :200] = -in_off[:200] + 25.0 / sc[:200]
    X[4 * k:5 * k, :200] = -in_off[:200] + 3.0 * (-1.0) ** np.arange(200) / sc[:200]
    sign = np.random.default_rng(seed + 1).choice([-8.0, 8.0], size=(k, in_off.size - 200))
    X[5 * k:6 * k, 200:] = sign / sc[200:] - in_off[200:]
    return X


class StatePool:
    """P (prime) policy states and torch's outputs for them; call c gives env e row (e + 37 c) mod P, so an env sees a different
    state on every call (P exceeds the number of calls a test makes) and the envs of one call get distinct rows"""

    def __init__(self, net, n, special, seed, extra=257):
        blobs, io, isc, oo, osc = net
        self.P = _next_prime(n + extra)
        X = torch_net.typical_inputs(io, isc, self.P, seed)
        special = np.asarray(special, float).reshape(-1, io.size)
        X[np.linspace(0, self.P - 1, len(special)).astype(int)] = special     # spread, so that every rotation meets some
        self.X = X
        self.Y = torch_net.forward(blobs, io, isc, oo, osc, X)
        self.calls = 0

    def rows(self, ids):
        r = (np.asarray(ids, np.int64) + 37 * self.calls) % self.P
        self.calls += 1
        return r


def snapshot(sc, envs, n_out):
    """what a decision of env e may change: its net output, its controller block, its policy state"""
    return {int(e): (sc.GetNetOut(int(e), n_out), sc.GetCtrl(int(e)), sc.GetPoliState(int(e))) for e in envs}


def assert_unchanged(sc, before, n_out, what):
    after = snapshot(sc, before.keys(), n_out)
    for e, old in before.items():
        for name, a, b in zip(("net_out", "ctrl", "poli_state"), old, after[e]):
            assert np.array_equal(a, b), (what, "env %d not in the list changed its %s" % (e, name))


def opt_index(sc):
    """the controller parameters an actor writes, in the order of its outputs (cDogControllerMACE / cRaptorControllerMACE)"""
    return np.flatnonzero(RAPTOR_OPT) if sc.num_joints == 19 else np.arange(1, 30)


def check_decision(sc, env, y, ctrl):
    """the action id is torch's critic arg-max (where the top two differ), the actor's outputs are the committed parameters
    (after decide_one's abs() of TransTime, Cv and, for the raptor, Cd).  Control block: [state, phase, first_cycle, cur / prev
    cycle time, cur / prev stumble, prev_com(2), prev_dist(2), action_id, params, ...] (oracle/capi.cpp: orc_get_ctrl)"""
    nf, fs = sc.num_frags, sc.frag_size
    crit = y[:nf]
    top = np.sort(crit)[::-1]
    if top[0] - top[1] <= 1e-9 * (1.0 + abs(top[0])):
        return
    a = int(np.argmax(crit))
    assert int(ctrl[11]) == a, ("action id", env, int(ctrl[11]), a, crit)
    opt = opt_index(sc)
    want = y[nf + a * fs:nf + (a + 1) * fs].copy()
    absolute = [0, 1, 2] if sc.num_joints == 19 else [0, 1]
    for k, p in enumerate(opt):
        if p in absolute:
            want[k] = abs(want[k])
    got = ctrl[12 + opt]
    assert _relerr(got, want) <= TOL, ("actor parameters", env, _relerr(got, want))


def decide_and_check(sc, pool, ids, n_out, watch=None):
    """one pass over `ids` with fresh states; returns the worst relative error against torch over the listed envs"""
    ids = np.asarray(ids, np.int32)
    if watch is None:
        watch = np.setdiff1d(np.arange(sc.num_envs), ids)
    before = snapshot(sc, watch, n_out)
    q0 = sc.GetStateAll()
    r = pool.rows(ids)
    sc.DebugDecide(ids, pool.X[r])
    worst = 0.0
    for e, row in zip(ids, r):
        g = sc.GetNetOut(int(e), n_out)
        err = _relerr(g, pool.Y[row])
        assert err <= TOL, ("net output", int(e), err, len(ids))
        worst = max(worst, err)
        check_decision(sc, int(e), pool.Y[row], sc.GetCtrl(int(e)))
    assert_unchanged(sc, before, n_out, len(ids))
    for a, b in zip(q0, sc.GetStateAll()):
        assert np.array_equal(a, b)            # a decision commits an action; the pose and velocity of every env stay
    return worst


def watch_set(n, ids, rng, cap):
    """the envs outside the list whose blocks are compared: all of them up to `cap`; beyond, the ones a row / env mix-up or an
    overlong row bound reaches first (ids below the row count + 64, the listed envs' neighbours) plus `cap` drawn at random"""
    rest = np.setdiff1d(np.arange(n), ids)
    if rest.size <= cap:
        return rest
    near = np.concatenate([np.arange(min(n, len(ids) + 64)), np.asarray(ids) - 1, np.asarray(ids) + 1])
    return np.union1d(np.intersect1d(near, rest), rng.choice(rest, cap, replace=False))


def batch_invariance(sc, pool, envs, positions, batch, n_out, seed=0):
    """env e's outputs and control block are bit-identical whether it is decided alone or at row p of a `batch`-row pass, with the
    same state each time and other envs (not in `envs`) around it.  (Deciding e twice in a row leaves the same control block: the
    second commit sees the same stashed COM, so prev_dist is 0 both times.)"""
    rng = np.random.default_rng(seed)
    others = np.setdiff1d(np.arange(sc.num_envs), envs)
    for j, e in enumerate(envs):
        x = pool.X[(e * 7 + 11 * j) % pool.P][None]
        sc.DebugDecide([e], x)
        sc.DebugDecide([e], x)
        ref = (sc.GetNetOut(e, n_out), sc.GetCtrl(e))
        for p in positions:
            ids = rng.choice(others, batch - 1, replace=False)
            ids = np.insert(ids, p, e).astype(np.int32)
            X = pool.X[pool.rows(ids)]
            X[p] = x[0]
            sc.DebugDecide(ids, X)
            got = (sc.GetNetOut(e, n_out), sc.GetCtrl(e))
            assert np.array_equal(got[0], ref[0]), ("net output depends on the batch", e, p, np.max(np.abs(got[0] - ref[0])))
            assert np.array_equal(got[1], ref[1]), ("control block depends on the batch", e, p)


def refuses_bad_lists(sc):
    n = sc.num_envs
    for ids, msg in (([0, n], "out of range"), ([-1], "out of range"), ([3, 1, 3], "listed twice")):
        with pytest.raises(RuntimeError, match=msg):
            sc.DebugDecide(ids)
    import ctypes as C
    ids = np.arange(n, dtype=np.int32)
    assert sc.L.trl_debug_decide(sc.h, ids.ctypes.data_as(C.c_void_p), n + 1, None) != 0
    assert b"count out of range" in sc.L.trl_last_error()
    assert sc.L.trl_debug_decide(None, None, 0, None) != 0 and b"null handle" in sc.L.trl_last_error()


# ------------------------------------------------------------------------------------------------ GPU
def _net(assets, scene):
    from pack_scene import read_pack
    return torch_net.blobs_from_pack(read_pack(os.path.join(assets, scene + ".trlpack")))


_RECORDED = {}


def recorded_states(assets, scene):
    """policy states of a real run: 32 envs after 1 s, every one of them past its first decision"""
    if scene not in _RECORDED:
        import deepterrainrl_b200 as trl
        sc = trl.ScenarioPoliEval(os.path.join(assets, scene + ".trlpack"), 32)
        for _ in range(30):
            sc.Update()
        _RECORDED[scene] = np.stack([sc.GetPoliState(e) for e in range(32)])
        sc.close()
    return _RECORDED[scene]


def _special(assets, scene, seed):
    net = _net(assets, scene)
    return net, np.concatenate([recorded_states(assets, scene), edge_states(net[1], net[2], 4, seed)])


@pytest.mark.parametrize("scene,n", [("dog_slopes_mixed", 8), ("dog_slopes_mixed", 1000), ("dog_slopes_mixed", 4096),
                                     ("goat_cliffs", 8), ("goat_cliffs", 1000), ("raptor_narrow_gaps", 8),
                                     ("raptor_narrow_gaps", 1000)])
def test_decision_batches_match_torch(assets, scene, n):
    """every pending count x every id order: outputs of the listed envs vs torch, the committed action vs torch's arg-max and actor,
    every other env untouched (all of them up to 1024, beyond that the nearest ones + 1024 at random)"""
    import deepterrainrl_b200 as trl
    n_out = SCENES[scene]
    net, special = _special(assets, scene, 3)
    pool = StatePool(net, n, special, seed=n)
    sc = trl.ScenarioPoliEval(os.path.join(assets, scene + ".trlpack"), n)
    # policy evaluation: reset leaves no commanded action (I_CMD = -1), so decide_one takes the net path and writes net_out from the
    # first pass on; the first pass, all envs in order, also fills every pending-list entry
    worst = decide_and_check(sc, pool, env_ids("identity", n, n), n_out, watch=[])
    rng = np.random.default_rng(n)
    for order in ORDERS:
        for count in counts_for(n):
            ids = env_ids(order, count, n, seed=1)
            worst = max(worst, decide_and_check(sc, pool, ids, n_out, watch=watch_set(n, ids, rng, 1024)))
    print(f"\n{scene} n={n}: worst max|g - t| / (1 + |t|) = {worst:.3e} over {pool.calls} passes")
    sc.close()


@pytest.mark.parametrize("scene", list(SCENES))
def test_decision_is_independent_of_batch_position(assets, scene):
    """alone, row 0 and rows 200 / 230 / 256 of a 257-row pass (cluster 0's 4th chunk, cluster 1's 4th, cluster 0's 5th = a 1-row
    chunk): each output element is a fixed-order DMMA chain plus a rank-order DSMEM sum of its own row, so it is bit-identical"""
    import deepterrainrl_b200 as trl
    n = 1000
    net, special = _special(assets, scene, 5)
    pool = StatePool(net, n, special, seed=17)
    sc = trl.ScenarioPoliEval(os.path.join(assets, scene + ".trlpack"), n)
    batch_invariance(sc, pool, [0, 5, 600, 999], [0, 31, 32, 200, 230, 256], 257, SCENES[scene], seed=2)
    refuses_bad_lists(sc)
    # n = 0 changes nothing
    before = snapshot(sc, range(0, n, 7), SCENES[scene])
    sc.DebugDecide([])
    assert_unchanged(sc, before, SCENES[scene], 0)
    sc.close()


@pytest.mark.parametrize("scene", list(SCENES))
def test_batched_pass_matches_one_cluster_pass(assets, scene, monkeypatch):
    """trl_decide2.cuh's claim: the batched pass differs from the one-cluster-per-decision pass (trl_decide.cuh, TRL_DECIDE_V1=1)
    only in summation order, <= 1e-13 relative on the net outputs"""
    import deepterrainrl_b200 as trl
    n, n_out = 300, SCENES[scene]
    net, special = _special(assets, scene, 7)
    pool = StatePool(net, n, special, seed=23)
    pack = os.path.join(assets, scene + ".trlpack")
    v2 = trl.ScenarioPoliEval(pack, n)
    monkeypatch.setenv("TRL_DECIDE_V1", "1")
    v1 = trl.ScenarioPoliEval(pack, n)
    monkeypatch.delenv("TRL_DECIDE_V1")
    gap = 0.0
    for order, count in (("permuted", n), ("reversed", 257), ("strided", 67), ("last", 33)):
        ids = env_ids(order, count, n, seed=4)
        X = pool.X[pool.rows(ids)]
        v2.DebugDecide(ids, X)
        v1.DebugDecide(ids, X)
        for e in ids:
            a, b = v2.GetNetOut(int(e), n_out), v1.GetNetOut(int(e), n_out)
            gap = max(gap, _relerr(a, b))
            assert np.abs(a).max() > 0
    print(f"\n{scene}: batched vs one-cluster pass, max |a - b| / (1 + |b|) = {gap:.3e}")
    assert gap <= 1e-13, gap
    v1.close(); v2.close()


def test_perturbed_weights(assets):
    """weights uploaded through SetWeights (blob order pack_scene.NET_LAYERS) reach every stage of the batched pass"""
    import deepterrainrl_b200 as trl
    from pack_scene import NET_LAYERS
    scene, n = "dog_slopes_mixed", 1000
    n_out = SCENES[scene]
    blobs, io, isc, oo, osc = _net(assets, scene)
    rng = np.random.default_rng(31)
    pert = {k: (w * (1.0 + 0.1 * rng.normal(size=w.shape)), b + 0.05 * rng.normal(size=b.shape)) for k, (w, b) in blobs.items()}
    special = np.concatenate([recorded_states(assets, scene), edge_states(io, isc, 4, 9)])
    pool = StatePool((pert, io, isc, oo, osc), n, special, seed=41)
    base = StatePool((blobs, io, isc, oo, osc), n, special, seed=41)
    assert np.max(np.abs(pool.Y - base.Y)) > 1e-2              # the perturbation matters
    sc = trl.ScenarioPoliEval(os.path.join(assets, scene + ".trlpack"), n)
    flat = []
    for name in NET_LAYERS:
        flat += [pert[name][0], pert[name][1]]
    sc.SetWeights(flat, io, isc, oo, osc)
    worst = 0.0
    for order, count in (("identity", n), ("permuted", 257), ("reversed", 129), ("last", 65), ("strided", 33), ("permuted", 1)):
        ids = env_ids(order, count, n, seed=6)
        worst = max(worst, decide_and_check(sc, pool, ids, n_out, watch=watch_set(n, ids, rng, 256)))
    print(f"\nperturbed weights: worst max|g - t| / (1 + |t|) = {worst:.3e}")
    sc.close()


def test_exploring_decision_is_independent_of_batch(assets):
    """exploration on (Boltzmann actor choice, parameter noise, base actions): env e decided alone in one handle and at row >= 200
    of a 257-row pass in a second handle with the same rng_seed commits the same action, flags and outputs, bit for bit; a further
    decision on both agrees too, so the stored random-stream position matched"""
    import deepterrainrl_b200 as trl
    scene, n = "dog_slopes_mixed", 300
    n_out = SCENES[scene]
    pack = os.path.join(assets, scene + ".trlpack")
    net, special = _special(assets, scene, 11)
    pool = StatePool(net, n, special, seed=29)
    a = trl.ScenarioExpMACE(pack, n, rng_seed=77)
    b = trl.ScenarioExpMACE(pack, n, rng_seed=77)
    X0 = pool.X[pool.rows(np.arange(n))]
    for sc in (a, b):
        sc.EnableExplore(1, 0.2, 0.025, 0.002)
        sc.DebugDecide(np.arange(n), X0)      # the commanded actions of the exploration reset; from here on decisions use the net
    test_envs = [3, 64, 150, 299, 0, 200, 101, 17]
    others = np.setdiff1d(np.arange(n), test_envs)
    rng = np.random.default_rng(5)
    explored = 0
    for j, e in enumerate(test_envs):
        x = pool.X[(13 * e + j) % pool.P]
        a.DebugDecide([e], x[None])
        p = 200 + 7 * j
        ids = np.insert(rng.choice(others, 256, replace=False), p, e).astype(np.int32)
        X = pool.X[pool.rows(ids)]
        X[p] = x
        b.DebugDecide(ids, X)
        for step in ("alone vs in a batch", "the next decision"):
            ca, cb = a.GetCtrl(e), b.GetCtrl(e)
            assert np.array_equal(ca, cb), (e, step)               # action, parameters, exp_critic / exp_actor flags
            assert np.array_equal(a.GetNetOut(e, n_out), b.GetNetOut(e, n_out)), (e, step)
            explored += int(ca[-4] + ca[-3] > 0)
            x2 = pool.X[(29 * e + j + 1) % pool.P][None]
            a.DebugDecide([e], x2)
            b.DebugDecide([e], x2)
    assert explored > 0                           # the comparison covered exploring decisions
    a.close(); b.close()
