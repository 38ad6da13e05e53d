"""The CUDA kernel *sources* executed on the CPU, thread for thread, by the test-only SIMT emulator (tests/simt/): every CUDA
thread is a fiber, warp collectives / __syncthreads / cluster.sync() are barriers, streams run in issue order, graphs replay.

What this tier pins without a GPU (the `-m gpu` tests remain the parity tests proper -- the emulator's arithmetic is not
FMA-contracted, so it is not the GPU's rounding):
  * the env-step, decision, terrain, reset, statistics and trainer kernels, driven through the real host code behind the C ABI
    (graph capture, overlapped two-stream schedule, pending lists), against the CPU oracle;
  * convergence: a collective some live lane does not reach deadlocks the fibers and aborts the test;
  * races: with a seeded scheduler the lanes of a warp run in varying orders between collectives, so a shared-memory hand-off
    without its barrier gives seed-dependent results -- results must be bit-identical across seeds;
  * experimental kernel variants (TRL_NVCC_EXTRA knobs of the nvcc build) are bit-identical to the default build before any
    GPU time is spent on them.
Nothing here is a fallback of the product: the library is built under tests/simt/_build/ and only this file loads it."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "simt"))
from loader import open_simt, simt_library  # noqa: E402

H = 1.0 / 600.0
pytestmark = pytest.mark.skipif(__import__("platform").machine() != "x86_64",
                                reason="the emulator's fiber switch is written for x86-64")


def _relerr(a, b):
    return np.max(np.abs(a - b) / (1.0 + np.abs(b)))


# ------------------------------------------------------------------------------------------------ the emulator itself
def _selftest(L, which, arg=0, seed=0):
    out = np.zeros(4096, np.int32)
    L.simt_set_sched_seed(C.c_ulonglong(seed))
    try:
        assert L.simt_selftest(which, out.ctypes.data_as(C.c_void_p), arg) == 0
    finally:
        L.simt_set_sched_seed(C.c_ulonglong(0))
    return out


def test_emulator_collectives_clusters_and_race_detection():
    L = open_simt()
    o = _selftest(L, 0)   # shuffle from lane+1, ballot of the odd lanes, xor-butterfly sum, double shuffle
    for blk in range(3):
        for t in range(64):
            lane = t & 31
            assert o[blk * 64 + t] == 100 * blk + (t & 32) + ((lane + 1) & 31) + 1000 * 16 + 100000 * 496
    # shared-memory neighbour exchange: with its __syncwarp the result does not depend on the schedule ...
    ref = _selftest(L, 1, 1)
    for r in range(4):
        for t in range(64):
            assert ref[r * 64 + t] == 10 * r + ((t & 32) | ((t + 1) & 31))
    assert all(np.array_equal(ref, _selftest(L, 1, 1, s)) for s in (7, 77, 123456))
    # ... without it, it does: this is how the kernel tests below would see a missing barrier
    assert any(not np.array_equal(_selftest(L, 1, 0), _selftest(L, 1, 0, s)) for s in (7, 77, 123456))
    o = _selftest(L, 2)   # 2 clusters x 4 CTAs x 96 threads: rank r reads rank r+1's dynamic shared memory
    for blk in range(8):
        peer = (blk // 4) * 4 + (blk % 4 + 1) % 4
        for t in range(96):
            assert o[blk * 96 + t] == 1000 * peer + (t + 3) % 96
    o = _selftest(L, 3)   # __syncthreads_or + barriers after two of four warps have exited
    assert (o[:64] == 100000 + 2016).all() and (o[64:256] == 0).all()


# ------------------------------------------------------------------------------------------------ kernels vs the oracle
def _pair(assets, name, n, mode=0, rng_seed=1234):
    from pyoracle import Oracle
    import deepterrainrl_b200 as trl
    pack = os.path.join(assets, name)
    cls = trl.ScenarioExpMACE if mode else trl.ScenarioPoliEval
    return cls(pack, n, rng_seed=rng_seed), Oracle(pack, n, mode, rng_seed=rng_seed)


def test_step_kernel_flat_dog_vs_oracle(assets):
    """BASELINE config 1 through the kernel source: q, qd, torques, contact bits, gait state every step."""
    with simt_library():
        g, o = _pair(assets, "dog_flat.trlpack", 1)
        for k in range(120):
            g.EnvStep(H)
            o.env_step(0, H)
            gq, gqd, gt, gc = g.GetState(0)
            oq, oqd, ot, oc = o.get_state(0)
            assert _relerr(gq, oq) < 1e-9 and _relerr(gqd, oqd) < 1e-8 and _relerr(gt, ot) < 1e-8, k
            np.testing.assert_array_equal(gc, oc)
            assert g.GetCtrl(0)[0] == o.get_ctrl(0)[0]
        g.close()


@pytest.mark.parametrize("scene,steps", [("dog_slopes_mixed", 140), ("raptor_narrow_gaps", 100), ("goat_cliffs", 100)])
def test_step_and_decision_kernels_vs_oracle(assets, scene, steps):
    """Policy in the loop: terrain bit-exact, the cluster decision kernel's network output, states after the decisions."""
    n = 3
    with simt_library():
        g, o = _pair(assets, scene + ".trlpack", n)
        for env in range(n):
            for seg in (0, 1):
                gd, gmx, gfl = g.GetTerrain(env, seg)
                od, omx, ofl = o.terrain(env, seg)
                assert gmx == omx and gfl == ofl
                np.testing.assert_array_equal(gd, od)
        for k in range(steps):
            g.EnvStep(H)
            for e in range(n):
                o.env_step(e, H)
        for e in range(n):
            gq, gqd, gt, gc = g.GetState(e)
            oq, oqd, ot, oc = o.get_state(e)
            assert _relerr(gq, oq) < 1e-8 and _relerr(gqd, oqd) < 1e-7, (scene, e)
            np.testing.assert_array_equal(gc, oc)
        np.testing.assert_allclose(g.GetPoliState(0), o.poli_state(0), rtol=1e-9, atol=1e-9)
        np.testing.assert_allclose(g.GetNetOut(0), o.net_out(0), rtol=1e-8, atol=1e-8)
        g.close()


@pytest.mark.parametrize("scene", ["dog_slopes_mixed", "raptor_narrow_gaps"])
def test_kernel_sources_reproduce_the_compiled_reference(assets, scene):
    """tests/test_gpu_ref_golden.py without the GPU: the kernel sources against the torques / gait states the reference's own
    compiled controller stack + cJoint clamp produced (tests/golden/ref_scenario_*.npz, tools/make_ref_golden.py)."""
    import deepterrainrl_b200 as trl
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_scenario_%s.npz" % scene))
    applied, fsm = g["applied"], g["fsm"]
    with simt_library():
        sc = trl.ScenarioPoliEval(os.path.join(assets, scene + ".trlpack"), 1, terrain_seeds=[int(g["seed"])])
        n = min(400, len(applied))
        for k in range(n):
            sc.EnvStep(H)
            _, _, tau, _ = sc.GetState(0)
            err = np.max(np.abs(tau - applied[k]) / (1.0 + np.abs(applied[k])))
            assert err < 1e-7, (scene, k, err)
            assert int(sc.GetCtrl(0)[0]) == int(fsm[k, 0]), (scene, k, "gait state")
        sc.close()


@pytest.mark.parametrize("scene,vertex", [("dog_slopes_mixed", False), ("raptor_narrow_gaps", False), ("goat_cliffs", True)])
def test_forced_steps_and_stress_states_vs_oracle(assets, monkeypatch, scene, vertex):
    """tests/test_gpu_step_forced.py in miniature: 3 envs, 40 forced env-steps (each from the oracle's state), then one instance
    of every stress kind (two of friction: below and above v_eps), 5 forced steps each.  Without FMA contraction q, the
    controller block, the policy state and the net output agree to 1e-12.  qd and the held torque come out of the two
    different solves (articulated-body passes here, CRBA + LDL^T in the oracle): the oracle itself moves them by 1e-12 .. 4e-12
    when its input state is perturbed by 1e-15 relative, so they are held to 5e-11, and q, which integrates qd over the step,
    to 5e-12; a stiff stress state, where 100x that sensitivity is larger, is held to that instead (F.Sensitivity).  The goat runs the vertex contact model
    (TRL_VERTEX_CONTACTS=1 / ORC_VTX=1), with two more states that put a convex terrain vertex into a box.

    Planted one at a time in trl_step.cu, each of these makes this test fail (and each also fails some older test of this file):
    the dt * cl joint-limit armature dropped from the chain pass (all three cases; qd off by 1e-2 .. 2), the touching test
    pen > -contact_tol changed to pen > 0 (all three; contact bits differ), kClearMargin = 0 (raptor and goat; a contact bit of
    a corner in the touching band above the window maximum differs), ci & 3 changed to ci & 1 in the vertex rounds (goat; qd
    off by 0.36)."""
    import test_gpu_step_forced as F
    n = 3
    kinds = F.KINDS + ("friction",) + (("vertex", "vertex") if vertex else ())
    if vertex:
        monkeypatch.setenv("TRL_VERTEX_CONTACTS", "1")
        monkeypatch.setenv("ORC_VTX", "1")
    with simt_library():
        g, o, m = F.make_pair(assets, scene, n)
        sens = F.Sensitivity(assets, scene, n)
        worst = F.Worst({"default": 1e-12, "q": 5e-12, "qd": 5e-11, "tau": 5e-11})
        F.forced_steps(g, o, m, range(n), 40, worst, scene, sens=sens)
        cov = F.stress_rounds(g, o, m, n, 4 if vertex else 3, worst, scene, seed=11, kinds=kinds, sens=sens)
        g.close()
    worst.report()
    cov.check(scene, kinds)


def test_update_graph_overlapped_schedule_and_tuples_vs_oracle(assets):
    """trl_update: captured graph, two-stream schedule with catch-up launches, exploration on; tuples and counters."""
    n = 4
    with simt_library():
        g, o = _pair(assets, "dog_slopes_mixed.trlpack", n, mode=1)
        g.EnableExplore(1, 0.2, 0.025, 0.002)
        o.set_explore(1, 0.2, 0.025, 0.002)
        for k in range(45):
            g.Update(1.0 / 30.0)
            o.update(1.0 / 30.0, threads=4)
        gr, gf, ge = g.GetTuples(f64=True)
        orr, of, oe = o.tuples()
        assert gr.shape == orr.shape and gr.shape[0] > 0
        gi = np.lexsort((np.arange(len(ge)), ge))
        oi = np.lexsort((np.arange(len(oe)), oe))
        np.testing.assert_array_equal(ge[gi], oe[oi])
        np.testing.assert_array_equal(gf[gi], of[oi])
        np.testing.assert_allclose(gr[gi], orr[oi], rtol=1e-7, atol=1e-7)
        g.close()


def test_serial_schedule_single_env_reset_and_two_scenes(assets, monkeypatch):
    """Host paths of tests/test_gpu_scenarios.py in miniature: the overlapped two-stream schedule equals the serial one bit for
    bit (states, counters, tuples as sets); trl_reset of one env / trl_set_state leave the neighbours alone; two handles with
    different scenes interleave (the constant-memory model is re-uploaded on every switch)."""
    import deepterrainrl_b200 as trl
    dog = os.path.join(assets, "dog_slopes_mixed.trlpack")
    rap = os.path.join(assets, "raptor_narrow_gaps.trlpack")
    with simt_library():
        n = 5
        monkeypatch.setenv("TRL_SERIAL_SCHEDULE", "1")
        ser = trl.ScenarioExpMACE(dog, n, rng_seed=7)
        monkeypatch.setenv("TRL_SERIAL_SCHEDULE", "0")
        ovl = trl.ScenarioExpMACE(dog, n, rng_seed=7)
        for sc in (ser, ovl):
            sc.EnableExplore(True, 0.2, 0.025, 0.01)
        l0s, l0o = ser.KernelLaunches(), ovl.KernelLaunches()
        for _ in range(36):
            ser.Update(1.0 / 30.0)
            ovl.Update(1.0 / 30.0)
        assert ser.KernelLaunches() - l0s == 36 * 62 and ovl.KernelLaunches() - l0o == 36 * 80   # terrain + 21 steps + 20 x (conv + FC) decision launches (+ 19 catch-ups)
        for a, b in zip(ser.GetStateAll(), ovl.GetStateAll()):
            np.testing.assert_array_equal(a, b)
        assert ser._stats() == ovl._stats()
        ra, fa, ea = ser.GetTuples(f64=True)
        rb, fb, eb = ovl.GetTuples(f64=True)
        assert ra.shape == rb.shape and ra.shape[0] >= n
        ka = np.lexsort(np.column_stack([ea, fa, ra]).T[::-1])
        kb = np.lexsort(np.column_stack([eb, fb, rb]).T[::-1])
        np.testing.assert_array_equal(ea[ka], eb[kb])
        np.testing.assert_array_equal(fa[ka], fb[kb])
        np.testing.assert_array_equal(ra[ka], rb[kb])
        # one env reset / state installed, neighbours untouched
        q0 = trl.ScenarioExpMACE(dog, 1, rng_seed=7).GetState(0)
        q1, qd1, tau1, c1 = ovl.GetState(3)
        other = ovl.GetState(4)[0].copy()
        ovl.Reset([3])
        q2, qd2, tau2, _ = ovl.GetState(3)
        np.testing.assert_array_equal(q2[2:], q0[0][2:])
        np.testing.assert_array_equal(qd2, q0[1])
        assert np.all(tau2 == 0)
        np.testing.assert_array_equal(ovl.GetState(4)[0], other)
        ovl.SetState(2, q=q1, qd=qd1, tau=tau1, contact=c1)
        q3, qd3, tau3, c3 = ovl.GetState(2)
        assert all(np.array_equal(x, y) for x, y in ((q3, q1), (qd3, qd1), (tau3, tau1), (c3, c1)))
        ser.close(); ovl.close()
        # two scenes alive at once
        a = trl.ScenarioPoliEval(dog, 3)
        for _ in range(4):
            a.Update(1.0 / 30.0)
        qa = a.GetStateAll()[0].copy()
        b = trl.ScenarioPoliEval(rap, 3)
        for _ in range(4):
            b.Update(1.0 / 30.0)
        qb = b.GetStateAll()[0].copy()
        a2, b2 = trl.ScenarioPoliEval(dog, 3), trl.ScenarioPoliEval(rap, 3)
        for _ in range(4):
            a2.Update(1.0 / 30.0)
            b2.Update(1.0 / 30.0)
        np.testing.assert_array_equal(a2.GetStateAll()[0], qa)
        np.testing.assert_array_equal(b2.GetStateAll()[0], qb)
        for sc in (a, b, a2, b2):
            sc.close()


def test_env_groups_match_the_monolithic_launch(assets, monkeypatch):
    """TRL_GROUPS=G splits every main step launch into G launches over contiguous env ranges on G streams (they only meet at the
    decision / catch-up launches): states, counters and tuples are bit-identical to the one-launch schedule; a group count that
    would leave a group empty is reduced.  (The same comparison runs at 1000 envs and G = 1 / 3 / 8 on the GPU:
    tests/test_gpu_scenarios.py::test_env_groups_match_monolithic_launch.)"""
    import deepterrainrl_b200 as trl
    dog = os.path.join(assets, "dog_slopes_mixed.trlpack")
    with simt_library():
        n = 18           # G = 2 -> chunk 16: groups [0,16) [16,18)
        scs = []
        for G in ("1", "2"):
            monkeypatch.setenv("TRL_GROUPS", G)
            scs.append(trl.ScenarioExpMACE(dog, n, rng_seed=7))
        monkeypatch.setenv("TRL_GROUPS", "8")
        tiny = trl.ScenarioExpMACE(dog, 5, rng_seed=7)     # 8 groups of >= 16 envs cannot be filled from 5 envs
        monkeypatch.delenv("TRL_GROUPS")
        lt = tiny.KernelLaunches()
        tiny.Update(1.0 / 30.0)
        assert tiny.KernelLaunches() - lt == 80
        tiny.close()
        for sc in scs:
            sc.EnableExplore(True, 0.2, 0.025, 0.01)
        l0 = [sc.KernelLaunches() for sc in scs]
        nu = 8           # 160 env-steps: every env has taken its first decision through the pending lists (tuples come later: GPU test)
        for _ in range(nu):
            for sc in scs:
                sc.Update(1.0 / 30.0)
        got = [sc.KernelLaunches() - a for sc, a in zip(scs, l0)]
        assert got == [nu * 80, nu * 100], got
        ref = scs[0]
        for sc in scs[1:]:
            for a, b in zip(ref.GetStateAll(), sc.GetStateAll()):
                np.testing.assert_array_equal(a, b)
            assert ref._stats() == sc._stats()
            for e in (0, 15, 16, 17):
                np.testing.assert_array_equal(ref.GetPoliState(e), sc.GetPoliState(e))
        for sc in scs:
            sc.close()


def test_trainer_kernels_vs_oracle(assets):
    from pyoracle import OracleTrainer
    from test_gpu_trainer import _synthetic_tuples
    import deepterrainrl_b200 as trl
    pack = os.path.join(assets, "dog_slopes_mixed.trlpack")
    kw = dict(num_init_samples=96, num_steps_per_iter=1, freeze_target_iters=3, init_input_offset_scale=1, seed=21)
    with simt_library():
        sc = trl.ScenarioExpMACE(pack, 4)
        g = trl.MACETrainer(sc, replay_mem_size=160, **kw)
        o = OracleTrainer(pack, replay_cap=160, **kw)
        rows, flags = _synthetic_tuples(128, g.S, g.A, o.get("in_off"), o.get("in_scale"), 3)
        g.AddTuples(rows, flags)
        o.add_tuples(rows, flags)
        for it in range(2):   # the second iteration includes an actor step
            l0 = g.KernelLaunches()
            g.Train(1)
            assert g.KernelLaunches() - l0 == 40
            o.train()
            cg, co = g.counters(), o.counters()
            for k in ("iter", "actor_iter", "stage", "num", "head", "total", "critic", "actor", "actor_batch"):
                assert cg[k] == co[k], (it, k)
            np.testing.assert_array_equal(g.lists("critic"), o.lists("critic"))
            tg, to = g.get("theta"), o.get("theta")
            assert np.max(np.abs(tg - to)) <= 1e-12 * max(1.0, np.max(np.abs(to))), it
        assert co["actor_iter"] >= 1
        # a second batch wraps the 160-slot ring onto used slots: the warp-cooperative slot assignment must fall back to the reference's
        # sequential order (buffers move between the critic and the actor list, the pending actor batch loses overwritten slots)
        rows2, flags2 = _synthetic_tuples(100, g.S, g.A, o.get("in_off"), o.get("in_scale"), 4)
        g.AddTuples(rows2, flags2)
        o.add_tuples(rows2, flags2)
        cg, co2 = g.counters(), o.counters()
        for k in ("num", "head", "total", "critic", "actor", "actor_batch"):
            assert cg[k] == co2[k], k
        for which in ("critic", "actor", "actor_batch"):
            np.testing.assert_array_equal(g.lists(which), o.lists(which))
        # ... and a small ring that wraps several times with mixed flags (list tails inside and outside the batch's own slots)
        kw2 = dict(kw, num_init_samples=10 ** 6)
        sc2 = trl.ScenarioExpMACE(pack, 4)
        g2 = trl.MACETrainer(sc2, replay_mem_size=96, **kw2)
        o2 = OracleTrainer(pack, replay_cap=96, **kw2)
        for rnd in range(7):
            rw, fl = _synthetic_tuples(37 + 11 * rnd, g.S, g.A, o.get("in_off"), o.get("in_scale"), 10 + rnd)
            g2.AddTuples(rw, fl)
            o2.add_tuples(rw, fl)
            c1, c2 = g2.counters(), o2.counters()
            for k in ("num", "head", "total", "critic", "actor", "actor_batch"):
                assert c1[k] == c2[k], (rnd, k)
            for which in ("critic", "actor"):
                np.testing.assert_array_equal(g2.lists(which), o2.lists(which))
        g2.close(); sc2.close()
        # destroying the scenario first leaves the trainer an inert shell: calls fail with a message, destroy is harmless
        sc.close()
        with pytest.raises(RuntimeError, match="has been destroyed"):
            g.Train(1)
        g.close()


def test_trainer_kernels_have_no_schedule_dependent_results(assets):
    """The trainer's kernels lean on __syncthreads and shared-memory staging: same race check as for the
    step / decision kernels -- a permuted thread schedule must not change a single weight."""
    from test_gpu_trainer import _synthetic_tuples
    import deepterrainrl_b200 as trl
    pack = os.path.join(assets, "raptor_narrow_gaps.trlpack")
    kw = dict(num_init_samples=64, num_steps_per_iter=1, freeze_target_iters=3, init_input_offset_scale=1, seed=5)
    thetas = []
    with simt_library() as L:
        for seed in (0, 31337):
            sc = trl.ScenarioExpMACE(pack, 2)
            g = trl.MACETrainer(sc, replay_mem_size=128, **kw)
            rows, flags = _synthetic_tuples(96, g.S, g.A, g.get("in_off"), g.get("in_scale"), 8)
            L.simt_set_sched_seed(C.c_ulonglong(seed))
            try:
                g.AddTuples(rows, flags)
                g.Train(1)
            finally:
                L.simt_set_sched_seed(C.c_ulonglong(0))
            assert g.counters()["iter"] >= 1
            thetas.append(g.get("theta"))
            g.close(); sc.close()
    assert np.array_equal(thetas[0], thetas[1])


# ------------------------------------------------------------------------------------------------ schedules and variants
_REF_CACHE = {}


def _trajectory(defines, pack, n, steps, seed=0, updates=0, net_out=False):
    """(cached for the product build at seed 0: every variant test compares with the same reference run)"""
    key = (pack, n, steps, updates, net_out)
    if not defines and seed == 0:
        if key not in _REF_CACHE:
            _REF_CACHE[key] = _trajectory_run(defines, pack, n, steps, seed, updates, net_out)
        return _REF_CACHE[key]
    return _trajectory_run(defines, pack, n, steps, seed, updates, net_out)


def _trajectory_run(defines, pack, n, steps, seed, updates, net_out):
    import deepterrainrl_b200 as trl
    with simt_library(defines) as L:
        L.simt_set_sched_seed(C.c_ulonglong(seed))
        try:
            g = trl.ScenarioPoliEval(pack, n)
            out = []
            for k in range(steps):
                g.EnvStep(H)
                if k % 10 == 9:
                    q, qd = g.GetStateAll()
                    out.append(np.concatenate([q, qd]).copy())
            for k in range(updates):
                g.Update(1.0 / 30.0)
                q, qd = g.GetStateAll()
                out.append(np.concatenate([q, qd]).copy())
            y = np.stack([g.GetNetOut(e) for e in range(n)]) if net_out else None
            g.close()
        finally:
            L.simt_set_sched_seed(C.c_ulonglong(0))
        return (np.stack(out), y) if net_out else np.stack(out)


def test_kernels_have_no_schedule_dependent_results(assets):
    """Race check: the lanes of every warp run in seed-dependent orders between collectives; a shared-memory hand-off
    (mass matrix, L^T read-back, corner tables, decision activations, pending lists) without its barrier would show."""
    pack = os.path.join(assets, "dog_slopes_mixed.trlpack")
    ref = _trajectory([], pack, 3, 130, 0, updates=2)
    for seed in (11, 2024):
        assert np.array_equal(ref, _trajectory([], pack, 3, 130, seed, updates=2)), seed


VARIANTS = [
    ["-DTRL_ACCUM_SMEM=1"],
    ["-DTRL_LDLT_SMEM=1"],
    ["-DTRL_KIN_SMEM=1"],
    ["-DTRL_OUTWARD_SMEM=1"],
    ["-DTRL_CONTACT_SMEM=1"],
    ["-DTRL_SMEM_XCHG=1"],
    ["-DTRL_SMEM_XCHG=1", "-DTRL_REUSE_KIN=1"],
    ["-DTRL_DECIDE_TILE=1", "-DTRL_CONV_TILE=2"],
    ["-DTRL_DECIDE_TILE=1", "-DTRL_CONV_TILE=4"],
    ["-DTRL_LINK_SMEM=0"],
    ["-DTRL_FIELD_SMEM=1"],
    ["-DTRL_TABLE_MIRROR=0"],
    ["-DTRL_HOIST_LIMITS=0"],
]


@pytest.fixture(scope="module")
def variant_builds():
    """compile every experiment build up front, several at a time (g++ is the slow part of this file, not the emulation)"""
    from concurrent.futures import ThreadPoolExecutor
    import build as simt_build
    simt_build.build([])
    with ThreadPoolExecutor(4) as ex:
        list(ex.map(simt_build.build, VARIANTS))


@pytest.mark.parametrize("defines", VARIANTS, ids=lambda d: " ".join(d))
@pytest.mark.parametrize("scene", ["dog_slopes_mixed", "raptor_narrow_gaps", "goat_cliffs"])
def test_experimental_variant_is_bit_identical(assets, defines, scene, variant_builds):
    """Opt-in builds of the step kernel only move data differently: same values,
    same operation order -> bit-identical trajectories, also under a permuted lane schedule."""
    if "-DTRL_DECIDE_TILE=1" in defines:
        # decision-kernel variants: what matters is the network output of every decision, compared bit for bit
        if scene != "raptor_narrow_gaps" and defines[-1] != "-DTRL_CONV_TILE=4":
            pytest.skip("one scene per tile size (suite time)")
        pack = os.path.join(assets, scene + ".trlpack")
        ref_t, ref_y = _trajectory([], pack, 3, 130, updates=1, net_out=True)
        t, y = _trajectory(defines, pack, 3, 130, updates=1, net_out=True)
        assert np.array_equal(ref_y, y) and np.array_equal(ref_t, t) and np.abs(y).max() > 0
        return
    if scene == "goat_cliffs" and "-DTRL_SMEM_XCHG=1" not in defines:
        pytest.skip("third scene only for the all-on build (suite time)")
    pack = os.path.join(assets, scene + ".trlpack")
    ref = _trajectory([], pack, 3, 130, updates=1)
    assert np.array_equal(ref, _trajectory(defines, pack, 3, 130, updates=1))
    if "-DTRL_SMEM_XCHG=1" in defines or scene == "dog_slopes_mixed":
        assert np.array_equal(ref, _trajectory(defines, pack, 3, 130, seed=99, updates=1))


def test_decision_batches_vs_torch(assets):
    """The batched decision pass on chosen env lists (trl_debug_decide), the sweep of tests/test_gpu_decide_batches.py in miniature:
    70 envs, so 2 FC clusters x 32-row chunks and (4 emulated SMs) 2 conv clusters.  67 decisions = a second chunk on cluster 0, ragged,
    running past row 70 of act2 into the zero fill; permuted / reversed / tail / strided lists.  Outputs vs torch f64, the committed
    action vs torch's arg-max, every other env untouched, an env's output bit-identical alone and at rows 0 / 66.  The emulator copies
    the tiles TMA would load, so this pins the row / env / chunk indexing, not the TMA ring (that is the GPU test's part)."""
    import torch_net
    from pack_scene import read_pack
    from test_gpu_decide_batches import StatePool, assert_unchanged, batch_invariance, decide_and_check, edge_states, env_ids, \
        refuses_bad_lists, snapshot
    import deepterrainrl_b200 as trl
    pack = os.path.join(assets, "dog_slopes_mixed.trlpack")
    net = torch_net.blobs_from_pack(read_pack(pack))
    recorded = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "first_decision.npz"))["poli_state"]
    n = 70
    pool = StatePool(net, n, np.concatenate([recorded[None], edge_states(net[1], net[2], 2, 3)]), seed=1)
    with simt_library():
        sc = trl.ScenarioPoliEval(pack, n)
        worst = decide_and_check(sc, pool, env_ids("identity", n, n), 90, watch=[])
        for order, count in (("permuted", 67), ("reversed", 65), ("last", 33), ("strided", 5)):
            worst = max(worst, decide_and_check(sc, pool, env_ids(order, count, n, seed=1), 90))
        assert worst <= 1e-10, worst
        before = snapshot(sc, range(n), 90)
        sc.DebugDecide([])
        assert_unchanged(sc, before, 90, 0)
        batch_invariance(sc, pool, [4], [0, 66], 67, 90)
        refuses_bad_lists(sc)
        sc.close()


def test_layer_state_probe_vs_oracle(assets):
    """trl_get_layer_state (csrc/trl_probe.cu; cNeuralNet::GetLayerState behind RecordNNActivation) on the emulator against the oracle's
    blobs (oracle/net.h: layer_state, itself checked against torch in tests/test_net_torch_cpu.py) for every top of the deploy net"""
    import ctypes as C
    from pyoracle import Oracle
    import deepterrainrl_b200 as trl
    pack = os.path.join(assets, "raptor_narrow_gaps.trlpack")
    names = ["data", "data_terrain", "data_char", "char_flatten0", "terr_conv0", "terr_relu0", "terr_conv1", "terr_relu1", "terr_conv2", "terr_relu2",
             "terr_ip0", "terr_relu3", "concat0", "ip0", "relu0", "output"] + [h + s for h in ("val", "a0", "a1", "a2") for s in ("_ip0", "_relu0", "_ip1")]
    with simt_library():
        sc = trl.ScenarioPoliEval(pack, 3)
        for _ in range(3):
            sc.Update()
        x = sc.GetPoliState(2)
        o = Oracle(pack, 1, 0)
        o.L.orc_net_layer.restype = C.c_int
        for name in names:
            buf = np.zeros(8192)
            n = o.L.orc_net_layer(o.h, x.ctypes.data_as(C.c_void_p), name.encode(), buf.ctypes.data_as(C.c_void_p), 8192)
            g = sc.GetLayerState(name, 2)
            assert n == g.size > 0, name
            assert np.max(np.abs(g - buf[:n]) / (1.0 + np.abs(buf[:n]))) <= 1e-13, name
        sc.close()


def _loopback_comm(sc):
    """a single-rank communicator whose collectives are memory copies (trl_comm_init_external)"""
    from deepterrainrl_b200.parallel import _Collectives

    def all_gather(ctx, send, recv, nbytes, stream):
        C.memmove(recv, send, nbytes)
        return 0
    fns = (_Collectives.AG(all_gather), _Collectives.BC(lambda ctx, buf, nbytes, root, stream: 0), _Collectives.AR(lambda ctx, buf, count, stream: 0))
    coll = _Collectives(None, *fns)
    assert sc.L.trl_comm_init_external(sc.h, C.byref(coll), 0, 1) == 0, sc.L.trl_last_error().decode()
    return coll, fns


def test_asynchronous_trainer_loop(assets):
    """trl_trainer_set_async + trl_train_run_timed (the reference's asynchronous trainer semantics): hand-over and training on their
    own stream, policy snapshot refreshed between updates: the mechanics on the emulator -- one trainer job per update, the last one
    flushed, mode switch back (tuple flow and reproducibility of the overlapped run: tests/test_gpu_comm.py on the GPU)."""
    import deepterrainrl_b200 as trl
    pack = os.path.join(assets, "dog_slopes_mixed.trlpack")
    sp = np.array([0.5, 0.2, 20.0, 0.025, 0.3, 0.002, 12.0, 8.0, 0.0])
    with simt_library() as L:
        L.trl_train_run_timed.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_double, C.c_int, C.c_void_p, C.c_void_p]
        sc = trl.ScenarioExpMACE(pack, 6, rng_seed=31)
        tr = trl.MACETrainer(sc, replay_mem_size=320, num_init_samples=16, freeze_target_iters=3, seed=9)
        # a critic batch needs 32 tuples: seed the replay memory so that the short rollout below trains from its first job on
        rng = np.random.default_rng(1)
        rows = rng.normal(size=(48, tr.W)) * 0.1
        rows[:, 1 + tr.S] = rng.integers(0, 3, 48)
        tr.AddTuples(rows, np.zeros(48, np.uint32))
        keep = _loopback_comm(sc)
        assert L.trl_trainer_set_async(tr.h, 1) == 0, L.trl_last_error().decode()
        theta0 = tr.get("theta")
        state, ms = C.c_int64(0), C.c_double(0)
        updates, iters = 4, 1
        assert L.trl_train_run_timed(tr.h, sp.ctypes.data_as(C.c_void_p), updates, iters, 32, C.c_double(1.0 / 30.0), 0, C.byref(state),
                                     C.byref(ms)) == 0, L.trl_last_error().decode()
        c = tr.counters()
        assert state.value == updates * iters and c["iter"] == updates * iters             # one trainer job per update, the last one flushed
        assert c["total"] >= 48 and c["stage"] == 1 and sc.GetNumTuples() == 0               # (tuple flow itself: tests/test_gpu_comm.py, test_distributed_cpu.py)
        assert np.max(np.abs(tr.get("theta") - theta0)) > 0
        assert L.trl_trainer_set_async(tr.h, 0) == 0                                        # back to the pointer binding
        sc.Update(); sc.Sync()
        tr.close(); sc.close(); del keep


def test_vertex_contacts_opt_in_vs_oracle(assets, monkeypatch):
    """The opt-in contact model (terrain vertices inside body boxes, DESIGN §3) in the kernel sources against the oracle's: goat /
    cliffs, where step edges do enter boxes -- the trajectories differ from the default model's and agree with each other."""
    from pyoracle import Oracle
    import deepterrainrl_b200 as trl
    pack = os.path.join(assets, "goat_cliffs.trlpack")
    n, updates = 3, 26
    base = Oracle(pack, n, 0)
    for _ in range(updates):
        base.update(1.0 / 30.0, 1)
    monkeypatch.setenv("ORC_VTX", "1")
    monkeypatch.setenv("TRL_VERTEX_CONTACTS", "1")
    o = Oracle(pack, n, 0)                           # the switch is read when a scene is loaded
    with simt_library():
        g = trl.ScenarioPoliEval(pack, n)
        for _ in range(updates):
            g.Update(1.0 / 30.0); o.update(1.0 / 30.0, 1)
        gq, _ = g.GetStateAll()
        g.close()
    oq = np.stack([o.get_state(e)[0] for e in range(n)], axis=1)
    bq = np.stack([base.get_state(e)[0] for e in range(n)], axis=1)
    assert np.max(np.abs(gq - oq) / (1.0 + np.abs(oq))) < 1e-8
    assert np.max(np.abs(bq - oq)) > 1e-6            # the opt-in model did change the motion
