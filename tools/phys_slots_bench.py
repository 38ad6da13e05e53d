"""Physics slots on the GPU: Q contact settings evaluated in ONE handle (Q x M envs, envs on slots in contiguous blocks) against the
same Q settings evaluated one after another in handles of M envs whose trl_set_phys_params holds the setting (the plain step kernels).
The scene is dog / slopes_mixed with the pack's policy; setting 0 is the scene's own, settings 1.. vary the friction and the ground
stiffness.  Every arm: an untimed pre-roll to a steady state, warm-up updates, then K updates device-timed on the engine's stream with
an L2 flush between updates (trl_bench_updates, as bench.py times them).

    python tools/phys_slots_bench.py [--steps K] [--presim SECONDS] [--settings 1,2,4,8] [--envs 512,4096]
    python tools/phys_slots_bench.py --table [--table-envs M] [--seconds S]

The first form prints one JSON line per (Q, M) with env-steps/s of both arms.  --table runs, in one batch each, the pack's dog policy on
slopes_mixed across a friction x stiffness grid and the raptor pack on narrow_gaps across contact settings with and without vertex
contacts, and prints per setting the episodes, the mean distance at a fall and the share of envs whose run had no logged fall.  Both
print the card's name and power limit."""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from policy_slots_bench import card  # noqa: E402

DOG = os.path.join(ROOT, "assets", "dog_slopes_mixed.trlpack")
RAPTOR = os.path.join(ROOT, "assets", "raptor_narrow_gaps.trlpack")
DT = 1.0 / 30.0
DEFAULT = [2.0e5, 2.0e3, 0.81, 0.01, 0.00025, 2.0e4, 20.0]


def phys(kn=2.0e5, dn=2.0e3, mu=0.81, tol=0.00025, vertex=False):
    return dict(kn=kn, dn=dn, mu=mu, tol=tol, vertex=vertex)


def p7(s):
    return [s["kn"], s["dn"], s["mu"], DEFAULT[3], s["tol"], DEFAULT[5], DEFAULT[6]]


# throughput: the scene's own setting, then friction and stiffness variations
SWEEP = [phys(), phys(mu=0.5), phys(mu=1.2), phys(kn=1e5, dn=1e3), phys(mu=0.5, kn=1e5, dn=1e3), phys(mu=1.2, kn=1e5, dn=1e3),
         phys(mu=0.3), phys(kn=5e4, dn=5e2)]
# --table: slot 0 is each scene's own setting
DOG_GRID = [phys(mu=mu, kn=kn, dn=kn / 100) for kn in (2e5, 1e5) for mu in (0.81, 0.5, 1.2)]
RAPTOR_GRID = [phys(mu=mu, tol=tol, vertex=v) for v in (False, True) for tol in (0.00025, 0.001) for mu in (0.81, 1.2)]


def handle(trl, pack, n, settings, slots, seed0=1):
    """a pack handle with settings[1:] in physics slots 1.., envs on `slots` from their first episode on"""
    sc = trl.ScenarioPoliEval(pack, n, terrain_seeds=np.arange(seed0, seed0 + n, dtype=np.uint64))
    for q, s in enumerate(settings[1:], 1):
        sc.LoadPhysics(q, p7(s), s["vertex"])
    if len(settings) > 1:
        sc.SetEnvPhysics(slots)
        sc.SetRandSeed(np.arange(seed0, seed0 + n, dtype=np.uint64))
    return sc


def timed(sc, args):
    sc.BenchUpdates(int(round(args.presim / DT)), DT, flush_l2=False)
    sc.BenchUpdates(args.warmup, DT, flush_l2=True)
    return sc.BenchUpdates(args.steps, DT, flush_l2=True)


def throughput(trl, args, name, power):
    for M in [int(x) for x in args.envs.split(",")]:
        for Q in [int(x) for x in args.settings.split(",")]:
            steps = args.steps * 20 * Q * M
            sc = handle(trl, DOG, Q * M, SWEEP[:Q], np.repeat(np.arange(Q), M))
            mixed_ms = timed(sc, args)
            sc.close()
            seq_ms = 0.0
            for q in range(Q):
                sc = handle(trl, DOG, M, [SWEEP[0]], None, seed0=1 + q * M)
                sc.SetPhysParams(p7(SWEEP[q]))
                seq_ms += timed(sc, args)
                sc.close()
            print(json.dumps(dict(settings=Q, envs_per_setting=M, steps=args.steps, mixed_ms=round(mixed_ms, 3), sequential_ms=round(seq_ms, 3),
                                  mixed_env_steps_per_s=steps / (mixed_ms * 1e-3), sequential_env_steps_per_s=steps / (seq_ms * 1e-3),
                                  speedup=seq_ms / mixed_ms, gpu=name, power_limit=power)), flush=True)


def table(trl, args, name, power):
    M = args.table_envs
    for scene, pack, grid in (("dog/slopes_mixed", DOG, DOG_GRID), ("raptor/narrow_gaps", RAPTOR, RAPTOR_GRID)):
        slots = np.repeat(np.arange(len(grid)), M)
        sc = handle(trl, pack, len(grid) * M, grid, slots)
        for _ in range(int(round(args.seconds / DT))):
            sc.Update(DT)
        sc.Sync()
        dist, env = sc.GetDistLog()
        for q, s in enumerate(grid):
            st = sc.GetEvalStats(None, physics=q)
            on = np.flatnonzero(slots == q)
            print(json.dumps(dict(scene=scene, slot=q, setting=s, envs=M, seconds=args.seconds, episodes=st["episodes"],
                                  mean_dist=st["avg_dist"], no_fall_share=float(1.0 - np.isin(on, env).mean()), gpu=name,
                                  power_limit=power)), flush=True)
        sc.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--presim", type=float, default=2.0)
    ap.add_argument("--settings", default="1,2,4,8")
    ap.add_argument("--envs", default="512,4096", help="envs per setting (M)")
    ap.add_argument("--table", action="store_true", help="the behaviour tables instead of the throughput comparison")
    ap.add_argument("--table-envs", type=int, default=1024)
    ap.add_argument("--seconds", type=float, default=20.0)
    args = ap.parse_args()
    import deepterrainrl_b200 as trl
    name, power = card()
    (table if args.table else throughput)(trl, args, name, power)


if __name__ == "__main__":
    main()
