"""Terrain slots on the GPU: T terrains evaluated in ONE handle (T x M envs, envs on slots in contiguous blocks) against the same T
terrains evaluated one after another in single-terrain handles of M envs each.  The scene is dog / slopes_mixed with the pack's policy;
slot 0 is the pack's terrain (slopes_mixed), slots 1.. are the committed terrain files mixed, narrow_gaps, tight_gaps, flat,
cliffs_rugged.  A single-terrain handle of terrain t > 0 is a pack handle with every env on slot t, which computes exactly what a
handle created with that file as -terrain_file does.  Every arm: an untimed pre-roll to a steady state, warm-up updates, then K updates
device-timed on the engine's stream with an L2 flush between updates (trl_bench_updates, as bench.py times them).

    python tools/terrain_slots_bench.py [--steps K] [--presim SECONDS] [--terrains 1,2,4,6] [--envs 512,4096]
    python tools/terrain_slots_bench.py --table [--table-envs M] [--seconds S]

The first form prints one JSON line per (T, M) with env-steps/s of both arms.  --table runs the pack's policy on all six terrains in one
handle for S seconds of simulated time and prints, per terrain, episodes, mean distance and the share of envs whose run had no logged
fall.  Both print the card's name and power limit."""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from policy_slots_bench import card  # noqa: E402

PACK = os.path.join(ROOT, "assets", "dog_slopes_mixed.trlpack")
TERRAIN_DIR = os.path.join(ROOT, "tests", "golden", "reference", "data", "terrain")
TERRAINS = ["slopes_mixed", "mixed", "narrow_gaps", "tight_gaps", "flat", "cliffs_rugged"]
DT = 1.0 / 30.0


def handle(trl, n, terrains, slots, seed0=1):
    """a pack handle with terrains[1:] in slots 1.., envs on `slots` from their first episode on"""
    sc = trl.ScenarioPoliEval(PACK, n, terrain_seeds=np.arange(seed0, seed0 + n, dtype=np.uint64))
    for t, name in enumerate(terrains[1:], 1):
        sc.LoadTerrain(t, os.path.join(TERRAIN_DIR, name + ".txt"))
    if len(terrains) > 1:
        sc.SetEnvTerrain(slots)
        sc.SetRandSeed(np.arange(seed0, seed0 + n, dtype=np.uint64))
    return sc


def timed(sc, args):
    sc.BenchUpdates(int(round(args.presim / DT)), DT, flush_l2=False)
    sc.BenchUpdates(args.warmup, DT, flush_l2=True)
    return sc.BenchUpdates(args.steps, DT, flush_l2=True)


def throughput(trl, args, name, power):
    for M in [int(x) for x in args.envs.split(",")]:
        for T in [int(x) for x in args.terrains.split(",")]:
            steps = args.steps * 20 * T * M
            sc = handle(trl, T * M, TERRAINS[:T], np.repeat(np.arange(T), M))
            mixed_ms = timed(sc, args)
            sc.close()
            seq_ms = 0.0
            for t in range(T):
                terr = [TERRAINS[0]] if t == 0 else [TERRAINS[0], TERRAINS[t]]
                sc = handle(trl, M, terr, np.full(M, 1 if t else 0), seed0=1 + t * M)
                seq_ms += timed(sc, args)
                sc.close()
            print(json.dumps(dict(terrains=T, envs_per_terrain=M, steps=args.steps, mixed_ms=round(mixed_ms, 3), sequential_ms=round(seq_ms, 3),
                                  mixed_env_steps_per_s=steps / (mixed_ms * 1e-3), sequential_env_steps_per_s=steps / (seq_ms * 1e-3),
                                  speedup=seq_ms / mixed_ms, gpu=name, power_limit=power)), flush=True)


def table(trl, args, name, power):
    M, T = args.table_envs, len(TERRAINS)
    slots = np.repeat(np.arange(T), M)
    sc = handle(trl, T * M, TERRAINS, slots)
    for _ in range(int(round(args.seconds / DT))):
        sc.Update(DT)
    sc.Sync()
    dist, env = sc.GetDistLog()
    for t, terr in enumerate(TERRAINS):
        st = sc.GetEvalStats(None, terrain=t)
        on = np.flatnonzero(slots == t)
        no_fall = 1.0 - np.isin(on, env).mean()
        print(json.dumps(dict(terrain=terr, envs=M, seconds=args.seconds, episodes=st["episodes"], mean_dist=st["avg_dist"],
                              no_fall_share=float(no_fall), gpu=name, power_limit=power)), flush=True)
    sc.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--presim", type=float, default=2.0)
    ap.add_argument("--terrains", default="1,2,4,6")
    ap.add_argument("--envs", default="512,4096", help="envs per terrain (M)")
    ap.add_argument("--table", action="store_true", help="the behaviour table instead of the throughput comparison")
    ap.add_argument("--table-envs", type=int, default=1024)
    ap.add_argument("--seconds", type=float, default=20.0)
    args = ap.parse_args()
    import deepterrainrl_b200 as trl
    name, power = card()
    (table if args.table else throughput)(trl, args, name, power)


if __name__ == "__main__":
    main()
