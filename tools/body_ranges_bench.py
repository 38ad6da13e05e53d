"""Ranged slots on the GPU: what drawing bodies and physics at episode resets costs.  4096 dog envs on dog_slopes_mixed (the pack's
policy) in these configurations, alternated in one process:

  body1       the body-slot build with one fixed body: an unmodified copy of dog.txt in body slot 1, every env on slot 0;
  rbody       every env on a ranged body (masses x0.8-1.25, Kp / Kd x0.8-1.2, TorqueLim x0.7-1.0);
  rphys       every env on a ranged physics slot (mu 0.5-1.1 x the scene's 0.81, kn +-20 %);
  rboth       both;
  body1_fall  body1 with every env tipped over before every timed update, so that every env resets inside every update;
  rboth_fall  rboth likewise: every env draws a body and physics inside every update.

Every handle gets an untimed pre-roll to a steady state; then, round by round, each configuration runs warm-up updates and K updates
device-timed on the engine's stream with an L2 flush between updates (trl_bench_updates, as bench.py times them).  The *_fall arms
time one update at a time, each after the host has tipped every env over (untimed).  Prints one JSON line per configuration with the
median env-steps/s over the rounds and the card's name and power limit.

    python tools/body_ranges_bench.py [--steps K] [--rounds R] [--envs N] [--presim SECONDS]"""
import argparse
import json
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from policy_slots_bench import card  # noqa: E402

DOG = os.path.join(ROOT, "assets", "dog_slopes_mixed.trlpack")
REF = os.path.join(ROOT, "tests", "golden", "reference")
DT = 1.0 / 30.0
DEFAULT = np.array([2.0e5, 2.0e3, 0.81, 0.01, 0.00025, 2.0e4, 20.0])
PHYS_LO = DEFAULT * np.array([0.8, 1.0, 0.5 / 0.81, 1.0, 1.0, 1.0, 1.0])
PHYS_HI = DEFAULT * np.array([1.2, 1.0, 1.1 / 0.81, 1.0, 1.0, 1.0, 1.0])
RANGES = {"Mass": (0.8, 1.25), "Kp": (0.8, 1.2), "Kd": (0.8, 1.2), "TorqueLim": (0.7, 1.0)}


def body_files(dst):
    """dog.txt and the lo / hi ends of its ranged body under dst, controller files by absolute path (a pack handle has no data root)"""
    with open(os.path.join(REF, "data", "characters", "dog.txt")) as f:
        base = json.load(f)
    base["Controllers"]["Files"] = [os.path.join(REF, p) for p in base["Controllers"]["Files"]]
    out = []
    for end in (None, 0, 1):
        c = json.loads(json.dumps(base))
        if end is not None:
            for name, ab in RANGES.items():
                for x in (c["BodyDefs"] if name == "Mass" else c["PDControllers"]):
                    x[name] = x.get(name, 0.0) * ab[end]
        path = os.path.join(dst, "dog_%s.txt" % ("copy" if end is None else ("lo", "hi")[end]))
        with open(path, "w") as f:
            json.dump(c, f)
        out.append(path)
    return out


def handles(trl, n, files):
    seeds = np.arange(1, n + 1, dtype=np.uint64)
    out = {}
    for k in ("body1", "rbody", "rphys", "rboth", "body1_fall", "rboth_fall"):
        sc = trl.ScenarioPoliEval(DOG, n, terrain_seeds=seeds)
        sc.LoadBody(1, files[0])
        if k in ("rbody", "rboth", "rboth_fall"):
            sc.LoadBodyRange(2, files[1], files[2])
            sc.SetEnvBody(np.full(n, 2, np.int32))
        if k in ("rphys", "rboth", "rboth_fall"):
            sc.LoadPhysicsRange(1, PHYS_LO, PHYS_HI)
            sc.SetEnvPhysics(np.ones(n, np.int32))
        sc.SetRandSeed(seeds)
        out[k] = sc
    return out


def tip_all(sc):
    """every env past the fall angle: it falls and resets inside the next update"""
    q, _ = sc.GetStateAll()
    for e in range(sc.num_envs):
        qe = q[:, e].copy()
        qe[2] = 3.0
        sc.SetState(e, q=qe)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--presim", type=float, default=2.0)
    args = ap.parse_args()
    import deepterrainrl_b200 as trl
    name, power = card()
    with tempfile.TemporaryDirectory() as d:
        hs = handles(trl, args.envs, body_files(d))
        for sc in hs.values():
            sc.BenchUpdates(int(round(args.presim / DT)), DT, flush_l2=False)
        ms = {k: [] for k in hs}
        for _ in range(args.rounds):
            for k, sc in hs.items():
                sc.BenchUpdates(args.warmup, DT, flush_l2=True)
                if k.endswith("_fall"):
                    t = 0.0
                    for _ in range(args.steps):
                        tip_all(sc)
                        t += sc.BenchUpdates(1, DT, flush_l2=True)
                    ms[k].append(t)
                else:
                    ms[k].append(sc.BenchUpdates(args.steps, DT, flush_l2=True))
        steps = args.steps * 20 * args.envs
        for k, v in ms.items():
            med = float(np.median(v))
            print(json.dumps(dict(config=k, envs=args.envs, steps=args.steps, rounds=args.rounds, median_ms=round(med, 3),
                                  env_steps_per_s=steps / (med * 1e-3), spread_ms=[round(min(v), 3), round(max(v), 3)], gpu=name,
                                  power_limit=power)), flush=True)
        for sc in hs.values():
            sc.close()


if __name__ == "__main__":
    main()
