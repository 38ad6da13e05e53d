"""Body slots on the GPU: what the body-slot build of the env-step kernels costs.  4096 dog envs on dog_slopes_mixed (the pack's policy)
in four configurations, alternated in one process:

  plain      a handle without slots (the plain step kernels);
  phys1      the physics-slot build: one extra physics slot loaded, every env on slot 0;
  body1      the body-slot build with one body: an unmodified copy of dog.txt in body slot 1, every env on slot 0;
  body8      the body-slot build with 8 bodies (dog.txt and 7 variants of its masses, leg lengths, gains and torque limits), envs round
             robin over the slots.

Every handle gets an untimed pre-roll to a steady state; then, round by round, each configuration runs warm-up updates and K updates
device-timed on the engine's stream with an L2 flush between updates (trl_bench_updates, as bench.py times them).  Prints one JSON line
per configuration with the median env-steps/s over the rounds and the card's name and power limit.

    python tools/body_slots_bench.py [--steps K] [--rounds R] [--envs N] [--presim SECONDS]"""
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
DEFAULT = [2.0e5, 2.0e3, 0.81, 0.01, 0.00025, 2.0e4, 20.0]
# (torso mass, leg length, Kp, torque limit) factors of the 8 bodies; body 0 is dog.txt itself
SCALES = [(1.0, 1.0, 1.0, 1.0), (1.3, 1.0, 1.0, 1.0), (0.8, 1.0, 1.0, 1.0), (1.0, 1.1, 1.0, 1.0), (1.0, 0.9, 1.0, 1.0),
          (1.0, 1.0, 0.8, 0.7), (1.0, 1.0, 1.2, 1.0), (1.2, 1.05, 0.9, 0.9)]


def body_files(dst):
    """dog.txt and its variants under dst, with the controller files named by absolute path (a pack handle has no data root)"""
    with open(os.path.join(REF, "data", "characters", "dog.txt")) as f:
        base = json.load(f)
    base["Controllers"]["Files"] = [os.path.join(REF, p) for p in base["Controllers"]["Files"]]
    out = []
    for k, (mass, leg, kp, tlim) in enumerate(SCALES):
        c = json.loads(json.dumps(base))
        B, J, P = c["BodyDefs"], c["Skeleton"]["Joints"], c["PDControllers"]
        B[5]["Mass"] *= mass                                    # torso
        for j in (13, 14, 17, 18):                              # thighs and shins with the joints below them
            for key in ("AttachX", "AttachY", "Param1"):
                B[j][key] *= leg
        for jt in J:
            if jt["Parent"] in (13, 14, 17, 18):
                jt["AttachY"] *= leg
        for p in P:
            p["Kp"] *= kp
            p["TorqueLim"] *= tlim
        path = os.path.join(dst, "dog_body%d.txt" % k)
        with open(path, "w") as f:
            json.dump(c, f)
        out.append(path)
    return out


def handles(trl, n, files):
    seeds = np.arange(1, n + 1, dtype=np.uint64)
    plain = trl.ScenarioPoliEval(DOG, n, terrain_seeds=seeds)
    phys1 = trl.ScenarioPoliEval(DOG, n, terrain_seeds=seeds)
    phys1.LoadPhysics(1, DEFAULT)
    body1 = trl.ScenarioPoliEval(DOG, n, terrain_seeds=seeds)
    body1.LoadBody(1, files[0])
    body8 = trl.ScenarioPoliEval(DOG, n, terrain_seeds=seeds)
    for b, f in enumerate(files[1:], 1):
        body8.LoadBody(b, f)
    body8.SetEnvBody(np.arange(n) % len(files))
    body8.SetRandSeed(seeds)
    return {"plain": plain, "phys1": phys1, "body1": body1, "body8": body8}


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
