"""Evaluation envs on the GPU: K training slots of M exploring envs each, evaluated while they train.

  (a) one exploration handle: K x (M exploring + E evaluating) envs, one trainer per slot (trl_set_env_eval);
  (b) the same training with no evaluation envs, plus what a user does without them: one evaluation handle of E envs per slot, its net
      refreshed from the slot's trainer every update (trl_trainer_get -> trl_set_weights).

Both arms run one update per call (train_run_slots(..., 1, ITERS)) so that (b) can refresh its nets between updates; each is
warmed up, then timed with a host clock around calls that end in a device synchronise.  The scene is dog / slopes_mixed with the
pack's policy in every slot.

    python tools/eval_envs_bench.py [--slots 1,4,8] [--envs 512,4096] [--eval 64,512] [--updates U] [--warmup W]

Prints one JSON line per (K, M, E): env-steps/s of the training and of the evaluation envs in both arms, and the card's name and power
limit."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from policy_slots_bench import card  # noqa: E402

DOG = os.path.join(ROOT, "assets", "dog_slopes_mixed.trlpack")
DT = 1.0 / 30.0
ITERS = 1
TRAINER = dict(replay_mem_size=50000, num_init_samples=1000)
STEPS_PER_UPDATE = 20


def sync(sc):
    sc.GetEvalStats(None)       # reads device memory after the handle's stream is idle


def net_of(tr):
    blobs = tr.blobs()
    return [x for k in blobs for x in blobs[k]], *[tr.get(v) for v in ("in_off", "in_scale", "out_off", "out_scale")]


def arm_a(trl, sched, K, M, E, updates, warmup):
    from deepterrainrl_b200.train import train_run_slots
    n = K * (M + E)
    sc = trl.ScenarioExpMACE(DOG, n, rng_seed=5)
    trs = [trl.MACETrainer(sc, slot=p, seed=10 + p, **TRAINER) for p in range(K)]
    slot = np.arange(n) // (M + E)
    if K > 1:
        sc.SetEnvPolicy(slot.astype(np.int32))
    sc.SetEnvEval((np.arange(n) % (M + E) >= M).astype(np.int32))
    sc.Reset()
    for _ in range(warmup):
        train_run_slots(trs, sched, 1, ITERS)
    sync(sc)
    t0 = time.perf_counter()
    for _ in range(updates):
        train_run_slots(trs, sched, 1, ITERS)
    sync(sc)
    t = time.perf_counter() - t0
    for o in trs + [sc]:
        o.close()
    return t


def arm_b(trl, sched, K, M, E, updates, warmup):
    from deepterrainrl_b200.train import train_run_slots
    n = K * M
    sc = trl.ScenarioExpMACE(DOG, n, rng_seed=5)
    trs = [trl.MACETrainer(sc, slot=p, seed=10 + p, **TRAINER) for p in range(K)]
    if K > 1:
        sc.SetEnvPolicy((np.arange(n) // M).astype(np.int32))
    evs = [trl.ScenarioPoliEval(DOG, E, rng_seed=7 + p) for p in range(K)]

    def one():
        train_run_slots(trs, sched, 1, ITERS)
        for p in range(K):
            evs[p].SetWeights(*net_of(trs[p]))
            evs[p].Update(DT)

    for _ in range(warmup):
        one()
    for o in evs + [sc]:
        sync(o)
    t0 = time.perf_counter()
    for _ in range(updates):
        one()
    for o in evs + [sc]:
        sync(o)
    t = time.perf_counter() - t0
    for o in trs + evs + [sc]:
        o.close()
    return t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--slots", default="1,4,8")
    ap.add_argument("--envs", default="512,4096")
    ap.add_argument("--eval", default="64,512")
    ap.add_argument("--updates", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    import deepterrainrl_b200 as trl
    from deepterrainrl_b200.train import TrainSchedule
    trl.load_library()
    sched = TrainSchedule(init_exp_rate=0.2, exp_rate=0.2, init_exp_temp=0.025, exp_temp=0.025, init_exp_base_rate=0.01, exp_base_rate=0.01)
    name, power = card()
    for K in [int(x) for x in args.slots.split(",")]:
        for M in [int(x) for x in args.envs.split(",")]:
            for E in [int(x) for x in args.eval.split(",")]:
                ta = arm_a(trl, sched, K, M, E, args.updates, args.warmup)
                tb = arm_b(trl, sched, K, M, E, args.updates, args.warmup)
                steps = args.updates * STEPS_PER_UPDATE
                print(json.dumps(dict(slots=K, train_envs=M, eval_envs=E, updates=args.updates,
                                      one_handle_train_steps_per_s=K * M * steps / ta, one_handle_eval_steps_per_s=K * E * steps / ta,
                                      separate_train_steps_per_s=K * M * steps / tb, separate_eval_steps_per_s=K * E * steps / tb,
                                      one_handle_s=ta, separate_s=tb, speedup=tb / ta, gpu=name, power_limit=power)), flush=True)


if __name__ == "__main__":
    main()
