"""Training slots on the GPU: K policies trained in ONE exploration handle (K x M envs, envs on slots in contiguous blocks, one MACE
trainer per slot, trl_train_run_slots) against the same K policies trained one after another in single-trainer handles of M envs each
(trl_train_run_timed).  dog / slopes_mixed, `--iters` trainer iterations per update (bench.py's config-4 default: 4); slot 0 starts
from the pack's model, slots 1.. from perturbed copies of it.  Every arm is pre-rolled until each of its trainers has left the init
stage (a small num_init_samples keeps that short), then `--steps` updates are timed: the slot handle with a host clock around
trl_train_run_slots + trl_sync, the single handles with trl_train_run_timed's device events, summed over the K handles.

    python tools/train_slots_bench.py [--steps 20] [--iters 4] [--ks 1,2,4,8] [--ms 512,4096] [--out FILE]

prints one JSON line per (K, M): env-steps/s and trainer iterations/s of both arms, the card's name and power limit.  Each trainer's
replay memory is replay_mem_size x (1 + 2 S + A) f32 (dog: 1 + 2 x 283 + 30 = 597 floats a row)."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from policy_slots_bench import PACK, perturbed_models  # noqa: E402

DT = 1.0 / 30.0
TRAINER = dict(replay_mem_size=100000, num_init_samples=2000)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else "unknown"


def slots_arm(trl, k, m, models, args, sched):
    from deepterrainrl_b200.train import train_run_slots
    n = k * m
    sc = trl.ScenarioExpMACE(PACK, n, rng_seed=1)
    trs = [trl.MACETrainer(sc, slot=p, model=models[p], seed=1 + p, **TRAINER) for p in range(k)]
    sc.SetEnvPolicy((np.arange(n) * k) // n)
    while min(t.counters()["stage"] for t in trs) == 0:
        train_run_slots(trs, sched, 20, args.iters)
    train_run_slots(trs, sched, 3, args.iters)       # warm-up: every captured graph of the timed window exists
    sc.Sync()
    t0 = time.perf_counter()
    train_run_slots(trs, sched, args.steps, args.iters)
    sc.Sync()
    s = time.perf_counter() - t0
    for t in trs:
        t.close()
    sc.close()
    return s


def single_arm(trl, k, m, models, args, sp):
    total = 0.0
    for p in range(k):
        sc = trl.ScenarioExpMACE(PACK, m, rng_seed=1)
        tr = trl.MACETrainer(sc, model=models[p], seed=1 + p, **TRAINER)
        L = tr.L
        st = C.c_int64(0)
        ms = C.c_double(0)

        def run(u):
            rc = L.trl_train_run_timed(tr.h, sp.ctypes.data_as(C.c_void_p), int(u), args.iters, 0, C.c_double(DT), 0, C.byref(st),
                                       C.byref(ms))
            if rc != 0:
                raise RuntimeError(L.trl_last_error().decode())
            return ms.value / 1e3
        while tr.counters()["stage"] == 0:
            run(20)
        run(3)
        total += run(args.steps)
        tr.close()
        sc.close()
    return total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--iters", type=int, default=4)
    ap.add_argument("--ks", default="1,2,4,8")
    ap.add_argument("--ms", default="512,4096")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import deepterrainrl_b200 as trl
    from deepterrainrl_b200.train import TrainSchedule
    sched = TrainSchedule()
    sp = np.array([sched.p[k] for k in TrainSchedule.KEYS], float)
    ks = [int(x) for x in args.ks.split(",")]
    d = tempfile.mkdtemp()
    files = perturbed_models(d, max(ks) - 1)
    models = [None] + [(f, os.path.splitext(f)[0] + "_scale.txt") for f in files]
    gpu = card()
    out = open(args.out, "a") if args.out else None
    for m in [int(x) for x in args.ms.split(",")]:
        for k in ks:
            s_slots = slots_arm(trl, k, m, models, args, sched)
            s_single = single_arm(trl, k, m, models, args, sp)
            env_steps = k * m * 20 * args.steps
            iters = k * args.iters * args.steps
            rec = dict(K=k, M=m, iters_per_update=args.iters, updates=args.steps, card=gpu,
                       slots_env_steps_per_s=env_steps / s_slots, single_env_steps_per_s=env_steps / s_single,
                       slots_trainer_iters_per_s=iters / s_slots, single_trainer_iters_per_s=iters / s_single,
                       speedup=s_single / s_slots)
            line = json.dumps(rec)
            print(line, flush=True)
            if out:
                out.write(line + "\n")
    if out:
        out.close()


if __name__ == "__main__":
    main()
