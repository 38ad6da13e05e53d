"""An exploration sweep on the GPU: K policies, each under its own exploration schedule, trained in ONE exploration handle (K x M envs,
envs on slots in contiguous blocks, one MACE trainer per slot, trl_train_run_slots_sched) against the same K policies trained one
after another in single-trainer handles of M envs each (trl_train_run with the same pacing).  dog / slopes_mixed; slot 0 starts from
the pack's model, slots 1.. from perturbed copies of it; schedule p spreads the reference's exp_rate / exp_temp / exp_base_rate
(args/opt_args_train_mace.txt) over a factor of 4 across the K policies.

Two pacings: `--iters` trainer iterations per update in lock-step, and tuple pacing (iters_per_update = 0: one iteration per 32 fresh
tuples of the trainer's slot, the reference's -tuple_buffer_size).  Paced runs read every trainer's counters back twice per update
(one round trip each for all K trainers in the slot handle; two per handle and update for the single handles).

Every arm is pre-rolled until each of its trainers has left the init stage, warmed up for 3 updates in the measured pacing, then
`--steps` updates are timed with a host clock around the run call and a final synchronisation.  Trainer iterations are the ones
requested: K x iters x steps in lock-step, and the fresh tuples of every trainer over the timed window / 32 when paced (exact up to
the carries: less than one iteration per trainer).  `*_steps_applied_per_s` is the growth of the trainers' iteration counters, which
count only the iterations that found a critic minibatch and applied a step.

    python tools/train_sweep_bench.py [--steps 20] [--iters 4] [--ks 1,2,4,8] [--ms 512,4096] [--out FILE]

prints one JSON line per (pacing, K, M): env-steps/s and trainer iterations/s of both arms, the card's name and power limit."""
import argparse
import ctypes as C
import json
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from policy_slots_bench import PACK, perturbed_models  # noqa: E402
from train_slots_bench import TRAINER, card  # noqa: E402

DT = 1.0 / 30.0
BASE = dict(init_exp_rate=0.9, exp_rate=0.2, init_exp_temp=20.0, exp_temp=0.025, init_exp_base_rate=0.9, exp_base_rate=0.002,
            trainer_num_anneal_iters=50000, exp_base_anneal_iters=50000, trainer_curriculum_iters=0)


def sweep(k):
    from deepterrainrl_b200.train import TrainSchedule
    out = []
    for p in range(k):
        f = 0.5 * 4.0 ** (p / max(1, k - 1))          # 0.5 .. 2 x the reference's final settings
        out.append(TrainSchedule(**dict(BASE, exp_rate=BASE["exp_rate"] * f, exp_temp=BASE["exp_temp"] * f,
                                        exp_base_rate=BASE["exp_base_rate"] * f)))
    return out


def progress(trs):
    """(steps applied, tuples taken) summed over the trainers"""
    cs = [t.counters() for t in trs]
    return np.array([sum(c["iter"] for c in cs), sum(c["total"] for c in cs)])


def requested(delta, k, ipu, args):
    return k * ipu * args.steps if ipu else delta[1] // 32


def slots_arm(trl, k, m, models, ipu, args):
    from deepterrainrl_b200.train import train_run_slots
    n = k * m
    scheds = sweep(k)
    sc = trl.ScenarioExpMACE(PACK, n, rng_seed=1)
    trs = [trl.MACETrainer(sc, slot=p, model=models[p], seed=1 + p, **TRAINER) for p in range(k)]
    sc.SetEnvPolicy((np.arange(n) * k) // n)
    while min(t.counters()["stage"] for t in trs) == 0:
        train_run_slots(trs, scheds, 20, args.iters)
    train_run_slots(trs, scheds, 3, ipu)      # warm-up: every captured graph of the timed window exists
    sc.Sync()
    p0 = progress(trs)
    t0 = time.perf_counter()
    train_run_slots(trs, scheds, args.steps, ipu)
    sc.Sync()
    s = time.perf_counter() - t0
    d1 = progress(trs) - p0
    delta = np.array([d1[0], requested(d1, k, ipu, args)])
    for t in trs:
        t.close()
    sc.close()
    return s, delta


def single_arm(trl, k, m, models, ipu, args):
    from deepterrainrl_b200.train import TrainSchedule
    total, delta = 0.0, np.zeros(2, np.int64)
    for p, sched in enumerate(sweep(k)):
        sp = np.array([sched.p[key] for key in TrainSchedule.KEYS], float)
        sc = trl.ScenarioExpMACE(PACK, m, rng_seed=1)
        tr = trl.MACETrainer(sc, model=models[p], seed=1 + p, **TRAINER)
        L = tr.L

        def run(u, i):
            if L.trl_train_run(tr.h, sp.ctypes.data_as(C.c_void_p), int(u), int(i), 32, C.c_double(DT)) != 0:
                raise RuntimeError(L.trl_last_error().decode())
        while tr.counters()["stage"] == 0:
            run(20, args.iters)
        run(3, ipu)
        sc.Sync()
        p0 = progress([tr])
        t0 = time.perf_counter()
        run(args.steps, ipu)
        sc.Sync()
        total += time.perf_counter() - t0
        d1 = progress([tr]) - p0
        delta += np.array([d1[0], requested(d1, 1, ipu, args)])
        tr.close()
        sc.close()
    return total, delta


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--iters", type=int, default=4)
    ap.add_argument("--ks", default="1,2,4,8")
    ap.add_argument("--ms", default="512,4096")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import deepterrainrl_b200 as trl
    ks = [int(x) for x in args.ks.split(",")]
    d = tempfile.mkdtemp()
    files = perturbed_models(d, max(ks) - 1)
    models = [None] + [(f, os.path.splitext(f)[0] + "_scale.txt") for f in files]
    gpu = card()
    out = open(args.out, "a") if args.out else None
    for pacing, ipu in (("tuples", None), ("fixed", args.iters)):
        for m in [int(x) for x in args.ms.split(",")]:
            for k in ks:
                s_slots, d_slots = slots_arm(trl, k, m, models, ipu, args)
                s_single, d_single = single_arm(trl, k, m, models, 0 if ipu is None else ipu, args)
                it_slots, it_single = int(d_slots[1]), int(d_single[1])
                env_steps = k * m * 20 * args.steps
                rec = dict(pacing=pacing, K=k, M=m, iters_per_update=ipu or 0, updates=args.steps, card=gpu,
                           slots_env_steps_per_s=env_steps / s_slots, single_env_steps_per_s=env_steps / s_single,
                           slots_trainer_iters_per_s=it_slots / s_slots, single_trainer_iters_per_s=it_single / s_single,
                           slots_steps_applied_per_s=int(d_slots[0]) / s_slots, single_steps_applied_per_s=int(d_single[0]) / s_single,
                           speedup=s_single / s_slots)
                line = json.dumps(rec)
                print(line, flush=True)
                if out:
                    out.write(line + "\n")
    if out:
        out.close()


if __name__ == "__main__":
    main()
