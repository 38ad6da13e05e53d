"""Training slots with and without the tuple exchange: env-steps/s and applied trainer iterations/s of K slot trainers on one handle.

dog / slopes_mixed, 4 trainer iterations per update, K in {1, 2, 4, 8} policies, M in {512, 4096} envs per policy (round robin), three
runs per (K, M):
  local   trl_train_run_slots_sched without a communicator (the one-GPU loop);
  sync    trl_train_run_slots_comm: one all-gather per update, each trainer's slot-filtered intake + iterations on its own stream;
  async   the same with every trainer asynchronous (intake + iterations beside the next update, a policy snapshot per slot).
Timed with a host clock around `--updates` updates that end in a device synchronise, after `--warmup` updates of the same shape
that also take every trainer past its init stage (num_init_samples 256), so the timed window applies the requested iterations.

One GPU (a world-1 NCCL communicator):   python tools/comm_slots_bench.py
N GPUs of one node (envs sharded by rank; local runs are skipped):
    python -m torch.distributed.run --nproc_per_node N tools/comm_slots_bench.py
Each rank prints one JSON line per run; rank 0's rates are per rank (multiply by N for the node)."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ks", default="1,2,4,8")
    ap.add_argument("--ms", default="512,4096")
    ap.add_argument("--modes", default="local,sync,async")
    ap.add_argument("--updates", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--iters", type=int, default=4)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    device = int(os.environ.get("LOCAL_RANK", "0"))
    import torch
    torch.cuda.set_device(device)
    group = None
    if world > 1:
        import torch.distributed as dist
        dist.init_process_group("nccl")
        group = dist.group.WORLD
    import deepterrainrl_b200 as trl
    from deepterrainrl_b200 import parallel
    from deepterrainrl_b200.train import TrainSchedule, train_run_slots
    pack = os.path.join(ROOT, "assets", "dog_slopes_mixed.trlpack")
    sched = TrainSchedule(init_exp_rate=0.5, exp_rate=0.2, init_exp_temp=5, exp_temp=0.025, init_exp_base_rate=0.2,
                          exp_base_rate=0.002, trainer_num_anneal_iters=1000, exp_base_anneal_iters=1000)
    # a small init stage: the warm-up leaves it behind, so the timed window trains at every update (steady state)
    kw = dict(replay_mem_size=200000, num_init_samples=256, freeze_target_iters=500)
    name = torch.cuda.get_device_name(device)
    lines = []
    for K in [int(x) for x in a.ks.split(",")]:
        for M in [int(x) for x in a.ms.split(",")]:
            for mode in a.modes.split(","):
                if mode == "local" and world > 1:
                    continue
                n = K * M
                sc = trl.ScenarioExpMACE(pack, n, device=device, terrain_seeds=parallel.shard_seeds(rank, n), rng_seed=7 + rank)
                trs = [trl.MACETrainer(sc, slot=p, seed=3 + p, **kw) for p in range(K)]
                sc.SetEnvPolicy(np.arange(n) % K)
                comm = None
                if mode != "local":
                    uid = None
                    if world == 1:
                        import ctypes as C
                        buf = (C.c_ubyte * 128)()
                        if sc.L.trl_comm_unique_id(buf) != 0:
                            raise RuntimeError(sc.L.trl_last_error().decode())
                        uid = bytes(buf)
                    comm = parallel.Comm(sc, rank, world, backend="nccl", unique_id=uid, group=group)
                    if mode == "async":
                        for t in trs:
                            t.SetAsync(True)
                run = lambda u: train_run_slots(trs, [sched] * K, u, a.iters, comm=comm, block_rows=n)  # noqa: E731
                run(a.warmup)
                sc.Sync()
                it0 = sum(t.counters()["iter"] for t in trs)
                s0 = sc.GetNumEnvSteps()
                t0 = time.perf_counter()
                run(a.updates)
                sc.Sync()
                dt = time.perf_counter() - t0
                its = sum(t.counters()["iter"] for t in trs) - it0
                steps = sc.GetNumEnvSteps() - s0
                rec = dict(mode=mode, K=K, envs_per_policy=M, envs=n, world=world, rank=rank, updates=a.updates, iters_per_update=a.iters,
                           env_steps_per_s=steps / dt, trainer_iters_per_s=its / dt, applied_iters=its, seconds=dt, gpu=name)
                if comm is not None:
                    rec["replica_spread"] = max(comm.ReplicaSpread(t) for t in trs)
                    comm.close()
                print(json.dumps(rec), flush=True)
                lines.append(rec)
                for t in trs:
                    t.close()
                sc.close()
    if a.out and rank == 0:
        with open(a.out, "w") as f:
            for r in lines:
                f.write(json.dumps(r) + "\n")
    if world > 1:
        import torch.distributed as dist
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
