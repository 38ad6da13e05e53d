"""Policy slots on the GPU: P models evaluated in ONE handle (P x M envs, envs on slots in contiguous blocks) against the same P models
evaluated one after another in single-policy handles of M envs each.  dog / slopes_mixed; slot 0 is the pack's model, slots 1.. are
perturbed copies of it (same topology, different decisions).  Every arm: an untimed pre-roll to a steady state, warm-up updates, then
K updates device-timed on the engine's stream with an L2 flush between updates (trl_bench_updates, as bench.py times them).

    python tools/policy_slots_bench.py [--steps K] [--presim SECONDS] [--out FILE]

prints one JSON line per (P, M) with env-steps/s of both arms, the card's name and power limit."""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
PACK = os.path.join(ROOT, "assets", "dog_slopes_mixed.trlpack")
DT = 1.0 / 30.0
LAYERS = ["terr_conv0", "terr_conv1", "terr_conv2", "terr_ip0", "ip0", "val_ip0", "val_ip1",
          "a0_ip0", "a0_ip1", "a1_ip0", "a1_ip1", "a2_ip0", "a2_ip1"]


def card():
    import torch
    q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return torch.cuda.get_device_name(0), (q.stdout.strip() if q.returncode == 0 else "unknown")


def perturbed_models(d, count, rel=0.05):
    from pack_scene import read_pack
    from deepterrainrl_b200.model_io import write_model_native
    rec = read_pack(PACK)
    vec = [np.asarray(rec[k], float) for k in ("net_in_offset", "net_in_scale", "net_out_offset", "net_out_scale")]
    paths = []
    for s in range(1, count + 1):
        rng = np.random.default_rng(s)
        blobs = {}
        for n in LAYERS:
            b = np.asarray(rec["net_" + n + "_b"], float).ravel()
            w = np.asarray(rec["net_" + n + "_w"], float).reshape(b.size, -1)
            blobs[n] = (w * (1 + rel * rng.standard_normal(w.shape)), b * (1 + rel * rng.standard_normal(b.shape)))
        p = os.path.join(d, "dog_p%d.h5" % s)
        write_model_native(p, blobs, *vec)
        paths.append(p)
    return paths


def timed(sc, args):
    sc.BenchUpdates(int(round(args.presim / DT)), DT, flush_l2=False)
    sc.BenchUpdates(args.warmup, DT, flush_l2=True)
    return sc.BenchUpdates(args.steps, DT, flush_l2=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--presim", type=float, default=2.0)
    ap.add_argument("--slots", default="1,2,4,8")
    ap.add_argument("--envs", default="512,4096", help="envs per model (M)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import deepterrainrl_b200 as trl
    name, power = card()
    d = tempfile.mkdtemp()
    P_list = [int(x) for x in args.slots.split(",")]
    models = [None] + perturbed_models(d, max(P_list) - 1)
    lines = []
    for M in [int(x) for x in args.envs.split(",")]:
        for P in P_list:
            steps = args.steps * 20 * P * M
            sc = trl.ScenarioPoliEval(PACK, P * M, terrain_seeds=np.arange(1, P * M + 1, dtype=np.uint64))
            for p in range(1, P):
                sc.LoadPolicy(p, models[p])
            if P > 1:
                sc.SetEnvPolicy(np.repeat(np.arange(P), M))
            mixed_ms = timed(sc, args)
            sc.close()
            seq_ms = 0.0
            for p in range(P):
                sc = trl.ScenarioPoliEval(PACK, M, terrain_seeds=np.arange(1 + p * M, 1 + (p + 1) * M, dtype=np.uint64))
                if models[p] is not None:
                    sc.LoadModel(models[p])
                seq_ms += timed(sc, args)
                sc.close()
            line = dict(slots=P, envs_per_slot=M, steps=args.steps, mixed_ms=round(mixed_ms, 3), sequential_ms=round(seq_ms, 3),
                        mixed_env_steps_per_s=steps / (mixed_ms * 1e-3), sequential_env_steps_per_s=steps / (seq_ms * 1e-3),
                        speedup=seq_ms / mixed_ms, gpu=name, power_limit=power)
            print(json.dumps(line), flush=True)
            lines.append(line)
    if args.out:
        with open(args.out, "w") as f:
            for line in lines:
                f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
