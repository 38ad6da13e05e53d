"""Save and restore times of checkpoints (trl_checkpoint_save / trl_create_from_checkpoint) at the sizes of a real run, and the file
sizes computed from the shapes.  Two cases on the dog (4096 envs, dog_slopes_mixed): one trainer with a full 500,000-row replay
memory (the shipped trainer_replay_mem_size), and 8 training slots whose trainers hold --slot-rows rows each.  The replay rows are
handed in through trl_trainer_add_tuples (random finite rows; a checkpoint's cost does not depend on their values).  Prints one JSON
line; the files go to a temporary directory and are removed.

    python tools/checkpoint_bench.py [--rows 500000] [--slot-rows 62500]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def fill(tr, rows, rng):
    """`rows` replay rows through the host hand-over, in blocks"""
    block = 8192
    for b in range(0, rows, block):
        k = min(block, rows - b)
        r = rng.standard_normal((k, tr.W))
        r[:, 1 + tr.S] = rng.integers(0, 3, k)
        tr.AddTuples(r, np.where(rng.uniform(size=k) < 0.4, 4, 0).astype(np.uint32))


def case(trl, pack, n, slots, rows, tmp):
    from deepterrainrl_b200.checkpoint import sections
    rng = np.random.default_rng(0)
    kw = dict(replay_mem_size=500000, num_init_samples=50000)
    sc = trl.ScenarioExpMACE(pack, n, rng_seed=1)
    trs = [trl.MACETrainer(sc, slot=p, seed=p + 1, **kw) for p in range(slots)]
    if slots > 1:
        sc.SetEnvPolicy(np.arange(n) % slots)
    for tr in trs:
        fill(tr, rows, rng)
    for _ in range(3):
        sc.Update(1.0 / 30.0)
    sc.Sync()
    path = os.path.join(tmp, "bench.ckpt")
    t0 = time.perf_counter()
    sc.SaveCheckpoint(path)
    t_save = time.perf_counter() - t0
    size = os.path.getsize(path)
    secs = sections(path)
    rows_bytes = sum(s[4] for s in secs if s[0].endswith(".mem"))
    for tr in trs:
        tr.close()
    sc.close()
    t0 = time.perf_counter()
    sc2, trs2, _ = trl.load_checkpoint(path)
    sc2.Sync()
    t_load = time.perf_counter() - t0
    for tr in trs2.values():
        tr.close()
    sc2.close()
    os.remove(path)
    return dict(envs=n, trainers=slots, rows_per_trainer=rows, file_bytes=size, replay_row_bytes=rows_bytes, sections=len(secs),
                save_s=round(t_save, 3), restore_s=round(t_load, 3))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=500000)
    ap.add_argument("--slot-rows", type=int, default=62500)
    ap.add_argument("--envs", type=int, default=4096)
    a = ap.parse_args()
    import deepterrainrl_b200 as trl
    pack = os.path.join(ROOT, "assets", "dog_slopes_mixed.trlpack")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    with tempfile.TemporaryDirectory() as tmp:
        out = dict(gpu=gpu, one_trainer=case(trl, pack, a.envs, 1, a.rows, tmp), eight_slots=case(trl, pack, a.envs, 8, a.slot_rows, tmp))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
