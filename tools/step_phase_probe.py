"""Per-phase cycles of the env-step kernel in the bench configuration (dog / slopes_mixed, 4096 envs, 4 s pre-roll).

Needs the measurement build of the step kernel: run as `TRL_VARIANT=phase_clocks python tools/step_phase_probe.py` (the variant is
compiled on first use).  Every warp's lane 0 sums clock64() deltas per phase (trl_debug_step_phases); the table is cycles per
env-step of one warp, i.e. the latency one environment sees, including the issue slots its neighbours on the same scheduler take."""
import argparse
import ctypes as C
import os
import sys

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
import deepterrainrl_b200 as trl  # noqa: E402
from deepterrainrl_b200 import scenario  # noqa: E402

NAMES = ["state load / store", "controller RNEA", "mass-matrix solve", "rest of controller", "kinematics", "contacts",
         "inward pass", "base + outward pass", "terrain / FSM / policy state"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scene", default="dog_slopes_mixed")
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--presim", type=float, default=4.0)
    ap.add_argument("--updates", type=int, default=30)
    args = ap.parse_args()
    if os.environ.get("TRL_VARIANT") != "phase_clocks":
        sys.exit("run with TRL_VARIANT=phase_clocks (the product build has no phase clocks)")
    scenario.build_library()
    pack = os.path.join(ROOT, "assets", args.scene + ".trlpack")
    n = args.envs
    sc = trl.ScenarioPoliEval(pack, n, terrain_seeds=np.arange(1, n + 1, dtype=np.uint64))
    sc.BenchUpdates(int(round(args.presim * 30)), 1.0 / 30.0, flush_l2=False)
    sc.L.trl_debug_step_phases.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int]
    out = np.zeros(10, np.uint64)
    ptr = out.ctypes.data_as(C.c_void_p)
    assert sc.L.trl_debug_step_phases(sc.h, ptr, 10, 1) == 0, sc.L.trl_last_error().decode()
    sc.BenchUpdates(args.updates, 1.0 / 30.0, flush_l2=False)
    assert sc.L.trl_debug_step_phases(sc.h, ptr, 10, 0) == 0, sc.L.trl_last_error().decode()
    steps = int(out[9])
    cyc = out[:9].astype(np.float64) / max(steps, 1)
    print(f"{args.scene}, {n} envs, {args.updates} updates after {args.presim} s pre-roll: {steps} env-steps counted")
    print(f"{'phase':32s} {'cycles / env-step':>18s} {'share':>7s}")
    for name, c in zip(NAMES, cyc):
        print(f"{name:32s} {c:18.0f} {100 * c / cyc.sum():6.1f}%")
    print(f"{'total':32s} {cyc.sum():18.0f}")
    sc.close()


if __name__ == "__main__":
    main()
