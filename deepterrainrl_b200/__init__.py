"""deepterrainrl_b200 -- H100-native batched rollout engine behind DeepTerrainRL's scenario API.

The compute path is hand-written CUDA (csrc/, built into lib/libterrainrl_b200.so and reached through the C ABI in
include/terrainrl_b200.h).  This package is the thin host-side mirror of the reference's scenario interface
(cScenarioPoliEval / cScenarioExpMACE method names) used by the tests and bench.py.  There is no CPU fallback:
importing works anywhere, creating a scenario without the built library or without a GPU raises.
"""
from .scenario import (BatchedScenario, ScenarioExpMACE, ScenarioPoliEval, build_library, library_path,  # noqa: F401
                       load_library, pack_from_args)

__all__ = ["BatchedScenario", "ScenarioExpMACE", "ScenarioPoliEval", "build_library", "library_path", "load_library", "pack_from_args"]
from .trainer import MACETrainer  # noqa: F401,E402
from .checkpoint import load_checkpoint  # noqa: F401,E402
