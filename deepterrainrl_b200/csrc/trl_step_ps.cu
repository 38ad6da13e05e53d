// deepterrainrl_b200 -- physics-slot build of the env-step kernels (trl_load_physics), terrain slots included; see trl_step.cu.
#define TRL_TERRAIN_SLOTS_VARIANT 1
#define TRL_PHYS_SLOTS_VARIANT 1
#include "trl_step.cu"
