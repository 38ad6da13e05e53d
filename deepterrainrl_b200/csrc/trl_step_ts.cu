// deepterrainrl_b200 -- terrain-slot build of the env-step kernels (trl_load_terrain); see trl_step.cu.
#define TRL_TERRAIN_SLOTS_VARIANT 1
#include "trl_step.cu"
