// deepterrainrl_b200 -- body-slot build of the env-step kernels (trl_load_body), terrain and physics slots included; see trl_step.cu.
#define TRL_TERRAIN_SLOTS_VARIANT 1
#define TRL_PHYS_SLOTS_VARIANT 1
#define TRL_BODY_SLOTS_VARIANT 1
#include "trl_step.cu"
