// deepterrainrl_b200 -- body-slot build of the L1-bypassing env-step kernel (compile with -Xptxas -dlcm=cg); see trl_step.cu.
#define TRL_CG_VARIANT 1
#define TRL_TERRAIN_SLOTS_VARIANT 1
#define TRL_PHYS_SLOTS_VARIANT 1
#define TRL_BODY_SLOTS_VARIANT 1
#include "trl_step.cu"
