// deepterrainrl_b200 -- the splitmix64 finaliser, shared by the trainer's counter RNG (trl_train.cu) and the checkpoint digest
// (trl_checkpoint.cu), on the device and on the host
#pragma once
#include "trl_types.h"

namespace trl {

#if defined(__CUDACC__) && !defined(TRL_SIMT_EMU)
__host__ __device__ __forceinline__
#else
inline
#endif
unsigned long long mix64(unsigned long long z) {
    z += 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

}  // namespace trl
