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

// The draws of ranged body and physics slots (trl_types.h: kBodyDrawTag).  Draw number `draw` of one kind (`tag`) of env `env` has
// the key mix64(mix64(mix64(rng_seed ^ tag) + env) + draw); its i-th number is the top 53 bits of mix64(key + i), scaled into [0, 1)
// (exact: a 53-bit integer times 2^-53).  The keys are their own, so a draw never moves the env's counter RNG.
#if defined(__CUDACC__) && !defined(TRL_SIMT_EMU)
__host__ __device__ __forceinline__
#else
inline
#endif
unsigned long long draw_key(unsigned long long rng_seed, unsigned long long tag, int env, long long draw) {
    return mix64(mix64(mix64(rng_seed ^ tag) + (unsigned long long)env) + (unsigned long long)draw);
}
#if defined(__CUDACC__) && !defined(TRL_SIMT_EMU)
__host__ __device__ __forceinline__
#else
inline
#endif
double draw_unit(unsigned long long key, int i) {
    return (double)(mix64(key + (unsigned long long)i) >> 11) * 0x1.0p-53;
}

}  // namespace trl
