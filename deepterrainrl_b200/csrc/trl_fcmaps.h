// deepterrainrl_b200 -- what the host hands the batched decision kernel (trl_decide2.cuh) besides the buffers: the two TMA
// descriptors (CUDA build) and the plain pointers they describe (the test-only emulator build reads through those)
#pragma once
#ifndef TRL_SIMT_EMU
#include <cuda.h>      // CUtensorMap (type only; the encoder is resolved at run time, nothing links against libcuda)
#define TRL_GRID_CONSTANT __grid_constant__
#else
#define TRL_GRID_CONSTANT
#endif

namespace trl {
struct FcMaps {
#ifndef TRL_SIMT_EMU
    CUtensorMap w;      // terr_ip0 weights  [64 rows][5984] f64, box [64][16], 128-byte swizzle
    CUtensorMap a;      // conv2 outputs     [rows][5984]   f64, box [32][16], 128-byte swizzle
#endif
    const double* w_ptr;
    const double* a_ptr;
    int a_rows;
    unsigned long long* prof;    // measurement only (trl_debug_fc_phases): rank 0 / thread 0 of cluster 0 stamps %globaltimer at phase ends
};

// the terr_ip0 weight descriptor of every policy slot (slot build of the FC kernel; 8 x 128 B, a __grid_constant__ parameter)
struct FcSlotMaps {
#ifndef TRL_SIMT_EMU
    CUtensorMap w[8];
#endif
    const double* w_ptr[8];
};

// the same two kernels as the forward pass of a TRAINER batch (trl_train.cu): rows = the minibatch, inputs already normalised, every
// activation the backward pass needs written out, raw (normalised) outputs, no decisions.  All-null in the decision path.
struct FwdTrain {
    const double* xn;                 // [rows][S] normalised net inputs
    int rows, S, cat, n_out, n_frags, frag;
    const int* gate;                  // device word: the launch is a no-op while it is 0 (the trainer's on-device control flow)
    double *a0, *a1;                  // post-ReLU conv0 / conv1 activations [rows][16 * 193], [rows][32 * 190] (null: not kept)
    double *t, *catb, *h, *hh, *y;    // [rows][64], [rows][cat], [rows][256], [4][rows][128] (null: not kept), raw outputs [rows][n_out]
};
}  // namespace trl
