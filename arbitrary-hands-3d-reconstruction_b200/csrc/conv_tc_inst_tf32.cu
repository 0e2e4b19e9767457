// Conv kernel instances (conv_tc.cuh) for fp32 activations on the tf32 tensor cores (the TF32 plan): 64- and 32-byte-
// channel chunks (32 / 16 fp32 channels) in one translation unit.
#include "conv_tc.cuh"

namespace acr {

int conv_tc_launch_tf32(const ConvTcPlan* pl, cudaStream_t st) {
  return pl->ck == 64 ? launch_mode<64, float>(pl, st) : launch_mode<32, float>(pl, st);
}

}  // namespace acr
