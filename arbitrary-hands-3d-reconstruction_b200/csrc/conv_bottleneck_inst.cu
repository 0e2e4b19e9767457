// Fused Bottleneck kernel instances (conv_bottleneck.cuh): {bf16, fp16} x {C_in = 64, C_in = 256}.
#include "conv_bottleneck.cuh"

namespace acr {

template <typename T, int CCHUNKS>
static int launch_bottleneck(const ConvBottleneckPlan* pl, cudaStream_t st) {
  static unsigned long long configured = 0;
  ACR_CHECK_CUDA(ensure_dynamic_smem(conv_bottleneck_kernel<T, CCHUNKS>, (int)BNK_SMEM, &configured));
  return launch_pdl(conv_bottleneck_kernel<T, CCHUNKS>, pl->p, pl->grid, BNK_SMEM, st);
}

int conv_bottleneck_launch(const ConvBottleneckPlan* pl, cudaStream_t st) {
  if (pl->act_dtype == ACR_DT_BF16)
    return pl->cchunks == 1 ? launch_bottleneck<__nv_bfloat16, 1>(pl, st) : launch_bottleneck<__nv_bfloat16, 4>(pl, st);
  return pl->cchunks == 1 ? launch_bottleneck<__half, 1>(pl, st) : launch_bottleneck<__half, 4>(pl, st);
}

}  // namespace acr
