// Fused BasicBlock kernel instances (conv_block.cuh): {bf16, fp16} x {64-channel, x-paired 32-channel}.
#include "conv_block.cuh"

namespace acr {

template <typename T, bool XPAIR>
static int launch_block(const ConvBlockPlan* pl, cudaStream_t st) {
  static unsigned long long configured = 0;
  ACR_CHECK_CUDA(ensure_dynamic_smem(conv_block_kernel<T, XPAIR>, (int)BLK_SMEM, &configured));
  return launch_pdl(conv_block_kernel<T, XPAIR>, pl->p, pl->grid, BLK_SMEM, st);
}

int conv_block_launch(const ConvBlockPlan* pl, cudaStream_t st) {
  if (pl->act_dtype == ACR_DT_BF16)
    return pl->xpair ? launch_block<__nv_bfloat16, true>(pl, st) : launch_block<__nv_bfloat16, false>(pl, st);
  return pl->xpair ? launch_block<__half, true>(pl, st) : launch_block<__half, false>(pl, st);
}

}  // namespace acr
