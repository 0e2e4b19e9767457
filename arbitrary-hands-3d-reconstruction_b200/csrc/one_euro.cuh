// One step of the OneEuro filter on one element (acr/utils.py:1485-1527), shared by the per-hand-type smoothing
// (smooth.cu) and the per-track smoothing of the tracker (track.cu), so that both run the same arithmetic:
//   x_hat = lowpass(x, alpha(mincutoff + beta*|lowpass(dx, alpha(dcutoff))|)),  dx = (x - x_prev)*freq,
//   alpha(c) = 1 / (1 + (1/(2 pi c)) / (1/freq)),  freq = 30 (te = 1/30 whatever the gap), beta = 0.7, dcutoff = 1.
#pragma once
#include <cuda_runtime.h>

namespace acr {

__device__ __forceinline__ float one_euro_alpha(float cutoff) {
  const float te = 1.0f / 30.0f;
  const float tau = 1.0f / (2.0f * 3.14159265358979323846f * cutoff);
  return 1.0f / (1.0f + tau / te);
}

// x: the new raw value; raw, filt, fdx: the bank's previous raw value, filtered value and filtered derivative.
// Writes the filtered value xh and the filtered derivative edx.  The roundings are spelled out (which product each
// FMA absorbs), so every kernel that inlines this step computes the same bits whatever its surrounding code.
__device__ __forceinline__ void one_euro_step(float x, float mincut, float raw, float filt, float fdx, float& xh,
                                              float& edx) {
  const float dx = __fmul_rn(__fsub_rn(x, raw), 30.0f);
  const float ad = one_euro_alpha(1.0f);
  edx = __fmaf_rn(fdx, 1.0f - ad, __fmul_rn(dx, ad));
  const float a = one_euro_alpha(__fmaf_rn(fabsf(edx), 0.7f, mincut));
  xh = __fmaf_rn(a, x, __fmul_rn(1.0f - a, filt));
}

}  // namespace acr
