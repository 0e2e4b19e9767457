// Closed-form camera translation of one hand, shared by acr_b200_cam_trans (mano.cu) and the least-squares
// branches of acr_b200_cam_trans_pnp (pnp.cu).
#pragma once
#include "common.cuh"

namespace acr {

// estimate_translation_np (acr/utils.py:430-472) for one hand, fp64 like the numpy original:
// rows [f,0,cx-u | (u-cx)*Z - f*X] and [0,f,cy-v | (v-cy)*Z - f*Y] of every usable joint, normal equations.
// j3d (21,3), pj2d (21,2) of the hand -> o (3); fewer than 4 usable joints -> (-1,-1,-1).
__device__ __forceinline__ void cam_trans_lstsq(const float* __restrict__ j3d, const float* __restrict__ pj2d,
                                                float focal, float img_size, float* __restrict__ o) {
  const double f = focal, c0 = (double)(img_size * 0.5f);
  double A00 = 0, A01 = 0, A02 = 0, A11 = 0, A12 = 0, A22 = 0, b0 = 0, b1 = 0, b2 = 0;
  int used = 0;
  for (int j = 0; j < 21; ++j) {
    const float X = j3d[j * 3 + 0], Y = j3d[j * 3 + 1], Z = j3d[j * 3 + 2];
    const float u = (pj2d[j * 2 + 0] + 1.f) * (img_size * 0.5f);
    const float v = (pj2d[j * 2 + 1] + 1.f) * (img_size * 0.5f);
    if (!(v > -2.f) || Z == -2.f) continue;   // the reference's "confidence" tests (acr/utils.py:489-492)
    ++used;
    const double qx = c0 - (double)u, qy = c0 - (double)v;        // third column of the two rows
    const double cx = ((double)u - c0) * (double)Z - f * (double)X, cy = ((double)v - c0) * (double)Z - f * (double)Y;
    A00 += f * f; A02 += f * qx; b0 += f * cx;
    A11 += f * f; A12 += f * qy; b1 += f * cy;
    A22 += qx * qx + qy * qy; b2 += qx * cx + qy * cy;
  }
  if (used < 4) { o[0] = o[1] = o[2] = -1.f; return; }
  // symmetric 3x3 solve (A01 = 0): Cramer's rule in fp64
  const double det = A00 * (A11 * A22 - A12 * A12) - A01 * (A01 * A22 - A12 * A02) + A02 * (A01 * A12 - A11 * A02);
  const double d0 = b0 * (A11 * A22 - A12 * A12) - A01 * (b1 * A22 - A12 * b2) + A02 * (b1 * A12 - A11 * b2);
  const double d1 = A00 * (b1 * A22 - A12 * b2) - b0 * (A01 * A22 - A12 * A02) + A02 * (A01 * b2 - b1 * A02);
  const double d2 = A00 * (A11 * b2 - b1 * A12) - A01 * (A01 * b2 - b1 * A02) + b0 * (A01 * A12 - A11 * A02);
  o[0] = (float)(d0 / det); o[1] = (float)(d1 / det); o[2] = (float)(d2 / det);
}

}  // namespace acr
