// Device-side rotation chain, float32, op-for-op the reference's order of evaluation so that the
// same branches are taken on the same inputs.
//   rodrigues()     : batch_rodrigues + quat2mat      /root/reference/mano/manolayer.py:423-434, 396-421
//   rot6d_to_aa()   : rot6d_to_rotmat -> rotation_matrix_to_quaternion -> quaternion_to_angle_axis
//                     -> NaN->0                         /root/reference/acr/utils.py:362-376, 826-906,
//                                                       773-823, 334-360
#pragma once
#include <cuda_runtime.h>

namespace acr {

// separately rounded products/sums (no FMA contraction), like the reference's element-wise ATen
// kernels: keeps the Gram-Schmidt residual of near-degenerate 6D inputs identical to the reference's
__device__ __forceinline__ float dot3_rn(float ax, float ay, float az, float bx, float by, float bz) {
  return __fadd_rn(__fadd_rn(__fmul_rn(ax, bx), __fmul_rn(ay, by)), __fmul_rn(az, bz));
}

// sin / cos of half the rotation angle.  kPiTrig selects sincospif, whose argument reduction is exact and needs no
// local memory (sincosf's large-argument path keeps a scratch array there); the two agree to an ulp or two.
template <bool kPiTrig>
__device__ __forceinline__ void half_angle_sincos(float ang, float* s, float* c) {
  if constexpr (kPiTrig) sincospif(ang * 0.159154943f, s, c);   // ang / (2 pi)
  else sincosf(ang * 0.5f, s, c);
}

template <bool kPiTrig = false>
__device__ __forceinline__ void rodrigues(float ax, float ay, float az, float* R) {
  // angle = || aa + 1e-8 ||, axis = aa / angle, q = [cos(a/2), sin(a/2) axis], q /= ||q||
  const float bx = ax + 1e-8f, by = ay + 1e-8f, bz = az + 1e-8f;
  const float ang = sqrtf(bx * bx + by * by + bz * bz);
  const float nx = ax / ang, ny = ay / ang, nz = az / ang;
  float s, c;
  half_angle_sincos<kPiTrig>(ang, &s, &c);
  float w = c, x = s * nx, y = s * ny, z = s * nz;
  const float qn = sqrtf(w * w + x * x + y * y + z * z);
  w /= qn; x /= qn; y /= qn; z /= qn;
  const float w2 = w * w, x2 = x * x, y2 = y * y, z2 = z * z;
  const float wx = w * x, wy = w * y, wz = w * z, xy = x * y, xz = x * z, yz = y * z;
  R[0] = w2 + x2 - y2 - z2; R[1] = 2 * xy - 2 * wz;   R[2] = 2 * wy + 2 * xz;
  R[3] = 2 * wz + 2 * xy;   R[4] = w2 - x2 + y2 - z2; R[5] = 2 * yz - 2 * wx;
  R[6] = 2 * xz - 2 * wy;   R[7] = 2 * wx + 2 * yz;   R[8] = w2 - x2 - y2 + z2;
}

// Vector-Jacobian product of rodrigues(): dR (row-major 3x3 cotangent) -> da, the exact derivative of the
// quaternion form above (the 1e-8 offset sits in the angle only, the axis numerator is `a`).  Written in n = a/angle
// and s/angle = sin(angle/2)/angle, which stay bounded, so it is finite at a = 0 (angle = sqrt(3)*1e-8).
__device__ __forceinline__ void rodrigues_vjp(float ax, float ay, float az, const float* g, float* da) {
  const float bx = ax + 1e-8f, by = ay + 1e-8f, bz = az + 1e-8f;
  const float ang = sqrtf(bx * bx + by * by + bz * bz);
  const float nx = ax / ang, ny = ay / ang, nz = az / ang;
  float s, c;
  half_angle_sincos<true>(ang, &s, &c);
  const float q[4] = {c, s * nx, s * ny, s * nz};
  const float qn = sqrtf(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
  const float w = q[0] / qn, x = q[1] / qn, y = q[2] / qn, z = q[3] / qn;
  // quat2mat: d/d(w,x,y,z) of the nine entries, contracted with g
  float dq[4];
  dq[0] = 2.f * (w * (g[0] + g[4] + g[8]) + x * (g[7] - g[5]) + y * (g[2] - g[6]) + z * (g[3] - g[1]));
  dq[1] = 2.f * (x * (g[0] - g[4] - g[8]) + y * (g[1] + g[3]) + z * (g[2] + g[6]) + w * (g[7] - g[5]));
  dq[2] = 2.f * (y * (g[4] - g[0] - g[8]) + x * (g[1] + g[3]) + w * (g[2] - g[6]) + z * (g[5] + g[7]));
  dq[3] = 2.f * (z * (g[8] - g[0] - g[4]) + w * (g[3] - g[1]) + x * (g[2] + g[6]) + y * (g[5] + g[7]));
  // q / ||q||
  const float proj = w * dq[0] + x * dq[1] + y * dq[2] + z * dq[3];
  dq[0] = (dq[0] - w * proj) / qn; dq[1] = (dq[1] - x * proj) / qn;
  dq[2] = (dq[2] - y * proj) / qn; dq[3] = (dq[3] - z * proj) / qn;
  // q = [cos(ang/2), sin(ang/2) a/ang], ang = ||a + 1e-8||
  const float sa = s / ang;
  const float nd = nx * dq[1] + ny * dq[2] + nz * dq[3];
  const float dang = 0.5f * (c * nd - s * dq[0]) - sa * nd;
  da[0] = sa * dq[1] + dang * (bx / ang);
  da[1] = sa * dq[2] + dang * (by / ang);
  da[2] = sa * dq[3] + dang * (bz / ang);
}

// Jacobian-vector product of rodrigues(): da (tangent of the axis angle) -> dR (row-major).  The forward-mode twin
// of rodrigues_vjp, in the same bounded quantities n = a/angle and s/angle, so it is finite at a = 0 as well.
__device__ __forceinline__ void rodrigues_jvp(float ax, float ay, float az, const float* da, float* dR) {
  const float bx = ax + 1e-8f, by = ay + 1e-8f, bz = az + 1e-8f;
  const float ang = sqrtf(bx * bx + by * by + bz * bz);
  const float nx = ax / ang, ny = ay / ang, nz = az / ang;
  float s, c;
  half_angle_sincos<true>(ang, &s, &c);
  const float q[4] = {c, s * nx, s * ny, s * nz};
  const float qn = sqrtf(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
  const float w = q[0] / qn, x = q[1] / qn, y = q[2] / qn, z = q[3] / qn;
  // q = [cos(ang/2), (s/ang) a]:  d ang = (b/ang) . da,  d(s/ang) a = n (c/2 - s/ang) d ang
  const float sa = s / ang;
  const float dang = (bx / ang) * da[0] + (by / ang) * da[1] + (bz / ang) * da[2];
  const float k = (0.5f * c - sa) * dang;
  float dq[4] = {-0.5f * s * dang, sa * da[0] + nx * k, sa * da[1] + ny * k, sa * da[2] + nz * k};
  // q / ||q||
  const float proj = w * dq[0] + x * dq[1] + y * dq[2] + z * dq[3];
  const float dw = (dq[0] - w * proj) / qn, dx = (dq[1] - x * proj) / qn;
  const float dy = (dq[2] - y * proj) / qn, dz = (dq[3] - z * proj) / qn;
  // quat2mat, differentiated entry by entry
  dR[0] = 2.f * (w * dw + x * dx - y * dy - z * dz);
  dR[1] = 2.f * (dx * y + x * dy - dw * z - w * dz);
  dR[2] = 2.f * (dw * y + w * dy + dx * z + x * dz);
  dR[3] = 2.f * (dw * z + w * dz + dx * y + x * dy);
  dR[4] = 2.f * (w * dw - x * dx + y * dy - z * dz);
  dR[5] = 2.f * (dy * z + y * dz - dw * x - w * dx);
  dR[6] = 2.f * (dx * z + x * dz - dw * y - w * dy);
  dR[7] = 2.f * (dw * x + w * dx + dy * z + y * dz);
  dR[8] = 2.f * (w * dw - x * dx - y * dy + z * dz);
}

// ------------------------------------------------------------------------------ SO(3) projection (batch_rotprojs)
// The reference (mano/manolayer.py:436-453) takes the SVD M = U S V^T of every input matrix, forms the orthogonal
// polar factor Q = U V^T and negates column 2 of Q when det Q < 0.  Here, per thread and in fp64: a fixed-sweep
// cyclic Jacobi eigensolve of A = M^T M gives V (a proper rotation) and S^2; then u_i = M v_i normalised for the two
// largest singular values (Gram-Schmidt on the second), u_3 = sign(det M) (u_1 x u_2), and Q = sum_i u_i v_i^T.
// Contract: M of rank >= 2 gives a finite orthogonal Q (at rank 2, det M is zero up to rounding and its computed
// sign picks the orientation).  Rank <= 1 is outside it -- the reference's own result is arbitrary there -- and
// gives NaN.  All indexing is compile-time, so nothing lives in local memory.
template <int p, int q>
__device__ __forceinline__ void jacobi_rotate(double (&a)[3][3], double (&v)[3][3]) {
  constexpr int r = 3 - p - q;
  const double apq = a[p][q];
  if (apq == 0.0) return;
  const double th = (a[q][q] - a[p][p]) / (2.0 * apq);
  const double t = copysign(1.0, th) / (fabs(th) + sqrt(fma(th, th, 1.0)));   // th = +-inf -> t = 0
  const double c = rsqrt(fma(t, t, 1.0)), s = t * c;
  const double app = a[p][p] - t * apq, aqq = a[q][q] + t * apq;
  const double arp = c * a[r][p] - s * a[r][q], arq = s * a[r][p] + c * a[r][q];
  a[p][p] = app; a[q][q] = aqq; a[p][q] = a[q][p] = 0.0;
  a[r][p] = a[p][r] = arp; a[r][q] = a[q][r] = arq;
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    const double vp = v[i][p], vq = v[i][q];
    v[i][p] = c * vp - s * vq; v[i][q] = s * vp + c * vq;
  }
}

// swap eigenpairs i < k so that lam[i] >= lam[k]; negating one column keeps det V = +1
template <int i, int k>
__device__ __forceinline__ void eig_order(double (&lam)[3], double (&v)[3][3]) {
  if (lam[i] >= lam[k]) return;
  const double l = lam[i]; lam[i] = lam[k]; lam[k] = l;
#pragma unroll
  for (int e = 0; e < 3; ++e) { const double x = v[e][i]; v[e][i] = v[e][k]; v[e][k] = -x; }
}

// M (row-major 3x3, fp32) -> its orthogonal polar factor Q (fp64, row-major) and whether det Q < 0 (`flip`; the
// reference then negates column 2 of Q).  The output rotation is Q diag(1, 1, flip ? -1 : 1).
__device__ __forceinline__ void polar_factor(const float* __restrict__ Mf, double (&Q)[3][3], bool& flip) {
  double M[3][3], a[3][3], v[3][3];
#pragma unroll
  for (int r = 0; r < 3; ++r)
#pragma unroll
    for (int c = 0; c < 3; ++c) { M[r][c] = (double)Mf[r * 3 + c]; v[r][c] = r == c ? 1.0 : 0.0; }
#pragma unroll
  for (int r = 0; r < 3; ++r)
#pragma unroll
    for (int c = 0; c < 3; ++c) a[r][c] = M[0][r] * M[0][c] + M[1][r] * M[1][c] + M[2][r] * M[2][c];
  // quadratic convergence: 6 cyclic sweeps take any 3x3 well below fp64 rounding
#pragma unroll 1
  for (int sweep = 0; sweep < 6; ++sweep) {
    jacobi_rotate<0, 1>(a, v);
    jacobi_rotate<0, 2>(a, v);
    jacobi_rotate<1, 2>(a, v);
  }
  double lam[3] = {a[0][0], a[1][1], a[2][2]};
  eig_order<0, 1>(lam, v);
  eig_order<1, 2>(lam, v);
  eig_order<0, 1>(lam, v);
  double u[2][3];
#pragma unroll
  for (int k = 0; k < 2; ++k)
#pragma unroll
    for (int r = 0; r < 3; ++r) u[k][r] = M[r][0] * v[0][k] + M[r][1] * v[1][k] + M[r][2] * v[2][k];
  double n0 = rsqrt(u[0][0] * u[0][0] + u[0][1] * u[0][1] + u[0][2] * u[0][2]);
#pragma unroll
  for (int r = 0; r < 3; ++r) u[0][r] *= n0;
  const double d01 = u[0][0] * u[1][0] + u[0][1] * u[1][1] + u[0][2] * u[1][2];
#pragma unroll
  for (int r = 0; r < 3; ++r) u[1][r] -= d01 * u[0][r];
  double n1 = rsqrt(u[1][0] * u[1][0] + u[1][1] * u[1][1] + u[1][2] * u[1][2]);
#pragma unroll
  for (int r = 0; r < 3; ++r) u[1][r] *= n1;
  const double detM = M[0][0] * (M[1][1] * M[2][2] - M[1][2] * M[2][1]) - M[0][1] * (M[1][0] * M[2][2] - M[1][2] * M[2][0]) +
                      M[0][2] * (M[1][0] * M[2][1] - M[1][1] * M[2][0]);
  flip = detM < 0.0;
  const double sg = flip ? -1.0 : 1.0;
  const double u2[3] = {sg * (u[0][1] * u[1][2] - u[0][2] * u[1][1]), sg * (u[0][2] * u[1][0] - u[0][0] * u[1][2]),
                        sg * (u[0][0] * u[1][1] - u[0][1] * u[1][0])};
#pragma unroll
  for (int r = 0; r < 3; ++r)
#pragma unroll
    for (int c = 0; c < 3; ++c) Q[r][c] = u[0][r] * v[c][0] + u[1][r] * v[c][1] + u2[r] * v[c][2];
}

// batch_rotprojs of one matrix: M (row-major, fp32) -> R = Q D (row-major, fp32)
__device__ __forceinline__ void so3_project(const float* __restrict__ M, float* __restrict__ R) {
  double Q[3][3];
  bool flip;
  polar_factor(M, Q, flip);
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    R[r * 3 + 0] = (float)Q[r][0]; R[r * 3 + 1] = (float)Q[r][1];
    R[r * 3 + 2] = (float)(flip ? -Q[r][2] : Q[r][2]);
  }
}

// Vector-Jacobian product of so3_project(): g (cotangent of R, row-major) -> dM.  With P = Q^T M (symmetric),
// B = Q^T (g D) and k = axial(B - B^T):  z = ((tr P) I - P)^-1 k,  dM = Q [z]x.  (tr P) I - P has the eigenvalues
// s_j + s_k, so this is finite whenever no two singular values sum to zero -- in particular at exact rotations,
// where the SVD's own derivative (1 / (s_i^2 - s_j^2)) is not.
__device__ __forceinline__ void so3_project_vjp(const float* __restrict__ Mf, const float* __restrict__ g,
                                                float* __restrict__ dM) {
  double Q[3][3];
  bool flip;
  polar_factor(Mf, Q, flip);
  double P[3][3], B[3][3];
#pragma unroll
  for (int r = 0; r < 3; ++r)
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const double gd = c == 2 && flip ? -1.0 : 1.0;
      P[r][c] = Q[0][r] * (double)Mf[0 * 3 + c] + Q[1][r] * (double)Mf[1 * 3 + c] + Q[2][r] * (double)Mf[2 * 3 + c];
      B[r][c] = gd * (Q[0][r] * (double)g[0 * 3 + c] + Q[1][r] * (double)g[1 * 3 + c] + Q[2][r] * (double)g[2 * 3 + c]);
    }
  const double k0 = B[2][1] - B[1][2], k1 = B[0][2] - B[2][0], k2 = B[1][0] - B[0][1];
  const double tr = P[0][0] + P[1][1] + P[2][2];
  // A = tr I - P (symmetrised), solved through its adjugate
  const double a00 = tr - P[0][0], a11 = tr - P[1][1], a22 = tr - P[2][2];
  const double a01 = -0.5 * (P[0][1] + P[1][0]), a02 = -0.5 * (P[0][2] + P[2][0]), a12 = -0.5 * (P[1][2] + P[2][1]);
  const double c00 = a11 * a22 - a12 * a12, c01 = a02 * a12 - a01 * a22, c02 = a01 * a12 - a02 * a11;
  const double c11 = a00 * a22 - a02 * a02, c12 = a01 * a02 - a00 * a12, c22 = a00 * a11 - a01 * a01;
  const double inv = 1.0 / (a00 * c00 + a01 * c01 + a02 * c02);
  const double z0 = (c00 * k0 + c01 * k1 + c02 * k2) * inv;
  const double z1 = (c01 * k0 + c11 * k1 + c12 * k2) * inv;
  const double z2 = (c02 * k0 + c12 * k1 + c22 * k2) * inv;
  // [z]x = [[0, -z2, z1], [z2, 0, -z0], [-z1, z0, 0]]
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    dM[r * 3 + 0] = (float)(Q[r][1] * z2 - Q[r][2] * z1);
    dM[r * 3 + 1] = (float)(Q[r][2] * z0 - Q[r][0] * z2);
    dM[r * 3 + 2] = (float)(Q[r][0] * z1 - Q[r][1] * z0);
  }
}

// Jacobian-vector product of so3_project(), for several tangents of one matrix.  M = Q P with P = Q^T M symmetric,
// so dM = dQ P + Q dP with dQ = Q [w]x and dP symmetric: the skew part of X = Q^T dM is that of [w]x P + P [w]x =
// [((tr P) I - P) w]x, hence w = ((tr P) I - P)^-1 axial(X - X^T) and dR = Q [w]x D.  The same matrix as in the VJP
// (finite unless two singular values sum to zero, so at exact rotations too); set up once, then apply per tangent.
struct So3ProjectJvp {
  double Q[3][3];
  double c00, c01, c02, c11, c12, c22;   // adjugate of (tr P) I - P (symmetrised), divided by its determinant
  bool flip;

  __device__ __forceinline__ void setup(const float* __restrict__ Mf) {
    polar_factor(Mf, Q, flip);
    double P[3][3];
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
      for (int c = 0; c < 3; ++c)
        P[r][c] = Q[0][r] * (double)Mf[0 * 3 + c] + Q[1][r] * (double)Mf[1 * 3 + c] + Q[2][r] * (double)Mf[2 * 3 + c];
    const double tr = P[0][0] + P[1][1] + P[2][2];
    const double a00 = tr - P[0][0], a11 = tr - P[1][1], a22 = tr - P[2][2];
    const double a01 = -0.5 * (P[0][1] + P[1][0]), a02 = -0.5 * (P[0][2] + P[2][0]), a12 = -0.5 * (P[1][2] + P[2][1]);
    c00 = a11 * a22 - a12 * a12; c01 = a02 * a12 - a01 * a22; c02 = a01 * a12 - a02 * a11;
    c11 = a00 * a22 - a02 * a02; c12 = a01 * a02 - a00 * a12; c22 = a00 * a11 - a01 * a01;
    const double inv = 1.0 / (a00 * c00 + a01 * c01 + a02 * c02);
    c00 *= inv; c01 *= inv; c02 *= inv; c11 *= inv; c12 *= inv; c22 *= inv;
  }

  // dM (tangent of M, row-major, fp32) -> dR (row-major, fp32)
  __device__ __forceinline__ void apply(const float* __restrict__ dMf, float* __restrict__ dR) const {
    double X[3][3];
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
      for (int c = 0; c < 3; ++c)
        X[r][c] = Q[0][r] * (double)dMf[0 * 3 + c] + Q[1][r] * (double)dMf[1 * 3 + c] + Q[2][r] * (double)dMf[2 * 3 + c];
    const double k0 = X[2][1] - X[1][2], k1 = X[0][2] - X[2][0], k2 = X[1][0] - X[0][1];
    const double z0 = c00 * k0 + c01 * k1 + c02 * k2;
    const double z1 = c01 * k0 + c11 * k1 + c12 * k2;
    const double z2 = c02 * k0 + c12 * k1 + c22 * k2;
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      dR[r * 3 + 0] = (float)(Q[r][1] * z2 - Q[r][2] * z1);
      dR[r * 3 + 1] = (float)(Q[r][2] * z0 - Q[r][0] * z2);
      const double d2 = Q[r][0] * z1 - Q[r][1] * z0;
      dR[r * 3 + 2] = (float)(flip ? -d2 : d2);
    }
  }
};

// rotation_matrix_to_angle_axis (acr/utils.py:334-360) of a row-major 3x3 (not necessarily orthonormal)
// matrix: 4-case quaternion on the TRANSPOSED matrix (:862-906), atan2 form (:803-823), NaN -> 0.
__device__ __forceinline__ void rotmat_to_aa(const float* __restrict__ R, float* __restrict__ aa) {
  // t = R^T, i.e. t(i,j) = R(j,i)
  const float t00 = R[0], t01 = R[3], t02 = R[6], t10 = R[1], t11 = R[4], t12 = R[7], t20 = R[2], t21 = R[5], t22 = R[8];
  float qw, qx, qy, qz, tt;
  if (t22 < 1e-6f) {
    if (t00 > t11) {
      tt = 1 + t00 - t11 - t22;
      qw = t12 - t21; qx = tt; qy = t01 + t10; qz = t20 + t02;
    } else {
      tt = 1 - t00 + t11 - t22;
      qw = t20 - t02; qx = t01 + t10; qy = tt; qz = t12 + t21;
    }
  } else {
    if (t00 < -t11) {
      tt = 1 - t00 - t11 + t22;
      qw = t01 - t10; qx = t20 + t02; qy = t12 + t21; qz = tt;
    } else {
      tt = 1 + t00 + t11 + t22;
      qw = tt; qx = t12 - t21; qy = t20 - t02; qz = t01 - t10;
    }
  }
  const float sc = sqrtf(tt);
  qw = qw / sc * 0.5f; qx = qx / sc * 0.5f; qy = qy / sc * 0.5f; qz = qz / sc * 0.5f;
  const float s2 = qx * qx + qy * qy + qz * qz;
  const float sn = sqrtf(s2);
  const float two_theta = 2.0f * ((qw < 0.0f) ? atan2f(-sn, -qw) : atan2f(sn, qw));
  const float k = (s2 > 0.0f) ? two_theta / sn : 2.0f;
  const float ox = qx * k, oy = qy * k, oz = qz * k;
  aa[0] = isnan(ox) ? 0.f : ox;
  aa[1] = isnan(oy) ? 0.f : oy;
  aa[2] = isnan(oz) ? 0.f : oz;
}

__device__ __forceinline__ void rot6d_to_aa(const float* __restrict__ r6, float* __restrict__ aa) {
  // the 6 numbers are a row-major (3,2) matrix: a1 = column 0, a2 = column 1
  const float a1x = r6[0], a1y = r6[2], a1z = r6[4];
  const float a2x = r6[1], a2y = r6[3], a2z = r6[5];
  // b1 = a1 / max(||a1||, 1e-6)
  float n1 = fmaxf(sqrtf(dot3_rn(a1x, a1y, a1z, a1x, a1y, a1z)), 1e-6f);
  const float b1x = a1x / n1, b1y = a1y / n1, b1z = a1z / n1;
  const float d = dot3_rn(b1x, b1y, b1z, a2x, a2y, a2z);
  const float ux = __fsub_rn(a2x, __fmul_rn(d, b1x)), uy = __fsub_rn(a2y, __fmul_rn(d, b1y)),
              uz = __fsub_rn(a2z, __fmul_rn(d, b1z));
  float n2 = fmaxf(sqrtf(dot3_rn(ux, uy, uz, ux, uy, uz)), 1e-6f);
  const float b2x = ux / n2, b2y = uy / n2, b2z = uz / n2;
  const float b3x = __fsub_rn(__fmul_rn(b1y, b2z), __fmul_rn(b1z, b2y)),
              b3y = __fsub_rn(__fmul_rn(b1z, b2x), __fmul_rn(b1x, b2z)),
              b3z = __fsub_rn(__fmul_rn(b1x, b2y), __fmul_rn(b1y, b2x));
  // R = [b1 b2 b3] (columns), row-major
  const float R[9] = {b1x, b2x, b3x, b1y, b2y, b3y, b1z, b2z, b3z};
  rotmat_to_aa(R, aa);
}

}  // namespace acr
