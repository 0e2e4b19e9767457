// Camera translation of every hand as the reference computes it: cv2.solvePnPRansac(SOLVEPNP_EPNP,
// reprojectionError=20, iterationsCount=100) on the usable joints (estimate_translation, acr/utils.py:414-428,
// 474-519), with the closed-form least squares (cam_trans.cuh) where the reference falls back to it.
//
// One warp per hand, everything in fp64 except what OpenCV itself rounds to fp32:
//   * the usable joints are compacted into shared memory (ballot + prefix count);
//   * RANSAC runs uniformly on all lanes: OpenCV's RNG (multiply-with-carry, state all ones), subsets of 5
//     distinct points, a model replaces the best one iff its inlier count > max(best, 4), and then the iteration
//     bound becomes RANSACUpdateNumIters(0.99, outlier ratio, 5, bound) -- 0 once every point is an inlier, so the
//     typical hand costs one hypothesis plus the final fit;
//   * the inlier test runs one point per lane: projection in fp64, rounded to fp32, (dx^2 + dy^2) <= 400 in fp32;
//   * EPnP (Lepetit et al. 2009, as OpenCV states it) runs on the warp: per-point work (alphas, M^T M, the
//     reductions of the R, t fit, the reprojection error) one point per lane with butterfly sums, so every lane
//     ends with the same bits and runs the small scalar parts (3x3 SVDs, L_6x10, the beta approximations and
//     their Gauss-Newton steps) redundantly; the 12x12 M^T M goes through a round-robin parallel one-sided
//     Jacobi in shared memory, six disjoint column pairs at a time, four lanes per pair.
// The SVDs are one-sided Jacobi with OpenCV's rotation rule and threshold, and, as in OpenCV, the singular vectors
// EPnP uses are the normalised rotated columns.  The hypothesis' rotation is used as a matrix (OpenCV's Rodrigues
// round trip moves it by an ulp).  Exactly 4 usable joints would be OpenCV's P3P; this path returns the least
// squares there instead.  Planar or collinear usable joints have no EPnP control points: such a hypothesis has no
// inliers, and a final or 5-point fit on them returns the least squares with mask 0 (OpenCV carries on with a
// pseudo-inverse, in a null space where round-off decides the answer).
#include <float.h>

#include "common.cuh"
#include "cam_trans.cuh"

namespace acr {
namespace {

constexpr int NJ = 21;
constexpr int PNP_WARPS = 4;     // hands per CTA
constexpr unsigned FULL = 0xffffffffu;
constexpr double JAC_EPS = 10 * DBL_EPSILON;   // OpenCV's JacobiSVD threshold
constexpr int MODEL_PTS = 5, RANSAC_ITERS = 100;
constexpr float THRESH2 = 400.f;  // reprojectionError 20 px, squared

struct PnpSmem {
  double A[12][12];      // M^T M; the Jacobi sweeps rotate its columns (= rows, it is symmetric) in place
  double ut[4][12];      // EPnP's v[0..3]: the left singular vectors of the four smallest singular values
  double L[6][10], rho[6];
  double cws[4][3];      // control points
  double R[3][3], t[3];  // pose of the last epnp() call
  double al[NJ][4];      // barycentric alphas of the current point set
  double du[NJ], dv[NJ]; // c - u, c - v of the current point set
  float S[NJ][3], J[NJ][2];  // usable joints (world, pixel), compacted
  int idx[NJ];           // their joint index
};

// a shared-memory read the compiler may not hoist out of a loop (keeps the 6x10 L and the null vectors out of
// registers, which the Gauss-Newton steps need)
__device__ __forceinline__ double vld(const double& x) { return *(const volatile double*)&x; }

__device__ __forceinline__ double wsum(double v) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(FULL, v, o);
  return v;
}

// OpenCV's one-sided Jacobi rotation of two columns with squared norms a, b and inner product p;
// false when they are orthogonal to the threshold.
__device__ __forceinline__ bool jacobi_rot(double a, double b, double p, double& c, double& s) {
  if (fabs(p) <= JAC_EPS * sqrt(a * b)) return false;
  p *= 2;
  const double beta = a - b, gamma = hypot(p, beta);
  if (beta < 0) {
    s = sqrt((gamma - beta) * 0.5 / gamma);
    c = p / (gamma * s * 2);
  } else {
    c = sqrt((gamma + beta) / (gamma * 2));
    s = p / (gamma * c * 2);
  }
  return true;
}

// SVD of a 3x3 matrix given as its transpose At (rows = columns of A).  On return w is descending, the rows of At
// are the left singular vectors and the rows of Vt the right ones.
__device__ __forceinline__ void svd3(double (&At)[3][3], double (&w)[3], double (&Vt)[3][3]) {
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    w[i] = At[i][0] * At[i][0] + At[i][1] * At[i][1] + At[i][2] * At[i][2];
#pragma unroll
    for (int k = 0; k < 3; ++k) Vt[i][k] = i == k ? 1.0 : 0.0;
  }
#pragma unroll 1
  for (int sweep = 0; sweep < 30; ++sweep) {
    bool changed = false;
#pragma unroll
    for (int pr = 0; pr < 3; ++pr) {
      const int i = pr == 2 ? 1 : 0, j = pr == 0 ? 1 : 2;
      double c, s;
      const double p = At[i][0] * At[j][0] + At[i][1] * At[j][1] + At[i][2] * At[j][2];
      if (jacobi_rot(w[i], w[j], p, c, s)) {
        double a = 0, b = 0;
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          const double t0 = c * At[i][k] + s * At[j][k], t1 = -s * At[i][k] + c * At[j][k];
          At[i][k] = t0; At[j][k] = t1;
          a += t0 * t0; b += t1 * t1;
          const double v0 = c * Vt[i][k] + s * Vt[j][k], v1 = -s * Vt[i][k] + c * Vt[j][k];
          Vt[i][k] = v0; Vt[j][k] = v1;
        }
        w[i] = a; w[j] = b;
        changed = true;
      }
    }
    if (!changed) break;
  }
#pragma unroll
  for (int i = 0; i < 3; ++i) w[i] = sqrt(At[i][0] * At[i][0] + At[i][1] * At[i][1] + At[i][2] * At[i][2]);
#pragma unroll
  for (int pr = 0; pr < 3; ++pr) {   // descending
    const int i = pr == 2 ? 1 : 0, j = pr == 0 ? 1 : 2;
    if (w[i] < w[j]) {
      double t = w[i]; w[i] = w[j]; w[j] = t;
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        t = At[i][k]; At[i][k] = At[j][k]; At[j][k] = t;
        t = Vt[i][k]; Vt[i][k] = Vt[j][k]; Vt[j][k] = t;
      }
    }
  }
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    const double s = w[i] > DBL_MIN ? 1.0 / w[i] : 0.0;
#pragma unroll
    for (int k = 0; k < 3; ++k) At[i][k] *= s;
  }
}

// One-sided Jacobi on the 12 columns of sm.A in round-robin order: the six disjoint pairs of a round at once, four
// lanes per pair, three elements per lane.  Then the four columns of smallest norm, normalised, go to sm.ut,
// smallest first.
__device__ void jacobi12(PnpSmem& sm, int lane) {
  const int pr = lane >> 2, q = (lane & 3) * 3;
  const bool act = lane < 24;
#pragma unroll 1
  for (int sweep = 0; sweep < 30; ++sweep) {
    bool changed = false;
#pragma unroll 1
    for (int r = 0; r < 11; ++r) {
      const int a = pr == 0 ? 0 : (pr - 1 + r) % 11 + 1, b = (10 - pr + r) % 11 + 1;
      const int i = act ? min(a, b) : 0, j = act ? max(a, b) : 1;
      double xi[3], xj[3], sa = 0, sb = 0, sp = 0;
#pragma unroll
      for (int e = 0; e < 3; ++e) {
        xi[e] = sm.A[i][q + e]; xj[e] = sm.A[j][q + e];
        sa += xi[e] * xi[e]; sb += xj[e] * xj[e]; sp += xi[e] * xj[e];
      }
#pragma unroll
      for (int o = 1; o <= 2; o <<= 1) {
        sa += __shfl_xor_sync(FULL, sa, o); sb += __shfl_xor_sync(FULL, sb, o); sp += __shfl_xor_sync(FULL, sp, o);
      }
      double c, s;
      __syncwarp();
      if (act && jacobi_rot(sa, sb, sp, c, s)) {
#pragma unroll
        for (int e = 0; e < 3; ++e) {
          sm.A[i][q + e] = c * xi[e] + s * xj[e];
          sm.A[j][q + e] = -s * xi[e] + c * xj[e];
        }
        changed = true;
      }
      __syncwarp();
    }
    if (!__any_sync(FULL, changed)) break;
  }
  double nrm = 0;
  if (lane < 12) {
#pragma unroll
    for (int k = 0; k < 12; ++k) nrm += sm.A[lane][k] * sm.A[lane][k];
    nrm = sqrt(nrm);
  }
  int rank = 0;   // position in the descending order of the 12 norms
#pragma unroll
  for (int k = 0; k < 12; ++k) {
    const double o = __shfl_sync(FULL, nrm, k);
    rank += (o > nrm) || (o == nrm && k < lane);
  }
  if (lane < 12 && rank >= 8) {
    const double s = nrm > DBL_MIN ? 1.0 / nrm : 0.0;
#pragma unroll
    for (int k = 0; k < 12; ++k) sm.ut[11 - rank][k] = sm.A[lane][k] * s;
  }
  __syncwarp();
}

// EPnP's Householder least squares on a 6 x NC system; false (x untouched) when A is singular.  The column scale
// eta is the largest magnitude in rows k..4, as in OpenCV.
template <int NC>
__device__ __forceinline__ bool qr_solve(double (&A)[6][NC], double (&b)[6], double (&x)[NC]) {
  double A1[NC], A2[NC];
#pragma unroll
  for (int k = 0; k < NC; ++k) {
    double eta = fabs(A[k][k]);
#pragma unroll
    for (int i = k + 1; i < 5; ++i) eta = fmax(eta, fabs(A[i][k]));
    if (eta == 0) return false;
    const double inv_eta = 1. / eta;
    double sum2 = 0;
#pragma unroll
    for (int i = k; i < 6; ++i) {
      A[i][k] *= inv_eta;
      sum2 += A[i][k] * A[i][k];
    }
    double sigma = sqrt(sum2);
    if (A[k][k] < 0) sigma = -sigma;
    A[k][k] += sigma;
    A1[k] = sigma * A[k][k];
    A2[k] = -eta * sigma;
#pragma unroll
    for (int j = k + 1; j < NC; ++j) {
      double sum = 0;
#pragma unroll
      for (int i = k; i < 6; ++i) sum += A[i][k] * A[i][j];
      const double tau = sum / A1[k];
#pragma unroll
      for (int i = k; i < 6; ++i) A[i][j] -= tau * A[i][k];
    }
  }
#pragma unroll
  for (int j = 0; j < NC; ++j) {
    double tau = 0;
#pragma unroll
    for (int i = j; i < 6; ++i) tau += A[i][j] * b[i];
    tau /= A1[j];
#pragma unroll
    for (int i = j; i < 6; ++i) b[i] -= tau * A[i][j];
  }
  x[NC - 1] = b[NC - 1] / A2[NC - 1];
#pragma unroll
  for (int i = NC - 2; i >= 0; --i) {
    double sum = 0;
#pragma unroll
    for (int j = i + 1; j < NC; ++j) sum += A[i][j] * x[j];
    x[i] = (b[i] - sum) / A2[i];
  }
  return true;
}

// least squares of rho on NC columns of L_6x10
template <int NC>
__device__ __forceinline__ bool solve_l(const PnpSmem& sm, const int (&cols)[NC], double (&x)[NC]) {
  double A[6][NC], b[6];
#pragma unroll
  for (int i = 0; i < 6; ++i) {
    b[i] = vld(sm.rho[i]);
#pragma unroll
    for (int k = 0; k < NC; ++k) A[i][k] = vld(sm.L[i][cols[k]]);
  }
#pragma unroll
  for (int k = 0; k < NC; ++k) x[k] = 0;
  return qr_solve<NC>(A, b, x);
}

// the three beta approximations (N = 1: B11 B12 B13 B14, N = 2: B11 B12 B22, N = 3: B11 B12 B22 B13 B23)
__device__ __forceinline__ void betas_approx(const PnpSmem& sm, int N, double (&beta)[4]) {
  if (N == 1) {
    const int cols[4] = {0, 1, 3, 6};
    double b[4];
    solve_l<4>(sm, cols, b);
    const double b0 = b[0] < 0 ? sqrt(-b[0]) : sqrt(b[0]), sg = b[0] < 0 ? -1.0 : 1.0;
    beta[0] = b0; beta[1] = sg * b[1] / b0; beta[2] = sg * b[2] / b0; beta[3] = sg * b[3] / b0;
    return;
  }
  double b[5];
  if (N == 2) {
    const int cols[3] = {0, 1, 2};
    double b3[3];
    solve_l<3>(sm, cols, b3);
    b[0] = b3[0]; b[1] = b3[1]; b[2] = b3[2]; b[3] = 0; b[4] = 0;
  } else {
    const int cols[5] = {0, 1, 2, 3, 4};
    solve_l<5>(sm, cols, b);
  }
  if (b[0] < 0) {
    beta[0] = sqrt(-b[0]);
    beta[1] = b[2] < 0 ? sqrt(-b[2]) : 0.0;
  } else {
    beta[0] = sqrt(b[0]);
    beta[1] = b[2] > 0 ? sqrt(b[2]) : 0.0;
  }
  if (b[1] < 0) beta[0] = -beta[0];
  beta[2] = N == 3 ? b[3] / beta[0] : 0.0;
  beta[3] = 0.0;
}

__device__ __forceinline__ void gauss_newton(const PnpSmem& sm, double (&beta)[4]) {
  double x[4] = {0, 0, 0, 0};
#pragma unroll 1
  for (int it = 0; it < 5; ++it) {
    double A[6][4], b[6];
#pragma unroll
    for (int i = 0; i < 6; ++i) {
      double l[10];
#pragma unroll
      for (int k = 0; k < 10; ++k) l[k] = vld(sm.L[i][k]);
      A[i][0] = 2 * l[0] * beta[0] + l[1] * beta[1] + l[3] * beta[2] + l[6] * beta[3];
      A[i][1] = l[1] * beta[0] + 2 * l[2] * beta[1] + l[4] * beta[2] + l[7] * beta[3];
      A[i][2] = l[3] * beta[0] + l[4] * beta[1] + 2 * l[5] * beta[2] + l[8] * beta[3];
      A[i][3] = l[6] * beta[0] + l[7] * beta[1] + l[8] * beta[2] + 2 * l[9] * beta[3];
      b[i] = vld(sm.rho[i]) - (l[0] * beta[0] * beta[0] + l[1] * beta[0] * beta[1] + l[2] * beta[1] * beta[1] +
                          l[3] * beta[0] * beta[2] + l[4] * beta[1] * beta[2] + l[5] * beta[2] * beta[2] +
                          l[6] * beta[0] * beta[3] + l[7] * beta[1] * beta[3] + l[8] * beta[2] * beta[3] +
                          l[9] * beta[3] * beta[3]);
    }
    qr_solve<4>(A, b, x);
#pragma unroll
    for (int i = 0; i < 4; ++i) beta[i] += x[i];
  }
}

// R, t of one beta vector and its mean reprojection error; this lane's point (pw, u, v, alphas) if has.
__device__ __forceinline__ double r_and_t(const PnpSmem& sm, bool has, int np, const double (&pw)[3],
                                          const double (&pw0)[3], const double (&a)[4], double u, double v,
                                          double f, double c, const double (&beta)[4], double (&R)[3][3],
                                          double (&t)[3]) {
  double ccs[4][3];
#pragma unroll
  for (int j = 0; j < 4; ++j)
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      double s = 0.0;
#pragma unroll
      for (int i = 0; i < 4; ++i) s += beta[i] * vld(sm.ut[i][3 * j + k]);
      ccs[j][k] = s;
    }
  double pc[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) pc[k] = a[0] * ccs[0][k] + a[1] * ccs[1][k] + a[2] * ccs[2][k] + a[3] * ccs[3][k];
  if (__shfl_sync(FULL, pc[2], 0) < 0.0) {   // the first point must lie in front of the camera
#pragma unroll
    for (int k = 0; k < 3; ++k) pc[k] = -pc[k];
  }
  double pc0[3], At[3][3];
#pragma unroll
  for (int k = 0; k < 3; ++k) pc0[k] = wsum(has ? pc[k] : 0.0) / np;
#pragma unroll
  for (int j = 0; j < 3; ++j)
#pragma unroll
    for (int k = 0; k < 3; ++k) At[k][j] = wsum(has ? (pc[j] - pc0[j]) * (pw[k] - pw0[k]) : 0.0);
  double w[3], Vt[3][3];
  svd3(At, w, Vt);
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) R[i][j] = At[0][i] * Vt[0][j] + At[1][i] * Vt[1][j] + At[2][i] * Vt[2][j];
  const double det = R[0][0] * R[1][1] * R[2][2] + R[0][1] * R[1][2] * R[2][0] + R[0][2] * R[1][0] * R[2][1] -
                     R[0][2] * R[1][1] * R[2][0] - R[0][1] * R[1][0] * R[2][2] - R[0][0] * R[1][2] * R[2][1];
  if (det < 0) {
    R[2][0] = -R[2][0]; R[2][1] = -R[2][1]; R[2][2] = -R[2][2];
  }
#pragma unroll
  for (int i = 0; i < 3; ++i) t[i] = pc0[i] - (R[i][0] * pw0[0] + R[i][1] * pw0[1] + R[i][2] * pw0[2]);
  double e = 0.0;
  if (has) {
    const double Xc = R[0][0] * pw[0] + R[0][1] * pw[1] + R[0][2] * pw[2] + t[0];
    const double Yc = R[1][0] * pw[0] + R[1][1] * pw[1] + R[1][2] * pw[2] + t[1];
    const double iz = 1.0 / (R[2][0] * pw[0] + R[2][1] * pw[1] + R[2][2] * pw[2] + t[2]);
    const double ue = c + f * Xc * iz, ve = c + f * Yc * iz;
    e = sqrt((u - ue) * (u - ue) + (v - ve) * (v - ve));
  }
  return wsum(e) / np;
}

// EPnP on np <= 21 points, this lane's point (X, Y, Z) -> pixel (u, v) if lane < np; K = [f 0 c; 0 f c; 0 0 1].
// The pose goes to sm.R, sm.t; t is NaN when the points are planar or collinear (the smallest eigenvalue of their
// covariance at most 10 eps of the largest), where the control-point matrix has no inverse.
__device__ void epnp(PnpSmem& sm, int lane, int np, double X, double Y, double Z, double u, double v, double f,
                     double c) {
  __syncwarp();
  const bool has = lane < np;
  // control points: centroid + PCA
  double c0[3] = {wsum(has ? X : 0.0) / np, wsum(has ? Y : 0.0) / np, wsum(has ? Z : 0.0) / np};
  const double pw[3] = {X, Y, Z};
  const double d[3] = {has ? X - c0[0] : 0.0, has ? Y - c0[1] : 0.0, has ? Z - c0[2] : 0.0};
  double At[3][3], dc[3], Vt[3][3];
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = i; j < 3; ++j) At[i][j] = At[j][i] = wsum(d[i] * d[j]);
  svd3(At, dc, Vt);
  if (!(dc[2] > JAC_EPS * dc[0])) {   // planar or collinear points: no control points, no alphas (warp-uniform)
    if (lane == 0) sm.t[0] = sm.t[1] = sm.t[2] = __longlong_as_double(0x7ff8000000000000ll);
    __syncwarp();
    return;
  }
  double cws[4][3];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const double k = i ? sqrt(dc[i - 1] / np) : 0.0;
#pragma unroll
    for (int j = 0; j < 3; ++j) cws[i][j] = i ? c0[j] + k * At[i - 1][j] : c0[j];
  }
  // barycentric coordinates: CC[i][j-1] = cws[j][i] - cws[0][i], alphas = CC^-1 (p - c0)
  double C[3][3], Ci[3][3];
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) C[i][j] = cws[j + 1][i] - cws[0][i];
  Ci[0][0] = C[1][1] * C[2][2] - C[1][2] * C[2][1];
  Ci[0][1] = C[0][2] * C[2][1] - C[0][1] * C[2][2];
  Ci[0][2] = C[0][1] * C[1][2] - C[0][2] * C[1][1];
  Ci[1][0] = C[1][2] * C[2][0] - C[1][0] * C[2][2];
  Ci[1][1] = C[0][0] * C[2][2] - C[0][2] * C[2][0];
  Ci[1][2] = C[0][2] * C[1][0] - C[0][0] * C[1][2];
  Ci[2][0] = C[1][0] * C[2][1] - C[1][1] * C[2][0];
  Ci[2][1] = C[0][1] * C[2][0] - C[0][0] * C[2][1];
  Ci[2][2] = C[0][0] * C[1][1] - C[0][1] * C[1][0];
  const double idet = 1.0 / (C[0][0] * Ci[0][0] + C[0][1] * Ci[1][0] + C[0][2] * Ci[2][0]);
  double a[4];
#pragma unroll
  for (int j = 0; j < 3; ++j) a[1 + j] = (Ci[j][0] * d[0] + Ci[j][1] * d[1] + Ci[j][2] * d[2]) * idet;
  a[0] = 1.0 - a[1] - a[2] - a[3];
  if (has) {
#pragma unroll
    for (int k = 0; k < 4; ++k) sm.al[lane][k] = a[k];
    sm.du[lane] = c - u;
    sm.dv[lane] = c - v;
  }
  if (lane == 0) {
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 3; ++j) sm.cws[i][j] = cws[i][j];
  }
  __syncwarp();
  // M^T M, M = [a_k f, 0, a_k (c-u)] / [0, a_k f, a_k (c-v)] per point: one entry per lane and pass
#pragma unroll 1
  for (int e = lane; e < 144; e += 32) {
    const int ra = e / 12, rb = e % 12, ka = ra / 3, kb = rb / 3, pa = ra % 3, pb = rb % 3;
    double s = 0.0;
#pragma unroll 1
    for (int i = 0; i < np; ++i) {
      const double aa = sm.al[i][ka], ab = sm.al[i][kb];
      const double m1a = pa == 0 ? aa * f : pa == 1 ? 0.0 : aa * sm.du[i];
      const double m1b = pb == 0 ? ab * f : pb == 1 ? 0.0 : ab * sm.du[i];
      const double m2a = pa == 0 ? 0.0 : pa == 1 ? aa * f : aa * sm.dv[i];
      const double m2b = pb == 0 ? 0.0 : pb == 1 ? ab * f : ab * sm.dv[i];
      s += m1a * m1b;
      s += m2a * m2b;
    }
    sm.A[ra][rb] = s;
  }
  __syncwarp();
  jacobi12(sm, lane);
  // L_6x10 and rho: one control-point pair (ca, cb) per lane
  if (lane < 6) {
    const int ca = lane < 3 ? 0 : lane < 5 ? 1 : 2, cb = lane < 3 ? lane + 1 : lane < 5 ? lane - 1 : 3;
    double dv[4][3];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int k = 0; k < 3; ++k) dv[i][k] = sm.ut[i][3 * ca + k] - sm.ut[i][3 * cb + k];
    auto dot = [&](int x, int y) { return dv[x][0] * dv[y][0] + dv[x][1] * dv[y][1] + dv[x][2] * dv[y][2]; };
    double* l = sm.L[lane];
    l[0] = dot(0, 0); l[1] = 2.0 * dot(0, 1); l[2] = dot(1, 1); l[3] = 2.0 * dot(0, 2); l[4] = 2.0 * dot(1, 2);
    l[5] = dot(2, 2); l[6] = 2.0 * dot(0, 3); l[7] = 2.0 * dot(1, 3); l[8] = 2.0 * dot(2, 3); l[9] = dot(3, 3);
    double r = 0.0;
#pragma unroll
    for (int k = 0; k < 3; ++k) r += (sm.cws[ca][k] - sm.cws[cb][k]) * (sm.cws[ca][k] - sm.cws[cb][k]);
    sm.rho[lane] = r;
  }
  __syncwarp();
  double best = 0.0;
#pragma unroll 1
  for (int N = 1; N <= 3; ++N) {
    double beta[4], Rc[3][3], tc[3];
    betas_approx(sm, N, beta);
    gauss_newton(sm, beta);
    const double err = r_and_t(sm, has, np, pw, c0, a, u, v, f, c, beta, Rc, tc);
    if (N == 1 || err < best) {
      best = err;
      if (lane == 0) {
#pragma unroll
        for (int i = 0; i < 3; ++i) {
          sm.t[i] = tc[i];
#pragma unroll
          for (int j = 0; j < 3; ++j) sm.R[i][j] = Rc[i][j];
        }
      }
    }
  }
  __syncwarp();
}

// OpenCV's RANSACUpdateNumIters(0.99, ep, 5, max_iters)
__device__ __forceinline__ int ransac_update_iters(double ep, int max_iters) {
  ep = fmin(fmax(ep, 0.0), 1.0);
  const double num = log(1.0 - 0.99);
  const double den = 1.0 - pow(1.0 - ep, (double)MODEL_PTS);
  if (den < DBL_MIN) return 0;
  const double ld = log(den);
  return (ld >= 0 || -num >= max_iters * (-ld)) ? max_iters : __double2int_rn(num / ld);
}

__device__ __forceinline__ unsigned rng_next(unsigned long long& state) {
  state = (unsigned long long)(unsigned)state * 4164903690ull + (unsigned)(state >> 32);
  return (unsigned)state;
}

// undistortPoints without distortion: (p - c) * (1/f); OpenCV keeps the input's precision
__device__ __forceinline__ double pix_fp32_normalised(float p, double f, double c) {
  const float x = __double2float_rn(__dmul_rn(__dsub_rn((double)p, c), 1.0 / f));
  return __dadd_rn(__dmul_rn((double)x, f), c);
}
__device__ __forceinline__ double pix_fp64_normalised(float p, double f, double c) {
  return __dadd_rn(__dmul_rn(__dmul_rn(__dsub_rn((double)p, c), 1.0 / f), f), c);
}

// projectPoints of one point (fp64, rounded to fp32) and OpenCV's squared-error test in fp32
__device__ __forceinline__ bool is_inlier(const double (&R)[3][3], const double (&t)[3], float X, float Y, float Z,
                                          float u, float v, double f, double c) {
  double p[3];
#pragma unroll
  for (int i = 0; i < 3; ++i)
    p[i] = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(R[i][0], X), __dmul_rn(R[i][1], Y)), __dmul_rn(R[i][2], Z)), t[i]);
  const double iz = p[2] != 0.0 ? 1.0 / p[2] : 1.0;
  const float pu = __double2float_rn(__dadd_rn(__dmul_rn(__dmul_rn(p[0], iz), f), c));
  const float pv = __double2float_rn(__dadd_rn(__dmul_rn(__dmul_rn(p[1], iz), f), c));
  const float dx = __fsub_rn(u, pu), dy = __fsub_rn(v, pv);
  return __fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)) <= THRESH2;
}

// the EPnP answer and its inlier mask; a non-finite t (EPnP failed) takes the least squares and mask 0, as when
// RANSAC finds no consensus
__device__ __forceinline__ void store_epnp(const PnpSmem& sm, const float* jh, const float* ph, float focal,
                                           float img_size, float* o, int32_t* inl, unsigned joints) {
  if (isfinite(sm.t[0]) && isfinite(sm.t[1]) && isfinite(sm.t[2])) {
    o[0] = (float)sm.t[0]; o[1] = (float)sm.t[1]; o[2] = (float)sm.t[2];
  } else {
    cam_trans_lstsq(jh, ph, focal, img_size, o);
    joints = 0;
  }
  if (inl) *inl = (int32_t)joints;
}

__global__ void __launch_bounds__(PNP_WARPS * 32)
cam_trans_pnp_kernel(const float* __restrict__ j3d, const float* __restrict__ pj2d, const int32_t* __restrict__ n_dev,
                     int n_max, float focal, float img_size, float* __restrict__ out, int32_t* __restrict__ inl_out) {
  __shared__ PnpSmem smem[PNP_WARPS];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int n = n_dev ? min(*n_dev, n_max) : n_max;
  const int h = blockIdx.x * PNP_WARPS + w;
  if (h >= n) return;   // warp-uniform
  PnpSmem& sm = smem[w];
  const float* jh = j3d + (size_t)h * NJ * 3;
  const float* ph = pj2d + (size_t)h * NJ * 2;
  float* o = out + (size_t)h * 3;
  const float half = img_size * 0.5f;

  // usable joints (acr/utils.py:487-502: pixel y > -2, z != -2), compacted in joint order
  float jx = 0.f, jy = 0.f, jz = 0.f, ju = 0.f, jv = 0.f;
  if (lane < NJ) {
    jx = jh[lane * 3 + 0]; jy = jh[lane * 3 + 1]; jz = jh[lane * 3 + 2];
    ju = (ph[lane * 2 + 0] + 1.f) * half; jv = (ph[lane * 2 + 1] + 1.f) * half;
  }
  const bool ok = lane < NJ && (jv > -2.f) && jz != -2.f;
  const unsigned use = __ballot_sync(FULL, ok);
  const int cnt = __popc(use);
  if (ok) {
    const int s = __popc(use & ((1u << lane) - 1));
    sm.S[s][0] = jx; sm.S[s][1] = jy; sm.S[s][2] = jz;
    sm.J[s][0] = ju; sm.J[s][1] = jv;
    sm.idx[s] = lane;
  }
  __syncwarp();
  if (cnt <= 4) {   // < 4: (-1,-1,-1); 4: the least squares in place of OpenCV's P3P
    if (lane == 0) {
      cam_trans_lstsq(jh, ph, focal, img_size, o);
      if (inl_out) inl_out[h] = 0;
    }
    return;
  }
  const double f = focal, c = (double)half;
  if (cnt == MODEL_PTS) {   // OpenCV runs one fp32 EPnP and calls every point an inlier
    const bool has = lane < cnt;
    epnp(sm, lane, cnt, has ? sm.S[lane][0] : 0.f, has ? sm.S[lane][1] : 0.f, has ? sm.S[lane][2] : 0.f,
         has ? pix_fp32_normalised(sm.J[lane][0], f, c) : 0.0, has ? pix_fp32_normalised(sm.J[lane][1], f, c) : 0.0,
         f, c);
    if (lane == 0) store_epnp(sm, jh, ph, focal, img_size, o, inl_out ? inl_out + h : nullptr, use);
    return;
  }
  // this lane's point for the inlier test
  const bool mine = lane < cnt;
  const float X = mine ? sm.S[lane][0] : 0.f, Y = mine ? sm.S[lane][1] : 0.f, Z = mine ? sm.S[lane][2] : 0.f;
  const float u = mine ? sm.J[lane][0] : 0.f, v = mine ? sm.J[lane][1] : 0.f;
  unsigned long long state = ~0ull;
  int niters = RANSAC_ITERS, best = 0;
  unsigned best_mask = 0;
#pragma unroll 1
  for (int it = 0; it < niters; ++it) {
    int sub[MODEL_PTS];
#pragma unroll
    for (int i = 0; i < MODEL_PTS; ++i) {
      int k;
      bool dup;
      do {
        k = (int)(rng_next(state) % (unsigned)cnt);
        dup = false;
#pragma unroll
        for (int j = 0; j < i; ++j) dup |= sub[j] == k;
      } while (dup);
      sub[i] = k;
    }
    const int s = lane == 0 ? sub[0] : lane == 1 ? sub[1] : lane == 2 ? sub[2] : lane == 3 ? sub[3] : sub[4];
    const bool hs = lane < MODEL_PTS;
    epnp(sm, lane, MODEL_PTS, hs ? sm.S[s][0] : 0.f, hs ? sm.S[s][1] : 0.f, hs ? sm.S[s][2] : 0.f,
         hs ? pix_fp32_normalised(sm.J[s][0], f, c) : 0.0, hs ? pix_fp32_normalised(sm.J[s][1], f, c) : 0.0, f, c);
    double R[3][3], t[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      t[i] = sm.t[i];
#pragma unroll
      for (int j = 0; j < 3; ++j) R[i][j] = sm.R[i][j];
    }
    const unsigned inl = __ballot_sync(FULL, mine && is_inlier(R, t, X, Y, Z, u, v, f, c));
    const int good = __popc(inl);
    if (good > max(best, MODEL_PTS - 1)) {
      best = good;
      best_mask = inl;
      niters = ransac_update_iters((double)(cnt - good) / cnt, niters);
    }
  }
  if (best == 0) {   // no consensus: the reference's except-branch, least squares on the usable joints
    if (lane == 0) {
      cam_trans_lstsq(jh, ph, focal, img_size, o);
      if (inl_out) inl_out[h] = 0;
    }
    return;
  }
  // final fit: EPnP on the inliers in fp64; lane l takes the l-th inlier (the source lane is the one whose inlier
  // prefix count is l)
  const bool inl_me = (best_mask >> lane) & 1u;
  const int rank = __popc(best_mask & ((1u << lane) - 1));
  int sl = 0;
#pragma unroll 1
  for (int k = 0; k < cnt; ++k) {
    const int rk = __shfl_sync(FULL, inl_me ? rank : -1, k);
    if (rk == lane) sl = k;
  }
  const float fX = __shfl_sync(FULL, X, sl), fY = __shfl_sync(FULL, Y, sl), fZ = __shfl_sync(FULL, Z, sl);
  const float fu = __shfl_sync(FULL, u, sl), fv = __shfl_sync(FULL, v, sl);
  const bool hf = lane < best;
  epnp(sm, lane, best, hf ? fX : 0.f, hf ? fY : 0.f, hf ? fZ : 0.f, hf ? pix_fp64_normalised(fu, f, c) : 0.0,
       hf ? pix_fp64_normalised(fv, f, c) : 0.0, f, c);
  const unsigned joints = __reduce_or_sync(FULL, (mine && inl_me) ? 1u << sm.idx[lane] : 0u);
  if (lane == 0) store_epnp(sm, jh, ph, focal, img_size, o, inl_out ? inl_out + h : nullptr, joints);
}

}  // namespace

extern "C" int acr_b200_cam_trans_pnp(const float* j3d, const float* pj2d, const int32_t* n_dev, int n_max,
                                      float focal_length, float img_size, float* cam_trans, int32_t* inlier_mask,
                                      void* stream) {
  ACR_CHECK_ARG(n_max >= 0 && (n_max == 0 || (j3d && pj2d && cam_trans)), "cam_trans_pnp: bad arguments");
  if (n_max == 0) return ACR_B200_OK;
  cam_trans_pnp_kernel<<<ceil_div(n_max, PNP_WARPS), PNP_WARPS * 32, 0, (cudaStream_t)stream>>>(
      j3d, pj2d, n_dev, n_max, focal_length, img_size, cam_trans, inlier_mask);
  ACR_CHECK_LAUNCH();
  return ACR_B200_OK;
}

}  // namespace acr
