"""numpy float64 restatement of the reference's camera translation: estimate_translation (acr/utils.py:474-519)
around cv2.solvePnPRansac(..., flags=SOLVEPNP_EPNP, reprojectionError=20, iterationsCount=100) (:414-428), with
its least-squares fall-back (:430-472).  Test infrastructure only: the product path is csrc/pnp.cu.

What it restates (checked against cv2 4.13 by tests/test_cpu_pnp.py):
  * RANSAC: cv::RNG seeded with all ones (next() = (uint32)state * 4164903690 + (state >> 32), uniform(0, n) =
    next() % n); subsets of 5 distinct indices, a repeated index is redrawn; the loop runs while iter < niters,
    niters = 100 at first; a model replaces the best one iff its inlier count > max(best, 4), and then
    niters = RANSACUpdateNumIters(0.99, outlier ratio, 5, niters), which is 0 once every point is an inlier.
  * Inlier test: the hypothesis projects every point (float64, x * (1/z), then rounded to float32), and a
    point is an inlier iff (dx^2 + dy^2) <= 400 in float32 arithmetic.
  * Hypotheses are EPnP on the 5 float32 points, the image points normalised ((u - c) * (1/f)) and rounded to
    float32; the answer is EPnP on all inliers in float64.  With exactly 5 points: one float32 EPnP, no RANSAC.
  * EPnP (Lepetit, Moreno-Noguer, Fua 2009) as OpenCV states it: centroid + PCA control points, barycentric
    alphas, the 2n x 12 M and the four smallest singular vectors of M^T M, L_6x10 / rho, the beta approximations
    N = 1, 2, 3 each refined by 5 Gauss-Newton steps (Householder QR), R, t from a 3x3 SVD (det < 0: negate the
    last row) with the depth sign check, smallest mean reprojection error wins.  The SVDs are one-sided
    (Hestenes) Jacobi, and the left singular vectors are the normalised rotated columns, as in OpenCV.
  * The hypothesis' rotation is used as a matrix: OpenCV's Rodrigues round trip (matrix -> vector -> matrix)
    moves it by an ulp, which decides an inlier only when a squared error lands on 400 to float32 precision.
"""
from __future__ import annotations

import numpy as np

from . import mano_ref

F = np.float32
THRESH2 = F(400.0)          # reprojectionError = 20 px, squared in float32
ITERS, CONF, MODEL_PTS = 100, 0.99, 5

# status codes (one per hand)
ST_INVALID, ST_LSTSQ_4, ST_LSTSQ_FAIL, ST_EPNP = 0, 1, 2, 3


class CvRNG:
    """cv::RNG: multiply-with-carry, 64-bit state."""

    def __init__(self, state=0xFFFFFFFFFFFFFFFF):
        self.state = state

    def next(self) -> int:
        s = self.state
        self.state = ((s & 0xFFFFFFFF) * 4164903690 + (s >> 32)) & 0xFFFFFFFFFFFFFFFF
        return self.state & 0xFFFFFFFF

    def uniform(self, n: int) -> int:
        return self.next() % n


def jacobi_svd(A, dtype=np.float64, sweeps=None):
    """One-sided Jacobi SVD of an (m, n) matrix, m >= n, OpenCV's ordering: returns (w descending, Ut, Vt) where the
    rows of Ut are the left singular vectors (rotated columns of A, normalised; zero for w == 0) and the rows of Vt
    the right ones.  Every operation is in ``dtype``; the rotation threshold is 10 eps of ``dtype``, so a long double
    run converges further than a float64 one.  ``sweeps`` caps the number of sweeps (default max(m, 30))."""
    At = np.array(A, dtype).T.copy()
    n = At.shape[0]
    m = At.shape[1]
    eps = np.finfo(dtype).eps * 10
    W = np.array([np.dot(At[i], At[i]) for i in range(n)], dtype)
    Vt = np.eye(n, dtype=dtype)
    for _ in range(max(m, 30) if sweeps is None else sweeps):
        changed = False
        for i in range(n - 1):
            for j in range(i + 1, n):
                a, b = W[i], W[j]
                p = np.dot(At[i], At[j])
                if abs(p) <= eps * np.sqrt(a * b):
                    continue
                p *= 2
                beta = a - b
                gamma = np.hypot(p, beta)
                if beta < 0:
                    s = np.sqrt((gamma - beta) * 0.5 / gamma)
                    c = p / (gamma * s * 2)
                else:
                    c = np.sqrt((gamma + beta) / (gamma * 2))
                    s = p / (gamma * c * 2)
                t0 = c * At[i] + s * At[j]
                t1 = -s * At[i] + c * At[j]
                At[i], At[j] = t0, t1
                W[i], W[j] = np.dot(t0, t0), np.dot(t1, t1)
                v0 = c * Vt[i] + s * Vt[j]
                v1 = -s * Vt[i] + c * Vt[j]
                Vt[i], Vt[j] = v0, v1
                changed = True
        if not changed:
            break
    W = np.sqrt(np.einsum("ij,ij->i", At, At))
    order = np.argsort(-W, kind="stable")
    W, At, Vt = W[order], At[order], Vt[order]
    Ut = At / np.where(W > 0, W, 1.0)[:, None]
    return W, Ut, Vt


def svd_solve(A, b):
    """Minimum-norm least squares through jacobi_svd, OpenCV's cvSolve(CV_SVD): singular values at or below
    10 eps * w_max (eps of A's dtype) count as zero."""
    w, Ut, Vt = jacobi_svd(A, A.dtype)
    keep = w > np.finfo(A.dtype).eps * 10 * w[0]
    return Vt[keep].T @ ((Ut[keep] @ b) / w[keep])


def _qr_solve(A, b):
    """EPnP's Householder least squares (6 x nc); None when A is singular (the caller keeps its step)."""
    A = A.copy()
    b = b.copy()
    nr, nc = A.shape
    A1, A2 = np.zeros(nc, A.dtype), np.zeros(nc, A.dtype)
    for k in range(nc):
        eta = np.abs(A[k:nr - 1, k]).max()           # OpenCV's scan stops one row short
        if eta == 0:
            return None
        A[k:, k] *= 1.0 / eta
        sigma = np.sqrt(np.sum(A[k:, k] ** 2))
        if A[k, k] < 0:
            sigma = -sigma
        A[k, k] += sigma
        A1[k] = sigma * A[k, k]
        A2[k] = -eta * sigma
        for j in range(k + 1, nc):
            tau = np.dot(A[k:, k], A[k:, j]) / A1[k]
            A[k:, j] -= tau * A[k:, k]
    for j in range(nc):
        tau = np.dot(A[j:, j], b[j:]) / A1[j]
        b[j:] -= tau * A[j:, j]
    x = np.zeros(nc, A.dtype)
    x[nc - 1] = b[nc - 1] / A2[nc - 1]
    for i in range(nc - 2, -1, -1):
        x[i] = (b[i] - np.dot(A[i, i + 1:], x[i + 1:])) / A2[i]
    return x


_PAIRS = [(0, 1), (0, 2), (0, 3), (1, 2), (1, 3), (2, 3)]
DEGENERATE = 10 * np.finfo(np.float64).eps   # smallest / largest PCA eigenvalue at or below this: no control points


def _det3(R):
    return (R[0, 0] * R[1, 1] * R[2, 2] + R[0, 1] * R[1, 2] * R[2, 0] + R[0, 2] * R[1, 0] * R[2, 1]
            - R[0, 2] * R[1, 1] * R[2, 0] - R[0, 1] * R[1, 0] * R[2, 2] - R[0, 0] * R[1, 2] * R[2, 1])


def _barycentric(d, cws):
    """alphas 1..3 of the centred points d: C^-1 d with C = (cws[1:] - cws[0])^T.  C^-1 is LAPACK's float64 inverse
    (which the golden pins: on a 5-point hand the null-space basis, and so t, follows its round-off), refined by one
    Newton step X + X (I - C X) when ``d`` is wider than float64 (numpy.linalg has no long double); the step squares
    the relative error, so the result is accurate to the wider type.  The caller has ruled out a singular C."""
    C = (cws[1:] - cws[0]).T
    Ci = np.linalg.inv(C.astype(np.float64)).astype(d.dtype)
    if np.finfo(d.dtype).eps < np.finfo(np.float64).eps:
        Ci = Ci + Ci @ (np.eye(3, dtype=d.dtype) - C @ Ci)
    return d @ Ci.T


def epnp(pw, uv, fu, fv, uc, vc, dtype=np.float64, basis_angle=0.0, all_sols=False):
    """EPnP on world points pw (n,3) and pixel points uv (n,2) in ``dtype`` -> (R, t, mean reprojection error), or
    with ``all_sols`` the list of the three (R, t, error) of the beta approximations N = 1, 2, 3 and the index of
    the one chosen.

    ``basis_angle`` rotates the two smallest singular vectors of M^T M within their span before L is built: a
    5-point M has a two-dimensional null space, and which basis of it the SVD returns is decided by round-off.

    When the smallest PCA eigenvalue is at or below DEGENERATE times the largest (planar or
    collinear points) the alphas do not exist: R and t are NaN, the error inf.  OpenCV inverts C by SVD and
    carries on in a null space of four or more dimensions, where its answer is decided by round-off; this
    statement, like csrc/pnp.cu, reports the failure instead."""
    pw = np.asarray(pw, dtype)
    uv = np.asarray(uv, dtype)
    n = pw.shape[0]
    c0 = np.cumsum(pw, 0)[-1] / n
    d = pw - c0
    dc, uct, _ = jacobi_svd(d.T @ d, dtype)
    if not dc[2] > DEGENERATE * dc[0]:
        nan = (np.full((3, 3), np.nan, dtype), np.full(3, np.nan, dtype), np.inf)
        return ([nan] * 3, 0) if all_sols else nan
    cws = np.zeros((4, 3), dtype)
    cws[0] = c0
    k = np.sqrt(dc / n)
    for i in range(1, 4):
        cws[i] = c0 + k[i - 1] * uct[i - 1]
    alphas = np.zeros((n, 4), dtype)
    alphas[:, 1:] = _barycentric(d, cws)
    alphas[:, 0] = 1 - alphas[:, 1] - alphas[:, 2] - alphas[:, 3]
    M = np.zeros((2 * n, 12), dtype)
    M[0::2, 0::3] = alphas * fu
    M[0::2, 2::3] = alphas * (uc - uv[:, 0:1])
    M[1::2, 1::3] = alphas * fv
    M[1::2, 2::3] = alphas * (vc - uv[:, 1:2])
    _, ut, _ = jacobi_svd(M.T @ M, dtype)
    v = [ut[11 - i].reshape(4, 3) for i in range(4)]
    if basis_angle:
        co, si = np.cos(dtype(basis_angle)), np.sin(dtype(basis_angle))
        v[0], v[1] = co * v[0] + si * v[1], co * v[1] - si * v[0]
    dv = [np.array([v[i][a] - v[i][b] for a, b in _PAIRS]) for i in range(4)]
    dot = lambda x, y: np.sum(x * y, 1)
    L = np.stack([dot(dv[0], dv[0]), 2 * dot(dv[0], dv[1]), dot(dv[1], dv[1]), 2 * dot(dv[0], dv[2]),
                  2 * dot(dv[1], dv[2]), dot(dv[2], dv[2]), 2 * dot(dv[0], dv[3]), 2 * dot(dv[1], dv[3]),
                  2 * dot(dv[2], dv[3]), dot(dv[3], dv[3])], 1)
    rho = np.array([np.sum((cws[a] - cws[b]) ** 2) for a, b in _PAIRS])
    lsq = lambda A: svd_solve(A, rho)

    def approx1():
        b = lsq(L[:, [0, 1, 3, 6]])
        if b[0] < 0:
            b0 = np.sqrt(-b[0])
            return np.array([b0, -b[1] / b0, -b[2] / b0, -b[3] / b0])
        b0 = np.sqrt(b[0])
        return np.array([b0, b[1] / b0, b[2] / b0, b[3] / b0])

    def approx23(cols):
        b = lsq(L[:, cols])
        zero = dtype(0)
        if b[0] < 0:
            b0, b1 = np.sqrt(-b[0]), (np.sqrt(-b[2]) if b[2] < 0 else zero)
        else:
            b0, b1 = np.sqrt(b[0]), (np.sqrt(b[2]) if b[2] > 0 else zero)
        if b[1] < 0:
            b0 = -b0
        return np.array([b0, b1, b[3] / b0 if len(cols) == 5 else zero, zero])

    def gauss_newton(beta):
        x = np.zeros(4, dtype)
        for _ in range(5):
            B = beta
            A = np.stack([2 * L[:, 0] * B[0] + L[:, 1] * B[1] + L[:, 3] * B[2] + L[:, 6] * B[3],
                          L[:, 1] * B[0] + 2 * L[:, 2] * B[1] + L[:, 4] * B[2] + L[:, 7] * B[3],
                          L[:, 3] * B[0] + L[:, 4] * B[1] + 2 * L[:, 5] * B[2] + L[:, 8] * B[3],
                          L[:, 6] * B[0] + L[:, 7] * B[1] + L[:, 8] * B[2] + 2 * L[:, 9] * B[3]], 1)
            q = (L[:, 0] * B[0] * B[0] + L[:, 1] * B[0] * B[1] + L[:, 2] * B[1] * B[1] + L[:, 3] * B[0] * B[2]
                 + L[:, 4] * B[1] * B[2] + L[:, 5] * B[2] * B[2] + L[:, 6] * B[0] * B[3] + L[:, 7] * B[1] * B[3]
                 + L[:, 8] * B[2] * B[3] + L[:, 9] * B[3] * B[3])
            xn = _qr_solve(A, rho - q)
            if xn is not None:
                x = xn
            beta = beta + x
        return beta

    def r_and_t(beta):
        ccs = sum(beta[i] * v[i] for i in range(4))
        pcs = alphas @ ccs
        if pcs[0, 2] < 0:
            pcs = -pcs
        pc0 = np.cumsum(pcs, 0)[-1] / n
        pw0 = c0
        abt = (pcs - pc0).T @ (pw - pw0)
        _, Ut, Vt = jacobi_svd(abt, dtype)
        R = Ut.T @ Vt
        if _det3(R) < 0:
            R[2] = -R[2]
        t = pc0 - R @ pw0
        Xc = pw @ R.T + t
        ue = uc + fu * Xc[:, 0] * (1 / Xc[:, 2])
        ve = vc + fv * Xc[:, 1] * (1 / Xc[:, 2])
        err = np.mean(np.sqrt((uv[:, 0] - ue) ** 2 + (uv[:, 1] - ve) ** 2))
        return R, t, err

    sols = [r_and_t(gauss_newton(approx1())), r_and_t(gauss_newton(approx23([0, 1, 2]))),
            r_and_t(gauss_newton(approx23([0, 1, 2, 3, 4])))]
    best = 0
    if sols[1][2] < sols[0][2]:
        best = 1
    if sols[2][2] < sols[best][2]:
        best = 2
    return (sols, best) if all_sols else sols[best]


def _update_num_iters(p, ep, model_points, max_iters):
    num = max(1.0 - p, np.finfo(np.float64).tiny)
    denom = 1.0 - (1.0 - ep) ** model_points
    if denom < np.finfo(np.float64).tiny:
        return 0
    num, denom = np.log(num), np.log(denom)
    return max_iters if (denom >= 0 or -num >= max_iters * (-denom)) else int(round(num / denom))


def _sq_errors(S, J, R, t, f, c):
    """float32 squared reprojection error of every point under (R, t); NaN for a failed hypothesis"""
    X, Y, Z = (S[:, k].astype(np.float64) for k in range(3))
    R, t = np.asarray(R, np.float64), np.asarray(t, np.float64)
    x = R[0, 0] * X + R[0, 1] * Y + R[0, 2] * Z + t[0]
    y = R[1, 0] * X + R[1, 1] * Y + R[1, 2] * Z + t[1]
    z = R[2, 0] * X + R[2, 1] * Y + R[2, 2] * Z + t[2]
    z = np.where(z != 0, 1.0 / np.where(z != 0, z, 1.0), 1.0)
    u = (x * z * f + c).astype(F)
    w = (y * z * f + c).astype(F)
    dx, dy = J[:, 0] - u, J[:, 1] - w
    return dx * dx + dy * dy


def normalised(J, f, c, fp32=False):
    """undistortPoints without distortion, back in pixels: ((p - c) * (1/f)) * f + c in float64, with the
    normalised point rounded to float32 first when ``fp32`` (OpenCV keeps the input's precision: the hypotheses
    see float32 points, the final fit float64 ones)."""
    x = (np.asarray(J, F).astype(np.float64) - c) * (1.0 / f)
    return (x.astype(F).astype(np.float64) if fp32 else x) * f + c


def final_fit(S, uv, f, c, dtype=np.float64, **kw):
    """EPnP of float32 world points S on already normalised pixels uv (see ``normalised``), in ``dtype``"""
    return epnp(np.asarray(S, F).astype(dtype), np.asarray(uv, np.float64).astype(dtype), f, f, c, c, dtype, **kw)


def solve_pnp_ransac(S, J, f=1265.0, c=256.0, trace=False):
    """cv2.solvePnPRansac(S, J, K, None, flags=EPNP, reprojectionError=20, iterationsCount=100) for float32
    S (n,3), J (n,2), n >= 5, K = [[f,0,c],[0,f,c],[0,0,1]] -> (t (3,) float64 or None, inlier bool mask (n,)).
    None also where EPnP fails (degenerate control points or a non-finite t; see ``epnp``).
    With ``trace`` a third value: {"hyps": [(subset, inlier count, float32 squared error of every point)],
    "iters": hypotheses evaluated, "changes": how often the best hypothesis was replaced}."""
    S = np.asarray(S, F)
    J = np.asarray(J, F)
    n = S.shape[0]
    tr = {"hyps": [], "iters": 0, "changes": 0}
    ret = (lambda t, m: (t, m, tr)) if trace else (lambda t, m: (t, m))
    if n == MODEL_PTS:
        t = epnp(S, normalised(J, f, c, fp32=True), f, f, c, c)[1]
        return ret(t, np.ones(n, bool)) if np.isfinite(t).all() else ret(None, np.zeros(n, bool))
    norm32 = normalised(J, f, c, fp32=True)
    rng = CvRNG()
    niters, best, best_mask = ITERS, 0, None
    it = 0
    while it < niters:
        idx = []
        for _ in range(MODEL_PTS):
            k = rng.uniform(n)
            while k in idx:
                k = rng.uniform(n)
            idx.append(k)
        R, t, _ = epnp(S[idx], norm32[idx], f, f, c, c)
        err2 = _sq_errors(S, J, R, t, f, c)
        mask = err2 <= THRESH2
        good = int(mask.sum())
        if trace:
            tr["hyps"].append((idx, good, err2))
        if good > max(best, MODEL_PTS - 1):
            best, best_mask = good, mask
            tr["changes"] += 1
            niters = _update_num_iters(CONF, (n - good) / n, MODEL_PTS, niters)
        it += 1
    tr["iters"] = it
    if best == 0:
        return ret(None, np.zeros(n, bool))
    t = final_fit(S[best_mask], normalised(J[best_mask], f, c), f, c)[1]
    if not np.isfinite(t).all():
        return ret(None, np.zeros(n, bool))
    return ret(t, best_mask)


def cam_trans_pnp(j3d, pj2d, focal_length=1265.0, img_size=512.0):
    """estimate_translation(j3d, (pj2d+1)*img_size/2, focal_length) of the reference, per hand ->
    (cam_trans (n,3) float64 (the reference rounds it to float32), inlier bitmask (n,) int32 over the 21 joints, status (n,) int32: ST_*).
    Fewer than 4 usable joints -> (-1,-1,-1); exactly 4 -> least squares (OpenCV would switch to P3P); no
    RANSAC consensus, or an EPnP that fails (planar or collinear usable joints) -> least squares on the usable
    joints, the reference's except-branch, with status ST_LSTSQ_FAIL."""
    j3d = np.asarray(j3d, F)
    j2d = ((np.asarray(pj2d, F) + 1) * F(img_size / 2)).astype(F)
    n = j3d.shape[0]
    out = np.zeros((n, 3))
    masks = np.zeros(n, np.int32)
    status = np.zeros(n, np.int32)
    lsq = mano_ref.cam_trans_lstsq(j3d, pj2d, focal_length, img_size)
    for i in range(n):
        use = (j2d[i, :, 1] > -2.0) & (j3d[i, :, 2] != -2.0)
        cnt = int(use.sum())
        if cnt < 4:
            out[i], status[i] = -1, ST_INVALID
            continue
        if cnt == 4:
            out[i], status[i] = lsq[i], ST_LSTSQ_4
            continue
        t, inl = solve_pnp_ransac(j3d[i][use], j2d[i][use], focal_length, img_size / 2)
        if t is None:
            out[i], status[i] = lsq[i], ST_LSTSQ_FAIL
            continue
        out[i], status[i] = t, ST_EPNP
        joints = np.nonzero(use)[0][inl]
        masks[i] = int(np.sum(1 << joints))
    return out, masks, status
