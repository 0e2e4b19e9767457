"""ORACLE (test infrastructure, never on the product path).

CPU/numpy restatement of the reference's rotation chain.  Pinned against the
reference itself through tests/golden/rot_golden.npz (made by
tests/golden/make_golden.py importing /root/reference unmodified).

Reference functions restated (all in /root/reference/):
  rot6d_to_rotmat               acr/utils.py:362-376
  rotation_matrix_to_quaternion acr/utils.py:826-906
  quaternion_to_angle_axis      acr/utils.py:773-823
  rotation_matrix_to_angle_axis acr/utils.py:334-360   (NaN -> 0)
  rot6D_to_angular              acr/utils.py:378-382
  batch_rodrigues / quat2mat    mano/manolayer.py:423-434 / :396-421
All arithmetic is float32, like the reference (MANO/parse always run in fp32).
"""
import numpy as np

F = np.float32


def _dtype(dtype):
    """The type a function computes in: its ``dtype`` argument, or the module's F (float32, the reference's)."""
    return globals()["F"] if dtype is None else dtype


def _normalize(v, eps):
    # torch.nn.functional.normalize: v / max(||v||, eps)
    F = v.dtype.type
    n = np.sqrt((v * v).sum(-1, keepdims=True, dtype=F))
    return v / np.maximum(n, F(eps))


def rot6d_to_rotmat(x, dtype=None):
    """(M,6) -> (M,3,3); the 6 numbers are read as a row-major (3,2) matrix whose two
    columns are the raw basis vectors (acr/utils.py:363 ``x.view(-1,3,2)``).
    ``dtype`` (here and below): the type of every operation, float32 like the reference or float64."""
    F = _dtype(dtype)
    x = np.asarray(x, F).reshape(-1, 3, 2)
    a1, a2 = x[:, :, 0], x[:, :, 1]
    b1 = _normalize(a1, 1e-6)
    d = (b1 * a2).sum(-1, keepdims=True, dtype=F)
    b2 = _normalize(a2 - d * b1, 1e-6)
    b3 = np.cross(b1, b2).astype(F)
    return np.stack([b1, b2, b3], axis=-1)  # columns b1,b2,b3


def rotmat_to_quaternion(R, eps=1e-6, dtype=None):
    """(M,3,3) -> (M,4) wxyz; 4-case selection evaluated on the TRANSPOSED matrix
    (acr/utils.py:862 ``rmat_t = transpose(rotation_matrix)``)."""
    F = _dtype(dtype)
    R = np.asarray(R, F)
    t = np.transpose(R, (0, 2, 1))
    m = lambda i, j: t[:, i, j]
    mask_d2 = m(2, 2) < F(eps)
    mask_d0_d1 = m(0, 0) > m(1, 1)
    mask_d0_nd1 = m(0, 0) < -m(1, 1)
    t0 = 1 + m(0, 0) - m(1, 1) - m(2, 2)
    q0 = np.stack([m(1, 2) - m(2, 1), t0, m(0, 1) + m(1, 0), m(2, 0) + m(0, 2)], -1)
    t1 = 1 - m(0, 0) + m(1, 1) - m(2, 2)
    q1 = np.stack([m(2, 0) - m(0, 2), m(0, 1) + m(1, 0), t1, m(1, 2) + m(2, 1)], -1)
    t2 = 1 - m(0, 0) - m(1, 1) + m(2, 2)
    q2 = np.stack([m(0, 1) - m(1, 0), m(2, 0) + m(0, 2), m(1, 2) + m(2, 1), t2], -1)
    t3 = 1 + m(0, 0) + m(1, 1) + m(2, 2)
    q3 = np.stack([t3, m(1, 2) - m(2, 1), m(2, 0) - m(0, 2), m(0, 1) - m(1, 0)], -1)
    c0 = (mask_d2 & mask_d0_d1)[:, None]
    c1 = (mask_d2 & ~mask_d0_d1)[:, None]
    c2 = (~mask_d2 & mask_d0_nd1)[:, None]
    c3 = (~mask_d2 & ~mask_d0_nd1)[:, None]
    q = np.where(c0, q0, np.where(c1, q1, np.where(c2, q2, q3))).astype(F)
    tt = np.where(c0[:, 0], t0, np.where(c1[:, 0], t1, np.where(c2[:, 0], t2, t3))).astype(F)
    with np.errstate(invalid="ignore", divide="ignore"):
        q = q / np.sqrt(tt)[:, None] * F(0.5)
    return q.astype(F)


def quaternion_to_angle_axis(q, dtype=None):
    F = _dtype(dtype)
    q = np.asarray(q, F)
    q1, q2, q3 = q[:, 1], q[:, 2], q[:, 3]
    s2 = q1 * q1 + q2 * q2 + q3 * q3
    s = np.sqrt(s2)
    c = q[:, 0]
    two_theta = F(2.0) * np.where(c < 0, np.arctan2(-s, -c), np.arctan2(s, c)).astype(F)
    with np.errstate(invalid="ignore", divide="ignore"):
        k = np.where(s2 > 0, two_theta / s, F(2.0)).astype(F)
    return np.stack([q1 * k, q2 * k, q3 * k], -1).astype(F)


def rotmat_to_angle_axis(R, dtype=None):
    aa = quaternion_to_angle_axis(rotmat_to_quaternion(R, dtype=dtype), dtype)
    aa[np.isnan(aa)] = 0.0
    return aa


def rot6d_to_angular(rot6d):
    """(N, 6*J) -> (N, 3*J)   (acr/utils.py:378-382)."""
    rot6d = np.asarray(rot6d, F)
    n = rot6d.shape[0]
    return rotmat_to_angle_axis(rot6d_to_rotmat(rot6d.reshape(-1, 6))).reshape(n, -1)


def batch_rodrigues(aa, dtype=None):
    """(M,3) -> (M,9) row-major rotation, via the half-angle quaternion with the
    reference's 1e-8 offset inside the norm (mano/manolayer.py:425).  ``dtype`` is the type of every
    operation: float32 is the reference's, float64 the high-precision statement the kernels are bounded against."""
    F = _dtype(dtype)
    aa = np.asarray(aa, F)
    ang = np.sqrt(((aa + F(1e-8)) ** 2).sum(-1, keepdims=True, dtype=F))
    axis = aa / ang
    h = ang * F(0.5)
    q = np.concatenate([np.cos(h), np.sin(h) * axis], -1).astype(F)
    q = q / np.sqrt((q * q).sum(-1, keepdims=True, dtype=F))
    w, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    w2, x2, y2, z2 = w * w, x * x, y * y, z * z
    wx, wy, wz, xy, xz, yz = w * x, w * y, w * z, x * y, x * z, y * z
    return np.stack([w2 + x2 - y2 - z2, 2 * xy - 2 * wz, 2 * wy + 2 * xz,
                     2 * wz + 2 * xy, w2 - x2 + y2 - z2, 2 * yz - 2 * wx,
                     2 * xz - 2 * wy, 2 * wx + 2 * yz, w2 - x2 - y2 + z2], -1).astype(F)


# ---------------------------------------------------------------------------------------------------------
# Temporal smoothing (acr/utils.py:1466-1527, acr/main.py:69-83)
# ---------------------------------------------------------------------------------------------------------
class OneEuroBank:
    """numpy restatement of create_OneEuroFilter + smooth_results for one hand type: OneEuroFilter(c,0.7) on the
    hand pose, OneEuroFilter(0.6,0.7) on betas, OneEuroFilter(c,0.7) on the root rotation MATRIX (float32)."""

    def __init__(self, smooth_coeff=4.0, freq=30.0):
        self.c, self.freq = F(smooth_coeff), F(freq)
        self.prev = None       # (raw, filtered, filtered_dx) of the 64-vector [pose45 | betas10 | R9]

    def _alpha(self, cutoff):
        te = F(1.0) / self.freq
        tau = F(1.0) / (F(2 * np.pi) * cutoff)
        return (F(1.0) / (F(1.0) + tau / te)).astype(F)

    def process(self, pose48, betas10):
        pose48, betas10 = np.asarray(pose48, F), np.asarray(betas10, F)
        R = batch_rodrigues(pose48[None, :3])[0]
        x = np.concatenate([pose48[3:], betas10, R]).astype(F)
        minc = np.concatenate([np.full(45, self.c, F), np.full(10, 0.6, F), np.full(9, self.c, F)])
        if self.prev is None:
            xh, edx = x.copy(), np.zeros_like(x)
        else:
            raw, filt, fdx = self.prev
            dx = (x - raw) * self.freq
            ad = self._alpha(F(1.0))
            edx = (ad * dx + (F(1.0) - ad) * fdx).astype(F)
            a = self._alpha(minc + F(0.7) * np.abs(edx))
            xh = (a * x + (F(1.0) - a) * filt).astype(F)
        self.prev = (x, xh, edx)
        root = rotmat_to_angle_axis(xh[55:].reshape(1, 3, 3))[0]
        return np.concatenate([root, xh[:45]]).astype(F), xh[45:55].astype(F)
