"""float64 statements of the MANO layer kernels of csrc/mano.cu -- the layer forward (axis angles or matrices through
the SO(3) projection, with or without root_palm), the backward (vertex + chain kernels, Rodrigues / projection VJP) and
the JVP (full and joints-only forms) -- with a per-element bound |got - exp| <= b on every output of the fp32 kernels.

The bound is derived mechanically.  Every quantity is an ``EV``: its value in the statement's dtype and a float64
bound on the fp32 kernel's error in it.  The kernel is restated stage by stage in its own operation order, and each
operation propagates the bound by the rules

    sum / difference     e_a + e_b + U |a + b|                  U = 2**-24, one fp32 rounding
    product              |a| e_b + |b| e_a + e_a e_b + U |ab|   (exact for a power of two)
    quotient             (e_a + |a / b| e_b) / |b| + U |a / b|
    square root          e / (2 sqrt a) + U sqrt a              (IEEE: no -use_fast_math in build.py)
    fmaf (explicit)      |a| e_b + |b| e_a + e_a e_b + e_c + U |ab + c|
    sequential chain     sum of the terms' bounds + U sum_i |s_i|   (s_i its partial sums: ``partial_sums``)

The long sums -- 145 blend rows, 16 skinning weights, <= 128 vertices per chunk of the backward's reductions -- are
chains of explicit fmaf (or adds) and are charged U per partial sum, which stays rigorous and loses far less to
cancellation than k U sum |terms|.  Elsewhere nvcc may contract a * b + c (build.py has no -fmad=false); counting
the product and the sum separately bounds either evaluation.  Intrinsics enter at the CUDA C Programming Guide's
maximum ulp errors (1 ulp <= 2 U relative): sincosf 2 ulp (the forward's rebuild_transforms<false>), sincospif 1 ulp
with its argument's product by the fp32 constant 0.159154943f (rebuild_transforms<true>, rodrigues_vjp / _jvp).  The
fp64 SO(3) projection enters as one rounding to fp32 plus an fp64 term with one assumed constant
(``so3_conditioning``).  Magnitudes are those of the float64 run; no count is fitted to a measurement.

With ``dtype=torch.float32`` the same statements are an fp32 implementation in the kernels' order of operations
(explicit fmaf fused, other products and sums rounded separately), whose error the float64 run's bounds must hold:
tests/test_cpu_mano_layer_bounds.py checks that, and pins the float64 values to the autograd / torch.func
restatements of tests/mano_torch_ref.py, mano_rotmat_ref.py and mano_jvp_ref.py.
"""
import math

import numpy as np
import torch

from oracle.mano_ref import JOINT_REORDER, LEVELS, TIPS
from tests.mano_torch_ref import rodrigues as rodrigues64

U = 2.0 ** -24
EPS64 = 2.0 ** -53
F32, F64 = torch.float32, torch.float64
NV, NVP, NK, VPB, NCHUNK = 778, 784, 145, 128, 7
PALM = (95, 22)                                  # PALM_VA, PALM_VB
CHAIN = [(LEVELS[lev][f], 0 if lev == 0 else LEVELS[lev - 1][f]) for lev in range(3) for f in range(5)]
JOINT_INV = [JOINT_REORDER.index(s) for s in range(21)]   # c_joint_inv: out-joint index of source joint s
C_2PI = float(np.float32(0.159154943))          # the kernel's fp32 1 / (2 pi)
C_2PI_REL = abs(C_2PI * 2 * math.pi - 1.0)      # its relative error, 0.68 U
OFF8 = float(np.float32(1e-8))                  # the kernel's fp32 1e-8 (Rodrigues' angle offset)
ROT_CUT = 1e-3                                  # see so3_project
FP64_TERM = 64                                  # an assumed first-order constant, see so3_conditioning


# --------------------------------------------------------------------------------------------- value with a bound
class EV:
    """A value of the fp32 computation (in the statement's dtype) and a float64 bound on its error."""
    __slots__ = ("v", "e")

    def __init__(self, v, e=None):
        self.v = v
        self.e = torch.zeros(v.shape, dtype=F64) if e is None else e.expand(v.shape) if e.dim() < v.dim() else e

    @property
    def a(self):
        return self.v.abs().to(F64)

    def __getitem__(self, i):
        return EV(self.v[i], self.e.expand(self.v.shape)[i])

    def reshape(self, *s):
        return EV(self.v.reshape(*s), self.e.expand(self.v.shape).reshape(*s))

    def _c(self, o):
        if isinstance(o, EV):
            return o
        return EV(torch.as_tensor(o, dtype=self.v.dtype), torch.zeros((), dtype=F64))

    def __neg__(self):
        return EV(-self.v, self.e)

    def __add__(self, o):
        o = self._c(o)
        r = self.v + o.v
        return EV(r, self.e + o.e + U * r.abs().to(F64))

    __radd__ = __add__

    def __sub__(self, o):
        o = self._c(o)
        r = self.v - o.v
        return EV(r, self.e + o.e + U * r.abs().to(F64))

    def __rsub__(self, o):
        return self._c(o) - self

    def __mul__(self, o):
        if isinstance(o, (int, float)) and o != 0 and math.frexp(abs(o))[0] == 0.5:   # a power of two: exact
            return EV(self.v * o, self.e * abs(o))
        o = self._c(o)
        r = self.v * o.v
        return EV(r, self.a * o.e + o.a * self.e + self.e * o.e + U * r.abs().to(F64))

    __rmul__ = __mul__

    def __truediv__(self, o):
        o = self._c(o)
        r = self.v / o.v
        ar = r.abs().to(F64)
        return EV(r, (self.e + ar * o.e) / o.a + U * ar)

    def sqrt(self):
        r = self.v.sqrt()
        ar = r.to(F64)
        return EV(r, self.e / (2 * ar) + U * ar)


def ev_stack(xs, dim):
    return EV(torch.stack([x.v for x in xs], dim), torch.stack([x.e.expand(x.v.shape) for x in xs], dim))


def ev_cat(xs, dim):
    return EV(torch.cat([x.v for x in xs], dim), torch.cat([x.e.expand(x.v.shape) for x in xs], dim))


def ev_sum(xs):
    """Left to right, as the kernel's a*b + c*d + ... expressions."""
    acc = xs[0]
    for x in xs[1:]:
        acc = acc + x
    return acc


def fma(a, b, c):
    """fmaf(a, b, c): one rounding of the exact a b + c.  In float32 the product and sum are formed in float64 and
    rounded to fp32 (within 2**-53 relative of the fused result)."""
    if a.v.dtype == F32:
        r = (a.v.double() * b.v.double() + c.v.double()).float()
    else:
        r = a.v * b.v + c.v
    return EV(r, a.a * b.e + b.a * a.e + a.e * b.e + c.e + U * r.abs().to(F64))


def _fma32(acc, a, b):
    """acc = fmaf(a, b, acc) on fp32 tensors (float32 runs of the long sums)."""
    return (a.double() * b.double() + acc.double()).float()


def partial_sums(terms, dim, init=None, valid=None):
    """A sequential chain s_i = s_(i-1) + t_i along ``dim`` (FMAs or adds, one rounding each) -> (its value, the
    rounding term U sum_i |s_i|).  Each step rounds once, with error <= U |s_i| of its own result, so this is the
    first-order bound of the chain; it is the k U sum |terms| of a k-term chain less what cancellation saves in the
    partial sums.  ``valid`` masks steps the kernel does not take (a chunk's padding)."""
    s = torch.cumsum(terms, dim)
    if init is not None:
        s = s + init.unsqueeze(dim)
    a = s.abs()
    if valid is not None:
        a = a * valid
    return s.select(dim, -1), U * a.sum(dim)


def ev_set(x, idx, val):
    v, e = x.v.clone(), x.e.expand(x.v.shape).clone()
    v[idx], e[idx] = val.v, val.e.expand(val.v.shape)
    return EV(v, e)


def exact(t, dtype):
    """An fp32 input (or model constant) as an EV with no error."""
    return EV(torch.as_tensor(t).to(dtype))


def zeros(shape, dtype):
    return EV(torch.zeros(shape, dtype=dtype))


# ----------------------------------------------------------------------------------------------------- the model
def model_from_packed(packed):
    """The kernel's packed model (ops.pack_mano_model / ManoLayer.packed_model, offsets as in mano.cu) -> dict of
    float64 tensors: dirs (778,3,145) with the 135 pose-map rows then the 10 shape rows, vt (778,3), W (778,16),
    JT (16,3), JS (16,3,10), hm (16,3).  These are exactly the fp32 constants the kernels read."""
    m = torch.as_tensor(packed).detach().cpu().to(F64).reshape(-1)
    o_vt = NK * 3 * NVP
    o_w = o_vt + 3 * NVP
    o_jt = o_w + 16 * NVP
    o_js = o_jt + 48
    o_hm = o_js + 480
    return dict(dirs=m[:o_vt].view(NK, 3, NVP)[:, :, :NV].permute(2, 1, 0).contiguous(),
                vt=m[o_vt:o_w].view(3, NVP)[:, :NV].t().contiguous(), W=m[o_w:o_jt].view(16, NVP)[:, :NV].t().contiguous(),
                JT=m[o_jt:o_js].view(16, 3).clone(), JS=m[o_js:o_hm].view(16, 3, 10).clone(), hm=m[o_hm:o_hm + 48].view(16, 3).clone())


def model_from_asset(asset, flat_hand_mean=True, round_joints=True):
    """The same dict from a MANO asset (its fp32 arrays).  JT = J_regressor . v_template and JS = J_regressor .
    shapedirs in float64, rounded to fp32 like acr_b200_mano_pack_model when ``round_joints`` (then this is
    model_from_packed of the packed asset); unrounded, the statement is the layer of tests/mano_torch_ref.py."""
    t = lambda k: torch.as_tensor(np.asarray(asset[k], np.float32)).to(F64)
    sd, pd, vt, jr = t("shapedirs"), t("posedirs"), t("v_template"), t("J_regressor")
    JT, JS = jr @ vt, torch.einsum("jv,vck->jck", jr, sd)
    if round_joints:
        JT, JS = JT.float().double(), JS.float().double()
    hm = torch.zeros(16, 3, dtype=F64)
    if not flat_hand_mean:
        hm[1:] = t("hands_mean").view(15, 3)
    return dict(dirs=torch.cat([pd, sd], 2), vt=vt, W=t("weights"), JT=JT, JS=JS, hm=hm)


# ---------------------------------------------------------------------------------------------------- rotations
def half_angle_sincos(ang, pi_trig, dtype):
    """sin, cos of ang / 2 (half_angle_sincos in rotation.cuh).
    pi_trig: sincospif(ang * 0.159154943f) -- the product rounds once (U) and the constant is 0.68 U off 1 / (2 pi),
    so the argument x carries e_ang / (2 pi) + (U + 0.68 U) |x|; sincospif is within 1 ulp (2 U relative) of
    sin / cos(pi x), whose argument error is pi times x's.  Otherwise sincosf(ang * 0.5f): the halving is exact,
    sincosf within 2 ulp (4 U relative).  The float64 statement takes the exact half angle."""
    if pi_trig:
        x = ang.v * torch.tensor(C_2PI, dtype=F32) if dtype == F32 else ang.v / (2 * math.pi)
        h = math.pi * x.to(F64)
        e_h = ang.e / 2 + math.pi * (U + C_2PI_REL) * x.abs().to(F64)
        ulp = 1
    else:
        h = ang.v.to(F64) * 0.5
        e_h = ang.e * 0.5
        ulp = 2
    s, c = torch.sin(h), torch.cos(h)
    return (EV(s.to(dtype), c.abs() * e_h + ulp * 2 * U * s.abs()),
            EV(c.to(dtype), s.abs() * e_h + ulp * 2 * U * c.abs()))


def _offset(a, dtype):
    """b = a + 1e-8f: the fp32 constant differs from 1e-8 by 6e-17, an input error of b."""
    off = EV(torch.tensor(OFF8 if dtype == F32 else 1e-8, dtype=dtype), torch.tensor(abs(OFF8 - 1e-8), dtype=F64))
    return [a[..., i] + off for i in range(3)]


def _quat(a, pi_trig, dtype):
    """rotation.cuh's common head: b, ang, n = a / ang, s, c and the unit quaternion (w, x, y, z), qn."""
    b = _offset(a, dtype)
    ang = (b[0] * b[0] + b[1] * b[1] + b[2] * b[2]).sqrt()
    nv = [a[..., i] / ang for i in range(3)]
    s, c = half_angle_sincos(ang, pi_trig, dtype)
    q = [c, s * nv[0], s * nv[1], s * nv[2]]
    qn = (q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]).sqrt()
    return b, ang, nv, s, c, [qi / qn for qi in q], qn


def rodrigues(a, pi_trig, dtype):
    """rodrigues<kPiTrig>: a EV (...,3) -> R EV (...,3,3)."""
    _, _, _, _, _, (w, x, y, z), _ = _quat(a, pi_trig, dtype)
    w2, x2, y2, z2 = w * w, x * x, y * y, z * z
    wx, wy, wz, xy, xz, yz = w * x, w * y, w * z, x * y, x * z, y * z
    R = [w2 + x2 - y2 - z2, xy * 2 - wz * 2, wy * 2 + xz * 2,
         wz * 2 + xy * 2, w2 - x2 + y2 - z2, yz * 2 - wx * 2,
         xz * 2 - wy * 2, wx * 2 + yz * 2, w2 - x2 - y2 + z2]
    return ev_stack(R, -1).reshape(*a.v.shape[:-1], 3, 3)


def rodrigues_vjp(a, g, dtype):
    """rodrigues_vjp: a EV (...,3), g EV (...,3,3) cotangent -> da EV (...,3)."""
    b, ang, nv, s, c, (w, x, y, z), qn = _quat(a, True, dtype)
    g = [g[..., i // 3, i % 3] for i in range(9)]
    dq = [(w * (g[0] + g[4] + g[8]) + x * (g[7] - g[5]) + y * (g[2] - g[6]) + z * (g[3] - g[1])) * 2,
          (x * (g[0] - g[4] - g[8]) + y * (g[1] + g[3]) + z * (g[2] + g[6]) + w * (g[7] - g[5])) * 2,
          (y * (g[4] - g[0] - g[8]) + x * (g[1] + g[3]) + w * (g[2] - g[6]) + z * (g[5] + g[7])) * 2,
          (z * (g[8] - g[0] - g[4]) + w * (g[3] - g[1]) + x * (g[2] + g[6]) + y * (g[5] + g[7])) * 2]
    proj = w * dq[0] + x * dq[1] + y * dq[2] + z * dq[3]
    dq = [(dq[i] - qi * proj) / qn for i, qi in enumerate((w, x, y, z))]
    sa = s / ang
    nd = nv[0] * dq[1] + nv[1] * dq[2] + nv[2] * dq[3]
    dang = (c * nd - s * dq[0]) * 0.5 - sa * nd
    return ev_stack([sa * dq[i + 1] + dang * (b[i] / ang) for i in range(3)], -1)


def rodrigues_jvp(a, da, dtype):
    """rodrigues_jvp: a EV (...,3), da EV (...,3) tangent -> dR EV (...,3,3)."""
    b, ang, nv, s, c, (w, x, y, z), qn = _quat(a, True, dtype)
    da = [da[..., i] for i in range(3)]
    sa = s / ang
    dang = (b[0] / ang) * da[0] + (b[1] / ang) * da[1] + (b[2] / ang) * da[2]
    k = (c * 0.5 - sa) * dang
    dq = [-(s * 0.5) * dang, sa * da[0] + nv[0] * k, sa * da[1] + nv[1] * k, sa * da[2] + nv[2] * k]
    proj = w * dq[0] + x * dq[1] + y * dq[2] + z * dq[3]
    dw, dx, dy, dz = [(dq[i] - qi * proj) / qn for i, qi in enumerate((w, x, y, z))]
    dR = [(w * dw + x * dx - y * dy - z * dz) * 2, (dx * y + x * dy - dw * z - w * dz) * 2,
          (dw * y + w * dy + dx * z + x * dz) * 2, (dw * z + w * dz + dx * y + x * dy) * 2,
          (w * dw - x * dx + y * dy - z * dz) * 2, (dy * z + y * dz - dw * x - w * dx) * 2,
          (dx * z + x * dz - dw * y - w * dy) * 2, (dw * x + w * dx + dy * z + y * dz) * 2,
          (w * dw - x * dx - y * dy + z * dz) * 2]
    return ev_stack(dR, -1).reshape(*a.v.shape[:-1], 3, 3)


def _skew(z):
    o = torch.zeros_like(z[..., 0])
    return torch.stack([o, -z[..., 2], z[..., 1], z[..., 2], o, -z[..., 0], -z[..., 1], z[..., 0], o], -1).view(
        *z.shape[:-1], 3, 3)


def _axial(X):
    return torch.stack([X[..., 2, 1] - X[..., 1, 2], X[..., 0, 2] - X[..., 2, 0], X[..., 1, 0] - X[..., 0, 1]], -1)


def polar64(M):
    """M (...,3,3) float64 -> Q (the orthogonal polar factor), D (...,3) = (1, 1, -1 where det Q < 0), the singular
    values S (...,3) in decreasing order, and the solve matrix (tr P) I - P, P = Q^T M, of the projection's
    derivatives (its eigenvalues are the sums s_j + s_k)."""
    Uu, S, Vh = torch.linalg.svd(M)
    Q = Uu @ Vh
    D = torch.ones(*M.shape[:-2], 3, dtype=F64)
    D[..., 2] = torch.where(torch.linalg.det(Q) < 0, -1.0, 1.0)
    P = Q.transpose(-1, -2) @ M
    A = P.diagonal(dim1=-2, dim2=-1).sum(-1)[..., None, None] * torch.eye(3, dtype=F64) - P
    return Q, D, S, A


def so3_conditioning(S):
    """-> (kappa, m, ok): m = s_2 + s_3 (the smallest s_j + s_k), kappa = s_1 / m, and ok = kappa <= 1 / ROT_CUT.

    The kernel's projection (polar_factor, fp64) takes V from a Jacobi eigensolve of M^T M and u_i = M v_i: its
    error in Q is of order eps64 kappa^2 (the squared conditioning of M^T M's eigenvectors where they matter), and the
    adjugate solve of the derivatives adds eps64 kappa.  ``so3_project`` charges FP64_TERM * eps64 * kappa^2 per unit
    of output.  FP64_TERM = 64 is an assumed constant, not a count: it is meant to cover the six Jacobi sweeps, the
    Gram-Schmidt and the 3x3 products to first order.  At the cutoff kappa = 1e3 the term is 7e-9, a tenth of U, so
    below the cutoff the fp32 rounding dominates whatever the constant.  Past it (rank <= 2 up to 1e-3 of ||M||: rank <= 1 is outside the contract and gives NaN, DESIGN.md;
    det M so small that its fp64 sign is not the float64 statement's) no bound is claimed, only finiteness where
    the rank is 3.  Note that M = -R is not singular here: the kernel's P = Q^T M uses the unflipped polar factor,
    so (tr P) I - P = 2 I there and the flip of column 2 is a constant factor."""
    m = S[..., 1] + S[..., 2]
    kappa = S[..., 0] / m
    return kappa, m, (m >= ROT_CUT * S[..., 0]) & (S[..., 2] >= 1e-9 * S[..., 0])


def so3_project(M, dtype):
    """so3_project: M (...,3,3) fp32 values -> R EV, ok (...).  fp64 throughout, one rounding to fp32:
    e = U |R| + FP64_TERM eps64 kappa^2 (entries of R are <= 1); e = 0 where not ok (no bound is claimed)."""
    Q, D, S, _ = polar64(M.to(F64))
    kappa, _, ok = so3_conditioning(S)
    R = Q * D[..., None, :]
    e = U * R.abs() + (FP64_TERM * EPS64 * kappa ** 2)[..., None, None]
    return EV(R.to(dtype), torch.where(ok[..., None, None], e, 0.0)), ok


def so3_project_vjp(M, g, dtype):
    """so3_project_vjp: with B = Q^T (g D), k = axial(B - B^T), z = ((tr P) I - P)^-1 k, dM = Q [z]x, in fp64 and
    rounded once.  g's own error: ||dB||_F = ||e_g||_F, ||axial(.)|| <= sqrt 2 ||dB||_F, ||dz|| <= ||dk|| / m, and
    an entry of dM is at most ||[dz]x||_F = sqrt 2 ||dz||: 2 ||e_g||_F / m.  The fp64 term as in so3_project on the
    scale ||z|| <= 2 ||g||_F / m."""
    M = M.to(F64)
    Q, D, S, A = polar64(M)
    kappa, m, ok = so3_conditioning(S)
    gv = g.v.to(F64)
    B = Q.transpose(-1, -2) @ (gv * D[..., None, :])
    z = torch.linalg.solve(A, _axial(B))
    dM = Q @ _skew(z)
    gF = gv.square().sum((-1, -2)).sqrt()
    eF = g.e.expand(g.v.shape).square().sum((-1, -2)).sqrt()
    e = U * dM.abs() + (FP64_TERM * EPS64 * kappa ** 2 * 2 * gF / m + 2 * eF / m)[..., None, None]
    return EV(dM.to(dtype), torch.where(ok[..., None, None], e, 0.0))


def so3_project_jvp(M, dM, dtype):
    """So3ProjectJvp.apply: X = Q^T dM, w = ((tr P) I - P)^-1 axial(X - X^T), dR = Q [w]x D; fp64, one rounding.
    dM is an fp32 input (exact); the fp64 term as in so3_project_vjp on the scale 2 ||dM||_F / m."""
    M, dM = M.to(F64), torch.as_tensor(dM).to(F64)
    Q, D, S, A = polar64(M)
    kappa, m, ok = so3_conditioning(S)
    w = torch.linalg.solve(A, _axial(Q.transpose(-1, -2) @ dM))
    dR = (Q @ _skew(w)) * D[..., None, :]
    e = U * dR.abs() + (FP64_TERM * EPS64 * kappa ** 2 * 2 * dM.square().sum((-1, -2)).sqrt() / m)[..., None, None]
    return EV(dR.to(dtype), torch.where(ok[..., None, None], e, 0.0))


# -------------------------------------------------------------------------------------------- phase 1: transforms
def _mm3(A, B):
    """sum_k A[..., :, k] B[..., k, :] left to right: the kernel's 3-term row . column expressions."""
    return ev_sum([A[..., :, k, None] * B[..., None, k, :] for k in range(3)])


def _mv3(A, x):
    return ev_sum([A[..., :, k] * x[..., None, k] for k in range(3)])


def transforms(model, pose, betas, mode, pi_trig, center_src, dtype):
    """rebuild_transforms<kPiTrig, kPose>: -> dict R (n,16,3,3), J (n,16,3), G (n,16,3,4), A (n,16,3,4), ctr (n,3),
    bounded (n,) (False where a matrix is past the projection's cutoff), a (n,16,3) the Rodrigues input.
    Axis angles: the mean pose is added in fp32, then rodrigues<kPiTrig>.  J = JT + 10 fmaf on JS . beta.
    The chain: N = Gp [Rl | rel] + [0 | t_p], rel = J_idx - J_par, each entry a left-to-right 3-term sum.
    A_j = [R_g | t_g - R_g J_j]."""
    n = pose.shape[0]
    out = {}
    if mode == "aa":
        a = exact(torch.as_tensor(pose).reshape(n, 16, 3), dtype) + exact(model["hm"], dtype)
        R = rodrigues(a, pi_trig, dtype)
        out["a"], out["bounded"] = a, torch.ones(n, dtype=torch.bool)
    else:
        R, ok = so3_project(torch.as_tensor(pose).reshape(n, 16, 3, 3), dtype)
        out["bounded"] = ok.all(1)
    b = exact(betas, dtype)
    JS = exact(model["JS"], dtype)
    J = exact(model["JT"], dtype)[None].reshape(1, 16, 3)
    for k in range(10):
        J = fma(JS[None, :, :, k], b[:, None, None, k], J)
    G = [None] * 16
    G[0] = ev_cat([R[:, 0], J[:, 0, :, None]], -1)
    for idx, par in CHAIN:
        rel = J[:, idx] - J[:, par]
        Gp = G[par]
        G[idx] = ev_cat([_mm3(Gp[:, :, :3], R[:, idx]), (_mv3(Gp[:, :, :3], rel) + Gp[:, :, 3])[..., None]], -1)
    G = ev_stack(G, 1)
    At = G[..., 3] - _mv3(G[..., :3], J)
    out.update(R=R, J=J, G=G, A=ev_cat([G[..., :3], At[..., None]], -1), b=b)
    out["ctr"] = G[:, center_src, :, 3] if center_src is not None else zeros((n, 3), dtype)
    return out


def blend(model, R, b, dtype, tangent=False):
    """blend_vertex / blend_tangents: v_posed = v_template + 145 FMAs over the blend rows (R_j - I for j >= 1, then
    beta), or its tangent from zero over (dR_j, dbeta).  -> (v_posed EV (n,778,3), the 145 coefficients EV)."""
    n = R.v.shape[0]
    pm = R[:, 1:] if tangent else R[:, 1:] - exact(torch.eye(3, dtype=F64), dtype)
    pm = ev_cat([pm.reshape(n, 135), b], 1)
    dirs = model["dirs"]
    order = list(range(135, NK)) + list(range(135))          # the kernel's order: the shape rows first
    init = None if tangent else model["vt"][None].expand(n, NV, 3)
    if dtype == F32:
        v = torch.zeros(n, NV, 3, dtype=F32) if tangent else init.to(F32)
        d32 = dirs.to(F32)
        for k in order:
            v = _fma32(v, d32[None, :, :, k], pm.v[:, None, None, k])
        rnd = 0.0
    else:
        v, rnd = partial_sums(dirs[None][..., order] * pm.v[:, None, None, order], -1, init)
    return EV(v, torch.einsum("vck,nk->nvc", dirs.abs(), pm.e) + rnd), pm


def skin(model, A, dtype):
    """skin_transform: T = sum_j w_j A_j, 16 FMAs from zero -> EV (n,778,3,4)."""
    W = model["W"]
    if dtype == F32:
        v = torch.zeros(A.v.shape[0], NV, 3, 4, dtype=F32)
        for j in range(16):
            v = _fma32(v, W.to(F32)[None, :, j, None, None], A.v[:, None, j])
        rnd = 0.0
    else:
        v, rnd = partial_sums(W[None, :, None, None, :] * A.v.permute(0, 2, 3, 1)[:, None], -1)
    return EV(v, torch.einsum("vj,njrc->nvrc", W, A.e) + rnd)


def _centre_src(center_idx):
    if center_idx is None:
        return None
    cs = JOINT_REORDER[center_idx]
    assert cs < 16, "centring on a fingertip is not supported"
    return cs


def _joints(src16, verts, side, palm):
    """Output joints (n,21,3) from the 16 kinematic joints (already centred) and the centred vertices."""
    if palm:
        src16 = ev_cat([((verts[:, PALM[0]] + verts[:, PALM[1]]) * 0.5)[:, None], src16[:, 1:]], 1)
    src = ev_cat([src16, verts[:, TIPS[side]]], 1)
    return src[:, JOINT_REORDER]


# ------------------------------------------------------------------------------------------------------- forward
def layer_forward(model, side, pose, betas, mode, center_idx, palm, dtype=F64):
    """mano_forward_body<kPose, kPalm> (the pipeline's mano_forward_kernel is mode 'aa' without the palm):
    x_r = T[r,0] vp_0 + T[r,1] vp_1 + T[r,2] vp_2 + T[r,3] - ctr_r; kinematic joints t_g - ctr; tips the vertices;
    the palm (x_95 + x_22) * 0.5 of the centred vertices.  mode 'aa' (pose (n,48), mean pose model['hm']) or 'rotmat'
    (pose (n,16,3,3)).  -> dict verts, joints, center (EVs) and bounded (n,)."""
    cs = _centre_src(center_idx)
    tr = transforms(model, pose, betas, mode, False, cs, dtype)
    vp, _ = blend(model, tr["R"], tr["b"], dtype)
    T = skin(model, tr["A"], dtype)
    verts = _mv3(T[..., :3], vp) + T[..., 3] - tr["ctr"][:, None]
    joints = _joints(tr["G"][..., 3] - tr["ctr"][:, None], verts, side, palm)
    return dict(verts=verts, joints=joints, center=tr["ctr"], bounded=tr["bounded"])


# ------------------------------------------------------------------------------------------------------ backward
def _chunked(x):
    """(n,778,...) -> (n,7,128,...) with zero padding: the vertex kernel's chunks of VPB vertices."""
    pad = torch.zeros((x.shape[0], NCHUNK * VPB - NV) + tuple(x.shape[2:]), dtype=x.dtype)
    return torch.cat([x, pad], 1).reshape((x.shape[0], NCHUNK, VPB) + tuple(x.shape[2:]))


VALID = (torch.arange(NCHUNK * VPB) < NV).to(F64).view(NCHUNK, VPB)   # vertices a chunk's loops visit


def _over_chunks(p):
    """The chain kernel's in-order sum of the seven partials."""
    return ev_sum([p[:, c] for c in range(NCHUNK)])


def layer_backward(model, side, pose, betas, mode, center_idx, palm, dverts=None, djoints=None, dcenter=None,
                   dtype=F64, defect=None):
    """mano_backward_{vertex,chain}_body<kPose, kPalm> -> dict dpose EV ((n,48) or (n,16,3,3)), dbetas EV (n,10),
    bounded (n,).  The cotangents are fp32 inputs (None: zero).

    Vertex kernel (per hand and chunk of 128 vertices), from the rebuilt transforms (sincospif):
      du     = dverts + the tip's joint cotangent (+ 0.5 * joint 0's on vertices 95 and 22 with the palm): adds;
      dvp_c  = T[0,c] du_0 + T[1,c] du_1 + T[2,c] du_2;
      dA_j   = sum_v (w_vj du_r) [vp_c | 1]: wd = w du rounded first, then <= 128 FMAs (adds) per chunk;
      su     = sum_v du, <= 128 adds per chunk;
      dpm_k  = sum over 3 coordinates of <= 128 FMAs dirs_k,c . dvp_c each, the three then added in order.
    Chain kernel: the seven partials summed in order; dctr = dcenter - the seven su - the source joints' cotangents
    (joint 0 excluded with the palm), in order; dG = [dA[:, :3] - dA[:, 3] J^T | dt + dA[:, 3]] with dt the joint's
    cotangent (+ dctr at the centre); dJ = -G[:, :3]^T dA[:, 3]; the three-level finger walks from the tip (dR = Gp^T
    dN[:, :3], drel = Gp^T dN[:, 3], dGp = dN [Rl | rel]^T-part, each a 3- or 4-term sum); the five fingers' root
    contributions in order; g = dR + dpm; rodrigues_vjp / so3_project_vjp; dbetas = dpb + 48 FMAs JS . dJ.

    ``defect`` plants one error for tests/test_cpu_mano_layer_bounds.py: 'tip445' (tip 2 read from vertex 445 on
    the right hand), 'palm96' (half the palm's cotangent on vertex 96 instead of 95), 'js' (1e-3 relative error on
    the JS . dJ term of dbetas), 'centre0' (the centre term also subtracting joint 0's cotangent with the palm)."""
    cs = _centre_src(center_idx)
    n = betas.shape[0]
    tr = transforms(model, pose, betas, mode, True, cs, dtype)
    G, J, R = tr["G"], tr["J"], tr["R"]
    partials = dverts is not None or djoints is not None
    dj = exact(djoints, dtype) if djoints is not None else None
    if partials:
        vp, _ = blend(model, R, tr["b"], dtype)
        T = skin(model, tr["A"], dtype)
        du = exact(dverts, dtype) if dverts is not None else zeros((n, NV, 3), dtype)
        if dj is not None:
            for s, v in enumerate(TIPS[side]):
                if defect == "tip445" and s == 2:
                    v = 445
                du = ev_set(du, (slice(None), v), du[:, v] + dj[:, JOINT_INV[16 + s]])
            if palm:
                for v in ((96,) + PALM[1:] if defect == "palm96" else PALM):
                    du = ev_set(du, (slice(None), v), du[:, v] + dj[:, 0] * 0.5)
        dvp = ev_sum([T[..., r, :3] * du[..., r, None] for r in range(3)])          # (n,778,3)
        W = model["W"]
        wd = EV(du.v[:, :, None, :] * W.to(dtype)[None, :, :, None], None)            # (n,778,16,3)
        wd.e = W[None, :, :, None] * du.e[:, :, None, :] + U * wd.a
        cw, cvp, cdu, cdvp = _chunked(wd.v), _chunked(vp.v), _chunked(du.v), _chunked(dvp.v)
        awd, ewd, avp, evp = _chunked(wd.a), _chunked(wd.e), _chunked(vp.a), _chunked(vp.e)
        dirs = _chunked(model["dirs"][None])[0]                                          # (7,128,3,145)
        if dtype == F32:      # the kernel's order: vertex by vertex within a chunk
            v_rc = torch.zeros(n, NCHUNK, 16, 3, 3, dtype=F32)
            v_t, v_su = 0, 0
            v_pm = torch.zeros(n, NCHUNK, 3, NK, dtype=F32)
            d32 = dirs.to(F32)
            for i in range(VPB):
                v_rc = _fma32(v_rc, cw[:, :, i, :, :, None], cvp[:, :, i, None, None, :])
                v_t, v_su = v_t + cw[:, :, i], v_su + cdu[:, :, i]
                v_pm = _fma32(v_pm, d32[None, :, i], cdvp[:, :, i, :, None])
            r_rc = r_t = r_su = r_pm = 0.0
        else:
            val = lambda k: VALID.view((1, NCHUNK, VPB) + (1,) * k)
            v_rc, r_rc = partial_sums(cw[..., None] * cvp[:, :, :, None, None, :], 2, valid=val(3))
            v_t, r_t = partial_sums(cw, 2, valid=val(2))
            v_su, r_su = partial_sums(cdu, 2, valid=val(1))
            v_pm, r_pm = partial_sums(dirs[None] * cdvp[..., None], 2, valid=val(2))
        dA_rc = EV(v_rc, torch.einsum("nhvjr,nhvc->nhjrc", awd, evp) + torch.einsum("nhvjr,nhvc->nhjrc", ewd, avp)
                   + torch.einsum("nhvjr,nhvc->nhjrc", ewd, evp) + r_rc)
        dA_t = EV(v_t, ewd.sum(2) + r_t)
        su = EV(v_su, _chunked(du.e).sum(2) + r_su)
        dpm3 = EV(v_pm, torch.einsum("hvck,nhvc->nhck", dirs.abs(), _chunked(dvp.e)) + r_pm)
        dpm_p = dpm3[:, :, 0] + dpm3[:, :, 1] + dpm3[:, :, 2]                            # (n,7,145)
        dA = _over_chunks(ev_cat([dA_rc, dA_t[..., None]], -1))                          # (n,16,3,4)
        dpm = _over_chunks(dpm_p)
    else:
        dA, dpm = zeros((n, 16, 3, 4), dtype), zeros((n, NK), dtype)
    # centre
    if cs is not None:
        d = exact(dcenter.reshape(n, 3), dtype) if dcenter is not None else zeros((n, 3), dtype)
        if partials:
            for c in range(NCHUNK):
                d = d - su[:, c]
        if dj is not None:
            for s in range(1 if palm and defect != "centre0" else 0, 16):
                d = d - dj[:, JOINT_INV[s]]
        dctr = d
    else:
        dctr = zeros((n, 3), dtype)
    # dG, dJ
    dt = zeros((n, 16, 3), dtype)
    if dj is not None:
        dt = dj[:, JOINT_INV[:16]]
        if palm:
            dt = ev_cat([zeros((n, 1, 3), dtype), dt[:, 1:]], 1)
    if cs is not None:
        dt = ev_set(dt, (slice(None), cs), dt[:, cs] + dctr)
    dAt = dA[..., 3]
    dG = ev_cat([dA[..., :3] - dAt[..., None] * J[:, :, None, :], (dt + dAt)[..., None]], -1)
    dJ = -ev_sum([G[..., r, :3] * dAt[..., r, None] for r in range(3)])                   # (n,16,3)
    dG = [dG[:, j] for j in range(16)]
    dJ = [dJ[:, j] for j in range(16)]
    dR = [None] * 16
    root = []
    for f in range(5):
        dN = dG[3 * f + 3]
        for lev in (2, 1, 0):
            idx = 3 * f + 1 + lev
            par = idx - 1 if lev else 0
            Gp, Rl = G[:, par], R[:, idx]
            rel = J[:, idx] - J[:, par]
            dR[idx] = ev_sum([Gp[:, r, :3, None] * dN[:, r, None, :3] for r in range(3)])
            drel = ev_sum([Gp[:, r, :3] * dN[:, r, 3, None] for r in range(3)])
            dP = ev_cat([_dP_rot(dN, Rl, rel), dN[:, :, 3, None]], -1)
            dJ[idx] = dJ[idx] + drel
            if lev:
                dJ[par] = dJ[par] - drel
                dN = dG[par] + dP
            else:
                root.append((dP, -drel))
    dG0, dJ0 = dG[0], dJ[0]
    for f in range(5):
        dG0 = dG0 + root[f][0]
        dJ0 = dJ0 + root[f][1]
    dR[0] = dG0[..., :3]
    dJ[0] = dJ0 + dG0[..., 3]
    dR = ev_stack(dR, 1)                                                                  # (n,16,3,3)
    dJ = ev_stack(dJ, 1)                                                                  # (n,16,3)
    g = dR + ev_cat([zeros((n, 1, 3, 3), dtype), dpm[:, :135].reshape(n, 15, 3, 3)], 1)
    if mode == "aa":
        dpose = rodrigues_vjp(tr["a"], g, dtype).reshape(n, 48)
    else:
        dpose = so3_project_vjp(torch.as_tensor(pose).reshape(n, 16, 3, 3), g, dtype)
    JS = exact(model["JS"], dtype)
    d = dpm[:, 135:]
    js = EV(JS.v * (1 + 1e-3)) if defect == "js" else JS
    for s in range(16):
        for c in range(3):
            d = fma(js[None, s, c, :], dJ[:, s, c, None], d)
    return dict(dpose=dpose, dbetas=d, bounded=tr["bounded"])


def _dP_rot(dN, Rl, rel):
    """dGp[r, i] = dN[r,0] Rl[i,0] + dN[r,1] Rl[i,1] + dN[r,2] Rl[i,2] + dN[r,3] rel[i]."""
    return ev_sum([dN[:, :, c, None] * Rl[:, None, :, c] for c in range(3)] + [dN[:, :, 3, None] * rel[:, None, :]])


# ----------------------------------------------------------------------------------------------------------- JVP
def layer_jvp(model, side, pose, betas, mode, center_idx, palm, tpose=None, tbetas=None, dtype=F64):
    """mano_layer_jvp_kernel / mano_layer_jvp_joints_kernel<kPose, kPalm> -> dict tverts (T,n,778,3), tjoints
    (T,n,21,3), tcenter (T,n,3) (EVs) and bounded (n,).  tpose (T,n,48) / (T,n,16,3,3), tbetas (T,n,10), fp32.

    Per tangent, from the rebuilt primal (sincospif): dR_j by rodrigues_jvp / So3ProjectJvp; dJ = 10 FMAs JS . dbeta
    from zero; the chain dN = dP [Rl | rel] + Gp [dRl | drel] (+ dt_p), each entry one left-to-right sum of 6 (7)
    products; dctr = dG_centre[:, 3]; the joint tangents dG[:, 3] - dctr; dA_j = [dG | dt - dG J - G dJ];
    d v_posed = 145 FMAs from zero over (dR_j, dbeta); dT = 16 FMAs; tan_row: a = dT[r,3], then six FMAs
    dT[r,:3] . vp and T[r,:3] . dvp in that order, minus dctr.  The joints-only form runs the same operations on the
    tips and palm vertices only, so one statement covers both."""
    cs = _centre_src(center_idx)
    n = betas.shape[0]
    nt = (tpose if tpose is not None else tbetas).shape[0]
    tr = transforms(model, pose, betas, mode, True, cs, dtype)
    G, J, R = tr["G"], tr["J"], tr["R"]
    vp, _ = blend(model, R, tr["b"], dtype)
    T = skin(model, tr["A"], dtype)
    JS = exact(model["JS"], dtype)
    outs = {"tverts": [], "tjoints": [], "tcenter": []}
    for u in range(nt):
        if tpose is None:
            dR = zeros((n, 16, 3, 3), dtype)
        elif mode == "aa":
            dR = rodrigues_jvp(tr["a"], exact(torch.as_tensor(tpose[u]).reshape(n, 16, 3), dtype), dtype)
        else:
            dR = so3_project_jvp(torch.as_tensor(pose).reshape(n, 16, 3, 3), torch.as_tensor(tpose[u]).reshape(n, 16, 3, 3),
                                 dtype)
        db = exact(tbetas[u], dtype) if tbetas is not None else zeros((n, 10), dtype)
        dJ = zeros((n, 16, 3), dtype)
        for k in range(10):
            dJ = fma(JS[None, :, :, k], db[:, None, None, k], dJ)
        dG = [None] * 16
        dG[0] = ev_cat([dR[:, 0], dJ[:, 0, :, None]], -1)
        for idx, par in CHAIN:
            dP, Gp, Rl, dRl = dG[par], G[:, par], R[:, idx], dR[:, idx]
            rel, drel = J[:, idx] - J[:, par], dJ[:, idx] - dJ[:, par]
            rot = ev_sum([dP[:, :, k, None] * Rl[:, None, k, :] for k in range(3)]
                         + [Gp[:, :, k, None] * dRl[:, None, k, :] for k in range(3)])
            t = ev_sum([dP[:, :, k] * rel[:, None, k] for k in range(3)] + [Gp[:, :, k] * drel[:, None, k] for k in range(3)]
                       + [dP[:, :, 3]])
            dG[idx] = ev_cat([rot, t[..., None]], -1)
        dG = ev_stack(dG, 1)
        dctr = dG[:, cs, :, 3] if cs is not None else zeros((n, 3), dtype)
        dAt = dG[..., 3] - _mv3(dG[..., :3], J) - _mv3(G[..., :3], dJ)
        dA = ev_cat([dG[..., :3], dAt[..., None]], -1)
        dvp, _ = blend(model, dR, db, dtype, tangent=True)
        dT = skin(model, dA, dtype)
        a = dT[..., 3]
        for c in range(3):
            a = fma(dT[..., c], vp[:, :, None, c], a)
        for c in range(3):
            a = fma(T[..., c], dvp[:, :, None, c], a)
        tv = a - dctr[:, None]
        outs["tverts"].append(tv)
        outs["tjoints"].append(_joints(dG[..., 3] - dctr[:, None], tv, side, palm))
        outs["tcenter"].append(dctr)
    out = {k: ev_stack(v, 0) for k, v in outs.items()}
    out["bounded"] = tr["bounded"]
    return out


# ----------------------------------------------------------------------------------------------------- test inputs
def _r32(x):
    return x.float().double()


def edge_poses(n, g):
    """(n,48) axis angles: seeded random rows, then (as far as n allows) rows whose 16 joints cycle through 0, 1e-6,
    pi - 1e-6, pi, 4 (beyond pi) and 2 pi - 0.1 about +-x, +-y, +-z and seeded axes (for a flat mean pose)."""
    pose = torch.randn(n, 48, generator=g, dtype=torch.float64) * 0.5
    axes = [torch.eye(3, dtype=torch.float64)[i] * s for i in range(3) for s in (1.0, -1.0)]
    axes += list(torch.nn.functional.normalize(torch.randn(4, 3, generator=g, dtype=torch.float64), dim=1))
    rows = [ax * th for ax in axes for th in (0.0, 1e-6, torch.pi - 1e-6, torch.pi, 4.0, 2 * torch.pi - 0.1)]
    rows = torch.stack(rows)
    for i in range(min(n, (len(rows) + 15) // 16 + 1)):
        pose[i] = rows[(torch.arange(16) + 16 * i) % len(rows)].reshape(48)
    return _r32(pose)


def matrices(n, g):
    """(n,16,3,3): the five classes of test_gpu_mano_rotmat._matrices (exact, noisy, det < 0, 2 R, Gaussian) mixed
    per joint, the identity, and in one joint a rank-3 matrix diag(1, s2, s3) between two rotations: s2 + s3 = 2e-3
    (inside the projection's cutoff) in every fourth hand from hand 1, 5e-4 (past it: that hand's outputs are only
    required finite) in every 64th from hand 3."""
    R = rodrigues64(torch.randn(n * 16, 3, generator=g, dtype=torch.float64)).view(n, 16, 3, 3)
    noise = torch.randn(n, 16, 3, 3, generator=g, dtype=torch.float64)
    h = torch.arange(n)[:, None]
    cls = (h + torch.arange(16)[None, :]) % 6
    one = torch.arange(16)[None, :] == h % 16                      # one joint of some hands is near-singular
    cls = torch.where(one & (h % 4 == 1), 6, torch.where(one & (h % 64 == 3), 7, cls))
    out = torch.where((cls == 0)[..., None, None], R, R + 0.1 * noise)
    out = torch.where((cls == 2)[..., None, None], -(R + 0.05 * noise), out)
    out = torch.where((cls == 3)[..., None, None], 2 * R, out)
    out = torch.where((cls == 4)[..., None, None], noise, out)
    out = torch.where((cls == 5)[..., None, None], torch.eye(3, dtype=torch.float64), out)
    R2 = rodrigues64(torch.randn(n * 16, 3, generator=g, dtype=torch.float64)).view(n, 16, 3, 3)
    for c, m in ((6, 2e-3), (7, 5e-4)):
        S = torch.diag(torch.tensor([1.0, 0.6 * m, 0.4 * m], dtype=torch.float64))
        out = torch.where((cls == c)[..., None, None], R @ S @ R2.transpose(-1, -2), out)
    return _r32(out)
