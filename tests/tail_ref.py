"""float64 statements of the fp32 tail (rotations, the pipeline's MANO forward with its projection, the least-squares
camera translation, the OneEuro smoothing) and the per-element error bounds the kernels are held to.

The statements are the numpy oracles of ``oracle/`` run in float64 (their ``dtype`` argument), so there is one
restatement of each operation; what is added here is the bookkeeping a bound needs.  Every bound has the form

    |got - exp| <= c * U * S            U = 2**-24, the unit roundoff of fp32 (half an ulp)

with S a sum of magnitudes taken from the float64 evaluation and c counted from the operations the kernel performs
(each fp32 operation has relative error <= U; a chain of k of them <= k U to first order).  The counts are derived in
the docstrings; none is fitted to a measurement.  tests/test_cpu_tail_ref.py shows that the float32 oracles satisfy
the bounds and that an error the old max-norm criterion accepted violates them.
"""
import numpy as np

from oracle import mano_ref, rotation_ref
from oracle.mano_ref import JOINT_REORDER, TIPS

U = 2.0 ** -24
F32, F64 = np.float32, np.float64
I3 = np.eye(3)


# ------------------------------------------------------------------------------------------------------ rotations
def rodrigues64(aa):
    """(M,3) -> (M,3,3), the half-angle quaternion form with the 1e-8 offset inside the angle."""
    return rotation_ref.batch_rodrigues(np.asarray(aa, F64).reshape(-1, 3), F64).reshape(-1, 3, 3)


def rodrigues_angle(aa):
    return np.sqrt(((np.asarray(aa, F64) + 1e-8) ** 2).sum(-1))


def rodrigues_bound(aa):
    """Per-entry bound of the fp32 Rodrigues, (M,) in absolute units.

    b = a + 1e-8 (U each), b^2 (3 U), their sum (5 U), ang = sqrt: relative error <= 3.5 U.  The half angle is exact;
    sincosf is within 2 ulp (2 U absolute: its values are <= 1) of the sine / cosine of the ROUNDED argument, whose
    absolute error is 3.5 U ang / 2: d(sin, cos) <= (2 + 1.75 ang) U.  n = a / ang: 4.5 U relative; s n: 1 more; the
    renormalisation (4 squares, 3 sums, sqrt, divide) moves each component by <= 4 U.  So every quaternion component
    is within dq = (11.5 + 1.75 ang) U.  An entry of R is a sum of four products of two components, sum |q_a| <= 2:
    |dR| <= 2 * 2 * dq + 4 U (its own four roundings, magnitudes summing to <= 1) = (50 + 7 ang) U.  In the MANO
    kernel the mean pose is added in fp32 first (U relative on a, i.e. U ang on the rotation): (50 + 8 ang) U."""
    return (50.0 + 8.0 * rodrigues_angle(aa)) * U


def rodrigues_bound2(aa):
    """The same as a 2-norm, for products of rotations: ||dq||_2 <= 2 dq (four components) turns the rotation by the
    angle 2 ||dq||, so ||dR||_2 <= 4 dq = (46 + 7 ang) U, + 12 U for the nine entries' own roundings (4 U each, as a
    Frobenius norm), + U ang for the mean pose: (58 + 8 ang) U -- a third of 3 x the per-entry bound."""
    return (58.0 + 8.0 * rodrigues_angle(aa)) * U


ORTHO_BOUND = 40 * U   # max |R R^T - I| of the fp32 Rodrigues: |q|^2 is within 8 U of 1 (the renormalisation), R R^T =
#                        |q|^4 I for the quaternion form, plus 4 U per entry of R entering twice in each of 3 products


def aa_to_rotmat64(aa):
    """Exact exponential map (no offset), (M,3) -> (M,3,3): what an axis angle MEANS, used to compare as rotations."""
    aa = np.asarray(aa, F64).reshape(-1, 3)
    th = np.sqrt((aa * aa).sum(-1))
    with np.errstate(invalid="ignore", divide="ignore"):
        a = np.where(th > 1e-4, np.sin(th) / th, 1 - th * th / 6)
        b = np.where(th > 1e-4, (1 - np.cos(th)) / (th * th), 0.5 - th * th / 24)
    K = np.zeros((aa.shape[0], 3, 3))
    K[:, 0, 1], K[:, 0, 2], K[:, 1, 0] = -aa[:, 2], aa[:, 1], aa[:, 2]
    K[:, 1, 2], K[:, 2, 0], K[:, 2, 1] = -aa[:, 0], -aa[:, 1], aa[:, 0]
    return I3 + a[:, None, None] * K + b[:, None, None] * (K @ K)


def rot6d_to_rotmat64(x):
    """(M,6) -> R (M,3,3) and cond (M,) = 1 / sin angle(a1, a2), the conditioning of the Gram-Schmidt step; inf where
    a column (or the residual of the second) is within a factor 2 of the 1e-6 clamp, or the input is not finite:
    there fp32 and fp64 may clamp differently and the result is no rotation, so only finiteness is required."""
    x = np.asarray(x, F64).reshape(-1, 6)
    with np.errstate(invalid="ignore", divide="ignore"):
        R = rotation_ref.rot6d_to_rotmat(x, F64)
        a1, a2 = x.reshape(-1, 3, 2)[:, :, 0], x.reshape(-1, 3, 2)[:, :, 1]
        n1, n2 = np.linalg.norm(a1, axis=1), np.linalg.norm(a2, axis=1)
        u = np.linalg.norm(a2 - (a1 * a2).sum(1, keepdims=True) * a1 / (n1 * n1)[:, None], axis=1)
        cond = n2 / u
    bad = ~np.isfinite(x).all(1) | ~(n1 > 2e-6) | ~(u > 2e-6) | ~np.isfinite(cond)
    return R, np.where(bad, np.inf, cond)


def rotmat_to_aa64(R):
    """(M,3,3) -> aa (M,3), branch (M,) in 0..3 (the order of the kernel's four cases), qw (M,) the quaternion's
    scalar before the sign case, and dist (M,3): t22 - 1e-6, t00 - t11, t00 + t11 (t = R^T), the signed distances to
    the three branch boundaries (the second matters when t22 < 1e-6, the third otherwise)."""
    R = np.asarray(R, F64).reshape(-1, 3, 3)
    q = rotation_ref.rotmat_to_quaternion(R, dtype=F64)
    aa = rotation_ref.quaternion_to_angle_axis(q, F64)
    aa[np.isnan(aa)] = 0.0
    t22, t00, t11 = R[:, 2, 2], R[:, 0, 0], R[:, 1, 1]
    d2 = t22 < 1e-6
    branch = np.where(d2, np.where(t00 > t11, 0, 1), np.where(t00 < -t11, 2, 3))
    return aa, branch, q[:, 0], np.stack([t22 - 1e-6, t00 - t11, t00 + t11], 1)


def rot6d_rotation_bound(cond):
    """Bound on ||R(aa_got) - R_exp||_F for rot6d_to_aa, (M,).

    Gram-Schmidt in fp32, every product and sum rounded separately: b1 = a1 / ||a1|| is within 3 U per unit length.
    d = b1 . a2 (5 operations on b1's 3 U): <= 6 U ||a2||; u = a2 - d b1 adds d's error, b1's (3 U), a product and a
    difference: <= 11 U ||a2|| absolute, which is 11 U / sin(a1, a2) relative to ||u||, + 3 U for its normalisation.
    b3 = b1 x b2 inherits both and adds 2 U.  ||dR||_F <= (3 + (11 c + 3) + (3 + 11 c + 3 + 2)) U = (14 + 22 c) U,
    c = cond.  The quaternion case that is taken has tt >= 1 - 1e-6, so q = v / (2 sqrt tt) is linear in the entries
    with coefficients <= 1 and the map to a rotation doubles a perturbation at most: 2 (14 + 22 c) U.  Quaternion ->
    axis angle -> rotation: atan2f within 2 ulp on an angle <= pi (13 U), the division and three products, the
    square root: 40 U covers it.  Total (68 + 44 c) U."""
    return (68.0 + 44.0 * np.asarray(cond, F64)) * U


PI_CUT = 1e-3   # axis angles are compared as vectors only when pi - theta exceeds this


def aa_vector_bound(rot_bound, theta):
    """Bound on ||aa_got - aa_exp|| given the rotation bound, inf within PI_CUT of theta = pi.
    The logarithm's Jacobian has norm (theta/2) / sin(theta/2) <= pi/2 below pi, and a rotation error d (as a vector)
    has ||dR||_F = sqrt(2) ||d||: ||d aa|| <= (pi/2) rot_bound / sqrt(2).  At pi the axis angle jumps from +pi n to
    -pi n, so nearer than PI_CUT (far more than any rot_bound that is not itself vacuous) only the rotation is
    compared."""
    b = (np.pi / 2) * np.asarray(rot_bound) / np.sqrt(2.0)
    return np.where(np.pi - np.asarray(theta) > PI_CUT, b, np.inf)


def _euler_zxz(al, be, ga):
    ca, sa, cb, sb, cg, sg = np.cos(al), np.sin(al), np.cos(be), np.sin(be), np.cos(ga), np.sin(ga)
    return np.array([[ca * cg - sa * cb * sg, -ca * sg - sa * cb * cg, sa * sb],
                     [sa * cg + ca * cb * sg, -sa * sg + ca * cb * cg, -ca * sb],
                     [sb * sg, sb * cg, cb]])


def structured_rot6d(seed=0):
    """The rotation test set: fp32 (M,6) inputs and a tag per row.

    'angle'    rotations by theta in {0, 1e-7..1e-3, 1, pi-1e-2..pi-1e-6, pi} about 8 seeded axes, the three
               coordinate axes and their negatives (the latter give qw < 0 in the t22 < 1e-6 cases);
    'edge'     rotations a distance +-d, d in {1e-7, 1e-6, 1e-5}, from each of the three branch boundaries of
               rotmat_to_aa (in Z-X-Z Euler angles R22 = cos b, R00 - R11 = (1 - cos b) cos(a - g) and
               R00 + R11 = (1 + cos b) cos(a + g), so each boundary is one angle condition);
    'scale'    the first two columns of a seeded rotation times 1e-3..1e3 each, the second sheared by k b1 with
               k in {0, 1, 1e2, 1e4} (nearly parallel columns);
    'degenerate' columns shorter than the 1e-6 clamp, a zero row, exactly parallel columns;
    'nan'      a NaN or inf in each of the six positions."""
    rng = np.random.default_rng(seed)
    rows, tags = [], []

    def put(R, tag):
        rows.append(np.asarray(R)[:, :2].reshape(6)); tags.append(tag)

    axes = [v / np.linalg.norm(v) for v in rng.standard_normal((8, 3))]
    axes += [s * e for e in np.eye(3) for s in (1.0, -1.0)]
    thetas = [0.0] + [10.0 ** -k for k in range(7, 2, -1)] + [1.0] + [np.pi - 10.0 ** -k for k in range(2, 7)] + [np.pi]
    for ax in axes:
        for th in thetas:
            put(aa_to_rotmat64(ax * th)[0], "angle")
    for _ in range(6):
        a, g = rng.uniform(0, 2 * np.pi, 2)
        for d in (1e-7, 1e-6, 1e-5):
            for s in (1, -1):
                put(_euler_zxz(a, np.arccos(1e-6 + s * d), g), "edge")                    # t22 = 1e-6 +- d
                b = rng.uniform(np.pi / 2 + 0.1, np.pi - 0.1)                            # t22 < 0: t00 = t11 +- ...
                put(_euler_zxz(g + np.pi / 2 + s * d, b, g), "edge")
                b = rng.uniform(0.1, np.pi / 2 - 0.1)                                    # t22 > 0: t00 = -t11 +- ...
                put(_euler_zxz(np.pi / 2 - g + s * d, b, g), "edge")
    for _ in range(8):
        R = aa_to_rotmat64(rng.standard_normal(3))[0]
        for s1 in (1e-3, 1.0, 1e3):
            for s2 in (1e-3, 1.0, 1e3):
                for k in (0.0, 1.0, 1e2, 1e4):
                    M = R.copy()
                    M[:, 1] = s2 * (R[:, 1] + k * R[:, 0]); M[:, 0] = s1 * R[:, 0]
                    put(M, "scale")
    R = aa_to_rotmat64(rng.standard_normal(3))[0]
    for s1, s2 in ((1e-7, 1.0), (1.0, 1e-7), (1e-8, 1e-8), (0.0, 0.0), (0.0, 1.0), (1.0, 0.0)):
        put(np.stack([s1 * R[:, 0], s2 * R[:, 1], R[:, 2]], 1), "degenerate")
    put(np.stack([R[:, 0], 2 * R[:, 0], R[:, 2]], 1), "degenerate")
    for i in range(6):
        for bad in (np.nan, np.inf):
            r = R[:, :2].reshape(6).copy(); r[i] = bad
            rows.append(r); tags.append("nan")
    return np.asarray(rows, F64).astype(F32), np.asarray(tags)


def check_rot6d(x32, aa_got):
    """All rot6d_to_aa assertions for inputs x32 (M,6) and the kernel's (M,3): returns worst err/bound of the
    rotation and of the vector comparison."""
    x32, aa_got = np.asarray(x32, F32).reshape(-1, 6), np.asarray(aa_got, F64).reshape(-1, 3)
    assert not np.isnan(aa_got).any(), "NaN in an axis angle (the kernel writes 0 instead)"
    R, cond = rot6d_to_rotmat64(x32)
    nonfinite = ~np.isfinite(x32).all(1)
    assert (aa_got[np.isnan(x32).any(1)] == 0).all(), "a NaN input row must give the zero axis angle"
    ok = np.isfinite(cond)
    assert np.isfinite(aa_got[~nonfinite]).all()
    rb = rot6d_rotation_bound(cond[ok])
    err = np.sqrt(((aa_to_rotmat64(aa_got[ok]) - R[ok]) ** 2).sum((1, 2)))
    bad = np.flatnonzero(err > rb)
    assert bad.size == 0, f"rotation off: rows {np.flatnonzero(ok)[bad][:5]} err {err[bad][:5]} bound {rb[bad][:5]}"
    # the principal value: |aa| <= pi (2 atan2f <= fl(pi) = pi (1 + 0.45 U), three products)
    nrm = np.sqrt((aa_got[ok] ** 2).sum(1))
    assert (nrm <= np.pi * (1 + 4 * U)).all(), f"axis angle longer than pi: {nrm.max()}"
    aa_exp, _, _, _ = rotmat_to_aa64(R[ok])
    vb = aa_vector_bound(rb, np.sqrt((aa_exp ** 2).sum(1)))
    verr = np.sqrt(((aa_got[ok] - aa_exp) ** 2).sum(1))
    fin = np.isfinite(vb)
    bad = np.flatnonzero(verr[fin] > vb[fin])
    assert bad.size == 0, f"axis angle off: {verr[fin][bad][:5]} bound {vb[fin][bad][:5]}"
    return float((err / rb).max()), float((verr[fin] / vb[fin]).max())


# ----------------------------------------------------------------------------------------------------- MANO forward
CHAIN = [(3 * f + 1 + lev, 0 if lev == 0 else 3 * f + lev) for lev in range(3) for f in range(5)]   # (joint, parent)


def mano_forward64(asset, poses, betas, side, center_idx):
    """The layer in float64 (oracle.mano_ref.mano_forward, dtype=float64) for fp32 inputs: dict with verts
    (n,778,3), joints (n,21,3), center (n,3) (zero without a centre), their per-element bounds b_verts, b_joints,
    b_center, and S (n,778,3), the magnitude sum of a vertex.  ``side`` is 'left' / 'right'; the left model's
    shapedirs are x-flipped as the pipeline's are; center_idx None or an out-joint index that is no fingertip.

    The bound follows the kernel's stages.  U-multiples, all magnitudes from the float64 run:
      e_R   per entry of a local rotation: rodrigues_bound (the mean pose's addition included).
      v_posed_c = v_template + 145 FMAs: 145 roundings + the R - I subtraction's, on
              S_vp = |v_template| + sum_k |dirs_k| |pm_k|, plus the coefficients' own error:
              e_vp = 146 U S_vp + sum_k |posedirs_k| (e_R + 2 U).
      J     = JT + JS . beta, 10 FMAs on model constants rounded from fp64: e_J = 12 U (|JT| + sum |JS_k| |beta_k|).
      chain ||dRg||_2 of a joint at depth d: the sum of its d local rotations' rodrigues_bound2 + 16 U per 3x3
              product; the translation adds ||dRg_parent|| ||rel|| + e_J of both joints + U ||rel|| +
              4 U (||rel|| + ||t_parent||) for its four operations on a unit row.
      A_j   = [Rg | t - Rg J]: e_At = e_t + ||dRg|| ||J|| + e_J + 4 U (||J|| + ||t||).
      T     = sum_j w_j A_j, 16 FMAs: dT <= sum_j w_j (error of A_j) + 16 U sum_j w_j |A_j|.
      x_r   = T[r,:3] . v_posed + T[r,3] - ctr_r, 5 operations on S = sum_j w_j (sum_c |A_j[r,c]| |v_posed_c| +
              |A_j[r,3]|) + |ctr_r|:  b = dT . |v_posed| + |T| . e_vp + dT_t + e_ctr + 5 U S.
    The leading terms are (16 + 5) U S from the skinning and 146 U S_vp from the blend; the chain and Rodrigues
    terms carry the joints' own magnitudes."""
    poses = np.asarray(poses, F32).astype(F64).reshape(-1, 48)
    betas = np.asarray(betas, F32).astype(F64).reshape(-1, 10)
    n = poses.shape[0]
    d = {}
    # the fp32 kernel adds the mean pose in fp32; float64 here, its rounding is inside e_R
    verts, joints, center = mano_ref.mano_forward(asset, poses, betas, side, center_idx, dtype=F64, detail=d)
    cs = None if center_idx is None else JOINT_REORDER[center_idx]
    assert cs is None or cs < 16
    eR = rodrigues_bound(d["full_pose"])                                        # (n,16)
    R, J, G, A, vp = d["R"], d["J"], d["G"], d["A"], d["v_posed"]
    sd, pdirs, vt, W = np.abs(d["shapedirs"]), np.abs(d["posedirs"]), np.abs(d["v_template"]), np.abs(d["weights"])
    pm = np.abs((R[:, 1:] - I3).reshape(n, 135))
    S_vp = vt[None] + np.einsum("vck,nk->nvc", sd, np.abs(betas)) + np.einsum("vck,nk->nvc", pdirs, pm)
    e_vp = 146 * U * S_vp + np.einsum("vcj,nj->nvc", pdirs.reshape(778, 3, 15, 9).sum(-1), eR[:, 1:] + 2 * U)
    JT = np.abs(d["J_regressor"] @ d["v_template"])
    JS = np.abs(np.einsum("jv,vck->jck", d["J_regressor"], d["shapedirs"]))
    e_J = np.linalg.norm(12 * U * (JT[None] + np.einsum("jck,nk->njc", JS, np.abs(betas))), axis=-1)   # (n,16)
    tg = G[:, :, :3, 3]
    nrm = lambda a: np.linalg.norm(a, axis=-1)
    eG, e_t = np.zeros((n, 16)), np.zeros((n, 16))
    eR2 = rodrigues_bound2(d["full_pose"])
    eG[:, 0], e_t[:, 0] = eR2[:, 0], e_J[:, 0]
    for idx, par in CHAIN:
        rel = nrm(J[:, idx] - J[:, par])
        eG[:, idx] = eG[:, par] + eR2[:, idx] + 16 * U
        e_t[:, idx] = (e_t[:, par] + eG[:, par] * rel + e_J[:, idx] + e_J[:, par] + U * rel
                       + 4 * U * (rel + nrm(tg[:, par])))
    e_At = e_t + eG * nrm(J) + e_J + 4 * U * (nrm(J) + nrm(tg))
    absA = np.abs(A[:, :, :3, :])
    Tabs = np.einsum("vj,njrc->nvrc", W, absA)
    dT_R = np.einsum("vj,nj->nv", W, eG)[:, :, None, None] + 16 * U * Tabs[..., :3]
    dT_t = np.einsum("vj,nj->nv", W, e_At)[:, :, None] + 16 * U * Tabs[..., 3]
    ctr = np.zeros((n, 3)) if cs is None else tg[:, cs]
    e_ctr = np.zeros(n) if cs is None else e_t[:, cs]
    avp = np.abs(vp)
    S = np.einsum("nvrc,nvc->nvr", Tabs[..., :3], avp) + Tabs[..., 3] + np.abs(ctr)[:, None]
    b_verts = (np.einsum("nvrc,nvc->nvr", dT_R, avp) + np.einsum("nvrc,nvc->nvr", Tabs[..., :3], e_vp) + dT_t
               + e_ctr[:, None, None] + 5 * U * S)
    b_src = np.concatenate([(e_t + e_ctr[:, None])[:, :, None] + U * (np.abs(tg) + np.abs(ctr)[:, None]),
                            b_verts[:, TIPS[side]]], 1)
    return dict(verts=verts, joints=joints, center=ctr, b_verts=b_verts, b_joints=b_src[:, JOINT_REORDER],
                b_center=np.repeat(e_t[:, cs][:, None], 3, 1) if cs is not None else np.zeros((n, 3)), S=S)


def project64(verts, joints, cam, offsets=None, b_verts=None, b_joints=None):
    """Weak-perspective projection in float64 from float64 verts / joints and the fp32 cam (n,3) = (s, tx, ty) and
    offsets (n,10): verts_camed = (s x + tx, s y + ty, z); pj2d likewise for the joints; pj2d_org =
    ((pj2d + 1) * (o[0], o[1]) / 2 + (o[5] - o[9], o[2] - o[6])).  With the inputs' bounds it returns the composed
    ones: a product and a sum, or one FMA, on the error of x: |s| b + 2 U (|s x| + |t|); pj2d_org adds a sum, a
    product, an exact halving and a sum: b_pj pad / 2 + 4 U (|pj2d + 1| pad / 2 + |lt|)."""
    cam = np.asarray(cam, F32).astype(F64).reshape(-1, 1, 3)
    s, t = cam[:, :, 0:1], cam[:, :, 1:]
    out = dict(verts_camed=np.concatenate([verts[..., :2] * s + t, verts[..., 2:]], -1), pj2d=joints[..., :2] * s + t)
    if b_verts is not None:
        out["b_verts_camed"] = np.concatenate(
            [np.abs(s) * b_verts[..., :2] + 2 * U * (np.abs(s * verts[..., :2]) + np.abs(t)), b_verts[..., 2:]], -1)
        out["b_pj2d"] = np.abs(s) * b_joints[..., :2] + 2 * U * (np.abs(s * joints[..., :2]) + np.abs(t))
    if offsets is not None:
        o = np.asarray(offsets, F32).astype(F64)
        pad = o[:, None, 0:2]
        lt = np.stack([o[:, 5] - o[:, 9], o[:, 2] - o[:, 6]], 1)[:, None]
        out["pj2d_org"] = (out["pj2d"] + 1) * pad / 2 + lt
        if b_verts is not None:
            out["b_pj2d_org"] = out["b_pj2d"] * pad / 2 + 4 * U * (np.abs(out["pj2d"] + 1) * pad / 2 + np.abs(lt))
    return out


def project_step_bound(x, s, t):
    """Bound of ONE fp32 evaluation of s x + t from the kernel's own fp32 x: a product and a sum, each within half an
    ulp (one FMA is within half an ulp of the result alone)."""
    return U * (np.abs(s * x) + np.abs(s * x + t)) + 1e-45


def org_step_bound(pj, pad, lt):
    """Bound of one fp32 evaluation of (pj + 1) * pad / 2 + lt from the kernel's own pj2d: three rounded operations
    (the halving is exact)."""
    h = np.abs(pj + 1) * pad / 2
    return U * (2 * h + np.abs((pj + 1) * pad / 2 + lt)) + 1e-45


# ------------------------------------------------------------------------------------------------ camera translation
def cam_trans64(j3d, pj2d, focal_length=1265.0, img_size=512.0):
    """Least-squares camera translation per hand, (n,21,3), (n,21,2) fp32 -> exp (n,3) float64 and bound (n,3).

    The kernel's fp32 step u = (pj2d + 1) * (img_size / 2) is restated in fp32 (a sum, then a product: nothing to
    contract), then rows [f, 0, c - u | (u - c) Z - f X] and [0, f, c - v | (v - c) Z - f Y] of every joint with
    v > -2 and Z != -2 go into normal equations solved in long double.  Fewer than 4 such joints give (-1,-1,-1)
    with a zero bound.  The kernel accumulates and solves in float64 and rounds once to fp32:
    |got - exp| <= U |exp| + 64 * 2**-53 * cond(A) * ||exp||_inf (Cramer's rule on a 3x3 system whose 9 sums have at
    most 42 terms; 64 covers them to first order)."""
    j3d, pj2d = np.asarray(j3d, F32).reshape(-1, 21, 3), np.asarray(pj2d, F32).reshape(-1, 21, 2)
    half = F32(F32(img_size) * F32(0.5))
    uv = ((pj2d + F32(1.0)) * half).astype(F32)
    n = j3d.shape[0]
    exp, bound = np.zeros((n, 3)), np.zeros((n, 3))
    LD = np.longdouble
    f, c0 = LD(F32(focal_length)), LD(half)
    for i in range(n):
        m = (uv[i, :, 1] > F32(-2.0)) & (j3d[i, :, 2] != F32(-2.0))
        if m.sum() < 4:
            exp[i] = -1.0
            continue
        X, Y, Z = (j3d[i, m, k].astype(LD) for k in range(3))
        u, v = uv[i, m, 0].astype(LD), uv[i, m, 1].astype(LD)
        k = int(m.sum())
        Q = np.zeros((2 * k, 3), LD)
        Q[0::2, 0], Q[1::2, 1], Q[0::2, 2], Q[1::2, 2] = f, f, c0 - u, c0 - v
        c = np.zeros(2 * k, LD)
        c[0::2], c[1::2] = (u - c0) * Z - f * X, (v - c0) * Z - f * Y
        A, b = Q.T @ Q, Q.T @ c
        # 3x3 solve by Gaussian elimination in long double (numpy.linalg has no long double)
        M = np.concatenate([A, b[:, None]], 1)
        for p in range(3):
            M[p] = M[p] / M[p, p]
            for r in range(3):
                if r != p:
                    M[r] = M[r] - M[r, p] * M[p]
        x = M[:, 3].astype(F64)
        exp[i] = x
        bound[i] = U * np.abs(x) + 64 * 2.0 ** -53 * np.linalg.cond(A.astype(F64)) * np.abs(x).max()
    return exp, bound


# ---------------------------------------------------------------------------------------------------------- smoothing
class OneEuro64:
    """One bank of the OneEuro filter in float64 (45 pose + 10 betas + 9 root-rotation entries) with a running bound
    of the fp32 kernel's error on every filtered element.

        x_hat = a x + (1 - a) x_hat_prev,   a = alpha(mincutoff + 0.7 |edx|),
        edx = ad dx + (1 - ad) edx_prev,    dx = (x - x_prev) * 30,   ad = alpha(1),
        alpha(c) = 1 / (1 + 30 / (2 pi c)),  mincutoff = smooth_coeff (pose, rotation) | 0.6 (betas).

    Bound, per element and frame (first order, every quantity from the float64 run):
        e_dx  = 30 (dxin + dxin_prev) + 2 U |dx|            dxin: the input's error, 0 for pose / betas (fp32 data),
                                                            rodrigues_bound for the rotation entries
        e_edx = ad e_dx + (1 - ad) e_edx_prev + 3 U (|ad dx| + |(1 - ad) edx_prev|) + 4 U |dx|   (ad itself: 4 U)
        e_a   = a (1 - a) (0.7 e_edx / c + 2 U) + 4 U a     (d alpha / d c = a (1 - a) / c; alpha's own 4 operations)
        e     = (1 - a) e_prev + a dxin + |x - x_hat_prev| e_a + 3 U (|a x| + |(1 - a) x_hat_prev|)
    The low-pass is a contraction: 0 < a_min <= a <= 1 with a_min = alpha(mincutoff), so e <= (1 - a_min) e_prev + g
    with g bounded by the inputs' range, and e stays below sup g / a_min whatever the number of frames; e_edx
    likewise with ad.  The recursion is evaluated, not its supremum, so the bound follows the data."""

    def __init__(self, smooth_coeff):
        self.minc = np.concatenate([np.full(45, float(F32(smooth_coeff))), np.full(10, float(F32(0.6))),
                                    np.full(9, float(F32(smooth_coeff)))])
        self.prev = None

    @staticmethod
    def alpha(c):
        return 1.0 / (1.0 + (1.0 / (2 * np.pi * c)) / (1.0 / 30.0))

    def process(self, pose48, betas10):
        """fp32 pose (48), betas (10) -> dict: pose (45), betas (10), M (3,3) the filtered root matrix, aa (3) its
        axis angle, qnorm the norm of its quaternion, and bounds b_pose, b_betas, b_M (per entry)."""
        pose48, betas10 = np.asarray(pose48, F32).astype(F64), np.asarray(betas10, F32).astype(F64)
        x = np.concatenate([pose48[3:], betas10, rodrigues64(pose48[:3]).reshape(9)])
        dxin = np.concatenate([np.zeros(55), np.full(9, rodrigues_bound(pose48[:3]))])
        if self.prev is None:
            xh, edx, e, e_edx = x.copy(), np.zeros(64), dxin.copy(), np.zeros(64)
        else:
            raw, filt, fdx, dxin_p, e_p, e_edx_p = self.prev
            dx = (x - raw) * 30.0
            ad = self.alpha(1.0)
            edx = ad * dx + (1 - ad) * fdx
            c = self.minc + 0.7 * np.abs(edx)
            a = self.alpha(c)
            xh = a * x + (1 - a) * filt
            e_dx = 30 * (dxin + dxin_p) + 2 * U * np.abs(dx)
            e_edx = ad * e_dx + (1 - ad) * e_edx_p + 3 * U * (np.abs(ad * dx) + np.abs((1 - ad) * fdx)) + 4 * U * np.abs(dx)
            e_a = a * (1 - a) * (0.7 * e_edx / c + 2 * U) + 4 * U * a
            e = (1 - a) * e_p + a * dxin + np.abs(x - filt) * e_a + 3 * U * (np.abs(a * x) + np.abs((1 - a) * filt))
        self.prev = (x, xh, edx, dxin, e, e_edx)
        M = xh[55:].reshape(1, 3, 3)
        aa, _, _, _ = rotmat_to_aa64(M)
        q = rotation_ref.rotmat_to_quaternion(M, dtype=F64)
        return dict(pose=xh[:45], betas=xh[45:55], M=M[0], aa=aa[0], qnorm=float(np.linalg.norm(q)),
                    b_pose=e[:45], b_betas=e[45:55], b_M=float(e[55:].max()))


def smoothed_root_bound(b_M, qnorm):
    """Bound on ||R(aa_got) - R(aa_exp)||_F for the root: the filtered matrix M (a blend of rotations, not orthonormal)
    goes through the quaternion cases.  With tt >= 1 in the case taken, q = v / (2 sqrt tt) moves by <= 2 b_M per
    component (v's entries sum two of M's; tt's own error through the square root), ||dq|| <= 4 b_M; the axis
    angle ignores ||q||, so the rotation moves by the angle 2 ||dq|| / ||q||, i.e. sqrt(2) * 8 b_M / ||q|| in the
    Frobenius norm (12 covers it); + 40 U for quaternion -> axis angle as in rot6d_rotation_bound."""
    return 12.0 * b_M / qnorm + 40 * U
