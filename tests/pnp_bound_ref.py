"""Fresh hands for the RANSAC-EPnP camera translation (csrc/pnp.cu) and the bounds the kernel is held to.

The statement is oracle/pnp_ref.py, run in float64 for the RANSAC decisions and in long double for the final fit;
what is added here is the bookkeeping.

Final fit on >= 6 inliers.  The statement runs in long double on the joints of the kernel's own inlier mask, with
the pixels normalised in float64 exactly as the kernel does, and per component

    |t_dev,k - t_ld,k| <= 1/2 ulp32(|t_ld,k| + e64) + e64
    e64 = 16 max_r ||t64_r - t_ld||_inf + 2**-50 ||t_ld||_inf

over 8 float64 runs r of the same statement on the points in a random order, each coordinate moved by up to 2**-52
relative.  The first term is the kernel's one rounding to fp32; e64 is an a-posteriori estimate of what float64
evaluation order and the hand's conditioning allow, not a proof.  Where a second beta approximation's reprojection
error is within both errors' own uncertainty (16 times their float64 spread) of the chosen one, the kernel may pick
either, and t may lie within the bound of either.

Five points (exactly 5 usable joints, or a final fit on 5 inliers) leave M^T M a two-dimensional null space whose
basis round-off picks, so t is determined only up to that choice: t must lie within 1/2 ulp32 + s of the long-double
result, s the largest distance between the results at 16 basis angles and at angle 0, plus the largest step between
neighbouring angles (the kernel's basis lies between two of them), plus the float64 spread.

Inlier sets.  The kernel's mask and status must equal the statement's, except where a joint's squared error straddles
400 (min <= 400 < max) across the basis-angle sweep of a hypothesis the statement evaluated: from there the RANSAC
path (inlier counts, the best hypothesis, the iteration bound) is not determined by the algorithm, and the kernel may
evaluate hypotheses the statement never reaches.
"""
import numpy as np

from oracle import mano_ref, pnp_ref

F, LD = np.float32, np.longdouble
INTRINSICS = [(f, s) for f in (500.0, 1265.0, 5000.0) for s in (256.0, 512.0, 1024.0)]
RUNS, ANGLES = 8, np.arange(16) * np.pi / 16
THRESH2 = float(pnp_ref.THRESH2)


# ------------------------------------------------------------------------------------------------------ fresh hands
def fresh_hands(seed, n):
    """n seeded hands, the intrinsics cycling through INTRINSICS -> dict of j3d (n,21,3), pj2d (n,21,2) float32,
    focal, img (n,) and labels: outliers (any joint moved off its projection), noise (px), planar, zero_pose, dup,
    top (partly above the top edge), v_edge (a joint at pixel v == -2 and one just above)."""
    from acr_b200.synth import make_synthetic_mano
    rng = np.random.default_rng(seed)
    assets = {s: make_synthetic_mano(s) for s in ("left", "right")}
    i = np.arange(n)
    focal = np.array([INTRINSICS[k % 9][0] for k in i])
    img = np.array([INTRINSICS[k % 9][1] for k in i])
    right = (i // 9) % 2 == 1
    kind = rng.integers(0, 16, n)
    lab = {"planar": (kind == 0) | (i % 97 == 5), "zero_pose": kind == 1, "dup": kind == 2, "top": kind == 3,
           "v_edge": kind == 4, "noise": rng.choice([0.0, 0.5, 3.0], n), "outliers": np.zeros(n, bool),
           "thresh": np.zeros(n, bool)}
    poses = (0.5 * rng.standard_normal((n, 48))).astype(F)
    betas = rng.standard_normal((n, 10)).astype(F)
    poses[lab["zero_pose"]] = 0
    betas[lab["zero_pose"]] = 0
    j3d = np.zeros((n, 21, 3), F)
    for side, sel in (("left", ~right), ("right", right)):
        if sel.any():
            j3d[sel] = mano_ref.mano_forward(assets[side], poses[sel], betas[sel], side)[1]
    j3d[lab["planar"], :, 2] = F(0.01)
    # depth log-uniform from 0.3 m to 30 m (nearly orthographic at the far end), off-centre by up to 40 % of the
    # image; "top" hands straddle the top edge, so joints above v = -2 are masked
    tz = np.exp(rng.uniform(np.log(0.3), np.log(30.0), n))
    tz[i % 41 == 0], tz[i % 41 == 1] = 0.3, 30.0
    tz = np.maximum(tz, 0.2 - j3d[:, :, 2].min(1))
    off = rng.uniform(-0.4, 0.4, (n, 2)) * img[:, None]
    off[lab["top"], 1] = -img[lab["top"]] / 2 + rng.uniform(-30, 10, lab["top"].sum())
    t = np.stack([off[:, 0] * tz / focal, off[:, 1] * tz / focal, tz], 1)
    X = j3d.astype(np.float64) + t[:, None]
    c = img[:, None, None] / 2
    pix = focal[:, None, None] * X[:, :, :2] / X[:, :, 2:] + c
    pix += lab["noise"][:, None, None] * rng.standard_normal(pix.shape)
    for h in range(n):
        if rng.random() < 0.5:                                  # 1..8 joints moved 30..150 px
            k = rng.integers(1, 9)
            idx = rng.choice(21, k, replace=False)
            pix[h, idx] += rng.uniform(30, 150, (k, 2)) * rng.choice([-1, 1], (k, 2))
            lab["outliers"][h] = True
        if rng.random() < 0.15:                                 # a joint 19.9 or 20.1 px off: on the threshold
            j, r, a = rng.integers(21), rng.choice([19.9, 20.1]), rng.uniform(0, 2 * np.pi)
            pix[h, j] += r * np.array([np.cos(a), np.sin(a)])
            lab["outliers"][h] = lab["thresh"][h] = True
        if lab["dup"][h]:
            a, b = rng.choice(21, 2, replace=False)
            j3d[h, b], pix[h, b] = j3d[h, a], pix[h, a]
    half = (img / 2).astype(F)[:, None, None]
    pj2d = (pix / half - 1).astype(F)
    for h in np.nonzero(lab["v_edge"])[0]:                      # pixel v == -2 exactly (masked), and just above
        a, b = rng.choice(21, 2, replace=False)
        pj2d[h, a, 1] = F(-1) - F(2) / half[h, 0, 0]
        pj2d[h, b, 1] = np.nextafter(pj2d[h, a, 1], F(0))
        lab["outliers"][h] = True
    # z = -2 masks a joint: the usable count cycles through 3..21 on a third of the hands (5 on some planar ones)
    want = np.full(n, 21)
    sel = rng.random(n) < 0.35
    want[sel] = 3 + (np.cumsum(sel)[sel] % 19)
    want[lab["planar"] & (i % 2 == 0)] = 5
    for h in range(n):
        if want[h] < 21:
            j3d[h, rng.choice(21, 21 - want[h], replace=False), 2] = F(-2)
    return {"j3d": j3d, "pj2d": pj2d, "focal": focal, "img": img, **lab}


def usable(j3d, pj2d, img):
    """the kernel's joint test for one hand: pixel v > -2 and z != -2"""
    j2d = ((np.asarray(pj2d, F) + 1) * F(img / 2)).astype(F)
    return (j2d[:, 1] > -2.0) & (j3d[:, 2] != -2.0), j2d


# ----------------------------------------------------------------------------------------------- the statement
def statement(j3d, pj2d, f, img):
    """pnp_ref.cam_trans_pnp for one hand with the RANSAC trace -> dict t, mask (bitmask over 21 joints), status,
    cnt (usable joints), best (inliers of the final fit), iters, changes, trace (None below 6 usable joints)"""
    use, j2d = usable(j3d, pj2d, img)
    cnt = int(use.sum())
    r = {"t": None, "mask": 0, "cnt": cnt, "best": 0, "iters": 0, "changes": 0, "trace": None}
    if cnt < 4:
        return {**r, "status": pnp_ref.ST_INVALID}
    if cnt == 4:
        return {**r, "status": pnp_ref.ST_LSTSQ_4}
    t, inl, tr = pnp_ref.solve_pnp_ransac(j3d[use], j2d[use], f, img / 2, trace=True)
    r.update(iters=tr["iters"], changes=tr["changes"], trace=tr if cnt > 5 else None)
    if t is None:
        return {**r, "status": pnp_ref.ST_LSTSQ_FAIL}
    return {**r, "t": t, "status": pnp_ref.ST_EPNP, "best": int(inl.sum()),
            "mask": int(np.sum(1 << np.nonzero(use)[0][inl].astype(np.int64)))}


def device_status(cnt, mask):
    """the status the kernel's outputs imply"""
    if cnt < 4:
        return pnp_ref.ST_INVALID
    if cnt == 4:
        return pnp_ref.ST_LSTSQ_4
    return pnp_ref.ST_EPNP if mask else pnp_ref.ST_LSTSQ_FAIL


# ------------------------------------------------------------------------------------------------------ the bounds
def half_ulp32(x):
    """half the fp32 ulp of |x| (normal range; 2**-150 below it)"""
    m, e = np.frexp(np.abs(np.asarray(x, np.float64)))
    return np.where(np.abs(x) >= 2.0 ** -126, np.ldexp(1.0, e - 25), 2.0 ** -150)


def _runs64(S, uv, f, c, rng):
    """RUNS float64 fits on permuted, 2**-52-perturbed inputs -> list of (sols, best)"""
    out = []
    S64, uv64 = np.asarray(S, F).astype(np.float64), np.asarray(uv, np.float64)
    for _ in range(RUNS):
        p = rng.permutation(S64.shape[0])
        ps = (S64[p].astype(LD) * (1 + LD(2.0 ** -52) * rng.uniform(-1, 1, S64.shape).astype(LD))).astype(np.float64)
        pu = (uv64[p].astype(LD) * (1 + LD(2.0 ** -52) * rng.uniform(-1, 1, uv64.shape).astype(LD))).astype(np.float64)
        out.append(pnp_ref.epnp(ps, pu, f, f, c, c, np.float64, all_sols=True))
    return out


def fit_bound(S, uv, f, c, seed=0, five=None):
    """The bound of the final fit (or the 5-usable EPnP) of float32 points S (m,3) on normalised pixels uv (m,2) ->
    list of candidates (t_ld (3,) float64, e) with e the per-hand slack (e64, or spread + float64 spread on five
    points), or None where the long-double statement fails (the kernel must then fall back)."""
    rng = np.random.default_rng(seed)
    five = S.shape[0] == 5 if five is None else five
    sols, best = pnp_ref.final_fit(S, uv, f, c, LD, all_sols=True)
    if not np.isfinite(sols[best][1].astype(np.float64)).all():
        return None
    runs = _runs64(S, uv, f, c, rng)
    tl = [np.asarray(s[1], np.float64) for s in sols]
    el = [float(s[2]) for s in sols]
    if five:
        sweep = [tl[best]] + [np.asarray(pnp_ref.final_fit(S, uv, f, c, LD, basis_angle=a)[1], np.float64)
                              for a in ANGLES[1:]]
        step = max(np.abs(sweep[k] - sweep[k - 1]).max() for k in range(len(sweep)))   # cyclic: t has period pi
        spread = max(np.abs(s - tl[best]).max() for s in sweep) + step
        d64 = max(np.abs(np.asarray(r[0][r[1]][1]) - tl[best]).max() for r in runs)
        return [(tl[best], spread + d64 + 2.0 ** -50 * np.abs(tl[best]).max())]
    e, u = [], []
    for k in range(3):
        dt = max(np.abs(np.asarray(r[0][k][1]) - tl[k]).max() for r in runs)
        de = max(abs(float(r[0][k][2]) - el[k]) for r in runs)
        e.append(16 * dt + 2.0 ** -50 * np.abs(tl[k]).max())
        u.append(16 * de + 2.0 ** -50 * abs(el[k]))
    return [(tl[k], e[k]) for k in range(3)
            if k == best or (np.isfinite(el[k]) and el[k] - el[best] <= u[k] + u[best])]


def ratio(t_dev, cands):
    """max over components of |t_dev - t_ld| / bound, for the candidate that fits best (<= 1: within the bound)"""
    t_dev = np.asarray(t_dev, np.float64)
    return min(float((np.abs(t_dev - t) / (half_ulp32(np.abs(t) + e) + e)).max()) for t, e in cands)


def straddles(S, J, f, c, trace):
    """True iff some hypothesis the statement evaluated has a joint whose float32 squared error lies on both sides of
    400 across the basis-angle sweep: from that hypothesis on, the inlier counts, and with them the best hypothesis
    and the iteration bound, are not determined, so the final inlier sets may differ in any joint"""
    S, J = np.asarray(S, F), np.asarray(J, F)
    norm32 = pnp_ref.normalised(J, f, c, fp32=True)
    for idx, _, err2 in trace["hyps"]:
        lo = hi = err2.astype(np.float64)
        for a in ANGLES[1:]:
            R, t, _ = pnp_ref.epnp(S[idx], norm32[idx], f, f, c, c, basis_angle=a)
            e = pnp_ref._sq_errors(S, J, R, t, f, c).astype(np.float64)
            lo, hi = np.fmin(lo, e), np.fmax(hi, e)
        if ((lo <= THRESH2) & (hi > THRESH2)).any():
            return True
    return False


def check_hand(args):
    """One hand against the kernel's outputs (t_dev float32 (3,), mask_dev): the statement, the inlier-set rule and
    the bound of the fit the kernel made -> dict with cls ('fit6', 'fit5', 'usable5', 'lstsq', 'invalid'), ratio
    (NaN where no fit bound applies), same (mask and status equal the statement's), exempt, and the trace counts."""
    h, j3d, pj2d, f, img, t_dev, mask_dev = args
    c = img / 2
    st = statement(j3d, pj2d, f, img)
    use, j2d = usable(j3d, pj2d, img)
    S, J = j3d[use], j2d[use]
    cnt = st["cnt"]
    sd = device_status(cnt, mask_dev)
    same = sd == st["status"] and mask_dev == st["mask"]
    exempt = False
    if not same and st["trace"] is not None:
        exempt = straddles(S, J, f, c, st["trace"])
    r = {k: st[k] for k in ("status", "cnt", "best", "iters", "changes")}
    r.update(h=h, dev_status=sd, same=same, exempt=exempt, ratio=np.nan, cls="invalid" if cnt < 4 else "lstsq")
    if sd != pnp_ref.ST_EPNP:
        return r
    if cnt == 5:
        cands, r["cls"] = fit_bound(S, pnp_ref.normalised(J, f, c, fp32=True), f, c, h), "usable5"
    else:
        inl = (mask_dev >> np.nonzero(use)[0]) & 1 == 1
        cands = fit_bound(S[inl], pnp_ref.normalised(J[inl], f, c), f, c, h)
        r["cls"] = "fit5" if inl.sum() == 5 else "fit6"
    r["ratio"] = np.inf if cands is None else ratio(t_dev, cands)
    return r


def pool_map(fn, items):
    """fn over items on every CPU (spawned workers: the parent may hold a CUDA context)"""
    import concurrent.futures as cf
    import multiprocessing as mp
    import os
    workers = len(os.sched_getaffinity(0))
    with cf.ProcessPoolExecutor(workers, mp_context=mp.get_context("spawn")) as ex:
        return list(ex.map(fn, items, chunksize=max(1, len(items) // (8 * workers))))
