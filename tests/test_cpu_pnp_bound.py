"""CPU: the bounds of tests/pnp_bound_ref.py on fresh hands.  The long-double statement agrees with the float64 one
within e64; a second float64 implementation (LAPACK's least squares for the beta approximations, the control-point
matrix inverted by its adjugate) satisfies the bound on every fit; perturbed statements violate it; and the fresh
hands reach every RANSAC regime the kernel has."""
import contextlib

import numpy as np
import pytest

from tests import pnp_bound_ref as B

N_HANDS = 360


@contextlib.contextmanager
def _variant(name):
    """a perturbed or alternative statement, patched into oracle.pnp_ref for the duration of a block"""
    from oracle import pnp_ref
    saved = pnp_ref.svd_solve, pnp_ref._barycentric, pnp_ref.jacobi_svd
    if name == "lapack":
        def adjugate(d, cws):
            C = (cws[1:] - cws[0]).T
            adj = np.array([np.cross(C[:, 1], C[:, 2]), np.cross(C[:, 2], C[:, 0]), np.cross(C[:, 0], C[:, 1])])
            return d @ (adj / (C[:, 0] @ adj[0])).T
        pnp_ref.svd_solve = lambda A, b: np.linalg.lstsq(A.astype(np.float64), b, rcond=None)[0]
        pnp_ref._barycentric = adjugate
    elif name == "jacobi3":                 # the 12 x 12 Jacobi stops after 3 sweeps
        orig = pnp_ref.jacobi_svd
        pnp_ref.jacobi_svd = lambda A, dtype=np.float64, sweeps=None: orig(A, dtype, 3 if len(A) == 12 else sweeps)
    try:
        yield
    finally:
        pnp_ref.svd_solve, pnp_ref._barycentric, pnp_ref.jacobi_svd = saved


def _hand(args):
    """statement, bound and the alternative fits of one fresh hand"""
    from oracle import pnp_ref
    h, j3d, pj2d, f, img = args
    st = B.statement(j3d, pj2d, f, img)
    r = {k: v for k, v in st.items() if k != "trace"}
    if st["status"] != pnp_ref.ST_EPNP:
        return r
    use, j2d = B.usable(j3d, pj2d, img)
    inl = (st["mask"] >> np.nonzero(use)[0]) & 1 == 1
    S, J, c = j3d[use][inl], j2d[use][inl], img / 2
    five = st["cnt"] == 5
    uv = pnp_ref.normalised(J, f, c, fp32=five)
    cands = B.fit_bound(S, uv, f, c, h)
    r["cls"] = "usable5" if five else "fit5" if inl.sum() == 5 else "fit6"
    r["ld_agree"] = min(float(np.abs(st["t"] - t).max() / e) if e else np.inf for t, e in cands)
    fits = {}
    with _variant("lapack"):
        fits["lapack"] = pnp_ref.final_fit(S, uv, f, c)[1]
    fits["fp32px"] = pnp_ref.final_fit(S, pnp_ref.normalised(J, f, c, fp32=True), f, c)[1]
    with _variant("jacobi3"):
        fits["jacobi3"] = pnp_ref.final_fit(S, uv, f, c)[1]
    fits["n1"] = pnp_ref.final_fit(S, uv, f, c, all_sols=True)[0][0][1]
    r.update({k: B.ratio(np.asarray(t).astype(np.float32), cands) for k, t in fits.items()})
    return r


@pytest.fixture(scope="module")
def hands():
    d = B.fresh_hands(11, N_HANDS)
    res = B.pool_map(_hand, [(h, d["j3d"][h], d["pj2d"][h], d["focal"][h], d["img"][h]) for h in range(N_HANDS)])
    return d, res


def _col(res, k, cls=None):
    return np.array([r[k] for r in res if k in r and (cls is None or r.get("cls") in cls)], np.float64)


def test_fresh_hands_cover_every_regime(hands):
    from oracle import pnp_ref
    d, res = hands
    st = np.array([r["status"] for r in res])
    cnt = np.array([r["cnt"] for r in res])
    iters, changes, best = (np.array([r[k] for r in res]) for k in ("iters", "changes", "best"))
    print(f"{N_HANDS} hands: iters >= 50 on {(iters >= 50).sum()}, no consensus on "
          f"{((st == pnp_ref.ST_LSTSQ_FAIL) & (cnt > 5)).sum()}, best changed >= 2 times on {(changes >= 2).sum()}, "
          f"5-inlier fits {((best == 5) & (cnt > 5)).sum()}, 5 usable {(cnt == 5).sum()}")
    assert (iters >= 50).sum() >= 3
    assert ((st == pnp_ref.ST_LSTSQ_FAIL) & (cnt > 5)).sum() >= 3
    assert (changes >= 2).sum() >= 3
    assert ((best == 5) & (cnt > 5)).sum() >= 2
    assert set(range(4, 22)) <= set(cnt.tolist())
    for f, s in B.INTRINSICS:
        assert ((d["focal"] == f) & (d["img"] == s) & (st == pnp_ref.ST_EPNP)).sum() >= 10
    for k in ("planar", "zero_pose", "dup", "top", "v_edge", "thresh"):
        assert d[k].sum() >= 3, k
    # planar usable joints have no EPnP: the least squares, whatever the count
    pl = d["planar"] & (cnt >= 5)
    assert pl.sum() >= 3 and (st[pl] == pnp_ref.ST_LSTSQ_FAIL).all()
    assert ((cnt == 5) & d["planar"]).sum() >= 1 and ((cnt > 5) & d["planar"]).sum() >= 1


def test_planar_hands_fall_back():
    """every z equal: the 5-usable path and RANSAC both end in the least squares with mask 0"""
    from oracle import mano_ref, pnp_ref
    j3d = B.fresh_hands(5, 18)["j3d"]
    j3d[:, :, 2] = 0.01
    X = j3d.astype(np.float64) + [0.02, -0.01, 0.6]
    pj2d = (1265.0 * X[:, :, :2] / X[:, :, 2:] / 256).astype(np.float32)
    j3d[:9, 5:, 2] = -2                  # 5 usable joints on the first 9 hands, 21 on the rest
    t, mask, st = pnp_ref.cam_trans_pnp(j3d, pj2d)
    lsq = mano_ref.cam_trans_lstsq(j3d, pj2d)
    assert (st == pnp_ref.ST_LSTSQ_FAIL).all() and (mask == 0).all()
    np.testing.assert_array_equal(t, lsq)


def test_long_double_agrees_with_float64(hands):
    _, res = hands
    a = _col(res, "ld_agree")
    print(f"float64 vs long double over {a.size} EPnP hands: worst |t64 - t_ld| / e64 {a.max():.3f}, "
          f"median {np.median(a):.3f}")
    assert a.size >= 150 and (a <= 1).all()


def test_bound_is_not_too_tight(hands):
    """LAPACK's least squares in place of the SVD solve and the adjugate in place of LAPACK's inverse: a float64
    implementation the statement did not write, rounded to fp32, within the bound on every fit"""
    _, res = hands
    for cls in (("fit6",), ("fit5", "usable5")):
        r = _col(res, "lapack", cls)
        print(f"{cls}: second float64 implementation, worst err/bound {r.max():.3f} over {r.size} hands")
        assert (r <= 1).all()
    assert _col(res, "lapack", ("fit6",)).max() > 0.1


@pytest.mark.parametrize("variant,share", [("fp32px", 0.5), ("jacobi3", 0.9), ("n1", 0.15)])
def test_bound_is_not_too_loose(hands, variant, share):
    """perturbed statements on >= 6-inlier fits: float32-normalised pixels in the final fit, the 12 x 12 Jacobi
    capped at 3 sweeps, the N = 1 approximation always taken"""
    _, res = hands
    r = _col(res, variant, ("fit6",))
    print(f"{variant}: violates the bound on {(r > 1).mean():.1%} of {r.size} fits; violation factors p50 "
          f"{np.median(r):.2g}, p90 {np.quantile(r, 0.9):.2g}, max {r.max():.2g}")
    assert (r > 1).mean() >= share
