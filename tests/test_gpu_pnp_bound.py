"""GPU: acr_b200_cam_trans_pnp on fresh hands (tests/pnp_bound_ref.py) at every intrinsic pair, held to the
long-double statement per component: the final fit on >= 6 inliers within 1/2 ulp32 + e64, five-point fits within
the basis-angle spread, the inlier sets and statuses equal to the statement's except where a differing joint
straddles the 20 px threshold across the basis sweep, the least-squares rows bit for bit, and the outputs the same
at every batch size and n_dev."""
import time

import numpy as np
import pytest
import torch

from tests import pnp_bound_ref as B

pytestmark = pytest.mark.gpu
N_HANDS = 1512                   # 168 per intrinsic pair
GUARD = 8
ST_INVALID, ST_LSTSQ_4, ST_LSTSQ_FAIL, ST_EPNP = 0, 1, 2, 3   # oracle/pnp_ref status codes


def _run(j3d, pj2d, f, img, n_dev=None):
    """the C ABI on NaN-prefilled outputs with guard rows on both sides -> (t (n,3), mask (n,)) as the kernel left
    them; the guards must be untouched"""
    from acr_b200 import lib as L
    n = j3d.shape[0]
    out = torch.full((n + 2 * GUARD, 3), float("nan"), device="cuda")
    mask = torch.full((n + 2 * GUARD,), -7, dtype=torch.int32, device="cuda")
    nd = None if n_dev is None else torch.tensor([n_dev], dtype=torch.int32, device="cuda")
    L.check(L.load().acr_b200_cam_trans_pnp(L.ptr(j3d), L.ptr(pj2d), L.ptr(nd), n, f, img, L.ptr(out[GUARD:]),
                                            L.ptr(mask[GUARD:]), L.current_stream()), "cam_trans_pnp")
    torch.cuda.synchronize()
    g = torch.cat([out[:GUARD], out[-GUARD:]])
    assert g.isnan().all() and (torch.cat([mask[:GUARD], mask[-GUARD:]]) == -7).all()
    return out[GUARD:-GUARD], mask[GUARD:-GUARD]


@pytest.fixture(scope="module")
def run():
    from acr_b200 import ops
    t0 = time.time()
    d = B.fresh_hands(2027, N_HANDS)
    t_dev = np.zeros((N_HANDS, 3), np.float32)
    m_dev = np.zeros(N_HANDS, np.int64)
    lsq = np.zeros((N_HANDS, 3), np.float32)
    groups = {}
    for f, s in B.INTRINSICS:
        sel = np.nonzero((d["focal"] == f) & (d["img"] == s))[0]
        j3d, pj2d = torch.from_numpy(d["j3d"][sel]).cuda(), torch.from_numpy(d["pj2d"][sel]).cuda()
        t, m = _run(j3d, pj2d, f, s)
        t_dev[sel], m_dev[sel] = t.cpu().numpy(), m.cpu().numpy()
        lsq[sel] = ops.cam_trans(j3d, pj2d, f, s).cpu().numpy()
        groups[(f, s)] = (sel, j3d, pj2d, t, m)
    res = B.pool_map(B.check_hand, [(h, d["j3d"][h], d["pj2d"][h], d["focal"][h], d["img"][h], t_dev[h],
                                     int(m_dev[h])) for h in range(N_HANDS)])
    print(f"\n{N_HANDS} fresh hands: kernel and statement in {time.time() - t0:.1f} s")
    return d, res, t_dev, m_dev, lsq, groups


def test_fit_bounds(run):
    d, res, *_ = run
    ratio = np.array([r["ratio"] for r in res])
    cls = np.array([r["cls"] for r in res])
    for f, s in B.INTRINSICS:
        at = (d["focal"] == f) & (d["img"] == s)
        parts = []
        for c in ("fit6", "fit5", "usable5"):
            r = ratio[at & (cls == c)]
            parts.append(f"{c} {r.size} worst {r.max():.3f}" if r.size else f"{c} 0")
        print(f"f {f:g} img {s:g}: " + ", ".join(parts))
        assert (at & (cls == "fit6")).sum() >= 30
    bad = np.nonzero(~(ratio <= 1) & np.isin(cls, ["fit6", "fit5", "usable5"]))[0]
    assert bad.size == 0, [(int(h), cls[h], float(ratio[h])) for h in bad[:10]]


def test_inlier_sets_and_status(run):
    d, res, *_ = run
    same = np.array([r["same"] for r in res])
    exempt = np.array([r["exempt"] for r in res])
    out, quiet = d["outliers"], ~d["outliers"] & (d["noise"] == 0)
    print(f"inlier set or status differs on {(~same).sum()} hands, exempted (a joint straddles 400 across the basis "
          f"sweep of a hypothesis) {(exempt & ~same).sum()}: {(~same & quiet).sum()} of {quiet.sum()} noise-free "
          f"hands without outliers, {(~same & ~out).sum()} of {(~out).sum()} without outliers, "
          f"{(~same & out).sum()} of {out.sum()} with")
    assert (same | exempt).all(), [res[h] for h in np.nonzero(~(same | exempt))[0][:5]]
    # measured on an H100: 0 / 3 (pixel noise 3 px, where a 5-point hypothesis moves joints by tens of px) / 21 of
    # 924.  The hands are seeded and the kernel deterministic, so the counts are exact; the limit on hands with
    # outliers (23) fails a kernel that also replaces the best hypothesis on an equal inlier count (29)
    assert same[quiet].all()
    assert (~same & ~out).sum() <= 0.01 * (~out).sum()
    assert (~same & out).sum() <= 0.025 * out.sum()
    st = np.array([r["status"] for r in res])
    cnt = np.array([r["cnt"] for r in res])
    assert set(range(4, 22)) <= set(cnt.tolist()) and ((st == ST_LSTSQ_FAIL) & (cnt > 5)).sum() >= 3


def test_fallback_rows_bitwise(run):
    d, res, t_dev, m_dev, lsq, _ = run
    sd = np.array([r["dev_status"] for r in res])
    assert np.isfinite(t_dev).all()
    fb = sd != ST_EPNP
    np.testing.assert_array_equal(t_dev[fb], lsq[fb])
    np.testing.assert_array_equal(t_dev[sd == ST_INVALID], -1.0)
    assert (m_dev[fb] == 0).all() and (sd == ST_INVALID).sum() >= 3 and (sd == ST_LSTSQ_4).sum() >= 3
    # planar usable joints: the least squares with mask 0 at every count
    pl = d["planar"] & (np.array([r["cnt"] for r in res]) >= 5)
    assert pl.sum() >= 3 and (sd[pl] == ST_LSTSQ_FAIL).all()


def test_planar_hands_fall_back():
    """every z equal, 5 and 21 usable joints: finite, ops.cam_trans's bits, mask 0"""
    from acr_b200 import ops
    j3d = B.fresh_hands(5, 18)["j3d"]
    j3d[:, :, 2] = 0.01
    X = j3d.astype(np.float64) + [0.02, -0.01, 0.6]
    pj2d = (1265.0 * X[:, :, :2] / X[:, :, 2:] / 256).astype(np.float32)
    j3d[:9, 5:, 2] = -2
    j3d, pj2d = torch.from_numpy(j3d).cuda(), torch.from_numpy(pj2d).cuda()
    t, m = _run(j3d, pj2d, 1265.0, 512.0)
    assert t.isfinite().all() and (m == 0).all()
    assert torch.equal(t, ops.cam_trans(j3d, pj2d, 1265.0, 512.0))


def test_batch_sizes_and_n_dev(run):
    """a hand's result does not depend on the batch around it, its position, or n_dev; rows past n_dev untouched"""
    *_, groups = run
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    for (f, s), (sel, j3d, pj2d, t, m) in groups.items():
        n = len(sel)
        for b in (1, 3, 4, 5, 4 * sms + 1):
            idx = torch.arange(b, device="cuda") * 7 % n
            tb, mb = _run(j3d[idx].contiguous(), pj2d[idx].contiguous(), f, s)
            assert torch.equal(tb, t[idx]) and torch.equal(mb, m[idx]), (f, s, b)
        for nd in (0, n - 3):
            tb, mb = _run(j3d, pj2d, f, s, n_dev=nd)
            assert torch.equal(tb[:nd], t[:nd]) and torch.equal(mb[:nd], m[:nd]), (f, s, nd)
            assert tb[nd:].isnan().all() and (mb[nd:] == -7).all(), (f, s, nd)
