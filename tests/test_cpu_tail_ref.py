"""The float64 statements and bounds of tests/tail_ref.py, checked without a GPU: they reproduce the reference goldens,
the float32 oracles satisfy every bound (the bounds are not too tight for a correct fp32 implementation), an error the
old max-norm criterion accepted violates them (they are not vacuous), and the structured rotation set reaches every
branch of rotmat_to_aa."""
import os

import numpy as np
import pytest

from acr_b200.synth import make_synthetic_mano
from oracle import mano_ref, rotation_ref
from tests import tail_ref as T
from tests.helpers import GOLDEN

U = T.U


@pytest.fixture(scope="module")
def assets():
    return {"left": make_synthetic_mano("left"), "right": make_synthetic_mano("right")}


def seeded_hands(n, seed, scale=0.5):
    rng = np.random.default_rng(seed)
    poses = (rng.standard_normal((n, 48)) * scale).astype(np.float32)
    betas = rng.standard_normal((n, 10)).astype(np.float32)
    poses[0] = 0
    if n > 2:
        poses[1, :3] = [np.pi, 0, 0]
        poses[2] = 1e-6
    return poses, betas


def worst(err, bound):
    return float((np.abs(err) / bound).max())


# ------------------------------------------------------------------------------------------------------- rotations
def test_rotation_statements_reproduce_the_golden():
    g = np.load(os.path.join(GOLDEN, "rot_golden.npz"))
    x = g["rot6d"].reshape(-1, 6)
    # rows 4, 5 of the golden are degenerate inputs: check_rot6d gives them an infinite bound and asks for finiteness
    r, v = T.check_rot6d(x, g["aa"].reshape(-1, 3))
    print(f"golden rot6d: worst err/bound as rotation {r:.3f}, as vector {v:.3f}")
    R = T.rodrigues64(g["aa_in"])
    assert (np.abs(R.reshape(-1, 9) - g["rodrigues"]) <= T.rodrigues_bound(g["aa_in"])[:, None]).all()


def test_float32_rotation_oracle_satisfies_the_bounds():
    x, tags = T.structured_rot6d(0)
    rng = np.random.default_rng(3)
    x = np.concatenate([x, rng.standard_normal((4096 * 16, 6)).astype(np.float32)])
    with np.errstate(all="ignore"):
        aa = rotation_ref.rot6d_to_angular(x)
    r, v = T.check_rot6d(x, aa)
    print(f"fp32 oracle rot6d_to_aa: worst err/bound as rotation {r:.3f}, as vector {v:.3f}")
    assert r > 1e-3, "a correct fp32 implementation sits three orders below the bound: the bound says nothing"
    aa_in = np.concatenate([rng.standard_normal((512, 3)), rng.standard_normal((64, 3)) * 100, np.zeros((1, 3)),
                            np.full((1, 3), 1e-7)]).astype(np.float32)
    R32 = rotation_ref.batch_rodrigues(aa_in)
    e = np.abs(R32 - T.rodrigues64(aa_in).reshape(-1, 9)) / T.rodrigues_bound(aa_in)[:, None]
    print(f"fp32 oracle rodrigues: worst err/bound {e.max():.3f}")
    assert 1e-3 < e.max() <= 1


def test_rotation_bounds_reject_wrong_branches():
    """What the two rotation defects a branch bug produces look like: the sign case dropped (the axis angle leaves the
    principal range) and the wrong case of the quaternion (tt near 0)."""
    x = (T.aa_to_rotmat64(np.array([[-3.0, 0.2, 0.1]]))[0][:, :2].reshape(1, 6)).astype(np.float32)
    R, _ = T.rot6d_to_rotmat64(x)
    aa, branch, qw, _ = T.rotmat_to_aa64(R)
    assert qw[0] < 0
    T.check_rot6d(x, aa)
    n = aa / np.linalg.norm(aa)
    with pytest.raises(AssertionError):
        T.check_rot6d(x, -n * (2 * np.pi - np.linalg.norm(aa)))     # the same rotation, the long way round
    with pytest.raises(AssertionError):
        T.check_rot6d(x, aa * (1 + 2e-4))
    with pytest.raises(AssertionError):
        T.check_rot6d(np.full((1, 6), np.nan, np.float32), np.full((1, 3), np.nan))


def test_structured_set_reaches_every_branch():
    x, tags = T.structured_rot6d(0)
    R, cond = T.rot6d_to_rotmat64(x)
    ok = np.isfinite(cond)
    aa, branch, qw, dist = T.rotmat_to_aa64(R[ok])
    theta = np.linalg.norm(aa, axis=1)
    for b in range(4):
        assert (branch == b).sum() >= 20, (b, (branch == b).sum())
    for b in range(3):
        assert ((branch == b) & (qw < 0)).sum() >= 5, b          # case 3 has qw = tt > 0
    near = 1e-4
    lo = dist[:, 0] < 0
    for name, d, where in (("t22 = 1e-6", dist[:, 0], np.ones(len(d0 := dist[:, 0]), bool)),
                           ("t00 = t11", dist[:, 1], lo), ("t00 = -t11", dist[:, 2], ~lo)):
        below, above = (where & (d < 0) & (d > -near)).sum(), (where & (d >= 0) & (d < near)).sum()
        assert below >= 6 and above >= 6, (name, below, above)
    assert (theta < 1e-6).sum() >= 10 and (np.pi - theta < 1e-4).sum() >= 20
    assert (tags == "nan").sum() == 12 and (~ok).sum() >= 12 + 6


# ------------------------------------------------------------------------------------------------------------ MANO
def test_mano_statement_reproduces_the_golden(assets):
    g = np.load(os.path.join(GOLDEN, "mano_golden.npz"))
    L = int(g["L"])
    for side, sl in (("left", slice(0, L)), ("right", slice(L, None))):
        m = T.mano_forward64(assets[side], g["poses"][sl], g["betas"][sl], side, 9)
        p = T.project64(m["verts"], m["joints"], g["cam"][sl], g["offsets"][sl], m["b_verts"], m["b_joints"])
        # the golden is the reference's own fp32 run, with other summation orders: it satisfies the bounds too
        for k, exp, b in (("verts", m["verts"], m["b_verts"]), ("j3d", m["joints"], m["b_joints"]),
                          ("center", m["center"], m["b_center"]), ("verts_camed", p["verts_camed"], p["b_verts_camed"]),
                          ("pj2d", p["pj2d"], p["b_pj2d"]), ("pj2d_org", p["pj2d_org"], p["b_pj2d_org"])):
            w = worst(g[k][sl].reshape(exp.shape) - exp, b)
            print(f"golden {side} {k}: worst err/bound {w:.3f}")
            assert w <= 1, (side, k, w)
    ct, b = T.cam_trans64(g["j3d"], g["pj2d"])
    assert (np.abs(g["cam_trans"] - ct) <= b).all()


def test_float32_mano_oracle_satisfies_the_bounds(assets):
    poses, betas = seeded_hands(24, 11)
    poses[3, 12:15] = [20 * np.pi, 0, 0]
    betas[4], betas[5] = 3, -3
    cam = np.random.default_rng(1).uniform(-1, 1, (24, 3)).astype(np.float32)
    cam[:, 0] = np.linspace(0.3, 3, 24)
    offs = np.tile(np.array([1920, 1920, 0, 0, 0, 0, 420, 0, 420, 0], np.float32), (24, 1))
    for side in ("left", "right"):
        for cidx in (9, None, 0):
            m = T.mano_forward64(assets[side], poses, betas, side, cidx)
            v, j, c = mano_ref.mano_forward(assets[side], poses, betas, side, cidx)
            wv, wj = worst(v - m["verts"], m["b_verts"]), worst(j - m["joints"], m["b_joints"])
            print(f"fp32 oracle {side} center {cidx}: verts {wv:.3f} joints {wj:.3f} of the bound")
            assert 1e-3 < wv <= 1 and wj <= 1
            if cidx is not None:
                assert worst(c[:, 0] - m["center"], m["b_center"]) <= 1
        p = T.project64(m["verts"], m["joints"], cam, offs, m["b_verts"], m["b_joints"])
        o = mano_ref.project(v, j, cam, offs)
        for k in ("verts_camed", "pj2d", "pj2d_org"):
            assert worst(o[k] - p[k], p["b_" + k]) <= 1, k


def test_mano_bound_rejects_what_the_max_norm_accepted(assets):
    """An error just inside the old tolerance (1e-4 of the largest magnitude) on ONE element: max-norm passes it, the
    per-element bound does not -- on a vertex, near the centre and far from it, and on a pixel of pj2d_org."""
    from tests.helpers import rel_err
    poses, betas = seeded_hands(4, 12)
    cam = np.array([[1.2, 0.3, -0.2]] * 4, np.float32)
    offs = np.tile(np.array([1920, 1920, 0, 0, 0, 0, 420, 0, 420, 0], np.float32), (4, 1))
    m = T.mano_forward64(assets["right"], poses, betas, "right", 9)
    p = T.project64(m["verts"], m["joints"], cam, offs, m["b_verts"], m["b_joints"])
    v32, j32, _ = mano_ref.mano_forward(assets["right"], poses, betas, "right", 9)
    o32 = mano_ref.project(v32, j32, cam, offs)["pj2d_org"]
    for got, exp, b in ((v32, m["verts"], m["b_verts"]), (o32, p["pj2d_org"], p["b_pj2d_org"])):
        for pick in (np.argmin, np.argmax):
            i = np.unravel_index(pick(np.abs(exp)), exp.shape)
            bad = got.copy()
            bad[i] += np.float32(0.9e-4 * np.abs(got).max())
            assert rel_err(bad, got) < 1e-4
            print(f"old tolerance / new bound on element {i}: {np.abs(bad - exp)[i] / b[i]:.1f}")
            assert np.abs(bad - exp)[i] > 2 * b[i]
    # the projection steps are held to the rounding of one evaluation: 3 ulp on one coordinate is out
    x = v32[..., 0].astype(np.float64)
    s, t = 1.7, -0.4
    exp = s * x + t
    got = (np.float32(s) * v32[..., 0] + np.float32(t)).astype(np.float32)
    s, t = float(np.float32(s)), float(np.float32(t))
    assert (np.abs(got - (s * x + t)) <= T.project_step_bound(x, s, t)).all()
    got[0, 0] = np.nextafter(np.nextafter(np.nextafter(got[0, 0], np.float32(9)), np.float32(9)), np.float32(9))
    assert np.abs(got - (s * x + t))[0, 0] > T.project_step_bound(x, s, t)[0, 0]


# ------------------------------------------------------------------------------------------------- camera translation
def test_cam_trans_statement_agrees_with_the_oracle(assets):
    poses, betas = seeded_hands(16, 13)
    v, j, _ = mano_ref.mano_forward(assets["right"], poses, betas, "right", 9)
    cam = np.random.default_rng(2).uniform(-0.8, 0.8, (16, 3)).astype(np.float32)
    cam[:, 0] = np.linspace(0.3, 3, 16)
    pj = mano_ref.project(v, j, cam)["pj2d"]
    j = j.copy()
    j[1, :16, 2] = -2.0          # 5 usable
    j[2, :17, 2] = -2.0          # 4 usable
    j[3, :18, 2] = -2.0          # 3 usable -> (-1,-1,-1)
    pj[4, :, 1] = -1.1           # v < -2 at either size: none usable
    pj[5, :18, 1] = -1.0078125   # v == -2.0 exactly at img_size 512 (not > -2): 3 usable
    for f, s in ((1265.0, 512.0), (500.0, 256.0), (5000.0, 512.0)):
        exp, b = T.cam_trans64(j, pj, f, s)
        ref = mano_ref.cam_trans_lstsq(j, pj, f, s)
        assert (exp[3] == -1).all() and (exp[4] == -1).all() and (b[3] == 0).all() and (exp[2] != -1).any()
        assert (exp[5] == -1).all() == (s == 512.0)
        w = worst(ref - exp, np.maximum(b, 1e-30))
        print(f"fp64 oracle cam_trans f={f} size={s}: worst err/bound {w:.3f}")
        assert w <= 1


# --------------------------------------------------------------------------------------------------------- smoothing
def test_one_euro_statement_reproduces_the_golden_and_bounds_the_oracle():
    g = np.load(os.path.join(GOLDEN, "smooth_golden.npz"))
    banks = [T.OneEuro64(4.0), T.OneEuro64(4.0)]
    ora = [rotation_ref.OneEuroBank(4.0), rotation_ref.OneEuroBank(4.0)]
    wp = wb = wr = 0.0
    for t in range(g["poses"].shape[0]):
        for h in range(2):
            if not g["det"][t, h] > 0:
                continue
            r = banks[h].process(g["poses"][t, h], g["betas"][t, h])
            op, ob = ora[h].process(g["poses"][t, h], g["betas"][t, h])
            for got_p, got_b in ((g["out_poses"][t, h], g["out_betas"][t, h]), (op, ob)):
                wp = max(wp, worst(got_p[3:] - r["pose"], r["b_pose"] + 1e-30))
                wb = max(wb, worst(got_b - r["betas"], r["b_betas"] + 1e-30))
                e = np.linalg.norm(T.aa_to_rotmat64(got_p[:3])[0] - T.aa_to_rotmat64(r["aa"])[0])
                wr = max(wr, e / T.smoothed_root_bound(r["b_M"], r["qnorm"]))
    print(f"golden + fp32 oracle smoothing: worst err/bound pose {wp:.3f} betas {wb:.3f} root {wr:.3f}")
    assert wp <= 1 and wb <= 1 and wr <= 1 and wp > 1e-3


def test_one_euro_bound_does_not_grow_with_the_frame_count():
    rng = np.random.default_rng(5)
    bank = T.OneEuro64(4.0)
    pose, betas = rng.standard_normal(48) * 0.3, rng.standard_normal(10)
    b = []
    for t in range(600):
        pose = pose + rng.standard_normal(48) * 0.02
        betas = betas + rng.standard_normal(10) * 0.01
        r = bank.process(pose.astype(np.float32), betas.astype(np.float32))
        b.append(max(r["b_pose"].max(), r["b_betas"].max(), r["b_M"]))
    assert max(b[300:]) <= 1.5 * max(b[10:300]) and max(b) < 1e-4
