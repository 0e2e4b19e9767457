#!/usr/bin/env python
"""Generate tests/golden/pnp_golden.npz: the reference's camera translation, estimate_translation
(acr/utils.py:474-519) around cv2.solvePnPRansac(EPNP, reprojectionError=20, iterationsCount=100), run with
OpenCV on the CPU.  Needs cv2 where it runs; the npz it writes is committed and is all the GPU tests read.

    python oracle/make_pnp_golden.py

Inputs are (j3d, pj2d) pairs as MANOWrapper produces them (synthetic MANO of acr_b200.synth through
oracle/mano_ref), in classes (CLASSES): clean hands over cam scales 0.3-3; 1-8 joints moved 30-150 px; joints
above the top edge (pixel y <= -2) or with z == -2, masked out; exactly 4, 5 and 6 usable joints; fewer than 4;
garbage points where RANSAC finds no model; and the rows of tests/golden/mano_golden.npz (reference outputs).

Per hand: cv2's t (float64) and inlier bitmask, a status (oracle/pnp_ref ST_*), and two conditioning
measures from the same seeded perturbation (1e-6 relative on j3d, 1e-7 on the pixels, PERTURB draws):
``cond`` = cv2's largest relative change of t, ``mask_stable`` = cv2's inlier set never changes.
"""
import os
import sys

import numpy as np

ROOT = os.path.abspath(os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
OUT = os.path.join(ROOT, "tests", "golden", "pnp_golden.npz")
CLASSES = ("clean", "outliers", "masked", "usable4", "usable5", "usable6", "fewer4", "garbage", "mano_golden")
COUNTS = dict(clean=120, outliers=120, masked=20, usable4=8, usable5=8, usable6=8, fewer4=8, garbage=16)
FOCAL, IMG = 1265.0, 512.0
PERTURB = 3


def _hands(rng, n):
    sys.path.insert(0, os.path.join(ROOT, "arbitrary-hands-3d-reconstruction_b200"))
    from acr_b200.synth import make_synthetic_mano
    from oracle import mano_ref
    assets = {s: make_synthetic_mano(s) for s in ("left", "right")}
    poses = (0.5 * rng.standard_normal((n, 48))).astype(np.float32)
    betas = rng.standard_normal((n, 10)).astype(np.float32)
    cam = np.stack([rng.uniform(0.3, 3.0, n), rng.uniform(-.6, .6, n), rng.uniform(-.6, .6, n)], 1).astype(np.float32)
    out = mano_ref.mano_wrapper_forward(assets, poses, betas, n // 2, n - n // 2, cam)
    return out["j3d"].astype(np.float32), out["pj2d"].astype(np.float32)


def _inputs(rng):
    j3d, pj2d, cls = [], [], []
    total = sum(v for k, v in COUNTS.items() if k != "garbage")
    J, P = _hands(rng, total)
    k = 0
    for name, cnt in COUNTS.items():
        ci = CLASSES.index(name)
        for _ in range(cnt):
            if name == "garbage":
                s = (rng.standard_normal((21, 3)) * 0.05).astype(np.float32)
                p = rng.uniform(-1, 1, (21, 2)).astype(np.float32)
            else:
                s, p = J[k].copy(), P[k].copy()
                k += 1
                if name == "outliers":
                    m = rng.integers(1, 9)
                    idx = rng.choice(21, m, replace=False)
                    px = rng.uniform(30, 150, (m, 2)) * rng.choice([-1, 1], (m, 2))
                    p[idx] = (p[idx] + px / (IMG / 2)).astype(np.float32)
                elif name == "masked":
                    m = rng.integers(1, 8)
                    idx = rng.choice(21, m, replace=False)
                    p[idx[: (m + 1) // 2], 1] = rng.uniform(-1.6, -1.01)   # pixel y < -2: above the image
                    s[idx[(m + 1) // 2:], 2] = -2.0                       # z == -2: the reference's 3D mask
                elif name in ("usable4", "usable5", "usable6", "fewer4"):
                    keep = int(name[-1]) if name != "fewer4" else int(rng.integers(0, 4))
                    drop = rng.choice(21, 21 - keep, replace=False)
                    p[drop, 1] = -1.5
            j3d.append(s)
            pj2d.append(p)
            cls.append(ci)
    g = np.load(os.path.join(ROOT, "tests", "golden", "mano_golden.npz"))
    for i in range(g["j3d"].shape[0]):
        j3d.append(g["j3d"][i].astype(np.float32))
        pj2d.append(g["pj2d"][i].astype(np.float32))
        cls.append(CLASSES.index("mano_golden"))
    return np.stack(j3d), np.stack(pj2d), np.array(cls, np.int32)


def main():
    import cv2
    sys.path.insert(0, ROOT)
    from oracle import mano_ref, pnp_ref
    rng = np.random.default_rng(20261015)
    j3d, pj2d, cls = _inputs(rng)
    n = j3d.shape[0]
    K = np.eye(3)
    K[0, 0] = K[1, 1] = FOCAL
    K[:2, 2] = IMG // 2
    lsq = mano_ref.cam_trans_lstsq(j3d, pj2d, FOCAL, IMG)

    def ransac(S, J):
        r = cv2.solvePnPRansac(S, J, K, None, flags=cv2.SOLVEPNP_EPNP, reprojectionError=20, iterationsCount=100)
        return (None, None) if r[3] is None else (r[2][:, 0], r[3][:, 0])

    t = np.zeros((n, 3))
    mask = np.zeros(n, np.int32)
    status = np.zeros(n, np.int32)
    cond = np.zeros(n)
    stable = np.ones(n, bool)
    prng = np.random.default_rng(7)
    j2d = ((pj2d + 1) * np.float32(IMG / 2)).astype(np.float32)          # acr/utils.py:404
    for i in range(n):
        use = (j2d[i, :, 1] > -2.0) & (j3d[i, :, 2] != -2.0)
        joints = np.nonzero(use)[0]
        if use.sum() < 4:
            t[i], status[i] = -1, pnp_ref.ST_INVALID
            continue
        S, J = j3d[i][use], j2d[i][use]
        ti, inl = ransac(S, J)
        if use.sum() == 4:                  # cv2 runs P3P; recorded, the device returns the least squares
            t[i], status[i] = ti if ti is not None else lsq[i], pnp_ref.ST_LSTSQ_4
            continue
        if ti is None:
            t[i], status[i] = lsq[i], pnp_ref.ST_LSTSQ_FAIL
            continue
        t[i], status[i], mask[i] = ti, pnp_ref.ST_EPNP, int(np.sum(1 << joints[inl]))
        for _ in range(PERTURB):
            Sp = (S * (1 + 1e-6 * prng.standard_normal(S.shape))).astype(np.float32)
            Jp = (J * (1 + 1e-7 * prng.standard_normal(J.shape))).astype(np.float32)
            tp, ip = ransac(Sp, Jp)
            if tp is None or not np.array_equal(np.sort(ip), np.sort(inl)):
                stable[i] = False
                cond[i] = np.inf
                continue
            cond[i] = max(cond[i], np.abs(tp - ti).max() / np.abs(ti).max())
    np.savez_compressed(OUT, j3d=j3d, pj2d=pj2d, classes=cls, class_names=np.array(CLASSES), t=t, inlier_mask=mask,
                        status=status, cond=cond, mask_stable=stable, focal=FOCAL, img_size=IMG)
    print("wrote", OUT, n, "hands;", {c: int((cls == k).sum()) for k, c in enumerate(CLASSES)},
          "status", np.bincount(status, minlength=4).tolist(), "unstable masks", int((~stable).sum()))


if __name__ == "__main__":
    main()
