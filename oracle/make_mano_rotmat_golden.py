#!/usr/bin/env python
"""Generate tests/golden/mano_rotmat_golden.npz by running the UNMODIFIED reference ManoLayer on the CPU: its
rotation-matrix branch (use_pca=False, joint_rot_mode='rotmat', mano/manolayer.py:151-162, batch_rotprojs :436-453)
and root_palm (:248-250), in both pose modes.  Runs only where a checkout of the reference exists; the npz it
writes is committed and is all the GPU tests read.

    python oracle/make_mano_rotmat_golden.py REFERENCE_ROOT

Per side: one batch of (n,16,3,3) matrices mixing five input classes per joint (exact rotations, rotations + 0.1
sigma noise, det < 0 matrices, 2 R, plain Gaussian matrices; hand 0 is all exact rotations), one batch of (n,48)
axis angles, betas and th_trans, and the outputs of every case in CASES (vertices at VERT_IDX only).
"""
import os
import sys

import numpy as np

ROOT = os.path.abspath(os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
OUT = os.path.join(ROOT, "tests", "golden", "mano_rotmat_golden.npz")
N = 10
CLASSES = ("exact", "noisy", "negdet", "scaled", "gaussian")
# vertices kept in the fixture (it stays small): every 8th, plus the palm and fingertip vertices
VERT_IDX = np.array(sorted(set(range(0, 778, 8)) | {22, 95, 317, 444, 445, 556, 673, 745}), np.int64)
# name -> (pose mode, center_idx, root_palm, th_trans)
CASES = {
    "rotmat_c9": ("rotmat", 9, False, False),
    "rotmat_c9_palm": ("rotmat", 9, True, False),
    "rotmat_none": ("rotmat", None, False, False),
    "rotmat_none_palm": ("rotmat", None, True, False),
    "rotmat_trans": ("rotmat", 9, False, True),
    "rotmat_trans_palm": ("rotmat", 9, True, True),
    "axisang_c9_palm": ("axisang", 9, True, False),
    "axisang_none_palm": ("axisang", None, True, False),
    "axisang_trans_palm": ("axisang", 9, True, True),
}


def inputs(batch_rodrigues, torch, side):
    g = np.random.default_rng({"left": 11, "right": 12}[side])
    aa = (g.standard_normal((N * 16, 3)) * 0.8).astype(np.float32)
    R = batch_rodrigues(torch.from_numpy(aa)).numpy().reshape(N, 16, 3, 3)
    cls = (np.arange(N)[:, None] + np.arange(16)[None, :]) % len(CLASSES)
    cls[0] = 0
    noise = g.standard_normal((N, 16, 3, 3)).astype(np.float32)
    mats = np.where((cls == 0)[..., None, None], R, 0)
    mats = np.where((cls == 1)[..., None, None], R + 0.1 * noise, mats)
    mats = np.where((cls == 2)[..., None, None], -(R + 0.05 * noise), mats)
    mats = np.where((cls == 3)[..., None, None], 2 * R, mats)
    mats = np.where((cls == 4)[..., None, None], noise, mats).astype(np.float32)
    pose_aa = (g.standard_normal((N, 48)) * 0.5).astype(np.float32)
    betas = g.standard_normal((N, 10)).astype(np.float32)
    trans = (g.standard_normal((N, 3)) * 0.1).astype(np.float32)
    return dict(mats=mats, classes=cls.astype(np.int32), aa=pose_aa, betas=betas, trans=trans)


def main(ref_root):
    sys.path.insert(0, ROOT)
    from oracle import ref_harness
    torch = ref_harness.import_reference(ref_root, "make_mano_rotmat_golden")
    import mano.manolayer as ml
    out = {"N": N, "vert_idx": VERT_IDX, "classes_names": np.array(CLASSES), "case_names": np.array(list(CASES))}
    for side in ("right", "left"):
        d = inputs(ml.batch_rodrigues, torch, side)
        for k, v in d.items():
            out[f"{side}__{k}"] = v
        for name, (mode, center, palm, use_trans) in CASES.items():
            if mode == "rotmat":
                layer = ml.ManoLayer(center_idx=center, side=side, use_pca=False, joint_rot_mode="rotmat")
                pose = torch.from_numpy(d["mats"])
            else:
                layer = ml.ManoLayer(center_idx=center, side=side, use_pca=False, flat_hand_mean=False, ncomps=45)
                pose = torch.from_numpy(d["aa"])
            kw = dict(th_betas=torch.from_numpy(d["betas"]), root_palm=torch.Tensor([int(palm)]))
            if use_trans:
                kw["th_trans"] = torch.from_numpy(d["trans"])
            with torch.no_grad():
                v, j, c = layer(pose, **kw)
            out[f"{side}__{name}__verts"] = v.numpy()[:, VERT_IDX]
            out[f"{side}__{name}__joints"] = j.numpy()
            if c is not None:
                out[f"{side}__{name}__center"] = c.numpy()
        if side == "right":
            out["buffer_names"] = np.array(sorted(n for n, _ in
                                                  ml.ManoLayer(use_pca=False, joint_rot_mode="rotmat").named_buffers()))
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, len(out), "arrays")


if __name__ == "__main__":
    if len(sys.argv) != 2:
        sys.exit(__doc__)
    main(sys.argv[1])
