"""ORACLE (test infrastructure, never on the product path).

CPU/numpy restatement of the reference MANO layer as ACR configures it
(``use_pca=False, flat_hand_mean=False, root_rot_mode='axisang',
center_idx=9``; /root/reference/acr/mano_wrapper.py:17-35) and of the
weak-perspective projection that follows it.  Pinned against the reference
through tests/golden/mano_golden.npz.

Reference functions restated (in /root/reference/):
  ManoLayer.forward            mano/manolayer.py:104-276
  th_posemap_axisang           mano/manolayer.py:281-287
  subtract_flat_id             mano/manolayer.py:308-316
  MANOWrapper.forward          acr/mano_wrapper.py:37-50 (left shapedirs x-flip :35)
  batch_orth_proj              acr/utils.py:384-390
  convert_kp2d_from_input_to_orgimg  acr/utils.py:392-397
"""
import numpy as np

from .rotation_ref import batch_rodrigues

F = np.float32


def _dtype(dtype):
    """The type a function computes in: its ``dtype`` argument, or the module's F (float32, the reference's)."""
    return globals()["F"] if dtype is None else dtype
LEVELS = ([1, 4, 7, 10, 13], [2, 5, 8, 11, 14], [3, 6, 9, 12, 15])      # manolayer.py:191-193
CHAIN_REORDER = [0, 1, 6, 11, 2, 7, 12, 3, 8, 13, 4, 9, 14, 5, 10, 15]   # manolayer.py:222
JOINT_REORDER = [0, 13, 14, 15, 16, 1, 2, 3, 17, 4, 5, 6, 18, 10, 11, 12, 19, 7, 8, 9, 20]  # :254
TIPS = {"right": [745, 317, 444, 556, 673], "left": [745, 317, 445, 556, 673]}  # :244-247


def _with_zeros(m34):
    pad = np.zeros((m34.shape[0], 1, 4), m34.dtype)
    pad[:, 0, 3] = 1
    return np.concatenate([m34, pad], 1)


def mano_forward(asset, pose, betas, side, center_idx=9, flip_shapedirs_x=None, dtype=None, detail=None):
    """pose (n,48) axis-angle [root3 | hand45], betas (n,10) -> verts (n,778,3),
    joints (n,21,3), center (n,1,3).

    ``flip_shapedirs_x`` defaults to ``side == 'left'`` which is what MANOWrapper does
    to the left layer after construction (acr/mano_wrapper.py:35).
    ``dtype`` is the type of every operation: float32 (the default, which the goldens pin) is the reference's;
    float64 is the statement the kernels' per-element bounds are taken against (tests/tail_ref.py).  A dict passed
    as ``detail`` receives the intermediates those bounds are built from: full_pose (n,16,3), R (n,16,3,3) local
    rotations, J (n,16,3) rest joints, v_posed (n,778,3), G (n,16,4,4) global transforms, A (n,16,4,4) with the rest
    pose removed, and the model arrays as used (shapedirs after the flip)."""
    F = _dtype(dtype)
    pose = np.asarray(pose, F).reshape(-1, 48)
    betas = np.asarray(betas, F).reshape(-1, 10)
    n = pose.shape[0]
    shapedirs = np.asarray(asset["shapedirs"], F).copy()
    if flip_shapedirs_x is None:
        flip_shapedirs_x = side == "left"
    if flip_shapedirs_x:
        shapedirs[:, 0, :] *= -1
    posedirs = np.asarray(asset["posedirs"], F)
    v_template = np.asarray(asset["v_template"], F)
    Jreg = np.asarray(asset["J_regressor"], F)
    weights = np.asarray(asset["weights"], F)
    hands_mean = np.asarray(asset["hands_mean"], F)

    # (i) full pose = [root | mean + hand]            manolayer.py:125-137
    full = np.concatenate([pose[:, :3], hands_mean[None] + pose[:, 3:]], 1).astype(F)
    # (ii) 16 rotations; pose_map = R - I for joints 1..15      :140-143, 281-287
    rots = batch_rodrigues(full.reshape(-1, 3), F).reshape(n, 16, 9)
    root_rot = rots[:, 0].reshape(n, 3, 3)
    rot_map = rots[:, 1:].reshape(n, 135)
    pose_map = rot_map - np.tile(np.eye(3, dtype=F).reshape(9), 15)[None]
    # (iii) shape blend, (iv) joint regression              :175-178
    v_shaped = np.einsum("vck,nk->nvc", shapedirs, betas).astype(F) + v_template[None]
    J = np.einsum("jv,nvc->njc", Jreg, v_shaped).astype(F)
    # (v) pose blend                                            :181-182
    v_posed = v_shaped + np.einsum("vck,nk->nvc", posedirs, pose_map).astype(F)
    # (vi) kinematic chain by levels                            :187-223
    all_rots = rot_map.reshape(n, 15, 3, 3)
    root_tr = _with_zeros(np.concatenate([root_rot, J[:, 0].reshape(n, 3, 1)], 2))
    chain = [root_tr[:, None]]
    prev_tr = np.repeat(root_tr[:, None], 5, 1)
    prev_j = np.repeat(J[:, 0][:, None], 5, 1)
    for lev in LEVELS:
        r = all_rots[:, [i - 1 for i in lev]]
        jl = J[:, lev]
        rel = np.concatenate([r, (jl - prev_j)[..., None]], 3).reshape(-1, 3, 4)
        cur = np.matmul(prev_tr.reshape(-1, 4, 4), _with_zeros(rel)).astype(F).reshape(n, 5, 4, 4)
        chain.append(cur)
        prev_tr, prev_j = cur, jl
    G = np.concatenate(chain, 1)[:, CHAIN_REORDER]                       # (n,16,4,4)
    # (vii) remove rest-pose joint location                     :226-228
    jh = np.concatenate([J, np.zeros((n, 16, 1), F)], 2)
    tmp = np.matmul(G, jh[..., None]).astype(F)                          # (n,16,4,1)
    G2 = G.copy()
    G2[:, :, :, 3:4] -= tmp
    # (viii)+(ix) linear blend skinning                         :230-240
    T = np.einsum("njab,vj->nvab", G2, weights).astype(F)               # (n,778,4,4)
    vh = np.concatenate([v_posed, np.ones((n, 778, 1), F)], 2)
    verts = np.einsum("nvab,nvb->nva", T, vh).astype(F)[:, :, :3]
    # (x) joints = chain translations + 5 fingertip vertices     :241-251
    jtr = np.concatenate([G[:, :, :3, 3], verts[:, TIPS[side]]], 1)
    # (xi) reorder, (xii) centre on joint ``center_idx``         :254-261
    jtr = jtr[:, JOINT_REORDER]
    if detail is not None:
        detail.update(full_pose=full.reshape(n, 16, 3), R=rots.reshape(n, 16, 3, 3), J=J, v_posed=v_posed, G=G, A=G2,
                      shapedirs=shapedirs, posedirs=posedirs, v_template=v_template, J_regressor=Jreg, weights=weights)
    center = None
    if center_idx is not None:
        center = jtr[:, center_idx][:, None].copy()
        jtr = jtr - center
        verts = verts - center
    return verts.astype(F), jtr.astype(F), center


def project(verts, j3d, cam, offsets=None):
    """batch_orth_proj for vertices (keeps z) and joints, plus the mapping of pj2d
    back to original-image pixels (acr/utils.py:384-397, 399-412 minus cam_trans)."""
    cam = np.asarray(cam, F).reshape(-1, 1, 3)
    vc = verts[:, :, :2] * cam[:, :, 0:1] + cam[:, :, 1:]
    verts_camed = np.concatenate([vc, verts[:, :, 2:3]], -1).astype(F)
    pj2d = (j3d[:, :, :2] * cam[:, :, 0:1] + cam[:, :, 1:]).astype(F)
    out = dict(verts_camed=verts_camed, pj2d=pj2d)
    if offsets is not None:
        off = np.asarray(offsets, F)
        pad, crop, padt = off[:, :2], off[:, 2:6], off[:, 6:10]
        lt = np.stack([crop[:, 3] - padt[:, 3], crop[:, 0] - padt[:, 0]], 1)
        out["pj2d_org"] = ((pj2d + 1) * pad[:, None] / 2 + lt[:, None]).astype(F)
    return out


def cam_trans_lstsq(j3d, pj2d, focal_length=1265.0, img_size=512.0):
    """Closed-form camera translation per hand: estimate_translation_np (acr/utils.py:430-472) with the
    joint-validity tests of estimate_translation (:489-500): pixel y > -2 and z != -2; <4 valid -> (-1,-1,-1)
    (ROMP's INVALID_TRANS; the reference's own constant is undefined, :425,504).  float64 like numpy."""
    j3d = np.asarray(j3d, F)
    j2d = ((np.asarray(pj2d, F) + 1) * F(img_size / 2)).astype(F)       # acr/utils.py:404
    out = np.zeros((j3d.shape[0], 3), np.float64)
    f = np.array([focal_length, focal_length], np.float64)
    center = np.array([img_size / 2.0, img_size / 2.0])
    for i in range(j3d.shape[0]):
        m = (j2d[i, :, -1] > -2.0) & (j3d[i, :, -1] != -2.0)
        if m.sum() < 4:
            out[i] = -1
            continue
        S, J = j3d[i][m], j2d[i][m]
        n = S.shape[0]
        Z = np.reshape(np.tile(S[:, 2], (2, 1)).T, -1)
        XY = np.reshape(S[:, 0:2], -1)
        O = np.tile(center, n)
        Fv = np.tile(f, n)
        Q = np.array([Fv * np.tile(np.array([1, 0]), n), Fv * np.tile(np.array([0, 1]), n), O - np.reshape(J, -1)]).T
        c = (np.reshape(J, -1) - O) * Z - Fv * XY
        out[i] = np.linalg.solve(Q.T @ Q, Q.T @ c)
    return out.astype(F)


def mano_wrapper_forward(assets, poses, betas, L, R, cam=None, offsets=None):
    """MANOWrapper.forward: rows [:L] go through the left layer, [L:L+R] through the
    right one; results concatenated left-first (acr/mano_wrapper.py:40-48)."""
    lv, lj, _ = mano_forward(assets["left"], poses[:L], betas[:L], "left")
    rv, rj, _ = mano_forward(assets["right"], poses[L:L + R], betas[L:L + R], "right")
    out = dict(verts=np.concatenate([lv, rv]), j3d=np.concatenate([lj, rj]),
               output_hand_type=np.concatenate([np.zeros(L), np.ones(R)]).astype(np.int32))
    if cam is not None:
        out.update(project(out["verts"], out["j3d"], cam, offsets))
    return out
