"""Thin Python wrappers over the C ABI for the fp32 tail of the hot path
(rotations, centre parsing, MANO).  torch only owns the memory and the stream."""
from __future__ import annotations

from typing import Dict, Optional

import numpy as np
import torch

from . import lib as L


# ----------------------------------------------------------------------------- MANO model
def pack_mano_model(asset: Dict[str, np.ndarray], flip_x: bool, device) -> torch.Tensor:
    """Pack a MANO asset (dict of numpy arrays, see acr_b200.synth.make_synthetic_mano or
    mano.assets.load_mano_pkl) into the kernel's constant layout and upload it."""
    lib = L.load()
    n = lib.acr_b200_mano_model_floats()
    out = np.zeros(n, np.float32)
    arrs = [np.ascontiguousarray(asset[k], np.float32) for k in
            ("shapedirs", "posedirs", "v_template", "J_regressor", "weights", "hands_mean")]
    assert arrs[0].shape == (778, 3, 10) and arrs[1].shape == (778, 3, 135) and arrs[2].shape == (778, 3)
    assert arrs[3].shape == (16, 778) and arrs[4].shape == (778, 16) and arrs[5].shape == (45,)
    L.check(lib.acr_b200_mano_pack_model(*[a.ctypes.data for a in arrs], int(bool(flip_x)), out.ctypes.data),
            "mano_pack_model")
    return torch.from_numpy(out).to(device)


def mano_forward(model_l: Optional[torch.Tensor], model_r: Optional[torch.Tensor], poses: torch.Tensor,
                 betas: torch.Tensor, hand_type: Optional[torch.Tensor] = None, default_side: int = 1,
                 center_idx: Optional[int] = 9, cam: Optional[torch.Tensor] = None,
                 offsets: Optional[torch.Tensor] = None, n_dev: Optional[torch.Tensor] = None,
                 want_camed: bool = True, peers=None, counts: Optional[torch.Tensor] = None):
    """-> dict(verts, joints, center[, verts_camed, pj2d, pj2d_org]); all (n, ...) fp32 CUDA tensors.
    ``peers`` (acr_b200.dist.PeerVertexGather) fuses the cross-GPU vertex all-gather into the kernel; ``counts``
    (8 int32, acr_b200_parse's row counts) then travels with the vertices."""
    dev = L.require_cuda(poses, betas, hand_type, cam, offsets, n_dev, model_l, model_r)
    n = poses.shape[0]
    poses = poses.contiguous().float()
    betas = betas.contiguous().float()
    out = dict(verts=torch.empty(n, 778, 3, device=dev), joints=torch.empty(n, 21, 3, device=dev),
               center=torch.empty(n, 1, 3, device=dev))
    if cam is not None:
        cam = cam.contiguous().float()
        if want_camed:
            out["verts_camed"] = torch.empty(n, 778, 3, device=dev)
        out["pj2d"] = torch.empty(n, 21, 2, device=dev)
        if offsets is not None:
            offsets = offsets.contiguous().float()
            out["pj2d_org"] = torch.empty(n, 21, 2, device=dev)
    if hand_type is not None:
        hand_type = hand_type.contiguous().to(torch.int32)
    if n == 0:
        return out
    lib = L.load()
    common = (L.ptr(model_l), L.ptr(model_r), L.ptr(poses), L.ptr(betas), L.ptr(hand_type),
              int(default_side), L.ptr(n_dev), n, -1 if center_idx is None else int(center_idx),
              L.ptr(cam), L.ptr(offsets), L.ptr(out["verts"]), L.ptr(out["joints"]),
              L.ptr(out["center"]), L.ptr(out.get("verts_camed")), L.ptr(out.get("pj2d")),
              L.ptr(out.get("pj2d_org")))
    with L.on(dev):
        if peers is None:
            rc = lib.acr_b200_mano_forward(*common, L.current_stream(dev))
        else:
            assert n <= peers.rows, "gather buffer too small"
            import ctypes as C
            rc = lib.acr_b200_mano_forward_gather(*common, L.ptr(counts), C.byref(peers.desc), L.current_stream(dev))
            if rc == L.OK:
                peers.note_launch()
    L.check(rc, "mano_forward")
    return out


def mano_backward(model: torch.Tensor, side: int, poses: torch.Tensor, betas: torch.Tensor,
                  center_idx: Optional[int], dverts: Optional[torch.Tensor], djoints: Optional[torch.Tensor],
                  dcenter: Optional[torch.Tensor], want_poses: bool = True, want_betas: bool = True):
    """Gradient of one side's ``mano_forward`` (verts, joints, center) -> (dposes (n,48), dbetas (n,10)); a
    cotangent of None is zero, an output not wanted comes back as None."""
    dev = L.require_cuda(model, poses, betas, dverts, djoints, dcenter)
    n = poses.shape[0]
    poses = poses.contiguous().float()
    betas = betas.contiguous().float()
    dverts, djoints, dcenter = [None if t is None else t.contiguous().float() for t in (dverts, djoints, dcenter)]
    dposes = torch.empty(n, 48, device=dev) if want_poses else None
    dbetas = torch.empty(n, 10, device=dev) if want_betas else None
    if n == 0 or not (want_poses or want_betas):
        return dposes, dbetas
    lib = L.load()
    ws = None
    if dverts is not None or djoints is not None:
        ws = torch.empty(int(lib.acr_b200_mano_backward_workspace_floats(n)), device=dev)
    with L.on(dev):
        rc = lib.acr_b200_mano_backward(L.ptr(model), int(side), L.ptr(poses), L.ptr(betas), n,
                                        -1 if center_idx is None else int(center_idx), L.ptr(dverts), L.ptr(djoints),
                                        L.ptr(dcenter), L.ptr(ws), L.ptr(dposes), L.ptr(dbetas), L.current_stream(dev))
    L.check(rc, "mano_backward")
    return dposes, dbetas


def mano_layer_forward(model: torch.Tensor, side: int, pose: torch.Tensor, pose_mode: int, betas: torch.Tensor,
                       center_idx: Optional[int], root_palm: bool):
    """One side's ManoLayer.forward for any pose input (``L.POSE_AXISANG``: (n,48) without the mean pose;
    ``L.POSE_ROTMAT``: (n,16,3,3) matrices, projected onto SO(3)) and ``root_palm`` -> (verts, joints, center)."""
    dev = L.require_cuda(model, pose, betas)
    n = pose.shape[0]
    pose = pose.contiguous().float()
    betas = betas.contiguous().float()
    verts, joints = torch.empty(n, 778, 3, device=dev), torch.empty(n, 21, 3, device=dev)
    center = torch.empty(n, 1, 3, device=dev)
    lib = L.load()
    with L.on(dev):
        rc = lib.acr_b200_mano_layer_forward(L.ptr(model), int(side), L.ptr(pose), int(pose_mode), L.ptr(betas), n,
                                             -1 if center_idx is None else int(center_idx), int(bool(root_palm)),
                                             L.ptr(verts), L.ptr(joints), L.ptr(center), L.current_stream(dev))
    L.check(rc, "mano_layer_forward")
    return verts, joints, center


def mano_layer_backward(model: torch.Tensor, side: int, pose: torch.Tensor, pose_mode: int, betas: torch.Tensor,
                        center_idx: Optional[int], root_palm: bool, dverts: Optional[torch.Tensor],
                        djoints: Optional[torch.Tensor], dcenter: Optional[torch.Tensor], want_pose: bool = True,
                        want_betas: bool = True):
    """Gradient of ``mano_layer_forward`` -> (dpose shaped like pose, dbetas (n,10)); a cotangent of None is zero,
    an output not wanted comes back as None."""
    dev = L.require_cuda(model, pose, betas, dverts, djoints, dcenter)
    n = pose.shape[0]
    pose = pose.contiguous().float()
    betas = betas.contiguous().float()
    dverts, djoints, dcenter = [None if t is None else t.contiguous().float() for t in (dverts, djoints, dcenter)]
    dpose = torch.empty(pose.shape, device=dev) if want_pose else None
    dbetas = torch.empty(n, 10, device=dev) if want_betas else None
    lib = L.load()
    ws = None
    if n and (dverts is not None or djoints is not None):
        ws = torch.empty(int(lib.acr_b200_mano_backward_workspace_floats(n)), device=dev)
    with L.on(dev):
        rc = lib.acr_b200_mano_layer_backward(L.ptr(model), int(side), L.ptr(pose), int(pose_mode), L.ptr(betas), n,
                                              -1 if center_idx is None else int(center_idx), int(bool(root_palm)),
                                              L.ptr(dverts), L.ptr(djoints), L.ptr(dcenter), L.ptr(ws), L.ptr(dpose),
                                              L.ptr(dbetas), L.current_stream(dev))
    L.check(rc, "mano_layer_backward")
    return dpose, dbetas


def mano_layer_jvp(model: torch.Tensor, side: int, pose: torch.Tensor, pose_mode: int, betas: torch.Tensor,
                   center_idx: Optional[int], root_palm: bool, tpose: Optional[torch.Tensor],
                   tbetas: Optional[torch.Tensor], want_verts: bool = True):
    """Forward-mode derivative of ``mano_layer_forward``: ``tpose`` (T, n, *pose.shape[1:]) and ``tbetas`` (T, n, 10)
    are T tangents per hand (None is zero) -> (tverts (T,n,778,3) or None, tjoints (T,n,21,3), tcenter (T,n,1,3)).
    Without ``want_verts`` the kernel computes the joints only (no vertex pass)."""
    dev = L.require_cuda(model, pose, betas, tpose, tbetas)
    n = pose.shape[0]
    T = (tpose if tpose is not None else tbetas).shape[0] if (tpose is not None or tbetas is not None) else 0
    pose = pose.contiguous().float()
    betas = betas.contiguous().float()
    tpose, tbetas = [None if t is None else t.contiguous().float() for t in (tpose, tbetas)]
    assert tpose is None or tpose.shape == (T,) + tuple(pose.shape)
    assert tbetas is None or tbetas.shape == (T, n, 10)
    idle = T == 0 or n == 0 or (tpose is None and tbetas is None)
    alloc = torch.zeros if idle else torch.empty     # the kernel writes every element
    tverts = alloc(T, n, 778, 3, device=dev) if want_verts else None
    tjoints, tcenter = alloc(T, n, 21, 3, device=dev), alloc(T, n, 1, 3, device=dev)
    if idle:
        return tverts, tjoints, tcenter
    lib = L.load()
    with L.on(dev):
        rc = lib.acr_b200_mano_layer_jvp(L.ptr(model), int(side), L.ptr(pose), int(pose_mode), L.ptr(betas), n,
                                         -1 if center_idx is None else int(center_idx), int(bool(root_palm)), T,
                                         L.ptr(tpose), L.ptr(tbetas), None, None, None, L.ptr(tverts), L.ptr(tjoints),
                                         L.ptr(tcenter), L.current_stream(dev))
    L.check(rc, "mano_layer_jvp")
    return tverts, tjoints, tcenter


def cam_trans(j3d: torch.Tensor, pj2d: torch.Tensor, focal_length: float = 1265.0, img_size: float = 512.0,
              n_dev: Optional[torch.Tensor] = None) -> torch.Tensor:
    """(n,21,3), (n,21,2) -> (n,3) camera translation (closed-form least squares on the device)."""
    dev = L.require_cuda(j3d, pj2d, n_dev)
    n = j3d.shape[0]
    out = torch.empty(n, 3, device=j3d.device)
    if n:
        with L.on(dev):
            L.check(L.load().acr_b200_cam_trans(L.ptr(j3d.contiguous().float()), L.ptr(pj2d.contiguous().float()),
                                                L.ptr(n_dev), n, float(focal_length), float(img_size), L.ptr(out),
                                                L.current_stream(dev)), "cam_trans")
    return out


def cam_trans_pnp(j3d: torch.Tensor, pj2d: torch.Tensor, focal_length: float = 1265.0, img_size: float = 512.0,
                  n_dev: Optional[torch.Tensor] = None, return_inliers: bool = False):
    """(n,21,3), (n,21,2) -> (n,3) camera translation as the reference's cv2.solvePnPRansac(EPNP,
    reprojectionError=20, iterationsCount=100) computes it, on the device; with ``return_inliers`` also the (n,)
    int32 inlier bitmask over the 21 joints (0 where the result is the least squares or (-1,-1,-1))."""
    dev = L.require_cuda(j3d, pj2d, n_dev)
    n = j3d.shape[0]
    out = torch.empty(n, 3, device=j3d.device)
    inl = torch.empty(n, dtype=torch.int32, device=j3d.device) if return_inliers else None
    if n:
        with L.on(dev):
            L.check(L.load().acr_b200_cam_trans_pnp(L.ptr(j3d.contiguous().float()), L.ptr(pj2d.contiguous().float()),
                                                    L.ptr(n_dev), n, float(focal_length), float(img_size), L.ptr(out),
                                                    L.ptr(inl), L.current_stream(dev)), "cam_trans_pnp")
    return (out, inl) if return_inliers else out


def cam_trans_mode(mode: str, j3d: torch.Tensor, pj2d: torch.Tensor, focal_length: float = 1265.0,
                   img_size: float = 512.0, n_dev: Optional[torch.Tensor] = None) -> Optional[torch.Tensor]:
    """``args().cam_trans_mode`` dispatch: 'lstsq' -> cam_trans, 'pnp' -> cam_trans_pnp, anything else
    ('none') -> None."""
    if mode == "lstsq":
        return cam_trans(j3d, pj2d, focal_length, img_size, n_dev=n_dev)
    if mode == "pnp":
        return cam_trans_pnp(j3d, pj2d, focal_length, img_size, n_dev=n_dev)
    return None


class OneEuroState:
    """Device-side history of the temporal filter (one bank per hand type); zero = no history."""

    def __init__(self, device):
        self.state = torch.zeros(int(L.load().acr_b200_one_euro_state_floats()), device=device)

    def reset(self) -> None:
        self.state.zero_()


def one_euro_smooth(poses: torch.Tensor, betas: torch.Tensor, state: OneEuroState, smooth_coeff: float = 4.0,
                    hand_type: Optional[torch.Tensor] = None, detection_flag: Optional[torch.Tensor] = None,
                    n_dev: Optional[torch.Tensor] = None) -> None:
    """In-place temporal smoothing of (n,48) poses and (n,10) betas (drop-in for acr.utils.smooth_results
    applied per hand as in acr/main.py:69-83).  The state has one bank per hand type, so at most two rows (one per
    type; row r uses bank r without ``hand_type``): more raise AcrB200Error, like the C entry point."""
    dev = L.require_cuda(poses, betas, hand_type, detection_flag, n_dev, state.state)
    assert poses.is_contiguous() and betas.is_contiguous() and poses.dtype == betas.dtype == torch.float32
    if poses.shape[0] > 2:
        raise L.AcrB200Error(f"one_euro_smooth: at most 2 rows, one per hand type (got {poses.shape[0]})")
    if poses.shape[0]:
        with L.on(dev):
            L.check(L.load().acr_b200_one_euro_smooth(L.ptr(poses), L.ptr(betas), L.ptr(hand_type), L.ptr(detection_flag),
                                                      L.ptr(n_dev), poses.shape[0], L.ptr(state.state), float(smooth_coeff),
                                                      L.current_stream(dev)), "one_euro_smooth")


# ------------------------------------------------------------------------------ rotations
def rot6d_to_aa(rot6d: torch.Tensor) -> torch.Tensor:
    """(N, 6*J) -> (N, 3*J); drop-in for acr.utils.rot6D_to_angular."""
    dev = L.require_cuda(rot6d)
    x = rot6d.contiguous().float()
    nrot = x.numel() // 6
    out = torch.empty(x.shape[0], x.shape[1] // 2, device=x.device)
    if nrot:
        with L.on(dev):
            L.check(L.load().acr_b200_rot6d_to_aa(L.ptr(x), nrot, L.ptr(out), L.current_stream(dev)), "rot6d_to_aa")
    return out


def rodrigues(aa: torch.Tensor) -> torch.Tensor:
    """(M,3) -> (M,9); drop-in for mano.manolayer.batch_rodrigues."""
    dev = L.require_cuda(aa)
    x = aa.contiguous().float()
    out = torch.empty(x.shape[0], 9, device=x.device)
    if x.shape[0]:
        with L.on(dev):
            L.check(L.load().acr_b200_rodrigues(L.ptr(x), x.shape[0], L.ptr(out), L.current_stream(dev)), "rodrigues")
    return out


# --------------------------------------------------------------------------------- parse
MAX_HANDS_PER_SIDE = 16


class ParseBuffers:
    """Worst-case (2KB rows: up to K hands per image and side) output buffers of acr_b200_parse (K = 1) /
    acr_b200_parse_topk, allocated once per (batch size, K).  ``top_idx`` / ``top_score`` are (B, 2) at K = 1 and
    (B, 2, K) above."""

    def __init__(self, B: int, device, K: int = 1):
        if not 1 <= int(K) <= MAX_HANDS_PER_SIDE:
            raise ValueError(f"hands per side must be in 1..{MAX_HANDS_PER_SIDE}, got {K}")
        f = lambda *s: torch.zeros(*s, device=device, dtype=torch.float32)
        i64 = lambda *s: torch.zeros(*s, device=device, dtype=torch.int64)
        i32 = lambda *s: torch.zeros(*s, device=device, dtype=torch.int32)
        K = int(K)
        R = 2 * K * B
        self.B, self.K = B, K
        self.params_pred, self.cam, self.global_orient = f(R, 109), f(R, 3), f(R, 3)
        self.hand_pose, self.betas, self.poses = f(R, 45), f(R, 10), f(R, 48)
        self.detection_flag, self.reorganize_idx, self.batch_ids = f(R), i64(R), i64(R)
        self.centers_pred, self.centers_conf, self.hand_type = i64(R, 2), f(R), i32(R)
        self.offsets_out, self.counts = f(R, 10), i32(8)
        top = (B, 2) if K == 1 else (B, 2, K)
        self.top_idx, self.top_score, self.row_src = i32(*top), f(*top), i32(R, 4)

    def struct(self) -> L.ParseOut:
        o = L.ParseOut()
        for name, _ in L.ParseOut._fields_:
            setattr(o, name, getattr(self, name).data_ptr())
        return o


def parse_maps(maps: Dict[str, tuple], B: int, bufs: ParseBuffers, meta_batch_ids: Optional[torch.Tensor],
               offsets: Optional[torch.Tensor], conf_thresh: float = 0.35, K: int = 1) -> None:
    """maps[name] = (fp32 CUDA tensor in NHWC layout, pix_stride) for l/r_center, l/r_params, l/r_prior.
    Fills ``bufs`` (built for this B and K) asynchronously on the current stream (no host sync).  K = 1 is the
    reference's inference parse (acr_b200_parse); K > 1 keeps up to K hands per image and side
    (acr_b200_parse_topk)."""
    if bufs.B != B or bufs.K != K:
        raise ValueError(f"parse buffers are sized for B={bufs.B}, K={bufs.K}, not B={B}, K={K}")
    lib = L.load()
    ms = []
    dev = L.require_cuda(bufs.counts, *[maps[k][0] for k in maps])
    for k in ("l_center", "r_center", "l_params", "r_params", "l_prior", "r_prior"):
        t, stride = maps[k]
        assert t.dtype == torch.float32
        m = L.Map()
        m.ptr, m.pix_stride = t.data_ptr(), int(stride)
        ms.append(m)
    if meta_batch_ids is not None:
        meta_batch_ids = meta_batch_ids.to(device=bufs.counts.device, dtype=torch.int64).contiguous()
    if offsets is not None:
        offsets = offsets.to(device=bufs.counts.device, dtype=torch.float32).contiguous()
    with L.on(dev):
        if K == 1:
            rc = lib.acr_b200_parse(*ms, B, float(conf_thresh), L.ptr(meta_batch_ids), L.ptr(offsets), bufs.struct(),
                                    L.current_stream(dev))
        else:
            rc = lib.acr_b200_parse_topk(*ms, B, int(K), float(conf_thresh), L.ptr(meta_batch_ids), L.ptr(offsets),
                                         bufs.struct(), L.current_stream(dev))
    L.check(rc, "parse")
    # keep the inputs alive until the kernels have run
    bufs._keep = (meta_batch_ids, offsets, [m for m in maps.values()])
