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


# K = 1 with the gate open and no miss limit is the reference's per-hand-type OneEuro smoothing (one bank per side)
TRACK_GATE_OPEN = 90                # cells: 63^2 + 63^2 < 90^2, so no pair on the 64x64 map is out of the gate
TRACK_NO_MISS_LIMIT = 2 ** 31 - 1   # frames: a track is never ended for missing frames


class HandTracker:
    """Device-side state of multi-hand tracking (acr_b200_track_hands): K track slots per side, each with its id, last
    cell, missed-frame count and OneEuro bank, for one stream or, with ``streams`` = S > 1, for S streams whose frames
    share a batch (acr_b200_track_streams; every call then says which stream each image belongs to).  ``gate`` is in
    centre-map cells (8 cells = 64 px on the 512 input; >= 90 never rejects), ``max_missed`` in frames (15 = half a
    second at 30 fps); ``smooth_coeff`` None tracks ids only, a positive value also filters poses and betas per track.
    ``state`` is S consecutive slots of acr_b200_track_state_bytes(K) bytes, slot s byte for byte a single-stream
    tracker's state.  Owns one (2KB,) int32 id buffer (and, for several streams, one workspace) per batch size, reused
    by every call (zero copy, like ParseBuffers)."""

    def __init__(self, device, K: int, gate: int = 8, max_missed: int = 15, smooth_coeff: Optional[float] = 4.0,
                 streams: int = 1):
        if not 1 <= int(K) <= MAX_HANDS_PER_SIDE:
            raise ValueError(f"hands per side must be in 1..{MAX_HANDS_PER_SIDE}, got {K}")
        if int(gate) < 0 or int(max_missed) < 0:
            raise ValueError(f"gate and max_missed must be >= 0, got {gate}, {max_missed}")
        if smooth_coeff is not None and not float(smooth_coeff) > 0:
            raise ValueError(f"smooth_coeff must be positive or None, got {smooth_coeff}")
        if not 1 <= int(streams) <= MAX_TRACK_STREAMS:
            raise ValueError(f"streams must be in 1..{MAX_TRACK_STREAMS}, got {streams}")
        self.device, self.K, self.gate, self.max_missed = torch.device(device), int(K), int(gate), int(max_missed)
        self.smooth_coeff = None if smooth_coeff is None else float(smooth_coeff)
        self.streams = int(streams)
        self.slot_bytes = int(L.load().acr_b200_track_state_bytes(self.K))
        self.state = torch.zeros(self.streams * self.slot_bytes, dtype=torch.uint8, device=self.device)
        self._ids, self._ws = {}, {}

    def ids(self, B: int) -> torch.Tensor:
        """The (2KB,) id buffer of batch size B."""
        if B not in self._ids:
            self._ids[B] = torch.full((2 * self.K * B,), -1, dtype=torch.int32, device=self.device)
        return self._ids[B]

    def workspace(self, B: int) -> torch.Tensor:
        """The device scratch of acr_b200_track_streams at batch size B (2KB rows)."""
        if B not in self._ws:
            nb = int(L.load().acr_b200_track_streams_workspace_bytes(2 * self.K * B, int(B), self.streams))
            self._ws[B] = torch.empty(nb, dtype=torch.uint8, device=self.device)
        return self._ws[B]

    def slot(self, s: int) -> torch.Tensor:
        """Stream s's state (a view): byte for byte the state of a single-stream tracker after the same frames."""
        return self.state[s * self.slot_bytes:(s + 1) * self.slot_bytes]

    def reset(self) -> None:
        """No tracks, birth counters at zero, in every stream; in place, so a captured graph stays valid."""
        self.state.zero_()


def _frame_ints(t: Optional[torch.Tensor], B: int, name: str) -> Optional[torch.Tensor]:
    if t is None:
        return None
    if not (isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == torch.int32 and t.is_contiguous()
            and tuple(t.shape) == (B,)):
        raise ValueError(f"{name} must be a contiguous ({B},) int32 CUDA tensor")
    return t


def track_rows(tracker: HandTracker, B: int, row_src: torch.Tensor, detection_flag: Optional[torch.Tensor],
               poses: Optional[torch.Tensor] = None, betas: Optional[torch.Tensor] = None,
               n_dev: Optional[torch.Tensor] = None, frame_stream: Optional[torch.Tensor] = None,
               frame_begin: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Track the rows of a batch of B images (``row_src`` (n,4) int32 in the parse's layout, n <= 2KB) on the current
    stream, no host sync.  With one stream the images are B consecutive frames.  ``frame_stream`` (B,) int32 on the
    device gives each image's stream slot in 0..streams-1 (a multi-stream tracker needs it; another value leaves the
    image's rows untracked), the frames of one stream in ascending batch index; ``frame_begin`` (B,) int32 starts a
    stream over (zeroed slot) at each nonzero frame.  With the tracker's ``smooth_coeff`` set, ``poses`` (n,48) and
    ``betas`` (n,10) (contiguous fp32) are filtered in place.  Returns the tracker's id buffer for B; rows
    [0, min(n, n_dev)) are valid."""
    dev = L.require_cuda(row_src, detection_flag, poses, betas, n_dev, frame_stream, frame_begin, tracker.state)
    n = row_src.shape[0]
    assert row_src.dtype == torch.int32 and row_src.is_contiguous() and row_src.shape[1:] == (4,)
    assert detection_flag is None or (detection_flag.dtype == torch.float32 and detection_flag.is_contiguous())
    smooth = tracker.smooth_coeff is not None
    if smooth:
        assert poses is not None and betas is not None, "a smoothing tracker needs poses and betas"
        assert poses.is_contiguous() and betas.is_contiguous() and poses.dtype == betas.dtype == torch.float32
    frame_stream = _frame_ints(frame_stream, int(B), "frame_stream")
    frame_begin = _frame_ints(frame_begin, int(B), "frame_begin")
    if frame_stream is None and tracker.streams > 1:
        raise ValueError(f"this tracker follows {tracker.streams} streams: give frame_stream, the stream of each image")
    if frame_stream is None and frame_begin is not None:
        frame_stream = torch.zeros(int(B), dtype=torch.int32, device=dev)
    ids = tracker.ids(B)
    P = lambda t: L.ptr(t) if smooth else None
    with L.on(dev):
        if frame_stream is None:
            L.check(L.load().acr_b200_track_hands(P(poses), P(betas), L.ptr(row_src), L.ptr(detection_flag),
                                                  L.ptr(n_dev), n, int(B), tracker.K, tracker.gate, tracker.max_missed,
                                                  tracker.smooth_coeff or 0.0, L.ptr(tracker.state), L.ptr(ids),
                                                  L.current_stream(dev)), "track_hands")
        else:
            L.check(L.load().acr_b200_track_streams(P(poses), P(betas), L.ptr(row_src), L.ptr(detection_flag),
                                                    L.ptr(n_dev), n, int(B), tracker.K, tracker.gate,
                                                    tracker.max_missed, tracker.smooth_coeff or 0.0,
                                                    L.ptr(tracker.state), L.ptr(ids), L.ptr(frame_stream),
                                                    L.ptr(frame_begin), tracker.streams,
                                                    L.ptr(tracker.workspace(int(B))), L.current_stream(dev)),
                    "track_streams")
    return ids


def track_hands(bufs: "ParseBuffers", tracker: HandTracker, frame_stream: Optional[torch.Tensor] = None,
                frame_begin: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Track the hands of a parse (ParseBuffers of B frames: consecutive frames of one stream, or with
    ``frame_stream`` / ``frame_begin`` as in track_rows, frames of several) on the current stream, no host sync:
    poses / betas are filtered in place when the tracker smooths (params_pred, global_orient and hand_pose stay raw).
    Returns the tracker's (2KB,) int32 id buffer, valid over rows [0, counts[2])."""
    if tracker.K != bufs.K:
        raise ValueError(f"this tracker is built for K={tracker.K}, the parse buffers for K={bufs.K}")
    return track_rows(tracker, bufs.B, bufs.row_src, bufs.detection_flag, bufs.poses, bufs.betas,
                      n_dev=bufs.counts[2:3], frame_stream=frame_stream, frame_begin=frame_begin)


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
MAX_TRACK_STREAMS = 4096            # acr_b200_track_streams' S


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


# --------------------------------------------------------------------------------- part labels
PART_LABELS_MAX_SIDE = 16384                       # ACR_B200_PART_LABELS_MAX_SIDE
PART_LABELS_INVALID, PART_LABELS_OVER_CAPACITY = 1, 2   # ACR_B200_PART_LABELS_* flags
PART_LABEL_CLASSES = 33                           # 0 background, 1-16 right-hand parts, 17-32 left-hand parts


def part_label_geometry(offsets) -> np.ndarray:
    """The packing rule of acr_b200_part_labels on the host: (n,10) offsets rows -> (n,3) int64 [first label byte, H,
    W], (0, 0) for an invalid row (which then takes no bytes).  ``part_label_layout`` adds the flags."""
    o = np.asarray(offsets, np.float32).reshape(-1, 10)
    ok = np.all((o >= 0) & (o == np.floor(o)), axis=1) & (o[:, 0] == o[:, 1]) & (o[:, 0] >= 1) \
        & (o[:, 0] <= PART_LABELS_MAX_SIDE) & (o[:, 6] + o[:, 8] < o[:, 0]) & (o[:, 7] + o[:, 9] < o[:, 0])
    geo = np.zeros((len(o), 3), np.int64)
    with np.errstate(invalid="ignore"):
        geo[ok, 1] = (o[ok, 0] - o[ok, 6] - o[ok, 8]).astype(np.int64)
        geo[ok, 2] = (o[ok, 0] - o[ok, 7] - o[ok, 9]).astype(np.int64)
    sizes = geo[:, 1] * geo[:, 2]
    geo[:, 0] = np.cumsum(sizes) - sizes
    return geo


def part_label_layout(offsets, capacity: int):
    """-> (geometry (n,3) as ``part_label_geometry``, flags (n,) int32, total label bytes of the valid frames): what
    acr_b200_part_labels computes on the device for these offsets and this capacity."""
    geo = part_label_geometry(offsets)
    valid = geo[:, 1] > 0
    flags = np.where(valid, 0, PART_LABELS_INVALID).astype(np.int32)
    flags[valid & (geo[:, 0] + geo[:, 1] * geo[:, 2] > capacity)] = PART_LABELS_OVER_CAPACITY
    return geo, flags, int((geo[:, 1] * geo[:, 2]).sum())


class PartLabels:
    """Output buffer of ``part_labels``: ``capacity`` label bytes and per-frame offsets / flags for up to
    ``max_frames`` images, allocated once and written in place (zero copy, like ParseBuffers: a later launch into the
    same buffer overwrites the labels, so consume or copy them first).  ``labels[i]`` is image i's (H_i, W_i) uint8
    CUDA view (0 background, 1-16 right-hand parts, 17-32 left-hand parts); a frame flagged invalid or over capacity
    raises.  When the launch had its offsets on the host the views need no device read; otherwise the first index
    reads the offsets and flags back (one synchronisation)."""

    def __init__(self, capacity: int, max_frames: int, device=None):
        if int(capacity) < 0 or int(max_frames) < 1:
            raise ValueError(f"PartLabels: need capacity >= 0 and max_frames >= 1 (got {capacity}, {max_frames})")
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        self.capacity, self.max_frames = int(capacity), int(max_frames)
        self.data = torch.empty(max(self.capacity, 1), dtype=torch.uint8, device=self.device)
        self.frame_offset = torch.zeros(self.max_frames, dtype=torch.int64, device=self.device)
        self.flags = torch.zeros(self.max_frames, dtype=torch.int32, device=self.device)
        self.n = 0
        self._host = None        # (geometry, flags) of the last launch when its offsets were on the host
        self._offsets = None     # the device offsets of the last launch

    def __len__(self) -> int:
        return self.n

    def expect(self, offsets) -> None:
        """Check the frames of the next launch, (n,10) host offsets rows, against the capacity (ValueError before
        anything is enqueued) and keep their geometry for the views; None forgets it (device offsets: the views read
        the launch's offsets back)."""
        if offsets is None:
            self._host = None
            return
        geo, flags, total = part_label_layout(offsets, self.capacity)
        if (flags == PART_LABELS_OVER_CAPACITY).any():
            raise ValueError(f"part_labels: the frames need {total} label bytes, over the capacity of {self.capacity}")
        self._host = (geo, flags)

    def _layout(self):
        if self._host is None:
            self._host = part_label_layout(self._offsets[:self.n].cpu().numpy(), self.capacity)[:2]
        return self._host

    def __getitem__(self, i: int) -> torch.Tensor:
        if not -self.n <= i < self.n:
            raise IndexError(f"image {i} of {self.n}")
        i %= self.n
        geo, flags = self._layout()
        if flags[i]:
            why = "its offsets row is not a valid geometry" if flags[i] == PART_LABELS_INVALID else \
                f"its labels end past the capacity of {self.capacity} bytes"
            raise ValueError(f"image {i} has no part labels: {why}")
        o, H, W = (int(v) for v in geo[i])
        return self.data[o:o + H * W].view(H, W)

    def views(self):
        """Every image's (H, W) view, in batch order."""
        return [self[i] for i in range(self.n)]


def part_labels(segms: torch.Tensor, offsets, out: PartLabels) -> PartLabels:
    """Enqueue acr_b200_part_labels on the current stream: ``segms`` the (n, M, M, stride) NHWC logit map as it lies in
    the arena (Engine.view('segms'): bf16 / fp16 / fp32, stride 48), ``offsets`` (n,10) the frames' offsets rows, on
    the host or the device.  Host offsets are checked against ``out``'s capacity before anything is enqueued
    (ValueError); device offsets are checked on the device, which flags what does not fit.  Returns ``out``."""
    n = int(segms.shape[0])
    dt = {torch.bfloat16: L.DT_BF16, torch.float16: L.DT_F16, torch.float32: L.DT_F32}.get(segms.dtype)
    if dt is None or segms.dim() != 4 or segms.shape[1] != segms.shape[2] or segms.stride(3) != 1 \
            or segms.stride(2) * segms.shape[2] != segms.stride(1) or segms.stride(1) * segms.shape[1] != segms.stride(0):
        raise ValueError("part_labels: segms must be an (n, M, M, stride) NHWC bf16 / fp16 / fp32 map with "
                         "contiguous rows")
    if n > out.max_frames:
        raise ValueError(f"part_labels: {n} images exceed the buffer's {out.max_frames} frames")
    offsets = torch.as_tensor(offsets)
    if tuple(offsets.shape) != (n, 10):
        raise ValueError(f"part_labels: offsets must have shape ({n}, 10), got {tuple(offsets.shape)}")
    host = None
    if not offsets.is_cuda:
        host = offsets.to(torch.float32).numpy()
        out.expect(host)
    dev = L.require_cuda(segms, out.data)
    offs_dev = offsets.to(device=dev, dtype=torch.float32).contiguous()
    with L.on(dev):
        L.check(L.load().acr_b200_part_labels(L.ptr(segms), dt, int(segms.stride(2)), int(segms.shape[1]),
                                              L.ptr(offs_dev), n, out.capacity, L.ptr(out.data),
                                              L.ptr(out.frame_offset), L.ptr(out.flags), L.current_stream(dev)),
                "part_labels")
    out.n, out._offsets = n, offs_dev
    out._host = None if host is None else part_label_layout(host, out.capacity)[:2]
    return out
