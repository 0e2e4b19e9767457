"""Drop-in ``ManoLayer`` backed by one fused sm_90a kernel.

Mirrors the constructor, buffers and ``forward`` signature of the reference
(/root/reference/mano/manolayer.py:13-22, :65-93, :104-110, :273-276); the ~124 ATen launches of
the reference forward (:104-276) become a single ``acr_b200_mano_forward`` call.

The layer is differentiable with respect to the pose (or PCA coefficients), betas and ``th_trans``: with grad
enabled and pose or betas requiring grad, the kernel runs inside ``_ManoFunction``, whose backward is the fused
``acr_b200_mano_backward``.  Otherwise the forward makes exactly the launch it makes without autograd.
"""
from __future__ import annotations

from typing import Optional

import numpy as np
import torch
from torch.autograd.function import once_differentiable
from torch.nn import Module

from acr_b200 import ops as _ops
from mano.assets import get_asset

_ZERO1 = torch.zeros(1)


class _ManoFunction(torch.autograd.Function):
    """(pose (n,48) without the mean pose, betas (n,10)) -> (verts, joints, center) of one side; the backward is the
    fused MANO backward kernel (first order only)."""

    @staticmethod
    def forward(ctx, pose, betas, model, side, center_idx):
        out = _ops.mano_forward(model if side == 0 else None, model if side == 1 else None, pose, betas, None, side,
                                center_idx)
        ctx.save_for_backward(pose, betas)
        ctx.model, ctx.side, ctx.center_idx = model, side, center_idx
        ctx.set_materialize_grads(False)     # an unused output's cotangent stays None and reaches the kernel as NULL
        return out["verts"], out["joints"], out["center"]

    @staticmethod
    @once_differentiable
    def backward(ctx, dverts, djoints, dcenter):
        pose, betas = ctx.saved_tensors
        want_pose, want_betas = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        if ctx.center_idx is None:
            dcenter = None                   # the centre output is zero and does not depend on the inputs
        if dverts is None and djoints is None and dcenter is None:
            return None, None, None, None, None
        dpose, dbetas = _ops.mano_backward(ctx.model, ctx.side, pose, betas, ctx.center_idx, dverts, djoints, dcenter,
                                           want_pose, want_betas)
        return dpose, dbetas, None, None, None


class ManoLayer(Module):
    __constants__ = ['use_pca', 'rot', 'ncomps', 'kintree_parents', 'side', 'center_idx', 'joint_rot_mode']

    def __init__(self, center_idx=None, flat_hand_mean=True, ncomps=6, side='right', mano_root='model_data/mano/',
                 use_pca=True, root_rot_mode='axisang', joint_rot_mode='axisang', robust_rot=False, asset=None):
        super().__init__()
        if root_rot_mode != 'axisang' or joint_rot_mode != 'axisang':
            # the reference's 6D-root branch references an undefined name (manolayer.py:148-150)
            raise NotImplementedError("only root_rot_mode='axisang', joint_rot_mode='axisang' are supported")
        self.center_idx = center_idx
        self.robust_rot = robust_rot
        self.rot = 3
        self.flat_hand_mean = flat_hand_mean
        self.side = side
        self.use_pca = use_pca
        self.joint_rot_mode = joint_rot_mode
        self.root_rot_mode = root_rot_mode
        self.ncomps = ncomps if use_pca else 45
        smpl_data = asset if asset is not None else get_asset(mano_root, side)
        self.smpl_data = smpl_data
        hands_components = np.asarray(smpl_data['hands_components'], np.float32)
        T = lambda a, dt=np.float32: torch.from_numpy(np.array(a, dtype=dt, copy=True, order='C'))  # copies, like torch.Tensor(a)
        self.register_buffer('th_betas', T(smpl_data['betas']).unsqueeze(0))
        self.register_buffer('th_shapedirs', T(smpl_data['shapedirs']))
        self.register_buffer('th_posedirs', T(smpl_data['posedirs']))
        self.register_buffer('th_v_template', T(smpl_data['v_template']).unsqueeze(0))
        self.register_buffer('th_J_regressor', T(smpl_data['J_regressor']))
        self.register_buffer('th_weights', T(smpl_data['weights']))
        self.register_buffer('th_faces', T(np.asarray(smpl_data['f']).astype(np.int32), np.int32).long())
        hands_mean = np.zeros(hands_components.shape[1], np.float32) if flat_hand_mean \
            else np.asarray(smpl_data['hands_mean'], np.float32).copy()
        self.register_buffer('th_hands_mean', T(hands_mean).unsqueeze(0))
        self.register_buffer('th_comps', T(hands_components))
        self.register_buffer('th_selected_comps', T(hands_components[:ncomps]))
        self.kintree_table = smpl_data['kintree_table']
        self.kintree_parents = list(np.asarray(self.kintree_table)[0].tolist())
        self._packed = None
        self._packed_key = None

    # packed constants follow the *current* buffers (MANOWrapper flips th_shapedirs in place)
    def packed_model(self) -> torch.Tensor:
        bufs = (self.th_shapedirs, self.th_posedirs, self.th_v_template, self.th_J_regressor, self.th_weights,
                self.th_hands_mean)
        key = tuple((b._version, b.data_ptr(), str(b.device)) for b in bufs)
        if self._packed is None or key != self._packed_key:
            asset = dict(shapedirs=self.th_shapedirs.detach().cpu().numpy(),
                         posedirs=self.th_posedirs.detach().cpu().numpy(),
                         v_template=self.th_v_template[0].detach().cpu().numpy(),
                         J_regressor=self.th_J_regressor.detach().cpu().numpy(),
                         weights=self.th_weights.detach().cpu().numpy(),
                         hands_mean=self.th_hands_mean[0].detach().cpu().numpy())
            self._packed = _ops.pack_mano_model(asset, False, self.th_shapedirs.device)
            self._packed_key = key
        return self._packed

    def forward(self, th_pose_coeffs, th_betas=_ZERO1, th_trans=_ZERO1, root_palm=torch.Tensor([0]),
                share_betas=torch.Tensor([0])):
        if bool(root_palm):
            raise NotImplementedError("root_palm=True is not on the ACR hot path")
        batch_size = th_pose_coeffs.shape[0]
        pose = th_pose_coeffs
        if self.use_pca:
            pose = torch.cat([pose[:, :3], pose[:, 3:3 + self.ncomps].mm(self.th_selected_comps)], 1)
        if th_betas is None or th_betas.numel() == 1:
            betas = self.th_betas.expand(batch_size, 10)
        else:
            betas = th_betas
            if bool(share_betas):
                betas = betas.mean(0, keepdim=True).expand(betas.shape[0], 10)
        use_trans = not (th_trans is None or th_trans is _ZERO1 or bool(torch.norm(th_trans) == 0))
        center_idx = None if use_trans else self.center_idx
        side = 1 if self.side == 'right' else 0
        model = self.packed_model()
        if torch.is_grad_enabled() and (pose.requires_grad or betas.requires_grad):
            verts, jtr, center = _ManoFunction.apply(pose[:, :48], betas, model, side, center_idx)
        else:
            out = _ops.mano_forward(model if side == 0 else None, model if side == 1 else None, pose[:, :48],
                                    betas, None, side, center_idx)
            verts, jtr, center = out["verts"], out["joints"], out["center"]
        if use_trans:
            verts = verts + th_trans.unsqueeze(1)
            jtr = jtr + th_trans.unsqueeze(1)
            return verts, jtr, th_trans.unsqueeze(1)
        if self.center_idx is None:
            return verts, jtr, None
        return verts, jtr, center
