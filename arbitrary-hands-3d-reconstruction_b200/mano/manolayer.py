"""Drop-in ``ManoLayer`` backed by one fused sm_90a kernel.

Mirrors the constructor, buffers and ``forward`` signature of the reference
(/root/reference/mano/manolayer.py:13-22, :65-93, :104-110, :273-276); the ~124 ATen launches of
the reference forward (:104-276) become a single ``acr_b200_mano_forward`` call.

The layer is differentiable with respect to the pose (or PCA coefficients), betas and ``th_trans``: with grad
enabled and pose or betas requiring grad, the kernel runs inside ``_ManoFunction``, whose backward is the fused
``acr_b200_mano_backward``.  Otherwise the forward makes exactly the launch it makes without autograd.

Rotation-matrix joints (``use_pca=False, joint_rot_mode='rotmat'``, reference :151-162) and ``root_palm``
(:248-250) run through ``acr_b200_mano_layer_forward`` / ``_backward`` instead: the SO(3) projection of every input
matrix and its gradient are fused into the same kernels.

Forward mode (``torch.func.jvp`` / ``jacfwd``, ``torch.autograd.forward_ad``) runs the fused JVP kernel
``acr_b200_mano_layer_jvp``, and every torch.func transform composes with the layer (``vmap``, ``grad``, ``jacrev``):
the Functions' vmap rules fold a vmapped batch into more hands, or into more tangents / cotangent rows.
"""
from __future__ import annotations

from typing import Optional

import numpy as np
import torch
import torch.autograd.forward_ad as _fwAD
from torch.nn import Module

from acr_b200 import lib as _lib
from acr_b200 import ops as _ops
from mano.assets import get_asset

_ZERO1 = torch.zeros(1)


_SECOND_ORDER = ("ManoLayer has first-order derivatives only: double backward and forward-over-reverse "
                 "(torch.func.hessian, jvp of grad) are not supported")


def _batch_first(x, bdim, size):
    """A vmapped tensor with its batch dim (None: unbatched) moved to the front, of length ``size``."""
    return x.expand(size, *x.shape) if bdim is None else x.movedim(bdim, 0)


def _fold_hands(x, bdim, size, hand_dim=0):
    """Fold a vmap batch of ``size`` into the hand dimension ``hand_dim``: batch b, hand i -> hand b*n + i.  None
    (no tensor) passes through."""
    if x is None:
        return None
    x = _batch_first(x, bdim, size).movedim(0, hand_dim)
    return x.reshape(*x.shape[:hand_dim], -1, *x.shape[hand_dim + 2:])


def _unfold_hands(x, size, hand_dim=0):
    return x.reshape(*x.shape[:hand_dim], size, -1, *x.shape[hand_dim + 1:])


class _ManoFunction(torch.autograd.Function):
    """(pose: (n,48) axis angles without the mean pose or (n,16,3,3) matrices, betas (n,10)) -> (verts, joints,
    center) of one side, with ``root_palm``.  Axis angles without the palm run the plain fused forward, the other forms
    ``acr_b200_mano_layer_forward``.  The backward is the fused backward kernel pair and the JVP the fused JVP kernel,
    each behind a Function of its own with a vmap rule, so torch.func's transforms compose with them; first order
    only."""

    @staticmethod
    def forward(pose, betas, model, side, pose_mode, center_idx, root_palm):
        if pose_mode == _lib.POSE_AXISANG and not root_palm:
            out = _ops.mano_forward(model if side == 0 else None, model if side == 1 else None, pose, betas, None, side,
                                    center_idx)
            return out["verts"], out["joints"], out["center"]
        return _ops.mano_layer_forward(model, side, pose, pose_mode, betas, center_idx, root_palm)

    @staticmethod
    def setup_context(ctx, inputs, output):
        pose, betas = inputs[:2]
        ctx.save_for_backward(pose, betas)
        ctx.save_for_forward(pose, betas)
        ctx.args = inputs[2:]
        ctx.set_materialize_grads(False)     # an unused output's cotangent stays None and reaches the kernel as NULL

    @staticmethod
    def backward(ctx, dverts, djoints, dcenter):
        pose, betas = ctx.saved_tensors
        none = (None,) * 5
        if ctx.args[3] is None:
            dcenter = None                   # the centre output is zero and does not depend on the inputs
        if dverts is None and djoints is None and dcenter is None:
            return (None, None) + none
        dpose, dbetas = _ManoVjp.apply(pose, betas, dverts, djoints, dcenter, *ctx.args)
        return (dpose if ctx.needs_input_grad[0] else None, dbetas if ctx.needs_input_grad[1] else None) + none

    @staticmethod
    def jvp(ctx, tpose, tbetas, *_):
        pose, betas = ctx.saved_tensors
        tv, tj, tc = _ManoJvp.apply(pose, betas, None if tpose is None else tpose.unsqueeze(0),
                                    None if tbetas is None else tbetas.unsqueeze(0), *ctx.args)
        return tv[0], tj[0], tc[0]

    @staticmethod
    def vmap(info, in_dims, pose, betas, *args):
        # the vmapped dims become more hands
        B = info.batch_size
        outs = _ManoFunction.apply(_fold_hands(pose, in_dims[0], B), _fold_hands(betas, in_dims[1], B), *args)
        return tuple(_unfold_hands(o, B) for o in outs), (0, 0, 0)


class _ManoVjp(torch.autograd.Function):
    """Cotangents of ``_ManoFunction``'s (verts, joints, center) -> (dpose, dbetas): the fused backward kernels."""

    @staticmethod
    def forward(pose, betas, dverts, djoints, dcenter, model, side, pose_mode, center_idx, root_palm):
        return _ops.mano_layer_backward(model, side, pose, pose_mode, betas, center_idx, root_palm, dverts, djoints,
                                        dcenter)

    @staticmethod
    def setup_context(ctx, inputs, output):
        pass

    @staticmethod
    def backward(ctx, *grads):
        raise RuntimeError(_SECOND_ORDER)

    @staticmethod
    def jvp(ctx, *tangents):
        raise RuntimeError(_SECOND_ORDER)

    @staticmethod
    def vmap(info, in_dims, pose, betas, dverts, djoints, dcenter, *args):
        # a batch of cotangents (jacrev) becomes more rows: pose and betas are repeated for each
        B = info.batch_size
        f = [_fold_hands(x, d, B) for x, d in zip((pose, betas, dverts, djoints, dcenter), in_dims)]
        dpose, dbetas = _ManoVjp.apply(*f, *args)
        return (_unfold_hands(dpose, B), _unfold_hands(dbetas, B)), (0, 0)


class _ManoJvp(torch.autograd.Function):
    """(pose, betas, tangents tpose (T,n,...) and tbetas (T,n,10), either None) -> the T tangents of
    ``_ManoFunction``'s outputs, tangent-major: the fused JVP kernel."""

    @staticmethod
    def forward(pose, betas, tpose, tbetas, model, side, pose_mode, center_idx, root_palm):
        return _ops.mano_layer_jvp(model, side, pose, pose_mode, betas, center_idx, root_palm, tpose, tbetas)

    @staticmethod
    def setup_context(ctx, inputs, output):
        pass

    @staticmethod
    def backward(ctx, *grads):
        raise RuntimeError(_SECOND_ORDER)

    @staticmethod
    def jvp(ctx, *tangents):
        raise RuntimeError(_SECOND_ORDER)

    @staticmethod
    def vmap(info, in_dims, pose, betas, tpose, tbetas, *args):
        B = info.batch_size
        if in_dims[0] is None and in_dims[1] is None:
            # only the tangents are batched (jacfwd): they become more tangents of the same hands, one launch
            f = [None if x is None else _batch_first(x, d, B).flatten(0, 1) for x, d in ((tpose, in_dims[2]),
                                                                                        (tbetas, in_dims[3]))]
            outs = _ManoJvp.apply(pose, betas, *f, *args)
            return tuple(o.unflatten(0, (B, -1)) for o in outs), (0, 0, 0)
        # the hands are batched: the batch becomes more hands, each with its own tangents
        outs = _ManoJvp.apply(_fold_hands(pose, in_dims[0], B), _fold_hands(betas, in_dims[1], B),
                              _fold_hands(tpose, in_dims[2], B, 1), _fold_hands(tbetas, in_dims[3], B, 1), *args)
        return tuple(_unfold_hands(o, B, 1) for o in outs), (1, 1, 1)


def _differentiated(*ts) -> bool:
    """Whether the forward must run inside ``_ManoFunction``: autograd will differentiate it, a torch.func transform
    is active (its wrapped tensors cannot go to the kernels directly), or an input is a forward-AD dual tensor.
    Otherwise the forward makes the plain launch."""
    if torch._C._are_functorch_transforms_active():
        return True
    if torch.is_grad_enabled() and any(t.requires_grad for t in ts):
        return True
    return _fwAD._current_level >= 0 and any(_fwAD.unpack_dual(t).tangent is not None for t in ts)


def _rodrigues(aa: torch.Tensor) -> torch.Tensor:
    """(M,3) axis angles -> (M,3,3), the reference's half-angle quaternion form (its batch_rodrigues); used once, for
    the ``th_hands_mean_rotmat`` buffer."""
    ang = torch.norm(aa + 1e-8, dim=1, keepdim=True)
    q = torch.cat([torch.cos(ang * 0.5), torch.sin(ang * 0.5) * (aa / ang)], 1)
    w, x, y, z = (q / q.norm(dim=1, keepdim=True)).unbind(1)
    return torch.stack([w * w + x * x - y * y - z * z, 2 * x * y - 2 * w * z, 2 * w * y + 2 * x * z,
                        2 * w * z + 2 * x * y, w * w - x * x + y * y - z * z, 2 * y * z - 2 * w * x,
                        2 * x * z - 2 * w * y, 2 * w * x + 2 * y * z, w * w - x * x - y * y + z * z], 1).view(-1, 3, 3)


class ManoLayer(Module):
    __constants__ = ['use_pca', 'rot', 'ncomps', 'kintree_parents', 'side', 'center_idx', 'joint_rot_mode']

    def __init__(self, center_idx=None, flat_hand_mean=True, ncomps=6, side='right', mano_root='model_data/mano/',
                 use_pca=True, root_rot_mode='axisang', joint_rot_mode='axisang', robust_rot=False, asset=None):
        super().__init__()
        # as in the reference, any joint_rot_mode but 'axisang' without PCA takes (n,16,3,3) matrices, and that
        # branch ignores root_rot_mode
        self.rotmat = not use_pca and joint_rot_mode != 'axisang'
        if not self.rotmat and root_rot_mode != 'axisang':
            # the reference's 6D-root branch references an undefined name (manolayer.py:148-150)
            raise NotImplementedError("only root_rot_mode='axisang' is supported with axis-angle joints")
        self.center_idx = center_idx
        self.robust_rot = robust_rot
        self.rot = 3 if root_rot_mode == 'axisang' else 6
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
        if self.rotmat:
            # the reference keeps the mean pose as matrices and never applies it in forward
            self.register_buffer('th_hands_mean_rotmat', _rodrigues(T(hands_mean).view(15, 3)).reshape(15, 3, 3))
        else:
            self.register_buffer('th_hands_mean', T(hands_mean).unsqueeze(0))
            self.register_buffer('th_comps', T(hands_components))
            self.register_buffer('th_selected_comps', T(hands_components[:ncomps]))
        self.kintree_table = smpl_data['kintree_table']
        self.kintree_parents = list(np.asarray(self.kintree_table)[0].tolist())
        self._packed = None
        self._packed_key = None

    # packed constants follow the *current* buffers (MANOWrapper flips th_shapedirs in place)
    def packed_model(self) -> torch.Tensor:
        # rotation-matrix layers have no axis-angle mean pose: the packed one is zero and unused
        hm = None if self.rotmat else self.th_hands_mean
        bufs = (self.th_shapedirs, self.th_posedirs, self.th_v_template, self.th_J_regressor, self.th_weights) + \
            (() if hm is None else (hm,))
        key = tuple((b._version, b.data_ptr(), str(b.device)) for b in bufs)
        if self._packed is None or key != self._packed_key:
            # the buffers are constants: read them as such also when the first call runs inside a torch.func transform
            with torch._C._DisableFuncTorch():
                asset = dict(shapedirs=self.th_shapedirs.detach().cpu().numpy(),
                             posedirs=self.th_posedirs.detach().cpu().numpy(),
                             v_template=self.th_v_template[0].detach().cpu().numpy(),
                             J_regressor=self.th_J_regressor.detach().cpu().numpy(),
                             weights=self.th_weights.detach().cpu().numpy(),
                             hands_mean=np.zeros(45, np.float32) if hm is None else hm[0].detach().cpu().numpy())
                self._packed = _ops.pack_mano_model(asset, False, self.th_shapedirs.device)
            self._packed_key = key
        return self._packed

    def forward(self, th_pose_coeffs, th_betas=_ZERO1, th_trans=_ZERO1, root_palm=torch.Tensor([0]),
                share_betas=torch.Tensor([0])):
        palm = bool(root_palm)
        batch_size = th_pose_coeffs.shape[0]
        pose = th_pose_coeffs
        if self.rotmat:
            assert pose.dim() == 4, ('When not self.use_pca, th_pose_coeffs should have 4 dims, got {}'.format(
                pose.dim()))
            assert pose.shape[2:4] == (3, 3), ('When not self.use_pca, th_pose_coeffs have 3x3 matrix for two '
                                               'last dims, got {}'.format(pose.shape[2:4]))
            if pose.shape[1] != 16:
                raise ValueError(f"rotation-matrix pose must be (n,16,3,3), got {tuple(pose.shape)}")
        elif self.use_pca:
            pose = torch.cat([pose[:, :3], pose[:, 3:3 + self.ncomps].mm(self.th_selected_comps)], 1)
        if th_betas is None or th_betas.numel() == 1:
            betas = self.th_betas.expand(batch_size, 10)
        else:
            betas = th_betas
            if bool(share_betas):
                betas = betas.mean(0, keepdim=True).expand(betas.shape[0], 10)
        use_trans = not (th_trans is None or th_trans is _ZERO1 or bool(torch.norm(th_trans) == 0))
        center_idx = None if use_trans else self.center_idx
        if palm and center_idx == 0:
            raise NotImplementedError("centring on the palm (center_idx=0 with root_palm) is not supported")
        side = 1 if self.side == 'right' else 0
        model = self.packed_model()
        mode = _lib.POSE_ROTMAT if self.rotmat else _lib.POSE_AXISANG
        p = pose if self.rotmat else pose[:, :48]
        if _differentiated(p, betas):
            verts, jtr, center = _ManoFunction.apply(p, betas, model, side, mode, center_idx, palm)
        elif self.rotmat or palm:
            verts, jtr, center = _ops.mano_layer_forward(model, side, p, mode, betas, center_idx, palm)
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
