"""Differentiable torch restatement of the reference ``ManoLayer.forward`` (mano/manolayer.py:104-276 of the
reference), used as the gradient reference of the fused MANO backward: autograd through it, in float64, is what
the kernel's gradients are compared with.  It covers what the drop-in ``mano.manolayer.ManoLayer`` supports:
axis-angle root, ``use_pca`` / ``ncomps``, ``flat_hand_mean``, ``center_idx``, ``th_trans``, ``share_betas`` and
the default-betas buffer.  Its forward is pinned to ``oracle.mano_ref`` and the reference goldens by
tests/test_cpu_mano_grad.py.  Written for clarity, not speed: one einsum per stage.
"""
import numpy as np
import torch

from oracle.mano_ref import JOINT_REORDER, LEVELS, TIPS


def rodrigues(aa: torch.Tensor) -> torch.Tensor:
    """(M,3) -> (M,3,3): half-angle quaternion with the 1e-8 offset inside the norm only (manolayer.py:423-434)."""
    ang = torch.norm(aa + 1e-8, dim=1, keepdim=True)
    half = ang * 0.5
    q = torch.cat([torch.cos(half), torch.sin(half) * (aa / ang)], 1)
    q = q / q.norm(dim=1, keepdim=True)
    w, x, y, z = q.unbind(1)
    return torch.stack([w * w + x * x - y * y - z * z, 2 * x * y - 2 * w * z, 2 * w * y + 2 * x * z,
                        2 * w * z + 2 * x * y, w * w - x * x + y * y - z * z, 2 * y * z - 2 * w * x,
                        2 * x * z - 2 * w * y, 2 * w * x + 2 * y * z, w * w - x * x - y * y + z * z], 1).view(-1, 3, 3)


class TorchMano:
    """One side's MANO layer over the buffers of a MANO asset (dict of numpy arrays, unflipped like ManoLayer's)."""

    def __init__(self, asset, side="right", use_pca=True, ncomps=6, flat_hand_mean=True, center_idx=None,
                 dtype=torch.float64, device="cpu"):
        t = lambda a: torch.as_tensor(np.asarray(a, np.float64), dtype=dtype, device=device)
        self.side, self.use_pca, self.center_idx = side, use_pca, center_idx
        self.ncomps = ncomps if use_pca else 45
        self.shapedirs, self.posedirs = t(asset["shapedirs"]), t(asset["posedirs"])          # (778,3,10), (778,3,135)
        self.v_template, self.J_regressor = t(asset["v_template"]), t(asset["J_regressor"])  # (778,3), (16,778)
        self.weights = t(asset["weights"])                                                  # (778,16)
        self.comps = t(np.asarray(asset["hands_components"])[:self.ncomps])                 # (ncomps,45)
        self.hands_mean = torch.zeros(45, dtype=dtype, device=device) if flat_hand_mean else t(asset["hands_mean"])
        self.default_betas = t(np.asarray(asset["betas"]).reshape(10))
        self.eye = torch.eye(3, dtype=dtype, device=device)

    def full_pose(self, pose_coeffs):
        """(n, 3+ncomps) or (n,48) coefficients -> (n,48) axis angles with the mean pose added."""
        hand = pose_coeffs[:, 3:3 + self.ncomps]
        if self.use_pca:
            hand = hand.mm(self.comps)
        return torch.cat([pose_coeffs[:, :3], self.hands_mean + hand], 1)

    def __call__(self, pose_coeffs, betas=None, trans=None, share_betas=False):
        n = pose_coeffs.shape[0]
        R = rodrigues(self.full_pose(pose_coeffs).reshape(-1, 3)).view(n, 16, 3, 3)
        pose_map = (R[:, 1:] - self.eye).reshape(n, 135)
        if betas is None:
            b = self.default_betas.expand(n, 10)
        else:
            b = betas.mean(0, keepdim=True).expand(n, 10) if share_betas else betas
        v_shaped = self.v_template + torch.einsum("vck,nk->nvc", self.shapedirs, b)
        J = torch.einsum("jv,nvc->njc", self.J_regressor, v_shaped)
        v_posed = v_shaped + torch.einsum("vck,nk->nvc", self.posedirs, pose_map)
        # kinematic chain: every finger hangs off the root, three levels deep
        Rg, tg = [None] * 16, [None] * 16
        Rg[0], tg[0] = R[:, 0], J[:, 0]
        for lev in range(3):
            for f in range(5):
                idx = LEVELS[lev][f]
                par = 0 if lev == 0 else LEVELS[lev - 1][f]
                Rg[idx] = Rg[par] @ R[:, idx]
                tg[idx] = (Rg[par] @ (J[:, idx] - J[:, par]).unsqueeze(-1)).squeeze(-1) + tg[par]
        Rg, tg = torch.stack(Rg, 1), torch.stack(tg, 1)                  # (n,16,3,3), (n,16,3)
        # skinning with the rest pose removed: A_j = [R_g | t_g - R_g J_j]
        At = tg - (Rg @ J.unsqueeze(-1)).squeeze(-1)
        TR = torch.einsum("vj,njab->nvab", self.weights, Rg)
        Tt = torch.einsum("vj,nja->nva", self.weights, At)
        verts = (TR @ v_posed.unsqueeze(-1)).squeeze(-1) + Tt
        jtr = torch.cat([tg, verts[:, TIPS[self.side]]], 1)[:, JOINT_REORDER]
        if trans is None or bool(torch.norm(trans) == 0):
            if self.center_idx is None:
                return verts, jtr, None
            c = jtr[:, self.center_idx].unsqueeze(1)
            return verts - c, jtr - c, c
        return verts + trans.unsqueeze(1), jtr + trans.unsqueeze(1), trans.unsqueeze(1)
