"""Float64 torch restatement of the reference ``ManoLayer.forward``'s rotation-matrix branch (use_pca=False,
joint_rot_mode='rotmat', mano/manolayer.py:151-162 of the reference, batch_rotprojs :436-453) and of ``root_palm``
(:248-250), used as the gradient reference of the fused kernels in those forms.  ``TorchManoRot`` extends
``tests.mano_torch_ref.TorchMano`` with ``from_rotations`` (everything after the joint rotations) and
``from_rotmats`` (the SO(3) projection, then ``from_rotations``); its ``__call__`` is rodrigues plus
``from_rotations`` and gives results identical to ``TorchMano.__call__`` (tests/test_cpu_mano_rotmat.py pins both,
and pins the restatement to the reference's own outputs).
"""
import torch

from oracle.mano_ref import JOINT_REORDER, LEVELS, TIPS
from tests.mano_torch_ref import TorchMano, rodrigues


def _skew(z):
    o = torch.zeros_like(z[:, 0])
    return torch.stack([o, -z[:, 2], z[:, 1], z[:, 2], o, -z[:, 0], -z[:, 1], z[:, 0], o], 1).view(-1, 3, 3)


class SO3Project(torch.autograd.Function):
    """batch_rotprojs (manolayer.py:436-453): Q = U V^T of M = U S V^T, column 2 negated where det Q < 0.  The
    backward is the closed-form VJP of the polar factor -- with P = Q^T M, B = Q^T (G D), k = axial(B - B^T):
    z = (tr(P) I - P)^-1 k and dM = Q [z]x -- rather than torch.svd's, which is NaN when singular values coincide
    (every exact rotation)."""

    @staticmethod
    def forward(ctx, M):
        U, _, Vh = torch.linalg.svd(M)
        Q = U @ Vh
        flip = torch.linalg.det(Q) < 0
        D = torch.ones(M.shape[0], 3, dtype=M.dtype, device=M.device)
        D[:, 2] = torch.where(flip, -1.0, 1.0).to(M.dtype)
        ctx.save_for_backward(M, Q, D)
        return Q * D[:, None, :]

    @staticmethod
    def backward(ctx, G):
        M, Q, D = ctx.saved_tensors
        P = Q.transpose(1, 2) @ M
        B = Q.transpose(1, 2) @ (G * D[:, None, :])
        k = torch.stack([B[:, 2, 1] - B[:, 1, 2], B[:, 0, 2] - B[:, 2, 0], B[:, 1, 0] - B[:, 0, 1]], 1)
        A = P.diagonal(dim1=1, dim2=2).sum(1)[:, None, None] * torch.eye(3, dtype=M.dtype, device=M.device) - P
        z = torch.linalg.solve(A, k)
        return Q @ _skew(z)


class TorchManoRot(TorchMano):
    """TorchMano with rotation-matrix input and root_palm."""

    def __call__(self, pose_coeffs, betas=None, trans=None, share_betas=False, root_palm=False):
        n = pose_coeffs.shape[0]
        R = rodrigues(self.full_pose(pose_coeffs).reshape(-1, 3)).view(n, 16, 3, 3)
        return self.from_rotations(R, betas, trans, share_betas, root_palm)

    def from_rotmats(self, mats, betas=None, trans=None, share_betas=False, root_palm=False):
        """(n,16,3,3) matrices, each projected onto SO(3) like batch_rotprojs; no mean pose, as in the reference."""
        n = mats.shape[0]
        R = SO3Project.apply(mats.reshape(-1, 3, 3)).view(n, 16, 3, 3)
        return self.from_rotations(R, betas, trans, share_betas, root_palm)

    def from_rotations(self, R, betas=None, trans=None, share_betas=False, root_palm=False):
        """Everything after the joint rotations R (n,16,3,3): the stages of TorchMano.__call__, op for op, plus the
        palm, (v95 + v22) / 2, in place of the wrist before the reorder and the centring."""
        n = R.shape[0]
        pose_map = (R[:, 1:] - self.eye).reshape(n, 135)
        if betas is None:
            b = self.default_betas.expand(n, 10)
        else:
            b = betas.mean(0, keepdim=True).expand(n, 10) if share_betas else betas
        v_shaped = self.v_template + torch.einsum("vck,nk->nvc", self.shapedirs, b)
        J = torch.einsum("jv,nvc->njc", self.J_regressor, v_shaped)
        v_posed = v_shaped + torch.einsum("vck,nk->nvc", self.posedirs, pose_map)
        Rg, tg = [None] * 16, [None] * 16
        Rg[0], tg[0] = R[:, 0], J[:, 0]
        for lev in range(3):
            for f in range(5):
                idx = LEVELS[lev][f]
                par = 0 if lev == 0 else LEVELS[lev - 1][f]
                Rg[idx] = Rg[par] @ R[:, idx]
                tg[idx] = (Rg[par] @ (J[:, idx] - J[:, par]).unsqueeze(-1)).squeeze(-1) + tg[par]
        Rg, tg = torch.stack(Rg, 1), torch.stack(tg, 1)
        At = tg - (Rg @ J.unsqueeze(-1)).squeeze(-1)
        TR = torch.einsum("vj,njab->nvab", self.weights, Rg)
        Tt = torch.einsum("vj,nja->nva", self.weights, At)
        verts = (TR @ v_posed.unsqueeze(-1)).squeeze(-1) + Tt
        if root_palm:
            tg = torch.cat([((verts[:, 95] + verts[:, 22]) / 2).unsqueeze(1), tg[:, 1:]], 1)
        jtr = torch.cat([tg, verts[:, TIPS[self.side]]], 1)[:, JOINT_REORDER]
        if trans is None or bool(torch.norm(trans) == 0):
            if self.center_idx is None:
                return verts, jtr, None
            c = jtr[:, self.center_idx].unsqueeze(1)
            return verts - c, jtr - c, c
        return verts + trans.unsqueeze(1), jtr + trans.unsqueeze(1), trans.unsqueeze(1)
