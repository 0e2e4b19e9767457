"""Float64 restatement of ``ManoLayer`` that every torch.func transform can differentiate, for the forward-mode tests.
The axis-angle layer is ``tests.mano_torch_ref.TorchMano`` itself (plain torch ops).  The rotation-matrix branch needs
a projection with derivatives that exist at exact rotations, where ``torch.linalg.svd``'s do not: ``SO3ProjectFn`` is
``tests.mano_rotmat_ref.SO3Project`` in the ``setup_context`` form, with the polar factor's closed-form JVP next to its
closed-form VJP, so ``jvp`` / ``jacfwd`` / ``jacrev`` / ``vmap`` all apply.  Its JVP is pinned to central differences
by tests/test_cpu_mano_jvp.py.
"""
import torch

from tests.mano_rotmat_ref import TorchManoRot, _skew


def _axial_skew(X):
    """axial(X - X^T) of a batch of 3x3 matrices."""
    return torch.stack([X[:, 2, 1] - X[:, 1, 2], X[:, 0, 2] - X[:, 2, 0], X[:, 1, 0] - X[:, 0, 1]], 1)


class SO3ProjectFn(torch.autograd.Function):
    """batch_rotprojs: Q = U V^T of M = U S V^T, column 2 negated where det Q < 0.  With P = Q^T M (symmetric) and
    A = (tr P) I - P: JVP  w = A^-1 axial(Q^T dM - dM^T Q),  dR = Q [w]x D;  VJP as ``SO3Project``."""
    generate_vmap_rule = True

    @staticmethod
    def forward(M):
        U, _, Vh = torch.linalg.svd(M)
        Q = U @ Vh
        flip = torch.where(torch.linalg.det(Q) < 0, -1.0, 1.0).to(M.dtype)
        D = torch.stack([torch.ones_like(flip), torch.ones_like(flip), flip], -1)
        return Q * D[:, None, :], Q, D

    @staticmethod
    def setup_context(ctx, inputs, output):
        _, Q, D = output
        ctx.save_for_backward(inputs[0], Q, D)
        ctx.save_for_forward(inputs[0], Q, D)
        ctx.mark_non_differentiable(Q, D)

    @staticmethod
    def _solve(M, Q, k):
        P = Q.transpose(1, 2) @ M
        A = P.diagonal(dim1=1, dim2=2).sum(1)[:, None, None] * torch.eye(3, dtype=M.dtype, device=M.device) - P
        return torch.linalg.solve(A, k)

    @staticmethod
    def backward(ctx, G, _gQ, _gD):
        M, Q, D = ctx.saved_tensors
        B = Q.transpose(1, 2) @ (G * D[:, None, :])
        return Q @ _skew(SO3ProjectFn._solve(M, Q, _axial_skew(B)))

    @staticmethod
    def jvp(ctx, dM):
        M, Q, D = ctx.saved_tensors
        w = SO3ProjectFn._solve(M, Q, _axial_skew(Q.transpose(1, 2) @ dM))
        return (Q @ _skew(w)) * D[:, None, :], None, None


class TorchManoFunc(TorchManoRot):
    """TorchManoRot with the transform-friendly projection."""

    def from_rotmats(self, mats, betas=None, trans=None, share_betas=False, root_palm=False):
        n = mats.shape[0]
        R = SO3ProjectFn.apply(mats.reshape(-1, 3, 3))[0].view(n, 16, 3, 3)
        return self.from_rotations(R, betas, trans, share_betas, root_palm)
