"""GPU: ManoLayer's forward-mode derivatives (the fused JVP kernel behind torch.func and torch.autograd.forward_ad)
against torch.func on the float64 restatements (tests/mano_torch_ref.py, tests/mano_jvp_ref.py), against the fused
backward kernel (jacrev, the dot-product test), and the kernel's own properties: the joints-only form, determinism,
and independence of the tangent tiling."""
import pytest
import torch
import torch.autograd.forward_ad as fwAD
from torch.func import grad, hessian, jacfwd, jacrev, jvp, vmap

from tests.helpers import rel_err
from tests.mano_jvp_ref import TorchManoFunc
from tests.mano_torch_ref import rodrigues

pytestmark = pytest.mark.gpu
TOL = 1e-4   # BASELINE.json: 1e-4 relative fp32 tolerance


@pytest.fixture(scope="module")
def assets():
    from acr_b200.synth import make_synthetic_mano
    return {"left": make_synthetic_mano("left"), "right": make_synthetic_mano("right")}


def _matrices(n, g, exact=False):
    """(n,16,3,3) float64: exact rotations, + 0.1 sigma noise, det < 0, 2 R and Gaussian, mixed per joint."""
    R = rodrigues(torch.randn(n * 16, 3, generator=g, dtype=torch.float64)).view(n, 16, 3, 3)
    if exact:
        return R
    noise = torch.randn(n, 16, 3, 3, generator=g, dtype=torch.float64)
    cls = (torch.arange(n)[:, None] + torch.arange(16)[None, :]) % 5
    out = torch.where((cls == 0)[..., None, None], R, R + 0.1 * noise)
    out = torch.where((cls == 2)[..., None, None], -(R + 0.05 * noise), out)
    out = torch.where((cls == 3)[..., None, None], 2 * R, out)
    return torch.where((cls == 4)[..., None, None], noise, out)


class Case:
    """A layer configuration, its float64 restatement and seeded inputs (axis-angle edge poses: zero, 1e-6, pi)."""

    def __init__(self, assets, side="right", n=9, center_idx=9, rotmat=False, use_pca=False, ncomps=45, flat=False,
                 betas_mode="given", trans=False, palm=False, exact=False, seed=0):
        from mano.manolayer import ManoLayer
        g = torch.Generator().manual_seed(seed)
        self.rotmat, self.palm, self.betas_mode = rotmat, palm, betas_mode
        if rotmat:
            self.layer = ManoLayer(center_idx=center_idx, side=side, use_pca=False, joint_rot_mode="rotmat",
                                   asset=assets[side]).cuda()
            self.ref = TorchManoFunc(assets[side], side, use_pca=False, center_idx=center_idx, device="cuda")
            self.pose = _matrices(n, g, exact)
        else:
            self.layer = ManoLayer(center_idx=center_idx, flat_hand_mean=flat, ncomps=ncomps, side=side,
                                   use_pca=use_pca, asset=assets[side]).cuda()
            self.ref = TorchManoFunc(assets[side], side, use_pca=use_pca, ncomps=ncomps, flat_hand_mean=flat,
                                     center_idx=center_idx, device="cuda")
            self.pose = torch.randn(n, 3 + (ncomps if use_pca else 45), generator=g, dtype=torch.float64) * 0.5
            if n >= 3:
                self.pose[0] = 0.0
                self.pose[1] = 1e-6
                self.pose[2, :3] = torch.tensor([3.14159, 0.0, 0.0])
        self.betas = torch.randn(n, 10, generator=g, dtype=torch.float64)
        self.trans = torch.randn(n, 3, generator=g, dtype=torch.float64) * 0.1 if trans else None
        self.tangents = [torch.randn(x.shape, generator=g, dtype=torch.float64) for x in self.primals(torch.float64)]

    def primals(self, dtype):
        out = [self.pose, self.betas] + ([self.trans] if self.trans is not None else [])
        return [x.to("cuda", dtype) for x in out]

    def fn(self, impl):
        """impl 'gpu' or 'ref' -> f(pose, betas[, trans]) -> (verts, joints[, center])."""
        def f(pose, betas, trans=None):
            b = None if self.betas_mode == "default" else betas
            if impl == "ref":
                call = self.ref.from_rotmats if self.rotmat else self.ref
                out = call(pose, b, trans, share_betas=self.betas_mode == "shared", root_palm=self.palm)
            else:
                kw = dict(root_palm=torch.Tensor([int(self.palm)]))
                if b is not None:
                    kw["th_betas"] = b
                if trans is not None:
                    kw["th_trans"] = trans
                if self.betas_mode == "shared":
                    kw["share_betas"] = torch.Tensor([1])
                out = self.layer(pose, **kw)
            return tuple(o for o in out if o is not None)
        return f


def _close(got, exp, what):
    for i, (a, e) in enumerate(zip(got, exp)):
        a = a.detach().double().cpu()
        assert torch.isfinite(a).all(), (what, i)
        err = rel_err(a.numpy(), e.detach().cpu().numpy())
        assert err < TOL, (what, i, err)


CASES = [dict(), dict(center_idx=0), dict(center_idx=None), dict(use_pca=True, ncomps=6), dict(flat=True),
         dict(betas_mode="default"), dict(betas_mode="shared"), dict(trans=True), dict(palm=True),
         dict(palm=True, center_idx=None), dict(rotmat=True), dict(rotmat=True, palm=True),
         dict(rotmat=True, center_idx=None, trans=True), dict(rotmat=True, exact=True)]


@pytest.mark.parametrize("side", ["right", "left"])
@pytest.mark.parametrize("kw", CASES, ids=lambda kw: ",".join(f"{k}={v}" for k, v in kw.items()) or "default")
def test_jvp_and_forward_ad_match_float64_restatement(assets, side, kw):
    c = Case(assets, side=side, seed=len(str(kw)), **kw)
    prim32, tan = c.primals(torch.float32), [t.to("cuda") for t in c.tangents]
    out, t32 = jvp(c.fn("gpu"), tuple(prim32), tuple(t.float() for t in tan))
    ref_out, t64 = jvp(c.fn("ref"), tuple(c.primals(torch.float64)), tuple(tan))
    assert len(t32) == len(t64)
    _close(out, ref_out, "primal")
    _close(t32, t64, "jvp")
    with fwAD.dual_level():
        duals = [fwAD.make_dual(p, t.float()) for p, t in zip(prim32, tan)]
        fa = [fwAD.unpack_dual(o).tangent for o in c.fn("gpu")(*duals)]
    _close(fa, t64, "forward_ad")


@pytest.mark.parametrize("kw", [dict(), dict(use_pca=True, ncomps=6, center_idx=None), dict(rotmat=True),
                                dict(rotmat=True, palm=True, side="left"), dict(palm=True, trans=True)])
def test_jacfwd_matches_float64_and_jacrev(assets, kw):
    c = Case(assets, n=5, seed=3, **kw)
    argnums = tuple(range(len(c.primals(torch.float32))))
    joints = lambda impl: (lambda *a: c.fn(impl)(*a)[1])
    jf = jacfwd(joints("gpu"), argnums=argnums)(*c.primals(torch.float32))
    jr = jacrev(joints("gpu"), argnums=argnums)(*c.primals(torch.float32))
    je = jacfwd(joints("ref"), argnums=argnums)(*c.primals(torch.float64))
    _close(jf, je, "jacfwd")
    _close(jf, [x.double() for x in jr], "jacfwd vs jacrev")


def test_per_hand_joint_jacobian_vmapped_over_hands(assets):
    """The fitting use: the (21*3) x 58 Jacobian of every hand, vmap over hands of jacfwd (one JVP launch)."""
    c = Case(assets, n=64, seed=4)
    f = lambda impl: (lambda p, b: c.fn(impl)(p[None], b[None])[1][0])
    got = vmap(jacfwd(f("gpu"), argnums=(0, 1)))(*c.primals(torch.float32))
    exp = vmap(jacfwd(f("ref"), argnums=(0, 1)))(*c.primals(torch.float64))
    assert got[0].shape == (64, 21, 3, 48) and got[1].shape == (64, 21, 3, 10)
    _close(got, exp, "per-hand jacobian")


@pytest.mark.parametrize("rotmat,palm,center_idx", [(False, False, 9), (False, True, None), (True, False, 0),
                                                    (True, True, 9)])
def test_dot_product_jvp_kernel_vs_backward_kernel(assets, rotmat, palm, center_idx):
    """<g, J t> == <J^T g, t>, between acr_b200_mano_layer_jvp and the fused backward."""
    from acr_b200 import lib as L
    from acr_b200 import ops
    c = Case(assets, n=37, rotmat=rotmat, palm=palm, center_idx=center_idx, seed=5)
    model, side = c.layer.packed_model(), 1
    mode = L.POSE_ROTMAT if rotmat else L.POSE_AXISANG
    pose = c.pose.cuda().float() if rotmat else c.pose.cuda().float()[:, :48]
    betas = c.betas.cuda().float()
    g = torch.Generator().manual_seed(6)
    T = 6
    tp = torch.randn((T,) + tuple(pose.shape), generator=g).cuda()
    tb = torch.randn(T, 37, 10, generator=g).cuda()
    gv, gj, gc = torch.randn(37, 778, 3, generator=g).cuda(), torch.randn(37, 21, 3, generator=g).cuda(), \
        torch.randn(37, 1, 3, generator=g).cuda()
    tv, tj, tc = ops.mano_layer_jvp(model, side, pose, mode, betas, center_idx, palm, tp, tb)
    dp, db = ops.mano_layer_backward(model, side, pose, mode, betas, center_idx, palm, gv, gj,
                                     gc if center_idx is not None else None)
    for t in range(T):
        lhs = (gv.double() * tv[t]).sum() + (gj.double() * tj[t]).sum()
        if center_idx is not None:
            lhs = lhs + (gc.double() * tc[t]).sum()
        rhs = (dp.double() * tp[t]).sum() + (db.double() * tb[t]).sum()
        assert abs(float(lhs - rhs)) <= 1e-4 * max(abs(float(rhs)), float((dp.double() * tp[t]).abs().sum())), t


@pytest.mark.parametrize("palm", [False, True])
def test_rotmat_tangents_finite_at_exact_rotations(assets, palm):
    c = Case(assets, n=33, rotmat=True, exact=True, palm=palm, seed=7)
    eye = torch.eye(3, dtype=torch.float64).expand(3, 16, 3, 3)
    c.pose = torch.cat([c.pose, eye])              # the identity too
    c.betas = torch.cat([c.betas, c.betas[:3]])
    t = torch.randn(c.pose.shape, generator=torch.Generator().manual_seed(8), dtype=torch.float64)
    _, t32 = jvp(lambda p: c.fn("gpu")(p, c.betas.cuda().float())[:2], (c.pose.cuda().float(),), (t.cuda().float(),))
    _, t64 = jvp(lambda p: c.fn("ref")(p, c.betas.cuda())[:2], (c.pose.cuda(),), (t.cuda(),))
    _close(t32, t64, "exact rotations")


@pytest.mark.parametrize("rotmat", [False, True])
def test_vmap_forward_bit_identical_to_unbatched(assets, rotmat):
    c = Case(assets, n=11, rotmat=rotmat, seed=9)
    f = c.fn("gpu")
    P = torch.stack([c.pose, c.pose * 0.9, c.pose * 1.1]).cuda().float()
    B = torch.stack([c.betas, c.betas, -c.betas]).cuda().float()
    got = vmap(f)(P, B)
    with torch.no_grad():
        for i in range(3):
            for a, e in zip(got, f(P[i], B[i])):
                assert torch.equal(a[i], e)


def test_vmap_of_grad(assets):
    c = Case(assets, n=16, seed=10, use_pca=True, ncomps=12)
    loss = lambda impl: (lambda p, b: c.fn(impl)(p[None], b[None])[1].square().sum())
    got = vmap(grad(loss("gpu"), argnums=(0, 1)))(*c.primals(torch.float32))
    exp = vmap(grad(loss("ref"), argnums=(0, 1)))(*c.primals(torch.float64))
    _close(got, exp, "vmap grad")


@pytest.mark.parametrize("rotmat,palm", [(False, False), (False, True), (True, False), (True, True)])
def test_joints_only_form_and_tangent_tiling(assets, rotmat, palm):
    """Without tverts the kernel runs the joints-only form: its joints agree with the full form's.  A tangent's
    result is the same bits alone or among 58, and repeated calls are bit-identical."""
    from acr_b200 import lib as L
    from acr_b200 import ops
    c = Case(assets, n=21, rotmat=rotmat, palm=palm, center_idx=None if palm else 9, seed=11)
    model, mode = c.layer.packed_model(), L.POSE_ROTMAT if rotmat else L.POSE_AXISANG
    pose = c.pose.cuda().float() if rotmat else c.pose.cuda().float()[:, :48]
    betas, center = c.betas.cuda().float(), None if palm else 9
    g = torch.Generator().manual_seed(12)
    tp = torch.randn((58,) + tuple(pose.shape), generator=g).cuda()
    tb = torch.randn(58, 21, 10, generator=g).cuda()
    run = lambda tp_, tb_, verts: ops.mano_layer_jvp(model, 1, pose, mode, betas, center, palm, tp_, tb_, verts)
    full, joints = run(tp, tb, True), run(tp, tb, False)
    assert joints[0] is None
    assert rel_err(joints[1].cpu().numpy(), full[1].cpu().numpy()) < 1e-6
    assert rel_err(joints[2].cpu().numpy(), full[2].cpu().numpy()) < 1e-6
    again = run(tp, tb, True)
    for a, b in zip(full, again):
        assert torch.equal(a, b)
    for t in (0, 5, 57):
        alone = run(tp[t:t + 1], tb[t:t + 1], True)
        for a, b in zip(alone, full):
            assert torch.equal(a[0], b[t]), t
        alone_j = run(tp[t:t + 1], tb[t:t + 1], False)
        assert torch.equal(alone_j[1][0], joints[1][t])


@pytest.mark.parametrize("rotmat", [False, True])
def test_second_order_raises(assets, rotmat):
    c = Case(assets, n=4, rotmat=rotmat, seed=13)
    p, b = c.primals(torch.float32)
    loss = lambda p_: c.fn("gpu")(p_, b)[1].square().sum()
    with pytest.raises(RuntimeError, match="first-order"):
        hessian(loss)(p)
    with pytest.raises(RuntimeError, match="first-order"):
        jvp(grad(loss), (p,), (torch.ones_like(p),))
    x = p.clone().requires_grad_()
    dx, = torch.autograd.grad(loss(x), x, create_graph=True)
    with pytest.raises(RuntimeError, match="first-order"):
        torch.autograd.grad(dx.sum(), x)
