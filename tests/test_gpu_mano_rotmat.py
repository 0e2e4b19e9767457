"""GPU: ManoLayer's rotation-matrix mode and root_palm (the SO(3) projection and its VJP fused into the MANO
kernels) against the reference's own outputs (tests/golden/mano_rotmat_golden.npz) and against autograd of the
float64 restatement (tests/mano_rotmat_ref.py)."""
import os

import numpy as np
import pytest
import torch

from tests.helpers import GOLDEN, rel_err
from tests.mano_rotmat_ref import TorchManoRot
from tests.mano_torch_ref import rodrigues

pytestmark = pytest.mark.gpu
TOL = 1e-4   # BASELINE.json: 1e-4 relative fp32 tolerance


@pytest.fixture(scope="module")
def assets():
    from acr_b200.synth import make_synthetic_mano
    return {"left": make_synthetic_mano("left"), "right": make_synthetic_mano("right")}


def _layer(assets, side, center_idx, rotmat=True, flat=False):
    from mano.manolayer import ManoLayer
    if rotmat:
        return ManoLayer(center_idx=center_idx, side=side, use_pca=False, joint_rot_mode="rotmat", asset=assets[side]).cuda()
    return ManoLayer(center_idx=center_idx, side=side, use_pca=False, flat_hand_mean=flat, asset=assets[side]).cuda()


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


# ----------------------------------------------------------------------------------------------- forward
@pytest.mark.parametrize("side", ["right", "left"])
def test_forward_matches_reference_golden(assets, side):
    g = np.load(os.path.join(GOLDEN, "mano_rotmat_golden.npz"))
    vi = g["vert_idx"]
    for name in g["case_names"]:
        name = str(name)
        mode = name.split("_")[0]
        center = None if "_none" in name else 9
        layer = _layer(assets, side, center, rotmat=mode == "rotmat")
        pose = torch.from_numpy(g[f"{side}__{'mats' if mode == 'rotmat' else 'aa'}"]).cuda()
        kw = dict(th_betas=torch.from_numpy(g[f"{side}__betas"]).cuda(), root_palm=torch.Tensor([int(name.endswith("_palm"))]))
        if "_trans" in name:
            kw["th_trans"] = torch.from_numpy(g[f"{side}__trans"]).cuda()
        v, j, c = layer(pose, **kw)
        assert rel_err(v.cpu().numpy()[:, vi], g[f"{side}__{name}__verts"]) < TOL, name
        assert rel_err(j.cpu().numpy(), g[f"{side}__{name}__joints"]) < TOL, name
        if f"{side}__{name}__center" in g.files:
            assert rel_err(c.cpu().numpy(), g[f"{side}__{name}__center"]) < TOL, name
        else:
            assert c is None


def run_case(assets, side="right", n=9, center_idx=9, rotmat=True, palm=False, trans=False, loss="all", exact=False,
             seed=0, want_grad=True):
    """-> (forward pairs, gradient pairs): each (name, gpu, float64 reference)."""
    g = torch.Generator().manual_seed(seed)
    pose = _matrices(n, g, exact) if rotmat else torch.randn(n, 48, generator=g, dtype=torch.float64) * 0.5
    betas = torch.randn(n, 10, generator=g, dtype=torch.float64)
    tr = torch.randn(n, 3, generator=g, dtype=torch.float64) * 0.1 if trans else None
    gv, gj, gc = (torch.randn(n, 778, 3, generator=g, dtype=torch.float64), torch.randn(n, 21, 3, generator=g, dtype=torch.float64),
                  torch.randn(n, 1, 3, generator=g, dtype=torch.float64))
    layer = _layer(assets, side, center_idx, rotmat)
    ref = TorchManoRot(assets[side], side, use_pca=False, flat_hand_mean=rotmat, center_idx=center_idx, device="cuda")

    def go(fn, dtype):
        p = pose.to("cuda", dtype).requires_grad_(want_grad)
        b = betas.to("cuda", dtype).requires_grad_(want_grad)
        t = tr.to("cuda", dtype).requires_grad_(want_grad) if tr is not None else None
        if fn is ref:
            outs = (ref.from_rotmats if rotmat else ref)(p, b, t, root_palm=palm)
        else:
            kw = dict(th_betas=b, root_palm=torch.Tensor([int(palm)]))
            if t is not None:
                kw["th_trans"] = t
            outs = fn(p, **kw)
        if not want_grad:
            return outs, ()
        terms = {"verts": (gv, outs[0]), "joints": (gj, outs[1]), "center": (gc, outs[2])}
        use = ["verts", "joints", "center"] if loss == "all" else [loss]
        total = sum((terms[k][0].to("cuda", dtype) * terms[k][1]).sum() for k in use if terms[k][1] is not None)
        total.backward()
        return outs, (p.grad, b.grad, None if t is None else t.grad)

    got_o, got_g = go(layer, torch.float32)
    exp_o, exp_g = go(ref, torch.float64)
    fwd = [(k, a, e) for k, a, e in zip(("verts", "joints", "center"), got_o, exp_o)]
    grads = [(k, a, e) for k, a, e in zip(("pose", "betas", "trans"), got_g, exp_g)]
    return fwd, grads


def _check(pairs):
    for name, a, e in pairs:
        assert (a is None) == (e is None), name
        if a is None:
            continue
        a = a.detach().double().cpu()
        assert torch.isfinite(a).all(), name
        err = rel_err(a.numpy(), e.detach().cpu().numpy())
        assert err < TOL, (name, err)


@pytest.mark.parametrize("side", ["right", "left"])
@pytest.mark.parametrize("n", [1, 7, 8, 9, 512, 4096])
def test_forward_sizes(assets, side, n):
    with torch.no_grad():
        _check(run_case(assets, side=side, n=n, seed=n, want_grad=False)[0])


@pytest.mark.parametrize("side", ["right", "left"])
@pytest.mark.parametrize("rotmat", [True, False])
@pytest.mark.parametrize("center_idx,palm,trans", [(9, False, False), (0, False, False), (None, False, False),
                                                   (9, True, False), (None, True, False), (9, True, True),
                                                   (9, False, True)])
def test_forward_modes(assets, side, rotmat, center_idx, palm, trans):
    if not rotmat and not palm:
        pytest.skip("axis angles without the palm are covered by test_gpu_mano_grad.py")
    with torch.no_grad():
        _check(run_case(assets, side=side, n=19, center_idx=center_idx, rotmat=rotmat, palm=palm, trans=trans, seed=3,
                        want_grad=False)[0])


# ----------------------------------------------------------------------------------------------- gradients
@pytest.mark.parametrize("side", ["right", "left"])
@pytest.mark.parametrize("n", [1, 7, 8, 9, 512, 4096])
def test_grad_sizes(assets, side, n):
    fwd, grads = run_case(assets, side=side, n=n, seed=100 + n)
    _check(fwd)
    _check(grads)


@pytest.mark.parametrize("side", ["right", "left"])
@pytest.mark.parametrize("rotmat,palm", [(True, False), (True, True), (False, True)])
@pytest.mark.parametrize("center_idx,loss", [(c, l) for c in (9, 0, None) for l in ("all", "joints", "verts", "center")
                                             if not (c is None and l == "center")])
def test_grad_centre_and_losses(assets, side, rotmat, palm, center_idx, loss):
    if palm and center_idx == 0:
        pytest.skip("centring on the palm is not supported")
    _check(run_case(assets, side=side, n=9, center_idx=center_idx, rotmat=rotmat, palm=palm, loss=loss, seed=11)[1])


@pytest.mark.parametrize("rotmat,palm", [(True, False), (True, True), (False, True)])
@pytest.mark.parametrize("loss", ["all", "center"])
def test_grad_trans(assets, rotmat, palm, loss):
    _, grads = run_case(assets, n=10, rotmat=rotmat, palm=palm, trans=True, loss=loss, seed=8)
    if loss == "center":        # with th_trans the third output is th_trans itself: only th_trans gets a gradient
        assert grads[0][1] is None and grads[1][1] is None
        grads = grads[2:]
    _check(grads)


@pytest.mark.parametrize("palm", [False, True])
def test_grad_finite_at_exact_rotations(assets, palm):
    fwd, grads = run_case(assets, n=33, palm=palm, exact=True, seed=12)
    _check(fwd)
    _check(grads)


def test_backward_deterministic_and_first_order_only(assets):
    layer = _layer(assets, "left", 9)
    g = torch.Generator().manual_seed(10)
    mats = _matrices(300, g).float().cuda()
    betas = torch.randn(300, 10, generator=g).cuda()
    gv = torch.randn(300, 778, 3, generator=g).cuda()

    def grads(create_graph=False):
        p, b = mats.clone().requires_grad_(), betas.clone().requires_grad_()
        v, j, c = layer(p, th_betas=b, root_palm=torch.Tensor([1]))
        loss = (gv * v).sum() + j.square().sum() + c.sum()
        return p, torch.autograd.grad(loss, (p, b), create_graph=create_graph)

    _, (p1, b1) = grads()
    _, (p2, b2) = grads()
    assert p1.shape == mats.shape
    assert torch.equal(p1, p2) and torch.equal(b1, b2)
    p, (dp, _) = grads(create_graph=True)
    with pytest.raises(RuntimeError):
        torch.autograd.grad(dp.sum(), p)


def test_forward_identical_with_and_without_grad(assets):
    layer = _layer(assets, "right", 9)
    g = torch.Generator().manual_seed(9)
    mats, betas = _matrices(37, g).float().cuda(), torch.randn(37, 10, generator=g).cuda()
    with torch.no_grad():
        ref = layer(mats, th_betas=betas)
    out = layer(mats.clone().requires_grad_(), th_betas=betas.clone().requires_grad_())
    assert out[0].requires_grad
    for a, b in zip(out, ref):
        assert torch.equal(a.detach(), b)


def test_fit_rotmat_joints(assets):
    """Adam fit of 64 hands' rotation matrices and betas to target joints, from exact rotations."""
    side, n, steps = "right", 64, 300
    g = torch.Generator().manual_seed(7)
    aa0 = torch.randn(n * 16, 3, generator=g, dtype=torch.float64) * 0.4
    m0 = rodrigues(aa0).view(n, 16, 3, 3)
    mt = rodrigues(aa0 + torch.randn(n * 16, 3, generator=g, dtype=torch.float64) * 0.15).view(n, 16, 3, 3)
    b0 = torch.randn(n, 10, generator=g, dtype=torch.float64)
    bt = b0 + torch.randn(n, 10, generator=g, dtype=torch.float64) * 0.5
    ref = TorchManoRot(assets[side], side, use_pca=False, center_idx=9, device="cuda")
    layer = _layer(assets, side, 9)
    with torch.no_grad():
        target = ref.from_rotmats(mt.cuda(), bt.cuda())[1]

    def fit(fn, dtype):
        p, b = m0.to("cuda", dtype).requires_grad_(), b0.to("cuda", dtype).requires_grad_()
        tgt = target.to(dtype)
        opt = torch.optim.Adam([p, b], lr=0.01)
        first = None
        for _ in range(steps):
            opt.zero_grad()
            loss = (fn(p, b) - tgt).square().sum()
            loss.backward()
            assert torch.isfinite(p.grad).all()
            opt.step()
            first = loss.item() if first is None else first
        with torch.no_grad():
            last = (fn(p, b) - tgt).square().sum().item()
        return first, last

    g0, g1 = fit(lambda p, b: layer(p, th_betas=b)[1], torch.float32)
    r0, r1 = fit(lambda p, b: ref.from_rotmats(p, b)[1], torch.float64)
    print(f"rotmat fit: gpu {g0:.4e} -> {g1:.4e} ({g0 / g1:.0f}x), float64 reference {r0:.4e} -> {r1:.4e} ({r0 / r1:.0f}x)")
    assert g0 / g1 >= 100 and r0 / r1 >= 100
    assert g1 <= 2 * r1
