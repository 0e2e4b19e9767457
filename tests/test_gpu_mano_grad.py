"""GPU: ManoLayer gradients (fused MANO backward kernel, through autograd) against autograd of the float64 torch
restatement (tests/mano_torch_ref.py), plus the properties of the autograd wiring."""
import pytest
import torch

from tests.helpers import rel_err
from tests.mano_torch_ref import TorchMano

pytestmark = pytest.mark.gpu
TOL = 1e-4   # BASELINE.json: 1e-4 relative fp32 tolerance


@pytest.fixture(scope="module")
def assets():
    from acr_b200.synth import make_synthetic_mano
    return {"left": make_synthetic_mano("left"), "right": make_synthetic_mano("right")}


def _layer(assets, side, center_idx, use_pca, ncomps, flat):
    from mano.manolayer import ManoLayer
    return ManoLayer(center_idx=center_idx, flat_hand_mean=flat, ncomps=ncomps, side=side, use_pca=use_pca,
                     asset=assets[side]).cuda()


def run_case(assets, side="right", n=9, center_idx=9, use_pca=False, ncomps=45, flat=False, betas_mode="given",
             trans=False, loss="all", edges=True, seed=0):
    """-> list of (name, gpu grad, float64 reference grad)."""
    g = torch.Generator().manual_seed(seed)
    ncoef = 3 + (ncomps if use_pca else 45)
    pose = torch.randn(n, ncoef, generator=g, dtype=torch.float64) * 0.5
    if edges and n >= 3:
        pose[0] = 0.0
        pose[1] = 1e-6
        pose[2, :3] = torch.tensor([3.14159, 0.0, 0.0])
    betas = torch.randn(n, 10, generator=g, dtype=torch.float64)
    tr = torch.randn(n, 3, generator=g, dtype=torch.float64) * 0.1 if trans else None
    gv, gj, gc = (torch.randn(n, 778, 3, generator=g, dtype=torch.float64), torch.randn(n, 21, 3, generator=g, dtype=torch.float64),
                  torch.randn(n, 1, 3, generator=g, dtype=torch.float64))
    layer = _layer(assets, side, center_idx, use_pca, ncomps, flat)
    ref = TorchMano(assets[side], side, use_pca=use_pca, ncomps=ncomps, flat_hand_mean=flat, center_idx=center_idx,
                    device="cuda")

    def go(fn, dtype):
        p = pose.to("cuda", dtype).requires_grad_()
        b = betas.to("cuda", dtype).requires_grad_() if betas_mode != "default" else None
        t = tr.to("cuda", dtype).requires_grad_() if tr is not None else None
        kw = {}
        if b is not None:
            kw["th_betas"] = b
        if t is not None:
            kw["th_trans"] = t
        if betas_mode == "shared":
            kw["share_betas"] = torch.Tensor([1])
        if fn is ref:
            v, j, c = ref(p, b, t, share_betas=betas_mode == "shared")
        else:
            v, j, c = fn(p, **kw)
        terms = {"verts": (gv, v), "joints": (gj, j), "center": (gc, c)}
        use = ["verts", "joints", "center"] if loss == "all" else [loss]
        total = sum((terms[k][0].to("cuda", dtype) * terms[k][1]).sum() for k in use if terms[k][1] is not None)
        total.backward()
        return p.grad, (None if b is None else b.grad), (None if t is None else t.grad)

    got = go(layer, torch.float32)
    exp = go(ref, torch.float64)
    out = []
    for name, a, e in zip(("pose", "betas", "trans"), got, exp):
        assert (a is None) == (e is None), name
        if a is not None:
            out.append((name, a.double().cpu(), e.cpu()))
    return out


def _check(res):
    for name, a, e in res:
        assert torch.isfinite(a).all(), name
        err = rel_err(a.numpy(), e.numpy())
        assert err < TOL, (name, err)


@pytest.mark.parametrize("side", ["right", "left"])
@pytest.mark.parametrize("n", [1, 7, 8, 9, 512, 4096])
def test_grad_sizes(assets, side, n):
    _check(run_case(assets, side=side, n=n, seed=n))


@pytest.mark.parametrize("side", ["right", "left"])
@pytest.mark.parametrize("center_idx,loss", [(c, l) for c in (9, 0, None) for l in ("all", "joints", "verts", "center")
                                             if not (c is None and l == "center")])   # no centre output without one
def test_grad_centre_and_losses(assets, side, center_idx, loss):
    _check(run_case(assets, side=side, n=9, center_idx=center_idx, loss=loss, seed=11))


@pytest.mark.parametrize("ncomps", [6, 45])
@pytest.mark.parametrize("flat", [True, False])
def test_grad_pca(assets, ncomps, flat):
    res = run_case(assets, n=33, use_pca=True, ncomps=ncomps, flat=flat, seed=ncomps)
    assert [r[0] for r in res] == ["pose", "betas"]
    _check(res)


@pytest.mark.parametrize("flat", [True, False])
def test_grad_flat_hand_mean_axisang(assets, flat):
    _check(run_case(assets, n=17, flat=flat, seed=5))


def test_grad_share_betas(assets):
    _check(run_case(assets, n=12, betas_mode="shared", seed=6))


def test_grad_default_betas_is_none(assets):
    res = run_case(assets, n=10, betas_mode="default", seed=7)
    assert [r[0] for r in res] == ["pose"]
    _check(res)


@pytest.mark.parametrize("loss", ["all", "center"])
def test_grad_trans(assets, loss):
    res = run_case(assets, n=10, trans=True, loss=loss, seed=8)
    # with th_trans the third output is th_trans itself: a loss on it alone reaches only th_trans
    assert [r[0] for r in res] == (["pose", "betas", "trans"] if loss == "all" else ["trans"])
    _check(res)


def test_forward_identical_with_and_without_grad(assets):
    layer = _layer(assets, "right", 9, True, 12, False)
    g = torch.Generator().manual_seed(9)
    pose, betas = torch.randn(37, 15, generator=g).cuda(), torch.randn(37, 10, generator=g).cuda()
    with torch.no_grad():
        ref = layer(pose, th_betas=betas)
    out = layer(pose.clone().requires_grad_(), th_betas=betas.clone().requires_grad_())
    assert out[0].requires_grad and out[2].requires_grad
    for a, b in zip(out, ref):
        assert torch.equal(a.detach(), b)
    plain = layer(pose, th_betas=betas)     # grad mode on, nothing requires grad: today's launch
    assert not plain[0].requires_grad
    for a, b in zip(plain, ref):
        assert torch.equal(a, b)


def test_backward_deterministic_and_first_order_only(assets):
    layer = _layer(assets, "left", 9, False, 45, False)
    g = torch.Generator().manual_seed(10)
    pose, betas = torch.randn(300, 48, generator=g).cuda() * 0.5, torch.randn(300, 10, generator=g).cuda()
    gv = torch.randn(300, 778, 3, generator=g).cuda()

    def grads(create_graph=False):
        p, b = pose.clone().requires_grad_(), betas.clone().requires_grad_()
        v, j, c = layer(p, th_betas=b)
        loss = (gv * v).sum() + j.square().sum() + c.sum()
        return p, torch.autograd.grad(loss, (p, b), create_graph=create_graph)

    _, (p1, b1) = grads()
    _, (p2, b2) = grads()
    assert torch.equal(p1, p2) and torch.equal(b1, b2)
    p, (dp, _) = grads(create_graph=True)
    with pytest.raises(RuntimeError):
        torch.autograd.grad(dp.sum(), p)


def test_fit_joints(assets):
    """Adam fit of 64 hands' pose and betas to target joints: the GPU layer tracks the float64 restatement."""
    side, n, steps = "right", 64, 300
    g = torch.Generator().manual_seed(7)
    p0 = torch.randn(n, 48, generator=g, dtype=torch.float64) * 0.4
    b0 = torch.randn(n, 10, generator=g, dtype=torch.float64)
    pt = p0 + torch.randn(n, 48, generator=g, dtype=torch.float64) * 0.15
    bt = b0 + torch.randn(n, 10, generator=g, dtype=torch.float64) * 0.5
    ref = TorchMano(assets[side], side, use_pca=False, flat_hand_mean=False, center_idx=9, device="cuda")
    layer = _layer(assets, side, 9, False, 45, False)
    with torch.no_grad():
        target = ref(pt.cuda(), bt.cuda())[1]

    def fit(fn, dtype):
        p, b = p0.to("cuda", dtype).requires_grad_(), b0.to("cuda", dtype).requires_grad_()
        tgt = target.to(dtype)
        opt = torch.optim.Adam([p, b], lr=0.01)
        first = None
        for _ in range(steps):
            opt.zero_grad()
            j = fn(p, b)
            loss = (j - tgt).square().sum()
            loss.backward()
            opt.step()
            first = loss.item() if first is None else first
        with torch.no_grad():
            last = (fn(p, b) - tgt).square().sum().item()
        return first, last

    g0, g1 = fit(lambda p, b: layer(p, th_betas=b)[1], torch.float32)
    r0, r1 = fit(lambda p, b: ref(p, b)[1], torch.float64)
    print(f"fit: gpu {g0:.4e} -> {g1:.4e}, float64 reference {r0:.4e} -> {r1:.4e}")
    assert g0 / g1 >= 100 and r0 / r1 >= 100
    assert g1 <= 2 * r1
