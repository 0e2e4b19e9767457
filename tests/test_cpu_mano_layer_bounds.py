"""CPU: the float64 statements and bounds of tests/mano_layer_ref.py.  The statements equal the autograd / torch.func
restatements per element, their float32 runs (the kernels' operation order) stay within the bounds, and errors that the
old max-norm criterion (rel_err < 1e-4) accepts are rejected by them."""
import pytest
import torch
from torch.func import jvp

from tests import mano_layer_ref as L
from tests.helpers import rel_err
from tests.mano_jvp_ref import TorchManoFunc
from tests.mano_rotmat_ref import TorchManoRot
from tests.tail_ref import mano_forward64
from tests.mano_layer_ref import _r32, edge_poses, matrices

F64 = torch.float64


@pytest.fixture(scope="module")
def assets():
    from acr_b200.synth import make_synthetic_mano
    return {"left": make_synthetic_mano("left"), "right": make_synthetic_mano("right")}


def _data(n, mode, seed):
    g = torch.Generator().manual_seed(seed)
    pose = matrices(n, g) if mode == "rotmat" else edge_poses(n, g)
    r = lambda *s: _r32(torch.randn(*s, generator=g, dtype=F64))
    return pose, r(n, 10), r(n, 778, 3), r(n, 21, 3), r(n, 3)


def _same(label, got, exp, bounded, hand_axis=0):
    """float64 statement == float64 restatement: per element within 1e-6 of the bound, and 1e-12 in max norm."""
    exp = exp.detach().reshape(got.v.shape)
    shape = [1] * exp.dim()
    shape[hand_axis] = -1
    keep = bounded.view(shape).expand(exp.shape)
    d = (got.v - exp).abs()[keep]
    assert float(d.max()) <= 1e-12 * float(exp.abs().max()), (label, float(d.max()))
    assert (d <= 1e-6 * got.e.expand(got.v.shape)[keep]).all(), label


@pytest.mark.parametrize("side", ["right", "left"])
@pytest.mark.parametrize("mode,flat", [("aa", True), ("aa", False), ("rotmat", True)])
@pytest.mark.parametrize("palm", [False, True])
def test_statements_equal_autograd(assets, side, mode, flat, palm):
    n = 16
    pose, betas, gv, gj, gc = _data(n, mode, 1)
    model = L.model_from_asset(assets[side], flat_hand_mean=flat, round_joints=False)
    ref = TorchManoRot(assets[side], side, use_pca=False, flat_hand_mean=flat, center_idx=9)
    p, b = pose.clone().requires_grad_(), betas.clone().requires_grad_()
    v, j, c = (ref.from_rotmats if mode == "rotmat" else ref)(p, b, root_palm=palm)
    ((gv * v).sum() + (gj * j).sum() + (gc[:, None] * c).sum()).backward()
    fw = L.layer_forward(model, side, pose, betas, mode, 9, palm)
    bw = L.layer_backward(model, side, pose, betas, mode, 9, palm, gv, gj, gc)
    ok = fw["bounded"]
    for k, e in (("verts", v), ("joints", j), ("center", c)):
        _same(k, fw[k], e, ok)
    _same("dpose", bw["dpose"], p.grad, ok)
    _same("dbetas", bw["dbetas"], b.grad, ok)


@pytest.mark.parametrize("mode", ["aa", "rotmat"])
@pytest.mark.parametrize("palm", [False, True])
def test_jvp_statement_equals_torch_func(assets, mode, palm):
    n, T, side = 12, 3, "right"
    pose, betas, _, _, _ = _data(n, mode, 2)
    g = torch.Generator().manual_seed(3)
    tpose = _r32(torch.randn((T,) + tuple(pose.shape), generator=g, dtype=F64))
    tbetas = _r32(torch.randn(T, n, 10, generator=g, dtype=F64))
    model = L.model_from_asset(assets[side], round_joints=False)
    ref = TorchManoFunc(assets[side], side, use_pca=False, flat_hand_mean=True, center_idx=9)
    f = (lambda p, b: ref.from_rotmats(p, b, root_palm=palm)) if mode == "rotmat" else (lambda p, b: ref(p, b, root_palm=palm))
    out = L.layer_jvp(model, side, pose, betas, mode, 9, palm, tpose, tbetas)
    for u in range(T):
        _, (tv, tj, tc) = jvp(f, (pose, betas), (tpose[u], tbetas[u]))
        for k, e in (("tverts", tv), ("tjoints", tj), ("tcenter", tc)):
            _same(k, out[k][u], e, out["bounded"])


def test_forward_statement_equals_tail_ref(assets):
    n = 16
    pose, betas, _, _, _ = _data(n, "aa", 4)
    exp = mano_forward64(assets["right"], pose.numpy(), betas.numpy(), "right", 9)
    model = L.model_from_asset(assets["right"], flat_hand_mean=False, round_joints=False)   # the oracle adds the mean
    got = L.layer_forward(model, "right", pose, betas, "aa", 9, False)
    for k in ("verts", "joints", "center"):
        _same(k, got[k], torch.as_tensor(exp[k]), got["bounded"])


def _ratio(got32, exp):
    err = (got32.v.double() - exp.v).abs()
    b = exp.e.expand(exp.v.shape)
    return float(torch.where(b > 0, err / b, torch.where(err > 0, torch.inf, 0.0)).max())


@pytest.mark.parametrize("mode", ["aa", "rotmat"])
@pytest.mark.parametrize("palm", [False, True])
def test_float32_run_within_bounds(assets, mode, palm):
    n, side = 24, "left" if palm else "right"
    pose, betas, gv, gj, gc = _data(n, mode, 5)
    model = L.model_from_asset(assets[side])
    g = torch.Generator().manual_seed(6)
    tpose = _r32(torch.randn((2,) + tuple(pose.shape), generator=g, dtype=F64))
    tbetas = _r32(torch.randn(2, n, 10, generator=g, dtype=F64))
    runs = {}
    for dt in (torch.float64, torch.float32):
        runs[dt] = {**L.layer_forward(model, side, pose, betas, mode, 9, palm, dtype=dt),
                    **L.layer_backward(model, side, pose, betas, mode, 9, palm, gv, gj, gc, dtype=dt),
                    **L.layer_jvp(model, side, pose, betas, mode, 9, palm, tpose, tbetas, dtype=dt)}
    ok = runs[torch.float64]["bounded"]
    assert ok.sum() >= n // 2
    for k in ("verts", "joints", "center", "dpose", "dbetas", "tverts", "tjoints", "tcenter"):
        ax = 1 if k.startswith("t") else 0
        sel = lambda x: x[:, ok] if ax else x[ok]
        r = _ratio(sel(runs[torch.float32][k]), sel(runs[torch.float64][k]))
        print(f"  {mode}{' palm' if palm else ''} {k}: float32 worst err/bound {r:.3e}")
        assert 1e-3 < r <= 1.0, (k, r)


@pytest.mark.parametrize("defect,palm", [("tip445", False), ("palm96", True), ("centre0", True)])
def test_planted_defects(assets, defect, palm):
    """A fingertip read from a neighbouring vertex, half the palm's cotangent on the wrong vertex, the centre term
    also subtracting the palm's cotangent.  On evenly scaled cotangents these errors are large enough (1e-2 .. 1e-1
    of the batch maximum) for the max-norm check to reject them too.  This batch shows the weakness that check has
    whenever hands differ in scale: hand 0 carries 1e4 times the vertex and centre cotangents of the others (and no
    joint cotangent), the max-norm check normalises by it and accepts, the per-element bound does not."""
    n = 32
    pose, betas, gv, gj, gc = _data(n, "aa", 7)
    gv[0] *= 1e4
    gc[0] *= 1e4
    gj[0] = 0.0
    model = L.model_from_asset(assets["right"])
    exp = L.layer_backward(model, "right", pose, betas, "aa", 9, palm, gv, gj, gc)
    bad = L.layer_backward(model, "right", pose, betas, "aa", 9, palm, gv, gj, gc, dtype=torch.float32, defect=defect)
    for k in ("dpose", "dbetas"):
        old = rel_err(bad[k].v.double().numpy(), exp[k].v.numpy())
        r = _ratio(bad[k], exp[k])
        print(f"  {defect} {k}: rel_err {old:.2e} (accepted by < 1e-4), worst err/bound {r:.1f}")
        assert old < 1e-4 and r > 1.0, (k, old, r)


def test_js_defect_rejected(assets):
    """A 1e-3 relative error on the J_regressor . shapedirs term of dbetas, on the inputs of test_gpu_mano_grad's
    test_grad_sizes (seed = n, all three cotangents).  The max-norm check rejects it there too (rel_err ~ 5e-4); the
    point is that the per-element bound is tight enough to see it."""
    n = 32
    g = torch.Generator().manual_seed(n)
    pose = _r32(torch.randn(n, 48, generator=g, dtype=F64) * 0.5)
    betas = _r32(torch.randn(n, 10, generator=g, dtype=F64))
    gv, gj, gc = (_r32(torch.randn(n, 778, 3, generator=g, dtype=F64)), _r32(torch.randn(n, 21, 3, generator=g, dtype=F64)),
                  _r32(torch.randn(n, 1, 3, generator=g, dtype=F64)))
    model = L.model_from_asset(assets["right"], flat_hand_mean=False)
    exp = L.layer_backward(model, "right", pose, betas, "aa", 9, False, gv, gj, gc)
    good = L.layer_backward(model, "right", pose, betas, "aa", 9, False, gv, gj, gc, dtype=torch.float32)
    bad = L.layer_backward(model, "right", pose, betas, "aa", 9, False, gv, gj, gc, dtype=torch.float32, defect="js")
    r_good, r_bad = _ratio(good["dbetas"], exp["dbetas"]), _ratio(bad["dbetas"], exp["dbetas"])
    print(f"  js dbetas: worst err/bound {r_good:.3e} without the defect, {r_bad:.2f} with it")
    assert r_good <= 1.0 < r_bad
