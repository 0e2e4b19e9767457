"""GPU: the MANO layer kernels -- ops.mano_backward (the pipeline's backward), ops.mano_layer_forward,
ops.mano_layer_backward and ops.mano_layer_jvp (full and joints-only) -- against the float64 statements of
tests/mano_layer_ref.py, every output element within its derived bound.  Each test prints the worst err / bound per
output class.  The rel_err checks of test_gpu_mano_grad.py, _jvp.py and _rotmat.py stay; this file adds to them."""
import pytest
import torch

from tests import mano_layer_ref as L
from tests.mano_layer_ref import _r32, edge_poses, matrices

pytestmark = pytest.mark.gpu
GROUP = 64      # hands per float64 evaluation (bounds the host memory of the partial sums at n = 4096)


@pytest.fixture(scope="module")
def layers():
    """(side, mode, flat) -> (packed model on the GPU, its float64 unpacking)."""
    from acr_b200.synth import make_synthetic_mano
    from mano.manolayer import ManoLayer
    cache = {}

    def get(side, mode, flat=True):
        key = (side, mode, flat)
        if key not in cache:
            kw = dict(joint_rot_mode="rotmat") if mode == "rotmat" else dict(flat_hand_mean=flat)
            packed = ManoLayer(side=side, use_pca=False, asset=make_synthetic_mano(side), **kw).cuda().packed_model()
            cache[key] = packed, L.model_from_packed(packed)
        return cache[key]
    return get


def _inputs(n, mode, seed):
    g = torch.Generator().manual_seed(seed)
    pose = matrices(n, g) if mode == "rotmat" else edge_poses(n, g)
    return pose, _r32(torch.randn(n, 10, generator=g, dtype=torch.float64)), g


def _groups(fn, n):
    """fn(slice) -> dict of EVs / tensors with the hand axis first (``hand_axis`` 1 for the JVP): concatenated."""
    parts = [fn(slice(i, min(n, i + GROUP))) for i in range(0, n, GROUP)]
    out = {}
    for k, v in parts[0].items():
        ax = 1 if k.startswith("t") else 0
        if isinstance(v, L.EV):
            out[k] = L.ev_cat([p[k] for p in parts], ax)
        else:
            out[k] = torch.cat([p[k] for p in parts], 0)
    return out


def _check(worst, label, got, ev, bounded, hand_axis=0):
    """Every element of the kernel's output within its bound; hands past the projection's cutoff only finite."""
    got = got.detach().double().cpu().reshape(ev.v.shape)
    assert torch.isfinite(got).all(), f"{label}: non-finite output"
    shape = [1] * got.dim()
    shape[hand_axis] = -1
    keep = bounded.view(shape).expand(got.shape)
    err, b = (got - ev.v).abs()[keep], ev.e.expand(ev.v.shape)[keep]
    bad = err > b
    ratio = float(torch.where(b > 0, err / b, torch.where(err > 0, torch.inf, 0.0)).max()) if err.numel() else 0.0
    worst[label] = max(worst.get(label, 0.0), ratio)
    assert not bad.any(), (f"{label}: {int(bad.sum())} of {bad.numel()} elements above the bound, worst err/bound "
                           f"{ratio:.3g}, e.g. err {err[bad][:4].tolist()} bound {b[bad][:4].tolist()}")


def _report(worst):
    for k, v in sorted(worst.items()):
        print(f"  bound {k}: worst err/bound {v:.3e}")


CENTRES = [9, 0, None]


# ------------------------------------------------------------------------------------------------------- forward
@pytest.mark.parametrize("side", ["right", "left"])
@pytest.mark.parametrize("mode", ["aa", "rotmat"])
@pytest.mark.parametrize("palm", [False, True])
@pytest.mark.parametrize("center", CENTRES)
def test_layer_forward(layers, side, mode, palm, center):
    from acr_b200 import lib as Lib, ops
    n = 33
    packed, model = layers(side, mode)
    pose, betas, _ = _inputs(n, mode, 1)
    pm = Lib.POSE_ROTMAT if mode == "rotmat" else Lib.POSE_AXISANG
    if palm and center == 0:
        with pytest.raises(RuntimeError, match="rc=.*centring on the palm"):
            ops.mano_layer_forward(packed, int(side == "right"), pose.float().cuda(), pm, betas.float().cuda(), 0, True)
        return
    v, j, c = ops.mano_layer_forward(packed, int(side == "right"), pose.float().cuda(), pm, betas.float().cuda(), center,
                                     palm)
    exp = L.layer_forward(model, side, pose, betas, mode, center, palm)
    worst = {}
    for k, got in (("verts", v), ("joints", j), ("center", c)):
        _check(worst, f"forward {mode} {k}", got, exp[k], exp["bounded"])
    _report(worst)


@pytest.mark.parametrize("n", [1, 7, 8, 9, 33, 512, 4096])
def test_layer_forward_sizes(layers, n):
    from acr_b200 import lib as Lib, ops
    packed, model = layers("right", "rotmat")
    pose, betas, _ = _inputs(n, "rotmat", n)
    v, j, c = ops.mano_layer_forward(packed, 1, pose.float().cuda(), Lib.POSE_ROTMAT, betas.float().cuda(), 9, True)
    exp = _groups(lambda s: L.layer_forward(model, "right", pose[s], betas[s], "rotmat", 9, True), n)
    worst = {}
    for k, got in (("verts", v), ("joints", j), ("center", c)):
        _check(worst, f"forward rotmat palm {k}", got, exp[k], exp["bounded"])
    _report(worst)


# ------------------------------------------------------------------------------------------------------ backward
def _cotangents(n, g, which):
    r = lambda *s: _r32(torch.randn(*s, generator=g, dtype=torch.float64))
    gv, gj, gc = r(n, 778, 3), r(n, 21, 3), r(n, 3)
    return (gv if "v" in which else None, gj if "j" in which else None, gc if "c" in which else None)


def _backward(layers, side, mode, palm, center, n, which, seed, pipeline=False, flat=True):
    from acr_b200 import lib as Lib, ops
    packed, model = layers(side, mode, flat)
    pose, betas, g = _inputs(n, mode, seed)
    if not flat:
        pose = _r32(torch.randn(n, 48, generator=g, dtype=torch.float64) * 0.5)
    gv, gj, gc = _cotangents(n, g, which)
    cu = lambda t: None if t is None else t.float().cuda()
    sd = int(side == "right")
    if pipeline:
        dp, db = ops.mano_backward(packed, sd, cu(pose), cu(betas), center, cu(gv), cu(gj), cu(gc))
    else:
        pm = Lib.POSE_ROTMAT if mode == "rotmat" else Lib.POSE_AXISANG
        dp, db = ops.mano_layer_backward(packed, sd, cu(pose), pm, cu(betas), center, palm, cu(gv), cu(gj),
                                         None if gc is None else cu(gc).view(n, 1, 3))
    sl = lambda t, s: None if t is None else t[s]
    exp = _groups(lambda s: L.layer_backward(model, side, pose[s], betas[s], mode, center, palm, sl(gv, s), sl(gj, s),
                                             sl(gc, s)), n)
    worst = {}
    tag = "pipeline" if pipeline else f"layer {mode}{' palm' if palm else ''}"
    _check(worst, f"backward {tag} dpose", dp, exp["dpose"], exp["bounded"])
    _check(worst, f"backward {tag} dbetas", db, exp["dbetas"], exp["bounded"])
    _report(worst)


@pytest.mark.parametrize("side", ["right", "left"])
@pytest.mark.parametrize("mode", ["aa", "rotmat"])
@pytest.mark.parametrize("palm", [False, True])
@pytest.mark.parametrize("center", CENTRES)
def test_layer_backward_modes(layers, side, mode, palm, center):
    if palm and center == 0:
        from acr_b200 import lib as Lib, ops
        packed, _ = layers(side, mode)
        pose, betas, g = _inputs(9, mode, 2)
        gv, gj, gc = _cotangents(9, g, "vjc")
        with pytest.raises(RuntimeError, match="rc=.*centring on the palm"):
            ops.mano_layer_backward(packed, int(side == "right"), pose.float().cuda(),
                                    Lib.POSE_ROTMAT if mode == "rotmat" else Lib.POSE_AXISANG, betas.float().cuda(), 0,
                                    True, gv.float().cuda(), gj.float().cuda(), gc.float().cuda().view(9, 1, 3))
        return
    _backward(layers, side, mode, palm, center, 9, "vjc", 2)


@pytest.mark.parametrize("mode,palm", [("aa", False), ("aa", True), ("rotmat", False), ("rotmat", True)])
@pytest.mark.parametrize("which", ["v", "j", "c"])
def test_layer_backward_single_cotangent(layers, mode, palm, which):
    _backward(layers, "right", mode, palm, 9, 9, which, 3)


@pytest.mark.parametrize("n", [1, 7, 8, 9, 33, 512, 4096])
def test_pipeline_backward_sizes(layers, n):
    _backward(layers, "right" if n % 2 else "left", "aa", False, 9, n, "vjc", n, pipeline=True)


@pytest.mark.parametrize("center", CENTRES)
def test_pipeline_backward_mean_pose(layers, center):
    _backward(layers, "right", "aa", False, center, 33, "vjc", 4, pipeline=True, flat=False)


@pytest.mark.parametrize("n", [33, 512])
def test_layer_backward_rotmat_sizes(layers, n):
    _backward(layers, "left", "rotmat", True, 9, n, "vjc", 5 + n)


# ----------------------------------------------------------------------------------------------------------- JVP
def _jvp(layers, side, mode, palm, center, n, T, want_verts, seed):
    from acr_b200 import lib as Lib, ops
    packed, model = layers(side, mode)
    pose, betas, g = _inputs(n, mode, seed)
    tpose = _r32(torch.randn((T,) + tuple(pose.shape), generator=g, dtype=torch.float64))
    tbetas = _r32(torch.randn(T, n, 10, generator=g, dtype=torch.float64))
    pm = Lib.POSE_ROTMAT if mode == "rotmat" else Lib.POSE_AXISANG
    tv, tj, tc = ops.mano_layer_jvp(packed, int(side == "right"), pose.float().cuda(), pm, betas.float().cuda(), center,
                                    palm, tpose.float().cuda(), tbetas.float().cuda(), want_verts=want_verts)
    exp = L.layer_jvp(model, side, pose, betas, mode, center, palm, tpose, tbetas)
    worst = {}
    tag = f"jvp {mode}{' palm' if palm else ''}{'' if want_verts else ' joints-only'}"
    if want_verts:
        _check(worst, f"{tag} tverts", tv, exp["tverts"], exp["bounded"], 1)
    else:
        assert tv is None
    _check(worst, f"{tag} tjoints", tj, exp["tjoints"], exp["bounded"], 1)
    _check(worst, f"{tag} tcenter", tc, exp["tcenter"], exp["bounded"], 1)
    _report(worst)


@pytest.mark.parametrize("side", ["right", "left"])
@pytest.mark.parametrize("mode", ["aa", "rotmat"])
@pytest.mark.parametrize("palm", [False, True])
@pytest.mark.parametrize("center", CENTRES)
@pytest.mark.parametrize("want_verts", [True, False])
def test_layer_jvp_modes(layers, side, mode, palm, center, want_verts):
    if palm and center == 0:
        from acr_b200 import lib as Lib, ops
        packed, _ = layers(side, mode)
        pose, betas, _ = _inputs(9, mode, 6)
        with pytest.raises(RuntimeError, match="rc=.*centring on the palm"):
            ops.mano_layer_jvp(packed, int(side == "right"), pose.float().cuda(),
                               Lib.POSE_ROTMAT if mode == "rotmat" else Lib.POSE_AXISANG, betas.float().cuda(), 0, True,
                               pose[None].float().cuda(), betas[None].float().cuda(), want_verts=want_verts)
        return
    _jvp(layers, side, mode, palm, center, 9, 3, want_verts, 6)


@pytest.mark.parametrize("T", [1, 3, 4, 5, 58])
@pytest.mark.parametrize("want_verts", [True, False])
def test_layer_jvp_tangent_counts(layers, T, want_verts):
    _jvp(layers, "right", "rotmat" if T % 2 else "aa", True, 9, 9, T, want_verts, 7 + T)


@pytest.mark.parametrize("n", [1, 8, 33])
def test_layer_jvp_sizes(layers, n):
    _jvp(layers, "left", "aa", False, 9, n, 5, True, 8 + n)
