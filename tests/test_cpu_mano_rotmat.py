"""CPU: ManoLayer's rotation-matrix mode and root_palm.  The float64 restatement (tests/mano_rotmat_ref.py) against
the reference's own outputs (tests/golden/mano_rotmat_golden.npz, oracle/make_mano_rotmat_golden.py), its gradients
against central differences, the layer's constructor / forward argument handling, and the built library's new
entry points (exports, argument checks, no local memory in the new kernels)."""
import os
import sys

import numpy as np
import pytest
import torch

from tests.helpers import GOLDEN, rel_err
from tests.mano_rotmat_ref import SO3Project, TorchManoRot
from tests.mano_torch_ref import TorchMano, rodrigues

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
LIB = os.path.join(ROOT, "arbitrary-hands-3d-reconstruction_b200", "lib", "libacr_b200.so")


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(GOLDEN, "mano_rotmat_golden.npz"))


@pytest.fixture(scope="module")
def assets():
    from acr_b200.synth import make_synthetic_mano
    return {"left": make_synthetic_mano("left"), "right": make_synthetic_mano("right")}


CASES = ["rotmat_c9", "rotmat_c9_palm", "rotmat_none", "rotmat_none_palm", "rotmat_trans", "rotmat_trans_palm",
         "axisang_c9_palm", "axisang_none_palm", "axisang_trans_palm"]


def golden_case(g, side, name):
    """-> (pose mode, center_idx, root_palm, use_trans) of a golden case, parsed from its name."""
    mode = name.split("_")[0]
    center = None if "_none" in name else 9
    return mode, center, name.endswith("_palm"), "_trans" in name


def restatement(assets, g, side, name):
    mode, center, palm, use_trans = golden_case(g, side, name)
    d = lambda k: torch.from_numpy(g[f"{side}__{k}"].astype(np.float64))
    trans = d("trans") if use_trans else None
    ref = TorchManoRot(assets[side], side, use_pca=False, flat_hand_mean=mode == "rotmat", center_idx=center)
    if mode == "rotmat":
        return ref.from_rotmats(d("mats"), d("betas"), trans, root_palm=palm)
    return ref(d("aa"), d("betas"), trans, root_palm=palm)


def test_golden_covers_the_cases(golden):
    assert list(golden["case_names"]) == CASES
    for side in ("left", "right"):
        cls = golden[f"{side}__classes"]
        assert set(np.unique(cls)) == set(range(5)) and (cls[0] == 0).all()
        m = golden[f"{side}__mats"].astype(np.float64)
        assert (np.linalg.det(m[cls == 2]) < 0).all()


@pytest.mark.parametrize("side", ["right", "left"])
@pytest.mark.parametrize("name", CASES)
def test_restatement_matches_reference_golden(assets, golden, side, name):
    v, j, c = restatement(assets, golden, side, name)
    vi = golden["vert_idx"]
    assert rel_err(v.numpy()[:, vi], golden[f"{side}__{name}__verts"]) < 1e-6
    assert rel_err(j.numpy(), golden[f"{side}__{name}__joints"]) < 1e-6
    key = f"{side}__{name}__center"
    if key in golden.files:
        assert rel_err(c.numpy(), golden[key]) < 1e-6
    else:
        assert c is None


@pytest.mark.parametrize("center_idx,trans", [(9, False), (None, False), (9, True)])
def test_from_rotations_is_torch_mano(assets, center_idx, trans):
    """Without the palm, rodrigues + from_rotations is TorchMano.__call__ (the restatement the axis-angle gradients
    are pinned to), bit for bit; with it, only output joint 0 changes."""
    g = torch.Generator().manual_seed(1)
    pose, betas = torch.randn(5, 48, generator=g, dtype=torch.float64) * 0.5, torch.randn(5, 10, generator=g, dtype=torch.float64)
    tr = torch.randn(5, 3, generator=g, dtype=torch.float64) * 0.1 if trans else None
    kw = dict(use_pca=False, flat_hand_mean=False, center_idx=center_idx)
    base = TorchMano(assets["right"], "right", **kw)
    ref = TorchManoRot(assets["right"], "right", **kw)
    R = rodrigues(ref.full_pose(pose).reshape(-1, 3)).view(5, 16, 3, 3)
    exp = base(pose, betas, tr)
    for a, b, e in zip(ref(pose, betas, tr), ref.from_rotations(R, betas, tr), exp):
        assert (a is None and b is None and e is None) or (torch.equal(a, e) and torch.equal(b, e))
    v, j, _ = ref(pose, betas, tr, root_palm=True)
    assert torch.equal(v, exp[0]) and torch.equal(j[:, 1:], exp[1][:, 1:])
    assert torch.allclose(j[:, 0], (v[:, 95] + v[:, 22]) / 2, rtol=0, atol=1e-12)


def _matrices(n, seed):
    """(n,16,3,3) float64: exact rotations, noisy, det < 0, 2 R and Gaussian, mixed per joint."""
    g = torch.Generator().manual_seed(seed)
    R = rodrigues(torch.randn(n * 16, 3, generator=g, dtype=torch.float64)).view(n, 16, 3, 3)
    noise = torch.randn(n, 16, 3, 3, generator=g, dtype=torch.float64)
    cls = (torch.arange(n)[:, None] + torch.arange(16)[None, :]) % 5
    out = torch.where((cls == 0)[..., None, None], R, R + 0.1 * noise)
    out = torch.where((cls == 2)[..., None, None], -(R + 0.05 * noise), out)
    out = torch.where((cls == 3)[..., None, None], 2 * R, out)
    return torch.where((cls == 4)[..., None, None], noise, out), cls


def test_projection_vjp_matches_svd_autograd_off_the_degenerate_set():
    M, cls = _matrices(4, 2)
    M = M.reshape(-1, 3, 3)[(cls.reshape(-1) != 0) & (cls.reshape(-1) != 3)]   # distinct singular values
    G = torch.randn(M.shape, generator=torch.Generator().manual_seed(3), dtype=torch.float64)
    a = M.clone().requires_grad_()
    (SO3Project.apply(a) * G).sum().backward()

    def svd_proj(x):
        U, _, Vh = torch.linalg.svd(x)
        Q = U @ Vh
        d = torch.where(torch.linalg.det(Q) < 0, -1.0, 1.0).to(x.dtype)
        return torch.cat([Q[:, :, :2], Q[:, :, 2:] * d[:, None, None]], 2)
    b = M.clone().requires_grad_()
    (svd_proj(b) * G).sum().backward()
    assert rel_err(a.grad.numpy(), b.grad.numpy()) < 1e-9


@pytest.mark.parametrize("side,center,palm,trans", [("right", 9, False, False), ("left", 9, True, False),
                                                     ("right", None, True, False), ("left", 9, True, True)])
def test_restatement_grad_matches_central_differences(assets, side, center, palm, trans):
    n = 5
    M, _ = _matrices(n, 4)                          # hand 0 / every 5th joint: exact rotations; class 2: det < 0
    g = torch.Generator().manual_seed(5)
    betas = torch.randn(n, 10, generator=g, dtype=torch.float64)
    tr = torch.randn(n, 3, generator=g, dtype=torch.float64) * 0.1 if trans else None
    gv, gj = torch.randn(n, 778, 3, generator=g, dtype=torch.float64), torch.randn(n, 21, 3, generator=g, dtype=torch.float64)
    gc = torch.randn(n, 1, 3, generator=g, dtype=torch.float64)
    ref = TorchManoRot(assets[side], side, use_pca=False, center_idx=center)

    def loss(m, b, t):
        v, j, c = ref.from_rotmats(m, b, t, root_palm=palm)
        out = (gv * v).sum() + (gj * j).sum()
        return out + ((gc * c).sum() if c is not None else 0.0)

    m, b = M.clone().requires_grad_(), betas.clone().requires_grad_()
    t = tr.clone().requires_grad_() if trans else None
    grads = torch.autograd.grad(loss(m, b, t), [x for x in (m, b, t) if x is not None])
    assert all(torch.isfinite(x).all() for x in grads)
    eps = 1e-6
    for _ in range(4):
        dirs = [torch.randn(x.shape, generator=g, dtype=torch.float64) for x in (M, betas)]
        dirs.append(torch.randn(3, generator=g, dtype=torch.float64).expand(n, 3) if trans else None)
        shift = lambda s: [None if x is None else x + s * eps * d for x, d in zip((M, betas, tr), dirs)]
        with torch.no_grad():
            fd = float(loss(*shift(1)) - loss(*shift(-1))) / (2 * eps)
        an = float(sum((x * d).sum() for x, d in zip(grads, [d for d in dirs if d is not None])))
        assert abs(fd - an) <= 1e-6 * max(abs(an), 1.0), (fd, an)


def test_projection_grad_finite_at_exact_rotations():
    R = rodrigues(torch.randn(32, 3, generator=torch.Generator().manual_seed(6), dtype=torch.float64))
    R = torch.cat([R, torch.eye(3, dtype=torch.float64)[None], -R[:4]])   # identity and exact det = -1 matrices
    a = R.clone().requires_grad_()
    (SO3Project.apply(a) * torch.randn(R.shape, generator=torch.Generator().manual_seed(7), dtype=torch.float64)).sum().backward()
    assert torch.isfinite(a.grad).all()


# ------------------------------------------------------------------------------------------------ the layer
def test_buffer_names_match_reference(golden, assets):
    from mano.manolayer import ManoLayer
    layer = ManoLayer(use_pca=False, joint_rot_mode="rotmat", asset=assets["right"])
    assert sorted(n for n, _ in layer.named_buffers()) == list(golden["buffer_names"])
    assert tuple(layer.th_hands_mean_rotmat.shape) == (15, 3, 3)
    flat = ManoLayer(use_pca=False, joint_rot_mode="rotmat", flat_hand_mean=True, asset=assets["right"])
    assert torch.equal(flat.th_hands_mean_rotmat, torch.eye(3).expand(15, 3, 3))


def test_constructor_modes(assets):
    from mano.manolayer import ManoLayer
    a = assets["left"]
    for root in ("axisang", "rot6d"):          # the rotation-matrix branch ignores root_rot_mode
        layer = ManoLayer(use_pca=False, joint_rot_mode="rotmat", root_rot_mode=root, side="left", asset=a)
        assert layer.rotmat and not hasattr(layer, "th_hands_mean")
    pca = ManoLayer(use_pca=True, joint_rot_mode="rotmat", asset=a)      # PCA takes the axis-angle path
    assert not pca.rotmat and tuple(pca.th_hands_mean.shape) == (1, 45)
    with pytest.raises(NotImplementedError):
        ManoLayer(use_pca=False, joint_rot_mode="axisang", root_rot_mode="rot6d", asset=a)
    with pytest.raises(NotImplementedError):
        ManoLayer(use_pca=True, joint_rot_mode="rotmat", root_rot_mode="rot6d", asset=a)


def test_forward_rejects_bad_input(assets):
    """All of these fail before any device work."""
    from mano.manolayer import ManoLayer
    rot = ManoLayer(use_pca=False, joint_rot_mode="rotmat", center_idx=9, asset=assets["right"])
    with pytest.raises(AssertionError):
        rot(torch.zeros(2, 48))
    with pytest.raises(AssertionError):
        rot(torch.zeros(2, 16, 3, 4))
    with pytest.raises(ValueError):
        rot(torch.zeros(2, 15, 3, 3))
    for layer, pose in ((ManoLayer(use_pca=False, joint_rot_mode="rotmat", center_idx=0, asset=assets["right"]),
                         torch.zeros(2, 16, 3, 3)),
                        (ManoLayer(use_pca=False, center_idx=0, asset=assets["right"]), torch.zeros(2, 48))):
        with pytest.raises(NotImplementedError):
            layer(pose, root_palm=torch.Tensor([1]))


# ------------------------------------------------------------------------------------------- the built library
def _lib():
    if not os.path.exists(LIB):
        pytest.skip("library not built")
    from acr_b200 import lib as L
    return L.load()


def test_packed_model_without_hands_mean(assets):
    _lib()
    from mano.manolayer import ManoLayer
    rot = ManoLayer(use_pca=False, joint_rot_mode="rotmat", flat_hand_mean=False, asset=assets["right"])
    aa = ManoLayer(use_pca=False, flat_hand_mean=True, asset=assets["right"])
    assert torch.equal(rot.packed_model(), aa.packed_model())     # zero mean pose, the rest identical


def test_layer_symbols_and_argument_checks():
    lib = _lib()
    from acr_b200 import lib as L
    for name in ("acr_b200_mano_layer_forward", "acr_b200_mano_layer_backward"):
        assert name in L.EXPORTS and hasattr(lib, name)
    assert (L.POSE_AXISANG, L.POSE_ROTMAT) == (0, 1)
    fwd, bwd = lib.acr_b200_mano_layer_forward, lib.acr_b200_mano_layer_backward
    assert fwd(None, 1, None, 1, None, 0, 9, 0, None, None, None, None) == 0
    assert bwd(None, 1, None, 1, None, 0, 9, 0, None, None, None, None, None, None, None) == 0
    # the checks run before anything touches a device, so host buffers stand in for device ones here
    buf = np.zeros(64, np.float32)
    p = (buf.ctypes.data + 15) // 16 * 16
    F = lambda side=1, mode=1, center=9, palm=0, model=p: fwd(model, side, p, mode, p, 2, center, palm, p, p, p, None)
    B = lambda side=1, mode=1, center=9, palm=0, ws=p: bwd(p, side, p, mode, p, 2, center, palm, p, None, None, ws, p, p, None)
    assert F(model=None) == -1
    for call in (F, B):
        assert call(side=2) == -1
        assert call(mode=2) == -1 and b"pose_mode" in lib.acr_b200_last_error()
        assert call(mode=-1) == -1
        assert call(center=21) == -1
        assert call(center=4) == -3                               # fingertip centre
        assert call(center=0, palm=1) == -3 and b"palm" in lib.acr_b200_last_error()
        assert call(mode=0, center=4, palm=1) == -3
    assert B(ws=None) == -1 and b"workspace" in lib.acr_b200_last_error()
    assert fwd(p, 1, p, 1, p, 2, 9, 0, p + 4, p, p, None) == -1     # verts not 16-byte aligned
    assert fwd(p, 1, p, 1, p, -1, 9, 0, p, p, p, None) == -1


def test_new_kernels_do_not_touch_local_memory():
    if not (os.path.exists(LIB) and os.path.exists("/usr/local/cuda/bin/cuobjdump")):
        pytest.skip("library not built or no cuobjdump")
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    try:
        import sass_audit
        rows = sass_audit.audit(LIB)
    finally:
        sys.path.pop(0)
    for k in ("mano_forward_kernel", "mano_backward_vertex_kernel", "mano_backward_chain_kernel"):
        assert k in rows, sorted(rows)                  # the axis-angle, no-palm kernels keep their names
    no_local = [f"mano_layer_backward_{s}_kernel<{m}, {p}>" for s in ("vertex", "chain") for m, p in
                (("0", "true"), ("1", "false"), ("1", "true"))]
    no_local += ["mano_layer_forward_kernel<1, false>", "mano_layer_forward_kernel<1, true>"]
    assert "mano_layer_forward_kernel<0, true>" in rows
    for k in no_local:
        assert k in rows, sorted(rows)
        assert rows[k]["LDL"] == 0 and rows[k]["STL"] == 0, (k, rows[k]["LDL"], rows[k]["STL"])
