"""CPU: the gradient reference of the MANO backward (tests/mano_torch_ref.py) against the numpy oracle and the
reference goldens, its autograd against finite differences of the oracle in float64, and the built library's
backward entry points (exports, argument checks, no local memory in the backward kernels)."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

from oracle import mano_ref, rotation_ref
from tests.helpers import GOLDEN, rel_err
from tests.mano_torch_ref import TorchMano

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
LIB = os.path.join(ROOT, "arbitrary-hands-3d-reconstruction_b200", "lib", "libacr_b200.so")


@pytest.fixture(scope="module")
def assets():
    from acr_b200.synth import make_synthetic_mano
    return {"left": make_synthetic_mano("left"), "right": make_synthetic_mano("right")}


@pytest.fixture
def oracle64(monkeypatch):
    """oracle.mano_ref evaluated in float64 (its arithmetic type is a module constant)."""
    monkeypatch.setattr(mano_ref, "F", np.float64)
    monkeypatch.setattr(rotation_ref, "F", np.float64)
    return mano_ref


def _inputs(n, seed, edges=True):
    g = np.random.default_rng(seed)
    pose = g.normal(size=(n, 48)) * 0.5
    betas = g.normal(size=(n, 10))
    if edges and n >= 3:
        pose[0] = 0.0
        pose[1] = 1e-6
        pose[2, :3] = [3.14159, 0.0, 0.0]
    return pose, betas


@pytest.mark.parametrize("side", ["right", "left"])
@pytest.mark.parametrize("center_idx", [9, 0, None])
def test_restatement_forward_matches_oracle(assets, oracle64, side, center_idx):
    pose, betas = _inputs(6, 1)
    ref = TorchMano(assets[side], side, use_pca=False, flat_hand_mean=False, center_idx=center_idx)
    v, j, c = ref(torch.from_numpy(pose), torch.from_numpy(betas))
    ov, oj, oc = oracle64.mano_forward(assets[side], pose, betas, side, center_idx, flip_shapedirs_x=False)
    assert rel_err(v.numpy(), ov) < 1e-10 and rel_err(j.numpy(), oj) < 1e-10
    if center_idx is None:
        assert c is None and oc is None
    else:
        assert rel_err(c.numpy(), oc) < 1e-10


def test_restatement_forward_matches_reference_golden(assets):
    """The goldens are the reference's own float32 outputs (MANOWrapper: left layer with x-flipped shapedirs)."""
    g = np.load(os.path.join(GOLDEN, "mano_golden.npz"))
    L = int(g["L"])
    for side, rows in (("left", slice(0, L)), ("right", slice(L, None))):
        a = dict(assets[side])
        if side == "left":
            a["shapedirs"] = np.asarray(a["shapedirs"]).copy()
            a["shapedirs"][:, 0, :] *= -1
        ref = TorchMano(a, side, use_pca=False, flat_hand_mean=False, center_idx=9)
        v, j, _ = ref(torch.from_numpy(g["poses"][rows].astype(np.float64)), torch.from_numpy(g["betas"][rows].astype(np.float64)))
        assert rel_err(v.numpy(), g["verts"][rows]) < 1e-5   # float32 goldens: their own rounding
        assert rel_err(j.numpy(), g["j3d"][rows]) < 1e-5


def _oracle_loss(oracle, asset, side, center_idx, pose, betas, gv, gj, gc):
    v, j, c = oracle.mano_forward(asset, pose, betas, side, center_idx, flip_shapedirs_x=False)
    out = float((gv * v).sum() + (gj * j).sum())
    return out + (float((gc * c).sum()) if c is not None else 0.0)


@pytest.mark.parametrize("side", ["right", "left"])
@pytest.mark.parametrize("center_idx", [9, None])
def test_restatement_grad_matches_oracle_finite_differences(assets, oracle64, side, center_idx):
    n = 4
    pose, betas = _inputs(n, 2)
    g = np.random.default_rng(3)
    gv, gj, gc = g.normal(size=(n, 778, 3)), g.normal(size=(n, 21, 3)), g.normal(size=(n, 1, 3))
    ref = TorchMano(assets[side], side, use_pca=False, flat_hand_mean=False, center_idx=center_idx)
    tp, tb = torch.from_numpy(pose).requires_grad_(), torch.from_numpy(betas).requires_grad_()
    v, j, c = ref(tp, tb)
    loss = (torch.from_numpy(gv) * v).sum() + (torch.from_numpy(gj) * j).sum()
    if c is not None:
        loss = loss + (torch.from_numpy(gc) * c).sum()
    dp, db = torch.autograd.grad(loss, (tp, tb))
    eps = 1e-6
    f = lambda p, b: _oracle_loss(oracle64, assets[side], side, center_idx, p, b, gv, gj, gc)
    # random directions, and each hand's own pose direction (hands 0-2 are the edge poses: 0, 1e-6, root ~ pi)
    dirs = [(g.normal(size=pose.shape), g.normal(size=betas.shape)) for _ in range(3)]
    for h in range(3):
        e = np.zeros_like(pose)
        e[h] = g.normal(size=48)
        dirs.append((e, np.zeros_like(betas)))
    for dpose, dbeta in dirs:
        fd = (f(pose + eps * dpose, betas + eps * dbeta) - f(pose - eps * dpose, betas - eps * dbeta)) / (2 * eps)
        an = float((dp.numpy() * dpose).sum() + (db.numpy() * dbeta).sum())
        assert abs(fd - an) <= 1e-6 * max(abs(an), 1.0), (fd, an)


def test_restatement_grad_pca_trans_share_betas():
    """The torch-op glue around the layer (PCA mm, share_betas, th_trans) through gradcheck on a small asset."""
    from acr_b200.synth import make_synthetic_mano
    a = make_synthetic_mano("right")
    ref = TorchMano(a, "right", use_pca=True, ncomps=6, flat_hand_mean=False, center_idx=9)
    g = torch.Generator().manual_seed(4)
    coeffs = (torch.randn(2, 9, generator=g, dtype=torch.float64) * 0.5).requires_grad_()
    betas = torch.randn(2, 10, generator=g, dtype=torch.float64).requires_grad_()
    trans = torch.randn(2, 3, generator=g, dtype=torch.float64).requires_grad_()
    fn = lambda c, b, t: tuple(o[:, :40:7] for o in ref(c, b, t, share_betas=True)[:2])
    assert torch.autograd.gradcheck(fn, (coeffs, betas, trans), eps=1e-6, atol=1e-6, rtol=1e-5)


# ------------------------------------------------------------------------------------------- the built library
def _lib():
    if not os.path.exists(LIB):
        pytest.skip("library not built")
    from acr_b200 import lib as L
    return L.load()


def test_backward_symbols_and_argument_checks():
    lib = _lib()
    from acr_b200 import lib as L
    for name in ("acr_b200_mano_backward_workspace_floats", "acr_b200_mano_backward"):
        assert name in L.EXPORTS and hasattr(lib, name)
    assert lib.acr_b200_mano_backward_workspace_floats(0) == 0
    assert lib.acr_b200_mano_backward_workspace_floats(3) == 3 * 7 * 340
    assert lib.acr_b200_mano_backward(None, 1, None, None, 0, 9, None, None, None, None, None, None, None) == 0
    # the checks run before anything touches a device, so host buffers stand in for device ones here
    buf = np.zeros(64, np.float32)
    p = buf.ctypes.data
    assert lib.acr_b200_mano_backward(None, 1, p, p, 2, 9, p, None, None, p, p, p, None) == -1
    assert lib.acr_b200_mano_backward(p, 2, p, p, 2, 9, p, None, None, p, p, p, None) == -1
    assert lib.acr_b200_mano_backward(p, 1, p, p, 2, 9, p, None, None, None, p, p, None) == -1   # no workspace
    assert b"workspace" in lib.acr_b200_last_error()
    assert lib.acr_b200_mano_backward(p, 1, p, p, 2, 4, p, None, None, p, p, p, None) == -3      # fingertip centre
    assert lib.acr_b200_mano_backward(p, 1, p, p, 2, 21, p, None, None, p, p, p, None) == -1


def test_backward_kernels_do_not_touch_local_memory():
    if not (os.path.exists(LIB) and os.path.exists("/usr/local/cuda/bin/cuobjdump")):
        pytest.skip("library not built or no cuobjdump")
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    try:
        import sass_audit
        rows = sass_audit.audit(LIB)
    finally:
        sys.path.pop(0)
    for k in ("mano_backward_vertex_kernel", "mano_backward_chain_kernel"):
        assert k in rows, sorted(rows)
        assert rows[k]["LDL"] == 0 and rows[k]["STL"] == 0, (k, rows[k]["LDL"], rows[k]["STL"])
