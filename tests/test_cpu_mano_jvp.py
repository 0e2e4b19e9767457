"""CPU: ManoLayer's forward-mode derivatives.  The float64 rotation-matrix restatement's JVP against central
differences and its VJP, the built library's JVP entry point (export, argument checks, no local memory in its
kernels), and the torch.func wiring of the layer's Functions, run with float64 torch stand-ins for the kernels."""
import os
import sys

import numpy as np
import pytest
import torch
from torch.func import grad, hessian, jacfwd, jacrev, jvp, vjp, vmap

from tests.mano_jvp_ref import SO3ProjectFn, TorchManoFunc
from tests.mano_rotmat_ref import SO3Project
from tests.mano_torch_ref import rodrigues

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
LIB = os.path.join(ROOT, "arbitrary-hands-3d-reconstruction_b200", "lib", "libacr_b200.so")


@pytest.fixture(scope="module")
def asset():
    from acr_b200.synth import make_synthetic_mano
    return make_synthetic_mano("right")


def _matrices(n, seed):
    g = torch.Generator().manual_seed(seed)
    R = rodrigues(torch.randn(n, 3, generator=g, dtype=torch.float64)).view(n, 3, 3)
    noise = torch.randn(n, 3, 3, generator=g, dtype=torch.float64)
    cls = torch.arange(n) % 4
    out = torch.where((cls == 1)[:, None, None], R + 0.1 * noise, R)            # 0: exact rotations
    out = torch.where((cls == 2)[:, None, None], -(R + 0.05 * noise), out)      # det < 0
    return torch.where((cls == 3)[:, None, None], 2 * R, out)


# ------------------------------------------------------------------------------------ the float64 restatement
def test_projection_jvp_matches_central_differences():
    M = _matrices(16, 1)
    dM = torch.randn(M.shape, generator=torch.Generator().manual_seed(2), dtype=torch.float64)
    _, t = jvp(lambda m: SO3ProjectFn.apply(m)[0], (M,), (dM,))
    eps = 1e-6
    fd = (SO3ProjectFn.apply(M + eps * dM)[0] - SO3ProjectFn.apply(M - eps * dM)[0]) / (2 * eps)
    assert torch.isfinite(t).all()
    assert float((t - fd).abs().max()) < 1e-7


def test_projection_vjp_is_so3project_and_adjoint_to_jvp():
    M = _matrices(16, 3)
    g = torch.Generator().manual_seed(4)
    G, dM = (torch.randn(M.shape, generator=g, dtype=torch.float64) for _ in range(2))
    a = M.clone().requires_grad_()
    (SO3Project.apply(a) * G).sum().backward()
    _, f = vjp(lambda m: SO3ProjectFn.apply(m)[0], M)
    assert torch.allclose(f(G)[0], a.grad, rtol=0, atol=1e-12)
    _, t = jvp(lambda m: SO3ProjectFn.apply(m)[0], (M,), (dM,))
    assert abs(float((G * t).sum() - (a.grad * dM).sum())) < 1e-10


@pytest.mark.parametrize("palm", [False, True])
def test_restatement_jacfwd_matches_jacrev(asset, palm):
    ref = TorchManoFunc(asset, "right", use_pca=False, center_idx=9)
    M = _matrices(32, 5).view(2, 16, 3, 3)
    b = torch.randn(2, 10, generator=torch.Generator().manual_seed(6), dtype=torch.float64)
    f = lambda m, bb: ref.from_rotmats(m, bb, root_palm=palm)[1]
    for a, r in zip(jacfwd(f, argnums=(0, 1))(M, b), jacrev(f, argnums=(0, 1))(M, b)):
        assert torch.isfinite(a).all()
        assert torch.allclose(a, r, rtol=0, atol=1e-10)


# ------------------------------------------------------------------------------------------- the built library
def _lib():
    if not os.path.exists(LIB):
        pytest.skip("library not built")
    from acr_b200 import lib as L
    return L.load()


def test_jvp_symbol_and_argument_checks():
    lib = _lib()
    from acr_b200 import lib as L
    assert "acr_b200_mano_layer_jvp" in L.EXPORTS and hasattr(lib, "acr_b200_mano_layer_jvp")
    f = lib.acr_b200_mano_layer_jvp
    # the checks run before anything touches a device, so host buffers stand in for device ones here
    buf = np.zeros(64, np.float32)
    p = buf.ctypes.data
    J = lambda model=p, pose=p, mode=0, n=2, n_tan=3, center=9, palm=0, side=1: f(
        model, side, pose, mode, p, n, center, palm, n_tan, p, p, None, None, None, None, p, None, None)
    assert J(n=0) == 0 and J(n=0, model=None) == 0
    assert J(model=None) == -1 and b"null" in lib.acr_b200_last_error()
    assert J(pose=None) == -1
    assert J(n_tan=-1) == -1 and b"n_tan" in lib.acr_b200_last_error()
    assert J(n=-1) == -1
    for mode in (2, -1):
        assert J(mode=mode) == -1 and b"pose_mode" in lib.acr_b200_last_error()
    assert J(side=2) == -1
    assert J(center=21) == -1
    assert J(center=4) == -3 and b"fingertip" in lib.acr_b200_last_error()    # as the forward
    assert J(mode=1, center=8) == -3
    assert J(center=0, palm=1) == -3 and b"palm" in lib.acr_b200_last_error()


def test_jvp_kernels_do_not_touch_local_memory():
    if not (os.path.exists(LIB) and os.path.exists("/usr/local/cuda/bin/cuobjdump")):
        pytest.skip("library not built or no cuobjdump")
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    try:
        import sass_audit
        rows = sass_audit.audit(LIB)
    finally:
        sys.path.pop(0)
    names = [f"mano_layer_jvp{s}_kernel<{m}, {p}>" for s in ("", "_joints") for m in (0, 1) for p in ("false", "true")]
    for k in names:
        assert k in rows, sorted(rows)
        assert rows[k]["LDL"] == 0 and rows[k]["STL"] == 0, (k, rows[k]["LDL"], rows[k]["STL"])


# ------------------------------------------------------------------------------ torch.func wiring of the layer
class _StandIn:
    """Float64 torch restatements of the four MANO ops the layer's Functions call, counting the calls."""

    def __init__(self, asset, rotmat):
        self.ref = TorchManoFunc(asset, "right", use_pca=False, flat_hand_mean=rotmat)
        self.calls = []

    def outputs(self, pose, mode, betas, center_idx, palm):
        from acr_b200 import lib as L
        self.ref.center_idx = center_idx
        if mode == L.POSE_ROTMAT:
            v, j, c = self.ref.from_rotmats(pose, betas, root_palm=palm)
        else:
            hm = torch.cat([torch.zeros(3, dtype=pose.dtype), self.ref.hands_mean])
            R = rodrigues((pose + hm).reshape(-1, 3)).view(pose.shape[0], 16, 3, 3)
            v, j, c = self.ref.from_rotations(R, betas, root_palm=palm)
        c = torch.zeros(pose.shape[0], 1, 3, dtype=pose.dtype) if c is None else c
        return v.clone(), j.clone(), c.clone()

    def mano_forward(self, model_l, model_r, pose, betas, hand_type, side, center_idx):
        self.calls.append(("forward", pose.shape[0]))
        return dict(zip(("verts", "joints", "center"), self.outputs(pose, 0, betas, center_idx, False)))

    def mano_layer_forward(self, model, side, pose, mode, betas, center_idx, palm):
        self.calls.append(("forward", pose.shape[0]))
        return self.outputs(pose, mode, betas, center_idx, palm)

    def mano_layer_backward(self, model, side, pose, mode, betas, center_idx, palm, dv, dj, dc):
        self.calls.append(("backward", pose.shape[0]))
        _, f = vjp(lambda p, b: self.outputs(p, mode, b, center_idx, palm), pose, betas)
        n, z = pose.shape[0], lambda t, *s: torch.zeros(s, dtype=pose.dtype) if t is None else t
        return f((z(dv, n, 778, 3), z(dj, n, 21, 3), z(dc, n, 1, 3)))

    def mano_layer_jvp(self, model, side, pose, mode, betas, center_idx, palm, tp, tb):
        T = (tp if tp is not None else tb).shape[0]
        self.calls.append(("jvp", pose.shape[0], T))
        outs = []
        for t in range(T):
            with torch.enable_grad():     # a reverse-mode JVP: forward AD does not nest
                outs.append(torch.autograd.functional.jvp(
                    lambda p, b: self.outputs(p, mode, b, center_idx, palm), (pose, betas),
                    (torch.zeros_like(pose) if tp is None else tp[t], torch.zeros_like(betas) if tb is None else tb[t]))[1])
        return tuple(torch.stack([o[k] for o in outs]) for k in range(3))


@pytest.mark.parametrize("rotmat,palm", [(False, False), (False, True), (True, False), (True, True)])
def test_layer_transforms_with_stand_in_ops(asset, monkeypatch, rotmat, palm):
    _lib()
    import mano.manolayer as ML
    stand = _StandIn(asset, rotmat)
    for name in ("mano_forward", "mano_layer_forward", "mano_layer_backward", "mano_layer_jvp"):
        monkeypatch.setattr(ML._ops, name, getattr(stand, name))
    layer = ML.ManoLayer(center_idx=9, use_pca=not rotmat, ncomps=6, flat_hand_mean=False,
                         joint_rot_mode="rotmat" if rotmat else "axisang", asset=asset).double()
    ref = TorchManoFunc(asset, "right", use_pca=not rotmat, ncomps=6, flat_hand_mean=rotmat, center_idx=9)
    g = torch.Generator().manual_seed(7)
    n = 3
    pose = (_matrices(n * 16, 8).view(n, 16, 3, 3) if rotmat else torch.randn(n, 9, generator=g, dtype=torch.float64))
    betas = torch.randn(n, 10, generator=g, dtype=torch.float64)
    pm = torch.Tensor([int(palm)])
    f = lambda p, b: layer(p, th_betas=b, root_palm=pm)[1]
    fr = lambda p, b: (ref.from_rotmats if rotmat else ref)(p, b, root_palm=palm)[1]
    close = lambda a, b: torch.allclose(a, b, rtol=0, atol=1e-9 * max(1.0, float(b.abs().max())))

    stand.calls.clear()
    Jh = vmap(jacfwd(lambda p, b: f(p[None], b[None])[0], argnums=(0, 1)))(pose, betas)
    assert stand.calls == [("forward", n), ("jvp", n, pose[0].numel() + 10)]      # one launch for all hands
    Jr = vmap(jacfwd(lambda p, b: fr(p[None], b[None])[0], argnums=(0, 1)))(pose, betas)
    assert all(close(a, e) for a, e in zip(Jh, Jr))
    stand.calls.clear()
    Jb = vmap(jacrev(lambda p, b: f(p[None], b[None])[0], argnums=(0, 1)))(pose, betas)
    assert stand.calls == [("forward", n), ("backward", n * 63)]                   # cotangents become rows
    assert all(close(a, e) for a, e in zip(Jb, Jr))
    V = vmap(f, in_dims=(0, None))(torch.stack([pose, pose * 0.9]), betas)
    assert close(V, torch.stack([f(pose, betas), f(pose * 0.9, betas)]))    # bits: tests/test_gpu_mano_jvp.py
    assert close(vmap(grad(lambda p, b: f(p[None], b[None]).square().sum()))(pose, betas),
                 vmap(grad(lambda p, b: fr(p[None], b[None]).square().sum()))(pose, betas))
    for second_order in (lambda: hessian(lambda p: f(p, betas).square().sum())(pose),
                         lambda: jvp(grad(lambda p: f(p, betas).square().sum()), (pose,), (pose,))):
        with pytest.raises(RuntimeError, match="first-order"):
            second_order()
    stand.calls.clear()
    with torch.no_grad():
        f(pose, betas)
    assert stand.calls == [("forward", n)]
