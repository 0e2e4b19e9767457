"""GPU parity: fused MANO / rotation kernels (through the C ABI) vs the oracle and the reference goldens."""
import os

import numpy as np
import pytest
import torch

from tests.helpers import GOLDEN, rel_err

pytestmark = pytest.mark.gpu
TOL = 1e-4   # BASELINE.json: 1e-4 relative fp32 tolerance


@pytest.fixture(scope="module")
def assets():
    from acr_b200.synth import make_synthetic_mano
    return {"left": make_synthetic_mano("left"), "right": make_synthetic_mano("right")}


@pytest.fixture(scope="module")
def wrapper(assets):
    from acr.mano_wrapper import MANOWrapper
    return MANOWrapper(assets).cuda()


def test_rot6d_and_rodrigues_golden():
    from acr_b200 import ops
    g = np.load(os.path.join(GOLDEN, "rot_golden.npz"))
    aa = ops.rot6d_to_aa(torch.from_numpy(g["rot6d"]).cuda()).cpu().numpy()
    assert not np.isnan(aa).any()
    d = np.abs(aa - g["aa"]).reshape(-1, 3).max(1)           # per rotation (64 of them)
    print("rot6d worst rows:", np.argsort(d)[-4:], np.sort(d)[-4:])
    # rows 4,5 are deliberately degenerate 6D inputs (zero-length / parallel columns): their second
    # basis vector is normalised rounding noise, so only finiteness is required of them
    well = np.ones(64, bool)
    well[[4, 5]] = False
    assert d[well].max() < 5e-5
    r = ops.rodrigues(torch.from_numpy(g["aa_in"]).cuda()).cpu().numpy()
    assert np.abs(r - g["rodrigues"]).max() < 2e-6


def test_rot6d_random_vs_oracle():
    from acr_b200 import ops
    from oracle import rotation_ref
    g = torch.Generator().manual_seed(5)
    x = torch.randn(4096, 96, generator=g)
    aa = ops.rot6d_to_aa(x.cuda()).cpu().numpy()
    ref = rotation_ref.rot6d_to_angular(x.numpy())
    # compare as rotations (axis-angle is discontinuous at pi): R(aa) must agree
    Ra = rotation_ref.batch_rodrigues(aa.reshape(-1, 3))
    Rb = rotation_ref.batch_rodrigues(ref.reshape(-1, 3))
    assert np.abs(Ra - Rb).max() < 2e-5
    assert np.mean(np.abs(aa - ref) < 1e-4) > 0.999


def test_mano_golden(wrapper):
    g = np.load(os.path.join(GOLDEN, "mano_golden.npz"))
    L, R = int(g["L"]), int(g["R"])
    outputs = {"params_dict": {"poses": torch.from_numpy(g["poses"]).cuda(), "betas": torch.from_numpy(g["betas"]).cuda(),
                               "cam": torch.from_numpy(g["cam"]).cuda()},
               "left_hand_num": torch.tensor([L]), "right_hand_num": torch.tensor([R])}
    out = wrapper(outputs, {"offsets": torch.from_numpy(g["offsets"])})
    for k, gk in (("verts", "verts"), ("j3d", "j3d"), ("verts_camed", "verts_camed"), ("pj2d", "pj2d"),
                  ("pj2d_org", "pj2d_org")):
        assert rel_err(out[k].cpu().numpy(), g[gk]) < TOL, k
    assert np.abs(out["verts"].cpu().numpy() - g["verts"]).max() < 3e-6
    assert out["output_hand_type"].tolist() == [0] * L + [1] * R
    # camera translation (device least squares) vs the reference's estimate_translation_np
    assert rel_err(out["cam_trans"].cpu().numpy(), g["cam_trans"]) < TOL


def test_manolayer_dropin_single_side(assets):
    from mano.manolayer import ManoLayer
    from oracle import mano_ref
    g = torch.Generator().manual_seed(1)
    pose = torch.randn(37, 48, generator=g) * 0.6
    betas = torch.randn(37, 10, generator=g)
    for side in ("right", "left"):
        layer = ManoLayer(ncomps=45, center_idx=9, side=side, use_pca=False, flat_hand_mean=False,
                          asset=assets[side]).cuda()
        v, j, c = layer(pose.cuda(), th_betas=betas.cuda())
        rv, rj, rc = mano_ref.mano_forward(assets[side], pose.numpy(), betas.numpy(), side, 9, flip_shapedirs_x=False)
        assert rel_err(v.cpu().numpy(), rv) < TOL and rel_err(j.cpu().numpy(), rj) < TOL
        assert rel_err(c.cpu().numpy(), rc) < TOL
        assert tuple(v.shape) == (37, 778, 3) and tuple(j.shape) == (37, 21, 3) and tuple(c.shape) == (37, 1, 3)
        # no centring / explicit translation paths of the reference signature
        layer.center_idx = None
        v2, j2, c2 = layer(pose[:3].cuda(), th_betas=betas[:3].cuda())
        rv2, rj2, _ = mano_ref.mano_forward(assets[side], pose[:3].numpy(), betas[:3].numpy(), side, None, False)
        assert c2 is None and rel_err(v2.cpu().numpy(), rv2) < TOL
        tr = torch.tensor([[0.1, -0.2, 0.3]] * 3)
        v3, j3, t3 = layer(pose[:3].cuda(), th_betas=betas[:3].cuda(), th_trans=tr.cuda())
        assert rel_err(v3.cpu().numpy(), rv2 + tr.numpy()[:, None]) < TOL


def test_mano_batch512_mixed_sides_and_edges(wrapper, assets):
    """BASELINE config 3 size (N=512 hands) incl. theta->0, theta~pi, ragged L/R and the n_dev row mask."""
    from acr_b200 import ops
    from oracle import mano_ref
    g = torch.Generator().manual_seed(2)
    N, L = 512, 200
    poses = torch.randn(N, 48, generator=g) * 0.5
    betas = torch.randn(N, 10, generator=g)
    poses[0] = 0
    poses[1, :3] = torch.tensor([3.14159, 0, 0])
    poses[2] = 1e-6
    cam = torch.rand(N, 3, generator=g) + 0.5
    offs = torch.tensor([[512., 512, 0, 0, 0, 0, 0, 0, 0, 0]]).repeat(N, 1)
    ht = torch.cat([torch.zeros(L), torch.ones(N - L)]).int()
    ml, mr = wrapper.models()
    n_dev = torch.tensor([N - 5], dtype=torch.int32).cuda()
    out = ops.mano_forward(ml, mr, poses.cuda(), betas.cuda(), ht.cuda(), 1, 9, cam.cuda(), offs.cuda(), n_dev=n_dev)
    ref = mano_ref.mano_wrapper_forward(assets, poses.numpy(), betas.numpy(), L, N - L, cam.numpy(), offs.numpy())
    v = out["verts"].cpu().numpy()
    assert rel_err(v[:N - 5], ref["verts"][:N - 5]) < TOL
    assert rel_err(out["joints"].cpu().numpy()[:N - 5], ref["j3d"][:N - 5]) < TOL
    assert rel_err(out["pj2d_org"].cpu().numpy()[:N - 5], ref["pj2d_org"][:N - 5]) < TOL


def test_open_gate_tracker_smoothing_golden():
    """The K = 1 tracker with the gate open and no miss limit (the per-hand-type smoothing of
    ACR.process_results) vs the reference's filter objects (smooth_golden.npz), frame by frame."""
    from acr_b200 import ops
    g = np.load(os.path.join(GOLDEN, "smooth_golden.npz"))
    tr = ops.HandTracker("cuda", 1, ops.TRACK_GATE_OPEN, ops.TRACK_NO_MISS_LIMIT, 4.0)
    rows = torch.tensor([[0, 0, 0, 0], [0, 1, 0, 0]], dtype=torch.int32).cuda()
    for t in range(g["poses"].shape[0]):
        poses = torch.from_numpy(g["poses"][t].copy()).cuda()
        betas = torch.from_numpy(g["betas"][t].copy()).cuda()
        ops.track_rows(tr, 1, rows, torch.from_numpy(g["det"][t].copy()).cuda(), poses, betas)
        assert np.abs(poses.cpu().numpy() - g["out_poses"][t]).max() < 5e-5, t
        assert np.abs(betas.cpu().numpy() - g["out_betas"][t]).max() < 1e-6, t
