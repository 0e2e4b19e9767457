"""GPU: multi-hand parsing (acr_b200_parse_topk, ``max_hands_per_side`` = K) against tests/parse_topk_ref.py, the
reference's selection (tests/golden/parse_topk_golden.npz) and, at K = 1, acr_b200_parse; then the pipeline at K = 4:
fused_forward + MANO on the synthetic network, CUDA-graph replay, the reference-schema forward and the errors."""
import contextlib
import functools
import os

import numpy as np
import pytest
import torch

from acr_b200 import lib as L
from tests.helpers import rel_err
from tests.parse_topk_ref import (GOLDEN_B, GOLDEN_KS, SCENES, flat, golden_seed, hand_built_maps, multi_peak_maps,
                                  parse_topk, topk_centers)

pytestmark = pytest.mark.gpu

NAMES = dict(l_center="l_center_map", r_center="r_center_map", l_params="l_params_maps", r_params="r_params_maps",
             l_prior="l_prior_maps", r_prior="r_prior_maps")
THRESH = 0.35


@contextlib.contextmanager
def hands_per_side(K):
    from acr.config import ConfigContext, parse_args
    ConfigContext(parse_args(["--max_hands_per_side", str(K)]))
    try:
        yield
    finally:
        ConfigContext(parse_args([]))


def _dev_maps(maps_np):
    out = {}
    for k, n in NAMES.items():
        t = torch.from_numpy(maps_np[n]).cuda().permute(0, 2, 3, 1).contiguous()
        out[k] = (t, t.shape[-1])
    return out


def _call(entry, dmaps, B, K, meta, offs, bufs):
    ms = []
    for k in NAMES:
        t, stride = dmaps[k]
        m = L.Map()
        m.ptr, m.pix_stride = t.data_ptr(), int(stride)
        ms.append(m)
    size = (B, K) if entry == "acr_b200_parse_topk" else (B,)
    return getattr(L.load(), entry)(*ms, *size, THRESH, L.ptr(meta), L.ptr(offs), bufs.struct(),
                                    L.current_stream(torch.device("cuda")))


def _parse(dmaps, B, K, meta=None, entry=None):
    """ParseBuffers(B, K) filled by ops.parse_maps (entry None) or by the named C entry point; synchronised."""
    from acr_b200 import ops
    bufs = ops.ParseBuffers(B, "cuda", K)
    offs = torch.arange(B * 10, dtype=torch.float32, device="cuda").view(B, 10)
    if entry is None:
        ops.parse_maps(dmaps, B, bufs, meta, offs, THRESH, K)
    else:
        L.check(_call(entry, dmaps, B, K, meta, offs, bufs), entry)
    torch.cuda.synchronize()
    bufs._offs = offs
    return bufs


def _check_vs_oracle(bufs, maps_np, K, meta_np):
    ref = parse_topk(maps_np, K, meta_np)
    Lr, Rr = int(ref["left_hand_num"][0]), int(ref["right_hand_num"][0])
    nl, nr = int(ref["detection_flag"][:Lr].sum()), int(ref["detection_flag"][Lr:].sum())
    c = bufs.counts.cpu().numpy()
    assert c[:6].tolist() == [Lr, Rr, Lr + Rr, nl + nr, nl, nr], (c.tolist(), Lr, Rr, nl, nr)
    N = Lr + Rr
    got = lambda t: t[:N].cpu().numpy()
    assert np.array_equal(got(bufs.row_src), ref["row_src"])
    assert np.array_equal(got(bufs.batch_ids), ref["batch_ids"])
    assert np.array_equal(got(bufs.reorganize_idx), ref["reorganize_idx"])
    assert np.array_equal(got(bufs.hand_type), ref["output_hand_type"])
    assert np.array_equal(got(bufs.centers_pred), np.concatenate([ref["l_centers_pred"], ref["r_centers_pred"]]))
    assert np.array_equal(got(bufs.detection_flag), ref["detection_flag"])
    conf = np.concatenate([ref["l_centers_conf"], ref["r_centers_conf"]]).ravel()
    assert np.array_equal(got(bufs.centers_conf), conf)
    assert np.abs(got(bufs.params_pred) - ref["params_pred"]).max() < 1e-6
    if hasattr(bufs, "_offs"):
        assert np.array_equal(got(bufs.offsets_out), bufs._offs.cpu().numpy()[ref["batch_ids"]])
    a, b = got(bufs.poses), ref["params_dict"]["poses"]
    assert np.mean(np.abs(a - b) < 1e-4) > 0.999
    return ref


@functools.lru_cache(maxsize=1)
def _random_case(B):
    maps = multi_peak_maps(900 + B, B)
    return maps, _dev_maps(maps)


@pytest.mark.parametrize("B", [1, 7, 256, 1500])
def test_random_multi_peak_maps(B):
    """K = 1 through acr_b200_parse_topk equals acr_b200_parse in every buffer; K = 2, 4, 16 equal the oracle."""
    from acr_b200.lib import ParseOut
    maps, dmaps = _random_case(B)
    meta = (torch.arange(B) * 3 + 1).cuda()
    old = _parse(dmaps, B, 1, meta, entry="acr_b200_parse")
    new = _parse(dmaps, B, 1, meta, entry="acr_b200_parse_topk")
    for name, _ in ParseOut._fields_:
        assert torch.equal(getattr(old, name), getattr(new, name)), name
    _check_vs_oracle(new, maps, 1, meta.cpu().numpy())
    most = 0
    for K in (2, 4, 16):
        bufs = _parse(dmaps, B, K, meta)
        ref = _check_vs_oracle(bufs, maps, K, meta.cpu().numpy())
        for side, s in enumerate("lr"):     # the whole top-K list, above the threshold or not
            idx, sc = topk_centers(maps[f"{s}_center_map"], K)
            assert np.array_equal(bufs.top_idx[:, side].cpu().numpy(), idx), (K, s)
            assert np.array_equal(bufs.top_score[:, side].cpu().numpy(), sc), (K, s)
        rows = ref["row_src"]
        most = max(most, max(np.sum((rows[:, 0] == b) & (rows[:, 1] == 0)) for b in range(B)))
    if B > 1:
        assert most > 4          # images with more than four hands of a side exist


def test_golden_indices(golden_dir):
    g = np.load(os.path.join(golden_dir, "parse_topk_golden.npz"))
    for K in GOLDEN_KS:
        maps = multi_peak_maps(golden_seed(K), GOLDEN_B)
        bufs = _parse(_dev_maps(maps), GOLDEN_B, K)
        nl, Lr = int(bufs.counts[4]), int(bufs.counts[0])
        rows = bufs.row_src.cpu().numpy()
        for s, sl in (("l", slice(0, nl)), ("r", slice(Lr, Lr + int(bufs.counts[5])))):
            assert np.array_equal(rows[sl, 0], g[f"K{K}__{s}_batch_ids"]), (K, s)
            assert np.array_equal(rows[sl, 2], g[f"K{K}__{s}_flat_inds"]), (K, s)
            yx = np.stack([rows[sl, 2] // 64, rows[sl, 2] % 64], 1).astype(np.float32)
            assert np.array_equal(yx, g[f"K{K}__{s}_center_yxs"]), (K, s)


@pytest.mark.parametrize("name", sorted(SCENES))
@pytest.mark.parametrize("K", [1, 4, 8])
def test_edge_cases(name, K):
    B = SCENES[name][0]
    maps = hand_built_maps(*SCENES[name])
    bufs = _parse(_dev_maps(maps), B, K)
    _check_vs_oracle(bufs, maps, K, None)
    rows = bufs.row_src[: int(bufs.counts[2])].cpu().numpy()
    if name == "five_peaks":
        assert int(bufs.counts[4]) == min(K, 5)
    if name == "plateau_border_thresh":
        assert flat(40, 40) not in rows[:, 2]                 # a score of exactly 0.35f is not a detection
        if K == 8:
            assert rows[:5, 2].tolist() == [flat(10, 10), flat(10, 11), flat(0, 0), flat(63, 63), flat(0, 63)]
    if name == "no_left":
        assert int(bufs.counts[4]) == 0 and float(bufs.detection_flag[0]) == 0.0 and rows[0].tolist() == [0, 0, 0, -1]


def test_k_out_of_range_raises():
    from acr_b200 import ops
    for K in (0, 17):
        with pytest.raises(ValueError):
            ops.ParseBuffers(1, "cuda", K)
    maps = hand_built_maps(*SCENES["scene"])
    dmaps = _dev_maps(maps)
    bufs = ops.ParseBuffers(3, "cuda", 16)
    offs = torch.zeros(3, 10, device="cuda")
    for K in (0, 17):
        assert _call("acr_b200_parse_topk", dmaps, 3, K, None, offs, bufs) == -1      # ACR_B200_EINVAL
    with pytest.raises(ValueError):
        ops.parse_maps(dmaps, 3, bufs, None, offs, THRESH, 4)                       # buffers sized for another K


# ------------------------------------------------------------------------------------------ pipeline at K = 4
def _frames(n, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, 256, (n, 512, 512, 3), generator=g, dtype=torch.uint8)


def _engine_maps(app, B):
    eng = app.model.engine(B, torch.device("cuda", torch.cuda.current_device()))
    return {n: eng.map_nchw(n).cpu().numpy() for n in NAMES.values()}


@pytest.fixture(scope="module")
def multi():
    """W32 bf16 synthetic network whose centre-head bias puts the threshold at the median of the second-best NMS
    peak of every (image, side): about half of them then show at least two hands."""
    from acr.main import ACR
    from acr_b200.synth import load_bn_calibration, make_synthetic_mano, synth_state_dict
    assets = {"left": make_synthetic_mano("left"), "right": make_synthetic_mano("right")}
    B = 6
    x, x2 = _frames(B, 5), _frames(B, 6)
    offs = torch.tensor([[512., 512, 0, 0, 0, 0, 0, 0, 0, 0]]).repeat(B, 1).cuda()
    with hands_per_side(4):
        app = ACR(state_dict=synth_state_dict(0, bn_stats=load_bn_calibration(0)), mano_assets=assets)
        app.fused_forward(x.cuda(), offs)
        torch.cuda.synchronize()
        maps = _engine_maps(app, B)
        second = np.concatenate([topk_centers(maps[f"{s}_center_map"], 2)[1][:, 1] for s in "lr"])
        t = float(np.median(second))
        app = ACR(state_dict=synth_state_dict(0, bn_stats=load_bn_calibration(0), center_bias=1.0 + THRESH - t),
                  mano_assets=assets)
        yield app, assets, B, x, x2, offs
    del app
    torch.cuda.empty_cache()


def test_fused_forward_rows_and_mano_vs_oracle(multi):
    from oracle import mano_ref
    app, assets, B, x, _, offs = multi
    with hands_per_side(4):
        bufs, mano = app.fused_forward(x.cuda(), offs)
        torch.cuda.synchronize()
        maps = _engine_maps(app, B)
    assert bufs.params_pred.shape[0] == 2 * 4 * B and mano["verts"].shape[0] == 2 * 4 * B
    ref = _check_vs_oracle(bufs, maps, 4, None)
    rows = ref["row_src"]
    per = [int(np.sum((rows[:, 0] == b) & (rows[:, 1] == s))) for b in range(B) for s in (0, 1)]
    print("hands per (image, side):", per)
    assert max(per) >= 2 and int(ref["detection_flag"].sum()) > 2
    N = rows.shape[0]
    Lr, Rr = int(ref["left_hand_num"][0]), int(ref["right_hand_num"][0])
    o = np.tile(np.array([512, 512, 0, 0, 0, 0, 0, 0, 0, 0], np.float32), (N, 1))
    pd = ref["params_dict"]
    m = mano_ref.mano_wrapper_forward(assets, pd["poses"], pd["betas"], Lr, Rr, pd["cam"], o)
    for k, mk in (("verts", "verts"), ("joints", "j3d"), ("pj2d_org", "pj2d_org")):
        e = rel_err(mano[k][:N].cpu().numpy(), m[mk])
        assert e < 1e-4, (k, e)
    ct = mano["cam_trans"][:N]
    assert ct.shape == (N, 3) and torch.isfinite(ct).all()


def test_graph_replay_at_k4_equals_eager(multi):
    app, _, B, x, x2, offs = multi
    with hands_per_side(4):
        replay = app.capture_graph(B)
        assert replay.hands_per_side == 4
        counts = []
        for frames in (x, x2):
            batch = frames.cuda()
            bufs, mano = app.fused_forward(batch, offs)
            torch.cuda.synchronize()
            n = int(bufs.counts[2])
            c, v, p = bufs.counts.clone(), mano["verts"][:n].clone(), bufs.params_pred[:n].clone()
            rs, ct = bufs.row_src[:n].clone(), mano["cam_trans"][:n].clone()
            bufs_g, mano_g = replay(batch, offs)
            torch.cuda.synchronize()
            assert torch.equal(bufs_g.counts, c)
            assert torch.equal(bufs_g.row_src[:n], rs) and torch.equal(bufs_g.params_pred[:n], p)
            assert torch.equal(mano_g["verts"][:n], v) and torch.equal(mano_g["cam_trans"][:n], ct)
            counts.append(c.tolist())
        print("graph replay counts:", counts)
    with hands_per_side(2):
        with pytest.raises(ValueError):
            replay(x.cuda(), offs)
    with pytest.raises(ValueError):                     # the default, K = 1
        replay(x.cuda(), offs)
    del replay


def test_reference_schema_forward_and_reorganize(multi):
    from acr.utils import justify_detection_state, reorganize_results
    app, _, B, x, _, offs = multi
    with hands_per_side(4):
        bufs, _ = app.fused_forward(x.cuda(), offs)
        torch.cuda.synchronize()
        want = bufs.row_src[: int(bufs.counts[2])].cpu().numpy().copy()
        nl = int(bufs.counts[0])
        out = app.batch_forward(x, offsets=offs.cpu())
    Lr, Rr = int(out["left_hand_num"]), int(out["right_hand_num"])
    assert Lr + Rr == want.shape[0] and Lr == nl
    cen = np.concatenate([out["l_centers_pred"].cpu().numpy(), out["r_centers_pred"].cpu().numpy()])
    assert np.array_equal(cen, np.stack([want[:, 2] % 64, want[:, 2] // 64], 1))
    assert out["l_centers_conf"].shape == (Lr, 1) and out["verts"].shape == (Lr + Rr, 778, 3)
    assert np.array_equal(out["reorganize_idx"].cpu().numpy(), want[:, 0])
    flag, reorg = justify_detection_state(out["detection_flag"], out["reorganize_idx"])
    assert flag
    reorg = reorg.cpu().numpy()
    res = reorganize_results(out, [f"img{b}.jpg" for b in reorg], reorg)
    det = out["detection_flag_cache"].cpu().numpy()
    for b in range(B):
        mine = want[det, :][want[det, 0] == b]
        hands = res.get(f"img{b}.jpg", [])
        assert len(hands) == len(mine), b
        assert [int(h["hand_type"]) for h in hands] == mine[:, 1].tolist(), b
    assert max(np.bincount(want[det, 0] * 2 + want[det, 1])) >= 2


def test_smoothing_with_several_hands_per_side_raises(multi):
    app, _, B, x, _, offs = multi
    with hands_per_side(4):
        out = app.model({"image": x, "offsets": offs.cpu(), "batch_ids": torch.arange(B)}, **app.demo_cfg)
        app.temporal_optimization = True
        try:
            with pytest.raises(ValueError, match="max_hands_per_side"):
                app.process_results(out)
        finally:
            app.temporal_optimization = False
