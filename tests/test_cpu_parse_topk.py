"""CPU: multi-hand parsing (``max_hands_per_side`` = K).  The oracle's top-K selection against the reference's own
(tests/golden/parse_topk_golden.npz), the oracle at K = 1 against ``oracle/parse_ref.parse``, the row / prior rules
on hand-built maps, the host checks of K, ``reorganize_results`` with several hands per image, and the SASS of the
new kernels."""
import os
import sys

import numpy as np
import pytest
import torch

from oracle import parse_ref
from tests.parse_topk_ref import (GOLDEN_B, GOLDEN_KS, SCENES, flat, golden_seed, hand_built_maps, multi_peak_maps,
                                  parse_centers_topk, parse_maps_topk, parse_topk)

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
KEYS = ("params_pred", "detection_flag", "reorganize_idx", "batch_ids", "l_centers_pred", "r_centers_pred",
        "l_centers_conf", "r_centers_conf", "left_hand_num", "right_hand_num", "output_hand_type")


def test_topk_selection_equals_reference_golden(golden_dir):
    g = np.load(os.path.join(golden_dir, "parse_topk_golden.npz"))
    assert tuple(g["ks"]) == GOLDEN_KS and int(g["B"]) == GOLDEN_B
    multi = 0
    for K in GOLDEN_KS:
        maps = multi_peak_maps(golden_seed(K), GOLDEN_B, with_params=False)
        for s in "lr":
            b, fi, yx, sc = parse_centers_topk(maps[f"{s}_center_map"], K)
            assert np.array_equal(b, g[f"K{K}__{s}_batch_ids"]), (K, s)
            assert np.array_equal(fi, g[f"K{K}__{s}_flat_inds"]), (K, s)
            assert np.array_equal(yx, g[f"K{K}__{s}_center_yxs"]), (K, s)
            assert np.array_equal(sc, g[f"K{K}__{s}_scores"]), (K, s)
            multi = max(multi, np.bincount(b, minlength=GOLDEN_B).max())
    assert multi == max(GOLDEN_KS)


def _random_maps(B, seed):
    """The maps of tests/test_gpu_parse.py::test_parse_random_vs_oracle."""
    g = np.random.default_rng(seed)
    maps = {}
    for s in "lr":
        cm = (g.standard_normal((B, 1, 64, 64)) * 0.12).astype(np.float32)
        on = g.random(B) < 0.7
        for b in np.nonzero(on)[0]:
            cm[b, 0, g.integers(0, 64), g.integers(0, 64)] = 0.5 + g.random()
        maps[f"{s}_center_map"] = cm
        maps[f"{s}_params_maps"] = g.standard_normal((B, 109, 64, 64)).astype(np.float32)
        maps[f"{s}_prior_maps"] = (g.standard_normal((B, 106, 64, 64)) * 0.1).astype(np.float32)
    return maps


@pytest.mark.parametrize("case", ["random_B1", "random_B7", "multi_peak_B24"])
def test_k1_equals_parse_ref(case):
    maps = {"random_B1": lambda: _random_maps(1, 0), "random_B7": lambda: _random_maps(7, 1),
            "multi_peak_B24": lambda: multi_peak_maps(5, 24)}[case]()
    B = maps["l_center_map"].shape[0]
    meta = np.arange(B) * 3 + 1
    ref = parse_ref.parse(maps, meta)
    got = parse_topk(maps, 1, meta)
    for k in KEYS:
        assert got[k].shape == np.asarray(ref[k]).shape and np.array_equal(got[k], ref[k]), k
    for k in ("cam", "global_orient", "hand_pose", "betas", "poses"):
        assert np.array_equal(got["params_dict"][k], ref["params_dict"][k]), k


# ------------------------------------------------------------------------------------------ hand-built maps
def scene(name):
    return hand_built_maps(*SCENES[name])


def test_row_order_counts_and_partners():
    out = parse_maps_topk(scene("scene"), 4)
    rows = out["row_src"].tolist()
    assert rows == [[0, 0, flat(10, 10), -1], [0, 0, flat(40, 40), -1], [0, 0, flat(20, 50), -1],
                    [2, 0, flat(5, 5), flat(6, 8)],
                    [1, 1, flat(30, 30), -1], [2, 1, flat(6, 8), flat(5, 5)], [2, 1, flat(50, 50), flat(5, 5)]]
    assert int(out["left_hand_num"][0]) == 4 and int(out["right_hand_num"][0]) == 3
    assert out["detection_flag"].tolist() == [1.0] * 7
    assert out["reorganize_idx"].tolist() == [0, 0, 0, 2, 1, 2, 2]
    assert out["l_centers_pred"].tolist() == [[10, 10], [40, 40], [50, 20], [5, 5]]
    # the prior is the own side's prior map at the partner, added to params 3..108
    maps = scene("scene")
    plain = maps["l_params_maps"][2, :, 5, 5].copy()
    plain[3:] += maps["l_prior_maps"][2, :, 6, 8]
    assert np.array_equal(out["params_pred"][3], plain)
    assert np.array_equal(out["params_pred"][0], maps["l_params_maps"][0, :, 10, 10])


def test_k_caps_hands_per_side_and_keeps_the_best():
    out = parse_maps_topk(scene("scene"), 2)
    assert [r[:3] for r in out["row_src"].tolist()][:3] == [[0, 0, flat(10, 10)], [0, 0, flat(40, 40)],
                                                           [2, 0, flat(5, 5)]]
    out = parse_maps_topk(scene("five_peaks"), 4)
    assert [r[2] for r in out["row_src"][:4]] == [flat(8 * i + 4, 9) for i in (4, 3, 2, 1)]


def test_partner_ties_go_to_the_lower_rank():
    # both right hands are at squared distance 16 from the left hand; rank 0 has the higher flat index
    rows = parse_maps_topk(scene("tie_partner"), 2)["row_src"]
    assert rows[0].tolist() == [0, 0, flat(20, 20), flat(20, 24)]


def test_dummy_row_and_gate():
    out = parse_maps_topk(scene("no_left"), 4)
    assert out["row_src"].tolist() == [[0, 0, 0, -1], [1, 1, flat(3, 3), -1], [1, 1, flat(40, 3), -1]]
    assert out["detection_flag"].tolist() == [0.0, 1.0, 1.0]
    assert int(out["left_hand_num"][0]) == 1 and int(out["right_hand_num"][0]) == 2
    # the batch's first left and first right rows are > 32 apart: no prior anywhere, even for close pairs
    assert (parse_maps_topk(scene("gate_off"), 4)["row_src"][:, 3] == -1).all()
    assert parse_maps_topk(scene("gate_on"), 4)["row_src"][:, 3].tolist() == [flat(20, 20), flat(31, 31), flat(0, 0), flat(30, 30)]


def test_plateau_border_and_threshold():
    out = parse_maps_topk(scene("plateau_border_thresh"), 8)
    fis = [r[2] for r in out["row_src"][: int(out["left_hand_num"][0])]]
    # the plateau survives the NMS twice (lower index first); the border peaks are found; exactly 0.35f is excluded
    assert fis == [flat(10, 10), flat(10, 11), flat(0, 0), flat(63, 63), flat(0, 63)]


# ------------------------------------------------------------------------------------------ host layers
def test_hands_per_side_is_validated():
    from acr.config import ConfigContext, parse_args
    from acr.result_parser import ResultParser
    from acr_b200.ops import ParseBuffers
    try:
        assert ResultParser.hands_per_side() == 1
        assert parse_args([]).max_hand == 4        # the reference's max_hand does not switch multi-hand parsing on
        ConfigContext(parse_args(["--max_hands_per_side", "4"]))
        assert ResultParser.hands_per_side() == 4
        for bad in ("0", "17"):
            ConfigContext(parse_args(["--max_hands_per_side", bad]))
            with pytest.raises(ValueError):
                ResultParser.hands_per_side()
    finally:
        ConfigContext(parse_args([]))
    with pytest.raises(ValueError):
        ParseBuffers(2, "cpu", 17)
    b = ParseBuffers(3, "cpu", 4)
    assert b.params_pred.shape == (24, 109) and b.row_src.shape == (24, 4) and b.top_idx.shape == (3, 2, 4)
    assert ParseBuffers(3, "cpu").top_idx.shape == (3, 2)


def test_parse_rows_is_2kb():
    from acr_b200.dist import gather_layout, parse_rows
    assert parse_rows(5) == 10 and parse_rows(5, 4) == 40
    gather_layout(2, parse_rows(3, 16))


def test_reorganize_results_lists_every_hand_under_its_image():
    from acr.utils import reorganize_results
    # four hands of image 0 (two left, two right), two of image 1, one undetected row
    n = 7
    g = torch.Generator().manual_seed(0)
    f = lambda *s: torch.randn(*s, generator=g)
    det = torch.tensor([1, 1, 1, 1, 1, 1, 0], dtype=torch.bool)
    outputs = {"detection_flag_cache": det, "params_dict": {"cam": f(n, 3), "poses": f(n, 48), "betas": f(n, 10)},
               "cam_trans": f(n, 3), "j3d": f(n, 21, 3), "verts": f(n, 778, 3), "pj2d": f(n, 21, 2),
               "pj2d_org": f(n, 21, 2), "output_hand_type": torch.tensor([0, 0, 0, 1, 1, 1, 0], dtype=torch.int32)}
    reorg = np.array([0, 0, 1, 0, 0, 1])            # detected rows only
    paths = ["a.jpg", "a.jpg", "b.jpg", "a.jpg", "a.jpg", "b.jpg"]
    res = reorganize_results(outputs, paths, reorg)
    assert sorted(res) == ["a.jpg", "b.jpg"]
    assert len(res["a.jpg"]) == 4 and len(res["b.jpg"]) == 2
    assert [int(h["hand_type"]) for h in res["a.jpg"]] == [0, 0, 1, 1]
    want = outputs["verts"][[0, 1, 3, 4]].numpy().astype(np.float16)
    assert np.array_equal(np.stack([h["verts"] for h in res["a.jpg"]]), want)


def test_topk_parse_kernels_do_not_spill():
    lib = os.path.join(ROOT, "arbitrary-hands-3d-reconstruction_b200", "lib", "libacr_b200.so")
    if not (os.path.exists(lib) and os.path.exists("/usr/local/cuda/bin/cuobjdump")):
        pytest.skip("library not built or no cuobjdump")
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    try:
        import sass_audit
        rows = sass_audit.audit(lib)
    finally:
        sys.path.pop(0)
    for name in ("parse_topk_kernel", "parse_topk_scan_kernel"):
        assert name in rows, sorted(n for n in rows if "parse" in n)
        r = rows[name]
        assert r["LDL"] == 0 and r["STL"] == 0, f"{name}: {r['LDL']} LDL / {r['STL']} STL"
