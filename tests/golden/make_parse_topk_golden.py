#!/usr/bin/env python
"""Generate tests/golden/parse_topk_golden.npz by running the UNMODIFIED reference's multi-hand centre selection,
``CenterMap.parse_centermap_heatmap_adaptive_scale_batch(train_flag=True)`` (acr/result_parser.py:218-243) with
``max_hand = K``, on seeded multi-peak centre maps (tests/parse_topk_ref.multi_peak_maps), K in GOLDEN_KS.  Runs only
where the reference exists, through the same harness as make_golden.py; the npz is committed.

    python tests/golden/make_parse_topk_golden.py

Per case ``K{K}``: the maps' seed and batch, and the reference's batch_ids, flat indices, centre [y, x] and
scores for each side.  Above-threshold scores in these maps are distinct, so torch.topk's order among equal
scores does not matter.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.abspath(os.path.join(HERE, "..", ".."))
REF = "/root/reference"


def main():
    sys.path.insert(0, ROOT)
    from tests.parse_topk_ref import GOLDEN_B as B, GOLDEN_KS as KS, golden_seed, multi_peak_maps
    from oracle import ref_harness
    torch = ref_harness.import_reference(REF, "make_parse_topk_golden")
    from acr.result_parser import CenterMap
    flat = {"ks": np.array(KS), "B": B}
    for K in KS:
        maps = multi_peak_maps(golden_seed(K), B, with_params=False)
        cm = CenterMap()
        cm.max_hand = K
        for s in "lr":
            m = maps[f"{s}_center_map"]
            above = np.sort(m[m > 0.35])
            assert (np.diff(above) > 0).all(), "above-threshold scores must be distinct"
            b, fi, yx, sc = cm.parse_centermap_heatmap_adaptive_scale_batch(torch.from_numpy(m), train_flag=True)
            flat[f"K{K}__{s}_batch_ids"] = b.numpy().astype(np.int64)
            flat[f"K{K}__{s}_flat_inds"] = fi.numpy().astype(np.int64)
            flat[f"K{K}__{s}_center_yxs"] = yx.numpy().astype(np.float32)
            flat[f"K{K}__{s}_scores"] = sc.numpy().astype(np.float32)
        print(f"K={K}: left {len(flat[f'K{K}__l_batch_ids'])} right {len(flat[f'K{K}__r_batch_ids'])} hands, "
              f"per image max {np.bincount(flat[f'K{K}__l_batch_ids'], minlength=B).max()}")
    out = os.path.join(HERE, "parse_topk_golden.npz")
    np.savez_compressed(out, **flat)
    print("wrote", out)


if __name__ == "__main__":
    main()
