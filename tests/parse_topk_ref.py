"""CPU/numpy statement of multi-hand parsing (``max_hands_per_side`` = K, acr_b200_parse_topk), built on the K = 1
oracle ``oracle/parse_ref.py``.  The selection is the reference's ``train_flag=True`` path of
``CenterMap.parse_centermap_heatmap_adaptive_scale_batch`` (acr/result_parser.py:218-243) with ``max_hand = K``,
pinned by tests/golden/parse_topk_golden.npz (tests/golden/make_parse_topk_golden.py).  The reference has no
working K > 1 form of ``parse_maps``, so the rows and the cross-hand prior are defined here (DESIGN.md,
"Multi-hand parsing"):

- rows: every left hand (image-major, rank-minor, ``torch.where(mask)`` order), then every right hand; a side with
  no detection in the batch gets the dummy row of the K = 1 parse;
- prior: hand (b, side, k) adds its own side's prior map sampled at the nearest opposite-side hand of image b
  (integer squared grid distance, ties to the lower rank), nothing when image b has none;
- gate: ``determine_coeff`` on the batch's first left and first right rows, as at K = 1.
At K = 1 this is ``parse_ref.parse`` exactly.
"""
import numpy as np

from oracle.parse_ref import CONF_THRESH, MAP, PART_IDX, F, _sample, nms5
from oracle.rotation_ref import rot6d_to_angular

GOLDEN_KS = (1, 2, 4, 8)     # tests/golden/parse_topk_golden.npz: K values, batch and map seeds
GOLDEN_B = 12


def golden_seed(K):
    return 4100 + K


def topk_centers(center_map, K):
    """-> (top_idx (B,K) int64, top_score (B,K) f32): the K best NMS scores of each map in descending order, equal
    scores to the lower flat index first."""
    s = nms5(np.asarray(center_map, F)).reshape(center_map.shape[0], -1)
    order = np.argsort(-s, axis=1, kind="stable")[:, :K]
    return order.astype(np.int64), np.take_along_axis(s, order, 1)


def parse_centers_topk(center_map, K, thresh=CONF_THRESH):
    """The reference's train_flag=True return: batch_ids (n,), flat_inds (n,), cyxs (n,2) [y,x], scores (n,)."""
    idx, sc = topk_centers(center_map, K)
    m = sc > F(thresh)
    b = np.nonzero(m)[0]
    fi = idx[m]
    return b.astype(np.int64), fi, np.stack([fi // MAP, fi % MAP], 1).astype(F), sc[m]


def nearest(fi, others):
    """Nearest of the flat indices ``others`` to ``fi`` on the 64-grid (ties: the first), or -1."""
    best, bd = -1, None
    for o in others:
        d = (fi // MAP - o // MAP) ** 2 + (fi % MAP - o % MAP) ** 2
        if bd is None or d < bd:
            best, bd = int(o), d
    return best


def parse_maps_topk(maps, K, batch_ids_meta=None, thresh=CONF_THRESH):
    """The ``parse_ref.parse_maps`` schema for up to K hands per image and side, plus ``row_src`` (N,4):
    image, side, flat index, partner's flat index or -1."""
    cms = {s: maps[f"{s}_center_map"] for s in "lr"}
    B = cms["l"].shape[0]
    det = {}
    for s in "lr":
        b, fi, _, _ = parse_centers_topk(cms[s], K, thresh)
        det[s] = (b, fi)
    per_img = {s: [det[s][1][det[s][0] == b] for b in range(B)] for s in "lr"}
    flags, rows = [], []
    for side, s in enumerate("lr"):
        if len(det[s][0]):
            rows += [[int(b), side, int(f), -1] for b, f in zip(*det[s])]
            flags += [True] * len(det[s][0])
        else:
            rows.append([0, side, 0, -1])
            flags.append(False)
    rows = np.array(rows, np.int64)
    nl, nr = len(det["l"][0]), len(det["r"][0])
    prior_on = False
    if nl and nr:
        il, ir = det["l"][1][0], det["r"][1][0]
        d = np.sqrt(F((il // MAP - ir // MAP) ** 2 + (il % MAP - ir % MAP) ** 2))
        prior_on = not d > 32
    if prior_on:
        for r in rows:
            r[3] = nearest(r[2], per_img["rl"[r[1]]][r[0]])
    params = np.zeros((len(rows), 109), F)
    for side, s in enumerate("lr"):
        sel = rows[:, 1] == side
        params[sel] = _sample(maps[f"{s}_params_maps"], rows[sel, 0], rows[sel, 2])
        pri = sel & (rows[:, 3] >= 0)
        if pri.any():
            params[pri, 3:] += _sample(maps[f"{s}_prior_maps"], rows[pri, 0], rows[pri, 3])
    L = max(nl, 1)
    lr, rr = rows[:L], rows[L:]
    out = {"row_src": rows.astype(np.int32), "detection_flag": np.asarray(flags, F), "params_pred": params,
           "l_params_pred": params[:L], "r_params_pred": params[L:]}
    out["l_centers_pred"] = np.stack([lr[:, 2] % MAP, lr[:, 2] // MAP], 1)
    out["r_centers_pred"] = np.stack([rr[:, 2] % MAP, rr[:, 2] // MAP], 1)
    out["l_centers_conf"] = _sample(maps["l_center_map"], lr[:, 0], lr[:, 2])
    out["r_centers_conf"] = _sample(maps["r_center_map"], rr[:, 0], rr[:, 2])
    out["left_hand_num"] = np.array([len(lr)], np.int64)
    out["right_hand_num"] = np.array([len(rr)], np.int64)
    meta = np.arange(B) if batch_ids_meta is None else np.asarray(batch_ids_meta)
    out["reorganize_idx"] = meta[rows[:, 0]]
    out["batch_ids"] = rows[:, 0]
    out["detection_flag_cache"] = out["detection_flag"].astype(bool)
    return out


def parse_topk(maps, K, batch_ids_meta=None, thresh=CONF_THRESH):
    """``parse_ref.parse`` for up to K hands per image and side."""
    out = parse_maps_topk(maps, K, batch_ids_meta, thresh)
    p = out["params_pred"]
    o = np.cumsum((0,) + PART_IDX)
    pd = dict(cam=p[:, o[0]:o[1]].copy(), global_orient=p[:, o[1]:o[2]].copy(),
              hand_pose=p[:, o[2]:o[3]].copy(), betas=p[:, o[3]:o[4]].copy())
    pd["hand_pose"] = rot6d_to_angular(pd["hand_pose"])
    pd["global_orient"] = rot6d_to_angular(pd["global_orient"])
    pd["poses"] = np.concatenate([pd["global_orient"], pd["hand_pose"]], 1)
    L, R = int(out["left_hand_num"][0]), int(out["right_hand_num"][0])
    out["output_hand_type"] = np.concatenate([np.zeros(L), np.ones(R)]).astype(np.int32)
    out["params_dict"] = pd
    return out


def multi_peak_maps(seed, B, max_peaks=10, with_params=True):
    """Seeded maps with 0..max_peaks centre peaks of distinct random heights in (0.36, 1.0) per image and side, on
    a 0.08-sigma noise floor (which itself crosses 0.35 now and then).  Peaks may fall within each other's NMS
    window; the NMS decides, as in the reference.  The parameter and prior maps come from their own stream, so the
    centre maps do not depend on ``with_params``."""
    g, gp = np.random.default_rng(seed), np.random.default_rng(seed + 1_000_000)
    maps = {}
    for s in "lr":
        cm = (g.standard_normal((B, 1, MAP, MAP)) * 0.08).astype(F)
        for b in range(B):
            n = int(g.integers(0, max_peaks + 1))
            ys, xs = g.integers(0, MAP, n), g.integers(0, MAP, n)
            cm[b, 0, ys, xs] = g.uniform(0.36, 1.0, n).astype(F)
        maps[f"{s}_center_map"] = cm
        if with_params:
            maps[f"{s}_params_maps"] = gp.standard_normal((B, 109, MAP, MAP), dtype=F)
            maps[f"{s}_prior_maps"] = gp.standard_normal((B, 106, MAP, MAP), dtype=F) * F(0.1)
    return maps


def flat(y, x):
    return y * MAP + x


def hand_built_maps(B, peaks):
    """peaks: {(side, b): [(y, x, score), ...]} on all-zero centre maps; seeded parameter / prior maps."""
    g = np.random.default_rng(11)
    maps = {}
    for s in "lr":
        cm = np.zeros((B, 1, MAP, MAP), F)
        for (side, b), pk in peaks.items():
            if side == s:
                for y, x, v in pk:
                    cm[b, 0, y, x] = v
        maps[f"{s}_center_map"] = cm
        maps[f"{s}_params_maps"] = g.standard_normal((B, 109, MAP, MAP), dtype=F)
        maps[f"{s}_prior_maps"] = g.standard_normal((B, 106, MAP, MAP), dtype=F) * F(0.1)
    return maps


# hand-built scenes (B, peaks); "scene" has three left hands in image 0, none in image 1 and one in image 2
SCENES = {
    "scene": (3, {("l", 0): [(10, 10, .9), (40, 40, .8), (20, 50, .7)], ("l", 2): [(5, 5, .6)],
                  ("r", 1): [(30, 30, .95)], ("r", 2): [(6, 8, .5), (50, 50, .45)]}),
    "five_peaks": (1, {("l", 0): [(8 * i + 4, 9, .4 + .1 * i) for i in range(5)], ("r", 0): [(60, 60, .9)]}),
    "tie_partner": (1, {("l", 0): [(20, 20, .9)], ("r", 0): [(20, 24, .9), (20, 16, .8)]}),
    "no_left": (2, {("r", 1): [(3, 3, .9), (40, 3, .8)]}),
    "gate_off": (2, {("l", 0): [(0, 0, .9)], ("r", 0): [(63, 63, .9)], ("l", 1): [(30, 30, .9)], ("r", 1): [(31, 31, .9)]}),
    "gate_on": (2, {("l", 0): [(0, 0, .9)], ("r", 0): [(20, 20, .9)], ("l", 1): [(30, 30, .9)], ("r", 1): [(31, 31, .9)]}),
    "plateau_border_thresh": (1, {("l", 0): [(10, 10, .7), (10, 11, .7), (0, 0, .6), (63, 63, .5), (0, 63, .4),
                                             (40, 40, .35)], ("r", 0): [(12, 12, .8)]}),
}
