"""GPU: multi-hand tracking (acr_b200_track_hands, acr_b200.ops.HandTracker) against the statement of
tests/track_ref.py: ids exactly, smoothed values within tests/tail_ref.OneEuro64's per-element bounds (one bank per
track), untouched rows bit for bit.  Then the pipeline at K = 4 on the multi-hand synthetic network: fused_forward,
CUDA-graph replay and the eager path."""
import numpy as np
import pytest
import torch

from acr_b200 import lib as L
from tests import tail_ref as T
from tests.test_cpu_track import random_scene
from tests.test_gpu_parse_topk import _frames, hands_per_side, multi  # noqa: F401  (the module's fixture)
from tests.track_ref import GATE_OPEN, NO_MISS_LIMIT, Tracker, parse_rows

pytestmark = pytest.mark.gpu
GUARD = 0x7FC0BEEF
EXTRA = 5          # guard rows past the row table


def dev(a, dtype=np.float32):
    return torch.from_numpy(np.ascontiguousarray(a, dtype)).cuda()


def stream():
    return torch.cuda.current_stream().cuda_stream


class Rig:
    """State, id buffer and guarded pose / beta buffers of one stream, driven through the C ABI."""

    def __init__(self, K):
        self.K = K
        self.state = torch.zeros(int(L.load().acr_b200_track_state_bytes(K)), dtype=torch.uint8, device="cuda")

    def run(self, rows, det, B, poses=None, betas=None, n_dev=None, gate=8, max_missed=15, coeff=4.0, n_max=None):
        """-> (rc, ids, poses out, betas out) as numpy; poses / betas None: ids only."""
        n = len(rows) if n_max is None else n_max
        ids = torch.full((n + EXTRA,), GUARD, dtype=torch.int32, device="cuda")
        rs = torch.zeros(n + EXTRA, 4, dtype=torch.int32, device="cuda")
        rs[:len(rows)] = dev(rows, np.int32)
        fl = torch.zeros(n + EXTRA, device="cuda")
        fl[:len(det)] = dev(det)
        p = b = None
        if poses is not None:
            p = torch.full((n + EXTRA, 48), GUARD, dtype=torch.int32, device="cuda")
            b = torch.full((n + EXTRA, 10), GUARD, dtype=torch.int32, device="cuda")
            p[:len(poses)] = dev(poses).view(torch.int32)
            b[:len(betas)] = dev(betas).view(torch.int32)
        nd = None if n_dev is None else dev([n_dev], np.int32)
        rc = L.load().acr_b200_track_hands(L.ptr(p), L.ptr(b), L.ptr(rs), L.ptr(fl), L.ptr(nd), n, B, self.K, gate,
                                          max_missed, float(coeff), L.ptr(self.state), L.ptr(ids), stream())
        torch.cuda.synchronize()
        ids = ids.cpu().numpy()
        assert (ids[n:] == GUARD).all(), "an id past n_max was written"
        out = [rc, ids[:n]]
        if p is not None:
            pb, bb = p.cpu().numpy(), b.cpu().numpy()
            assert (pb[n:] == GUARD).all() and (bb[n:] == GUARD).all(), "a row past n_max was written"
            out += [pb[:n].view(np.float32), bb[:n].view(np.float32)]
        return out


def scene_inputs(hands, K, seed):
    rows, det, _ = parse_rows(hands, K)
    rng = np.random.default_rng(seed)
    poses = (rng.standard_normal((len(rows), 48)) * 0.4).astype(np.float32)
    betas = rng.standard_normal((len(rows), 10)).astype(np.float32)
    return rows, det, poses, betas


# ------------------------------------------------------------------------------------------------- ids and values
@pytest.mark.parametrize("K", [1, 2, 4, 16])
@pytest.mark.parametrize("B", [1, 7, 256])
def test_ids_and_smoothed_values_follow_the_statement(K, B):
    calls = max(3, 60 // B)
    hands = random_scene(100 * K + B, B * calls, K)
    assert any(not h[s] for h in hands for s in (0, 1)), "a frame with no hands on a side"
    coeff = 4.0
    ref = Tracker(K, gate=6, max_missed=4, bank=lambda: T.OneEuro64(coeff))
    ids_ref = Tracker(K, gate=6, max_missed=4)
    rig, rig_ids = Rig(K), Rig(K)
    worst = dict(pose=0.0, betas=0.0, root=0.0)
    tracks = set()
    for c in range(calls):
        rows, det, poses, betas = scene_inputs(hands[c * B:(c + 1) * B], K, c)
        n = len(rows)
        want, out = ref.step(rows, det, n, B, poses, betas)
        rc, ids, p, b = rig.run(rows, det, B, poses, betas, gate=6, max_missed=4, coeff=coeff)
        assert rc == L.OK
        assert np.array_equal(ids, want), (c, ids, want)
        want2, _ = ids_ref.step(rows, det, n, B)
        rc, ids2 = rig_ids.run(rows, det, B, gate=6, max_missed=4)
        assert rc == L.OK and np.array_equal(ids2, want2)
        for r in range(n):
            if r not in out:            # no detection: untouched, bit for bit
                assert ids[r] == -1
                assert (p[r].view(np.int32) == poses[r].view(np.int32)).all()
                assert (b[r].view(np.int32) == betas[r].view(np.int32)).all()
                continue
            tid, born, res = out[r]
            tracks.add(tid)
            if born:
                assert (p[r, 3:].view(np.int32) == poses[r, 3:].view(np.int32)).all()
                assert (b[r].view(np.int32) == betas[r].view(np.int32)).all()
            e = np.abs(p[r, 3:].astype(np.float64) - res["pose"]) / (res["b_pose"] + 1e-45)
            worst["pose"] = max(worst["pose"], float(e.max()))
            e = np.abs(b[r].astype(np.float64) - res["betas"]) / (res["b_betas"] + 1e-45)
            worst["betas"] = max(worst["betas"], float(e.max()))
            er = np.linalg.norm(T.aa_to_rotmat64(p[r, :3])[0] - T.aa_to_rotmat64(res["aa"])[0])
            worst["root"] = max(worst["root"], er / T.smoothed_root_bound(res["b_M"], res["qnorm"]))
    print(f"K={K} B={B}: {len(tracks)} tracks, worst err/bound", worst)
    assert max(worst.values()) <= 1
    assert len(tracks) > 4                  # births, deaths and gate misses did happen


def test_rows_past_n_dev_and_malformed_rows_are_untouched():
    K, B = 4, 7
    hands = random_scene(9, B, K, p_on=1.0)
    rows, det, poses, betas = scene_inputs(hands, K, 1)
    n = len(rows)
    bad = rows.copy()
    bad[1, 0] = B            # image out of range
    bad[2, 2] = 4096         # cell off the map
    bad[3, 1] = 3            # no side
    nd = n - 2
    ref = Tracker(K)
    want, _ = ref.step(bad, det, nd, B)
    rc, ids, p, b = Rig(K).run(bad, det, B, poses, betas, n_dev=nd, n_max=2 * K * B)
    assert rc == L.OK and np.array_equal(ids[:n], want) and (ids[n:] == -1).all()
    for r in range(n):
        if want[r] < 0:
            assert (p[r].view(np.int32) == poses[r].view(np.int32)).all()
            assert (b[r].view(np.int32) == betas[r].view(np.int32)).all()
    assert (p[n:].view(np.int32) == GUARD).all() and (b[n:].view(np.int32) == GUARD).all()


# -------------------------------------------------------------------------------------------- bit-for-bit anchors
@pytest.mark.parametrize("K", [2, 16])
def test_one_launch_equals_single_frames_and_repeats(K):
    B = 40
    hands = random_scene(77 + K, B, K)
    rows, det, poses, betas = scene_inputs(hands, K, 5)
    many, again = Rig(K), Rig(K)
    rc, ids, p, b = many.run(rows, det, B, poses, betas, gate=6, max_missed=3)
    rc2, ids2, p2, b2 = again.run(rows, det, B, poses, betas, gate=6, max_missed=3)
    assert rc == rc2 == L.OK
    assert np.array_equal(ids, ids2) and (p.view(np.int32) == p2.view(np.int32)).all()
    assert (b.view(np.int32) == b2.view(np.int32)).all() and torch.equal(many.state, again.state)
    one = Rig(K)
    r0 = 0
    for f in range(B):
        r1, d1, _ = parse_rows([hands[f]], K)
        sel = [r for r in range(len(rows)) if rows[r, 0] == f and det[r] > 0]
        if not sel:                     # no hands this frame: the parse's dummy rows only
            rc, i1, p1, b1 = one.run(r1, d1, 1, np.zeros((len(r1), 48), np.float32),
                                     np.zeros((len(r1), 10), np.float32), gate=6, max_missed=3)
            assert rc == L.OK and (i1 == -1).all()
            continue
        rc, i1, p1, b1 = one.run(rows[sel] * [0, 1, 1, 1], det[sel], 1, poses[sel], betas[sel], gate=6,
                                 max_missed=3)
        assert rc == L.OK
        assert np.array_equal(i1, ids[sel]), f
        assert (p1.view(np.int32) == p[sel].view(np.int32)).all() and (b1.view(np.int32) == b[sel].view(np.int32)).all()
        r0 += len(sel)
    assert r0 == int((det > 0).sum())
    assert torch.equal(one.state, many.state)


def test_tracker_wrapper_errors_and_reset():
    from acr_b200 import ops
    t = ops.HandTracker("cuda", 4)
    with pytest.raises(ValueError):
        ops.track_hands(ops.ParseBuffers(2, "cuda", 2), t)
    for bad in (dict(K=0), dict(K=17), dict(K=2, gate=-1), dict(K=2, smooth_coeff=0.0)):
        with pytest.raises(ValueError):
            ops.HandTracker("cuda", **bad)
    t.state.fill_(7)
    t.reset()
    assert int(t.state.count_nonzero()) == 0


# ---------------------------------------------------------------------------------------------- the pipeline, K = 4
def _sequence(x, steps):
    """A stream of batches: the frames shifted a few pixels per step (hands move a little)."""
    return [torch.roll(x, shifts=(3 * i, 2 * i), dims=(1, 2)) for i in range(steps)]


def test_fused_forward_with_tracker_equals_separate_calls(multi):   # noqa: F811
    from acr_b200 import ops
    app, _, B, x, _, offs = multi
    with hands_per_side(4):
        t, twin = ops.HandTracker("cuda", 4), ops.HandTracker("cuda", 4)
        ml, mr = app.mano_regression.models()
        seen = set()
        for batch in _sequence(x.cuda(), 4):
            bufs, mano = app.fused_forward(batch, offs, tracker=t)
            torch.cuda.synchronize()
            n = int(bufs.counts[2])
            got = {k: mano[k][:n].clone() for k in ("verts", "track_id", "pj2d_org")}
            gp = bufs.poses[:n].clone()
            bufs, _ = app.fused_forward(batch, offs)
            ids = ops.track_hands(bufs, twin)
            m2 = ops.mano_forward(ml, mr, bufs.poses, bufs.betas, bufs.hand_type, 1, app.mano_regression.center_idx,
                                  bufs.cam, bufs.offsets_out, n_dev=bufs.counts[2:3])
            torch.cuda.synchronize()
            assert torch.equal(got["track_id"], ids[:n]) and torch.equal(gp, bufs.poses[:n])
            assert torch.equal(got["verts"], m2["verts"][:n]) and torch.equal(got["pj2d_org"], m2["pj2d_org"][:n])
            seen |= set(ids[:n].tolist())
        print("track ids seen:", sorted(seen))
        assert len(seen - {-1}) >= 2
        with pytest.raises(ValueError):
            app.fused_forward(x.cuda(), offs, tracker=t, peers=object())


def test_graph_replay_with_tracker_equals_eager(multi):   # noqa: F811
    from acr_b200 import ops
    app, _, B, x, _, offs = multi
    with hands_per_side(4):
        t, twin = ops.HandTracker("cuda", 4), ops.HandTracker("cuda", 4)
        replay = app.capture_graph(B, tracker=t)
        seq = _sequence(x.cuda(), 3)
        for rnd in range(2):
            for batch in seq:
                bufs, mano = app.fused_forward(batch, offs, tracker=twin)
                torch.cuda.synchronize()
                n = int(bufs.counts[2])
                ids, v, p = mano["track_id"][:n].clone(), mano["verts"][:n].clone(), bufs.poses[:n].clone()
                bufs_g, mano_g = replay(batch, offs)
                torch.cuda.synchronize()
                assert torch.equal(mano_g["track_id"][:n], ids), rnd
                assert torch.equal(bufs_g.poses[:n], p) and torch.equal(mano_g["verts"][:n], v)
            t.reset()
            twin.reset()
        with pytest.raises(ValueError):
            app.capture_graph(B, tracker=ops.HandTracker("cuda", 2))
        del replay


def test_eager_track_hands_gives_the_same_ids(multi):   # noqa: F811
    from acr_b200 import ops
    app, _, B, x, _, offs = multi
    with hands_per_side(4):
        t = ops.HandTracker("cuda", 4, smooth_coeff=None)
        app.track_hands, app._hand_tracker = True, None
        try:
            for batch in _sequence(x.cuda(), 3):
                bufs, mano = app.fused_forward(batch, offs, tracker=t)
                torch.cuda.synchronize()
                n = int(bufs.counts[2])
                want = mano["track_id"][:n].cpu()
                out = app.batch_forward(batch.cpu(), offsets=offs.cpu())
                assert torch.equal(out["track_id"].cpu(), want)
            with pytest.raises(ValueError, match="batch_ids"):
                app.batch_forward(x, offsets=offs.cpu(), batch_ids=torch.arange(B) + 1)
        finally:
            app.track_hands, app._hand_tracker = False, None


def test_k1_track_hands_with_smoothing_equals_temporal_optimization(multi):   # noqa: F811
    app, _, B, x, _, offs = multi
    frames = _sequence(x[:1].cuda(), 6)
    res = {}
    with hands_per_side(1):
        for mode in ("smooth", "track"):
            app.temporal_optimization, app.track_hands = True, mode == "track"
            app.track_gate, app.track_max_missed = GATE_OPEN, NO_MISS_LIMIT
            app._one_euro = app._hand_tracker = None
            try:
                res[mode] = []
                for f in frames:
                    out = app.batch_forward(f.cpu(), offsets=offs[:1].cpu())
                    res[mode].append((out["params_dict"]["poses"].clone(), out["verts"].clone()))
            finally:
                app.temporal_optimization = app.track_hands = False
                app.track_gate, app.track_max_missed = 8, 15
                app._one_euro = app._hand_tracker = None
    for (pa, va), (pb, vb) in zip(res["smooth"], res["track"]):
        assert torch.equal(pa, pb) and torch.equal(va, vb)
