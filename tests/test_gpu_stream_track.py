"""GPU: multi-hand tracking of several streams in one batch (acr_b200_track_streams, HandTracker(streams=S)) against
per-stream acr_b200_track_hands runs, bit for bit -- ids, filtered poses and betas, every state slot -- and against
the statement of tests/stream_track_ref.py; then the pipeline at K = 4: fused_forward with stream ids against
per-stream single-stream trackers on the same batch's rows, graph replays against eager calls, and the eager track_hands path."""
import numpy as np
import pytest
import torch

from acr_b200 import lib as L
from tests.stream_track_ref import StreamTracker, interleave, stream_detections
from tests.test_cpu_stream_track import batch_of, stream_scenes
from tests.test_gpu_parse_topk import hands_per_side, multi  # noqa: F401  (the module's fixture)
from tests.test_gpu_track import EXTRA, GUARD, Rig, _sequence, dev, stream
from tests.track_ref import parse_rows

pytestmark = pytest.mark.gpu
GATE, MISSED, COEFF = 6, 3, 4.0


def run_streams(state, S, K, rows, det, fs, begin, poses=None, betas=None, n_dev=None):
    """acr_b200_track_streams on guarded buffers -> (rc, ids, poses out, betas out) as numpy."""
    n, B = len(rows), len(fs)
    ids = torch.full((n + EXTRA,), GUARD, dtype=torch.int32, device="cuda")
    rs = torch.zeros(n + EXTRA, 4, dtype=torch.int32, device="cuda")
    rs[:n] = dev(rows, np.int32)
    fl = torch.zeros(n + EXTRA, device="cuda")
    fl[:n] = dev(det)
    p = b = None
    if poses is not None:
        p = torch.full((n + EXTRA, 48), GUARD, dtype=torch.int32, device="cuda")
        b = torch.full((n + EXTRA, 10), GUARD, dtype=torch.int32, device="cuda")
        p[:n] = dev(poses).view(torch.int32)
        b[:n] = dev(betas).view(torch.int32)
    nd = None if n_dev is None else dev([n_dev], np.int32)
    ws = torch.empty(int(L.load().acr_b200_track_streams_workspace_bytes(n, B, S)), dtype=torch.uint8, device="cuda")
    fsd, bd = dev(fs, np.int32), (None if begin is None else dev(begin, np.int32))
    rc = L.load().acr_b200_track_streams(L.ptr(p), L.ptr(b), L.ptr(rs), L.ptr(fl), L.ptr(nd), n, B, K, GATE, MISSED,
                                         COEFF, L.ptr(state), L.ptr(ids), L.ptr(fsd), L.ptr(bd), S, L.ptr(ws), stream())
    torch.cuda.synchronize()
    ids = ids.cpu().numpy()
    assert (ids[n:] == GUARD).all(), "an id past n_max was written"
    out = [rc, ids[:n]]
    if p is not None:
        pb, bb = p.cpu().numpy(), b.cpu().numpy()
        assert (pb[n:] == GUARD).all() and (bb[n:] == GUARD).all(), "a row past n_max was written"
        out += [pb[:n].view(np.float32), bb[:n].view(np.float32)]
    return out


def batch_case(seed, S, K, B):
    """A batch of B images from up to S streams, with random stream lengths (some streams absent), invalid stream
    ids, malformed rows and n_dev short of the table.  -> rows, det, poses, betas, frame_stream, n_dev."""
    rng = np.random.default_rng(seed)
    used = min(S, max(1, B // 2))
    lengths = np.bincount(rng.integers(0, used, B), minlength=used)
    scenes = stream_scenes(seed, lengths, K)
    order, _, _ = interleave(rng, list(lengths))
    hands, fs = batch_of(scenes, order, rng.permutation(S)[:used])
    fs[rng.choice(B, B // 16, replace=False)] = rng.choice([-1, S, S + 7, -100], B // 16)   # frames of no stream
    rows, det, _ = parse_rows(hands, K)
    rows = rows.copy()
    m = len(rows)
    for r in rng.choice(m, max(1, m // 40), replace=False):
        kind = rng.integers(4)
        if kind == 0:
            rows[r, 0] = rng.choice([-1, B, B + 3])             # image out of range
        elif kind == 1:
            rows[r, 2] = rng.choice([-1, 4096])                 # cell off the map
        elif kind == 2:
            rows[r, 1] = 2                                      # no side
        else:
            rows[r, 0] = rng.integers(B)                        # out of time order (most of the time)
    poses = (rng.standard_normal((m, 48)) * 0.4).astype(np.float32)
    betas = rng.standard_normal((m, 10)).astype(np.float32)
    return rows, det, poses, betas, fs, m - int(rng.integers(0, 3))


def per_stream_reference(rigs, S, K, rows, det, fs, begin, poses, betas, n_dev, smooth):
    """acr_b200_track_hands per stream on its detections alone (the rows its whole-call table keeps), split before
    each begin flag -> ids, poses, betas."""
    n = min(n_dev, len(rows))
    ids = np.full(len(rows), -1, np.int64)
    p, b = poses.copy(), betas.copy()
    for s in range(S):
        frames = np.flatnonzero(fs == s)
        if not len(frames):
            continue
        _, dets = stream_detections(rows, det, n, frames, K)
        cuts = [i for i in range(len(frames)) if begin[frames[i]]]
        bounds = sorted(set([0] + cuts + [len(frames)]))
        for lo, hi in zip(bounds[:-1], bounds[1:]):
            if lo in cuts:
                rigs[s].state.zero_()
            local = {int(f): i for i, f in enumerate(frames[lo:hi])}
            sel = [r for r in dets if int(rows[r, 0]) in local]
            sub = rows[sel].reshape(-1, 4).copy()
            sub[:, 0] = [local[int(i)] for i in sub[:, 0]]
            res = rigs[s].run(sub, det[sel], hi - lo, poses[sel] if smooth else None, betas[sel] if smooth else None,
                              gate=GATE, max_missed=MISSED, coeff=COEFF)
            assert res[0] == L.OK
            ids[sel] = res[1]
            if smooth:
                p[sel], b[sel] = res[2], res[3]
    return ids, p, b


@pytest.mark.parametrize("smooth", [True, False], ids=["smooth", "ids"])
@pytest.mark.parametrize("K", [1, 4, 16])
@pytest.mark.parametrize("S,B", [(1, 64), (3, 96), (64, 384), (256, 512)])
def test_streams_equal_per_stream_single_stream_calls(S, B, K, smooth):
    nbytes = int(L.load().acr_b200_track_state_bytes(K))
    state = torch.zeros(S * nbytes, dtype=torch.uint8, device="cuda")
    rigs = [Rig(K) for _ in range(S)]
    ref = StreamTracker(S, K, gate=GATE, max_missed=MISSED) if S * B <= 96 * 64 else None
    tracked = 0
    for call in range(2):
        rows, det, poses, betas, fs, n_dev = batch_case(1000 * S + 10 * K + call, S, K, B)
        rng = np.random.default_rng(call)
        begin = ((rng.random(B) < 0.05) & (call > 0)).astype(np.int32)
        res = run_streams(state, S, K, rows, det, fs, begin, poses if smooth else None, betas if smooth else None,
                          n_dev=n_dev)
        assert res[0] == L.OK
        ids = res[1]
        want, wp, wb = per_stream_reference(rigs, S, K, rows, det, fs, begin, poses, betas, n_dev, smooth)
        assert np.array_equal(ids, want), call
        if smooth:
            assert (res[2].view(np.int32) == wp.view(np.int32)).all()
            assert (res[3].view(np.int32) == wb.view(np.int32)).all()
        for s in range(S):
            assert torch.equal(state[s * nbytes:(s + 1) * nbytes], rigs[s].state), s
        if ref is not None:
            sid, _ = ref.step(rows, det, n_dev, fs, begin)
            assert np.array_equal(ids, sid), call
        # untouched: rows past n_dev, malformed rows and frames of invalid streams
        for r in np.flatnonzero(ids < 0):
            if smooth:
                assert (res[2][r].view(np.int32) == poses[r].view(np.int32)).all()
        assert (ids[n_dev:] == -1).all()
        img = rows[:, 0]
        inv = np.array([not (0 <= i < B) or not (0 <= fs[i] < S) for i in img])
        assert (ids[inv] == -1).all()
        tracked += int((ids >= 0).sum())
    assert tracked > 0


@pytest.mark.parametrize("K", [1, 4])
def test_repeated_launches_are_bit_identical_and_s1_is_track_hands(K):
    B, S = 128, 16
    rows, det, poses, betas, fs, n_dev = batch_case(77 + K, S, K, B)
    begin = (np.arange(B) % 37 == 5).astype(np.int32)
    nbytes = int(L.load().acr_b200_track_state_bytes(K))
    outs = []
    for _ in range(2):
        state = torch.zeros(S * nbytes, dtype=torch.uint8, device="cuda")
        outs.append((run_streams(state, S, K, rows, det, fs, begin, poses, betas, n_dev=n_dev), state))
    (a, sa), (b, sb) = outs
    assert np.array_equal(a[1], b[1]) and torch.equal(sa, sb)
    assert (a[2].view(np.int32) == b[2].view(np.int32)).all() and (a[3].view(np.int32) == b[3].view(np.int32)).all()
    # S = 1, every frame on stream 0, no begin flag: acr_b200_track_hands bit for bit
    rows1, det1, _ = parse_rows([([64 * 3 + 4, 64 * 30 + 7], [64 * 50 + 50])] * 5 + [([], [])] * 2, K)
    p1 = np.random.default_rng(1).standard_normal((len(rows1), 48)).astype(np.float32)
    b1 = np.random.default_rng(2).standard_normal((len(rows1), 10)).astype(np.float32)
    one, s1 = Rig(K), torch.zeros(nbytes, dtype=torch.uint8, device="cuda")
    for _ in range(2):
        want = one.run(rows1, det1, 7, p1, b1, gate=GATE, max_missed=MISSED, coeff=COEFF)
        got = run_streams(s1, 1, K, rows1, det1, np.zeros(7, np.int32), None, p1, b1)
        assert np.array_equal(got[1], want[1]) and (got[2].view(np.int32) == want[2].view(np.int32)).all()
        assert torch.equal(s1, one.state)


def test_tracker_wrapper_streams():
    from acr_b200 import ops
    t = ops.HandTracker("cuda", 2, streams=5)
    assert t.state.numel() == 5 * t.slot_bytes and t.slot(4).numel() == t.slot_bytes
    bufs = ops.ParseBuffers(3, "cuda", 2)
    with pytest.raises(ValueError, match="frame_stream"):
        ops.track_hands(bufs, t)
    with pytest.raises(ValueError):
        ops.track_hands(bufs, t, torch.zeros(4, dtype=torch.int32, device="cuda"))
    for bad in (0, 4097):
        with pytest.raises(ValueError):
            ops.HandTracker("cuda", 2, streams=bad)
    t.state.fill_(3)
    t.reset()
    assert int(t.state.count_nonzero()) == 0


# ---------------------------------------------------------------------------------------------- the pipeline, K = 4
ASSIGN = [[0, 1, 2, 0, 1, 2], [2, 2, 0, 1, 1, 0], [1, 0, 0, 2, 1, 2], [0, 2, 1, 1, 2, 0]]   # two frames per stream


def test_fused_forward_with_streams_equals_per_stream_trackers(multi):   # noqa: F811
    """The same batch without a tracker, then each stream's rows alone (images renumbered) through a single-stream
    tracker: ids, filtered poses / betas and every state slot bit for bit."""
    from acr_b200 import ops
    app, _, B, x, _, offs = multi
    with hands_per_side(4):
        t = ops.HandTracker("cuda", 4, streams=3)
        single = [ops.HandTracker("cuda", 4) for _ in range(3)]
        seen = set()
        for step, batch in enumerate(_sequence(x.cuda(), 4)):
            fs = torch.tensor(ASSIGN[step], dtype=torch.int32)
            bufs, mano = app.fused_forward(batch, offs, tracker=t, stream_ids=fs)
            torch.cuda.synchronize()
            n = int(bufs.counts[2])
            got = (mano["track_id"][:n].clone(), bufs.poses[:n].clone(), bufs.betas[:n].clone())
            bufs, _ = app.fused_forward(batch, offs)                 # raw rows of the same batch
            torch.cuda.synchronize()
            img = bufs.row_src[:n, 0].long()
            for s in range(3):
                frames = torch.nonzero(fs == s).flatten().cuda()
                sel = torch.nonzero(fs.cuda()[img] == s).flatten()
                local = torch.full((B,), -1, dtype=torch.int32, device="cuda")
                local[frames] = torch.arange(len(frames), dtype=torch.int32, device="cuda")
                rows = bufs.row_src[sel].clone()
                rows[:, 0] = local[rows[:, 0].long()]
                p, b = bufs.poses[sel].contiguous(), bufs.betas[sel].contiguous()
                ids = ops.track_rows(single[s], len(frames), rows.contiguous(),
                                     bufs.detection_flag[sel].contiguous(), p, b)
                torch.cuda.synchronize()
                assert torch.equal(got[0][sel], ids[:len(sel)]), (step, s)
                assert torch.equal(got[1][sel], p) and torch.equal(got[2][sel], b), (step, s)
                assert torch.equal(t.slot(s), single[s].state), (step, s)
                seen |= {(s, i) for i in ids[:len(sel)].tolist() if i >= 0}
        print("(stream, track id) seen:", sorted(seen))
        assert len(seen) >= 4
        with pytest.raises(ValueError, match="stream_ids"):
            app.fused_forward(x.cuda(), offs, tracker=t)


def test_graph_replays_with_streams_equal_eager(multi):   # noqa: F811
    from acr_b200 import ops
    from acr_b200.preprocess import RaggedFrames
    app, _, B, x, _, offs = multi
    seq = _sequence(x.cuda(), 4)
    begins = [None, None, [0, 0, 1, 0, 0, 0], None]        # step 2: slot 0 gets a new camera
    with hands_per_side(4):
        t, tf, twin, twin_f = (ops.HandTracker("cuda", 4, streams=3) for _ in range(4))
        replay = app.capture_graph(B, tracker=t)
        nbytes = max(f.numel() for f in seq) * B
        replay_f = app.capture_frames_graph(B, nbytes, tracker=tf)
        rf = RaggedFrames(B, nbytes, torch.device("cuda", torch.cuda.current_device()), 512, exact=True)
        with pytest.raises(ValueError):
            replay(seq[0], offs)
        with pytest.raises(ValueError):
            replay(seq[0], offs, [0, 1, 2])
        for step, batch in enumerate(seq):
            fs, beg = ASSIGN[step], begins[step]
            bgr = [f.flip(-1) for f in batch]                    # the frames graph takes BGR frames
            sid = torch.tensor(fs, dtype=torch.int32)
            sb = None if beg is None else torch.tensor(beg, dtype=torch.int32)
            bufs, mano = app.fused_forward(batch, offs, tracker=twin, stream_ids=sid, stream_begin=sb)
            torch.cuda.synchronize()
            n = int(bufs.counts[2])
            ids, v, p = mano["track_id"][:n].clone(), mano["verts"][:n].clone(), bufs.poses[:n].clone()
            bufs_g, mano_g = replay(batch, offs, sid, sb)
            torch.cuda.synchronize()
            assert torch.equal(mano_g["track_id"][:n], ids), step
            assert torch.equal(bufs_g.poses[:n], p) and torch.equal(mano_g["verts"][:n], v)
            assert torch.equal(t.state, twin.state)
            # from raw frames: the frames graph against eager preprocessing + fused_forward on a twin state
            bufs_f, mano_f = replay_f(bgr, sid, sb)
            torch.cuda.synchronize()
            nf = int(bufs_f.counts[2])
            idf, pf = mano_f["track_id"][:nf].clone(), bufs_f.poses[:nf].clone()
            rf.load(bgr)
            bufs_e, mano_e = app.fused_forward(*rf.launch(), tracker=twin_f, stream_ids=sid, stream_begin=sb)
            torch.cuda.synchronize()
            assert int(bufs_e.counts[2]) == nf
            assert torch.equal(mano_e["track_id"][:nf], idf) and torch.equal(bufs_e.poses[:nf], pf), step
            assert torch.equal(tf.state, twin_f.state)
        del replay, replay_f


def test_eager_track_streams_gives_the_same_ids(multi):   # noqa: F811
    from acr_b200 import ops
    app, _, B, x, _, offs = multi
    with hands_per_side(4):
        t = ops.HandTracker("cuda", 4, smooth_coeff=None, streams=3)
        app.track_hands, app.track_streams, app._hand_tracker = True, 3, None
        try:
            for step, batch in enumerate(_sequence(x.cuda(), 3)):
                sid = torch.tensor(ASSIGN[step], dtype=torch.int32)
                bufs, mano = app.fused_forward(batch, offs, tracker=t, stream_ids=sid)
                torch.cuda.synchronize()
                n = int(bufs.counts[2])
                want = mano["track_id"][:n].cpu()
                out = app.batch_forward(batch.cpu(), offsets=offs.cpu(), stream_ids=sid)
                assert torch.equal(out["track_id"].cpu(), want), step
            with pytest.raises(ValueError, match="stream_ids"):
                app.batch_forward(x, offsets=offs.cpu())
        finally:
            app.track_hands, app.track_streams, app._hand_tracker = False, 1, None
