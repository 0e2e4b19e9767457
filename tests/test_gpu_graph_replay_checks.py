"""GPU: a graph replay that raises has written nothing.  For each of capture_graph, capture_frames_graph and
capture_jpeg_graph, captured with a 3-stream tracker (and, for JPEG files, part labels of a fixed capacity): a valid
replay, then one that fails a check with new stream ids; it raises ValueError and leaves the graph's stream ids (and
the plain graph's frames and offsets) as they were, and the next valid replay equals the eager fused_forward on a twin
tracker bit for bit."""
import numpy as np
import pytest
import torch

from acr_b200 import jpeg, ops
from acr_b200.preprocess import RaggedFrames, preprocess_frames
from tests import jpeg_cases as JC

pytestmark = pytest.mark.gpu
B = 3
SID = [torch.tensor(s, dtype=torch.int32) for s in ([0, 1, 2], [2, 0, 1], [1, 2, 0])]   # valid, failing, valid


@pytest.fixture(scope="module")
def app():
    from acr.main import ACR
    from acr_b200.synth import load_bn_calibration, make_synthetic_mano, synth_state_dict
    assets = {"left": make_synthetic_mano("left"), "right": make_synthetic_mano("right")}
    a = ACR(state_dict=synth_state_dict(0, bn_stats=load_bn_calibration(0)), mano_assets=assets)
    yield a
    del a
    torch.cuda.empty_cache()


def _trackers():
    from acr.result_parser import ResultParser
    K = ResultParser.hands_per_side()
    return ops.HandTracker("cuda", K, streams=3), ops.HandTracker("cuda", K, streams=3)


def _snapshot(bufs, mano):
    torch.cuda.synchronize()
    n = int(bufs.counts[2])
    return [bufs.counts.clone(), bufs.params_pred[:n].clone(), bufs.poses[:n].clone(), mano["verts"][:n].clone(),
            mano["pj2d_org"][:n].clone(), mano["track_id"][:n].clone()]


def _assert_equal(got, exp, tracker, twin):
    assert len(got) == len(exp)
    for g, e in zip(got, exp):
        assert torch.equal(g, e)
    assert torch.equal(tracker.state, twin.state)


def _assert_raises_and_keeps(replay, args, kept, match):
    before = [t.clone() for t in kept]
    with pytest.raises(ValueError, match=match):
        replay(*args)
    torch.cuda.synchronize()
    for b, t in zip(before, kept):
        assert torch.equal(b, t)


def _bgr(shapes, seed):
    rng = np.random.default_rng(seed)
    return [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for h, w in shapes]


def test_plain_graph(app):
    t, twin = _trackers()
    replay = app.capture_graph(B, tracker=t)
    g = torch.Generator().manual_seed(0)
    x = [torch.randint(0, 256, (B, 512, 512, 3), generator=g, dtype=torch.uint8).cuda() for _ in range(2)]
    offs = torch.tensor([[512., 512, 0, 0, 0, 0, 0, 0, 0, 0]]).repeat(B, 1).cuda()
    got = _snapshot(*replay(x[0], offs, SID[0]))
    _assert_equal(got, _snapshot(*app.fused_forward(x[0], offs, tracker=twin, stream_ids=SID[0])), t, twin)
    wrong = torch.zeros(B + 1, 512, 512, 3, dtype=torch.uint8, device="cuda")      # no broadcast to (B, ...)
    _assert_raises_and_keeps(replay, (wrong, offs, SID[1]), replay.static_streams + replay.static_inputs,
                             "broadcast")
    got = _snapshot(*replay(x[1], offs, SID[2], [0, 1, 0]))
    exp = _snapshot(*app.fused_forward(x[1], offs, tracker=twin, stream_ids=SID[2], stream_begin=[0, 1, 0]))
    _assert_equal(got, exp, t, twin)


def test_frames_graph(app):
    t, twin = _trackers()
    shapes = [[(720, 1280), (37, 1001), (480, 640)], [(1080, 1920), (300, 257), (1, 1)]]
    frames = [_bgr(s, i) for i, s in enumerate(shapes)]
    cap = max(sum(f.size for f in fs) for fs in frames)
    replay = app.capture_frames_graph(B, cap, tracker=t)
    rf = RaggedFrames(B, cap, torch.device("cuda", torch.cuda.current_device()), 512, exact=True)

    def eager(fs, sid):
        rf.load(fs)
        return _snapshot(*app.fused_forward(*rf.launch(), tracker=twin, stream_ids=sid))

    _assert_equal(_snapshot(*replay(frames[0], SID[0])), eager(frames[0], SID[0]), t, twin)
    over = _bgr([(1080, 1920)] * B, 5)                                              # over max_frame_bytes
    _assert_raises_and_keeps(replay, (over, SID[1]), replay.static_streams, "capacity")
    _assert_equal(_snapshot(*replay(frames[1], SID[2])), eager(frames[1], SID[2]), t, twin)


MIX_A = [(720, 1280, 90, "420", 0, "smooth"), (17, 9, 100, "444", 1, "noisy"), (480, 640, 90, "422", 4, "smooth")]
MIX_B = [(480, 640, 85, "420", 2, "noisy"), (300, 257, 90, "444", 0, "smooth"), (720, 1280, 95, "422", 0, "noisy")]


def test_jpeg_graph(app):
    t, twin = _trackers()
    mixes = [[JC.encode(*s) for s in m] for m in (MIX_A, MIX_B)]
    big = [JC.encode(1080, 1920, 90, "420", 0, "smooth")] * B                       # within the caps, not the labels
    every = mixes + [big]
    coded = max(sum(jpeg.parse(b).scan_len for b in m) for m in every)
    frame_bytes = max(sum(jpeg.parse(b).H * jpeg.parse(b).W * 3 for b in m) for m in every)
    pixels = max(sum(jpeg.parse(b).H * jpeg.parse(b).W for b in m) for m in mixes)
    replay = app.capture_jpeg_graph(B, coded, frame_bytes, tracker=t, part_labels=pixels)
    labels = ops.PartLabels(pixels, B)

    def eager(mix, sid):
        img, offs = preprocess_frames([torch.from_numpy(JC.cv2_decode(b)).cuda() for b in mix])
        snap = _snapshot(*app.fused_forward(img, offs.cuda(), tracker=twin, stream_ids=sid, part_labels=labels))
        return snap + [v.clone() for v in labels.views()]

    def run(mix, sid):
        bufs, mano = replay(mix, sid)
        replay.jpeg.raise_on_status()
        return _snapshot(bufs, mano) + [v.clone() for v in mano["part_labels"].views()]

    got = run(mixes[0], SID[0])
    _assert_equal(got, eager(mixes[0], SID[0]), t, twin)
    _assert_raises_and_keeps(replay, (big, SID[1]), replay.static_streams, "label bytes")
    for g, v in zip(got[-B:], replay.part_labels.views()):                         # the views still read replay 1
        assert torch.equal(g, v)
    _assert_equal(run(mixes[1], SID[2]), eager(mixes[1], SID[2]), t, twin)
