"""CPU: the statement of multi-hand tracking over several streams in one batch (tests/stream_track_ref.py) against the
single-stream statement it is built on, and the argument checks of acr_b200_track_streams in the built library."""
import numpy as np
import pytest

from tests.stream_track_ref import StreamTracker, interleave
from tests.test_cpu_track import _lib, random_scene
from tests.track_ref import Tracker, parse_rows


def stream_scenes(seed, lengths, K):
    """One random-walk scene per stream: scenes[s][i] = (left cells, right cells) of stream s's frame i."""
    return [random_scene(seed * 1000 + s, n, K) for s, n in enumerate(lengths)]


def batch_of(scenes, order, slots=None):
    """The batch of one interleaving: image b is frame i of stream s where b is s's i-th image in ``order``.
    -> hands per image, frame_stream (stream s gets slot slots[s])."""
    B = len(order)
    hands = [None] * B
    seen = [0] * len(scenes)
    for b, s in enumerate(order):
        hands[b] = scenes[s][seen[s]]
        seen[s] += 1
    fs = np.asarray(order if slots is None else [slots[s] for s in order], np.int32)
    return hands, fs


def per_stream_ids(ids, rows, det, fs):
    """{(slot, image's frame number in its stream, side, cell): id} of the detections."""
    out = {}
    for r in range(len(rows)):
        if det[r] > 0 and ids[r] >= 0:
            b, side, c = (int(v) for v in rows[r, :3])
            out[(int(fs[b]), int((fs[:b] == fs[b]).sum()), side, c)] = int(ids[r])
    return out


def test_one_stream_is_the_single_stream_statement():
    K, B = 3, 30
    hands = random_scene(5, 2 * B, K)
    st, one = StreamTracker(1, K, gate=6, max_missed=3), Tracker(K, gate=6, max_missed=3)
    for c in range(2):
        rows, det, _ = parse_rows(hands[c * B:(c + 1) * B], K)
        ids, _ = st.step(rows, det, len(rows), np.zeros(B, np.int32))
        want, _ = one.step(rows, det, len(rows), B)
        assert np.array_equal(ids, want)


@pytest.mark.parametrize("seed", range(4))
def test_interleaving_and_slot_numbers_do_not_change_a_stream(seed):
    K, lengths = 2, [9, 1, 14, 6]
    rng = np.random.default_rng(seed)
    scenes = stream_scenes(seed, lengths, K)
    runs = []
    for slots in (None, [5, 0, 7, 2]):
        order, _, _ = interleave(rng, lengths)
        hands, fs = batch_of(scenes, order, slots)
        rows, det, _ = parse_rows(hands, K)
        ids, _ = StreamTracker(8, K, gate=5, max_missed=2).step(rows, det, len(rows), fs)
        got = per_stream_ids(ids, rows, det, fs)
        if slots is not None:               # back to stream numbers
            back = {v: s for s, v in enumerate(slots)}
            got = {(back[k[0]],) + k[1:]: v for k, v in got.items()}
        runs.append(got)
    assert runs[0] == runs[1] and len(runs[0]) > 10
    # and each stream is the single-stream statement on its own frames
    for s, n in enumerate(lengths):
        rows, det, _ = parse_rows(scenes[s], K)
        want, _ = Tracker(K, gate=5, max_missed=2).step(rows, det, len(rows), n)
        mine = per_stream_ids(want, rows, det, np.zeros(n, np.int32))
        assert {k[1:]: v for k, v in runs[0].items() if k[0] == s} == {k[1:]: v for k, v in mine.items()}


def test_begin_flag_is_a_fresh_tracker():
    K, lengths = 2, [12, 10]
    rng = np.random.default_rng(3)
    scenes = stream_scenes(7, lengths, K)
    order, frames, begin = interleave(rng, lengths, begins=[(0, 5)])
    hands, fs = batch_of(scenes, order)
    rows, det, _ = parse_rows(hands, K)
    ids, _ = StreamTracker(2, K).step(rows, det, len(rows), fs, begin)
    # stream 0's frames 5.. equal a fresh tracker on them alone; stream 1 does not notice
    got = per_stream_ids(ids, rows, det, fs)
    r5, d5, _ = parse_rows(scenes[0][5:], K)
    fresh, _ = Tracker(K).step(r5, d5, len(r5), lengths[0] - 5)
    want = {(0, i + 5, s, c): v for (_, i, s, c), v in per_stream_ids(fresh, r5, d5, np.zeros(7, np.int32)).items()}
    assert {k: v for k, v in got.items() if k[0] == 0 and k[1] >= 5} == want
    assert min(want.values()) in (0, 1)         # the birth counters started over
    r1, d1, _ = parse_rows(scenes[1], K)
    alone, _ = Tracker(K).step(r1, d1, len(r1), lengths[1])
    assert {k[1:]: v for k, v in got.items() if k[0] == 1} == \
        {k[1:]: v for k, v in per_stream_ids(alone, r1, d1, np.zeros(lengths[1], np.int32)).items()}


def test_invalid_streams_and_rows_past_n_dev_are_not_tracked():
    K = 2
    hands = [([64 * 10 + 10], [64 * 30 + 30])] * 6
    rows, det, _ = parse_rows(hands, K)
    fs = np.array([0, -1, 1, 2, 0, 1], np.int32)          # S = 2: -1 and 2 are invalid
    poses = np.ones((len(rows), 48), np.float32)
    ids, out = StreamTracker(2, K, bank=None).step(rows, det, len(rows) - 1, fs, poses=poses, betas=poses[:, :10])
    for r in range(len(rows)):
        bad = fs[rows[r, 0]] not in (0, 1) or r >= len(rows) - 1
        assert (ids[r] == -1) == bad and ((r in out) != bad), r


# ------------------------------------------------------------------------------------------- the built library
def test_abi_argument_checks():
    lib = _lib()
    from acr_b200 import lib as L
    assert {"acr_b200_track_streams_workspace_bytes", "acr_b200_track_streams"} <= set(L.EXPORTS)
    ws = lib.acr_b200_track_streams_workspace_bytes
    assert ws(64, 8, 4) > ws(64, 8, 1) > 0 and ws(64, 8, 16) == ws(64, 8, 8) and ws(128, 8, 4) > ws(64, 8, 4)
    assert ws(-1, 8, 4) == 0 and ws(8, 0, 4) == 0 and ws(8, 8, 0) == 0 and ws(8, 8, 4097) == 0 and ws(8, 8, 4096) > 0
    p = 4096   # never dereferenced: every call below fails its checks before any launch

    def call(poses=p, betas=p, rows=p, flag=p, n_max=8, B=1, K=4, gate=8, missed=15, coeff=4.0, state=p, ids=p,
             fs=p, begin=p, S=4, work=p):
        return lib.acr_b200_track_streams(poses, betas, rows, flag, None, n_max, B, K, gate, missed, coeff, state,
                                          ids, fs, begin, S, work, None)

    cases = [dict(K=0), dict(K=17), dict(B=0), dict(n_max=9), dict(n_max=-1), dict(gate=-1), dict(missed=-1),
             dict(state=None), dict(rows=None), dict(ids=None), dict(poses=None), dict(betas=None), dict(coeff=0.0),
             dict(coeff=-1.0), dict(coeff=float("nan")), dict(S=0), dict(S=-3), dict(S=4097), dict(fs=None),
             dict(work=None)]
    for kw in cases:
        assert call(**kw) == -1, kw                                  # ACR_B200_EINVAL
        assert b"track_streams" in lib.acr_b200_last_error(), kw
    assert b"frame_stream" in (call(fs=None), lib.acr_b200_last_error())[1]
    assert b"S must be" in (call(S=4097), lib.acr_b200_last_error())[1]
