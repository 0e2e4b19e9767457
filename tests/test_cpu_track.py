"""CPU: the statement of multi-hand tracking (tests/track_ref.py) on scripted scenes, its anchor to the reference's
filter objects (tests/golden/smooth_golden.npz), and the argument checks of acr_b200_track_hands in the built library."""
import os

import numpy as np
import pytest

from oracle import rotation_ref
from tests.helpers import GOLDEN
from tests.track_ref import GATE_OPEN, NO_MISS_LIMIT, Tracker, parse_rows

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
LIB = os.path.join(ROOT, "arbitrary-hands-3d-reconstruction_b200", "lib", "libacr_b200.so")


def cell(y, x):
    return y * 64 + x


def run(tr, frames, K):
    """frames[t] = (left cells, right cells) of one frame, one call per frame -> per frame {(side, rank): id}."""
    out = []
    for hands in frames:
        rows, det, _ = parse_rows([hands], K)
        ids, _ = tr.step(rows, det, len(rows), 1)
        got = {}
        for r, (b, s, c, _) in enumerate(rows):
            if det[r] > 0:
                got[(int(s), hands[s].index(int(c)))] = int(ids[r])
        out.append(got)
    return out


def test_parallel_hands_keep_their_ids():
    frames = [([cell(20, 10 + t), cell(40, 10 + t)], []) for t in range(20)]
    out = run(Tracker(2), frames, 2)
    assert all(f == {(0, 0): 0, (0, 1): 2} for f in out)


def test_rank_order_changes_do_not_swap_ids():
    frames = [([cell(20, 10), cell(40, 10)], []), ([cell(40, 11), cell(20, 11)], [])]
    out = run(Tracker(2), frames, 2)
    assert out[1] == {(0, 0): 2, (0, 1): 0}


@pytest.mark.parametrize("gap", [1, 5, 6, 9])
def test_occlusion_up_to_max_missed_keeps_the_id(gap):
    frames = [([cell(30, 30)], [])] * 3 + [([], [])] * gap + [([cell(30, 31)], [])]
    out = run(Tracker(1, max_missed=5), frames, 1)
    assert out[-1][(0, 0)] == (0 if gap <= 5 else 2)


def test_jump_beyond_the_gate_is_a_new_track():
    frames = [([cell(10, 10)], [])] * 2 + [([cell(10, 10 + 9)], [])] + [([cell(10, 19 + 8)], [])]
    tr = Tracker(1, gate=8, bank=lambda: rotation_ref.OneEuroBank(4.0))
    rng = np.random.default_rng(1)
    ids, born = [], []
    for hands in frames:
        rows, det, _ = parse_rows([hands], 1)
        p = rng.standard_normal((len(rows), 48)).astype(np.float32)
        b = rng.standard_normal((len(rows), 10)).astype(np.float32)
        got, o = tr.step(rows, det, len(rows), 1, p, b)
        ids.append(int(got[0]))
        born.append(o[0][1])
        pose, betas = o[0][2]
        if o[0][1]:                         # a first frame passes pose and betas through
            assert (pose[3:] == p[0, 3:]).all() and (betas == b[0]).all()
    assert ids == [0, 0, 2, 2] and born == [True, False, True, False]


def test_full_slots_evict_the_most_missed():
    # K = 2: A and B live; A misses 2 frames, B 1; a new far hand takes A's slot (most misses)
    A, B, C = cell(5, 5), cell(50, 50), cell(5, 60)
    frames = [([A, B], []), ([B], []), ([], []), ([B, C], [])]
    tr = Tracker(2, gate=8, max_missed=10)
    out = run(tr, frames, 2)
    assert out[0] == {(0, 0): 0, (0, 1): 2}
    assert out[3] == {(0, 0): 2, (0, 1): 4}
    assert tr.live[0].all() and tr.id[0].tolist() == [4, 2]
    # equal misses: the lower slot goes
    tr = Tracker(2, gate=8, max_missed=10)
    out = run(tr, [([A, B], []), ([], []), ([C], [])], 2)
    assert tr.id[0].tolist() == [4, 2]


def test_equal_distances_resolve_by_slot_then_row():
    # two slots at the same distance from one detection: the lower slot takes it
    tr = Tracker(2, gate=8)
    out = run(tr, [([cell(10, 10), cell(10, 14)], []), ([cell(10, 12)], [])], 2)
    assert out[1] == {(0, 0): 0}
    # one slot, two detections at the same distance: the earlier row (higher score) takes it, the other is born
    tr = Tracker(2, gate=8)
    out = run(tr, [([cell(10, 12)], []), ([cell(10, 10), cell(10, 14)], [])], 2)
    assert out[1] == {(0, 0): 0, (0, 1): 2}


def test_ids_even_left_odd_right_in_birth_order():
    frames = [([cell(1, 1)], [cell(60, 60)]), ([cell(1, 1), cell(30, 30)], [cell(60, 60), cell(2, 50)]),
              ([], [cell(60, 60), cell(2, 50), cell(40, 5)])]
    out = run(Tracker(4), frames, 4)
    assert out[1] == {(0, 0): 0, (0, 1): 2, (1, 0): 1, (1, 1): 3}
    assert out[2] == {(1, 0): 1, (1, 1): 3, (1, 2): 5}


def random_scene(seed, B, K, p_on=0.8):
    """Random-walk hands per side: births, deaths, occlusions and jumps; hands[b][s] = cells in a random rank order."""
    rng = np.random.default_rng(seed)
    hands = []
    pos = [[] for _ in range(2)]
    for _ in range(B):
        fr = []
        for s in range(2):
            if rng.random() < 0.1 and len(pos[s]) < K + 1:
                pos[s].append(rng.integers(0, 64, 2))
            if pos[s] and rng.random() < 0.05:
                pos[s].pop(int(rng.integers(len(pos[s]))))
            pos[s] = [np.clip(p + rng.integers(-3, 4, 2) + (rng.random() < 0.05) * rng.integers(-20, 21, 2), 0, 63)
                      for p in pos[s]]
            cells = sorted({int(p[0]) * 64 + int(p[1]) for p in pos[s] if rng.random() < p_on})
            rng.shuffle(cells)
            fr.append(cells[:K])
        hands.append(fr)
    return hands


@pytest.mark.parametrize("K", [1, 2, 4])
def test_batch_equals_single_frames(K):
    hands = random_scene(3 + K, 60, K)
    one, many = Tracker(K, gate=6, max_missed=3), Tracker(K, gate=6, max_missed=3)
    rows, det, _ = parse_rows(hands, K)
    ids, _ = many.step(rows, det, len(rows), len(hands))
    got = {}
    for b in range(len(hands)):
        r1, d1, _ = parse_rows([hands[b]], K)
        i1, _ = one.step(r1, d1, len(r1), 1)
        for r in range(len(r1)):
            if d1[r] > 0:
                got[(b, int(r1[r, 1]), int(r1[r, 2]))] = int(i1[r])
    want = {(int(rows[r, 0]), int(rows[r, 1]), int(rows[r, 2])): int(ids[r]) for r in range(len(rows)) if det[r] > 0}
    assert got == want and len(set(want.values())) > K
    for a in ("live", "id", "cell", "missed"):
        assert (getattr(one, a) == getattr(many, a)).all(), a


def test_malformed_rows_are_skipped():
    rows = np.array([[0, 0, 5, -1], [2, 0, 9, -1], [1, 0, 7, -1], [3, 0, 4096, -1], [5, 0, 3, -1], [2, 2, 3, -1],
                     [3, 1, 3, -1]], np.int32)
    det = np.ones(len(rows), np.float32)
    ids, _ = Tracker(2).step(rows, det, len(rows), 4)
    # image 1 after image 2: skipped; cell 4096 and image 5 >= B: skipped; side 2: no side; n_dev excludes the last
    assert ids.tolist()[:6] == [0, 0, -1, -1, -1, -1]
    ids, _ = Tracker(2).step(rows, det, 6, 4)
    assert ids[6] == -1


# ---------------------------------------------------------------------------------------------- reference anchor
def test_statement_reproduces_the_reference_filter_golden():
    """K = 1, gates open: the statement with the fp32 restatement of the reference's filter objects per track is the
    reference's per-hand-type smoothing (acr/main.py:69-83) on tests/golden/smooth_golden.npz."""
    g = np.load(os.path.join(GOLDEN, "smooth_golden.npz"))
    tr = Tracker(1, gate=GATE_OPEN, max_missed=NO_MISS_LIMIT, bank=lambda: rotation_ref.OneEuroBank(4.0))
    for t in range(g["poses"].shape[0]):
        rows = np.array([[0, 0, 0, -1], [0, 1, 0, -1]], np.int32)
        det = g["det"][t].astype(np.float32)
        ids, out = tr.step(rows, det, 2, 1, g["poses"][t], g["betas"][t])
        for h in range(2):
            if not det[h] > 0:
                assert ids[h] == -1
                continue
            assert ids[h] == h
            p, b = out[h][2]
            assert np.abs(p - g["out_poses"][t, h]).max() < 2e-5, (t, h)
            assert np.abs(b - g["out_betas"][t, h]).max() < 1e-6, (t, h)


# ------------------------------------------------------------------------------------------- the built library
def _lib():
    if not os.path.exists(LIB):
        pytest.skip("library not built")
    from acr_b200 import lib as L
    return L.load()


def test_abi_argument_checks():
    lib = _lib()
    from acr_b200 import lib as L
    assert {"acr_b200_track_state_bytes", "acr_b200_track_hands"} <= set(L.EXPORTS)
    assert lib.acr_b200_track_state_bytes(1) > 0 and lib.acr_b200_track_state_bytes(16) > lib.acr_b200_track_state_bytes(4)
    assert lib.acr_b200_track_state_bytes(0) == 0 and lib.acr_b200_track_state_bytes(17) == 0
    p = 4096   # never dereferenced: every call below fails its checks before any launch

    def call(poses=p, betas=p, rows=p, flag=p, n_max=8, B=1, K=4, gate=8, missed=15, coeff=4.0, state=p, ids=p):
        return lib.acr_b200_track_hands(poses, betas, rows, flag, None, n_max, B, K, gate, missed, coeff, state, ids,
                                        None)

    cases = [dict(K=0), dict(K=17), dict(B=0), dict(n_max=9), dict(n_max=-1), dict(gate=-1), dict(missed=-1),
             dict(state=None), dict(rows=None), dict(ids=None), dict(poses=None), dict(betas=None), dict(coeff=0.0),
             dict(coeff=-1.0), dict(coeff=float("nan"))]
    for kw in cases:
        assert call(**kw) == -1, kw                                  # ACR_B200_EINVAL
        assert b"track_hands" in lib.acr_b200_last_error(), kw
    assert b"smooth_coeff" in (call(coeff=0.0), lib.acr_b200_last_error())[1]
