"""numpy statement of multi-hand tracking (acr_b200_track_hands): per-track identities and one OneEuro bank per track
for up to K hands per side, over a batch of B consecutive frames of one stream.

Rows come in the parse's layout and order: ``row_src`` (n,4) = image, side, flat centre cell y*64+x on the 64x64
centre map, and a fourth column the tracker does not read; side-major, then image-major, then by rank (descending
score).  Each side is tracked on its own, in K slots.  A live slot holds its id, the cell of its last matched
detection, its count of consecutive missed frames and a 64-element OneEuro bank (45 pose values, 10 betas, 9 root-
matrix entries: the quantities of the reference's smooth_results).

Which rows are detections.  Walking the rows [0, min(n_dev, n_max)) of one side in table order, a row is skipped
(track id -1, left untouched) when its image is outside [0, B), its cell outside [0, 4096), or its image below that of
the last row kept before it; a kept row is a detection when detection_flag > 0, up to K per image (a further one is
skipped too; the parse never writes more).  Rows of no side, and rows at or past n_dev, get -1 as well.

Per frame b = 0..B-1 and side s, in this order:
  1. Match: the pairs (live slot k, detection r) with integer squared cell distance d2 <= gate^2; repeatedly take the
     smallest by (d2, k, r) -- a total order -- and drop its slot and row from further matching.
  2. Miss: a live slot left unmatched counts one more missed frame and is freed once that count exceeds max_missed
     (its id is never reused); a matched slot's count returns to 0 and its cell becomes the detection's.
  3. Birth: unmatched detections in row order each take the lowest free slot, or, with none free, evict the live
     slot not matched (nor born) in this frame with the most misses, ties to the lower slot.  One always exists:
     unmatched detections <= K - matched slots.
  4. A new track's id is 2 c_s + s with a per-side birth counter c_s: even ids on the left, odd on the right.
A frame with no detection of a side still runs steps 2 (every live slot misses).  gate >= 90 never rejects a pair
(63^2 + 63^2 < 90^2).

Filtering: each detection with a track goes through its track's bank with the reference's OneEuroFilter
(acr/utils.py:1485-1527, te = 1/30 whatever the gap).  A newborn track's first frame passes the pose's 45 values and
the betas through; the root, as every frame's, is the filtered matrix taken back to an axis angle (for a first frame
the Rodrigues round trip of the input, as the reference's filter returns a first frame unchanged).  Frames without a
detection leave the bank untouched.  A zeroed state is no tracks and both counters at zero.
"""
import numpy as np

GATE_OPEN = 90                 # never rejects a pair on the 64x64 map
NO_MISS_LIMIT = 2 ** 31 - 1    # a track is never freed for missing frames
NCELL = 64 * 64


def cell_d2(a, b):
    dy, dx = a // 64 - b // 64, a % 64 - b % 64
    return int(dy * dy + dx * dx)


class Tracker:
    """The state of one stream (both sides).  ``bank`` is a factory of filter banks with ``process(pose48, betas10)``
    (tests.tail_ref.OneEuro64 or oracle.rotation_ref.OneEuroBank), or None for ids only."""

    def __init__(self, K, gate=8, max_missed=15, bank=None):
        self.K, self.gate, self.max_missed, self.bank = int(K), int(gate), int(max_missed), bank
        self.reset()

    def reset(self):
        K = self.K
        self.live = np.zeros((2, K), bool)
        self.id = np.zeros((2, K), np.int64)
        self.cell = np.zeros((2, K), np.int64)
        self.missed = np.zeros((2, K), np.int64)
        self.banks = [[None] * K for _ in range(2)]
        self.births = [0, 0]

    def detections(self, row_src, det, n_dev, B):
        """-> frames[s][b] = detection rows of side s in image b (row order)."""
        row_src = np.asarray(row_src).reshape(-1, 4)
        n = max(0, min(int(n_dev), row_src.shape[0]))
        frames = [[[] for _ in range(B)] for _ in range(2)]
        last = [0, 0]
        for r in range(n):
            img, s, c = (int(v) for v in row_src[r, :3])
            if s not in (0, 1) or not (0 <= img < B and 0 <= c < NCELL) or img < last[s]:
                continue
            last[s] = img
            if det[r] > 0 and len(frames[s][img]) < self.K:
                frames[s][img].append(r)
        return frames

    def step(self, row_src, det, n_dev, B, poses=None, betas=None):
        """One call over B frames.  -> (ids (n_max,) int64, out): out[r] = (track id, born, bank result or None) for
        every tracked row r, in the order the rows were filtered."""
        row_src = np.asarray(row_src).reshape(-1, 4)
        det = np.asarray(det)
        ids = np.full(row_src.shape[0], -1, np.int64)
        out = {}
        frames = self.detections(row_src, det, n_dev, B)
        for b in range(B):
            for s in (0, 1):
                self._frame(s, frames[s][b], row_src, ids, out, poses, betas)
        return ids, out

    def _frame(self, s, rows, row_src, ids, out, poses, betas):
        K, g2 = self.K, self.gate * self.gate
        live, cell, missed = self.live[s], self.cell[s], self.missed[s]
        cells = {r: int(row_src[r, 2]) for r in rows}
        pairs = sorted((cell_d2(cell[k], cells[r]), k, r) for k in range(K) if live[k] for r in rows
                       if cell_d2(cell[k], cells[r]) <= g2)
        slot_of, matched = {}, set()
        for _, k, r in pairs:
            if k not in matched and r not in slot_of:
                matched.add(k)
                slot_of[r] = k
        for k in range(K):
            if not live[k]:
                continue
            if k in matched:
                missed[k] = 0
            else:
                missed[k] += 1
                if missed[k] > self.max_missed:
                    live[k] = False
        for r in rows:
            if r in slot_of:
                cell[slot_of[r]] = cells[r]
        born = set()
        for r in rows:
            if r in slot_of:
                continue
            free = [k for k in range(K) if not live[k]]
            if free:
                k = free[0]
            else:
                cand = [k for k in range(K) if k not in matched and k not in born]
                assert cand, "no slot to evict: more detections than slots"
                k = max(cand, key=lambda j: (missed[j], -j))
            live[k], cell[k], missed[k] = True, cells[r], 0
            self.id[s, k] = 2 * self.births[s] + s
            self.births[s] += 1
            self.banks[s][k] = self.bank() if self.bank is not None else None
            born.add(k)
            slot_of[r] = k
        for r in rows:
            k = slot_of[r]
            ids[r] = self.id[s, k]
            res = None
            if self.bank is not None and poses is not None:
                res = self.banks[s][k].process(poses[r], betas[r])
            out[r] = (int(self.id[s, k]), k in born, res)


def parse_rows(hands, K):
    """Row table of one batch in the parse's layout from ``hands[b][s]`` = cells of image b and side s in rank
    order (at most K): -> row_src (n,4) int32, detection flag (n,) float32, and the (L, R) row counts.  A side with
    no hand in the whole batch gets the parse's dummy row (image 0, cell 0, flag 0)."""
    rows, flags, counts = [], [], []
    for s in (0, 1):
        mine = [(b, c) for b in range(len(hands)) for c in hands[b][s][:K]]
        if not mine:
            rows.append((0, s, 0, -1)); flags.append(0.0)
        for b, c in mine:
            rows.append((b, s, c, -1)); flags.append(1.0)
        counts.append(max(len(mine), 1))
    return np.asarray(rows, np.int32), np.asarray(flags, np.float32), tuple(counts)
