"""numpy statement of multi-hand tracking over several streams in one batch (acr_b200_track_streams), built on the
single-stream statement tests/track_ref.py.

``frame_stream`` (B,) gives the stream slot of each image of the batch, in 0..S-1; the images of one stream are its
frames in time order, in ascending batch index.  For each stream s, the call is tests.track_ref.Tracker.step on s's
frames alone with s's own state: the row table restricted to the rows whose image is one of s's (rows [0, n_dev) only,
in their original order), with images renumbered 0..B_s-1 in batch order.  Every other row -- at or past n_dev, image
outside [0, B), or an image whose stream is outside 0..S-1 -- gets id -1 and is left untouched.  A nonzero
``frame_begin`` entry starts the frame's stream over (a fresh state, as HandTracker.reset()) just before that frame:
the stream's frames are then stepped in pieces, split before each begin flag.  Which rows are detections is decided
once over the stream's rows of the whole call, as one single-stream call decides it over its table (so a row out of
time order stays skipped even when the frame it went back behind lies in a later piece); a begin flag resets the
tracks, not that.  On the parse's tables, whose rows are in time order, the two readings agree.
"""
import numpy as np

from tests.track_ref import Tracker


class StreamTracker:
    """S single-stream trackers; ``step`` takes a whole batch of interleaved streams."""

    def __init__(self, S, K, gate=8, max_missed=15, bank=None):
        self.S, self.K = int(S), int(K)
        self.args = dict(gate=gate, max_missed=max_missed, bank=bank)
        self.streams = [Tracker(K, **self.args) for _ in range(self.S)]

    def reset(self):
        for t in self.streams:
            t.reset()

    def step(self, row_src, det, n_dev, frame_stream, frame_begin=None, poses=None, betas=None):
        """-> (ids (n_max,) int64, out): out[r] = (stream, track id, born, bank result or None) per tracked row r."""
        row_src = np.asarray(row_src).reshape(-1, 4)
        det = np.asarray(det)
        frame_stream = np.asarray(frame_stream).astype(np.int64)
        B = len(frame_stream)
        begin = np.zeros(B, bool) if frame_begin is None else np.asarray(frame_begin) != 0
        n = max(0, min(int(n_dev), row_src.shape[0]))
        ids = np.full(row_src.shape[0], -1, np.int64)
        out = {}
        for s in range(self.S):
            frames = np.flatnonzero(frame_stream == s)           # s's frames in time order
            if not len(frames):
                continue
            rows, dets = stream_detections(row_src, det, n, frames, self.K)
            # pieces between begin flags: a begin flag on frame i starts a fresh state before it
            cuts = [i for i in range(len(frames)) if begin[frames[i]]]
            bounds = sorted(set([0] + cuts + [len(frames)]))
            for a, b in zip(bounds[:-1], bounds[1:]):
                if a in cuts:
                    self.streams[s].reset()
                local = {int(f): i for i, f in enumerate(frames[a:b])}
                sel = [r for r in dets if int(row_src[r, 0]) in local]
                sub = row_src[sel].copy().reshape(-1, 4)           # no row: every frame still runs (misses)
                sub[:, 0] = [local[int(i)] for i in sub[:, 0]]
                p = None if poses is None else np.asarray(poses)[sel]
                bt = None if betas is None else np.asarray(betas)[sel]
                sid, sout = self.streams[s].step(sub, det[sel], len(sel), b - a, p, bt)
                for i, r in enumerate(sel):
                    ids[r] = sid[i]
                    if i in sout:
                        tid, born, res = sout[i]
                        out[r] = (s, tid, born, res)
        return ids, out


def stream_detections(row_src, det, n, frames, K):
    """The rows [0, n) of the images ``frames`` (one stream's, in time order) in table order, and those of them that
    are detections of that stream's single-stream call over its whole table (tests.track_ref.Tracker.detections)."""
    local = {int(f): i for i, f in enumerate(frames)}
    rows = [r for r in range(n) if int(row_src[r, 0]) in local]
    sub = row_src[rows].copy().reshape(-1, 4)
    sub[:, 0] = [local[int(i)] for i in sub[:, 0]]
    per = Tracker(K).detections(sub, np.asarray(det)[rows], len(rows), len(frames))
    return rows, sorted(rows[i] for side in per for img in side for i in img)


def interleave(rng, lengths, begins=()):
    """A random interleaving of streams with the given frame counts: -> frame_stream (B,) and, per stream, its
    frames' batch indices in time order.  ``begins``: (stream, frame number) pairs to flag."""
    order = np.concatenate([np.full(n, s) for s, n in enumerate(lengths)]).astype(np.int32)
    rng.shuffle(order)
    frames = [np.flatnonzero(order == s) for s in range(len(lengths))]
    begin = np.zeros(len(order), np.int32)
    for s, i in begins:
        begin[frames[s][i]] = 1
    return order, frames, begin

