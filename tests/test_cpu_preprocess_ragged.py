"""CPU: the ragged pre-processing's host side -- packing, descriptors, offsets vectors and the input checks that
must fire before anything is launched."""
import re

import numpy as np
import pytest
import torch

from acr_b200 import lib as L
from acr_b200.preprocess import (FRAME_DTYPE, check_ragged, offsets_vector, paddings_to_square, preprocess_frames,
                                 ragged_layout)

SHAPES = [(360, 640), (640, 360), (600, 600), (1, 1), (1, 7), (7, 1), (513, 511)]


def _frames(shapes, seed=0):
    rng = np.random.default_rng(seed)
    return [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for h, w in shapes]


def test_frame_descriptor_matches_the_c_struct():
    """FRAME_DTYPE is acr_b200_frame of include/acr_b200.h: int64 offset, then six int32, 32 bytes."""
    import os
    hdr = open(os.path.join(os.path.dirname(__file__), "..", "include", "acr_b200.h")).read()
    body = re.search(r"typedef struct acr_b200_frame \{(.*?)\} acr_b200_frame;", hdr, re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    fields = []
    for decl in body.split(";"):
        decl = decl.strip()
        if decl:
            ctype, names = decl.split(None, 1)
            fields += [(n.strip(), ctype) for n in names.split(",")]
    size = {"int64_t": 8, "int32_t": 4}
    assert [n for n, _ in fields] == list(FRAME_DTYPE.names)
    pos = 0
    for n, ctype in fields:
        assert FRAME_DTYPE.fields[n][1] == pos and FRAME_DTYPE.fields[n][0].itemsize == size[ctype], n
        pos += size[ctype]
    assert FRAME_DTYPE.itemsize == pos == 32


def test_layout_offsets_and_descriptors():
    frames = _frames(SHAPES)
    desc, offsets, total = ragged_layout(frames)
    sizes = [h * w * 3 for h, w in SHAPES]
    assert desc["offset"].tolist() == np.concatenate([[0], np.cumsum(sizes)[:-1]]).tolist()
    assert total == sum(sizes)
    for i, (h, w) in enumerate(SHAPES):
        t, r, b, l = paddings_to_square(h, w)
        assert (desc[i]["H"], desc[i]["W"], desc[i]["side"], desc[i]["pad_t"], desc[i]["pad_l"]) == (h, w, max(h, w), t, l)
        assert desc[i]["reserved"] == 0
        assert np.array_equal(offsets[i], offsets_vector(h, w))
        # the vector the kernel writes from the descriptor: [side, side, 0,0,0,0, t, side-W-l, side-H-t, l]
        s = max(h, w)
        assert offsets[i].tolist() == [s, s, 0, 0, 0, 0, t, s - w - l, s - h - t, l]
    assert offsets.dtype == np.float32


def test_layout_accepts_every_host_form():
    """numpy, CPU tensors and non-contiguous views give the same layout."""
    frames = _frames(SHAPES[:3])
    views = [np.ascontiguousarray(f.transpose(1, 0, 2)).transpose(1, 0, 2) for f in frames]
    assert not views[0].flags.c_contiguous
    ref = ragged_layout(frames)
    for alt in ([torch.from_numpy(f) for f in frames], views, [torch.from_numpy(v) for v in views]):
        got = ragged_layout(alt)
        assert np.array_equal(got[0], ref[0]) and np.array_equal(got[1], ref[1]) and got[2] == ref[2]


@pytest.fixture
def no_launch(monkeypatch):
    """Any attempt to reach the library fails the test: the checks must come first."""
    def refuse(*a, **k):
        raise AssertionError("the library was reached before the input was rejected")
    monkeypatch.setattr(L, "load", refuse)


@pytest.mark.parametrize("frames, exc", [
    ([], ValueError),
    ([np.zeros((4, 4, 3), np.float32)], TypeError),
    ([np.zeros((4, 4, 3), np.uint8), torch.zeros(4, 4, 3, dtype=torch.int16)], TypeError),
    ([np.zeros((4, 4, 4), np.uint8)], ValueError),
    ([np.zeros((4, 4), np.uint8)], ValueError),
    ([np.zeros((0, 4, 3), np.uint8)], ValueError),
    ([np.zeros((4, 0, 3), np.uint8)], ValueError),
    ([[[[0, 0, 0]]]], TypeError),
], ids=["empty", "float", "int16", "4-channels", "2-d", "zero-rows", "zero-cols", "nested-list"])
def test_bad_frames_are_rejected_before_launch(no_launch, frames, exc):
    with pytest.raises(exc):
        preprocess_frames(frames)
    from acr.utils import img_preprocess
    with pytest.raises(exc):
        img_preprocess(frames)


def test_path_count_is_checked_before_launch(no_launch):
    from acr.utils import img_preprocess
    with pytest.raises(ValueError):
        img_preprocess(_frames([(4, 4), (5, 6)]), ["a.jpg"])


def test_capacity_checks():
    frames = _frames([(10, 20), (30, 5)])
    total = 10 * 20 * 3 + 30 * 5 * 3
    desc, offsets, n_bytes, host = check_ragged(frames, 2, total, exact=True)
    assert n_bytes == total and host
    with pytest.raises(ValueError, match="bytes"):
        check_ragged(frames, 2, total - 1)
    with pytest.raises(ValueError, match="exceed"):
        check_ragged(frames, 1, 10 ** 6)
    for n in (1, 3):           # the graph form takes exactly its batch
        with pytest.raises(ValueError, match="exactly"):
            check_ragged(_frames([(4, 4)] * n), 2, 10 ** 6, exact=True)
    check_ragged(_frames([(4, 4)]), 2, 10 ** 6)        # the eager form takes fewer
