"""CPU: the part-label statement (tests/part_labels_ref.py) and the host side of acr_b200_part_labels.

* the statement equals F.interpolate(bilinear, align_corners=False) + argmax on random logits, over up- and
  downsampling sides and portrait / landscape pads;
* the host packing rule (acr_b200.ops.part_label_layout) equals the statement's: prefix of H*W, invalid rows, capacity;
* PartLabels / part_labels reject what does not fit before anything is enqueued;
* the kernel compiles for sm_90a with no stack frame and no spills.
"""
import os
import re
import subprocess

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from acr_b200 import ops
from acr_b200.lib import AcrB200Error
from acr_b200.preprocess import offsets_vector
from tests import part_labels_ref as ref

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
PKG = os.path.join(ROOT, "arbitrary-hands-3d-reconstruction_b200")


def _torch_labels(segm, row):
    side, pad_t, pad_l, H, W = ref.frame_geometry(row)
    x = torch.from_numpy(np.ascontiguousarray(segm.transpose(2, 0, 1)))[None].double()
    up = F.interpolate(x, size=(side, side), mode="bilinear", align_corners=False)[0]
    return up.argmax(0)[pad_t:pad_t + H, pad_l:pad_l + W].numpy().astype(np.uint8)


@pytest.mark.parametrize("hw", [(1, 1), (17, 17), (255, 255), (256, 256), (257, 257), (300, 300), (1920, 1920),
                                (300, 200), (200, 300), (1080, 1920), (1920, 1080), (1, 17), (17, 1)])
def test_statement_equals_interpolate_and_argmax(hw):
    rng = np.random.default_rng(hw[0] * 7919 + hw[1])
    segm = rng.standard_normal((256, 256, 33))
    row = offsets_vector(*hw)
    got = ref.part_labels(segm, row)
    assert got.shape == hw
    assert np.array_equal(got, _torch_labels(segm, row))


def test_statement_ties_go_to_the_lowest_channel():
    segm = np.zeros((256, 256, 33))
    segm[..., 5] = segm[..., 9] = 1.0
    assert (ref.part_labels(segm, offsets_vector(40, 30)) == 5).all()
    assert (ref.part_labels(np.zeros((256, 256, 33)), offsets_vector(3, 3)) == 0).all()


def _rows():
    good = [offsets_vector(720, 1280), offsets_vector(1, 1), offsets_vector(4032, 3024), offsets_vector(5, 9)]
    bad = [np.array([10, 10, 0, 0, 0, 0, 0.5, 0, 0, 0], np.float32),      # non-integer
           np.array([10, 10, 0, 0, 0, 0, -1, 0, 0, 0], np.float32),       # negative
           np.array([10, 10, 0, 0, 0, 0, 4, 0, 6, 0], np.float32),        # pad_t + pad_b >= side
           np.array([10, 10, 0, 0, 0, 0, 0, 5, 0, 5], np.float32),        # pad_l + pad_r >= side
           np.array([10, 12, 0, 0, 0, 0, 0, 0, 0, 0], np.float32),        # unequal sides
           np.array([0, 0, 0, 0, 0, 0, 0, 0, 0, 0], np.float32),          # empty
           np.array([16385, 16385, 0, 0, 0, 0, 0, 0, 0, 0], np.float32),  # over the side limit
           np.array([np.nan, np.nan, 0, 0, 0, 0, 0, 0, 0, 0], np.float32),
           np.array([1e30, 1e30, 0, 0, 0, 0, 0, 0, 0, 0], np.float32)]
    return good, bad


def test_host_packing_equals_the_statement():
    good, bad = _rows()
    rng = np.random.default_rng(3)
    rows = np.stack([r for pair in zip(good + good, bad) for r in pair] + [np.array([16384, 16384] + [0] * 8)])
    rows = rows[rng.permutation(len(rows))].astype(np.float32)
    for cap in (0, 1, 720 * 1280, 720 * 1280 + 1, 10 ** 7, 10 ** 9):
        geo, flags, total = ops.part_label_layout(rows, cap)
        start, H, W, rflags = ref.packing(rows, cap)
        assert np.array_equal(geo[:, 0], start) and np.array_equal(geo[:, 1], H) and np.array_equal(geo[:, 2], W)
        assert np.array_equal(flags, rflags), cap
        assert total == int((H * W).sum())
    assert ref.frame_geometry(np.array([16384, 16384] + [0] * 8)) == (16384, 0, 0, 16384, 16384)
    for r in bad:
        assert ref.frame_geometry(r) is None, r


def test_ragged_packing_is_the_bgr_packing_divided_by_three():
    from acr_b200.preprocess import shapes_layout
    shapes = [(720, 1280), (1, 1), (3024, 4032), (1080, 1920), (7, 1)]
    desc, offsets, total = shapes_layout(shapes)
    geo, flags, n = ops.part_label_layout(offsets, total // 3)
    assert not flags.any() and n == total // 3
    assert np.array_equal(geo[:, 0] * 3, desc["offset"])
    assert [tuple(g) for g in geo[:, 1:]] == shapes


def test_capacity_overflow_raises_before_launch():
    # the host checks come before anything touches a device, so they run here on CPU tensors
    segms = torch.zeros(2, 256, 256, 48, dtype=torch.bfloat16)
    offs = torch.from_numpy(np.stack([offsets_vector(10, 10), offsets_vector(10, 10)]))
    with pytest.raises(ValueError, match="over the capacity"):
        ops.part_labels(segms, offs, ops.PartLabels(199, 2, "cpu"))
    with pytest.raises(ValueError, match="exceed"):
        ops.part_labels(segms, offs, ops.PartLabels(200, 1, "cpu"))
    with pytest.raises(ValueError, match="NHWC"):
        ops.part_labels(segms.permute(0, 3, 1, 2), offs, ops.PartLabels(200, 2, "cpu"))
    with pytest.raises(ValueError):
        ops.PartLabels(-1, 1, "cpu")
    with pytest.raises(AcrB200Error):              # a fitting batch reaches the device check
        ops.part_labels(segms, offs, ops.PartLabels(200, 2, "cpu"))


def test_kernel_has_no_stack_or_spills(tmp_path):
    nvcc = "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("no nvcc")
    src = os.path.join(PKG, "csrc", "part_labels.cu")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-I",
                        os.path.join(ROOT, "include"), "--expt-relaxed-constexpr", "-Xptxas", "-v", "-c", src, "-o",
                        str(tmp_path / "part_labels.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    props = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    kernels = re.findall(r"Compiling entry function '(\S+)' for 'sm_90a'", r.stderr)
    assert len(kernels) == 4 and len(props) == 4, r.stderr        # the prefix and three map dtypes
    assert all(p == ("0", "0", "0") for p in props), r.stderr
