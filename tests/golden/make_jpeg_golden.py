#!/usr/bin/env python
"""Generate jpeg_pillow_golden.npz: JPEG files written by Pillow's encoder, which makes choices cv2.imencode does not
(SOF1 with 16-bit quantisation tables, restart intervals in MCU rows or blocks, EXIF, an ICC profile split over
several APP2 segments, COM, optimised Huffman tables, an RGB file).  The files are committed as data, so the tests
need no Pillow; tests/test_cpu_jpeg_conformance.py and tests/test_gpu_jpeg_conformance.py read them.

    python tests/golden/make_jpeg_golden.py      # writes jpeg_pillow_golden.npz next to this file

Each key is a file name; each value is the file's bytes as a uint8 array."""
import io
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.abspath(os.path.join(HERE, "..", ".."))
sys.path.insert(0, ROOT)

from tests import jpeg_cases as JC  # noqa: E402

EXIF_ORIENTATION_1 = (b"Exif\x00\x00MM\x00\x2a\x00\x00\x00\x08\x00\x01\x01\x12\x00\x03\x00\x00\x00\x01\x00\x01\x00\x00"
                      b"\x00\x00\x00\x00")


def content(h, w, seed):
    """Smooth gradients plus seeded noise, RGB (Pillow's order)."""
    rng = np.random.default_rng(seed)
    img = JC.image(h, w, "smooth").astype(np.int32) + rng.integers(-24, 25, (h, w, 3))
    return np.clip(img, 0, 255).astype(np.uint8)[:, :, ::-1].copy()


def cases():
    """name -> (height, width, Pillow save arguments)."""
    big_q = [[min(1 + 7 * k, 255) for k in range(64)], [min(200 + 13 * k, 1000) for k in range(64)]]
    icc = bytes(np.random.default_rng(1).integers(0, 256, 70000, dtype=np.uint8))
    return {
        "sof1_q16_420": (61, 83, dict(qtables=big_q, subsampling=2)),
        "sof1_q16_444": (40, 56, dict(qtables=big_q, subsampling=0)),
        "rst_rows_420": (77, 130, dict(quality=90, restart_marker_rows=1, subsampling=2)),
        "rst_blocks7_422": (50, 141, dict(quality=90, restart_marker_blocks=7, subsampling=1)),
        "exif_420": (45, 64, dict(quality=85, exif=EXIF_ORIENTATION_1)),
        "icc_app2x2_444": (24, 40, dict(quality=80, icc_profile=icc, subsampling=0)),
        "comment_optimize_444": (70, 49, dict(quality=95, optimize=True, subsampling=0, comment=b"a comment")),
        "optimize_422": (33, 95, dict(quality=75, optimize=True, subsampling=1)),
        "optimize_420": (96, 72, dict(quality=60, optimize=True, subsampling=2)),
        "rgb_keep_rgb": (21, 34, dict(quality=90, keep_rgb=True, subsampling=0)),
    }


def main():
    from PIL import Image
    out = {}
    for k, (name, (h, w, kw)) in enumerate(cases().items()):
        bio = io.BytesIO()
        Image.fromarray(content(h, w, k)).save(bio, "JPEG", **kw)
        out[name] = np.frombuffer(bio.getvalue(), np.uint8)
    path = os.path.join(HERE, "jpeg_pillow_golden.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes,", len(out), "files")


if __name__ == "__main__":
    main()
