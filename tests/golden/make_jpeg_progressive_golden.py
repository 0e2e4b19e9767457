#!/usr/bin/env python
"""Generate jpeg_progressive_sources.npz: the baseline cv2 files that tests/test_cpu_jpeg_progressive_sweep.py codes
again with tests/jpeg_progressive_writer.py to check that the writer's existing output stays byte for byte the
same.  The sources are committed as data, so that check does not depend on the installed cv2's encoder.

    python tests/golden/make_jpeg_progressive_golden.py      # writes jpeg_progressive_sources.npz next to this file

Keys: ``src-{h}x{w}-{sampling}``; each value is the file's bytes as a uint8 array."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.abspath(os.path.join(HERE, "..", ".."))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "arbitrary-hands-3d-reconstruction_b200"))

from tests import jpeg_cases as JC  # noqa: E402

WRITER = [(45, 83, s) for s in ("420", "422", "444", "440", "grey")]     # the script files' sources
MULTI = [(37, 53, s) for s in ("444", "422", "420", "440")]             # the multi-scan sequential files' sources


def main():
    out = {f"src-{h}x{w}-{s}": np.frombuffer(JC.encode(h, w, 90, s, 0, "noisy"), np.uint8) for h, w, s in WRITER + MULTI}
    np.savez_compressed(os.path.join(HERE, "jpeg_progressive_sources.npz"), **out)
    print({k: v.size for k, v in out.items()})


if __name__ == "__main__":
    main()
