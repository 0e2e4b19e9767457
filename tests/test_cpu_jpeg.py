"""CPU: the JPEG header parser (acr_b200.jpeg) and the numpy decode statement (oracle/jpeg_ref.py).

* the parser reads every file of the test matrix (tests/jpeg_cases.py) and lays the batch out consistently;
* the oracle equals cv2.imdecode with array_equal (every small file, the large smooth files and a noisy sample);
* progressive, 4:1:1 and 12-bit files are rejected with the feature named; truncated files raise;
* a file with a JPEG appended after its EOI decodes as its first image, like cv2; over-long scans are rejected;
* bit-flipped files give an image of the right shape or JpegError;
* the jpeg kernels in the built library touch no local memory.
"""
import os
import sys

import numpy as np
import pytest

from acr_b200 import jpeg
from oracle import jpeg_ref
from tests import jpeg_cases as JC

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
SMALL = JC.SIZES[:3]
LARGE = JC.SIZES[3:]


def test_parser_reads_every_file_of_the_matrix():
    for case in JC.matrix():
        h, w, q, s, r, c = case
        info = jpeg.parse(JC.encode(*case))
        assert (info.H, info.W, info.ncomp, info.restart) == (h, w, 1 if s == "grey" else 3, r), case
        if s != "grey":
            assert (info.hmax, info.vmax) == {"444": (1, 1), "422": (2, 1), "420": (2, 2), "440": (1, 2)}[s], case
        assert info.n_blocks == info.mcus_x * info.mcus_y * info.bpm


def test_batch_layout_packs_files_back_to_back():
    cases = JC.matrix(SMALL)[:40]
    bufs = [JC.encode(*c) for c in cases]
    lay = jpeg.layout(bufs)
    infos = [jpeg.parse(b) for b in bufs]
    assert lay.coded_bytes == sum(i.scan_len for i in infos)
    assert lay.out_bytes == sum(i.H * i.W * 3 for i in infos)
    assert lay.chunks == sum(i.n_chunks for i in infos) and lay.blocks == sum(i.n_blocks for i in infos)
    d = lay.desc
    assert np.array_equal(d["coded_offset"][1:], np.cumsum(d["coded_len"])[:-1])
    assert np.array_equal(d["chunk_begin"][1:], np.cumsum(d["n_chunks"])[:-1])
    assert np.array_equal(d["block_begin"], d["coef_offset"])


@pytest.mark.parametrize("case", JC.matrix(SMALL), ids=lambda c: "-".join(map(str, c)))
def test_oracle_equals_cv2_small(case):
    buf = JC.encode(*case)
    assert np.array_equal(jpeg_ref.decode(buf), JC.cv2_decode(buf))


@pytest.mark.parametrize("case", [c for c in JC.matrix(LARGE) if c[5] == "smooth" or (c[2] == 50 and c[4] == 0)],
                         ids=lambda c: "-".join(map(str, c)))
def test_oracle_equals_cv2_large(case):
    buf = JC.encode(*case)
    assert np.array_equal(jpeg_ref.decode(buf), JC.cv2_decode(buf))


def test_unsupported_streams_are_rejected_with_the_feature_named():
    import cv2
    with pytest.raises(jpeg.JpegUnsupported, match="progressive"):
        jpeg.parse(JC.encode(17, 9, 90, "420", 0, "smooth", progressive=True))
    img = JC.image(16, 32, "smooth")
    ok, buf = cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_411])
    with pytest.raises(jpeg.JpegUnsupported, match="sampling factors 4x1"):
        jpeg.parse(buf.tobytes())
    b = bytearray(JC.encode(7, 13, 90, "444", 0, "smooth"))
    sof = b.find(b"\xff\xc0")
    b[sof + 4] = 12                                   # SOF sample precision
    with pytest.raises(jpeg.JpegUnsupported, match="12-bit"):
        jpeg.parse(bytes(b))
    with pytest.raises(jpeg.JpegUnsupported, match="file 1: progressive"):
        jpeg.layout([JC.encode(7, 13, 90, "444", 0, "smooth"), JC.encode(7, 13, 90, "444", 0, "smooth", True)])


def test_exif_orientation_other_than_one_is_rejected():
    base = JC.encode(7, 13, 90, "444", 0, "smooth")
    for o, ok in ((1, True), (6, False)):
        tiff = b"MM\x00\x2a\x00\x00\x00\x08" + b"\x00\x01" + b"\x01\x12\x00\x03\x00\x00\x00\x01" + bytes([0, o, 0, 0]) \
            + b"\x00\x00\x00\x00"
        app1 = b"Exif\x00\x00" + tiff
        f = base[:2] + b"\xff\xe1" + (len(app1) + 2).to_bytes(2, "big") + app1 + base[2:]
        if ok:
            assert jpeg.parse(f).W == 13
        else:
            with pytest.raises(jpeg.JpegUnsupported, match="EXIF orientation 6"):
                jpeg.parse(f)


def test_data_after_the_first_eoi_is_ignored():
    """A second JPEG appended after the EOI (an MPF preview, a motion-photo trailer) is not part of the scan."""
    first = JC.encode(17, 9, 90, "420", 0, "smooth")
    f = first + JC.encode(7, 13, 90, "444", 4, "noisy")
    assert jpeg.parse(f).scan_len == jpeg.parse(first).scan_len
    assert np.array_equal(jpeg_ref.decode(f), JC.cv2_decode(f))
    assert np.array_equal(JC.cv2_decode(f), JC.cv2_decode(first))


def test_scans_past_the_position_range_are_rejected(monkeypatch):
    buf = JC.encode(17, 9, 90, "420", 0, "noisy")
    n = jpeg.parse(buf).scan_len
    monkeypatch.setattr(jpeg, "MAX_SCAN_BYTES", n)
    with pytest.raises(jpeg.JpegUnsupported, match="entropy-coded segment"):
        jpeg.parse(buf)
    monkeypatch.setattr(jpeg, "MAX_SCAN_BYTES", n + 1)
    assert jpeg.parse(buf).scan_len == n


def test_truncated_files_raise():
    good = JC.encode(720, 1280, 90, "420", 0, "noisy")
    info = jpeg.parse(good)
    for cut in (10, info.scan_offset - 5):            # inside the headers: the parser raises
        with pytest.raises(jpeg.JpegError):
            jpeg.parse(good[:cut])
    with pytest.raises(jpeg.JpegError, match="EOI"):
        jpeg.parse(good[:info.scan_offset + 1000])
    for cut in (info.scan_offset + info.scan_len // 3, info.scan_offset + info.scan_len - 40):
        with pytest.raises(jpeg.JpegError):           # inside the scan: the entropy decode raises
            jpeg_ref.decode(good[:cut] + b"\xff\xd9")


def test_bit_flipped_files_give_an_image_or_the_error():
    rng = np.random.default_rng(5)
    for case in [(17, 9, 100, "444", 0, "noisy"), (7, 13, 90, "420", 1, "noisy"), (17, 9, 50, "grey", 4, "smooth")]:
        b = JC.encode(*case)
        info = jpeg.parse(b)
        for _ in range(20):
            a = bytearray(b)
            p = info.scan_offset + int(rng.integers(0, info.scan_len))
            a[p] ^= 1 << int(rng.integers(0, 8))
            try:
                assert jpeg_ref.decode(bytes(a)).shape == (info.H, info.W, 3)
            except jpeg.JpegError:
                pass


def test_jpeg_kernels_do_not_touch_local_memory():
    lib = os.path.join(ROOT, "arbitrary-hands-3d-reconstruction_b200", "lib", "libacr_b200.so")
    if not (os.path.exists(lib) and os.path.exists("/usr/local/cuda/bin/cuobjdump")):
        pytest.skip("library not built or no cuobjdump")
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    try:
        import sass_audit
        rows = sass_audit.audit(lib)
    finally:
        sys.path.pop(0)
    names = {"jpeg_spec_kernel", "jpeg_sync_kernel", "jpeg_write_kernel", "jpeg_idct_kernel", "jpeg_color_kernel"}
    found = {n: r for n, r in rows.items() if n in names}
    assert set(found) == names, sorted(rows)[:10]
    for n, r in found.items():
        assert r["LDL"] == 0 and r["STL"] == 0, f"{n}: {r['LDL']} LDL / {r['STL']} STL"
