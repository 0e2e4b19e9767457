"""CPU: progressive and multi-scan sequential JPEG files in the header parser (acr_b200.jpeg, ``max_scans``) and the
numpy statement of their decode (tests/jpeg_progressive_ref.py).

* the statement equals cv2.imdecode on cv2 progressive files (with and without RST), on Pillow progressive files
  (optimised tables: a DHT before every scan) and on multi-scan sequential files;
* with ``max_scans = 0`` those files raise as before; single-scan files parse the same with any ``max_scans``;
* one-component scans cover the component's own blocks; scan segments end at the next non-RST marker;
* invalid scripts raise JpegError, scripts the device does not decode raise JpegUnsupported, including an
  incomplete script, whose cv2 output (libjpeg's block smoothing) differs from the plain IDCT;
* the batch cap on scans raises ValueError; the multi-scan kernels touch no local memory;
* the progressive script writer (tests/jpeg_progressive_writer.py): per-component and interleaved DC, spectral
  selection only, successive approximation four bits deep, one-coefficient bands (over 64 scans per component),
  components alternating in file order, DRI changing between scans, per-scan optimal and all-long tables, and an
  EOB run of 32767 blocks; its files equal cv2 and the source file's pixels, and put EOB runs, correction bits,
  RST markers and stuffed FF 00 across 256-byte chunk boundaries.
"""
import os
import sys

import numpy as np
import pytest

from acr_b200 import jpeg
from tests import jpeg_cases as JC
from tests import jpeg_progressive_ref as PR
from tests import jpeg_progressive_writer as PW

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
SMALL = [(1, 1), (7, 13), (17, 9), (37, 53)]
BIG = 64


def _scan_list(b):
    """[(SOS start, segment end)] of a multi-scan file."""
    info = jpeg.parse(b, BIG)
    out = []
    for s in info.scans:
        sos = b.rfind(b"\xff\xda", 0, s.offset)
        out.append((sos, s.offset + s.length))
    return info, out


def _with_scans(b, order):
    """The file with its scans in ``order`` (indices, repeats allowed), each with the table and DRI segments before
    its SOS."""
    _, sc = _scan_list(b)
    starts = [sc[0][0]] + [end for _, end in sc[:-1]]
    return b[:sc[0][0]] + b"".join(b[starts[k]:sc[k][1]] for k in order) + b"\xff\xd9"


def _patch_sos(b, k, ss=None, se=None, ah=None, al=None):
    _, sc = _scan_list(b)
    a = bytearray(b)
    p = sc[k][0]
    ns = a[p + 4]
    q = p + 5 + 2 * ns
    if ss is not None:
        a[q] = ss
    if se is not None:
        a[q + 1] = se
    if ah is not None or al is not None:
        a[q + 2] = ((a[q + 2] >> 4 if ah is None else ah) << 4) | ((a[q + 2] & 15) if al is None else al)
    return bytes(a)


@pytest.mark.parametrize("size", SMALL, ids=lambda s: f"{s[0]}x{s[1]}")
def test_statement_equals_cv2_on_cv2_progressive_files(size):
    bad = []
    for q in JC.QUALITIES:
        for s in JC.SAMPLINGS:
            for r in (0, 1, 3):
                b = PW.cv2_progressive(*size, q, s, r)
                if not np.array_equal(PR.decode(b), JC.cv2_decode(b)):
                    bad.append((q, s, r))
    assert not bad


def test_statement_equals_cv2_on_a_large_progressive_file():
    for s, r in (("420", 0), ("444", 4)):
        b = PW.cv2_progressive(240, 320, 90, s, r, "smooth")
        assert np.array_equal(PR.decode(b), JC.cv2_decode(b))


def test_statement_equals_cv2_on_pillow_progressive_files():
    for sub in (0, 1, 2):
        for q in (50, 95):
            b = PW.pillow_progressive(45, 83, q, sub)
            info = jpeg.parse(b, BIG)
            assert b.count(b"\xff\xc4") >= len(info.scans) - 1    # tables redefined between scans
            assert np.array_equal(PR.decode(b), JC.cv2_decode(b)), (sub, q)


MULTI = [([[0], [1], [2]], ()), ([[0], [1, 2]], (3, 0)), ([[2], [0, 1]], (0, 2)), ([[1], [0], [2]], (1, 5, 2))]


@pytest.mark.parametrize("sampling", ["444", "422", "420", "440"])
def test_statement_equals_cv2_on_multi_scan_sequential_files(sampling):
    for h, w in ((7, 13), (17, 9), (37, 53)):
        b0 = JC.encode(h, w, 90, sampling, 0, "noisy")
        for groups, rst in MULTI:
            b = PW.multi_scan_sequential(b0, groups, rst)
            assert len(jpeg.parse(b, BIG).scans) == len(groups)
            assert np.array_equal(PR.decode(b), JC.cv2_decode(b)), (h, w, groups)
            assert np.array_equal(JC.cv2_decode(b), JC.cv2_decode(b0))


def test_max_scans_zero_raises_as_before():
    prog = PW.cv2_progressive(17, 9, 90, "420", 0)
    with pytest.raises(jpeg.JpegUnsupported, match="progressive"):
        jpeg.parse(prog)
    multi = PW.multi_scan_sequential(JC.encode(17, 9, 90, "420", 0, "noisy"), [[0], [1, 2]])
    with pytest.raises(jpeg.JpegUnsupported, match="multi-scan sequential"):
        jpeg.parse(multi)
    with pytest.raises(jpeg.JpegUnsupported, match="file 1: progressive"):
        jpeg.layout([JC.encode(7, 13, 90, "444", 0, "smooth"), prog])
    assert len(jpeg.layout([prog, multi], max_scans=BIG).scans) == 10 + 2


def test_single_scan_files_parse_the_same_with_max_scans():
    for case in JC.matrix(SMALL[:3])[::7]:
        b = JC.encode(*case)
        a, c = jpeg.parse(b), jpeg.parse(b, BIG)
        assert not c.scans and (a.scan_offset, a.scan_len, a.n_chunks) == (c.scan_offset, c.scan_len, c.n_chunks)
    f = JC.encode(17, 9, 90, "420", 0, "smooth") + JC.encode(7, 13, 90, "444", 4, "noisy")
    assert jpeg.parse(f, BIG).scan_len == jpeg.parse(f).scan_len


def test_scan_geometry_and_segments():
    b = PW.cv2_progressive(17, 17, 90, "420", 3)
    info, sc = _scan_list(b)
    for s, (sos, end) in zip(info.scans, sc):
        assert b[end:end + 2] in (b"\xff\xc4", b"\xff\xda", b"\xff\xd9", b"\xff\xdd")   # the next marker
        if len(s.comps) == 1:
            w, h = info.comp_size(s.comps[0])
            assert (s.mcus_x, s.mcus_y) == (-(-w // 8), -(-h // 8))
        else:
            assert (s.mcus_x, s.mcus_y) == (info.mcus_x, info.mcus_y)
    luma = [s for s in info.scans if s.comps == [0]]
    assert luma and all(s.mcus_x == 3 for s in luma)          # W = 17: 3 luma blocks per row, not 4
    assert info.comp_blocks(0)[0] == 4
    assert info.n_chunks == sum(s.n_chunks for s in info.scans)


def test_invalid_scripts_raise_jpeg_error():
    b = PW.cv2_progressive(17, 9, 90, "420", 0)          # scans: 0 DC Al=1 (3 comps), 1 Y 1..5, ..., 5 Y refine
    for k, kw in ((1, dict(ss=6, se=5)), (1, dict(se=64)), (0, dict(se=3)), (0, dict(ss=1, se=5)),
                  (5, dict(ah=2, al=0)), (1, dict(al=14))):
        with pytest.raises(jpeg.JpegError, match="bad progression") as e:
            jpeg.parse(_patch_sos(b, k, **kw), BIG)
        assert not isinstance(e.value, jpeg.JpegUnsupported), (k, kw)


def test_scripts_the_device_does_not_decode_raise_unsupported():
    b = PW.cv2_progressive(17, 9, 90, "420", 0)
    n = len(jpeg.parse(b, BIG).scans)
    cases = {"Ah is not the previous Al": _patch_sos(b, 5, ah=3, al=2),
             "AC scan before the component's first DC": _with_scans(b, [1, 0] + list(range(2, n))),
             "two first scans": _with_scans(b, list(range(n)) + [1]),
             "incomplete progressive script": _with_scans(b, list(range(n - 1)))}
    for what, f in cases.items():
        with pytest.raises(jpeg.JpegUnsupported, match=what):
            jpeg.parse(f, BIG)
    _, sc = _scan_list(b)
    dqt = b[b.find(b"\xff\xdb"):]
    dqt = dqt[:2 + ((dqt[2] << 8) | dqt[3])]                  # the file's first DQT, sent again before scan 1
    with pytest.raises(jpeg.JpegUnsupported, match="DQT that redefines"):
        jpeg.parse(b[:sc[1][0]] + dqt + b[sc[1][0]:], BIG)


def test_incomplete_script_is_smoothed_by_cv2_and_rejected():
    b = PW.cv2_progressive(37, 53, 90, "420", 0, "smooth")
    info = jpeg.parse(b, BIG)
    n = len(info.scans)
    f = _with_scans(b, list(range(n - 1)))                   # without the last luma refinement
    with pytest.raises(jpeg.JpegUnsupported, match="incomplete progressive script"):
        jpeg.parse(f, BIG)
    fi = jpeg.parse(b, BIG)
    fi.scans = fi.scans[:n - 1]      # f's scans: the dropped one came last, so the others keep their offsets
    assert not np.array_equal(PR.decode(f, fi), JC.cv2_decode(f))


def test_scan_capacity_raises_value_error():
    files = [PW.cv2_progressive(7, 13, 90, "444", 0), PW.cv2_progressive(17, 9, 90, "grey", 0)]
    assert len(jpeg.plan(files, max_scans=16)[0].scans) == 16
    with pytest.raises(ValueError, match="capacity of 15"):
        jpeg.plan(files, max_scans=15)
    with pytest.raises(ValueError, match="capacity of 5"):
        jpeg.parse(files[1], 5)


def test_multi_scan_kernels_do_not_touch_local_memory():
    lib = os.path.join(ROOT, "arbitrary-hands-3d-reconstruction_b200", "lib", "libacr_b200.so")
    if not (os.path.exists(lib) and os.path.exists("/usr/local/cuda/bin/cuobjdump")):
        pytest.skip("library not built or no cuobjdump")
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    try:
        import sass_audit
        rows = sass_audit.audit(lib)
    finally:
        sys.path.pop(0)
    names = {"jpeg_scan_spec_kernel", "jpeg_scan_sync_kernel", "jpeg_scan_write_kernel", "jpeg_refine_kernel"}
    found = {n: r for n, r in rows.items() if n in names}
    assert set(found) == names, sorted(rows)[:10]
    for n, r in found.items():
        assert r["LDL"] == 0 and r["STL"] == 0, f"{n}: {r['LDL']} LDL / {r['STL']} STL"


# ---- the progressive script writer (tests/jpeg_progressive_writer.py) ----------------------------------------------
WRITER_SAMPLINGS = ["420", "422", "444", "440", "grey"]


def writer_files():
    """label -> (file, writer stats, source file) for every script, sampling and table kind."""
    out = {}
    for s in WRITER_SAMPLINGS:
        src = JC.encode(45, 83, 90, s, 0, "noisy")
        for name, (script, rst) in PW.scripts(1 if s == "grey" else 3).items():
            for tables in ("optimal", "long"):
                b, st = PW.progressive(src, script, rst, tables)
                out[f"{s}-{name}-{tables}"] = (b, st, src)
    return out


def long_eob_file():
    """A flat 1456 x 1456 grey frame (33124 blocks) whose AC scan is one EOB run of 32767 blocks and another."""
    import cv2
    flat = cv2.imencode(".jpg", np.full((1456, 1456), 117, np.uint8), [cv2.IMWRITE_JPEG_QUALITY, 90])[1].tobytes()
    return PW.progressive(flat, [([0], 0, 0, 0, 0), ([0], 1, 63, 0, 0)])[0], flat


@pytest.mark.parametrize("sampling", WRITER_SAMPLINGS)
def test_writer_scripts_equal_cv2_and_the_source(sampling):
    files = {k: v for k, v in writer_files().items() if k.startswith(sampling + "-")}
    for label, (b, _, src) in files.items():
        info = jpeg.parse(b, 4096)
        assert info.scans, label
        exp = JC.cv2_decode(src)
        assert np.array_equal(JC.cv2_decode(b), exp), label
        assert np.array_equal(PR.decode(b), exp), label


def test_writer_scripts_cover_the_issue():
    files = writer_files()
    one = jpeg.parse(files["420-one-coef-bands-optimal"][0], 4096)
    assert sum(1 for s in one.scans if s.comps == [0]) > 64                  # over 64 scans per component
    deep = jpeg.parse(files["420-deep-sa-optimal"][0], 4096)
    assert max(s.al for s in deep.scans) == 4 and len({s.restart for s in deep.scans}) > 1   # DRI changes
    mixed = jpeg.parse(files["444-components-interleaved-in-file-order-optimal"][0], 4096)
    order = [s.comps[0] for s in mixed.scans if s.ss > 0]
    assert order[:3] == [0, 1, 2] and order[3:6] == [0, 1, 2]                  # components alternate in file order
    assert any(s.se < 63 and s.ss > 1 for s in mixed.scans)                    # narrow bands, then refinements


def test_writer_files_cross_chunk_boundaries():
    """EOB runs with their correction bits, RST markers and stuffed FF 00 pairs straddle 256-byte chunk boundaries
    somewhere in the writer files, so the device's chunks start inside each of them."""
    tot = {}
    for _, st, _ in writer_files().values():
        for k, v in st.items():
            tot[k] = tot.get(k, 0) + v
    for k in ("eob_across", "corr_across", "rst_across", "ff00_across"):
        assert tot[k] > 0, (k, tot)


def test_longest_eob_run():
    b, src = long_eob_file()
    info = jpeg.parse(b, 16)
    assert info.scans[1].n_blocks == 182 * 182 > 32767
    seg = b[info.scans[1].offset:info.scans[1].offset + info.scans[1].length]
    assert len(seg) < 16                                                      # two EOBn codes: 32767 + 357 blocks
    assert np.array_equal(JC.cv2_decode(b), JC.cv2_decode(src))
    assert np.array_equal(PR.decode(b), JC.cv2_decode(b))
