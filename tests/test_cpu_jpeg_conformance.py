"""CPU: the JPEG parser and the numpy decode statement (oracle/jpeg_ref.py) on streams other encoders write.

* the test-side writer (tests/jpeg_writer.py) reproduces cv2's scan byte for byte with cv2's tables, and every
  variant it writes carries the source's coefficients (only the quantisation variants change pixels);
* its Huffman presets have the code lengths they promise, and parse() reads every header variant: per-component
  table ids 0-3, 8- and 16-bit quantisation tables with SOF1, several tables per segment, redefined tables, the last
  of two DRIs, component ids, APPn / COM segments and a grey frame with 2x2 sampling factors;
* the oracle equals cv2.imdecode on every writer variant, on cv2 files with optimised tables and separate luma /
  chroma qualities, on the committed Pillow files (SOF1 with 16-bit DQT, restarts per row and per 7 blocks, EXIF,
  an ICC profile over several APP2 segments, COM, optimised tables) and on every size of the small sweep.  The
  12 and 24 MP frames are left to the GPU test: the numpy Huffman decoder takes minutes on them;
* fill bytes before markers and a trailing RST after the last MCU decode as cv2 decodes them;
* the files put restart markers, stuffed FF 00 pairs and runs of fill bytes across 256-byte decoder chunks.
"""
import numpy as np
import pytest

from acr_b200 import jpeg
from oracle import jpeg_ref
from tests import jpeg_cases as JC
from tests import jpeg_writer as JW


def _all_coef_equal(a, b):
    return len(a) == len(b) and all(np.array_equal(x, y) for x, y in zip(a, b))


# ------------------------------------------------------------------------------------------------ the writer itself
@pytest.mark.parametrize("name", list(JC.WRITER_SOURCES))
def test_writer_with_the_source_tables_reproduces_the_cv2_scan(name):
    for rst in (0, 1, 4):
        case = JC.WRITER_SOURCES[name][:4] + (rst,) + JC.WRITER_SOURCES[name][5:]
        b = JC.encode(*case)
        src = JW.source(b)
        f = JW.write(src, restart=rst)
        assert JW.scan_of(f) == JW.scan_of(b), case
        assert np.array_equal(JC.cv2_decode(f), JC.cv2_decode(b)), case


@pytest.mark.parametrize("name", list(JC.WRITER_SOURCES))
def test_every_writer_variant_keeps_the_source_coefficients(name):
    src = JW.source(JC.encode(*JC.WRITER_SOURCES[name]))
    ref = JC.cv2_decode(JC.encode(*JC.WRITER_SOURCES[name]))
    files = {k: v for k, v in JC.writer_files().items() if k.startswith(f"writer-{name}-")}
    assert len(files) >= 40
    for label, (b, quant_changed) in files.items():
        assert _all_coef_equal(jpeg_ref.coefficients(b), src.coef), label
        same = np.array_equal(JC.cv2_decode(b), ref)
        assert same != quant_changed, label      # lowered quantisation tables change pixels, nothing else does


def test_huffman_presets_have_their_code_lengths():
    src = JW.source(JC.encode(*JC.WRITER_SOURCES["420"]))
    for kind in ("optimal", "long", "short", "skewed"):
        dc, ac = JW.preset_tables(src, kind)
        for t in dc + ac:
            parsed = jpeg.HuffTable(t.bits, t.vals)        # the parser's table: Kraft-valid, no all-ones code
            if kind == "long":
                assert min(t.lengths()) == 10 and max(t.lengths()) == 16
                assert not parsed.lut.any()                  # every code takes the maxcode path
                assert all(t.bits[l] for l in range(10, 17) if len(t.vals) >= 7)
            elif kind == "skewed":
                assert t.bits[1] == 1
        if kind == "short":
            assert set(dc[0].lengths()) == {4} and set(ac[0].lengths()) == {8}
        if kind == "optimal":                                # counted per component: Cb and Cr differ
            assert not JW._same(ac[1], ac[2])
    with pytest.raises(ValueError, match="Kraft"):
        JW.table_from_lengths({0: 1, 1: 1})                  # would need the all-ones code


# ------------------------------------------------------------------------------------------------------- headers
def test_parse_reads_every_header_variant():
    for name in JC.WRITER_SOURCES:
        src, variants = JC.writer_variants(name)
        for label, kw in variants.items():
            b = JW.write(src, **kw)
            info = jpeg.parse(b)
            nc = src.ncomp
            assert (info.H, info.W, info.ncomp) == (src.H, src.W, nc), label
            assert info.restart == (kw["dri"][-1] if "dri" in kw else kw.get("restart", 0)), label
            quant = kw.get("quant", src.quant)
            assert np.array_equal(info.quant, quant[:nc]), label
            dc, ac = JW.preset_tables(src, kw.get("tables", "source"), kw.get("restart", 0))
            for c in range(nc):
                for got, exp in ((info.dc[c], dc[c]), (info.ac[c], ac[c])):
                    assert np.array_equal(got.bits, exp.bits) and np.array_equal(got.vals, exp.vals), (label, c)
            if nc == 1:
                assert (info.mcus_x, info.mcus_y, info.bpm) == (-(-src.W // 8), -(-src.H // 8), 1), label
            else:
                assert [(info.comp_h[c], info.comp_v[c]) for c in range(3)] == src.comp_hv, label
            sof1 = any(kw.get("qprec", (0, 0, 0))[:nc])       # 16-bit tables are written with SOF1
            assert b.count(b"\xff\xc1") >= 1 if sof1 else b"\xff\xc1" not in b[:info.scan_offset], label


def test_pillow_files_carry_what_they_are_named_for():
    files = JC.pillow_files()
    q16 = files["pillow-sof1_q16_420"]
    assert b"\xff\xc1" in q16 and int(jpeg.parse(q16).quant.max()) > 255
    assert jpeg.parse(files["pillow-rst_rows_420"]).restart == jpeg.parse(files["pillow-rst_rows_420"]).mcus_x
    assert jpeg.parse(files["pillow-rst_blocks7_422"]).restart == 7
    assert files["pillow-icc_app2x2_444"].count(b"\xff\xe2") >= 2 and len(files["pillow-icc_app2x2_444"]) > 65536
    assert b"Exif\x00\x00" in files["pillow-exif_420"]
    assert b"\xff\xfe" in files["pillow-comment_optimize_444"]
    with pytest.raises(jpeg.JpegUnsupported, match="RGB"):
        jpeg.parse(files["pillow-rgb_keep_rgb"])


# ------------------------------------------------------------------------------------------ the oracle against cv2
def _mismatches(files):
    bad = []
    for name, b in files.items():
        try:
            if not np.array_equal(jpeg_ref.decode(b), JC.cv2_decode(b)):
                bad.append(name)
        except jpeg.JpegError as e:
            bad.append(f"{name}: {e}")
    return bad


def test_oracle_equals_cv2_on_the_writer_variants():
    files = {k: b for k, (b, _) in JC.writer_files().items()}
    bad = _mismatches(files)
    assert not bad, f"{len(bad)} of {len(files)}: {bad[:6]}"


def test_oracle_equals_cv2_on_cv2_optimized_and_pillow_files():
    files = dict(JC.cv2_optimized())
    files.update({k: b for k, b in JC.pillow_files().items() if "rgb" not in k})
    bad = _mismatches(files)
    assert not bad, f"{len(bad)} of {len(files)}: {bad[:6]}"


@pytest.mark.parametrize("sampling", JC.SAMPLINGS)
def test_oracle_equals_cv2_on_the_small_sweep(sampling):
    cases = [c for c in JC.small_sweep() if c[3] == sampling]
    bad = _mismatches({c: JC.encode(*c) for c in cases})
    assert not bad, f"{len(bad)} of {len(cases)}: {bad[:6]}"


def test_oracle_skips_fill_bytes_before_markers():
    """T.81 B.1.1.2: any marker may follow 0xFF fill bytes; libjpeg skips them."""
    b = JC.encode(17, 45, 90, "420", 1, "noisy")
    info = jpeg.parse(b)
    scan = b[info.scan_offset:info.scan_offset + info.scan_len]
    filled = bytearray()
    for i, x in enumerate(scan):
        if x == 0xFF and i + 1 < len(scan) and 0xD0 <= scan[i + 1] <= 0xD7:
            filled.append(0xFF)
        filled.append(x)
    f = b[:info.scan_offset] + bytes(filled) + b"\xff" + b[info.scan_offset + info.scan_len:]
    assert len(f) > len(b) + 1
    assert np.array_equal(JC.cv2_decode(f), JC.cv2_decode(b))
    assert np.array_equal(jpeg_ref.decode(f), JC.cv2_decode(b))


def test_oracle_accepts_a_trailing_restart_marker():
    """An RST after the last MCU, when the MCU count is a multiple of the interval, as some encoders write."""
    b = JC.encode(16, 64, 90, "444", 4, "noisy")            # 16 MCUs, interval 4: three markers, then one more
    info = jpeg.parse(b)
    e = info.scan_offset + info.scan_len
    f = b[:e] + b"\xff\xd3" + b[e:]
    assert np.array_equal(JC.cv2_decode(f), JC.cv2_decode(b))
    assert np.array_equal(jpeg_ref.decode(f), JC.cv2_decode(b))
    g = b[:e] + b"\xff\xd4" + b[e:]                          # out of sequence: still an error
    with pytest.raises(jpeg.JpegError, match="sequence"):
        jpeg_ref.coefficients(g)


# ---------------------------------------------------------------------------------- chunk-boundary coverage
def _scan_events(b):
    """Raw offsets in the scan of RST markers' FF, stuffed pairs' FF, and fill runs as (first, last)."""
    s = JW.scan_of(b)
    rst, stuffed, runs = [], [], []
    i, n = 0, len(s)
    while i < n:
        if s[i] != 0xFF:
            i += 1
            continue
        if i + 1 < n and s[i + 1] == 0:
            stuffed.append(i)
            i += 2
            continue
        j = i
        while j + 1 < n and s[j + 1] == 0xFF:
            j += 1
        if j > i or j + 1 >= n:
            runs.append((i, j - 1 if j + 1 < n else j))
        if j + 1 < n:
            rst.append(j)
        i = j + 2
    return rst, stuffed, runs


def test_markers_stuffing_and_fill_bytes_cross_chunk_boundaries():
    C = jpeg.CHUNK
    hit = {"rst-last": 0, "rst-first": 0, "stuffed-last": 0, "stuffed-first": 0, "fill-crosses": 0}
    files = [b for b, _ in JC.writer_files().values()]
    files += [b for k, b in JC.pillow_files().items() if "rgb" not in k]
    for b in files:
        rst, stuffed, runs = _scan_events(b)
        hit["rst-last"] += sum(p % C == C - 1 for p in rst)
        hit["rst-first"] += sum(p % C == 0 for p in rst)
        hit["stuffed-last"] += sum(p % C == C - 1 for p in stuffed)
        hit["stuffed-first"] += sum(p % C == 0 for p in stuffed)
        hit["fill-crosses"] += sum(a // C != b_ // C for a, b_ in runs)
    assert all(hit.values()), hit
