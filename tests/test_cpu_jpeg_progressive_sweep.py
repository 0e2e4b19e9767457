"""CPU: a sweep of progressive and multi-scan sequential JPEG files over every partial-MCU size, restart layout and
refinement code path, and the files tests/test_gpu_jpeg_progressive_sweep.py decodes on the device.

* the numpy statement (tests/jpeg_progressive_ref.py) equals cv2.imdecode on cv2 progressive files at every (h, w)
  in jpeg_cases.SWEEP^2, every sampling, RST interval 0 / 1 / 3, and their coefficients are the baseline file's;
* every script of tests/jpeg_progressive_writer.py, with optimal and all-long tables, at sizes from
  {1, 7, 8, 9, 16, 17, 33}^2, with no restarts and with restart layouts computed from each scan's geometry (with
  and without 0xFF fill bytes), multi-scan sequential files with per-scan restarts and fill bytes, grey frames whose
  SOF gives the one component 2x2, 1x2 or 2x1 sampling, and medium frames whose scans have more than 256 blocks
  (not a multiple of 256): each decodes in cv2 to its source's pixels, and the statement equals cv2;
* the restart layouts put RST markers where intended (mid-row in one-component chroma scans, at row ends, none at
  all, every block of a refinement scan, intervals that change between the scans of one component);
* the writer's stream features all occur: ZRL in first and refinement scans, EOBn codes of every length class
  (r = 0..14) in both, EOB runs cut by an RST and ending at the scan's last block, correction bits after a ZRL, and
  EOB runs, correction bits, RSTs and stuffed FF 00 across 256-byte chunk boundaries;
* the writer's existing output is byte for byte what it was before ``fill`` and the counters existed.
"""
import functools
import hashlib
import os
import re

import numpy as np
import pytest

from acr_b200 import jpeg
from tests import jpeg_cases as JC
from tests import jpeg_progressive_ref as PR
from tests import jpeg_progressive_writer as PW
from tests import jpeg_writer as JW

BIG = 4096
SAMPLINGS = ["420", "422", "444", "440", "grey"]
WSIZES = [(h, w) for h in (1, 7, 8, 9, 16, 17, 33) for w in (1, 7, 8, 9, 16, 17, 33)]
MEDIUM = [(127, 135), (129, 257), (257, 129)]
GROUPS = [[[0], [1, 2]], [[1], [0], [2]], [[2], [0, 1]]]
LAYOUTS = ["none", "rows", "mid-row", "refine-1", "past-end"]
FILLS = [(0,), (1, 3)]


# ---- the corpus --------------------------------------------------------------------------------------------------
def cv2_sweep(sizes=None):
    """label -> (cv2 progressive file, its baseline twin with the same coefficients)."""
    out = {}
    for h, w in sizes or [(h, w) for h in JC.SWEEP for w in JC.SWEEP]:
        for s in SAMPLINGS:
            for r in (0, 1, 3):
                out[f"cv2-{h}x{w}-{s}-r{r}"] = (PW.cv2_progressive(h, w, 90, s, r), JC.encode(h, w, 90, s, r, "noisy"))
    return out


def scan_geometry(src, comps):
    """(units per row, units) of a scan over ``comps`` of the source: MCUs, or the component's own blocks."""
    if len(comps) > 1:
        mx, my = src.mcus
        return mx, mx * my
    units = PW._scan_units(src, comps)
    return units[-1][0][2] + 1, len(units)


def layout(kind, src, script):
    """Per-scan restart intervals of a layout, from each scan's geometry."""
    if kind == "none":
        return None
    out = []
    for k, (comps, ss, se, ah, al) in enumerate(script):
        mx, n = scan_geometry(src, comps)
        if kind == "rows":                      # a boundary at every row end
            out.append(mx)
        elif kind == "mid-row":                 # boundaries inside rows (one past a row, then drifting)
            out.append(mx + 1)
        elif kind == "refine-1":                # every block in refinement scans; first scans change per scan
            out.append(1 if ah else (2, 3, 5, 7)[k % 4])
        else:                                   # a DRI longer than the scan: no RST at all
            out.append(min(n + 1, 65535))
    return out


def _writer_source(h, w, s, grey_hv=None):
    b = JC.encode(h, w, 90, s, 0, "noisy")
    if grey_hv is not None:      # the same coefficients under a SOF that gives the grey component these factors
        b = JW.write(JW.source(b), tables="source", grey_hv=grey_hv)
    return b


@functools.lru_cache(maxsize=None)
def writer_sweep():
    """label -> (file, writer stats, baseline source) for the writer's scripts at small sizes: each (sampling,
    script, tables) takes 14 of the sizes (every size comes up for every sampling), cycling through the restart
    layouts and fill bytes."""
    out = {}
    v = 0
    for s in SAMPLINGS:
        scripts = PW.scripts(1 if s == "grey" else 3)
        for name, (script, _) in scripts.items():
            for tables in ("optimal", "long"):
                for k in range(14):
                    h, w = WSIZES[(7 * v + k) % len(WSIZES)]
                    kind = LAYOUTS[(v + k) % len(LAYOUTS)]
                    fill = FILLS[((v + k) // len(LAYOUTS)) % 2] if kind != "none" else (0,)
                    src = _writer_source(h, w, s)
                    b, st = PW.progressive(src, script, layout(kind, JW.source(src), script), tables, fill)
                    out[f"w-{s}-{name}-{tables}-{h}x{w}-{kind}-f{fill[0]}"] = (b, st, src)
                v += 1
    return out


@functools.lru_cache(maxsize=None)
def grey_sampling_files():
    """label -> (file, stats, source): grey frames whose SOF gives the component 2x2, 1x2 or 2x1, every script."""
    out = {}
    for i, hv in enumerate(((2, 2), (1, 2), (2, 1))):
        for j, (name, (script, rst)) in enumerate(PW.scripts(1).items()):
            h, w = ((17, 33), (33, 9), (9, 17))[(i + j) % 3]
            src = _writer_source(h, w, "grey", hv)
            b, st = PW.progressive(src, script, rst, ("optimal", "long")[j % 2], ((0,), (2, 1))[(i + j) % 2])
            out[f"grey{hv[0]}x{hv[1]}-{name}-{h}x{w}"] = (b, st, src)
    return out


@functools.lru_cache(maxsize=None)
def medium_files():
    """label -> (file, stats, source): scans of more than 256 blocks, not a multiple of 256, every sampling and
    script, restart layouts cycling."""
    out = {}
    v = 0
    for s in SAMPLINGS:
        for name, (script, _) in PW.scripts(1 if s == "grey" else 3).items():
            h, w = MEDIUM[v % 3]
            kind = ("none", "refine-1", "mid-row")[v % 3]
            src = _writer_source(h, w, s)
            b, st = PW.progressive(src, script, layout(kind, JW.source(src), script), ("optimal", "long")[v % 2],
                                   ((0,), (1, 3))[v % 2])
            out[f"m-{s}-{name}-{h}x{w}-{kind}"] = (b, st, src)
            v += 1
    return out


@functools.lru_cache(maxsize=None)
def multi_sweep():
    """label -> (file, source): multi-scan sequential files at the small sizes, three component groupings, with
    no restarts, per-scan restarts, and per-scan restarts with fill bytes."""
    out = {}
    v = 0
    for s in ("420", "422", "444", "440"):
        for h, w in WSIZES:
            src = _writer_source(h, w, s)
            S = JW.source(src)
            for groups in GROUPS:
                variant = v % 3
                rst, fill = (), (0,)
                if variant:         # a row and one more, every unit, two units: changing from scan to scan
                    rst = [(scan_geometry(S, g)[0] + 1, 1, 2)[(k + v) % 3] for k, g in enumerate(groups)]
                if variant == 2:
                    fill = (1, 3)
                out[f"ms-{s}-{h}x{w}-{''.join(map(str, sum(groups, [])))}-v{variant}"] = (
                    PW.multi_scan_sequential(src, groups, rst, fill), src)
                v += 1
    return out


@functools.lru_cache(maxsize=None)
def eob_classes_file():
    """(file, stats, source): a 1664 x 1664 grey frame, flat but for noise blocks spaced so that the AC first and
    AC refinement scans code EOB runs of every length class 4..14 (runs of 1.25 * 2^r blocks), the last run ending
    at the scan's last block."""
    import cv2
    n = 208
    img = np.full((8 * n, 8 * n), 117, np.uint8)
    rng = np.random.default_rng(3)
    p = 0
    for r in range(4, 15):
        by, bx = divmod(p, n)
        img[8 * by:8 * by + 8, 8 * bx:8 * bx + 8] = rng.integers(0, 256, (8, 8))
        p += 1 + (1 << r) + (1 << (r - 2))
    src = cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, 90])[1].tobytes()
    b, st = PW.progressive(src, [([0], 0, 0, 0, 0), ([0], 1, 63, 0, 1), ([0], 1, 63, 1, 0)])
    return b, st, src


def all_stats():
    out = [st for _, st, _ in writer_sweep().values()] + [st for _, st, _ in grey_sampling_files().values()]
    out += [st for _, st, _ in medium_files().values()] + [eob_classes_file()[1]]
    return out


# ---- restart layouts ---------------------------------------------------------------------------------------------
def rst_count(b, s):
    """RST markers in scan s's segment (after any fill bytes)."""
    return len(re.findall(rb"\xff[\xd0-\xd7]", b[s.offset:s.offset + s.length]))


def boundaries(s):
    """Block-unit positions (MCUs, or blocks of a one-component scan) where scan s's restart intervals end."""
    n = s.mcus_x * s.mcus_y
    return list(range(s.restart, n, s.restart)) if s.restart else []


# ---- tests -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("h", JC.SWEEP)
def test_statement_equals_cv2_on_the_cv2_sweep(h):
    bad = []
    for label, (b, base) in cv2_sweep([(h, w) for w in JC.SWEEP]).items():
        exp = JC.cv2_decode(b)
        if not np.array_equal(PR.decode(b), exp) or not np.array_equal(exp, JC.cv2_decode(base)):
            bad.append(label)
    assert not bad, bad[:8]


def test_cv2_progressive_coefficients_are_the_baseline_files():
    from oracle import jpeg_ref
    for label, (b, base) in cv2_sweep([(1, 1), (9, 17), (17, 33), (33, 8)]).items():
        for c, (x, y) in enumerate(zip(PR.coefficients(b), jpeg_ref.coefficients(base, jpeg.parse(base)))):
            assert np.array_equal(x, y), (label, c)


def test_recoded_coefficients_are_the_sources_on_the_components_own_blocks():
    """A re-coded file carries its source's coefficients in each component's ceil(w / 8) x ceil(h / 8) blocks; the
    MCU padding past them, which a baseline file codes and a one-component scan does not, is not compared (it never
    reaches a pixel)."""
    from oracle import jpeg_ref
    files = {k: (v[0], v[2]) for k, v in writer_sweep().items()}
    files.update(multi_sweep())
    for label, (b, src) in list(files.items())[::10]:
        info = jpeg.parse(b, BIG)
        own = [(-(-info.comp_size(c)[1] // 8), -(-info.comp_size(c)[0] // 8)) for c in range(info.ncomp)]
        for c, (x, y, (h, w)) in enumerate(zip(PR.coefficients(b, info), jpeg_ref.coefficients(src, jpeg.parse(src)),
                                               own)):
            assert np.array_equal(x[:h, :w], y[:h, :w]), (label, c)


@pytest.mark.parametrize("sampling", SAMPLINGS)
def test_writer_sweep_equals_cv2_and_the_source(sampling):
    bad = []
    for label, (b, _, src) in writer_sweep().items():
        if not label.startswith(f"w-{sampling}-"):
            continue
        exp = JC.cv2_decode(src)
        if not np.array_equal(JC.cv2_decode(b), exp) or not np.array_equal(PR.decode(b), exp):
            bad.append(label)
    assert not bad, bad[:8]


def test_multi_scan_sweep_equals_cv2_and_the_source():
    bad = []
    for label, (b, src) in multi_sweep().items():
        exp = JC.cv2_decode(src)
        if not np.array_equal(JC.cv2_decode(b), exp) or not np.array_equal(PR.decode(b), exp):
            bad.append(label)
    assert not bad, bad[:8]


def test_grey_sampling_factors_and_medium_files_equal_cv2_and_the_source():
    bad = []
    files = dict(grey_sampling_files())
    files.update(medium_files())
    b, st, src = eob_classes_file()
    files["eob-classes"] = (b, st, src)
    for label, (b, _, src) in files.items():
        info = jpeg.parse(b, BIG)
        exp = JC.cv2_decode(src)
        if not np.array_equal(JC.cv2_decode(b), exp):
            bad.append(label)
        elif label.startswith("grey") and not np.array_equal(PR.decode(b, info), exp):
            bad.append(label)
    assert not bad, bad[:8]
    sof = {label[4:7] for label, (b, _, _) in grey_sampling_files().items()
           if b[b.find(b"\xff\xc2") + 11] == (int(label[4]) << 4 | int(label[6]))}
    assert sof == {"2x2", "1x2", "2x1"}                      # the SOF really carries the factors


def test_medium_files_have_scans_past_256_blocks():
    n = set()
    for label, (b, _, _) in medium_files().items():
        info = jpeg.parse(b, BIG)
        for s in info.scans:
            if s.n_blocks > 256 and s.n_blocks % 256:
                n.add((label.split("-")[1], s.ah > 0))
    assert n == {(s, a) for s in SAMPLINGS for a in (False, True)}, sorted(n)


def test_statement_on_medium_files():
    """The statement (slow on these sizes) on one medium file per sampling, the refinement-heavy scripts."""
    for label, (b, _, src) in medium_files().items():
        if "-deep-sa-" in label or "-interleaved-" in label:
            assert np.array_equal(PR.decode(b), JC.cv2_decode(src)), label


def test_restart_layouts_put_boundaries_where_intended():
    mid_chroma = row_end = past_end = refine_1 = differ = fill_rst = 0
    files = {k: v[0] for k, v in writer_sweep().items()}
    files.update({k: v[0] for k, v in medium_files().items()})
    files.update({k: v[0] for k, v in multi_sweep().items()})
    for label, b in files.items():
        info = jpeg.parse(b, BIG)
        per_comp = {}
        for s in info.scans:
            n = s.mcus_x * s.mcus_y
            bnd = boundaries(s)
            assert rst_count(b, s) == len(bnd), (label, s.comps, s.restart)
            if len(s.comps) == 1 and s.comps[0] > 0 and any(p % s.mcus_x for p in bnd):
                mid_chroma += 1
            row_end += any(p % s.mcus_x == 0 for p in bnd)
            past_end += s.restart >= n
            refine_1 += s.ah > 0 and s.restart == 1 and n > 1
            fill_rst += bool(re.search(rb"\xff\xff[\xd0-\xd7]", b[s.offset:s.offset + s.length]))
            for c in s.comps:
                per_comp.setdefault(c, set()).add(s.restart)
        differ += any(len(v - {0}) > 1 for v in per_comp.values())
    counts = dict(mid_chroma=mid_chroma, row_end=row_end, past_end=past_end, refine_1=refine_1, differ=differ,
                  fill_rst=fill_rst)
    assert all(v > 0 for v in counts.values()), counts


def test_writer_stream_features_all_occur():
    tot = dict.fromkeys(PW.STAT_KEYS, 0)
    for st in all_stats():
        for k, v in st.items():
            tot[k] += v
    missing = [k for k in PW.STAT_KEYS if tot[k] == 0]
    assert not missing, (missing, tot)


def test_one_coefficient_bands_at_both_ends():
    for label, (b, _, _) in writer_sweep().items():
        if "-one-coef-bands-" in label:
            bands = {(s.ss, s.se, s.ah) for s in jpeg.parse(b, BIG).scans}
            assert {(1, 1, 0), (1, 1, 1), (63, 63, 0), (63, 63, 1)} <= bands, label


# ---- the writer's existing output ------------------------------------------------------------------------------
# sha256 (first 32 hex digits) of every script file and the multi-scan sequential files the writer made from the
# committed sources (tests/golden/jpeg_progressive_sources.npz) before ``fill`` and the counters were added
WRITER_DIGESTS = {"420": "89c48998e862c50188985b9a2ad388f9", "422": "33b4e3dc4ac730f220c0cd51aa26b4a7",
                  "444": "f1e773b363b3a4aac41e12ce8b5a54f7", "440": "ed7a5a6ad7cfb386e46968c18dac6aeb",
                  "grey": "a3cdbc4de9bfd1efd5747a81e2d6fdc4"}
OLD_STATS = ("eob_across", "corr_across", "rst_across", "ff00_across", "max_eobrun")
MULTI = [([[0], [1], [2]], ()), ([[0], [1, 2]], (3, 0)), ([[2], [0, 1]], (0, 2)), ([[1], [0], [2]], (1, 5, 2))]


@pytest.mark.parametrize("sampling", SAMPLINGS)
def test_writer_output_is_unchanged(sampling):
    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "jpeg_progressive_sources.npz"))
    h = hashlib.sha256()
    src = z[f"src-45x83-{sampling}"].tobytes()
    for name, (script, rst) in PW.scripts(1 if sampling == "grey" else 3).items():
        for tables in ("optimal", "long"):
            b, st = PW.progressive(src, script, rst, tables)
            h.update(b)
            h.update(repr([st[k] for k in OLD_STATS]).encode())
    if sampling != "grey":
        src = z[f"src-37x53-{sampling}"].tobytes()
        for groups, rst in MULTI:
            h.update(PW.multi_scan_sequential(src, groups, rst))
    assert h.hexdigest()[:32] == WRITER_DIGESTS[sampling]
