"""Multi-scan sequential JPEG files for the tests (tests/test_*_jpeg_progressive.py): the coefficients of a cv2 file
(tests/jpeg_writer.py's ``Source``) coded again as several sequential scans (Ss = 0, Se = 63, Ah = Al = 0), each over
a group of the components, with the source's headers and Huffman tables (``Table`` and the bit writer of
tests/jpeg_writer.py).  A one-component scan codes the component's own ceil(w / 8) x ceil(h / 8) blocks; an
interleaved scan codes the frame's MCUs over its components.  ``restart`` sets a DRI before each scan; ``fill``
writes 0xFF fill bytes before each RST and at the end of each scan.  With the default ``fill`` every file is byte for
byte what the writer wrote before ``fill`` and the feature counters existed (tests/test_cpu_jpeg_progressive_sweep.py
holds it to digests)."""
from typing import Sequence

import numpy as np

import tests.jpeg_writer as JW


def _encode_block(bits, blk, pred, dc, ac):
    d = int(blk[0]) - pred
    s = abs(d).bit_length()
    bits.put(*dc[s])
    bits.put(d if d >= 0 else d + (1 << s) - 1, s)
    run = 0
    for z in range(1, 64):
        v = int(blk[JW.ZIGZAG[z]])
        if v == 0:
            run += 1
            continue
        while run > 15:
            bits.put(*ac[0xF0])
            run -= 16
        s = abs(v).bit_length()
        bits.put(*ac[(run << 4) | s])
        bits.put(v if v >= 0 else v + (1 << s) - 1, s)
        run = 0
    if run:
        bits.put(*ac[0x00])
    return int(blk[0])


def _codes(t):
    return {s: (c, l) for s, (c, l) in JW.Table(t.bits, t.vals).codes().items()}


def _fill(fill: Sequence[int], k: int) -> bytes:
    """The 0xFF fill bytes before the k-th RST of a scan (``fill`` cycled); k = -1: before the marker that ends a
    scan (the first entry)."""
    return b"\xff" * (fill[k % len(fill)] if k >= 0 else fill[0])


def multi_scan_sequential(buf: bytes, groups: Sequence[Sequence[int]], restart: Sequence[int] = (),
                          fill: Sequence[int] = (0,)) -> bytes:
    """``buf`` (a baseline cv2 file) coded again as one sequential scan per group of component indices, in order.
    ``restart[k]``: the restart interval of scan k (0 = none; missing = 0).  ``fill``: 0xFF fill bytes (T.81
    B.1.1.2) before each RST, cycling through the list, and ``fill[0]`` of them after each scan, before the next
    DRI or the EOI."""
    src = JW.source(buf)
    sos = buf.find(b"\xff\xda")
    head = buf[:sos]
    L = (buf[sos + 2] << 8) | buf[sos + 3]
    sel = buf[sos + 5:sos + 5 + 2 * src.ncomp]
    tsel = {k: sel[2 * k + 1] for k in range(src.ncomp)}
    mx, my = src.mcus
    out = bytearray(head)
    for k, grp in enumerate(groups):
        rst = restart[k] if k < len(restart) else 0
        out += JW._seg(0xDD, rst.to_bytes(2, "big"))
        payload = bytes([len(grp)]) + b"".join(bytes([sel[2 * c], tsel[c]]) for c in grp) + bytes([0, 63, 0])
        out += JW._seg(0xDA, payload)
        if len(grp) > 1:
            units = [[(c, my_ * src.comp_hv[c][1] + dy, mx_ * src.comp_hv[c][0] + dx)
                      for c in grp for dy in range(src.comp_hv[c][1]) for dx in range(src.comp_hv[c][0])]
                     for my_ in range(my) for mx_ in range(mx)]
        else:
            c = grp[0]
            w = -(-src.W * src.comp_hv[c][0] // src.hmax) if src.ncomp > 1 else src.W
            h = -(-src.H * src.comp_hv[c][1] // src.vmax) if src.ncomp > 1 else src.H
            units = [[(c, by, bx)] for by in range(-(-h // 8)) for bx in range(-(-w // 8))]
        dc = {c: _codes(src.dc[c]) for c in grp}
        ac = {c: _codes(src.ac[c]) for c in grp}
        bits = JW._Bits()
        pred = {c: 0 for c in grp}
        for u, unit in enumerate(units):
            if rst and u and u % rst == 0:
                bits.flush()
                bits.out += _fill(fill, u // rst - 1) + bytes([0xFF, 0xD0 + ((u // rst - 1) & 7)])
                pred = {c: 0 for c in grp}
            for c, by, bx in unit:
                pred[c] = _encode_block(bits, src.coef[c][by, bx], pred[c], dc[c], ac[c])
        bits.flush()
        out += bits.out + _fill(fill, -1)
    out += b"\xff\xd9"
    return bytes(out)


def cv2_progressive(h, w, q, sampling, rst, content="noisy") -> bytes:
    from tests import jpeg_cases as JC
    return JC.encode(h, w, q, sampling, rst, content, progressive=True)


def pillow_progressive(h, w, q, subsampling, optimize=True) -> bytes:
    """Pillow's progressive writer; ``optimize`` writes optimal tables, one DHT before each scan."""
    import io

    from PIL import Image

    from tests import jpeg_cases as JC
    img = Image.fromarray(np.ascontiguousarray(JC.image(h, w, "noisy", seed=q)[:, :, ::-1]))
    b = io.BytesIO()
    img.save(b, "JPEG", quality=q, progressive=True, optimize=optimize, subsampling=subsampling)
    return b.getvalue()


# ---- progressive scripts (T.81 G.1.2, the order of libjpeg's progressive Huffman encoder) ----------------------------
def _bitlen(v: int) -> int:
    return abs(v).bit_length()


class _Scan:
    """Events of one scan: ("H", class, comp, symbol), ("B", value, nbits), ("R", marker number); ``count``: the
    stream features of ``STAT_KEYS`` it contains."""

    def __init__(self):
        self.ev = []
        self.count = {}

    def note(self, key):
        self.count[key] = self.count.get(key, 0) + 1

    def huff(self, tc, c, sym):
        self.ev.append(("H", tc, c, sym))

    def bits(self, v, n):
        if n:
            self.ev.append(("B", v & ((1 << n) - 1), n))


def _scan_units(src, comps):
    mx, my = src.mcus
    if len(comps) > 1:
        return [[(c, y * src.comp_hv[c][1] + dy, x * src.comp_hv[c][0] + dx)
                 for c in comps for dy in range(src.comp_hv[c][1]) for dx in range(src.comp_hv[c][0])]
                for y in range(my) for x in range(mx)]
    c = comps[0]
    w = -(-src.W * src.comp_hv[c][0] // src.hmax) if src.ncomp > 1 else src.W
    h = -(-src.H * src.comp_hv[c][1] // src.vmax) if src.ncomp > 1 else src.H
    return [[(c, by, bx)] for by in range(-(-h // 8)) for bx in range(-(-w // 8))]


def _progressive_events(src, comps, ss, se, ah, al, restart):
    sc = _Scan()
    units = _scan_units(src, comps)
    state = {"eobrun": 0, "be": []}

    def emit_eobrun():
        n = state["eobrun"]
        if n:
            r = n.bit_length() - 1
            sc.note(f"eob{r}_{'refine' if ah else 'first'}")
            sc.ev.append(("EOB", r))
            sc.huff(1, comps[0], r << 4)
            sc.bits(n, r)
            for b in state["be"]:
                sc.bits(b, 1)
            sc.ev.append(("EOB_END",))
            state["eobrun"], state["be"] = 0, []

    pred = {c: 0 for c in comps}
    for u, unit in enumerate(units):
        if restart and u and u % restart == 0:
            if state["eobrun"]:
                sc.note("eobrun_at_rst")
            emit_eobrun()
            sc.ev.append(("R", (u // restart - 1) & 7))
            pred = {c: 0 for c in comps}
        for c, by, bx in unit:
            blk = src.coef[c][by, bx].astype(np.int64)
            if ss == 0 and ah == 0:                               # DC first
                v = int(blk[0]) >> al
                d = v - pred[c]
                pred[c] = v
                s = _bitlen(d)
                sc.huff(0, c, s)
                sc.bits(d if d >= 0 else d - 1, s)
            elif ss == 0:                                         # DC refinement
                sc.bits((int(blk[0]) >> al) & 1, 1)
            elif ah == 0:                                         # AC first
                r = 0
                for k in range(ss, se + 1):
                    v = int(blk[JW.ZIGZAG[k]])
                    mag = abs(v) >> al
                    if mag == 0:
                        r += 1
                        continue
                    emit_eobrun()
                    while r > 15:
                        sc.note("zrl_first")
                        sc.huff(1, c, 0xF0)
                        r -= 16
                    n = mag.bit_length()
                    sc.huff(1, c, (r << 4) | n)
                    sc.bits(mag if v >= 0 else ~mag, n)
                    r = 0
                if r:
                    state["eobrun"] += 1
                    if state["eobrun"] == 0x7FFF:
                        emit_eobrun()
            else:                                                 # AC refinement
                absv = [abs(int(blk[JW.ZIGZAG[k]])) >> al for k in range(64)]
                eob = max([k for k in range(ss, se + 1) if absv[k] == 1], default=0)
                r, br = 0, []
                for k in range(ss, se + 1):
                    t = absv[k]
                    if t == 0:
                        r += 1
                        continue
                    while r > 15 and k <= eob:
                        emit_eobrun()
                        sc.note("zrl_refine")
                        if br:
                            sc.note("corr_after_zrl")
                        sc.huff(1, c, 0xF0)
                        r -= 16
                        for b in br:
                            sc.bits(b, 1)
                        br = []
                    if t > 1:
                        br.append(t & 1)
                        continue
                    emit_eobrun()
                    sc.huff(1, c, (r << 4) | 1)
                    sc.bits(0 if blk[JW.ZIGZAG[k]] < 0 else 1, 1)
                    for b in br:
                        sc.bits(b, 1)
                    br, r = [], 0
                if r or br:
                    state["eobrun"] += 1
                    state["be"] += br
                    if state["eobrun"] == 0x7FFF or len(state["be"]) > 937:
                        emit_eobrun()
    if state["eobrun"]:
        sc.note("eobrun_at_end")
    emit_eobrun()
    return sc


STAT_KEYS = (["eob_across", "corr_across", "rst_across", "ff00_across", "max_eobrun", "zrl_first", "zrl_refine",
              "corr_after_zrl", "eobrun_at_rst", "eobrun_at_end"]
             + [f"eob{r}_{kind}" for kind in ("first", "refine") for r in range(15)])


def progressive(buf: bytes, script, restart=None, tables="optimal", fill: Sequence[int] = (0,)):
    """``buf`` (a baseline cv2 file) coded again as a progressive file with ``script``: a list of
    (component indices, Ss, Se, Ah, Al) in file order.  ``restart[k]``: scan k's restart interval (default none).
    Every scan gets its own DHT: per-scan ``optimal`` tables or ``long`` ones (codes of 10 to 16 bits).  ``fill``:
    0xFF fill bytes before each RST (cycling) and ``fill[0]`` after each scan, before the next DRI / DHT or the EOI.
    Returns (file bytes, stats), stats over ``STAT_KEYS``:
      *_across          EOBn codes, the correction-bit runs after them, RST markers and stuffed FF 00 pairs that
                        straddle a 256-byte boundary of their scan's segment;
      max_eobrun        the longest EOB run (rounded down to a power of two);
      zrl_first / zrl_refine   ZRL codes in AC first / AC refinement scans;
      corr_after_zrl    refinement ZRL codes followed by correction bits;
      eob{r}_first / eob{r}_refine   EOBn codes of length class r (runs of 2^r .. 2^(r+1) - 1 blocks);
      eobrun_at_rst / eobrun_at_end  EOB runs cut by a restart marker / ending at the scan's last block."""
    src = JW.source(buf)
    sos = buf.find(b"\xff\xda")
    head = bytearray(buf[:sos])
    sof = head.find(b"\xff\xc0")
    head[sof + 1] = 0xC2
    sel = buf[sos + 5:sos + 5 + 2 * src.ncomp]
    cid = [sel[2 * c] for c in range(src.ncomp)]
    out = bytearray(head)
    stats = dict.fromkeys(STAT_KEYS, 0)
    chunk = 256
    for k, (comps, ss, se, ah, al) in enumerate(script):
        rst = restart[k] if restart and k < len(restart) else 0
        sc = _progressive_events(src, comps, ss, se, ah, al, rst)
        for key, v in sc.count.items():
            stats[key] += v
        nres = 0
        freq = {}
        for e in sc.ev:
            if e[0] == "H":
                freq.setdefault((e[1], e[2]), {}).setdefault(e[3], 0)
                freq[(e[1], e[2])][e[3]] += 1
        codes = {}
        dht = b""
        for (tc, c), f in sorted(freq.items()):
            if tables == "long":
                syms = sorted(f)
                lengths = {s: 10 + min(6, i * 7 // max(len(syms), 1)) for i, s in enumerate(syms)}
                t = JW.table_from_lengths(lengths)
            else:
                t = JW.table_from_lengths(JW._optimal_lengths(f))
            codes[(tc, c)] = t.codes()
            dht += JW._dht(tc, c, t)
        out += JW._seg(0xDD, rst.to_bytes(2, "big"))
        if dht:
            out += JW._seg(0xC4, dht)
        payload = bytes([len(comps)]) + b"".join(bytes([cid[c], (c << 4) | c]) for c in comps) + \
            bytes([ss, se, (ah << 4) | al])
        out += JW._seg(0xDA, payload)
        bits = JW._Bits()
        eob_start = None
        for e in sc.ev:
            if e[0] == "H":
                bits.put(*codes[(e[1], e[2])][e[3]])
            elif e[0] == "B":
                bits.put(e[1], e[2])
            elif e[0] == "EOB":
                eob_start = len(bits.out)
                stats["max_eobrun"] = max(stats["max_eobrun"], 1 << e[1])
            elif e[0] == "EOB_END":
                if eob_start // chunk != len(bits.out) // chunk:
                    stats["eob_across"] += 1
                    if ah:
                        stats["corr_across"] += 1
            else:
                bits.flush()
                bits.out += _fill(fill, nres)
                nres += 1
                p = len(bits.out)
                bits.out += bytes([0xFF, 0xD0 + e[1]])
                if p // chunk != (p + 1) // chunk:
                    stats["rst_across"] += 1
        bits.flush()
        seg = bytes(bits.out)
        stats["ff00_across"] += sum(1 for i in range(chunk - 1, len(seg) - 1, chunk) if seg[i] == 0xFF and seg[i + 1] == 0)
        out += seg + _fill(fill, -1)
    out += b"\xff\xd9"
    return bytes(out), stats


def scripts(ncomp: int):
    """name -> (script, restart per scan) for a frame of ``ncomp`` components."""
    allc = list(range(ncomp))
    out = {}
    out["cv2-default"] = ([(allc, 0, 0, 0, 1)] + [([0], 1, 5, 0, 2)] + [([c], 1, 63, 0, 1) for c in allc[1:]]
                          + [([0], 6, 63, 0, 2), ([0], 1, 63, 2, 1), (allc, 0, 0, 1, 0)]
                          + [([c], 1, 63, 1, 0) for c in allc[1:]] + [([0], 1, 63, 1, 0)], None)
    out["per-comp-dc-spectral"] = ([([c], 0, 0, 0, 0) for c in allc]
                                   + [([c], lo, hi, 0, 0) for c in allc for lo, hi in ((1, 5), (6, 20), (21, 63))],
                                   [3, 0, 5, 1, 0, 2, 7, 0, 4, 1, 0, 9][:4 * ncomp])
    deep = [(allc, 0, 0, 0, 3)] + [([c], 1, 63, 0, 4) for c in allc]
    for a in (3, 2, 1, 0):
        deep += [([c], 1, 63, a + 1, a) for c in allc]
    for a in (2, 1, 0):
        deep += [(allc, 0, 0, a + 1, a)]
    out["deep-sa"] = (deep, [2 if k % 2 else 0 for k in range(len(deep))])
    one = [(allc, 0, 0, 0, 1), (allc, 0, 0, 1, 0)]
    for k in range(1, 64):
        for c in allc:
            one += [([c], k, k, 0, 1)]
    for k in range(1, 64):
        for c in allc:
            one += [([c], k, k, 1, 0)]
    out["one-coef-bands"] = (one, None)
    mixed = [([c], 0, 0, 0, 0) for c in allc[::-1]]
    for lo, hi in ((1, 2), (3, 9), (10, 63)):
        for c in allc:
            mixed += [([c], lo, hi, 0, 2)]
    for a in (1, 0):
        for c in allc[::-1]:
            mixed += [([c], 1, 63, a + 1, a)]
    out["components-interleaved-in-file-order"] = (mixed, [1, 4] * (len(mixed) // 2 + 1))
    return out
