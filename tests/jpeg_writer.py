"""A test-side baseline / extended-sequential JPEG stream writer (T.81 Annex B, F.1.2 and K.2).

It takes quantised coefficient planes (what ``oracle.jpeg_ref.coefficients`` returns for a real encoder's file)
and writes them again with other choices than cv2 makes, so the decoder sees the streams other encoders write:

* Huffman tables per component (ids 0-3): the source's own, optimal from symbol counts, ``long`` (every code 10-16
  bits, past the decoder's 9-bit lookup), ``short`` (fixed 4-bit DC and 8-bit AC codes), ``skewed`` (a 1-bit code
  for the most frequent symbol), or any Kraft-valid length assignment (``table_from_lengths``);
* quantisation tables per component (ids 0-3), 8-bit or 16-bit precision (``Pq = 1``, written with SOF1);
* restart intervals, an explicit DRI of 0, a DRI given twice, a trailing RST after the last MCU;
* 0xFF fill bytes before every RST and before the EOI (T.81 B.1.1.2);
* several tables per DHT / DQT segment, tables redefined before the SOS, component ids, JFIF / EXIF / Adobe / no
  APPn, COM and APP2 segments, and 2x2 sampling factors on a grey frame.

No forward DCT: the coefficients are written as given, so ``coefficients(write(src, ...))`` is ``src.coef``.
"""
from __future__ import annotations

import heapq
import struct
from dataclasses import dataclass
from typing import List, Optional, Sequence

import numpy as np

from acr_b200 import jpeg
from oracle import jpeg_ref

ZIGZAG = jpeg.ZIGZAG


@dataclass
class Source:
    """Quantised coefficients of one frame and the headers that place them."""
    H: int
    W: int
    comp_hv: List[tuple]        # SOF sampling factors (h, v) per component
    coef: List[np.ndarray]      # per component (block rows, blocks per row, 64) int16, natural order
    quant: np.ndarray           # (ncomp, 64) uint16, natural order
    dc: list                    # the source's HuffTables per component
    ac: list

    @property
    def ncomp(self) -> int:
        return len(self.coef)

    @property
    def hmax(self) -> int:
        return max(h for h, _ in self.comp_hv) if self.ncomp > 1 else 1

    @property
    def vmax(self) -> int:
        return max(v for _, v in self.comp_hv) if self.ncomp > 1 else 1

    @property
    def mcus(self) -> tuple:
        """(mcus_x, mcus_y): a one-component scan is not interleaved, one block per MCU."""
        return -(-self.W // (8 * self.hmax)), -(-self.H // (8 * self.vmax))


def source(buf: bytes) -> Source:
    info = jpeg.parse(buf)
    hv = [(info.comp_h[c], info.comp_v[c]) for c in range(info.ncomp)]
    return Source(info.H, info.W, hv, jpeg_ref.coefficients(buf, info), info.quant.copy(), info.dc, info.ac)


# ---- Huffman tables ------------------------------------------------------------------------------------------------
@dataclass
class Table:
    """A canonical Huffman table: ``bits[l]`` codes of length l (1..16), ``vals`` in code order."""
    bits: np.ndarray
    vals: np.ndarray

    def codes(self) -> dict:
        """symbol -> (code, length), canonical (T.81 C.2)."""
        out, code, k = {}, 0, 0
        for l in range(1, 17):
            for _ in range(int(self.bits[l])):
                out[int(self.vals[k])] = (code, l)
                code += 1
                k += 1
            code <<= 1
        return out

    def lengths(self) -> List[int]:
        return [l for l in range(1, 17) for _ in range(int(self.bits[l]))]


def table_from_lengths(length_of: dict) -> Table:
    """symbol -> code length (1..16) -> Table.  The lengths must leave the all-ones code of every length free."""
    if not length_of:
        raise ValueError("a Huffman table needs at least one symbol")
    if max(length_of.values()) > 16 or min(length_of.values()) < 1:
        raise ValueError("code lengths must be 1..16")
    if sum(2.0 ** -l for l in length_of.values()) >= 1.0:
        raise ValueError("lengths not Kraft-valid with the all-ones code reserved")
    bits = np.zeros(17, np.int32)
    for l in length_of.values():
        bits[l] += 1
    vals = np.array(sorted(length_of, key=lambda s: (length_of[s], s)), np.uint8)
    return Table(bits, vals)


def _optimal_lengths(freq: dict) -> dict:
    """Code lengths of a length-limited (16) Huffman code for symbol -> count, with the all-ones code reserved:
    T.81 K.2 (a pseudo-symbol of count 1 takes the all-ones code) and K.3 (lengths over 16 adjusted)."""
    syms = sorted(freq)
    items = [(max(int(freq[s]), 1), k, [k]) for k, s in enumerate(syms)] + [(1, len(syms), [len(syms)])]
    size = [0] * (len(syms) + 1)
    if len(items) == 1:
        size[0] = 1
    heapq.heapify(items)
    tie = len(items)
    while len(items) > 1:
        f1, _, a = heapq.heappop(items)
        f2, _, b = heapq.heappop(items)
        for k in a + b:
            size[k] += 1
        heapq.heappush(items, (f1 + f2, tie, a + b))
        tie += 1
    bits = np.zeros(40, np.int64)
    for s in size:
        bits[s] += 1
    for i in range(39, 16, -1):                      # K.3 Adjust_BITS
        while bits[i] > 0:
            j = i - 2
            while bits[j] == 0:
                j -= 1
            bits[i] -= 2
            bits[i - 1] += 1
            bits[j + 1] += 2
            bits[j] -= 1
    i = 16
    while bits[i] == 0:
        i -= 1
    bits[i] -= 1                                     # drop the pseudo-symbol's (longest) code
    order = sorted(range(len(syms)), key=lambda k: (-freq[syms[k]], syms[k]))
    lens = [l for l in range(1, 17) for _ in range(int(bits[l]))]
    return {syms[k]: l for k, l in zip(order, lens)}


def symbol_counts(src: Source, restart: int = 0) -> tuple:
    """Per component, the DC and AC symbol counts of src's coefficients as a scan with this restart interval
    codes them."""
    dc = [dict() for _ in range(src.ncomp)]
    ac = [dict() for _ in range(src.ncomp)]
    for c, tc, sym, _, _ in _symbols(src, restart):
        if c == RST:
            continue
        t = (ac if tc else dc)[c]
        t[sym] = t.get(sym, 0) + 1
    return dc, ac


def _all_symbols(counts: dict, ac: bool) -> dict:
    """counts plus every other symbol an 8-bit sequential scan may code (count 0), for the fixed-shape presets."""
    full = dict(counts)
    if ac:
        for r in range(16):
            for s in range(1, 11):
                full.setdefault((r << 4) | s, 0)
        full.setdefault(0xF0, 0)
    else:
        for s in range(12):
            full.setdefault(s, 0)
    return full


def preset_tables(src: Source, kind: str, restart: int = 0):
    """(dc tables, ac tables) per component for a preset: 'source', 'optimal' (from the symbol counts of a scan
    with this restart interval), 'long', 'short' or 'skewed'."""
    if kind == "source":
        return ([Table(t.bits, t.vals) for t in src.dc], [Table(t.bits, t.vals) for t in src.ac])
    dcs, acs = symbol_counts(src, restart)
    out = ([], [])
    for c in range(src.ncomp):
        for k, (cnt, is_ac) in enumerate(((dcs[c], False), (acs[c], True))):
            if kind == "optimal":
                lens = _optimal_lengths(cnt)
            elif kind == "skewed":
                top = max(cnt, key=lambda s: (cnt[s], -s))
                boosted = _all_symbols(cnt, is_ac)
                boosted[top] = 4 * sum(cnt.values()) + 4
                lens = _optimal_lengths(boosted)
                assert lens[top] == 1
            elif kind == "long":       # lengths cycle 10, 11, ..., 16 in frequency order
                syms = sorted(_all_symbols(cnt, is_ac), key=lambda s: (-cnt.get(s, 0), s))
                lens = {s: 10 + i % 7 for i, s in enumerate(syms)}
            elif kind == "short":      # fixed length: 4 bits DC, 8 bits AC
                syms = sorted(_all_symbols(cnt, is_ac))
                lens = {s: 8 if is_ac else 4 for s in syms}
            else:
                raise ValueError(kind)
            out[k].append(table_from_lengths(lens))
    return out


# ---- the scan ------------------------------------------------------------------------------------------------------
class _Bits:
    def __init__(self):
        self.out = bytearray()
        self.acc = 0
        self.n = 0

    def put(self, v: int, n: int):
        if n == 0:
            return
        self.acc = (self.acc << n) | (v & ((1 << n) - 1))
        self.n += n
        while self.n >= 8:
            self.n -= 8
            byte = (self.acc >> self.n) & 0xFF
            self.out.append(byte)
            if byte == 0xFF:
                self.out.append(0)                   # byte stuffing
        self.acc &= (1 << self.n) - 1

    def flush(self):
        """Pad the last byte with ones (T.81 F.1.2.3)."""
        if self.n:
            self.put((1 << (8 - self.n)) - 1, 8 - self.n)


def _slots(src: Source):
    if src.ncomp == 1:
        return [(0, 0, 0)]
    return [(c, dy, dx) for c, (h, v) in enumerate(src.comp_hv) for dy in range(v) for dx in range(h)]


RST = -1


def _symbols(src: Source, restart: int):
    """The scan as (component, table class 0 = DC / 1 = AC, symbol, extra bits value, extra bits length), with
    (RST, ...) where a restart interval ends (T.81 F.1.2)."""
    mx_n, my_n = src.mcus
    slots = _slots(src)
    pred = [0] * src.ncomp
    for m in range(mx_n * my_n):
        if restart and m and m % restart == 0:
            yield RST, 0, 0xD0 + (m // restart - 1) % 8, 0, 0
            pred = [0] * src.ncomp
        my, mx = divmod(m, mx_n)
        for c, dy, dx in slots:
            h, v = (1, 1) if src.ncomp == 1 else src.comp_hv[c]
            zz = src.coef[c][my * v + dy, mx * h + dx].astype(np.int64)[ZIGZAG]
            d = int(zz[0]) - pred[c]
            pred[c] = int(zz[0])
            s = abs(d).bit_length()
            yield c, 0, s, d if d >= 0 else d + (1 << s) - 1, s
            nz = np.flatnonzero(zz[1:]) + 1
            k0 = 1
            for k in nz:
                r = int(k) - k0
                while r > 15:
                    yield c, 1, 0xF0, 0, 0
                    r -= 16
                x = int(zz[k])
                s = abs(x).bit_length()
                yield c, 1, (r << 4) | s, x if x >= 0 else x + (1 << s) - 1, s
                k0 = int(k) + 1
            if k0 <= 63:
                yield c, 1, 0x00, 0, 0


def _scan(src: Source, dc: Sequence[Table], ac: Sequence[Table], restart: int, trailing_rst: bool,
          fill: Sequence[int]) -> bytes:
    codes = ([t.codes() for t in dc], [t.codes() for t in ac])
    bw = _Bits()
    nres = 0

    def marker(code):
        nonlocal nres
        bw.flush()
        bw.out += b"\xff" * fill[nres % len(fill)] + bytes([0xFF, code])
        nres += 1

    for c, tc, sym, v, n in _symbols(src, restart):
        if c == RST:
            marker(sym)
            continue
        bw.put(*codes[tc][c][sym])
        bw.put(v, n)
    if trailing_rst:
        mx_n, my_n = src.mcus
        total = mx_n * my_n
        assert restart and total % restart == 0, "a trailing RST follows a whole last interval"
        marker(0xD0 + (total // restart - 1) % 8)
    bw.flush()
    return bytes(bw.out)


# ---- headers -------------------------------------------------------------------------------------------------------
def _seg(m: int, payload: bytes) -> bytes:
    return bytes([0xFF, m]) + struct.pack(">H", len(payload) + 2) + payload


def _dht(tc: int, th: int, t: Table) -> bytes:
    return bytes([(tc << 4) | th]) + bytes(int(b) for b in t.bits[1:17]) + bytes(int(v) for v in t.vals)


def _dqt(tq: int, q: np.ndarray, pq: int) -> bytes:
    zz = q.astype(np.int64)[ZIGZAG]
    return bytes([(pq << 4) | tq]) + (b"".join(struct.pack(">H", int(v)) for v in zz) if pq else
                                      bytes(int(v) for v in zz))


def _same(s: Table, t: Table) -> bool:
    return np.array_equal(s.bits, t.bits) and np.array_equal(s.vals, t.vals)


JFIF = _seg(0xE0, b"JFIF\x00\x01\x01\x00\x00\x01\x00\x01\x00\x00")
ADOBE = _seg(0xEE, b"Adobe\x00\x64\x00\x00\x00\x00\x01")        # transform 1: YCbCr
EXIF = _seg(0xE1, b"Exif\x00\x00" + b"MM\x00\x2a\x00\x00\x00\x08" + b"\x00\x01"
            + b"\x01\x12\x00\x03\x00\x00\x00\x01\x00\x01\x00\x00" + b"\x00\x00\x00\x00")   # orientation 1
APPS = {"jfif": JFIF, "exif": EXIF, "adobe": ADOBE, "none": b""}


def write(src: Source, *, tables="source", quant: Optional[np.ndarray] = None, qprec=(0, 0, 0),
          comp_ids=(1, 2, 3), dc_ids=None, ac_ids=None, q_ids=None, restart=0, dri=None, trailing_rst=False,
          fill=(0,), app="jfif", com=False, app2=False, one_segment=False, redefine=False,
          grey_hv=(1, 1)) -> bytes:
    """One sequential Huffman JPEG file of src's coefficients.

    tables      a preset name (``preset_tables``) or (dc tables, ac tables) per component
    quant       (ncomp, 64) tables written instead of src.quant; qprec: 0 = 8-bit, 1 = 16-bit (then SOF1) each
    *_ids       the table ids (0-3) per component; comp_ids the SOF / SOS component ids
    restart     the restart interval in MCUs; ``dri`` lists the DRI values written in order (the last counts;
                default ``[restart]`` when restart, none otherwise)
    fill        0xFF fill bytes before each RST (cycling through the list) and before the EOI (the first entry)
    app         'jfif', 'exif', 'adobe' or 'none'; com / app2 add a COM and an APP2 segment
    one_segment every table in one DHT and one DQT segment; redefine: each table id first defined with a
                different table, then redefined before the SOS
    grey_hv     the sampling factors a grey frame's SOF gives its one component"""
    nc = src.ncomp
    dc, ac = preset_tables(src, tables, restart) if isinstance(tables, str) else tables
    quant = src.quant if quant is None else np.asarray(quant)
    default = lambda ts: [0] if nc == 1 else [0, 1, 1] if _same(ts[1], ts[2]) else [0, 1, 2]
    dc_ids = list(dc_ids if dc_ids is not None else default(dc))
    ac_ids = list(ac_ids if ac_ids is not None else default(ac))
    q_ids = list(q_ids if q_ids is not None else [0] if nc == 1 else
                 [0, 1, 1] if np.array_equal(quant[1], quant[2]) and qprec[1] == qprec[2] else [0, 1, 2])
    for a in range(nc):       # components that share a table id must share the table
        for b in range(a):
            assert dc_ids[a] != dc_ids[b] or _same(dc[a], dc[b]), ("DC table id", dc_ids[a])
            assert ac_ids[a] != ac_ids[b] or _same(ac[a], ac[b]), ("AC table id", ac_ids[a])
            assert q_ids[a] != q_ids[b] or (np.array_equal(quant[a], quant[b]) and qprec[a] == qprec[b]), \
                ("quantisation table id", q_ids[a])
    ext = any(qprec[c] for c in range(nc))
    out = bytearray(b"\xff\xd8") + APPS[app]
    if com:
        out += _seg(0xFE, b"written by tests/jpeg_writer.py")
    if app2:
        out += _seg(0xE2, b"ICC_PROFILE\x00\x01\x01" + bytes(range(256)) * 2)

    dqt = [_dqt(q_ids[c], quant[c], qprec[c]) for c in dict((q_ids[c], c) for c in range(nc)).values()]
    dht = [_dht(0, dc_ids[c], dc[c]) for c in dict((dc_ids[c], c) for c in range(nc)).values()]
    dht += [_dht(1, ac_ids[c], ac[c]) for c in dict((ac_ids[c], c) for c in range(nc)).values()]
    if redefine:     # a first definition of every id with other contents, superseded before the SOS
        bogus_q = np.full(64, 255, np.uint16)
        bogus_t = table_from_lengths({s: 8 for s in range(1, 200)})
        out += _seg(0xDB, b"".join(_dqt(q_ids[c], bogus_q, 0) for c in range(nc)))
        out += _seg(0xC4, b"".join(_dht(0, i, bogus_t) for i in set(dc_ids)) +
                    b"".join(_dht(1, i, bogus_t) for i in set(ac_ids)))
    if one_segment:
        out += _seg(0xDB, b"".join(dqt))
    else:
        for d in dqt:
            out += _seg(0xDB, d)

    hv = [grey_hv] if nc == 1 else src.comp_hv
    sof = struct.pack(">BHHB", 8, src.H, src.W, nc) + b"".join(
        bytes([comp_ids[c], (hv[c][0] << 4) | hv[c][1], q_ids[c]]) for c in range(nc))
    out += _seg(0xC1 if ext else 0xC0, sof)
    if one_segment:
        out += _seg(0xC4, b"".join(dht))
    else:
        for d in dht:
            out += _seg(0xC4, d)
    for v in (dri if dri is not None else ([restart] if restart else [])):
        out += _seg(0xDD, struct.pack(">H", v))
    sos = bytes([nc]) + b"".join(bytes([comp_ids[c], (dc_ids[c] << 4) | ac_ids[c]]) for c in range(nc)) + \
        b"\x00\x3f\x00"
    out += _seg(0xDA, sos)
    out += _scan(src, dc, ac, restart, trailing_rst, fill if any(fill) else (0,))
    out += b"\xff" * fill[0] + b"\xff\xd9"
    return bytes(out)


def scan_of(buf: bytes) -> bytes:
    info = jpeg.parse(buf)
    return bytes(buf[info.scan_offset:info.scan_offset + info.scan_len])
