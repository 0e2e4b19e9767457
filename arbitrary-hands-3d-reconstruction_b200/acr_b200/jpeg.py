"""JPEG decoding on the device (csrc/jpeg.cu): host header parser, frame and scan descriptors and ``decode``.

The host reads the markers only (SOI, APPn far enough for an EXIF orientation, DQT, SOF0/1/2, DHT, DRI, SOS, EOI)
and builds one ``acr_b200_jpeg_frame`` per file (include/acr_b200.h): sizes, sampling, the quantisation tables in
natural order and the Huffman tables as lookup tables.  The entropy-coded segments travel untouched, packed back
to back; byte stuffing and restart markers are handled on the device.  The output equals
``cv2.imdecode(buf, cv2.IMREAD_COLOR)`` byte for byte (libjpeg-turbo: islow IDCT, fancy upsampling).

Progressive (SOF2) and multi-scan sequential files are decoded when the call gives a scan capacity, ``max_scans`` >
0 (``parse``, ``layout``, ``plan``, ``decode``, ``JpegBatch``): each of their scans gets an ``acr_b200_jpeg_scan``
with the Huffman tables and restart interval in force at its SOS, and its own segment, which ends at the first
marker that is not a stuffed FF 00 or an RST.  The device decodes complete scripts only (every coefficient sent
once, then refined down to Al = 0); libjpeg smooths the blocks of an incomplete one, so those raise
``JpegUnsupported`` and the host fallback gives cv2's pixels.  With ``max_scans = 0`` multi-scan files raise as
single-scan-only decoding always did.

Streams the device does not decode (arithmetic, lossless / hierarchical, 12-bit, CMYK / YCCK / RGB, sampling other
than 4:4:4, 4:2:2, 4:2:0, 4:4:0 and grey, EXIF orientation other than 1, the scripts above) raise
``JpegUnsupported`` naming the feature; ``decode(..., host_fallback=True)`` decodes those with cv2 instead.
"""
from __future__ import annotations

import struct
from dataclasses import dataclass, field
from typing import List, Optional, Sequence, Tuple

import numpy as np

CHUNK = 256   # ACR_B200_JPEG_CHUNK: entropy-coded bytes per decoder thread
MAX_SCAN_BYTES = 1 << 28   # ACR_B200_JPEG_MAX_SCAN_BYTES: a decoder position (byte * 8 + bit) must fit an int32

ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20,
                   13, 6, 7, 14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52,
                   45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63], np.int32)   # zigzag index -> natural index


class JpegError(ValueError):
    """A malformed or truncated JPEG stream."""


class JpegUnsupported(JpegError):
    """A valid JPEG stream that uses a feature the device decoder does not implement."""


@dataclass
class HuffTable:
    bits: np.ndarray        # (17,) number of codes of each length 1..16 (index 0 unused)
    vals: np.ndarray        # symbols in code order
    maxcode: np.ndarray = field(init=False)   # (18,) largest code of each length, -1 if none; [17] sentinel
    valoff: np.ndarray = field(init=False)    # (18,) symbol index of code c of length l = c + valoff[l]
    lut: np.ndarray = field(init=False)       # (512,) 9-bit lookahead: (length << 8) | symbol, 0 for longer codes

    def __post_init__(self):
        self.maxcode = np.full(18, -1, np.int32)
        self.valoff = np.zeros(18, np.int32)
        self.lut = np.zeros(512, np.uint16)
        code, p = 0, 0
        for l in range(1, 17):
            n = int(self.bits[l])
            if n:
                if code + n >= (1 << l):
                    # the all-ones code of every length is reserved (T.81 C.2): padding bits are ones
                    raise JpegError("bad Huffman table: codes overflow or use the all-ones code")
                self.valoff[l] = p - code
                for k in range(n):
                    if l <= 9:
                        c = code + k
                        self.lut[c << (9 - l):(c + 1) << (9 - l)] = (l << 8) | int(self.vals[p + k])
                self.maxcode[l] = code + n - 1
                p += n
                code += n
            code <<= 1
        self.maxcode[17] = 0x7fffffff


@dataclass
class JpegInfo:
    H: int
    W: int
    ncomp: int
    comp_h: List[int]           # sampling factors per component (1 or 2; grey is (1, 1))
    comp_v: List[int]
    hmax: int
    vmax: int
    mcus_x: int
    mcus_y: int
    slots: List[Tuple[int, int, int]]    # (component, dy, dx) of each block of an MCU, in coding order
    quant: np.ndarray           # (ncomp, 64) uint16, natural order
    dc: List[HuffTable]
    ac: List[HuffTable]
    restart: int                # restart interval in MCUs, 0 = none
    scan_offset: int            # entropy-coded segment: bytes [scan_offset, scan_offset + scan_len) of the file
    scan_len: int               # (a multi-scan file: the first scan's offset and every scan's bytes together)
    scans: List["ScanInfo"] = field(default_factory=list)   # a multi-scan file's scans in file order, else empty

    @property
    def bpm(self) -> int:
        return len(self.slots)

    def comp_blocks(self, c: int) -> Tuple[int, int]:
        """(blocks per row, block rows) of component c's plane, padded to whole MCUs."""
        return self.mcus_x * self.comp_h[c], self.mcus_y * self.comp_v[c]

    def comp_size(self, c: int) -> Tuple[int, int]:
        """(width, height) in samples of component c (libjpeg's downsampled_width / _height)."""
        return (-(-self.W * self.comp_h[c] // self.hmax), -(-self.H * self.comp_v[c] // self.vmax))

    @property
    def n_blocks(self) -> int:
        return self.mcus_x * self.mcus_y * self.bpm

    @property
    def n_chunks(self) -> int:
        if self.scans:
            return sum(s.n_chunks for s in self.scans)
        return max(1, -(-self.scan_len // CHUNK))


@dataclass
class ScanInfo:
    """One scan of a multi-scan file.  An interleaved scan (several components) codes the frame's MCUs, with
    ``slots`` in scan order; a one-component scan codes that component's own blocks, ceil(w / 8) x ceil(h / 8) in
    raster order (``mcus_x`` x ``mcus_y``, one slot), not the MCU-padded plane."""
    comps: List[int]            # frame component indices, scan order
    ss: int
    se: int
    ah: int
    al: int
    restart: int                # restart interval in MCUs (in blocks for a one-component scan), 0 = none
    offset: int                 # entropy-coded segment: bytes [offset, offset + length) of the file
    length: int
    mcus_x: int
    mcus_y: int
    slots: List[Tuple[int, int, int]]
    dc: dict                    # frame component -> HuffTable the scan uses
    ac: dict

    @property
    def refine(self) -> bool:
        return self.ah != 0

    @property
    def n_blocks(self) -> int:
        return self.mcus_x * self.mcus_y * len(self.slots)

    @property
    def n_chunks(self) -> int:
        return max(1, -(-self.length // CHUNK))


_SOF_NAMES = {0xC2: "progressive", 0xC3: "lossless", 0xC5: "hierarchical (differential sequential)",
              0xC6: "hierarchical (differential progressive)", 0xC7: "hierarchical (differential lossless)",
              0xC9: "arithmetic coding", 0xCA: "arithmetic coding (progressive)",
              0xCB: "arithmetic coding (lossless)", 0xCD: "arithmetic coding (differential sequential)",
              0xCE: "arithmetic coding (differential progressive)", 0xCF: "arithmetic coding (differential lossless)"}
_SAMPLINGS = {(1, 1): "4:4:4", (2, 1): "4:2:2", (2, 2): "4:2:0", (1, 2): "4:4:0"}


def _exif_orientation(seg: bytes) -> Optional[int]:
    """Orientation tag (0x0112) of IFD0 of an APP1 Exif payload, or None."""
    if len(seg) < 14 or seg[:6] != b"Exif\x00\x00":
        return None
    t = seg[6:]
    if t[:2] == b"II":
        e = "<"
    elif t[:2] == b"MM":
        e = ">"
    else:
        return None
    try:
        ifd = struct.unpack(e + "I", t[4:8])[0]
        n = struct.unpack(e + "H", t[ifd:ifd + 2])[0]
        for k in range(n):
            o = ifd + 2 + 12 * k
            tag, typ, cnt = struct.unpack(e + "HHI", t[o:o + 8])
            if tag == 0x0112 and typ == 3:
                return struct.unpack(e + "H", t[o + 8:o + 10])[0]
    except struct.error:
        return None
    return None


def _dht(seg: bytes, dht: dict) -> None:
    i = 0
    while i < len(seg):
        if i + 17 > len(seg):
            raise JpegError("bad DHT segment")
        tc, th = seg[i] >> 4, seg[i] & 15
        bits = np.zeros(17, np.int32)
        bits[1:] = np.frombuffer(seg[i + 1:i + 17], np.uint8)
        cnt = int(bits.sum())
        if tc > 1 or th > 3 or cnt > 256 or i + 17 + cnt > len(seg):
            raise JpegError("bad DHT segment")
        dht[(tc, th)] = HuffTable(bits, np.frombuffer(seg[i + 17:i + 17 + cnt], np.uint8).copy())
        i += 17 + cnt


def _dqt(seg: bytes, qt: list, used=()) -> None:
    i = 0
    while i < len(seg):
        pq, tq = seg[i] >> 4, seg[i] & 15
        sz = 128 if pq else 64
        if tq > 3 or pq > 1 or i + 1 + sz > len(seg):
            raise JpegError("bad DQT segment")
        if tq in used:
            raise JpegUnsupported("a DQT that redefines a quantisation table a component has already used is not "
                                  "supported on the device")
        vals = (np.frombuffer(seg[i + 1:i + 1 + sz], ">u2") if pq else
                np.frombuffer(seg[i + 1:i + 65], np.uint8)).astype(np.uint16)
        q = np.zeros(64, np.uint16)
        q[ZIGZAG] = vals
        qt[tq] = q
        i += 1 + sz


def _geometry(H, W, comps, jfif, adobe_transform):
    """Sampling checks and the frame's MCU geometry -> (comp_h, comp_v, hmax, vmax, mcus_x, mcus_y, slots)."""
    nc = len(comps)
    ids = [c[0] for c in comps]
    if nc == 3:
        rgb = (not jfif) and (adobe_transform == 0 if adobe_transform is not None else ids == [82, 71, 66])
        if rgb:
            raise JpegUnsupported("RGB JPEG (no YCbCr transform) is not supported on the device")
        hv = [(h, v) for _, h, v, _ in comps]
        if hv[1] != (1, 1) or hv[2] != (1, 1) or hv[0] not in _SAMPLINGS:
            raise JpegUnsupported("sampling factors " + ",".join(f"{h}x{v}" for h, v in hv) + " are not supported "
                                  "on the device (4:4:4, 4:2:2, 4:2:0 and 4:4:0 only)")
        hmax, vmax = hv[0]
        comp_h, comp_v = [hmax, 1, 1], [vmax, 1, 1]
        mcus_x, mcus_y = -(-W // (8 * hmax)), -(-H // (8 * vmax))
        slots = [(0, dy, dx) for dy in range(vmax) for dx in range(hmax)] + [(1, 0, 0), (2, 0, 0)]
    else:
        hmax = vmax = 1      # a one-component scan is not interleaved: one block per MCU, whatever the factors
        comp_h, comp_v = [1], [1]
        mcus_x, mcus_y = -(-W // 8), -(-H // 8)
        slots = [(0, 0, 0)]
    return comp_h, comp_v, hmax, vmax, mcus_x, mcus_y, slots


def segment_end(b: bytes, pos: int) -> int:
    """End of the entropy-coded segment that starts at ``pos``: the FF of the first marker that is not a stuffed
    FF 00 or an RST, after any FF fill bytes (which stay in the segment); -1 when the file ends first."""
    n = len(b)
    i = pos
    while True:
        i = b.find(b"\xff", i)
        if i < 0:
            return -1
        j = i + 1
        while j < n and b[j] == 0xFF:
            j += 1
        if j >= n:
            return -1
        if b[j] == 0 or 0xD0 <= b[j] <= 0xD7:
            i = j + 1
            continue
        return j - 1


def parse(buf, max_scans: int = 0) -> JpegInfo:
    """Read the headers of one JPEG file (bytes-like) -> JpegInfo.  Raises JpegUnsupported (feature named) or
    JpegError.  Reads the markers only: the entropy-coded segment of a single-scan file runs from the end of the SOS
    header to the first EOI after it.

    ``max_scans`` > 0 also reads progressive (SOF2) and multi-scan sequential files (see ``_parse_scans``); such a
    file with more than ``max_scans`` scans raises ValueError.  With 0 they raise JpegUnsupported."""
    b = bytes(buf)
    n = len(b)
    if n < 4 or b[0] != 0xFF or b[1] != 0xD8:
        raise JpegError("not a JPEG stream (no SOI marker)")
    pos = 2
    qt = [None] * 4
    dht = {}
    restart = 0
    sof = None
    progressive = False
    adobe_transform = None
    jfif = False
    while True:
        while pos < n and b[pos] == 0xFF and pos + 1 < n and b[pos + 1] == 0xFF:
            pos += 1                                            # fill bytes
        if pos + 4 > n or b[pos] != 0xFF:
            raise JpegError("truncated or corrupt header: expected a marker")
        m = b[pos + 1]
        L = (b[pos + 2] << 8) | b[pos + 3]
        if L < 2 or pos + 2 + L > n:
            raise JpegError(f"truncated marker segment 0x{m:02X}")
        seg = b[pos + 4:pos + 2 + L]
        pos += 2 + L
        if m in _SOF_NAMES and not (m == 0xC2 and max_scans > 0):
            raise JpegUnsupported(f"{_SOF_NAMES[m]} JPEG is not supported on the device")
        if m == 0xCC:
            raise JpegUnsupported("arithmetic coding (DAC marker) is not supported on the device")
        if m == 0xE0 and seg[:5] == b"JFIF\x00":
            jfif = True
        elif m == 0xE1:
            o = _exif_orientation(seg)
            if o is not None and o != 1:
                raise JpegUnsupported(f"EXIF orientation {o} (a rotated or mirrored image) is not supported "
                                      "on the device")
        elif m == 0xEE and seg[:5] == b"Adobe" and len(seg) >= 12:
            adobe_transform = seg[11]
        elif m == 0xDB:
            _dqt(seg, qt)
        elif m == 0xC4:
            _dht(seg, dht)
        elif m == 0xDD:
            if len(seg) != 2:
                raise JpegError("bad DRI segment")
            restart = (seg[0] << 8) | seg[1]
        elif m in (0xC0, 0xC1, 0xC2):
            if len(seg) < 6:
                raise JpegError("bad SOF segment")
            P, H, W, nc = seg[0], (seg[1] << 8) | seg[2], (seg[3] << 8) | seg[4], seg[5]
            if P != 8:
                raise JpegUnsupported(f"{P}-bit samples are not supported on the device (8-bit only)")
            if H == 0:
                raise JpegUnsupported("a height defined by a DNL marker is not supported on the device")
            if W == 0 or len(seg) != 6 + 3 * nc:
                raise JpegError("bad SOF segment")
            if nc == 4:
                raise JpegUnsupported("CMYK / YCCK (4 components) is not supported on the device")
            if nc not in (1, 3):
                raise JpegUnsupported(f"{nc} components are not supported on the device")
            comps = [(seg[6 + 3 * k], seg[7 + 3 * k] >> 4, seg[7 + 3 * k] & 15, seg[8 + 3 * k]) for k in range(nc)]
            if any(not (1 <= h <= 4 and 1 <= v <= 4) or tq > 3 for _, h, v, tq in comps):
                raise JpegError("bad SOF segment")
            sof = (H, W, comps)
            progressive = m == 0xC2
        elif m == 0xDA:
            break
        elif m == 0xD9:
            raise JpegError("EOI before the first scan")
        elif 0xD0 <= m <= 0xD7 or m == 0x01:
            raise JpegError(f"unexpected marker 0x{m:02X} in the header")
    if sof is None:
        raise JpegError("no SOF marker before the scan")
    H, W, comps = sof
    nc = len(comps)
    if max_scans > 0 and len(seg) >= 1 and (progressive or seg[0] < nc):
        return _parse_scans(b, pos, seg, H, W, comps, _geometry(H, W, comps, jfif, adobe_transform), qt, dht,
                            restart, progressive, max_scans)
    if len(seg) < 1 or seg[0] != nc or len(seg) != 4 + 2 * nc:
        if len(seg) >= 1 and seg[0] < nc:
            raise JpegUnsupported("multi-scan sequential JPEG (a scan with fewer components than the frame) is "
                                  "not supported on the device")
        raise JpegError("bad SOS segment")
    ss, se, ahal = seg[1 + 2 * nc], seg[2 + 2 * nc], seg[3 + 2 * nc]
    if ss != 0 or se != 63 or ahal != 0:
        raise JpegError("bad SOS spectral selection for a sequential scan")
    ids = [c[0] for c in comps]
    sel = [(seg[1 + 2 * k], seg[2 + 2 * k] >> 4, seg[2 + 2 * k] & 15) for k in range(nc)]
    if [s[0] for s in sel] != ids:
        raise JpegError("SOS components do not match the frame's")
    comp_h, comp_v, hmax, vmax, mcus_x, mcus_y, slots = _geometry(H, W, comps, jfif, adobe_transform)
    quant = np.zeros((nc, 64), np.uint16)
    dc, ac = [], []
    for k, (_, _, _, tq) in enumerate(comps):
        if qt[tq] is None:
            raise JpegError(f"component {k} uses an undefined quantisation table")
        quant[k] = qt[tq]
        td, ta = sel[k][1], sel[k][2]
        if (0, td) not in dht or (1, ta) not in dht:
            raise JpegError(f"component {k} uses an undefined Huffman table")
        dc.append(dht[(0, td)])
        ac.append(dht[(1, ta)])
    # Inside entropy-coded data an FF is followed by 00 (stuffing) or D0..D7 (restart), so the first EOI after the
    # SOS header ends the scan; whatever follows it (an appended MPF preview, a motion-photo trailer) is not decoded.
    end = b.find(b"\xff\xd9", pos)
    if end < 0:
        raise JpegError("truncated stream: no EOI marker after the scan")
    if end - pos >= MAX_SCAN_BYTES:
        raise JpegUnsupported(f"an entropy-coded segment of {end - pos} bytes is not supported on the device "
                              f"(at most {MAX_SCAN_BYTES - 1})")
    return JpegInfo(H, W, nc, comp_h, comp_v, hmax, vmax, mcus_x, mcus_y, slots, quant, dc, ac, restart,
                    pos, end - pos)


def _parse_scans(b, pos, seg, H, W, comps, geom, qt, dht, restart, progressive, max_scans) -> JpegInfo:
    """The scans of a progressive or multi-scan sequential file, from the first SOS header (``seg``, which ends at
    ``pos``) to the EOI.  Each scan gets the Huffman tables and restart interval in force at its SOS, and its
    segment ends at the first marker that is not a stuffed FF 00 or an RST (``segment_end``).

    The device decodes complete scripts only, each coefficient sent once by a first scan and then refined bit by
    bit down to Al = 0: libjpeg smooths the blocks of an incomplete script (so no plain IDCT gives cv2's pixels),
    and it lets a later first scan overwrite a coefficient, which the device, running first scans in parallel,
    cannot.  Those scripts, and the ones libjpeg only warns about, raise JpegUnsupported; the ones libjpeg rejects
    (JERR_BAD_PROGRESSION) raise JpegError."""
    n = len(b)
    nc = len(comps)
    ids = [c[0] for c in comps]
    comp_h, comp_v, hmax, vmax, mcus_x, mcus_y, slots = geom
    info = JpegInfo(H, W, nc, comp_h, comp_v, hmax, vmax, mcus_x, mcus_y, slots, np.zeros((nc, 64), np.uint16),
                    [], [], 0, pos, 0)
    latched = [False] * nc
    used_q = set()
    sent = np.full((nc, 64), -1, np.int32)   # Al the last scan left each coefficient at, -1 = never sent
    scans = []
    while True:
        ns = seg[0] if len(seg) else 0
        if ns < 1 or ns > nc or len(seg) != 4 + 2 * ns:
            raise JpegError("bad SOS segment")
        sel = []
        for k in range(ns):
            cid = seg[1 + 2 * k]
            if cid not in ids:
                raise JpegError("SOS names a component the frame does not have")
            ci = ids.index(cid)
            if any(ci == s[0] for s in sel):
                raise JpegError("SOS names a component twice")
            sel.append((ci, seg[2 + 2 * k] >> 4, seg[2 + 2 * k] & 15))
        ss, se, ah, al = seg[1 + 2 * ns], seg[2 + 2 * ns], seg[3 + 2 * ns] >> 4, seg[3 + 2 * ns] & 15
        if progressive:
            bad = se != 0 if ss == 0 else (ss > se or se > 63 or ns != 1)
            if bad or (ah != 0 and al != ah - 1) or al > 13:
                raise JpegError(f"bad progression: Ss={ss} Se={se} Ah={ah} Al={al} over {ns} components")
        elif ss != 0 or se != 63 or ah or al:
            raise JpegError("bad SOS spectral selection for a sequential scan")
        dc, ac = {}, {}
        for ci, td, ta in sel:
            tq = comps[ci][3]
            if qt[tq] is None:
                raise JpegError(f"component {ci} uses an undefined quantisation table")
            if not latched[ci]:
                info.quant[ci] = qt[tq]
                latched[ci] = True
                used_q.add(tq)
            if ss == 0 and ah == 0:
                if (0, td) not in dht:
                    raise JpegError(f"component {ci} uses an undefined Huffman table")
                dc[ci] = dht[(0, td)]
            if se > 0:
                if (1, ta) not in dht:
                    raise JpegError(f"component {ci} uses an undefined Huffman table")
                ac[ci] = dht[(1, ta)]
            band = sent[ci, ss:se + 1]
            if not progressive:
                if (band >= 0).any():
                    raise JpegUnsupported("a multi-scan sequential file that codes a component twice is not "
                                          "supported on the device")
            elif ss > 0 and sent[ci, 0] < 0:
                raise JpegUnsupported("a progressive AC scan before the component's first DC scan is not supported "
                                      "on the device")
            elif ah == 0 and (band >= 0).any():
                raise JpegUnsupported("a progressive script that sends a coefficient by two first scans is not "
                                      "supported on the device")
            elif ah != 0 and (band != ah).any():
                raise JpegUnsupported("a progressive refinement scan whose Ah is not the previous Al of its "
                                      "coefficients is not supported on the device")
            band[:] = al
        if ns > 1:
            sx, sy = mcus_x, mcus_y
            sslots = [(ci, dy, dx) for ci, _, _ in sel for dy in range(comp_v[ci]) for dx in range(comp_h[ci])]
        else:
            w, h = info.comp_size(sel[0][0])
            sx, sy, sslots = -(-w // 8), -(-h // 8), [(sel[0][0], 0, 0)]
        end = segment_end(b, pos)
        if end < 0:
            raise JpegError("truncated stream: no marker after a scan")
        if end - pos >= MAX_SCAN_BYTES:
            raise JpegUnsupported(f"an entropy-coded segment of {end - pos} bytes is not supported on the device "
                                  f"(at most {MAX_SCAN_BYTES - 1})")
        scans.append(ScanInfo([s[0] for s in sel], ss, se, ah, al, restart, pos, end - pos, sx, sy, sslots, dc, ac))
        pos = end
        while True:                                           # the markers up to the next SOS or the EOI
            while pos + 1 < n and b[pos + 1] == 0xFF:
                pos += 1
            if pos + 1 >= n:
                raise JpegError("truncated or corrupt header: expected a marker")
            m = b[pos + 1]
            if m == 0xD9:
                break
            if pos + 4 > n:
                raise JpegError("truncated or corrupt header: expected a marker")
            L = (b[pos + 2] << 8) | b[pos + 3]
            if L < 2 or pos + 2 + L > n:
                raise JpegError(f"truncated marker segment 0x{m:02X}")
            seg = b[pos + 4:pos + 2 + L]
            pos += 2 + L
            if m == 0xDA:
                break
            if m == 0xC4:
                _dht(seg, dht)
            elif m == 0xDB:
                _dqt(seg, qt, used_q)
            elif m == 0xDD:
                if len(seg) != 2:
                    raise JpegError("bad DRI segment")
                restart = (seg[0] << 8) | seg[1]
            elif not (0xE0 <= m <= 0xEF or m == 0xFE):
                raise JpegError(f"unexpected marker 0x{m:02X} between scans")
            if pos >= n or b[pos] != 0xFF:
                raise JpegError("truncated or corrupt header: expected a marker")
        if m == 0xD9:
            break
    if progressive and (sent != 0).any():
        raise JpegUnsupported("an incomplete progressive script (a coefficient not refined down to Al = 0) is not "
                              "supported on the device")
    if not progressive and (sent != 0).any():
        raise JpegUnsupported("a multi-scan sequential file that leaves a component uncoded is not supported on "
                              "the device")
    if len(scans) > max_scans:
        raise ValueError(f"the file needs {len(scans)} scans, over the capacity of {max_scans}")
    info.scans = scans
    info.scan_len = sum(s.length for s in scans)
    return info


# ---- descriptors (include/acr_b200.h) -----------------------------------------------------------------------------
HUFF_DTYPE = np.dtype([("lut", "<u2", 512), ("maxcode", "<i4", 18), ("valoff", "<i4", 18), ("huffval", "u1", 256)],
                      align=True)
FRAME_DTYPE = np.dtype([("coded_offset", "<i8"), ("out_offset", "<i8"), ("coef_offset", "<i8"),
                        ("coded_len", "<i4"), ("H", "<i4"), ("W", "<i4"), ("ncomp", "<i4"),
                        ("mcus_x", "<i4"), ("mcus_y", "<i4"), ("bpm", "<i4"), ("restart", "<i4"),
                        ("chunk_begin", "<i4"), ("n_chunks", "<i4"), ("block_begin", "<i4"), ("n_blocks", "<i4"),
                        ("comp_h", "<i4", 3), ("comp_v", "<i4", 3), ("comp_bw", "<i4", 3), ("comp_bh", "<i4", 3),
                        ("comp_w", "<i4", 3), ("comp_hgt", "<i4", 3), ("comp_block0", "<i4", 3), ("n_scans", "<i4"),
                        ("slot_comp", "i1", 8), ("slot_dy", "i1", 8), ("slot_dx", "i1", 8),
                        ("quant", "<u2", (3, 64)), ("dc", HUFF_DTYPE, 3), ("ac", HUFF_DTYPE, 3)], align=True)
SCAN_DTYPE = np.dtype([("coded_offset", "<i8"), ("coded_len", "<i4"), ("frame", "<i4"), ("chunk_begin", "<i4"),
                       ("n_chunks", "<i4"), ("ncomp", "<i4"), ("ss", "<i4"), ("se", "<i4"), ("ah", "<i4"), ("al", "<i4"),
                       ("restart", "<i4"), ("mcus_x", "<i4"), ("mcus_y", "<i4"), ("bpm", "<i4"), ("n_blocks", "<i4"),
                       ("slot_comp", "i1", 8), ("slot_dy", "i1", 8), ("slot_dx", "i1", 8),
                       ("dc", HUFF_DTYPE, 3), ("ac", HUFF_DTYPE, 3)], align=True)
assert HUFF_DTYPE.itemsize == 1424 and FRAME_DTYPE.itemsize == 9112 and SCAN_DTYPE.itemsize == 8632

STATUS_BITS = {1: "a bad Huffman code or an AC run past the block", 2: "the data ends early (truncated file)",
               4: "a restart marker out of place", 8: "a marker inside the entropy-coded data",
               16: "more coded blocks than the frame has", 256: "a descriptor that does not fit the buffers"}


def _fill_huff(rec, t: HuffTable):
    rec["lut"] = t.lut
    rec["maxcode"] = t.maxcode
    rec["valoff"] = t.valoff
    hv = np.zeros(256, np.uint8)
    hv[:len(t.vals)] = t.vals
    rec["huffval"] = hv


@dataclass
class Layout:
    """A batch laid out for acr_b200_jpeg_decode: descriptors, where each file's segment goes in the packed coded
    buffer, and the totals the buffers must hold.  ``infos[i]`` is None for a frame the host decodes instead.
    ``scans``: one descriptor per scan of the multi-scan files, in file order (empty when there are none)."""
    desc: np.ndarray
    infos: list
    coded_bytes: int
    out_bytes: int
    chunks: int
    blocks: int
    scans: np.ndarray = field(default_factory=lambda: np.zeros(0, SCAN_DTYPE))


def layout(encoded: Sequence, host_fallback: bool = False, fallback_shapes=None, max_scans: int = 0) -> Layout:
    """Parse every file and build the batch's descriptors.  Unsupported files raise JpegUnsupported (naming the
    file's index and the feature) unless ``host_fallback``, in which case they get an ncomp = 0 descriptor and
    their (H, W) from ``fallback_shapes[i]`` (decoded by the caller).  ``max_scans`` > 0 lays out progressive and
    multi-scan sequential files too (``parse``): a multi-scan frame has n_scans > 0, and its scans' segments and
    chunks follow one another where a single-scan frame's one segment would be."""
    n = len(encoded)
    if n == 0:
        raise ValueError("a JPEG batch needs at least one file")
    desc = np.zeros(n, FRAME_DTYPE)
    infos = []
    scan_desc = []
    cpos = opos = chunks = blocks = 0
    for i, buf in enumerate(encoded):
        try:
            info = parse(buf, max_scans)
        except JpegUnsupported as e:
            if not host_fallback:
                raise JpegUnsupported(f"file {i}: {e}") from None
            info = None
        except JpegError as e:
            raise JpegError(f"file {i}: {e}") from None
        d = desc[i]
        if info is None:
            H, W = fallback_shapes[i]
            d["H"], d["W"], d["out_offset"] = H, W, opos
            d["chunk_begin"], d["block_begin"], d["coef_offset"] = chunks, blocks, blocks
            opos += H * W * 3
            infos.append(None)
            continue
        infos.append(info)
        d["coded_offset"], d["coded_len"] = cpos, info.scan_len
        d["out_offset"], d["H"], d["W"], d["ncomp"] = opos, info.H, info.W, info.ncomp
        d["mcus_x"], d["mcus_y"], d["bpm"], d["restart"] = info.mcus_x, info.mcus_y, info.bpm, info.restart
        d["chunk_begin"], d["n_chunks"] = chunks, info.n_chunks
        d["block_begin"], d["coef_offset"], d["n_blocks"] = blocks, blocks, info.n_blocks
        b0 = 0
        for c in range(info.ncomp):
            bw, bh = info.comp_blocks(c)
            w, h = info.comp_size(c)
            d["comp_h"][c], d["comp_v"][c], d["comp_bw"][c], d["comp_bh"][c] = info.comp_h[c], info.comp_v[c], bw, bh
            d["comp_w"][c], d["comp_hgt"][c], d["comp_block0"][c] = w, h, b0
            b0 += bw * bh
            d["quant"][c] = info.quant[c]
            if not info.scans:
                _fill_huff(d["dc"][c], info.dc[c])
                _fill_huff(d["ac"][c], info.ac[c])
        for k, (c, dy, dx) in enumerate(info.slots):
            d["slot_comp"][k], d["slot_dy"][k], d["slot_dx"][k] = c, dy, dx
        if info.scans:
            d["restart"] = 0
            d["n_scans"] = len(info.scans)
            sc, sp = chunks, cpos
            for si in info.scans:
                r = np.zeros((), SCAN_DTYPE)
                r["coded_offset"], r["coded_len"], r["frame"] = sp, si.length, i
                r["chunk_begin"], r["n_chunks"], r["ncomp"] = sc, si.n_chunks, len(si.comps)
                r["ss"], r["se"], r["ah"], r["al"], r["restart"] = si.ss, si.se, si.ah, si.al, si.restart
                r["mcus_x"], r["mcus_y"], r["bpm"], r["n_blocks"] = si.mcus_x, si.mcus_y, len(si.slots), si.n_blocks
                for k, (c, dy, dx) in enumerate(si.slots):
                    r["slot_comp"][k], r["slot_dy"][k], r["slot_dx"][k] = c, dy, dx
                for c, t in si.dc.items():
                    _fill_huff(r["dc"][c], t)
                for c, t in si.ac.items():
                    _fill_huff(r["ac"][c], t)
                scan_desc.append(r)
                sc += si.n_chunks
                sp += si.length
        cpos += info.scan_len
        opos += info.H * info.W * 3
        chunks += info.n_chunks
        blocks += info.n_blocks
    scans = np.array(scan_desc, SCAN_DTYPE) if scan_desc else np.zeros(0, SCAN_DTYPE)
    return Layout(desc, infos, cpos, opos, chunks, blocks, scans)


def _round_up(x: int, m: int) -> int:
    return (x + m - 1) // m * m


class JpegBatch:
    """Device buffers for decoding batches of up to ``max_frames`` JPEG files with at most ``max_coded_bytes``
    entropy-coded bytes, ``max_frame_bytes`` decoded BGR bytes, ``max_chunks`` chunks and ``max_blocks`` blocks in
    all, and at most ``max_scans`` scans over the multi-scan files (0: single-scan files only, the launches of
    acr_b200_jpeg_decode; otherwise acr_b200_jpeg_decode_scans, whatever the batch holds).  One device buffer holds
    the descriptors and then the packed coded bytes, so one H2D copy from one pinned staging buffer carries a batch.
    ``load`` checks and copies, ``launch`` enqueues the decode; the buffers never move, so a CUDA graph can capture
    ``launch`` once and replay it after every ``load``."""

    def __init__(self, max_frames: int, max_coded_bytes: int, max_frame_bytes: int, max_chunks: int,
                 max_blocks: int, device=None, out=None, max_scans: int = 0):
        import torch
        if min(max_frames, max_chunks, max_blocks) < 1 or max_frame_bytes < 3 * max_frames or max_coded_bytes < 0 \
                or max_scans < 0:
            raise ValueError("JpegBatch: capacities must be positive")
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        self.max_frames, self.max_coded_bytes, self.max_frame_bytes = max_frames, max_coded_bytes, max_frame_bytes
        self.max_chunks, self.max_blocks, self.max_scans = max_chunks, max_blocks, max_scans
        from . import lib as L
        self.frame_bytes = _round_up(max_frames * FRAME_DTYPE.itemsize, 256)
        self.meta_bytes = self.frame_bytes + _round_up(max_scans * SCAN_DTYPE.itemsize, 256)
        ws = (L.load().acr_b200_jpeg_scan_workspace_bytes(max_chunks, max_blocks, max_scans) if max_scans else
              L.load().acr_b200_jpeg_workspace_bytes(max_chunks, max_blocks))
        dev = self.device
        self.buf = torch.empty(self.meta_bytes + max(max_coded_bytes, 1), dtype=torch.uint8, device=dev)
        self.workspace = torch.empty(ws, dtype=torch.uint8, device=dev)
        # ``out``: a caller's uint8 device buffer of at least max_frame_bytes bytes to decode into
        self.out = torch.empty(max_frame_bytes, dtype=torch.uint8, device=dev) if out is None else out
        self.status = torch.zeros(max_frames, dtype=torch.int32, device=dev)
        self._stage = torch.empty(self.meta_bytes + max(max_coded_bytes, 1), dtype=torch.uint8, pin_memory=True)
        self._copied = None
        self.layout = None
        self.n = 0

    def check(self, lay: Layout, exact: bool = False) -> None:
        """Raise ValueError when a laid-out batch does not fit the capacities (before anything is enqueued)."""
        n = len(lay.desc)
        if exact and n != self.max_frames:
            raise ValueError(f"this JPEG batch takes exactly {self.max_frames} files, got {n}")
        for what, got, cap in (("files", n, self.max_frames), ("entropy-coded bytes", lay.coded_bytes,
                                                                 self.max_coded_bytes),
                               ("decoded BGR bytes", lay.out_bytes, self.max_frame_bytes),
                               ("decoder chunks", lay.chunks, self.max_chunks),
                               ("coefficient blocks", lay.blocks, self.max_blocks),
                               ("scans of multi-scan files", len(lay.scans), self.max_scans)):
            if got > cap:
                raise ValueError(f"the batch needs {got} {what}, over the capacity of {cap}")

    def load(self, encoded: Sequence, lay: Layout) -> None:
        """Copy the descriptors and the entropy-coded segments of ``encoded`` (laid out as ``lay``, which
        ``check`` accepted) into the device buffer, on the current stream: one H2D copy."""
        import torch
        if self._copied is not None:
            self._copied.synchronize()      # the previous H2D read of the staging buffer is done
        st = self._stage.numpy()
        n = len(lay.desc)
        st[:n * FRAME_DTYPE.itemsize] = lay.desc.view(np.uint8)
        if self.max_scans:
            # unused scan descriptors: no components, no chunks, after every real scan in chunk and frame order
            sd = np.zeros(self.max_scans, SCAN_DTYPE)
            sd[:len(lay.scans)] = lay.scans
            sd["chunk_begin"][len(lay.scans):] = lay.chunks
            sd["frame"][len(lay.scans):] = 0x7fffffff
            st[self.frame_bytes:self.frame_bytes + sd.nbytes] = sd.view(np.uint8)
        for buf, info, d in zip(encoded, lay.infos, lay.desc):
            if info is None:
                continue
            src = np.frombuffer(memoryview(buf), np.uint8)
            o = self.meta_bytes + int(d["coded_offset"])
            if info.scans:
                for si in info.scans:
                    st[o:o + si.length] = src[si.offset:si.offset + si.length]
                    o += si.length
            else:
                st[o:o + info.scan_len] = src[info.scan_offset:info.scan_offset + info.scan_len]
        nbytes = self.meta_bytes + lay.coded_bytes
        with torch.cuda.device(self.device):
            self.buf[:nbytes].copy_(self._stage[:nbytes], non_blocking=True)
            self._copied = torch.cuda.Event()
            self._copied.record()
        self.layout, self.n = lay, n

    def launch(self, n: int = None) -> None:
        """Enqueue acr_b200_jpeg_decode over the loaded batch (or over ``n`` descriptors) on the current stream."""
        from . import lib as L
        n = self.n if n is None else n
        if n == 0:
            raise ValueError("JpegBatch.launch before load")
        with L.on(self.device):
            if self.max_scans:
                L.check(L.load().acr_b200_jpeg_decode_scans(
                    self.buf.data_ptr() + self.meta_bytes, self.max_coded_bytes, self.buf.data_ptr(), n,
                    self.buf.data_ptr() + self.frame_bytes, self.max_scans, self.max_chunks, self.max_blocks,
                    L.ptr(self.workspace), self.workspace.numel(), L.ptr(self.out), self.max_frame_bytes,
                    L.ptr(self.status), L.current_stream(self.device)), "jpeg_decode_scans")
                return
            L.check(L.load().acr_b200_jpeg_decode(
                self.buf.data_ptr() + self.meta_bytes, self.max_coded_bytes, self.buf.data_ptr(), n,
                self.max_chunks, self.max_blocks, L.ptr(self.workspace), self.workspace.numel(), L.ptr(self.out),
                self.max_frame_bytes, L.ptr(self.status), L.current_stream(self.device)), "jpeg_decode")

    def prepare(self, encoded: Sequence, host_fallback: bool = False, exact: bool = False):
        """Parse, lay out and check a batch (raises before anything is enqueued) -> (layout, host-decoded frames by
        index, for the unsupported files when ``host_fallback``)."""
        lay, fallback = plan(encoded, host_fallback, self.max_scans)
        self.check(lay, exact)
        return lay, fallback

    def put_host_frames(self, fallback) -> None:
        """Copy host-decoded frames into their places of the packed output, on the current stream."""
        import torch
        for i, img in fallback.items():
            d = self.layout.desc[i]
            o = int(d["out_offset"])
            self.out[o:o + img.size].copy_(torch.from_numpy(np.ascontiguousarray(img)).reshape(-1), non_blocking=False)

    def frames(self):
        """(H_i, W_i, 3) uint8 views of the packed output for the loaded batch."""
        return [self.out[int(d["out_offset"]):int(d["out_offset"]) + 3 * int(d["H"]) * int(d["W"])]
                .view(int(d["H"]), int(d["W"]), 3) for d in self.layout.desc]

    def coefficients(self, i: int):
        """Quantised coefficients the last decode stored for file i: per component a (block rows, blocks per row, 64)
        int16 device view, natural order (what oracle/jpeg_ref.coefficients computes).  Undefined when its status
        word is set."""
        import torch
        from . import lib as L
        d = self.layout.desc[i]
        base = L.load().acr_b200_jpeg_coef_offset(self.max_chunks)
        coef = self.workspace[base:base + self.max_blocks * 128].view(torch.int16)
        out = []
        for c in range(int(d["ncomp"])):
            b0 = int(d["coef_offset"]) + int(d["comp_block0"][c])
            bw, bh = int(d["comp_bw"][c]), int(d["comp_bh"][c])
            out.append(coef[64 * b0:64 * (b0 + bw * bh)].view(bh, bw, 64))
        return out

    def raise_on_status(self) -> None:
        """Wait for the decode and raise JpegError for the first file whose status word is set."""
        st = self.status[:self.n].cpu().numpy()
        for i, s in enumerate(st):
            if s:
                why = "; ".join(v for k, v in STATUS_BITS.items() if s & k)
                raise JpegError(f"file {i}: corrupt entropy-coded data: {why}")


def _host_decode(buf):
    import cv2
    img = cv2.imdecode(np.frombuffer(memoryview(buf), np.uint8), cv2.IMREAD_COLOR)
    if img is None:
        raise JpegError("cv2.imdecode could not decode the file")
    return img


def plan(encoded: Sequence, host_fallback: bool = False, max_scans: int = 0):
    """``layout`` of a batch -> (layout, {index: host-decoded BGR frame} for the files the device does not decode
    when ``host_fallback``; otherwise those raise JpegUnsupported).  ``max_scans``: as in ``parse``, and the most
    scans the batch's multi-scan files may use together (ValueError above it, before any host decode)."""
    fallback = {}
    if host_fallback:
        for i, buf in enumerate(encoded):
            try:
                parse(buf, max_scans)
            except JpegUnsupported:
                fallback[i] = _host_decode(buf)
    lay = layout(encoded, host_fallback, {i: img.shape[:2] for i, img in fallback.items()}, max_scans)
    if len(lay.scans) > max_scans:
        raise ValueError(f"the batch needs {len(lay.scans)} scans of multi-scan files, over the capacity of "
                         f"{max_scans}")
    return lay, fallback


def decode(encoded_list: Sequence, device=None, host_fallback: bool = False, max_scans: int = 0):
    """Decode a list of JPEG files (bytes-like) on the device -> list of (H_i, W_i, 3) uint8 BGR CUDA views of one
    packed buffer (the layout ``preprocess_frames`` / ``RaggedFrames`` consume), each equal to
    ``cv2.imdecode(buf, cv2.IMREAD_COLOR)``.  Unsupported files raise JpegUnsupported before anything is enqueued,
    unless ``host_fallback``: those are decoded by cv2 on the host and copied into the same packed buffer.  Corrupt
    entropy-coded data raises JpegError after the decode (the call waits for it).  ``max_scans`` > 0 decodes
    progressive and multi-scan sequential files on the device too, as long as their scans number at most
    ``max_scans`` together (ValueError otherwise); a batch without them runs the single-scan launches."""
    encoded_list = list(encoded_list)
    lay, fallback = plan(encoded_list, host_fallback, max_scans)
    jb = JpegBatch(len(encoded_list), lay.coded_bytes, lay.out_bytes, max(lay.chunks, 1), max(lay.blocks, 1), device,
                   max_scans=len(lay.scans))
    jb.load(encoded_list, lay)
    jb.launch()
    jb.put_host_frames(fallback)
    out = jb.frames()
    jb.raise_on_status()
    return out
