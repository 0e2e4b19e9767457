"""Numpy statement of the device decode of progressive and multi-scan sequential JPEG files (csrc/jpeg.cu,
acr_b200_jpeg_decode_scans), pinned to ``cv2.imdecode(buf, cv2.IMREAD_COLOR)`` for complete scripts.

The scans are decoded one after another in file order, as ITU-T T.81 Annex G states them and in the order of
libjpeg's progressive Huffman decoder: DC first (the prediction << Al) and DC refinement (one bit per block), AC first
with EOB runs (each value << Al) and AC refinement with correction bits; a sequential scan over a subset of the
components decodes as in Annex F.  A one-component scan codes the component's own blocks, not the MCU-padded plane.
The islow IDCT, the upsampling and the colour conversion are oracle/jpeg_ref's single-scan stages.

    coefficients(buf)  -> per component (block rows, blocks per row, 64) int16, quantised, natural order
    decode(buf)        -> (H, W, 3) uint8 BGR

Single-scan files go through oracle/jpeg_ref unchanged.  Malformed entropy data raises acr_b200.jpeg.JpegError."""
import numpy as np

from acr_b200.jpeg import JpegError, JpegInfo, ZIGZAG, parse as _parse
from oracle import jpeg_ref
from oracle.jpeg_ref import _split_intervals

MAX_SCANS = 65535      # the statement reads multi-scan files of any length


def parse(buf) -> JpegInfo:
    return _parse(buf, MAX_SCANS)


class _Bits:
    """MSB-first reader over one restart interval's unstuffed bytes, zero-filled past the end."""

    def __init__(self, data: bytes):
        self.pad, self.n, self.p = data + b"\x00" * 8, 8 * len(data), 0

    def peek(self, n):
        j = self.p >> 3
        w = int.from_bytes(self.pad[j:j + 5], "big")
        return (w >> (40 - (self.p & 7) - n)) & ((1 << n) - 1)

    def get(self, n):
        v = self.peek(n) if n else 0
        self.p += n
        if self.p > self.n:
            raise JpegError("entropy-coded data ends early (truncated file)")
        return v

    def huff(self, t):
        e = int(t.lut[self.peek(9)])
        if e:
            l, sym = e >> 8, e & 0xFF
        else:
            l = 10
            while self.peek(l) > t.maxcode[l]:
                l += 1
                if l > 16:
                    raise JpegError("bad Huffman code")
            sym = int(t.vals[self.peek(l) + t.valoff[l]])
        self.get(l)
        return sym


def _extend(v, s):
    return v if v >= 1 << (s - 1) else v - (1 << s) + 1


def _i16(x):
    return ((x + 32768) & 0xFFFF) - 32768       # JCOEF is 16-bit


def _scan_blocks(info: JpegInfo, sc, coef):
    """Block views of scan ``sc`` in coding order: (component, block) per block."""
    out = []
    inter = len(sc.comps) > 1
    for m in range(sc.mcus_x * sc.mcus_y):
        my, mx = divmod(m, sc.mcus_x)
        for c, dy, dx in sc.slots:
            if inter:
                out.append((c, coef[c][my * info.comp_v[c] + dy, mx * info.comp_h[c] + dx]))
            else:
                out.append((c, coef[c][my, mx]))
    return out


def _multi_scan_coefficients(b: bytes, info: JpegInfo):
    coef = []
    for c in range(info.ncomp):
        bw, bh = info.comp_blocks(c)
        coef.append(np.zeros((bh, bw, 64), np.int16))
    for sc in info.scans:
        intervals, marks = _split_intervals(b[sc.offset:sc.offset + sc.length])
        blocks = _scan_blocks(info, sc, coef)
        per = sc.restart * len(sc.slots) if sc.restart else len(blocks)
        total = -(-len(blocks) // per)
        if sc.restart and len(blocks) % per == 0 and len(intervals) == total + 1 and not intervals[-1]:
            intervals.pop()
        if len(intervals) != total:
            raise JpegError(f"{len(intervals) - 1} restart markers where {total - 1} were expected")
        if any(m != k % 8 for k, m in enumerate(marks)):
            raise JpegError("restart markers out of sequence")
        p1 = 1 << sc.al
        for k, data in enumerate(intervals):
            r = _Bits(data)
            pred = [0] * info.ncomp
            eobrun = 0
            for c, blk in blocks[k * per:(k + 1) * per]:
                if sc.ss == 0 and sc.ah == 0:                 # DC first or sequential
                    s = r.huff(sc.dc[c])
                    if s > 15:
                        raise JpegError("bad DC magnitude category")
                    pred[c] += _extend(r.get(s), s) if s else 0
                    blk[0] = _i16(pred[c] << sc.al)
                    if sc.se == 63:
                        z = 1
                        while z < 64:
                            rs = r.huff(sc.ac[c])
                            rr, s = rs >> 4, rs & 15
                            if s:
                                z += rr
                                if z > 63:
                                    raise JpegError("AC run past the end of a block")
                                blk[ZIGZAG[z]] = _extend(r.get(s), s)
                                z += 1
                            elif rr == 15:
                                z += 16
                            else:
                                break
                elif sc.ss == 0:                              # DC refinement: one bit
                    if r.get(1):
                        blk[0] = _i16(int(blk[0]) | p1)
                elif sc.ah == 0:                              # AC first
                    if eobrun:
                        eobrun -= 1
                        continue
                    z = sc.ss
                    while z <= sc.se:
                        rs = r.huff(sc.ac[c])
                        rr, s = rs >> 4, rs & 15
                        if s:
                            z += rr
                            if z > sc.se:
                                raise JpegError("AC run past the end of the band")
                            blk[ZIGZAG[z]] = _i16(_extend(r.get(s), s) << sc.al)
                            z += 1
                        elif rr == 15:
                            z += 16
                        else:
                            eobrun = (1 << rr) + r.get(rr) - 1
                            break
                else:                                         # AC refinement (G.1.2.3)
                    z = sc.ss
                    if eobrun == 0:
                        while z <= sc.se:
                            rs = r.huff(sc.ac[c])
                            rr, s = rs >> 4, rs & 15
                            val = 0
                            if s:
                                if s != 1:
                                    raise JpegError("bad AC refinement magnitude")
                                val = p1 if r.get(1) else -p1
                            elif rr != 15:
                                eobrun = (1 << rr) + r.get(rr)
                                break
                            while z <= sc.se:
                                co = int(blk[ZIGZAG[z]])
                                if co:
                                    if r.get(1) and not co & p1:
                                        blk[ZIGZAG[z]] = _i16(co + (p1 if co >= 0 else -p1))
                                else:
                                    rr -= 1
                                    if rr < 0:
                                        break
                                z += 1
                            if val:
                                if z > sc.se:
                                    raise JpegError("AC refinement past the end of the band")
                                blk[ZIGZAG[z]] = val
                            z += 1
                    if eobrun > 0:
                        for zz in range(z, sc.se + 1):
                            co = int(blk[ZIGZAG[zz]])
                            if co and r.get(1) and not co & p1:
                                blk[ZIGZAG[zz]] = _i16(co + (p1 if co >= 0 else -p1))
                        eobrun -= 1
            if eobrun:
                raise JpegError("an EOB run past the end of a restart interval")
            if r.n - r.p >= 8:
                raise JpegError("extra entropy-coded data after the last block of an interval")
    return coef


def coefficients(buf, info: JpegInfo = None):
    """Huffman-decode every scan -> list (per component) of (block rows, blocks per row, 64) int16 arrays."""
    if info is None:
        info = parse(buf)
    if not info.scans:
        return jpeg_ref.coefficients(buf, info)
    return _multi_scan_coefficients(bytes(buf), info)


def planes(buf, info: JpegInfo = None):
    """Component sample planes, cropped to each component's size."""
    if info is None:
        info = parse(buf)
    out = []
    for c, cf in enumerate(coefficients(buf, info)):
        bh, bw = cf.shape[:2]
        s = jpeg_ref.idct_islow(cf.reshape(-1, 64), info.quant[c]).reshape(bh, bw, 8, 8).transpose(0, 2, 1, 3)
        w, h = info.comp_size(c)
        out.append(s.reshape(bh * 8, bw * 8)[:h, :w])
    return out


def decode(buf, info: JpegInfo = None):
    """One JPEG file (any number of scans) -> (H, W, 3) uint8 BGR."""
    if info is None:
        info = parse(buf)
    p = planes(buf, info)
    H, W = info.H, info.W
    if info.ncomp == 1:
        return np.repeat(p[0][:, :, None], 3, 2)
    y = p[0].astype(np.int64)
    cb = jpeg_ref.upsample(p[1], info.hmax, info.vmax)[:H, :W]
    cr = jpeg_ref.upsample(p[2], info.hmax, info.vmax)[:H, :W]
    cr_r, cb_b, cr_g, cb_g = jpeg_ref.color_tables()
    r = y + cr_r[cr]
    g = y + ((cb_g[cb] + cr_g[cr]) >> 16)
    bl = y + cb_b[cb]
    return np.clip(np.stack([bl, g, r], 2), 0, 255).astype(np.uint8)
