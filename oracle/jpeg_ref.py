"""Numpy statement of the baseline JPEG decode of csrc/jpeg.cu, pinned bit for bit to ``cv2.imdecode(buf,
cv2.IMREAD_COLOR)`` (libjpeg-turbo's defaults: JDCT_ISLOW, do_fancy_upsampling on, fixed-point YCbCr->BGR tables).
Written from the algorithms (ITU-T T.81 Annex F; the islow IDCT of Loeffler, Ligtenberg and Moschytz with 13-bit
constants and 2 pass-1 bits; the triangle upsampling filters; the 16-bit colour tables), not from library source.

    decode(buf)        -> (H, W, 3) uint8 BGR
    coefficients(buf)  -> per component (block rows, blocks per row, 64) int16, quantised, natural order

The headers come from acr_b200.jpeg.parse.  Malformed entropy data raises acr_b200.jpeg.JpegError."""
from __future__ import annotations

import numpy as np

from acr_b200.jpeg import JpegError, JpegInfo, ZIGZAG, parse

CONST_BITS, PASS1_BITS = 13, 2


def _fix(x: float) -> int:
    return int(x * (1 << CONST_BITS) + 0.5)


F_0_298, F_0_390, F_0_541, F_0_765 = _fix(0.298631336), _fix(0.390180644), _fix(0.541196100), _fix(0.765366865)
F_0_899, F_1_175, F_1_501, F_1_847 = _fix(0.899976223), _fix(1.175875602), _fix(1.501321110), _fix(1.847759065)
F_1_961, F_2_053, F_2_562, F_3_072 = _fix(1.961570560), _fix(2.053119869), _fix(2.562915447), _fix(3.072711026)


def _split_intervals(seg: bytes):
    """Remove byte stuffing and split at restart markers -> (list of data byte strings, list of RST numbers).
    A marker may be preceded by any number of 0xFF fill bytes (T.81 B.1.1.2); fill bytes that run to the end of
    the segment precede its EOI."""
    out, marks, cur, i, n = [], [], bytearray(), 0, len(seg)
    while i < n:
        x = seg[i]
        if x != 0xFF:
            cur.append(x)
            i += 1
            continue
        if i + 1 < n and seg[i + 1] == 0:
            cur.append(0xFF)
            i += 2
            continue
        while i + 1 < n and seg[i + 1] == 0xFF:
            i += 1
        if i + 1 >= n:
            break
        y = seg[i + 1]
        if not 0xD0 <= y <= 0xD7:
            raise JpegError(f"unexpected marker 0xFF{y:02X} inside the entropy-coded data")
        out.append(bytes(cur))
        marks.append(y - 0xD0)
        cur = bytearray()
        i += 2
    out.append(bytes(cur))
    return out, marks


def coefficients(buf, info: JpegInfo = None):
    """Huffman-decode the scan -> list (per component) of (block rows, blocks per row, 64) int16 arrays."""
    if info is None:
        info = parse(buf)
    b = bytes(buf)
    seg = b[info.scan_offset:info.scan_offset + info.scan_len]
    intervals, marks = _split_intervals(seg)
    total = info.mcus_x * info.mcus_y
    per = info.restart if info.restart else total
    if info.restart and total % per == 0 and len(intervals) == total // per + 1 and not intervals[-1]:
        intervals.pop()     # an RST after the last MCU, which some encoders write when the last interval is whole
    if len(intervals) != -(-total // per):
        raise JpegError(f"{len(intervals) - 1} restart markers where {-(-total // per) - 1} were expected")
    if any(m != k % 8 for k, m in enumerate(marks)):
        raise JpegError("restart markers out of sequence")
    coef = []
    for c in range(info.ncomp):
        bw, bh = info.comp_blocks(c)
        coef.append(np.zeros((bh, bw, 64), np.int16))
    slots = info.slots
    for k, data in enumerate(intervals):
        nbits = 8 * len(data)
        pad = data + b"\x00" * 8
        p = 0
        pred = [0] * info.ncomp

        def bits(p, n):   # n <= 27 bits at bit p, zero-filled past the end
            j = p >> 3
            w = int.from_bytes(pad[j:j + 5], "big")
            return (w >> (40 - (p & 7) - n)) & ((1 << n) - 1)

        def huff(p, t):
            look = bits(p, 9)
            e = int(t.lut[look])
            if e:
                l, sym = e >> 8, e & 0xFF
            else:
                l = 10
                while bits(p, l) > t.maxcode[l]:
                    l += 1
                    if l > 16:
                        raise JpegError("bad Huffman code")
                sym = int(t.vals[bits(p, l) + t.valoff[l]])
            return l, sym

        for m in range(k * per, min(total, (k + 1) * per)):
            my, mx = divmod(m, info.mcus_x)
            for c, dy, dx in slots:
                blk = coef[c][my * info.comp_v[c] + dy, mx * info.comp_h[c] + dx]
                l, s = huff(p, info.dc[c])
                p += l
                d = 0
                if s:
                    if s > 16:
                        raise JpegError("bad DC magnitude category")
                    v = bits(p, s)
                    d = v if v >= 1 << (s - 1) else v - (1 << s) + 1
                    p += s
                pred[c] += d
                blk[0] = ((pred[c] + 32768) & 0xFFFF) - 32768       # JCOEF is 16-bit
                z = 1
                while z < 64:
                    l, rs = huff(p, info.ac[c])
                    p += l
                    r, s = rs >> 4, rs & 15
                    if s:
                        z += r
                        if z > 63:
                            raise JpegError("AC run past the end of a block")
                        v = bits(p, s)
                        blk[ZIGZAG[z]] = v if v >= 1 << (s - 1) else v - (1 << s) + 1
                        p += s
                        z += 1
                    elif r == 15:
                        z += 16
                    else:
                        break
                if p > nbits:
                    raise JpegError("entropy-coded data ends early (truncated file)")
        if nbits - p >= 8:
            raise JpegError("extra entropy-coded data after the last MCU of an interval")
    return coef


def _descale(x, n):
    return (x + (1 << (n - 1))) >> n


def _idct_1d(s, shift):
    """One islow pass over axis 1 of s (N, 8, M) int64 -> (N, 8, M) descaled by `shift` (no range limit)."""
    z2, z3 = s[:, 2], s[:, 6]
    z1 = (z2 + z3) * F_0_541
    tmp2 = z1 - z3 * F_1_847
    tmp3 = z1 + z2 * F_0_765
    tmp0 = (s[:, 0] + s[:, 4]) << CONST_BITS
    tmp1 = (s[:, 0] - s[:, 4]) << CONST_BITS
    t10, t13, t11, t12 = tmp0 + tmp3, tmp0 - tmp3, tmp1 + tmp2, tmp1 - tmp2
    a0, a1, a2, a3 = s[:, 7], s[:, 5], s[:, 3], s[:, 1]
    z1, z2, z3, z4 = a0 + a3, a1 + a2, a0 + a2, a1 + a3
    z5 = (z3 + z4) * F_1_175
    a0, a1, a2, a3 = a0 * F_0_298, a1 * F_2_053, a2 * F_3_072, a3 * F_1_501
    z1, z2 = z1 * -F_0_899, z2 * -F_2_562
    z3, z4 = z3 * -F_1_961 + z5, z4 * -F_0_390 + z5
    a0, a1, a2, a3 = a0 + z1 + z3, a1 + z2 + z4, a2 + z2 + z3, a3 + z1 + z4
    out = [t10 + a3, t11 + a2, t12 + a1, t13 + a0, t13 - a0, t12 - a1, t11 - a2, t10 - a3]
    return np.stack([_descale(o, shift) for o in out], 1)


def _range_limit(x):
    """libjpeg's post-IDCT table, indexed by x & 1023 (x already centred on 0): -128..127 -> 0..255, 128..511 ->
    255, 512..895 -> 0, 896..1023 -> 0..127."""
    j = x & 1023
    return np.where(j < 128, j + 128, np.where(j < 512, 255, np.where(j < 896, 0, j - 896))).astype(np.uint8)


def idct_islow(coef, quant):
    """(N, 64) int16 quantised coefficients (natural order), (64,) quantisation table -> (N, 8, 8) uint8 samples."""
    x = coef.astype(np.int64).reshape(-1, 8, 8) * quant.astype(np.int64).reshape(8, 8)
    ws = _idct_1d(x, CONST_BITS - PASS1_BITS)                       # columns: axis 1 is the row index
    out = _idct_1d(ws.transpose(0, 2, 1), CONST_BITS + PASS1_BITS + 3)   # rows
    return _range_limit(out.transpose(0, 2, 1))


def planes(buf, info: JpegInfo = None):
    """Component sample planes, cropped to each component's size (libjpeg's downsampled_width x _height)."""
    if info is None:
        info = parse(buf)
    out = []
    for c, cf in enumerate(coefficients(buf, info)):
        bh, bw = cf.shape[:2]
        s = idct_islow(cf.reshape(-1, 64), info.quant[c]).reshape(bh, bw, 8, 8).transpose(0, 2, 1, 3)
        w, h = info.comp_size(c)
        out.append(s.reshape(bh * 8, bw * 8)[:h, :w])
    return out


def _up_h2(x):
    """h2v1 triangle filter (3/4 nearer + 1/4 further, biases 1 / 2), edge columns replicated."""
    x = x.astype(np.int32)
    left = np.concatenate([x[:, :1], x[:, :-1]], 1)
    right = np.concatenate([x[:, 1:], x[:, -1:]], 1)
    out = np.empty((x.shape[0], 2 * x.shape[1]), np.int32)
    out[:, 0::2] = (3 * x + left + 1) >> 2
    out[:, 1::2] = (3 * x + right + 2) >> 2
    return out


def _rows_pm(x):
    up = np.concatenate([x[:1], x[:-1]], 0)
    down = np.concatenate([x[1:], x[-1:]], 0)
    return up, down


def upsample(x, fx, fy):
    """libjpeg-turbo's fancy upsampling of one chroma plane by (fx, fy) in {1, 2}^2; h2v1 and h2v2 fall back to
    replication for planes at most 2 samples wide, as libjpeg-turbo does."""
    x = x.astype(np.int32)
    if (fx, fy) == (1, 1):
        return x
    if fx == 2 and x.shape[1] <= 2:
        return np.repeat(np.repeat(x, 2, 1), fy, 0)
    up, down = _rows_pm(x)
    if (fx, fy) == (2, 1):
        return _up_h2(x)
    if (fx, fy) == (1, 2):
        out = np.empty((2 * x.shape[0], x.shape[1]), np.int32)
        out[0::2] = (3 * x + up + 1) >> 2
        out[1::2] = (3 * x + down + 2) >> 2
        return out
    out = np.empty((2 * x.shape[0], 2 * x.shape[1]), np.int32)
    for r, cs in ((0, 3 * x + up), (1, 3 * x + down)):
        left = np.concatenate([cs[:, :1], cs[:, :-1]], 1)
        right = np.concatenate([cs[:, 1:], cs[:, -1:]], 1)
        out[r::2, 0::2] = (3 * cs + left + 8) >> 4
        out[r::2, 1::2] = (3 * cs + right + 7) >> 4
    return out


def color_tables():
    """libjpeg's YCbCr->RGB tables (16 fractional bits): Cr->R, Cb->B, Cr->G and Cb->G (with the rounding half)."""
    x = np.arange(256, dtype=np.int64) - 128
    fix = lambda v: int(v * 65536 + 0.5)
    half = 1 << 15
    cr_r = (fix(1.40200) * x + half) >> 16
    cb_b = (fix(1.77200) * x + half) >> 16
    cr_g = -fix(0.71414) * x
    cb_g = -fix(0.34414) * x + half
    return cr_r, cb_b, cr_g, cb_g


def decode(buf, info: JpegInfo = None):
    """One baseline JPEG -> (H, W, 3) uint8 BGR, equal to cv2.imdecode(buf, cv2.IMREAD_COLOR)."""
    if info is None:
        info = parse(buf)
    p = planes(buf, info)
    H, W = info.H, info.W
    if info.ncomp == 1:
        return np.repeat(p[0][:, :, None], 3, 2)
    y = p[0].astype(np.int64)
    cb = upsample(p[1], info.hmax, info.vmax)[:H, :W]
    cr = upsample(p[2], info.hmax, info.vmax)[:H, :W]
    cr_r, cb_b, cr_g, cb_g = color_tables()
    r = y + cr_r[cr]
    g = y + ((cb_g[cb] + cr_g[cr]) >> 16)
    bl = y + cb_b[cb]
    return np.clip(np.stack([bl, g, r], 2), 0, 255).astype(np.uint8)
