"""The statement of acr_b200_part_labels, in fp64 on the CPU (numpy).

For image i with offsets row [side, side, 0,0,0,0, pad_t, pad_r, pad_b, pad_l], its frame is H = side - pad_t - pad_b
by W = side - pad_l - pad_r, and

    labels_i[y, x] = argmax_c bilinear(segms_i[c], side)[y + pad_t, x + pad_l]     (uint8, ties to the lowest c)

where bilinear is F.interpolate(size=(side, side), mode='bilinear', align_corners=False): per axis the source
coordinate max((d + 0.5) * M / side - 0.5, 0) of an M-cell map, its floor i0, the upper neighbour min(i0 + 1, M - 1) and
the weights 1 - lambda, lambda with lambda = src - i0.  The same rule holds when side < M (no antialias).
"""
import numpy as np

U32 = 2.0 ** -24            # unit roundoff of fp32
MAX_SIDE = 16384            # ACR_B200_PART_LABELS_MAX_SIDE
INVALID, OVER_CAPACITY = 1, 2


def frame_geometry(row):
    """-> (side, pad_t, pad_l, H, W), or None when the row is not a valid geometry."""
    o = np.asarray(row, np.float64).reshape(10)
    if not (np.all(o >= 0) and np.all(o == np.floor(o))):
        return None
    side = o[0]
    if o[1] != side or not 1 <= side <= MAX_SIDE or o[6] + o[8] >= side or o[7] + o[9] >= side:
        return None
    side, pad_t, pad_r, pad_b, pad_l = (int(v) for v in (side, o[6], o[7], o[8], o[9]))
    return side, pad_t, pad_l, side - pad_t - pad_b, side - pad_l - pad_r


def packing(offsets, capacity):
    """-> (first label byte (n,), H (n,), W (n,), flags (n,)): the exclusive prefix of H*W over the valid frames; an
    invalid row is flagged INVALID and takes no bytes, a frame whose labels end past ``capacity`` is OVER_CAPACITY."""
    n = len(offsets)
    start, Hs, Ws, flags = (np.zeros(n, np.int64) for _ in range(4))
    pos = 0
    for i, row in enumerate(offsets):
        g = frame_geometry(row)
        start[i] = pos
        if g is None:
            flags[i] = INVALID
            continue
        Hs[i], Ws[i] = g[3], g[4]
        if pos + g[3] * g[4] > capacity:
            flags[i] = OVER_CAPACITY
        pos += g[3] * g[4]
    return start, Hs, Ws, flags


def axis(M, side, d):
    """Source cells and weights of padded output indices d on one axis -> (i0, i1, lambda)."""
    src = np.maximum((np.asarray(d, np.float64) + 0.5) * M / side - 0.5, 0.0)
    i0 = np.floor(src).astype(np.int64)
    return i0, np.minimum(i0 + 1, M - 1), src - i0


def interpolate(segm, side, ys, xs):
    """(M, M, C) logits -> (len(ys), len(xs), C) fp64 bilinear values at padded rows ys and columns xs."""
    s = np.asarray(segm, np.float64)
    M = s.shape[0]
    y0, y1, ly = axis(M, side, ys)
    x0, x1, lx = axis(M, side, xs)
    ly, lx = ly[:, None, None], lx[None, :, None]
    top = s[y0][:, x0] * (1 - lx) + s[y0][:, x1] * lx
    bot = s[y1][:, x0] * (1 - lx) + s[y1][:, x1] * lx
    return top * (1 - ly) + bot * ly


def part_labels(segm, row, rows_per_chunk=64):
    """(M, M, 33) logits of one image and its offsets row -> (H, W) uint8 labels."""
    side, pad_t, pad_l, H, W = frame_geometry(row)
    out = np.empty((H, W), np.uint8)
    xs = np.arange(pad_l, pad_l + W)
    for r in range(0, H, rows_per_chunk):
        ys = np.arange(pad_t + r, pad_t + min(H, r + rows_per_chunk))
        out[r:r + len(ys)] = np.argmax(interpolate(segm, side, ys, xs), axis=2)
    return out


def fp32_bound_scale(M):
    """Bound on how far the kernel's fp32 arithmetic moves the margin between two channels, per unit of the largest
    |logit| near the quad.  Per axis the source coordinate scale * (d + 0.5) - 0.5 (scale = M / side rounded, one
    fused multiply-add) is off by <= 3u(M + 1) and 1 - lambda by u more, and a weight error delta moves a value by <=
    2 delta A on each axis; the interpolation itself rounds by <= 4u A per channel.  Two channels: 8(3u(M + 1) + 2u) A
    <= 8u(3M + 5) A, taken twice over."""
    return 16.0 * U32 * (3 * M + 5)


def compare(segm, row, got, rows_per_chunk=64):
    """Kernel labels ``got`` (H, W) of one image against the statement -> (pixels that differ beyond the fp32 bound,
    pixels that differ within it).  A differing pixel is exempt when the fp64 margin between the statement's label and
    the kernel's is at most fp32_bound_scale(M) times the largest |logit| within two cells of its quad."""
    from scipy.ndimage import maximum_filter
    side, pad_t, pad_l, H, W = frame_geometry(row)
    s = np.asarray(segm, np.float64)
    M = s.shape[0]
    near = maximum_filter(np.abs(s).max(axis=2), size=5, mode="nearest")
    scale = fp32_bound_scale(M)
    xs = np.arange(pad_l, pad_l + W)
    x0 = axis(M, side, xs)[0]
    bad = exempt = 0
    for r in range(0, H, rows_per_chunk):
        ys = np.arange(pad_t + r, pad_t + min(H, r + rows_per_chunk))
        v = interpolate(s, side, ys, xs)
        want = np.argmax(v, axis=2)
        g = got[r:r + len(ys)].astype(np.int64)
        diff = g != want
        if not diff.any():
            continue
        yy, xx = np.nonzero(diff)
        margin = v[yy, xx, want[yy, xx]] - v[yy, xx, g[yy, xx]]
        y0 = axis(M, side, ys)[0]
        ok = (g[yy, xx] < s.shape[2]) & (margin <= scale * near[y0[yy], x0[xx]])
        exempt += int(ok.sum())
        bad += int((~ok).sum())
    return bad, exempt
