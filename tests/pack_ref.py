"""Restatement of the conv weight packer and the per-element fp64 error bound of the plan's ops (test infrastructure).

Packer (csrc/plan.cu acr_b200_pack_conv), in its fp32 operation order:
    scale = g / sqrt(var + eps)              (scale = 1 without BN)
    shift = beta - mean * scale (+ cb * scale)
    w'    = w * scale, rounded to the storage type: round to nearest even for bf16 / fp16, nearest tf32 with ties away
            from zero for TF32 (tests/tf32_ref.tf32_round), kept for fp32.
``pack_conv_ref`` restates that in numpy; the layout functions place its words the way each engine form does, indexed
from the original OIHW (or ConvTranspose) weight, so a packed buffer can be compared with them bit for bit.

Bound: a kernel whose fp32 result y is within ``acc`` of the exact value e and which rounds y to nearest in the output
type T stores some g with  |g - e| <= 1/2 ulp_T(|e| + acc) + acc  (``check_bound``).  ``direction_counts`` counts, among
the 16-bit outputs that differ from the correctly rounded exact value, how many went toward zero and how many away: a
conversion that rounds to nearest leaves none of them where the rounding of e +- acc is decided, a truncating one
moves about half of all outputs toward zero.
"""
import math

import numpy as np
import torch
import torch.nn.functional as Fn

from acr_b200 import lib as L

EPS = np.float32(1e-5)
U32 = 2.0 ** -24          # unit roundoff of fp32
# fp32 accumulation on the tensor cores: NVIDIA does not document how wgmma rounds its fp32 sums, so each addition is
# allowed twice fp32's machine epsilon (2^-23), which also covers an accumulator that truncates
U_ACC_TC = 2.0 ** -22


# ------------------------------------------------------------------------------------------------------- rounding
def bf16_bits(x: np.ndarray) -> np.ndarray:
    """fp32 -> bf16 words, round to nearest even (finite inputs)."""
    u = np.ascontiguousarray(x, np.float32).view(np.uint32)
    return ((u + np.uint32(0x7FFF) + ((u >> 16) & np.uint32(1))) >> 16).astype(np.uint16)


def round_storage(x: np.ndarray, dt) -> np.ndarray:
    """fp32 values -> the packer's stored words: uint16 for bf16 / fp16, float32 for TF32 / fp32."""
    x = np.ascontiguousarray(x, np.float32)
    if dt == L.DT_BF16:
        return bf16_bits(x)
    if dt == L.DT_F16:
        with np.errstate(over="ignore"):                     # |x| >= 65520 -> Inf, as __float2half_rn
            return x.astype(np.float16).view(np.uint16)      # numpy's conversion rounds to nearest even, subnormals included
    if dt == L.DT_TF32:
        from tests.tf32_ref import tf32_round
        return tf32_round(torch.from_numpy(x.copy())).numpy()
    return x.copy()


def words_to_f64(words: np.ndarray, dt) -> np.ndarray:
    if dt == L.DT_BF16:
        return (np.ascontiguousarray(words, np.uint16).astype(np.uint32) << 16).view(np.float32).astype(np.float64)
    if dt == L.DT_F16:
        return np.ascontiguousarray(words, np.uint16).view(np.float16).astype(np.float64)
    return np.asarray(words, np.float32).astype(np.float64)


def word_type(dt):
    return np.uint16 if dt in (L.DT_BF16, L.DT_F16) else np.float32


def fold_bn(cout, conv_bias=None, bn=None):
    """-> (scale, shift) fp32 in the packer's operation order."""
    if bn is not None:
        g, beta, mean, var = (np.asarray(b, np.float32) for b in bn)
        scale = g / np.sqrt(var + EPS)
        shift = beta - mean * scale
    else:
        scale, shift = np.ones(cout, np.float32), np.zeros(cout, np.float32)
    if conv_bias is not None:
        shift = shift + np.asarray(conv_bias, np.float32) * scale
    return scale.astype(np.float32), shift.astype(np.float32)


def pack_conv_ref(w, conv_bias=None, bn=None, dt=L.DT_BF16, scale_axis=0):
    """w (any layout with the output channel on ``scale_axis``) -> (rounded words in w's layout, fp32 bias (cout,))."""
    w = np.asarray(w, np.float32)
    scale, shift = fold_bn(w.shape[scale_axis], conv_bias, bn)
    sh = [1] * w.ndim
    sh[scale_axis] = -1
    return round_storage(w * scale.reshape(sh), dt), shift


def bn_of(sd, bnkey):
    return None if bnkey is None else [sd[f"{bnkey}.{n}"] for n in ("weight", "bias", "running_mean", "running_var")]


# -------------------------------------------------------------------------------------------------------- layouts
# Each takes rounded words in the original weight's layout and returns the packed buffer of one engine form: the packed
# index of every original weight is written out from the kernel's view of the operand; every other slot is zero.
def layout_plain(wq, cout_pad, cin_pad):
    """(co, ci, k, k) -> [co][ky*k+kx][ci]."""
    co, ci, k, _ = wq.shape
    out = np.zeros((cout_pad, k * k, cin_pad), wq.dtype)
    out[:co, :, :ci] = wq.transpose(0, 2, 3, 1).reshape(co, k * k, ci)
    return out


def layout_xpair(wq):
    """32 -> 32 3x3 on the x-paired grid: packed output channel dxo*32+co, input channel dxi*32+ci, tap ky*3+pt.  Output
    pixel 2j+dxo reads input pixel 2(j+pt-1)+dxi, i.e. original tap kx = 2(pt-1)+dxi-dxo+1 when that is 0..2."""
    co, ci = wq.shape[:2]
    out = np.zeros((2 * co, 9, 2 * ci), wq.dtype)
    for dxo in range(2):
        for dxi in range(2):
            for pt in range(3):
                kx = 2 * (pt - 1) + dxi - dxo + 1
                if 0 <= kx <= 2:
                    for ky in range(3):
                        out[dxo * co:(dxo + 1) * co, ky * 3 + pt, dxi * ci:(dxi + 1) * ci] = wq[:, :, ky, kx]
    return out


def layout_s2x(wq, cout_pad):
    """3x3 stride 2 of a dense 32-channel input read as x-pairs (even pixel | odd pixel): tap kx = 1 reads the even
    half, kx = 0 and 2 the odd half (of pair ox-1 and ox)."""
    co, ci = wq.shape[:2]
    out = np.zeros((cout_pad, 9, 2 * ci), wq.dtype)
    for ky in range(3):
        for kx in range(3):
            off = 0 if kx == 1 else ci
            out[:co, ky * 3 + kx, off:off + ci] = wq[:, :, ky, kx]
    return out


def layout_deconv(wq_t, cout_pad, cin_pad):
    """ConvTranspose2d(k4, s2, p1) words (ci, co, 4, 4) -> [parity py*2+px][co][tap ty*2+tx][ci]: output pixel
    (2m+py, 2n+px) takes input (m+py+ty-1, n+px+tx-1) through kernel element (3-py-2ty, 3-px-2tx)."""
    ci, co = wq_t.shape[:2]
    out = np.zeros((4, cout_pad, 4, cin_pad), wq_t.dtype)
    for py in range(2):
        for px in range(2):
            for ty in range(2):
                for tx in range(2):
                    out[py * 2 + px, :co, ty * 2 + tx, :ci] = wq_t[:, :, 3 - py - 2 * ty, 3 - px - 2 * tx].T
    return out


def layout_stem(wq, kch):
    """(64, 3, k, k) -> [co][1 tap][(ky*k+kx)*3+ci] with kch >= 3k^2 channels."""
    co, ci, k, _ = wq.shape
    out = np.zeros((co, 1, kch), wq.dtype)
    for ky in range(k):
        for kx in range(k):
            out[:, 0, (ky * k + kx) * ci:(ky * k + kx + 1) * ci] = wq[:, :, ky, kx]
    return out


# --------------------------------------------------------------------------------------------- engine conv records
def _f(sd, k):
    return np.asarray(sd[k], np.float32)


def engine_conv_expectation(eng, i, sd):
    """The i-th conv record of a built Engine -> dict(words=expected packed weights, bias=expected fp32 bias or None,
    w=OIHW restated weights (fp64) for a plain conv of the record's NCHW input, b=fp64 bias (None: per image),
    deconv=bool).  ``sd``: the state dict as fp32 numpy arrays."""
    r, o, dt = eng.recs[i], eng._cops[i], eng.plan_dt
    a = r.get("attrs", {})
    flags = o.shift[0]
    if a.get("deconv"):
        wt = _f(sd, a["w"] + ".weight")                                         # (ci, co, 4, 4)
        wq, b = pack_conv_ref(wt, None, bn_of(sd, a["bn"]), dt, scale_axis=1)
        return dict(words=layout_deconv(wq, o.cout_pad, o.cin_pad), bias=_pad(b, o.cout_pad), w=words_to_f64(wq, dt),
                    b=b.astype(np.float64), deconv=True)
    if "stem" in a:
        wq, b = pack_conv_ref(_f(sd, a["stem"]["w"] + ".weight"), None, bn_of(sd, a["stem"]["bn"]), dt)
        wf = words_to_f64(wq, dt)
        w1 = np.zeros((64, o.cin_pad, 1, 1))                                    # the 1x1 conv on the im2col channels
        w1[:, :27, 0, 0] = wf.transpose(0, 2, 3, 1).reshape(64, 27)
        return dict(words=layout_stem(wq, o.cin_pad), bias=b, w=w1, b=b.astype(np.float64))
    if "fold_side" in a:
        wq, _ = pack_conv_ref(eng.fold_weights(sd, a["fold_side"]), None, None, dt)
        return dict(words=layout_plain(wq, o.cout_pad, o.cin_pad), bias=None, w=words_to_f64(wq, dt), b=None)
    if a.get("merged"):
        each, ws, bs, wf, bf = a["merged"], [], [], [], []
        for wk, bk in zip(a["w"], a["bn"]):
            wq, b = pack_conv_ref(_f(sd, wk + ".weight"), _f(sd, wk + ".bias") if a["bias"] else None, bn_of(sd, bk), dt)
            ws.append(layout_plain(wq, each, o.cin_pad))
            bs.append(_pad(b, each))
            wf.append(np.pad(words_to_f64(wq, dt), ((0, each - wq.shape[0]), (0, 0), (0, 0), (0, 0))))
            bf.append(_pad(b, each).astype(np.float64))
        return dict(words=np.concatenate(ws), bias=np.concatenate(bs), w=np.concatenate(wf), b=np.concatenate(bf))
    wq, b = pack_conv_ref(_f(sd, a["w"] + ".weight"), _f(sd, a["w"] + ".bias") if a["bias"] else None,
                          bn_of(sd, a["bn"]), dt)
    if flags & 4:       # ACR_CONV_XPAIR: BN tiled over the two pixels of a pair
        words, bias = layout_xpair(wq), np.tile(b, 2)
    elif flags & 8:     # ACR_CONV_S2X
        words, bias = layout_s2x(wq, o.cout_pad), _pad(b, o.cout_pad)
    else:
        words, bias = layout_plain(wq, o.cout_pad, o.cin_pad), _pad(b, o.cout_pad)
    return dict(words=words, bias=bias, w=words_to_f64(wq, dt), b=b.astype(np.float64))


def _pad(b, n):
    out = np.zeros(n, np.float32)
    out[:len(b)] = b
    return out


def blob_words(blob: np.ndarray, offset: int, like: np.ndarray) -> np.ndarray:
    """The packed array at ``offset`` of a weight blob (uint8), shaped and typed as ``like``."""
    return blob[offset: offset + like.nbytes].view(like.dtype).reshape(like.shape)


# ---------------------------------------------------------------------------------------------------------- bound
_ULP = {  # (mantissa bits, smallest normal exponent) of each output type
    torch.bfloat16: (7, -126), torch.float16: (10, -14), torch.float32: (23, -126)}


def ulp(v: torch.Tensor, tdt) -> torch.Tensor:
    """Spacing of the type ``tdt`` at magnitude v >= 0 (fp64), subnormal range included."""
    m, emin = _ULP[tdt]
    e = torch.floor(torch.log2(v.clamp_min(2.0 ** emin)))
    return torch.exp2(e.clamp_min(emin) - m)


def conv_with_bound(x, w, b, stride, u_acc, residual=None, pow11=False, relu=False, deconv=False, pre_round=0.0):
    """fp64 conv of the stored input x (NCHW) with the weights the kernel reads, in the epilogue's order (+ bias,
    1.1 ** channel 0, + residual, ReLU), and its accumulation bound acc.

    The products of 16-bit (or tf32) operands are exact in fp32, so what the kernel adds to the exact result is the
    rounding of its n = K + 2 additions (K products, bias, residual): |y - e| <= n u_acc (S + |bias| + |residual|), S =
    the same conv on absolute values (the standard bound of recursive summation, n u << 1).  1.1 ** y propagates an
    input error d as ln(1.1) 1.1 ** y d, and powf adds at most 4 ulp (CUDA C Programming Guide, powf); the kernels raise
    the fp32 base 1.1f = 1.1 (1 + db), which scales the result by (1 + db) ** y, off by expm1(|y| ln(1 + db)); ReLU does not
    increase an error.  ``pre_round``: the unit roundoff of a conversion of the accumulator before the epilogue (the fp32
    validation plan sums in fp64 and rounds conv + bias to fp32 before 1.1 ** x and the residual)."""
    x, w = x.double(), torch.as_tensor(w).double()
    if deconv:       # ConvTranspose2d(k4, s2, p1): every output sums cin * 4 products
        conv = lambda xx, ww: Fn.conv_transpose2d(xx, ww, None, 2, 1)
        K = w.shape[0] * 4
    else:
        conv = lambda xx, ww: Fn.conv2d(xx, ww, None, stride, w.shape[-1] // 2)
        K = w.shape[1] * w.shape[2] * w.shape[3]
    y, S = conv(x, w), conv(x.abs(), w.abs())
    if b is not None:   # (cout,) or a per-image (B, cout, 1, 1) bias
        bb = torch.as_tensor(b).double()
        bb = bb.view(1, -1, 1, 1) if bb.dim() == 1 else bb
        y, S = y + bb, S + bb.abs()
    if residual is not None:
        S = S + residual.double().abs()
    acc = (K + 2) * u_acc * S
    acc = acc + pre_round * (y.abs() + acc)
    if pow11:
        e0 = torch.pow(1.1, y[:, :1])
        base = math.log(float(np.float32(1.1)) / 1.1)          # ln(1 + db) of the fp32 base, about 2.2e-8
        a0 = math.log(1.1) * e0 * acc[:, :1] * (1 + acc[:, :1]) + 4 * 2.0 ** -23 * e0 + e0 * torch.expm1(y[:, :1].abs() * base)
        acc = torch.cat([a0, acc[:, 1:]], 1)
        y = torch.cat([e0, y[:, 1:]], 1)
    if residual is not None:
        y = y + residual.double()
    if relu:
        y = torch.relu(y)
    return y, acc


def check_bound(got, exp, acc, tdt):
    """-> (worst err / bound, number of elements above their bound); got, exp, acc broadcast together."""
    got, exp = got.double(), exp.double()
    acc = torch.as_tensor(acc).double()
    bound = 0.5 * ulp(exp.abs() + acc, tdt) + acc
    err = (got - exp).abs()
    ratio = err / bound
    return float(ratio.max()) if ratio.numel() else 0.0, int((err > bound).sum())


def rne(exp: torch.Tensor, tdt) -> torch.Tensor:
    """fp64 -> nearest value of the 16-bit type, ties to even (via fp32, which is exact here: a double rounding only
    matters within 2^-29 relative of a 16-bit tie, below the accumulation bound of any of these ops)."""
    return exp.float().to(tdt).double()


def direction_counts(got, exp, acc, tdt):
    """-> ((toward zero, away) among the DECIDED elements where got != RNE_T(exp), (toward, away) among all of them).

    An element is decided when the whole interval exp +- acc rounds to one value of T: a kernel whose fp32 result is
    within acc of exp and whose output conversion rounds to nearest stores exactly that value, so a decided element off
    RNE_T(exp) is a conversion that does not round to nearest (a truncating one moves about half of all elements toward
    zero).  Undecided elements may go either way, and the way is not symmetric on the tensor cores: their fp32
    accumulation rounds toward zero (measured on an H100: the wgmma conv leaves 1.2 - 1.8 times more off-RNE outputs
    below the exact value than above, the CUDA-core conv on the same operands about as many either way), so
    ``direction_ok`` asserts the decided counts; the counts over all elements are reported."""
    got, exp = got.double(), exp.double()
    acc = torch.as_tensor(acc).double()
    r = rne(exp, tdt)
    diff = got != r
    down = got.abs() < r.abs()
    decided = rne(exp - acc, tdt) == rne(exp + acc, tdt)
    tw, n = int((diff & down).sum()), int(diff.sum())
    dtw, dn = int((diff & down & decided).sum()), int((diff & decided).sum())
    return (dtw, dn - dtw), (tw, n - tw)


def direction_ok(toward, away):
    """No decided element off RNE_T(exp) in either direction (see ``direction_counts``)."""
    return toward == 0 and away == 0
