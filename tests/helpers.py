"""Shared helpers for the parity tests (single-op harness around the C ABI)."""
import ctypes as C
import os

import numpy as np
import torch

from acr_b200 import lib as L

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def rup(x, m):
    return (x + m - 1) // m * m


def rel_err(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-12))


def to_nhwc_padded(x_nchw: torch.Tensor, stride: int, dtype) -> torch.Tensor:
    """(B,C,H,W) float -> (B,H,W,stride) `dtype`, zero padded channels."""
    B, Cc, H, W = x_nchw.shape
    out = torch.zeros(B, H, W, stride, dtype=dtype)
    out[..., :Cc] = x_nchw.permute(0, 2, 3, 1).to(dtype)
    return out


def ctensor(offset, Cc, H, W, stride, dt, external=0):
    t = L.Tensor()
    t.offset, t.C, t.H, t.W, t.pix_stride, t.dtype, t.external = offset, Cc, H, W, stride, dt, external
    return t


def pack_conv_host(w, conv_bias, bn, cin_pad, cout_pad, dt):
    """-> (packed uint16 (cout_pad,k*k,cin_pad), bias fp32 (cout_pad)) via the library's host packer."""
    lib = L.load()
    w = np.ascontiguousarray(w, np.float32)
    cout, cin, k, _ = w.shape
    wp = np.zeros((cout_pad, k * k, cin_pad), np.uint16)
    bias = np.zeros(cout_pad, np.float32)
    p = lambda a: None if a is None else np.ascontiguousarray(a, np.float32).ctypes.data
    keep = [None if a is None else np.ascontiguousarray(a, np.float32) for a in ([conv_bias] + list(bn or [None] * 4))]
    q = lambda a: None if a is None else a.ctypes.data
    L.check(lib.acr_b200_pack_conv(w.ctypes.data, q(keep[0]), q(keep[1]), q(keep[2]), q(keep[3]), q(keep[4]),
                                   1e-5, cout, cin, k, cout_pad, cin_pad, dt, wp.ctypes.data, bias.ctypes.data),
            "pack_conv")
    return wp, bias


def u16_to_float(a: np.ndarray, dt) -> torch.Tensor:
    t = torch.from_numpy(a.view(np.int16).copy())
    return t.view(torch.bfloat16 if dt == L.DT_BF16 else torch.float16).float()


CONV_BIAS_PER_IMAGE, CONV_POW11_CH0 = 1, 2     # ACR_CONV_* flag bits (shift[0]) of a CONV op


def run_conv_case(kind, B, H, W, cin, cout, k, s, relu, residual, bias, bn, out_f32, dt=L.DT_BF16, seed=0,
                  in_stride=None, cin_pad=None, flags=0, bias_img=None, ch_scale=False, bound=False):
    """Runs one conv through acr_b200_run_op on the GPU and returns (got, expected, pad_ok), fp32 NCHW got and fp64
    expected, plus the accumulation bound acc of tests.pack_ref.conv_with_bound when ``bound``.

    The expected output is computed in fp64 on the rounded input and on the restated rounding of the ORIGINAL weights
    (tests/pack_ref.py, pinned to the packer bit for bit by tests/test_cpu_packing.py), in the kernel's epilogue order:
    + bias, 1.1 ** channel 0, + residual, ReLU.
    flags: ACR_CONV_* bits of the op.  With CONV_BIAS_PER_IMAGE the bias is ``bias_img``, an fp32 (B, cout_pad) tensor
    placed in the arena as aux[0] (the folded part-head conv).  ``ch_scale`` multiplies input channel c by a power of
    two from 2^-6 (c = 0) to 2^6 (c = cin - 1), so that small channels matter to the bound."""
    from tests import pack_ref
    g = torch.Generator().manual_seed(seed)
    tdt = torch.bfloat16 if dt == L.DT_BF16 else torch.float16
    in_stride = in_stride or rup(cin, 16)
    cin_pad, cout_pad = cin_pad or rup(cin, 16), rup(cout, 16)
    Ho, Wo = H // s, W // s
    x = torch.randn(B, cin, H, W, generator=g)
    if ch_scale:
        x = x * torch.exp2(torch.round(torch.linspace(-6, 6, cin))).view(1, cin, 1, 1)
    w = torch.randn(cout, cin, k, k, generator=g) * (2.0 / (cin * k * k)) ** 0.5
    cb = torch.randn(cout, generator=g) * 0.1 if bias else None
    bnp = None
    if bn:
        bnp = [torch.rand(cout, generator=g) + 0.5, torch.randn(cout, generator=g) * 0.1,
               torch.randn(cout, generator=g) * 0.1, torch.rand(cout, generator=g) + 0.5]
    wp, bvec = pack_conv_host(w.numpy(), None if cb is None else cb.numpy(),
                              None if bnp is None else [t.numpy() for t in bnp], cin_pad, cout_pad, dt)
    xin = to_nhwc_padded(x, in_stride, tdt)
    res = torch.randn(B, cout, Ho, Wo, generator=g) if residual else None
    # arena layout: [x | res | out]
    esz = 2
    off_x = 0
    off_r = rup(xin.numel() * esz, 1024)
    res_stride = cout_pad
    rbytes = B * Ho * Wo * res_stride * esz if residual else 0
    off_o = rup(off_r + rbytes, 1024)
    oesz = 4 if out_f32 else 2
    obytes = B * Ho * Wo * cout_pad * oesz
    per_image = bool(flags & CONV_BIAS_PER_IMAGE)
    if per_image:
        assert bias_img is not None and tuple(bias_img.shape) == (B, cout_pad) and bias_img.dtype == torch.float32
    off_b = rup(off_o + obytes, 1024)
    arena = torch.zeros(off_b + (B * cout_pad * 4 if per_image else 0) + 1024, dtype=torch.uint8)
    if per_image:
        arena[off_b: off_b + B * cout_pad * 4] = bias_img.contiguous().view(torch.uint8).flatten()
    arena[off_x: off_x + xin.numel() * esz] = xin.view(torch.uint8).flatten()
    if residual:
        rin = to_nhwc_padded(res, res_stride, tdt)
        arena[off_r: off_r + rin.numel() * esz] = rin.view(torch.uint8).flatten()
    blob = np.concatenate([wp.view(np.uint8).reshape(-1), np.zeros((-wp.nbytes) % 256, np.uint8),
                           bvec.view(np.uint8).reshape(-1)])
    w_off, b_off = 0, wp.nbytes + ((-wp.nbytes) % 256)
    op = L.Op()
    op.kind = kind
    op.n_in = 2 if residual else 1
    op.in_[0] = ctensor(off_x, cin, H, W, in_stride, dt)
    if residual:
        op.in_[1] = ctensor(off_r, cout, Ho, Wo, res_stride, dt)
    op.out = ctensor(off_o, cout, Ho, Wo, cout_pad, L.DT_F32 if out_f32 else dt)
    if per_image:
        op.aux[0] = ctensor(off_b, cout_pad, 1, 1, cout_pad, L.DT_F32)
    op.w_offset[0], op.w_offset[1] = w_off, b_off
    op.k, op.stride, op.relu, op.has_residual = k, s, int(relu), int(residual)
    op.cin_pad, op.cout_pad = cin_pad, cout_pad
    op.shift[0] = flags
    d_arena = arena.cuda()
    d_blob = torch.from_numpy(blob).cuda()
    lib = L.load()
    L.check(lib.acr_b200_run_op(C.byref(op), B, d_arena.data_ptr(), d_blob.data_ptr(), None, dt,
                                torch.cuda.current_stream().cuda_stream), "run_op")
    torch.cuda.synchronize()
    raw = d_arena[off_o: off_o + obytes].cpu()
    got = raw.view(torch.float32 if out_f32 else tdt).view(B, Ho, Wo, cout_pad).float()
    pad_ok = bool((got[..., cout:] == 0).all())
    got = got[..., :cout].permute(0, 3, 1, 2).contiguous()
    # expected: the restated weights (not the packer's words) and the same rounded activations, fp64 on the CPU
    wq, bq = pack_ref.pack_conv_ref(w.numpy(), None if cb is None else cb.numpy(),
                                    None if bnp is None else [t.numpy() for t in bnp], dt)
    wf = torch.from_numpy(pack_ref.words_to_f64(wq, dt))
    xf = xin[..., :cin].float().permute(0, 3, 1, 2).contiguous()
    rf = rin[..., :cout].float().permute(0, 3, 1, 2) if residual else None
    bf = bias_img[:, :cout, None, None] if per_image else torch.from_numpy(bq)
    exp, acc = pack_ref.conv_with_bound(xf, wf, bf, s, pack_ref.U_ACC_TC, residual=rf,
                                        pow11=bool(flags & CONV_POW11_CH0), relu=relu)
    return (got, exp, pad_ok, acc) if bound else (got, exp, pad_ok)
