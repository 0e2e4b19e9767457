"""GPU parity of the conv kernel's ping-pong consumer teams (resident weights) at sizes where every persistent CTA runs
several tiles, some CTAs an odd number: the teams alternate their MMA turns over many tiles and the barrier phases wrap.
Tolerances as in test_gpu_conv.py."""
import ctypes as C

import pytest
import torch

from acr_b200 import lib as L
from tests.helpers import ctensor, run_conv_case, rup
from tests.test_gpu_conv import _check

pytestmark = pytest.mark.gpu

# (B, H, W, cin, cout, k, s, relu, residual, bias, bn, out_f32); virtual tiles over 132 CTAs in the comments
CASES = [
    (7, 128, 128, 64, 64, 3, 1, True, True, False, True, False),    # single box, 448 tiles: 3 or 4 per CTA
    (3, 128, 128, 64, 256, 1, 1, True, True, False, True, False),   # 1x1, N split in two: 384 virtual tiles, 2 or 3
    (35, 64, 64, 64, 128, 3, 2, True, False, False, True, False),   # stride 2, four parity views: 140 tiles, 1 or 2
    (34, 32, 32, 128, 128, 3, 1, True, True, False, True, False),   # streamed weights (lockstep): 136 tiles, 1 or 2
]


@pytest.mark.parametrize("case", CASES + [c + ((("dt", L.DT_F16),),) for c in CASES])
def test_conv_tc_many_tiles_per_cta(case):
    _check(L.OP_CONV, case)


@pytest.mark.parametrize("case", CASES[:2])
def test_conv_tc_many_tiles_per_cta_tma_store(case, monkeypatch):
    monkeypatch.setenv("ACR_B200_TMA_OUT", "1")
    _check(L.OP_CONV, case)


def _paired_case(form, B, H, W, cout, residual):
    """x-paired 32-channel convs packed through Engine._pack_conv: form "xpair" = 3x3 stride-1 32 -> 32 on the (H, W/2, 64)
    grid, "s2x" = 3x3 stride-2 32 -> cout reading the input as x-pairs.  -> (got, expected) fp32 NCHW."""
    import torch.nn.functional as Fn
    from acr_b200.engine import Engine, _Blob
    g = torch.Generator().manual_seed(B * H + cout)
    s = 2 if form == "s2x" else 1
    Ho, Wo = H // s, W // s
    x = torch.randn(B, 32, H, W, generator=g).bfloat16()
    res = torch.randn(B, cout, Ho, Wo, generator=g).bfloat16() if residual else None
    sd = {"c.weight": torch.randn(cout, 32, 3, 3, generator=g) * (2 / 288) ** 0.5,
          "b.weight": torch.rand(cout, generator=g) + 0.5, "b.bias": torch.randn(cout, generator=g) * 0.1,
          "b.running_mean": torch.randn(cout, generator=g) * 0.1, "b.running_var": torch.rand(cout, generator=g) + 0.5}
    blob = _Blob()
    eng = Engine(None, B, "cpu", dry_run=True)
    sdn = {k: v.numpy() for k, v in sd.items()}
    if form == "s2x":
        w_off, b_off = eng._pack_conv(sdn, blob, "c", "b", False, 64, cout, s2x=True)
    else:
        w_off, b_off = eng._pack_conv(sdn, blob, "c", "b", False, 64, 64, pair=True)
    xin = x.permute(0, 2, 3, 1).contiguous()
    nbytes = xin.numel() * 2
    obytes = B * Ho * Wo * cout * 2
    off_r = rup(nbytes, 1024)
    off_o = off_r + (rup(obytes, 1024) if residual else 0)
    arena = torch.zeros(off_o + rup(obytes, 1024), dtype=torch.uint8)
    arena[:nbytes] = xin.view(torch.uint8).flatten()
    if residual:
        arena[off_r: off_r + obytes] = res.permute(0, 2, 3, 1).contiguous().view(torch.uint8).flatten()
    op = L.Op()
    op.kind, op.n_in = L.OP_CONV, 2 if residual else 1
    op.in_[0] = ctensor(0, 64, H, W // 2, 64, L.DT_BF16)
    if form == "s2x":
        op.out = ctensor(off_o, cout, Ho, Wo, cout, L.DT_BF16)
        op.cin_pad, op.cout_pad, op.shift[0] = 64, cout, 8       # ACR_CONV_S2X
    else:
        if residual:
            op.in_[1] = ctensor(off_r, 64, Ho, Wo // 2, 64, L.DT_BF16)
        op.out = ctensor(off_o, 64, Ho, Wo // 2, 64, L.DT_BF16)
        op.cin_pad, op.cout_pad, op.shift[0] = 64, 64, 4         # ACR_CONV_XPAIR
    op.w_offset[0], op.w_offset[1] = w_off, b_off
    op.k, op.stride, op.relu, op.has_residual = 3, s, 1, int(residual)
    d_arena = arena.cuda()
    d_blob = torch.frombuffer(bytearray(blob.tobytes()), dtype=torch.uint8).cuda()
    L.check(L.load().acr_b200_run_op(C.byref(op), B, d_arena.data_ptr(), d_blob.data_ptr(), None, L.DT_BF16,
                                     torch.cuda.current_stream().cuda_stream), "run_op")
    torch.cuda.synchronize()
    got = d_arena[off_o: off_o + obytes].cpu().view(torch.bfloat16).view(B, Ho, Wo, cout).permute(0, 3, 1, 2).float()
    sc = sd["b.weight"] / torch.sqrt(sd["b.running_var"] + 1e-5)
    exp = Fn.conv2d(x.float(), sd["c.weight"], None, s, 1) * sc.view(1, -1, 1, 1) \
        + (sd["b.bias"] - sd["b.running_mean"] * sc).view(1, -1, 1, 1)
    if residual:
        exp = exp + res.float()
    return got, torch.relu(exp)


@pytest.mark.parametrize("tma_out", [0, 1])
def test_conv_tc_x_paired_many_tiles_per_cta(tma_out, monkeypatch):
    """x-paired 32 -> 32 with residual on a (128, 128) pair grid: 5 x 64 = 320 tiles, 2 or 3 per CTA."""
    monkeypatch.setenv("ACR_B200_TMA_OUT", str(tma_out))
    got, exp = _paired_case("xpair", 5, 128, 256, 32, True)
    assert (got - exp).abs().max().item() <= exp.abs().max().item() * 2 ** -6   # weights are rounded to bf16 here


@pytest.mark.parametrize("cout", [32, 64])
def test_conv_tc_stride2_x_paired_many_tiles_per_cta(cout):
    """x-paired stride-2 form, 256 x 256 input: 7 x 64 = 448 tiles, 3 or 4 per CTA."""
    got, exp = _paired_case("s2x", 7, 256, 256, cout, False)
    assert (got - exp).abs().max().item() <= exp.abs().max().item() * 2 ** -6   # weights are rounded to bf16 here
