"""GPU parity: the implicit-GEMM convolution (wgmma) and the CUDA-core reference conv, one op at a
time through acr_b200_run_op, vs fp32 CPU convolution on identically rounded operands."""
import numpy as np
import pytest
import torch

from acr_b200 import lib as L
from tests.helpers import run_conv_case

pytestmark = pytest.mark.gpu

# (B, H, W, cin, cout, k, s, relu, residual, bias, bn, out_f32)  -- every distinct conv class of the net
CASES = [
    (2, 32, 32, 64, 64, 1, 1, True, False, False, True, False),     # 1x1, CK=64
    (2, 32, 32, 64, 64, 3, 1, True, True, False, True, False),      # BasicBlock conv2 @64ch
    (2, 64, 64, 32, 32, 3, 1, True, False, False, True, False),     # CK=32 (64B swizzle)
    (1, 32, 32, 128, 128, 3, 1, True, True, False, True, False),    # 2 channel chunks
    (2, 16, 16, 256, 256, 3, 1, True, True, False, True, False),    # N=256, smallest map
    (1, 64, 64, 64, 256, 1, 1, True, True, False, True, False),     # bottleneck expand + residual
    (1, 64, 64, 256, 64, 1, 1, True, False, False, True, False),
    (2, 64, 64, 32, 64, 3, 2, False, False, False, True, False),    # stride-2 fuse conv (no relu)
    (1, 64, 64, 256, 64, 3, 2, True, False, False, True, False),    # transition1[1]
    (2, 32, 32, 64, 128, 3, 2, True, False, False, True, False),
    (2, 64, 64, 34, 64, 3, 2, True, False, True, True, False),      # head stem: cin 34 -> CK=16 x3, bias
    (1, 32, 32, 34, 256, 3, 1, True, False, True, True, False),     # contact conv
    (1, 64, 64, 16, 64, 3, 1, True, False, True, True, False),      # CK=16 (32B swizzle)
    (1, 64, 64, 32, 16, 3, 1, True, False, True, True, False),      # N=16
    (1, 64, 64, 64, 33, 3, 1, True, False, True, True, False),      # cout 33 -> 48
    (1, 64, 64, 33, 33, 3, 1, False, False, True, False, False),    # segm logits conv (no BN, no act)
    (2, 32, 32, 64, 106, 1, 1, False, False, True, False, True),    # head final conv, fp32 out
    (2, 32, 32, 64, 1, 1, 1, False, False, True, False, True),      # centre head
    (2, 16, 16, 128, 32, 1, 1, False, False, False, True, False),   # fuse 1x1
]


# more inputs for the same checks: a 13th element holds run_conv_case keywords (and "dt" to override the test's dtype)
EXTRA_CASES = [
    (1, 32, 32, 64, 48, 3, 1, True, False, False, True, False),     # N tails: cout_pad not a multiple of 128
    (1, 32, 32, 64, 112, 1, 1, True, False, True, True, False),
    (1, 32, 32, 64, 144, 3, 1, True, True, False, True, False),
    (1, 16, 16, 128, 400, 1, 1, False, False, True, False, False),
    (1, 32, 32, 48, 64, 3, 1, True, False, False, True, False, (("in_stride", 48), ("cin_pad", 64))),     # K tails
    (1, 32, 32, 96, 96, 3, 2, True, False, False, True, False, (("in_stride", 96), ("cin_pad", 128))),
    (2, 32, 32, 64, 64, 3, 1, True, True, False, True, False, (("ch_scale", True),)),   # channels 2^-6 .. 2^6
    (1, 32, 32, 128, 144, 1, 1, False, False, True, False, False, (("ch_scale", True),)),
    (1, 64, 64, 48, 109, 1, 1, False, False, True, False, True, (("ch_scale", True), ("in_stride", 48), ("cin_pad", 64))),
]


def _check(kind, case, dt=L.DT_BF16):
    """Every output element within the fp64 bound of tests/pack_ref.py (exact conv of the rounded operands; accumulation
    bound; one rounding to the output type), and 16-bit outputs whose rounding the bound decides rounded to nearest
    (tests.pack_ref.direction_counts)."""
    from tests.pack_ref import check_bound, direction_counts, direction_ok
    B, H, W, cin, cout, k, s, relu, res, bias, bn, f32 = case[:12]
    kw = dict(case[12]) if len(case) > 12 else {}
    dt = kw.pop("dt", dt)
    got, exp, pad_ok, acc = run_conv_case(kind, B, H, W, cin, cout, k, s, relu, res, bias, bn, f32, dt=dt,
                                          seed=hash(case[:12]) % 1000, bound=True, **kw)
    assert pad_ok, "padding channels of the output are not zero"
    tdt = torch.float32 if f32 else (torch.bfloat16 if dt == L.DT_BF16 else torch.float16)
    worst, n_bad = check_bound(got, exp, acc, tdt)
    (toward, away), (t_all, a_all) = ((0, 0), (0, 0)) if f32 else direction_counts(got, exp, acc, tdt)
    print(f"conv {case}: worst err/bound {worst:.3f}, off-RNE toward zero / away: decided {toward} / {away}, "
          f"all {t_all} / {a_all}")
    assert n_bad == 0, f"{n_bad} elements above their bound (worst err/bound {worst:.3f})"
    assert direction_ok(toward, away), f"rounding direction: {toward} toward zero vs {away} away"


@pytest.mark.parametrize("case", CASES + EXTRA_CASES)
def test_conv_ref(case):
    _check(L.OP_CONV_REF, case)


@pytest.mark.parametrize("case", CASES + EXTRA_CASES)
def test_conv_tc(case):
    _check(L.OP_CONV, case)


@pytest.mark.parametrize("case", [CASES[1], CASES[3], CASES[4], CASES[5]])
def test_conv_tc_tma_store_epilogue(case, monkeypatch):
    """Opt-in epilogue that stages 64-channel slabs in swizzled shared memory and writes them with TMA stores
    (ACR_B200_TMA_OUT=1 at plan creation): same results as the direct-store epilogue."""
    monkeypatch.setenv("ACR_B200_TMA_OUT", "1")
    _check(L.OP_CONV, case)


@pytest.mark.parametrize("case", CASES + EXTRA_CASES)
def test_conv_tc_fp16(case):
    _check(L.OP_CONV, case, dt=L.DT_F16)


@pytest.mark.parametrize("cin,cout,k,s", [(34, 64, 3, 2), (34, 256, 3, 1), (33, 33, 3, 1), (34, 64, 1, 1)])
def test_conv_tc_k_padded_by_tma_oob(cin, cout, k, s):
    """The engine feeds 33/34-channel tensors (48-wide buffers) as ONE 64-channel K chunk: channels
    48..63 do not exist in memory and must come back as TMA out-of-bounds zeros."""
    got, exp, pad_ok = run_conv_case(L.OP_CONV, 2, 64, 64, cin, cout, k, s, True, False, True, True, False,
                                     seed=cin + cout, in_stride=48, cin_pad=64)
    assert pad_ok
    assert (got - exp).abs().max().item() <= exp.abs().max().item() * 2 ** -8 + 1e-6


def test_conv_tc_full_resolution_property():
    """BASELINE-size property check: 64->64 3x3 @128x128, B=8 -- linearity in the input
    (conv(a*x) == a*conv(x) without bias/relu) on the tensor-core path."""
    c1 = (8, 128, 128, 64, 64, 3, 1, False, False, False, False, True)
    g1, e1, _ = run_conv_case(L.OP_CONV, *c1, seed=11)
    assert (g1 - e1).abs().max().item() <= e1.abs().max().item() * 2e-5 + 1e-6


@pytest.mark.parametrize("flags", [0, 4])
def test_conv_tc_x_paired_32ch(flags):
    """The engine runs dense 32->32 3x3 convs as 64->64 convs on the x-paired grid (two adjacent pixels =
    one 128-byte operand row).  Packed through Engine._pack_conv(pair=True); expected from the ORIGINAL
    weights with plain fp32 conv + BN + residual + ReLU.  flags = ACR_CONV_XPAIR makes the kernel multiply only
    the non-zero 32x32 corner of the two side taps (what the engine does); 0 = the full block-sparse weights."""
    import ctypes as C
    import torch.nn.functional as Fn
    from acr_b200.engine import Engine, _Blob
    from tests.helpers import ctensor, rup
    g = torch.Generator().manual_seed(9)
    B, H, W = 2, 32, 64
    x = torch.randn(B, 32, H, W, generator=g).bfloat16()
    res = torch.randn(B, 32, H, W, generator=g).bfloat16()
    sd = {"c.weight": torch.randn(32, 32, 3, 3, generator=g) * (2 / 288) ** 0.5,
          "b.weight": torch.rand(32, generator=g) + 0.5, "b.bias": torch.randn(32, generator=g) * 0.1,
          "b.running_mean": torch.randn(32, generator=g) * 0.1, "b.running_var": torch.rand(32, generator=g) + 0.5}
    eng = Engine(None, B, "cpu", dry_run=True)
    blob = _Blob()
    w_off, b_off = eng._pack_conv({k: v.numpy() for k, v in sd.items()}, blob, "c", "b", False, 64, 64, pair=True)
    xin = x.permute(0, 2, 3, 1).contiguous()          # NHWC, C=32 dense
    rin = res.permute(0, 2, 3, 1).contiguous()
    nbytes = xin.numel() * 2
    arena = torch.zeros(3 * rup(nbytes, 1024), dtype=torch.uint8)
    arena[:nbytes] = xin.view(torch.uint8).flatten()
    arena[rup(nbytes, 1024): rup(nbytes, 1024) + nbytes] = rin.view(torch.uint8).flatten()
    op = L.Op()
    op.kind, op.n_in = L.OP_CONV, 2
    op.in_[0] = ctensor(0, 64, H, W // 2, 64, L.DT_BF16)
    op.in_[1] = ctensor(rup(nbytes, 1024), 64, H, W // 2, 64, L.DT_BF16)
    op.out = ctensor(2 * rup(nbytes, 1024), 64, H, W // 2, 64, L.DT_BF16)
    op.w_offset[0], op.w_offset[1] = w_off, b_off
    op.k, op.stride, op.relu, op.has_residual, op.cin_pad, op.cout_pad = 3, 1, 1, 1, 64, 64
    op.shift[0] = flags
    d_arena = arena.cuda()
    d_blob = torch.frombuffer(bytearray(blob.tobytes()), dtype=torch.uint8).cuda()
    L.check(L.load().acr_b200_run_op(C.byref(op), B, d_arena.data_ptr(), d_blob.data_ptr(), None, L.DT_BF16,
                                     torch.cuda.current_stream().cuda_stream), "run_op")
    torch.cuda.synchronize()
    got = d_arena[2 * rup(nbytes, 1024): 2 * rup(nbytes, 1024) + nbytes].cpu().view(torch.bfloat16)
    got = got.view(B, H, W, 32).permute(0, 3, 1, 2).float()
    sc = sd["b.weight"] / torch.sqrt(sd["b.running_var"] + 1e-5)
    exp = Fn.conv2d(x.float(), sd["c.weight"], None, 1, 1) * sc.view(1, -1, 1, 1) \
        + (sd["b.bias"] - sd["b.running_mean"] * sc).view(1, -1, 1, 1) + res.float()
    exp = torch.relu(exp)
    assert (got - exp).abs().max().item() <= exp.abs().max().item() * 2 ** -6   # weights are rounded to bf16 here


@pytest.mark.parametrize("cout,H", [(32, 64), (64, 64), (128, 32), (256, 32)])
def test_conv_tc_stride2_x_paired_input(cout, H):
    """3x3 stride-2 convs of DENSE 32-channel tensors (fuse-layer / transition convs of branch 0) read the input as
    x-pairs (H, W/2, 64): two row-parity boxes per tile, taps = unaligned descriptor starts + K halves (MODE_S2X).
    Packed through Engine._pack_conv(s2x=True); expected from the ORIGINAL weights with a plain fp32 stride-2 conv."""
    import ctypes as C
    import torch.nn.functional as Fn
    from acr_b200.engine import Engine, _Blob
    from tests.helpers import ctensor, rup
    g = torch.Generator().manual_seed(cout + H)
    B, W = 2, H
    x = torch.randn(B, 32, H, W, generator=g).bfloat16()
    sd = {"c.weight": torch.randn(cout, 32, 3, 3, generator=g) * (2 / 288) ** 0.5,
          "b.weight": torch.rand(cout, generator=g) + 0.5, "b.bias": torch.randn(cout, generator=g) * 0.1,
          "b.running_mean": torch.randn(cout, generator=g) * 0.1, "b.running_var": torch.rand(cout, generator=g) + 0.5}
    eng = Engine(None, B, "cpu", dry_run=True)
    blob = _Blob()
    w_off, b_off = eng._pack_conv({k: v.numpy() for k, v in sd.items()}, blob, "c", "b", False, 64, cout, s2x=True)
    xin = x.permute(0, 2, 3, 1).contiguous()                      # NHWC, C = 32 dense
    nbytes = xin.numel() * 2
    obytes = B * (H // 2) * (W // 2) * cout * 2
    off_o = rup(nbytes, 1024)
    arena = torch.zeros(off_o + rup(obytes, 1024), dtype=torch.uint8)
    arena[:nbytes] = xin.view(torch.uint8).flatten()
    op = L.Op()
    op.kind, op.n_in = L.OP_CONV, 1
    op.in_[0] = ctensor(0, 64, H, W // 2, 64, L.DT_BF16)           # the x-paired view of the input
    op.out = ctensor(off_o, cout, H // 2, W // 2, cout, L.DT_BF16)
    op.w_offset[0], op.w_offset[1] = w_off, b_off
    op.k, op.stride, op.relu, op.has_residual, op.cin_pad, op.cout_pad = 3, 2, 1, 0, 64, cout
    op.shift[0] = 8                                               # ACR_CONV_S2X
    d_arena = arena.cuda()
    d_blob = torch.frombuffer(bytearray(blob.tobytes()), dtype=torch.uint8).cuda()
    L.check(L.load().acr_b200_run_op(C.byref(op), B, d_arena.data_ptr(), d_blob.data_ptr(), None, L.DT_BF16,
                                     torch.cuda.current_stream().cuda_stream), "run_op")
    torch.cuda.synchronize()
    got = d_arena[off_o: off_o + obytes].cpu().view(torch.bfloat16).view(B, H // 2, W // 2, cout).permute(0, 3, 1, 2).float()
    sc = sd["b.weight"] / torch.sqrt(sd["b.running_var"] + 1e-5)
    exp = Fn.conv2d(x.float(), sd["c.weight"], None, 2, 1) * sc.view(1, -1, 1, 1) + (sd["b.bias"] - sd["b.running_mean"] * sc).view(1, -1, 1, 1)
    exp = torch.relu(exp)
    assert (got - exp).abs().max().item() <= exp.abs().max().item() * 2 ** -6   # weights are rounded to bf16 here
