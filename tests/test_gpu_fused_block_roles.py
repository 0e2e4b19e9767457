"""GPU: the fused BasicBlock (csrc/conv_block.cuh) on data that exposes the tensor core's reduction order, bit-identical to the
block's two conv launches (ACR_B200_FUSE_BLOCKS=0).

The fused kernel's conv1 runs with the weights as the wgmma A operand (M = output channels) and the pixels as B, where the
standalone conv has the pixels as A and the weights as B.  Each output element is the same dot product either way, so the
results agree only if the tensor core reduces an element's products the same way whichever operand side they come from.
Seeded Gaussian networks rarely reach the truncation inside the tensor core's internal alignment; these inputs do:
activations over about 30 binades (fp16 subnormals included), weights over 11 more, and channel pairs whose products
nearly cancel inside each k-step.  Both 16-bit types, both forms, images whose every tile touches a border and images
with interior tiles, with the intermediate stored and not."""
import ctypes as C

import numpy as np
import pytest
import torch

from acr_b200 import lib as L
from tests.helpers import ctensor, pack_conv_host, rup

pytestmark = pytest.mark.gpu


def _spread(shape, lo, hi, g):
    """sign * (1 + u) * 2^e, e uniform over [lo, hi): magnitudes spread over hi - lo binades."""
    e = torch.floor(lo + (hi - lo) * torch.rand(shape, generator=g))
    m = 1 + torch.rand(shape, generator=g)
    s = torch.where(torch.rand(shape, generator=g) < 0.5, -1.0, 1.0)
    return (s * m * torch.exp2(e)).double()


def _cancelling_weights(c, g):
    """[c_out][c_in][3][3] over 11 binades; input channel 2i + 1 is -(channel 2i) times 1 + O(2^-8) for half of the pairs,
    so with equal activations in the pair (see _activations) their products nearly cancel."""
    w = _spread((c, c, 3, 3), -16, -5, g)
    pert = 1 + torch.randint(-3, 4, (c, c // 2, 3, 3), generator=g).double() * 2.0 ** -8
    keep = torch.rand((c, c // 2, 3, 3), generator=g) < 0.5
    w[:, 1::2] = torch.where(keep, -w[:, 0::2] * pert, w[:, 1::2])
    return w.float().numpy()


def _activations(B, H, W, c, dt, g):
    """[B][H][W][c]: fp16 down into its subnormals (2^-24), bf16 from 2^-20; channel 2i + 1 repeats channel 2i."""
    x = _spread((B, H, W, c), -24 if dt == L.DT_F16 else -20, 6, g)
    x[..., 1::2] = x[..., 0::2]
    return x


def _pack(form, dt, w, bn):
    """Packed (weights bytes, fp32 bias) of one conv, BN folded, as the engine packs it."""
    if form == "xpair":
        from acr_b200.engine import Engine, _Blob
        blob = _Blob()
        eng = Engine(None, 1, "cpu", torch.bfloat16 if dt == L.DT_BF16 else torch.float16, dry_run=True)
        sd = {"c.weight": w, "b.weight": bn[0], "b.bias": bn[1], "b.running_mean": bn[2], "b.running_var": bn[3]}
        eng._pack_conv(sd, blob, "c", "b", False, 64, 64, pair=True)
        raw = np.frombuffer(blob.tobytes(), np.uint8)
        nw = 64 * 9 * 64 * 2
        return raw[:nw].copy(), raw[rup(nw, 256): rup(nw, 256) + 256].view(np.float32).copy()
    wp, b = pack_conv_host(w, None, bn, 64, 64, dt)
    return wp.view(np.uint8).reshape(-1), b


def _run(form, dt, x, packed, fuse, store_mid, monkeypatch):
    """One BasicBlock as a two-op plan on the raw 16-bit input x (B, H, W', 64); -> (output, intermediate) as int16 bits."""
    monkeypatch.setenv("ACR_B200_FUSE_BLOCKS", "1" if fuse else "0")
    B, H, Wg, _ = x.shape
    (w1, b1), (w2, b2) = packed
    blob = np.zeros(4 * 65536, np.uint8)
    offs = [0, 65536, 2 * 65536, 3 * 65536]
    for o, a in zip(offs, [w1, b1.view(np.uint8), w2, b2.view(np.uint8)]):
        blob[o:o + a.nbytes] = a.view(np.uint8)
    nb = x.numel() * 2
    off_y = rup(nb, 1024)
    off_o = off_y + rup(nb, 1024)
    arena = torch.zeros(off_o + rup(nb, 1024), dtype=torch.uint8)
    arena[:nb] = x.contiguous().view(torch.uint8).flatten()
    d_arena, d_blob = arena.cuda(), torch.from_numpy(blob).cuda()
    xin = ctensor(0, 64, H, Wg, 64, dt)
    ops = (L.Op * 2)()
    for i, o in enumerate(ops):
        o.kind, o.k, o.stride, o.relu, o.cin_pad, o.cout_pad = L.OP_CONV, 3, 1, 1, 64, 64
        o.w_offset[0], o.w_offset[1] = offs[2 * i], offs[2 * i + 1]
        o.shift[0] = 4 if form == "xpair" else 0
    ops[0].n_in, ops[0].in_[0], ops[0].out = 1, xin, ctensor(off_y, 64, H, Wg, 64, dt)
    ops[0].shift[0] |= L.CONV_BLOCK | (L.CONV_BLOCK_MID if store_mid else 0)
    ops[1].n_in, ops[1].has_residual = 2, 1
    ops[1].in_[0], ops[1].in_[1], ops[1].out = ctensor(off_y, 64, H, Wg, 64, dt), xin, ctensor(off_o, 64, H, Wg, 64, dt)
    lib = L.load()
    plan = C.c_void_p()
    L.check(lib.acr_b200_plan_create(ops, 2, B, d_arena.data_ptr(), d_arena.numel(), d_blob.data_ptr(), d_blob.numel(),
                                     dt, C.byref(plan)), "plan_create")
    try:
        assert lib.acr_b200_plan_num_launches(plan) == (1 if fuse else 2)
        L.check(lib.acr_b200_plan_run(plan, None, torch.cuda.current_stream().cuda_stream), "plan_run")
        torch.cuda.synchronize()
    finally:
        lib.acr_b200_plan_destroy(plan)
    out = d_arena[off_o:off_o + nb].view(torch.int16).view(B, H, Wg, 64).cpu()
    mid = d_arena[off_y:off_y + nb].view(torch.int16).view(B, H, Wg, 64).cpu()
    return out, mid


# (B, H, W) in pixels: 16 x 8 tiles (16 pixel pairs wide in the x-paired form)
#   (2, 32, 16)  one tile column: every tile touches a border
#   (1, 64, 64)  the 64-channel head blocks' size: 12 of 32 tiles interior
#   (2, 48, 80)  interior tiles, a width that is not a power of two
SHAPES = [(2, 32, 16), (1, 64, 64), (2, 48, 80)]


@pytest.mark.parametrize("store_mid", [True, False])
@pytest.mark.parametrize("dt", [L.DT_BF16, L.DT_F16])
@pytest.mark.parametrize("form", ["64", "xpair"])
@pytest.mark.parametrize("shape", SHAPES)
def test_wide_range_cancelling_block_equals_two_launches(form, dt, shape, store_mid, monkeypatch):
    B, H, W = shape
    c = 32 if form == "xpair" else 64
    if form == "xpair":
        W *= 2
    g = torch.Generator().manual_seed(7 + W + (dt == L.DT_F16))
    tdt = torch.bfloat16 if dt == L.DT_BF16 else torch.float16
    x = _activations(B, H, W, c, dt, g).to(tdt).view(B, H, W * c // 64, 64)
    ident = [np.ones(c, np.float32), None, np.zeros(c, np.float32), np.ones(c, np.float32)]
    packed = []
    for _ in range(2):
        bn = list(ident)
        bn[1] = (_spread((c,), -12, -4, g)).float().numpy()
        packed.append(_pack(form, dt, _cancelling_weights(c, g), bn))
    ref_out, ref_mid = _run(form, dt, x, packed, False, True, monkeypatch)
    out, mid = _run(form, dt, x, packed, True, store_mid, monkeypatch)
    assert torch.equal(out, ref_out)
    if store_mid:
        assert torch.equal(mid, ref_mid)
    else:
        assert not mid.any()   # no reader: the fused launch does not store it
    assert ref_mid.any() and out.any()
