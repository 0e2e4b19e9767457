"""GPU: the fused BasicBlock launch (csrc/conv_block.cuh) is bit-identical to the block's two conv launches
(ACR_B200_FUSE_BLOCKS=0), for both forms (64 -> 64 and x-paired 32 -> 32), both 16-bit types, a one-tile image (every
border at once), tile counts that are not a multiple of the grid, batch 1 and 5, a channel-slice input, the stored
intermediate, and the whole Engine."""
import ctypes as C

import numpy as np
import pytest
import torch

from acr_b200 import lib as L
from tests.helpers import ctensor, pack_conv_host, rup

pytestmark = pytest.mark.gpu


def _weights(form, dt, g):
    """Packed (weights, bias) of conv1 and conv2 of one block, BN folded."""
    from acr_b200.engine import Engine, _Blob
    c = 32 if form == "xpair" else 64
    out = []
    for _ in range(2):
        w = (torch.randn(c, c, 3, 3, generator=g) * (2 / (9 * c)) ** 0.5).numpy()
        bn = [(torch.rand(c, generator=g) + 0.5).numpy(), (torch.randn(c, generator=g) * 0.1).numpy(),
              (torch.randn(c, generator=g) * 0.1).numpy(), (torch.rand(c, generator=g) + 0.5).numpy()]
        if form == "xpair":
            blob = _Blob()
            eng = Engine(None, 1, "cpu", torch.bfloat16 if dt == L.DT_BF16 else torch.float16, dry_run=True)
            sd = {"c.weight": w, "b.weight": bn[0], "b.bias": bn[1], "b.running_mean": bn[2], "b.running_var": bn[3]}
            eng._pack_conv(sd, blob, "c", "b", False, 64, 64, pair=True)
            raw = np.frombuffer(blob.tobytes(), np.uint8)
            nw = 64 * 9 * 64 * 2
            out.append((raw[:nw].copy(), raw[rup(nw, 256): rup(nw, 256) + 256].view(np.float32).copy()))
        else:
            wp, b = pack_conv_host(w, None, bn, 64, 64, dt)
            out.append((wp.view(np.uint8).reshape(-1), b))
    return out


def _run_block(form, dt, B, H, W, fuse, monkeypatch, in_stride=64, c_off=0, store_mid=True, seed=0):
    """Runs one BasicBlock as a two-op plan; -> (output, intermediate) as raw 16-bit tensors (B, H, W', 64)."""
    monkeypatch.setenv("ACR_B200_FUSE_BLOCKS", "1" if fuse else "0")
    g = torch.Generator().manual_seed(seed)
    tdt = torch.bfloat16 if dt == L.DT_BF16 else torch.float16
    Wg = W // 2 if form == "xpair" else W            # grid width: pixel pairs for the x-paired form
    x = torch.zeros(B, H, Wg, in_stride, dtype=tdt)
    x[..., c_off:c_off + 64] = torch.randn(B, H, Wg, 64, generator=g).to(tdt)
    (w1, b1), (w2, b2) = _weights(form, dt, g)
    blob = np.zeros(4 * 65536, np.uint8)
    offs = [0, 65536, 2 * 65536, 3 * 65536]
    for o, a in zip(offs, [w1, b1.view(np.uint8), w2, b2.view(np.uint8)]):
        blob[o:o + a.nbytes] = a.view(np.uint8)
    xb = x.numel() * 2
    yb = B * H * Wg * 64 * 2
    off_x, off_y = 0, rup(xb, 1024)
    off_o = off_y + rup(yb, 1024)
    arena = torch.zeros(off_o + rup(yb, 1024), dtype=torch.uint8)
    arena[:xb] = x.view(torch.uint8).flatten()
    d_arena, d_blob = arena.cuda(), torch.from_numpy(blob).cuda()
    xin = ctensor(off_x + 2 * c_off, 64, H, Wg, in_stride, dt)
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
    out = d_arena[off_o:off_o + yb].view(tdt).view(B, H, Wg, 64).cpu()
    mid = d_arena[off_y:off_y + yb].view(tdt).view(B, H, Wg, 64).cpu()
    return out, mid


# (B, H, W) of the grid the block runs on (the x-paired form: W pixels = W / 2 pairs)
SHAPES = [(1, 16, 16), (5, 48, 80), (1, 64, 64), (3, 128, 128)]


@pytest.mark.parametrize("dt", [L.DT_BF16, L.DT_F16])
@pytest.mark.parametrize("form", ["64", "xpair"])
@pytest.mark.parametrize("shape", SHAPES)
def test_fused_block_equals_two_launches(form, dt, shape, monkeypatch):
    B, H, W = shape
    if form == "xpair":
        W *= 2
    ref_out, ref_mid = _run_block(form, dt, B, H, W, False, monkeypatch)
    out, mid = _run_block(form, dt, B, H, W, True, monkeypatch)
    assert torch.equal(out, ref_out)
    assert torch.equal(mid, ref_mid)   # the stored intermediate
    assert out.float().abs().sum() > 0


@pytest.mark.parametrize("dt", [L.DT_BF16, L.DT_F16])
def test_fused_block_channel_slice_input(dt, monkeypatch):
    """64-channel block reading channels 64..127 of a 256-wide buffer (the head blocks read the merged stem conv)."""
    kw = dict(in_stride=256, c_off=64, store_mid=False)
    ref_out, _ = _run_block("64", dt, 2, 64, 64, False, monkeypatch, **kw)
    out, mid = _run_block("64", dt, 2, 64, 64, True, monkeypatch, **kw)
    assert torch.equal(out, ref_out)
    assert not mid.float().abs().sum()   # no reader, not stored


@pytest.fixture(scope="module")
def sd():
    from acr_b200.synth import load_bn_calibration, synth_state_dict
    return synth_state_dict(0, bn_stats=load_bn_calibration(0))


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_engine_fused_blocks_bit_identical(sd, dtype, monkeypatch):
    """Whole plan with and without fused blocks: every kept output, and (reuse_memory=False) every block intermediate."""
    from acr_b200.engine import Engine
    g = torch.Generator().manual_seed(3)
    image = torch.randint(0, 256, (2, 512, 512, 3), generator=g, dtype=torch.uint8).cuda()
    res = {}
    for fuse in ("1", "0"):
        monkeypatch.setenv("ACR_B200_FUSE_BLOCKS", fuse)
        eng = Engine(sd, 2, "cuda", dtype, reuse_memory=False)
        assert len(eng.block_starts) == 80
        assert eng.num_launches == eng.n_ops - (80 if fuse == "1" else 0)
        eng.run(image)
        torch.cuda.synchronize()
        names = ["segms", "l_center_map", "r_center_map", "l_params_maps", "r_params_maps", "l_prior_maps",
                 "r_prior_maps", "pooled"] + [eng.recs[i]["out"].name for i in eng.block_starts]
        res[fuse] = {n: eng.view(n).clone() for n in names}
        del eng
    for n, v in res["1"].items():
        assert torch.equal(v, res["0"][n]), n
