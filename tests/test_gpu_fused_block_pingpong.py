"""GPU: the ping-pong schedule of the fused BasicBlock launch (csrc/conv_block.cuh: 16 x 8 tiles, tile k of a CTA on team
k & 1 in box k & 1) is bit-identical to the block's two conv launches (ACR_B200_FUSE_BLOCKS=0), for both forms and both
16-bit types, at tile counts that exercise every way the two teams' turns can end: a CTA with one tile (the second team
never runs), fewer tiles than SMs, and CTAs with odd and even tile counts; batch 1, 3 and 133; a channel-slice input;
the stored intermediate; and the whole Engine at batch 3."""
import pytest
import torch

from acr_b200 import lib as L
from tests.test_gpu_fused_block import _run_block

pytestmark = pytest.mark.gpu

# (B, H, W) of the grid the block runs on (x-paired form: W pairs); tiles are 16 x 8, so with 132 SMs the CTAs get:
#   (1, 16, 16)     2 tiles:   one tile each, the second team of every CTA stays idle; far fewer tiles than SMs
#   (1, 64, 64)    32 tiles:   one tile each
#   (5, 48, 80)   150 tiles:   2 or 1 per CTA
#   (133, 16, 16) 266 tiles:   3 or 2 per CTA
#   (3, 128, 128) 384 tiles:   3 or 2 per CTA, a mostly odd count
#   (3, 128, 176) 528 tiles:   4 per CTA
SHAPES = [(1, 16, 16), (1, 64, 64), (5, 48, 80), (133, 16, 16), (3, 128, 128), (3, 128, 176)]


@pytest.mark.parametrize("dt", [L.DT_BF16, L.DT_F16])
@pytest.mark.parametrize("form", ["64", "xpair"])
@pytest.mark.parametrize("shape", SHAPES)
def test_pingpong_block_equals_two_launches(form, dt, shape, monkeypatch):
    B, H, W = shape
    if form == "xpair":
        W *= 2
    ref_out, ref_mid = _run_block(form, dt, B, H, W, False, monkeypatch, seed=11)
    out, mid = _run_block(form, dt, B, H, W, True, monkeypatch, seed=11)
    assert torch.equal(out, ref_out)
    assert torch.equal(mid, ref_mid)   # the stored intermediate: each tile's own 16 x 8 conv1 pixels
    assert out.float().abs().sum() > 0


@pytest.mark.parametrize("dt", [L.DT_BF16, L.DT_F16])
@pytest.mark.parametrize("shape", [(1, 16, 16), (3, 48, 80)])
def test_pingpong_block_channel_slice_input(dt, shape, monkeypatch):
    """64-channel block reading channels 64..127 of a 256-wide buffer, no stored intermediate."""
    B, H, W = shape
    kw = dict(in_stride=256, c_off=64, store_mid=False, seed=5)
    ref_out, _ = _run_block("64", dt, B, H, W, False, monkeypatch, **kw)
    out, mid = _run_block("64", dt, B, H, W, True, monkeypatch, **kw)
    assert torch.equal(out, ref_out)
    assert not mid.float().abs().sum()


@pytest.fixture(scope="module")
def sd():
    from acr_b200.synth import load_bn_calibration, synth_state_dict
    return synth_state_dict(0, bn_stats=load_bn_calibration(0))


def test_engine_fused_blocks_bit_identical_batch3(sd, monkeypatch):
    """Whole W32 plan at batch 3, fused blocks against unfused: every kept output and every block's output."""
    from acr_b200.engine import Engine
    g = torch.Generator().manual_seed(7)
    image = torch.randint(0, 256, (3, 512, 512, 3), generator=g, dtype=torch.uint8).cuda()
    res = {}
    for fuse in ("1", "0"):
        monkeypatch.setenv("ACR_B200_FUSE_BLOCKS", fuse)
        eng = Engine(sd, 3, "cuda", torch.bfloat16, reuse_memory=False)
        eng.run(image)
        torch.cuda.synchronize()
        names = ["segms", "l_center_map", "r_center_map", "l_params_maps", "r_params_maps", "l_prior_maps",
                 "r_prior_maps", "pooled"] + [eng.recs[i]["out"].name for i in eng.block_starts]
        res[fuse] = {n: eng.view(n).clone() for n in names}
        del eng
    for n, v in res["1"].items():
        assert torch.equal(v, res["0"][n]), n
