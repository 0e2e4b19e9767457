"""GPU: the two-team schedule of the fused Bottleneck launch (csrc/conv_bottleneck.cuh: 16 x 8 tiles, tile k of a CTA on
team k & 1 in box k & 1) is bit-identical to the block's three conv launches (ACR_B200_FUSE_BLOCKS=0), for C_in 64 and
256 and both 16-bit types, at tile counts that exercise every way the two teams' work can end: a CTA with one tile (the
second team never runs), fewer tiles than SMs, and CTAs with odd and even tile counts; batch 1, 3, 5 and 133; and a
one-tile-wide image, where every tile touches the left and right borders and one of the top and bottom."""
import pytest
import torch

from acr_b200 import lib as L
from tests.test_gpu_fused_bottleneck import _run_bottleneck

pytestmark = pytest.mark.gpu

# (B, H, W) of the block; tiles are 16 x 8, so with 132 SMs the CTAs get:
#   (1, 16, 16)     2 tiles:   one tile each, the second team of every CTA stays idle; a one-tile-wide image
#   (1, 64, 64)    32 tiles:   one tile each
#   (5, 48, 80)   150 tiles:   2 or 1 per CTA
#   (133, 16, 16) 266 tiles:   3 or 2 per CTA
#   (3, 128, 128) 384 tiles:   3 or 2 per CTA, a mostly odd count
#   (3, 128, 176) 528 tiles:   4 per CTA
SHAPES = [(1, 16, 16), (1, 64, 64), (5, 48, 80), (133, 16, 16), (3, 128, 128), (3, 128, 176)]


@pytest.mark.parametrize("dt", [L.DT_BF16, L.DT_F16])
@pytest.mark.parametrize("cin", [64, 256])
@pytest.mark.parametrize("shape", SHAPES)
def test_two_team_bottleneck_equals_three_launches(cin, dt, shape, monkeypatch):
    B, H, W = shape
    ref = _run_bottleneck(cin, dt, B, H, W, False, monkeypatch, seed=13)
    out = _run_bottleneck(cin, dt, B, H, W, True, monkeypatch, seed=13)
    assert torch.equal(out, ref)
    assert out.float().abs().sum() > 0
