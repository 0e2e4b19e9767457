"""GPU: the fused BasicBlock launch (csrc/conv_block.cuh) over longer tile chains per CTA, bit-identical to the block's two
conv launches (ACR_B200_FUSE_BLOCKS=0).  The producer pulls each box's next tile (k + 2) into L2 when it loads tile k, and
the conv1 epilogue stores whole M blocks with stmatrix; these shapes give every CTA 4 to 8 tiles, so both teams run
several turns in steady state, and the last prefetches fall on either side of a CTA's final tile."""
import pytest
import torch

from acr_b200 import lib as L
from tests.test_gpu_fused_block import _run_block

pytestmark = pytest.mark.gpu

# (B, H, W) of the grid (x-paired form: W pairs); 16 x 8 tiles over 132 SMs:
#   (5, 128, 128)   640 tiles: 5 or 4 per CTA
#   (7, 128, 128)   896 tiles: 7 or 6 per CTA
#   (3, 128, 352)  1056 tiles: 8 per CTA
SHAPES = [(5, 128, 128), (7, 128, 128), (3, 128, 352)]


@pytest.mark.parametrize("dt", [L.DT_BF16, L.DT_F16])
@pytest.mark.parametrize("form", ["64", "xpair"])
@pytest.mark.parametrize("shape", SHAPES)
def test_long_tile_chain_block_equals_two_launches(form, dt, shape, monkeypatch):
    B, H, W = shape
    if form == "xpair":
        W *= 2
    ref_out, ref_mid = _run_block(form, dt, B, H, W, False, monkeypatch, seed=13)
    out, mid = _run_block(form, dt, B, H, W, True, monkeypatch, seed=13)
    assert torch.equal(out, ref_out)
    assert torch.equal(mid, ref_mid)
    assert out.float().abs().sum() > 0
