"""CPU: which Bottlenecks the engine hands to the fused launch (csrc/conv_bottleneck.cuh), that the records stay one per
spec op, and the fused kernel instances in the built library (no spills; wgmma, TMA and mbarrier present)."""
import os
import sys

import pytest
import torch

from acr_b200 import lib as L

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))


def _dry(**kw):
    from acr_b200.engine import Engine
    return Engine(None, 2, "cpu", kw.pop("dtype", torch.bfloat16), dry_run=True, **kw)


@pytest.mark.parametrize("widths", [None, (48, 96, 192, 384)])
def test_marked_triples_are_the_hrnet_layer1_bottlenecks(widths):
    eng = _dry(widths=widths)
    assert eng.n_ops == 368 and sum(r["kind"] == L.OP_CONV for r in eng.recs) == 340   # records unchanged
    starts = eng.bottleneck_starts
    assert len(starts) == 4 and not set(starts) & set(eng.block_starts)
    for b, i in enumerate(starts):
        r1, r2, r3 = eng.recs[i: i + 3]
        names = [r["attrs"]["w"] for r in (r1, r2, r3)]
        assert names == [f"backbone.layer1.{b}.conv{c}" for c in (1, 2, 3)]
        assert r1["ins"][0].C == (64 if b == 0 else 256) and r1["ins"][0].H == 128
        res = r3["ins"][1]
        if b == 0:   # the downsample's output is block 0's residual
            assert eng.recs[i - 1]["attrs"]["w"] == "backbone.layer1.0.downsample.0" and eng.recs[i - 1]["out"] is res
        else:
            assert res is r1["ins"][0]
    assert sum(eng.recs[i].get("bottleneck", False) for i in range(eng.n_ops)) == 4


def test_resnet_block0_stays_three_launches():
    """ResNet's block 0 records its downsample between conv2 and conv3: only blocks 1 and 2 of layer1 are marked."""
    eng = _dry(backbone="resnet50")
    names = [eng.recs[i]["attrs"]["w"] for i in eng.bottleneck_starts]
    assert names == ["backbone.layer1.1.conv1", "backbone.layer1.2.conv1"]


def test_observable_intermediates_and_fp32_plans_are_not_fused():
    assert _dry(reuse_memory=False).bottleneck_starts == []
    assert _dry(dtype=torch.float32).bottleneck_starts == []
    assert _dry(dtype=torch.float32, tf32=True).bottleneck_starts == []
    first = _dry()
    i0, i1 = first.bottleneck_starts[:2]
    for kept in (first.recs[i0]["out"].name, first.recs[i1 + 1]["out"].name):   # conv1's output, conv2's output
        eng = _dry(keep_extra=(kept,))
        assert len(eng.bottleneck_starts) == 3 and all(eng.recs[i]["out"].name != kept and eng.recs[i + 1]["out"].name != kept
                                                       for i in eng.bottleneck_starts)


def test_fused_bottleneck_instances_do_not_spill():
    lib = os.path.join(ROOT, "arbitrary-hands-3d-reconstruction_b200", "lib", "libacr_b200.so")
    if not (os.path.exists(lib) and os.path.exists("/usr/local/cuda/bin/cuobjdump")):
        pytest.skip("library not built or no cuobjdump")
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    try:
        import sass_audit
        rows = sass_audit.audit(lib)
    finally:
        sys.path.pop(0)
    bnk = {n: r for n, r in rows.items() if n.startswith("conv_bottleneck_kernel<")}
    assert len(bnk) == 4   # {bf16, fp16} x {C_in 64, C_in 256}
    for n, r in bnk.items():
        assert r["LDL"] == 0 and r["STL"] == 0, f"{n}: {r['LDL']} LDL / {r['STL']} STL"
        assert r["HGMMA"] > 0 and r["UTMALDG"] > 0 and r["SYNCS"] > 0, n
        assert r["USETMAXREG"] == 2, n
