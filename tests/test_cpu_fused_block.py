"""CPU: which BasicBlocks the engine hands to the fused launch (csrc/conv_block.cuh), that the records stay one per spec op,
and the fused kernel instances in the built library (no spills; wgmma, TMA and mbarrier present)."""
import os
import sys

import pytest
import torch

from acr_b200 import lib as L

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))


def _dry(**kw):
    from acr_b200.engine import Engine
    return Engine(None, 2, "cpu", kw.pop("dtype", torch.bfloat16), dry_run=True, **kw)


def test_marked_pairs_are_the_narrow_branch_blocks():
    eng = _dry()
    assert eng.n_ops == 368 and sum(r["kind"] == L.OP_CONV for r in eng.recs) == 340   # records unchanged
    starts = eng.block_starts
    assert len(starts) == 80
    shapes = sorted((eng.recs[i]["ins"][0].C, eng.recs[i]["ins"][0].H) for i in starts)
    assert shapes.count((32, 128)) == 32 and shapes.count((64, 64)) == 48
    heads = [i for i in starts if "final_layers" in eng.recs[i]["attrs"]["w"]]
    assert len(heads) == 16
    for i in starts:
        r1, r2 = eng.recs[i], eng.recs[i + 1]
        assert r1["attrs"]["w"].endswith(".conv1") and r2["attrs"]["w"].endswith(".conv2")
        assert r2["ins"][0] is r1["out"] and r2["ins"][1] is r1["ins"][0] and r2["attrs"]["residual"]
        assert not r1["block_mid"]     # reuse_memory: nothing else reads the intermediate
    assert sum(eng.recs[i].get("block", False) for i in range(eng.n_ops)) == 80


def test_observable_intermediates_are_stored():
    eng = _dry(reuse_memory=False)
    assert len(eng.block_starts) == 80 and all(eng.recs[i]["block_mid"] for i in eng.block_starts)
    first = _dry()
    kept = first.recs[first.block_starts[0]]["out"].name
    eng = _dry(keep_extra=(kept,))
    marks = {eng.recs[i]["out"].name: eng.recs[i]["block_mid"] for i in eng.block_starts}
    assert marks[kept] and sum(marks.values()) == 1


def test_validation_plan_and_ref_conv_are_not_fused():
    assert _dry(dtype=torch.float32).block_starts == []
    assert _dry(debug_ref_conv=True).block_starts == []


def test_fused_block_instances_do_not_spill():
    lib = os.path.join(ROOT, "arbitrary-hands-3d-reconstruction_b200", "lib", "libacr_b200.so")
    if not (os.path.exists(lib) and os.path.exists("/usr/local/cuda/bin/cuobjdump")):
        pytest.skip("library not built or no cuobjdump")
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    try:
        import sass_audit
        rows = sass_audit.audit(lib)
    finally:
        sys.path.pop(0)
    blk = {n: r for n, r in rows.items() if n.startswith("conv_block_kernel<")}
    assert len(blk) == 4   # {bf16, fp16} x {64-channel, x-paired}
    for n, r in blk.items():
        assert r["LDL"] == 0 and r["STL"] == 0, f"{n}: {r['LDL']} LDL / {r['STL']} STL"
        assert r["HGMMA"] > 0 and r["UTMALDG"] > 0 and r["SYNCS"] > 0, n
        assert r["USETMAXREG"] == 2, n
