"""CPU: register budget of the conv kernel in the built library (cuobjdump of the sm_90a code): no conv_tc_kernel instance
touches local memory (no spills), and every instance keeps its wgmma / TMA / mbarrier pipeline and the producer-consumer
register split."""
import os
import sys

import pytest

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))


def test_conv_tc_instances_do_not_spill():
    lib = os.path.join(ROOT, "arbitrary-hands-3d-reconstruction_b200", "lib", "libacr_b200.so")
    if not (os.path.exists(lib) and os.path.exists("/usr/local/cuda/bin/cuobjdump")):
        pytest.skip("library not built or no cuobjdump")
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    try:
        import sass_audit
        rows = sass_audit.audit(lib)
    finally:
        sys.path.pop(0)
    conv = {n: r for n, r in rows.items() if n.startswith("conv_tc_kernel<")}
    assert len(conv) >= 30
    for n, r in conv.items():
        assert r["LDL"] == 0 and r["STL"] == 0, f"{n}: {r['LDL']} LDL / {r['STL']} STL"
        assert r["HGMMA"] > 0 and r["UTMALDG"] > 0 and r["SYNCS"] > 0, n
        assert r["USETMAXREG"] == 2, n   # producer gives registers up, consumers take them
