"""CPU: the restated conv plan (tests/conv_plan_ref.py) against the built library's conv_tc_kernel instances, its sweep
over every argument set conv_tc_prepare accepts, and the coverage of tests/test_gpu_conv_instances.MATRIX: every
reachable (instance, ping-pong, short epilogue, TMA store, fp32 output, N split) combination has a GPU case, and every
compiled instance the sweep cannot reach is listed below with its reason."""
import collections
import os
import sys

import pytest

from tests import conv_plan_ref as R

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
LIB = os.path.join(ROOT, "arbitrary-hands-3d-reconstruction_b200", "lib", "libacr_b200.so")

# compiled instances no accepted argument set reaches, with the reason
UNREACHABLE_INSTANCES = {
    ("__nv_bfloat16", 64, R.MODE_S2X, 64):
        "NT = 64 needs cout_pad <= 64, and then the nine 64 x cout_pad weight blocks (72 KB at most) fit resident next "
        "to the two 17 x 24-pixel boxes: a streamed S2X conv has cout_pad >= 112",
    ("__half", 64, R.MODE_S2X, 64): "as for bf16",
}
# reachable combinations (instance, pingpong, plain, tma_out, out_f32, nsplit > 1) with no GPU case: none
UNREACHABLE_COMBINATIONS = {}


@pytest.fixture(scope="module")
def swept():
    """-> (combination -> first ConvArgs that gives it, how many plans have each SB, the plans past the budget)."""
    combos, sbs, bad = collections.OrderedDict(), collections.Counter(), []
    for a, p in R.sweep():
        combos.setdefault(R.combination(p), a)
        sbs[p.SB] += 1
        if p.a_room < 0 or p.smem > R.SMEM_BUDGET:
            bad.append((a, p))
    return combos, sbs, bad


def test_compiled_instances_match_the_restated_launch_mode():
    """Every conv_tc_kernel instance of the built library is one launch_mode can launch, and the other way round: a new
    template instance fails here until conv_plan_ref knows about it."""
    if not (os.path.exists(LIB) and os.path.exists("/usr/local/cuda/bin/cuobjdump")):
        pytest.skip("library not built or no cuobjdump")
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    try:
        import sass_audit
        rows = sass_audit.audit(LIB)
    finally:
        sys.path.pop(0)
    compiled = {n for n in rows if n.startswith("conv_tc_kernel<")}
    restated = {R.kernel_name(k) for k in R.compiled_instances()}
    assert compiled == restated, (f"compiled, not restated: {sorted(compiled - restated)}; "
                                  f"restated, not compiled: {sorted(restated - compiled)}")
    assert len(compiled) == 78


def test_sweep_reaches_every_instance_but_the_listed_ones(swept):
    combos, _, _ = swept
    reached = {c[0] for c in combos}
    assert reached <= R.compiled_instances()
    assert set(UNREACHABLE_INSTANCES) == R.compiled_instances() - reached, \
        f"unreachable now: {sorted(R.compiled_instances() - reached)}"


def test_weight_ring_depth(swept):
    """Streamed weights always get the full four-block ring: the shared-memory plan never has to cut SB below 4 (the
    kernel's SB = 2 and 3 paths are not reachable); resident weights have no ring."""
    _, sbs, _ = swept
    assert set(sbs) == {0, 4}, sbs


def test_shared_memory_plan_stays_in_budget(swept):
    """conv_tc_prepare divides SMEM_BUDGET - fixed - B region as size_t: that difference is never negative for an
    accepted plan (the C++ would wrap where the restatement does not), and no plan asks for more than the budget."""
    _, _, bad = swept
    assert not bad, bad[:3]


def test_gpu_matrix_covers_every_reachable_combination(swept):
    from tests.test_gpu_conv_instances import MATRIX, conv_args
    combos, _, _ = swept
    by = collections.defaultdict(list)
    for c in MATRIX:
        by[R.combination(R.prepare(conv_args(c)))].append(c.id)
    assert set(by) <= set(combos), f"matrix cases the sweep does not produce: {sorted(set(by) - set(combos), key=str)}"
    missing = [c for c in combos if c not in by and c not in UNREACHABLE_COMBINATIONS]
    # the table: every compiled instance against its cases or its reason
    lines = []
    for key in sorted(R.compiled_instances(), key=lambda k: (k[0], -k[1], k[2], k[3])):
        ids = sorted({i for cb, v in by.items() if cb[0] == key for i in v})
        n_reach = sum(1 for cb in combos if cb[0] == key)
        n_cov = sum(1 for cb in by if cb[0] == key)
        what = UNREACHABLE_INSTANCES.get(key) or f"{n_cov}/{n_reach} combinations, {len(ids)} cases: {ids[0]} ..."
        lines.append(f"{R.kernel_name(key):42s} {R.mode_name(key[2]):22s} {what}")
    print("\n".join(lines))
    print(f"reachable combinations {len(combos)}, covered {len(set(by) & set(combos))}, cases {len(MATRIX)}")
    assert not missing, "combinations (instance, pingpong, plain, tma_out, out_f32, nsplit > 1) without a GPU case: " + \
        "; ".join(f"{R.kernel_name(c[0])} {c[1:]} e.g. {combos[c]}" for c in missing)
