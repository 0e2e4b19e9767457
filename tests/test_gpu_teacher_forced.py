"""GPU parity, teacher forced: EVERY launch of the network plan is compared with the oracle's restatement of
that op (oracle/op_ref.py, unrounded fp32 parameters) applied to the plan's OWN stored inputs.  No error
accumulates from op to op and the seeded random network cannot amplify storage round-off, so the bound is
the per-op one: storage rounding of weights and of the one output (2^-7 of the op's output range for bf16,
2^-10 for fp16, 2e-5 for the fp32 validation plan).  This pins fuse layers, bilinear up-sampling, coord
channels, every head stack, the attention pooling, the part head and the folded final conv individually --
a wrong align_corners, BN eps, coord formula, tap order or weight key shows up as an O(1) error of ONE op."""
import os

import pytest
import torch

from tests.helpers import rel_err

pytestmark = pytest.mark.gpu

TOL = {torch.bfloat16: 2.0 ** -7, torch.float16: 2.0 ** -10, torch.float32: 2e-5}


@pytest.fixture(scope="module")
def sd():
    from acr_b200.synth import load_bn_calibration, synth_state_dict
    return synth_state_dict(0, bn_stats=load_bn_calibration(0))


@pytest.fixture(scope="module")
def image():
    # one frame: the sweep re-computes every op on the CPU.  At batch 1 a kernel that reads another image's data reads its
    # own; the batch dimension is covered by tests/test_gpu_batch.py (every op teacher forced on three distinct frames,
    # every launch per image against batch 1)
    gi = torch.Generator().manual_seed(123)
    return torch.randint(0, 256, (2, 512, 512, 3), generator=gi, dtype=torch.uint8)[1:]


def _pare(eng, s):
    """(B,106) contact + shape offsets of side s: the part head packs them densely (106 floats per image)."""
    return eng.view(f"{s}_pare").float().cpu().reshape(-1)[: eng.batch * 106].view(eng.batch, 106)


def sweep(eng, sd, image, tol):
    """-> list of (op index, description, rel err); asserts nothing."""
    from acr_b200 import lib as L
    from oracle import op_ref
    sdf = {k: v.float() for k, v in sd.items() if v.dtype.is_floating_point}
    get = lambda t: eng.map_nchw(t).cpu()
    rows = []
    pool_in = None
    for i, r in enumerate(eng.recs):
        kind, a = r["kind"], r.get("attrs", {})
        checks = []      # (label, got, expected)
        if kind in (L.OP_CONV, L.OP_CONV_REF):
            if "stem" in a:
                checks.append(("stem 27->64 1x1 on im2col", get(r["out"]), op_ref.stem_from_cols(get(r["ins"][0])[:, :27], sdf)))
            elif "fold_side" in a:
                s = a["fold_side"]
                raw = eng.view(r["ins"][0]).float().cpu()                      # (B,64,64,128): params 0..105, cam 112..114
                prm, cam = raw[..., :106].permute(0, 3, 1, 2), raw[..., 112:115].permute(0, 3, 1, 2)
                pare = _pare(eng, s)
                checks.append((f"contact_layers[{'4' if s == 'l' else '5'}] folded 218->109", get(r["out"]),
                               op_ref.final_params(prm, cam, pare, sdf, s)))
            elif a.get("merged"):          # convs on the same input run as one wide conv: every slice against its own conv
                x, got, each = get(r["ins"][0]), get(r["out"]), a["merged"]
                for j, (wk, bk) in enumerate(zip(a["w"], a["bn"])):
                    checks.append((f"conv {wk} (slice {j} of a merged conv)", got[:, j * each:(j + 1) * each],
                                   op_ref.conv_bn_act(x, sdf, wk, bk, a["s"], a["relu"])))
            elif a.get("extra"):           # a fuse sum folded into the conv that produces one of its terms
                conv = op_ref.conv_bn_act(get(r["ins"][0]), sdf, a["w"], a["bn"], a["s"], False)
                others, shifts, pos = [get(t) for t in r["ins"][1:]], [sh for _, sh in a["extra"]], a["extra_pos"]
                exp = op_ref.fuse(others[:pos] + [conv] + others[pos:], shifts[:pos] + [0] + shifts[pos:], a["relu"])
                checks.append((f"conv {a['w']} + folded fuse sum of {len(others) + 1} terms", get(r["out"]), exp))
            else:
                res = get(r["ins"][1]) if a["residual"] else None
                exp = op_ref.conv_bn_act(get(r["ins"][0]), sdf, a["w"], a["bn"], a["s"], a["relu"], res, a["pow11"])
                checks.append((f"conv {a['w']} k{a['k']} s{a['s']}", get(r["out"]), exp))
        elif kind == L.OP_STEM:
            checks.append(("stem (CUDA-core form)", get(r["out"]), op_ref.stem(image, sdf)))
        elif kind == L.OP_STEM_TC:
            checks.append(("stem (wgmma, operand built in shared memory)", get(r["out"]), op_ref.stem(image, sdf)))
        elif kind == L.OP_IM2COL_STEM:
            checks.append(("im2col of the normalised frame", get(r["out"])[:, :27], op_ref.im2col_stem(image)))
        elif kind == L.OP_FUSE:
            checks.append((f"fuse x{len(r['ins'])}", get(r["out"]), op_ref.fuse([get(t) for t in r["ins"]], a["shifts"], a["relu"])))
        elif kind == L.OP_BILINEAR2X:
            checks.append(("bilinear x2", get(r["out"]), op_ref.bilinear2x(get(r["ins"][0]))))
        elif kind == L.OP_COORD:
            xc = eng.view(r["out"]).float().cpu()
            exp = op_ref.coord(xc.shape[1], xc.shape[2])[None].expand(xc.shape[0], -1, -1, -1)
            w0 = eng.spec.widths[0]
            checks.append(("coord channels", xc[..., w0:w0 + 2].permute(0, 3, 1, 2), exp))
            assert float(xc[..., w0 + 2:].abs().max()) == 0.0, "pad channels of the coord concat are not zero"
        elif kind == L.OP_POOL:
            pool_in = r["ins"]                                                  # partials are checked after the merge
        elif kind == L.OP_PARTHEAD:
            B = eng.batch
            pooled = eng.view("pooled").float().cpu().view(B, 256, 32)
            checks.append(("attention pooling (softmax over HW x features)", pooled,
                           op_ref.attention_pool(get(pool_in[0]), get(pool_in[1]))))
            for s in "lr":
                pare = _pare(eng, s)
                checks.append((f"part head {s}: LocallyConnected2d + Linear", pare, op_ref.part_offsets(pooled, sdf, s)))
        else:
            raise AssertionError(f"op kind {kind} has no teacher-forced check")
        for label, got, exp in checks:
            assert torch.isfinite(got).all(), (i, label)
            rows.append((i, label, rel_err(got.numpy(), exp.numpy())))
    return rows


def _run(sd, image, dtype, widths=None):
    from acr_b200.engine import Engine
    torch.set_num_threads(min(32, os.cpu_count()))   # > 64 threads oversubscribe these small convs (measured 40x slower at 128)
    eng = Engine(sd, image.shape[0], "cuda", dtype, reuse_memory=False, widths=widths)   # every intermediate tensor is kept
    eng.run(image.cuda())
    torch.cuda.synchronize()
    rows = sweep(eng, sd, image, TOL[dtype])
    worst = sorted(rows, key=lambda r: -r[2])[:5]
    print(f"teacher-forced sweep {dtype}: {len(rows)} checks over {len(eng.recs)} launches; worst:",
          [(i, l, f"{e:.2e}") for i, l, e in worst])
    assert len(rows) >= len(eng.recs) - 1
    bad = [(i, l, e) for i, l, e in rows if not e <= TOL[dtype]]
    assert not bad, f"{len(bad)} ops above {TOL[dtype]:.2e}: {bad[:8]}"


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_every_op_teacher_forced_16bit(sd, image, dtype):
    """The product plans (wgmma conv, x-paired 32-channel convs, tensor-core stem and pooling)."""
    _run(sd, image, dtype)


def test_every_op_teacher_forced_with_folded_fuse_sums(sd, image, monkeypatch):
    """Opt-in plan (ACR_B200_FOLD_FUSE=1): the fuse sums of the coarser HR-module outputs computed in the epilogue of the
    stride-2 conv that produces one of their terms (extra terms nearest-upsampled in the epilogue)."""
    monkeypatch.setenv("ACR_B200_FOLD_FUSE", "1")
    _run(sd, image, torch.bfloat16)


def test_every_op_teacher_forced_fp32_validation_plan(sd, image):
    """The fp32 validation plan (model_precision='fp32'): fp32 storage, fp64 accumulate."""
    _run(sd, image, torch.float32)


def test_every_op_teacher_forced_hrnet_w48(image):
    """The HRNet-W48 trunk of BASELINE configs[4]: the reference has no such network (parity unpinned: no golden can
    exist), so every launch of its plan is pinned against the oracle's per-op restatement instead -- 48/96/192/384-
    channel convs (zero-filled K tails, N split at 384 outputs), fuse layers, heads on the 50-channel coord concat."""
    from acr_b200.netspec import WIDTHS_W48, build_acr_spec
    from acr_b200.synth import synth_state_dict
    sd48 = synth_state_dict(3, spec=build_acr_spec(512, widths=WIDTHS_W48))
    _run(sd48, image, torch.bfloat16, widths=WIDTHS_W48)


def test_heads_only_plan_teacher_forced(sd, image):
    """The ACR.head_forward plan (ops after the trunk) on an external feature."""
    from acr_b200.engine import Engine
    from oracle import net_ref
    torch.set_num_threads(min(32, os.cpu_count()))   # > 64 threads oversubscribe these small convs (measured 40x slower at 128)
    x = net_ref._Net(sd).backbone(image)
    eng = Engine(sd, 1, "cuda", torch.bfloat16, reuse_memory=False, head_only=True)
    eng.run_heads(x.cuda())
    torch.cuda.synchronize()
    rows = sweep(eng, sd, image, TOL[torch.bfloat16])
    bad = [(i, l, e) for i, l, e in rows if not e <= TOL[torch.bfloat16]]
    assert len(rows) >= 55 and not bad, bad[:8]
