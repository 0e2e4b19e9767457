"""GPU: every launch plan per image at batch > 1, on distinct frames.

The network kernels work per image and use no atomics or other order-dependent sums, so an image's maps must not depend
on the batch it travels in or on its position in it -- bit for bit, in every plan.  The batch is taken past one tile per
SM (B = SMs + 5): the persistent conv and fused-block grids have one CTA per SM, and at 512 x 512 the branch-3 and head
convs have one 16 x 16 super-tile per image, so only at such a batch do some CTAs run a second tile of those classes.
Every frame comes from its own seed: a kernel that reads another image's per-image bias, pooling partials, part-head
offsets or batch coordinate gives a different answer for that image (a batch of repeated frames would hide it).

* per image == batch 1, every plan variant; the product batch (256) permuted == permuted outputs;
* every launch of the plan per image == batch 1 (names the first op that mixes images), every launch of a 3-frame plan
  teacher forced against the oracle;
* the per-image bias and 1.1 ** x of the 16-bit conv at op level against fp64;
* CUDA-graph replay == eager at batch 4 and SMs + 5, the parse / MANO tail at SMs + 5 against the oracle.
"""
import gc
import os
import time

import numpy as np
import pytest
import torch

from acr_b200 import lib as L
from tests.helpers import CONV_BIAS_PER_IMAGE, CONV_POW11_CH0, rel_err, rup, run_conv_case
from tests.test_gpu_network import sd  # noqa: F401  (module fixture)

pytestmark = pytest.mark.gpu

MAPS = ("segms", "l_center_map", "r_center_map", "l_params_maps", "r_params_maps", "l_prior_maps", "r_prior_maps")
KEPT = MAPS + ("pooled", "l_pare", "r_pare", "feat32", "l_bias_img", "r_bias_img")
EXTRA = ("feat32", "l_bias_img", "r_bias_img")    # kept beyond the plan's outputs (keep_extra)


def n_sm():
    return torch.cuda.get_device_properties(0).multi_processor_count


def big_batch():
    """More virtual tiles than CTAs for every one-tile-per-image conv class: some CTAs run a second tile, most do not."""
    return n_sm() + 5


def frames(n, first_seed=0):
    """(n, 512, 512, 3) uint8: frame i from seed first_seed + i, uniform noise over its own intensity range."""
    out = torch.empty(n, 512, 512, 3, dtype=torch.uint8)
    for i in range(n):
        g = torch.Generator().manual_seed(1000 + first_seed + i)
        lo, hi = int(torch.randint(0, 96, (1,), generator=g)), int(torch.randint(160, 257, (1,), generator=g))
        out[i] = torch.randint(lo, hi, (512, 512, 3), generator=g, dtype=torch.uint8)
    return out


def features(n, first_seed=0):
    """(n, 32, 128, 128) backbone features for the heads-only plan, feature i from seed first_seed + i."""
    return torch.stack([torch.randn(32, 128, 128, generator=torch.Generator().manual_seed(2000 + first_seed + i))
                        for i in range(n)])


def logical(eng, name):
    """(B, ...) view of a tensor's logical channels (the part head packs the 106 offsets of an image densely)."""
    t = eng.spec.tensors[name] if isinstance(name, str) else name
    if t.name.endswith("_pare"):
        return eng.view(t).reshape(-1)[: eng.batch * 106].view(eng.batch, 106)
    return eng.view(t)[..., : t.C]


def free():
    """Give the device memory of engines the caller has dropped back before the next big one is built."""
    gc.collect()
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------- plan variants
def _sd_w48():
    from acr_b200.netspec import WIDTHS_W48, build_acr_spec
    from acr_b200.synth import synth_state_dict
    return synth_state_dict(3, spec=build_acr_spec(512, widths=WIDTHS_W48))


def _sd_resnet():
    from acr_b200.netspec import build_acr_spec
    from acr_b200.synth import synth_state_dict
    return synth_state_dict(0, spec=build_acr_spec(512, backbone="resnet50"))


# name -> Engine keyword arguments, environment switches (read at plan creation), batches (big = SMs + 5), state dict
VARIANTS = {
    "w32-bf16": dict(),
    "w32-fp16": dict(kw=dict(act_dtype=torch.float16)),
    "w32-bf16-unfused-blocks": dict(env={"ACR_B200_FUSE_BLOCKS": "0"}),
    "w32-bf16-folded-fuse": dict(env={"ACR_B200_FOLD_FUSE": "1"}),
    "w32-bf16-tma-store": dict(env={"ACR_B200_TMA_OUT": "1"}),
    "w32-bf16-im2col-stem": dict(env={"ACR_B200_STEM_FUSED": "0"}),
    "w32-bf16-cuda-core-stem": dict(kw=dict(stem_on_tensor_cores=False)),
    "w48-bf16": dict(kw=dict(widths=(48, 96, 192, 384)), sd=_sd_w48),
    "tf32": dict(kw=dict(act_dtype=torch.float32, tf32=True)),
    "resnet50-bf16": dict(kw=dict(backbone="resnet50"), sd=_sd_resnet, batches=("big",)),
    "fp32-validation": dict(kw=dict(act_dtype=torch.float32), batches=(3,)),     # flat grids: a big batch adds nothing
    "heads-only-bf16": dict(kw=dict(head_only=True), batches=(3,)),
}


def _run(eng, inputs):
    if eng.head_only:
        eng.run_heads(inputs.cuda())
    else:
        eng.run(inputs.cuda())
    torch.cuda.synchronize()


@pytest.mark.parametrize("variant", list(VARIANTS))
def test_every_image_equals_its_batch_1_run(sd, variant, monkeypatch):
    """Each plan variant on B distinct frames: the kept outputs of the chosen images (0, 1, SMs - 1, SMs, B - 1 at
    B = SMs + 5; all three at B = 3) equal those of a batch-1 plan run on that frame alone, bit for bit."""
    from acr_b200.engine import Engine
    v = VARIANTS[variant]
    for k, val in v.get("env", {}).items():
        monkeypatch.setenv(k, val)
    kw = dict(v.get("kw", {}))
    dtype = kw.pop("act_dtype", torch.bfloat16)
    sdv = v["sd"]() if "sd" in v else sd
    make_inputs = features if kw.get("head_only") else frames
    B_big = big_batch()
    weights, want = None, {}          # image index -> {name: outputs of that image in the batched plan}
    for b in v.get("batches", ("big", 3)):
        B = B_big if b == "big" else b
        pick = sorted({0, 1, n_sm() - 1, n_sm(), B - 1}) if b == "big" else list(range(B))
        eng = Engine(sdv, B, "cuda", dtype, keep_extra=EXTRA, weights=weights, **kw)
        weights = eng.weights
        _run(eng, make_inputs(B))
        kept = {n: logical(eng, n) for n in KEPT}
        for i in pick:
            want.setdefault(i, []).append((B, {n: t[i].clone() for n, t in kept.items()}))
        del kept, eng
        free()
    one = Engine(sdv, 1, "cuda", dtype, keep_extra=EXTRA, weights=weights, **kw)
    for i, runs in sorted(want.items()):
        _run(one, make_inputs(1, first_seed=i))
        for B, w in runs:
            for n in KEPT:
                got = logical(one, n)[0]
                assert torch.isfinite(got).all(), (variant, n, i)
                assert torch.equal(w[n], got), f"{variant}: image {i} of a batch of {B}: {n} differs from its batch-1 run"


def test_permuted_product_batch_gives_permuted_outputs(sd):
    """W32 bf16 at the product batch (256): the frames in order and in a fixed permutation (pi(0) != 0); every kept output
    of every image comes back permuted, bit for bit."""
    from acr_b200.engine import Engine
    B = 256
    x = frames(B)
    perm = (7 * torch.arange(B) + 3) % B          # 7 is prime to 256: a permutation, pi(0) = 3
    eng = Engine(sd, B, "cuda", keep_extra=EXTRA)
    _run(eng, x)
    first = {n: logical(eng, n).clone() for n in KEPT}
    _run(eng, x[perm].contiguous())
    perm = perm.cuda()
    for n in KEPT:
        assert torch.equal(logical(eng, n), first[n][perm]), n
    del first, eng
    free()


# ---------------------------------------------------------------------------------------- launch by launch, B = 3
def _no_reuse(sdv, B, dtype, tf32, inputs, weights=None):
    from acr_b200.engine import Engine
    eng = Engine(sdv, B, "cuda", dtype, reuse_memory=False, tf32=tf32, weights=weights)   # every intermediate is kept
    _run(eng, inputs)
    return eng


@pytest.mark.parametrize("precision", ["bf16", "tf32"])
def test_every_launch_per_image_equals_batch_1(sd, precision):
    """Every record of the plan (block intermediates included: ACR_CONV_BLOCK_MID without memory reuse), its output and
    auxiliary tensors per image at B = 3 against the batch-1 plan on the same frame.  A failure names the first op that
    mixes images."""
    dtype, tf32 = (torch.bfloat16, False) if precision == "bf16" else (torch.float32, True)
    x = frames(3)
    eng = _no_reuse(sd, 3, dtype, tf32, x)
    assert any(r.get("block_mid") for r in eng.recs) or tf32
    one = _no_reuse(sd, 1, dtype, tf32, x[:1], weights=eng.weights)
    assert [r["kind"] for r in one.recs] == [r["kind"] for r in eng.recs]
    for i in range(3):
        if i:
            _run(one, x[i:i + 1])
        for k, (r, r1) in enumerate(zip(eng.recs, one.recs)):
            for t, t1 in zip([r["out"]] + r.get("aux", []), [r1["out"]] + r1.get("aux", [])):
                assert t.name == t1.name
                a, b = logical(eng, t)[i], logical(one, t1)[0]
                assert torch.equal(a, b), \
                    f"op {k} (kind {r['kind']}, {r.get('attrs', {}).get('w', '')}): image {i} of 3, tensor {t.name}: " \
                    f"max |diff| {float((a.float() - b.float()).abs().max()):.3g}"
    del eng, one
    free()


def test_every_op_teacher_forced_at_batch_3(sd):
    """tests/test_gpu_teacher_forced.sweep, unchanged, on a bf16 plan of three distinct frames: the numbers of every op for
    images 1 and 2 too are pinned against the oracle at the per-op bound 2^-7, not only their equality to another run."""
    from tests.test_gpu_teacher_forced import TOL, sweep
    torch.set_num_threads(min(32, os.cpu_count()))   # > 64 threads oversubscribe these small convs
    x = frames(3)
    eng = _no_reuse(sd, 3, torch.bfloat16, False, x)
    t0 = time.perf_counter()
    rows = sweep(eng, sd, x, TOL[torch.bfloat16])
    print(f"teacher-forced sweep, bf16, 3 frames: {len(rows)} checks over {len(eng.recs)} launches in "
          f"{time.perf_counter() - t0:.1f} s of CPU; worst:", [(i, l, f"{e:.2e}") for i, l, e in
                                                               sorted(rows, key=lambda r: -r[2])[:5]])
    assert len(rows) >= len(eng.recs) - 1
    bad = [(i, l, e) for i, l, e in rows if not e <= TOL[torch.bfloat16]]
    assert not bad, f"{len(bad)} ops above 2^-7: {bad[:8]}"
    del eng
    free()


# --------------------------------------------------------------------------------------------------- op level
# (B, H, W, cin, cout, k, s, relu, residual, bias, bn, out_f32, flags); B = 0 stands for SMs + 5
BIAS_CASES = [
    (3, 64, 64, 128, 109, 1, 1, False, False, False, False, True, CONV_BIAS_PER_IMAGE),    # folded final conv, fp32 out
    (3, 64, 64, 128, 109, 1, 1, False, False, False, False, False, CONV_BIAS_PER_IMAGE),   # ... 16-bit out
    (3, 64, 64, 64, 3, 3, 1, False, False, True, True, False, CONV_POW11_CH0),             # cam head, 1.1 ** channel 0
    (0, 16, 16, 128, 109, 1, 1, False, False, False, False, True, CONV_BIAS_PER_IMAGE),    # one super-tile per image:
    (0, 16, 16, 128, 109, 1, 1, False, False, False, False, False, CONV_BIAS_PER_IMAGE),   # CTAs on their second tile
    (0, 16, 16, 64, 3, 3, 1, False, False, True, True, False, CONV_POW11_CH0),             # read the bias too
]


@pytest.mark.parametrize("dt", [L.DT_BF16, L.DT_F16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("case", BIAS_CASES, ids=lambda c: f"B{c[0] or 'big'}-{c[1]}x{c[2]}-{c[3]}to{c[4]}-k{c[5]}-"
                         f"{'f32' if c[11] else '16bit'}-flags{c[12]}")
def test_conv_per_image_bias_and_pow11_vs_fp64(case, dt):
    """ACR_CONV_BIAS_PER_IMAGE (a (B, cout_pad) fp32 bias, one row per image, very different from image to image) and
    ACR_CONV_POW11_CH0 on the 16-bit wgmma conv, against fp64 on the same rounded operands at the bound of
    tests/test_gpu_conv.py."""
    B, H, W, cin, cout, k, s, relu, res, bias, bn, f32, flags = case
    B = B or big_batch()
    bimg = None
    if flags & CONV_BIAS_PER_IMAGE:     # zero past the real channels, as the part head writes it
        g = torch.Generator().manual_seed(B + cout)
        bimg = torch.zeros(B, rup(cout, 16))
        bimg[:, :cout] = torch.randn(B, cout, generator=g) * 0.3 + torch.randn(B, 1, generator=g) * 3.0
    got, exp, pad_ok = run_conv_case(L.OP_CONV, B, H, W, cin, cout, k, s, relu, res, bias, bn, f32, dt=dt,
                                     seed=hash(case) % 1000, flags=flags, bias_img=bimg)
    scale = float(exp.abs().max())
    err = (got.double() - exp).abs().amax(dim=(1, 2, 3))
    tol = scale * (2e-5 if f32 else (2 ** -8 if dt == L.DT_BF16 else 2 ** -10)) + 1e-6
    assert pad_ok, "padding channels of the output are not zero"
    worst = int(err.argmax())
    assert float(err[worst]) <= tol, f"image {worst} of {B}: max err {float(err[worst]):.4g} > tol {tol:.4g}"


# ------------------------------------------------------------------------------------------- graph and pipeline tail
def _assets():
    from acr_b200.synth import make_synthetic_mano
    return {"left": make_synthetic_mano("left"), "right": make_synthetic_mano("right")}


def test_graph_replay_equals_eager_beyond_batch_1():
    """ACR.capture_graph(B) for B = 4 and SMs + 5 (W32 bf16): replay == eager fused_forward bit for bit, on two frame batches
    with different detection counts (the n_dev row mask of MANO moves between replays).  The centre-head bias is set so
    that the detection threshold falls between the frames' centre-map maxima."""
    from acr.main import ACR
    from acr_b200.engine import Engine
    from acr_b200.synth import load_bn_calibration, synth_state_dict
    from oracle.parse_ref import CONF_THRESH
    B_big = big_batch()
    x = frames(B_big)
    sd1 = synth_state_dict(0, bn_stats=load_bn_calibration(0))        # centre bias 1.0
    eng = Engine(sd1, B_big, "cuda")
    _run(eng, x)
    peak = {s: logical(eng, f"{s}_center_map").float().amax(dim=(1, 2, 3)).cpu() for s in "lr"}
    del eng
    free()
    # threshold t in the widest gap of the middle half of the maxima: a frame's side is detected iff its maximum > t once
    # the bias is 1.0 + CONF_THRESH - t
    m = torch.cat([peak["l"], peak["r"]]).sort().values
    q = len(m) // 4
    gaps = m[q + 1: 3 * q + 1] - m[q: 3 * q]
    j = q + int(gaps.argmax())
    t = float(m[j] + m[j + 1]) / 2
    det = (peak["l"] > t).int() + (peak["r"] > t).int()
    app = ACR(state_dict=synth_state_dict(0, bn_stats=load_bn_calibration(0), center_bias=1.0 + CONF_THRESH - t),
              mano_assets=_assets())
    order = torch.argsort(-det, stable=True)
    for B in (4, B_big):
        offs = torch.tensor([[512., 512, 0, 0, 0, 0, 0, 0, 0, 0]]).repeat(B, 1).cuda()
        most, fewest = order[:B], order[-B:] if B < B_big else order[-((B + 1) // 2):].repeat(2)[:B]
        replay = app.capture_graph(B)
        counts = []
        for idx in (most, fewest):
            batch = x[idx].contiguous().cuda()
            bufs, mano = app.fused_forward(batch, offs)
            torch.cuda.synchronize()
            n = int(bufs.counts[2])
            v_eager, p_eager = mano["verts"][:n].clone(), bufs.params_pred[:n].clone()
            c_eager = bufs.counts.clone()
            bufs_g, mano_g = replay(batch, offs)
            torch.cuda.synchronize()
            assert torch.equal(bufs_g.counts, c_eager), (B, c_eager.tolist(), bufs_g.counts.tolist())
            assert torch.equal(mano_g["verts"][:n], v_eager) and torch.equal(bufs_g.params_pred[:n], p_eager), B
            counts.append(n)
        print(f"graph replay at batch {B}: {counts[0]} and {counts[1]} hands")
        assert counts[0] != counts[1], (B, counts)
        del replay
        free()
    del app
    free()


def test_pipeline_tail_at_a_big_batch_vs_oracle(sd):
    """batch_forward at B = SMs + 5 against parse_ref.parse and mano_ref.mano_wrapper_forward run on the plan's own maps:
    indices and centres bit-exact, params_pred within 1e-5, MANO within 1e-4.  (Parsing is batch-global on purpose --
    determine_coeff uses the batch's first left and first right centre, as the reference does -- so rows are compared
    with the oracle on the whole batch, not per image.)"""
    from acr.main import ACR
    from oracle import mano_ref, parse_ref
    B = big_batch()
    assets = _assets()
    app = ACR(state_dict=sd, mano_assets=assets)
    out = app.batch_forward(frames(B))
    torch.cuda.synchronize()
    maps = {k: out[k].cpu().numpy() for k in MAPS if k != "segms"}
    p = parse_ref.parse(maps)
    N = p["params_pred"].shape[0]
    assert out["params_pred"].shape[0] == N
    for k in ("reorganize_idx", "l_centers_pred", "r_centers_pred", "detection_flag"):
        assert (out[k].cpu().numpy() == p[k]).all(), k
    assert np.abs(out["params_pred"].cpu().numpy() - p["params_pred"]).max() < 1e-5
    L_, R_ = int(p["left_hand_num"][0]), int(p["right_hand_num"][0])
    offs = np.tile(np.array([512, 512, 0, 0, 0, 0, 0, 0, 0, 0], np.float32), (N, 1))
    m = mano_ref.mano_wrapper_forward(assets, p["params_dict"]["poses"], p["params_dict"]["betas"], L_, R_,
                                      p["params_dict"]["cam"], offs)
    for k in ("verts", "j3d", "pj2d_org"):
        e = rel_err(out[k].cpu().numpy(), m[k])
        assert e < 1e-4, (k, e)
    del out, app
    free()
