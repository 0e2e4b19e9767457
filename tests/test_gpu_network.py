"""GPU parity: the whole launch plan (backbone + heads), the fused pipeline and the drop-in API vs the
oracle / the reference goldens."""
import os

import numpy as np
import pytest
import torch

from tests.helpers import GOLDEN, rel_err

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def sd():
    from acr_b200.synth import load_bn_calibration, synth_state_dict
    return synth_state_dict(0, bn_stats=load_bn_calibration(0))


@pytest.fixture(scope="module")
def image():
    gi = torch.Generator().manual_seed(123)
    return torch.randint(0, 256, (2, 512, 512, 3), generator=gi, dtype=torch.uint8)


@pytest.fixture(scope="module")
def oracle_out(sd, image):
    from oracle import net_ref
    torch.set_num_threads(min(32, os.cpu_count()))   # > 64 threads oversubscribe these small convs (measured 40x slower at 128)
    return net_ref.net_forward(sd, image, return_backbone=True)


def _engine_maps(sd, image, ref_conv, dtype=torch.bfloat16):
    from acr_b200.engine import Engine
    eng = Engine(sd, image.shape[0], "cuda", dtype, debug_ref_conv=ref_conv, keep_extra=("feat32",))
    eng.run(image.cuda())
    torch.cuda.synchronize()
    names = ["l_center_map", "r_center_map", "l_params_maps", "r_params_maps", "l_prior_maps", "r_prior_maps", "segms"]
    out = {n: eng.map_nchw(n).cpu() for n in names}
    out["backbone"] = eng.view("feat32")[..., :32].permute(0, 3, 1, 2).float().cpu()
    out["pooled"] = eng.view("pooled").view(image.shape[0], 256, 32).cpu()
    return eng, out


# Tolerances of the whole-network comparisons.  The seeded random-weight network amplifies storage
# round-off: the ORACLE ITSELF, re-run with every conv/fuse output rounded to the storage type
# (net_ref.net_forward(act_dtype=...)), deviates from its own fp32 result by (max-abs / max-abs, measured
# here on this input):  bf16  0.06 (backbone) .. 0.12 (centre maps);  fp16  0.007 .. 0.019.
# Kernel-level parity is pinned op by op in test_gpu_conv.py (identical operands, fp32-accurate); the
# whole-network tests below pin the WIRING: a wrong tensor / weight / epilogue gives O(1) errors.
TOL_NET = {torch.bfloat16: 0.30, torch.float16: 0.06}


def _cmp(out, ref, tol):
    worst = {}
    for k in ("backbone", "segms", "l_center_map", "r_center_map", "l_params_maps", "r_params_maps",
              "l_prior_maps", "r_prior_maps", "pooled"):
        assert torch.isfinite(out[k]).all(), k
        worst[k] = rel_err(out[k].numpy(), ref[k].numpy())
    print("rel errors:", {k: f"{v:.3e}" for k, v in worst.items()})
    for k, v in worst.items():
        assert v < tol, (k, v)
    return worst


def _stem_out(sd, image, dtype, form):
    from acr_b200 import lib as L
    from acr_b200.engine import Engine
    os.environ["ACR_B200_STEM_FUSED"] = "0" if form == "im2col" else "1"
    try:
        eng = Engine(sd, image.shape[0], "cuda", dtype, keep_extra=("t1_stem1",), stem_on_tensor_cores=form != "cuda_cores")
    finally:
        del os.environ["ACR_B200_STEM_FUSED"]
    kinds = [r["kind"] for r in eng.recs]
    want = {"fused": L.OP_STEM_TC, "im2col": L.OP_IM2COL_STEM, "cuda_cores": L.OP_STEM}[form]
    assert kinds.count(want) == 1 and sum(kinds.count(k) for k in (L.OP_STEM_TC, L.OP_IM2COL_STEM, L.OP_STEM)) == 1
    eng.run(image.cuda())
    torch.cuda.synchronize()
    return eng.view("t1_stem1")[..., :64].permute(0, 3, 1, 2).float().cpu()


@pytest.mark.parametrize("form", ["fused", "im2col", "cuda_cores"])
@pytest.mark.parametrize("dtype,tol", [(torch.float16, 3e-3), (torch.bfloat16, 2e-2)])
def test_stem_vs_oracle(sd, image, form, dtype, tol):
    """conv1 + bn1 + ReLU on uint8 frames (acr/model.py:831-835) in its three forms -- one wgmma kernel that builds the
    im2col operand in shared memory (csrc/stem_tc.cu, the default), im2col + a 1x1 wgmma conv (ACR_B200_STEM_FUSED=0),
    the direct CUDA-core kernel -- against the oracle's fp32 conv (error = 16-bit rounding of taps/weights/output)."""
    from oracle import net_ref
    got = _stem_out(sd, image, dtype, form)
    net = net_ref._Net(sd)
    x = (image.float().permute(0, 3, 1, 2) / 255.0) * 2.0 - 1.0
    ref = net.cbr(x, "backbone.conv1", "backbone.bn1", stride=2)
    assert rel_err(got.numpy(), ref.numpy()) < tol


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_fused_stem_equals_the_im2col_form(sd, image, dtype):
    """Same 16-bit taps, same 16-bit folded weights, fp32 accumulation in both: the two tensor-core forms may differ only
    by the bias (added in fp32 by the conv epilogue, carried as a hi + lo 16-bit pair through the K dimension by the fused
    kernel: 2^-17 relative) and by the summation order -- at most one 16-bit ulp of the output, on a handful of pixels."""
    a, b = _stem_out(sd, image, dtype, "fused"), _stem_out(sd, image, dtype, "im2col")
    ulp = 2.0 ** -7 if dtype == torch.bfloat16 else 2.0 ** -10
    diff = (a - b).abs()
    assert (diff <= ulp * torch.maximum(a.abs(), b.abs()) + 1e-6).all(), float(diff.max())
    assert (diff > 0).float().mean() < 0.02


@pytest.mark.parametrize("dtype,tol", [(torch.float16, 1e-3), (torch.bfloat16, 4e-3)])
def test_attention_pooling_vs_torch(sd, image, dtype, tol):
    """Hadamard_product / part attention (acr/model.py:103-128) as the split-softmax tensor-core GEMM over
    pixels: compared on the engine's OWN stored feature map and logits with an fp32 softmax + einsum (the
    only difference is the one rounding of the softmax weights to the storage type)."""
    from acr_b200.engine import Engine
    spec = Engine(None, 1, "cpu", dry_run=True).spec
    contact = [n for n in spec.tensors if n.endswith("_contact")][0]
    eng = Engine(sd, image.shape[0], "cuda", dtype, keep_extra=(contact,))
    eng.run(image.cuda())
    torch.cuda.synchronize()
    B = image.shape[0]
    feat = eng.view(contact)[..., :256].float().reshape(B, -1, 256)
    logit = eng.view("segms")[:, ::2, ::2, 1:33].float().reshape(B, -1, 32)
    ref = torch.einsum("bpc,bpj->bcj", feat, torch.softmax(logit, dim=1))
    got = eng.view("pooled").view(B, 256, 32)
    assert rel_err(got.cpu().numpy(), ref.cpu().numpy()) < tol


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_pool_on_tcgen05_equals_the_mma_sync_form(sd, image, dtype):
    """csrc/pool_tc.cu (wgmma / TMA, one maximum per 1024-pixel chunk) against the warp-level mma.sync kernel it
    replaces (ACR_B200_POOL_TC=0, running maximum per 512 pixels) on the same plan and frames: the two differ only in
    which maximum the 16-bit weights were rounded against and in the summation order."""
    from acr_b200.engine import Engine
    eng = Engine(sd, image.shape[0], "cuda", dtype)
    got = {}
    for form in ("1", "0"):
        os.environ["ACR_B200_POOL_TC"] = form
        try:
            eng.run(image.cuda())
            torch.cuda.synchronize()
        finally:
            del os.environ["ACR_B200_POOL_TC"]
        got[form] = eng.view("pooled").view(image.shape[0], 256, 32).clone()
        assert torch.isfinite(got[form]).all()
    assert rel_err(got["1"].cpu().numpy(), got["0"].cpu().numpy()) < (2e-3 if dtype == torch.bfloat16 else 3e-4)


def test_plan_fp16_refconv_vs_oracle(sd, image, oracle_out):
    """Everything except the tensor-core conv (stem, fuse, bilinear, pooling, part head, plan wiring)."""
    _, out = _engine_maps(sd, image, ref_conv=True, dtype=torch.float16)
    _cmp(out, oracle_out, TOL_NET[torch.float16])


def test_plan_fp16_tcgen05_vs_oracle(sd, image, oracle_out):
    _, out = _engine_maps(sd, image, ref_conv=False, dtype=torch.float16)
    _cmp(out, oracle_out, TOL_NET[torch.float16])


def test_plan_bf16_tcgen05_vs_oracle(sd, image, oracle_out):
    """BASELINE configs[2] precision (bf16 storage, fp32 accumulate)."""
    _, out = _engine_maps(sd, image, ref_conv=False)
    _cmp(out, oracle_out, TOL_NET[torch.bfloat16])


# Bound (this test prints the observed values): engine(bf16) vs the same-rounding oracle <= 0.07 on every map, while the
# fp32 oracle and the same-rounding oracle are 0.13-0.18 apart.  Bound = 2x the largest observed value.
TOL_SAME_ROUNDING = {torch.bfloat16: 0.14, torch.float16: 0.03}


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_plan_vs_same_rounding_oracle(sd, image, oracle_out, dtype):
    """BASELINE dtype, whole network, same rounding points: the oracle with BN folded into weights that are
    rounded to the storage type, 16-bit stem taps / raw head outputs / softmax weights and every conv / fuse /
    bilinear output rounded (net_ref.net_forward(act_dtype, fold_round=True)).  What remains is fp32 summation
    order (tensor-core tiles vs MKL-DNN), which flips individual 16-bit roundings that the random network then
    amplifies -- the distance to this oracle must be well inside the distance between the two oracles."""
    from oracle import net_ref
    same = net_ref.net_forward(sd, image, dtype, return_backbone=True, fold_round=True)
    _, out = _engine_maps(sd, image, ref_conv=False, dtype=dtype)
    keys = ("backbone", "segms", "l_center_map", "r_center_map", "l_params_maps", "r_params_maps", "l_prior_maps",
            "r_prior_maps", "pooled")
    d_engine = {k: rel_err(out[k].numpy(), same[k].numpy()) for k in keys}
    d_oracles = {k: rel_err(same[k].numpy(), oracle_out[k].numpy()) for k in keys}
    print(f"{dtype} engine vs same-rounding oracle:", {k: f"{v:.3e}" for k, v in d_engine.items()})
    print(f"{dtype} same-rounding oracle vs fp32 oracle:", {k: f"{v:.3e}" for k, v in d_oracles.items()})
    for k in keys:
        assert d_engine[k] < TOL_SAME_ROUNDING[dtype], (k, d_engine[k])


def test_fp32_pipeline_vs_reference_golden(sd, image):
    """model_precision='fp32' (the reference's shipped default) = the fp32 validation plan.  The WHOLE pipeline
    -- frames -> maps -> centres -> parameters -> 6D->aa -> MANO -> vertices / joints / projection -- against the
    goldens written by the unmodified reference (tests/golden/net_golden.npz): identical centres, every
    floating-point output within the north star's 1e-4 (relative to the output's range)."""
    from acr.config import args
    from acr.main import ACR
    from acr_b200.synth import make_synthetic_mano
    g = np.load(os.path.join(GOLDEN, "net_golden.npz"))
    args().model_precision = "fp32"
    try:
        assets = {"left": make_synthetic_mano("left"), "right": make_synthetic_mano("right")}
        app = ACR(state_dict=sd, mano_assets=assets)
        out = app.batch_forward(image)
        torch.cuda.synchronize()
        errs = {}
        for k in ("l_center_map", "r_center_map"):
            errs[k] = rel_err(out[k].cpu().numpy(), g[k])
        errs["segms_crop"] = rel_err(out["segms"][:, :, 100:108, 100:108].cpu().numpy(), g["segms_crop"])
        for k, gk in (("l_params_maps", "l_params_crop"), ("r_params_maps", "r_params_crop"), ("l_prior_maps", "l_prior_crop")):
            errs[gk] = rel_err(out[k][:, :, 30:34, 30:34].cpu().numpy(), g[gk])
        assert (out["l_centers_pred"].cpu().numpy() == g["l_centers_pred"]).all()
        assert (out["r_centers_pred"].cpu().numpy() == g["r_centers_pred"]).all()
        assert (out["reorganize_idx"].cpu().numpy() == g["reorganize_idx"]).all()
        assert (out["detection_flag"].cpu().numpy() == g["detection_flag"]).all()
        errs["params_pred"] = rel_err(out["params_pred"].cpu().numpy(), g["params_pred"])
        for k in ("poses", "betas", "cam"):
            errs[k] = rel_err(out["params_dict"][k].cpu().numpy(), g[k])
        for k in ("verts", "j3d", "pj2d_org"):
            errs[k] = rel_err(out[k].cpu().numpy(), g[k])
        errs["verts_max_abs_m"] = float(np.abs(out["verts"].cpu().numpy() - g["verts"]).max())
        print("fp32 pipeline vs reference golden:", {k: f"{v:.2e}" for k, v in errs.items()})
        for k, v in errs.items():
            assert v < 1e-4, (k, v)
    finally:
        args().model_precision = "bf16"


@pytest.mark.parametrize("precision,tol", [("fp32", 1e-4), ("fp16", TOL_NET[torch.float16])])
def test_head_forward_on_external_feature(sd, image, oracle_out, precision, tol):
    """ACR.head_forward(x) (/root/reference/acr/model.py:47-65): the heads-only plan on the ORACLE's backbone
    output must reproduce the oracle's seven maps."""
    from acr.config import args
    from acr.model import ACR
    args().model_precision = precision
    try:
        model = ACR()
        model.load_state_dict(sd, strict=True)
        model = model.cuda()
        out = model.head_forward(oracle_out["backbone"].cuda())
        torch.cuda.synchronize()
        assert set(out) == {"l_params_maps", "r_params_maps", "l_center_map", "r_center_map", "l_prior_maps",
                            "r_prior_maps", "segms"}
        for k, v in out.items():
            assert v.dtype == torch.float32 and tuple(v.shape) == tuple(oracle_out[k].shape), k
            e = rel_err(v.cpu().numpy(), oracle_out[k].numpy())
            assert e < tol, (k, e)
    finally:
        args().model_precision = "bf16"


def test_outputs_survive_the_next_forward(sd, image):
    """Like the reference, every forward() returns its own tensors: a second call with the same batch size must
    not overwrite the first call's outputs; a map that was not read in time raises instead of going stale."""
    from acr.config import args
    from acr.model import ACR
    args().model_precision = "fp16"
    try:
        model = ACR()
        model.load_state_dict(sd, strict=True)
        model = model.cuda()
        meta = lambda im: {"image": im, "offsets": torch.tensor([[512., 512, 0, 0, 0, 0, 0, 0, 0, 0]] * 2),
                           "batch_ids": torch.arange(2)}
        a = model(meta(image))
        keep = {k: a[k].clone() for k in ("params_pred", "reorganize_idx", "l_centers_pred", "detection_flag")}
        keep_pd = {k: v.clone() for k, v in a["params_dict"].items()}
        centre = a["l_center_map"].clone()            # read in time
        b = model(meta(torch.flip(image, dims=[0, 2])))
        torch.cuda.synchronize()
        assert not torch.equal(b["params_pred"], keep["params_pred"])
        for k, v in keep.items():
            assert torch.equal(a[k], v), k
        for k, v in keep_pd.items():
            assert torch.equal(a["params_dict"][k], v), k
        assert torch.equal(a["l_center_map"], centre)
        with pytest.raises(RuntimeError):
            a["segms"]                                 # never read before the arena was re-used
        assert b.materialize()["segms"].shape == (2, 33, 256, 256)
    finally:
        args().model_precision = "bf16"


def test_engine_cache_is_bounded_and_shares_weights(sd):
    """Variable batch sizes (the last partial batch of a video) must not accumulate plans: LRU of 3, one packed
    weight blob for all of them."""
    from acr.model import ACR
    model = ACR()
    model.load_state_dict(sd, strict=True)
    model = model.cuda()
    engines = [model.engine(b, "cuda") for b in (1, 2, 3, 4, 1)]
    assert len(model._engines) == 3
    assert len({e.weights.data_ptr() for e in engines}) == 1
    assert engines[-1].batch == 1 and engines[-1] is not engines[0]      # batch 1 was evicted, then rebuilt


def test_channel_slice_view_starts_at_its_offset(sd, image):
    """Engine.view of a channel slice (cam head = channels 112..114 of the 128-wide head tensor)."""
    from acr_b200.engine import Engine
    eng = Engine(sd, 2, "cuda", torch.float16, keep_extra=("l_cam_raw",))   # the 128-wide head tensor must outlive the run
    eng.run(image.cuda())
    torch.cuda.synchronize()
    whole = eng.view(eng.spec.tensors["l_cam_raw"].base)
    assert torch.equal(eng.view("l_cam_raw")[..., :3], whole[..., 112:115])
    assert torch.equal(eng.map_nchw("l_cam_raw"), whole[..., 112:115].permute(0, 3, 1, 2).float())
    assert float(eng.map_nchw("l_cam_raw")[:, 0].min()) > 0.0          # channel 0 went through 1.1**x


def test_plan_tcgen05_matches_refconv(sd, image):
    """Same rounding points, different conv engine (fp16 storage): only summation order differs."""
    _, a = _engine_maps(sd, image, ref_conv=False, dtype=torch.float16)
    _, b = _engine_maps(sd, image, ref_conv=True, dtype=torch.float16)
    for k in a:
        assert rel_err(a[k].numpy(), b[k].numpy()) < 2e-2, k


def test_full_batch_256_is_batch_invariant(sd, image):
    """BASELINE configs[2] size (256 frames per GPU) through a size-independent property: every kernel of the plan
    works per image (conv super-tiles, pooling chunks, part head), so a frame's maps must not depend on the
    batch it travels in -- the 256-frame plan run on the two test frames repeated 128 times reproduces the
    2-frame plan (itself pinned against the oracle above) bit for bit, at every position of the batch.
    What this does NOT cover: a kernel that takes image b's per-image data (bias, pooling partials, part-head offsets,
    batch coordinate) from another image is wrong in the same way in both plans, and the 2-frame plan is pinned against
    the oracle only at TOL_NET.  Distinct frames, batch-1 parity of every plan and every launch, and a permuted
    256-frame batch are in tests/test_gpu_batch.py."""
    from acr_b200.engine import Engine
    B = 256
    names = ["segms", "l_center_map", "r_center_map", "l_params_maps", "r_params_maps", "l_prior_maps", "r_prior_maps"]
    small = Engine(sd, 2, "cuda")
    small.run(image.cuda())
    frames = image[torch.arange(B) % 2].contiguous().cuda()
    big = Engine(sd, B, "cuda")
    big.run(frames)
    torch.cuda.synchronize()
    for n in names + ["pooled"]:
        C = big.spec.tensors[n].C                      # logical channels (the rest of the pixel stride is padding)
        a, b = big.view(n)[..., :C], small.view(n)[..., :C]
        a = a.reshape(B // 2, 2, *a.shape[1:])
        assert torch.equal(a, b.unsqueeze(0).expand_as(a)), n


@pytest.mark.parametrize("precision", ["fp16", "bf16"])
def test_dropin_api_end_to_end(sd, image, precision):
    """acr.main.ACR -> acr.model.ACR.forward -> MANOWrapper.forward against (a) the oracle run on the
    engine's own maps (fp32 tail at 1e-4, bit-exact indices) and (b, fp16 only) the reference goldens:
    same centres and outputs within the 16-bit backbone's tolerance (a bf16 arg-max flip legitimately
    moves a centre, SURVEY.md section 7 hard part 2)."""
    from acr.config import args
    from acr.main import ACR
    from acr_b200.synth import make_synthetic_mano
    from oracle import mano_ref, parse_ref
    args().model_precision = precision
    assets = {"left": make_synthetic_mano("left"), "right": make_synthetic_mano("right")}
    app = ACR(state_dict=sd, mano_assets=assets)
    out = app.batch_forward(image)
    maps = {k: out[k].cpu().numpy() for k in ("l_center_map", "r_center_map", "l_params_maps", "r_params_maps",
                                              "l_prior_maps", "r_prior_maps")}
    p = parse_ref.parse(maps)
    N = p["params_pred"].shape[0]
    assert out["params_pred"].shape[0] == N
    assert (out["reorganize_idx"].cpu().numpy() == p["reorganize_idx"]).all()
    assert (out["l_centers_pred"].cpu().numpy() == p["l_centers_pred"]).all()
    assert (out["r_centers_pred"].cpu().numpy() == p["r_centers_pred"]).all()
    assert np.abs(out["params_pred"].cpu().numpy() - p["params_pred"]).max() < 1e-5
    L_, R_ = int(p["left_hand_num"][0]), int(p["right_hand_num"][0])
    offs = np.tile(np.array([512, 512, 0, 0, 0, 0, 0, 0, 0, 0], np.float32), (N, 1))
    m = mano_ref.mano_wrapper_forward(assets, p["params_dict"]["poses"], p["params_dict"]["betas"], L_, R_,
                                      p["params_dict"]["cam"], offs)
    assert rel_err(out["verts"].cpu().numpy(), m["verts"]) < 1e-4
    assert rel_err(out["j3d"].cpu().numpy(), m["j3d"]) < 1e-4
    assert rel_err(out["pj2d_org"].cpu().numpy(), m["pj2d_org"]) < 1e-4
    if precision == "fp16":
        g = np.load(os.path.join(GOLDEN, "net_golden.npz"))
        assert (out["l_centers_pred"].cpu().numpy() == g["l_centers_pred"]).all()
        assert (out["r_centers_pred"].cpu().numpy() == g["r_centers_pred"]).all()
        assert rel_err(out["params_pred"].cpu().numpy(), g["params_pred"]) < TOL_NET[torch.float16]
        assert out["verts"].shape == g["verts"].shape
    # fused sync-free pipeline gives the same rows
    bufs, mano = app.fused_forward(image.cuda(), torch.from_numpy(offs[:2]).cuda())
    torch.cuda.synchronize()
    assert int(bufs.counts[2]) == N
    assert torch.equal(mano["verts"][:N], out["verts"])
    args().model_precision = "bf16"


def test_cuda_graph_replay_matches_eager(sd):
    """acr.main.ACR.capture_graph: one CUDA graph for the ~380 launches of the pipeline (serving / webcam
    mode, batch 1..few) must reproduce the eager launches bit for bit."""
    from acr.main import ACR
    from acr_b200.synth import make_synthetic_mano
    assets = {"left": make_synthetic_mano("left"), "right": make_synthetic_mano("right")}
    app = ACR(state_dict=sd, mano_assets=assets)
    gi = torch.Generator().manual_seed(77)
    offs = torch.tensor([[512., 512, 0, 0, 0, 0, 0, 0, 0, 0]]).cuda()
    replay = app.capture_graph(1)
    for _ in range(3):
        frame = torch.randint(0, 256, (1, 512, 512, 3), generator=gi, dtype=torch.uint8).cuda()
        bufs, mano = app.fused_forward(frame, offs)
        torch.cuda.synchronize()
        n = int(bufs.counts[2])
        v_eager, p_eager = mano["verts"][:n].clone(), bufs.params_pred[:n].clone()
        bufs_g, mano_g = replay(frame, offs)
        torch.cuda.synchronize()
        assert int(bufs_g.counts[2]) == n
        assert torch.equal(mano_g["verts"][:n], v_eager) and torch.equal(bufs_g.params_pred[:n], p_eager)
