"""GPU: the TF32 plan (model_precision='tf32'): fp32 storage, every conv but the stem on the wgmma tensor cores with tf32
operands and fp32 accumulation.  Per conv against fp64 on the same operands, what becomes of raw fp32 operands (the
tensor cores truncate, the kernel rounds its activations to nearest first), every launch teacher-forced (W32 and W48), the whole network against the fp32 oracle and the TF32
same-rounding restatement, the pipeline against the reference goldens, head_forward and CUDA-graph replay."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from acr_b200 import lib as L
from tests.helpers import GOLDEN, ctensor, rel_err, rup
from tests.test_gpu_conv import CASES
from tests.test_gpu_network import image, oracle_out, sd  # noqa: F401  (module fixtures)
from tests.tf32_ref import tf32_round, tf32_truncate

pytestmark = pytest.mark.gpu

MAPS = ("backbone", "segms", "l_center_map", "r_center_map", "l_params_maps", "r_params_maps", "l_prior_maps",
        "r_prior_maps", "pooled")


def _pack_tf32(w, cb, bn, cin_pad, cout_pad):
    cout, cin, k, _ = w.shape
    wp = np.zeros((cout_pad, k * k, cin_pad), np.float32)
    bias = np.zeros(cout_pad, np.float32)
    keep = [None if a is None else np.ascontiguousarray(a, np.float32) for a in [w, cb] + list(bn or [None] * 4)]
    q = lambda a: None if a is None else a.ctypes.data
    L.check(L.load().acr_b200_pack_conv(*(q(a) for a in keep), 1e-5, cout, cin, k, cout_pad, cin_pad, L.DT_TF32,
                                        wp.ctypes.data, bias.ctypes.data), "pack_conv")
    return wp, bias


def run_tf32_conv(B, H, W, cin, cout, k, s, relu, residual, bias, bn, seed=0, in_stride=None, cin_pad=None, flags=0,
                  x=None, w=None, raw_w=False):
    """One conv through acr_b200_run_op(OP_CONV, act_dtype=DT_TF32).  Returns (got, x, packed weights, bias, residual,
    per-image bias, pad_ok): got fp32 NCHW; the operands as stored.  raw_w: the weights go into the blob as given (not
    rounded by the packer; no bias, no BN)."""
    g = torch.Generator().manual_seed(seed)
    in_stride = in_stride or rup(cin, 16)
    cin_pad, cout_pad = cin_pad or rup(cin, 16), rup(cout, 16)
    Ho, Wo = H // s, W // s
    if x is None:
        x = tf32_round(torch.randn(B, cin, H, W, generator=g))
    if w is None:
        w = torch.randn(cout, cin, k, k, generator=g) * (2.0 / (cin * k * k)) ** 0.5
    cb = torch.randn(cout, generator=g) * 0.1 if bias else None
    bnp = [torch.rand(cout, generator=g) + 0.5, torch.randn(cout, generator=g) * 0.1,
           torch.randn(cout, generator=g) * 0.1, torch.rand(cout, generator=g) + 0.5] if bn else None
    wp, bvec = _pack_tf32(w.numpy(), None if cb is None else cb.numpy(), None if bnp is None else [t.numpy() for t in bnp],
                          cin_pad, cout_pad)
    if raw_w:
        wp = np.zeros_like(wp)
        wp[:cout, :, :cin] = w.permute(0, 2, 3, 1).reshape(cout, k * k, cin).numpy()
    res = tf32_round(torch.randn(B, cout, Ho, Wo, generator=g)) if residual else None
    bimg = None
    if flags & 1:      # (the part head writes zero bias past the 109 real channels)
        bimg = torch.zeros(B, cout_pad)
        bimg[:, :cout] = torch.randn(B, cout, generator=g) * 0.1
    xin = torch.zeros(B, H, W, in_stride)
    xin[..., :cin] = x.permute(0, 2, 3, 1)
    # arena: [x | residual | out | per-image bias], fp32
    off_r = rup(xin.numel() * 4, 1024)
    off_o = rup(off_r + (B * Ho * Wo * cout_pad * 4 if residual else 0), 1024)
    obytes = B * Ho * Wo * cout_pad * 4
    off_b = rup(off_o + obytes, 1024)
    arena = torch.zeros(off_b + B * cout_pad * 4 + 1024, dtype=torch.uint8)
    arena[: xin.numel() * 4] = xin.view(torch.uint8).flatten()
    if residual:
        rin = torch.zeros(B, Ho, Wo, cout_pad)
        rin[..., :cout] = res.permute(0, 2, 3, 1)
        arena[off_r: off_r + rin.numel() * 4] = rin.view(torch.uint8).flatten()
    if bimg is not None:
        arena[off_b: off_b + bimg.numel() * 4] = bimg.contiguous().view(torch.uint8).flatten()
    blob = np.concatenate([wp.view(np.uint8).reshape(-1), np.zeros((-wp.nbytes) % 256, np.uint8), bvec.view(np.uint8)])
    op = L.Op()
    op.kind, op.n_in = L.OP_CONV, 2 if residual else 1
    op.in_[0] = ctensor(0, cin, H, W, in_stride, L.DT_F32)
    if residual:
        op.in_[1] = ctensor(off_r, cout, Ho, Wo, cout_pad, L.DT_F32)
    op.out = ctensor(off_o, cout, Ho, Wo, cout_pad, L.DT_F32)
    if bimg is not None:
        op.aux[0] = ctensor(off_b, cout_pad, 1, 1, cout_pad, L.DT_F32)
    op.w_offset[0], op.w_offset[1] = 0, wp.nbytes + ((-wp.nbytes) % 256)
    op.k, op.stride, op.relu, op.has_residual = k, s, int(relu), int(residual)
    op.cin_pad, op.cout_pad = cin_pad, cout_pad
    op.shift[0] = flags
    d_arena, d_blob = arena.cuda(), torch.from_numpy(blob).cuda()
    L.check(L.load().acr_b200_run_op(C.byref(op), B, d_arena.data_ptr(), d_blob.data_ptr(), None, L.DT_TF32,
                                     torch.cuda.current_stream().cuda_stream), "run_op")
    torch.cuda.synchronize()
    got = d_arena[off_o: off_o + obytes].cpu().view(torch.float32).view(B, Ho, Wo, cout_pad)
    pad_ok = bool((got[..., cout:] == 0).all())
    got = got[..., :cout].permute(0, 3, 1, 2).contiguous()
    wf = torch.from_numpy(wp).view(cout_pad, k, k, cin_pad)[:cout, :, :, :cin].permute(0, 3, 1, 2).contiguous()
    return got, x, wf, torch.from_numpy(bvec[:cout].copy()), res, bimg, pad_ok


def _expected64(x, wf, bvec, res, bimg, k, s, relu, pow11):
    """fp64 CPU conv on the same operands, with the kernel's epilogue order: + bias, (1.1 ** ch0), + residual, ReLU."""
    import torch.nn.functional as Fn
    cout = wf.shape[0]
    y = Fn.conv2d(x.double(), wf.double(), None, s, k // 2)
    y = y + (bimg[:, :cout, None, None].double() if bimg is not None else bvec.double().view(1, -1, 1, 1))
    if pow11:
        y = torch.cat([torch.pow(1.1, y[:, :1]), y[:, 1:]], 1)
    if res is not None:
        y = y + res.double()
    return torch.relu(y) if relu else y


# the conv classes of tests/test_gpu_conv.py, the 33/34-channel inputs fed as one zero-filled K chunk, the cam scale channel
# (1.1 ** x) and the per-image bias of the folded part-head conv
EXTRA = [
    dict(case=(2, 64, 64, 34, 64, 3, 2, True, False, True, True, False), in_stride=48, cin_pad=64),
    dict(case=(2, 64, 64, 34, 256, 3, 1, True, False, True, True, False), in_stride=48, cin_pad=64),
    dict(case=(2, 64, 64, 33, 33, 3, 1, True, False, True, True, False), in_stride=48, cin_pad=64),
    dict(case=(2, 64, 64, 34, 64, 1, 1, True, False, True, True, False), in_stride=48, cin_pad=64),
    dict(case=(2, 32, 32, 64, 3, 3, 1, False, False, True, True, False), flags=2),       # ACR_CONV_POW11_CH0
    dict(case=(2, 32, 32, 128, 109, 1, 1, False, False, False, False, False), flags=1),  # ACR_CONV_BIAS_PER_IMAGE
]


@pytest.mark.parametrize("spec", [dict(case=c) for c in CASES] + EXTRA,
                         ids=lambda d: "-".join(str(int(v) if isinstance(v, bool) else v) for v in d["case"][:11])
                         + "".join(f"-{k}{v}" for k, v in d.items() if k != "case"))
def test_conv_tf32_vs_fp64_on_the_same_operands(spec):
    """1x1, 3x3 single-box (MODE_P1) and three-box, stride 2 from parity views, N split, streamed weights, residual,
    K padded by TMA zero fill, 1.1 ** x and the per-image bias.  Inputs, residuals and weights are tf32-representable,
    so only fp32 summation separates the kernel from fp64."""
    B, H, W, cin, cout, k, s, relu, res, bias, bn, _ = spec["case"]
    flags = spec.get("flags", 0)
    got, x, wf, bvec, r, bimg, pad_ok = run_tf32_conv(B, H, W, cin, cout, k, s, relu, res, bias, bn,
                                                      seed=hash(spec["case"]) % 1000, in_stride=spec.get("in_stride"),
                                                      cin_pad=spec.get("cin_pad"), flags=flags)
    exp = _expected64(x, wf, bvec, r, bimg, k, s, relu, flags & 2)
    scale = float(exp.abs().max())
    err = float((got.double() - exp).abs().max())
    assert pad_ok, "padding channels of the output are not zero"
    assert err <= 2e-5 * scale + 1e-6, f"max err {err:.3g} > 2e-5 x {scale:.3g}"


def _rounding_errors(raw_operand):
    """Positive operands, K = 256, one of them raw fp32 (low 13 bits not zero), the other tf32-representable: truncation
    biases every product down by half a tf32 ulp on average (2.4e-4 relative), round-to-nearest is unbiased.  -> max
    relative error of the kernel vs fp64 convs on the truncated and on the rounded operand."""
    g = torch.Generator().manual_seed(5)
    B, H, W, cin, cout = 2, 32, 32, 256, 64
    x = torch.rand(B, cin, H, W, generator=g) + 1.0
    w = (torch.rand(cout, cin, 1, 1, generator=g) + 0.5) / cin
    if raw_operand == "activations":
        w = tf32_round(w)
    else:
        x = tf32_round(x)
    raw = x if raw_operand == "activations" else w
    assert (tf32_truncate(raw) != raw).float().mean() > 0.99
    got, _, _, bvec, _, _, _ = run_tf32_conv(B, H, W, cin, cout, 1, 1, False, False, False, False, x=x, w=w,
                                             raw_w=raw_operand == "weights")
    scale = float(got.abs().max())
    err = {}
    for name, fn in (("truncated", tf32_truncate), ("nearest", tf32_round)):
        xe, we = (fn(x), w) if raw_operand == "activations" else (x, fn(w))
        exp = _expected64(xe, we, bvec, None, None, 1, 1, False, False)
        err[name] = float((got.double() - exp).abs().max()) / scale
    print(f"tf32, raw fp32 {raw_operand}: max rel err vs fp64 on truncated operands {err['truncated']:.2e}, "
          f"on round-to-nearest {err['nearest']:.2e}")
    return err


def test_operand_rounding():
    """What becomes of the low 13 bits of an fp32 operand.  The tensor cores truncate: raw fp32 weights (B operand, put in
    the blob unrounded) give the truncated-operand result.  The kernel's activations (A operand) are rounded to nearest
    in shared memory first: raw fp32 activations give the round-to-nearest result."""
    e = _rounding_errors("weights")
    assert e["truncated"] <= 2e-5 and e["nearest"] > 10 * e["truncated"], e
    e = _rounding_errors("activations")
    assert e["nearest"] <= 2e-5 and e["truncated"] > 10 * e["nearest"], e


@pytest.fixture(scope="module")
def frame():
    gi = torch.Generator().manual_seed(123)
    return torch.randint(0, 256, (2, 512, 512, 3), generator=gi, dtype=torch.uint8)[1:]


# per-op bound of the teacher-forced sweep, from the operand rounding alone: a product of a weight and an activation, each
# rounded to the nearest tf32 (relative error <= 2^-11 each), is off by <= 2^-10; the sum of such products over K stays
# below 2^-9 of the op's output range unless the products cancel by more than a factor of 2
TOL_TEACHER_FORCED = 2.0 ** -9


@pytest.mark.parametrize("width", [32, 48])
def test_every_op_teacher_forced_tf32(frame, width):
    from acr_b200.engine import Engine
    from acr_b200.netspec import WIDTHS, WIDTHS_W48, build_acr_spec
    from acr_b200.synth import load_bn_calibration, synth_state_dict
    from tests.test_gpu_teacher_forced import sweep
    torch.set_num_threads(min(32, os.cpu_count()))
    widths = WIDTHS if width == 32 else WIDTHS_W48
    sdw = synth_state_dict(0, bn_stats=load_bn_calibration(0)) if width == 32 else \
        synth_state_dict(3, spec=build_acr_spec(512, widths=WIDTHS_W48))
    eng = Engine(sdw, 1, "cuda", torch.float32, reuse_memory=False, widths=widths, tf32=True)
    assert all(r["kind"] != L.OP_CONV_REF for r in eng.recs)
    eng.run(frame.cuda())
    torch.cuda.synchronize()
    rows = sweep(eng, sdw, frame, TOL_TEACHER_FORCED)
    worst = sorted(rows, key=lambda r: -r[2])[:6]
    print(f"teacher-forced sweep tf32 W{width}: {len(rows)} checks over {len(eng.recs)} launches; worst:",
          [(i, l, f"{e:.2e}") for i, l, e in worst])
    assert len(rows) >= len(eng.recs) - 1
    bad = [(i, l, e) for i, l, e in rows if not e <= TOL_TEACHER_FORCED]
    assert not bad, f"{len(bad)} ops above 2^-9: {bad[:8]}"


def _plan_maps(sd, image, dtype, tf32=False):
    from acr_b200.engine import Engine
    eng = Engine(sd, image.shape[0], "cuda", dtype, keep_extra=("feat32",), tf32=tf32)
    eng.run(image.cuda())
    torch.cuda.synchronize()
    out = {n: eng.map_nchw(n).cpu() for n in MAPS if n not in ("backbone", "pooled")}
    out["backbone"] = eng.view("feat32")[..., :32].permute(0, 3, 1, 2).float().cpu()
    out["pooled"] = eng.view("pooled").view(image.shape[0], 256, 32).float().cpu()
    return out


# Distance of the TF32 plan to its same-rounding restatement (tests/tf32_ref.py) on this input, max-abs / max-abs per map:
# measured on an H100 at most 1.12e-2 (segms; backbone 4.6e-3, pooled 2.2e-3); the bound is twice that.  What is left is
# fp32 summation order (tensor-core tiles vs the CPU's), which the random network amplifies: the restatement itself is
# 0.9e-2 .. 2.2e-2 from the fp32 oracle, the fp16 plan 1.0e-2 .. 2.5e-2.
MEASURED_SAME_ROUNDING = 1.12e-2
TOL_TF32_SAME_ROUNDING = 2 * MEASURED_SAME_ROUNDING


def test_network_tf32_is_closer_to_the_fp32_oracle_than_fp16(sd, image, oracle_out):
    """Whole network on the seeded frames: every compared map of the TF32 plan is closer to the fp32 oracle than the fp16
    plan's is, and within twice the measured distance of the TF32 same-rounding restatement."""
    from tests import tf32_ref
    tf = _plan_maps(sd, image, torch.float32, tf32=True)
    h = _plan_maps(sd, image, torch.float16)
    same = tf32_ref.net_forward(sd, image, return_backbone=True)
    e_tf = {k: rel_err(tf[k].numpy(), oracle_out[k].numpy()) for k in MAPS}
    e_16 = {k: rel_err(h[k].numpy(), oracle_out[k].numpy()) for k in MAPS}
    d_same = {k: rel_err(tf[k].numpy(), same[k].numpy()) for k in MAPS}
    d_oracles = {k: rel_err(same[k].numpy(), oracle_out[k].numpy()) for k in MAPS}
    print("tf32 plan vs fp32 oracle:", {k: f"{v:.3e}" for k, v in e_tf.items()})
    print("fp16 plan vs fp32 oracle:", {k: f"{v:.3e}" for k, v in e_16.items()})
    print("tf32 plan vs tf32 same-rounding restatement:", {k: f"{v:.3e}" for k, v in d_same.items()})
    print("tf32 restatement vs fp32 oracle:", {k: f"{v:.3e}" for k, v in d_oracles.items()})
    for k in MAPS:
        assert torch.isfinite(tf[k]).all(), k
        assert e_tf[k] < e_16[k], (k, e_tf[k], e_16[k])
        assert d_same[k] < TOL_TF32_SAME_ROUNDING, (k, d_same[k])


# Pipeline against the reference goldens (relative to each output's range), measured on an H100 at most these values; the
# bounds are twice that.  maps: centre / params / prior maps; params: params_pred, poses (the largest), betas, cam; mano:
# verts (the largest, 1.38e-1), joints, 2-D joints (9e-3).  The seeded random network amplifies the tf32 operand error
# (2^-11) to these; the top-2 centre margins (0.25 .. 0.44) keep the golden's centres.
MEASURED_GOLDEN = dict(maps=1.9e-2, params=6.0e-2, mano=1.38e-1)


def test_tf32_pipeline_vs_reference_golden(sd, image):
    """ACR(model_precision='tf32').batch_forward on the golden frames: the golden's centres, and parameters, vertices and
    joints within twice the measured distance.  Prints the margin between the two highest values of every centre map."""
    from acr.config import args
    from acr.main import ACR
    from acr_b200.synth import make_synthetic_mano
    g = np.load(os.path.join(GOLDEN, "net_golden.npz"))
    args().model_precision = "tf32"
    try:
        app = ACR(state_dict=sd, mano_assets={"left": make_synthetic_mano("left"), "right": make_synthetic_mano("right")})
        out = app.batch_forward(image)
        torch.cuda.synchronize()
        for s in "lr":
            top2 = out[f"{s}_center_map"].reshape(image.shape[0], -1).topk(2, dim=1).values
            print(f"tf32 {s} centre maps: top-2 margin per image", [f"{float(a - b):.3e}" for a, b in top2])
        assert (out["l_centers_pred"].cpu().numpy() == g["l_centers_pred"]).all()
        assert (out["r_centers_pred"].cpu().numpy() == g["r_centers_pred"]).all()
        assert (out["reorganize_idx"].cpu().numpy() == g["reorganize_idx"]).all()
        assert (out["detection_flag"].cpu().numpy() == g["detection_flag"]).all()
        errs = {k: rel_err(out[k].cpu().numpy(), g[k]) for k in ("l_center_map", "r_center_map")}
        for k, gk in (("l_params_maps", "l_params_crop"), ("r_params_maps", "r_params_crop"), ("l_prior_maps", "l_prior_crop")):
            errs[gk] = rel_err(out[k][:, :, 30:34, 30:34].cpu().numpy(), g[gk])
        errs["params_pred"] = rel_err(out["params_pred"].cpu().numpy(), g["params_pred"])
        for k in ("poses", "betas", "cam"):
            errs[k] = rel_err(out["params_dict"][k].cpu().numpy(), g[k])
        for k in ("verts", "j3d", "pj2d_org"):
            errs[k] = rel_err(out[k].cpu().numpy(), g[k])
        print("tf32 pipeline vs reference golden:", {k: f"{v:.2e}" for k, v in errs.items()})
        group = lambda k: "maps" if k.endswith(("_map", "_crop")) else ("mano" if k in ("verts", "j3d", "pj2d_org") else "params")
        for k, v in errs.items():
            assert v < 2 * MEASURED_GOLDEN[group(k)], (k, v)
    finally:
        args().model_precision = "bf16"


def test_head_forward_tf32_on_the_oracle_backbone(sd, oracle_out):
    """ACR.head_forward in 'tf32' on the oracle's backbone output: within the fp16 plan's tolerance of the oracle."""
    from acr.config import args
    from acr.model import ACR
    from tests.test_gpu_network import TOL_NET
    args().model_precision = "tf32"
    try:
        model = ACR()
        model.load_state_dict(sd, strict=True)
        model = model.cuda()
        out = model.head_forward(oracle_out["backbone"].cuda())
        torch.cuda.synchronize()
        assert model.engine(oracle_out["backbone"].shape[0], "cuda", head_only=True).tf32
        errs = {k: rel_err(v.cpu().numpy(), oracle_out[k].numpy()) for k, v in out.items()}
        print("tf32 head_forward vs oracle:", {k: f"{v:.2e}" for k, v in errs.items()})
        for k, v in out.items():
            assert v.dtype == torch.float32 and tuple(v.shape) == tuple(oracle_out[k].shape), k
            assert errs[k] < TOL_NET[torch.float16], (k, errs[k])
    finally:
        args().model_precision = "bf16"


def test_tf32_graph_replay_and_eager_runs_are_bit_identical(sd):
    """capture_graph in 'tf32' replays the eager fused_forward bit for bit, and two eager runs agree bit for bit (no
    atomics or order-dependent sums on the TF32 plan)."""
    from acr.config import args
    from acr.main import ACR
    from acr_b200.synth import make_synthetic_mano
    args().model_precision = "tf32"
    try:
        app = ACR(state_dict=sd, mano_assets={"left": make_synthetic_mano("left"), "right": make_synthetic_mano("right")})
        gi = torch.Generator().manual_seed(77)
        offs = torch.tensor([[512., 512, 0, 0, 0, 0, 0, 0, 0, 0]]).cuda()
        replay = app.capture_graph(1)
        assert app.model.engine(1, "cuda").tf32
        for _ in range(2):
            frame = torch.randint(0, 256, (1, 512, 512, 3), generator=gi, dtype=torch.uint8).cuda()
            runs = []
            for _ in range(2):
                bufs, mano = app.fused_forward(frame, offs)
                torch.cuda.synchronize()
                n = int(bufs.counts[2])
                runs.append((n, mano["verts"][:n].clone(), bufs.params_pred[:n].clone()))
            assert runs[0][0] == runs[1][0] and torch.equal(runs[0][1], runs[1][1]) and torch.equal(runs[0][2], runs[1][2])
            n, v_eager, p_eager = runs[0]
            bufs_g, mano_g = replay(frame, offs)
            torch.cuda.synchronize()
            assert int(bufs_g.counts[2]) == n
            assert torch.equal(mano_g["verts"][:n], v_eager) and torch.equal(bufs_g.params_pred[:n], p_eager)
    finally:
        args().model_precision = "bf16"
